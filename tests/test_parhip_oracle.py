"""CPU checks of the ParHIP oracle (tests/parhip_oracle.py): it reads the sample files as graph.read_parhip does, the
64-bit sample as the 32-bit one, every one of the 64 width / weight combinations of the version word back to the graph
written, ignores the version's high bits and trailing bytes, orders EXTERNAL as the preparation does (independently
computed) with forward lists, and refuses each kind at the first violation in file order."""
import os

import numpy as np
import pytest

from kaminpar_b200.graph import random_weights, read_parhip, rmat
from tests import parhip_oracle as PO
from tests import prepare_oracle as PRO
from tests.helpers import from_edges

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MISC = os.path.join(ROOT, "tests", "golden", "misc")


def small(weighted=True, seed=1):
    g = rmat(6, 4, seed=seed)
    return random_weights(g, seed=seed, max_vwgt=9, max_adjwgt=9) if weighted else g


def test_sample_files_match_the_fixture_reader():
    a = PO.read(open(os.path.join(MISC, "rgg2d-32bit.parhip"), "rb").read())
    b = PO.read(open(os.path.join(MISC, "rgg2d-64bit.parhip"), "rb").read())
    g = read_parhip(os.path.join(MISC, "rgg2d-32bit.parhip"))
    assert a["kind"] == b["kind"] == 0 and a["widths"] == 0x04040404 and b["widths"] == 0x08080808
    for f in ("xadj", "adjncy"):
        assert np.array_equal(a[f], getattr(g, f)) and np.array_equal(b[f], a[f])
    assert a["vwgt"] is None and a["adjwgt"] is None and b["vwgt"] is None


@pytest.mark.parametrize("version", range(64))
def test_every_width_and_weight_combination(version):
    g = small()
    vw, ew = (version & 2) == 0, (version & 1) == 0
    data = PO.write(g.xadj, g.adjncy, g.vwgt if vw else None, g.adjwgt if ew else None, version)
    r = PO.read(data + b"\x07" * (version % 5))  # trailing bytes are ignored
    assert r["kind"] == 0 and r["has_node_weights"] == int(vw) and r["has_edge_weights"] == int(ew)
    assert np.array_equal(r["xadj"], g.xadj) and np.array_equal(r["adjncy"], g.adjncy)
    assert (r["vwgt"] is None) != vw and (r["adjwgt"] is None) != ew
    if vw:
        assert np.array_equal(r["vwgt"], g.vwgt)
    if ew:
        assert np.array_equal(r["adjwgt"], g.adjwgt)
    hi = PO.read(PO.write(g.xadj, g.adjncy, g.vwgt if vw else None, g.adjwgt if ew else None, version | (0x5A << 6)))
    assert hi["kind"] == 0 and np.array_equal(hi["adjncy"], g.adjncy)


def test_unit_weights_stay():
    g = small(weighted=False)
    r = PO.read(PO.write(g.xadj, g.adjncy, np.ones(g.n, np.int32), np.ones(g.m, np.int32)))
    assert np.array_equal(r["vwgt"], np.ones(g.n)) and np.array_equal(r["adjwgt"], np.ones(g.m))


def test_external_is_the_preparation_order_with_forward_lists():
    g = random_weights(rmat(10, 8, seed=5), seed=3, max_vwgt=9, max_adjwgt=9)
    # isolated vertices in the middle and at the end
    xadj = np.concatenate([g.xadj[:100], np.full(7, g.xadj[99]), g.xadj[99:], np.full(3, g.xadj[-1])])
    n = len(xadj) - 1
    adj = g.adjncy.copy()
    vw = np.arange(1, n + 1, dtype=np.int32)
    data = PO.write(xadj, adj, vw, g.adjwgt)
    r = PO.read(data, PO.EXTERNAL)
    prep = PRO.rearrange(xadj, adj, vw, g.adjwgt)
    assert r["kind"] == 0 and r["sorted"] == 1
    assert np.array_equal(r["old_to_new"], prep["old_to_new"]) and np.array_equal(r["xadj"], prep["xadj"])
    assert np.array_equal(r["vwgt"], prep["vwgt"])
    o2n = r["old_to_new"]
    for u in range(n):  # forward: row u of the new graph is the file's row relabelled, in order
        nu = o2n[u]
        row = r["adjncy"][r["xadj"][nu]:r["xadj"][nu + 1]]
        assert np.array_equal(row, o2n[adj[xadj[u]:xadj[u + 1]]])
        assert np.array_equal(r["adjwgt"][r["xadj"][nu]:r["xadj"][nu + 1]], g.adjwgt[xadj[u]:xadj[u + 1]])
    # the reversed lists of the preparation hold the same edges
    assert sorted(map(tuple, np.stack([r["adjncy"], r["adjwgt"]], 1))) == \
        sorted(map(tuple, np.stack([prep["adjncy"], prep["adjwgt"]], 1)))
    assert PO.read(data, PO.IMPLICIT)["sorted"] == 1 and PO.read(data, PO.NATURAL)["sorted"] == 0


def _file(version=None, weighted=True):
    g = from_edges(4, [(0, 1), (1, 2), (2, 3)], vwgt=[1, 2, 3, 4], ew=[5, 6, 7]) if weighted else \
        from_edges(4, [(0, 1), (1, 2), (2, 3)])
    return g, bytearray(PO.write(g.xadj, g.adjncy, g.vwgt if weighted else None, g.adjwgt if weighted else None,
                                 version))


def _put(data, at, value, width, signed=False):
    data[at:at + width] = int(value).to_bytes(width, "little", signed=signed)


def test_refusals_in_file_order():
    g, d = _file()
    n, m = g.n, g.m  # 4, 6
    off_adj = 24 + 5 * 4
    off_vw = off_adj + m * 4
    off_ew = off_vw + n * 4
    end = off_ew + m * 4
    assert len(d) == end

    def kind(data, order=PO.NATURAL):
        r = PO.read(bytes(data), order)
        return PO.KINDS[r["kind"]], r["offset"], r["section"], r["index"]

    assert kind(d[:20]) == ("TRUNCATED", 20, PO.HEADER, -1)
    assert kind(d[:end - 1]) == ("TRUNCATED", end - 1, PO.ADJWGT, m - 1)
    assert kind(d[:off_adj + 5]) == ("TRUNCATED", off_adj + 5, PO.ADJNCY, 1)
    big = bytearray(d)
    _put(big, 8, 1 << 31, 8)
    assert kind(big) == ("TOO_LARGE", 8, PO.HEADER, -1)
    big = bytearray(d)
    _put(big, 16, 1 << 31, 8)
    assert kind(big) == ("TOO_LARGE", 16, PO.HEADER, -1)
    x = bytearray(d)
    _put(x, 24, off_adj + 4, 4)  # offsets[0] != base
    assert kind(x) == ("OFFSETS", 24, PO.OFFS, 0)
    x = bytearray(d)
    _put(x, 24 + 4 * 4, off_adj + 4 * 5, 4)  # offsets[n] != base + m * 4
    assert kind(x) == ("OFFSETS", 40, PO.OFFS, 4)
    x = bytearray(d)
    _put(x, 24 + 2 * 4, off_adj + 1, 4)  # not on an id boundary
    assert kind(x) == ("OFFSETS", 32, PO.OFFS, 2)
    x = bytearray(d)
    _put(x, off_adj + 5 * 4, 4, 4)
    _put(x, off_ew, 0, 4)
    assert kind(x) == ("NEIGHBOR_OUT_OF_RANGE", off_adj + 20, PO.ADJNCY, 5)
    assert kind(x, PO.EXTERNAL) == kind(x)
    x = bytearray(d)
    _put(x, off_vw + 12, -3, 4, signed=True)
    assert kind(x) == ("WEIGHT", off_vw + 12, PO.VWGT, 3)
    x = bytearray(d)
    for i in range(m):
        _put(x, off_ew + 4 * i, 1 << 30, 4)
    assert kind(x) == ("TOTAL_WEIGHT", end - 1, PO.ADJWGT, m)
    # 64-bit widths narrow only what fits
    g, d = _file(PO.version_of(True, True, True, True, True, True))
    base = 24 + 5 * 8
    x = bytearray(d)
    _put(x, base + 8, 1 << 32, 8)
    assert kind(x) == ("TOO_LARGE", base + 8, PO.ADJNCY, 1)
    x = bytearray(d)
    _put(x, base + 6 * 8 + 8, 1 << 31, 8)
    assert kind(x) == ("TOO_LARGE", base + 56, PO.VWGT, 1)
    # competing violations: the earliest byte wins
    x = bytearray(d)
    _put(x, base + 6 * 8 + 8, 0, 8)
    _put(x, base + 16, 9, 8)
    assert kind(x)[0] == "NEIGHBOR_OUT_OF_RANGE"
