"""GPU: the METIS reader on the device (include/kaminpar_b200_io.h, kmp_metis.cuh) against the oracle
(tests/metis_oracle.py): every report field and every array, through kmp_read_metis (a file) and
kmp_parse_metis_device (a torch uint8 tensor).
  M0  the valid corpus (tests/metis_corpus.py): misc/rgg2d.metis == graph_rgg2d.npz; the four formats with unit weights
      written out (dropped); comments before the header, between lines, after the last line, with leading spaces;
      blank and space-only lines; runs of spaces, leading zeros, no final newline; n = 0, m = 0; maximum weights and
      ids; a star whose hub line has 2^17 targets; a multi-tile file shifted byte by byte across the tile boundaries;
      KMP_GRID_CAP 1..3; a seq_strict handle
  M1  every refusal kind at the first line, the last line and inside the hub line; competing violations; garbage after
      vertex n; no graph is returned
  M2  weighted R-MAT 2^20 and rgg 2^20 written as METIS files
  M3  read -> kmp_prepare_graph_device -> set_graph_prepared -> kmp_lp_cluster equals the LP oracle on the host copy;
      a handle that clusters, reads and clusters again gives the clusterings of call indices 0 and 1"""
import functools
import os

import numpy as np
import pytest

from kaminpar_b200 import lp
from kaminpar_b200 import metis as ME
from kaminpar_b200.graph import random_weights, rgg2d, rmat
from tests import metis_corpus as MC
from tests import metis_oracle as MO

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _handle(schedule="sync"):
    eng = lp.EngineContext()
    eng.schedule = schedule
    return lp.LPHandle(lp._cluster_config(lp.LabelPropagationCoarseningContext(), eng))


@pytest.fixture(scope="module")
def handle():
    h = _handle()
    yield h
    h.close()


def _tensor(data: bytes):
    import torch

    if not data:
        return torch.empty(0, dtype=torch.uint8, device="cuda")
    return torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()


def _got(call):
    """(report dict, arrays dict) of one reader call; a refusal returns no graph."""
    try:
        g = call()
    except ME.MetisError as e:
        assert e.code == (-4 if e.report.kind in MO.UNSUPPORTED else -1)
        return e.report, None
    c = g.get()
    rep = g.report
    arrays = dict(xadj=c.xadj, adjncy=c.adjncy, vwgt=c.vwgt, adjwgt=c.adjwgt)
    g.close()
    return rep, arrays


def check(h, data: bytes, tmp_path, expect=None, name="case"):
    """Both entry points == the oracle, field for field; returns the oracle's dict."""
    expect = expect or MO.parse(data)
    p = tmp_path / f"{name}.metis"
    p.write_bytes(data)
    for how, call in (("file", lambda: ME.read_metis_device(h, str(p))),
                      ("device", lambda: ME.parse_metis_device(h, _tensor(data)))):
        rep, arrays = _got(call)
        got = MO.as_dict(rep)
        assert got == MO.report_of(expect), (name, how, got, MO.report_of(expect))
        if expect["kind"] != 0:
            assert arrays is None
            continue
        assert rep.message() == ("ignorning extra lines in input file" if expect["extra_lines"] else "")
        for f in ("xadj", "adjncy", "vwgt", "adjwgt"):
            assert (arrays[f] is None) == (expect[f] is None), (name, how, f)
            if expect[f] is not None:
                assert np.array_equal(arrays[f].astype(np.int64), np.asarray(expect[f], np.int64)), (name, how, f)
    return expect


# ---- M0 ----------------------------------------------------------------------------------------------------------
VALID = MC.valid_cases()


@pytest.mark.parametrize("name,data", VALID, ids=[c[0] for c in VALID])
def test_m0_valid_corpus(handle, tmp_path, name, data):
    r = check(handle, data, tmp_path, name=name)
    assert r["kind"] == 0


def test_m0_rgg2d_fixture(handle, tmp_path):
    data = open(os.path.join(ROOT, "tests", "golden", "misc", "rgg2d.metis"), "rb").read()
    check(handle, data, tmp_path)
    g = ME.read_metis_device(handle, os.path.join(ROOT, "tests", "golden", "misc", "rgg2d.metis")).get()
    gold = np.load(os.path.join(ROOT, "tests", "golden", "graph_rgg2d.npz"))
    assert np.array_equal(g.xadj, gold["xadj"]) and np.array_equal(g.adjncy, gold["adjncy"])
    assert g.vwgt is None and g.adjwgt is None


CAPPED = [c for c in VALID if c[0] in ("star_hub_w", "tiles_shift0", "tiles_shift13", "comments", "blank_lines")]


@pytest.mark.parametrize("cap", [1, 2, 3])
def test_m0_grid_cap(monkeypatch, tmp_path, cap):
    monkeypatch.setenv("KMP_GRID_CAP", str(cap))  # read by kmp_lp_create
    h = _handle()
    for name, data in CAPPED + [("self_loop_hub", dict((c[0], c[1]) for c in MC.refusal_cases())["self_loop_hub"])]:
        check(h, data, tmp_path, name=name)
    h.close()


def test_m0_seq_strict_handle(tmp_path):
    h = _handle("seq_strict")
    for name, data in CAPPED:
        check(h, data, tmp_path, name=name)
    h.close()


def test_m0_misaligned_or_host_bytes_are_refused(handle):
    import ctypes as C

    import torch

    t = torch.zeros(64, dtype=torch.uint8, device="cuda")
    with pytest.raises(RuntimeError, match="error -1"):
        ME.parse_metis_device(handle, t[1:])
    host = torch.frombuffer(bytearray(b"2 1\n2\n1\n" + b" " * 56), dtype=torch.uint8)
    with pytest.raises(ValueError, match="CUDA tensor"):
        ME.parse_metis_device(handle, host)
    pinned = host.pin_memory()  # host memory reached through the C ABI: refused, never read by a kernel
    rep, out = ME.MetisReport(), C.c_void_p()
    for ptr in (host.data_ptr() & ~15, pinned.data_ptr()):
        assert ME._lib().kmp_parse_metis_device(handle._h, C.c_void_p(ptr), C.c_uint64(8), C.byref(out),
                                                C.byref(rep)) == -1
        assert out.value is None


# ---- M1 ----------------------------------------------------------------------------------------------------------
REFUSED = MC.refusal_cases()


@pytest.mark.parametrize("name,data,kind", REFUSED, ids=[c[0] for c in REFUSED])
def test_m1_refusals(handle, tmp_path, name, data, kind):
    r = check(handle, data, tmp_path, name=name)
    assert MO.KINDS[r["kind"]] == kind


def test_m1_every_kind_and_no_graph(handle, tmp_path):
    assert {c[2] for c in REFUSED} == set(MO.KINDS[1:])
    p = tmp_path / "bad.metis"
    p.write_bytes(b"2 1\n2\n9\n")
    with pytest.raises(ME.MetisError) as e:
        ME.read_metis_device(handle, str(p))
    assert e.value.report.kind_name == "NEIGHBOR_OUT_OF_RANGE" and e.value.report.vertex == 1
    assert e.value.report.message() == "neighbor out of range at byte 6 (line 3, vertex 1)"


# ---- M2 ----------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def large(name):
    if name == "rmat20_w":
        g = random_weights(rmat(20, 8, seed=3), seed=4, max_vwgt=20, max_adjwgt=100)
    else:
        g = rgg2d(1 << 20, seed=2)
    return MO.write_metis(g.xadj, g.adjncy, g.vwgt, g.adjwgt), g


@pytest.mark.parametrize("name", ["rmat20_w", "rgg20"])
def test_m2_large(handle, tmp_path, name):
    data, g = large(name)
    r = check(handle, data, tmp_path, name=name)
    assert np.array_equal(r["xadj"], g.xadj) and np.array_equal(r["adjncy"], g.adjncy)


# ---- M3 ----------------------------------------------------------------------------------------------------------
def test_m3_read_prepare_cluster(tmp_path):
    from kaminpar_b200 import prepare as PR
    from oracle import bindings as B

    g0 = random_weights(rmat(14, 8, seed=6), seed=2, max_adjwgt=9)
    p = tmp_path / "g.metis"
    p.write_bytes(MO.write_metis(g0.xadj, g0.adjncy, adjwgt=g0.adjwgt))
    h = _handle()
    ctx = lp.create_default_context()
    ctx.partition.setup(g0, 8, 0.03)
    mcw = lp.compute_max_cluster_weight(ctx.coarsening, ctx.partition, g0.n, g0.total_node_weight())

    # a clustering before the read: call index 0
    first, _ = B.oracle_rearrange(g0)
    h.set_graph(first)
    c0, _ = h.cluster(mcw)
    assert np.array_equal(c0, B.oracle_lp_cluster(first, 0, mcw, schedule=B.SYNC, call_index=0))

    mg = ME.read_metis_device(h, str(p))
    host = mg.get()
    assert np.array_equal(host.xadj, g0.xadj) and np.array_equal(host.adjncy, g0.adjncy)
    assert np.array_equal(host.adjwgt, g0.adjwgt)
    pg = PR.rearrange_by_degree_buckets_device(h, mg.n, mg.m, *mg.device_arrays())
    expect, _ = B.oracle_rearrange(host)  # the oracle's preparation of the host copy of what was read
    prepared = pg.get()
    for f in ("xadj", "adjncy", "vwgt", "adjwgt"):
        a, b = getattr(prepared, f), getattr(expect, f)
        assert (a is None) == (b is None) and (a is None or np.array_equal(a, b)), f
    pg.set_on(h)
    c1, _ = h.cluster(mcw)
    assert np.array_equal(c1, B.oracle_lp_cluster(expect, 0, mcw, schedule=B.SYNC, call_index=1))
    pg.close()
    mg.close()
    h.close()
