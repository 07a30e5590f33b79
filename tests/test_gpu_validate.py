"""GPU: graph validation on the device (include/kaminpar_b200_validate.h, kmp_validate.cuh) against the oracle
(tests/validate_oracle.py, held to the reference by tests/test_validate_bridge.py and the golden verdicts): every field
of the report, from host and from device arrays.
  V1  valid graphs: the golden graphs, weighted R-MAT 2^20 and 2^16, rgg 2^20, a 3-D grid, a star whose hub has
      degree 2^17 (CUB's large-segment path), isolated vertices, n = 0, m = 0
  V2  the small corpus: each kind at the first and last edge, inside a hub row and in a degree-1 row, competing
      kinds, duplicates, broken xadj (start, end, decreasing entries, entries near 2^32)
  V3  the same kinds on weighted R-MAT 2^16, the 3-D grid and the star
  V4  KMP_GRID_CAP 1..3; adjncy 4-byte but not 16-byte aligned
  V5  one handle clusters, validates and clusters again: both clusterings equal the oracle's at call indices 0 and 1
Malformed arrays go only to the validator."""
import functools

import numpy as np
import pytest

from kaminpar_b200 import lp
from kaminpar_b200 import validate as VA
from kaminpar_b200.graph import CSRGraph, grid3d, random_weights, rgg2d, rmat
from tests import test_validate_bridge as TB
from tests import validate_oracle as V

pytestmark = pytest.mark.gpu


def _handle():
    return lp.LPHandle(lp._cluster_config(lp.LabelPropagationCoarseningContext(), lp.EngineContext()))


@pytest.fixture(scope="module")
def handle():
    h = _handle()
    yield h
    h.close()


def _device(a, pad=0):
    """A device copy of a uint32 / int32 array (None stays None), `pad` elements into its allocation."""
    import torch

    if a is None:
        return None, 0
    t = torch.zeros(len(a) + pad + 1, dtype=torch.int32, device="cuda")
    if len(a):
        t[pad:pad + len(a)] = torch.from_numpy(np.ascontiguousarray(a).view(np.int32)).cuda()
    return t, t.data_ptr() + 4 * pad


def check(h, xadj, adj, w, expect=None, pad=0):
    """Host and device report == the oracle, field for field; returns the oracle's report."""
    expect = expect or V.validate(xadj, adj, w)
    want = V.as_dict(expect)
    got = VA.validate_graph(h, CSRGraph(xadj, adj, adjwgt=w))
    assert V.as_dict(got) == want, ("host", got)
    assert got.message() == V.message(expect)
    assert got.n == len(xadj) - 1 and got.m == len(adj)
    keep = [_device(xadj), _device(adj, pad), _device(w)]
    got = VA.validate_graph_device(h, len(xadj) - 1, len(adj), keep[0][1], keep[1][1] if len(adj) else 0, keep[2][1])
    assert V.as_dict(got) == want, ("device", got)
    return expect


# ---- V1 ----------------------------------------------------------------------------------------------------------
LARGE = ("rmat20_w", "rgg20", "grid48", "star2^17", "rmat16_w")


@functools.lru_cache(maxsize=None)
def large(name):
    if name == "rmat20_w":
        g = random_weights(rmat(20, 8, seed=3), seed=4, max_adjwgt=100)
    elif name == "rmat16_w":
        g = random_weights(rmat(16, 8, seed=3), seed=4, max_adjwgt=100)
    elif name == "rgg20":
        g = rgg2d(1 << 20, seed=2)
    elif name == "grid48":
        g = grid3d(48)
    else:
        g = CSRGraph(*V.star(1 << 17, isolated=3))
    return name, g.xadj, g.adjncy, g.adjwgt


SMALL = V.small_bases() + V.empty_graphs()


@pytest.mark.parametrize("name", [c[0] for c in SMALL] + list(LARGE))
def test_v1_valid_graphs(handle, name):
    _, xadj, adj, w = large(name) if name in LARGE else SMALL[[c[0] for c in SMALL].index(name)]
    r = check(handle, xadj, adj, w)
    assert r["valid"] and r["duplicates"] == 0


# ---- V2 ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", TB.CASES, ids=[c[0] for c in TB.CASES])
def test_v2_small_corpus(handle, case):
    check(handle, *case[1:])


# ---- V3 ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["rmat16_w", "grid48", "star2^17"])  # the oracle takes ~1 s per 10^6 edges
def test_v3_large_mutations(handle, name):
    base = large(name)
    cases = V.mutations(*base) + [c for c in V.broken_xadj(*base) if "several" in c[0] or "2^32" in c[0]]
    kinds = set()
    for _, xadj, adj, w in cases:
        kinds.add(check(handle, xadj, adj, w)["kind"])
    assert set(range(V.XADJ_DECREASING, V.NUM_KINDS)) <= kinds


# ---- V4 ----------------------------------------------------------------------------------------------------------
CAPPED = [c for c in TB.CASES if c[0].startswith(("rmat9_w", "star300_iso"))]


@pytest.mark.parametrize("cap", [1, 2, 3])
def test_v4_grid_cap(monkeypatch, cap):
    monkeypatch.setenv("KMP_GRID_CAP", str(cap))  # read by kmp_lp_create
    h = _handle()
    for _, xadj, adj, w in CAPPED + [large("star2^17")]:
        check(h, xadj, adj, w)
    h.close()


def test_v4_adjncy_not_16_byte_aligned(handle):
    for name, xadj, adj, w in [c for c in TB.CASES if c[0].startswith("rmat9_w")] + [large("rmat16_w")]:
        check(handle, xadj, adj, w, pad=1)


# ---- V5 ----------------------------------------------------------------------------------------------------------
def test_v5_validation_leaves_the_handle_alone():
    from oracle import bindings as B

    g, _ = B.oracle_rearrange(rmat(14, 8, seed=6))
    ctx = lp.create_default_context()
    ctx.partition.setup(g, 8, 0.03)
    mcw = lp.compute_max_cluster_weight(ctx.coarsening, ctx.partition, g.n, g.total_node_weight())
    h = _handle()
    h.set_graph(g)
    c0, _ = h.cluster(mcw)
    assert np.array_equal(c0, B.oracle_lp_cluster(g, 0, mcw, schedule=B.SYNC, call_index=0))
    bad = TB.CASES[[c[0] for c in TB.CASES].index("rmat9_w/missing_reverse@hub")]
    r = check(h, *bad[1:])
    assert r["kind"] == V.MISSING_REVERSE
    assert np.array_equal(h.download_labels(), c0)  # labels untouched
    c1, _ = h.cluster(mcw)
    assert np.array_equal(c1, B.oracle_lp_cluster(g, 0, mcw, schedule=B.SYNC, call_index=1))
    h.close()


def test_v5_seq_strict_handle():
    eng = lp.EngineContext()
    eng.schedule = "seq_strict"
    h = lp.LPHandle(lp._cluster_config(lp.LabelPropagationCoarseningContext(), eng))
    for _, xadj, adj, w in [c for c in TB.CASES if c[0].startswith("rgg16_w")]:
        check(h, xadj, adj, w)
    h.close()
