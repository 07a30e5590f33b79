"""Parity tests of threshold edge sparsification on the device (-m gpu, DESIGN.md §13): kmp_coarse_sparsify,
called through the C ABI (include/kaminpar_b200_contraction.h), against the CPU oracle (tests/sparsify_oracle.py) --
bit-exact coarse CSR, weights, mapping and selection stats in the canonical form."""
import numpy as np
import pytest

from kaminpar_b200 import contraction as KC
from kaminpar_b200 import lp
from kaminpar_b200.graph import CSRGraph, grid3d, random_weights, rgg2d, rmat
from oracle import bindings as B
from oracle import contraction_oracle as CO
from tests import helpers as H
from tests import sparsify_oracle as S
from tests.test_gpu_parity import NAMES, ctx_for, get_graph

pytestmark = pytest.mark.gpu

SEEDS = (0, 0x9E3779B97F4A7C15, 2**64 - 1)


def gpu_result(cg):
    c = cg.get()
    return dict(c_n=cg.n, c_xadj=c.xadj, c_adjncy=c.adjncy, c_vwgt=c.vwgt, c_adjwgt=c.adjwgt, mapping=cg.mapping())


def new_handle():
    ctx = lp.create_default_context()
    return lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))


def check_sparsify(handle, g, cl, target, seed):
    """Contract g by cl on the handle, sparsify to `target`, compare with the oracle. Returns the oracle result."""
    cg = KC.contract_on_handle(handle, cl)
    con = CO.contract(g.xadj, g.adjncy, g.vwgt, g.adjwgt, cl)
    assert CO.equal(gpu_result(cg), con)
    c_m = len(con["c_adjncy"])
    target = min(target, c_m)
    st = cg.sparsify(handle, target, seed)
    o = S.sparsify_contracted(con, target, seed)
    assert CO.equal(gpu_result(cg), o), (target, seed)
    assert cg.m == len(o["c_adjncy"])
    assert (st.c_m_before, st.c_m_after, st.target_m) == (c_m, len(o["c_adjncy"]), target)
    assert (st.threshold, st.smaller, st.equal, st.equal_kept) == (o["threshold"], o["smaller"], o["equal"],
                                                                    o["equal_kept"])
    cg.close()
    return o


def identity_level(handle, g, target, seed):
    return check_sparsify(handle, g, np.arange(g.n, dtype=np.uint32), target, seed)


@pytest.mark.parametrize("name", NAMES)
def test_sparsify_after_lp_cluster_matches_oracle(name):
    g = get_graph(name)
    ctx, mcw = ctx_for(g, 8, seed=1)
    h = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
    h.set_graph(g)
    cl, _ = h.cluster(mcw)
    c_n = len(np.unique(cl))
    default_target = KC.sparsification_target(g.m, g.n, c_n)
    for target in (default_target, g.m // 7):
        for seed in SEEDS[:2]:
            check_sparsify(h, g, cl, target, seed)


def _generated():
    yield "rmat16", rmat(16, 16, 3)
    yield "rmat16_w", random_weights(rmat(16, 16, 4), 5, max_vwgt=3, max_adjwgt=50)
    yield "grid32", grid3d(32)
    yield "grid24_w", random_weights(grid3d(24), 6, max_adjwgt=4)
    yield "rgg", rgg2d(1 << 15, seed=3)
    yield "rgg_w", random_weights(rgg2d(1 << 15, seed=4), 7, max_adjwgt=1000)


@pytest.mark.parametrize("name,g", list(_generated()))
def test_generated_levels(name, g):
    ctx, mcw = ctx_for(g, 16, seed=2)
    h = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
    h.set_graph(g)
    cl, _ = h.cluster(mcw)
    c_n = len(np.unique(cl))
    for seed in SEEDS:
        check_sparsify(h, g, cl, KC.sparsification_target(g.m, g.n, c_n), seed)


def _weighted_grid(weights_fn, rows=64, cols=64):
    """2-D grid whose undirected edge i has weight weights_fn(i, count)."""
    g = H.grid2d(rows, cols)
    src = np.repeat(np.arange(g.n), np.diff(g.xadj.astype(np.int64)))
    lo, hi = np.minimum(src, g.adjncy), np.maximum(src, g.adjncy)
    key = lo.astype(np.int64) * g.n + hi
    uniq, inv = np.unique(key, return_inverse=True)
    w = np.asarray(weights_fn(np.arange(len(uniq)), len(uniq)), np.int64)
    return CSRGraph(g.xadj, g.adjncy, None, w[inv].astype(np.int32))


def _cases():
    rng = np.random.default_rng(11)
    yield "all_equal", H.grid2d(48, 48)
    yield "small_random", _weighted_grid(lambda i, c: rng.integers(1, 9, c))
    yield "near_int_max", _weighted_grid(lambda i, c: 2**31 - 1 - rng.integers(0, 64, c))
    yield "wide_range", _weighted_grid(lambda i, c: rng.integers(1, 2**31 - 1, c))
    # two weights on either side of a pass-0 (2^21) and of a pass-1 (2^10) digit boundary
    yield "bin21", _weighted_grid(lambda i, c: np.where(i % 2 == 0, 2**21 - 1, 2**21))
    yield "bin10", _weighted_grid(lambda i, c: np.where(i % 3 == 0, 2**10 - 1, 2**10))


@pytest.mark.parametrize("name,g", list(_cases()))
def test_selection_edge_cases(name, g):
    h = new_handle()
    h.set_graph(g)
    c_m = g.m
    w = np.sort(g.adjwgt.astype(np.int64)) if g.adjwgt is not None else np.ones(c_m, np.int64)
    targets = {c_m, c_m - 1, c_m // 2, 3, 2, 1, 0}
    # T at the minimum (target = c_m: k = 1) and at the maximum (target = 2: k = c_m - 1, the heaviest edge is
    # stored twice); k at the last and the first key of a digit bin
    low = int(np.count_nonzero(w == w[0]))
    targets |= {c_m - low + 1, c_m - low, c_m - low + 2}
    for t in sorted(x for x in targets if 0 <= x <= c_m):
        for seed in SEEDS[:2]:
            o = identity_level(h, g, t, seed)
            if t == c_m:
                assert o["threshold"] == w[0] and o["probability"] == 1.0
            if t == 2:
                assert o["threshold"] == w[-1]
            if t < 2:
                assert len(o["c_adjncy"]) == 0 and o["threshold"] == 0


def test_many_ctas():
    g = random_weights(rmat(18, 16, 9), 3, max_adjwgt=20)
    h = new_handle()
    h.set_graph(g)
    cl = (np.arange(g.n) // 2).astype(np.uint32)
    for t in (g.m // 3, g.m // 50):
        check_sparsify(h, g, cl, t, SEEDS[1])


@pytest.mark.parametrize("cap", [1, 2, 3])
def test_grid_cap(cap, monkeypatch):
    monkeypatch.setenv("KMP_GRID_CAP", str(cap))  # read by kmp_lp_create
    h = new_handle()
    for g in (random_weights(rmat(14, 16, 2), 3, max_adjwgt=7), H.grid2d(40, 40),
              _weighted_grid(lambda i, c: np.where(i % 2 == 0, 2**21 - 1, 2**21))):
        h.set_graph(g)
        cl = (np.arange(g.n) // 3).astype(np.uint32)
        check_sparsify(h, g, cl, max(2, g.m // 5), SEEDS[1])
        identity_level(h, g, g.m, SEEDS[0])


def test_device_resident_level():
    """cluster -> contract -> sparsify -> kmp_lp_set_graph_device -> cluster, next to the host path on the oracle."""
    g = B.oracle_rearrange(rmat(15, 16, 21))[0]
    ctx, mcw = ctx_for(g, 8, seed=2)
    h0 = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
    h0.set_graph(g)
    h0.cluster(mcw, fetch=False)
    cg = KC.contract_on_handle(h0, None)
    seed = 77
    assert KC.sparsify_level(h0, cg, g.m, g.n, KC.SparsificationClusterCoarseningContext(laziness_factor=0.5), seed)
    d_xadj, d_adj, d_vw, d_ew, _ = cg.device_arrays()
    h1 = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
    h1.set_graph_device(cg.n, cg.m, d_xadj, d_adj, d_vw, d_ew)
    mcw1 = 2 * mcw
    c1, _ = h1.cluster(mcw1)
    # host path
    cl0 = B.oracle_lp_cluster(g, 2, mcw, schedule=B.SYNC)
    con = CO.contract(g.xadj, g.adjncy, g.vwgt, g.adjwgt, cl0)
    o = S.sparsify_contracted(con, S.sparsification_target(g.m, g.n, con["c_n"]), seed)
    assert CO.equal(gpu_result(cg), o)
    cgraph = CSRGraph(o["c_xadj"], o["c_adjncy"], o["c_vwgt"], o["c_adjwgt"])
    assert np.array_equal(c1, B.oracle_lp_cluster(cgraph, 2, mcw1, schedule=B.SYNC))
    h2 = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
    h2.set_graph(cgraph)
    assert np.array_equal(c1, h2.cluster(mcw1)[0])


def test_laziness_and_seed_draw():
    g = rmat(13, 16, 5)
    h = new_handle()
    h.set_graph(g)
    draws = []
    cg = KC.contract_on_handle(h, np.arange(g.n, dtype=np.uint32))
    m0 = cg.m
    assert not KC.sparsify_level(h, cg, g.m, g.n, KC.SparsificationClusterCoarseningContext(), lambda: draws.append(1))
    assert cg.m == m0 and draws == []  # c_m <= 4 x target: lazy, no draw
    # target < 2 sparsifies without a draw
    assert KC.sparsify_level(h, cg, g.m, g.n, KC.SparsificationClusterCoarseningContext(0.5, 1e-9, 0.0),
                             lambda: draws.append(1))
    assert cg.m == 0 and draws == []
    cg.close()
    # sparsification with target >= 2 draws exactly once and uses the drawn value
    cg = KC.contract_on_handle(h, np.arange(g.n, dtype=np.uint32))
    con = CO.contract(g.xadj, g.adjncy, g.vwgt, g.adjwgt, np.arange(g.n, dtype=np.uint32))
    s_ctx = KC.SparsificationClusterCoarseningContext(laziness_factor=1.0)
    target = KC.sparsification_target(g.m, g.n, cg.n)
    assert target >= 2 and cg.m > target

    def draw():
        draws.append(77)
        return 77

    assert KC.sparsify_level(h, cg, g.m, g.n, s_ctx, draw)
    assert draws == [77]
    o = S.sparsify_contracted(con, target, 77)
    assert CO.equal(gpu_result(cg), o)
    assert not CO.equal(o, S.sparsify_contracted(con, target, 0))  # the seed matters on this level
    cg.close()
    # laziness_factor < 1 can ask for a target above the level's edge count: refused before any draw or device work
    cg = KC.contract_on_handle(h, (np.arange(g.n) // (g.n // 2)).astype(np.uint32))  # two clusters
    m_before = cg.m
    big = KC.sparsification_target(g.m, g.n, cg.n)
    assert big > m_before
    with pytest.raises(ValueError, match="exceeds"):
        KC.sparsify_level(h, cg, g.m, g.n, KC.SparsificationClusterCoarseningContext(laziness_factor=0.01), draw)
    assert draws == [77] and cg.m == m_before
    cg.close()


def test_projections_unchanged():
    g = random_weights(rmat(14, 16, 8), 2, max_adjwgt=5)
    h = new_handle()
    h.set_graph(g)
    cl = np.random.default_rng(3).integers(0, g.n // 4, g.n).astype(np.uint32)
    cg = KC.contract_on_handle(h, cl)
    coarse = np.random.default_rng(1).integers(0, 16, cg.n).astype(np.uint32)
    up, mapping = cg.project_up(coarse), cg.mapping().copy()
    down = cg.project_down(up)
    vw = cg.get().vwgt.copy()
    cg.sparsify(h, cg.m // 4, 5)
    assert np.array_equal(cg.project_up(coarse), up) and np.array_equal(cg.project_down(up), down)
    cg._mapping = None
    assert np.array_equal(cg.mapping(), mapping) and np.array_equal(cg.get().vwgt, vw)
    cg.close()


def test_refusals():
    lib = lp.load_library()
    g = H.grid2d(8, 8)
    h = new_handle()
    h.set_graph(g)
    cg = KC.contract_on_handle(h, np.arange(g.n, dtype=np.uint32))
    with pytest.raises(RuntimeError, match="exceeds"):
        cg.sparsify(h, cg.m + 1, 0)
    assert cg.m == g.m  # untouched
    assert lib.kmp_coarse_sparsify(None, cg._g, 2, 0, None) != 0
    assert lib.kmp_coarse_sparsify(h._h, None, 2, 0, None) != 0
    assert lib.kmp_coarse_sparsify(h._h, cg._g, 2, 0, None) == 0  # stats may be NULL
    cg.close()
    # an empty coarse graph: target 0 is the only valid target
    e = H.empty_graph(4)
    h.set_graph(e)
    cg = KC.contract_on_handle(h, np.arange(4, dtype=np.uint32))
    st = cg.sparsify(h, 0, 0)
    assert cg.m == 0 and st.c_m_after == 0 and list(cg.get().xadj) == [0] * 5
    cg.close()
