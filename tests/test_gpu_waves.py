"""Parity when launches need more than one pass over their grid, and along the sub-round axis (-m gpu).

Every grid-stride loop, work-queue refill and persistent-kernel iteration of an LP round only runs its second
pass once a work list outgrows the launch's grid. The inputs of the other parity tests are too small for that, so
here the grids are made small instead (KMP_GRID_CAP) or the inputs large, and the sub-round count, a public
setting, is varied. All of it is integer work: the GPU must equal the oracle's `sync` schedule bit for bit.

W1  capped grids (KMP_GRID_CAP = 1, 2, 3 CTAs) on ladders, R-MAT, grid and road graphs, clustering through the
    library and through the stepping API; each case asserts from the schedule's work lists that the loops it
    relies on take more than two passes
W2  sync_subrounds in {0, 1, .., 31} (0: the default 8; 32 is refused), granule_log2 in {0, 4, 12}: the small-group
    rule, move stamps only while 4 * S <= 64, the proposal-counter parity carried from group to group
W3  the refiner's commit at k up to 40000 (shared-memory privatisation limits, per-block loops at large k),
    the stepping API, min block weights
W4  production grids at a scale where lists exceed what an H100 holds resident (132 SMs x 2048 threads)
"""
import ctypes as C
import functools

import numpy as np
import pytest

from kaminpar_b200 import lp
from kaminpar_b200.graph import grid3d, random_weights, rgg2d, rmat
from oracle import bindings as B
from tests import helpers as H
from tests.test_gpu_edges import ctx_for, ladder, oracle_params, run_cluster, run_refine
from tests.test_gpu_parity import get_graph

pytestmark = pytest.mark.gpu

SEED = 3
UINT32_MAX = 0xFFFFFFFF
CTA_THREADS = 256                     # sweep_thread, the persistent low-group kernel, the commits
TEAMS_PER_CTA = {3: 8, 4: 4, 5: 1, 6: 1}  # sweep_team: vertices a CTA holds at once, by tier
RESIDENT_THREADS = 132 * 2048         # the most threads an H100 (132 SMs) holds resident
TIER3_TEAMS = 132 * 6 * 8             # tier-3 grid: 6 resident CTAs of 8 warp teams per SM


def graph(name):
    return ladder(name) if name in ("dense_w", "wide_unit") else get_graph(name)


def kernel_tiers(g):
    """Kernel tier of every vertex (tests/helpers.py tier_of, vectorised); degree 0 gives tier 0 but is never listed"""
    hub = H.HUB_MIN_DEGREE_W if g.adjwgt is not None else H.HUB_MIN_DEGREE_UNIT
    return np.searchsorted(np.array([8, 17, 32, 256, 1024, 4096, hub]), g.degrees().astype(np.int64), side="right")


def largest_lists(g, seed, S, granule_log2):
    """Largest work list of each kernel tier over the sub-rounds of the schedule (the oracle's sub-round index of
    every vertex; unvisited vertices, e.g. isolated ones, are in no list). 'g1': tiers 1 and 2 together, the one
    loop of degree group 1 in the persistent kernel."""
    sg = np.zeros(g.n, np.uint32)
    B.oracle().lpo_sync_subround_index(C.c_uint32(g.n), g.xadj.ctypes.data_as(C.c_void_p), C.c_int(seed),
                                       C.c_uint32(S), C.c_uint32(granule_log2), C.c_uint32(UINT32_MAX),
                                       sg.ctypes.data_as(C.c_void_p))
    t = kernel_tiers(g)
    listed = sg != UINT32_MAX
    out = {}
    for key, sel in [(tier, t == tier) for tier in range(8)] + [("g1", (t == 1) | (t == 2))]:
        m = listed & sel
        out[key] = int(np.bincount(sg[m]).max()) if m.any() else 0
    return out


def refine_case(g, seed, k, part, mbw, subrounds=8, granule_log2=4, min_bw=None, oracle_subrounds=None):
    """run_refine against the oracle, plus the visited-vertex count"""
    expect = B.oracle_lp_refine(g, seed, k, mbw, part, schedule=B.SYNC,
                                params=oracle_params(1, subrounds=subrounds if oracle_subrounds is None else
                                                     oracle_subrounds, granule_log2=granule_log2),
                                min_block_weights=min_bw, return_stats=True)
    gs, _ = run_refine(g, seed, k, part.copy(), mbw, subrounds=subrounds, granule_log2=granule_log2, min_bw=min_bw,
                       expect=expect)
    assert gs.nodes_visited == expect[2].nodes_visited
    return gs, expect


def random_refine(g, k, seed, subrounds=8, granule_log2=4):
    ctx, _ = ctx_for(g, k)
    part = np.random.default_rng(k + seed).integers(0, k, g.n).astype(np.uint32)
    return refine_case(g, seed, k, part, ctx.partition.max_block_weights(), subrounds, granule_log2)


# ------------------------------------------------------------------------------------------------
# W1: capped grids
# ------------------------------------------------------------------------------------------------
# graph, KMP_GRID_CAP, sync_subrounds, clustering driver, other knobs, the tiers (or 'g1') whose loops must take
# > 2 passes. 'library' clusters through LPClustering: degree groups 0 and 1 run as one persistent launch each per
# round. 'stepping' clusters through the stepping API at world 1: every sub-round is a sweep launch per tier
# (sweep_thread in tiers 0..2) and a commit that unpacks the gathered proposals.
W1 = [
    ("grid20", 1, 8, "library", {}, (0,)),
    ("grid20", 3, 1, "library", {"KMP_ACTIVATION": "push"}, (0,)),
    ("road60", 2, 1, "stepping", {}, (0,)),
    ("road60", 3, 1, "library", {"KMP_FORCE_P64": "1"}, (0,)),
    ("rmat16_hubs", 1, 8, "library", {"KMP_ACTIVATION": "pull"}, (0, "g1", 3)),
    ("rmat16_hubs", 2, 1, "library", {"KMP_ACTIVATION": "push"}, (0, "g1", 3, 4)),
    ("rmat16_hubs", 3, 1, "stepping", {}, (0, 1, 2, 3, 4)),
    ("rmat15_hubs_w", 1, 1, "library", {"KMP_FORCE_P64": "1", "KMP_ACTIVATION": "push"}, (0, "g1", 3, 4)),
    ("rmat15_hubs_w", 3, 1, "library", {}, (0, "g1", 3)),
    ("rmat15_hubs_w", 3, 1, "stepping", {"KMP_ACTIVATION": "pull"}, (0, 1, 2, 3)),
    ("wide_unit", 2, 1, "stepping", {"KMP_ACTIVATION": "push"}, (0, 1)),
    ("wide_unit", 3, 1, "library", {"KMP_FORCE_P64": "1"}, (0, "g1")),
    ("dense_w", 1, 8, "stepping", {}, (4,)),
    ("dense_w", 3, 1, "library", {"KMP_ACTIVATION": "push"}, (4,)),
]


def w1_id(case):
    name, cap, S, driver, env, _ = case
    parts = [name, f"cap{cap}", f"S{S}"] + ([driver] if driver != "library" else [])
    return "-".join(parts + [f"{k[4:].lower()}={v}" for k, v in env.items()])


def stepping_cluster(g, seed, mcw, subrounds):
    """Clustering through the stepping API at world 1 (ShardedLP + CudaBackend): labels, moves per round, edges and
    vertices scanned equal the oracle's, as run_cluster checks for the library path"""
    import torch

    from kaminpar_b200.dist import CudaBackend, ShardedLP

    ctx, _ = ctx_for(g, 8, seed)
    ctx.engine.sync_subrounds = subrounds
    h = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
    try:
        h.set_graph(g)
        drv = ShardedLP(CudaBackend(h, torch.device("cuda", 0)), g.n, ctx.coarsening.clustering.lp.num_iterations, 0, 1)
        c, moved, gs = drv.compute_clustering(mcw)
    finally:
        h.close()
    expect, st = B.oracle_lp_cluster(g, seed, mcw, schedule=B.SYNC, params=oracle_params(0, subrounds=subrounds),
                                     return_stats=True)
    assert np.array_equal(c, expect)
    assert list(moved) == list(st[0].moved[: st[0].iterations])
    assert gs.edges_scanned == st[0].edges_scanned and gs.nodes_visited == st[0].nodes_visited


@pytest.mark.parametrize("case", W1, ids=[w1_id(c) for c in W1])
def test_w1_capped_grids(case, monkeypatch):
    name, cap, S, driver, env, relies = case
    monkeypatch.setenv("KMP_GRID_CAP", str(cap))
    for key, value in env.items():
        monkeypatch.setenv(key, value)
    g = graph(name)
    sizes = largest_lists(g, SEED, S, 4)
    for t in relies:
        thread_loop = t == "g1" or t <= 2
        per_pass = cap * (CTA_THREADS if thread_loop else TEAMS_PER_CTA.get(t, 8))
        assert sizes[t] > 2 * per_pass, (t, sizes[t], per_pass)
    _, mcw = ctx_for(g, 8)
    if driver == "stepping":
        stepping_cluster(g, SEED, mcw, S)
    else:
        gs = run_cluster(g, SEED, mcw, subrounds=S)  # labels, moves per round, edges and vertices scanned
        rounds = gs.iterations
        assert rounds > 0
        launches = [rounds if sizes[0] else 0, rounds if sizes["g1"] else 0]  # one persistent launch per group, round
        assert list(gs.group_launches[:2]) == launches, list(gs.group_launches)
    random_refine(g, 8, SEED, subrounds=S)


# ------------------------------------------------------------------------------------------------
# W2: the sub-round axis
# ------------------------------------------------------------------------------------------------
# graph, sync_subrounds, sync_granule_log2: every S in {1, 2, 3, 4, 5, 7, 16, 17, 31} and every granule in {0, 4, 12}
W2 = [
    ("rmat16_hubs", 1, 0), ("rmat16_hubs", 3, 4), ("rmat16_hubs", 17, 12),
    ("ladder_wide", 2, 12), ("ladder_wide", 31, 4),
    ("grid20", 5, 0), ("grid20", 16, 4),
    ("star_hub", 7, 12), ("star_hub", 4, 0),
    ("with_isolated", 31, 0), ("with_isolated", 1, 12),
]


@pytest.mark.parametrize("name,S,G", W2)
def test_w2_subround_axis(name, S, G, monkeypatch):
    """Pull activation is forced: it needs a move stamp per sub-round, which exist while 4 * S <= 64; from S = 17 on
    every round pushes."""
    monkeypatch.setenv("KMP_ACTIVATION", "pull")
    g = graph(name)
    _, mcw = ctx_for(g, 8)
    gs = run_cluster(g, SEED, mcw, subrounds=S, granule_log2=G)
    assert gs.pull_rounds == (gs.iterations if S <= 16 else 0), (gs.pull_rounds, gs.iterations)
    gs, _ = random_refine(g, 8, SEED, subrounds=S, granule_log2=G)
    assert gs.pull_rounds == (gs.iterations if S <= 16 else 0), (gs.pull_rounds, gs.iterations)


def test_w2_low_group_parity_carries_over():
    """With S = 3 group 0 of rmat16_hubs has three non-empty sub-rounds: group 1 starts on the other proposal
    counter. The persistent kernels must hand the parity on as the per-sub-round path does."""
    g = graph("rmat16_hubs")
    sizes = largest_lists(g, SEED, 3, 4)
    assert sizes[0] > 0 and sizes["g1"] > 0
    _, mcw = ctx_for(g, 8)
    for seed in (SEED, 11):
        gs = run_cluster(g, seed, mcw, subrounds=3)
        assert gs.group_launches[0] == gs.iterations and gs.group_launches[1] == gs.iterations


def test_w2_zero_subrounds_mean_the_default():
    """sync_subrounds = 0 is the default (8) in the engine; the oracle's S = 0 would be one sub-round, which gives
    another clustering on this graph."""
    g = graph("rmat16_hubs")
    _, mcw = ctx_for(g, 8)
    one = B.oracle_lp_cluster(g, SEED, mcw, schedule=B.SYNC, params=oracle_params(0, subrounds=1))
    eight = B.oracle_lp_cluster(g, SEED, mcw, schedule=B.SYNC, params=oracle_params(0, subrounds=8))
    assert not np.array_equal(one, eight)
    run_cluster(g, SEED, mcw, subrounds=0, oracle_subrounds=8)
    k = 8
    ctx, _ = ctx_for(g, k)
    part = np.random.default_rng(1).integers(0, k, g.n).astype(np.uint32)
    refine_case(g, SEED, k, part, ctx.partition.max_block_weights(), subrounds=0, oracle_subrounds=8)


def test_w2_more_than_31_subrounds_are_refused():
    """The work-list keys are 8 bits (8 tiers x S sub-rounds + the unvisited key): S = 31 is the largest."""
    g = graph("with_isolated")
    ctx, mcw = ctx_for(g, 8)
    ctx.engine.sync_subrounds = 32
    clusterer = lp.LPClustering(ctx.coarsening, ctx.engine)
    clusterer.set_max_cluster_weight(mcw)
    with pytest.raises(RuntimeError, match=r"error -1:.*sync_subrounds too large \(max 31\)"):
        clusterer.compute_clustering(g)
    p_graph = lp.PartitionedGraph(g, 8, np.arange(g.n, dtype=np.uint32) % 8)
    refiner = lp.LabelPropagationRefiner(ctx)
    with pytest.raises(RuntimeError, match=r"error -1:.*sync_subrounds too large \(max 31\)"):
        refiner.initialize(p_graph)
        refiner.refine(p_graph, ctx.partition)


# ------------------------------------------------------------------------------------------------
# W3: the refiner's commit at large k
# ------------------------------------------------------------------------------------------------
# 512 / 8192: k * 16 and k ints of shared memory (kSmemPrivLimit); 16896: k * 16 = 2112 x 128 histogram entries;
# 40000: more than twice that. The commit loops over blocks and histogram entries grid-stride, in several passes here.
W3_KS = (512, 513, 8192, 8193, 16896, 16897, 40000)
W3_SEED = 2


@functools.lru_cache(maxsize=None)
def grid64():
    return grid3d(64)  # 2^18 vertices: blocks still hold ~6 vertices at k = 40000


@functools.lru_cache(maxsize=None)
def w3_expect(k, kind):
    """(partition, max / min block weights, oracle result) of a W3 case, shared by its engine paths"""
    g = grid64()
    ctx, _ = ctx_for(g, k)
    mbw = ctx.partition.max_block_weights().copy()
    part = np.random.default_rng(k).integers(0, k, g.n).astype(np.uint32)
    min_bw = None
    if kind == "min":
        min_bw = np.full(k, max(1, g.n // k - 2), np.int32)
    elif kind == "hot":
        # Block k - 1 (past the first 16896 blocks) holds every vertex with three even coordinates. Each vertex with
        # exactly one odd coordinate has two neighbours there and none in its own random block: it proposes into
        # block k - 1 in every sub-round, and the block's room (a few thousand) keeps the commit contended, so its
        # level histogram decides every sub-round.
        x = np.arange(g.n)
        hot = ((x % 64) % 2 == 0) & (((x // 64) % 64) % 2 == 0) & ((x // 4096) % 2 == 0)
        part = np.random.default_rng(k).integers(0, k - 1, g.n).astype(np.uint32)
        part[hot] = k - 1
        mbw[k - 1] = int(hot.sum()) + 5000
    expect = B.oracle_lp_refine(g, W3_SEED, k, mbw, part, schedule=B.SYNC, params=oracle_params(1),
                                min_block_weights=min_bw, return_stats=True)
    assert sum(expect[2].moved[: expect[2].iterations]) > 0
    return part, mbw, min_bw, expect


def w3_run(k, kind):
    g = grid64()
    part, mbw, min_bw, expect = w3_expect(k, kind)
    gs, _ = run_refine(g, W3_SEED, k, part.copy(), mbw, min_bw=min_bw, expect=expect)
    assert gs.nodes_visited == expect[2].nodes_visited
    return expect


@pytest.mark.parametrize("k", W3_KS)
def test_w3_refiner_at_large_k(k):
    w3_run(k, "random")


def test_w3_blocks_past_the_reset_grid_stay_contended():
    """k = 16897: only block 16896 lies past the first 2112 x 128 histogram entries, and it is proposed into in every
    sub-round; a histogram left from an earlier sub-round would lower what it accepts."""
    w3_run(16897, "hot")


def test_w3_min_block_weights_at_large_k():
    w3_run(40000, "min")


def test_w3_stepping_api_at_large_k():
    """The stepping API at world 1 (ShardedLP + CudaBackend): proposals packed, then unpacked, accumulated and
    committed by one cooperative launch"""
    import torch

    from kaminpar_b200.dist import CudaBackend, ShardedLP

    k = 40000
    g = grid64()
    part, mbw, _, (ep, ebw, st) = w3_expect(k, "random")
    ctx, _ = ctx_for(g, k, W3_SEED)
    h = lp.LPHandle(lp._refine_config(ctx.refinement.lp, ctx.engine))
    h.set_graph(g)
    drv = ShardedLP(CudaBackend(h, torch.device("cuda", 0)), g.n, ctx.refinement.lp.num_iterations, 0, 1)
    p, bw, moved, _ = drv.refine(k, mbw, part.copy())
    h.close()
    assert np.array_equal(p, ep) and np.array_equal(bw, ebw)
    assert list(moved) == list(st.moved[: st.iterations])


# ------------------------------------------------------------------------------------------------
# W4: natural scale, production grids
# ------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def w4_graph(name):
    if name == "grid144":
        return grid3d(144)
    if name == "rgg21":
        return rgg2d(1 << 21, 7)
    return random_weights(rmat(20, 8, 3), 5, max_vwgt=3, max_adjwgt=5)  # "rmat20_w"


def test_w4_grid144_group0_beyond_the_resident_grid():
    g = w4_graph("grid144")
    sizes = largest_lists(g, SEED, 8, 4)
    assert sizes[0] > RESIDENT_THREADS, sizes
    _, mcw = ctx_for(g, 8)
    gs = run_cluster(g, SEED, mcw)
    assert gs.group_launches[0] == gs.iterations


def test_w4_rgg_group1_in_one_list():
    g = w4_graph("rgg21")
    sizes = largest_lists(g, SEED, 1, 4)
    assert sizes["g1"] > RESIDENT_THREADS, sizes
    _, mcw = ctx_for(g, 8)
    gs = run_cluster(g, SEED, mcw, subrounds=1)
    assert gs.group_launches[1] == gs.iterations
    random_refine(g, 64, SEED, subrounds=1)


def test_w4_weighted_rmat_team_queue_refills():
    g = w4_graph("rmat20_w")
    sizes = largest_lists(g, SEED, 2, 4)
    assert sizes[3] > TIER3_TEAMS, sizes
    _, mcw = ctx_for(g, 8)
    run_cluster(g, SEED, mcw, subrounds=2)
