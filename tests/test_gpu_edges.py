"""Parity at the edges of the sweep kernels (-m gpu). The inputs are built to land where one of the eight sweep
kernels could be subtly wrong: degrees on both sides of every tier boundary, rating tables just below and above
the size at which they switch from direct indexing to hashing, labels whose hashes collide (probe chains that wrap
around, an overflowing hub bucket, multi-pass hub selection), cluster and block weights exactly at a limit or one
above it, vertex weights near 2^24, neighbour limits that cut inside a hub chunk, labels at the limit of the 24-bit
gather word, and a device graph whose adjacency is not 16-byte aligned. All of it is integer work: the GPU must
equal the oracle's `sync` schedule bit for bit.

T0  kmp_lp_select_all == lpo_sync_select_all on crafted frozen states
T1  full clustering / refinement == oracle sync (labels, block weights, moves per round, edges scanned); every
    kernel tier the input covers must have run (last_stats.group_nodes), so a change of the tier rule cannot turn
    a case into a no-op.
"""
import functools
import zlib

import numpy as np
import pytest

from kaminpar_b200 import lp
from kaminpar_b200.graph import CSRGraph, rmat
from oracle import bindings as B
from tests import helpers as H

pytestmark = pytest.mark.gpu

UINT32_MAX = 0xFFFFFFFF
SEED = 3
NC = len(H.LADDER_DEGREES)  # centres per ladder
DENSE_POOL = 256            # parallel edges: n = 278 < 512, so every team table can also be direct-indexed
WIDE_POOL = 18436           # distinct neighbours for the largest ladder degree (18433)
MAG_POOL = 112              # 128 vertices of weight ~2^24: total weight just below 2^31 - 1
# team table sizes (SLOTS) are 512 / 2048 / 8192 / 16384 (edge weights) / 32768 (unit): label counts on both sides
DENSE_NUM_LABELS = (512, 513, 2048, 2049, 8192, 8193, 16384, 16385, 32768, 32769)
WIDE_NUM_LABELS = (None, 32768, 32769, 1 << 20)  # None: n; 2^20: > 640 colliding labels in one hub bucket


@functools.lru_cache(maxsize=None)
def ladder(name):
    degs = sorted(H.LADDER_DEGREES)  # the largest hub is the last vertex: its adjacency ends adjncy
    if name == "dense_unit":
        return H.degree_ladder(degs, DENSE_POOL, multi=True, seed=1)
    if name == "dense_w":
        return H.degree_ladder(degs, DENSE_POOL, weighted=True, multi=True, seed=2)
    if name == "wide_unit":
        return H.degree_ladder(degs, WIDE_POOL, seed=3)
    if name == "wide_w":
        return H.degree_ladder(degs, WIDE_POOL, weighted=True, seed=4)
    if name.startswith("tail"):  # m % 4 == 1, 2, 3: the hub's last chunk ends inside a 16-byte block
        return H.degree_ladder(degs, WIDE_POOL, seed=5, m_mod4=int(name[4:]))
    if name == "mag_small":  # vertex weights ~2^24, total weight just below 2^31 - 1
        g = H.degree_ladder(sorted(H.TIER_EDGE_DEGREES), MAG_POOL, weighted=True, multi=True, seed=6)
        return H.magnified(g, MAG_POOL, seed=6)
    raise KeyError(name)


def npool(name):
    return {"dense_unit": DENSE_POOL, "dense_w": DENSE_POOL, "mag_small": MAG_POOL}.get(name, WIDE_POOL)


def seed_of(*parts):
    return zlib.crc32(repr(parts).encode())


def num_labels_for(g):
    return DENSE_NUM_LABELS if g.n < 512 else tuple(g.n if x is None else x for x in WIDE_NUM_LABELS)


def ctx_for(g, k, seed=SEED):
    ctx = lp.create_default_context()
    ctx.engine.seed = seed
    ctx.partition.setup(g, k, 0.03)
    mcw = lp.compute_max_cluster_weight(ctx.coarsening, ctx.partition, g.n, g.total_node_weight())
    return ctx, mcw


def handle(g, mode, max_num_neighbors=UINT32_MAX, large_degree_threshold=UINT32_MAX):
    ctx, _ = ctx_for(g, 8)
    c = ctx.coarsening.clustering.lp if mode == 0 else ctx.refinement.lp
    c.max_num_neighbors, c.large_degree_threshold = max_num_neighbors, large_degree_threshold
    h = lp.LPHandle(lp._cluster_config(c, ctx.engine) if mode == 0 else lp._refine_config(c, ctx.engine))
    h.set_graph(g)
    return h


def oracle_params(mode, max_num_neighbors=UINT32_MAX, large_degree_threshold=UINT32_MAX, commit_passes=None,
                  subrounds=B.SYNC_SUBROUNDS_DEFAULT, granule_log2=B.SYNC_GRANULE_LOG2_DEFAULT):
    p = B.default_cluster_params() if mode == 0 else B.default_refine_params()
    p.max_num_neighbors, p.large_degree_threshold = max_num_neighbors, large_degree_threshold
    return B.oracle_params(p, subrounds, granule_log2, commit_passes=commit_passes or (1 if mode == 0 else 4))


def check_t0(h, g, mode, labels, weights, params=None, **kw):
    t_gpu, f_gpu = h.select_all(mode, labels, weights, call_index=1, iteration=2, **kw)
    t_cpu, f_cpu = B.oracle_sync_select_all(mode, g, labels, weights, seed=SEED, call=1, iteration=2, params=params,
                                            **kw)
    bad = np.nonzero(t_gpu != t_cpu)[0]
    assert bad.size == 0, (bad[:8], g.degrees()[bad[:8]], t_gpu[bad[:8]], t_cpu[bad[:8]])
    if mode == 0:
        deg = g.degrees()
        assert np.array_equal(f_gpu[deg > 0], f_cpu[deg > 0])
    return t_cpu


def test_ladders_cover_every_tier():
    """The ladders reach all eight kernel tiers, and their degrees sit on both sides of every boundary."""
    for name in ("dense_unit", "dense_w", "wide_unit", "wide_w", "tail1"):
        assert H.tiers_present(ladder(name)) == list(range(8)), name
    for d in H.TIER_EDGE_DEGREES[::2]:
        assert H.tier_of(d, False) + 1 == H.tier_of(d + 1, False) or d == 8191
    assert H.tier_of(8191, True) == 6 and H.tier_of(8192, True) == 7
    assert H.tier_of(16383, False) == 6 and H.tier_of(16384, False) == 7
    assert [ladder(f"tail{r}").m % 4 for r in (1, 2, 3)] == [1, 2, 3]
    assert ladder("mag_small").total_node_weight() < (1 << 31) - 1
    assert ladder("mag_small").total_node_weight() > (1 << 30)


# ------------------------------------------------------------------------------------------------
# T0: frozen-state selection
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pattern", H.LABEL_PATTERNS)
@pytest.mark.parametrize("name", ["dense_unit", "dense_w", "wide_unit", "wide_w"])
def test_t0_cluster_selection_at_the_edges(name, pattern):
    g = ladder(name)
    pool = npool(name)
    rng = np.random.default_rng(seed_of(name, pattern))
    graphs = [(g, 1000)]
    if g.vwgt is not None:
        graphs.append((H.magnified(g, pool), H.MAG_LIMIT))
    h = handle(g, 0)
    for gg, mcw in graphs:
        if gg is not g:
            h.set_graph(gg)
        for nl in num_labels_for(g):
            for feas in ("lo", "hi", "mix"):
                labels, weights = H.frozen_cluster_state(gg, pool, nl, pattern, feas, rng, mcw=mcw)
                t = check_t0(h, gg, 0, labels, weights, max_cluster_weight=mcw)
                if pattern == "one" and feas != "mix":  # the centres' single candidate: exactly (in)feasible
                    moved = t[pool:] != labels[pool:]
                    assert moved.all() if feas == "lo" else not moved.any()
    h.close()


@pytest.mark.parametrize("pattern", H.LABEL_PATTERNS)
@pytest.mark.parametrize("name", ["dense_unit", "dense_w", "wide_unit", "wide_w"])
def test_t0_refine_selection_at_the_edges(name, pattern):
    g = ladder(name)
    pool = npool(name)
    rng = np.random.default_rng(seed_of(name, pattern, 1))
    h = handle(g, 1)
    cases = [(g, k, 10000) for k in num_labels_for(g)]
    if g.vwgt is not None:
        gm = H.magnified(g, pool)
        cases += [(gm, k, H.MAG_LIMIT) for k in num_labels_for(g)[:2]]
    cur = g
    for gg, k, limit in cases:
        if gg is not cur:
            h.set_graph(gg)
            cur = gg
        cw = 1 if gg.vwgt is None else int(gg.vwgt[pool])
        for regime in ("fit", "over"):
            for feas in ("lo", "hi", "mix"):
                labels, bw, maxw, own = H.frozen_refine_state(gg, pool, k, pattern, regime, feas, rng, limit=limit)
                mins = [None]
                if feas == "mix":  # weight[own] - w(u) == min (may leave) and == min - 1 (stays)
                    for d in (0, 1):
                        mn = np.zeros(k, np.int32)
                        mn[own] = int(bw[own]) - cw + d
                        mins.append(mn)
                for mn in mins:
                    t = check_t0(h, gg, 1, labels, bw, max_weights=maxw, min_weights=mn)
                    if pattern == "one" and feas != "mix":
                        moved = t[pool:] != own
                        assert moved.all() if feas == "lo" else not moved.any()
    h.close()


@pytest.mark.parametrize("mnn", [7, 8, 31, 255, 2047, 2049, 8191, 16385])
@pytest.mark.parametrize("name", ["dense_w", "wide_unit"])
def test_t0_neighbour_limits(name, mnn):
    """max_num_neighbors cuts every scan -- inside a 2048-edge hub chunk and a 256-edge slice for 2047 / 2049 /
    8191 / 16385; a vertex whose degree reaches large_degree_threshold (a ladder degree) is not visited."""
    g = ladder(name)
    pool = npool(name)
    rng = np.random.default_rng(mnn)
    for thr in (UINT32_MAX, 4096, 16640):
        for mode in (0, 1):
            h = handle(g, mode, mnn, thr)
            params = oracle_params(mode, mnn, thr)
            for pattern in ("distinct", "tie", "collide"):
                if mode == 0:
                    labels, w = H.frozen_cluster_state(g, pool, 1 << 20 if pattern == "collide" else g.n, pattern,
                                                       "mix", rng)
                    check_t0(h, g, 0, labels, w, params=params, max_cluster_weight=1000)
                else:
                    k = 1 << 20 if pattern == "collide" else 600
                    labels, bw, maxw, _ = H.frozen_refine_state(g, pool, k, pattern, "over", "mix", rng)
                    check_t0(h, g, 1, labels, bw, params=params, max_weights=maxw)
            h.close()


# ------------------------------------------------------------------------------------------------
# T1: full calls
# ------------------------------------------------------------------------------------------------
def assert_tiers_ran(stats, g, thr=UINT32_MAX):
    expect = H.tiers_present(g, thr)
    ran = [t for t in range(8) if stats.group_nodes[t] > 0]
    assert ran == expect, (ran, expect)


def run_cluster(g, seed, mcw, mnn=UINT32_MAX, thr=UINT32_MAX, passes=1, subrounds=8, granule_log2=4,
                oracle_subrounds=None):
    """oracle_subrounds: the oracle's sub-round count where it differs from the engine's (default: the same)"""
    ctx, _ = ctx_for(g, 8, seed)
    ctx.coarsening.clustering.lp.max_num_neighbors = mnn
    ctx.coarsening.clustering.lp.large_degree_threshold = thr
    ctx.engine.cluster_commit_passes = passes
    ctx.engine.sync_subrounds, ctx.engine.sync_granule_log2 = subrounds, granule_log2
    clusterer = lp.LPClustering(ctx.coarsening, ctx.engine)
    clusterer.set_max_cluster_weight(mcw)
    c = clusterer.compute_clustering(g)
    params = oracle_params(0, mnn, thr, passes, subrounds if oracle_subrounds is None else oracle_subrounds,
                           granule_log2)
    expect, st = B.oracle_lp_cluster(g, seed, mcw, schedule=B.SYNC, params=params, return_stats=True)
    assert np.array_equal(c, expect)
    gs = clusterer.last_stats
    assert gs.moved_list() == list(st[0].moved[: st[0].iterations])
    assert gs.edges_scanned == st[0].edges_scanned and gs.nodes_visited == st[0].nodes_visited
    assert gs.num_clusters == st[0].num_clusters and gs.two_hop_ran == st[0].two_hop_ran
    assert H.cluster_weights_ok(g, c, mcw)
    return gs


def run_refine(g, seed, k, part, mbw, mnn=UINT32_MAX, thr=UINT32_MAX, passes=4, subrounds=8, granule_log2=4,
               min_bw=None, expect=None):
    """expect: the oracle's (partition, block weights, stats) of this call when the caller already has them"""
    ctx, _ = ctx_for(g, k, seed)
    ctx.refinement.lp.max_num_neighbors = mnn
    ctx.refinement.lp.large_degree_threshold = thr
    ctx.engine.refine_commit_passes = passes
    ctx.engine.sync_subrounds, ctx.engine.sync_granule_log2 = subrounds, granule_log2
    ctx.partition.setup(g, [int(x) for x in mbw])
    if min_bw is not None:
        ctx.partition.setup_min_block_weights([int(x) for x in min_bw])
    p_graph = lp.PartitionedGraph(g, k, part)
    refiner = lp.LabelPropagationRefiner(ctx)
    refiner.initialize(p_graph)
    refiner.refine(p_graph, ctx.partition)
    if expect is None:
        expect = B.oracle_lp_refine(g, seed, k, mbw, part, schedule=B.SYNC,
                                    params=oracle_params(1, mnn, thr, passes, subrounds, granule_log2),
                                    min_block_weights=min_bw, return_stats=True)
    ep, ebw, st = expect
    assert np.array_equal(p_graph.partition, ep)
    assert np.array_equal(p_graph.block_weights(), ebw)
    gs = refiner.last_stats
    assert gs.moved_list() == list(st.moved[: st.iterations]) and gs.edges_scanned == st.edges_scanned
    return gs, ep


LADDERS = ["dense_unit", "dense_w", "wide_unit", "wide_w", "tail1", "tail2", "tail3", "mag_small"]


@pytest.mark.parametrize("name", LADDERS)
def test_t1_ladder_clustering_and_refinement(name):
    g = ladder(name)
    _, mcw = ctx_for(g, 8)
    for seed in (0, 5):
        assert_tiers_ran(run_cluster(g, seed, mcw), g)
    for k in (4, 513, 2049):
        ctx, _ = ctx_for(g, k)
        part = np.random.default_rng(k).integers(0, k, g.n).astype(np.uint32)
        gs, _ = run_refine(g, 2, k, part, ctx.partition.max_block_weights())
        assert_tiers_ran(gs, g)


@pytest.mark.parametrize("mnn,thr", [(8, UINT32_MAX), (255, UINT32_MAX), (2049, UINT32_MAX), (8191, 16640),
                                     (16385, 16384), (UINT32_MAX, 4096)])
@pytest.mark.parametrize("name", ["dense_w", "wide_unit", "tail3"])
def test_t1_neighbour_limits(name, mnn, thr):
    g = ladder(name)
    _, mcw = ctx_for(g, 8)
    assert_tiers_ran(run_cluster(g, 1, mcw, mnn, thr), g, thr)
    k = 16
    ctx, _ = ctx_for(g, k)
    part = np.random.default_rng(3).integers(0, k, g.n).astype(np.uint32)
    gs, _ = run_refine(g, 1, k, part, ctx.partition.max_block_weights(), mnn, thr)
    assert_tiers_ran(gs, g, thr)


def test_t1_contended_cluster_commit():
    """Round 0 on the dense ladder: nearly every pool vertex proposes the same hub's cluster. Sweeping the cluster
    weight limit over small values lets the room of that cluster end exactly at one priority level of the commit
    ladder for some of them (w_t + cum == max)."""
    g = ladder("dense_unit")
    for mcw in range(2, 48):
        run_cluster(g, 7, mcw)


def test_cluster_commit_passes_other_than_one_are_refused():
    """The clusterer's commit kernels decide in one pass (no departure credit, unlike the refiner's): a config
    asking for more passes would silently differ from the oracle's multi-pass rule, so it is refused."""
    g = ladder("dense_unit")
    ctx, mcw = ctx_for(g, 8)
    ctx.engine.cluster_commit_passes = 4
    clusterer = lp.LPClustering(ctx.coarsening, ctx.engine)
    clusterer.set_max_cluster_weight(mcw)
    with pytest.raises(RuntimeError, match="error -4:.*single-pass"):
        clusterer.compute_clustering(g)


@pytest.mark.parametrize("passes", [1, 4])
@pytest.mark.parametrize("name", ["dense_unit", "dense_w"])
def test_t1_contended_refine_commit(name, passes):
    """All centres in block 0, the pool spread over blocks 1..3: every pool vertex proposes block 0, whose room
    (max - weight) is swept so that it ends exactly at one priority level for some of the runs."""
    g = ladder(name)
    pool = npool(name)
    k = 4
    part = np.concatenate([1 + np.arange(pool) % 3, np.zeros(g.n - pool)]).astype(np.uint32)
    bw = H.block_weights(g, part, k)
    for room in range(0, 40):
        mbw = np.full(k, int(bw.sum()), np.int32)
        mbw[0] = int(bw[0]) + room
        run_refine(g, 4, k, part, mbw, passes=passes)


# ------------------------------------------------------------------------------------------------
# 24-bit gather word: labels up to 0xFFFFFF (4-byte word) and above 2^24 (8-byte word, switched automatically)
# ------------------------------------------------------------------------------------------------
def top_block_graph(n):
    """n vertices, all isolated except an R-MAT block (2^12 vertices) on the highest ids; R-MAT's vertex 0 (its
    largest hub) becomes vertex n - 1, so label n - 1 is on many neighbour lists from the first round on."""
    b = rmat(12, 8, 21)
    src = n - 1 - np.repeat(np.arange(b.n, dtype=np.int64), b.degrees().astype(np.int64))
    dst = n - 1 - b.adjncy.astype(np.int64)
    order = np.argsort(src, kind="stable")
    xadj = np.zeros(n + 1, np.int64)
    xadj[1:] = np.cumsum(np.bincount(src, minlength=n))
    return CSRGraph(xadj.astype(np.uint32), dst[order].astype(np.uint32))


@pytest.mark.parametrize("n", [1 << 24, (1 << 24) + 4096])
def test_t1_labels_at_the_24_bit_word_limit(n):
    g = top_block_graph(n)
    assert g.adjncy.max() == n - 1
    _, mcw = ctx_for(g, 8)
    gs = run_cluster(g, 2, mcw)  # incl. the isolated-vertex post pass
    assert gs.two_hop_ran
    h = handle(g, 0)
    labels = np.arange(n, dtype=np.uint32)
    w = np.ones(n, np.int32)
    check_t0(h, g, 0, labels, w, max_cluster_weight=mcw)
    h.close()


# ------------------------------------------------------------------------------------------------
# kmp_lp_set_graph_device alignment contract
# ------------------------------------------------------------------------------------------------
def device_arrays(g, adj_offset=0):
    import torch

    xadj = torch.from_numpy(g.xadj.view(np.int32).copy()).cuda()
    buf = torch.zeros(g.m + 4, dtype=torch.int32, device="cuda")
    buf[adj_offset: adj_offset + g.m] = torch.from_numpy(g.adjncy.view(np.int32).copy()).cuda()
    vw = None if g.vwgt is None else torch.from_numpy(g.vwgt.copy()).cuda()
    ew = None if g.adjwgt is None else torch.from_numpy(g.adjwgt.copy()).cuda()
    return xadj, buf, vw, ew


def test_set_graph_device_refuses_unaligned_pointers():
    g = ladder("dense_w")
    xadj, buf, vw, ew = device_arrays(g)
    ptrs = [xadj.data_ptr(), buf.data_ptr(), vw.data_ptr(), ew.data_ptr()]
    h = handle(g, 0)
    for i in range(4):
        for off in (1, 2, 3):
            p = list(ptrs)
            p[i] += off
            with pytest.raises(RuntimeError, match="error -1:.*4-byte aligned"):
                h.set_graph_device(g.n, g.m, *p)
    h.set_graph_device(g.n, g.m, *ptrs)  # aligned: accepted
    h.close()


@pytest.mark.parametrize("off", [1, 2, 3])
@pytest.mark.parametrize("name", ["tail1", "wide_w"])
def test_adjncy_view_off_a_16_byte_boundary(name, off):
    """adjncy as a view 4, 8 or 12 bytes past a 16-byte boundary (e.g. d_adj[1:] of a larger buffer): the hub tier
    must not bulk-copy from it; clustering and refinement stay the oracle's."""
    g = ladder(name)
    xadj, buf, vw, ew = device_arrays(g, off)
    adj_ptr = buf.data_ptr() + 4 * off
    assert adj_ptr % 16 == 4 * off
    ptrs = (xadj.data_ptr(), adj_ptr, 0 if vw is None else vw.data_ptr(), 0 if ew is None else ew.data_ptr())
    _, mcw = ctx_for(g, 8)
    h = handle(g, 0)
    h.set_graph_device(g.n, g.m, *ptrs)
    c, st = h.cluster(mcw)
    assert np.array_equal(c, B.oracle_lp_cluster(g, SEED, mcw, schedule=B.SYNC))
    assert st.group_nodes[7] > 0
    h.close()
    k = 8
    ctx, _ = ctx_for(g, k)
    part = np.random.default_rng(off).integers(0, k, g.n).astype(np.uint32)
    h = handle(g, 1)
    h.set_graph_device(g.n, g.m, *ptrs)
    p = part.copy()
    _, bw, st = h.refine(k, ctx.partition.max_block_weights(), p)
    ep, ebw = B.oracle_lp_refine(g, SEED, k, ctx.partition.max_block_weights(), part, schedule=B.SYNC,
                                 params=oracle_params(1))
    assert np.array_equal(p, ep) and np.array_equal(bw, ebw)
    assert st.group_nodes[7] > 0
    h.close()
