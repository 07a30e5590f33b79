"""Parity tests proper (-m gpu): the CUDA path, called through the C ABI, against the CPU oracle's
`sync` schedule -- bit-exact label vectors, block weights and statistics (all integer work).

T0  per-vertex decision on frozen state  (kmp_lp_select_all == lpo_sync_select_all)
T1  full compute_clustering / refine     (GPU == oracle sync), incl. golden-input graphs
T3  GPU vs reference (seq): validity, feasibility and quality side by side (not bit-identical by
    construction -- the reference is asynchronous; see DESIGN.md)
"""
import numpy as np
import pytest

from kaminpar_b200 import lp
from kaminpar_b200.graph import grid3d, random_weights, rgg2d, rmat, road_like
from oracle import bindings as B
from tests import helpers as H

pytestmark = pytest.mark.gpu


def ctx_for(g, k, seed=0):
    ctx = lp.create_default_context()
    ctx.engine.seed = seed
    ctx.partition.setup(g, k, 0.03)
    mcw = lp.compute_max_cluster_weight(ctx.coarsening, ctx.partition, g.n, g.total_node_weight())
    return ctx, mcw


def graphs():
    out = {}
    for name in ("rgg2d_k4", "walshaw_k16", "walshaw_unsorted", "rmat13_w", "grid12", "road60", "star30000"):
        out[name] = H.load_case(name)[0]
    g0 = rmat(15, 16, 7)
    out["rmat15_sorted"] = B.oracle_rearrange(g0)[0]          # hubs up to deg ~ 10^4 (sweep_block)
    out["rmat14_unsorted_w"] = random_weights(rmat(14, 8, 9), 3, max_vwgt=4, max_adjwgt=7)
    out["rmat16_hubs"] = B.oracle_rearrange(rmat(16, 32, 5))[0]  # vertices in every kernel tier (deg 1 .. > 8192)
    out["rmat15_hubs_w"] = random_weights(B.oracle_rearrange(rmat(15, 48, 11))[0], 5, max_vwgt=3, max_adjwgt=5)
    out["grid20"] = B.oracle_rearrange(grid3d(20))[0]
    out["rgg_2e15"] = B.oracle_rearrange(rgg2d(1 << 15, 4))[0]
    out["star_hub"] = H.big_star(40000)                        # global-table path (distinct > 4096)
    out["path"] = H.path_graph(300)
    out["complete"] = H.complete_graph(40)
    out["bipartite"] = H.complete_bipartite(30, 50)
    out["with_isolated"] = H.from_edges(40, [(i, i + 1) for i in range(0, 20)])
    # both sides of every kernel-tier boundary; parallel edges keep n below every direct-indexing size (n = 278)
    out["ladder_dense_w"] = H.degree_ladder(sorted(H.LADDER_DEGREES), 256, weighted=True, multi=True, seed=2)
    out["ladder_wide"] = H.degree_ladder(sorted(H.LADDER_DEGREES), 18436, seed=3)  # distinct neighbours
    return out


GRAPHS = None


def get_graph(name):
    global GRAPHS
    if GRAPHS is None:
        GRAPHS = graphs()
    return GRAPHS[name]


NAMES = ["rgg2d_k4", "walshaw_k16", "walshaw_unsorted", "rmat13_w", "grid12", "road60", "star30000", "rmat15_sorted",
         "rmat14_unsorted_w", "rmat16_hubs", "rmat15_hubs_w", "grid20", "rgg_2e15", "star_hub", "path", "complete",
         "bipartite", "with_isolated", "ladder_dense_w", "ladder_wide"]


# ------------------------------------------------------------------------------------------------
# T0
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_t0_cluster_selection(name):
    g = get_graph(name)
    ctx, mcw = ctx_for(g, 8, seed=3)
    h = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
    h.set_graph(g)
    rng = np.random.default_rng(1)
    # a mid-run state: labels of a previous oracle run, cluster weights consistent with them
    labels = B.oracle_lp_cluster(g, 5, mcw, schedule=B.SYNC)
    flip = rng.random(g.n) < 0.3
    labels = np.where(flip, np.arange(g.n, dtype=np.uint32), labels).astype(np.uint32)
    w = np.ones(g.n, np.int64) if g.vwgt is None else g.vwgt.astype(np.int64)
    weights = np.bincount(labels, weights=w, minlength=g.n).astype(np.int32)
    deg = g.degrees()
    for it in (0, 2):
        t_gpu, f_gpu = h.select_all(0, labels, weights, max_cluster_weight=mcw, call_index=1, iteration=it)
        t_cpu, f_cpu = B.oracle_sync_select_all(0, g, labels, weights, max_cluster_weight=mcw, seed=3, call=1,
                                                iteration=it)
        assert np.array_equal(t_gpu, t_cpu)
        assert np.array_equal(f_gpu[deg > 0], f_cpu[deg > 0])
    h.close()


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("k", [2, 16, 600])
def test_t0_refine_selection(name, k):
    g = get_graph(name)
    ctx, _ = ctx_for(g, k, seed=11)
    h = lp.LPHandle(lp._refine_config(ctx.refinement.lp, ctx.engine))
    h.set_graph(g)
    rng = np.random.default_rng(k)
    labels = rng.integers(0, k, g.n).astype(np.uint32)
    weights = H.block_weights(g, labels, k).astype(np.int32)
    mbw = ctx.partition.max_block_weights().copy()
    mbw[rng.integers(0, k)] = max(1, int(mbw[0] * 0.9))  # one overloaded block exercises the overload rule
    minw = np.zeros(k, np.int32)
    minw[rng.integers(0, k)] = int(weights.max())  # one block may not shrink (lp_refiner.cc:160-162)
    for mn in (None, minw):
        t_gpu, _ = h.select_all(1, labels, weights, max_weights=mbw, min_weights=mn, iteration=1)
        t_cpu, _ = B.oracle_sync_select_all(1, g, labels, weights, max_weights=mbw, min_weights=mn, seed=11,
                                            iteration=1)
        assert np.array_equal(t_gpu, t_cpu)
    h.close()


# ------------------------------------------------------------------------------------------------
# T1
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("seed", [0, 5])
def test_t1_clustering_matches_oracle_sync(name, seed):
    g = get_graph(name)
    ctx, mcw = ctx_for(g, 8, seed=seed)
    clusterer = lp.LPClustering(ctx.coarsening, ctx.engine)
    clusterer.set_max_cluster_weight(mcw)
    c = clusterer.compute_clustering(g)
    expect, st = B.oracle_lp_cluster(g, seed, mcw, schedule=B.SYNC, return_stats=True)
    assert np.array_equal(c, expect)
    gs = clusterer.last_stats
    assert gs.moved_list() == list(st[0].moved[: st[0].iterations])
    assert gs.edges_scanned == st[0].edges_scanned and gs.nodes_visited == st[0].nodes_visited
    assert gs.num_clusters == st[0].num_clusters and gs.two_hop_ran == st[0].two_hop_ran
    assert (c < max(g.n, 1)).all() and H.cluster_weights_ok(g, c, mcw)
    # second call on the same object: different clustering (overlay coarsener), still oracle-exact
    c2 = clusterer.compute_clustering(g)
    expect2 = B.oracle_lp_cluster(g, seed, mcw, schedule=B.SYNC, num_calls=2)[1]
    assert np.array_equal(c2, expect2)


@pytest.mark.parametrize("name", ["rmat15_sorted", "star_hub", "rmat14_unsorted_w", "rmat16_hubs", "rmat15_hubs_w"])
@pytest.mark.parametrize("knobs", [("8", "200", "6000"), ("64", "0", "40000"), ("3072", "0", "20000")])
def test_t1_hub_bucket_layout_does_not_change_results(name, knobs, monkeypatch):
    """Bucket capacity, the claim limit of the select map and the wave budget of the hub tier are performance
    knobs (read once per handle). Tiny buckets push almost every entry through the overflow list and a tiny claim
    limit forces the multi-pass (hash class) selection; one-hub waves reuse the bucket memory: all of them must
    give the oracle's clustering and refinement."""
    monkeypatch.setenv("KMP_HUB_BUCKET_CAP", knobs[0])
    monkeypatch.setenv("KMP_HUB_SEL_LIMIT", knobs[1])
    monkeypatch.setenv("KMP_HUB_WAVE_SLOTS", knobs[2])
    g = get_graph(name)
    ctx, mcw = ctx_for(g, 8, seed=3)
    clusterer = lp.LPClustering(ctx.coarsening, ctx.engine)
    clusterer.set_max_cluster_weight(mcw)
    c = clusterer.compute_clustering(g)
    assert np.array_equal(c, B.oracle_lp_cluster(g, 3, mcw, schedule=B.SYNC))
    k = 8
    part = np.random.default_rng(5).integers(0, k, g.n).astype(np.uint32)
    p_graph = lp.PartitionedGraph(g, k, part)
    refiner = lp.LabelPropagationRefiner(ctx)
    refiner.initialize(p_graph)
    refiner.refine(p_graph, ctx.partition)
    rp = B.oracle_params(B.default_refine_params(), commit_passes=4)
    ep, ebw = B.oracle_lp_refine(g, 3, k, ctx.partition.max_block_weights(), part, schedule=B.SYNC, params=rp)
    assert np.array_equal(p_graph.partition, ep) and np.array_equal(p_graph.block_weights(), ebw)


@pytest.mark.parametrize("mode", ["push", "pull"])
@pytest.mark.parametrize("name", ["rmat16_hubs", "rmat15_hubs_w", "grid20", "walshaw_k16", "star_hub"])
def test_t1_activation_mode_does_not_change_results(name, mode, monkeypatch):
    """Pull activation (move stamps read with the neighbour labels) and push activation (movers flag their
    neighbours, label_propagation.h:848-870) are two implementations of the same active set."""
    monkeypatch.setenv("KMP_ACTIVATION", mode)
    g = get_graph(name)
    ctx, mcw = ctx_for(g, 8, seed=6)
    clusterer = lp.LPClustering(ctx.coarsening, ctx.engine)
    clusterer.set_max_cluster_weight(mcw)
    c = clusterer.compute_clustering(g)
    expect, st = B.oracle_lp_cluster(g, 6, mcw, schedule=B.SYNC, return_stats=True)
    assert np.array_equal(c, expect)
    gs = clusterer.last_stats
    assert gs.edges_scanned == st[0].edges_scanned and gs.nodes_visited == st[0].nodes_visited
    assert (gs.pull_rounds == 0) if mode == "push" else (gs.pull_rounds == gs.iterations)
    k = 8
    part = np.random.default_rng(3).integers(0, k, g.n).astype(np.uint32)
    p_graph = lp.PartitionedGraph(g, k, part)
    refiner = lp.LabelPropagationRefiner(ctx)
    refiner.initialize(p_graph)
    refiner.refine(p_graph, ctx.partition)
    rp = B.oracle_params(B.default_refine_params(), commit_passes=4)
    ep, ebw = B.oracle_lp_refine(g, 6, k, ctx.partition.max_block_weights(), part, schedule=B.SYNC, params=rp)
    assert np.array_equal(p_graph.partition, ep) and np.array_equal(p_graph.block_weights(), ebw)


@pytest.mark.parametrize("knob", ["timing", "KMP_FORCE_P64=1"])
@pytest.mark.parametrize("name", ["rmat16_hubs", "rmat15_hubs_w", "road60"])
def test_t1_launch_structure_knobs_do_not_change_results(name, knob, monkeypatch):
    """The side-stream overlap of the tiers of a sub-round (timing mode launches them serially, one event pair
    each) and the width of the packed (label, stamp) gather word (8 bytes once n > 2^24, e.g. the 512^3 grid;
    forced here) are implementation choices only."""
    timing = knob == "timing"
    if not timing:
        monkeypatch.setenv(*knob.split("="))
    g = get_graph(name)
    ctx, mcw = ctx_for(g, 8, seed=4)
    clusterer = lp.LPClustering(ctx.coarsening, ctx.engine)
    clusterer._handle.set_timing(timing)
    clusterer.set_max_cluster_weight(mcw)
    c = clusterer.compute_clustering(g)
    assert np.array_equal(c, B.oracle_lp_cluster(g, 4, mcw, schedule=B.SYNC))
    k = 8
    part = np.random.default_rng(9).integers(0, k, g.n).astype(np.uint32)
    p_graph = lp.PartitionedGraph(g, k, part)
    refiner = lp.LabelPropagationRefiner(ctx)
    refiner._handle.set_timing(timing)
    refiner.initialize(p_graph)
    refiner.refine(p_graph, ctx.partition)
    rp = B.oracle_params(B.default_refine_params(), commit_passes=4)
    ep, ebw = B.oracle_lp_refine(g, 4, k, ctx.partition.max_block_weights(), part, schedule=B.SYNC, params=rp)
    assert np.array_equal(p_graph.partition, ep) and np.array_equal(p_graph.block_weights(), ebw)


@pytest.mark.parametrize("name", ["rmat16_hubs", "grid20", "rgg_2e15"])
def test_t1_long_refinement_switches_to_push_activation(name):
    """Twelve rounds: once few vertices move the engine switches from pull to push activation on its own
    (kmp_lp.cu choose_activation); results stay the oracle's, round by round."""
    g = get_graph(name)
    k = 16
    ctx, _ = ctx_for(g, k, seed=8)
    ctx.refinement.lp.num_iterations = 12
    part = np.random.default_rng(5).integers(0, k, g.n).astype(np.uint32)
    p_graph = lp.PartitionedGraph(g, k, part)
    refiner = lp.LabelPropagationRefiner(ctx)
    refiner.initialize(p_graph)
    refiner.refine(p_graph, ctx.partition)
    base = B.default_refine_params()
    base.num_iterations = 12
    rp = B.oracle_params(base, commit_passes=4)
    ep, ebw, st = B.oracle_lp_refine(g, 8, k, ctx.partition.max_block_weights(), part, schedule=B.SYNC, params=rp,
                                     return_stats=True)
    assert np.array_equal(p_graph.partition, ep) and np.array_equal(p_graph.block_weights(), ebw)
    gs = refiner.last_stats
    assert gs.moved_list() == list(st.moved[: st.iterations]) and gs.edges_scanned == st.edges_scanned
    assert gs.pull_rounds >= 2 and gs.pull_rounds + gs.push_rounds >= gs.iterations


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("k", [2, 4, 64])
def test_t1_refinement_matches_oracle_sync(name, k):
    g = get_graph(name)
    ctx, _ = ctx_for(g, k, seed=2)
    rng = np.random.default_rng(7)
    part = rng.integers(0, k, g.n).astype(np.uint32)
    p_graph = lp.PartitionedGraph(g, k, part)
    refiner = lp.LabelPropagationRefiner(ctx)
    refiner.initialize(p_graph)
    assert refiner.refine(p_graph, ctx.partition) is True
    rp = B.oracle_params(B.default_refine_params(), commit_passes=4)
    ep, ebw, st = B.oracle_lp_refine(g, 2, k, ctx.partition.max_block_weights(), part, schedule=B.SYNC, params=rp,
                                     return_stats=True)
    assert np.array_equal(p_graph.partition, ep)
    assert np.array_equal(p_graph.block_weights(), ebw)
    assert refiner.last_stats.moved_list() == list(st.moved[: st.iterations])
    assert refiner.last_stats.edges_scanned == st.edges_scanned
    assert np.array_equal(H.block_weights(g, p_graph.partition, k), ebw)


def test_t1_refinement_min_block_weights_and_unbalanced_start():
    g = get_graph("walshaw_k16")
    k = 8
    ctx, _ = ctx_for(g, k, seed=4)
    part = (np.arange(g.n) * k // g.n).astype(np.uint32)
    bw0 = H.block_weights(g, part, k)
    ctx.partition.setup_min_block_weights([int(0.97 * w) for w in bw0])
    p_graph = lp.PartitionedGraph(g, k, part)
    refiner = lp.LabelPropagationRefiner(ctx)
    refiner.initialize(p_graph)
    refiner.refine(p_graph, ctx.partition)
    rp = B.oracle_params(B.default_refine_params(), commit_passes=4)
    ep, ebw = B.oracle_lp_refine(g, 4, k, ctx.partition.max_block_weights(), part, schedule=B.SYNC, params=rp,
                                 min_block_weights=ctx.partition.min_block_weights())
    assert np.array_equal(p_graph.partition, ep) and np.array_equal(p_graph.block_weights(), ebw)
    assert (ebw >= ctx.partition.min_block_weights()).all()
    # a move never pushes a block above its maximum (blocks that start overloaded may only shrink)
    assert (ebw <= np.maximum(ctx.partition.max_block_weights(), bw0)).all()


def test_t1_communities_and_limits():
    g = get_graph("rmat13_w")
    ctx, mcw = ctx_for(g, 8, seed=9)
    comm = (np.arange(g.n) % 3).astype(np.uint32)
    ctx.coarsening.clustering.lp.max_num_neighbors = 6
    ctx.coarsening.clustering.lp.large_degree_threshold = 300
    clusterer = lp.LPClustering(ctx.coarsening, ctx.engine)
    clusterer.set_max_cluster_weight(mcw)
    clusterer.set_communities(comm)
    c = clusterer.compute_clustering(g)
    cp = B.default_cluster_params()
    cp.max_num_neighbors, cp.large_degree_threshold = 6, 300
    expect = B.oracle_lp_cluster(g, 9, mcw, schedule=B.SYNC, params=cp, communities=comm)
    assert np.array_equal(c, expect)


def test_t1_free_memory_afterwards_and_regraph():
    g1, g2 = get_graph("grid12"), get_graph("road60")
    ctx, mcw = ctx_for(g1, 4)
    clusterer = lp.LPClustering(ctx.coarsening, ctx.engine)
    clusterer.set_max_cluster_weight(mcw)
    a = clusterer.compute_clustering(g1, free_memory_afterwards=True)
    b = clusterer.compute_clustering(g2)
    c = clusterer.compute_clustering(g1)
    # one handle: the second and third clustering run with call indices 1 and 2
    assert np.array_equal(a, B.oracle_lp_cluster(g1, 0, mcw, schedule=B.SYNC))
    assert np.array_equal(b, B.oracle_lp_cluster(g2, 0, mcw, schedule=B.SYNC, call_index=1))
    assert np.array_equal(c, B.oracle_lp_cluster(g1, 0, mcw, schedule=B.SYNC, call_index=2))


def test_empty_graph_and_isolated_only():
    ctx = lp.create_default_context()
    clusterer = lp.LPClustering(ctx.coarsening)
    clusterer.set_max_cluster_weight(10)
    assert len(clusterer.compute_clustering(H.empty_graph(0))) == 0
    g = H.empty_graph(7)
    c = clusterer.compute_clustering(g)
    assert np.array_equal(c, B.oracle_lp_cluster(g, 0, 10, schedule=B.SYNC))


# ------------------------------------------------------------------------------------------------
# T3: against the reference's own (sequential) outputs stored in the golden files
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["rgg2d_k4", "walshaw_k16", "rmat14", "grid12", "road60"])
def test_t3_quality_next_to_reference(name):
    g, d = H.load_case(name)
    k = int(d["k"][0])
    mcw = int(d["max_cluster_weight"][0])
    ctx, mcw2 = ctx_for(g, k)
    assert mcw == mcw2
    clusterer = lp.LPClustering(ctx.coarsening, ctx.engine)
    clusterer.set_max_cluster_weight(mcw)
    c = clusterer.compute_clustering(g)
    ref_c = d["clustering_s0"]
    assert H.cluster_weights_ok(g, c, mcw)
    n_gpu, n_ref = len(np.unique(c)), len(np.unique(ref_c))
    assert n_gpu <= 1.6 * n_ref + 8  # same order of shrinkage as the reference
    part = d["part_in_s0"]
    p_graph = lp.PartitionedGraph(g, k, part)
    refiner = lp.LabelPropagationRefiner(ctx)
    refiner.initialize(p_graph)
    refiner.refine(p_graph, ctx.partition)
    cut_gpu = B.oracle_edge_cut(g, p_graph.partition)
    cut_ref = int(d["cut_s0"][0])
    cut_in = B.oracle_edge_cut(g, part)
    feasible_gpu = (p_graph.block_weights() <= d["max_block_weights"]).all()
    feasible_ref = (d["bw_out_s0"] <= d["max_block_weights"]).all()
    assert feasible_gpu == feasible_ref or feasible_gpu
    assert cut_gpu < cut_in
    assert cut_gpu <= 1.25 * cut_ref + 16


# ------------------------------------------------------------------------------------------------
# k = 256 (BASELINE config 5), weighted coarse level, device-side metrics
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["rmat16_hubs", "rmat15_hubs_w", "grid20", "road60", "rgg_2e15"])
def test_t1_refinement_k256_and_device_edge_cut(name):
    """k = 256 blocks (block-weight arrays privatised in shared memory, tables direct-indexed); afterwards
    kmp_lp_edge_cut on the device == metrics::edge_cut (metrics.cc:36-53) of the same labels."""
    g = get_graph(name)
    k = 256
    if k > g.n // 4:
        pytest.skip("k too large for this graph")
    ctx, _ = ctx_for(g, k, seed=12)
    part = np.random.default_rng(12).integers(0, k, g.n).astype(np.uint32)
    p_graph = lp.PartitionedGraph(g, k, part)
    refiner = lp.LabelPropagationRefiner(ctx)
    refiner.initialize(p_graph)
    refiner.refine(p_graph, ctx.partition)
    rp = B.oracle_params(B.default_refine_params(), commit_passes=4)
    ep, ebw = B.oracle_lp_refine(g, 12, k, ctx.partition.max_block_weights(), part, schedule=B.SYNC, params=rp)
    assert np.array_equal(p_graph.partition, ep) and np.array_equal(p_graph.block_weights(), ebw)
    assert refiner._handle.edge_cut() == B.oracle_edge_cut(g, ep)
    assert B.oracle_edge_cut(g, ep) < B.oracle_edge_cut(g, part)


@pytest.mark.parametrize("name", ["rmat16_hubs", "walshaw_k16", "star_hub"])
def test_device_edge_cut_of_a_clustering(name):
    g = get_graph(name)
    ctx, mcw = ctx_for(g, 8, seed=1)
    clusterer = lp.LPClustering(ctx.coarsening, ctx.engine)
    clusterer.set_max_cluster_weight(mcw)
    c = clusterer.compute_clustering(g)
    assert clusterer._handle.edge_cut() == B.oracle_edge_cut(g, c)


@pytest.mark.parametrize("ths,iso", [(4, 3), (4, 4), (2, 2), (4, 2), (2, 1)])
@pytest.mark.parametrize("name", ["star30000", "star_hub", "road60", "with_isolated", "rmat13_w"])
def test_t1_cluster_post_pass_variants(name, ths, iso):
    """CLUSTER_THREADWISE two-hop and the CLUSTER isolated-node variants (next-fit packing in id order, the reference's
    one-thread outcome: label_propagation.h:884-917, :977-1002) == oracle sync, weights never exceed the limit."""
    g = get_graph(name)
    ctx, mcw = ctx_for(g, 8, seed=13)
    ctx.coarsening.clustering.lp.two_hop_strategy = ths
    ctx.coarsening.clustering.lp.isolated_nodes_strategy = iso
    clusterer = lp.LPClustering(ctx.coarsening, ctx.engine)
    clusterer.set_max_cluster_weight(mcw)
    c = clusterer.compute_clustering(g)
    cp = B.default_cluster_params()
    cp.two_hop_strategy, cp.isolated_nodes_strategy = ths, iso
    expect, st = B.oracle_lp_cluster(g, 13, mcw, schedule=B.SYNC, params=cp, return_stats=True)
    assert np.array_equal(c, expect)
    assert clusterer.last_stats.two_hop_ran == st[0].two_hop_ran
    assert H.cluster_weights_ok(g, c, mcw)
