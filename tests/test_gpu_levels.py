"""Parity across levels and calls (-m gpu): one handle reused through a sequence of graphs and through a whole
multilevel cycle, checked call by call and level by level against the CPU oracles -- bit-exact labels, block
weights, statistics, coarse graphs and balancer rounds (all integer work).

The sync schedule keys its hashes on the number of clusterings the handle computed before, on any graph (the call
index, DESIGN.md "parity across levels and calls"): level L of a hierarchy clustered on one handle runs with call
index L. A refinement uses the handle's cluster-call count too; each balancer counts its own calls that reached the
device.

L1  one clusterer across graphs of changing size, tier mix and optional inputs
L2  one refiner and one of each balancer across graphs and k; a handle that clusters and then refines
L3  a device-resident V-cycle on two handles: cluster -> contract -> sparsify -> set_graph_device on the same handle,
    then project_up -> overload balance -> LP refine -> underload balance per level
L4  the cycle again on the same handles, grow-only buffers sized by the first cycle or too small for the second
L5  labels that do not belong to the graph, or are not a k-way partition, are refused; the handle works afterwards
"""
import numpy as np
import pytest
import torch

from kaminpar_b200 import contraction as KC
from kaminpar_b200 import lp
from kaminpar_b200.graph import CSRGraph, rmat
from oracle import bindings as B
from oracle import contraction_oracle as CO
from tests import balance_oracle as O
from tests import helpers as H
from tests import sparsify_oracle as S
from tests import underload_oracle as U
from tests.test_gpu_parity import get_graph

pytestmark = pytest.mark.gpu

REFINE_PARAMS = B.oracle_params(B.default_refine_params(), commit_passes=4)


def assert_stats(gs, st):
    """Device kmp_lp_stats == oracle lpo_stats: per-round moves, scan counters, clusters, two-hop."""
    assert gs.moved_list() == list(st.moved[: st.iterations])
    assert gs.edges_scanned == st.edges_scanned and gs.nodes_visited == st.nodes_visited
    assert gs.num_clusters == st.num_clusters and gs.two_hop_ran == st.two_hop_ran


def isolated_heavy():
    """Half of the vertices isolated: the isolated-node post pass runs on every level."""
    g = rmat(13, 8, seed=17)
    pad = g.n
    xadj = np.concatenate([g.xadj, np.full(pad, g.xadj[-1], np.uint32)])
    return CSRGraph(xadj, g.adjncy)


def weighted_rmat():
    return get_graph("rmat14_unsorted_w")


# ------------------------------------------------------------------------------------------------
# L1: one clusterer across a sequence of graphs
# ------------------------------------------------------------------------------------------------
def l1_sequence():
    return [get_graph("rmat16_hubs"), get_graph("path"), weighted_rmat(), H.empty_graph(0), H.empty_graph(7),
            get_graph("star_hub"), get_graph("grid20"), get_graph("rmat16_hubs")]


def _mcw(g, i):
    # changes between calls: the limit for k = 8, halved or doubled on alternate calls
    base = max(1, B.oracle_max_cluster_weight(g, 8)) if g.n else 10
    return base * (2 if i % 3 == 1 else 1) // (2 if i % 3 == 2 else 1) or 1


def _check_cluster_call(c, gs, g, seed, mcw, i, params=None, desired=0, communities=None):
    assert len(c) == g.n
    if g.n == 0:  # no vertices: nothing to compare, but the call still counts
        return
    cp = B.oracle_params(params or B.default_cluster_params())
    want, st = B.oracle_lp_cluster(g, seed, mcw, schedule=B.SYNC, params=cp, desired=desired, communities=communities,
                                   return_stats=True, call_index=i)
    assert np.array_equal(c, want), f"call {i}"
    assert_stats(gs, st[0])


def _device_graph(g):
    """torch tensors on cuda:0 holding g (kept alive by the caller while the handle uses them)."""
    t = dict(xadj=torch.from_numpy(g.xadj.astype(np.int32)).cuda(),
             adjncy=torch.from_numpy(g.adjncy.astype(np.int32)).cuda())
    if g.vwgt is not None:
        t["vwgt"] = torch.from_numpy(g.vwgt.astype(np.int32)).cuda()
    if g.adjwgt is not None:
        t["adjwgt"] = torch.from_numpy(g.adjwgt.astype(np.int32)).cuda()
    return t


def test_l1_set_graph_device_sequence():
    seed = 3
    ctx = lp.create_default_context()
    ctx.engine.seed = seed
    h = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
    for i, g in enumerate(l1_sequence()):
        t = _device_graph(g)
        h.set_graph_device(g.n, g.m, t["xadj"].data_ptr(), t["adjncy"].data_ptr() if g.m else 0,
                           t["vwgt"].data_ptr() if "vwgt" in t else 0, t["adjwgt"].data_ptr() if "adjwgt" in t else 0)
        mcw = _mcw(g, i)
        c, gs = h.cluster(mcw)
        torch.cuda.synchronize()
        _check_cluster_call(c, gs, g, seed, mcw, i)
        del t
    h.close()


def test_l1_free_memory_on_alternate_calls():
    seed = 5
    ctx = lp.create_default_context()
    ctx.engine.seed = seed
    clusterer = lp.LPClustering(ctx.coarsening, ctx.engine)
    for i, g in enumerate(l1_sequence()):
        mcw = _mcw(g, i)
        clusterer.set_max_cluster_weight(mcw)
        c = clusterer.compute_clustering(g, free_memory_afterwards=i % 2 == 0)
        _check_cluster_call(c, clusterer.last_stats, g, seed, mcw, i)


@pytest.mark.parametrize("max_num_neighbors", [0xFFFFFFFF, 6])
def test_l1_optional_inputs_come_and_go(max_num_neighbors):
    seed = 7
    ctx = lp.create_default_context()
    ctx.engine.seed = seed
    ctx.coarsening.clustering.lp.max_num_neighbors = max_num_neighbors
    cp = B.default_cluster_params()
    cp.max_num_neighbors = max_num_neighbors
    clusterer = lp.LPClustering(ctx.coarsening, ctx.engine)
    for i, g in enumerate(l1_sequence()):
        mcw = _mcw(g, i)
        clusterer.set_max_cluster_weight(mcw)
        comm = (np.arange(g.n) * 5 // max(g.n, 1)).astype(np.uint32) if i % 2 == 0 and g.n else None
        desired = g.n // 3 if i % 3 == 0 else 0
        clusterer.set_communities(comm)
        clusterer.set_desired_cluster_count(desired)
        c = clusterer.compute_clustering(g)
        _check_cluster_call(c, clusterer.last_stats, g, seed, mcw, i, params=cp, desired=desired, communities=comm)


# ------------------------------------------------------------------------------------------------
# L2: one refiner and one of each balancer across graphs and k
# ------------------------------------------------------------------------------------------------
L2_STEPS = [  # (graph, k, min block weights, communities)
    ("walshaw_k16", 2, False, False),
    ("rmat15_hubs_w", 600, True, True),
    ("path", 4, False, False),
    ("rgg_2e15", 20000, True, False),
    ("grid20", 3, False, True),
    ("walshaw_k16", 2, True, False),
]


def test_l2_refiner_and_balancers_across_graphs_and_k():
    seed = 9
    ctx = lp.create_default_context()
    ctx.engine.seed = seed
    refiner = lp.LabelPropagationRefiner(ctx)
    over = lp.OverloadBalancer(ctx)
    under = lp.UnderloadBalancer(ctx)
    ob_calls = ub_calls = skipped = 0
    for step, (name, k, with_min, with_comm) in enumerate(L2_STEPS):
        g = get_graph(name)
        p_ctx = lp.PartitionContext().setup(g, k, 0.03)
        mbw, pbw = p_ctx.max_block_weights(), p_ctx.perfectly_balanced_block_weights()
        mnw = U.min_block_weights(pbw, 0.1) if with_min else None
        if with_min:
            p_ctx.setup_min_block_weights(mnw)
        comm = (np.arange(g.n) % 3).astype(np.uint32) if with_comm else None
        # overload balancer; the last step starts feasible (round robin on a unit-weight graph): the operator skips
        # the device and the balancer's call count stays
        last = step == len(L2_STEPS) - 1
        part = (np.arange(g.n) % k).astype(np.uint32) if last else O.overload_input(g, k, step, 0.15, (0,))
        pg = lp.PartitionedGraph(g, k, part)
        over.initialize(pg)
        over.refine(pg, p_ctx)
        assert (over.last_stats is None) == last
        if over.last_stats is None:
            skipped += 1
            want_labels = part
        else:
            want = O.overload_balance(g, k, part, mbw, pbw, seed=seed, call=ob_calls)
            ob_calls += 1
            want_labels = want["labels"]
            assert np.array_equal(pg.partition, want["labels"]), f"step {step}"
            assert np.array_equal(pg.block_weights(), want["block_weights"])
            assert over.last_stats.moved_list() == want["moved"] and over.last_stats.rounds == want["rounds"]
        # LP refiner (a handle that never clusters: call index 0 on every call)
        refiner.set_communities(comm)
        refiner.initialize(pg)
        refiner.refine(pg, p_ctx)
        ep, ebw, st = B.oracle_lp_refine(g, seed, k, mbw, want_labels, schedule=B.SYNC, params=REFINE_PARAMS,
                                         min_block_weights=mnw, communities=comm, return_stats=True)
        assert np.array_equal(pg.partition, ep), f"step {step}"
        assert np.array_equal(pg.block_weights(), ebw)
        assert refiner.last_stats.moved_list() == list(st.moved[: st.iterations])
        assert refiner.last_stats.edges_scanned == st.edges_scanned
        # underload balancer on an underloaded input; no minimum weights: no device work
        upart = U.underload_input(g, k, step, 0.3)
        ug = lp.PartitionedGraph(g, k, upart)
        under.initialize(ug)
        under.refine(ug, p_ctx)
        if under.last_stats is None:
            skipped += 1
            assert np.array_equal(ug.partition, upart)
        else:
            want = U.underload_balance(g, k, upart, mbw, mnw, seed=seed, call=ub_calls)
            ub_calls += 1
            assert np.array_equal(ug.partition, want["labels"]), f"step {step}"
            assert np.array_equal(ug.block_weights(), want["block_weights"])
            assert under.last_stats.moved_list() == want["moved"] and under.last_stats.rounds == want["rounds"]
    # the call counts are the calls that reached the device, not the operator calls
    assert skipped >= 2 and ob_calls + ub_calls + skipped == 2 * len(L2_STEPS)


def test_l2_a_handle_that_clusters_then_refines():
    """A refinement hashes with the number of clusterings the handle computed before (here 2 and then 3)."""
    seed = 4
    ctx = lp.create_default_context()
    ctx.engine.seed = seed
    ctx.engine.refine_commit_passes = 1  # kmp_lp_cluster runs single-pass commits
    h = lp.LPHandle(lp._refine_config(ctx.refinement.lp, ctx.engine))
    # the handle's configuration as oracle parameters: the refiner's LP settings, one commit pass
    params = B.oracle_params(B.default_refine_params(), commit_passes=1)
    calls = 0
    for name, k in (("walshaw_k16", 8), ("rmat15_hubs_w", 64), ("grid20", 4)):
        g = get_graph(name)
        h.set_graph(g)
        mcw = B.oracle_max_cluster_weight(g, k)
        for _ in range(2 if calls == 0 else 1):
            c, gs = h.cluster(mcw)
            want, st = B.oracle_lp_cluster(g, seed, mcw, schedule=B.SYNC, params=params, return_stats=True,
                                           call_index=calls)
            assert np.array_equal(c, want)
            assert_stats(gs, st[0])
            calls += 1
        mbw = B.oracle_max_block_weights(g, k)
        part = np.random.default_rng(k).integers(0, k, g.n).astype(np.uint32)
        got = part.copy()
        _, bw, rs = h.refine(k, mbw, got)
        ep, ebw, st = B.oracle_lp_refine(g, seed, k, mbw, part, schedule=B.SYNC, params=params, return_stats=True,
                                         call_index=calls)
        assert np.array_equal(got, ep) and np.array_equal(bw, ebw), name
        assert rs.moved_list() == list(st.moved[: st.iterations])
    h.close()


# ------------------------------------------------------------------------------------------------
# L3 / L4: device-resident V-cycles
# ------------------------------------------------------------------------------------------------
class Cycle:
    """A clusterer handle and a refiner handle, with the call counts the oracles need."""

    def __init__(self, seed):
        self.seed = seed
        self.ctx = lp.create_default_context()
        self.ctx.engine.seed = seed
        self.hc = lp.LPHandle(lp._cluster_config(self.ctx.coarsening.clustering.lp, self.ctx.engine))
        self.hr = lp.LPHandle(lp._refine_config(self.ctx.refinement.lp, self.ctx.engine))
        self.cluster_calls = self.ob_calls = self.ub_calls = 0

    def close(self):
        self.hc.close()
        self.hr.close()


def _coarse_dict(cg):
    c = cg.get()
    return dict(c_n=cg.n, c_xadj=c.xadj, c_adjncy=c.adjncy, c_vwgt=c.vwgt, c_adjwgt=c.adjwgt, mapping=cg.mapping())


def run_cycle(cy: Cycle, g0, k, sparsify, sp_seed):
    """One V-cycle of g0 on cy's handles, every step checked against the oracles."""
    ctx = cy.ctx
    ctx.partition.setup(g0, k, 0.03)
    s_ctx = KC.SparsificationClusterCoarseningContext(laziness_factor=1.0)
    # ---- coarsening: one clusterer handle, every level on the device ----
    levels = [g0]   # oracle graphs, level 0 = the input
    coarse = []     # device CoarseGraphs, coarse[L] = level L + 1
    cy.hc.set_graph(g0)
    while True:
        L = len(coarse)
        g = levels[-1]
        mcw = lp.compute_max_cluster_weight(ctx.coarsening, ctx.partition, g.n, g.total_node_weight())
        _, gs = cy.hc.cluster(mcw, fetch=False)
        want, st = B.oracle_lp_cluster(g, cy.seed, mcw, schedule=B.SYNC, return_stats=True,
                                       call_index=cy.cluster_calls)
        cy.cluster_calls += 1
        assert np.array_equal(cy.hc.download_labels(), want), f"level {L}: clustering"
        assert_stats(gs, st[0])
        cg = KC.contract_on_handle(cy.hc, None)
        coarse.append(cg)
        con = CO.contract(g.xadj, g.adjncy, g.vwgt, g.adjwgt, want)
        assert CO.equal(_coarse_dict(cg), con), f"level {L}: contraction"
        if sparsify:
            seed = sp_seed * 1000 + L
            did = KC.sparsify_level(cy.hc, cg, g.m, g.n, s_ctx, seed)
            target = S.sparsification_target(g.m, g.n, con["c_n"])
            assert did == (len(con["c_adjncy"]) > s_ctx.laziness_factor * target)
            if did:
                con = S.sparsify_contracted(con, target, seed if target >= 2 else 0)
                st_sp = cg.sparsify_stats
                assert (st_sp.threshold, st_sp.smaller, st_sp.equal, st_sp.equal_kept) == (
                    con["threshold"], con["smaller"], con["equal"], con["equal_kept"]), f"level {L}: sparsification"
                assert CO.equal(_coarse_dict(cg), con), f"level {L}: sparsification"
        levels.append(CSRGraph(con["c_xadj"], con["c_adjncy"], con["c_vwgt"], con["c_adjwgt"]))
        c_n = con["c_n"]
        if c_n <= 160 * k or c_n > 0.95 * g.n or len(coarse) == 12:
            break
        d_xadj, d_adj, d_vw, d_ew, _ = cg.device_arrays()
        cy.hc.set_graph_device(cg.n, cg.m, d_xadj, d_adj, d_vw, d_ew)
    # ---- uncoarsening: one refiner handle ----
    mbw, pbw = ctx.partition.max_block_weights(), ctx.partition.perfectly_balanced_block_weights()
    mnw = U.min_block_weights(pbw, 0.1)
    n_top = levels[-1].n
    part = (np.arange(n_top, dtype=np.int64) * k // max(n_top, 1)).astype(np.uint32)
    for L in range(len(levels) - 1, -1, -1):
        g = levels[L]
        if L < len(levels) - 1:
            cg = coarse[L]
            up = cg.project_up(part)
            assert np.array_equal(up, CO.project_up(cg.mapping(), part)), f"level {L}: project_up"
            part = up
        if L == 0:
            cy.hr.set_graph(g)
        else:
            d_xadj, d_adj, d_vw, d_ew, _ = coarse[L - 1].device_arrays()
            cy.hr.set_graph_device(g.n, g.m, d_xadj, d_adj, d_vw, d_ew)
        cy.hr.upload_partition(part)
        _, bw, ost = cy.hr.overload_balance(k, mbw, pbw, None)
        ob = O.overload_balance(g, k, part, mbw, pbw, seed=cy.seed, call=cy.ob_calls)
        cy.ob_calls += 1
        assert np.array_equal(bw, ob["block_weights"]), f"level {L}: overload balance"
        assert ost.moved_list() == ob["moved"] and ost.rounds == ob["rounds"]
        _, bw, rst = cy.hr.refine(k, mbw, None, min_block_weights=mnw)
        ep, ebw, st = B.oracle_lp_refine(g, cy.seed, k, mbw, ob["labels"], schedule=B.SYNC, params=REFINE_PARAMS,
                                         min_block_weights=mnw, return_stats=True)
        assert np.array_equal(bw, ebw), f"level {L}: refinement"
        assert rst.moved_list() == list(st.moved[: st.iterations]) and rst.edges_scanned == st.edges_scanned
        _, bw, ust = cy.hr.underload_balance(k, mbw, mnw, None)
        ub = U.underload_balance(g, k, ep, mbw, mnw, seed=cy.seed, call=cy.ub_calls)
        cy.ub_calls += 1
        part = cy.hr.download_labels()
        assert np.array_equal(part, ub["labels"]), f"level {L}: underload balance"
        assert np.array_equal(bw, ub["block_weights"])
        assert ust.moved_list() == ub["moved"] and ust.rounds == ub["rounds"]
    assert cy.hr.edge_cut() == B.oracle_edge_cut(levels[0], part)
    for cg in coarse:  # after the uncoarsening has passed every level
        cg.close()
    return len(coarse)


L3_GRAPHS = {
    "rmat16_hubs": lambda: get_graph("rmat16_hubs"),      # hub tier on level 0 only
    "rmat15_hubs_w": lambda: get_graph("rmat15_hubs_w"),  # edge weights from level 0
    "grid20": lambda: get_graph("grid20"),                # many levels, down to direct-indexed table sizes
    "isolated": isolated_heavy,                           # post passes on every level
}
L3_CASES = [(name, k, sp, seed) for name in L3_GRAPHS for k in (4, 64) for sp in (False, True)
            for seed in ((0,) if name == "rmat16_hubs" else (0, 1))]


@pytest.mark.parametrize("name,k,sparsify,seed", L3_CASES)
def test_l3_v_cycle(name, k, sparsify, seed):
    cy = Cycle(seed)
    levels = run_cycle(cy, L3_GRAPHS[name](), k, sparsify, seed)
    assert levels >= 1
    cy.close()


@pytest.mark.parametrize("order", ["large_first", "small_first"])
def test_l4_cycles_on_the_same_handles(order):
    """Large first: the second cycle finds every grow-only buffer sized by the first. Small first: every buffer
    has to grow. The call counts carry over from one cycle to the next."""
    graphs = [("rmat15_hubs_w", 64, True, 3), ("grid20", 4, False, 4)]
    if order == "small_first":
        graphs.reverse()
    cy = Cycle(2)
    for name, k, sp, sp_seed in graphs:
        run_cycle(cy, L3_GRAPHS[name](), k, sp, sp_seed)
    assert cy.cluster_calls >= 3
    cy.close()


# ------------------------------------------------------------------------------------------------
# L5: refusals
# ------------------------------------------------------------------------------------------------
def test_l5_labels_of_another_graph_are_refused():
    seed = 6
    ctx = lp.create_default_context()
    ctx.engine.seed = seed
    ctx.engine.refine_commit_passes = 1
    h = lp.LPHandle(lp._refine_config(ctx.refinement.lp, ctx.engine))
    params = B.oracle_params(B.default_refine_params(), commit_passes=1)
    ga, gb = get_graph("walshaw_k16"), get_graph("grid20")
    k = 4
    p_ctx = lp.PartitionContext().setup(gb, k, 0.03)
    mbw, pbw = p_ctx.max_block_weights(), p_ctx.perfectly_balanced_block_weights()
    mnw = U.min_block_weights(pbw, 0.1)
    h.set_graph(ga)
    h.cluster(B.oracle_max_cluster_weight(ga, k))  # labels of ga stay on the device
    calls = 1

    def refused_without_labels():
        with pytest.raises(RuntimeError, match="error -1"):
            KC.contract_on_handle(h, None)
        with pytest.raises(RuntimeError, match="error -1"):
            h.refine(k, mbw, None)
        with pytest.raises(RuntimeError, match="error -1"):
            h.overload_balance(k, mbw, pbw, None)
        with pytest.raises(RuntimeError, match="error -1"):
            h.underload_balance(k, mbw, mnw, None)
        with pytest.raises(RuntimeError, match="error -1"):
            h.edge_cut()

    h.set_graph(gb)
    refused_without_labels()
    # the next valid call equals the oracle (refusals do not count as calls)
    part = (np.arange(gb.n) * k // gb.n).astype(np.uint32)
    h.upload_partition(part)
    _, bw, _ = h.refine(k, mbw, None)
    ep, ebw = B.oracle_lp_refine(gb, seed, k, mbw, part, schedule=B.SYNC, params=params, call_index=calls)
    assert np.array_equal(h.download_labels(), ep) and np.array_equal(bw, ebw)
    assert h.edge_cut() == B.oracle_edge_cut(gb, ep)
    # releasing the scratch releases the labels
    h.free_scratch()
    refused_without_labels()
    # a clustering on the device is not a k-way partition
    mcw = B.oracle_max_cluster_weight(gb, k)
    c, _ = h.cluster(mcw)
    assert int(c.max()) >= k
    assert np.array_equal(c, B.oracle_lp_cluster(gb, seed, mcw, schedule=B.SYNC, params=params, call_index=calls))
    calls += 1
    with pytest.raises(RuntimeError, match="error -1"):
        h.refine(k, mbw, None)
    # ... but it contracts, and the device edge cut of a clustering is defined
    cg = KC.contract_on_handle(h, None)
    assert CO.equal(_coarse_dict(cg), CO.contract(gb.xadj, gb.adjncy, gb.vwgt, gb.adjwgt, c))
    cg.close()
    assert h.edge_cut() == B.oracle_edge_cut(gb, c)
    # a host partition with a block id == k
    bad = part.copy()
    bad[gb.n // 2] = k
    with pytest.raises(RuntimeError, match="error -1"):
        h.refine(k, mbw, bad.copy())
    with pytest.raises(RuntimeError, match="error -1"):
        h.refine(k, mbw, None)  # the refused partition is still on the device
    got = part.copy()
    _, bw, _ = h.refine(k, mbw, got)
    ep, ebw = B.oracle_lp_refine(gb, seed, k, mbw, part, schedule=B.SYNC, params=params, call_index=calls)
    assert np.array_equal(got, ep) and np.array_equal(bw, ebw)
    h.close()


def test_l5_seq_strict_refiner_refuses_out_of_range_blocks():
    g = H.load_case("rgg2d_k4")[0]
    ctx = lp.create_default_context()
    ctx.engine.schedule = "seq_strict"
    h = lp.LPHandle(lp._refine_config(ctx.refinement.lp, ctx.engine))
    h.set_graph(g)
    k = 4
    mbw = B.oracle_max_block_weights(g, k)
    with pytest.raises(RuntimeError, match="error -1"):
        h.refine(k, mbw, None)
    bad = (np.arange(g.n) % (k + 1)).astype(np.uint32)
    with pytest.raises(RuntimeError, match="error -1"):
        h.refine(k, mbw, bad)
    h.close()
