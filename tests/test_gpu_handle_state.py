"""-m gpu: kmp_lp_free_scratch between any two calls changes no result.

kmp_lp_free_scratch releases the handle's scratch (the LP labels and weights, the commit, hub, list-building,
graph-operation and balancer scratch) and keeps its state: the graph, the work lists and hub metadata, the call
counters of the LP calls and of both balancers, and the seq_strict engine's random stream. Each sequence below runs
twice on a fresh handle, once plainly and once with free_scratch() after every call, and every output of the two
runs must be equal; where an oracle exists, each step is also held to it. A call that would read the device labels
of the call before it gets them from the host in both runs (free_scratch clears them, and such a call is refused).
"""
import numpy as np
import pytest

from kaminpar_b200 import contraction as KC
from kaminpar_b200 import lp
from oracle import bindings as B
from oracle import contraction_oracle as CO
from tests import balance_oracle as O
from tests import helpers as H
from tests import overlay_oracle as OV
from tests import sparsify_oracle as S
from tests import underload_oracle as U
from tests.test_gpu_parity import ctx_for, get_graph
from tests.test_gpu_strict import _ctx as strict_ctx

pytestmark = pytest.mark.gpu


class Run:
    """Records the outputs of a sequence of calls; with free=True, frees the handles' scratch after each call."""

    def __init__(self, free):
        self.free = free
        self.outputs = []

    def done(self, handle, *outputs):
        self.outputs.append(outputs)
        if self.free:
            handle.free_scratch()


def both_runs(sequence):
    plain, freed = Run(False), Run(True)
    sequence(plain)
    sequence(freed)
    assert len(plain.outputs) == len(freed.outputs)
    for i, (a, b) in enumerate(zip(plain.outputs, freed.outputs)):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            if isinstance(x, dict):
                assert CO.equal(x, y), f"call {i}"
            else:
                assert np.array_equal(x, y), f"call {i}"


def coarse_dict(cg):
    c = cg.get()
    return dict(c_n=cg.n, c_xadj=c.xadj, c_adjncy=c.adjncy, c_vwgt=c.vwgt, c_adjwgt=c.adjwgt, mapping=cg.mapping())


def moves(st):
    return np.array(st.moved[: st.iterations], np.int64)


def test_sync_handle_clusters_refines_and_balances():
    """Cluster twice (call indices 0 and 1), refine, both balancers, refine again: on a graph with hubs, so the hub
    metadata is kept and the hub scratch released."""
    g = get_graph("rmat15_hubs_w")
    seed, k = 9, 8
    ctx = lp.create_default_context()
    ctx.engine.seed = seed
    ctx.engine.refine_commit_passes = 1  # kmp_lp_cluster runs single-pass commits
    params = B.oracle_params(B.default_refine_params(), commit_passes=1)
    p_ctx = lp.PartitionContext().setup(g, k, 0.03)
    mbw, pbw = p_ctx.max_block_weights(), p_ctx.perfectly_balanced_block_weights()
    mnw = U.min_block_weights(pbw, 0.1)
    mcw = B.oracle_max_cluster_weight(g, k)

    def sequence(run):
        h = lp.LPHandle(lp._refine_config(ctx.refinement.lp, ctx.engine))
        h.set_graph(g)
        for call in (0, 1):
            c, st = h.cluster(mcw)
            want, ws = B.oracle_lp_cluster(g, seed, mcw, schedule=B.SYNC, params=params, return_stats=True,
                                           call_index=call)
            assert np.array_equal(c, want), f"cluster call {call}"
            assert st.moved_list() == list(ws[0].moved[: ws[0].iterations])
            run.done(h, c, moves(st))
        part = np.random.default_rng(k).integers(0, k, g.n).astype(np.uint32)
        got = part.copy()
        _, bw, st = h.refine(k, mbw, got)
        ep, ebw, ws = B.oracle_lp_refine(g, seed, k, mbw, part, schedule=B.SYNC, params=params, return_stats=True,
                                         call_index=2)
        assert np.array_equal(got, ep) and np.array_equal(bw, ebw), "refine"
        assert st.moved_list() == list(ws.moved[: ws.iterations])
        run.done(h, got, bw, moves(st))

        part = O.overload_input(g, k, 1, 0.15, (0,))
        got = part.copy()
        improved, bw, st = h.overload_balance(k, mbw, pbw, got)
        want = O.overload_balance(g, k, part, mbw, pbw, seed=seed, call=0)
        assert np.array_equal(got, want["labels"]) and np.array_equal(bw, want["block_weights"]), "overload balance"
        assert improved == want["improved"] and st.moved_list() == want["moved"]
        run.done(h, got, bw, np.array([improved]), np.array(st.moved_list()))

        part = U.underload_input(g, k, 2, 0.3)
        got = part.copy()
        improved, bw, st = h.underload_balance(k, mbw, mnw, got)
        want = U.underload_balance(g, k, part, mbw, mnw, seed=seed, call=0)
        assert np.array_equal(got, want["labels"]) and np.array_equal(bw, want["block_weights"]), "underload balance"
        assert improved == want["improved"] and st.moved_list() == want["moved"]
        run.done(h, got, bw, np.array([improved]), np.array(st.moved_list()))

        part = got.copy()
        _, bw, st = h.refine(k, mbw, got, min_block_weights=mnw)
        ep, ebw, ws = B.oracle_lp_refine(g, seed, k, mbw, part, schedule=B.SYNC, params=params, min_block_weights=mnw,
                                         return_stats=True, call_index=2)
        assert np.array_equal(got, ep) and np.array_equal(bw, ebw), "second refine"
        run.done(h, got, bw, moves(st))
        h.close()

    both_runs(sequence)


def test_cluster_contract_sparsify():
    g = get_graph("rmat15_hubs_w")
    seed, sp_seed = 3, 11
    ctx, mcw = ctx_for(g, 8, seed=seed)

    def sequence(run):
        h = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
        h.set_graph(g)
        c, st = h.cluster(mcw)
        want = B.oracle_lp_cluster(g, seed, mcw, schedule=B.SYNC)
        assert np.array_equal(c, want), "clustering"
        run.done(h, c, moves(st))
        cg = KC.contract_on_handle(h, c)
        con = CO.contract(g.xadj, g.adjncy, g.vwgt, g.adjwgt, want)
        coarse = coarse_dict(cg)
        assert CO.equal(coarse, con), "contraction"
        run.done(h, coarse)
        target = max(2, cg.m // 2)
        cg.sparsify(h, target, sp_seed)
        sparse = coarse_dict(cg)
        assert CO.equal(sparse, S.sparsify_contracted(con, target, sp_seed)), "sparsification"
        run.done(h, sparse)
        cg.close()
        h.close()

    both_runs(sequence)


def test_cluster_overlay_twice():
    g = get_graph("rmat13_w")
    seed = 4
    ctx, mcw = ctx_for(g, 8, seed=seed)
    calls = B.oracle_lp_cluster(g, seed, mcw, schedule=B.SYNC, num_calls=4)

    def sequence(run):
        h = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
        h.set_graph(g)
        for i in range(2):  # clusterings 2i and 2i + 1: the call counter survives free_scratch
            out, st = h.cluster_overlay(1, mcw)
            assert np.array_equal(out, OV.overlay_tree(list(calls[2 * i: 2 * i + 2]))), f"overlay {i}"
            run.done(h, out, np.array([st.num_clusters]))
        h.close()

    both_runs(sequence)


@pytest.mark.parametrize("name", ["grid12", "walshaw_k16"])
def test_seq_strict_handle(name):
    """Cluster twice and refine on one seq_strict handle: the engine's random stream continues across
    free_scratch. The first clustering and a refinement on a fresh refiner handle are the reference's."""
    g, d = H.load_case(name)
    k = int(d["k"][0])
    mcw = int(d["max_cluster_weight"][0])
    seed = int(d["seeds"][0])
    ctx = strict_ctx(d, seed)
    ctx.partition.setup(g, k, 0.03)
    mbw = ctx.partition.max_block_weights()
    exp = d[f"clustering_s{seed}"]
    part_in = np.ascontiguousarray(d[f"part_in_s{seed}"], np.uint32)

    def sequence(run):
        h = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
        h.set_graph(g)
        for call in range(2):
            c, st = h.cluster(mcw)
            if call == 0:
                assert np.array_equal(c, exp if exp.ndim == 1 else exp[0]), "first clustering"
            run.done(h, c, moves(st))
        got = part_in.copy()
        _, bw, st = h.refine(k, mbw, got)
        run.done(h, got, bw, moves(st))
        h.close()
        hr = lp.LPHandle(lp._refine_config(ctx.refinement.lp, ctx.engine))
        hr.set_graph(g)
        got = part_in.copy()
        _, bw, st = hr.refine(k, mbw, got)
        assert np.array_equal(got, d[f"part_out_s{seed}"]) and np.array_equal(bw, d[f"bw_out_s{seed}"]), "refine"
        run.done(hr, got, bw, moves(st))
        hr.close()

    both_runs(sequence)
