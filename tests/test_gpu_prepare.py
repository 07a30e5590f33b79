"""-m gpu: the input preparation on the device (kmp_prepare.cuh, DESIGN.md §15) equals the NumPy oracle
(tests/prepare_oracle.py, pinned against the unmodified reference by tests/test_prepare_oracle.py) bit for bit.

P0  the rearrangement on the oracle's CPU inputs, from host and from device arrays
P1  sizes where the tiles matter: R-MAT 20 with weights, rgg 2^20, a star whose hub spans many edge tiles; an adjncy
    view off 16-byte alignment
P2  malformed input is refused with KMP_ERR_INVALID and the handle works afterwards
P3  finish: output vector and block weights, from a host partition and from the handle's device labels; the device
    labels are refused once the handle holds another graph
P4  the facade's first step from the raw graph: prepare -> kmp_lp_set_graph_prepared -> seq_strict cluster and
    refine == the reference goldens (computed on the reference's own rearrangement)
P5  both ends of a device-resident V-cycle: prepare -> sync cluster -> contract -> LP on the coarse graph -> project
    up -> overload balance -> LP refine -> underload balance -> finish, every step against the oracles
"""
import numpy as np
import pytest
import torch

from kaminpar_b200 import contraction as KC
from kaminpar_b200 import lp
from kaminpar_b200 import prepare as PR
from kaminpar_b200.graph import CSRGraph, random_weights, rgg2d, rmat
from oracle import bindings as B
from oracle import contraction_oracle as CO
from tests import balance_oracle as O
from tests import helpers as H
from tests import prepare_oracle as P
from tests import underload_oracle as U
from tests.test_prepare_oracle import GOLDEN_INPUTS, live_inputs, raw_cases, sorted_golden_cases, star

pytestmark = pytest.mark.gpu

REFINE_PARAMS = B.oracle_params(B.default_refine_params(), commit_passes=4)


def _handle(seed=0, refine=False, schedule="sync"):
    ctx = lp.create_default_context()
    ctx.engine.seed = seed
    ctx.engine.schedule = schedule
    cfg = (lp._refine_config(ctx.refinement.lp, ctx.engine) if refine else
           lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
    return lp.LPHandle(cfg)


def assert_prepared(pg: PR.PreparedGraph, g: CSRGraph):
    exp = P.rearrange(g.xadj, g.adjncy, g.vwgt, g.adjwgt)
    assert pg.n == exp["n_prime"] and pg.num_isolated == exp["num_isolated"] and pg.m == g.m
    assert pg.stats.n_nonisolated == exp["n_prime"] and pg.stats.num_isolated == exp["num_isolated"]
    xadj, adj, vw, ew, o2n = pg._download()
    assert np.array_equal(xadj, exp["xadj"]), "xadj"
    assert np.array_equal(adj, exp["adjncy"]), "adjncy"
    assert np.array_equal(o2n, exp["old_to_new"]), "old_to_new"
    for got, want in ((vw, exp["vwgt"]), (ew, exp["adjwgt"])):
        assert (got is None) == (want is None)
        if want is not None:
            assert np.array_equal(got, want)
    gl = pg.get()
    assert gl.sorted and gl.n == exp["n_prime"]
    return exp


def _device_csr(g: CSRGraph, misalign=False):
    """torch copies of g on cuda:0; misalign: adjncy is a view 4 bytes past a 16-byte boundary."""
    t = lambda a: torch.from_numpy(a.view(np.int32).copy()).cuda()
    adj = t(g.adjncy)
    if misalign:
        buf = torch.zeros(g.m + 1, dtype=torch.int32, device="cuda")
        buf[1:] = adj
        adj = buf[1:]
        assert adj.data_ptr() % 16 != 0
    return dict(xadj=t(g.xadj), adjncy=adj, vwgt=None if g.vwgt is None else t(g.vwgt),
                adjwgt=None if g.adjwgt is None else t(g.adjwgt))


def _prepare_device(h, g, misalign=False):
    d = _device_csr(g, misalign)
    torch.cuda.synchronize()  # the copies ran on torch's stream, the preparation runs on the handle's
    ptr = lambda x: 0 if x is None else x.data_ptr()
    pg = PR.rearrange_by_degree_buckets_device(h, g.n, g.m, ptr(d["xadj"]), ptr(d["adjncy"]), ptr(d["vwgt"]),
                                               ptr(d["adjwgt"]))
    return pg, d


# ---- P0 ------------------------------------------------------------------------------------------------------
P0_INPUTS = list(live_inputs()) + list(raw_cases())


@pytest.mark.parametrize("name,g", P0_INPUTS, ids=[n for n, _ in P0_INPUTS])
def test_p0_equals_oracle(name, g):
    h = _handle()
    pg = PR.rearrange_by_degree_buckets(h, g)
    assert_prepared(pg, g)
    pg.close()
    pg, _ = _prepare_device(h, g)
    assert_prepared(pg, g)
    pg.close()
    h.close()


# ---- P1 ------------------------------------------------------------------------------------------------------
def _p1_graphs():
    yield "rmat20_w", lambda: random_weights(rmat(20, 16, seed=5), 3, max_vwgt=7, max_adjwgt=9)
    yield "rgg2^20", lambda: rgg2d(1 << 20, seed=2)
    yield "star2^20", lambda: star(1 << 20)  # the hub's 2^20 - 1 edges span 512 edge tiles


@pytest.mark.parametrize("name,make", list(_p1_graphs()), ids=[n for n, _ in _p1_graphs()])
def test_p1_large_inputs(name, make):
    g = make()
    h = _handle()
    pg = PR.rearrange_by_degree_buckets(h, g)
    exp = assert_prepared(pg, g)
    pg.close()
    pg, _ = _prepare_device(h, g, misalign=True)
    assert_prepared(pg, g)
    assert pg.stats.device_ms > 0 and exp["n_prime"] == pg.n
    pg.close()
    h.close()


# ---- P2 ------------------------------------------------------------------------------------------------------
def test_p2_malformed_input_is_refused_and_the_handle_stays_usable():
    g = H.load_graph("walshaw_data")
    h = _handle()
    bad = []
    x = g.xadj.copy()
    x[0] = 1
    bad.append(("xadj[0] != 0", CSRGraph(x, g.adjncy)))
    x = g.xadj.copy()
    x[100] = x[101] + 1
    bad.append(("decreasing xadj", CSRGraph(x, g.adjncy)))
    x = g.xadj.copy()
    x[-1] -= 1
    bad.append(("xadj[n] != m", CSRGraph(x, g.adjncy)))
    a = g.adjncy.copy()
    a[g.m // 2] = g.n
    bad.append(("target >= n", CSRGraph(g.xadj, a)))
    a = g.adjncy.copy()
    a[-1] = 0xFFFFFFFF
    bad.append(("target 2^32 - 1", CSRGraph(g.xadj, a)))
    bad.append(("n = 0, m = 1", CSRGraph(np.zeros(1, np.uint32), np.zeros(1, np.uint32))))
    for what, b in bad:
        with pytest.raises(RuntimeError, match="error -1"):
            PR.rearrange_by_degree_buckets(h, b)
        with pytest.raises(RuntimeError, match="error -1"):
            _prepare_device(h, b)
        pg = PR.rearrange_by_degree_buckets(h, g)  # the handle works afterwards
        assert_prepared(pg, g)
        pg.close()
    assert h._children == 0


# ---- P3 ------------------------------------------------------------------------------------------------------
def _with_isolated(g, extra, seed, heavy=False):
    from tests.test_prepare_oracle import _with_isolated as wi

    return wi(g, extra, seed, (lambda r, c: r.integers(10, 60, c)) if heavy else None)


P3_CASES = [
    ("walshaw+3000", lambda: _with_isolated(H.load_graph("walshaw_data"), 3000, 2), 8),
    ("rmat14w+isolated", lambda: random_weights(rmat(14, 4, seed=3), 5, max_vwgt=6), 64),
    ("path+heavy", lambda: _with_isolated(H.path_graph(60), 50, 4, heavy=True), 8),
    ("all_isolated", lambda: H.empty_graph(1000), 7),
    ("no_isolated_k1", lambda: H.load_graph("rgg2d"), 1),
]


@pytest.mark.parametrize("name,make,k", P3_CASES, ids=[c[0] for c in P3_CASES])
def test_p3_finish_equals_oracle(name, make, k):
    g = make()
    h = _handle(refine=True)
    pg = PR.rearrange_by_degree_buckets(h, g)
    exp = assert_prepared(pg, g)
    p_ctx = lp.PartitionContext().setup(g, k, 0.03)  # on the raw graph
    rng = np.random.default_rng(k)
    part = rng.integers(0, k, pg.n).astype(np.uint32)
    want, want_bw = P.finish(exp, k, p_ctx.max_block_weights(), part)
    got, bw = pg.finish(h, k, p_ctx, part)
    assert np.array_equal(got, want) and np.array_equal(bw, want_bw)
    if pg.n > 0:
        pg.set_on(h)
        h.upload_partition(part)
        got, bw = pg.finish(h, k, p_ctx)  # the handle's device labels
        assert np.array_equal(got, want) and np.array_equal(bw, want_bw)
    if pg.n > 0:
        with pytest.raises(RuntimeError, match="error -1"):  # a label >= k
            pg.finish(h, k, p_ctx, np.full(pg.n, k, np.uint32))
    h.set_graph(H.load_graph("rgg16"))  # the handle moves on: its labels are not this graph's
    h.upload_partition(np.zeros(16, np.uint32))
    with pytest.raises(RuntimeError, match="error -1"):
        pg.finish(h, k, p_ctx)
    got, _ = pg.finish(h, k, p_ctx, part)  # a host partition still works
    assert np.array_equal(got, want)
    pg.close()
    h.close()


# ---- P4 ------------------------------------------------------------------------------------------------------
def _strict_ctx(d, seed):
    from tests.test_gpu_strict import _ctx

    return _ctx(d, seed)


@pytest.mark.parametrize("case", sorted_golden_cases())
def test_p4_seq_strict_from_the_raw_graph_equals_the_reference(case):
    g0 = GOLDEN_INPUTS[case]()
    _, d = H.load_case(case)
    k = int(d["k"][0])
    mcw = int(d["max_cluster_weight"][0])
    num_calls = int(d["num_calls"][0])
    for seed in d["seeds"]:
        seed = int(seed)
        ctx = _strict_ctx(d, seed)
        hc = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
        pg = PR.rearrange_by_degree_buckets(hc, g0)
        assert np.array_equal(pg.old_to_new(), d["old_to_new"])
        pg.set_on(hc)
        exp = d[f"clustering_s{seed}"]
        for call in range(num_calls):
            c, _ = hc.cluster(mcw)
            assert np.array_equal(c, exp if num_calls == 1 else exp[call]), f"clustering (seed {seed}, call {call})"
        hr = lp.LPHandle(lp._refine_config(ctx.refinement.lp, ctx.engine))
        pg.set_on(hr)
        part = np.ascontiguousarray(d[f"part_in_s{seed}"], np.uint32).copy()
        p, bw, _ = hr.refine(k, d["max_block_weights"], part)
        assert np.array_equal(p, d[f"part_out_s{seed}"]) and np.array_equal(bw, d[f"bw_out_s{seed}"])
        hr.close()
        pg.close()
        hc.close()


# ---- P5 ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [4, 64])
def test_p5_device_resident_v_cycle(k):
    seed = 1
    g0 = _with_isolated(random_weights(rmat(14, 8, seed=21), 6, max_vwgt=4, max_adjwgt=5), 900, 7)
    ctx = lp.create_default_context()
    ctx.engine.seed = seed
    p_ctx = ctx.partition.setup(g0, k, 0.03)  # on the raw graph, isolated vertices included
    hc = _handle(seed)
    hr = _handle(seed, refine=True)
    pg = PR.rearrange_by_degree_buckets(hc, g0)
    exp = assert_prepared(pg, g0)
    g = CSRGraph(exp["xadj"][: pg.n + 1], exp["adjncy"], exp["vwgt"][: pg.n], exp["adjwgt"], sorted=True)
    # ---- coarsening: the prepared graph, one level down, all on the device ----
    pg.set_on(hc)
    mcw = lp.compute_max_cluster_weight(ctx.coarsening, p_ctx, g.n, g.total_node_weight())
    hc.cluster(mcw, fetch=False)
    want = B.oracle_lp_cluster(g, seed, mcw, schedule=B.SYNC, call_index=0)
    assert np.array_equal(hc.download_labels(), want), "clustering"
    cg = KC.contract_on_handle(hc, None)
    con = CO.contract(g.xadj, g.adjncy, g.vwgt, g.adjwgt, want)
    c = cg.get()
    assert CO.equal(dict(c_n=cg.n, c_xadj=c.xadj, c_adjncy=c.adjncy, c_vwgt=c.vwgt, c_adjwgt=c.adjwgt,
                         mapping=cg.mapping()), con), "contraction"
    gc = CSRGraph(con["c_xadj"], con["c_adjncy"], con["c_vwgt"], con["c_adjwgt"])
    mbw, pbw = p_ctx.max_block_weights(), p_ctx.perfectly_balanced_block_weights()
    mnw = U.min_block_weights(pbw, 0.1)
    d_xadj, d_adj, d_vw, d_ew, _ = cg.device_arrays()
    hr.set_graph_device(cg.n, cg.m, d_xadj, d_adj, d_vw, d_ew)
    part = (np.arange(gc.n, dtype=np.int64) * k // max(gc.n, 1)).astype(np.uint32)
    cpart, cbw, _ = hr.refine(k, mbw, part.copy())  # refined in place
    ep, ebw = B.oracle_lp_refine(gc, seed, k, mbw, part, schedule=B.SYNC, params=REFINE_PARAMS)
    assert np.array_equal(cpart, ep) and np.array_equal(cbw, ebw), "coarse LP"
    # ---- uncoarsening on the prepared graph ----
    up = cg.project_up(cpart)
    assert np.array_equal(up, CO.project_up(cg.mapping(), cpart)), "project_up"
    pg.set_on(hr)
    hr.upload_partition(up)
    _, bw, _ = hr.overload_balance(k, mbw, pbw, None)
    ob = O.overload_balance(g, k, up, mbw, pbw, seed=seed, call=0)
    assert np.array_equal(bw, ob["block_weights"]), "overload balance"
    _, bw, _ = hr.refine(k, mbw, None, min_block_weights=mnw)
    # the refiner's handle never clusters: its refinements hash with call index 0 (DESIGN.md, parity across calls)
    ep, ebw = B.oracle_lp_refine(g, seed, k, mbw, ob["labels"], schedule=B.SYNC, params=REFINE_PARAMS,
                                 min_block_weights=mnw, call_index=0)
    assert np.array_equal(bw, ebw), "refinement"
    _, bw, _ = hr.underload_balance(k, mbw, mnw, None)
    ub = U.underload_balance(g, k, ep, mbw, mnw, seed=seed, call=0)
    assert np.array_equal(bw, ub["block_weights"]), "underload balance"
    # ---- finish from the device labels ----
    out, fbw = pg.finish(hr, k, p_ctx)
    want_out, want_bw = P.finish(exp, k, mbw, ub["labels"])
    assert np.array_equal(out, want_out) and np.array_equal(fbw, want_bw), "finish"
    cg.close()
    pg.close()
    hr.close()
    hc.close()
