"""-m gpu: block-induced subgraph extraction and the copy-back on the device (kmp_subgraph.cuh, DESIGN.md §16) equal
the NumPy oracle (tests/subgraph_oracle.py) bit for bit.

G0  extraction from a host and from the device partition, weighted and unweighted: k in {1, 2, 3, 64, 1000, 70000}
    (the sort above 16 key bits), R-MAT 20, rgg 2^20, a star whose hub spans 512 edge tiles with mixed blocks, an
    adjncy off 16-byte alignment, KMP_GRID_CAP = 1..3, seq_strict and sharded handles; the refusals
G1  copy-back for k' = 2k and k' = input_k (input_k in {3, 11, 37, 1000}) from host and device sub-partitions; the
    refusals leave the labels and the handle usable; refused once the handle moved to another graph
G2  a block's device_view on a second handle: LP refinement at k = 2 and LP clustering on it == the oracles on the
    host subgraph
G3  deep-style uncoarsening on one refiner handle: project up -> overload -> LP refine -> extract -> sub-partitions
    (a fixed split and the G2 LP result) -> copy-back -> overload -> LP refine at k', every step against its oracle
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from kaminpar_b200 import contraction as KC
from kaminpar_b200 import lp
from kaminpar_b200 import subgraphs as SG
from kaminpar_b200.graph import CSRGraph, random_weights, rgg2d, rmat
from oracle import bindings as B
from oracle import contraction_oracle as CO
from tests import balance_oracle as O
from tests import helpers as H
from tests import subgraph_oracle as S
from tests.test_prepare_oracle import star

pytestmark = pytest.mark.gpu

REFINE_PARAMS = B.oracle_params(B.default_refine_params(), commit_passes=4)


def _handle(seed=0, refine=True, schedule="sync"):
    ctx = lp.create_default_context()
    ctx.engine.seed = seed
    ctx.engine.schedule = schedule
    cfg = (lp._refine_config(ctx.refinement.lp, ctx.engine) if refine else
           lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
    return lp.LPHandle(cfg)


def assert_extracted(sg: SG.Subgraphs, g: CSRGraph, part, k):
    exp = S.lazy_extract_np(g.xadj, g.adjncy, g.vwgt, g.adjwgt, part, k)
    assert sg.k == k and sg.n == g.n and sg.m == int(exp["edge_off"][-1])
    assert sg.stats.m_internal == sg.m and sg.stats.m == g.m
    no, eo = sg.offsets()
    assert np.array_equal(no, exp["node_off"]) and np.array_equal(eo, exp["edge_off"])
    xadj, adj, vw, ew, mapping, bn = sg._download()
    for what, got, want in (("xadj", xadj, exp["xadj"]), ("adjncy", adj, exp["adjncy"]), ("mapping", mapping,
                            exp["mapping"]), ("block_nodes", bn, exp["block_nodes"])):
        assert np.array_equal(got, want), what
    for got, want in ((vw, exp["vwgt"]), (ew, exp["adjwgt"])):
        assert (got is None) == (want is None)
        if want is not None:
            assert np.array_equal(got, want)
    return exp


def _part(n, k, how, seed=0):
    if how == "contiguous":
        return (np.arange(n, dtype=np.int64) * k // max(n, 1)).astype(np.uint32)
    return np.random.default_rng(seed).integers(0, k, n).astype(np.uint32)


def _extract_both(h, g, part, k):
    """From a host partition, then from the same labels on the device."""
    sg = SG.extract_subgraphs(h, k, part)
    exp = assert_extracted(sg, g, part, k)
    sg.close()
    h.upload_partition(part)
    sg = SG.extract_subgraphs(h, k)
    assert_extracted(sg, g, part, k)
    assert np.array_equal(h.download_labels(), part)  # the labels are read, not changed
    sg.close()
    return exp


# ---- G0 ------------------------------------------------------------------------------------------------------
G0_SMALL = [
    ("rmat14", lambda: rmat(14, 8, seed=3)),
    ("rmat14_w", lambda: random_weights(rmat(14, 8, seed=3), 4, max_vwgt=6, max_adjwgt=9)),
    ("rgg16_vw_ew", lambda: H.load_graph("rgg16_vwgt_adjwgt")),
]


@pytest.mark.parametrize("k", [1, 2, 3, 64, 1000, 70000])
@pytest.mark.parametrize("name,make", G0_SMALL, ids=[n for n, _ in G0_SMALL])
def test_g0_equals_oracle(name, make, k):
    g = make()
    h = _handle()
    h.set_graph(g)
    _extract_both(h, g, _part(g.n, k, "random", k), k)
    if k >= 64:  # most blocks empty or one vertex: every vertex can be its block's only member
        _extract_both(h, g, _part(g.n, k, "contiguous"), k)
    h.close()


def _g0_large():
    yield "rmat20_w", lambda: random_weights(rmat(20, 16, seed=5), 3, max_vwgt=7, max_adjwgt=9), 64
    yield "rgg2^20", lambda: rgg2d(1 << 20, seed=2), 64
    yield "star2^20", lambda: star(1 << 20), 5  # the hub's 2^20 - 1 edges span 512 edge tiles


@pytest.mark.parametrize("name,make,k", list(_g0_large()), ids=[n for n, _, _ in _g0_large()])
def test_g0_large_inputs_and_misaligned_adjncy(name, make, k):
    g = make()
    h = _handle()
    h.set_graph(g)
    for how in ("contiguous", "random"):
        part = _part(g.n, k, how, 1)
        if name.startswith("star"):
            part[0] = 1  # the hub's edges: mixed blocks, in every tile
        _extract_both(h, g, part, k)
    # the same from device arrays with adjncy a view 4 bytes past a 16-byte boundary
    t = lambda a: torch.from_numpy(a.view(np.int32).copy()).cuda()
    buf = torch.zeros(g.m + 1, dtype=torch.int32, device="cuda")
    buf[1:] = t(g.adjncy)
    adj = buf[1:]
    assert adj.data_ptr() % 16 != 0
    d = [t(g.xadj), adj, None if g.vwgt is None else t(g.vwgt), None if g.adjwgt is None else t(g.adjwgt)]
    torch.cuda.synchronize()
    h.set_graph_device(g.n, g.m, *[0 if x is None else x.data_ptr() for x in d])
    part = _part(g.n, k, "random", 2)
    sg = SG.extract_subgraphs(h, k, part)
    assert_extracted(sg, g, part, k)
    assert sg.stats.device_ms > 0
    sg.close()
    h.close()


@pytest.mark.parametrize("cap", [1, 2, 3])
def test_g0_grid_cap(cap, monkeypatch):
    monkeypatch.setenv("KMP_GRID_CAP", str(cap))
    g = random_weights(rmat(13, 8, seed=6), 1, max_vwgt=3, max_adjwgt=4)
    h = _handle()
    h.set_graph(g)
    for k in (3, 1000):
        _extract_both(h, g, _part(g.n, k, "random", cap), k)
    h.close()


def test_g0_seq_strict_and_sharded_handles_extract():
    g = H.load_graph("walshaw_data")
    part = _part(g.n, 8, "random", 4)
    h = _handle(schedule="seq_strict")
    h.set_graph(g)
    _extract_both(h, g, part, 8)
    h.close()
    h = _handle()
    h.set_graph(g)
    lp._check(lp.load_library().kmp_lp_set_shard(h._h, C.c_uint32(1), C.c_uint32(3)))
    _extract_both(h, g, part, 8)  # each rank holds the whole graph: extraction is the same on every rank
    h.close()


def test_g0_refusals():
    g = H.load_graph("walshaw_data")
    h = _handle()
    with pytest.raises(RuntimeError, match="error -1"):  # no graph
        SG.extract_subgraphs(h, 4, np.zeros(4, np.uint32))
    h.set_graph(g)
    with pytest.raises(RuntimeError, match="error -1"):  # no labels on the device
        SG.extract_subgraphs(h, 4)
    with pytest.raises(RuntimeError, match="error -1"):
        SG.extract_subgraphs(h, 0, np.zeros(g.n, np.uint32))
    bad = _part(g.n, 4, "random")
    bad[g.n // 2] = 4
    h.upload_partition(_part(g.n, 4, "random"))
    with pytest.raises(RuntimeError, match="error -1"):  # a label >= k
        SG.extract_subgraphs(h, 4, bad)
    with pytest.raises(RuntimeError, match="error -1"):  # the refused partition was loaded: no valid labels remain
        SG.extract_subgraphs(h, 4)
    with pytest.raises(RuntimeError, match="error -4"):  # n + k >= 2^32
        SG.extract_subgraphs(h, 0xFFFFFFFF - g.n + 1, np.zeros(g.n, np.uint32))
    lib = lp.load_library()
    mbw = np.full(2, g.n, np.int32)
    p2 = _part(g.n, 2, "random")
    sg = SG.extract_subgraphs(h, 2, p2)
    lp._check(lib.kmp_lp_step_begin_refine(h._h, C.c_uint32(2), lp._ptr(mbw), None, None, lp._ptr(p2)))
    with pytest.raises(RuntimeError, match="error -1"):  # inside a stepping call
        SG.extract_subgraphs(h, 2, p2)
    with pytest.raises(RuntimeError, match="error -1"):  # the copy-back neither
        sg.copy_partitions(h, np.zeros(g.n, np.uint32), 4, 4)
    lp._check(lib.kmp_lp_step_finish(h._h, None, None, None))
    assert np.array_equal(h.download_labels(), p2)
    sg.close()
    _extract_both(h, g, p2, 2)  # the handle works afterwards
    assert h._children == 0
    h.close()


# ---- G1 ------------------------------------------------------------------------------------------------------
def _sub_partitions(sg, exp, k, k_prime, input_k, seed):
    k0 = S.sub_block_offsets(k, k_prime, input_k)
    counts = k0[1:] - k0[:-1]
    rng = np.random.default_rng(seed)
    sub = np.zeros(sg.n, np.uint32)
    no = exp["node_off"]
    for b in range(k):
        sub[no[b]:no[b + 1]] = rng.integers(0, counts[b], int(no[b + 1] - no[b]))
    return sub, counts


G1_CASES = [(k, 2 * k, input_k) for k, input_k in ((2, 1000), (8, 37))] + \
    [(k, input_k, input_k) for k, input_k in ((2, 3), (8, 11), (32, 37), (512, 1000), (2, 2))]


@pytest.mark.parametrize("k,k_prime,input_k", G1_CASES)
def test_g1_copy_back_equals_oracle(k, k_prime, input_k):
    g = random_weights(rmat(14, 8, seed=9), 2, max_vwgt=5)
    h = _handle()
    h.set_graph(g)
    part = _part(g.n, k, "random", k)
    sg = SG.extract_subgraphs(h, k, part)
    exp = assert_extracted(sg, g, part, k)
    sub, counts = _sub_partitions(sg, exp, k, k_prime, input_k, 3)
    want, want_bw = S.copy_back(part, exp["mapping"], exp["node_off"], sub, k, k_prime, input_k, g.vwgt)
    out, bw = sg.copy_partitions(h, sub, k_prime, input_k)
    assert np.array_equal(out, want) and np.array_equal(bw, want_bw)
    assert np.array_equal(h.download_labels(), want)
    # from device sub-partitions
    h.upload_partition(part)
    d_sub = torch.from_numpy(sub.view(np.int32).copy()).cuda()
    torch.cuda.synchronize()
    out, bw = sg.copy_partitions(h, d_sub.data_ptr(), k_prime, input_k)
    assert np.array_equal(out, want) and np.array_equal(bw, want_bw)
    # refusals leave the labels untouched
    h.upload_partition(part)
    if counts.min() > 0:
        b = int(np.argmax(np.diff(exp["node_off"].astype(np.int64)) > 0))
        bad = sub.copy()
        bad[exp["node_off"][b]] = counts[b]
        with pytest.raises(RuntimeError, match="error -1"):
            sg.copy_partitions(h, bad, k_prime, input_k)
    with pytest.raises(RuntimeError, match="error -1"):
        sg.copy_partitions(h, sub, k - 1, input_k) if k > 1 else sg.copy_partitions(h, sub, 0, input_k)
    if k > 1:
        with pytest.raises(RuntimeError, match="error -1"):  # not a multiple of k on the way to input_k
            sg.copy_partitions(h, sub, 2 * k + 1, 10 * k)
    assert np.array_equal(h.download_labels(), part)
    # the handle is usable: LP refinement at k' from the copied-back labels
    sg.copy_partitions(h, sub, k_prime, input_k, fetch=False)
    mbw = np.full(k_prime, int(g.vwgt.sum()), np.int32)
    _, bw, _ = h.refine(k_prime, mbw, None)
    ep, ebw = B.oracle_lp_refine(g, 0, k_prime, mbw, want, schedule=B.SYNC, params=REFINE_PARAMS)
    assert np.array_equal(h.download_labels(), ep) and np.array_equal(bw, ebw)
    # refused once the handle moved to another graph, even the same arrays again
    h.set_graph(g)
    with pytest.raises(RuntimeError, match="error -1"):
        sg.copy_partitions(h, sub, k_prime, input_k)
    sg.close()
    h.close()


def test_g1_non_power_of_two_k_on_the_final_k_path_is_refused():
    g = H.load_graph("walshaw_data")
    h = _handle()
    h.set_graph(g)
    part = _part(g.n, 3, "random")
    sg = SG.extract_subgraphs(h, 3, part)
    if sum(S.compute_final_k(b, 3, 10) for b in range(3)) != 10:
        with pytest.raises(RuntimeError, match="error -1"):
            sg.copy_partitions(h, np.zeros(g.n, np.uint32), 10, 10)
    sg.close()
    h.close()


# ---- G2 ------------------------------------------------------------------------------------------------------
def test_g2_device_view_on_a_second_handle():
    g = random_weights(rmat(13, 8, seed=11), 5, max_vwgt=4, max_adjwgt=6)
    h = _handle()
    h.set_graph(g)
    k = 4
    part = _part(g.n, k, "contiguous")
    sg = SG.extract_subgraphs(h, k, part)
    exp = assert_extracted(sg, g, part, k)
    for b in range(k):
        x, adj, vw, ew = S.block_of(exp, b)
        gb = CSRGraph(x.copy(), adj.copy(), vw.copy(), ew.copy())
        hb = _handle(seed=b)
        hb.set_graph_device(*sg.device_view(b))
        mbw = np.full(2, int(gb.vwgt.sum() * 0.55) + 1, np.int32)
        p0 = (np.arange(gb.n) % 2).astype(np.uint32)
        p, bw, _ = hb.refine(2, mbw, p0.copy())
        ep, ebw = B.oracle_lp_refine(gb, b, 2, mbw, p0, schedule=B.SYNC, params=REFINE_PARAMS)
        assert np.array_equal(p, ep) and np.array_equal(bw, ebw), f"refine block {b}"
        hb.close()
        hc = _handle(seed=b, refine=False)
        hc.set_graph_device(*sg.device_view(b))
        c, _ = hc.cluster(20)
        assert np.array_equal(c, B.oracle_lp_cluster(gb, b, 20, schedule=B.SYNC)), f"cluster block {b}"
        hc.close()
    sg.close()
    h.close()


# ---- G3 ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("split", ["fixed", "lp"])
def test_g3_deep_uncoarsening_with_extension(split):
    seed, k, input_k = 1, 2, 8
    g = random_weights(rmat(14, 8, seed=21), 6, max_vwgt=4, max_adjwgt=5)
    ctx = lp.create_default_context()
    ctx.engine.seed = seed
    hc = _handle(seed, refine=False)
    hr = _handle(seed)
    # one level down on the clusterer's handle
    hc.set_graph(g)
    p_ctx = ctx.partition.setup(g, k, 0.03)
    mcw = lp.compute_max_cluster_weight(ctx.coarsening, p_ctx, g.n, g.total_node_weight())
    clustering, _ = hc.cluster(mcw)
    assert np.array_equal(clustering, B.oracle_lp_cluster(g, seed, mcw, schedule=B.SYNC)), "clustering"
    cg = KC.contract_on_handle(hc, None)
    con = CO.contract(g.xadj, g.adjncy, g.vwgt, g.adjwgt, clustering)
    cpart = (np.arange(cg.n, dtype=np.int64) * k // max(cg.n, 1)).astype(np.uint32)
    # uncoarsening at k on the refiner's handle
    up = cg.project_up(cpart)
    assert np.array_equal(up, CO.project_up(con["mapping"], cpart)), "project_up"
    hr.set_graph(g)
    hr.upload_partition(up)
    mbw, pbw = p_ctx.max_block_weights(), p_ctx.perfectly_balanced_block_weights()
    _, bw, _ = hr.overload_balance(k, mbw, pbw, None)
    ob = O.overload_balance(g, k, up, mbw, pbw, seed=seed, call=0)
    assert np.array_equal(bw, ob["block_weights"]), "overload balance"
    _, bw, _ = hr.refine(k, mbw, None)
    ep, ebw = B.oracle_lp_refine(g, seed, k, mbw, ob["labels"], schedule=B.SYNC, params=REFINE_PARAMS)
    assert np.array_equal(bw, ebw) and np.array_equal(hr.download_labels(), ep), "refinement"
    # extension to k' = 2k from the refined labels on the device
    sg = SG.extract_subgraphs(hr, k)
    exp = assert_extracted(sg, g, ep, k)
    k_prime = 2 * k
    sub = np.zeros(g.n, np.uint32)
    for b in range(k):
        lo, hi = int(exp["node_off"][b]), int(exp["node_off"][b + 1])
        x, adj, vw, ew = S.block_of(exp, b)
        gb = CSRGraph(x.copy(), adj.copy(), vw.copy(), ew.copy())
        p0 = (np.arange(gb.n, dtype=np.int64) * 2 // max(gb.n, 1)).astype(np.uint32)
        if split == "lp":  # a bipartition refined on a second handle that views the block in place
            hb = _handle(seed)
            hb.set_graph_device(*sg.device_view(b))
            bmbw = np.full(2, int(gb.vwgt.sum() * 0.53) + 1, np.int32)
            p0, _, _ = hb.refine(2, bmbw, p0.copy())
            hb.close()
            ep0, _ = B.oracle_lp_refine(gb, seed, 2, bmbw, (np.arange(gb.n, dtype=np.int64) * 2 //
                                                           max(gb.n, 1)).astype(np.uint32), schedule=B.SYNC,
                                        params=REFINE_PARAMS)
            assert np.array_equal(p0, ep0), f"block {b} bipartition"
        sub[lo:hi] = p0
    want, want_bw = S.copy_back(ep, exp["mapping"], exp["node_off"], sub, k, k_prime, input_k, g.vwgt)
    _, bw = sg.copy_partitions(hr, sub, k_prime, input_k, fetch=False)
    assert np.array_equal(hr.download_labels(), want), "copy-back"
    # balance and refine at k' from the device labels
    p2 = ctx.partition.setup(g, k_prime, 0.03)
    mbw2, pbw2 = p2.max_block_weights(), p2.perfectly_balanced_block_weights()
    _, bw, _ = hr.overload_balance(k_prime, mbw2, pbw2, None)
    ob2 = O.overload_balance(g, k_prime, want, mbw2, pbw2, seed=seed, call=1)
    assert np.array_equal(bw, ob2["block_weights"]), "overload balance at k'"
    _, bw, _ = hr.refine(k_prime, mbw2, None)
    ep2, ebw2 = B.oracle_lp_refine(g, seed, k_prime, mbw2, ob2["labels"], schedule=B.SYNC, params=REFINE_PARAMS)
    assert np.array_equal(bw, ebw2) and np.array_equal(hr.download_labels(), ep2), "refinement at k'"
    sg.close()
    cg.close()
    hr.close()
    hc.close()
