"""Parity tests of the overlay of clusterings on the device (-m gpu, DESIGN.md §14): kmp_overlay_clusterings and
kmp_lp_cluster_overlay through the C ABI (include/kaminpar_b200_contraction.h) against the overlay oracle
(tests/overlay_oracle.py) over the LP oracle's and the reference's own clusterings, bit for bit.

    T0  the tree over crafted clusterings, also under KMP_GRID_CAP
    T1  2^L LP calls + tree == overlay_tree of the oracle's 2^L consecutive calls (sync), of the reference's (seq_strict)
    T2  overlay -> contraction from the device labels -> next level on the device; overlay_level and max_level
    T3  refusals"""
import ctypes as C
import os

import numpy as np
import pytest

from kaminpar_b200 import contraction as KC
from kaminpar_b200 import lp
from kaminpar_b200.graph import CSRGraph, rmat
from oracle import bindings as B
from oracle import contraction_oracle as CO
from tests import helpers as H
from tests import overlay_oracle as O
from tests.test_gpu_parity import NAMES, ctx_for, get_graph
from tests.test_gpu_strict import _ctx as strict_ctx

pytestmark = pytest.mark.gpu


def new_handle(seed=0):
    ctx = lp.create_default_context()
    ctx.engine.seed = seed
    return lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))


def clog2(x):
    return int(x - 1).bit_length() if x > 1 else 0


def tree_sort_bits(cls):
    """max over the tree's pairs of ceil(log2 n) + ceil(log2 c_a)"""
    c = [np.asarray(x, np.uint32) for x in cls]
    n, bits, half = len(c[0]), 0, len(c) // 2
    while half >= 1:
        for p in range(half):
            bits = max(bits, clog2(n) + clog2(len(np.unique(c[p]))))
            c[p] = O.overlay(c[p], c[half + p])
        half //= 2
    return bits


def check_tree(h, cls):
    cls = np.ascontiguousarray(np.asarray(cls, np.uint32))
    out, st = h.overlay(cls)
    exp = O.overlay_tree(list(cls))
    assert np.array_equal(out, exp)
    assert np.array_equal(h.download_labels(), exp)  # the result is the handle's device labels
    assert st.num_clusterings == len(cls) and st.num_clusters == len(np.unique(exp))
    assert st.sort_bits == (tree_sort_bits(cls) if len(cls) > 1 else 0)
    return exp


def crafted():
    rng = np.random.default_rng(5)
    yield "n1", 1, [[0], [0]]
    n = 1000
    ident = np.arange(n)
    x = rng.integers(0, 40, n) * 17
    yield "identity", n, [ident, x]
    yield "identity_b", n, [x, ident]
    yield "all_equal", n, [np.zeros(n), np.zeros(n)]
    yield "all_equal_a", n, [np.zeros(n), x]
    yield "a_eq_b", n, [x, x]
    w, hgt = 50, 40  # rows x columns of a grid: every (row, column) pair is one vertex
    u = np.arange(w * hgt)
    yield "grid_rows_cols", w * hgt, [u // w, u % w]
    yield "grid_cols_rows", w * hgt, [u % w, u // w]
    yield "labels_n_minus_1", n, [np.full(n, n - 1), np.where(rng.random(n) < 0.5, n - 1, x)]
    big = 1 << 20  # one cluster of a spans every CTA of the sort and of the scatter
    yield "one_big_cluster", big, [np.zeros(big), rng.integers(0, big, big)]
    yield "count4", n, [rng.integers(0, k, n) * (n // k) for k in (3, 10, 50, 7)]
    yield "count8", 5000, [rng.integers(0, 5000, 5000) // d * d for d in (1, 2, 3, 5, 8, 13, 21, 34)]
    yield "count1", n, [x]


@pytest.mark.parametrize("name,n,cls", list(crafted()))
def test_t0_crafted(name, n, cls):
    h = new_handle()
    h.set_graph(H.empty_graph(n))
    check_tree(h, cls)


@pytest.mark.parametrize("cap", [1, 2, 3])
def test_t0_grid_cap(cap, monkeypatch):
    monkeypatch.setenv("KMP_GRID_CAP", str(cap))  # read by kmp_lp_create
    h = new_handle()
    for name, n, cls in crafted():
        if n <= 5000:
            h.set_graph(H.empty_graph(n))
            check_tree(h, cls)
    g = get_graph("rmat13_w")
    ctx, mcw = ctx_for(g, 8, seed=4)
    h = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
    h.set_graph(g)
    out, _ = h.cluster_overlay(2, mcw)
    calls = B.oracle_lp_cluster(g, 4, mcw, schedule=B.SYNC, num_calls=4)
    assert np.array_equal(out, O.overlay_tree(list(calls)))


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("levels", [0, 1, 2])
def test_t1_cluster_overlay_matches_oracle_sync(name, levels):
    g = get_graph(name)
    seed = 3
    ctx, mcw = ctx_for(g, 8, seed=seed)
    h = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
    h.set_graph(g)
    count = 1 << levels
    out, st = h.cluster_overlay(levels, mcw)
    calls = B.oracle_lp_cluster(g, seed, mcw, schedule=B.SYNC, num_calls=count + 1)
    exp = O.overlay_tree(list(calls[:count]))
    assert np.array_equal(out, exp)
    assert st.num_clusterings == count and st.num_clusters == len(np.unique(exp))
    assert st.sort_bits == (tree_sort_bits(calls[:count]) if count > 1 else 0)
    assert st.lp_device_ms > 0
    # the call counter advanced by 2^L: the next clustering is the oracle's call 2^L
    nxt, _ = h.cluster(mcw)
    assert np.array_equal(nxt, calls[count])


def strict_case(name):
    """(graph, max cluster weight, seed, the reference's consecutive clusterings on one LPClustering object, cluster
    config) from an existing multi-call golden (ref_*.npz) or an overlay golden (overlay_*.npz,
    tests/golden/make_overlay_golden.py)."""
    if name.startswith("overlay_"):
        d = np.load(os.path.join(H.GOLDEN, f"{name}.npz"))
        g = CSRGraph(d["xadj"], d["adjncy"], sorted=True, buckets=d["buckets"])
        seed = int(d["seed"][0])
        ctx = lp.create_default_context()
        ctx.engine.seed = seed
        ctx.engine.schedule = "seq_strict"
        return g, int(d["max_cluster_weight"][0]), d["clusterings"], ctx
    g, d = H.load_case(name)
    seed = int(d["seeds"][0])
    return g, int(d["max_cluster_weight"][0]), d[f"clustering_s{seed}"], strict_ctx(d, seed)


STRICT_CASES = [("walshaw_3calls", 1), ("overlay_walshaw", 1), ("overlay_walshaw", 2), ("overlay_rgg2d", 1),
                ("overlay_rgg2d", 2)]


@pytest.mark.parametrize("name,levels", STRICT_CASES)
def test_t1_strict_overlay_matches_reference_clusterings(name, levels):
    g, mcw, ref, ctx = strict_case(name)
    h = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
    h.set_graph(g)
    count = 1 << levels
    out, st = h.cluster_overlay(levels, mcw)
    exp = O.overlay_tree(list(ref[:count]))
    assert np.array_equal(out, exp) and st.num_clusters == len(np.unique(exp))
    if count < len(ref):  # the random stream continued across the calls
        assert np.array_equal(h.cluster(mcw)[0], ref[count])


def gpu_result(cg):
    c = cg.get()
    return dict(c_n=cg.n, c_xadj=c.xadj, c_adjncy=c.adjncy, c_vwgt=c.vwgt, c_adjwgt=c.adjwgt, mapping=cg.mapping())


def test_t2_device_resident_level():
    """overlay -> kmp_contract_clustering(h, NULL) -> kmp_lp_set_graph_device -> cluster, next to the host path."""
    g = B.oracle_rearrange(rmat(15, 16, 21))[0]
    ctx, mcw = ctx_for(g, 8, seed=2)
    h0 = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
    h0.set_graph(g)
    out, _ = h0.cluster_overlay(1, mcw, fetch=False)
    assert out is None
    ov = O.overlay_tree(list(B.oracle_lp_cluster(g, 2, mcw, schedule=B.SYNC, num_calls=2)))
    # the calls that read the device labels see the overlay (weights they need are recomputed from the labels)
    assert h0.edge_cut() == B.oracle_edge_cut(g, ov)
    cg = KC.contract_on_handle(h0, None)
    con = CO.contract(g.xadj, g.adjncy, g.vwgt, g.adjwgt, ov)
    assert CO.equal(gpu_result(cg), con)
    hh = new_handle()
    hh.set_graph(g)
    cg_host = KC.contract_on_handle(hh, ov)  # host path: the downloaded overlay contracted from the host
    assert CO.equal(gpu_result(cg_host), con)
    cg_host.close()
    d_xadj, d_adj, d_vw, d_ew, _ = cg.device_arrays()
    h1 = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
    h1.set_graph_device(cg.n, cg.m, d_xadj, d_adj, d_vw, d_ew)
    c1, _ = h1.cluster(2 * mcw)
    cgraph = CSRGraph(con["c_xadj"], con["c_adjncy"], con["c_vwgt"], con["c_adjwgt"])
    assert np.array_equal(c1, B.oracle_lp_cluster(cgraph, 2, 2 * mcw, schedule=B.SYNC))
    h1.close()
    cg.close()


def test_t2_overlay_level_and_max_level():
    g = get_graph("rmat13_w")
    ctx, mcw = ctx_for(g, 8, seed=6)
    h = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
    h.set_graph(g)
    calls = B.oracle_lp_cluster(g, 6, mcw, schedule=B.SYNC, num_calls=7)

    def expect(cl):
        return CO.contract(g.xadj, g.adjncy, g.vwgt, g.adjwgt, cl)

    cg = KC.overlay_level(h, 0, KC.OverlayClusterCoarseningContext(1, 0), mcw)  # level 0 <= max_level 0: overlay
    assert CO.equal(gpu_result(cg), expect(O.overlay_tree(list(calls[:2]))))
    cg.close()
    cg = KC.overlay_level(h, 1, KC.OverlayClusterCoarseningContext(1, 0), mcw)  # above max_level: one clustering
    assert CO.equal(gpu_result(cg), expect(calls[2]))
    cg.close()
    # a negative max_level compares as a huge unsigned value in the reference: it never turns the overlay off
    cg = KC.overlay_level(h, 9, KC.OverlayClusterCoarseningContext(2, -1), mcw)
    assert CO.equal(gpu_result(cg), expect(O.overlay_tree(list(calls[3:7]))))
    cg.close()
    cg = KC.overlay_level(h, 0, None, mcw)  # defaults: num_levels 1, max_level INT_MAX
    nxt = B.oracle_lp_cluster(g, 6, mcw, schedule=B.SYNC, num_calls=9)
    assert CO.equal(gpu_result(cg), expect(O.overlay_tree(list(nxt[7:9]))))
    cg.close()


def test_t3_refusals():
    lib = lp.load_library()
    n = 64
    h = new_handle()
    st = lp.KmpOverlayStats()
    cl = np.zeros((4, n), np.uint32)
    # no graph
    assert lib.kmp_overlay_clusterings(h._h, C.c_uint32(1), cl.ctypes.data_as(C.c_void_p), None, None) != 0
    assert lib.kmp_lp_cluster_overlay(h._h, C.c_int(1), C.c_int32(10), C.c_uint32(0), None, None, None) != 0
    assert lib.kmp_lp_cluster_overlay(None, C.c_int(1), C.c_int32(10), C.c_uint32(0), None, None, None) != 0
    g = H.grid2d(8, 8)
    h.set_graph(g)
    rng = np.random.default_rng(2)
    good = rng.integers(0, n, (2, n)).astype(np.uint32)
    before = check_tree(h, good)
    for count in (0, 3, 5, 6):
        assert lib.kmp_overlay_clusterings(h._h, C.c_uint32(count), cl.ctypes.data_as(C.c_void_p), None,
                                           C.byref(st)) != 0
    for levels in (-1, 17):
        assert lib.kmp_lp_cluster_overlay(h._h, C.c_int(levels), C.c_int32(10), C.c_uint32(0), None, None, None) != 0
    with pytest.raises(ValueError):
        h.overlay(np.zeros((2, n + 1), np.uint32))
    # a label >= n in any input, at any tree position: refused, the device labels stay as they were
    for count in (1, 2, 4, 8):
        for pos in {0, count - 1, count // 2}:
            bad = rng.integers(0, n, (count, n)).astype(np.uint32)
            bad[pos, 7] = n
            with pytest.raises(RuntimeError, match=">= n"):
                h.overlay(bad)
            assert np.array_equal(h.download_labels(), before)
    assert h.edge_cut() == B.oracle_edge_cut(g, before)  # still valid labels
    # sharded handles are refused
    hs = new_handle()
    hs.set_graph(g)
    assert lib.kmp_lp_set_shard(hs._h, C.c_uint32(0), C.c_uint32(2)) == 0
    with pytest.raises(RuntimeError, match="one GPU"):
        hs.overlay(good)
    with pytest.raises(RuntimeError, match="one GPU"):
        hs.cluster_overlay(1, 10)
    # n = 0: no device work, the calls still count
    he = new_handle()
    he.set_graph(H.empty_graph(0))
    out, st0 = he.overlay(np.zeros((2, 0), np.uint32))
    assert len(out) == 0 and st0.num_clusterings == 2 and st0.num_clusters == 0
    out, st0 = he.cluster_overlay(2, 10)
    assert len(out) == 0 and st0.num_clusterings == 4
    # free_scratch releases the stash and the labels; the next call works from scratch
    h.free_scratch()
    with pytest.raises(RuntimeError):
        KC.contract_on_handle(h, None)
    check_tree(h, rng.integers(0, n, (4, n)))
