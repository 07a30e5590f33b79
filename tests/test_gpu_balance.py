"""The overload balancer on the device (-m gpu) against the NumPy oracle of DESIGN.md §11, bit for bit.

T0  kmp_balance_select_all == balance_oracle.select_all on frozen states: targets exactly at capacity and one
    above, gain ties across blocks, vertices without a feasible neighbour block, isolated vertices, vertex weights
    near 2^24, hub vertices, degrees on both sides of the thread / warp / CTA tiers (8|9, 256|257), k above the
    CTA tier's 8192-block range.
T1  kmp_overload_balance == balance_oracle.overload_balance: labels, block weights, moves per round, return value;
    again with every launch capped at 1..3 CTAs (KMP_GRID_CAP).
T2  the device-resident chain upload -> balance(NULL) -> refine(NULL) -> download equals the host chain and the
    oracles (balance, then the LP refiner's sync schedule).
T3  refusals: seq_strict handles, labels that are a clustering.
"""
import zlib

import numpy as np
import pytest

from kaminpar_b200 import lp
from kaminpar_b200.graph import CSRGraph, rmat
from oracle import bindings as B
from tests import balance_oracle as O
from tests import helpers as H

pytestmark = pytest.mark.gpu


def _handle(schedule="sync", seed=0):
    ctx = lp.create_default_context()
    ctx.engine.schedule = schedule
    ctx.engine.seed = seed
    return lp.LPHandle(lp._refine_config(ctx.refinement.lp, ctx.engine))


def _weighted(g, lo, hi, seed, edges=False):
    rng = np.random.default_rng(seed)
    ew = None
    if edges:  # symmetric edge weights
        src = np.repeat(np.arange(g.n), np.diff(g.xadj.astype(np.int64)))
        a, b = np.minimum(src, g.adjncy), np.maximum(src, g.adjncy)
        ew = ((a.astype(np.int64) * 7919 + b * 104729) % 5 + 1).astype(np.int32)
    return CSRGraph(g.xadj, g.adjncy, rng.integers(lo, hi, g.n).astype(np.int32), ew)


def _ladder():
    degs = (7, 8, 9, 255, 256, 257, 3000)
    return H.degree_ladder(degs, 4000, weighted=True, seed=1)


def _select_graphs():
    iso = H.from_edges(50, [(i, i + 1) for i in range(30)])  # vertices 31..49 isolated
    return {
        "rmat11": rmat(11, 8, seed=5),
        "rmat11_w": _weighted(rmat(11, 8, seed=5), 1, 6, 2, edges=True),
        "grid": H.grid2d(30, 30),
        "iso": iso,
        "star": H.big_star(5000),
        "ladder": _ladder(),
        "mag": _weighted(rmat(6, 8, seed=2), (1 << 24) - 8, 1 << 24, 3),  # total weight < 2^31
    }


def _frozen(g, k, regime, rng):
    labels = rng.integers(0, k, g.n).astype(np.uint32)
    vw = np.ones(g.n, np.int64) if g.vwgt is None else g.vwgt.astype(np.int64)
    W = np.bincount(labels, weights=vw, minlength=k).astype(np.int64)
    if regime == "capacity":  # every block exactly at capacity for some vertex weight, or one above
        w = rng.choice(vw, k)
        maxw = W + w - rng.integers(0, 2, k)
    elif regime == "tight":   # about half the blocks cannot take anything
        maxw = W + np.where(rng.random(k) < 0.5, -1, int(vw.max()))
    else:
        maxw = W + int(vw.max()) * 4
    return labels, W.astype(np.int32), np.minimum(maxw, (1 << 31) - 1).astype(np.int32)


@pytest.mark.parametrize("name", ["rmat11", "rmat11_w", "grid", "iso", "star", "ladder", "mag"])
@pytest.mark.parametrize("k", [2, 16, 300, 20000])
@pytest.mark.parametrize("regime", ["capacity", "tight", "loose"])
def test_select_all_matches_oracle(name, k, regime):
    g = _select_graphs()[name]
    rng = np.random.default_rng(zlib.crc32(f"{name}/{k}/{regime}".encode()))
    labels, W, maxw = _frozen(g, k, regime, rng)
    h = _handle(seed=3)
    h.set_graph(g)
    for call, rnd in ((0, 0), (2, 5)):
        t, key = h.balance_select_all(k, labels, W, maxw, call_index=call, round=rnd)
        et, ekey = O.select_all(g, k, labels, W, maxw, seed=3, call=call, rnd=rnd)
        assert np.array_equal(t, et), f"targets differ at {np.nonzero(t != et)[0][:10]}"
        assert np.array_equal(key.view(np.uint32), ekey.view(np.uint32))
    h.close()


def _balance_cases():
    return [
        ("rmat12", rmat(12, 8, seed=3), 16, 0.10, (0,)),
        ("rmat12_w", _weighted(rmat(12, 8, seed=3), 1, 9, 1, edges=True), 64, 0.20, (0, 5, 9)),
        ("grid", H.grid2d(60, 60), 4, 0.30, (1,)),
        ("walshaw", H.load_graph("walshaw_data"), 2, 0.10, (0,)),
        ("walshaw256", H.load_graph("walshaw_data"), 256, 0.10, (0, 1)),
        ("rgg16w", H.load_graph("rgg16_vwgt_adjwgt"), 16, 0.05, (3,)),
        ("star", H.big_star(3000), 4, 0.5, (2,)),
    ]


def _check_balance(g, k, part, p, seed=0, handle=None):
    mbw, pbw = p.max_block_weights(), p.perfectly_balanced_block_weights()
    h = handle or _handle(seed=seed)
    h.set_graph(g)
    got = part.copy()
    improved, bw, st = h.overload_balance(k, mbw, pbw, got)
    want = O.overload_balance(g, k, part, mbw, pbw, seed=seed)
    assert np.array_equal(got, want["labels"])
    assert np.array_equal(bw, want["block_weights"])
    assert improved == want["improved"]
    assert st.moved_list() == want["moved"]
    assert (st.overload_before, st.overload_after) == (want["before"], want["after"])
    if handle is None:
        h.close()
    return want


@pytest.mark.parametrize("case", range(7))
def test_overload_balance_matches_oracle(case):
    name, g, k, share, blocks = _balance_cases()[case]
    p = lp.create_default_context().partition.setup(g, k, 0.03)
    part = O.overload_input(g, k, 11, share, blocks)
    want = _check_balance(g, k, part, p, seed=2)
    assert want["improved"] and want["rounds"] > 0


@pytest.mark.parametrize("cap", [1, 2, 3])
def test_overload_balance_grid_cap(cap, monkeypatch):
    monkeypatch.setenv("KMP_GRID_CAP", str(cap))  # read by kmp_lp_create
    for case in (0, 1, 6):
        name, g, k, share, blocks = _balance_cases()[case]
        p = lp.create_default_context().partition.setup(g, k, 0.03)
        _check_balance(g, k, O.overload_input(g, k, 5, share, blocks), p, seed=1)


def test_feasible_input_returns_false_untouched():
    g = H.load_graph("walshaw_data")
    k = 8
    p = lp.create_default_context().partition.setup(g, k, 0.03)
    part = (np.arange(g.n) % k).astype(np.uint32)
    h = _handle()
    h.set_graph(g)
    got = part.copy()
    improved, bw, st = h.overload_balance(k, p.max_block_weights(), p.perfectly_balanced_block_weights(), got)
    assert not improved and st.rounds == 0 and np.array_equal(got, part)
    assert np.array_equal(bw, O.block_weights(g, part, k))


def test_device_resident_chain():
    g = _weighted(rmat(12, 8, seed=3), 1, 5, 4)
    k = 16
    p = lp.create_default_context().partition.setup(g, k, 0.03)
    mbw, pbw = p.max_block_weights(), p.perfectly_balanced_block_weights()
    part = O.overload_input(g, k, 9, 0.15, (0, 3))
    # device-resident: nothing crosses the bus between the two calls
    hd = _handle()
    hd.set_graph(g)
    hd.upload_partition(part)
    improved, bw_bal, _ = hd.overload_balance(k, mbw, pbw, None)
    _, bw_dev, _ = hd.refine(k, mbw, None)
    dev = hd.download_labels()
    # host chain on another handle
    hh = _handle()
    hh.set_graph(g)
    host = part.copy()
    hh.overload_balance(k, mbw, pbw, host)
    hh.refine(k, mbw, host)
    assert improved
    assert np.array_equal(dev, host)
    # oracles: the balancer, then the refiner's sync schedule on the balanced partition
    want = O.overload_balance(g, k, part, mbw, pbw)
    assert np.array_equal(bw_bal, want["block_weights"])
    rp = B.oracle_params(B.default_refine_params(), commit_passes=4)
    ep, ebw = B.oracle_lp_refine(g, 0, k, mbw, want["labels"], schedule=B.SYNC, params=rp)
    assert np.array_equal(dev, ep) and np.array_equal(bw_dev, ebw)
    hd.close()
    hh.close()


def test_overload_balancer_operator():
    g = H.load_graph("walshaw_data")
    k = 16
    ctx = lp.create_default_context()
    ctx.partition.setup(g, k, 0.03)
    part = O.overload_input(g, k, 2, 0.2, (0,))
    pg = lp.PartitionedGraph(g, k, part)
    bal = lp.OverloadBalancer(ctx)
    assert bal.name() == "Overload Balancer"
    bal.initialize(pg)
    assert bal.refine(pg, ctx.partition)
    want = O.overload_balance(g, k, part, ctx.partition.max_block_weights(),
                              ctx.partition.perfectly_balanced_block_weights())
    assert np.array_equal(pg.partition, want["labels"])
    assert np.array_equal(pg.block_weights(), want["block_weights"])
    assert want["after"] == 0
    assert not bal.refine(pg, ctx.partition)  # now feasible: no device work
    assert bal.last_stats is None


def test_refusals():
    g = rmat(10, 8, seed=1)
    k = 4
    p = lp.create_default_context().partition.setup(g, k, 0.03)
    mbw, pbw = p.max_block_weights(), p.perfectly_balanced_block_weights()
    part = O.overload_input(g, k, 1, 0.3)
    hs = _handle(schedule="seq_strict")
    hs.set_graph(g)
    with pytest.raises(RuntimeError, match="error -4"):
        hs.overload_balance(k, mbw, pbw, part.copy())
    with pytest.raises(RuntimeError, match="error -4"):
        hs.balance_select_all(k, part, O.block_weights(g, part, k), mbw)
    hs.close()
    # the device labels are a clustering (ids in [0, n)), not a k-way partition
    ctx = lp.create_default_context()
    hc = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
    hc.set_graph(g)
    hc.cluster(max_cluster_weight=20)
    with pytest.raises(RuntimeError, match="error -1"):
        hc.overload_balance(k, mbw, pbw, None)
    hc.close()


def test_refuses_a_clustering_of_a_large_graph():
    """Labels up to n - 1 with n >> k: refused before any kernel reads a [k] array at a label."""
    g = rmat(16, 8, seed=2)
    k = 4
    p = lp.create_default_context().partition.setup(g, k, 0.03)
    ctx = lp.create_default_context()
    hc = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
    hc.set_graph(g)
    clustering, _ = hc.cluster(max_cluster_weight=40)
    assert int(clustering.max()) > 1000 * k
    with pytest.raises(RuntimeError, match="error -1"):
        hc.overload_balance(k, p.max_block_weights(), p.perfectly_balanced_block_weights(), None)
    # the handle still works afterwards: a valid partition balances
    part = O.overload_input(g, k, 3, 0.3)
    improved, _, _ = hc.overload_balance(k, p.max_block_weights(), p.perfectly_balanced_block_weights(), part)
    assert improved
    hc.close()


def test_refuses_sharded_and_stepping_handles():
    import ctypes as C

    g = rmat(10, 8, seed=1)
    k = 4
    p = lp.create_default_context().partition.setup(g, k, 0.03)
    mbw, pbw = p.max_block_weights(), p.perfectly_balanced_block_weights()
    part = O.overload_input(g, k, 1, 0.3)
    lib = lp.load_library()
    hs = _handle()
    hs.set_graph(g)
    assert lib.kmp_lp_set_shard(hs._h, C.c_uint32(0), C.c_uint32(2)) == 0  # rank 0 of 2: a sharded handle
    with pytest.raises(RuntimeError, match="error -4"):
        hs.overload_balance(k, mbw, pbw, part.copy())
    hs.close()
    ht = _handle()
    ht.set_graph(g)
    mb = np.ascontiguousarray(mbw, np.int32)
    assert lib.kmp_lp_step_begin_refine(ht._h, C.c_uint32(k), mb.ctypes.data_as(C.c_void_p), None, None,
                                        part.ctypes.data_as(C.c_void_p)) == 0
    with pytest.raises(RuntimeError, match="error -4"):
        ht.overload_balance(k, mbw, pbw, part.copy())
    ht.close()
