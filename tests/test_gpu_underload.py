"""The underload balancer on the device (-m gpu) against the NumPy oracle of DESIGN.md §12, bit for bit.

T0  kmp_underload_select_all == underload_oracle.underload_select_all on frozen states: targets exactly at their
    maximum and one above, sources exactly at min + w and one below, gain ties across underloaded blocks, vertices
    without an underloaded neighbour block, isolated vertices, vertex weights near 2^24, hub vertices, degrees on
    both sides of the thread / warp / CTA tiers (8|9, 256|257), k above the CTA tier's 8192-block range.
T1  kmp_underload_balance == underload_oracle.underload_balance: labels, block weights, moves per round, underload
    before / after, return value; again with every launch capped at 1..3 CTAs (KMP_GRID_CAP).
T2  the device-resident chain upload -> overload balance(NULL) -> LP refine(NULL, min weights) -> underload
    balance(NULL) -> download equals the host chain and the oracles; LP and overload results do not depend on an
    earlier underload call on the handle.
T3  refusals: seq_strict, sharded and stepping handles, labels that are a clustering.
"""
import ctypes as C
import zlib

import numpy as np
import pytest

from kaminpar_b200 import lp
from kaminpar_b200.graph import CSRGraph, rmat
from oracle import bindings as B
from tests import balance_oracle as O
from tests import helpers as H
from tests import underload_oracle as U

pytestmark = pytest.mark.gpu

I32_MAX = (1 << 31) - 1


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


def _select_graphs():
    iso = H.from_edges(50, [(i, i + 1) for i in range(30)])  # vertices 31..49 isolated
    return {
        "rmat11": rmat(11, 8, seed=5),
        "rmat11_w": _weighted(rmat(11, 8, seed=5), 1, 6, 2, edges=True),
        "grid": H.grid2d(30, 30),
        "iso": iso,
        "star": H.big_star(5000),
        "ladder": H.degree_ladder((7, 8, 9, 255, 256, 257, 3000), 4000, weighted=True, seed=1),
        "mag": _weighted(rmat(6, 8, seed=2), (1 << 24) - 8, 1 << 24, 3),  # total weight < 2^31
    }


def _frozen(g, k, regime, rng):
    """labels, W, max, min with about half the blocks underloaded (W < min)."""
    labels = rng.integers(0, k, g.n).astype(np.uint32)
    vw = np.ones(g.n, np.int64) if g.vwgt is None else g.vwgt.astype(np.int64)
    W = np.bincount(labels, weights=vw, minlength=k).astype(np.int64)
    vmax = int(vw.max())
    under = rng.random(k) < 0.5
    under[0] = True
    if regime == "edge":  # targets exactly at max for some vertex weight or one above; sources at min + w or below
        w = rng.choice(vw, k)
        maxw = np.where(under, W + w - rng.integers(0, 2, k), W + 4 * vmax)
        minw = np.where(under, W + 1 + rng.integers(0, vmax, k), W - w + rng.integers(0, 2, k))
    elif regime == "tight":  # half the targets cannot take anything, half the sources cannot lose anything
        half = rng.random(k) < 0.5
        maxw = np.where(under & half, W - 1, W + 4 * vmax)
        minw = np.where(under, W + vmax, np.where(half, W, W - 4 * vmax))
    else:
        maxw = W + 4 * vmax
        minw = np.where(under, W + 2 * vmax, W - 4 * vmax)
    clip = lambda a: np.clip(a, 0, I32_MAX).astype(np.int32)  # noqa: E731
    return labels, W.astype(np.int32), clip(maxw), clip(minw)


@pytest.mark.parametrize("name", ["rmat11", "rmat11_w", "grid", "iso", "star", "ladder", "mag"])
@pytest.mark.parametrize("k", [2, 16, 300, 20000])
@pytest.mark.parametrize("regime", ["edge", "tight", "loose"])
def test_underload_select_all_matches_oracle(name, k, regime):
    g = _select_graphs()[name]
    rng = np.random.default_rng(zlib.crc32(f"under/{name}/{k}/{regime}".encode()))
    labels, W, maxw, minw = _frozen(g, k, regime, rng)
    h = _handle(seed=3)
    h.set_graph(g)
    for call, rnd in ((0, 0), (2, 5)):
        t, key = h.underload_select_all(k, labels, W, maxw, minw, call_index=call, round=rnd)
        et, ekey = U.underload_select_all(g, k, labels, W, maxw, minw, seed=3, call=call, rnd=rnd)
        assert np.array_equal(t, et), f"targets differ at {np.nonzero(t != et)[0][:10]}"
        assert np.array_equal(key.view(np.uint32), ekey.view(np.uint32))
    h.close()


def _cases():
    return [
        ("rmat12", rmat(12, 8, seed=3), 16, 0.10),
        ("rmat12_w", _weighted(rmat(12, 8, seed=3), 1, 9, 1, edges=True), 64, 0.30),
        ("grid", H.grid2d(60, 60), 4, 0.20),
        ("walshaw", H.load_graph("walshaw_data"), 2, 0.10),
        ("walshaw256", H.load_graph("walshaw_data"), 256, 0.30),
        ("rgg16w", H.load_graph("rgg16_vwgt_adjwgt"), 16, 0.10),
        ("star", H.big_star(3000), 4, 0.5),
    ]


def _min_weights(p, min_eps=0.03):
    return U.min_block_weights(p.perfectly_balanced_block_weights(), min_eps)


def _check(g, k, part, p, seed=0, handle=None):
    mbw, mnw = p.max_block_weights(), _min_weights(p)
    h = handle or _handle(seed=seed)
    h.set_graph(g)
    got = part.copy()
    improved, bw, st = h.underload_balance(k, mbw, mnw, got)
    want = U.underload_balance(g, k, part, mbw, mnw, seed=seed)
    assert np.array_equal(got, want["labels"])
    assert np.array_equal(bw, want["block_weights"])
    assert improved == want["improved"]
    assert st.moved_list() == want["moved"]
    assert (st.underload_before, st.underload_after) == (want["before"], want["after"])
    if handle is None:
        h.close()
    return want


@pytest.mark.parametrize("case", range(7))
def test_underload_balance_matches_oracle(case):
    name, g, k, share = _cases()[case]
    p = lp.create_default_context().partition.setup(g, k, 0.03)
    want = _check(g, k, U.underload_input(g, k, 11, share), p, seed=2)
    assert want["improved"] and want["rounds"] > 0


@pytest.mark.parametrize("cap", [1, 2, 3])
def test_underload_balance_grid_cap(cap, monkeypatch):
    monkeypatch.setenv("KMP_GRID_CAP", str(cap))  # read by kmp_lp_create
    for case in (0, 1, 6):
        name, g, k, share = _cases()[case]
        p = lp.create_default_context().partition.setup(g, k, 0.03)
        _check(g, k, U.underload_input(g, k, 5, share), p, seed=1)


def test_no_min_weights_or_min_balanced_input():
    g = H.load_graph("walshaw_data")
    k = 8
    p = lp.create_default_context().partition.setup(g, k, 0.03)
    part = (np.arange(g.n) % k).astype(np.uint32)
    h = _handle()
    h.set_graph(g)
    got = part.copy()
    improved, bw, st = h.underload_balance(k, p.max_block_weights(), _min_weights(p), got)
    assert not improved and st.rounds == 0 and np.array_equal(got, part)
    assert np.array_equal(bw, O.block_weights(g, part, k))
    skewed = U.underload_input(g, k, 3, 0.5)
    got = skewed.copy()
    improved, bw, st = h.underload_balance(k, p.max_block_weights(), None, got)
    assert not improved and bw is None and st.rounds == 0 and np.array_equal(got, skewed)
    h.close()


def _chain_input():
    g = _weighted(rmat(12, 8, seed=3), 1, 5, 4)
    k = 16
    p = lp.create_default_context().partition.setup(g, k, 0.03)
    part = O.overload_input(g, k, 9, 0.15, (0, 3))
    rng = np.random.default_rng(4)
    part[np.flatnonzero((part == 5) & (rng.random(g.n) < 0.3))] = 0  # block 5 underloaded, block 0 overloaded
    # minimum = perfectly balanced weight: the LP refiner leaves some underload for the last stage
    return g, k, p.max_block_weights(), p.perfectly_balanced_block_weights(), _min_weights(p, 0.0), part


def test_device_resident_chain():
    g, k, mbw, pbw, mnw, part = _chain_input()
    # device-resident: nothing crosses the bus between the stages
    hd = _handle()
    hd.set_graph(g)
    hd.upload_partition(part)
    hd.overload_balance(k, mbw, pbw, None)
    hd.refine(k, mbw, None, min_block_weights=mnw)
    improved, bw_dev, st = hd.underload_balance(k, mbw, mnw, None)
    dev = hd.download_labels()
    # host chain on another handle
    hh = _handle()
    hh.set_graph(g)
    host = part.copy()
    hh.overload_balance(k, mbw, pbw, host)
    hh.refine(k, mbw, host, min_block_weights=mnw)
    hh.underload_balance(k, mbw, mnw, host)
    assert np.array_equal(dev, host)
    # oracles: overload balance, the refiner's sync schedule with minimum weights, underload balance
    ob = O.overload_balance(g, k, part, mbw, pbw)
    rp = B.oracle_params(B.default_refine_params(), commit_passes=4)
    ep, _ = B.oracle_lp_refine(g, 0, k, mbw, ob["labels"], schedule=B.SYNC, params=rp, min_block_weights=mnw)
    ub = U.underload_balance(g, k, ep, mbw, mnw)
    assert ub["improved"] and improved
    assert np.array_equal(dev, ub["labels"]) and np.array_equal(bw_dev, ub["block_weights"])
    assert st.moved_list() == ub["moved"]
    hd.close()
    hh.close()


def test_lp_and_overload_results_do_not_depend_on_an_earlier_underload_call():
    g, k, mbw, pbw, mnw, part = _chain_input()
    results = []
    for first in (False, True):
        h = _handle()
        h.set_graph(g)
        if first:
            assert h.underload_balance(k, mbw, mnw, U.underload_input(g, k, 1, 0.3))[0]
        x = part.copy()
        _, bw_o, st_o = h.overload_balance(k, mbw, pbw, x)
        y = x.copy()
        _, bw_r, st_r = h.refine(k, mbw, y, min_block_weights=mnw)
        results.append((x, bw_o, st_o.moved_list(), y, bw_r, st_r.moved_list()))
        h.close()
    for a, b in zip(*results):
        assert np.array_equal(a, b) if isinstance(a, np.ndarray) else a == b


def test_underload_balancer_operator():
    g = H.load_graph("walshaw_data")
    k = 16
    ctx = lp.create_default_context()
    ctx.partition.setup(g, k, 0.03)
    part = U.underload_input(g, k, 2, 0.2)
    pg = lp.PartitionedGraph(g, k, part)
    bal = lp.UnderloadBalancer(ctx)
    assert bal.name() == "Underload Balancer"
    bal.initialize(pg)
    assert not bal.refine(pg, ctx.partition)  # no minimum weights: no device work
    assert bal.last_stats is None and np.array_equal(pg.partition, part)
    mnw = _min_weights(ctx.partition)
    ctx.partition.setup_min_block_weights(mnw)
    assert bal.refine(pg, ctx.partition)
    want = U.underload_balance(g, k, part, ctx.partition.max_block_weights(), mnw)
    assert np.array_equal(pg.partition, want["labels"])
    assert np.array_equal(pg.block_weights(), want["block_weights"])
    assert want["after"] == 0
    assert not bal.refine(pg, ctx.partition)  # now min-balanced: no device work
    assert bal.last_stats is None


def test_refusals():
    g = rmat(10, 8, seed=1)
    k = 4
    p = lp.create_default_context().partition.setup(g, k, 0.03)
    mbw, mnw = p.max_block_weights(), _min_weights(p)
    part = U.underload_input(g, k, 1, 0.3)
    hs = _handle(schedule="seq_strict")
    hs.set_graph(g)
    with pytest.raises(RuntimeError, match="error -4"):
        hs.underload_balance(k, mbw, mnw, part.copy())
    with pytest.raises(RuntimeError, match="error -4"):
        hs.underload_select_all(k, part, O.block_weights(g, part, k), mbw, mnw)
    hs.close()
    lib = lp.load_library()
    hsh = _handle()
    hsh.set_graph(g)
    assert lib.kmp_lp_set_shard(hsh._h, C.c_uint32(0), C.c_uint32(2)) == 0  # rank 0 of 2: a sharded handle
    with pytest.raises(RuntimeError, match="error -4"):
        hsh.underload_balance(k, mbw, mnw, part.copy())
    hsh.close()
    ht = _handle()
    ht.set_graph(g)
    mb = np.ascontiguousarray(mbw, np.int32)
    assert lib.kmp_lp_step_begin_refine(ht._h, C.c_uint32(k), mb.ctypes.data_as(C.c_void_p), None, None,
                                        part.ctypes.data_as(C.c_void_p)) == 0
    with pytest.raises(RuntimeError, match="error -4"):
        ht.underload_balance(k, mbw, mnw, part.copy())
    ht.close()


def test_refuses_a_clustering_of_a_large_graph():
    """Labels up to n - 1 with n >> k: refused before any kernel reads a [k] array at a label."""
    g = rmat(16, 8, seed=2)
    k = 4
    p = lp.create_default_context().partition.setup(g, k, 0.03)
    mbw, mnw = p.max_block_weights(), _min_weights(p)
    ctx = lp.create_default_context()
    hc = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
    hc.set_graph(g)
    clustering, _ = hc.cluster(max_cluster_weight=40)
    assert int(clustering.max()) > 1000 * k
    with pytest.raises(RuntimeError, match="error -1"):
        hc.underload_balance(k, mbw, mnw, None)
    # the handle still works afterwards: a valid partition balances
    improved, _, _ = hc.underload_balance(k, mbw, mnw, U.underload_input(g, k, 3, 0.3))
    assert improved
    hc.close()
