"""CPU properties of the order-free underload balancer (DESIGN.md §12), on the oracle in tests/underload_oracle.py:
no block ends below its minimum because a vertex left it and none ends above its maximum by an arrival, the total
underload never rises and falls in every round that accepts a move, input without minimum weights or already
min-balanced is left untouched, and the same seed gives the same result. The source side of the commit ladder
(minimum weights) is checked on a hand-made input."""
import numpy as np
import pytest

from kaminpar_b200 import lp
from kaminpar_b200.graph import CSRGraph, rmat
from tests import balance_oracle as O
from tests import helpers as H
from tests import underload_oracle as U

MIN_EPS = 0.03


def _weights(g, k, eps=0.03, min_eps=MIN_EPS):
    p = lp.create_default_context().partition.setup(g, k, eps)
    return p.max_block_weights().astype(np.int64), U.min_block_weights(p.perfectly_balanced_block_weights(), min_eps)


def _weighted(g, seed):
    rng = np.random.default_rng(seed)
    return CSRGraph(g.xadj, g.adjncy, rng.integers(1, 9, g.n).astype(np.int32), None)


def _graph(name):
    if name == "rmat12":
        return rmat(12, 8, seed=3)
    if name == "rmat12w":
        return _weighted(rmat(12, 8, seed=3), 1)
    if name == "grid":
        return H.grid2d(40, 40)
    if name == "walshaw":
        return H.load_graph("walshaw_data")
    if name == "rgg16w":
        return H.load_graph("rgg16_vwgt_adjwgt")
    raise ValueError(name)


CASES = [("rmat12", 4, 0.10), ("rmat12", 16, 0.10), ("rmat12w", 64, 0.20), ("grid", 2, 0.08), ("walshaw", 16, 0.10),
         ("rgg16w", 256, 0.30)]


@pytest.mark.parametrize("name,k,share", CASES)
def test_underload_properties(name, k, share):
    g = _graph(name)
    mbw, mnw = _weights(g, k)
    part = U.underload_input(g, k, 7, share)
    W0 = O.block_weights(g, part, k)
    assert W0[0] < mnw[0]
    res = U.underload_balance(g, k, part, mbw, mnw, seed=1)
    W1 = res["block_weights"].astype(np.int64)
    assert np.array_equal(W1, O.block_weights(g, res["labels"], k))
    assert res["improved"] and res["before"] == U.total_underload(W0, mnw)
    lost, gained = W1 < W0, W1 > W0
    assert np.all(W1[lost] >= mnw[lost])                     # no block drops below its minimum by a departure
    assert np.all(W1[gained] <= mbw[gained])                 # no block rises above its maximum by an arrival
    assert np.all(W0[gained] < mnw[gained])                  # only underloaded blocks receive
    assert np.all(W0[lost] >= mnw[lost])                     # underloaded blocks never lose
    moved = np.flatnonzero(res["labels"] != part)
    assert np.all(W0[res["labels"][moved]] < mnw[res["labels"][moved]])
    again = U.underload_balance(g, k, part, mbw, mnw, seed=1)
    assert np.array_equal(again["labels"], res["labels"]) and again["moved"] == res["moved"]


@pytest.mark.parametrize("name,k,share", CASES)
def test_each_round_lowers_the_underload(name, k, share):
    g = _graph(name)
    mbw, mnw = _weights(g, k)
    res = U.underload_balance(g, k, U.underload_input(g, k, 3, share), mbw, mnw, seed=4)
    trace, moved = res["underload"], res["moved"]
    assert len(trace) == res["rounds"] + 1 and trace[0] == res["before"] and trace[-1] == res["after"]
    for r in range(res["rounds"]):
        assert trace[r + 1] <= trace[r]
        assert (trace[r + 1] < trace[r]) == (moved[r] > 0)
    assert res["rounds"] == O.MAX_ROUNDS or res["after"] == 0 or moved[-1] == 0


def test_reaches_zero_underload_on_the_bench_shape():
    g = _graph("rmat12")
    k = 16
    mbw, mnw = _weights(g, k)
    res = U.underload_balance(g, k, U.underload_input(g, k, 11, 0.10), mbw, mnw)
    assert res["before"] > 0 and res["after"] == 0


def test_no_min_weights_or_min_balanced_input_is_untouched():
    g = _graph("walshaw")
    k = 8
    mbw, mnw = _weights(g, k)
    part = (np.arange(g.n) % k).astype(np.uint32)
    assert U.total_underload(O.block_weights(g, part, k), mnw) == 0
    res = U.underload_balance(g, k, part, mbw, mnw)
    assert not res["improved"] and res["rounds"] == 0 and np.array_equal(res["labels"], part)
    skewed = U.underload_input(g, k, 2, 0.5)
    res = U.underload_balance(g, k, skewed, mbw, None)
    assert not res["improved"] and res["rounds"] == 0 and np.array_equal(res["labels"], skewed)


def test_seed_determinism():
    g = _graph("rmat12w")
    k = 16
    mbw, mnw = _weights(g, k)
    part = U.underload_input(g, k, 5, 0.2)
    a = U.underload_balance(g, k, part, mbw, mnw, seed=1)
    b = U.underload_balance(g, k, part, mbw, mnw, seed=1)
    c = U.underload_balance(g, k, part, mbw, mnw, seed=2)
    assert np.array_equal(a["labels"], b["labels"]) and a["moved"] == b["moved"]
    assert a["after"] == c["after"] == 0


def test_source_side_ladder():
    """Block 0 (weight 4, minimum 3) has two accepted departures but can afford one: the one at the higher ladder
    level leaves; without minimum weights both leave."""
    g = H.from_edges(6, [(0, 4), (1, 5), (2, 3)])
    labels = np.array([0, 0, 0, 0, 1, 2], np.int64)
    W = O.block_weights(g, labels, 3)
    maxw = np.array([10, 10, 10], np.int64)
    mv_u, mv_t = np.array([0, 1]), np.array([1, 2])
    for base in range(64):
        lvl = O.ladder_level(O.bijective32(mv_u, base))
        if lvl[0] != lvl[1]:
            break
    assert np.all(O.commit_ladder(g, labels, W, maxw, mv_u, mv_t, base))
    acc = U.commit_ladder(g, labels, W, maxw, mv_u, mv_t, base, np.array([3, 0, 0]))
    assert list(acc) == [lvl[0] > lvl[1], lvl[1] > lvl[0]]
    assert np.all(U.commit_ladder(g, labels, W, maxw, mv_u, mv_t, base, np.array([2, 0, 0])))


def test_select_all_keeps_blocked_sources():
    g = _graph("grid")
    k = 4
    mbw, mnw = _weights(g, k)
    part = U.underload_input(g, k, 1, 0.2)
    W = O.block_weights(g, part, k)
    t, key = U.underload_select_all(g, k, part, W, mbw, mnw)
    under = W < mnw
    assert np.all(t[under[part]] == part[under[part]])             # underloaded blocks keep their vertices
    moved = t != part
    assert moved.any() and np.all(under[t[moved]])                 # targets are underloaded
    assert np.all(key[~moved] == O.relative_gain(np.full(int((~moved).sum()), O.INT32_MIN), 1))
