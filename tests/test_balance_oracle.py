"""CPU properties of the order-free overload balancer (DESIGN.md §11), on the oracle in tests/balance_oracle.py:
a block that was not overloaded never ends above its maximum, the total overload decreases in every round that
moves a vertex, a feasible input is left untouched, an overloaded block loses less than its overload plus the
heaviest vertex, and the same seed gives the same result.
The key against the reference's own relative_gain.h: tests/test_balance_bridge.py."""
import numpy as np
import pytest

from kaminpar_b200 import lp
from kaminpar_b200.graph import CSRGraph, rmat
from tests import balance_oracle as O
from tests import helpers as H


def _ctx(g, k, eps=0.03):
    ctx = lp.create_default_context()
    ctx.partition.setup(g, k, eps)
    return ctx.partition


def _weighted(g, seed):
    rng = np.random.default_rng(seed)
    return CSRGraph(g.xadj, g.adjncy, rng.integers(1, 9, g.n).astype(np.int32), None)


CASES = [
    ("rmat12", 4, 0.10, (0,)),
    ("rmat12", 16, 0.10, (0,)),
    ("rmat12w", 64, 0.20, (0, 5, 9)),
    ("grid", 2, 0.30, (1,)),
    ("walshaw", 16, 0.10, (0, 1)),
    ("rgg16w", 256, 0.05, (3,)),
]


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


@pytest.mark.parametrize("name,k,share,blocks", CASES)
def test_balance_properties(name, k, share, blocks):
    g = _graph(name)
    p = _ctx(g, k)
    mbw, pbw = p.max_block_weights().astype(np.int64), p.perfectly_balanced_block_weights()
    part = O.overload_input(g, k, 7, share, blocks)
    W0 = O.block_weights(g, part, k)
    over0 = np.maximum(W0 - mbw, 0)
    assert over0.sum() > 0
    res = O.overload_balance(g, k, part, mbw, pbw, seed=1)
    W1 = res["block_weights"].astype(np.int64)
    assert np.array_equal(W1, O.block_weights(g, res["labels"], k))
    assert res["improved"]
    assert np.all(W1[over0 == 0] <= mbw[over0 == 0])            # no block becomes overloaded
    vmax = int(g.vwgt.max()) if g.vwgt is not None else 1
    lost = W0 - W1
    assert np.all(lost[over0 > 0] < over0[over0 > 0] + vmax)     # never more than the overload plus one vertex
    assert np.all(W1[over0 > 0] <= W0[over0 > 0])                # overloaded blocks only lose weight
    assert res["after"] <= res["before"]
    again = O.overload_balance(g, k, part, mbw, pbw, seed=1)
    assert np.array_equal(again["labels"], res["labels"])
    assert again["moved"] == res["moved"]


def test_each_round_lowers_the_overload():
    g = _graph("rmat12w")
    k = 16
    p = _ctx(g, k)
    mbw, pbw = p.max_block_weights().astype(np.int64), p.perfectly_balanced_block_weights()
    part = O.overload_input(g, k, 3, 0.3, (0, 1))
    labels, totals = part.copy(), []
    res = O.overload_balance(g, k, part, mbw, pbw, seed=4)
    # replay round by round: a call capped at r rounds equals the first r rounds of the full call
    for r in range(1, res["rounds"] + 1):
        cap = O.MAX_ROUNDS
        O.MAX_ROUNDS = r
        try:
            totals.append(O.overload_balance(g, k, labels, mbw, pbw, seed=4)["after"])
        finally:
            O.MAX_ROUNDS = cap
    seq = [res["before"]] + totals
    moved = res["moved"]
    for r in range(res["rounds"]):
        assert (seq[r + 1] < seq[r]) == (moved[r] > 0)
        assert seq[r + 1] <= seq[r]


def test_feasible_input_is_untouched():
    g = _graph("walshaw")
    k = 8
    p = _ctx(g, k)
    part = (np.arange(g.n) % k).astype(np.uint32)
    res = O.overload_balance(g, k, part, p.max_block_weights(), p.perfectly_balanced_block_weights())
    assert not res["improved"] and res["rounds"] == 0 and np.array_equal(res["labels"], part)


def test_seed_changes_the_result():
    g = _graph("rmat12")
    k = 16
    p = _ctx(g, k)
    part = O.overload_input(g, k, 7, 0.1)
    a = O.overload_balance(g, k, part, p.max_block_weights(), p.perfectly_balanced_block_weights(), seed=1)
    b = O.overload_balance(g, k, part, p.max_block_weights(), p.perfectly_balanced_block_weights(), seed=2)
    assert not np.array_equal(a["labels"], b["labels"])


def test_perfectly_balanced_block_weight():
    """kaminpar.h:436-438: ceil(unrelaxed max / (1 + inferred epsilon)); uniform k: ceil(total / k) up to rounding."""
    g = _graph("rmat12w")
    for k in (2, 16, 64):
        p = _ctx(g, k)
        total = g.total_node_weight()
        for b in (0, k - 1):
            assert abs(p.perfectly_balanced_block_weight(b) - -(-total // k)) <= 1


def test_desc_bits_order():
    keys = np.array([-np.inf, -3e9, -1.5, -1e-30, 0.0, 1e-30, 1.0, 2.5, 3e9, np.inf], np.float32)
    d = O.desc_bits(keys)
    assert np.all(np.diff(d.astype(np.int64)) < 0)
