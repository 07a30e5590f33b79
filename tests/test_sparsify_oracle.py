"""CPU properties of the sparsification oracle (tests/sparsify_oracle.py, DESIGN.md §13), and the library's host-side
target formula (kmp_sparsification_target) against hand-computed doubles."""
import numpy as np
import pytest

from kaminpar_b200 import contraction as KC
from kaminpar_b200.graph import random_weights, rmat
from oracle import contraction_oracle as CO
from tests import helpers as H
from tests import sparsify_oracle as S


def _level(seed=1, max_adjwgt=5):
    g = random_weights(rmat(11, 8, seed), seed, max_adjwgt=max_adjwgt)
    cl = (np.arange(g.n) // 3).astype(np.uint32)
    return CO.contract(g.xadj, g.adjncy, g.vwgt, g.adjwgt, cl)


def _edges(d):
    return S.edge_set(d["c_xadj"], d["c_adjncy"], d["c_adjwgt"])


@pytest.mark.parametrize("seed", [0, 3, 2**64 - 1])
def test_symmetric_and_threshold_respected(seed):
    con = _level()
    c_m = len(con["c_adjncy"])
    for target in (c_m // 2, c_m // 5, c_m - 1, 2):
        o = S.sparsify_contracted(con, target, seed)
        kept = _edges(o)
        assert kept == {(v, u, w) for (u, v, w) in kept}  # undirected
        t = o["threshold"]
        before = _edges(con)
        assert {e for e in before if e[2] > t} <= kept
        assert not any(e[2] < t for e in kept)
        larger = c_m - o["smaller"] - o["equal"]
        assert len(kept) == larger + o["equal_kept"] == len(o["c_adjncy"])
        assert o["smaller"] == sum(e[2] < t for e in before) and o["equal"] == sum(e[2] == t for e in before)
        assert o["smaller"] < c_m - target + 1 <= o["smaller"] + o["equal"]  # T is the k-th smallest
        assert np.all(np.diff(o["c_xadj"].astype(np.int64)) >= 0) and int(o["c_xadj"][-1]) == len(kept)


def test_target_below_two_keeps_nothing():
    con = _level()
    for target in (0, 1):
        o = S.sparsify_contracted(con, target, 9)
        assert len(o["c_adjncy"]) == 0 and list(o["c_xadj"]) == [0] * (con["c_n"] + 1)
        assert o["c_n"] == con["c_n"] and np.array_equal(o["c_vwgt"], con["c_vwgt"])


def test_p_one_quirk_on_a_constructed_hash():
    """target == c_m gives p == 1.0, and dice(u, v) < 1.0 fails for h = 2^32 - 1: such an edge is dropped."""
    g = H.from_edges(3, [(0, 1), (1, 2)])
    # the seed that maps the pair (0, 1) to a hash whose low 32 bits are all ones: invert fmix64 on the target
    want = np.uint64(0xFFFFFFFF) | (np.uint64(0x1234) << np.uint64(32))
    key = _unfmix64(want)
    assert int(S.fmix64(np.array([key], np.uint64))[0]) == int(want)
    seed = (int(key) - (1 << 32 | 0)) % 2**64  # key = ((max << 32) | min) + seed with (u, v) = (0, 1)
    assert int(S.dice_hash(0, 1, seed)) == 0xFFFFFFFF and S.dice(0, 1, seed) == 1.0
    con = CO.contract(g.xadj, g.adjncy, None, None, np.arange(3, dtype=np.uint32))
    o = S.sparsify_contracted(con, 4, seed)
    assert o["probability"] == 1.0 and o["equal"] == 4
    assert _edges(o) == {(1, 2, 1), (2, 1, 1)}  # both directions of (0, 1) dropped


def _unfmix64(h):
    """Inverse of murmur3's fmix64 (its two multipliers are odd, the xor-shifts by 33 are self-inverse on 64 bits)."""
    M = 2**64
    inv1 = pow(0xFF51AFD7ED558CCD, -1, M)
    inv2 = pow(0xC4CEB9FE1A85EC53, -1, M)
    x = int(h)
    x ^= x >> 33
    x = (x * inv2) % M
    x ^= x >> 33
    x = (x * inv1) % M
    x ^= x >> 33
    return np.uint64(x)


def test_deterministic_for_a_seed():
    con = _level(2)
    c_m = len(con["c_adjncy"])
    a = S.sparsify_contracted(con, c_m // 3, 42)
    b = S.sparsify_contracted(con, c_m // 3, 42)
    c = S.sparsify_contracted(con, c_m // 3, 43)
    assert CO.equal(a, b)
    assert not CO.equal(a, c)  # the seed changes which edges at T survive


def test_select_matches_sort():
    rng = np.random.default_rng(5)
    for _ in range(20):
        w = rng.integers(-5, 6, rng.integers(2, 200))
        target = int(rng.integers(2, len(w) + 1))
        t, smaller, equal = S.select(w, target)
        assert t == np.sort(w)[len(w) - target]
        assert smaller == np.count_nonzero(w < t) and equal == np.count_nonzero(w == t)


# (prev_m, prev_n, c_n, density, edge) -> hand-computed target
TARGET_CASES = [
    ((1000, 100, 50, 0.5, 0.5), 250),     # density: 0.5 * 1000 / 100 * 50 = 250 < 500
    ((1000, 100, 100, 0.5, 0.5), 500),    # tie: both 500
    ((1001, 100, 100, 0.5, 0.5), 500),    # 500.5 truncated
    ((999, 7, 3, 0.5, 0.5), 214),         # 0.5 * 999 / 7 * 3 = 214.07...
    ((10, 3, 3, 0.5, 2.0), 5),            # density 5.000000000000001 -> 5
    ((10, 3, 6, 1.0, 2.0), 10),           # min(20, 20) >= prev_m: prev_m
    ((100, 10, 5, 0.5, 1e-9), 0),         # edge target 1e-7 truncated to 0
    ((0, 0, 0, 0.5, 0.5), 0),             # nan density: std::min keeps the edge target (0), not below prev_m
    ((4294967295, 4294967295, 4294967295, 0.5, 0.5), 2147483647),
]


@pytest.mark.parametrize("args,want", TARGET_CASES)
def test_target_formula(args, want):
    assert S.sparsification_target(*args) == want
    assert KC.sparsification_target(*args) == want


def test_target_formula_random_against_library():
    rng = np.random.default_rng(8)
    for _ in range(2000):
        prev_n = int(rng.integers(1, 2**31))
        prev_m = int(rng.integers(0, 2**32))
        c_n = int(rng.integers(0, prev_n + 1))
        d, e = (float(x) for x in rng.uniform(0, 1.5, 2))
        assert S.sparsification_target(prev_m, prev_n, c_n, d, e) == KC.sparsification_target(prev_m, prev_n, c_n, d, e)
