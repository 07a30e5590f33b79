"""CPU properties of the overlay oracle (tests/overlay_oracle.py, DESIGN.md §14): the intersection property the
reference asserts after every overlay, the id ranges the rule implies, degenerate inputs, and a hand-computed tree
whose ids change when the tree pairs the clusterings differently."""
import numpy as np
import pytest

from tests import overlay_oracle as O


def overlay_literal(a, b):
    """The rule word for word, O(n^2): for tiny inputs only."""
    n = len(a)
    distinct_a = sorted(set(int(x) for x in a))
    ra = {x: i for i, x in enumerate(distinct_a)}
    out = np.zeros(n, np.uint32)
    for u in range(n):
        index = sum(1 for v in range(n) if ra[int(a[v])] < ra[int(a[u])])
        below = {int(b[v]) for v in range(n) if a[v] == a[u] and b[v] < b[u]}
        out[u] = index + len(below)
    return out


@pytest.mark.parametrize("seed", range(8))
def test_matches_the_literal_rule(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 60))
    a = rng.integers(0, n, n).astype(np.uint32)
    b = rng.integers(0, max(1, n // 3), n).astype(np.uint32)
    assert np.array_equal(O.overlay(a, b), overlay_literal(a, b))


@pytest.mark.parametrize("seed", range(6))
def test_intersection_and_id_ranges(seed):
    rng = np.random.default_rng(100 + seed)
    n = int(rng.integers(2, 5000))
    a = rng.integers(0, int(rng.integers(1, n + 1)), n).astype(np.uint32)
    b = rng.integers(0, n, n).astype(np.uint32)
    out = O.overlay(a, b)
    # out[u] == out[v] iff a[u] == a[v] and b[u] == b[v]: the classes are those of the pair (a, b)
    _, pair_class = np.unique(a.astype(np.int64) * n + b, return_inverse=True)
    _, out_class = np.unique(out, return_inverse=True)
    classes = pair_class.max() + 1
    assert out_class.max() + 1 == classes
    assert np.unique(np.stack([pair_class, out_class]), axis=1).shape[1] == classes  # a bijection between them
    # ids of cluster c of a lie in [index(c), index(c + 1)), all below n
    _, ra = np.unique(a, return_inverse=True)
    index = np.concatenate([[0], np.cumsum(np.bincount(ra))])
    assert (out >= index[ra]).all() and (out < index[ra + 1]).all() and (out < n).all()
    # the smallest b of every a-cluster gets index(c) itself
    for c in np.unique(ra)[:20]:
        members = ra == c
        assert out[members][b[members] == b[members].min()][0] == index[c]


def test_identity_all_equal_and_self():
    n = 37
    ident = np.arange(n, dtype=np.uint32)
    zeros = np.zeros(n, np.uint32)
    rng = np.random.default_rng(3)
    x = rng.integers(0, 9, n).astype(np.uint32)
    assert np.array_equal(O.overlay(ident, x), ident)  # singletons stay singletons, numbered in order
    # b = identity: all singletons, numbered by (a-rank, vertex): the stable argsort of a, inverted
    expect = np.empty(n, np.uint32)
    expect[np.argsort(x, kind="stable")] = np.arange(n)
    assert np.array_equal(O.overlay(x, ident), expect)
    assert np.array_equal(O.overlay(zeros, zeros), zeros)
    # all equal a: the result is the dense rank of b
    assert np.array_equal(O.overlay(zeros, x), np.unique(x, return_inverse=True)[1].astype(np.uint32))
    # a == b: the start of each cluster's block, index(ra(a[u]))
    _, ra = np.unique(x, return_inverse=True)
    index = np.concatenate([[0], np.cumsum(np.bincount(ra))])
    assert np.array_equal(O.overlay(x, x), index[ra].astype(np.uint32))
    assert np.array_equal(O.overlay_tree([x]), x)
    assert len(O.overlay(np.zeros(0, np.uint32), np.zeros(0, np.uint32))) == 0


def test_tree_order_is_pinned():
    """Level 2 pairs C0 with C2 and C1 with C3; pairing C0 with C1 instead gives the same classes, other ids."""
    c = [np.array(x, np.uint32) for x in ([0, 0, 0, 0, 4, 4, 4, 4], [1, 1, 2, 2, 1, 1, 2, 2],
                                          [0, 3, 0, 3, 0, 3, 0, 3], [5, 5, 5, 5, 5, 5, 7, 7])]
    # by hand: overlay(C0, C2) = [0 1 0 1 4 5 4 5], overlay(C1, C3) = [0 0 4 4 0 0 5 5], then their overlay
    assert np.array_equal(O.overlay(c[0], c[2]), [0, 1, 0, 1, 4, 5, 4, 5])
    assert np.array_equal(O.overlay(c[1], c[3]), [0, 0, 4, 4, 0, 0, 5, 5])
    assert np.array_equal(O.overlay_tree(c), [0, 2, 1, 3, 4, 6, 5, 7])
    assert np.array_equal(O.overlay(O.overlay(c[0], c[1]), O.overlay(c[2], c[3])), np.arange(8))


def test_tree_of_eight_matches_nested_pairs():
    rng = np.random.default_rng(8)
    n = 300
    c = [rng.integers(0, 20, n).astype(np.uint32) * 7 for _ in range(8)]
    lvl3 = [O.overlay(c[p], c[4 + p]) for p in range(4)]
    lvl2 = [O.overlay(lvl3[p], lvl3[2 + p]) for p in range(2)]
    assert np.array_equal(O.overlay_tree(c), O.overlay(lvl2[0], lvl2[1]))


def test_refusals():
    with pytest.raises(ValueError):
        O.overlay([0, 3, 1], [0, 0, 0])
    with pytest.raises(ValueError):
        O.overlay([0, 1], [0])
    with pytest.raises(ValueError):
        O.overlay_tree([np.zeros(3, np.uint32)] * 3)
    with pytest.raises(ValueError):
        O.overlay_tree([])
