"""Bridge between the `sync` selection rule (what the GPU computes, T0/T1) and the REFERENCE.

The `seq` oracle's select_best_cluster code (oracle/lp_oracle.cc ClusterPolicy / RefinePolicy) is pinned
bit-for-bit to the unmodified reference by tests/test_oracle_golden.py. Here the SAME code is run on frozen
mid-run states (lpo_seq_select_all) next to the sync rule (lpo_sync_select_all, separate code):

  * a vertex whose set of maximal feasible candidates is a singleton (or empty) has ONE answer; sync must give it;
  * otherwise the reference draws uniformly from that set (lp_clusterer.cc:238-241, lp_refiner.cc:233-236);
    sync's hash-chosen target must be a member of exactly that set.

Same for the favored cluster of the clusterer (lp_clusterer.cc:243-248). Together with T0 (GPU == sync on
frozen state) this ties the GPU's per-vertex decision to the reference's selection rule.
"""
import numpy as np
import pytest

from oracle import bindings as B
from tests.helpers import (LABEL_PATTERNS, LADDER_DEGREES, degree_ladder, frozen_cluster_state, frozen_refine_state,
                           golden_cases, load_case)


def cluster_states(g, mcw):
    """frozen clusterer states: initial singletons, and the sync schedule after 1, 2 and 4 rounds"""
    w = np.ones(g.n, np.int64) if g.vwgt is None else g.vwgt.astype(np.int64)
    yield "init", np.arange(g.n, dtype=np.uint32), w.astype(np.int32)
    for rounds in (1, 2, 4):
        p = B.default_cluster_params()
        p.num_iterations = rounds
        p.two_hop_strategy = 0
        p.isolated_nodes_strategy = 0
        labels = B.oracle_lp_cluster(g, 0, mcw, schedule=B.SYNC, params=p)
        cw = np.bincount(labels, weights=w, minlength=g.n).astype(np.int32)
        yield f"sync{rounds}", labels, cw


def assert_sync_in_reference_ties(g, mode, labels, weights, max_cluster_weight=0, max_weights=None, min_weights=None,
                                  seed=1, iteration=0, tag=()):
    """On one frozen state (graph, labels, weights, limits): the sync rule's target is a member of the reference's
    tie set and equals the reference's choice where that set is a singleton (or empty); the same for the favored
    cluster of the clusterer. Returns (vertices checked, vertices with a unique answer)."""
    lim = dict(max_cluster_weight=max_cluster_weight) if mode == 0 else dict(max_weights=max_weights,
                                                                             min_weights=min_weights)
    tgt, fav = B.oracle_sync_select_all(mode, g, labels, weights, seed=seed, iteration=iteration, **lim)
    fav_chk = np.where(fav == 0xFFFFFFFF, labels, fav).astype(np.uint32) if mode == 0 else None
    r = B.oracle_seq_select_all(mode, g, labels, weights, check_target=tgt, check_favored=fav_chk, **lim)
    bad = np.nonzero(r["check_in_ties"] == 0)[0]
    assert bad.size == 0, (tag, bad[:5], tgt[bad[:5]], r["target"][bad[:5]])
    single = r["num_ties"] <= 1
    assert np.array_equal(tgt[single], r["target"][single]), tag
    if mode == 0:
        # favored: stored for the same vertices, member of the reference's tie set, equal when unique
        assert np.array_equal(fav == 0xFFFFFFFF, r["favored"] == 0xFFFFFFFF), tag
        assert (r["check_fav_in_ties"] == 1).all(), tag
        fs = (r["num_fav_ties"] <= 1) & (fav != 0xFFFFFFFF)
        assert np.array_equal(fav[fs], r["favored"][fs]), tag
    return g.n, int(single.sum())


@pytest.mark.parametrize("case", golden_cases())
def test_sync_cluster_selection_is_the_references(case):
    g, d = load_case(case)
    if g.n == 0:
        pytest.skip("empty")
    k = int(d["k"][0]) if "k" in d else 8
    mcw = max(int(B.oracle_max_cluster_weight(g, k)), 1)
    checked = singles = 0
    for name, labels, cw in cluster_states(g, mcw):
        for it in (0, 3):
            c, s = assert_sync_in_reference_ties(g, 0, labels, cw, max_cluster_weight=mcw, iteration=it,
                                                 tag=(case, name, it))
            checked += c
            singles += s
    assert checked > 0 and singles > 0


@pytest.mark.parametrize("case", golden_cases())
def test_sync_refine_selection_is_the_references(case):
    g, d = load_case(case)
    if g.n == 0:
        pytest.skip("empty")
    w = np.ones(g.n, np.int64) if g.vwgt is None else g.vwgt.astype(np.int64)
    for k in (2, 4, 16):
        if k > g.n:
            continue
        rng = np.random.default_rng(k)
        part = rng.integers(0, k, g.n).astype(np.uint32)
        mbw = B.oracle_max_block_weights(g, k)
        states = [("random", part)]
        p = B.default_refine_params()
        p.num_iterations = 2
        part2, _ = B.oracle_lp_refine(g, 0, k, mbw, part, schedule=B.SYNC, params=p)
        states.append(("sync2", part2))
        for name, lab in states:
            bw = np.bincount(lab, weights=w, minlength=k).astype(np.int32)
            for min_w in (None, np.full(k, int(bw.min()), np.int32)):
                assert_sync_in_reference_ties(g, 1, lab, bw, max_weights=mbw, min_weights=min_w, seed=2, iteration=1,
                                              tag=(case, k, name))


# ---- the same on the states of the kernel-edge suite (tests/test_gpu_edges.py): degree ladders with labels that
# are all one, all distinct, exactly tied or hash-colliding, and weights exactly at a limit or one above it
LADDERS = {
    "dense_w": (lambda: degree_ladder(sorted(LADDER_DEGREES), 256, weighted=True, multi=True, seed=2), 256),
    "wide_unit": (lambda: degree_ladder(sorted(LADDER_DEGREES), 18436, seed=3), 18436),
}


@pytest.mark.parametrize("pattern", LABEL_PATTERNS)
@pytest.mark.parametrize("name", sorted(LADDERS))
def test_sync_selection_is_the_references_at_the_kernel_edges(name, pattern):
    make, pool = LADDERS[name]
    g = make()
    rng = np.random.default_rng(len(name) * 10 + LABEL_PATTERNS.index(pattern))
    singles = 0
    for nl in (513, 32769) if g.n < 512 else (g.n, 1 << 20):
        for feas in ("lo", "hi", "mix"):
            labels, weights = frozen_cluster_state(g, pool, nl, pattern, feas, rng)
            singles += assert_sync_in_reference_ties(g, 0, labels, weights, max_cluster_weight=1000,
                                                     tag=(name, pattern, nl, feas))[1]
        cw = 1 if g.vwgt is None else int(g.vwgt[pool])
        for regime in ("fit", "over"):
            labels, bw, maxw, own = frozen_refine_state(g, pool, nl, pattern, regime, "mix", rng)
            for d in (None, 0, 1):
                mn = None
                if d is not None:
                    mn = np.zeros(nl, np.int32)
                    mn[own] = int(bw[own]) - cw + d
                singles += assert_sync_in_reference_ties(g, 1, labels, bw, max_weights=maxw, min_weights=mn,
                                                         tag=(name, pattern, nl, regime, d))[1]
    assert singles > 0
