"""CPU oracle of the order-free underload balancer (DESIGN.md §12), in NumPy.

It is the specification the device code (kaminpar_b200/csrc/kmp_underload.cuh) is tested against bit for bit. It
builds on the overload balancer's oracle (tests/balance_oracle.py): the same hashes, the same float relative gain,
the same target evaluation restricted to the underloaded blocks, and the same one-pass commit ladder followed by
the source side that commit_refine_fused (lp_commit.cuh) applies with minimum block weights.
"""
import math

import numpy as np

from tests import balance_oracle as O

SALT_UBAL_TIE, SALT_UBAL_COMMIT = 8, 9
_NO_ROOM = -(1 << 62)  # a maximum no block weight plus a vertex weight stays at or below


def min_block_weights(pbw, min_epsilon):
    """PartitionContext::setup_min_block_weights(min_epsilon) (context.cc:72-81): ceil((1 - eps) * perfectly)."""
    return np.array([math.ceil((1 - min_epsilon) * int(w)) for w in pbw], np.int32)


def total_underload(W, minw):
    return int(np.maximum(np.asarray(minw, np.int64) - np.asarray(W, np.int64), 0).sum())


def _node_weights(g):
    return np.ones(g.n, np.int64) if g.vwgt is None else g.vwgt.astype(np.int64)


def best_targets(g, k, labels, W, maxw, base_tie, verts, tmask):
    """balance_oracle.best_targets with the targets restricted to the blocks with tmask[c]: a block outside the mask
    gets a maximum nothing fits under, which is the device's mask test (bal_offer) in the oracle's terms."""
    masked_max = np.where(np.asarray(tmask, bool), np.asarray(maxw, np.int64), _NO_ROOM)
    return O.best_targets(g, k, labels, W, masked_max, base_tie, verts)


def commit_ladder(g, labels, W, maxw, mv_u, mv_t, base_commit, minw):
    """One pass of the refiner's ladder commit with minimum weights: balance_oracle.commit_ladder's target side,
    then the source side of commit_refine_fused (lp_commit.cuh): of the moves the target side accepted, a source b
    keeps those at levels >= the lowest level j at which W[b] minus the accepted departures at levels >= j stays
    >= minw[b]."""
    acc = O.commit_ladder(g, labels, W, maxw, mv_u, mv_t, base_commit)
    vw = _node_weights(g)
    lvl = O.ladder_level(O.bijective32(mv_u, base_commit))
    k = len(W)
    src = np.asarray(labels, np.int64)[mv_u]
    hist = np.zeros((k, O.LADDER_LEVELS), np.int64)
    np.add.at(hist, (src[acc], lvl[acc]), vw[mv_u][acc])
    out = np.cumsum(hist[:, ::-1], axis=1)[:, ::-1]  # out[b][j] = accepted departures at level >= j
    ok = np.asarray(W, np.int64)[:, None] - out >= np.asarray(minw, np.int64)[:, None]
    ojmin = np.where(ok.any(axis=1), ok.argmax(axis=1), O.LADDER_LEVELS)
    return acc & (lvl >= ojmin[src])


def _movable_from(g, labels, W, minw, under):
    """underload_balancer.cc:241-244: the own block is not underloaded and stays >= its minimum without u."""
    return ~under[labels] & (W[labels] - _node_weights(g) >= minw[labels])


def underload_select_all(g, k, labels, W, maxw, minw, seed=0, call=0, rnd=0):
    """kmp_underload_select_all: target and key of every vertex; a vertex that may not leave its block, or has no
    adjacent underloaded block with room, keeps its block (key from gain INT32_MIN)."""
    labels = np.asarray(labels).astype(np.int64)
    W = np.asarray(W, np.int64)
    maxw = np.asarray(maxw, np.int64)
    minw = np.asarray(minw, np.int64)
    under = W < minw
    t, _, key = best_targets(g, k, labels, W, maxw, O.sync_base(seed, call, rnd, SALT_UBAL_TIE), np.arange(g.n),
                             under)
    keep = ~_movable_from(g, labels, W, minw, under)
    t[keep] = labels[keep]
    key[keep] = O.relative_gain(np.full(int(keep.sum()), O.INT32_MIN), _node_weights(g)[keep])
    return t.astype(np.uint32), key


def underload_balance(g, k, labels, maxw, minw, seed=0, call=0):
    """kmp_underload_balance. Returns dict(labels, block_weights, improved, moved, before, after, rounds,
    underload) with underload[r] the total underload at the start of round r (and at the end)."""
    labels = np.asarray(labels).astype(np.int64).copy()
    maxw = np.asarray(maxw, np.int64)
    vw = _node_weights(g)
    W = O.block_weights(g, labels, k)
    if minw is None:  # no minimum weights: nothing to do
        return dict(labels=labels.astype(np.uint32), block_weights=W.astype(np.int32), improved=False, moved=[],
                    before=0, after=0, rounds=0, underload=[0])
    minw = np.asarray(minw, np.int64)
    before = total_underload(W, minw)
    moved, trace = [], []
    prev = None
    r = 0
    while True:
        deficit = np.maximum(minw - W, 0)
        total = int(deficit.sum())
        trace.append(total)
        if total == 0 or (r > 0 and prev == 0) or r == O.MAX_ROUNDS:  # prev: proposals of the last round
            break
        under = deficit > 0
        cand = np.nonzero(_movable_from(g, labels, W, minw, under))[0]
        tgt, _, key = best_targets(g, k, labels, W, maxw, O.sync_base(seed, call, r, SALT_UBAL_TIE), cand, under)
        has = tgt != labels[cand]
        cs, ts, ks = cand[has], tgt[has], key[has]
        order = np.lexsort((cs, O.desc_bits(ks), ts))  # per target: key desc, vertex id asc
        cs, ts = cs[order], ts[order]
        wts = vw[cs]
        incl = np.cumsum(wts)
        seg_start = np.ones(len(cs), bool)
        seg_start[1:] = ts[1:] != ts[:-1]
        base = np.maximum.accumulate(np.where(seg_start, incl - wts, 0))
        sel = incl - wts - base < deficit[ts]
        mv_u, mv_t = cs[sel], ts[sel]
        prev = len(mv_u)
        acc = commit_ladder(g, labels, W, maxw, mv_u, mv_t, O.sync_base(seed, call, r, SALT_UBAL_COMMIT), minw)
        mu, mt = mv_u[acc], mv_t[acc]
        np.add.at(W, labels[mu], -vw[mu])
        np.add.at(W, mt, vw[mu])
        labels[mu] = mt
        moved.append(int(len(mu)))
        r += 1
    return dict(labels=labels.astype(np.uint32), block_weights=W.astype(np.int32), improved=before > 0, moved=moved,
                before=before, after=total_underload(W, minw), rounds=r, underload=trace)


def underload_input(g, k, seed, share, block=0):
    """A hashed k-way partition with a seeded share of `block`'s vertices moved to hashed other blocks."""
    rng = np.random.default_rng(seed)
    part = rng.integers(0, k, g.n).astype(np.uint32)
    pick = np.flatnonzero((part == block) & (rng.random(g.n) < share))
    other = (block + 1 + (O.draw_hash(seed, pick) % max(k - 1, 1)).astype(np.int64)) % k
    part[pick] = other.astype(np.uint32)
    return part
