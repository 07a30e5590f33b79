"""CPU oracle of the order-free overload balancer (DESIGN.md §11), in NumPy.

It is the specification the device code (kaminpar_b200/csrc/kmp_balance.cuh) is tested against bit for bit:
the same hashes (lp_device.cuh), the same float relative gain (refinement/balancer/relative_gain.h), the same
one-pass commit ladder as the LP refiner's sync commit (oracle/lp_oracle.cc sync_commit, commit_refine_fused).
"""
import numpy as np

MASK32 = 0xFFFFFFFF
MASK64 = (1 << 64) - 1
INT32_MIN = -(1 << 31)
SALT_BAL_TIE, SALT_BAL_DRAW, SALT_BAL_COMMIT = 5, 6, 7
MAX_ROUNDS = 64  # KMP_BALANCE_MAX_ROUNDS
LADDER_LEVELS = 16


def _splitmix64(x):
    x = (x + 0x9E3779B97F4A7C15) & MASK64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & MASK64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & MASK64
    return x ^ (x >> 31)


def sync_base(seed, call, it, salt):
    a = _splitmix64(((seed & MASK32) << 32) | (call & MASK32))
    b = _splitmix64(((it & MASK32) << 32) | salt)
    return _splitmix64(a ^ b) >> 32


def lowbias32(x):
    x = np.asarray(x, np.uint64) & MASK32
    x ^= x >> 16
    x = (x * 0x7FEB352D) & MASK32
    x ^= x >> 15
    x = (x * 0x846CA68B) & MASK32
    x ^= x >> 16
    return x


def tie_hash(base, u, c):
    u = np.asarray(u, np.uint64)
    c = np.asarray(c, np.uint64)
    return lowbias32(((u * 0x9E3779B1) & MASK32) ^ ((c * 0x85EBCA77) & MASK32) ^ np.uint64(base))


def draw_hash(base, u):
    u = np.asarray(u, np.uint64)
    return lowbias32(((u * 0x9E3779B1) & MASK32) ^ np.uint64(base))


def bijective32(x, base):
    x = (np.asarray(x, np.uint64) ^ np.uint64(base)) & MASK32
    x = (x * 0x9E3779B1) & MASK32
    x ^= x >> 15
    x = (x * 0x85EBCA77) & MASK32
    x ^= x >> 13
    x = (x * 0xC2B2AE3D) & MASK32
    x ^= x >> 16
    return x


def ladder_level(prio):
    prio = np.asarray(prio, np.uint64)
    lvl = np.zeros(prio.shape, np.int64)
    for j in range(1, LADDER_LEVELS):  # level >= j  <=>  prio < 2^(32 - j)
        lvl += prio < (1 << (32 - j))
    return lvl


def relative_gain(gain, weight):
    """compute_relative_gain: float(gain) * w if gain > 0, else float(gain) / w, in float32."""
    g = np.asarray(gain, np.int64).astype(np.float32)
    w = np.asarray(weight, np.int64).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(np.asarray(gain) > 0, g * w, g / w).astype(np.float32)


def desc_bits(key):
    b = np.asarray(key, np.float32).view(np.uint32).astype(np.uint64)
    ordered = np.where(b >> 31 != 0, b ^ 0xFFFFFFFF, b ^ 0x80000000)
    return (~ordered) & MASK32


def _node_weights(g):
    return np.ones(g.n, np.int64) if g.vwgt is None else g.vwgt.astype(np.int64)


def block_weights(g, labels, k):
    return np.bincount(labels, weights=_node_weights(g), minlength=k).astype(np.int64)


def best_targets(g, k, labels, W, maxw, base_tie, verts):
    """(target, gain, key) of the vertices `verts`: the best adjacent block c != own with W[c] + w(u) <= max[c] by
    (gain desc, tie_hash asc, c asc); none: own block, gain INT32_MIN."""
    verts = np.asarray(verts, np.int64)
    labels = labels.astype(np.int64)
    vw = _node_weights(g)
    deg = (g.xadj[verts + 1].astype(np.int64) - g.xadj[verts])
    idx = np.repeat(np.arange(len(verts)), deg)
    starts = np.repeat(g.xadj[verts].astype(np.int64) - np.concatenate(([0], np.cumsum(deg)[:-1])), deg)
    e = starts + np.arange(len(idx))
    c = labels[g.adjncy[e].astype(np.int64)]
    w = np.ones(len(e), np.int64) if g.adjwgt is None else g.adjwgt[e].astype(np.int64)
    own = labels[verts]
    conn_own = np.bincount(idx, weights=np.where(c == own[idx], w, 0), minlength=len(verts)).astype(np.int64)
    pair = idx * np.int64(k) + c
    uniq, inv = np.unique(pair, return_inverse=True)
    conn = np.bincount(inv, weights=w).astype(np.int64)
    pi, pc = uniq // k, uniq % k
    u = verts[pi]
    ok = (pc != own[pi]) & (W[pc] + vw[u] <= maxw[pc])
    pi, pc, u, conn = pi[ok], pc[ok], u[ok], conn[ok]
    gain = (conn - conn_own[pi]).astype(np.int32).astype(np.int64)  # EdgeWeight arithmetic
    h = tie_hash(base_tie, u, pc).astype(np.int64)
    order = np.lexsort((pc, h, -gain, pi))
    pi, pc, gain = pi[order], pc[order], gain[order]
    first = np.ones(len(pi), bool)
    first[1:] = pi[1:] != pi[:-1]
    target = own.copy()
    best_gain = np.full(len(verts), INT32_MIN, np.int64)
    target[pi[first]] = pc[first]
    best_gain[pi[first]] = gain[first]
    return target, best_gain, relative_gain(best_gain, vw[verts])


def select_all(g, k, labels, W, maxw, seed=0, call=0, rnd=0):
    """kmp_balance_select_all."""
    W = np.asarray(W, np.int64)
    maxw = np.asarray(maxw, np.int64)
    t, _, key = best_targets(g, k, np.asarray(labels), W, maxw, sync_base(seed, call, rnd, SALT_BAL_TIE), np.arange(g.n))
    return t.astype(np.uint32), key


def commit_ladder(g, labels, W, maxw, mv_u, mv_t, base_commit):
    """One pass of the refiner's ladder commit (no departure credit, no minimum weights)."""
    vw = _node_weights(g)
    lvl = ladder_level(bijective32(mv_u, base_commit))
    k = len(W)
    hist = np.zeros((k, LADDER_LEVELS), np.int64)
    np.add.at(hist, (mv_t, lvl), vw[mv_u])
    cum = np.cumsum(hist[:, ::-1], axis=1)[:, ::-1]  # cum[t][j] = weight at level >= j
    fits = W[:, None] + cum <= maxw[:, None]
    jmin = np.where(fits.any(axis=1), fits.argmax(axis=1), LADDER_LEVELS)
    return lvl >= jmin[mv_t]


def overload_balance(g, k, labels, maxw, pbw, seed=0, call=0):
    """kmp_overload_balance. Returns dict(labels, block_weights, improved, moved, before, after, rounds)."""
    labels = np.asarray(labels).astype(np.int64).copy()
    maxw = np.asarray(maxw, np.int64)
    pbw = np.asarray(pbw, np.int64)
    vw = _node_weights(g)
    W = block_weights(g, labels, k)
    before = int(np.maximum(W - maxw, 0).sum())
    moved = []
    prev = None
    r = 0
    while True:
        over = np.maximum(W - maxw, 0)
        total = int(over.sum())
        if total == 0 or (r > 0 and prev == 0) or r == MAX_ROUNDS:  # prev: proposals of the last round
            break
        cand = np.nonzero(over[labels] > 0)[0]
        tgt, _, key = best_targets(g, k, labels, W, maxw, sync_base(seed, call, r, SALT_BAL_TIE), cand)
        blk = labels[cand]
        order = np.lexsort((cand, desc_bits(key), blk))
        cs, bs, ts = cand[order], blk[order], tgt[order]
        wts = vw[cs]
        incl = np.cumsum(wts)
        seg_start = np.ones(len(cs), bool)
        seg_start[1:] = bs[1:] != bs[:-1]
        base = np.maximum.accumulate(np.where(seg_start, incl - wts, 0))
        prefix = incl - wts - base
        sel = prefix < over[bs]
        cs, bs, ts = cs[sel], bs[sel], ts[sel]
        under = np.nonzero(W < pbw)[0]
        internal = np.nonzero(ts == bs)[0]
        if len(under) > 0 and len(internal) > 0:
            # the first underloaded block with room, cyclically from a hashed start
            start = draw_hash(sync_base(seed, call, r, SALT_BAL_DRAW), cs[internal]).astype(np.int64) % len(under)
            todo = np.ones(len(internal), bool)
            for q in range(len(under)):
                c = under[(start + q) % len(under)]
                hit = todo & (W[c] + vw[cs[internal]] <= maxw[c])
                ts[internal[hit]] = c[hit]
                todo &= ~hit
                if not todo.any():
                    break
        prop = ts != bs
        mv_u, mv_t = cs[prop], ts[prop]
        prev = len(mv_u)
        acc = commit_ladder(g, labels, W, maxw, mv_u, mv_t, sync_base(seed, call, r, SALT_BAL_COMMIT))
        mu, mt = mv_u[acc], mv_t[acc]
        np.add.at(W, labels[mu], -vw[mu])
        np.add.at(W, mt, vw[mu])
        labels[mu] = mt
        moved.append(int(len(mu)))
        r += 1
    return dict(labels=labels.astype(np.uint32), block_weights=W.astype(np.int32), improved=before > 0, moved=moved,
                before=before, after=int(np.maximum(W - maxw, 0).sum()), rounds=r)


def edge_cut(g, labels):
    src = np.repeat(np.arange(g.n), np.diff(g.xadj.astype(np.int64)))
    w = np.ones(len(src), np.int64) if g.adjwgt is None else g.adjwgt.astype(np.int64)
    lab = np.asarray(labels).astype(np.int64)
    return int(w[lab[src] != lab[g.adjncy.astype(np.int64)]].sum()) // 2


def overload_input(g, k, seed, share, blocks=(0,)):
    """A hashed k-way partition with a seeded share of the vertices moved into `blocks`."""
    rng = np.random.default_rng(seed)
    part = rng.integers(0, k, g.n).astype(np.uint32)
    pick = rng.random(g.n) < share
    part[pick] = np.asarray(blocks, np.uint32)[rng.integers(0, len(blocks), int(pick.sum()))]
    return part
