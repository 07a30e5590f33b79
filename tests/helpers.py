"""Shared test helpers (graph families mirror tests/shm/graph_factories.h:16-183 of the reference)."""
import glob
import os

import numpy as np

from kaminpar_b200.graph import CSRGraph

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_graph(name: str) -> CSRGraph:
    d = np.load(os.path.join(GOLDEN, f"graph_{name}.npz"))
    return CSRGraph(d["xadj"], d["adjncy"], d["vwgt"] if "vwgt" in d else None, d["adjwgt"] if "adjwgt" in d else None)


def golden_cases():
    return sorted(os.path.basename(p)[4:-4] for p in glob.glob(os.path.join(GOLDEN, "ref_*.npz")))


def load_case(name: str):
    d = np.load(os.path.join(GOLDEN, f"ref_{name}.npz"))
    g = CSRGraph(d["xadj"], d["adjncy"], d["vwgt"] if "vwgt" in d else None, d["adjwgt"] if "adjwgt" in d else None,
                 sorted=bool(d["sorted"][0]), buckets=d["buckets"] if "buckets" in d else None)
    return g, d


def from_edges(n, edges, vwgt=None, ew=None) -> CSRGraph:
    """Undirected edge list -> symmetric CSR (tests/shm/graph_builder.h)."""
    adj = [[] for _ in range(n)]
    wts = [[] for _ in range(n)]
    for i, (u, v) in enumerate(edges):
        w = 1 if ew is None else ew[i]
        adj[u].append(v)
        wts[u].append(w)
        adj[v].append(u)
        wts[v].append(w)
    xadj = np.zeros(n + 1, np.uint32)
    for u in range(n):
        xadj[u + 1] = xadj[u] + len(adj[u])
    adjncy = np.array([v for a in adj for v in a], np.uint32)
    adjwgt = None if ew is None else np.array([w for a in wts for w in a], np.int32)
    return CSRGraph(xadj, adjncy, None if vwgt is None else np.asarray(vwgt, np.int32), adjwgt)


def empty_graph(n=0):
    return CSRGraph(np.zeros(n + 1, np.uint32), np.zeros(0, np.uint32))


def path_graph(n):
    return from_edges(n, [(i, i + 1) for i in range(n - 1)])


def star_graph(leaves):
    return from_edges(leaves + 1, [(0, i + 1) for i in range(leaves)])


def complete_graph(n):
    return from_edges(n, [(i, j) for i in range(n) for j in range(i + 1, n)])


def complete_bipartite(a, b):
    return from_edges(a + b, [(i, a + j) for i in range(a) for j in range(b)])


def grid2d(rows, cols):
    e = []
    for r in range(rows):
        for c in range(cols):
            u = r * cols + c
            if c + 1 < cols:
                e.append((u, u + 1))
            if r + 1 < rows:
                e.append((u, u + cols))
    return from_edges(rows * cols, e)


def matching_graph(pairs):
    return from_edges(2 * pairs, [(2 * i, 2 * i + 1) for i in range(pairs)])


def big_star(n: int) -> CSRGraph:
    xadj = np.zeros(n + 1, np.int64)
    xadj[1] = n - 1
    xadj[2:] = n - 1 + np.arange(1, n)
    adj = np.concatenate([np.arange(1, n), np.zeros(n - 1, np.int64)])
    return CSRGraph(xadj.astype(np.uint32), adj.astype(np.uint32))


# ------------------------------------------------------------------------------------------------
# Inputs at the edges of the sweep kernels (kaminpar_b200/csrc/kmp_lp.cu tier_of, lp_sweep.cuh)
# ------------------------------------------------------------------------------------------------
HUB_MIN_DEGREE_W, HUB_MIN_DEGREE_UNIT = 8192, 16384  # kHubMinDegree / kHubMinDegreeUnit

# both sides of every tier boundary: 7|8 (tier 0|1), 16|17 (1|2), 31|32 (2|3), 255|256 (3|4), 1023|1024 (4|5),
# 4095|4096 (5|6), 8191|8192 (6|hub with edge weights), 16383|16384 (6|hub with unit weights)
TIER_EDGE_DEGREES = (7, 8, 16, 17, 31, 32, 255, 256, 1023, 1024, 4095, 4096, 8191, 8192, 16383, 16384)
# hub degrees ending 1 before, at and 1 after a multiple of the 256-edge slice (65 * 256) and of the 2048-edge chunk
# (9 * 2048)
HUB_CHUNK_DEGREES = (16639, 16640, 16641, 18431, 18432, 18433)
LADDER_DEGREES = TIER_EDGE_DEGREES + HUB_CHUNK_DEGREES


def tier_of(d, weighted):
    """Kernel tier of a vertex of degree d >= 1 (kmp_lp.cu tier_of)."""
    hub = HUB_MIN_DEGREE_W if weighted else HUB_MIN_DEGREE_UNIT
    return 0 if d < 8 else 1 if d <= 16 else 2 if d < 32 else 3 if d < 256 else 4 if d < 1024 else \
        5 if d < 4096 else 6 if d < hub else 7


def tiers_present(g: CSRGraph, large_degree_threshold=0xFFFFFFFF):
    d = g.degrees()
    d = d[(d > 0) & (d < large_degree_threshold)]
    return sorted({tier_of(int(x), g.adjwgt is not None) for x in np.unique(d)})


def degree_ladder(degrees, n, weighted=False, multi=False, seed=0, m_mod4=None, centre_weight=2):
    """One centre vertex per requested degree, its neighbours drawn from a pool of n vertices.

    Ids: the pool is 0..n-1, the centres follow in the order of `degrees` (pass them ascending and the largest
    hub's adjacency is the tail of adjncy). A centre's neighbours come in pairs (2i, 2i+1) of pool vertices with
    equal edge weights, so a labelling that tells even from odd pool vertices gives every even-degree centre an
    exact tie. multi=False: distinct neighbours (needs n > max degree); multi=True: the pairs are drawn with
    replacement (parallel edges), so a hub can live in a graph small enough for direct-indexed rating tables.
    m_mod4: append single self-loop entries to pool vertices until m % 4 == m_mod4 (a symmetric graph alone has
    an even m). weighted: edge weights 1..7, pool vertex weights 1..4 and `centre_weight` on every centre."""
    rng = np.random.default_rng(seed)
    pairs = n // 2
    src, dst, ew = [], [], []
    for i, d in enumerate(degrees):
        c = n + i
        np_ = (d + 1) // 2
        if multi:
            pi = rng.integers(0, pairs, np_)
        else:
            assert np_ <= pairs, "degree_ladder(multi=False) needs n > degree"
            pi = rng.choice(pairs, np_, replace=False)
        nb = np.stack([2 * pi, 2 * pi + 1], axis=1).reshape(-1)[:d]
        w = np.repeat(rng.integers(1, 8, np_), 2)[:d]
        src.append(np.full(d, c, np.int64))
        dst.append(nb.astype(np.int64))
        ew.append(w)
    src = np.concatenate(src)
    dst = np.concatenate(dst)
    ew = np.concatenate(ew)
    u = np.concatenate([src, dst])
    v = np.concatenate([dst, src])
    w = np.concatenate([ew, ew])
    if m_mod4 is not None:
        loops = (m_mod4 - len(u)) % 4
        u = np.concatenate([u, np.arange(loops)])
        v = np.concatenate([v, np.arange(loops)])
        w = np.concatenate([w, np.ones(loops, np.int64)])
    order = np.argsort(u, kind="stable")  # keeps each centre's neighbour order
    total = n + len(degrees)
    xadj = np.zeros(total + 1, np.int64)
    xadj[1:] = np.cumsum(np.bincount(u, minlength=total))
    vwgt = adjwgt = None
    if weighted:
        vwgt = np.concatenate([rng.integers(1, 5, n), np.full(len(degrees), centre_weight)])
        adjwgt = w[order]
    return CSRGraph(xadj.astype(np.uint32), v[order].astype(np.uint32), vwgt, adjwgt)


def colliding_labels(count, mask_bits, limit, exclude=()):
    """`count` ids v < limit (ascending) whose lowbias32(v) has all of its low `mask_bits` bits set: they share the
    last slot of every open-addressing table of <= 2^mask_bits slots keyed by lowbias32 (probe chains wrap
    around at once), the last hub bucket of every vertex with <= 2^mask_bits buckets, and the hash-class bits
    (lowbias32 >> pbits) of the hub tier's multi-pass selection up to bit mask_bits - 1."""
    from tests.test_hash_bijection import lowbias32

    mask = np.uint32((1 << mask_bits) - 1)
    v = np.arange(limit, dtype=np.uint32)
    ids = v[(lowbias32(v) & mask) == mask]
    if len(exclude):
        ids = np.setdiff1d(ids, np.asarray(exclude, np.uint32))
    if count is None:
        return ids
    assert len(ids) >= count, f"only {len(ids)} colliding ids below {limit}"
    return ids[:count]


LABEL_PATTERNS = ("one", "distinct", "tie", "collide")
MAG_LIMIT = (1 << 31) - 1 - (1 << 25)  # a weight limit near 2^31 that leaves room for one 2^24-sized vertex on top


def collide_bits(num_labels):
    """Low hash bits the colliding labels share: >= 32 of them below num_labels; 10 bits (> 640 labels in one
    hub bucket, hash classes shared up to K = 16) once num_labels >= 2^20."""
    return 10 if num_labels >= 1 << 20 else max(4, int(np.log2(num_labels)) - 5)


def pattern_labels(n, npool, num_labels, pattern, rng, centre_labels=None):
    """Labels in [0, num_labels) for a degree ladder: the centres (ids npool..n-1) get `centre_labels` or distinct
    labels of their own; the pool's labels follow `pattern`:
      one      : a single label (a centre's top rating is its whole degree: at a tier's largest degree the
                 16-bit counters of tier 6 hold their largest value),
      distinct : all different (with multi=False ladders: a table full of rating-1 ties, decided by the tie hash),
      tie      : even pool vertices one label, odd ones another (every even-degree centre: an exact tie),
      collide  : labels whose lowbias32 share the low collide_bits(num_labels) bits (probe chains that wrap
                 around, one overflowing hub bucket, multi-pass hub selection)."""
    coll = colliding_labels(None, collide_bits(num_labels), num_labels) if pattern == "collide" else None
    free = np.arange(num_labels, dtype=np.int64)
    if coll is not None:
        free = np.setdiff1d(free, coll)
    if centre_labels is not None:  # one shared label (the refiner's block O): not a candidate of the centres
        free = free[free != centre_labels]
        coll = None if coll is None else coll[coll != centre_labels]
    nc = n - npool
    pick = rng.choice(free, size=min(len(free), n), replace=False)
    labels = np.empty(n, np.int64)
    labels[npool:] = pick[:nc] if centre_labels is None else centre_labels
    rest = pick[nc:]
    if pattern == "one":
        labels[:npool] = rest[0]
    elif pattern == "distinct":
        labels[:npool] = rest[np.arange(npool) % len(rest)]
    elif pattern == "tie":
        labels[:npool] = np.where(np.arange(npool) % 2 == 0, rest[0], rest[1])
    else:
        labels[:npool] = coll[np.arange(npool) % len(coll)]
    return labels.astype(np.uint32)


def frozen_cluster_state(g, npool, num_labels, pattern, feas, rng, mcw=1000):
    """A clusterer state on a degree ladder whose pool labels are the centres' candidates. Every candidate's
    cluster weight is exactly at the limit for a centre (weight + w(centre) == mcw: feas "lo"), one above it ("hi"),
    or either at random ("mix"); a centre's own cluster holds only itself (so it stores a favored cluster).
    Returns (labels, weights[num_labels])."""
    labels = pattern_labels(g.n, npool, num_labels, pattern, rng)
    cw = 1 if g.vwgt is None else int(g.vwgt[npool])
    weights = rng.integers(1, max(2, min(mcw // 2, 1 << 24)), num_labels).astype(np.int64)
    cand = np.unique(labels[:npool])
    bump = {"lo": 0, "hi": 1}.get(feas)
    weights[cand] = mcw - cw + (rng.integers(0, 2, len(cand)) if bump is None else bump)
    weights[labels[npool:]] = cw
    return labels, weights.astype(np.int32)


def frozen_refine_state(g, npool, k, pattern, regime, feas, rng, limit=10000):
    """A refiner state on a degree ladder: all centres in one block O, the pool's blocks follow `pattern`.
    regime "fit": O is light, a candidate block c fits a centre exactly (bw[c] + w(u) == max: feas "lo") or misses
    by one ("hi"); regime "over": O is overloaded by 7 and a candidate is overloaded by 6 ("lo": overload(c) ==
    overload(O) - 1, feasible) or 7 ("hi": equal, infeasible); "mix" draws either per block.
    Returns (labels, block weights, max block weights, O)."""
    own = int(rng.integers(0, k))
    labels = pattern_labels(g.n, npool, k, pattern, rng, centre_labels=own)
    cw = 1 if g.vwgt is None else int(g.vwgt[npool])
    maxw = np.full(k, limit, np.int64)
    bw = rng.integers(0, limit // 2, k).astype(np.int64)
    cand = np.unique(labels[:npool])
    bump = {"lo": 0, "hi": 1}.get(feas)
    b = rng.integers(0, 2, len(cand)) if bump is None else bump
    if regime == "fit":
        bw[own] = limit // 2
        bw[cand] = limit - cw + b
    else:
        bw[own] = limit + 7
        bw[cand] = limit + 6 + b
    return labels, bw.astype(np.int32), maxw.astype(np.int32), own


def magnified(g, npool, seed=0):
    """The same ladder with vertex weights near 2^24: 2^24 + 5 on every centre, [2^24 - 2^20, 2^24) on the pool
    (112 pool vertices and 16 centres: total weight in (2^31 - 2^27, 2^31 - 1))."""
    rng = np.random.default_rng(seed)
    vw = np.concatenate([rng.integers((1 << 24) - (1 << 20), 1 << 24, npool), np.full(g.n - npool, (1 << 24) + 5)])
    return CSRGraph(g.xadj, g.adjncy, vw.astype(np.int32), g.adjwgt)


def block_weights(g: CSRGraph, part, k):
    w = np.ones(g.n, np.int64) if g.vwgt is None else g.vwgt.astype(np.int64)
    return np.bincount(part, weights=w, minlength=k).astype(np.int64)


def cluster_weights_ok(g: CSRGraph, clustering, max_w):
    w = np.ones(g.n, np.int64) if g.vwgt is None else g.vwgt.astype(np.int64)
    cw = np.bincount(clustering, weights=w, minlength=g.n)
    mx = max(int(max_w), int(w.max()) if g.n else 0)
    return bool((cw <= mx).all())
