"""CPU oracle of threshold edge sparsification (DESIGN.md §13) -- TEST INFRASTRUCTURE ONLY.

NumPy restatement of SparsificationClusterCoarsener (kaminpar-shm/coarsening/sparsification_cluster_coarsener.cc):

  * target(prev_m, prev_n, c_n) = min(edge_target_factor * prev_m, density_target_factor * prev_m / prev_n * c_n)
    in double, truncated if below prev_m, else prev_m (:41-48);
  * T = the (c_m - target + 1)-th smallest edge weight with the exact counts smaller / equal
    (quickselect_k_smallest, kaminpar-common/parallel/quickselect.h); p = (target - larger) / equal in double
    (:177-193);
  * an edge (u, v, w) is kept iff w > T, or w == T and dice(u, v) < p, where dice hashes the ordered pair plus the
    seed with murmur3's fmix64 and scales the low 32 bits by 1 / (2^32 - 1) (:201-218); target < 2 keeps nothing
    (:166-175).

It works on the canonical coarse CSR of oracle/contraction_oracle.py (coarse ids = ranks of the leaders, adjacency
sorted by target), so `dice` hashes the canonical ids.
"""
from __future__ import annotations

import numpy as np

M32 = np.uint64(0xFFFFFFFF)


def sparsification_target(prev_m, prev_n, c_n, density_target_factor=0.5, edge_target_factor=0.5) -> int:
    # IEEE doubles (prev_n = 0 gives inf / nan as in C++), operands in the reference's order
    f = np.float64
    with np.errstate(all="ignore"):
        edge = f(edge_target_factor) * f(prev_m)
        dens = f(density_target_factor) * f(prev_m) / f(prev_n) * f(c_n)
    target = dens if dens < edge else edge  # std::min(edge, dens) = (dens < edge) ? dens : edge
    return int(target) if target < f(prev_m) else int(prev_m)


def select(adjwgt, target_m):
    """(T, smaller, equal) of the (c_m - target_m + 1)-th smallest weight."""
    w = np.asarray(adjwgt, np.int64)
    k = len(w) - int(target_m) + 1
    t = int(np.partition(w, k - 1)[k - 1])
    return t, int(np.count_nonzero(w < t)), int(np.count_nonzero(w == t))


def fmix64(x):
    x = np.asarray(x, np.uint64).copy()
    x ^= x >> np.uint64(33)
    x *= np.uint64(0xFF51AFD7ED558CCD)
    x ^= x >> np.uint64(33)
    x *= np.uint64(0xC4CEB9FE1A85EC53)
    x ^= x >> np.uint64(33)
    return x


def dice_hash(u, v, seed):
    """Low 32 bits h of the hash; dice = h / (2^32 - 1)."""
    u = np.asarray(u, np.uint64)
    v = np.asarray(v, np.uint64)
    key = (np.maximum(u, v) << np.uint64(32)) | np.minimum(u, v)
    with np.errstate(over="ignore"):
        key = key + np.uint64(int(seed) & 0xFFFFFFFFFFFFFFFF)
        return fmix64(key) & M32


def dice(u, v, seed):
    return dice_hash(u, v, seed).astype(np.float64) / 4294967295.0


def sparsify(c_xadj, c_adjncy, c_adjwgt, target_m, seed):
    """Returns dict(c_xadj, c_adjncy, c_adjwgt, threshold, smaller, equal, equal_kept, probability)."""
    c_xadj = np.asarray(c_xadj, np.int64)
    adj = np.asarray(c_adjncy, np.int64)
    w = np.asarray(c_adjwgt, np.int64)
    c_n, c_m = len(c_xadj) - 1, len(adj)
    assert 0 <= target_m <= c_m
    if target_m < 2:
        keep = np.zeros(c_m, bool)
        t = smaller = equal = 0
        p = 0.0
    else:
        t, smaller, equal = select(w, target_m)
        larger = c_m - smaller - equal
        assert larger <= target_m
        p = float(target_m - larger) / float(equal)
        src = np.repeat(np.arange(c_n, dtype=np.int64), np.diff(c_xadj))
        at = w == t
        keep = w > t
        keep[at] = dice(src[at], adj[at], seed) < p
    kept_before = np.concatenate([[0], np.cumsum(keep)])
    return dict(c_xadj=kept_before[c_xadj].astype(np.uint32), c_adjncy=adj[keep].astype(np.uint32),
                c_adjwgt=w[keep].astype(np.int32), threshold=t, smaller=smaller, equal=equal,
                equal_kept=int(np.count_nonzero(keep & (w == t))) if target_m >= 2 else 0, probability=p)


def sparsify_contracted(contracted: dict, target_m, seed) -> dict:
    """sparsify() of an oracle/contraction_oracle.py result: a full coarse graph dict with the same c_n, c_vwgt
    and mapping, plus the selection's numbers."""
    s = sparsify(contracted["c_xadj"], contracted["c_adjncy"], contracted["c_adjwgt"], target_m, seed)
    out = dict(contracted)
    out.update(s)
    return out


def edge_set(c_xadj, c_adjncy, c_adjwgt=None):
    src = np.repeat(np.arange(len(c_xadj) - 1, dtype=np.int64), np.diff(np.asarray(c_xadj, np.int64)))
    if c_adjwgt is None:
        return set(zip(src.tolist(), np.asarray(c_adjncy).tolist()))
    return set(zip(src.tolist(), np.asarray(c_adjncy).tolist(), np.asarray(c_adjwgt).tolist()))
