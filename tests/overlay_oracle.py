"""NumPy oracle of the overlay of clusterings (DESIGN.md §14), written from the rule of the reference's
OverlayClusterCoarsener (kaminpar-shm/coarsening/overlay_cluster_coarsener.cc:34-151):

    out[u] = index(ra(a[u])) + |{distinct b[v] : a[v] == a[u], b[v] < b[u]}|

where ra(x) is the rank of x among the distinct values of a and index(c) the number of vertices whose a-rank is
below c (fill_leader_mapping / compute_mapping / fill_cluster_buckets). 2^L clusterings are reduced in the tree order
of coarsen(): for level = L .. 1, h = 2^(level-1), C[p] = overlay(C[p], C[h + p]) for p < h; the result is C[0]."""
import numpy as np


def overlay(a, b) -> np.ndarray:
    a = np.asarray(a, np.int64)
    b = np.asarray(b, np.int64)
    n = len(a)
    if len(b) != n:
        raise ValueError("clusterings of different lengths")
    if n == 0:
        return np.zeros(0, np.uint32)
    if a.min() < 0 or b.min() < 0 or a.max() >= n or b.max() >= n:
        raise ValueError("a clustering holds an id outside [0, n)")
    _, ra = np.unique(a, return_inverse=True)  # ra(a[u])
    index = np.concatenate([[0], np.cumsum(np.bincount(ra))])  # index(c): vertices whose a-rank is below c
    pairs, inv = np.unique(ra * n + b, return_inverse=True)  # distinct (ra, b), sorted by ra then b
    first = np.searchsorted(pairs, (pairs // n) * n)  # first distinct pair of the same a-cluster
    below = np.arange(len(pairs)) - first  # distinct b of that cluster below this one
    return (index[ra] + below[inv]).astype(np.uint32)


def overlay_tree(clusterings) -> np.ndarray:
    c = [np.asarray(x, np.uint32) for x in clusterings]
    count = len(c)
    if count == 0 or count & (count - 1):
        raise ValueError("the number of clusterings must be a power of two")
    half = count // 2
    while half >= 1:
        for p in range(half):
            c[p] = overlay(c[p], c[half + p])
        half //= 2
    return c[0]
