"""NumPy oracle of the input preparation (DESIGN.md §15): a literal restatement of what KaMinPar::compute_partition
does with the caller's graph before and after partitioning.

    rearrange(...)  graph::rearrange_by_degree_buckets (graphutils/permutator.h:28-209) and the isolated-vertex cut
                    (count_isolated_nodes, permutator.cc:266-282; CSRGraph::remove_isolated_nodes, csr_graph.cc:150-174)
    finish(...)     CSRGraph::integrate_isolated_nodes + graph::assign_isolated_nodes (permutator.cc:236-264) + the
                    map back to the caller's ids (kaminpar.cc:419-445)

The device (kaminpar_b200/csrc/kmp_prepare.cuh) equals it bit for bit; tests/test_prepare_oracle.py pins it against
the unmodified reference.
"""
import numpy as np

ISOLATED_BUCKET = 32  # kNumberOfDegreeBuckets<uint32_t> - 1 (degree_buckets.h:17, permutator.h:105-107)


def buckets(xadj) -> np.ndarray:
    """bucket(u) = floor(log2 deg(u)) + 1, and 32 for deg(u) == 0."""
    deg = np.diff(np.asarray(xadj, np.int64))
    b = np.full(deg.shape, ISOLATED_BUCKET, np.int64)
    for j in range(32):  # floor(log2 d) + 1 == j + 1  <=>  2^j <= d < 2^(j+1)
        b[(deg >= (1 << j)) & (deg < (1 << (j + 1)))] = j + 1
    return b


def rearrange(xadj, adjncy, vwgt=None, adjwgt=None) -> dict:
    """The permuted graph on all n vertices (isolated ones last) and n' = n - #isolated. xadj has n + 1 entries;
    the LP's graph is xadj[:n'+1] with vwgt[:n']."""
    xadj = np.asarray(xadj, np.int64)
    adjncy = np.asarray(adjncy, np.int64)
    n = len(xadj) - 1
    b = buckets(xadj)
    new_to_old = np.argsort(b, kind="stable")
    old_to_new = np.empty(n, np.int64)
    old_to_new[new_to_old] = np.arange(n)
    deg = np.diff(xadj)
    new_xadj = np.zeros(n + 1, np.int64)
    np.cumsum(deg[new_to_old], out=new_xadj[1:])
    # permutator.h:196-207: p_e = --new_nodes[u] walks old_u's list forwards and writes it backwards, so the i-th
    # edge of old_u lands at new_xadj[u + 1] - 1 - i
    m = len(adjncy)
    src = np.repeat(np.arange(n), deg)
    pos = new_xadj[old_to_new[src] + 1] - 1 - (np.arange(m) - xadj[src])
    new_adj = np.empty(m, np.int64)
    new_adj[pos] = old_to_new[adjncy]
    new_ew = None
    if adjwgt is not None:
        new_ew = np.empty(m, np.int32)
        new_ew[pos] = np.asarray(adjwgt, np.int32)
    num_isolated = int((deg == 0).sum())
    return dict(
        xadj=new_xadj.astype(np.uint32), adjncy=new_adj.astype(np.uint32),
        vwgt=None if vwgt is None else np.asarray(vwgt, np.int32)[new_to_old],
        adjwgt=new_ew, old_to_new=old_to_new.astype(np.uint32), new_to_old=new_to_old.astype(np.uint32),
        n_prime=n - num_isolated, num_isolated=num_isolated,
    )


def finish(prepared: dict, k: int, max_block_weights, partition):
    """partition: blocks of the n' vertices. Returns (the partition of the caller's n vertices, block weights)."""
    n_prime, n = prepared["n_prime"], len(prepared["old_to_new"])
    vw = prepared["vwgt"]
    w = np.ones(n, np.int64) if vw is None else np.asarray(vw, np.int64)
    partition = np.asarray(partition, np.int64)
    assert len(partition) == n_prime and (partition < k).all()
    bw = np.zeros(k, np.int64)
    np.add.at(bw, partition, w[:n_prime])
    p = np.empty(n, np.int64)
    p[:n_prime] = partition
    b = 0
    for u in range(n_prime, n):  # permutator.cc:255-261
        while b + 1 < k and bw[b] + w[u] > int(max_block_weights[b]):
            b += 1
        p[u] = b
        bw[b] += w[u]
    return p[prepared["old_to_new"]].astype(np.uint32), bw
