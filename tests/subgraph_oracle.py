"""NumPy oracle of the partition extension's graph passes (DESIGN.md §16), at the reference's one-thread order:

    lazy_extract(...)       graph::lazy_extract_subgraphs_preprocessing + graph::extract_subgraph for every block
                            (graphutils/subgraph_extractor.cc:181-324), in the device's n + k layout
    extract_nonlazy(...)    graph::extract_subgraphs (:334-490): per block the same graph and the same mapping
    compute_final_k(...)    partitioning::compute_final_k (partitioning/partition_utils.cc:21-49)
    copy_back(...)          graph::copy_subgraph_partitions (:492-533)

Written as the reference's loops, not as the device's sort and scans, so that the two are independent.
"""
from __future__ import annotations

import numpy as np


def lazy_extract(xadj, adjncy, vwgt, adjwgt, part, k):
    """Returns dict(node_off, edge_off, block_nodes, mapping, xadj (n + k), adjncy, vwgt, adjwgt)."""
    xadj = np.asarray(xadj, np.int64)
    adjncy = np.asarray(adjncy, np.int64)
    part = np.asarray(part, np.int64)
    n = len(xadj) - 1
    counts = np.bincount(part, minlength=k)[:k] if n > 0 else np.zeros(k, np.int64)
    node_off = np.zeros(k + 1, np.int64)
    node_off[1:] = np.cumsum(counts)
    block_nodes = np.zeros(n, np.int64)
    mapping = np.zeros(n, np.int64)
    index = np.zeros(k, np.int64)
    for u in range(n):  # the second parallel_for at one thread: __atomic_fetch_add hands out ranks in id order
        b = part[u]
        block_nodes[node_off[b] + index[b]] = u
        mapping[u] = index[b]
        index[b] += 1
    xcat = np.zeros(n + k, np.int64)
    out_adj, out_ew = [], []
    edge_off = np.zeros(k + 1, np.int64)
    cur_total = 0
    for b in range(k):
        edge_off[b] = cur_total
        cur = 0
        for i in range(node_off[b], node_off[b + 1]):
            u = block_nodes[i]
            xcat[i + b] = cur
            for e in range(xadj[u], xadj[u + 1]):
                v = adjncy[e]
                if part[v] == b:
                    out_adj.append(mapping[v])
                    if adjwgt is not None:
                        out_ew.append(adjwgt[e])
                    cur += 1
        xcat[node_off[b + 1] + b] = cur
        cur_total += cur
    edge_off[k] = cur_total
    return dict(
        node_off=node_off.astype(np.uint32), edge_off=edge_off.astype(np.uint32),
        block_nodes=block_nodes.astype(np.uint32), mapping=mapping.astype(np.uint32), xadj=xcat.astype(np.uint32),
        adjncy=np.asarray(out_adj, np.uint32),
        vwgt=None if vwgt is None else np.asarray(vwgt, np.int32)[block_nodes],
        adjwgt=None if adjwgt is None else np.asarray(out_ew, np.int32))


def lazy_extract_np(xadj, adjncy, vwgt, adjwgt, part, k):
    """lazy_extract vectorised (stable argsorts instead of the loops), for graphs of millions of edges. The CPU
    tests hold it equal to lazy_extract."""
    xadj = np.asarray(xadj, np.int64)
    adjncy = np.asarray(adjncy, np.int64)
    part = np.asarray(part, np.int64)
    n = len(xadj) - 1
    deg = np.diff(xadj)
    node_off = np.zeros(k + 1, np.int64)
    node_off[1:] = np.cumsum(np.bincount(part, minlength=k)[:k]) if n > 0 else 0
    order = np.argsort(part, kind="stable")
    newpos = np.empty(n, np.int64)
    newpos[order] = np.arange(n)
    mapping = newpos - node_off[part] if n > 0 else np.zeros(0, np.int64)
    src = np.repeat(np.arange(n), deg)
    internal = np.nonzero(part[adjncy] == part[src])[0] if len(adjncy) else np.zeros(0, np.int64)
    internal = internal[np.argsort(newpos[src[internal]], kind="stable")]
    ideg = np.bincount(src[internal], minlength=n)[order] if n > 0 else np.zeros(0, np.int64)
    edge_pos = np.zeros(n + 1, np.int64)
    edge_pos[1:] = np.cumsum(ideg)
    blk = part[order]
    xcat = np.zeros(n + k, np.int64)
    xcat[np.arange(n) + blk] = edge_pos[:n] - edge_pos[node_off[blk]]
    b = np.arange(k)
    xcat[node_off[1:] + b] = edge_pos[node_off[1:]] - edge_pos[node_off[:-1]]
    return dict(
        node_off=node_off.astype(np.uint32), edge_off=edge_pos[node_off].astype(np.uint32),
        block_nodes=order.astype(np.uint32), mapping=mapping.astype(np.uint32), xadj=xcat.astype(np.uint32),
        adjncy=mapping[adjncy[internal]].astype(np.uint32),
        vwgt=None if vwgt is None else np.asarray(vwgt, np.int32)[order],
        adjwgt=None if adjwgt is None else np.asarray(adjwgt, np.int32)[internal])


def extract_nonlazy(xadj, adjncy, vwgt, adjwgt, part, k):
    """graph::extract_subgraphs at one thread: per block (xadj, adjncy, vwgt, adjwgt) and the mapping. The reference
    lays the blocks out with padding slots between them; the blocks themselves are what a caller reads."""
    xadj = np.asarray(xadj, np.int64)
    part = np.asarray(part, np.int64)
    n = len(xadj) - 1
    mapping = np.zeros(n, np.int64)
    members = [[] for _ in range(k)]
    for u in range(n):
        b = part[u]
        mapping[u] = len(members[b])
        members[b].append(u)
    blocks = []
    for b in range(k):
        bx, ba, bw = [0], [], []
        for u in members[b]:
            for e in range(xadj[u], xadj[u + 1]):
                v = adjncy[e]
                if part[v] == b:
                    ba.append(mapping[v])
                    if adjwgt is not None:
                        bw.append(adjwgt[e])
            bx.append(len(ba))
        blocks.append(dict(xadj=np.asarray(bx, np.uint32), adjncy=np.asarray(ba, np.uint32),
                           vwgt=None if vwgt is None else np.asarray(vwgt, np.int32)[np.asarray(members[b], np.int64)],
                           adjwgt=None if adjwgt is None else np.asarray(bw, np.int32)))
    return blocks, mapping.astype(np.uint32)


def block_of(res, b):
    """Block b of a lazy_extract result as (xadj, adjncy, vwgt, adjwgt)."""
    no, eo = res["node_off"], res["edge_off"]
    n0, n1, e0, e1 = int(no[b]), int(no[b + 1]), int(eo[b]), int(eo[b + 1])
    return (res["xadj"][n0 + b: n1 + b + 1], res["adjncy"][e0:e1],
            None if res["vwgt"] is None else res["vwgt"][n0:n1], None if res["adjwgt"] is None else res["adjwgt"][e0:e1])


_LUT = [0, 8, 4, 12, 2, 10, 6, 14, 1, 9, 5, 13, 3, 11, 7, 15]


def compute_final_k(block: int, current_k: int, input_k: int) -> int:
    """partition_utils.cc:21-49, with its nibble lookup table."""
    if current_k == input_k:
        return 1
    level = current_k.bit_length() - 1  # floor_log2
    base = input_k >> level
    num_plus_one = input_k & ((1 << level) - 1)
    rev = 0
    for i in range(8):
        rev |= _LUT[(block >> (4 * (7 - i))) & 0xF] << (4 * i)
    reversed_block = rev >> (32 - level)
    return base + (1 if reversed_block < num_plus_one else 0)


def sub_block_offsets(k: int, k_prime: int, input_k: int) -> np.ndarray:
    """k0 of copy_subgraph_partitions (k + 1 entries)."""
    k0 = [k_prime // k] * (k + 1)
    if k_prime == input_k:
        for b in range(k):
            k0[b + 1] = compute_final_k(b, k, input_k)
    k0[0] = 0
    return np.cumsum(np.asarray(k0, np.int64))


def copy_back(part, mapping, node_off, sub_block_major, k, k_prime, input_k, vwgt=None):
    """(partition[n], block weights[k']) of copy_subgraph_partitions; sub_block_major: block b's sub-partition at
    node_off[b]."""
    part = np.asarray(part, np.int64)
    k0 = sub_block_offsets(k, k_prime, input_k)
    assert k0[-1] == k_prime
    sub = np.asarray(sub_block_major, np.int64)
    s = sub[np.asarray(node_off, np.int64)[part] + np.asarray(mapping, np.int64)] if len(part) else sub
    assert np.all(s < (k0[1:] - k0[:-1])[part])
    out = (k0[part] + s).astype(np.uint32)
    w = np.ones(len(part), np.int64) if vwgt is None else np.asarray(vwgt, np.int64)
    bw = np.bincount(out, weights=w, minlength=k_prime).astype(np.int32) if len(part) else np.zeros(k_prime, np.int32)
    return out, bw
