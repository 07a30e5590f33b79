"""NumPy oracle of graph validation (include/kaminpar_b200_validate.h, DESIGN.md §17): the reference's
debug::validate_graph (kaminpar-shm/datastructures/csr_graph.cc:266-356, check_undirected = true, num_pseudo_nodes = 0)
with the library's two shape checks in front, carried on past the first violation to count every edge under its first
kind, plus the duplicate-neighbour count.

Two forms that must agree: `validate_loop` follows the reference's loops (for each edge, a scan of the neighbour's row
in input order; quadratic in hub degrees, for small graphs), `validate` is vectorised (one sort of (row, target) keys).
Both return the same dict; `message(report)` is the reference's warning line.
"""
from __future__ import annotations

import numpy as np

VALID, XADJ_START, XADJ_END, XADJ_DECREASING, NEIGHBOR_OUT_OF_GRAPH, SELF_LOOP, \
    NEIGHBOR_OF_NEIGHBOR_OUT_OF_GRAPH, MISSING_REVERSE, WEIGHT_MISMATCH = range(9)
NUM_KINDS = 9
FIELDS = ("valid", "kind", "u", "e", "v", "e_rev", "v_rev", "w", "w_rev", "count", "duplicates", "dup_u", "dup_e")


def _report(n, m):
    return dict(valid=1, kind=VALID, n=n, m=m, u=0, e=0, v=0, e_rev=0, v_rev=0, w=0, w_rev=0, count=[0] * NUM_KINDS,
                duplicates=0, dup_u=0, dup_e=0)


def _shape(r, xadj, n, m):
    """Steps 1-2; True when they pass (and the rows may be read)."""
    xadj = np.asarray(xadj, np.int64)
    r["count"][XADJ_START] = int(xadj[0] != 0)
    r["count"][XADJ_END] = int(xadj[n] != m)
    dec = np.nonzero(xadj[:-1] > xadj[1:])[0]
    r["count"][XADJ_DECREASING] = len(dec)
    if xadj[0] != 0:
        r.update(kind=XADJ_START, e=int(xadj[0]))
    elif xadj[n] != m:
        r.update(kind=XADJ_END, u=n, e=int(xadj[n]))
    elif len(dec):
        r.update(kind=XADJ_DECREASING, u=int(dec[0]))
    r["valid"] = int(r["kind"] == VALID)
    return r["valid"] == 1


def validate_loop(xadj, adjncy, adjwgt=None) -> dict:
    xadj = [int(x) for x in xadj]
    adjncy = [int(x) for x in adjncy]
    adjwgt = None if adjwgt is None else [int(x) for x in adjwgt]
    n, m = len(xadj) - 1, len(adjncy)
    r = _report(n, m)
    if not _shape(r, xadj, n, m):
        return r
    first = None
    for u in range(n):
        seen = set()
        for e in range(xadj[u], xadj[u + 1]):
            v = adjncy[e]
            if v in seen:
                r["duplicates"] += 1
                if r["duplicates"] == 1:
                    r["dup_u"], r["dup_e"] = u, e
            seen.add(v)
            det = dict(u=u, e=e, v=v)
            if v >= n:
                kind = NEIGHBOR_OUT_OF_GRAPH
            elif u == v:
                kind = SELF_LOOP
            else:
                kind = MISSING_REVERSE  # csr_graph.cc:318-350: scan v's row in input order
                for e_prime in range(xadj[v], xadj[v + 1]):
                    u_prime = adjncy[e_prime]
                    if u_prime >= n:
                        kind = NEIGHBOR_OF_NEIGHBOR_OUT_OF_GRAPH
                        det.update(e_rev=e_prime, v_rev=u_prime)
                        break
                    if u != u_prime:
                        continue
                    kind = VALID
                    if adjwgt is not None and adjwgt[e] != adjwgt[e_prime]:
                        kind = WEIGHT_MISMATCH
                        det.update(e_rev=e_prime, v_rev=u, w=adjwgt[e], w_rev=adjwgt[e_prime])
                    break
            if kind != VALID:
                r["count"][kind] += 1
                if first is None:
                    first = dict(det, kind=kind)
    if first is not None:
        r.update(first)
        r["valid"] = 0
    return r


def validate(xadj, adjncy, adjwgt=None) -> dict:
    xadj = np.asarray(xadj, np.int64)
    adj = np.asarray(adjncy, np.int64)
    n, m = len(xadj) - 1, len(adj)
    r = _report(n, m)
    if not _shape(r, xadj, n, m) or m == 0:
        return r
    owner = np.repeat(np.arange(n, dtype=np.int64), np.diff(xadj))
    pos = np.arange(m, dtype=np.int64)
    # first occurrence of every (row, target): np.unique's indices are the first positions in input order
    keys = (owner << 32) | adj
    ukeys, ufirst = np.unique(keys, return_index=True)
    dup = np.ones(m, bool)
    dup[ufirst] = False
    r["duplicates"] = int(dup.sum())
    if r["duplicates"]:
        e = int(np.argmax(dup))  # rows are contiguous and ascending: the smallest position is in the smallest row
        r["dup_u"], r["dup_e"] = int(owner[e]), e
    none = np.int64(1) << 40
    bad = adj >= n
    q = np.full(n, none, np.int64)  # first position with a target >= n per row
    brow, bidx = np.unique(owner[bad], return_index=True)
    q[brow] = pos[bad][bidx]
    kind = np.zeros(m, np.int64)
    kind[bad] = NEIGHBOR_OUT_OF_GRAPH
    selfl = ~bad & (adj == owner)
    kind[selfl] = SELF_LOOP
    rest = ~bad & ~selfl
    v = np.where(rest, adj, 0)
    want = (v << 32) | owner
    i = np.minimum(np.searchsorted(ukeys, want), len(ukeys) - 1)
    p = np.where(ukeys[i] == want, ufirst[i], none)
    qv = q[v]
    non = rest & (qv < p)
    kind[non] = NEIGHBOR_OF_NEIGHBOR_OUT_OF_GRAPH
    miss = rest & ~non & (p == none)
    kind[miss] = MISSING_REVERSE
    if adjwgt is not None:
        w = np.asarray(adjwgt, np.int64)
        wm = rest & ~non & ~miss & (w != w[np.minimum(p, m - 1)])
        kind[wm] = WEIGHT_MISMATCH
    for k in range(NEIGHBOR_OUT_OF_GRAPH, NUM_KINDS):
        r["count"][k] = int((kind == k).sum())
    viol = np.nonzero(kind)[0]
    if len(viol):
        e = int(viol[0])
        k = int(kind[e])
        r.update(valid=0, kind=k, u=int(owner[e]), e=e, v=int(adj[e]))
        if k == NEIGHBOR_OF_NEIGHBOR_OUT_OF_GRAPH:
            r.update(e_rev=int(qv[e]), v_rev=int(adj[qv[e]]))
        elif k == WEIGHT_MISMATCH:
            r.update(e_rev=int(p[e]), v_rev=int(owner[e]), w=int(w[e]), w_rev=int(w[p[e]]))
    return r


def message(r: dict) -> str:
    """csr_graph.cc:276-350, word for word (the shape kinds are the library's own)."""
    k = r["kind"]
    if k == XADJ_START:
        return f"xadj[0] is {r['e']}, not 0"
    if k == XADJ_END:
        return f"xadj[{r['u']}] is {r['e']}, not the number of edges {r['m']}"
    if k == XADJ_DECREASING:
        return f"Bad node array at position {r['u']}"
    if k == NEIGHBOR_OUT_OF_GRAPH:
        return f"Neighbor {r['v']} of {r['u']} is out-of-graph"
    if k == SELF_LOOP:
        return f"Self-loop at {r['u']}: {r['e']} --> {r['v']}"
    if k == NEIGHBOR_OF_NEIGHBOR_OUT_OF_GRAPH:
        return f"Neighbor {r['v_rev']} of neighbor {r['v']} of {r['u']} is out-of-graph"
    if k == MISSING_REVERSE:
        return f"Edge {r['u']} --> {r['v']} exists with edge {r['e']}, but the reverse edges does not exist"
    if k == WEIGHT_MISMATCH:
        return (f"Weight of edge {r['e']} ({r['w']}) differs from the weight of its reverse edge {r['e_rev']} "
                f"({r['w_rev']})")
    return ""


def as_dict(report) -> dict:
    """The oracle's fields of a GraphReport (kaminpar_b200.validate) or of a golden record."""
    if isinstance(report, dict):
        return {f: (list(report[f]) if f == "count" else int(report[f])) for f in FIELDS}
    return {f: (list(getattr(report, f)) if f == "count" else int(getattr(report, f))) for f in FIELDS}


# ---- corpus: valid graphs and their mutations --------------------------------------------------------------------
# A case is (name, xadj, adjncy, adjwgt or None), arrays as numpy (uint32 / int32).

def _case(name, xadj, adj, w=None):
    return (name, np.asarray(xadj, np.uint32), np.asarray(adj, np.uint32), None if w is None else np.asarray(w, np.int32))


def insert_edge(xadj, adj, w, row, index, target, weight=1):
    """Insert `target` (and its weight) at `index` of `row` (0 <= index <= degree)."""
    xadj = xadj.astype(np.int64)
    at = int(xadj[row] + index)
    adj = np.insert(adj.astype(np.int64), at, target).astype(np.uint32)
    if w is not None:
        w = np.insert(w, at, weight).astype(np.int32)
    xadj[row + 1:] += 1
    return xadj.astype(np.uint32), adj, w


def owner_of(xadj, e):
    return int(np.searchsorted(xadj.astype(np.int64), e, side="right") - 1)


def star(leaves, isolated=0):
    """Vertex 0 joined to `leaves` leaves, then `isolated` isolated vertices."""
    xadj = np.concatenate([[0], leaves + np.arange(0, leaves + 1), np.full(isolated, 2 * leaves)])
    adj = np.concatenate([np.arange(1, leaves + 1), np.zeros(leaves)])
    return xadj, adj


def positions(xadj, adj):
    """Named edge positions of a graph: its first and last edge, the middle of its largest row and the edge of its
    first degree-1 row."""
    deg = np.diff(xadj.astype(np.int64))
    m = len(adj)
    out = {"first": 0, "last": m - 1}
    hub = int(np.argmax(deg))
    out["hub"] = int(xadj[hub] + deg[hub] // 2)
    ones = np.nonzero(deg == 1)[0]
    if len(ones):
        out["deg1"] = int(xadj[ones[0]])
    return out


def _non_neighbor(xadj, adj, u, n):
    row = set(int(x) for x in adj[xadj[u]:xadj[u + 1]])
    for d in range(1, n):
        t = (u + n // 2 + d) % n
        if t != u and t not in row:
            return t
    return None


def mutations(name, xadj, adj, w):
    """Each edge kind at each named position, the competing kinds and the duplicate cases."""
    n, m = len(xadj) - 1, len(adj)
    out = []
    weighted = w if w is not None else np.ones(m, np.int32)
    for where, e in positions(xadj, adj).items():
        u, v = owner_of(xadj, e), int(adj[e])
        a = adj.copy(); a[e] = n
        out.append(_case(f"{name}/out_of_graph@{where}", xadj, a, w))
        a = adj.copy(); a[e] = u
        out.append(_case(f"{name}/self_loop@{where}", xadj, a, w))
        t = _non_neighbor(xadj, adj, u, n)
        if t is not None:
            a = adj.copy(); a[e] = t
            out.append(_case(f"{name}/missing_reverse@{where}", xadj, a, w))
        ww = weighted.copy(); ww[e] += 1
        out.append(_case(f"{name}/weight_mismatch@{where}", xadj, adj, ww))
        # an out-of-range entry in v's row before / after u's first occurrence
        row = adj[xadj[v]:xadj[v + 1]]
        i = int(np.nonzero(row == u)[0][0])
        out.append(_case(f"{name}/neighbor_of_neighbor_before@{where}", *insert_edge(xadj, adj, w, v, i, n + 3, 1)))
        out.append(_case(f"{name}/neighbor_of_neighbor_after@{where}", *insert_edge(xadj, adj, w, v, i + 1, 0xFFFFFFFF, 1)))
    # competing kinds: a missing reverse edge before a self-loop (both in the largest row)
    deg = np.diff(xadj.astype(np.int64))
    hub = int(np.argmax(deg))
    if deg[hub] >= 2:
        t = _non_neighbor(xadj, adj, hub, n)
        if t is not None:
            a = adj.copy(); a[xadj[hub]] = t; a[xadj[hub + 1] - 1] = hub
            out.append(_case(f"{name}/missing_then_self_loop", xadj, a, w))
    # duplicates of the first edge (u, v) with reverse p: v's row gets u a second time right after p
    e = 0
    u, v = owner_of(xadj, e), int(adj[e])
    i = int(np.nonzero(adj[xadj[v]:xadj[v + 1]] == u)[0][0])
    x2, a2, w2 = insert_edge(xadj, adj, weighted, v, i + 1, u, 0)
    p = int(x2[v] + i)
    w_first = w2.copy(); w_first[p] = w2[e] + 7; w_first[p + 1] = w2[e]  # mismatching first, matching duplicate
    out.append(_case(f"{name}/dup_mismatching_first", x2, a2, w_first))
    w_later = w2.copy(); w_later[p + 1] = w2[e] + 7  # matching first, mismatching duplicate
    out.append(_case(f"{name}/dup_mismatching_later", x2, a2, w_later))
    # a consistent multi-edge, next to its first occurrence in both rows (weights kept)
    x3, a3, w3 = insert_edge(xadj, adj, weighted, u, 1, v, int(weighted[e]))
    x3, a3, w3 = insert_edge(x3, a3, w3, v, i + 1, u, int(weighted[e]))
    out.append(_case(f"{name}/dup_consecutive", x3, a3, None if w is None else w3))
    # ... and one that is not next to it ([v, ..., v] in u's row, likewise in v's)
    du, dv = int(xadj[u + 1] - xadj[u]), int(xadj[v + 1] - xadj[v])
    if du >= 2 and i + 1 < dv:  # v is first in u's row, u at i in v's: appending both puts them apart
        x4, a4, w4 = insert_edge(xadj, adj, weighted, u, du, v, int(weighted[e]))
        x4, a4, w4 = insert_edge(x4, a4, w4, v, dv, u, int(weighted[e]))
        out.append(_case(f"{name}/dup_apart", x4, a4, None if w is None else w4))
    return out


def broken_xadj(name, xadj, adj, w):
    n, m = len(xadj) - 1, len(adj)
    out = []
    x = xadj.copy(); x[0] = 1
    out.append(_case(f"{name}/xadj_start", x, adj, w))
    for d in (1, -1):
        x = xadj.astype(np.int64); x[n] = m + d
        out.append(_case(f"{name}/xadj_end{d:+d}", x, adj, w))
    x = xadj.copy(); x[0] = 5  # a decrease at u = 0 needs xadj[0] > 0
    out.append(_case(f"{name}/xadj_decreasing@0", x, adj, w))
    if n >= 2:
        x = xadj.copy(); x[n - 1] = m + 1
        out.append(_case(f"{name}/xadj_decreasing@n-1", x, adj, w))
    if n >= 8:
        x = xadj.copy()
        for u in (n // 4, n // 2, 3 * n // 4):
            x[u] = x[u + 1] + 1 if x[u + 1] < 0xFFFFFFFF else x[u]
        out.append(_case(f"{name}/xadj_decreasing@several", x, adj, w))
        x = xadj.astype(np.int64)
        k = min(n - 1, 5)
        x[1:k + 1] = (1 << 32) - 64 + np.arange(k)  # monotone-looking up to k, then back below
        out.append(_case(f"{name}/xadj_near_2^32", x, adj, w))
    return out


def small_bases():
    """Valid graphs small enough for the loop form and the reference bridge."""
    import os

    from kaminpar_b200.graph import grid3d, random_weights, rmat

    gold = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    out = []
    for name, f in (("rgg2d", "graph_rgg2d"), ("walshaw_data", "graph_walshaw_data"), ("rgg16_w", "graph_rgg16_vwgt_adjwgt")):
        d = np.load(os.path.join(gold, f + ".npz"))
        out.append(_case(name, d["xadj"], d["adjncy"], d["adjwgt"] if "adjwgt" in d.files else None))
    g = random_weights(rmat(9, 4, seed=5), seed=2, max_adjwgt=9)
    out.append(_case("rmat9_w", g.xadj, g.adjncy, g.adjwgt))
    g = grid3d(5)
    out.append(_case("grid5", g.xadj, g.adjncy))
    out.append(_case("star300_iso", *star(300, isolated=4)))
    return out


def empty_graphs():
    return [_case("n0", [0], []), _case("m0", np.zeros(6), [])]
