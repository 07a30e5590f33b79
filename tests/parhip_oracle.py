"""NumPy oracle of the ParHIP reader on the device (include/kaminpar_b200_parhip.h, DESIGN.md §19): the rule of the
header, written out section by section, and the three orderings of io::parhip::read_graph
(kaminpar-io/parhip_parser.cc:179-336).

    read(data, ordering)   -> dict: the report fields and, for a graph, xadj / adjncy / vwgt / adjwgt / old_to_new
    write(xadj, adjncy, vwgt, adjwgt, version) -> bytes: a ParHIP file at the widths the version's bits give

The EXTERNAL permutation is computed here by bucketing with frexp and concatenating the buckets' vertex lists, not by
the preparation oracle's stable sort, and the adjacency lists are copied forward (csr_read_deg_buckets, :306-325).
"""
import numpy as np

KINDS = ("OK", "TRUNCATED", "TOO_LARGE", "OFFSETS", "NEIGHBOR_OUT_OF_RANGE", "WEIGHT", "TOTAL_WEIGHT")
OK, TRUNCATED, TOO_LARGE, OFFSETS, NEIGHBOR_OUT_OF_RANGE, WEIGHT, TOTAL_WEIGHT = range(7)
HEADER, OFFS, ADJNCY, VWGT, ADJWGT = range(5)  # sections
NATURAL, DEGREE_BUCKETS, EXTERNAL, IMPLICIT = range(4)  # NodeOrdering
INT32_MAX = (1 << 31) - 1
REPORT_FIELDS = ("kind", "section", "has_node_weights", "has_edge_weights", "sorted", "ordering", "version", "n", "m",
                 "bytes", "offset", "index", "widths")


def version_of(vw: bool, ew: bool, offsets64=False, ids64=False, vw64=False, ew64=False, high=0) -> int:
    """The version word: a bit CLEAR means present / 64-bit (ParHIPHeader::version, :51-68); `high` sets bits >= 6."""
    return ((0 if ew else 1) | (0 if vw else 2) | (0 if offsets64 else 4) | (0 if ids64 else 8) |
            (0 if vw64 else 16) | (0 if ew64 else 32) | (high << 6))


def widths(version: int):
    """Bytes per entry of offsets, ids, node weights, edge weights."""
    return tuple(4 if (version >> b) & 1 else 8 for b in (2, 3, 4, 5))


def write(xadj, adjncy, vwgt=None, adjwgt=None, version=None) -> bytes:
    """The file of a graph; `version` defaults to 32-bit widths with the weights that are given."""
    xadj = np.asarray(xadj, np.int64)
    n, m = len(xadj) - 1, len(adjncy)
    if version is None:
        version = version_of(vwgt is not None, adjwgt is not None)
    wo, wi, wv, we = widths(version)
    base = 24 + (n + 1) * wo
    parts = [np.array([version, n, m], "<u8").tobytes(),
             (xadj * wi + base).astype(f"<u{wo}").tobytes(),
             np.asarray(adjncy, np.int64).astype(f"<u{wi}").tobytes()]
    if (version & 2) == 0:
        parts.append(np.asarray(vwgt, np.int64).astype(f"<i{wv}").tobytes())
    if (version & 1) == 0:
        parts.append(np.asarray(adjwgt, np.int64).astype(f"<i{we}").tobytes())
    return b"".join(parts)


def _u(b, start, count, w):
    return np.frombuffer(b[start:start + count * w], f"<u{w}").astype(np.uint64)


def read(data, ordering: int = NATURAL) -> dict:
    """The rule of kaminpar_b200_parhip.h on the file's bytes."""
    b = bytes(data)
    L = len(b)
    r = dict(kind=OK, section=HEADER, has_node_weights=0, has_edge_weights=0,
             sorted=int(ordering in (EXTERNAL, IMPLICIT)), ordering=ordering, version=0, n=0, m=0, bytes=L, offset=0,
             index=0, widths=0, xadj=None, adjncy=None, vwgt=None, adjwgt=None, old_to_new=None)

    def refuse(kind, offset, section, index):
        r.update(kind=kind, offset=offset, section=section, index=index)
        return r

    if L >= 8:
        v = int(np.frombuffer(b[:8], "<u8")[0])
        r["version"] = v
        r["has_edge_weights"], r["has_node_weights"] = int((v & 1) == 0), int((v & 2) == 0)
        w = widths(v)
        r["widths"] = w[0] | (w[1] << 8) | (w[2] << 16) | (w[3] << 24)
    if L >= 16:
        r["n"] = n = int(np.frombuffer(b[8:16], "<u8")[0])
        if n >= 1 << 31:
            return refuse(TOO_LARGE, 8, HEADER, -1)
    if L < 24:
        return refuse(TRUNCATED, L, HEADER, -1)
    r["m"] = m = int(np.frombuffer(b[16:24], "<u8")[0])
    if m >= 1 << 31:
        return refuse(TOO_LARGE, 16, HEADER, -1)
    v = r["version"]
    vw, ew = bool(r["has_node_weights"]), bool(r["has_edge_weights"])
    wo, wi, wv, we = widths(v)
    count = [0, n + 1, m, n if vw else 0, m if ew else 0]
    width = [0, wo, wi, wv, we]
    start = [0, 24]
    for s in range(1, 5):
        start.append(start[s] + count[s] * width[s])
    end = start[5]
    base = start[ADJNCY]
    cands = []  # (key, section, index)

    def first(section, flags, kinds):
        idx = np.flatnonzero(flags)
        if len(idx):
            i = int(idx[0])
            k = int(kinds[i]) if np.ndim(kinds) else int(kinds)
            cands.append((((start[section] + i * width[section]) << 8) | k, section, i))

    def complete(s):
        return int(min(count[s], max(0, (L - start[s]) // width[s]))) if count[s] else 0

    vals = {s: _u(b, start[s], complete(s), width[s]) for s in range(1, 5)}
    # offsets
    off = vals[OFFS]  # uint64: differences wrap modulo 2^64, which keeps their residues modulo the id width
    c = len(off)
    bad = np.zeros(c, bool)
    if c:
        bad[0] |= off[0] != np.uint64(base)
        bad[1:] |= off[1:] < off[:-1]
        bad |= ((off - np.uint64(base)) & np.uint64(wi - 1)) != 0
        if c == n + 1:
            bad[n] |= off[n] != np.uint64(base + m * wi)
    first(OFFS, bad, OFFSETS)
    # targets
    t = vals[ADJNCY]
    first(ADJNCY, ((t >> np.uint64(32)) != 0) | (t >= np.uint64(n)),
          np.where((t >> np.uint64(32)) != 0, TOO_LARGE, NEIGHBOR_OUT_OF_RANGE))
    # weights
    sums = {}
    for s, ww in ((VWGT, wv), (ADJWGT, we)):
        x = vals[s].astype(np.uint64)
        sx = x.view(np.int64) if ww == 8 else x.astype(np.uint32).view(np.int32).astype(np.int64)
        first(s, (sx < 1) | (sx > INT32_MAX), np.where(sx < 1, WEIGHT, TOO_LARGE))
        ok = (sx >= 1) & (sx <= INT32_MAX)
        sums[s] = int(sx[ok].sum())
        if count[s] and start[s + 1] <= L and sums[s] > INT32_MAX:
            cands.append((((start[s + 1] - 1) << 8) | TOTAL_WEIGHT, s, count[s]))
    if L < end:
        s = 1
        while start[s + 1] <= L:
            s += 1
        cands.append(((L << 8) | TRUNCATED, s, (L - start[s]) // width[s]))
    if cands:
        key, s, i = min(cands)
        return refuse(key & 0xFF, key >> 8, s, i)
    xadj = ((np.asarray(off, np.uint64) - np.uint64(base)) // np.uint64(wi)).astype(np.uint32)
    adj = t.astype(np.uint32)
    vwgt = vals[VWGT].astype(np.uint32).view(np.int32) if vw else None
    adjwgt = vals[ADJWGT].astype(np.uint32).view(np.int32) if ew else None
    if ordering == EXTERNAL:
        xadj, adj, vwgt, adjwgt, o2n = external(xadj, adj, vwgt, adjwgt)
        r["old_to_new"] = o2n
    r.update(xadj=xadj, adjncy=adj, vwgt=vwgt, adjwgt=adjwgt)
    return r


def external(xadj, adjncy, vwgt=None, adjwgt=None):
    """csr_read_deg_buckets on a checked graph: (xadj, adjncy, vwgt, adjwgt, old_to_new) in the new order."""
    xadj = np.asarray(xadj, np.int64)
    n = len(xadj) - 1
    deg = np.diff(xadj)
    bucket = np.frexp(deg.astype(np.float64))[1].astype(np.int64)  # floor(log2 d) + 1 for d > 0 (exact: d < 2^31)
    bucket[deg == 0] = 32
    new_to_old = np.concatenate([np.flatnonzero(bucket == k) for k in range(33)] + [np.zeros(0, np.int64)])
    old_to_new = np.empty(n, np.int64)
    old_to_new[new_to_old] = np.arange(n)
    new_deg = deg[new_to_old]
    new_xadj = np.zeros(n + 1, np.int64)
    np.cumsum(new_deg, out=new_xadj[1:])
    e = np.concatenate([np.arange(xadj[u], xadj[u + 1]) for u in new_to_old] + [np.zeros(0, np.int64)]) \
        if n < 4096 else np.repeat(xadj[new_to_old] - new_xadj[:-1], new_deg) + np.arange(new_xadj[-1])
    e = e.astype(np.int64)
    adj = old_to_new[np.asarray(adjncy, np.int64)[e]] if len(e) else np.zeros(0, np.int64)
    return (new_xadj.astype(np.uint32), adj.astype(np.uint32),
            None if vwgt is None else np.asarray(vwgt, np.int32)[new_to_old],
            None if adjwgt is None else np.asarray(adjwgt, np.int32)[e],
            old_to_new.astype(np.uint32))


def report_of(r: dict) -> dict:
    return {f: r[f] for f in REPORT_FIELDS}


def as_dict(rep) -> dict:
    return {f: getattr(rep, f) for f in REPORT_FIELDS}
