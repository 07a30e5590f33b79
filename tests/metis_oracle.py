"""NumPy oracle of the METIS reader on the device (include/kaminpar_b200_io.h, DESIGN.md §18): the rule that restates
csr_read (kaminpar-io/metis_parser.cc:158-245), written twice.

    parse_loop(data)  one pass over the lines and bytes, as the rule reads
    parse(data)       vectorised over the bytes (for files of hundreds of MB)

Both return the same dict: the report's fields (KIND names in KINDS) and, for a graph, xadj / adjncy / vwgt / adjwgt
(None when absent or dropped). The header is parsed by one function shared by both (it is host code on the device
path too). test_metis_oracle.py holds the two forms to each other and to graph.read_metis.
"""
from __future__ import annotations

import numpy as np

KINDS = ("OK", "EMPTY", "HEADER", "FORMAT", "TOO_LARGE", "BAD_BYTE", "MISSING_NODE_WEIGHT", "MISSING_EDGE_WEIGHT",
         "ZERO_WEIGHT", "WEIGHT_TOO_LARGE", "NEIGHBOR_OUT_OF_RANGE", "SELF_LOOP", "TOO_FEW_LINES", "EDGE_COUNT",
         "TOTAL_WEIGHT")
K = {name: i for i, name in enumerate(KINDS)}
UNSUPPORTED = (K["FORMAT"], K["TOO_LARGE"])
CAP = 1 << 40  # a token's value saturates here: above every id and weight
I32 = (1 << 31) - 1
REPORT = ("kind", "offset", "line", "vertex", "n", "m", "format", "has_node_weights", "has_edge_weights",
          "node_weights_dropped", "edge_weights_dropped", "extra_lines", "bytes")
SP, NL, PCT = 32, 10, 37


def _report(data: bytes) -> dict:
    r = dict.fromkeys(REPORT, 0)
    r.update(bytes=len(data), xadj=None, adjncy=None, vwgt=None, adjwgt=None)
    return r


def _refuse(r: dict, data: bytes, kind: int, offset: int, vertex: int) -> dict:
    r.update(kind=kind, offset=offset, line=data.count(b"\n", 0, offset) + 1, vertex=vertex, extra_lines=0)
    return r


def _is_digit(c: int) -> bool:
    return 48 <= c <= 57


def header(data: bytes, r: dict):
    """parse_header (metis_parser.cc:36-80) under the rule: (first byte after the header, n, m, vw, ew) or None with
    the refusal in r."""
    L = len(data)
    if L == 0:
        _refuse(r, data, K["EMPTY"], 0, -1)
        return None
    i = 0
    while True:  # comment lines before the header
        while i < L and data[i] == SP:
            i += 1
        if i < L and data[i] == PCT:
            j = data.find(b"\n", i)
            i = L if j < 0 else j + 1
            continue
        break
    toks = []  # (value, offset)

    def values():  # the value checks of the tokens read so far, in file order
        if len(toks) >= 1 and toks[0][0] >= 1 << 32:
            return K["TOO_LARGE"], toks[0][1]
        if len(toks) >= 2 and 2 * toks[1][0] >= 1 << 32:
            return K["TOO_LARGE"], toks[1][1]
        if len(toks) >= 2 and toks[1][0] > toks[0][0] * (toks[0][0] - 1) // 2:
            return K["HEADER"], toks[1][1]
        if len(toks) >= 3 and toks[2][0] not in (0, 1, 10, 11):
            return K["FORMAT"], toks[2][1]
        return None

    def malformed(off):
        v = values()
        kind, off = v if v is not None else (K["HEADER"], off)
        _refuse(r, data, kind, off, -1)

    def publish():
        r["n"] = toks[0][0] if toks else 0
        r["m"] = toks[1][0] if len(toks) > 1 else 0
        fmt = toks[2][0] if len(toks) > 2 else 0
        r["format"] = min(fmt, (1 << 32) - 1)
        r["has_node_weights"] = int((fmt % 100) // 10 != 0)
        r["has_edge_weights"] = int(fmt % 10 != 0)

    for t in range(3):
        if t == 2 and (i >= L or data[i] == NL):
            break
        if i >= L or not _is_digit(data[i]):
            publish()
            malformed(i)
            return None
        j = i
        while j < L and _is_digit(data[j]):
            j += 1
        toks.append((min(int(data[i:j]), CAP), i))
        i = j
        while i < L and data[i] == SP:
            i += 1
    publish()
    if i >= L or data[i] != NL:
        malformed(i)
        return None
    v = values()
    if v is not None:
        _refuse(r, data, v[0], v[1], -1)
        return None
    fmt = toks[2][0] if len(toks) > 2 else 0
    return i + 1, toks[0][0], toks[1][0], (fmt % 100) // 10 != 0, fmt % 10 != 0


def _finish(r, data, n, m2, vw, ew, lines, xadj, adj, vwgt, adjwgt, extra):
    """The end-of-file checks, the dropped weights and the arrays."""
    L = len(data)
    if lines < n:
        return _refuse(r, data, K["TOO_FEW_LINES"], L, lines)
    if int(xadj[-1]) != m2:
        return _refuse(r, data, K["EDGE_COUNT"], L, n)
    svw = int(np.sum(vwgt, dtype=np.int64)) if vw else 0
    sew = int(np.sum(adjwgt, dtype=np.int64)) if ew else 0
    if svw > I32 or sew > I32:
        return _refuse(r, data, K["TOTAL_WEIGHT"], L, n)
    r["extra_lines"] = int(extra)
    r["xadj"] = np.asarray(xadj, np.uint32)
    r["adjncy"] = np.asarray(adj, np.uint32)
    if vw and svw != n:
        r["vwgt"] = np.asarray(vwgt, np.int32)
    r["node_weights_dropped"] = int(bool(vw) and svw == n)
    if ew and sew != m2:
        r["adjwgt"] = np.asarray(adjwgt, np.int32)
    r["edge_weights_dropped"] = int(bool(ew) and sew == m2)
    return r


def parse_loop(data: bytes) -> dict:
    """The rule, line by line and byte by byte."""
    data = bytes(data)
    r = _report(data)
    h = header(data, r)
    if h is None:
        return r
    pos, n, m, vw, ew = h
    m2, L = 2 * m, len(data)
    v, extra = 0, False
    xadj, adj, vwgt, adjwgt = [0], [], [], []
    while pos < L:
        j = data.find(b"\n", pos)
        term = L if j < 0 else j
        if v >= n and data[pos] != PCT:
            extra = True
        body = data[pos:term]
        if not body.lstrip(b" ").startswith(b"%"):  # a data line: vertex v
            if v < n:
                bad, toks = [], []
                for k in range(len(body)):
                    c = body[k]
                    if _is_digit(c):
                        if k == 0 or not _is_digit(body[k - 1]):
                            e = k
                            while e < len(body) and _is_digit(body[e]):
                                e += 1
                            toks.append((pos + k, min(int(body[k:e]), CAP)))
                    elif c != SP:
                        bad.append(pos + k)
                viol = [(b, K["BAD_BYTE"]) for b in bad[:1]]
                if vw and not toks:
                    viol.append((term, K["MISSING_NODE_WEIGHT"]))
                elif ew and (len(toks) - vw) % 2:
                    viol.append((term, K["MISSING_EDGE_WEIGHT"]))
                rest = toks
                if vw and toks:
                    off, val = toks[0]
                    if val == 0:
                        viol.append((off, K["ZERO_WEIGHT"]))
                    elif val > I32:
                        viol.append((off, K["WEIGHT_TOO_LARGE"]))
                    vwgt.append(val)
                    rest = toks[1:]
                for q, (off, val) in enumerate(rest):
                    if ew and q % 2 == 1:
                        if val == 0:
                            viol.append((off, K["ZERO_WEIGHT"]))
                        elif val > I32:
                            viol.append((off, K["WEIGHT_TOO_LARGE"]))
                        adjwgt.append(val)
                    else:
                        if val == 0 or val > n:
                            viol.append((off, K["NEIGHBOR_OUT_OF_RANGE"]))
                        elif val - 1 == v:
                            viol.append((off, K["SELF_LOOP"]))
                        adj.append(val - 1)
                if viol:
                    off, kind = min(viol)
                    return _refuse(r, data, kind, off, v)
                xadj.append(len(adj))
            v += 1
        pos = L if j < 0 else j + 1
    return _finish(r, data, n, m2, vw, ew, v, xadj, adj, vwgt, adjwgt, extra)


def parse(data) -> dict:
    """The rule, vectorised over the bytes."""
    data = bytes(data) if not isinstance(data, bytes) else data
    r = _report(data)
    h = header(data, r)
    if h is None:
        return r
    base, n, m, vw, ew = h
    vw, ew = int(vw), int(ew)
    m2 = 2 * m
    d = np.frombuffer(data, np.uint8)[base:]
    N = len(d)
    nlpos = np.flatnonzero(d == NL)
    starts = np.concatenate([[0], nlpos + 1]).astype(np.int64)
    starts = starts[starts < N]
    k = np.searchsorted(nlpos, starts)
    ends = np.where(k < len(nlpos), nlpos[np.minimum(k, max(len(nlpos) - 1, 0))] if len(nlpos) else N, N)
    nonsp = np.flatnonzero(d != SP)
    k = np.searchsorted(nonsp, starts)
    fns = np.where(k < len(nonsp), nonsp[np.minimum(k, max(len(nonsp) - 1, 0))] if len(nonsp) else N, N)
    comment = (fns < ends) & (d[np.minimum(fns, max(N - 1, 0))] == PCT) if N else np.zeros(0, bool)
    dl = np.flatnonzero(~comment)
    lines = len(dl)
    vl = dl[:n]
    vs, ve = starts[vl], ends[vl]
    after = 0 if n == 0 else (int(dl[n - 1]) + 1 if lines >= n else len(starts))
    extra = bool(np.any(d[starts[after:]] != PCT))
    mark = np.zeros(N + 1, np.int64)
    np.add.at(mark, vs, 1)
    np.add.at(mark, ve, -1)
    judged = np.cumsum(mark)[:N] > 0
    digit = (d >= 48) & (d <= 57)
    bad = np.flatnonzero(judged & ~digit & (d != SP))
    prevdig = np.concatenate([[False], digit[:-1]])
    ts = np.flatnonzero(digit & ~prevdig & judged)
    nondig = np.flatnonzero(~digit)
    k = np.searchsorted(nondig, ts)
    te = np.where(k < len(nondig), nondig[np.minimum(k, max(len(nondig) - 1, 0))] if len(nondig) else N, N)
    nz = np.flatnonzero(digit & (d != 48))
    k = np.searchsorted(nz, ts)
    fnz = np.where(k < len(nz), nz[np.minimum(k, max(len(nz) - 1, 0))] if len(nz) else N, N)
    fnz = np.minimum(fnz, te)
    sig = te - fnz
    big = sig > 13
    val = np.zeros(len(ts), np.int64)
    for j in range(13):
        sel = np.flatnonzero((j < sig) & ~big)
        val[sel] = val[sel] * 10 + (d[fnz[sel] + j].astype(np.int64) - 48)
    val = np.where(big, CAP, np.minimum(val, CAP))
    first_tok = np.searchsorted(ts, vs)
    ntok = np.diff(np.append(first_tok, len(ts)))
    tv = np.searchsorted(vs, ts, side="right") - 1
    j = np.arange(len(ts)) - first_tok[tv] if len(ts) else np.zeros(0, np.int64)
    isvw = (j == 0) & bool(vw)
    r2 = ((j - vw) & 1) if ew else np.zeros(len(ts), np.int64)
    target = ~isvw & (r2 == 0)
    weight = ~isvw & (r2 == 1)
    cand = []  # (offset, kind, vertex) arrays, offsets relative to base

    def add(mask_idx, offs, kind, verts):
        if len(mask_idx):
            cand.append((offs[mask_idx], np.full(len(mask_idx), kind), verts[mask_idx]))

    vline = np.searchsorted(vs, bad, side="right") - 1
    add(np.arange(len(bad)), bad, K["BAD_BYTE"], vline)
    wtok = isvw | weight
    add(np.flatnonzero(wtok & (val == 0)), ts, K["ZERO_WEIGHT"], tv)
    add(np.flatnonzero(wtok & (val > I32)), ts, K["WEIGHT_TOO_LARGE"], tv)
    add(np.flatnonzero(target & ((val == 0) | (val > n))), ts, K["NEIGHBOR_OUT_OF_RANGE"], tv)
    add(np.flatnonzero(target & (val >= 1) & (val <= n) & (val - 1 == tv)), ts, K["SELF_LOOP"], tv)
    verts = np.arange(len(vl))
    if vw:
        add(np.flatnonzero(ntok == 0), ve, K["MISSING_NODE_WEIGHT"], verts)
    if ew:
        add(np.flatnonzero((ntok > 0 if vw else True) & ((ntok - vw) % 2 == 1)), ve, K["MISSING_EDGE_WEIGHT"], verts)
    if cand:
        offs = np.concatenate([c[0] for c in cand]).astype(np.int64)
        kinds = np.concatenate([c[1] for c in cand]).astype(np.int64)
        vts = np.concatenate([c[2] for c in cand]).astype(np.int64)
        i = int(np.lexsort((kinds, offs))[0])
        return _refuse(r, data, int(kinds[i]), base + int(offs[i]), int(vts[i]))
    nt = (ntok - vw) >> ew
    xadj = np.concatenate([[0], np.cumsum(nt)]).astype(np.int64)
    return _finish(r, data, n, m2, vw, ew, lines, xadj, val[target] - 1, val[isvw], val[weight], extra)


def as_dict(rep) -> dict:
    """A MetisReport's fields as the oracle's dict (device_ms left out)."""
    return {f: int(getattr(rep, f)) for f in REPORT}


def report_of(r: dict) -> dict:
    return {f: int(r[f]) for f in REPORT}


def equal(a: dict, b: dict) -> bool:
    """Report fields and arrays equal (arrays None on both sides or equal)."""
    if report_of(a) != report_of(b):
        return False
    for f in ("xadj", "adjncy", "vwgt", "adjwgt"):
        x, y = a.get(f), b.get(f)
        if (x is None) != (y is None) or (x is not None and not np.array_equal(np.asarray(x, np.int64), np.asarray(y, np.int64))):
            return False
    return True


def write_metis(xadj, adjncy, vwgt=None, adjwgt=None, fmt=None) -> bytes:
    """A vectorised METIS writer (graph.write_metis loops per vertex): one line per vertex, the node weight first,
    targets 1-based, each edge weight after its target, one space between tokens. `fmt` defaults to the arrays given;
    an array of ones is written as given (unit weights written explicitly)."""
    xadj = np.asarray(xadj, np.int64)
    n = len(xadj) - 1
    adj = np.asarray(adjncy, np.int64)
    vw, ew = int(vwgt is not None), int(adjwgt is not None)
    if fmt is None:
        fmt = 10 * vw + ew
    deg = np.diff(xadj)
    per_row = vw + deg * (1 + ew)
    slots = np.maximum(per_row, 1)  # an empty row is one token of no digits: its newline
    rs = np.concatenate([[0], np.cumsum(slots)])
    T = int(rs[-1])
    val = np.zeros(T, np.int64)
    nd = np.zeros(T, np.int64)
    live = np.zeros(T, bool)
    if vw:
        val[rs[:-1]] = np.asarray(vwgt, np.int64)
        live[rs[:-1]] = True
    row = np.repeat(np.arange(n), deg)
    pos = rs[:-1][row] + vw + (np.arange(len(adj)) - xadj[:-1][row]) * (1 + ew)
    val[pos] = adj + 1
    live[pos] = True
    if ew:
        val[pos + 1] = np.asarray(adjwgt, np.int64)
        live[pos + 1] = True
    nd[live] = 1
    p10 = 10
    while True:
        more = live & (val >= p10)
        if not more.any():
            break
        nd[more] += 1
        p10 *= 10
    sep = np.full(T, SP, np.uint8)
    sep[rs[1:] - 1] = NL
    head = (f"{n} {len(adj) // 2}" + (f" {fmt:02d}" if fmt else "") + "\n").encode()
    offs = len(head) + np.concatenate([[0], np.cumsum(nd + 1)[:-1]]) if T else np.zeros(0, np.int64)
    out = np.empty(len(head) + int(np.sum(nd + 1)), np.uint8)
    out[: len(head)] = np.frombuffer(head, np.uint8)
    out[offs + nd] = sep
    for k in range(int(nd.max()) if T else 0):  # digit k from the right
        sel = np.flatnonzero(nd > k)
        out[offs[sel] + nd[sel] - 1 - k] = 48 + (val[sel] // 10 ** k) % 10
    return out.tobytes()
