"""The unmodified reference's ParHIP reader on a corpus of small files, through the program oracle/_ref/parhip_read
(oracle/ref_parhip_read.cc + kaminpar-io/parhip_parser.cc, Release build), and the corpus itself.

    corpus() -> [(name, bytes)]   valid 32-bit files (weights present or not, unit weights, isolated vertices, a hub,
                                  n = 0, m = 0, high version bits, trailing bytes) and the same graphs at 64-bit widths
    run(data, ordering)           the reference's read: dict(exit, xadj, adjncy, vwgt, adjwgt, old_to_new, sorted), or
                                  dict(exit, log) when it exited with an error, or None where it was not built
Files outside the parity domain are never handed to the reference: it would read outside its mapping."""
import os
import re
import subprocess
import tempfile

import numpy as np

from tests import parhip_oracle as PO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "parhip_read")
GOLDEN = os.path.join(ROOT, "tests", "golden", "parhip_cases.npz")


def _graph(n, deg, seed, isolated=0):
    rng = np.random.default_rng(seed)
    src = rng.integers(0, n, n * deg // 2)
    dst = rng.integers(0, n, n * deg // 2)
    keep = src != dst
    a = np.concatenate([src[keep], dst[keep]])
    b = np.concatenate([dst[keep], src[keep]])
    key = np.unique(a * n + b)
    u, v = key // n, key % n
    u = u + isolated * (u >= n // 2)  # a run of isolated vertices in the middle
    v = v + isolated * (v >= n // 2)
    N = n + isolated
    xadj = np.zeros(N + 1, np.int64)
    np.add.at(xadj, u + 1, 1)
    return np.cumsum(xadj), v, rng


def corpus():
    out = []
    x, adj, rng = _graph(300, 6, 1, isolated=40)
    n, m = len(x) - 1, len(adj)
    vw, ew = rng.integers(1, 50, n), rng.integers(1, 1000, m)
    out.append(("plain", PO.write(x, adj)))
    out.append(("weighted", PO.write(x, adj, vw, ew)))
    out.append(("node_weights", PO.write(x, adj, vw, None)))
    out.append(("edge_weights", PO.write(x, adj, None, ew)))
    out.append(("unit_weights", PO.write(x, adj, np.ones(n), np.ones(m))))
    out.append(("high_bits_trailing", PO.write(x, adj, vw, ew, PO.version_of(True, True, high=0x3FF)) + b"\x00" * 9))
    hx = np.concatenate([[0, 2000], 2000 + np.arange(1, 2001)])  # a hub of degree 2000 and its leaves
    hadj = np.concatenate([np.arange(1, 2001), np.zeros(2000, np.int64)])
    out.append(("hub", PO.write(hx, hadj, None, rng.integers(1, 9, len(hadj)))))
    out.append(("m0", PO.write(np.zeros(6, np.int64), [], np.arange(1, 6), [])))
    out.append(("n0", PO.write([0], [])))
    out.append(("rgg2d", open(os.path.join(ROOT, "tests", "golden", "misc", "rgg2d-32bit.parhip"), "rb").read()))
    for name, data in list(out):  # the same graphs at 64-bit widths, which the reference's build refuses
        r = PO.read(data)
        v = r["version"] & 3
        out.append((name + "_64", PO.write(r["xadj"], r["adjncy"], r["vwgt"], r["adjwgt"], v)))
    r = PO.read(dict(out)["weighted"])  # one 64-bit width at a time: each of validate's four refusals
    for tag, widths in (("offsets", dict(offsets64=True)), ("vwgt", dict(vw64=True)), ("adjwgt", dict(ew64=True))):
        out.append((f"weighted_64{tag}", PO.write(r["xadj"], r["adjncy"], r["vwgt"], r["adjwgt"],
                                                  PO.version_of(True, True, **widths))))
    return out


def run(data: bytes, ordering: int):
    if not os.path.exists(REF):
        return None
    with tempfile.TemporaryDirectory() as d:
        path, dump = os.path.join(d, "g.parhip"), os.path.join(d, "g.bin")
        with open(path, "wb") as f:
            f.write(data)
        p = subprocess.run([REF, path, str(ordering), dump], capture_output=True, text=True)
        if p.returncode != 0:  # the log line the reference printed before it exited, without its colours
            return dict(exit=p.returncode, log=re.sub(r"\x1b\[[0-9;]*m", "", p.stdout + p.stderr).strip())
        raw = np.fromfile(dump, np.uint8)
    n, m, srt, hv, he, perm = (int(x) for x in raw[:48].view("<u8"))
    words = raw[48:].view("<u4")
    out = dict(exit=0, sorted=srt, xadj=words[:n + 1].copy())
    at = n + 1
    out["adjncy"] = words[at:at + m].copy()
    at += m
    out["vwgt"] = words[at:at + n].view("<i4").copy() if hv else None
    at += n if hv else 0
    out["adjwgt"] = words[at:at + m].view("<i4").copy() if he else None
    at += m if he else 0
    out["old_to_new"] = words[at:at + n].copy() if perm else None
    return out
