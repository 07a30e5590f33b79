"""Building and calling tests/cpp/ref_metis_bridge.cc: the unmodified reference's METIS reader (metis_parser.cc),
compiled here against the reference headers, the rest of the reference linked from
oracle/_ref/libkaminpar_ref_full.so. Used by tests/test_metis_bridge.py and tests/golden/make_metis_golden.py."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import re
import shutil
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("KMP_REFERENCE", "/root/reference")
REF_LIB_DIR = os.path.join(ROOT, "oracle", "_ref")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")


def available() -> bool:
    return (CXX is not None and os.path.exists(os.path.join(REF, "kaminpar-io", "metis_parser.cc"))
            and os.path.exists(os.path.join(REF_LIB_DIR, "libkaminpar_ref_full.so")))


def compile_bridge(out_dir: str, release: bool):
    """The bridge with the reader in the Release build (-DNDEBUG) or with its assertions on."""
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, f"ref_metis_bridge_{'release' if release else 'assert'}.so")
    cmd = [CXX, "-std=c++20", "-O2", "-fPIC", "-w", "-mcx16", "-shared", "-Wl,-Bsymbolic"] + \
          (["-DNDEBUG"] if release else []) + \
          ["-I" + os.path.join(ROOT, "oracle", "ref_shim"), "-I" + REF, "-I" + os.path.join(REF, "include"),
           "-I" + os.path.join(REF, "include", "kaminpar-shm"),
           os.path.join(ROOT, "tests", "cpp", "ref_metis_bridge.cc"), os.path.join(REF, "kaminpar-io", "metis_parser.cc"),
           "-o", so, "-L" + REF_LIB_DIR, "-lkaminpar_ref_full", "-Wl,-rpath," + REF_LIB_DIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lib = C.CDLL(so)
    lib.bridge_read.argtypes = [C.c_char_p, C.c_char_p, C.c_size_t]
    lib.bridge_assert.argtypes = [C.c_char_p, C.c_char_p, C.c_size_t]
    lib.bridge_sizes.argtypes = [C.c_void_p] * 4
    lib.bridge_copy.argtypes = [C.c_void_p] * 4
    return lib


def read(lib, path: str) -> dict:
    """csr_read in the Release build: None for nullopt, else the arrays (weights None when dropped) and the printed
    warning lines (colour codes and '[Warning] ' removed)."""
    msg = C.create_string_buffer(1 << 16)
    ok = lib.bridge_read(path.encode(), msg, len(msg))
    text = msg.value.decode(errors="replace")
    warnings = [re.sub(r"\x1b\[[0-9;]*m", "", ln.split("[Warning] ", 1)[1]).strip()
                for ln in text.splitlines() if "[Warning] " in ln]
    if not ok:
        return dict(graph=None, warnings=warnings)
    n, m = C.c_uint64(), C.c_uint64()
    vw, ew = C.c_int(), C.c_int()
    lib.bridge_sizes(C.byref(n), C.byref(m), C.byref(vw), C.byref(ew))
    xadj = np.zeros(n.value + 1, np.uint32)
    adj = np.zeros(m.value, np.uint32)
    vwgt = np.zeros(n.value, np.int32) if vw.value else None
    adjwgt = np.zeros(m.value, np.int32) if ew.value else None
    p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    lib.bridge_copy(p(xadj), p(adj), p(vwgt), p(adjwgt))
    return dict(graph=dict(xadj=xadj, adjncy=adj, vwgt=vwgt, adjwgt=adjwgt), warnings=warnings)


def assertion(lib, path: str):
    """The read with assertions on, in a forked child: None if it returned, else 'file:line' of the assertion."""
    where = C.create_string_buffer(512)
    rc = lib.bridge_assert(path.encode(), where, len(where))
    assert rc in (0, 3), rc
    if rc == 0:
        return None
    file, line = where.value.decode().rsplit(":", 1)
    return f"{os.path.basename(file)}:{line}"


def digest(g: dict) -> str:
    """sha256 prefix of a graph's arrays (absent weights marked)."""
    h = hashlib.sha256()
    for f, t in (("xadj", np.uint32), ("adjncy", np.uint32), ("vwgt", np.int32), ("adjwgt", np.int32)):
        a = g[f]
        h.update(b"-" if a is None else np.ascontiguousarray(a, t).tobytes() + b"|")
    return h.hexdigest()[:24]


def case_digest(data: bytes) -> str:
    return hashlib.sha256(data).hexdigest()[:24]


def skipped(name: str, kind: str) -> bool:
    """Cases the reference is not run on: TOO_FEW_LINES reads past its mapping, and a header m in [2^31, 2^32)
    passes its assertions and allocates 2^32 edge entries (the rule refuses it: edge ids are 32-bit)."""
    return kind == "TOO_FEW_LINES" or name == "too_large_m"


def verdict(rel, asr, path: str, name: str, kind: str) -> dict:
    """The reference's verdict on one file: the assertion that fires (with assertions on), and, in the Release build,
    the graph's digest and the warnings printed (files without an assertion only, and EMPTY / FORMAT)."""
    out = dict(where="", digest="", warnings="", graph=0)
    if skipped(name, kind):
        return out
    out["where"] = assertion(asr, path) or ""
    if not out["where"] or kind in ("EMPTY", "FORMAT"):
        r = read(rel, path)
        out["graph"] = int(r["graph"] is not None)
        # outside the domain (FORMAT) the Release build's arrays are garbage: only a graph's digest is kept
        out["digest"] = digest(r["graph"]) if r["graph"] is not None and kind == "OK" else ""
        out["warnings"] = "|".join(r["warnings"])
    return out
