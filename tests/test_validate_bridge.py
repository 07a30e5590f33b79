"""CPU: the validation oracle (tests/validate_oracle.py) against the UNMODIFIED reference's two validators, called
through tests/cpp/ref_validate_bridge.cc (compiled here against the reference headers, linked against
oracle/_ref/libkaminpar_ref_full.so; skipped where either is absent):
  - verdict and warning line of debug::validate_graph (csr_graph.cc:266-356) equal the oracle's `valid` and
    message() on every case of the corpus whose shape the reference can read (xadj[0] == 0, xadj[n] == m);
  - validate_undirected_graph's exit status (the CLI's --validate, run in a forked child since it calls exit(1))
    equals `valid and duplicates == 0` on graphs with in-range targets, no self-loops and duplicates (if any) next to
    each other in their row; on a row such as [a, b, a] the reference passes and the oracle flags a duplicate."""
import ctypes as C
import hashlib
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from tests import validate_oracle as V

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("KMP_REFERENCE", "/root/reference")
REF_LIB_DIR = os.path.join(ROOT, "oracle", "_ref")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")


def corpus():
    cases = []
    for base in V.small_bases() + V.empty_graphs():
        cases.append(base)
        if len(base[2]):
            cases += V.mutations(*base)
        cases += V.broken_xadj(*base)
    return cases


def digest(xadj, adj, w):
    h = hashlib.sha256()
    for a in (xadj, adj, w):
        h.update(b"-" if a is None else np.ascontiguousarray(a).tobytes() + b"|")
    return h.hexdigest()[:16]


def shape_ok(xadj, adj):
    return int(xadj[0]) == 0 and int(xadj[-1]) == len(adj)


def in_undirected_domain(xadj, adj):
    if not shape_ok(xadj, adj) or np.any(np.diff(xadj.astype(np.int64)) < 0):
        return False
    n = len(xadj) - 1
    for u in range(n):
        row = adj[xadj[u]:xadj[u + 1]].astype(np.int64)
        if np.any(row >= n) or np.any(row == u):
            return False
        vals, first, counts = np.unique(row, return_index=True, return_counts=True)
        last = np.array([np.nonzero(row == x)[0][-1] for x in vals[counts > 1]], np.int64)
        if np.any(last - first[counts > 1] + 1 != counts[counts > 1]):
            return False  # a duplicate not next to its first occurrence
    return True


def compile_bridge(out_dir):
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "ref_validate_bridge.so")
    cmd = [CXX, "-std=c++20", "-O2", "-fPIC", "-w", "-mcx16", "-DNDEBUG", "-shared",
           "-I" + os.path.join(ROOT, "oracle", "ref_shim"), "-I" + REF, "-I" + os.path.join(REF, "include"),
           "-I" + os.path.join(REF, "include", "kaminpar-shm"),
           os.path.join(ROOT, "tests", "cpp", "ref_validate_bridge.cc"),
           "-o", so, "-L" + REF_LIB_DIR, "-lkaminpar_ref_full", "-Wl,-rpath," + REF_LIB_DIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return C.CDLL(so)


def _p(a):
    return None if a is None else np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)


def reference_validate(bridge, xadj, adj, w):
    """(verdict, warning line without colour codes, "[Warning] " and newline) of debug::validate_graph."""
    buf = C.create_string_buffer(4096)
    ok = bridge.bridge_validate_graph(C.c_uint32(len(xadj) - 1), C.c_uint32(len(adj)), _p(xadj), _p(adj), _p(w), buf,
                                      C.c_size_t(len(buf)))
    text = re.sub(r"\x1b\[[0-9;]*m", "", buf.value.decode()).strip()
    return ok, text.removeprefix("[Warning] ")


def reference_undirected(bridge, xadj, adj, w):
    return bridge.bridge_validate_undirected(C.c_uint32(len(xadj) - 1), C.c_uint32(len(adj)), _p(xadj), _p(adj), _p(w))


@pytest.fixture(scope="module")
def bridge():
    if not (os.path.isdir(os.path.join(REF, "kaminpar-shm")) and
            os.path.exists(os.path.join(REF_LIB_DIR, "libkaminpar_ref_full.so")) and CXX):
        pytest.skip("the reference sources / oracle/_ref/libkaminpar_ref_full.so are not present")
    with tempfile.TemporaryDirectory() as d:
        yield compile_bridge(d)


CASES = corpus()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_oracle_equals_reference_validate_graph(bridge, case):
    _, xadj, adj, w = case
    r = V.validate(xadj, adj, w)
    assert V.as_dict(V.validate_loop(xadj, adj, w)) == V.as_dict(r)
    if not shape_ok(xadj, adj):
        assert r["kind"] in (V.XADJ_START, V.XADJ_END) and not r["valid"]
        return
    ok, msg = reference_validate(bridge, xadj, adj, w)
    assert ok == r["valid"]
    assert msg == V.message(r)


UNDIRECTED = [c for c in CASES if in_undirected_domain(c[1], c[2])]


@pytest.mark.parametrize("case", UNDIRECTED, ids=[c[0] for c in UNDIRECTED])
def test_oracle_equals_reference_validate_undirected_graph(bridge, case):
    _, xadj, adj, w = case
    r = V.validate(xadj, adj, w)
    assert reference_undirected(bridge, xadj, adj, w) == (0 if r["valid"] and r["duplicates"] == 0 else 1)


def test_apart_duplicates_pass_the_reference_cli_check_but_are_counted(bridge):
    apart = [c for c in CASES if c[0].endswith("/dup_apart")]
    assert apart
    for _, xadj, adj, w in apart:
        r = V.validate(xadj, adj, w)
        assert r["valid"] and r["duplicates"] == 2
        assert reference_undirected(bridge, xadj, adj, w) == 0
