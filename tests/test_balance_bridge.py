"""Bridge of the order-free overload balancer (DESIGN.md §11) to the UNMODIFIED reference's OverloadBalancer
(overload_balancer.cc) and compute_relative_gain (relative_gain.h), compiled on the host (CPU tests; skipped where
the reference sources or its build under oracle/_ref are absent). The device equals the oracle bit for bit
(tests/test_gpu_balance.py), so what holds for the oracle here holds for the GPU.

* the key: the oracle's float relative gain equals the reference's own function over a sweep of (gain, weight);
* single-move inputs (overload <= the lightest vertex of the block, a unique top key, a unique best target): the
  oracle moves the same vertex to the same block as the reference;
* on the golden graphs plus a contracted (weighted) level, k in {2, 4, 16, 64, 256}: the oracle reaches zero
  overload wherever the reference does, and its cut stays within 1.25 x the reference's + 16 (DESIGN.md §11).
"""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from kaminpar_b200 import lp
from kaminpar_b200.graph import CSRGraph
from tests import balance_oracle as O
from tests import helpers as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("KMP_REFERENCE", "/root/reference")
REF_LIB_DIR = os.path.join(ROOT, "oracle", "_ref")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
EPS = 0.03
KS = (2, 4, 16, 64, 256)


@pytest.fixture(scope="module")
def bridge(tmp_path_factory):
    if not (os.path.isdir(os.path.join(REF, "kaminpar-shm")) and
            os.path.exists(os.path.join(REF_LIB_DIR, "libkaminpar_ref_full.so")) and CXX):
        pytest.skip("the reference sources / oracle/_ref/libkaminpar_ref_full.so are not present")
    so = str(tmp_path_factory.mktemp("bridge") / "ref_balance_bridge.so")
    cmd = [CXX, "-std=c++20", "-O2", "-fPIC", "-w", "-mcx16", "-DNDEBUG", "-shared",
           "-I" + os.path.join(ROOT, "oracle", "ref_shim"), "-I" + REF, "-I" + os.path.join(REF, "include"),
           "-I" + os.path.join(REF, "include", "kaminpar-shm"), os.path.join(ROOT, "tests", "cpp", "ref_balance_bridge.cc"),
           "-o", so, "-L" + REF_LIB_DIR, "-lkaminpar_ref_full", "-Wl,-rpath," + REF_LIB_DIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lib = C.CDLL(so)
    lib.bridge_relative_gain.restype = C.c_float
    lib.bridge_relative_gain.argtypes = [C.c_int32, C.c_int32]
    return lib


def ref_balance(lib, g, k, part, seed=0):
    p = np.ascontiguousarray(part, np.uint32).copy()
    arr = lambda a, t: None if a is None else np.ascontiguousarray(a, t).ctypes.data_as(C.c_void_p)  # noqa: E731
    improved = lib.bridge_overload_balance(
        C.c_uint32(g.n), C.c_uint32(g.m), arr(g.xadj, np.uint32), arr(g.adjncy, np.uint32), arr(g.vwgt, np.int32),
        arr(g.adjwgt, np.int32), C.c_uint32(k), C.c_double(EPS), C.c_int(seed), p.ctypes.data_as(C.c_void_p))
    return bool(improved), p


def _contracted():
    d = np.load(os.path.join(H.GOLDEN, "contract_rmat13_w.npz"))
    return CSRGraph(d["c_xadj"], d["c_adjncy"], d["c_vwgt"], d["c_adjwgt"])


GRAPHS = {
    "walshaw": lambda: H.load_graph("walshaw_data"),
    "rgg16": lambda: H.load_graph("rgg16"),
    "rgg16w": lambda: H.load_graph("rgg16_vwgt_adjwgt"),
    "rgg2d": lambda: H.load_graph("rgg2d"),
    "rmat13_contracted": _contracted,
}


def _ctx(g, k):
    return lp.create_default_context().partition.setup(g, k, EPS)


def test_relative_gain_equals_reference(bridge):
    gains = [-(1 << 31), -(1 << 24) - 1, -(1 << 24), -12345, -2, -1, 0, 1, 2, 7, 12345, (1 << 24) - 1, 1 << 24,
             (1 << 24) + 1, (1 << 31) - 1]
    weights = [1, 2, 3, 7, 1000, (1 << 24) - 1, 1 << 24, (1 << 24) + 1, (1 << 31) - 1]
    G, W = np.meshgrid(np.array(gains, np.int64), np.array(weights, np.int64))
    ours = O.relative_gain(G.ravel(), W.ravel()).view(np.uint32)
    ref = np.array([bridge.bridge_relative_gain(int(a), int(b)) for a, b in zip(G.ravel(), W.ravel())], np.float32)
    assert np.array_equal(ours, ref.view(np.uint32))


def _single_move_cases(g, k, mref, rng, want):
    """Inputs under the reference's own maxima: every block but b within its maximum, b over it by at most its
    lightest vertex (a single move covers it), a unique top key in b and a unique best target of that vertex."""
    vw = np.ones(g.n, np.int64) if g.vwgt is None else g.vwgt.astype(np.int64)
    out = []
    for _ in range(80):
        if len(out) >= want:
            break
        part = (rng.permutation(g.n) % k).astype(np.uint32)
        b = int(rng.integers(0, k))
        others = rng.permutation(np.flatnonzero(part != b))
        W = O.block_weights(g, part, k)
        for v in others:  # fill b until it just exceeds its maximum
            if W[b] > mref[b]:
                break
            W[part[v]] -= vw[v]
            W[b] += vw[v]
            part[v] = b
        inb = part == b
        if W[b] <= mref[b] or np.any(np.delete(W - mref, b) > 0) or W[b] - mref[b] > vw[inb].min():
            continue
        cand = np.flatnonzero(inb)
        t, gain, key = O.best_targets(g, k, part, W, mref, 0, cand)
        top = np.flatnonzero(key == key.max())
        if len(top) != 1 or t[top[0]] == b:
            continue
        u = int(cand[top[0]])
        conn = {}
        for e in range(int(g.xadj[u]), int(g.xadj[u + 1])):
            c = int(part[g.adjncy[e]])
            conn[c] = conn.get(c, 0) + (1 if g.adjwgt is None else int(g.adjwgt[e]))
        feas = sorted((v - conn.get(b, 0) for c, v in conn.items() if c != b and W[c] + vw[u] <= mref[c]), reverse=True)
        if len(feas) > 1 and feas[0] == feas[1]:
            continue
        out.append((part, u, int(t[top[0]])))
    return out


@pytest.mark.parametrize("name", sorted(GRAPHS))
def test_single_move_same_vertex_and_block(bridge, name):
    g = GRAPHS[name]()
    rng = np.random.default_rng(17)
    found = 0
    for k in (2, 4, 16, 64):
        p = _ctx(g, k)
        mref, pbw = p.max_block_weights().astype(np.int64), p.perfectly_balanced_block_weights()
        for part, u, t in _single_move_cases(g, k, mref, rng, 2):
            improved, ref = ref_balance(bridge, g, k, part)
            res = O.overload_balance(g, k, part, mref, pbw)
            assert improved and res["improved"]
            assert list(np.flatnonzero(ref != part)) == [u]
            assert list(np.flatnonzero(res["labels"] != part)) == [u]
            assert ref[u] == res["labels"][u] == t
            found += 1
    assert found >= 1, "no single-move inputs: the generator no longer produces the shape"


def _overloaded_inputs(g, k):
    yield "one_block", O.overload_input(g, k, 7, 0.10, (0,))
    yield "three_blocks", O.overload_input(g, k, 8, 0.20, tuple(range(min(3, k))))


CUT_FACTOR, CUT_SLACK = 1.25, 16


@pytest.mark.parametrize("name", sorted(GRAPHS))
@pytest.mark.parametrize("k", KS)
def test_zero_overload_and_cut_against_reference(bridge, name, k):
    g = GRAPHS[name]()
    p = _ctx(g, k)
    mref, pbw = p.max_block_weights().astype(np.int64), p.perfectly_balanced_block_weights()
    for label, part in _overloaded_inputs(g, k):
        improved, ref = ref_balance(bridge, g, k, part)
        res = O.overload_balance(g, k, part, mref, pbw)
        assert improved == res["improved"]
        ref_over = int(np.maximum(O.block_weights(g, ref, k) - mref, 0).sum())
        if ref_over == 0:
            assert res["after"] == 0, (label, res["moved"])
        assert O.edge_cut(g, res["labels"]) <= CUT_FACTOR * O.edge_cut(g, ref) + CUT_SLACK, label
