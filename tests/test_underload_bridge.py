"""Bridge of the order-free underload balancer (DESIGN.md §12) to the UNMODIFIED reference's UnderloadBalancer
(underload_balancer.cc), compiled on the host (CPU tests; skipped where the reference sources or its build under
oracle/_ref are absent). The device equals the oracle bit for bit (tests/test_gpu_underload.py), so what holds for
the oracle here holds for the GPU. The reference runs with one thread, PartitionContext::setup(graph, k, 0.03) and
setup_min_block_weights(0.03).

* the minimum weights: underload_oracle.min_block_weights equals what the reference's context computes;
* single-candidate inputs (exactly one vertex may leave its block for an adjacent underloaded block, and that move
  covers the deficit): the oracle moves the same vertex to the same block as the reference;
* on the golden graphs plus a contracted (weighted) level, k in {2, 4, 16, 64, 256}: the oracle reaches zero
  underload wherever the reference does, creates no overload, and its cut stays within 1.25 x the reference's + 16.
"""
import ctypes as C
import os
import shutil
import subprocess
from collections import deque

import numpy as np
import pytest

from kaminpar_b200 import lp
from kaminpar_b200.graph import CSRGraph
from tests import balance_oracle as O
from tests import helpers as H
from tests import underload_oracle as U

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("KMP_REFERENCE", "/root/reference")
REF_LIB_DIR = os.path.join(ROOT, "oracle", "_ref")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
EPS = MIN_EPS = 0.03
KS = (2, 4, 16, 64, 256)
CUT_FACTOR, CUT_SLACK = 1.25, 16


@pytest.fixture(scope="module")
def bridge(tmp_path_factory):
    if not (os.path.isdir(os.path.join(REF, "kaminpar-shm")) and
            os.path.exists(os.path.join(REF_LIB_DIR, "libkaminpar_ref_full.so")) and CXX):
        pytest.skip("the reference sources / oracle/_ref/libkaminpar_ref_full.so are not present")
    so = str(tmp_path_factory.mktemp("bridge") / "ref_underload_bridge.so")
    cmd = [CXX, "-std=c++20", "-O2", "-fPIC", "-w", "-mcx16", "-DNDEBUG", "-shared",
           "-I" + os.path.join(ROOT, "oracle", "ref_shim"), "-I" + REF, "-I" + os.path.join(REF, "include"),
           "-I" + os.path.join(REF, "include", "kaminpar-shm"),
           os.path.join(ROOT, "tests", "cpp", "ref_underload_bridge.cc"),
           "-o", so, "-L" + REF_LIB_DIR, "-lkaminpar_ref_full", "-Wl,-rpath," + REF_LIB_DIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return C.CDLL(so)


def ref_underload(lib, g, k, part, seed=0):
    p = np.ascontiguousarray(part, np.uint32).copy()
    mnw = np.zeros(k, np.int32)
    arr = lambda a, t: None if a is None else np.ascontiguousarray(a, t).ctypes.data_as(C.c_void_p)  # noqa: E731
    improved = lib.bridge_underload_balance(
        C.c_uint32(g.n), C.c_uint32(g.m), arr(g.xadj, np.uint32), arr(g.adjncy, np.uint32), arr(g.vwgt, np.int32),
        arr(g.adjwgt, np.int32), C.c_uint32(k), C.c_double(EPS), C.c_double(MIN_EPS), C.c_int(seed),
        p.ctypes.data_as(C.c_void_p), mnw.ctypes.data_as(C.c_void_p))
    return bool(improved), p, mnw


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


def _weights(g, k):
    p = lp.create_default_context().partition.setup(g, k, EPS)
    return p.max_block_weights().astype(np.int64), U.min_block_weights(p.perfectly_balanced_block_weights(), MIN_EPS)


def _single_candidate_cases(g, k, mbw, mnw, rng, want):
    """Block b = a BFS ball just below its minimum; one boundary vertex u of the ball in block s, whose weight covers
    the deficit; every other block at its minimum (nothing may leave it); s takes the rest. Kept when the oracle's
    frozen-state selection finds exactly one vertex with a target."""
    vw = np.ones(g.n, np.int64) if g.vwgt is None else g.vwgt.astype(np.int64)
    xadj = g.xadj.astype(np.int64)
    out = []
    for _ in range(30):
        if len(out) >= want:
            break
        b, s = (int(x) for x in rng.choice(k, 2, replace=False))
        part = np.full(g.n, k, np.int64)
        W = np.zeros(k, np.int64)
        seen, queue = {int(rng.integers(0, g.n))}, deque()
        queue.append(next(iter(seen)))
        while queue:  # the ball: BFS order while it stays below min[b]
            v = queue.popleft()
            if W[b] + vw[v] >= mnw[b]:
                continue
            part[v], W[b] = b, W[b] + vw[v]
            for x in g.adjncy[xadj[v]:xadj[v + 1]]:
                if int(x) not in seen:
                    seen.add(int(x))
                    queue.append(int(x))
        if W[b] == 0:
            continue
        inb = part == b
        src = np.repeat(np.arange(g.n), np.diff(xadj))
        boundary = np.unique(src[inb[g.adjncy.astype(np.int64)] & ~inb[src]])
        heavy = boundary[vw[boundary] >= mnw[b] - W[b]]
        if len(heavy) == 0:
            continue
        u = int(rng.choice(heavy))
        part[u], W[s] = s, vw[u]
        others = [c for c in range(k) if c not in (b, s)]
        oi = 0
        for v in boundary:  # the rest of the boundary into the other blocks, none above its minimum
            if part[v] != k:
                continue
            while oi < len(others) and W[others[oi]] + vw[v] > mnw[others[oi]]:
                oi += 1
            if oi == len(others):
                break
            part[v], W[others[oi]] = others[oi], W[others[oi]] + vw[v]
        if np.any(part[boundary] == k):
            continue
        pool = {}  # the other vertices by weight: top each other block up to exactly its minimum where possible
        for v in rng.permutation(np.flatnonzero(part == k)):
            pool.setdefault(int(vw[v]), []).append(int(v))
        for c in others:
            while W[c] < mnw[c] and pool:
                need = int(mnw[c] - W[c])
                fit = [w for w in pool if w <= need]
                w = need if need in pool else (max(fit) if fit else min(pool))
                v = pool[w].pop()
                if not pool[w]:
                    del pool[w]
                part[v], W[c] = c, W[c] + w
        for vs in pool.values():
            part[vs] = s
            W[s] += vw[vs].sum()
        part = part.astype(np.uint32)
        t, _ = U.underload_select_all(g, k, part, W, mbw, mnw)
        movers = np.flatnonzero(t != part)
        if list(movers) != [u] or W[s] < mnw[s] or np.any(np.delete(W, b) < np.delete(mnw, b)):
            continue
        out.append((part, u, b))
    return out


def test_min_weights_equal_reference(bridge):
    for name in ("walshaw", "rmat13_contracted"):
        g = GRAPHS[name]()
        for k in KS:
            _, mnw = _weights(g, k)
            _, _, ref_mnw = ref_underload(bridge, g, k, np.zeros(g.n, np.uint32))
            assert np.array_equal(mnw, ref_mnw), (name, k)


@pytest.mark.parametrize("name", sorted(GRAPHS))
def test_single_candidate_same_vertex_and_block(bridge, name):
    g = GRAPHS[name]()
    rng = np.random.default_rng(23)
    found = 0
    for k in (4, 16):
        mbw, mnw = _weights(g, k)
        for part, u, b in _single_candidate_cases(g, k, mbw, mnw, rng, 2):
            improved, ref, _ = ref_underload(bridge, g, k, part)
            res = U.underload_balance(g, k, part, mbw, mnw)
            assert improved and res["improved"]
            assert list(np.flatnonzero(ref != part)) == [u]
            assert list(np.flatnonzero(res["labels"] != part)) == [u]
            assert ref[u] == res["labels"][u] == b
            found += 1
    assert found >= 1, "no single-candidate inputs: the generator no longer produces the shape"


def _underloaded_inputs(g, k):
    yield "one_block", U.underload_input(g, k, 7, 0.10)
    yield "heavy_share", U.underload_input(g, k, 8, 0.40, block=k - 1)


@pytest.mark.parametrize("name", sorted(GRAPHS))
@pytest.mark.parametrize("k", KS)
def test_zero_underload_and_cut_against_reference(bridge, name, k):
    g = GRAPHS[name]()
    mbw, mnw = _weights(g, k)
    for label, part in _underloaded_inputs(g, k):
        W0 = O.block_weights(g, part, k)
        improved, ref, _ = ref_underload(bridge, g, k, part)
        res = U.underload_balance(g, k, part, mbw, mnw)
        assert improved == res["improved"]
        if U.total_underload(O.block_weights(g, ref, k), mnw) == 0:
            assert res["after"] == 0, (label, res["moved"])
        W1 = res["block_weights"].astype(np.int64)
        assert np.all((W1 <= mbw) | (W1 <= W0)), label  # no overload created
        assert O.edge_cut(g, res["labels"]) <= CUT_FACTOR * O.edge_cut(g, ref) + CUT_SLACK, label
