"""Bridge of the sparsification oracle (tests/sparsify_oracle.py, DESIGN.md §13) to the UNMODIFIED reference's
SparsificationClusterCoarsener, compiled on the host (CPU tests; skipped where the reference sources or its build
under oracle/_ref are absent). The device equals the oracle bit for bit (tests/test_gpu_sparsify.py), so what holds
for the oracle here holds for the GPU. The reference runs one coarsen() with one thread.

* NOOP clustering, laziness factor <= 1 (so that it sparsifies): the reference's first-level mapping is the identity
  on these inputs, so its coarse ids are the canonical ones, and the seed it draws is the first random_index() after
  the reseed. The oracle with that seed gives the reference's coarse graph edge for edge.
  One of the inputs is a contracted level (the committed reference contraction of R-MAT 13 with weights), so the
  rule is pinned on summed coarse edge weights, too.
* With the reference's default laziness factor 4 a level that is not dense enough is left as contracted.
* The reference's own LP clustering (a real, non-identity clustering makes the coarse ids and summed weights): the
  reference's mapping, taken as a clustering, is contracted by oracle/contraction_oracle.py. After canonicalisation
  the coarse vertices and weights are equal; T, smaller, equal and the set of edges heavier than T are equal; no kept
  edge is lighter than T. The kept edges at T are decided by a hash, per undirected pair, so their count is close to
  2 * Binomial(equal / 2, p), with mean include = target - larger and standard deviation
  sigma = sqrt(2 * equal * p * (1 - p)): the reference's count and the oracle's must both lie within 4 sigma + 2 of
  include. Inputs: R-MAT 13 with weights, grid and a random-weight R-MAT 12, which LP clusters, and the 16-vertex
  weighted RGG golden, which it leaves unclustered. The walshaw golden is not among them: the reference crashes in
  this configuration (LP clustering inside the coarsener, serial stand-in build) on that input.
"""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

from kaminpar_b200.graph import CSRGraph, random_weights, rmat
from oracle import contraction_oracle as CO
from tests import helpers as H
from tests import sparsify_oracle as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("KMP_REFERENCE", "/root/reference")
REF_LIB_DIR = os.path.join(ROOT, "oracle", "_ref")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")


@pytest.fixture(scope="module")
def bridge(tmp_path_factory):
    if not (os.path.isdir(os.path.join(REF, "kaminpar-shm")) and
            os.path.exists(os.path.join(REF_LIB_DIR, "libkaminpar_ref_full.so")) and CXX):
        pytest.skip("the reference sources / oracle/_ref/libkaminpar_ref_full.so are not present")
    so = str(tmp_path_factory.mktemp("bridge") / "ref_sparsify_bridge.so")
    cmd = [CXX, "-std=c++20", "-O2", "-fPIC", "-w", "-mcx16", "-DNDEBUG", "-shared",
           "-I" + os.path.join(ROOT, "oracle", "ref_shim"), "-I" + REF, "-I" + os.path.join(REF, "include"),
           "-I" + os.path.join(REF, "include", "kaminpar-shm"),
           os.path.join(ROOT, "tests", "cpp", "ref_sparsify_bridge.cc"),
           "-o", so, "-L" + REF_LIB_DIR, "-lkaminpar_ref_full", "-Wl,-rpath," + REF_LIB_DIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lib = C.CDLL(so)
    lib.bridge_first_draw.restype = C.c_uint64
    lib.bridge_sparsify_coarsen.restype = C.c_uint32
    return lib


def _arr(a, t):
    return None if a is None else np.ascontiguousarray(a, t).ctypes.data_as(C.c_void_p)


def ref_coarsen(lib, g, lp_clustering, laziness, seed, k=8, density=0.5, edge=0.5):
    n, m = g.n, g.m
    c_n = np.zeros(1, np.uint32)
    xadj, adj = np.zeros(n + 1, np.uint32), np.zeros(max(m, 1), np.uint32)
    vw, ew, mapping = np.zeros(max(n, 1), np.int32), np.zeros(max(m, 1), np.int32), np.zeros(max(n, 1), np.uint32)
    keep = [np.ascontiguousarray(a, t) if a is not None else None
            for a, t in ((g.xadj, np.uint32), (g.adjncy, np.uint32), (g.vwgt, np.int32), (g.adjwgt, np.int32))]
    c_m = lib.bridge_sparsify_coarsen(
        C.c_uint32(n), C.c_uint32(m), *[_arr(a, a.dtype) if a is not None else None for a in keep],
        C.c_int(lp_clustering), C.c_uint32(k), C.c_double(0.03), C.c_double(density), C.c_double(edge),
        C.c_double(laziness), C.c_int(seed), _arr(c_n, np.uint32), _arr(xadj, np.uint32), _arr(adj, np.uint32),
        _arr(vw, np.int32), _arr(ew, np.int32), _arr(mapping, np.uint32))
    cn = int(c_n[0])
    return dict(c_n=cn, c_xadj=xadj[: cn + 1].copy(), c_adjncy=adj[:c_m].copy(), c_vwgt=vw[:cn].copy(),
                c_adjwgt=ew[:c_m].copy(), mapping=mapping[:n].copy())


def ref_first_mapping(lib, g, clustering):
    out = np.zeros(g.n, np.uint32)
    keep = [np.ascontiguousarray(a, t) if a is not None else None
            for a, t in ((g.xadj, np.uint32), (g.adjncy, np.uint32), (g.vwgt, np.int32), (g.adjwgt, np.int32))]
    lib.bridge_contract_mapping(C.c_uint32(g.n), C.c_uint32(g.m), *[_arr(a, a.dtype) if a is not None else None
                                                                   for a in keep],
                                _arr(np.ascontiguousarray(clustering, np.uint32), np.uint32), _arr(out, np.uint32))
    return out


def _contracted_golden():
    d = np.load(os.path.join(H.GOLDEN, "contract_rmat13_w.npz"))
    return CSRGraph(d["c_xadj"], d["c_adjncy"], d["c_vwgt"], d["c_adjwgt"])


def _golden(name):
    return lambda: H.load_case(name)[0]


GRAPHS = {
    "walshaw": lambda: H.load_graph("walshaw_data"),
    "rgg16w": lambda: H.load_graph("rgg16_vwgt_adjwgt"),
    "rmat13_w": _golden("rmat13_w"),
    "grid12": _golden("grid12"),
    "rmat12_randw": lambda: random_weights(rmat(12, 8, 5), 3, max_vwgt=1, max_adjwgt=6),
    "rmat13_contracted": _contracted_golden,
}


def _contracted(g, cl):
    return CO.contract(g.xadj, g.adjncy, g.vwgt, g.adjwgt, cl)


@pytest.mark.parametrize("name", sorted(GRAPHS))
@pytest.mark.parametrize("laziness", [1.0, 0.5])
def test_noop_clustering_edge_for_edge(bridge, name, laziness):
    g = GRAPHS[name]()
    ident = np.arange(g.n, dtype=np.uint32)
    assert np.array_equal(ref_first_mapping(bridge, g, ident), ident), "the reference's first mapping is not the identity"
    for seed in (0, 7):
        ref = ref_coarsen(bridge, g, 0, laziness, seed)
        assert np.array_equal(ref["mapping"], ident)
        con = _contracted(g, ident)
        target = S.sparsification_target(g.m, g.n, con["c_n"])
        assert len(con["c_adjncy"]) > laziness * target  # the reference sparsified
        o = S.sparsify_contracted(con, target, bridge.bridge_first_draw(seed))
        r = CO.canonicalize(ref["c_n"], ref["c_xadj"], ref["c_adjncy"], ref["c_vwgt"], ref["c_adjwgt"],
                            ref["mapping"], ident)
        assert CO.equal(r, o), (name, seed)
        assert 0 < len(o["c_adjncy"]) < len(con["c_adjncy"])


def test_noop_lazy_level_is_the_contraction(bridge):
    """laziness 4 (the default): a level whose edge count is at most 4 x target is left as contracted."""
    g = GRAPHS["grid12"]()
    ident = np.arange(g.n, dtype=np.uint32)
    ref = ref_coarsen(bridge, g, 0, 4.0, 0)
    r = CO.canonicalize(ref["c_n"], ref["c_xadj"], ref["c_adjncy"], ref["c_vwgt"], ref["c_adjwgt"], ref["mapping"],
                        ident)
    assert CO.equal(r, _contracted(g, ident))


@pytest.mark.parametrize("name", ["rmat13_w", "grid12", "rmat12_randw", "rgg16w"])
def test_lp_clustering_threshold_and_heavy_edges(bridge, name):
    g = GRAPHS[name]()
    laziness = 0.5
    ref = ref_coarsen(bridge, g, 1, laziness, 3)
    cl = ref["mapping"]  # a clustering whose canonical coarse ids are the reference's coarse ids
    if name != "rgg16w":  # the 16-vertex weighted RGG stays unclustered under its heavy vertex weights
        assert ref["c_n"] < g.n
    con = _contracted(g, cl)
    r = CO.canonicalize(ref["c_n"], ref["c_xadj"], ref["c_adjncy"], ref["c_vwgt"], ref["c_adjwgt"], cl, cl)
    assert r["c_n"] == con["c_n"]
    assert np.array_equal(r["c_vwgt"], con["c_vwgt"]) and np.array_equal(r["mapping"], con["mapping"])
    c_m = len(con["c_adjncy"])
    target = S.sparsification_target(g.m, g.n, con["c_n"])
    assert c_m > laziness * target and 2 <= target <= c_m  # the reference sparsified
    o = S.sparsify_contracted(con, target, 12345)
    t, smaller, equal = o["threshold"], o["smaller"], o["equal"]
    con_set = S.edge_set(con["c_xadj"], con["c_adjncy"], con["c_adjwgt"])
    ref_set = S.edge_set(r["c_xadj"], r["c_adjncy"], r["c_adjwgt"])
    # the reference's threshold: its kept edges contain every edge above T and none below, so the lightest kept
    # weight is T, and smaller / equal follow from the contracted level
    ref_t = int(r["c_adjwgt"].min())
    assert ref_t == t
    assert sum(e[2] < t for e in con_set) == smaller and sum(e[2] == t for e in con_set) == equal
    assert ref_set <= con_set
    assert {e for e in ref_set if e[2] > t} == {e for e in con_set if e[2] > t}
    larger = c_m - smaller - equal
    include = target - larger
    p = include / equal
    sigma = math.sqrt(2 * equal * p * (1 - p))
    ref_eq = sum(e[2] == t for e in ref_set)
    assert abs(ref_eq - include) <= 4 * sigma + 2, (ref_eq, include, sigma)
    assert abs(o["equal_kept"] - include) <= 4 * sigma + 2, (o["equal_kept"], include, sigma)
