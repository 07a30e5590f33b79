"""Bridge of the overlay oracle (tests/overlay_oracle.py, DESIGN.md §14) to the UNMODIFIED reference's
OverlayClusterCoarsener, compiled on the host (CPU tests; skipped where the reference sources or its build under
oracle/_ref are absent). The device equals the oracle bit for bit (tests/test_gpu_overlay.py), so what holds for the
oracle here holds for the GPU.

The reference runs one coarsen() with one thread and its own LP clusterer, for num_levels L in {1, 2} and two seeds.
Next to it a standalone reference LP clusterer, reseeded the same way and given the same max cluster weight, computes
2^L consecutive clusterings. Then:
  * the reference's own contract_clustering of overlay_tree(clusterings) is the coarsener's level exactly (coarse CSR,
    vertex weights and mapping): the tree order and the ids of the oracle are the reference's;
  * the oracle contraction of overlay_tree(clusterings) equals that level after canonicalize();
  * max_level = 0 still overlays on the first level (level() = 0), while with L = 0 the level is the contraction of
    the first clustering. A negative max_level is compared as std::size_t in the reference and never disables the
    overlay; kaminpar_b200.contraction.overlay_level mirrors that.
Inputs: the golden graphs rgg2d, rgg16 (vertex and edge weights) and walshaw, and a grid. No input is left out: the
serial stand-in build of the reference runs this coarsener on all of them (unlike the sparsification coarsener on
walshaw, tests/test_sparsify_bridge.py).
"""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import contraction_oracle as CO
from tests import helpers as H
from tests import overlay_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("KMP_REFERENCE", "/root/reference")
REF_LIB_DIR = os.path.join(ROOT, "oracle", "_ref")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
K, EPS = 8, 0.03


@pytest.fixture(scope="module")
def bridge(tmp_path_factory):
    if not (os.path.isdir(os.path.join(REF, "kaminpar-shm")) and
            os.path.exists(os.path.join(REF_LIB_DIR, "libkaminpar_ref_full.so")) and CXX):
        pytest.skip("the reference sources / oracle/_ref/libkaminpar_ref_full.so are not present")
    so = str(tmp_path_factory.mktemp("bridge") / "ref_overlay_bridge.so")
    cmd = [CXX, "-std=c++20", "-O2", "-fPIC", "-w", "-mcx16", "-DNDEBUG", "-shared",
           "-I" + os.path.join(ROOT, "oracle", "ref_shim"), "-I" + REF, "-I" + os.path.join(REF, "include"),
           "-I" + os.path.join(REF, "include", "kaminpar-shm"),
           os.path.join(ROOT, "tests", "cpp", "ref_overlay_bridge.cc"),
           "-o", so, "-L" + REF_LIB_DIR, "-lkaminpar_ref_full", "-Wl,-rpath," + REF_LIB_DIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lib = C.CDLL(so)
    lib.bridge_contract.restype = C.c_uint32
    lib.bridge_overlay_coarsen.restype = C.c_uint32
    return lib


def _arr(a, t):
    return None if a is None else np.ascontiguousarray(a, t).ctypes.data_as(C.c_void_p)


def _graph_args(g):
    keep = [None if a is None else np.ascontiguousarray(a, t)
            for a, t in ((g.xadj, np.uint32), (g.adjncy, np.uint32), (g.vwgt, np.int32), (g.adjwgt, np.int32))]
    return keep, [C.c_uint32(g.n), C.c_uint32(g.m)] + [None if a is None else _arr(a, a.dtype) for a in keep]


def _level(call, n, m):
    c_n = np.zeros(1, np.uint32)
    xadj, adj = np.zeros(n + 1, np.uint32), np.zeros(max(m, 1), np.uint32)
    vw, ew, mapping = np.zeros(max(n, 1), np.int32), np.zeros(max(m, 1), np.int32), np.zeros(max(n, 1), np.uint32)
    c_m = call(_arr(c_n, np.uint32), _arr(xadj, np.uint32), _arr(adj, np.uint32), _arr(vw, np.int32),
               _arr(ew, np.int32), _arr(mapping, np.uint32))
    cn = int(c_n[0])
    return dict(c_n=cn, c_xadj=xadj[: cn + 1].copy(), c_adjncy=adj[:c_m].copy(), c_vwgt=vw[:cn].copy(),
                c_adjwgt=ew[:c_m].copy(), mapping=mapping[:n].copy())


def ref_clusterings(lib, g, seed, count):
    keep, args = _graph_args(g)
    out = np.zeros((count, g.n), np.uint32)
    lib.bridge_lp_clusterings(*args, C.c_uint32(K), C.c_double(EPS), C.c_int(seed), C.c_int(count), _arr(out, np.uint32))
    return out


def ref_contract(lib, g, clustering):
    keep, args = _graph_args(g)
    cl = np.ascontiguousarray(clustering, np.uint32)
    return _level(lambda *o: lib.bridge_contract(*args, _arr(cl, np.uint32), *o), g.n, g.m)


def ref_coarsen(lib, g, num_levels, max_level, seed):
    keep, args = _graph_args(g)
    return _level(lambda *o: lib.bridge_overlay_coarsen(*args, C.c_uint32(K), C.c_double(EPS), C.c_int(num_levels),
                                                        C.c_int(max_level), C.c_int(seed), *o), g.n, g.m)


def inputs():
    yield "rgg2d", H.load_graph("rgg2d")
    yield "rgg16_vwgt_adjwgt", H.load_graph("rgg16_vwgt_adjwgt")
    yield "walshaw_data", H.load_graph("walshaw_data")
    yield "grid40", H.grid2d(40, 40)


INPUTS = dict(inputs())


@pytest.mark.parametrize("name", sorted(INPUTS))
@pytest.mark.parametrize("levels", [1, 2])
@pytest.mark.parametrize("seed", [0, 7])
def test_coarsener_level_is_the_contracted_overlay_tree(bridge, name, levels, seed):
    g = INPUTS[name]
    cls = ref_clusterings(bridge, g, seed, 1 << levels)
    ov = O.overlay_tree(list(cls))
    level = ref_coarsen(bridge, g, levels, 2**31 - 1, seed)
    assert CO.equal(level, ref_contract(bridge, g, ov))
    oracle = CO.contract(g.xadj, g.adjncy, g.vwgt, g.adjwgt, ov)
    keys = ("c_n", "c_xadj", "c_adjncy", "c_vwgt", "c_adjwgt", "mapping")
    assert CO.equal(CO.canonicalize(*(level[key] for key in keys), ov), oracle)
    if g.n > 100:  # the overlay is a real intersection on these inputs
        assert level["c_n"] > len(np.unique(cls[0]))


@pytest.mark.parametrize("name", sorted(INPUTS))
def test_max_level_and_no_overlay(bridge, name):
    g = INPUTS[name]
    cls = ref_clusterings(bridge, g, 7, 2)
    # level() is 0 on the first coarsen(): max_level = 0 still overlays, and so does a negative max_level
    for max_level in (0, -1):
        assert CO.equal(ref_coarsen(bridge, g, 1, max_level, 7), ref_contract(bridge, g, O.overlay_tree(list(cls))))
    assert CO.equal(ref_coarsen(bridge, g, 0, 2**31 - 1, 7), ref_contract(bridge, g, cls[0]))
