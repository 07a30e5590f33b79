"""-m gpu: the drop-in claim, compiled and run. oracle/_ref/libkaminpar_ref_b200.so is the UNMODIFIED reference
partitioner (every kaminpar-shm / kaminpar-common translation unit) whose factories.cc returns the GPU glue
classes for the two LABEL_PROPAGATION cases (integration/, INTEGRATION.md §2; `make -C oracle ref_b200`), linked
against libkaminpar_b200.so. KaMinPar::compute_partition then coarsens with the GPU LP clusterer and refines with
the GPU LP refiner on every level, everything else (contraction, initial partitioning, balancers) is the reference.

Asserted: the reference's own end-to-end properties (tests/endtoend/shm_endtoend_test.cc:142-247) and the
quality next to the pure-CPU reference build (libkaminpar_ref_full.so)."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import bindings as B
from tests import helpers as H

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_B200 = os.path.join(ROOT, "oracle", "_ref", "libkaminpar_ref_b200.so")
LIB_FULL = os.path.join(ROOT, "oracle", "_ref", "libkaminpar_ref_full.so")


def _load(path):
    if not os.path.exists(path):
        pytest.skip(f"{path} not built (needs /root/reference at build time: make -C oracle ref_full ref_b200)")
    lib = C.CDLL(path)
    lib.kmpfull_compute_partition.restype = C.c_longlong
    return lib


def partition(lib, g, k, eps=0.03, seed=0):
    out = np.zeros(g.n, np.uint32)
    cut = lib.kmpfull_compute_partition(
        C.c_uint32(g.n), g.xadj.ctypes.data_as(C.c_void_p), g.adjncy.ctypes.data_as(C.c_void_p),
        None if g.vwgt is None else g.vwgt.ctypes.data_as(C.c_void_p),
        None if g.adjwgt is None else g.adjwgt.ctypes.data_as(C.c_void_p), C.c_uint32(k), C.c_double(eps),
        C.c_int(seed), C.c_int(1), out.ctypes.data_as(C.c_void_p))
    return int(cut), out


@pytest.mark.parametrize("name,k,cut_bound", [("rgg2d", 4, None), ("walshaw_data", 16, 2000), ("rgg16", 8, None)])
def test_compute_partition_through_swapped_factories(name, k, cut_bound):
    g = H.load_graph(name)
    lib = _load(LIB_B200)
    cut, p = partition(lib, g, k)
    assert len(p) == g.n and (p < k).all()                       # test_pykaminpar.py:95-104
    assert cut == B.oracle_edge_cut(g, p)                        # shm_endtoend_test.cc:142-173: reported == recomputed
    if cut_bound is not None:
        assert cut <= cut_bound                                  # :170 (Walshaw data, k = 16, eps = 0.03, seed 0)
    w = np.ones(g.n, np.int64) if g.vwgt is None else g.vwgt.astype(np.int64)
    bw = np.bincount(p, weights=w, minlength=k)
    assert bw.max() <= (1 + 0.03) * np.ceil(w.sum() / k) + w.max()   # feasible up to the max node weight
    cut2, p2 = partition(lib, g, k)
    assert cut2 == cut and np.array_equal(p, p2)                 # :189-217 same seed, same partition
    cut3, p3 = partition(lib, g, k, seed=1)
    assert not np.array_equal(p, p3)                             # :219-247 different seed, different partition
    ref_cut, _ = partition(_load(LIB_FULL), g, k)
    print(f"{name} k={k}: cut with the GPU LP {cut}, pure reference {ref_cut}")
    assert cut <= 1.25 * ref_cut + 16


def test_python_facade_over_the_integrated_build():
    """integration.facade.KaMinPar mirrors the reference's facade (kaminpar.h:857-997) on top of the integrated
    build: copy_graph / set_k / set_uniform_max_block_weights / compute_partition / reseed."""
    if not os.path.exists(LIB_B200):
        pytest.skip("integrated build not available")
    from integration.facade import KaMinPar

    g = H.load_graph("walshaw_data")
    KaMinPar.reseed(0)
    shm = KaMinPar(num_threads=1)
    shm.copy_graph(g.xadj, g.adjncy)
    shm.set_k(16)
    shm.set_uniform_max_block_weights(0.03)
    cut, part = shm.compute_partition()
    assert (part < 16).all() and cut == B.oracle_edge_cut(g, part) and cut <= 2000
    cut2, part2 = shm.compute_partition()
    assert cut2 == cut and np.array_equal(part, part2)
