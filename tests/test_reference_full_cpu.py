"""CPU: the whole UNMODIFIED reference partitioner (oracle/_ref/libkaminpar_ref_full.so: every kaminpar-shm /
kaminpar-common translation unit on the serial oneTBB stand-in, `make -C oracle ref_full`) through the same C entry
point the GPU-integrated build exports (integration/partition_driver.cc). Pins the harness of
tests/test_gpu_integration.py against the reference's own end-to-end properties
(tests/endtoend/shm_endtoend_test.cc:142-247)."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import bindings as B
from tests import helpers as H

LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libkaminpar_ref_full.so")


def test_reference_compute_partition_properties():
    if not os.path.exists(LIB):
        pytest.skip("oracle/_ref/libkaminpar_ref_full.so not built (needs /root/reference)")
    lib = C.CDLL(LIB)
    lib.kmpfull_compute_partition.restype = C.c_longlong

    def run(g, k, seed=0):
        out = np.zeros(g.n, np.uint32)
        cut = lib.kmpfull_compute_partition(C.c_uint32(g.n), g.xadj.ctypes.data_as(C.c_void_p),
                                            g.adjncy.ctypes.data_as(C.c_void_p), None, None, C.c_uint32(k),
                                            C.c_double(0.03), C.c_int(seed), C.c_int(1), out.ctypes.data_as(C.c_void_p))
        return int(cut), out

    g = H.load_graph("walshaw_data")
    cut, p = run(g, 16)
    assert (p < 16).all() and cut == B.oracle_edge_cut(g, p) and cut <= 2000
    cut2, p2 = run(g, 16)
    assert np.array_equal(p, p2)
    _, p3 = run(g, 16, seed=1)
    assert not np.array_equal(p, p3)
    g = H.load_graph("rgg2d")
    cut, p = run(g, 4)
    assert g.n == 1024 and g.m == 8226 and cut == B.oracle_edge_cut(g, p)
