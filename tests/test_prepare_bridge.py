"""CPU: the oracle's finish (tests/prepare_oracle.py) against the UNMODIFIED reference's graph::assign_isolated_nodes,
called directly on crafted states through tests/cpp/ref_prepare_bridge.cc (compiled here against the reference
headers, linked against oracle/_ref/libkaminpar_ref_full.so; skipped where either is absent): a block already above
its maximum, zero-weight isolated vertices, k = 1, and weights that fit a block exactly."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests import prepare_oracle as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("KMP_REFERENCE", "/root/reference")
REF_LIB_DIR = os.path.join(ROOT, "oracle", "_ref")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")


@pytest.fixture(scope="module")
def bridge(tmp_path_factory):
    if not (os.path.isdir(os.path.join(REF, "kaminpar-shm")) and
            os.path.exists(os.path.join(REF_LIB_DIR, "libkaminpar_ref_full.so")) and CXX):
        pytest.skip("the reference sources / oracle/_ref/libkaminpar_ref_full.so are not present")
    so = str(tmp_path_factory.mktemp("bridge") / "ref_prepare_bridge.so")
    cmd = [CXX, "-std=c++20", "-O2", "-fPIC", "-w", "-mcx16", "-DNDEBUG", "-shared",
           "-I" + os.path.join(ROOT, "oracle", "ref_shim"), "-I" + REF, "-I" + os.path.join(REF, "include"),
           "-I" + os.path.join(REF, "include", "kaminpar-shm"),
           os.path.join(ROOT, "tests", "cpp", "ref_prepare_bridge.cc"),
           "-o", so, "-L" + REF_LIB_DIR, "-lkaminpar_ref_full", "-Wl,-rpath," + REF_LIB_DIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return C.CDLL(so)


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def sorted_cycle_with_isolated(n_prime, ni):
    """A cycle over the first n' >= 3 vertices (all of degree 2: the graph is sorted by degree bucket as it stands)
    and ni isolated vertices after them."""
    adj = []
    xadj = [0]
    for u in range(n_prime):
        adj += sorted(((u - 1) % n_prime, (u + 1) % n_prime))
        xadj.append(len(adj))
    xadj += [len(adj)] * ni
    return np.array(xadj, np.uint32), np.array(adj, np.uint32)


STATES = [
    # name, n', vwgt, k, max block weights, partition of the n' vertices
    ("block0_over_max", 6, [5, 5, 5, 1, 1, 1, 2, 2, 2, 2, 2], 3, [10, 8, 8], [0, 0, 0, 1, 2, 2]),
    ("zero_weight_isolated", 4, [1, 1, 1, 1, 0, 0, 3, 0, 2, 0], 2, [3, 5], [0, 0, 1, 1]),
    ("k1", 4, [1, 2, 3, 4, 5, 6, 7], 1, [10], [0, 0, 0, 0]),
    ("exact_fit", 4, [2, 2, 2, 2, 2, 4, 1, 3, 2], 3, [6, 6, 8], [0, 1, 1, 2]),
    ("unit_weights", 8, None, 4, [4, 4, 4, 4], [0, 0, 1, 1, 1, 2, 2, 3]),
    ("all_blocks_full", 6, [3, 3, 3, 3, 3, 3, 1, 1, 1], 3, [6, 6, 6], [0, 0, 1, 1, 2, 2]),
]


@pytest.mark.parametrize("state", STATES, ids=[s[0] for s in STATES])
def test_oracle_finish_equals_reference_assign_isolated_nodes(bridge, state):
    _, n_prime, vwgt, k, mbw, part = state
    n = n_prime + (len(vwgt) - n_prime if vwgt is not None else 5)
    ni = n - n_prime
    xadj, adj = sorted_cycle_with_isolated(n_prime, ni)
    vw = None if vwgt is None else np.array(vwgt, np.int32)
    mbw = np.array(mbw, np.int32)
    part = np.array(part, np.uint32)
    out = np.zeros(n, np.uint32)
    bw = np.zeros(k, np.int32)
    rc = bridge.bridge_assign_isolated_nodes(C.c_uint32(n), C.c_uint32(len(adj)), _p(xadj), _p(adj), _p(vw),
                                             C.c_uint32(ni), C.c_uint32(k), _p(mbw), _p(part), _p(out), _p(bw))
    assert rc == 0
    prep = P.rearrange(xadj, adj, vw)  # already sorted: the identity arrangement
    assert np.array_equal(prep["old_to_new"], np.arange(n)) and prep["n_prime"] == n_prime
    got, got_bw = P.finish(prep, k, mbw, part)
    assert np.array_equal(got, out)
    assert np.array_equal(got_bw, bw.astype(np.int64))
