"""CPU: the subgraph oracle (tests/subgraph_oracle.py) against the UNMODIFIED reference, called through
tests/cpp/ref_subgraph_bridge.cc (compiled here against the reference headers, linked against
oracle/_ref/libkaminpar_ref_full.so; skipped where either is absent):

  lazy_extract_subgraphs_preprocessing + extract_subgraph per block, and extract_subgraphs per block + its mapping
  copy_subgraph_partitions for k' < input_k and k' == input_k
  compute_final_k over current_k = 2^0 .. 2^12 and input_k = 2 .. 10 000

Cases: the golden graphs, weighted R-MAT, empty blocks, all vertices in one block, isolated vertices, k > n, a path
cut in two. The same bridge generates the pinned fixtures tests/golden/subgraph_*.npz (make_subgraph_golden.py)."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from kaminpar_b200.graph import random_weights, rmat
from tests import helpers as H
from tests import subgraph_oracle as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("KMP_REFERENCE", "/root/reference")
REF_LIB_DIR = os.path.join(ROOT, "oracle", "_ref")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")


def reference_present():
    return (os.path.isdir(os.path.join(REF, "kaminpar-shm")) and
            os.path.exists(os.path.join(REF_LIB_DIR, "libkaminpar_ref_full.so")) and CXX is not None)


def compile_bridge(out_dir):
    so = os.path.join(str(out_dir), "ref_subgraph_bridge.so")
    cmd = [CXX, "-std=c++20", "-O2", "-fPIC", "-w", "-mcx16", "-DNDEBUG", "-shared",
           "-I" + os.path.join(ROOT, "oracle", "ref_shim"), "-I" + REF, "-I" + os.path.join(REF, "include"),
           "-I" + os.path.join(REF, "include", "kaminpar-shm"),
           os.path.join(ROOT, "tests", "cpp", "ref_subgraph_bridge.cc"),
           "-o", so, "-L" + REF_LIB_DIR, "-lkaminpar_ref_full", "-Wl,-rpath," + REF_LIB_DIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return C.CDLL(so)


@pytest.fixture(scope="module")
def bridge(tmp_path_factory):
    if not reference_present():
        pytest.skip("the reference sources / oracle/_ref/libkaminpar_ref_full.so are not present")
    return compile_bridge(tmp_path_factory.mktemp("bridge"))


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def ref_lazy(lib, g, part, k):
    n, m = g.n, g.m
    out = dict(node_off=np.zeros(k + 1, np.uint32), block_nodes=np.zeros(n, np.uint32), mapping=np.zeros(n, np.uint32),
               edge_off=np.zeros(k + 1, np.uint32), xadj=np.zeros(n + k, np.uint32), adjncy=np.zeros(m, np.uint32),
               vwgt=np.zeros(n, np.int32), adjwgt=np.zeros(m, np.int32))
    weighted = np.zeros(2, np.int32)
    rc = lib.bridge_lazy_extract(C.c_uint32(n), C.c_uint32(m), _p(g.xadj), _p(g.adjncy), _p(g.vwgt), _p(g.adjwgt),
                                 C.c_uint32(k), _p(part), _p(out["node_off"]), _p(out["block_nodes"]),
                                 _p(out["mapping"]), _p(out["edge_off"]), _p(out["xadj"]), _p(out["adjncy"]),
                                 _p(out["vwgt"]), _p(out["adjwgt"]), _p(weighted))
    assert rc == 0
    m_int = int(out["edge_off"][-1])
    out["adjncy"] = out["adjncy"][:m_int]
    out["vwgt"] = out["vwgt"] if weighted[0] else None
    out["adjwgt"] = out["adjwgt"][:m_int] if weighted[1] else None
    return out


def ref_nonlazy(lib, g, part, k, input_k, node_off):
    n, m = g.n, g.m
    mapping = np.zeros(n, np.uint32)
    xadj, adj = np.zeros(n + k, np.uint32), np.zeros(m, np.uint32)
    vw, ew = np.zeros(n, np.int32), np.zeros(m, np.int32)
    weighted = np.zeros(2, np.int32)
    rc = lib.bridge_extract_subgraphs(C.c_uint32(n), C.c_uint32(m), _p(g.xadj), _p(g.adjncy), _p(g.vwgt),
                                      _p(g.adjwgt), C.c_uint32(k), C.c_uint32(input_k), _p(part), _p(node_off),
                                      _p(mapping), _p(xadj), _p(adj), _p(vw), _p(ew), _p(weighted))
    assert rc == 0
    return mapping, xadj, adj, vw if weighted[0] else None, ew if weighted[1] else None


def ref_copy_back(lib, g, part, k, k_prime, input_k, sub):
    out = np.zeros(g.n, np.uint32)
    rc = lib.bridge_copy_subgraph_partitions(C.c_uint32(g.n), C.c_uint32(g.m), _p(g.xadj), _p(g.adjncy),
                                             C.c_uint32(k), _p(part), C.c_uint32(k_prime), C.c_uint32(input_k),
                                             _p(sub), _p(out))
    assert rc == 0
    return out


def ref_final_k(lib, input_k, levels=13):
    out = np.zeros((1 << levels) - 1, np.uint32)
    lib.bridge_compute_final_k(C.c_uint32(input_k), C.c_uint32(levels), _p(out))
    return out


def bridge_cases():
    """(name, graph, k, partition) of the bridge tests and the pinned fixtures."""
    rng = np.random.default_rng(7)
    g = H.load_graph("walshaw_data")
    yield "walshaw_k16", g, 16, rng.integers(0, 16, g.n).astype(np.uint32)
    g = H.load_graph("rgg16_vwgt_adjwgt")
    yield "rgg16_w_k5", g, 5, (np.arange(g.n) * 5 // g.n).astype(np.uint32)
    g = H.load_graph("rgg2d")
    yield "rgg2d_k3", g, 3, rng.integers(0, 3, g.n).astype(np.uint32)
    g = random_weights(rmat(12, 8, seed=4), 2, max_vwgt=5, max_adjwgt=9)
    yield "rmat12_w_k8", g, 8, rng.integers(0, 8, g.n).astype(np.uint32)
    g = H.path_graph(60)
    yield "empty_blocks", g, 8, (2 * rng.integers(0, 4, g.n)).astype(np.uint32)
    g = H.grid2d(20, 20)
    yield "one_block", g, 4, np.full(g.n, 2, np.uint32)
    g = H.from_edges(30, [(0, 1), (1, 2), (5, 6), (10, 11), (11, 12), (12, 10)])
    yield "isolated", g, 3, rng.integers(0, 3, g.n).astype(np.uint32)
    g = H.path_graph(10)
    yield "k_gt_n", g, 37, rng.integers(0, 37, g.n).astype(np.uint32)
    g = H.path_graph(101)
    yield "path_cut", g, 2, (np.arange(g.n) >= 50).astype(np.uint32)


CASES = list(bridge_cases())


def assert_same(exp, got):
    for key in ("node_off", "edge_off", "block_nodes", "mapping", "xadj", "adjncy", "vwgt", "adjwgt"):
        assert (exp[key] is None) == (got[key] is None), key
        if exp[key] is not None:
            assert np.array_equal(np.asarray(exp[key]), np.asarray(got[key])), key


@pytest.mark.parametrize("name,g,k,part", CASES, ids=[c[0] for c in CASES])
def test_lazy_extraction_equals_reference(bridge, name, g, k, part):
    ref = ref_lazy(bridge, g, part, k)
    assert_same(S.lazy_extract(g.xadj, g.adjncy, g.vwgt, g.adjwgt, part, k), ref)
    assert_same(S.lazy_extract_np(g.xadj, g.adjncy, g.vwgt, g.adjwgt, part, k), ref)


@pytest.mark.parametrize("name,g,k,part", CASES, ids=[c[0] for c in CASES])
def test_nonlazy_extraction_equals_reference(bridge, name, g, k, part):
    exp = S.lazy_extract_np(g.xadj, g.adjncy, g.vwgt, g.adjwgt, part, k)
    mapping, xadj, adj, vw, ew = ref_nonlazy(bridge, g, part, k, 4 * k, exp["node_off"])
    assert np.array_equal(mapping, exp["mapping"])
    blocks, omap = S.extract_nonlazy(g.xadj, g.adjncy, g.vwgt, g.adjwgt, part, k)
    assert np.array_equal(omap, mapping)
    cursor = 0
    for b in range(k):
        n0, n1 = int(exp["node_off"][b]), int(exp["node_off"][b + 1])
        bx = xadj[n0 + b: n1 + b + 1]
        mb = int(bx[-1])
        assert np.array_equal(bx, blocks[b]["xadj"]), f"xadj of block {b}"
        assert np.array_equal(adj[cursor:cursor + mb], blocks[b]["adjncy"]), f"adjncy of block {b}"
        if blocks[b]["vwgt"] is not None:
            assert vw is not None and np.array_equal(vw[n0:n1], blocks[b]["vwgt"])
        if blocks[b]["adjwgt"] is not None:
            assert ew is not None and np.array_equal(ew[cursor:cursor + mb], blocks[b]["adjwgt"])
        cursor += mb


def _subs(exp, k, k_prime, input_k, seed):
    k0 = S.sub_block_offsets(k, k_prime, input_k)
    counts = k0[1:] - k0[:-1]
    rng = np.random.default_rng(seed)
    sub = np.zeros(len(exp["mapping"]), np.uint32)
    no = exp["node_off"]
    for b in range(k):
        sub[no[b]:no[b + 1]] = rng.integers(0, max(int(counts[b]), 1), int(no[b + 1] - no[b]))
    return sub


@pytest.mark.parametrize("name,g,k,part", CASES, ids=[c[0] for c in CASES])
def test_copy_back_equals_reference(bridge, name, g, k, part):
    exp = S.lazy_extract_np(g.xadj, g.adjncy, None, None, part, k)
    for k_prime, input_k in ((2 * k, 8 * k), (4 * k, 4 * k + 1), (k, k)):  # k' < input_k twice, then k' == input_k
        sub = _subs(exp, k, k_prime, input_k, k_prime)
        want, _ = S.copy_back(part, exp["mapping"], exp["node_off"], sub, k, k_prime, input_k)
        assert np.array_equal(ref_copy_back(bridge, g, part, k, k_prime, input_k, sub), want)
    if k & (k - 1) == 0:  # k' == input_k with differing sub-block counts (the final_k path needs a power-of-two k)
        for input_k in (k + 1, 3 * k - 1, 10 * k + 3):
            sub = _subs(exp, k, input_k, input_k, input_k)
            want, _ = S.copy_back(part, exp["mapping"], exp["node_off"], sub, k, input_k, input_k)
            assert np.array_equal(ref_copy_back(bridge, g, part, k, input_k, input_k, sub), want)


def test_compute_final_k_equals_reference(bridge):
    for input_k in list(range(2, 70)) + list(range(70, 10001, 97)) + [1023, 1024, 1025, 4096, 8191, 10000]:
        ref = ref_final_k(bridge, input_k)
        i = 0
        for level in range(13):
            cur = 1 << level
            got = [S.compute_final_k(b, cur, input_k) for b in range(cur)]
            assert got == ref[i:i + cur].tolist(), (input_k, cur)
            i += cur
