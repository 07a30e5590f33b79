"""The host twin of the device initial bipartitioner (tests/cpp/ip_host_check.cc: kmp_bipartition.cuh and
kmp_ip_params.h compiled with g++ without FMA contraction), through ctypes. Used by the CPU tests against the live
reference and by the GPU tests, which hold the device to it block for block."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

from kaminpar_b200.bipartition import IPConfig
from tests import subgraph_oracle as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
TWIN = os.path.join(ROOT, "build", "ip_host_check.so")
TWIN_SRCS = [os.path.join(ROOT, "tests", "cpp", "ip_host_check.cc"),
             os.path.join(ROOT, "kaminpar_b200", "csrc", "kmp_bipartition.cuh"),
             os.path.join(ROOT, "kaminpar_b200", "csrc", "kmp_ip_params.h"),
             os.path.join(ROOT, "kaminpar_b200", "csrc", "kmp_rng.cuh"),
             os.path.join(ROOT, "include", "kaminpar_b200_bipartition.h")]
REF = os.environ.get("KMP_REFERENCE", "/root/reference")
BRIDGE = os.path.join(ROOT, "oracle", "_ref", "ref_ip_bridge.so")
_LIB = None


def _fresh(target, sources):
    return os.path.exists(target) and all(os.path.getmtime(s) <= os.path.getmtime(target) for s in sources)


def _compile_twin(out):
    cmd = [CXX, "-std=c++17", "-O2", "-fPIC", "-shared", "-ffp-contract=off", TWIN_SRCS[0], "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def build_twin():
    """build/ip_host_check.so, unless it is newer than its sources."""
    if not _fresh(TWIN, TWIN_SRCS):
        os.makedirs(os.path.dirname(TWIN), exist_ok=True)
        _compile_twin(TWIN)
    return TWIN


def build_bridge(out=BRIDGE):
    """tests/cpp/ref_ip_bridge.cc against the reference headers and oracle/_ref/libkaminpar_ref_full.so."""
    src = os.path.join(ROOT, "tests", "cpp", "ref_ip_bridge.cc")
    if out == BRIDGE and _fresh(out, [src, os.path.join(ROOT, "oracle", "_ref", "libkaminpar_ref_full.so")]):
        return out
    lib_dir = os.path.join(ROOT, "oracle", "_ref")
    cmd = [CXX, "-std=c++20", "-O2", "-fPIC", "-w", "-mcx16", "-DNDEBUG", "-shared",
           "-I" + os.path.join(ROOT, "oracle", "ref_shim"), "-I" + REF, "-I" + os.path.join(REF, "include"),
           "-I" + os.path.join(REF, "include", "kaminpar-shm"), src, "-o", out, "-L" + lib_dir,
           "-lkaminpar_ref_full", "-Wl,-rpath," + lib_dir]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return out


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def lib():
    global _LIB
    if _LIB is None:
        if _fresh(TWIN, TWIN_SRCS):  # as build() left it
            out = TWIN
        else:  # a read-only or stale tree: compile into a temporary directory
            out = os.path.join(tempfile.mkdtemp(prefix="kmp_ip_host_"), "ip_host_check.so")
            _compile_twin(out)
        L = C.CDLL(out)
        L.ip_default_config.restype = IPConfig
        L.ip_block_params.restype = C.c_int
        L.ip_block_params.argtypes = [C.c_uint32, C.c_void_p, C.c_int, C.c_int32, C.c_double, C.c_void_p, C.c_uint32,
                                      C.c_uint32, C.c_uint32, C.c_uint32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
        L.ip_host_bipartition.argtypes = [C.c_uint32, C.c_uint32] + [C.c_void_p] * 6 + [C.c_int32, C.c_uint64,
                                                                                        C.c_void_p, C.c_void_p]
        L.ip_host_bipartition.restype = C.c_int
        L.ip_compute_final_k.restype = C.c_uint32
        L.ip_compute_final_k.argtypes = [C.c_uint32] * 3
        _LIB = L
    return _LIB


def block_arrays(res, b):
    bx, ba, bv, be = S.block_of(res, b)
    return (np.ascontiguousarray(bx, np.uint32), np.ascontiguousarray(ba, np.uint32),
            None if bv is None else np.ascontiguousarray(bv, np.int32),
            None if be is None else np.ascontiguousarray(be, np.int32))


def block_params(cfg, input_k, mbw, uniform, total, eps, b, k, bx, ba, bv, be):
    nb, mb = len(bx) - 1, len(ba)
    tnw = int(bv.sum()) if bv is not None else nb
    mnw = int(bv.max()) if bv is not None and nb > 0 else 1
    tew = int(be.sum()) if be is not None else mb
    out = np.zeros(6, np.int32)
    ok = lib().ip_block_params(input_k, _p(np.ascontiguousarray(mbw, np.int32)), int(uniform), total, eps,
                               C.byref(cfg), b, k, nb, mb, tnw, mnw, tew, _p(out))
    assert ok, "block %d's sub-block range runs past input_k = %d at k = %d" % (b, input_k, k)
    return out


def bipartition_block(cfg, params, seed, bx, ba, bv, be, arena_bytes=0):
    nb = len(bx) - 1
    out = np.zeros(nb, np.uint32)
    cnt = np.zeros(2, np.uint32)
    rc = lib().ip_host_bipartition(nb, len(ba), _p(bx), _p(ba), _p(bv), _p(be), C.byref(cfg), _p(params),
                                   int(np.int32(np.uint32(seed))), arena_bytes, _p(out), _p(cnt))
    return rc, out, cnt


def expected_sub_partitions(g, part, k, k_prime, input_k, mbw, seed, cfg=None, uniform=True, eps=0.03):
    """The block-major sub-partitions kmp_bipartition_subgraphs must produce, from the host twin."""
    cfg = cfg if cfg is not None else IPConfig()
    res = S.lazy_extract_np(g.xadj, g.adjncy, g.vwgt, g.adjwgt, part, k)
    total = int(g.vwgt.sum()) if g.vwgt is not None else g.n
    sub = np.zeros(g.n, np.uint32)
    for b in range(k):
        s_b = lib().ip_compute_final_k(b, k, input_k) if k_prime == input_k else k_prime // k
        bx, ba, bv, be = block_arrays(res, b)
        if s_b != 2 or len(bx) == 1:
            continue
        params = block_params(cfg, input_k, mbw, uniform, total, eps, b, k, bx, ba, bv, be)
        rc, out, _ = bipartition_block(cfg, params, (seed + b) & 0xFFFFFFFF, bx, ba, bv, be)
        assert rc == 0
        no = res["node_off"]
        sub[int(no[b]):int(no[b + 1])] = out
    return sub


def max_block_weights(total, input_k, eps=0.03, uniform=True, seed=0):
    if uniform:
        return np.full(input_k, int((1 + eps) * np.ceil(total / input_k)), np.int32)
    rng = np.random.default_rng(seed)
    return (np.ceil(total / input_k) * (1 + rng.uniform(0.0, 0.2, input_k))).astype(np.int32)
