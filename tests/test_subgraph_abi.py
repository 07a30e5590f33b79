"""CPU checks of the subgraph extraction's C ABI (include/kaminpar_b200_subgraph.h): the library exports every symbol
the header declares, refuses null arguments with an error instead of touching them, and the Python layer fails loudly
(no fallback) without a GPU. The new kernels (kmp_subgraph.cuh) neither spill nor use a stack frame
(cuobjdump -res-usage of the built library)."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from kaminpar_b200 import lp
from kaminpar_b200 import subgraphs as SG

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "kaminpar_b200", "csrc", "libkaminpar_b200.so")
KMP_ERR_INVALID = -1
KERNELS = ("k_sub_count", "k_sub_node_off", "k_sub_map", "k_sub_xadj", "k_sub_edges", "k_sub_copy_back")


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "kaminpar_b200_subgraph.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(kmp_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    lib = lp.load_library()
    syms = declared_symbols()
    assert len(syms) == 10 and "kmp_extract_subgraphs" in syms
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in the header but not exported"
    assert lib.kmp_lp_abi_version() == 3
    assert C.sizeof(SG.SubgraphStats) == 24


def test_null_arguments_are_refused():
    lib = SG._lib()
    out = C.c_void_p()
    part = np.zeros(4, np.uint32)
    assert lib.kmp_extract_subgraphs(None, 2, part.ctypes.data, C.byref(out), None) == KMP_ERR_INVALID
    assert lib.kmp_subgraphs_copy_partitions(None, None, 4, 4, None, None, None) == KMP_ERR_INVALID
    assert lib.kmp_subgraphs_copy_partitions_device(None, None, 4, 4, None, None, None) == KMP_ERR_INVALID
    assert lib.kmp_subgraphs_offsets(None, None, None) == KMP_ERR_INVALID
    assert lib.kmp_subgraphs_download(None, None, None, None, None, None, None) == KMP_ERR_INVALID
    assert lib.kmp_subgraphs_device_arrays(None, None, None, None, None, None, None, None, None) == KMP_ERR_INVALID
    assert lib.kmp_subgraphs_k(None) == 0 and lib.kmp_subgraphs_n(None) == 0 and lib.kmp_subgraphs_m(None) == 0
    lib.kmp_subgraphs_destroy(None)


def test_no_silent_cpu_fallback():
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError, match="no CUDA device"):
        handle = lp.LPHandle(lp._refine_config(lp.create_default_context().refinement.lp, lp.EngineContext()))
        SG.extract_subgraphs(handle, 2, np.zeros(4, np.uint32))


def test_subgraph_kernels_do_not_spill():
    tool = next((c for c in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump"),
                             shutil.which("cuobjdump")) if c and os.path.exists(c)), None)
    if tool is None:
        pytest.skip("cuobjdump (CUDA toolkit) not found")
    out = subprocess.run([tool, "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    res, name = [], None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        if name and "REG:" in line:
            k = re.search(r"\d+(k_sub_[a-z_]+?)(?:E|I)", name)
            if k:
                res.append((k.group(1), name, {a: int(b) for a, b in re.findall(r"([A-Z]+(?:\[\d\])?):(\d+)", line)}))
            name = None
    assert sorted({k for k, _, _ in res}) == sorted(KERNELS)
    assert len(res) == len(KERNELS) + 1  # the edge pass with and without edge weights
    for k, name, r in res:
        assert r["LOCAL"] == 0 and r["STACK"] == 0, (name, r)
        assert r["SHARED"] <= 48 * 1024, (name, r)
