"""CPU checks of the preparation's C ABI (include/kaminpar_b200_prepare.h): the library exports every symbol the
header declares, refuses null arguments with an error instead of touching them, and the Python layer fails loudly
(no fallback) without a GPU. The new kernels (kmp_prepare.cuh) neither spill nor use a stack frame
(cuobjdump -res-usage of the built library)."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from kaminpar_b200 import lp
from kaminpar_b200 import prepare as PR
from kaminpar_b200.graph import rmat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "kaminpar_b200", "csrc", "libkaminpar_b200.so")
KMP_ERR_INVALID = -1
KERNELS = ("k_prep_count", "k_prep_scatter", "k_prep_edges", "k_prep_iso_weights", "k_prep_next_fit",
           "k_prep_map_back")


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "kaminpar_b200_prepare.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(kmp_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    lib = lp.load_library()
    syms = declared_symbols()
    assert len(syms) == 10 and "kmp_prepared_finish" in syms
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in the header but not exported"
    assert lib.kmp_lp_abi_version() == 3
    assert C.sizeof(PR.PrepareStats) == 24


def test_null_arguments_are_refused():
    lib = PR._lib()
    out = C.c_void_p()
    xadj = np.zeros(1, np.uint32)
    assert lib.kmp_prepare_graph(None, 0, 0, xadj.ctypes.data, None, None, None, C.byref(out), None) == KMP_ERR_INVALID
    assert lib.kmp_prepare_graph_device(None, 0, 0, xadj.ctypes.data, None, None, None, C.byref(out),
                                        None) == KMP_ERR_INVALID
    assert lib.kmp_prepared_finish(None, None, 4, None, None, None, None) == KMP_ERR_INVALID
    assert lib.kmp_lp_set_graph_prepared(None, None) == KMP_ERR_INVALID
    assert lib.kmp_prepared_download(None, None, None, None, None, None) == KMP_ERR_INVALID
    assert lib.kmp_prepared_n(None) == 0 and lib.kmp_prepared_m(None) == 0
    lib.kmp_prepared_destroy(None)


def test_no_silent_cpu_fallback():
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError, match="no CUDA device"):
        handle = lp.LPHandle(lp._cluster_config(lp.LabelPropagationCoarseningContext(), lp.EngineContext()))
        PR.rearrange_by_degree_buckets(handle, rmat(8, 4, seed=1))


def test_prepare_kernels_do_not_spill():
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
            k = re.search(r"\d+(k_prep_[a-z_]+?)(?:E|I)", name)
            if k:
                res.append((k.group(1), name, {a: int(b) for a, b in re.findall(r"([A-Z]+(?:\[\d\])?):(\d+)", line)}))
            name = None
    assert sorted({k for k, _, _ in res}) == sorted(KERNELS)
    assert len(res) == len(KERNELS) + 1  # the edge copy with and without edge weights
    for k, name, r in res:
        assert r["LOCAL"] == 0 and r["STACK"] == 0, (name, r)
        assert r["SHARED"] <= 48 * 1024, (name, r)
