"""Checks of the validation's C ABI (include/kaminpar_b200_validate.h). CPU: the library exports every symbol the
header declares with the struct size the Python layer mirrors, refuses null arguments with an error instead of
touching them, formats every report of the corpus as the oracle (and so the reference) words it, and the Python layer
fails loudly (no fallback) without a GPU; the k_val_* kernels neither spill nor use a stack frame (cuobjdump
-res-usage of the built library). GPU: misaligned device pointers, n or m >= 2^31 and a handle inside a stepping call
are refused."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from kaminpar_b200 import lp
from kaminpar_b200 import validate as VA
from kaminpar_b200.graph import rmat
from tests import test_validate_bridge as TB
from tests import validate_oracle as V

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "kaminpar_b200", "csrc", "libkaminpar_b200.so")
KMP_ERR_INVALID, KMP_ERR_UNSUPPORTED = -1, -4
KERNELS = ("k_val_xadj", "k_val_iota", "k_val_first_bad", "k_val_edges", "k_val_dups", "k_val_detail")


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "kaminpar_b200_validate.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(kmp_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    lib = lp.load_library()
    syms = declared_symbols()
    assert syms == ["kmp_graph_report_message", "kmp_validate_graph", "kmp_validate_graph_device"]
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in the header but not exported"
    assert lib.kmp_lp_abi_version() == 3
    assert C.sizeof(VA.GraphReport) == 96
    assert len(VA.KINDS) == V.NUM_KINDS


def test_null_arguments_are_refused():
    lib = VA._lib()
    xadj = np.zeros(1, np.uint32)
    rep = VA.GraphReport()
    assert lib.kmp_validate_graph(None, 0, 0, xadj.ctypes.data, None, None, C.byref(rep)) == KMP_ERR_INVALID
    assert lib.kmp_validate_graph_device(None, 0, 0, xadj.ctypes.data, None, None, C.byref(rep)) == KMP_ERR_INVALID
    assert lib.kmp_graph_report_message(None, None, 0) == KMP_ERR_INVALID


def report_of(r: dict) -> VA.GraphReport:
    rep = VA.GraphReport()
    for f in V.FIELDS + ("n", "m"):
        if f == "count":
            for k in range(V.NUM_KINDS):
                rep.count[k] = r["count"][k]
        else:
            setattr(rep, f, r[f])
    return rep


def test_message_is_the_references_line():
    seen = set()
    for _, xadj, adj, w in TB.CASES:
        r = V.validate(xadj, adj, w)
        assert report_of(r).message() == V.message(r)
        seen.add(r["kind"])
    assert seen == set(range(V.NUM_KINDS))
    r = V.validate(*TB.CASES[0][1:3])
    rep = report_of(dict(r, kind=V.MISSING_REVERSE, u=4000000000, v=7, e=2147483646))
    assert rep.message() == "Edge 4000000000 --> 7 exists with edge 2147483646, but the reverse edges does not exist"
    buf = C.create_string_buffer(8)  # truncated, NUL-terminated, full length returned
    assert VA._lib().kmp_graph_report_message(C.byref(rep), buf, 8) == len(rep.message()) and buf.value == b"Edge 40"


def test_no_silent_cpu_fallback():
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError, match="no CUDA device"):
        handle = lp.LPHandle(lp._cluster_config(lp.LabelPropagationCoarseningContext(), lp.EngineContext()))
        VA.validate_graph(handle, rmat(8, 4, seed=1))


def test_validate_kernels_do_not_spill():
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
            k = re.search(r"\d+(k_val_[a-z_]+?)(?:E|I)", name)
            if k:
                res.append((k.group(1), name, {a: int(b) for a, b in re.findall(r"([A-Z]+(?:\[\d\])?):(\d+)", line)}))
            name = None
    assert sorted({k for k, _, _ in res}) == sorted(KERNELS)
    assert len(res) == len(KERNELS) + 1  # the edge probe with and without edge weights
    for k, name, r in res:
        assert r["LOCAL"] == 0 and r["STACK"] == 0, (name, r)
        assert r["SHARED"] <= 48 * 1024, (name, r)


@pytest.mark.gpu
def test_refusals_on_gpu():
    import torch

    lib = VA._lib()
    handle = lp.LPHandle(lp._cluster_config(lp.LabelPropagationCoarseningContext(), lp.EngineContext()))
    x = torch.zeros(8, dtype=torch.int32, device="cuda")
    rep = VA.GraphReport()
    base = x.data_ptr()
    assert lib.kmp_validate_graph_device(handle._h, 1, 0, C.c_void_p(base + 2), None, None, C.byref(rep)) == KMP_ERR_INVALID
    assert lib.kmp_validate_graph_device(handle._h, 1, 1, C.c_void_p(base), C.c_void_p(base + 1), None,
                                         C.byref(rep)) == KMP_ERR_INVALID
    assert lib.kmp_validate_graph_device(handle._h, 1, 1, C.c_void_p(base), C.c_void_p(base), C.c_void_p(base + 3),
                                         C.byref(rep)) == KMP_ERR_INVALID
    assert lib.kmp_validate_graph_device(handle._h, 1, 0, C.c_void_p(base), None, None, None) == KMP_ERR_INVALID
    assert lib.kmp_validate_graph_device(handle._h, 1 << 31, 0, C.c_void_p(base), None, None,
                                         C.byref(rep)) == KMP_ERR_UNSUPPORTED
    assert lib.kmp_validate_graph_device(handle._h, 0, 1 << 31, C.c_void_p(base), C.c_void_p(base), None,
                                         C.byref(rep)) == KMP_ERR_UNSUPPORTED
    handle.close()


@pytest.mark.gpu
def test_stepping_handle_is_refused_and_works_afterwards():
    from kaminpar_b200.graph import random_weights

    lib = VA._lib()
    g = random_weights(rmat(10, 8, seed=2), seed=1, max_adjwgt=5)
    h = lp.LPHandle(lp._refine_config(lp.LabelPropagationRefinementContext(), lp.EngineContext()))
    h.set_graph(g)
    mbw = np.full(2, g.n, np.int32)
    part = (np.arange(g.n) % 2).astype(np.uint32)
    lp._check(lib.kmp_lp_step_begin_refine(h._h, C.c_uint32(2), lp._ptr(mbw), None, None, lp._ptr(part)))
    with pytest.raises(RuntimeError, match="error -1"):
        VA.validate_graph(h, g)
    lp._check(lib.kmp_lp_step_finish(h._h, None, None, None))
    assert np.array_equal(h.download_labels(), part)
    rep = VA.validate_graph(h, g)
    assert V.as_dict(rep) == V.as_dict(V.validate(g.xadj, g.adjncy, g.adjwgt)) and rep.valid == 1
    h.close()
