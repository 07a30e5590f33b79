"""Checks of the METIS reader's C ABI (include/kaminpar_b200_io.h). CPU: the library exports every symbol the header
declares with the struct size the Python layer mirrors, refuses null arguments with an error instead of touching them,
formats the report's line, fails loudly (no fallback) without a GPU, and the k_metis_* kernels neither spill nor use a
stack frame (cuobjdump -res-usage of the built library). GPU: null, misaligned and oversized arguments, an unreadable
path, a header of unsupported size and a handle inside a stepping call are refused; the handle works afterwards."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from kaminpar_b200 import lp
from kaminpar_b200 import metis as ME
from tests import metis_oracle as MO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "kaminpar_b200", "csrc", "libkaminpar_b200.so")
KMP_ERR_INVALID, KMP_ERR_UNSUPPORTED = -1, -4
KERNELS = ("k_metis_summary", "k_metis_write", "k_metis_finish")


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "kaminpar_b200_io.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(kmp_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    lib = lp.load_library()
    syms = declared_symbols()
    assert syms == ["kmp_metis_destroy", "kmp_metis_device_arrays", "kmp_metis_download", "kmp_metis_m",
                    "kmp_metis_n", "kmp_metis_report_message", "kmp_parse_metis_device", "kmp_read_metis"]
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in the header but not exported"
    assert lib.kmp_lp_abi_version() == 3
    assert C.sizeof(ME.MetisReport) == 80
    assert ME.KINDS == MO.KINDS
    text = open(os.path.join(ROOT, "include", "kaminpar_b200_io.h")).read()
    assert f"#define KMP_METIS_TILE_BYTES {ME.TILE_BYTES} " in text


def test_null_arguments_are_refused():
    lib = ME._lib()
    rep = ME.MetisReport()
    out = C.c_void_p()
    assert lib.kmp_read_metis(None, b"x", C.byref(out), C.byref(rep)) == KMP_ERR_INVALID
    assert lib.kmp_parse_metis_device(None, None, 0, C.byref(out), C.byref(rep)) == KMP_ERR_INVALID
    assert lib.kmp_metis_report_message(None, None, 0) == KMP_ERR_INVALID
    assert lib.kmp_metis_device_arrays(None, None, None, None, None) == KMP_ERR_INVALID
    assert lib.kmp_metis_download(None, None, None, None, None) == KMP_ERR_INVALID
    assert lib.kmp_metis_n(None) == 0 and lib.kmp_metis_m(None) == 0
    lib.kmp_metis_destroy(None)
    assert out.value is None


def test_message():
    rep = ME.MetisReport()
    assert rep.message() == ""
    rep.extra_lines = 1
    assert rep.message() == "ignorning extra lines in input file"  # metis_parser.cc:151, word for word
    rep.kind, rep.offset, rep.line, rep.vertex = MO.K["SELF_LOOP"], 123456789012, 40, 7
    assert rep.message() == "self-loop at byte 123456789012 (line 40, vertex 7)"
    rep.kind, rep.vertex = MO.K["HEADER"], -1
    assert rep.message() == "malformed header at byte 123456789012 (line 40, vertex -1)"
    buf = C.create_string_buffer(8)
    assert ME._lib().kmp_metis_report_message(C.byref(rep), buf, 8) == len(rep.message()) and buf.value == b"malform"


def test_no_silent_cpu_fallback(tmp_path):
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    p = tmp_path / "g.metis"
    p.write_bytes(b"2 1\n2\n1\n")
    with pytest.raises(RuntimeError, match="no CUDA device"):
        handle = lp.LPHandle(lp._cluster_config(lp.LabelPropagationCoarseningContext(), lp.EngineContext()))
        ME.read_metis_device(handle, str(p))


def test_metis_kernels_do_not_spill():
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
            k = re.search(r"\d+(k_metis_[a-z_]+?)(?:E|I)", name)
            if k:
                res.append((k.group(1), name, {a: int(b) for a, b in re.findall(r"([A-Z]+(?:\[\d\])?):(\d+)", line)}))
            name = None
    assert sorted({k for k, _, _ in res}) == sorted(KERNELS)
    assert len(res) == len(KERNELS) + 1  # the write pass and its detail form
    for k, name, r in res:
        assert r["LOCAL"] == 0 and r["STACK"] == 0, (name, r)
        assert r["SHARED"] <= 48 * 1024, (name, r)


@pytest.mark.gpu
def test_refusals_on_gpu(tmp_path):
    import torch

    lib = ME._lib()
    handle = lp.LPHandle(lp._cluster_config(lp.LabelPropagationCoarseningContext(), lp.EngineContext()))
    x = torch.zeros(64, dtype=torch.uint8, device="cuda")
    base = x.data_ptr()
    rep = ME.MetisReport()
    out = C.c_void_p()
    assert lib.kmp_parse_metis_device(handle._h, None, 8, C.byref(out), C.byref(rep)) == KMP_ERR_INVALID
    assert lib.kmp_parse_metis_device(handle._h, C.c_void_p(base + 4), 8, C.byref(out), C.byref(rep)) == KMP_ERR_INVALID
    assert lib.kmp_parse_metis_device(handle._h, C.c_void_p(base), 1 << 56, C.byref(out),
                                      C.byref(rep)) == KMP_ERR_UNSUPPORTED
    assert lib.kmp_parse_metis_device(handle._h, C.c_void_p(base), 8, None, C.byref(rep)) == KMP_ERR_INVALID
    assert lib.kmp_parse_metis_device(handle._h, C.c_void_p(base), 8, C.byref(out), None) == KMP_ERR_INVALID
    assert lib.kmp_read_metis(handle._h, None, C.byref(out), C.byref(rep)) == KMP_ERR_INVALID
    assert lib.kmp_read_metis(handle._h, str(tmp_path / "missing").encode(), C.byref(out), C.byref(rep)) == KMP_ERR_INVALID
    assert rep.kind == 0 and out.value is None
    p = tmp_path / "big.metis"
    p.write_bytes(b"5000000000 1\n")
    assert lib.kmp_read_metis(handle._h, str(p).encode(), C.byref(out), C.byref(rep)) == KMP_ERR_UNSUPPORTED
    assert rep.kind_name == "TOO_LARGE" and out.value is None
    g = ME.parse_metis_device(handle, torch.frombuffer(bytearray(b"2 1\n2\n1\n"), dtype=torch.uint8).cuda())
    assert g.n == 2 and g.m == 2 and np.array_equal(g.get().adjncy, [1, 0])
    g.close()
    handle.close()


@pytest.mark.gpu
def test_stepping_handle_is_refused_and_works_afterwards(tmp_path):
    from kaminpar_b200.graph import random_weights, rmat

    lib = ME._lib()
    g = random_weights(rmat(10, 8, seed=2), seed=1, max_adjwgt=5)
    p = tmp_path / "g.metis"
    p.write_bytes(MO.write_metis(g.xadj, g.adjncy, adjwgt=g.adjwgt))
    h = lp.LPHandle(lp._refine_config(lp.LabelPropagationRefinementContext(), lp.EngineContext()))
    h.set_graph(g)
    mbw = np.full(2, g.n, np.int32)
    part = (np.arange(g.n) % 2).astype(np.uint32)
    lp._check(lib.kmp_lp_step_begin_refine(h._h, C.c_uint32(2), lp._ptr(mbw), None, None, lp._ptr(part)))
    with pytest.raises(RuntimeError, match="error -1"):
        ME.read_metis_device(h, str(p))
    lp._check(lib.kmp_lp_step_finish(h._h, None, None, None))
    assert np.array_equal(h.download_labels(), part)
    mg = ME.read_metis_device(h, str(p))
    c = mg.get()
    assert np.array_equal(c.xadj, g.xadj) and np.array_equal(c.adjncy, g.adjncy) and np.array_equal(c.adjwgt, g.adjwgt)
    mg.close()
    h.close()
