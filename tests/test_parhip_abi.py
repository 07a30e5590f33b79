"""Checks of the ParHIP reader's C ABI (include/kaminpar_b200_parhip.h). CPU: the library exports exactly the symbols
the header declares, the report's size is the one the Python layer mirrors, null arguments and unknown orderings are
refused without being touched, the report's line is formatted, there is no CPU fallback, and the k_parhip_* kernels
neither spill nor use a stack frame (cuobjdump -res-usage of the built library)."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

from kaminpar_b200 import lp
from kaminpar_b200 import parhip as PH
from tests import parhip_oracle as PO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "kaminpar_b200", "csrc", "libkaminpar_b200.so")
KMP_ERR_INVALID, KMP_ERR_UNSUPPORTED = -1, -4


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "kaminpar_b200_parhip.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(kmp_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    lib = lp.load_library()
    syms = declared_symbols()
    assert syms == ["kmp_parhip_destroy", "kmp_parhip_device_arrays", "kmp_parhip_download", "kmp_parhip_m",
                    "kmp_parhip_n", "kmp_parhip_report_message", "kmp_parhip_sorted", "kmp_parse_parhip_device",
                    "kmp_parse_parhip_device_prepared", "kmp_pool_usage", "kmp_read_parhip", "kmp_read_parhip_prepared"]
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in the header but not exported"
    assert lib.kmp_lp_abi_version() == 3
    assert C.sizeof(PH.ParhipReport) == 80
    assert PH.KINDS == PO.KINDS
    assert tuple(f for f, _ in PH.ParhipReport._fields_ if f != "device_ms") == \
        ("kind", "section", "has_node_weights", "has_edge_weights", "sorted", "ordering", "version", "n", "m", "bytes",
         "offset", "index", "widths")
    assert set(PO.REPORT_FIELDS) <= {f for f, _ in PH.ParhipReport._fields_}
    assert PH.ORDERINGS == {"natural": PO.NATURAL, "degree_buckets": PO.DEGREE_BUCKETS,
                            "external_degree_buckets": PO.EXTERNAL, "implicit_degree_buckets": PO.IMPLICIT}


def test_null_arguments_are_refused():
    lib = PH._lib()
    rep = PH.ParhipReport()
    out = C.c_void_p()
    assert lib.kmp_read_parhip(None, b"x", 0, C.byref(out), C.byref(rep)) == KMP_ERR_INVALID
    assert lib.kmp_parse_parhip_device(None, None, 0, 0, C.byref(out), C.byref(rep)) == KMP_ERR_INVALID
    assert lib.kmp_read_parhip_prepared(None, b"x", C.byref(out), C.byref(rep)) == KMP_ERR_INVALID
    assert lib.kmp_parse_parhip_device_prepared(None, None, 0, C.byref(out), C.byref(rep)) == KMP_ERR_INVALID
    assert lib.kmp_parhip_report_message(None, None, 0) == KMP_ERR_INVALID
    assert lib.kmp_parhip_device_arrays(None, None, None, None, None, None) == KMP_ERR_INVALID
    assert lib.kmp_parhip_download(None, None, None, None, None, None) == KMP_ERR_INVALID
    assert lib.kmp_parhip_n(None) == 0 and lib.kmp_parhip_m(None) == 0 and lib.kmp_parhip_sorted(None) == 0
    assert lib.kmp_pool_usage(None, 0, C.byref(C.c_uint64()), C.byref(C.c_uint64())) == KMP_ERR_INVALID
    lib.kmp_parhip_destroy(None)
    assert out.value is None


def test_message():
    rep = PH.ParhipReport()
    assert rep.message() == ""
    rep.kind, rep.offset, rep.section, rep.index = PO.NEIGHBOR_OUT_OF_RANGE, 123456789012, PO.ADJNCY, 7
    assert rep.message() == "neighbor out of range at byte 123456789012 (adjncy entry 7)"
    rep.kind, rep.offset, rep.section, rep.index = PO.TRUNCATED, 20, PO.HEADER, -1
    assert rep.message() == "truncated at byte 20 (header entry -1)"
    rep.kind, rep.section, rep.index = PO.TOTAL_WEIGHT, PO.VWGT, 9
    assert rep.message() == "total weight too large at byte 20 (vwgt entry 9)"
    buf = C.create_string_buffer(8)
    assert PH._lib().kmp_parhip_report_message(C.byref(rep), buf, 8) == len(rep.message()) and buf.value == b"total w"


def test_no_silent_cpu_fallback(tmp_path):
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    p = tmp_path / "g.parhip"
    p.write_bytes(PO.write([0, 1, 2], [1, 0]))
    with pytest.raises(RuntimeError, match="no CUDA device"):
        handle = lp.LPHandle(lp._cluster_config(lp.LabelPropagationCoarseningContext(), lp.EngineContext()))
        PH.read_parhip_device(handle, str(p))


def test_parhip_kernels_do_not_spill():
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
            k = re.search(r"\d+(k_parhip_[a-z_]+?)(?:E|I)", name)
            if k:
                res.append((k.group(1), name, {a: int(b) for a, b in re.findall(r"([A-Z]+(?:\[\d\])?):(\d+)", line)}))
            name = None
    assert sorted({k for k, _, _ in res}) == ["k_parhip_edges", "k_parhip_pass"]
    assert len(res) == 9  # four sections at two widths, and the edge copy
    for k, name, r in res:
        assert r["LOCAL"] == 0 and r["STACK"] == 0, (name, r)
        assert r["SHARED"] <= 48 * 1024, (name, r)


@pytest.mark.gpu
def test_refusals_on_gpu(tmp_path):
    import torch

    lib = PH._lib()
    handle = lp.LPHandle(lp._cluster_config(lp.LabelPropagationCoarseningContext(), lp.EngineContext()))
    x = torch.zeros(64, dtype=torch.uint8, device="cuda")
    base = x.data_ptr()
    rep = PH.ParhipReport()
    out = C.c_void_p()
    assert lib.kmp_parse_parhip_device(handle._h, None, 8, 0, C.byref(out), C.byref(rep)) == KMP_ERR_INVALID
    assert lib.kmp_parse_parhip_device(handle._h, C.c_void_p(base + 4), 8, 0, C.byref(out),
                                       C.byref(rep)) == KMP_ERR_INVALID
    assert lib.kmp_parse_parhip_device(handle._h, C.c_void_p(base), 1 << 56, 0, C.byref(out),
                                       C.byref(rep)) == KMP_ERR_UNSUPPORTED
    assert lib.kmp_parse_parhip_device(handle._h, C.c_void_p(base), 8, 4, C.byref(out), C.byref(rep)) == KMP_ERR_INVALID
    assert lib.kmp_parse_parhip_device(handle._h, C.c_void_p(base), 8, PH.COMPRESS, C.byref(out),
                                       C.byref(rep)) == KMP_ERR_UNSUPPORTED
    assert lib.kmp_read_parhip(handle._h, None, 0, C.byref(out), C.byref(rep)) == KMP_ERR_INVALID
    assert lib.kmp_read_parhip(handle._h, str(tmp_path / "missing").encode(), 0, C.byref(out),
                               C.byref(rep)) == KMP_ERR_INVALID
    assert rep.kind == 0 and out.value is None
    host = torch.zeros(64, dtype=torch.uint8).pin_memory()  # host memory through the C ABI: never read by a kernel
    assert lib.kmp_parse_parhip_device(handle._h, C.c_void_p(host.data_ptr()), 64, 0, C.byref(out),
                                       C.byref(rep)) == KMP_ERR_INVALID
    assert out.value is None
    handle.close()
