"""Host-side mirror of graph validation on the device, over the C ABI in include/kaminpar_b200_validate.h (device code:
kaminpar_b200/csrc/kmp_validate.cuh, DESIGN.md §17).

    validate_graph(handle, graph) -> GraphReport
        debug::validate_graph(graph) (csr_graph.cc:266-356) + the multi-edge count of validate_undirected_graph
    validate_graph_device(handle, n, m, d_xadj, d_adjncy, d_adjwgt=None) -> GraphReport
        the same on device arrays (e.g. torch tensors' data_ptr())

The report's verdict and first violation are those of the reference's debug::validate_graph; `message()` is its
warning line. A malformed graph is a report, not an exception: only a refused call raises.

There is no CPU fallback: without the CUDA library / a GPU every call raises.
"""
from __future__ import annotations

import ctypes as C

from . import lp
from .graph import CSRGraph

NUM_KINDS = 9
KINDS = ("VALID", "XADJ_START", "XADJ_END", "XADJ_DECREASING", "NEIGHBOR_OUT_OF_GRAPH", "SELF_LOOP",
         "NEIGHBOR_OF_NEIGHBOR_OUT_OF_GRAPH", "MISSING_REVERSE", "WEIGHT_MISMATCH")  # KMP_GRAPH_*


class GraphReport(C.Structure):
    """kmp_graph_report: `valid`, `kind` (an index into KINDS), the first violation's u, e, v, e_rev, v_rev, w,
    w_rev, the per-kind `count`, `duplicates` with the first duplicate (dup_u, dup_e), and device_ms."""

    _fields_ = [
        ("valid", C.c_int32),
        ("kind", C.c_int32),
        ("n", C.c_uint32),
        ("m", C.c_uint32),
        ("u", C.c_uint32),
        ("e", C.c_uint32),
        ("v", C.c_uint32),
        ("e_rev", C.c_uint32),
        ("v_rev", C.c_uint32),
        ("w", C.c_int32),
        ("w_rev", C.c_int32),
        ("count", C.c_uint32 * NUM_KINDS),
        ("duplicates", C.c_uint32),
        ("dup_u", C.c_uint32),
        ("dup_e", C.c_uint32),
        ("device_ms", C.c_float),
    ]

    @property
    def kind_name(self) -> str:
        return KINDS[self.kind]

    def message(self) -> str:
        """The reference's warning line for the first violation ("" when valid)."""
        lib = _lib()
        size = lib.kmp_graph_report_message(C.byref(self), None, 0)
        buf = C.create_string_buffer(size + 1)
        lib.kmp_graph_report_message(C.byref(self), buf, size + 1)
        return buf.value.decode()

    def __repr__(self) -> str:
        return (f"GraphReport({self.kind_name}, u={self.u}, e={self.e}, v={self.v}, e_rev={self.e_rev}, "
                f"count={list(self.count)}, duplicates={self.duplicates})")


def _lib():
    lib = lp.load_library()
    if not getattr(lib, "_validate_ready", False):
        for sym in ("kmp_validate_graph", "kmp_validate_graph_device", "kmp_graph_report_message"):
            if not hasattr(lib, sym):
                raise RuntimeError(f"{lp.library_path()} lacks {sym}; rebuild the library")
        lib.kmp_validate_graph.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32] + [C.c_void_p] * 4
        lib.kmp_validate_graph_device.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32] + [C.c_void_p] * 4
        lib.kmp_graph_report_message.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
        lib._validate_ready = True
    return lib


def validate_graph(handle: lp.LPHandle, graph: CSRGraph) -> GraphReport:
    """Validate a host graph on the device of `handle` (its graph and state are not touched)."""
    out = GraphReport()
    lp._check(_lib().kmp_validate_graph(handle._h, graph.n, graph.m, lp._ptr(graph.xadj), lp._ptr(graph.adjncy),
                                        lp._ptr(graph.adjwgt), C.byref(out)))
    return out


def validate_graph_device(handle: lp.LPHandle, n: int, m: int, d_xadj: int, d_adjncy: int,
                          d_adjwgt: int = None) -> GraphReport:
    """The same from device arrays (integers, e.g. torch tensors' data_ptr(); 4-byte aligned)."""
    out = GraphReport()
    lp._check(_lib().kmp_validate_graph_device(handle._h, n, m, C.c_void_p(d_xadj), C.c_void_p(d_adjncy or None),
                                               C.c_void_p(d_adjwgt or None), C.byref(out)))
    return out
