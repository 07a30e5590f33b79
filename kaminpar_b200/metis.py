"""Host-side mirror of the METIS reader on the device, over the C ABI in include/kaminpar_b200_io.h (device code:
kaminpar_b200/csrc/kmp_metis.cuh, DESIGN.md §18).

    read_metis_device(handle, path) -> MetisGraph
        csr_read(path) (kaminpar-io/metis_parser.cc:158-245), the file streamed to the device and parsed there
    parse_metis_device(handle, tensor) -> MetisGraph
        the same on bytes already on the device (a torch uint8 tensor, 16-byte aligned)

A malformed file raises MetisError, which carries the report of its first violation. graph.read_metis stays the
host reader for fixtures.

There is no CPU fallback: without the CUDA library / a GPU every call raises.
"""
from __future__ import annotations

import ctypes as C

from . import lp
from .graph import CSRGraph

KINDS = ("OK", "EMPTY", "HEADER", "FORMAT", "TOO_LARGE", "BAD_BYTE", "MISSING_NODE_WEIGHT", "MISSING_EDGE_WEIGHT",
         "ZERO_WEIGHT", "WEIGHT_TOO_LARGE", "NEIGHBOR_OUT_OF_RANGE", "SELF_LOOP", "TOO_FEW_LINES", "EDGE_COUNT",
         "TOTAL_WEIGHT")  # KMP_METIS_*
TILE_BYTES = 4096  # KMP_METIS_TILE_BYTES


class MetisReport(C.Structure):
    """kmp_metis_report: `kind` (an index into KINDS), the header's weight flags, the dropped weights, `extra_lines`,
    n, m, the file's `bytes`, the first violation's `offset`, `line` and `vertex`, device_ms and the header's
    `format`."""

    _fields_ = [
        ("kind", C.c_int32),
        ("has_node_weights", C.c_int32),
        ("has_edge_weights", C.c_int32),
        ("node_weights_dropped", C.c_int32),
        ("edge_weights_dropped", C.c_int32),
        ("extra_lines", C.c_int32),
        ("n", C.c_uint64),
        ("m", C.c_uint64),
        ("bytes", C.c_uint64),
        ("offset", C.c_uint64),
        ("line", C.c_uint64),
        ("vertex", C.c_int64),
        ("device_ms", C.c_float),
        ("format", C.c_uint32),
    ]

    @property
    def kind_name(self) -> str:
        return KINDS[self.kind]

    def message(self) -> str:
        """'<kind> at byte <offset> (line <line>, vertex <vertex>)' for a refusal; for a graph the reference's
        warning line when extra lines were ignored, else ''."""
        return lp.report_message(_lib().kmp_metis_report_message, self)

    def __repr__(self) -> str:
        return (f"MetisReport({self.kind_name}, offset={self.offset}, line={self.line}, vertex={self.vertex}, "
                f"n={self.n}, m={self.m}, bytes={self.bytes})")


class MetisError(lp.ReportError):
    """A refused METIS input; `report` (a MetisReport) holds its first violation, `code` the library's error code."""


def _lib():
    lib = lp.load_library()
    if not getattr(lib, "_metis_ready", False):
        lp.require_symbols(lib, "kmp_read_metis", "kmp_parse_metis_device", "kmp_metis_download",
                           "kmp_metis_report_message")
        for sym in ("kmp_metis_n", "kmp_metis_m"):
            getattr(lib, sym).restype = C.c_uint32
            getattr(lib, sym).argtypes = [C.c_void_p]
        lib.kmp_metis_destroy.restype = None
        lib.kmp_metis_destroy.argtypes = [C.c_void_p]
        lib.kmp_read_metis.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_void_p]
        lib.kmp_parse_metis_device.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
        lib.kmp_metis_download.argtypes = [C.c_void_p] * 5
        lib.kmp_metis_report_message.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
        lib._metis_ready = True
    return lib


class MetisGraph(lp.DeviceResult):
    """A METIS file parsed on the device: n vertices, m adjacency entries, weights None when absent or dropped. Owns
    device memory of the reading handle's pool, freed on its stream."""

    _destroy = "kmp_metis_destroy"

    def __init__(self, ptr, report: MetisReport, handle: lp.LPHandle):
        super().__init__(ptr, report, handle)
        self.report = report
        ptrs = self.device_arrays()
        self._has_vwgt, self._has_adjwgt = ptrs[2] != 0, ptrs[3] != 0
        self._host = None

    @property
    def n(self) -> int:
        return int(_lib().kmp_metis_n(self._g))

    @property
    def m(self) -> int:
        return int(_lib().kmp_metis_m(self._g))

    def get(self) -> CSRGraph:
        """The graph, copied to the host."""
        if self._host is None:
            xadj, adj, vw, ew = self._download_csr("kmp_metis_download", self.n, self.m, self._has_vwgt,
                                                   self._has_adjwgt)
            self._host = CSRGraph(xadj=xadj, adjncy=adj, vwgt=vw, adjwgt=ew)
        return self._host

    def device_arrays(self):
        """(d_xadj, d_adjncy, d_vwgt, d_adjwgt) as integers (0: absent); valid while this object lives."""
        return self._device_ptrs("kmp_metis_device_arrays", 4)

    def set_on(self, handle: lp.LPHandle):
        """kmp_lp_set_graph_device on these arrays: keep this object open while `handle` uses them."""
        handle.set_graph_device(self.n, self.m, *self.device_arrays())


def _finish(rc: int, out, report: MetisReport, handle: lp.LPHandle) -> MetisGraph:
    lp.check_report(rc, report, MetisError)
    return MetisGraph(out, report, handle)


def read_metis_device(handle: lp.LPHandle, path: str) -> MetisGraph:
    """csr_read of the METIS file at `path` on the device of `handle` (its graph and state are not touched)."""
    out = C.c_void_p()
    report = MetisReport()
    rc = _lib().kmp_read_metis(handle._h, str(path).encode(), C.byref(out), C.byref(report))
    return _finish(rc, out, report, handle)


def parse_metis_device(handle: lp.LPHandle, tensor) -> MetisGraph:
    """The same on the bytes of a contiguous torch uint8 CUDA tensor (16-byte aligned) on the handle's device. Work
    queued on torch's current stream is waited for first, so a tensor just written by a kernel is read whole."""
    ptr, size = lp.device_bytes(tensor)
    out = C.c_void_p()
    report = MetisReport()
    rc = _lib().kmp_parse_metis_device(handle._h, ptr, size, C.byref(out), C.byref(report))
    return _finish(rc, out, report, handle)
