"""Host-side mirror of the ParHIP reader on the device, over the C ABI in include/kaminpar_b200_parhip.h (device code:
kaminpar_b200/csrc/kmp_parhip.cuh, DESIGN.md §19).

    read_parhip_device(handle, path, ordering="natural") -> ParhipGraph
        io::parhip::read_graph(path, compress=false, ordering) (kaminpar-io/parhip_parser.cc:179-336), the file
        streamed to the device and read there
    parse_parhip_device(handle, tensor, ordering="natural") -> ParhipGraph
        the same on bytes already on the device (a torch uint8 tensor, 16-byte aligned)
    read_parhip_prepared(handle, path) / parse_parhip_prepared(handle, tensor) -> prepare.PreparedGraph
        the external degree-bucket read straight into a prepared graph (isolated vertices last)

A malformed file raises ParhipError, which carries the report of its first violation. graph.read_parhip stays the
host reader for fixtures.

There is no CPU fallback: without the CUDA library / a GPU every call raises.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import lp, prepare
from .graph import CSRGraph

KINDS = ("OK", "TRUNCATED", "TOO_LARGE", "OFFSETS", "NEIGHBOR_OUT_OF_RANGE", "WEIGHT", "TOTAL_WEIGHT")  # KMP_PARHIP_*
SECTIONS = ("header", "offsets", "adjncy", "vwgt", "adjwgt")  # KMP_PARHIP_SECTION_*
ORDERINGS = {"natural": 0, "degree_buckets": 1, "external_degree_buckets": 2, "implicit_degree_buckets": 3}
COMPRESS = 0x100


class ParhipReport(C.Structure):
    """kmp_parhip_report: `kind` (an index into KINDS), the `section` and entry `index` of the first violation and its
    byte `offset`, the header's weight flags, `sorted`, the `ordering` asked for, version, n, m, the file's `bytes`,
    device_ms and the section `widths` (one byte each: offsets, ids, node weights, edge weights)."""

    _fields_ = [
        ("kind", C.c_int32),
        ("section", C.c_int32),
        ("has_node_weights", C.c_int32),
        ("has_edge_weights", C.c_int32),
        ("sorted", C.c_int32),
        ("ordering", C.c_int32),
        ("version", C.c_uint64),
        ("n", C.c_uint64),
        ("m", C.c_uint64),
        ("bytes", C.c_uint64),
        ("offset", C.c_uint64),
        ("index", C.c_int64),
        ("device_ms", C.c_float),
        ("widths", C.c_uint32),
    ]

    @property
    def kind_name(self) -> str:
        return KINDS[self.kind]

    def message(self) -> str:
        """'<kind> at byte <offset> (<section> entry <index>)' for a refusal, '' for a graph."""
        return lp.report_message(_lib().kmp_parhip_report_message, self)

    def __repr__(self) -> str:
        return (f"ParhipReport({self.kind_name}, offset={self.offset}, section={SECTIONS[self.section]}, "
                f"index={self.index}, n={self.n}, m={self.m}, bytes={self.bytes})")


class ParhipError(lp.ReportError):
    """A refused ParHIP input; `report` (a ParhipReport) holds its first violation, `code` the library's error code."""


def _lib():
    lib = lp.load_library()
    if not getattr(lib, "_parhip_ready", False):
        lp.require_symbols(lib, "kmp_read_parhip", "kmp_parse_parhip_device", "kmp_read_parhip_prepared",
                           "kmp_parse_parhip_device_prepared", "kmp_parhip_download", "kmp_parhip_report_message")
        for sym in ("kmp_parhip_n", "kmp_parhip_m"):
            getattr(lib, sym).restype = C.c_uint32
            getattr(lib, sym).argtypes = [C.c_void_p]
        lib.kmp_parhip_sorted.argtypes = [C.c_void_p]
        lib.kmp_parhip_destroy.restype = None
        lib.kmp_parhip_destroy.argtypes = [C.c_void_p]
        lib.kmp_read_parhip.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_void_p, C.c_void_p]
        lib.kmp_parse_parhip_device.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_void_p, C.c_void_p]
        lib.kmp_read_parhip_prepared.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_void_p]
        lib.kmp_parse_parhip_device_prepared.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
        lib.kmp_parhip_download.argtypes = [C.c_void_p] * 6
        lib.kmp_parhip_report_message.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
        lib._parhip_ready = True
    return lib


class ParhipGraph(lp.DeviceResult):
    """A ParHIP file read on the device: n vertices, m adjacency entries, weights None when absent, `sorted` for the
    implicit and external degree-bucket orderings, `old_to_new()` the external ordering's permutation. Owns device
    memory of the reading handle's pool, freed on its stream."""

    _destroy = "kmp_parhip_destroy"

    def __init__(self, ptr, report: ParhipReport, handle: lp.LPHandle):
        super().__init__(ptr, report, handle)
        self.report = report
        ptrs = self.device_arrays()
        self._has_vwgt, self._has_adjwgt, self._has_perm = ptrs[2] != 0, ptrs[3] != 0, ptrs[4] != 0
        self._host = None

    @property
    def n(self) -> int:
        return int(_lib().kmp_parhip_n(self._g))

    @property
    def m(self) -> int:
        return int(_lib().kmp_parhip_m(self._g))

    @property
    def sorted(self) -> bool:
        return bool(_lib().kmp_parhip_sorted(self._g))

    def _download(self):
        if self._host is None:
            n = self.n
            perm = np.zeros(n, np.uint32) if self._has_perm else None
            xadj, adj, vw, ew = self._download_csr("kmp_parhip_download", n, self.m, self._has_vwgt,
                                                   self._has_adjwgt, perm)
            self._host = (CSRGraph(xadj=xadj, adjncy=adj, vwgt=vw, adjwgt=ew, sorted=self.sorted), perm)
        return self._host

    def get(self) -> CSRGraph:
        """The graph, copied to the host."""
        return self._download()[0]

    def old_to_new(self) -> Optional[np.ndarray]:
        """The external ordering's permutation (file id -> graph id), else None."""
        return self._download()[1]

    def device_arrays(self):
        """(d_xadj, d_adjncy, d_vwgt, d_adjwgt, d_old_to_new) as integers (0: absent); valid while this object lives."""
        return self._device_ptrs("kmp_parhip_device_arrays", 5)

    def set_on(self, handle: lp.LPHandle):
        """kmp_lp_set_graph_device on these arrays: keep this object open while `handle` uses them."""
        handle.set_graph_device(self.n, self.m, *self.device_arrays()[:4])


def _ordering(ordering) -> int:
    return ORDERINGS[ordering] if isinstance(ordering, str) else int(ordering)


def read_parhip_device(handle: lp.LPHandle, path: str, ordering="natural") -> ParhipGraph:
    """read_graph of the ParHIP file at `path` on the device of `handle` (its graph and state are not touched)."""
    out = C.c_void_p()
    report = ParhipReport()
    rc = _lib().kmp_read_parhip(handle._h, str(path).encode(), _ordering(ordering), C.byref(out), C.byref(report))
    lp.check_report(rc, report, ParhipError)
    return ParhipGraph(out, report, handle)


def parse_parhip_device(handle: lp.LPHandle, tensor, ordering="natural") -> ParhipGraph:
    """The same on the bytes of a contiguous torch uint8 CUDA tensor (16-byte aligned) on the handle's device. Work
    queued on torch's current stream is waited for first, so a tensor just written by a kernel is read whole."""
    ptr, size = lp.device_bytes(tensor)
    out = C.c_void_p()
    report = ParhipReport()
    rc = _lib().kmp_parse_parhip_device(handle._h, ptr, size, _ordering(ordering), C.byref(out), C.byref(report))
    lp.check_report(rc, report, ParhipError)
    return ParhipGraph(out, report, handle)


def _prepared(rc: int, out, report: ParhipReport, handle: lp.LPHandle) -> prepare.PreparedGraph:
    lp.check_report(rc, report, ParhipError)
    prepare._lib()
    pg = prepare.PreparedGraph(out, prepare.PrepareStats(), handle)
    pg.report = report
    return pg


def read_parhip_prepared(handle: lp.LPHandle, path: str) -> prepare.PreparedGraph:
    """The external degree-bucket read of `path` as a prepared graph: `set_on` and `finish` take it as it is, and
    `finish` returns the partition in the file's vertex ids."""
    out = C.c_void_p()
    report = ParhipReport()
    rc = _lib().kmp_read_parhip_prepared(handle._h, str(path).encode(), C.byref(out), C.byref(report))
    return _prepared(rc, out, report, handle)


def parse_parhip_prepared(handle: lp.LPHandle, tensor) -> prepare.PreparedGraph:
    """The same on bytes already on the device."""
    ptr, size = lp.device_bytes(tensor)
    out = C.c_void_p()
    report = ParhipReport()
    rc = _lib().kmp_parse_parhip_device_prepared(handle._h, ptr, size, C.byref(out), C.byref(report))
    return _prepared(rc, out, report, handle)
