"""Host-side mirror of the reference's cluster contraction interface, over the C ABI in
include/kaminpar_b200_contraction.h (device code: kaminpar_b200/csrc/kmp_contract.cuh).

    contract_clustering(graph, clustering, con_ctx) -> CoarseGraph
        kaminpar-shm/coarsening/contraction/cluster_contraction.h:47-56
    CoarseGraph.get() / project_up() / project_down()
        kaminpar-shm/coarsening/contraction/cluster_contraction.h:22-32

There is no CPU fallback: without the CUDA library / a GPU every call raises.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import lp
from .graph import CSRGraph


class ContractionStats(C.Structure):
    """kmp_contraction_stats."""

    _fields_ = [
        ("c_n", C.c_uint32),
        ("c_m", C.c_uint32),
        ("cut_edges", C.c_uint64),
        ("sort_bits", C.c_uint32),
        ("kernel_launches", C.c_uint32),
        ("device_ms", C.c_float),
    ]


class ContractionCoarseningContext:  # kaminpar.h (ContractionCoarseningContext), defaults presets.cc:181-185
    """Accepted for interface compatibility. The reference's `algorithm` / `unbuffered_implementation`
    choose between CPU data structures with the same result; the device path has one algorithm."""

    def __init__(self):
        self.algorithm = 1  # UNBUFFERED
        self.unbuffered_implementation = 0
        self.edge_buffer_fill_fraction = 1.0


def _lib():
    lib = lp.load_library()
    if not getattr(lib, "_contraction_ready", False):
        lib.kmp_coarse_n.restype = C.c_uint32
        lib.kmp_coarse_m.restype = C.c_uint32
        lib.kmp_coarse_fine_n.restype = C.c_uint32
        lib.kmp_coarse_destroy.restype = None
        lib._contraction_ready = True
    return lib


class CoarseGraph:
    """``kaminpar::shm::CoarseGraph`` (cluster_contraction.h:22-32). The coarse graph lives on the
    device; `get()` downloads it once, `device_arrays()` hands it to the next level's LP handle."""

    def __init__(self, handle_ptr, stats: ContractionStats, keepalive=None):
        self._g = handle_ptr
        self.stats = stats
        self._keepalive = keepalive  # the LPHandle whose graph was contracted (owns the stream)
        if keepalive is not None:
            keepalive._children += 1  # the handle is destroyed after this graph (see close)
        self._host: Optional[CSRGraph] = None
        self._mapping: Optional[np.ndarray] = None

    @property
    def n(self) -> int:
        return int(_lib().kmp_coarse_n(self._g))

    @property
    def m(self) -> int:
        return int(_lib().kmp_coarse_m(self._g))

    def get(self) -> CSRGraph:
        if self._host is None:
            n, m = self.n, self.m
            xadj = np.zeros(n + 1, np.uint32)
            adj = np.zeros(m, np.uint32)
            vw = np.zeros(n, np.int32)
            ew = np.zeros(m, np.int32)
            lp._check(_lib().kmp_coarse_download(self._g, lp._ptr(xadj), lp._ptr(adj), lp._ptr(vw), lp._ptr(ew), None))
            self._host = CSRGraph(xadj=xadj, adjncy=adj, vwgt=vw, adjwgt=ew, sorted=False)
        return self._host

    def mapping(self) -> np.ndarray:
        """fine -> coarse (CoarseGraphImpl::get_mapping, cluster_contraction_preprocessing.h:32-34)."""
        if self._mapping is None:
            out = np.zeros(int(_lib().kmp_coarse_fine_n(self._g)), np.uint32)
            lp._check(_lib().kmp_coarse_download(self._g, None, None, None, None, lp._ptr(out)))
            self._mapping = out
        return self._mapping

    def device_arrays(self):
        """(d_xadj, d_adjncy, d_vwgt, d_adjwgt, d_mapping) as integers; valid while this object lives."""
        ptrs = [C.c_void_p() for _ in range(5)]
        lp._check(_lib().kmp_coarse_device_arrays(self._g, *[C.byref(p) for p in ptrs]))
        return tuple(int(p.value or 0) for p in ptrs)

    def project_up(self, coarse, fine: Optional[np.ndarray] = None) -> np.ndarray:
        coarse = np.ascontiguousarray(coarse, np.uint32)
        if len(coarse) != self.n:
            raise ValueError("coarse partition has the wrong length")
        if fine is None:
            fine = np.zeros(int(_lib().kmp_coarse_fine_n(self._g)), np.uint32)
        lp._check(_lib().kmp_coarse_project_up(self._g, lp._ptr(coarse), lp._ptr(fine)))
        return fine

    def project_down(self, fine, coarse: Optional[np.ndarray] = None) -> np.ndarray:
        fine = np.ascontiguousarray(fine, np.uint32)
        if len(fine) != int(_lib().kmp_coarse_fine_n(self._g)):
            raise ValueError("fine partition has the wrong length")
        if coarse is None:
            coarse = np.zeros(self.n, np.uint32)
        lp._check(_lib().kmp_coarse_project_down(self._g, lp._ptr(fine), lp._ptr(coarse)))
        return coarse

    def close(self):
        if getattr(self, "_g", None):
            _lib().kmp_coarse_destroy(self._g)  # frees on the handle's stream: the handle must still exist
            self._g = None
            k = self._keepalive
            if k is not None:
                k._children -= 1
                if k._close_pending and k._children == 0:
                    k.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def contract_on_handle(handle: lp.LPHandle, clustering: Optional[np.ndarray]) -> CoarseGraph:
    """Contract the graph `handle` holds. clustering=None: by the labels the last
    LPHandle.cluster() left on the device (no D2H / H2D of the clustering)."""
    cl = None if clustering is None else np.ascontiguousarray(clustering, np.uint32)
    out = C.c_void_p()
    stats = ContractionStats()
    lp._check(_lib().kmp_contract_clustering(handle._h, lp._ptr(cl), C.byref(out), C.byref(stats)))
    return CoarseGraph(out, stats, keepalive=handle)


def contract_clustering(graph: CSRGraph, clustering, con_ctx: Optional[ContractionCoarseningContext] = None,
                        engine: Optional[lp.EngineContext] = None) -> CoarseGraph:
    """``contract_clustering(graph, clustering, con_ctx)`` (cluster_contraction.cc:22-29)."""
    del con_ctx  # see ContractionCoarseningContext
    if len(clustering) != graph.n:
        raise ValueError("clustering has the wrong length")
    ctx = lp.create_default_context()
    handle = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, engine or ctx.engine))
    handle.set_graph(graph)
    return contract_on_handle(handle, clustering)
