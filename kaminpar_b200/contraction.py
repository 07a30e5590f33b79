"""Host-side mirror of the reference's cluster contraction interface, over the C ABI in
include/kaminpar_b200_contraction.h (device code: kaminpar_b200/csrc/kmp_contract.cuh).

    contract_clustering(graph, clustering, con_ctx) -> CoarseGraph
        kaminpar-shm/coarsening/contraction/cluster_contraction.h:47-56
    CoarseGraph.get() / project_up() / project_down()
        kaminpar-shm/coarsening/contraction/cluster_contraction.h:22-32
    sparsification_target(...), CoarseGraph.sparsify(...), sparsify_level(...)
        kaminpar-shm/coarsening/sparsification_cluster_coarsener.cc:41-228 (DESIGN.md §13)
    overlay_level(...)
        kaminpar-shm/coarsening/overlay_cluster_coarsener.cc:34-80 (DESIGN.md §14)

There is no CPU fallback: without the CUDA library / a GPU every call raises.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import lp
from .graph import CSRGraph

INT_MAX = 2**31 - 1


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


class SparsifyStats(C.Structure):
    """kmp_sparsify_stats."""

    _fields_ = [
        ("c_m_before", C.c_uint32),
        ("c_m_after", C.c_uint32),
        ("target_m", C.c_uint32),
        ("threshold", C.c_int32),
        ("smaller", C.c_uint32),
        ("equal", C.c_uint32),
        ("equal_kept", C.c_uint32),
        ("kernel_launches", C.c_uint32),
        ("device_ms", C.c_float),
    ]


class SparsificationClusterCoarseningContext:  # kaminpar.h:185-189, defaults presets.cc:172-177
    def __init__(self, density_target_factor: float = 0.5, edge_target_factor: float = 0.5,
                 laziness_factor: float = 4.0):
        self.density_target_factor = density_target_factor
        self.edge_target_factor = edge_target_factor
        self.laziness_factor = laziness_factor


class OverlayClusterCoarseningContext:  # kaminpar.h (OverlayClusterCoarseningContext), defaults presets.cc:167-171
    def __init__(self, num_levels: int = 1, max_level: int = INT_MAX):
        self.num_levels = num_levels
        self.max_level = max_level


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
        for sym in ("kmp_sparsification_target", "kmp_coarse_sparsify"):
            if not hasattr(lib, sym):
                raise RuntimeError(f"{lp.library_path()} lacks {sym}; rebuild the library")
        lib.kmp_sparsification_target.restype = C.c_uint32
        lib.kmp_sparsification_target.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_double, C.c_double]
        lib.kmp_coarse_sparsify.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p]
        lib._contraction_ready = True
    return lib


class CoarseGraph(lp.DeviceResult):
    """``kaminpar::shm::CoarseGraph`` (cluster_contraction.h:22-32). The coarse graph lives on the
    device; `get()` downloads it once, `device_arrays()` hands it to the next level's LP handle."""

    _destroy = "kmp_coarse_destroy"

    def __init__(self, ptr, stats: ContractionStats, handle: lp.LPHandle):
        super().__init__(ptr, stats, handle)
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
        return self._device_ptrs("kmp_coarse_device_arrays", 5)

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

    def sparsify(self, handle: lp.LPHandle, target_m: int, seed: int) -> SparsifyStats:
        """kmp_coarse_sparsify: keep the edges above the threshold weight and a hashed share of those at it, until
        about `target_m` directed edges remain (DESIGN.md §13). `handle` is the one that contracted this graph.
        Vertices, vertex weights and the mapping stay; earlier `device_arrays()` pointers become invalid."""
        stats = SparsifyStats()
        lp._check(_lib().kmp_coarse_sparsify(handle._h, self._g, C.c_uint32(int(target_m)),
                                              C.c_uint64(int(seed) & 0xFFFFFFFFFFFFFFFF), C.byref(stats)))
        self._host = None
        self.sparsify_stats = stats
        return stats


def sparsification_target(prev_m: int, prev_n: int, c_n: int, density_target_factor: float = 0.5,
                          edge_target_factor: float = 0.5) -> int:
    """SparsificationClusterCoarsener::sparsification_target (sparsification_cluster_coarsener.cc:41-48), computed by
    the library so that every caller evaluates the same double expression."""
    return int(_lib().kmp_sparsification_target(int(prev_m), int(prev_n), int(c_n), float(density_target_factor),
                                                float(edge_target_factor)))


def sparsify_level(handle: lp.LPHandle, cg: CoarseGraph, prev_m: int, prev_n: int,
                   ctx: Optional[SparsificationClusterCoarseningContext] = None, seed=0) -> bool:
    """The sparsification step of SparsificationClusterCoarsener::coarsen() (:50-156) on a contracted level:
    sparsify iff c_m > laziness_factor * target (:89). `prev_m` / `prev_n` belong to the previous level's graph (the
    input graph on the first level). `seed` is an int or a callable that draws one; it is called only when the
    reference draws its seed, i.e. when sparsification runs with target >= 2. Returns whether it sparsified.

    With laziness_factor < 1 the rule can ask to sparsify a level whose target exceeds its edge count; the
    reference's selection rank c_m - target + 1 underflows there, so this is refused with ValueError (no seed is
    drawn, the graph is left as it is)."""
    ctx = ctx or SparsificationClusterCoarseningContext()
    target = sparsification_target(prev_m, prev_n, cg.n, ctx.density_target_factor, ctx.edge_target_factor)
    if not float(cg.m) > ctx.laziness_factor * target:
        return False
    if target > cg.m:
        raise ValueError(f"sparsification target {target} exceeds the level's {cg.m} edges (laziness_factor "
                         f"{ctx.laziness_factor} < 1): the reference's threshold selection is undefined there")
    s = 0
    if target >= 2:
        s = seed() if callable(seed) else seed
    cg.sparsify(handle, target, s)
    return True


def contract_on_handle(handle: lp.LPHandle, clustering: Optional[np.ndarray]) -> CoarseGraph:
    """Contract the graph `handle` holds. clustering=None: by the labels the last
    LPHandle.cluster() left on the device (no D2H / H2D of the clustering)."""
    cl = None if clustering is None else np.ascontiguousarray(clustering, np.uint32)
    out = C.c_void_p()
    stats = ContractionStats()
    lp._check(_lib().kmp_contract_clustering(handle._h, lp._ptr(cl), C.byref(out), C.byref(stats)))
    return CoarseGraph(out, stats, handle)


def overlay_level(handle: lp.LPHandle, level: int, ctx: Optional[OverlayClusterCoarseningContext],
                  max_cluster_weight: int, desired: int = 0, communities=None) -> CoarseGraph:
    """One level of OverlayClusterCoarsener::coarsen() (:34-80) on the graph `handle` holds: 2^num_levels clusterings
    intersected on the device if `level` (the number of coarse graphs built so far, AbstractClusterCoarsener::level())
    is at most max_level, else one clustering; then the contraction, with the clustering left on the device.

    The comparison is the reference's, `level <= static_cast<std::size_t>(max_level)`: a negative max_level converts
    to a huge unsigned value, so it never turns the overlay off."""
    ctx = ctx or OverlayClusterCoarseningContext()
    if level <= int(ctx.max_level) % 2**64:
        handle.cluster_overlay(ctx.num_levels, max_cluster_weight, desired, communities, fetch=False)
    else:
        handle.cluster(max_cluster_weight, desired, communities, fetch=False)
    return contract_on_handle(handle, None)


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
