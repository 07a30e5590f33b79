"""Host-side mirror of the input preparation on the device, over the C ABI in include/kaminpar_b200_prepare.h
(device code: kaminpar_b200/csrc/kmp_prepare.cuh, DESIGN.md §15).

    rearrange_by_degree_buckets(handle, graph) -> PreparedGraph
        graph::rearrange_by_degree_buckets + the isolated-vertex cut (kaminpar.cc:368-402,
        graphutils/permutator.cc:19-91, csr_graph.cc:150-174)
    PreparedGraph.finish(handle, k, max_block_weights, partition=None)
        integrate_isolated_nodes + graph::assign_isolated_nodes + map_original_node (kaminpar.cc:419-445)

Set the PartitionContext up on the RAW graph, before preparing it, as compute_partition does (kaminpar.cc:316 runs
before the removal at :391): its max block weights count the isolated vertices. `finish` accepts that context.

There is no CPU fallback: without the CUDA library / a GPU every call raises.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import lp
from .graph import CSRGraph


class PrepareStats(C.Structure):
    """kmp_prepare_stats."""

    _fields_ = [
        ("n", C.c_uint32),
        ("n_nonisolated", C.c_uint32),
        ("num_isolated", C.c_uint32),
        ("m", C.c_uint32),
        ("kernel_launches", C.c_uint32),
        ("device_ms", C.c_float),
    ]


def _lib():
    lib = lp.load_library()
    if not getattr(lib, "_prepare_ready", False):
        lp.require_symbols(lib, "kmp_prepare_graph", "kmp_prepare_graph_device", "kmp_prepared_finish",
                           "kmp_lp_set_graph_prepared")
        for sym in ("kmp_prepared_n", "kmp_prepared_num_isolated", "kmp_prepared_m"):
            getattr(lib, sym).restype = C.c_uint32
            getattr(lib, sym).argtypes = [C.c_void_p]
        lib.kmp_prepared_destroy.restype = None
        lib.kmp_prepared_destroy.argtypes = [C.c_void_p]
        lib.kmp_prepare_graph.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32] + [C.c_void_p] * 6
        lib.kmp_prepare_graph_device.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32] + [C.c_void_p] * 6
        lib.kmp_prepared_finish.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32] + [C.c_void_p] * 4
        lib._prepare_ready = True
    return lib


class PreparedGraph(lp.DeviceResult):
    """The caller's graph rearranged by degree bucket on the device, its isolated vertices last. The LP sees the
    first `n` (non-isolated) vertices: `set_on(handle)`; `finish(...)` maps a partition of them back to the caller's
    ids with the isolated vertices placed. Owns device memory of the preparing handle's pool, freed on its stream."""

    _destroy = "kmp_prepared_destroy"

    def __init__(self, ptr, stats: PrepareStats, handle: lp.LPHandle):
        super().__init__(ptr, stats, handle)
        ptrs = self.device_arrays()
        self._has_vwgt, self._has_adjwgt = ptrs[2] != 0, ptrs[3] != 0
        self._host = None

    @property
    def n(self) -> int:
        """n': the vertices the LP sees."""
        return int(_lib().kmp_prepared_n(self._g))

    @property
    def num_isolated(self) -> int:
        return int(_lib().kmp_prepared_num_isolated(self._g))

    @property
    def m(self) -> int:
        return int(_lib().kmp_prepared_m(self._g))

    def _download(self):
        if self._host is None:
            n_all = self.n + self.num_isolated
            o2n = np.zeros(n_all, np.uint32)
            self._host = self._download_csr("kmp_prepared_download", n_all, self.m, self._has_vwgt, self._has_adjwgt,
                                            o2n) + (o2n,)
        return self._host

    def old_to_new(self) -> np.ndarray:
        """Original id -> prepared id, for all n vertices (ids >= self.n are the isolated ones)."""
        return self._download()[4]

    def node_weights(self) -> Optional[np.ndarray]:
        """Weights of all n vertices in prepared order, the isolated ones included (None: unit weights)."""
        return self._download()[2]

    def get(self) -> CSRGraph:
        """The graph the LP sees (n' vertices, sorted=True), copied to the host."""
        xadj, adj, vw, ew, _ = self._download()
        n = self.n
        return CSRGraph(xadj=xadj[: n + 1].copy(), adjncy=adj, vwgt=None if vw is None else vw[:n].copy(), adjwgt=ew,
                        sorted=True)

    def device_arrays(self):
        """(d_xadj, d_adjncy, d_vwgt, d_adjwgt, d_old_to_new, d_new_to_old) as integers (0: absent); valid while this
        object lives."""
        return self._device_ptrs("kmp_prepared_device_arrays", 6)

    def set_on(self, handle: lp.LPHandle):
        """kmp_lp_set_graph_prepared: the handle's graph becomes the n' prepared vertices, marked sorted."""
        lp._check(_lib().kmp_lp_set_graph_prepared(handle._h, self._g))
        handle._graph_id = None
        handle._n = self.n

    def finish(self, handle: lp.LPHandle, k: int, max_block_weights, partition: Optional[np.ndarray] = None):
        """Returns (partition of the caller's n vertices in its own ids, block weights incl. the isolated vertices).
        `max_block_weights`: k weights or a PartitionContext set up on the raw graph. partition: n' block ids of the
        prepared vertices, or None for the labels `handle` holds on the device for this graph."""
        if isinstance(max_block_weights, lp.PartitionContext):
            max_block_weights = max_block_weights.max_block_weights()
        mbw = np.ascontiguousarray(max_block_weights, np.int32)
        if len(mbw) != k:
            raise ValueError("max_block_weights needs k entries")
        part = None
        if partition is not None:
            part = np.ascontiguousarray(partition, np.uint32)
            if len(part) != self.n:
                raise ValueError("partition needs one block per prepared (non-isolated) vertex")
        out = np.zeros(self.n + self.num_isolated, np.uint32)
        bw = np.zeros(k, np.int32)
        lp._check(_lib().kmp_prepared_finish(handle._h, self._g, C.c_uint32(int(k)), lp._ptr(mbw), lp._ptr(part),
                                             lp._ptr(out), lp._ptr(bw)))
        return out, bw


def rearrange_by_degree_buckets(handle: lp.LPHandle, graph: CSRGraph) -> PreparedGraph:
    """graph::rearrange_by_degree_buckets + the isolated-vertex cut on the device of `handle` (host input)."""
    out = C.c_void_p()
    stats = PrepareStats()
    lp._check(_lib().kmp_prepare_graph(handle._h, graph.n, graph.m, lp._ptr(graph.xadj), lp._ptr(graph.adjncy),
                                       lp._ptr(graph.vwgt), lp._ptr(graph.adjwgt), C.byref(out), C.byref(stats)))
    return PreparedGraph(out, stats, handle)


def rearrange_by_degree_buckets_device(handle: lp.LPHandle, n: int, m: int, d_xadj: int, d_adjncy: int,
                                       d_vwgt: int = 0, d_adjwgt: int = 0) -> PreparedGraph:
    """The same from device arrays (integers, e.g. torch tensors' data_ptr(); 4-byte aligned)."""
    out = C.c_void_p()
    stats = PrepareStats()
    lp._check(_lib().kmp_prepare_graph_device(handle._h, n, m, C.c_void_p(d_xadj), C.c_void_p(d_adjncy),
                                              C.c_void_p(d_vwgt or None), C.c_void_p(d_adjwgt or None), C.byref(out),
                                              C.byref(stats)))
    return PreparedGraph(out, stats, handle)
