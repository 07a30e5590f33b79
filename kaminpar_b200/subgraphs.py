"""Host-side mirror of the partition extension's device steps, over the C ABI in include/kaminpar_b200_subgraph.h
(device code: kaminpar_b200/csrc/kmp_subgraph.cuh, DESIGN.md §16).

    extract_subgraphs(handle, k, partition=None) -> Subgraphs
        graph::lazy_extract_subgraphs_preprocessing + graph::extract_subgraph for every block
        (graphutils/subgraph_extractor.cc:181-324)
    Subgraphs.copy_partitions(handle, sub_partitions, k_prime, input_k)
        graph::copy_subgraph_partitions (subgraph_extractor.cc:492-533)

Between the two, a caller bipartitions each block (on the host: `block(b)`, or on another handle: `device_view(b)`)
and lays the sub-partitions out block-major, block b's at [node_off[b], node_off[b + 1]).

There is no CPU fallback: without the CUDA library / a GPU every call raises.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import lp
from .graph import CSRGraph


class SubgraphStats(C.Structure):
    """kmp_subgraph_stats."""

    _fields_ = [
        ("n", C.c_uint32),
        ("k", C.c_uint32),
        ("m", C.c_uint32),
        ("m_internal", C.c_uint32),
        ("kernel_launches", C.c_uint32),
        ("device_ms", C.c_float),
    ]


def _lib():
    lib = lp.load_library()
    if not getattr(lib, "_subgraph_ready", False):
        for sym in ("kmp_extract_subgraphs", "kmp_subgraphs_copy_partitions", "kmp_subgraphs_copy_partitions_device"):
            if not hasattr(lib, sym):
                raise RuntimeError(f"{lp.library_path()} lacks {sym}; rebuild the library")
        for sym in ("kmp_subgraphs_k", "kmp_subgraphs_n", "kmp_subgraphs_m"):
            getattr(lib, sym).restype = C.c_uint32
            getattr(lib, sym).argtypes = [C.c_void_p]
        lib.kmp_subgraphs_destroy.restype = None
        lib.kmp_subgraphs_destroy.argtypes = [C.c_void_p]
        lib.kmp_extract_subgraphs.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.kmp_subgraphs_offsets.argtypes = [C.c_void_p] * 3
        lib.kmp_subgraphs_download.argtypes = [C.c_void_p] * 7
        for sym in ("kmp_subgraphs_copy_partitions", "kmp_subgraphs_copy_partitions_device"):
            getattr(lib, sym).argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32] + [C.c_void_p] * 3
        lib._subgraph_ready = True
    return lib


class Subgraphs(lp.DeviceResult):
    """The k block-induced subgraphs of a handle's graph on the device, in one n + k xadj (block b's local xadj at
    node_off[b] + b), one adjncy and the vertex order block_nodes. Owns device memory of the extracting handle's pool,
    freed on its stream."""

    _destroy = "kmp_subgraphs_destroy"

    def __init__(self, ptr, stats: SubgraphStats, handle: lp.LPHandle):
        super().__init__(ptr, stats, handle)
        ptrs = self.device_arrays()
        self._has_vwgt, self._has_adjwgt = ptrs[2] != 0, ptrs[3] != 0
        self._host = None
        self._offsets = None

    @property
    def k(self) -> int:
        return int(_lib().kmp_subgraphs_k(self._g))

    @property
    def n(self) -> int:
        return int(_lib().kmp_subgraphs_n(self._g))

    @property
    def m(self) -> int:
        """Internal directed edges of all blocks."""
        return int(_lib().kmp_subgraphs_m(self._g))

    def offsets(self):
        """(node_off[k + 1], edge_off[k + 1])."""
        if self._offsets is None:
            no = np.zeros(self.k + 1, np.uint32)
            eo = np.zeros(self.k + 1, np.uint32)
            lp._check(_lib().kmp_subgraphs_offsets(self._g, lp._ptr(no), lp._ptr(eo)))
            self._offsets = (no, eo)
        return self._offsets

    def _download(self):
        if self._host is None:
            n, k, m = self.n, self.k, self.m
            xadj = np.zeros(n + k, np.uint32)
            adj = np.zeros(m, np.uint32)
            vw = np.zeros(n, np.int32) if self._has_vwgt else None
            ew = np.zeros(m, np.int32) if self._has_adjwgt else None
            mapping = np.zeros(n, np.uint32)
            bn = np.zeros(n, np.uint32)
            lp._check(_lib().kmp_subgraphs_download(self._g, lp._ptr(xadj), lp._ptr(adj), lp._ptr(vw), lp._ptr(ew),
                                                    lp._ptr(mapping), lp._ptr(bn)))
            self._host = (xadj, adj, vw, ew, mapping, bn)
        return self._host

    def xadj_cat(self) -> np.ndarray:
        """The n + k xadj entries of all blocks, block b's at node_off[b] + b."""
        return self._download()[0]

    def mapping(self) -> np.ndarray:
        """Vertex -> its rank within its block."""
        return self._download()[4]

    def block_nodes(self) -> np.ndarray:
        """Vertices by block, ascending id within a block."""
        return self._download()[5]

    def block(self, b: int) -> CSRGraph:
        """Block b's subgraph, copied to the host."""
        xadj, adj, vw, ew, _, _ = self._download()
        no, eo = self.offsets()
        n0, n1, e0, e1 = int(no[b]), int(no[b + 1]), int(eo[b]), int(eo[b + 1])
        return CSRGraph(xadj=xadj[n0 + b: n1 + b + 1].copy(), adjncy=adj[e0:e1].copy(),
                        vwgt=None if vw is None else vw[n0:n1].copy(), adjwgt=None if ew is None else ew[e0:e1].copy())

    def device_arrays(self):
        """(d_xadj, d_adjncy, d_vwgt, d_adjwgt, d_mapping, d_block_nodes, d_node_off, d_edge_off) as integers (0:
        absent); valid while this object lives."""
        return self._device_ptrs("kmp_subgraphs_device_arrays", 8)

    def device_view(self, b: int):
        """Block b in place as (n_b, m_b, d_xadj, d_adjncy, d_vwgt, d_adjwgt) for LPHandle.set_graph_device: no copy.
        The view is valid while this object lives."""
        d_xadj, d_adj, d_vw, d_ew = self.device_arrays()[:4]
        no, eo = self.offsets()
        n0, n1, e0, e1 = int(no[b]), int(no[b + 1]), int(eo[b]), int(eo[b + 1])
        return (n1 - n0, e1 - e0, d_xadj + 4 * (n0 + b), d_adj + 4 * e0, d_vw + 4 * n0 if d_vw else 0,
                d_ew + 4 * e0 if d_ew else 0)

    def copy_partitions(self, handle: lp.LPHandle, sub_partitions, k_prime: int, input_k: int, fetch=True):
        """copy_subgraph_partitions: the k'-way partition from the block-major sub-partitions (a host array of n ids,
        or an integer device pointer). It becomes `handle`'s labels and block weights. Returns (partition or None,
        block weights or None)."""
        lib = _lib()
        out = np.zeros(self.n, np.uint32) if fetch else None
        bw = np.zeros(k_prime, np.int32) if fetch else None
        if isinstance(sub_partitions, int):
            lp._check(lib.kmp_subgraphs_copy_partitions_device(handle._h, self._g, C.c_uint32(k_prime),
                                                               C.c_uint32(input_k), C.c_void_p(sub_partitions),
                                                               lp._ptr(out), lp._ptr(bw)))
        else:
            sub = np.ascontiguousarray(sub_partitions, np.uint32)
            if len(sub) != self.n:
                raise ValueError("sub_partitions needs one sub-block id per vertex, block-major")
            lp._check(lib.kmp_subgraphs_copy_partitions(handle._h, self._g, C.c_uint32(k_prime), C.c_uint32(input_k),
                                                        lp._ptr(sub), lp._ptr(out), lp._ptr(bw)))
        return out, bw


def extract_subgraphs(handle: lp.LPHandle, k: int, partition: Optional[np.ndarray] = None) -> Subgraphs:
    """The k block-induced subgraphs of the graph `handle` holds. partition: n block ids (host), loaded as the
    handle's labels, or None for the labels it holds on the device."""
    part = None
    if partition is not None:
        part = np.ascontiguousarray(partition, np.uint32)
        if getattr(handle, "_n", None) is not None and len(part) != handle._n:  # no graph: the library refuses
            raise ValueError("partition needs one block per vertex")
    out = C.c_void_p()
    stats = SubgraphStats()
    lp._check(_lib().kmp_extract_subgraphs(handle._h, C.c_uint32(int(k)), lp._ptr(part), C.byref(out),
                                           C.byref(stats)))
    return Subgraphs(out, stats, handle)
