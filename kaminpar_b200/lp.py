"""Python mirror of the reference's operator interface for the LP hot path, over the C ABI
(include/kaminpar_b200_lp.h -> kaminpar_b200/csrc/libkaminpar_b200.so).

Same names, argument meaning and error behaviour as the reference:

* ``LPClustering(c_ctx)`` with ``set_max_cluster_weight`` / ``set_desired_cluster_count`` /
  ``set_communities`` / ``compute_clustering(graph, free_memory_afterwards)``
  (kaminpar-shm/coarsening/clusterer.h:35-46, clustering/lp_clusterer.cc:376-399),
* ``LabelPropagationRefiner(ctx)`` with ``initialize(p_graph)`` / ``refine(p_graph, p_ctx)``
  (kaminpar-shm/refinement/refiner.h:34-56, refinement/lp/lp_refiner.cc:357-376),
* ``OverloadBalancer(ctx)`` with ``initialize(p_graph)`` / ``refine(p_graph, p_ctx)``
  (refinement/balancer/overload_balancer.cc:40-160, include/kaminpar_b200_balancer.h),
* ``UnderloadBalancer(ctx)`` with ``initialize(p_graph)`` / ``refine(p_graph, p_ctx)``
  (refinement/balancer/underload_balancer.cc:35-104, include/kaminpar_b200_balancer.h),
* ``PartitionContext.setup`` (kaminpar-shm/context.cc:27-70), ``compute_max_cluster_weight``
  (kaminpar-shm/coarsening/max_cluster_weights.h:17-46), ``create_default_context``
  (kaminpar-shm/presets.cc:109-450, LP fields only).

There is NO CPU fallback: if the CUDA library is missing or no device is present every compute call
raises ``RuntimeError``. Nothing here imports ``oracle/``.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from dataclasses import dataclass, field
from typing import Optional, Sequence

import numpy as np

from .graph import CSRGraph

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libkaminpar_b200.so")
_lib = None
ABI_VERSION = 3  # include/kaminpar_b200_lp.h: KMP_LP_ABI_VERSION

UINT32_MAX = 0xFFFFFFFF


class KmpConfig(C.Structure):
    _fields_ = [
        ("num_iterations", C.c_uint32),
        ("large_degree_threshold", C.c_uint32),
        ("max_num_neighbors", C.c_uint32),
        ("impl", C.c_int32),
        ("tie_breaking_strategy", C.c_int32),
        ("two_hop_strategy", C.c_int32),
        ("two_hop_threshold", C.c_double),
        ("isolated_nodes_strategy", C.c_int32),
        ("relabel_before_second_phase", C.c_int32),
        ("seed", C.c_int32),
        ("sync_subrounds", C.c_uint32),
        ("sync_granule_log2", C.c_uint32),
        ("sync_commit_passes", C.c_uint32),
        ("device", C.c_int32),
        ("schedule", C.c_int32),
    ]


class KmpStats(C.Structure):
    _fields_ = [
        ("iterations", C.c_uint32),
        ("moved", C.c_uint32 * 64),
        ("edges_scanned", C.c_uint64),
        ("nodes_visited", C.c_uint64),
        ("proposals", C.c_uint64),
        ("num_clusters", C.c_uint32),
        ("two_hop_ran", C.c_uint32),
        ("device_ms", C.c_float),
        ("sweep_ms", C.c_float),
        ("sweep_launches", C.c_uint64),
        ("kernel_launches", C.c_uint64),
        ("group_edges", C.c_uint64 * 12),
        ("group_nodes", C.c_uint64 * 12),
        ("group_launches", C.c_uint64 * 12),
        ("group_sweep_ms", C.c_float * 16),
        ("pull_rounds", C.c_uint32),
        ("push_rounds", C.c_uint32),
    ]

    def moved_list(self):
        return list(self.moved[: self.iterations])


class KmpBalanceStats(C.Structure):  # include/kaminpar_b200_balancer.h
    _fields_ = [
        ("rounds", C.c_uint32),
        ("moved", C.c_uint32 * 64),
        ("overload_before", C.c_int64),
        ("overload_after", C.c_int64),
        ("candidates", C.c_uint64),
        ("edges_scanned", C.c_uint64),
        ("kernel_launches", C.c_uint64),
        ("device_ms", C.c_float),
    ]

    def moved_list(self):
        return list(self.moved[: self.rounds])


class KmpUnderloadStats(C.Structure):  # include/kaminpar_b200_balancer.h
    _fields_ = [
        ("rounds", C.c_uint32),
        ("moved", C.c_uint32 * 64),
        ("underload_before", C.c_int64),
        ("underload_after", C.c_int64),
        ("candidates", C.c_uint64),
        ("edges_scanned", C.c_uint64),
        ("kernel_launches", C.c_uint64),
        ("device_ms", C.c_float),
    ]

    def moved_list(self):
        return list(self.moved[: self.rounds])


class KmpOverlayStats(C.Structure):  # include/kaminpar_b200_contraction.h
    _fields_ = [
        ("num_clusterings", C.c_uint32),
        ("num_clusters", C.c_uint32),
        ("sort_bits", C.c_uint32),
        ("kernel_launches", C.c_uint32),
        ("lp_device_ms", C.c_float),
        ("overlay_device_ms", C.c_float),
    ]


def library_path() -> str:
    return _LIB_PATH


def load_library():
    """Load the CUDA library. Fails loudly when it has not been built (no fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            raise RuntimeError(
                f"{_LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). kaminpar_b200 has no CPU fallback."
            )
        lib = C.CDLL(_LIB_PATH)
        lib.kmp_last_error.restype = C.c_char_p
        lib.kmp_lp_labels_device.restype = C.c_void_p
        require_symbols(lib, "kmp_overload_balance", "kmp_balance_select_all",  # include/kaminpar_b200_balancer.h
                        "kmp_underload_balance", "kmp_underload_select_all",
                        "kmp_lp_cluster_overlay", "kmp_overlay_clusterings")  # include/kaminpar_b200_contraction.h
        if lib.kmp_lp_abi_version() != ABI_VERSION:  # the ctypes structs below mirror exactly this header version
            raise RuntimeError(f"{_LIB_PATH}: ABI version {lib.kmp_lp_abi_version()} != {ABI_VERSION}; rebuild the library")
        _lib = lib
    return _lib


def require_symbols(lib, *symbols):
    """Refuses a library built before one of `symbols` existed."""
    for sym in symbols:
        if not hasattr(lib, sym):
            raise RuntimeError(f"{_LIB_PATH} lacks {sym}; rebuild the library")


def _check(rc: int):
    if rc != 0:
        msg = load_library().kmp_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"kaminpar_b200 error {rc}: {msg}")


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def report_message(fn, report) -> str:
    """The message the C function `fn` (a kmp_*_report_message) formats for `report`."""
    size = fn(C.byref(report), None, 0)
    buf = C.create_string_buffer(size + 1)
    fn(C.byref(report), buf, size + 1)
    return buf.value.decode()


class ReportError(RuntimeError):
    """An input refused with a report; `report` holds its first violation, `code` the library's error code."""

    def __init__(self, code: int, report):
        super().__init__(f"kaminpar_b200 error {code}: {report.message()}")
        self.code = code
        self.report = report


def check_report(rc: int, report, error):
    """_check, except that a call refused with a violation in `report` raises error(rc, report)."""
    if rc != 0 and report.kind != 0:
        raise error(rc, report)
    _check(rc)


def device_bytes(tensor):
    """(pointer, length) of the bytes of a contiguous torch CUDA tensor, for a reader that parses them on the
    device. The library reads them on its handle's stream, so the work torch has queued on its current stream is
    waited for first: a tensor just written by a kernel is read whole."""
    import torch

    if tensor.dtype.itemsize != 1 or not tensor.is_contiguous():
        raise ValueError("a device read needs a contiguous tensor of bytes")
    if not tensor.is_cuda:  # the library refuses device memory of another device than the handle's
        raise ValueError("a device read needs a CUDA tensor")
    torch.cuda.current_stream(tensor.device).synchronize()
    return C.c_void_p(tensor.data_ptr() or None), C.c_uint64(tensor.numel())


# --------------------------------------------------------------------------------------------
# Context mirror (LP fields of include/kaminpar-shm/kaminpar.h)
# --------------------------------------------------------------------------------------------
@dataclass
class LabelPropagationCoarseningContext:  # kaminpar.h:140-154, defaults presets.cc:140-153
    num_iterations: int = 5
    large_degree_threshold: int = UINT32_MAX
    max_num_neighbors: int = UINT32_MAX
    impl: int = 1  # TWO_PHASE
    relabel_before_second_phase: bool = False
    two_hop_strategy: int = 2  # MATCH_THREADWISE
    two_hop_threshold: float = 0.5
    isolated_nodes_strategy: int = 3  # MATCH_DURING_TWO_HOP
    tie_breaking_strategy: int = 1  # UNIFORM


@dataclass
class LabelPropagationRefinementContext:  # kaminpar.h:221-228, defaults presets.cc:339-347
    num_iterations: int = 5
    large_degree_threshold: int = UINT32_MAX
    max_num_neighbors: int = UINT32_MAX
    impl: int = 0  # SINGLE_PHASE
    tie_breaking_strategy: int = 1  # UNIFORM


@dataclass
class EngineContext:
    """Knobs of the GPU engine that have no reference counterpart (DESIGN.md "sync schedule")."""

    seed: int = 0
    sync_subrounds: int = 8
    sync_granule_log2: int = 4
    cluster_commit_passes: int = 1
    refine_commit_passes: int = 4
    device: int = -1
    # "sync": deterministic synchronous sub-rounds (any size, any number of GPUs); "seq_strict": the
    # reference's own one-thread order and random draws on one thread block -- bit-identical to the
    # unmodified reference at one thread, small inputs only (include/kaminpar_b200_lp.h KMP_SCHEDULE_*)
    schedule: str = "sync"


@dataclass
class ClusteringContext:
    lp: LabelPropagationCoarseningContext = field(default_factory=LabelPropagationCoarseningContext)
    cluster_weight_limit: str = "EPSILON_BLOCK_WEIGHT"  # presets.cc:155
    cluster_weight_multiplier: float = 1.0


@dataclass
class CoarseningContext:
    clustering: ClusteringContext = field(default_factory=ClusteringContext)
    contraction_limit: int = 2000  # presets.cc


@dataclass
class RefinementContext:
    lp: LabelPropagationRefinementContext = field(default_factory=LabelPropagationRefinementContext)


class PartitionContext:
    """kaminpar.h:417-531, context.cc:27-90 (the parts the LP path reads)."""

    def __init__(self):
        self.k = 0
        self.n = 0
        self.m = 0
        self.total_node_weight = 0
        self.original_total_node_weight = 0
        self.max_node_weight = 1
        self._epsilon = -1.0
        self._max_block_weights: list[int] = []
        self._unrelaxed: list[int] = []
        self._min_block_weights: list[int] = []
        self._uniform = False

    def setup(self, graph: CSRGraph, k_or_weights, epsilon: Optional[float] = None, relax: bool = False):
        if isinstance(k_or_weights, (int, np.integer)):
            k = int(k_or_weights)
            self._epsilon = float(epsilon)
            perfectly = int(math.ceil(1.0 * graph.total_node_weight() / k))
            weights = [int((1.0 + self._epsilon) * perfectly)] * k  # context.cc:33-36 (truncation)
            self._setup(graph, weights, relax)
            self._uniform = True
        else:
            self._setup(graph, [int(w) for w in k_or_weights], relax)
        return self

    def _setup(self, graph, weights, relax):
        self.n, self.m = graph.n, graph.m
        self.total_node_weight = self.original_total_node_weight = graph.total_node_weight()
        self.max_node_weight = graph.max_node_weight()
        self.k = len(weights)
        self._max_block_weights = list(weights)
        self._unrelaxed = list(weights)
        self._uniform = False
        if relax:  # context.cc:61-69
            eps = self.inferred_epsilon()
            self._max_block_weights = [
                max(w, int(math.ceil(1.0 * w / (1.0 + eps))) + self.max_node_weight) for w in weights
            ]

    def infer_epsilon(self, actual_total_node_weight: int) -> float:  # kaminpar.h:477-487
        if actual_total_node_weight == 0:
            return 0.0
        if self._uniform:
            mx = (1.0 + self._epsilon) * math.ceil(1.0 * self.original_total_node_weight / self.k)
            return mx / math.ceil(1.0 * actual_total_node_weight / self.k) - 1.0
        return 1.0 * sum(self._max_block_weights) / actual_total_node_weight - 1.0

    def inferred_epsilon(self) -> float:
        return self.infer_epsilon(self.total_node_weight)

    def max_block_weight(self, b: int) -> int:
        return self._max_block_weights[b]

    def max_block_weights(self) -> np.ndarray:
        return np.asarray(self._max_block_weights, dtype=np.int32)

    def perfectly_balanced_block_weight(self, b: int) -> int:  # kaminpar.h:436-438
        return int(math.ceil(1.0 * self._unrelaxed[b] / (1 + self.inferred_epsilon())))

    def perfectly_balanced_block_weights(self) -> np.ndarray:
        return np.asarray([self.perfectly_balanced_block_weight(b) for b in range(self.k)], dtype=np.int32)

    def min_block_weight(self, b: int) -> int:
        return self._min_block_weights[b] if self._min_block_weights else 0

    def has_min_block_weights(self) -> bool:
        return bool(self._min_block_weights)

    def setup_min_block_weights(self, weights: Sequence[int]):
        assert len(weights) == self.k
        self._min_block_weights = [int(w) for w in weights]

    def min_block_weights(self) -> Optional[np.ndarray]:
        return np.asarray(self._min_block_weights, dtype=np.int32) if self._min_block_weights else None


@dataclass
class Context:
    coarsening: CoarseningContext = field(default_factory=CoarseningContext)
    refinement: RefinementContext = field(default_factory=RefinementContext)
    partition: PartitionContext = field(default_factory=PartitionContext)
    engine: EngineContext = field(default_factory=EngineContext)


def create_default_context() -> Context:
    return Context()


def compute_max_cluster_weight(c_ctx: CoarseningContext, p_ctx: PartitionContext, n: int,
                               total_node_weight: int) -> int:
    """coarsening/max_cluster_weights.h:17-46."""
    limit = c_ctx.clustering.cluster_weight_limit
    if limit == "EPSILON_BLOCK_WEIGHT":
        div = min(max(n // c_ctx.contraction_limit, 2), p_ctx.k)
        mcw = (p_ctx.infer_epsilon(total_node_weight) * total_node_weight) / div
    elif limit == "BLOCK_WEIGHT":
        mcw = (1.0 + p_ctx.inferred_epsilon()) * total_node_weight / p_ctx.k
    elif limit == "ONE":
        mcw = 1.0
    else:
        mcw = 0.0
    return int(mcw * c_ctx.clustering.cluster_weight_multiplier)


class PartitionedGraph:
    """kaminpar-shm/datastructures/partitioned_graph.h:50-456 (labels + block weights)."""

    def __init__(self, graph: CSRGraph, k: int, partition: np.ndarray):
        self.graph = graph
        self._k = int(k)
        self.partition = np.ascontiguousarray(partition, dtype=np.uint32).copy()
        w = np.ones(graph.n, np.int64) if graph.vwgt is None else graph.vwgt.astype(np.int64)
        self._block_weights = np.bincount(self.partition, weights=w, minlength=k).astype(np.int32)

    def k(self) -> int:
        return self._k

    def block(self, u: int) -> int:
        return int(self.partition[u])

    def block_weight(self, b: int) -> int:
        return int(self._block_weights[b])

    def block_weights(self) -> np.ndarray:
        return self._block_weights


# --------------------------------------------------------------------------------------------
# Device handle
# --------------------------------------------------------------------------------------------
class LPHandle:
    """Owns one kmp_lp_handle (one CUDA stream on one device)."""

    def __init__(self, cfg: KmpConfig):
        self._lib = load_library()
        self._h = C.c_void_p()
        # results made on this handle (DeviceResult) free their arrays on its stream: while any is open, close() is
        # deferred to the last one's close -- also when the garbage collector finalises a reference cycle holding
        # both in arbitrary order
        self._children = 0
        self._close_pending = False
        _check(self._lib.kmp_lp_create(C.byref(cfg), C.byref(self._h)))
        self._graph_id = None

    def _adopt(self):
        """A DeviceResult of this handle opened: the handle outlives it."""
        self._children += 1

    def _release_child(self):
        """A DeviceResult of this handle closed: a deferred close() runs after the last one."""
        self._children -= 1
        if self._close_pending and self._children == 0:
            self.close()

    def close(self):
        if getattr(self, "_children", 0) > 0:
            self._close_pending = True
            return
        if getattr(self, "_h", None) is not None and self._h:
            self._lib.kmp_lp_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_graph(self, g: CSRGraph):
        _check(self._lib.kmp_lp_set_graph(self._h, C.c_uint32(g.n), C.c_uint32(g.m), _ptr(g.xadj), _ptr(g.adjncy),
                                          _ptr(g.vwgt), _ptr(g.adjwgt)))
        if g.sorted:  # CSRGraph::sorted(): only the seq_strict schedule reads it (the reference's chunk order)
            _check(self._lib.kmp_lp_set_graph_sorted(self._h, C.c_int(1)))
        self._graph_id = id(g)
        self._n = g.n

    def set_graph_device(self, n, m, d_xadj, d_adjncy, d_vwgt=0, d_adjwgt=0):
        """Device pointers (ints), e.g. torch tensors' data_ptr()."""
        _check(self._lib.kmp_lp_set_graph_device(self._h, C.c_uint32(n), C.c_uint32(m), C.c_void_p(d_xadj),
                                                 C.c_void_p(d_adjncy), C.c_void_p(d_vwgt or None),
                                                 C.c_void_p(d_adjwgt or None)))
        self._graph_id = None
        self._n = n

    def dist_init(self, rank: int, world: int, group=None):
        """One process per GPU: create the NCCL communicator inside the library (kmp_lp_dist_init). The id of
        rank 0 travels through torch.distributed (plumbing only); afterwards cluster() / refine() run the
        frontier-sharded schedule themselves, collectives included."""
        uid = (C.c_ubyte * 128)()
        if world > 1:
            import torch
            import torch.distributed as dist

            if rank == 0:
                _check(self._lib.kmp_lp_dist_unique_id(uid))
            t = torch.tensor(list(uid), dtype=torch.uint8, device="cuda")
            dist.broadcast(t, src=0, group=group)
            for i, b in enumerate(t.cpu().tolist()):
                uid[i] = b
        _check(self._lib.kmp_lp_dist_init(self._h, uid, C.c_uint32(rank), C.c_uint32(world)))

    def set_timing(self, enabled: bool):
        _check(self._lib.kmp_lp_set_timing(self._h, C.c_int(1 if enabled else 0)))

    def cluster(self, max_cluster_weight, desired=0, communities=None, out: Optional[np.ndarray] = None,
                fetch=True):
        stats = KmpStats()
        if fetch and out is None:
            out = np.empty(self._n, np.uint32)
        comm = None if communities is None else np.ascontiguousarray(communities, np.uint32)
        _check(self._lib.kmp_lp_cluster(self._h, C.c_int32(int(max_cluster_weight)), C.c_uint32(int(desired)),
                                        _ptr(comm), _ptr(out) if fetch else None, C.byref(stats)))
        return out, stats

    def cluster_overlay(self, num_levels, max_cluster_weight, desired=0, communities=None,
                        out: Optional[np.ndarray] = None, fetch=True):
        """kmp_lp_cluster_overlay: 2^num_levels clusterings of the graph (the same arguments, consecutive calls),
        intersected in OverlayClusterCoarsener's tree order (DESIGN.md §14). The result stays on the device as the
        handle's labels (contract_on_handle(handle, None) contracts it). Returns (clustering or None, stats)."""
        stats = KmpOverlayStats()
        if fetch and out is None:
            out = np.empty(self._n, np.uint32)
        comm = None if communities is None else np.ascontiguousarray(communities, np.uint32)
        _check(self._lib.kmp_lp_cluster_overlay(self._h, C.c_int(int(num_levels)), C.c_int32(int(max_cluster_weight)),
                                                C.c_uint32(int(desired)), _ptr(comm), _ptr(out) if fetch else None,
                                                C.byref(stats)))
        return out, stats

    def overlay(self, clusterings, out: Optional[np.ndarray] = None, fetch=True):
        """kmp_overlay_clusterings: the overlay tree over given clusterings of the handle's graph (a power of two of
        them, each n ids in [0, n)). The result becomes the handle's device labels. Returns (overlay or None, stats)."""
        cl = np.ascontiguousarray(np.asarray(clusterings, np.uint32))
        if cl.ndim != 2 or cl.shape[1] != self._n:
            raise ValueError("clusterings must be a sequence of clusterings of the graph's n vertices")
        stats = KmpOverlayStats()
        if fetch and out is None:
            out = np.empty(self._n, np.uint32)
        _check(self._lib.kmp_overlay_clusterings(self._h, C.c_uint32(cl.shape[0]), _ptr(cl),
                                                 _ptr(out) if fetch else None, C.byref(stats)))
        return out, stats

    def refine(self, k, max_block_weights, partition: Optional[np.ndarray], min_block_weights=None,
               communities=None):
        stats = KmpStats()
        mbw = np.ascontiguousarray(max_block_weights, np.int32)
        mnw = None if min_block_weights is None else np.ascontiguousarray(min_block_weights, np.int32)
        comm = None if communities is None else np.ascontiguousarray(communities, np.uint32)
        bw = np.zeros(k, np.int32)
        _check(self._lib.kmp_lp_refine(self._h, C.c_uint32(int(k)), _ptr(mbw), _ptr(mnw), _ptr(comm),
                                       _ptr(partition), _ptr(bw), C.byref(stats)))
        return partition, bw, stats

    def upload_partition(self, partition: np.ndarray):
        p = np.ascontiguousarray(partition, np.uint32)
        _check(self._lib.kmp_lp_upload_partition(self._h, _ptr(p)))

    def download_labels(self) -> np.ndarray:
        out = np.empty(self._n, np.uint32)
        _check(self._lib.kmp_lp_download_labels(self._h, _ptr(out)))
        return out

    def select_all(self, mode, labels, weights, max_weights=None, max_cluster_weight=0, min_weights=None,
                   call_index=0, iteration=0):
        labels = np.ascontiguousarray(labels, np.uint32)
        weights = np.ascontiguousarray(weights, np.int32)
        mw = None if max_weights is None else np.ascontiguousarray(max_weights, np.int32)
        mn = None if min_weights is None else np.ascontiguousarray(min_weights, np.int32)
        tgt = np.empty(self._n, np.uint32)
        fav = np.empty(self._n, np.uint32)
        _check(self._lib.kmp_lp_select_all(self._h, C.c_int(mode), _ptr(labels), _ptr(weights),
                                           C.c_uint32(len(weights)), _ptr(mw), C.c_int32(int(max_cluster_weight)),
                                           _ptr(mn), C.c_uint32(call_index), C.c_uint32(iteration), _ptr(tgt),
                                           _ptr(fav)))
        return tgt, fav

    def overload_balance(self, k, max_block_weights, perfectly_balanced_block_weights, partition: Optional[np.ndarray]):
        """kmp_overload_balance: partition (uint32, balanced in place) or None = the labels on the device.
        Returns (improved, block_weights, stats)."""
        stats = KmpBalanceStats()
        mbw = np.ascontiguousarray(max_block_weights, np.int32)
        pbw = np.ascontiguousarray(perfectly_balanced_block_weights, np.int32)
        bw = np.zeros(k, np.int32)
        improved = C.c_int(0)
        if partition is not None:
            assert partition.dtype == np.uint32 and partition.flags.c_contiguous
        _check(self._lib.kmp_overload_balance(self._h, C.c_uint32(int(k)), _ptr(mbw), _ptr(pbw), _ptr(partition), _ptr(bw),
                                              C.byref(improved), C.byref(stats)))
        return bool(improved.value), bw, stats

    def balance_select_all(self, k, labels, block_weights, max_block_weights, call_index=0, round=0):
        """kmp_balance_select_all: (target[n] uint32, key[n] float32) against frozen state."""
        labels = np.ascontiguousarray(labels, np.uint32)
        bw = np.ascontiguousarray(block_weights, np.int32)
        mbw = np.ascontiguousarray(max_block_weights, np.int32)
        tgt = np.empty(self._n, np.uint32)
        key = np.empty(self._n, np.float32)
        _check(self._lib.kmp_balance_select_all(self._h, C.c_uint32(int(k)), _ptr(labels), _ptr(bw), _ptr(mbw),
                                                C.c_uint32(call_index), C.c_uint32(round), _ptr(tgt), _ptr(key)))
        return tgt, key

    def underload_balance(self, k, max_block_weights, min_block_weights, partition: Optional[np.ndarray]):
        """kmp_underload_balance: partition (uint32, balanced in place) or None = the labels on the device;
        min_block_weights None = no minimum weights (no device work, block weights None).
        Returns (improved, block_weights, stats)."""
        stats = KmpUnderloadStats()
        mbw = np.ascontiguousarray(max_block_weights, np.int32)
        mnw = None if min_block_weights is None else np.ascontiguousarray(min_block_weights, np.int32)
        bw = np.zeros(k, np.int32)
        improved = C.c_int(0)
        if partition is not None:
            assert partition.dtype == np.uint32 and partition.flags.c_contiguous
        _check(self._lib.kmp_underload_balance(self._h, C.c_uint32(int(k)), _ptr(mbw), _ptr(mnw), _ptr(partition),
                                               _ptr(bw), C.byref(improved), C.byref(stats)))
        return bool(improved.value), (bw if mnw is not None else None), stats

    def underload_select_all(self, k, labels, block_weights, max_block_weights, min_block_weights, call_index=0,
                             round=0):
        """kmp_underload_select_all: (target[n] uint32, key[n] float32) against frozen state."""
        labels = np.ascontiguousarray(labels, np.uint32)
        bw = np.ascontiguousarray(block_weights, np.int32)
        mbw = np.ascontiguousarray(max_block_weights, np.int32)
        mnw = np.ascontiguousarray(min_block_weights, np.int32)
        tgt = np.empty(self._n, np.uint32)
        key = np.empty(self._n, np.float32)
        _check(self._lib.kmp_underload_select_all(self._h, C.c_uint32(int(k)), _ptr(labels), _ptr(bw), _ptr(mbw),
                                                  _ptr(mnw), C.c_uint32(call_index), C.c_uint32(round), _ptr(tgt),
                                                  _ptr(key)))
        return tgt, key

    def edge_cut(self) -> int:
        cut = C.c_int64(0)
        _check(self._lib.kmp_lp_edge_cut(self._h, C.byref(cut)))
        return int(cut.value)

    def free_scratch(self):
        _check(self._lib.kmp_lp_free_scratch(self._h))


def pool_usage(handle: LPHandle, reset: bool = False):
    """(bytes in use, most bytes in use since the last reset) of the device pool the handle and its results allocate
    from; reset restarts the high-water mark at the current use."""
    used, high = C.c_uint64(), C.c_uint64()
    _check(load_library().kmp_pool_usage(handle._h, C.c_int(int(reset)), C.byref(used), C.byref(high)))
    return int(used.value), int(high.value)


class DeviceResult:
    """A result object of a graph operation on an LPHandle (a coarse graph, a prepared graph, extracted subgraphs).
    It owns device memory of the handle's pool, freed on the handle's stream when it closes, so the handle stays open
    until the last of its results is closed. A subclass names the C symbol that destroys it in `_destroy`."""

    _destroy: str

    def __init__(self, ptr, stats, handle: LPHandle):
        self._g = ptr
        self.stats = stats
        self._handle = handle
        handle._adopt()

    def _device_ptrs(self, symbol: str, count: int):
        """The `count` device pointers `symbol` hands out, as integers (0: absent)."""
        ptrs = [C.c_void_p() for _ in range(count)]
        _check(getattr(load_library(), symbol)(self._g, *[C.byref(p) for p in ptrs]))
        return tuple(int(p.value or 0) for p in ptrs)

    def _download_csr(self, symbol: str, n: int, m: int, vwgt: bool, adjwgt: bool, *extra):
        """(xadj, adjncy, vwgt, adjwgt) of n vertices and m edges copied to the host by `symbol`, the weights None
        unless present; `extra` are the host arrays (or None) that `symbol` fills after adjwgt."""
        xadj = np.zeros(n + 1, np.uint32)
        adj = np.zeros(m, np.uint32)
        vw = np.zeros(n, np.int32) if vwgt else None
        ew = np.zeros(m, np.int32) if adjwgt else None
        _check(getattr(load_library(), symbol)(self._g, _ptr(xadj), _ptr(adj), _ptr(vw), _ptr(ew),
                                               *[_ptr(a) for a in extra]))
        return xadj, adj, vw, ew

    def close(self):
        if getattr(self, "_g", None):
            getattr(load_library(), self._destroy)(self._g)  # frees on the handle's stream: the handle must still exist
            self._g = None
            self._handle._release_child()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_SCHEDULES = {"sync": 0, "seq_strict": 1}


def _cluster_config(lp: LabelPropagationCoarseningContext, eng: EngineContext) -> KmpConfig:
    return KmpConfig(
        lp.num_iterations, lp.large_degree_threshold, lp.max_num_neighbors, lp.impl, lp.tie_breaking_strategy,
        lp.two_hop_strategy, lp.two_hop_threshold, lp.isolated_nodes_strategy, int(lp.relabel_before_second_phase),
        eng.seed, eng.sync_subrounds, eng.sync_granule_log2, eng.cluster_commit_passes, eng.device,
        _SCHEDULES[eng.schedule],
    )


def _refine_config(lp: LabelPropagationRefinementContext, eng: EngineContext) -> KmpConfig:
    return KmpConfig(
        lp.num_iterations, lp.large_degree_threshold, lp.max_num_neighbors, lp.impl, lp.tie_breaking_strategy,
        0, 0.5, 0, 0, eng.seed, eng.sync_subrounds, eng.sync_granule_log2, eng.refine_commit_passes, eng.device,
        _SCHEDULES[eng.schedule],
    )


# --------------------------------------------------------------------------------------------
# Reference-shaped operators
# --------------------------------------------------------------------------------------------
class LPClustering:
    """Drop-in for ``kaminpar::shm::LPClustering : Clusterer`` (lp_clusterer.h:19, clusterer.h:19-47)."""

    def __init__(self, c_ctx: CoarseningContext, engine: Optional[EngineContext] = None):
        self._c_ctx = c_ctx
        self._engine = engine or EngineContext()
        self._handle = LPHandle(_cluster_config(c_ctx.clustering.lp, self._engine))
        self._max_cluster_weight = None  # kInvalidBlockWeight until set (lp_clusterer.cc:287)
        self._desired = 0
        self._communities = None
        self._graph = None
        self.last_stats: Optional[KmpStats] = None

    def invalidate_graph(self):
        """The graph object is recognised by identity: call this when its arrays were rewritten in place."""
        self._graph = None

    def set_max_cluster_weight(self, weight: int):
        self._max_cluster_weight = int(weight)

    def set_desired_cluster_count(self, count: int):
        self._desired = int(count)

    def set_communities(self, communities):
        self._communities = None if communities is None or len(communities) == 0 else np.asarray(communities)

    def compute_clustering(self, graph: CSRGraph, free_memory_afterwards: bool = False,
                           clustering: Optional[np.ndarray] = None) -> np.ndarray:
        """Returns clustering[u] in [0, n): id of the cluster's founding vertex, not compacted."""
        if self._max_cluster_weight is None:
            raise ValueError("set_max_cluster_weight() must be called before compute_clustering()")
        if self._graph is not graph:
            self._handle.set_graph(graph)
            self._graph = graph
        out, stats = self._handle.cluster(self._max_cluster_weight, self._desired, self._communities, out=clustering)
        self.last_stats = stats
        if free_memory_afterwards:
            self._handle.free_scratch()
        return out


class LabelPropagationRefiner:
    """Drop-in for ``kaminpar::shm::LabelPropagationRefiner : Refiner`` (lp_refiner.h:19,
    refiner.h:18-57)."""

    def __init__(self, ctx: Context):
        self._ctx = ctx
        self._handle = LPHandle(_refine_config(ctx.refinement.lp, ctx.engine))
        self._communities = None
        self._graph = None
        self.last_stats: Optional[KmpStats] = None

    def name(self) -> str:
        return "Label Propagation"

    def invalidate_graph(self):
        self._graph = None

    def set_communities(self, communities):
        self._communities = None if communities is None or len(communities) == 0 else np.asarray(communities)

    def initialize(self, p_graph: PartitionedGraph):
        if self._graph is not p_graph.graph:
            self._handle.set_graph(p_graph.graph)
            self._graph = p_graph.graph

    def refine(self, p_graph: PartitionedGraph, p_ctx: PartitionContext) -> bool:
        if self._graph is not p_graph.graph:
            raise ValueError("initialize(p_graph) must be called before refine()")
        assert p_graph.k() <= p_ctx.k
        _, bw, stats = self._handle.refine(p_ctx.k, p_ctx.max_block_weights(), p_graph.partition,
                                           p_ctx.min_block_weights(), self._communities)
        p_graph._block_weights = bw
        self.last_stats = stats
        return True  # lp_refiner.cc:88


class OverloadBalancer:
    """Drop-in for ``kaminpar::shm::OverloadBalancer : Refiner`` (overload_balancer.h, refiner.h:18-57) on the
    device. Its selection rule is the reference's without thread order (DESIGN.md §11)."""

    def __init__(self, ctx: Context):
        self._ctx = ctx
        self._handle = LPHandle(_refine_config(ctx.refinement.lp, ctx.engine))
        self._graph = None
        self.last_stats: Optional[KmpBalanceStats] = None

    def name(self) -> str:
        return "Overload Balancer"

    def invalidate_graph(self):
        self._graph = None

    def initialize(self, p_graph: PartitionedGraph):
        pass  # overload_balancer.cc:40-43: nothing until refine() finds an overloaded block

    def refine(self, p_graph: PartitionedGraph, p_ctx: PartitionContext) -> bool:
        assert p_graph.k() <= p_ctx.k
        mbw = p_ctx.max_block_weights()
        w = p_graph.block_weights().astype(np.int64)
        if int(np.maximum(w - mbw[: len(w)], 0).sum()) == 0:  # metrics::total_overload == 0: no device work
            self.last_stats = None
            return False
        if self._graph is not p_graph.graph:
            self._handle.set_graph(p_graph.graph)
            self._graph = p_graph.graph
        improved, bw, stats = self._handle.overload_balance(p_ctx.k, mbw, p_ctx.perfectly_balanced_block_weights(),
                                                            p_graph.partition)
        p_graph._block_weights = bw
        self.last_stats = stats
        return improved


class UnderloadBalancer:
    """Drop-in for ``kaminpar::shm::UnderloadBalancer : Refiner`` (underload_balancer.h, refiner.h:18-57) on the
    device. Its selection rule is the reference's without thread order (DESIGN.md §12)."""

    def __init__(self, ctx: Context):
        self._ctx = ctx
        self._handle = LPHandle(_refine_config(ctx.refinement.lp, ctx.engine))
        self._graph = None
        self.last_stats: Optional[KmpUnderloadStats] = None

    def name(self) -> str:
        return "Underload Balancer"

    def invalidate_graph(self):
        self._graph = None

    def initialize(self, p_graph: PartitionedGraph):
        pass  # underload_balancer.cc:35-37: nothing to do

    def refine(self, p_graph: PartitionedGraph, p_ctx: PartitionContext) -> bool:
        assert p_graph.k() <= p_ctx.k
        mnw = p_ctx.min_block_weights()
        if mnw is None:  # underload_balancer.cc:47: no minimum weights
            self.last_stats = None
            return False
        w = p_graph.block_weights().astype(np.int64)
        if bool(np.all(w >= mnw[: len(w)])):  # metrics::is_min_balanced: no device work
            self.last_stats = None
            return False
        if self._graph is not p_graph.graph:
            self._handle.set_graph(p_graph.graph)
            self._graph = p_graph.graph
        improved, bw, stats = self._handle.underload_balance(p_ctx.k, p_ctx.max_block_weights(), mnw, p_graph.partition)
        p_graph._block_weights = bw
        self.last_stats = stats
        return improved
