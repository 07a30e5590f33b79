"""Block bipartitioning on the device, over the C ABI in include/kaminpar_b200_bipartition.h (device code:
kaminpar_b200/csrc/kmp_bipartition.cuh, DESIGN.md §20): KaMinPar's multilevel initial bipartitioner on every block of
a Subgraphs that is split in two, between extract_subgraphs and Subgraphs.copy_partitions.

    IPConfig                     kmp_ip_config, the supported fields of InitialPartitioningContext
    default_config()             the default preset's values
    bipartition(subgraphs, handle, k_prime, input_k, max_block_weights, seed=..., total_node_weight=..., ...)
                                 -> torch tensor of n sub-block ids on the handle's device (block-major)

There is no CPU fallback: without the CUDA library / a GPU every call raises.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import lp

NOOP, TWOWAY_SIMPLE_FM, TWOWAY_ADAPTIVE_FM, TWOWAY_FLOW = 0, 1, 2, 3
EPSILON_BLOCK_WEIGHT, BLOCK_WEIGHT, ONE, ZERO = 0, 1, 2, 3


class IPRefinement(C.Structure):
    """kmp_ip_refinement: a list of at most one algorithm (num_algorithms 0 = NOOP) and its FM settings."""

    _fields_ = [
        ("num_algorithms", C.c_uint32),
        ("algorithm", C.c_int32),
        ("num_fruitless_moves", C.c_uint32),
        ("alpha", C.c_double),
        ("num_iterations", C.c_uint64),
        ("improvement_abortion_threshold", C.c_double),
    ]


class IPConfig(C.Structure):
    """kmp_ip_config. IPConfig() holds the default preset's values."""

    _fields_ = [
        ("contraction_limit", C.c_uint32),
        ("convergence_threshold", C.c_double),
        ("large_degree_threshold", C.c_uint32),
        ("cluster_weight_limit", C.c_int32),
        ("cluster_weight_multiplier", C.c_double),
        ("pool_refinement", IPRefinement),
        ("repetition_multiplier", C.c_double),
        ("min_num_repetitions", C.c_int32),
        ("min_num_non_adaptive_repetitions", C.c_int32),
        ("max_num_repetitions", C.c_int32),
        ("num_seed_iterations", C.c_int32),
        ("use_adaptive_bipartitioner_selection", C.c_int32),
        ("enable_bfs_bipartitioner", C.c_int32),
        ("enable_ggg_bipartitioner", C.c_int32),
        ("enable_random_bipartitioner", C.c_int32),
        ("refinement", IPRefinement),
        ("refine_pool_partition", C.c_int32),
        ("use_adaptive_epsilon", C.c_int32),
    ]

    def __init__(self, **kw):
        super().__init__()
        fm = dict(num_algorithms=1, algorithm=TWOWAY_SIMPLE_FM, num_fruitless_moves=100, alpha=1.0, num_iterations=5,
                  improvement_abortion_threshold=0.0001)
        defaults = dict(contraction_limit=20, convergence_threshold=0.05, large_degree_threshold=1000000,
                        cluster_weight_limit=BLOCK_WEIGHT, cluster_weight_multiplier=1.0 / 12.0,
                        pool_refinement=IPRefinement(**fm), repetition_multiplier=1.0, min_num_repetitions=10,
                        min_num_non_adaptive_repetitions=5, max_num_repetitions=50, num_seed_iterations=1,
                        use_adaptive_bipartitioner_selection=1, enable_bfs_bipartitioner=1,
                        enable_ggg_bipartitioner=1, enable_random_bipartitioner=1, refinement=IPRefinement(**fm),
                        refine_pool_partition=0, use_adaptive_epsilon=1)
        defaults.update(kw)
        for key, value in defaults.items():
            setattr(self, key, value)


def preset(name: str) -> IPConfig:
    """The initial-partitioning fields of KaMinPar's presets default, fast, largek and largek-fast (presets.cc)."""
    c = IPConfig()
    if name == "default":
        return c
    if name == "fast":
        c.min_num_repetitions = c.min_num_non_adaptive_repetitions = c.max_num_repetitions = 1
        return c
    if name in ("largek", "largek-fast"):
        c.min_num_repetitions, c.min_num_non_adaptive_repetitions, c.max_num_repetitions = 4, 2, 4
        if name == "largek-fast":
            c.min_num_repetitions, c.min_num_non_adaptive_repetitions, c.max_num_repetitions = 2, 1, 2
            c.enable_ggg_bipartitioner = 0
            c.pool_refinement.algorithm = NOOP
            c.pool_refinement.num_iterations = 1
            c.refine_pool_partition = 1
        return c
    raise ValueError("unknown preset " + name)


class BipartitionStats(C.Structure):
    """kmp_bipartition_stats."""

    _fields_ = [
        ("blocks_split", C.c_uint32),
        ("pool_runs", C.c_uint32),
        ("coarsening_levels", C.c_uint32),
        ("arena_retries", C.c_uint32),
        ("kernel_launches", C.c_uint32),
        ("device_ms", C.c_float),
    ]


def _lib():
    lib = lp.load_library()
    if not getattr(lib, "_bipartition_ready", False):
        lp.require_symbols(lib, "kmp_bipartition_subgraphs", "kmp_ip_default_config", "kmp_lp_handle_device")
        lib.kmp_lp_handle_device.restype = C.c_int
        lib.kmp_lp_handle_device.argtypes = [C.c_void_p]
        lib.kmp_ip_default_config.restype = IPConfig
        lib.kmp_ip_default_config.argtypes = []
        lib.kmp_bipartition_subgraphs.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p,
                                                  C.c_int, C.c_int64, C.c_double, C.c_void_p, C.c_int32, C.c_void_p,
                                                  C.c_void_p]
        lib._bipartition_ready = True
    return lib


def default_config() -> IPConfig:
    """kmp_ip_default_config() from the library."""
    return _lib().kmp_ip_default_config()


def bipartition_into(subgraphs, handle: lp.LPHandle, k_prime: int, input_k: int, max_block_weights, out_ptr: int, *,
                     seed: int, total_node_weight: int, ip_config: Optional[IPConfig] = None, uniform: bool = True,
                     epsilon: float = 0.03) -> BipartitionStats:
    """kmp_bipartition_subgraphs into a device buffer given as an integer pointer (n uint32 entries)."""
    mbw = np.ascontiguousarray(max_block_weights, np.int32)
    if len(mbw) != input_k:
        raise ValueError("max_block_weights needs input_k entries")
    cfg = ip_config if ip_config is not None else IPConfig()
    stats = BipartitionStats()
    lp._check(_lib().kmp_bipartition_subgraphs(handle._h, subgraphs._g, C.c_uint32(k_prime), C.c_uint32(input_k),
                                               lp._ptr(mbw), int(bool(uniform)), C.c_int64(int(total_node_weight)),
                                               C.c_double(epsilon), C.byref(cfg), C.c_int32(int(seed)),
                                               C.c_void_p(out_ptr) if out_ptr else None, C.byref(stats)))
    return stats


def bipartition(subgraphs, handle: lp.LPHandle, k_prime: int, input_k: int, max_block_weights, *, seed: int,
                total_node_weight: int, ip_config: Optional[IPConfig] = None, uniform: bool = True,
                epsilon: float = 0.03):
    """The blocks' sub-partitions as a torch tensor of n sub-block ids on the handle's device, block-major: its
    data_ptr() goes straight into Subgraphs.copy_partitions. max_block_weights, total_node_weight, uniform and epsilon
    describe the input graph's partition context at input_k. Returns (tensor, BipartitionStats)."""
    import torch

    dev = torch.device("cuda", int(_lib().kmp_lp_handle_device(handle._h)))
    out = torch.empty(max(subgraphs.n, 1), dtype=torch.int32, device=dev)[:subgraphs.n]
    torch.cuda.current_stream(dev).synchronize()
    stats = bipartition_into(subgraphs, handle, k_prime, input_k, max_block_weights, out.data_ptr(), seed=seed,
                             ip_config=ip_config, uniform=uniform, total_node_weight=total_node_weight,
                             epsilon=epsilon)
    return out, stats
