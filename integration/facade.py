"""`KaMinPar` facade (include/kaminpar-shm/kaminpar.h:857-997): CSRGraph in, partition vector out.

This is NOT a re-implementation of the multilevel partitioner. It drives the UNMODIFIED reference partitioner
(coarsening loop, contraction, initial partitioning, balancers) compiled by `make -C oracle ref_b200` with the
GPU label-propagation clusterer / refiner swapped in behind `factories.cc` (integration/, INTEGRATION.md §2).
The library only exists where the reference sources were available at build time; without it the constructor
fails loudly -- there is no fallback partitioner.

Lives in integration/ (demo / test infrastructure), NOT in the product package: it loads a build of the reference
from oracle/_ref/, which nothing under kaminpar_b200/ may do."""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import numpy as np

from kaminpar_b200.graph import CSRGraph

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB_B200 = os.path.join(_ROOT, "oracle", "_ref", "libkaminpar_ref_b200.so")


class KaMinPar:
    """Mirrors `kaminpar::KaMinPar`: `copy_graph` / `borrow_and_mutate_graph`, `set_k`,
    `set_uniform_max_block_weights`, `compute_partition` (returns the edge cut), `reseed`. Default preset, one
    host thread (the configuration in which the reference is deterministic)."""

    _seed = 0

    def __init__(self, num_threads: int = 1):
        if not os.path.exists(_LIB_B200):
            raise RuntimeError(f"{_LIB_B200} is missing: build it with `make -C oracle ref_b200` where the KaMinPar "
                               "sources are available (it is the reference partitioner with the GPU LP plugged in)")
        self._lib = C.CDLL(_LIB_B200)
        self._lib.kmpfull_compute_partition.restype = C.c_longlong
        self._threads = int(num_threads)
        self._graph: Optional[CSRGraph] = None
        self._k = 2
        self._eps = 0.03

    @classmethod
    def reseed(cls, seed: int):  # kaminpar.h:869
        cls._seed = int(seed)

    def copy_graph(self, xadj, adjncy, vwgt=None, adjwgt=None):  # kaminpar.h:925-930
        self._graph = CSRGraph(np.array(xadj, np.uint32), np.array(adjncy, np.uint32),
                               None if vwgt is None else np.array(vwgt, np.int32),
                               None if adjwgt is None else np.array(adjwgt, np.int32))

    borrow_and_mutate_graph = copy_graph  # kaminpar.h:912-917 (the driver copies either way)

    def set_graph(self, graph: CSRGraph):
        self._graph = graph

    def set_k(self, k: int):
        self._k = int(k)

    def set_uniform_max_block_weights(self, epsilon: float):
        self._eps = float(epsilon)

    def compute_partition(self, partition: Optional[np.ndarray] = None):
        """Returns (edge_cut, partition)."""
        g = self._graph
        if g is None:
            raise ValueError("no graph set")
        out = np.zeros(g.n, np.uint32) if partition is None else partition
        cut = self._lib.kmpfull_compute_partition(
            C.c_uint32(g.n), g.xadj.ctypes.data_as(C.c_void_p), g.adjncy.ctypes.data_as(C.c_void_p),
            None if g.vwgt is None else g.vwgt.ctypes.data_as(C.c_void_p),
            None if g.adjwgt is None else g.adjwgt.ctypes.data_as(C.c_void_p), C.c_uint32(self._k),
            C.c_double(self._eps), C.c_int(self._seed), C.c_int(self._threads), out.ctypes.data_as(C.c_void_p))
        return int(cut), out
