"""ctypes bindings for the CPU oracle (oracle/liblp_oracle.so) and, when it has been built in the
authoring container, for the unmodified reference compiled against the serial oneTBB stand-in
(oracle/_ref/libkaminpar_ref.so).

TEST INFRASTRUCTURE ONLY -- imported by tests/, __graft_entry__.smoke() and bench.py's CPU-baseline
legs. The product (kaminpar_b200/) never imports this module.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import numpy as np

# precaution for the OpenMP stand-in build of the reference (sizeable per-thread buffers on the stack);
# has to be in the environment before libgomp initialises
os.environ.setdefault("OMP_STACKSIZE", "64M")

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_LIB = os.path.join(_HERE, "_ref", "libkaminpar_ref.so")          # serial stand-in: deterministic, pins the oracle
REF_OMP_LIB = os.path.join(_HERE, "_ref", "libkaminpar_ref_omp.so")  # OpenMP stand-in: all host cores (CPU baseline)
ORACLE_LIB = os.path.join(_HERE, "liblp_oracle.so")

U32P = np.ctypeslib.ndpointer(dtype=np.uint32, flags="C_CONTIGUOUS")
I32P = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")


def _opt(a: Optional[np.ndarray], dtype):
    if a is None:
        return None
    a = np.ascontiguousarray(a, dtype=dtype)
    return a.ctypes.data_as(C.c_void_p)


class LPParams(C.Structure):
    """Mirror of LabelPropagationCoarseningContext / ...RefinementContext
    (include/kaminpar-shm/kaminpar.h:140-154, :221-228)."""

    _fields_ = [
        ("num_iterations", C.c_uint32),
        ("large_degree_threshold", C.c_uint32),
        ("max_num_neighbors", C.c_uint32),
        ("impl", C.c_int32),  # 0 SINGLE_PHASE, 1 TWO_PHASE, 2 GROWING_HASH_TABLES
        ("tie_breaking", C.c_int32),  # 0 GEOMETRIC, 1 UNIFORM
        ("two_hop_strategy", C.c_int32),  # 0 DISABLE 1 MATCH 2 MATCH_THREADWISE 3 CLUSTER 4 CLUSTER_THREADWISE
        ("two_hop_threshold", C.c_double),
        ("isolated_nodes_strategy", C.c_int32),  # 0 KEEP 1 MATCH 2 CLUSTER 3 MATCH_DURING_TWO_HOP 4 CLUSTER_DURING_TWO_HOP
    ]


def default_cluster_params() -> LPParams:
    # presets.cc:140-153
    return LPParams(5, 0xFFFFFFFF, 0xFFFFFFFF, 1, 1, 2, 0.5, 3)


def default_refine_params() -> LPParams:
    # presets.cc:339-347
    return LPParams(5, 0xFFFFFFFF, 0xFFFFFFFF, 0, 1, 0, 0.5, 0)


# ------------------------------------------------------------------------------------------------
# Reference (unmodified sources + serial TBB stand-in)
# ------------------------------------------------------------------------------------------------
_ref = None


def have_reference() -> bool:
    return os.path.exists(REF_LIB)


def ref():
    global _ref
    if _ref is None:
        lib = C.CDLL(REF_LIB)
        lib.kmpref_version.restype = C.c_char_p
        lib.kmpref_rearrange_by_degree_buckets.restype = C.c_uint32
        lib.kmpref_edge_cut.restype = C.c_int64
        lib.kmpref_max_cluster_weight.restype = C.c_int32
        _ref = lib
    return _ref


def _garrs(g):
    return (
        C.c_uint32(g.n), C.c_uint32(g.m),
        g.xadj.ctypes.data_as(C.c_void_p), g.adjncy.ctypes.data_as(C.c_void_p),
        _opt(g.vwgt, np.int32), _opt(g.adjwgt, np.int32),
    )


def ref_rearrange(g, remove_isolated=True):
    """graph::rearrange_by_degree_buckets (+ remove_isolated_nodes). Returns (graph, old_to_new)."""
    from kaminpar_b200.graph import CSRGraph

    xadj = np.zeros(g.n + 1, np.uint32)
    adj = np.zeros(g.m, np.uint32)
    vw = np.zeros(g.n, np.int32) if g.vwgt is not None else None
    ew = np.zeros(g.m, np.int32) if g.adjwgt is not None else None
    o2n = np.zeros(g.n, np.uint32)
    buckets = np.zeros(34, np.uint32)
    nb = C.c_uint32(0)
    n_lp = ref().kmpref_rearrange_by_degree_buckets(
        *_garrs(g), C.c_int(1 if remove_isolated else 0),
        xadj.ctypes.data_as(C.c_void_p), adj.ctypes.data_as(C.c_void_p), _opt(vw, np.int32), _opt(ew, np.int32),
        o2n.ctypes.data_as(C.c_void_p), buckets.ctypes.data_as(C.c_void_p), C.byref(nb),
    )
    out = CSRGraph(
        xadj=xadj[: n_lp + 1].copy(), adjncy=adj, vwgt=None if vw is None else vw[:n_lp].copy(), adjwgt=ew,
        sorted=True, buckets=buckets,
    )
    return out, o2n


_ref_omp = None


def have_parallel_reference() -> bool:
    return os.path.exists(REF_OMP_LIB)


def ref_omp():
    global _ref_omp
    if _ref_omp is None:
        _ref_omp = C.CDLL(REF_OMP_LIB)
    return _ref_omp


def ref_lp_cluster(g, seed, max_cluster_weight, desired=0, params=None, num_calls=1, parallel=False):
    """parallel=True: the same unmodified sources on all host cores (OpenMP mode of the stand-in);
    like the reference with T > 1 threads the result then depends on thread timing."""
    params = params or default_cluster_params()
    out = np.zeros(g.n * num_calls, np.uint32)
    (ref_omp() if parallel else ref()).kmpref_lp_cluster(
        *_garrs(g), C.c_int(1 if g.sorted else 0), C.c_int(seed), C.c_int32(max_cluster_weight),
        C.c_uint32(desired), C.byref(params), C.c_int(num_calls), out.ctypes.data_as(C.c_void_p),
    )
    return out if num_calls == 1 else out.reshape(num_calls, g.n)


def ref_lp_refine(g, seed, k, max_block_weights, partition, params=None, min_block_weights=None):
    params = params or default_refine_params()
    part = np.ascontiguousarray(partition, dtype=np.uint32).copy()
    bw = np.zeros(k, np.int32)
    mbw = np.ascontiguousarray(max_block_weights, dtype=np.int32)
    ref().kmpref_lp_refine(
        *_garrs(g), C.c_int(1 if g.sorted else 0), C.c_int(seed), C.c_uint32(k), mbw.ctypes.data_as(C.c_void_p),
        _opt(min_block_weights, np.int32), C.byref(params), part.ctypes.data_as(C.c_void_p),
        bw.ctypes.data_as(C.c_void_p),
    )
    return part, bw


def ref_edge_cut(g, k, partition) -> int:
    part = np.ascontiguousarray(partition, dtype=np.uint32)
    return int(ref().kmpref_edge_cut(*_garrs(g), C.c_uint32(k), part.ctypes.data_as(C.c_void_p)))


def ref_max_cluster_weight(g, k, eps=0.03) -> int:
    return int(ref().kmpref_max_cluster_weight(
        C.c_uint32(g.n), C.c_uint32(g.m), g.xadj.ctypes.data_as(C.c_void_p), g.adjncy.ctypes.data_as(C.c_void_p),
        _opt(g.vwgt, np.int32), C.c_uint32(k), C.c_double(eps)))


def ref_max_block_weights(g, k, eps=0.03) -> np.ndarray:
    out = np.zeros(k, np.int32)
    ref().kmpref_max_block_weights(
        C.c_uint32(g.n), C.c_uint32(g.m), g.xadj.ctypes.data_as(C.c_void_p), g.adjncy.ctypes.data_as(C.c_void_p),
        _opt(g.vwgt, np.int32), C.c_uint32(k), C.c_double(eps), out.ctypes.data_as(C.c_void_p))
    return out


def ref_contract(g, clustering, algorithm=1):
    """The unmodified reference's contract_clustering (0 BUFFERED, 1 UNBUFFERED = default preset,
    2 UNBUFFERED_NAIVE). Returns the raw (non-canonical) result dict."""
    cl = np.ascontiguousarray(clustering, np.uint32)
    c_xadj = np.zeros(g.n + 1, np.uint32)
    c_adj = np.zeros(max(g.m, 1), np.uint32)
    c_vw = np.zeros(max(g.n, 1), np.int32)
    c_ew = np.zeros(max(g.m, 1), np.int32)
    mapping = np.zeros(max(g.n, 1), np.uint32)
    c_m = C.c_uint32(0)
    lib = ref()
    lib.kmpref_contract.restype = C.c_uint32
    c_n = int(lib.kmpref_contract(
        *_garrs(g), cl.ctypes.data_as(C.c_void_p), C.c_int(algorithm), c_xadj.ctypes.data_as(C.c_void_p),
        c_adj.ctypes.data_as(C.c_void_p), c_vw.ctypes.data_as(C.c_void_p), c_ew.ctypes.data_as(C.c_void_p),
        mapping.ctypes.data_as(C.c_void_p), C.byref(c_m)))
    return dict(c_n=c_n, c_xadj=c_xadj[: c_n + 1].copy(), c_adjncy=c_adj[: c_m.value].copy(), c_vwgt=c_vw[:c_n].copy(),
                c_adjwgt=c_ew[: c_m.value].copy(), mapping=mapping[: g.n].copy())


# ------------------------------------------------------------------------------------------------
# Oracle restatement (oracle/lp_oracle.cc)
# ------------------------------------------------------------------------------------------------
class OracleParams(C.Structure):
    _fields_ = LPParams._fields_ + [
        ("sync_subrounds", C.c_uint32),
        ("sync_granule_log2", C.c_uint32),
        ("sync_commit_passes", C.c_uint32),
    ]


class OracleStats(C.Structure):
    _fields_ = [
        ("iterations", C.c_uint32),
        ("moved", C.c_uint32 * 64),
        ("edges_scanned", C.c_uint64),
        ("nodes_visited", C.c_uint64),
        ("num_clusters", C.c_uint32),
        ("two_hop_ran", C.c_uint32),
    ]


SYNC_SUBROUNDS_DEFAULT = 8
SYNC_GRANULE_LOG2_DEFAULT = 4


def oracle_params(base: LPParams, subrounds=SYNC_SUBROUNDS_DEFAULT, granule_log2=SYNC_GRANULE_LOG2_DEFAULT,
                  commit_passes=1) -> OracleParams:
    p = OracleParams()
    for name, _ in LPParams._fields_:
        setattr(p, name, getattr(base, name))
    p.sync_subrounds, p.sync_granule_log2, p.sync_commit_passes = subrounds, granule_log2, commit_passes
    return p


_oracle = None


def build_oracle():
    import subprocess

    subprocess.check_call(["make", "-s", "-C", _HERE, "liblp_oracle.so"])


def oracle():
    global _oracle
    if _oracle is None:
        if not os.path.exists(ORACLE_LIB):
            build_oracle()
        lib = C.CDLL(ORACLE_LIB)
        lib.lpo_rearrange_by_degree_buckets.restype = C.c_uint32
        lib.lpo_edge_cut.restype = C.c_int64
        lib.lpo_max_cluster_weight.restype = C.c_int32
        lib.lpo_max_block_weight.restype = C.c_int32
        lib.lpo_max_cluster_weight.argtypes = [C.c_uint32, C.c_int64, C.c_uint32, C.c_double]
        lib.lpo_max_block_weight.argtypes = [C.c_int64, C.c_uint32, C.c_double]
        _oracle = lib
    return _oracle


def graph_buckets(g):
    """Bucket prefix array (34) + count, as the reference's CSRGraph ctor derives them."""
    if g.buckets is not None:
        b = np.ascontiguousarray(g.buckets, dtype=np.uint32)
        nb = 0
        for i in range(33, 0, -1):
            if b[i] != b[i - 1]:
                nb = i
                break
        return b, nb
    b = np.zeros(34, np.uint32)
    nb = C.c_uint32(0)
    oracle().lpo_degree_buckets(C.c_uint32(g.n), g.xadj.ctypes.data_as(C.c_void_p), C.c_int(1 if g.sorted else 0),
                                b.ctypes.data_as(C.c_void_p), C.byref(nb))
    return b, nb.value


def oracle_rearrange(g, remove_isolated=True):
    from kaminpar_b200.graph import CSRGraph

    xadj = np.zeros(g.n + 1, np.uint32)
    adj = np.zeros(g.m, np.uint32)
    vw = np.zeros(g.n, np.int32) if g.vwgt is not None else None
    ew = np.zeros(g.m, np.int32) if g.adjwgt is not None else None
    o2n = np.zeros(g.n, np.uint32)
    buckets = np.zeros(34, np.uint32)
    nb = C.c_uint32(0)
    n_lp = oracle().lpo_rearrange_by_degree_buckets(
        *_garrs(g), C.c_int(1 if remove_isolated else 0),
        xadj.ctypes.data_as(C.c_void_p), adj.ctypes.data_as(C.c_void_p), _opt(vw, np.int32), _opt(ew, np.int32),
        o2n.ctypes.data_as(C.c_void_p), buckets.ctypes.data_as(C.c_void_p), C.byref(nb),
    )
    out = CSRGraph(
        xadj=xadj[: n_lp + 1].copy(), adjncy=adj, vwgt=None if vw is None else vw[:n_lp].copy(), adjwgt=ew,
        sorted=True, buckets=buckets,
    )
    return out, o2n


SEQ, SYNC = 0, 1


def _sync_only(schedule, call_index):
    if call_index != 0 and schedule != SYNC:
        raise ValueError("call_index is a key of the sync schedule; seq replays earlier calls (num_calls)")


def oracle_lp_cluster(g, seed, max_cluster_weight, schedule=SEQ, desired=0, params=None, num_calls=1,
                      communities=None, return_stats=False, call_index=0):
    """call_index (sync): how many clusterings the device handle computed before this one, on any graph
    (DESIGN.md, "parity across levels and calls"); with num_calls > 1 the calls take call_index, call_index + 1, ..."""
    _sync_only(schedule, call_index)
    if not isinstance(params, OracleParams):
        params = oracle_params(params or default_cluster_params())
    b, nb = graph_buckets(g)
    out = np.zeros(g.n * num_calls, np.uint32)
    stats = (OracleStats * num_calls)()
    oracle().lpo_lp_cluster(
        C.c_int(schedule), *_garrs(g), b.ctypes.data_as(C.c_void_p), C.c_uint32(nb), C.c_int(seed),
        C.c_int32(max_cluster_weight), C.c_uint32(desired), _opt(communities, np.uint32), C.byref(params),
        C.c_int(num_calls), out.ctypes.data_as(C.c_void_p), stats, C.c_uint32(call_index),
    )
    res = out if num_calls == 1 else out.reshape(num_calls, g.n)
    return (res, stats) if return_stats else res


def oracle_lp_refine(g, seed, k, max_block_weights, partition, schedule=SEQ, params=None, min_block_weights=None,
                     communities=None, return_stats=False, call_index=0):
    """call_index (sync): the number of clusterings the device handle computed before this refinement (0 for a
    handle that only refines)."""
    _sync_only(schedule, call_index)
    if not isinstance(params, OracleParams):
        params = oracle_params(params or default_refine_params())
    b, nb = graph_buckets(g)
    part = np.ascontiguousarray(partition, dtype=np.uint32).copy()
    bw = np.zeros(k, np.int32)
    mbw = np.ascontiguousarray(max_block_weights, dtype=np.int32)
    stats = OracleStats()
    oracle().lpo_lp_refine(
        C.c_int(schedule), *_garrs(g), b.ctypes.data_as(C.c_void_p), C.c_uint32(nb), C.c_int(seed), C.c_uint32(k),
        mbw.ctypes.data_as(C.c_void_p), _opt(min_block_weights, np.int32), _opt(communities, np.uint32),
        C.byref(params), part.ctypes.data_as(C.c_void_p), bw.ctypes.data_as(C.c_void_p), C.byref(stats),
        C.c_uint32(call_index),
    )
    return (part, bw, stats) if return_stats else (part, bw)


def oracle_edge_cut(g, partition) -> int:
    part = np.ascontiguousarray(partition, dtype=np.uint32)
    return int(oracle().lpo_edge_cut(C.c_uint32(g.n), g.xadj.ctypes.data_as(C.c_void_p),
                                     g.adjncy.ctypes.data_as(C.c_void_p), _opt(g.adjwgt, np.int32),
                                     part.ctypes.data_as(C.c_void_p)))


def oracle_max_cluster_weight(g, k, eps=0.03) -> int:
    return int(oracle().lpo_max_cluster_weight(g.n, g.total_node_weight(), k, eps))


def oracle_max_block_weights(g, k, eps=0.03) -> np.ndarray:
    return np.full(k, oracle().lpo_max_block_weight(g.total_node_weight(), k, eps), np.int32)


def oracle_sync_select_all(mode, g, labels, weights, max_weights=None, max_cluster_weight=0, min_weights=None,
                           seed=0, call=0, iteration=0, params=None):
    """params (LPParams / OracleParams, optional): its max_num_neighbors and large_degree_threshold apply as in a
    full call -- a vertex of degree >= the threshold keeps its label and stores no favored cluster."""
    labels = np.ascontiguousarray(labels, np.uint32)
    weights = np.ascontiguousarray(weights, np.int32)
    tgt = np.zeros(g.n, np.uint32)
    fav = np.zeros(g.n, np.uint32)
    if params is not None and not isinstance(params, OracleParams):
        params = oracle_params(params)
    oracle().lpo_sync_select_all(
        C.c_int(mode), C.c_uint32(g.n), g.xadj.ctypes.data_as(C.c_void_p), g.adjncy.ctypes.data_as(C.c_void_p),
        _opt(g.vwgt, np.int32), _opt(g.adjwgt, np.int32), labels.ctypes.data_as(C.c_void_p),
        weights.ctypes.data_as(C.c_void_p), C.c_uint32(len(weights)), _opt(max_weights, np.int32),
        C.c_int32(max_cluster_weight), _opt(min_weights, np.int32), C.c_int(seed), C.c_uint32(call),
        C.c_uint32(iteration), tgt.ctypes.data_as(C.c_void_p), fav.ctypes.data_as(C.c_void_p),
        None if params is None else C.byref(params))
    return tgt, fav


def oracle_seq_select_all(mode, g, labels, weights, max_weights=None, max_cluster_weight=0, min_weights=None,
                          check_target=None, check_favored=None):
    """The reference-pinned `seq` selection code on frozen state (lpo_seq_select_all). Returns a dict with
    target, favored, num_ties, num_fav_ties, check_in_ties, check_fav_in_ties."""
    labels = np.ascontiguousarray(labels, np.uint32)
    weights = np.ascontiguousarray(weights, np.int32)
    tgt = np.zeros(g.n, np.uint32)
    fav = np.zeros(g.n, np.uint32)
    nt = np.zeros(g.n, np.uint32)
    nft = np.zeros(g.n, np.uint32)
    cin = np.ones(g.n, np.uint8)
    cfin = np.ones(g.n, np.uint8)
    oracle().lpo_seq_select_all(
        C.c_int(mode), C.c_uint32(g.n), g.xadj.ctypes.data_as(C.c_void_p), g.adjncy.ctypes.data_as(C.c_void_p),
        _opt(g.vwgt, np.int32), _opt(g.adjwgt, np.int32), labels.ctypes.data_as(C.c_void_p),
        weights.ctypes.data_as(C.c_void_p), C.c_uint32(len(weights)), _opt(max_weights, np.int32),
        C.c_int32(max_cluster_weight), _opt(min_weights, np.int32), _opt(check_target, np.uint32),
        _opt(check_favored, np.uint32), tgt.ctypes.data_as(C.c_void_p), fav.ctypes.data_as(C.c_void_p),
        nt.ctypes.data_as(C.c_void_p), nft.ctypes.data_as(C.c_void_p), cin.ctypes.data_as(C.c_void_p),
        cfin.ctypes.data_as(C.c_void_p))
    return dict(target=tgt, favored=fav, num_ties=nt, num_fav_ties=nft, check_in_ties=cin, check_fav_in_ties=cfin)
