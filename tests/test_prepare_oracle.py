"""CPU: the preparation oracle (tests/prepare_oracle.py, DESIGN.md §15) against the UNMODIFIED reference.

* The rearrangement equals the live reference's graph::rearrange_by_degree_buckets + remove_isolated_nodes
  (oracle/_ref/libkaminpar_ref.so; skipped where it is not built) and every committed golden the reference computed on
  its own rearrangement of a raw input.
* Next fit and the map back are pinned end to end through the reference's whole KaMinPar::compute_partition
  (oracle/_ref/libkaminpar_ref_full.so, one thread): from the reference's output vector, take the blocks of the
  non-isolated vertices, apply the oracle's finish with the same max block weights, and get the whole vector back.
"""
import ctypes as C
import os

import numpy as np
import pytest

from kaminpar_b200.graph import CSRGraph, grid3d, random_weights, rmat, road_like
from oracle import bindings as B
from tests import helpers as H
from tests import prepare_oracle as P

FULL_LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref",
                        "libkaminpar_ref_full.so")


def star(n: int) -> CSRGraph:  # tests/golden/make_golden.py
    xadj = np.zeros(n + 1, np.int64)
    xadj[1] = n - 1
    xadj[2:] = n - 1 + np.arange(1, n)
    adj = np.concatenate([np.arange(1, n), np.zeros(n - 1, np.int64)])
    return CSRGraph(xadj.astype(np.uint32), adj.astype(np.uint32))


# the raw input of every golden the reference computed on its own rearrangement (tests/golden/make_golden.py)
GOLDEN_INPUTS = {
    "rgg2d_k4": lambda: H.load_graph("rgg2d"),
    "rgg2d_k2": lambda: H.load_graph("rgg2d"),
    "rgg16_w": lambda: H.load_graph("rgg16_vwgt_adjwgt"),
    "walshaw_k16": lambda: H.load_graph("walshaw_data"),
    "walshaw_geometric": lambda: H.load_graph("walshaw_data"),
    "walshaw_3calls": lambda: H.load_graph("walshaw_data"),
    "grid12": lambda: grid3d(12),
    "rmat14": lambda: rmat(14, 16, 1),
    "road60": lambda: road_like(60, 2, 0.3, 0.5),
    "star30000": lambda: star(30000),
}


def sorted_golden_cases():
    return [c for c in H.golden_cases() if bool(np.load(os.path.join(H.GOLDEN, f"ref_{c}.npz"))["sorted"][0])]


def hubs(degrees, isolated_every=0) -> CSRGraph:
    """A simple symmetric graph with one hub per entry of `degrees`: hub i is joined to the leaves 0 .. d_i - 1 of a
    shared leaf pool, so the leaves' degrees vary too. Optionally an isolated vertex after every few hubs."""
    hub_ids, nxt = [], 0
    for i in range(len(degrees)):
        hub_ids.append(nxt)
        nxt += 1
        if isolated_every and (i + 1) % isolated_every == 0:
            nxt += 1  # an isolated vertex
    leaves = max(degrees)
    edges = [(h, nxt + j) for h, d in zip(hub_ids, degrees) for j in range(d)]
    n = nxt + leaves
    src = np.array([u for u, v in edges] + [v for u, v in edges], np.int64)
    dst = np.array([v for u, v in edges] + [u for u, v in edges], np.int64)
    order = np.lexsort((dst, src))
    xadj = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(src, minlength=n), out=xadj[1:])
    return CSRGraph(xadj.astype(np.uint32), dst[order].astype(np.uint32))


def raw_with_degrees(degrees, seed=0) -> CSRGraph:
    """Any CSR the device accepts: not symmetric, with self-loops and parallel edges (the reference's own graph
    validation refuses these, so they are checked against the oracle's properties only)."""
    rng = np.random.default_rng(seed)
    deg = np.asarray(degrees, np.int64)
    n = len(deg)
    xadj = np.zeros(n + 1, np.int64)
    np.cumsum(deg, out=xadj[1:])
    adj = rng.integers(0, max(n, 1), int(xadj[-1]))
    src = np.repeat(np.arange(n), deg)
    adj[::7] = src[::7]  # self-loops
    return CSRGraph(xadj.astype(np.uint32), adj.astype(np.uint32))


def raw_cases():
    yield "raw_selfloops", raw_with_degrees([5, 0, 1, 2, 0, 9, 3, 0, 70000, 0])
    yield "n1_selfloop", CSRGraph(np.array([0, 1], np.uint32), np.array([0], np.uint32))


def edge_cases():
    ladder = []
    for j in range(1, 17):
        ladder += [2**j - 1, 2**j, 2**j + 1]
    yield "ladder_to_2^16+1", hubs(ladder, isolated_every=5)
    yield "hub_above_2^16", hubs([70000, 3, 1, 2, 65535, 65536, 1], isolated_every=2)
    yield "n0", H.empty_graph(0)
    yield "n1", H.empty_graph(1)
    yield "all_isolated", H.empty_graph(37)
    g = rmat(10, 4, seed=9)
    rng = np.random.default_rng(3)
    perm = rng.permutation(g.n + 300)  # 300 isolated vertices spread through the id range
    deg = np.zeros(g.n + 300, np.int64)
    deg[perm[: g.n]] = np.diff(g.xadj.astype(np.int64))
    xadj = np.zeros(g.n + 301, np.int64)
    np.cumsum(deg, out=xadj[1:])
    adj = np.empty(g.m, np.int64)
    for u in range(g.n):
        adj[xadj[perm[u]]:xadj[perm[u] + 1]] = perm[g.adjncy[g.xadj[u]:g.xadj[u + 1]]]
    yield "isolated_spread", random_weights(CSRGraph(xadj.astype(np.uint32), adj.astype(np.uint32)), 4, 7, 9)


def live_inputs():
    for name in ("rgg2d", "rgg16", "rgg16_vwgt_adjwgt", "walshaw_data"):
        yield name, H.load_graph(name)
    for name in ("grid12", "rmat14", "road60", "star30000"):
        yield name, GOLDEN_INPUTS[name]()
    yield "rmat12_w", random_weights(rmat(12, 8, seed=4), 11, max_vwgt=9, max_adjwgt=13)
    yield from edge_cases()


def _check_against(prep, ref_graph, ref_o2n, n):
    n_prime = prep["n_prime"]
    assert n_prime == ref_graph.n and prep["num_isolated"] == n - n_prime
    assert np.array_equal(prep["xadj"][: n_prime + 1], ref_graph.xadj)
    assert np.all(prep["xadj"][n_prime:] == prep["xadj"][n])  # the isolated tail adds no edges
    assert np.array_equal(prep["adjncy"], ref_graph.adjncy)
    assert np.array_equal(prep["old_to_new"], ref_o2n)
    if ref_graph.vwgt is None:
        assert prep["vwgt"] is None
    else:
        assert np.array_equal(prep["vwgt"][:n_prime], ref_graph.vwgt)
    if ref_graph.adjwgt is None:
        assert prep["adjwgt"] is None
    else:
        assert np.array_equal(prep["adjwgt"], ref_graph.adjwgt)


@pytest.mark.parametrize("name,g", list(live_inputs()), ids=lambda x: x if isinstance(x, str) else "")
def test_oracle_equals_live_reference(name, g):
    if not B.have_reference():
        pytest.skip("oracle/_ref/libkaminpar_ref.so not built (needs the reference sources)")
    ref_graph, ref_o2n = B.ref_rearrange(g)
    prep = P.rearrange(g.xadj, g.adjncy, g.vwgt, g.adjwgt)
    _check_against(prep, ref_graph, ref_o2n, g.n)
    if g.vwgt is not None:  # the isolated vertices keep their weights, in new-id order
        assert np.array_equal(prep["vwgt"][prep["old_to_new"]], g.vwgt)


@pytest.mark.parametrize("case", sorted_golden_cases())
def test_oracle_equals_reference_goldens(case):
    g0 = GOLDEN_INPUTS[case]()
    gold, d = H.load_case(case)
    prep = P.rearrange(g0.xadj, g0.adjncy, g0.vwgt, g0.adjwgt)
    _check_against(prep, gold, d["old_to_new"], g0.n)


def test_oracle_edge_case_properties():
    for name, g in list(edge_cases()) + list(raw_cases()):
        prep = P.rearrange(g.xadj, g.adjncy, g.vwgt, g.adjwgt)
        b = P.buckets(g.xadj)
        o2n, n2o = prep["old_to_new"], prep["new_to_old"]
        assert np.array_equal(o2n[n2o], np.arange(g.n)), name
        nb = b[n2o]
        assert np.all(np.diff(nb) >= 0), name  # sorted by bucket ...
        assert np.all(np.diff(n2o.astype(np.int64))[np.diff(nb) == 0] > 0), name  # ... stably
        assert prep["num_isolated"] == int((b == 32).sum()), name
        for u in range(min(g.n, 200)):
            old = n2o[u]
            lst = g.adjncy[g.xadj[old]:g.xadj[old + 1]]
            assert np.array_equal(prep["adjncy"][prep["xadj"][u]:prep["xadj"][u + 1]], o2n[lst[::-1]]), name
    assert list(P.buckets(np.array([0, 0, 1, 3, 6, 10, 10 + 2**16]))) == [32, 1, 2, 2, 3, 17]


# ---- finish: next fit + map back, pinned through the reference's whole compute_partition -------------------------
def _with_isolated(g: CSRGraph, extra: int, seed: int, vw_iso=None) -> CSRGraph:
    """g plus `extra` isolated vertices, all ids shuffled (isolated vertices spread through the range)."""
    n = g.n + extra
    rng = np.random.default_rng(seed)
    perm = rng.permutation(n)
    deg = np.zeros(n, np.int64)
    deg[perm[: g.n]] = np.diff(g.xadj.astype(np.int64))
    xadj = np.zeros(n + 1, np.int64)
    np.cumsum(deg, out=xadj[1:])
    adj = np.empty(g.m, np.int64)
    ew = None if g.adjwgt is None else np.empty(g.m, np.int32)
    for u in range(g.n):
        s, e = g.xadj[u], g.xadj[u + 1]
        adj[xadj[perm[u]]:xadj[perm[u] + 1]] = perm[g.adjncy[s:e]]
        if ew is not None:
            ew[xadj[perm[u]]:xadj[perm[u] + 1]] = g.adjwgt[s:e]
    vw = None
    if g.vwgt is not None or vw_iso is not None:
        vw = np.ones(n, np.int32)
        if g.vwgt is not None:
            vw[perm[: g.n]] = g.vwgt
        if vw_iso is not None:
            vw[perm[g.n:]] = vw_iso(rng, extra)
    return CSRGraph(xadj.astype(np.uint32), adj.astype(np.uint32), vw, ew)


def finish_inputs():
    base = H.load_graph("walshaw_data")
    yield "walshaw+400", _with_isolated(base, 400, 1), 16
    yield "walshaw+3000", _with_isolated(base, 3000, 2), 8  # isolated weight spans several blocks
    yield "rgg16w+40_heavy", _with_isolated(H.load_graph("rgg16_vwgt_adjwgt"), 40, 3,
                                            lambda r, c: r.integers(5, 40, c)), 4
    path = H.path_graph(60)
    # heavy isolated vertices: next fit leaves room in every block it passes, so b advances again and again and the
    # last block takes what is left
    yield "path60+50_heavy", _with_isolated(path, 50, 4, lambda r, c: r.integers(20, 60, c)), 8
    yield "grid+600_w", _with_isolated(random_weights(grid3d(8), 5, max_vwgt=4, max_adjwgt=3), 600, 5,
                                       lambda r, c: r.integers(0, 6, c)), 6


@pytest.fixture(scope="module")
def full_ref():
    if not os.path.exists(FULL_LIB):
        pytest.skip("oracle/_ref/libkaminpar_ref_full.so not built (needs the reference sources)")
    lib = C.CDLL(FULL_LIB)
    lib.kmpfull_compute_partition.restype = C.c_longlong
    return lib


def _arr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


@pytest.mark.parametrize("name,g,k", list(finish_inputs()), ids=lambda x: x if isinstance(x, str) else "")
def test_finish_equals_reference_compute_partition(full_ref, name, g, k):
    out = np.zeros(g.n, np.uint32)
    full_ref.kmpfull_compute_partition(C.c_uint32(g.n), _arr(g.xadj), _arr(g.adjncy), _arr(g.vwgt), _arr(g.adjwgt),
                                       C.c_uint32(k), C.c_double(0.03), C.c_int(0), C.c_int(1), _arr(out))
    prep = P.rearrange(g.xadj, g.adjncy, g.vwgt, g.adjwgt)
    assert prep["num_isolated"] > 0
    mbw = B.ref_max_block_weights(g, k, 0.03)  # set up on the FULL graph, as compute_partition does
    part = out[prep["new_to_old"][: prep["n_prime"]]]
    got, bw = P.finish(prep, k, mbw, part)
    assert np.array_equal(got, out)
    w = np.ones(g.n, np.int64) if g.vwgt is None else g.vwgt.astype(np.int64)
    assert np.array_equal(bw, np.bincount(out, weights=w, minlength=k).astype(np.int64))
    iso_blocks = out[prep["new_to_old"][prep["n_prime"]:]]
    if name.endswith("_heavy"):  # the chain passed more than one block and ended in the last
        assert len(np.unique(iso_blocks)) > 2 and iso_blocks[-1] == k - 1
