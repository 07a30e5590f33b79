"""The clusterer's hub tier on class-sorted chunks (-m gpu): the gather counting-sorts every 2048-edge chunk of a
hub's staged labels by hash class and records the class offsets, and each rate item reads only its own class's
range of every chunk. These graphs put hubs of K = 1 (edge weights), 2, 4, 16, 32 and 512 hash classes
(hub_classes in lp_sweep.cuh) next to one another, at degrees that are not multiples of the chunk size, with one hub
whose first chunk holds a single class and whose class 3 sits entirely in its last chunk. The clusterer must stay bit-exact
to the oracle's sync schedule: labels, moves per round and scan counters; forcing the split path
(KMP_HUB_SEL_LIMIT) must not change the visited vertices or scanned edges of any kernel tier."""
import functools

import numpy as np
import pytest

from kaminpar_b200 import lp
from kaminpar_b200.graph import CSRGraph, random_weights
from oracle import bindings as B
from tests import test_gpu_shards as S
from tests.test_hash_bijection import lowbias32

pytestmark = pytest.mark.gpu

UINT32_MAX = 0xFFFFFFFF
N = 1 << 19
# hub degrees: K = 2 (16384, the smallest unit-weight hub), 4, 4, 16 and 32 hash classes; 8192 is a hub of one
# class with edge weights (its labels are read in edge order, each with its edge's weight) and tier 6 without
HUB_DEGREES = (16384, 20001, 30000, 70001, 140001, 8192)
SKEWED = 1  # the hub whose chunks are arranged by class


def _classes(ids, k):
    return lowbias32(ids.astype(np.uint32)) & np.uint32(k - 1)


def csr(n, u, v):
    a, b = np.concatenate([u, v]), np.concatenate([v, u])
    key = np.unique(a * n + b)
    a, b = key // n, key % n
    xadj = np.zeros(n + 1, np.uint32)
    np.cumsum(np.bincount(a, minlength=n), out=xadj[1:])
    return CSRGraph(xadj, b.astype(np.uint32))


@functools.lru_cache(maxsize=None)
def giant_hub():
    """one hub of 2^21 + 4097 edges: 512 hash classes, more than the 256 a chunk is sorted by"""
    n = (1 << 21) + 8192
    rng = np.random.default_rng(12)
    d = (1 << 21) + 4097
    bg = rng.integers(1, n, size=(n, 2))
    bg = bg[bg[:, 0] != bg[:, 1]]
    return csr(n, np.concatenate([np.zeros(d, np.int64), bg[:, 0]]), np.concatenate([np.arange(1, d + 1), bg[:, 1]]))


@functools.lru_cache(maxsize=None)
def hub_graph(weighted=False):
    rng = np.random.default_rng(11)
    hubs = np.arange(len(HUB_DEGREES), dtype=np.int64)
    src, dst = [], []
    pool = np.arange(len(HUB_DEGREES), N, dtype=np.int64)
    for h, d in zip(hubs, HUB_DEGREES):
        if h == SKEWED:
            # K = 4, rows sorted by id: the first chunk holds class 0 only, and the last (partial) chunk holds
            # class 3 only, which no other chunk has
            cls = _classes(pool, 4)
            head = pool[cls == 0][:2048]
            c3 = pool[cls == 3][-(d % 2048):]
            mid = pool[(pool > head[-1]) & (pool < c3[0]) & (cls != 3)]
            nb = np.concatenate([head, rng.choice(mid, size=d - 2048 - len(c3), replace=False), c3])
        else:
            nb = rng.choice(pool, size=d, replace=False)
        src.append(np.full(d, h))
        dst.append(nb)
    # a sparse background: labels move between rounds, so the hubs see changing label multisets
    bg = rng.integers(len(HUB_DEGREES), N, size=(3 * N, 2))
    bg = bg[bg[:, 0] != bg[:, 1]]
    src.append(bg[:, 0])
    dst.append(bg[:, 1])
    g = csr(N, np.concatenate(src), np.concatenate(dst))
    if weighted:
        g = random_weights(g, 7, max_vwgt=3, max_adjwgt=5)
    return g


def skewed_layout_holds():
    g = hub_graph()
    row = g.adjncy[g.xadj[SKEWED]:g.xadj[SKEWED + 1]].astype(np.int64)
    cls = _classes(row, 4)
    d = len(row)
    last = (d - 1) // 2048 * 2048
    return (cls[:2048] == 0).all() and (cls[:last] != 3).all() and (cls[last:] == 3).any()


def cluster(g, seed, mnn=UINT32_MAX):
    """one clustering, bit-exact to the oracle; returns the scanned edges and visited vertices per kernel tier"""
    ctx = lp.create_default_context()
    ctx.engine.seed = seed
    ctx.partition.setup(g, 16, 0.03)
    ctx.coarsening.clustering.lp.max_num_neighbors = mnn
    mcw = lp.compute_max_cluster_weight(ctx.coarsening, ctx.partition, g.n, g.total_node_weight())
    c = lp.LPClustering(ctx.coarsening, ctx.engine)
    c.set_max_cluster_weight(mcw)
    labels = c.compute_clustering(g)
    p = B.default_cluster_params()
    p.max_num_neighbors = mnn
    want, st = B.oracle_lp_cluster(g, seed, mcw, schedule=B.SYNC, params=B.oracle_params(p), return_stats=True)
    gs = c.last_stats
    assert np.array_equal(labels, want)
    assert gs.moved_list() == list(st[0].moved[: st[0].iterations])
    assert gs.edges_scanned == st[0].edges_scanned and gs.nodes_visited == st[0].nodes_visited
    return list(gs.group_edges), list(gs.group_nodes)


def test_graph_has_the_hub_classes():
    g = hub_graph()
    deg = np.diff(g.xadj.astype(np.int64))[: len(HUB_DEGREES)]
    assert sorted(int(x) for x in deg % 2048) != [0] * len(HUB_DEGREES)
    k = [1 << int(np.ceil(np.log2(-(-int(d) // 8192)))) for d in deg]
    assert k == [2, 4, 4, 16, 32, 1], k
    assert skewed_layout_holds()


def test_hub_with_more_classes_than_a_chunk_is_sorted_by():
    """K = 512 > 256 sort classes: an item reads its sort class's ranges and filters by the next hash bit"""
    g = giant_hub()
    assert int(g.xadj[1]) == (1 << 21) + 4097
    cluster(g, 2)


@pytest.mark.parametrize("limit", ["0", "300", "2"])
@pytest.mark.parametrize("weighted", [False, True], ids=["unit", "weighted"])
def test_hub_classes_match_the_oracle(weighted, limit, monkeypatch):
    """Every hub class read from its sorted ranges (limit 0), and with the claim limit forcing splits by the next
    hash bits, re-read over the class's ranges and filtered: labels, moves and the per-tier scan counts hold."""
    g = hub_graph(weighted)
    base = cluster(g, 3)
    monkeypatch.setenv("KMP_HUB_SEL_LIMIT", limit)
    assert cluster(g, 3) == base


@pytest.mark.parametrize("mnn", [10000, 20000, 65537])
def test_hub_classes_below_max_num_neighbors(mnn):
    """max_num_neighbors below a hub's degree: the row is cut inside a chunk, the classes keep the full degree's
    count"""
    cluster(hub_graph(), 5, mnn)


@pytest.mark.parametrize("world", [2, 3])
def test_hub_classes_sharded(world, monkeypatch):
    """Emulated ranks take the hub entries i % world == rank, gather and rate them from the sorted chunks"""
    graphs = {"hub_classes": hub_graph(), "hub_classes_w": hub_graph(True)}
    monkeypatch.setattr(S, "graph", lambda name: graphs[name] if name in graphs else S.get_graph(name))
    for name in graphs:
        S.run_sharded(S.Case(name, 0, 1), world, "rotated")
