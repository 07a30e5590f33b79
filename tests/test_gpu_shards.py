"""The sharded path at world 2, 3 and 5, emulated on one GPU (-m gpu): W handles on device 0, each the shard
(r, W) of the stepping API, all on torch's current stream, so the launch order is the program order. The
all-gather is made by copying tensors and the favored MAX all-reduce by a tensor maximum; no second process, no
NCCL. The round loop is ShardedLP._iterations (kaminpar_b200/dist.py) written out, with checks between its steps.

Per sub-round every rank sweeps its slice into its own send buffer, followed by a guard tail of `size` words
holding a sentinel. Before anything is committed the host checks that no rank reports more proposals than
kmp_lp_subround_cap allows, that no rank wrote past its buffer and that the ranks together propose at most `size`
moves. Each rank then commits the gathered buffers in rank order, reversed, or starting with its own (rotated):
the commit is order-free (DESIGN.md §3), so all three give the oracle's `sync` result.

Every case checks, bit for bit: the moves per round (equal on every rank), every rank's labels (and block weights),
the scan counters summed over the ranks (the frontier is partitioned: nothing scanned twice or skipped) and the
visited vertices per kernel tier summed over the ranks (== the world-1 run's, and every tier the input has ran).

What this cannot reach is the library's own NCCL path (kmp_lp_dist_init: sweeps that write straight into the
NCCL send buffer, ncclAllGather, the favored ncclAllReduce); the sweep and commit kernels are the same, reached
through k_pack_movers here. tests/test_gpu_dist.py runs that path where a box has two GPUs.
"""
import ctypes as C
import functools
import os
from dataclasses import dataclass

import numpy as np
import pytest

from kaminpar_b200 import lp
from kaminpar_b200.graph import CSRGraph, rmat
from oracle import bindings as B
from tests import helpers as H
from tests.test_gpu_edges import ladder
from tests.test_gpu_parity import get_graph

pytestmark = pytest.mark.gpu

UINT32_MAX = 0xFFFFFFFF
SENTINEL = 0x5A5A5A5A  # guard words after each send buffer (no vertex id or count of these graphs)
ORDERS = ("rank", "reversed", "rotated")
WORLDS = (2, 3, 5)
GRAPHS = ["rmat16_hubs", "rmat15_hubs_w", "star_hub", "star30000", "grid20", "walshaw_unsorted", "path", "complete",
          "bipartite", "with_isolated", "dense_w", "wide_unit"]
CLUSTER_SEEDS = (0, 5)
REFINE_SEED = 5
REFINE_KS = (2, 64, 600)  # 600 * 16 level-histogram entries exceed commit_refine_fused's shared-memory limit
# smallest world from which a sub-round of the graph has 0 < size < world, i.e. ranks with an empty slice of a
# non-empty list (or no hub of a one-hub list), at the default schedule and the seeds above
EMPTY_SLICES_FROM = {"dense_w": 2, "star_hub": 2, "star30000": 2, "bipartite": 3, "wide_unit": 3}


@functools.lru_cache(maxsize=None)
def graph(name):
    if name in ("dense_w", "wide_unit"):  # degree ladders: a few centres per tier, few hubs
        return ladder(name)
    if name == "rmat16":  # vertices of every kernel tier
        return B.oracle_rearrange(rmat(16, 16, 3))[0]
    return get_graph(name)


def gather_order(order, world, rank):
    """the ranks whose proposal buffers `rank` receives, in the order it receives them"""
    if order == "rank":
        return list(range(world))
    if order == "reversed":
        return list(range(world - 1, -1, -1))
    return [(rank + i) % world for i in range(world)]


@dataclass(frozen=True)
class Case:
    """One call sequence on one set of handles, and everything the oracle needs to replay it."""
    graph: str
    mode: int                     # 0 clustering, 1 refinement
    seed: int
    k: int = 8                    # blocks (refinement); the clustering's weight limit is sized for k = 8
    calls: int = 1                # clusterings on the same handles (call indices 0, 1, ...)
    mnn: int = UINT32_MAX         # max_num_neighbors
    thr: int = UINT32_MAX         # large_degree_threshold
    subrounds: int = 8
    two_hop: int = 2              # the clusterer's post passes (two_hop_strategy, isolated_nodes_strategy)
    isolated: int = 3
    start: str = "random"         # refinement start: random blocks, or "min": contiguous blocks, min block weights
    communities: bool = False


def engine_ctx(case):
    g = graph(case.graph)
    ctx = lp.create_default_context()
    ctx.engine.seed = case.seed
    ctx.engine.sync_subrounds = case.subrounds
    ctx.partition.setup(g, case.k, 0.03)
    c = ctx.coarsening.clustering.lp if case.mode == 0 else ctx.refinement.lp
    c.max_num_neighbors, c.large_degree_threshold = case.mnn, case.thr
    if case.mode == 0:
        c.two_hop_strategy, c.isolated_nodes_strategy = case.two_hop, case.isolated
    return ctx


def config(case):
    ctx = engine_ctx(case)
    if case.mode == 0:
        return lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine)
    return lp._refine_config(ctx.refinement.lp, ctx.engine)


def oracle_params(case):
    p = B.default_cluster_params() if case.mode == 0 else B.default_refine_params()
    p.max_num_neighbors, p.large_degree_threshold = case.mnn, case.thr
    if case.mode == 0:
        p.two_hop_strategy, p.isolated_nodes_strategy = case.two_hop, case.isolated
    return B.oracle_params(p, case.subrounds, commit_passes=1 if case.mode == 0 else 4)


def inputs(case):
    """(max cluster weight, communities) of a clustering; (k, max / min block weights, start, communities) of a
    refinement"""
    g = graph(case.graph)
    ctx = engine_ctx(case)
    comm = (np.arange(g.n) % 3).astype(np.uint32) if case.communities else None
    if case.mode == 0:
        mcw = lp.compute_max_cluster_weight(ctx.coarsening, ctx.partition, g.n, g.total_node_weight())
        return mcw, comm
    k = case.k
    min_bw = None
    if case.start == "min":  # test_t1_refinement_min_block_weights_and_unbalanced_start
        part = (np.arange(g.n) * k // g.n).astype(np.uint32)
        min_bw = np.array([int(0.97 * w) for w in H.block_weights(g, part, k)], np.int32)
    else:
        part = np.random.default_rng(k + case.seed).integers(0, k, g.n).astype(np.uint32)
    return k, ctx.partition.max_block_weights(), min_bw, part, comm


@functools.lru_cache(maxsize=None)
def expected(case):
    """[(labels, block weights or None, oracle stats)] per call of the case"""
    g = graph(case.graph)
    if case.mode == 0:
        mcw, comm = inputs(case)
        labels, st = B.oracle_lp_cluster(g, case.seed, mcw, schedule=B.SYNC, params=oracle_params(case),
                                         num_calls=case.calls, communities=comm, return_stats=True)
        labels = labels.reshape(case.calls, g.n)
        return [(labels[c], None, st[c]) for c in range(case.calls)]
    k, mbw, min_bw, part, comm = inputs(case)
    p, bw, st = B.oracle_lp_refine(g, case.seed, k, mbw, part, schedule=B.SYNC, params=oracle_params(case),
                                   min_block_weights=min_bw, communities=comm, return_stats=True)
    return [(p, bw, st)]


# ------------------------------------------------------------------------------------------------
# The lockstep harness
# ------------------------------------------------------------------------------------------------
@dataclass
class Result:
    labels: list       # per rank
    block_weights: list
    stats: list        # per rank: this rank's share of the scan counters
    moved: list        # per round, equal on every rank


class Shards:
    """`world` ranks of one sharded run: one handle each on device 0, all on torch's current stream."""

    def __init__(self, g, cfg, world, order):
        import torch

        from kaminpar_b200.dist import CudaBackend

        self.torch = torch
        self.dev = torch.device("cuda", 0)
        self.n, self.world, self.order = g.n, world, order
        self.num_iterations = cfg.num_iterations
        self.handles, self.ranks = [], []
        for r in range(world):
            h = lp.LPHandle(cfg)
            self.handles.append(h)
            h.set_graph(g)
            b = CudaBackend(h, self.dev)
            b.set_shard(r, world)
            self.ranks.append(b)
        self.small_subrounds = 0  # sub-rounds with 0 < size < world

    def close(self):
        for h in self.handles:
            h.close()

    def subround(self, it, sg):
        torch = self.torch
        caps = {b.subround_cap(sg) for b in self.ranks}
        assert len(caps) == 1, (it, sg, caps)
        cap, size = caps.pop()
        if size == 0:
            return
        self.small_subrounds += size < self.world
        words = 4 + 2 * cap
        send = torch.full((self.world, words + size), SENTINEL, dtype=torch.int32, device=self.dev)
        for r, b in enumerate(self.ranks):
            b.sweep(it, sg, send[r])
        host = send.cpu().numpy().view(np.uint32)  # waits for the sweeps
        counts = host[:, 0].astype(np.int64)
        assert (counts <= cap).all(), ("proposals over the cap", it, sg, counts.tolist(), cap)
        assert (host[:, words:] == SENTINEL).all(), ("a rank wrote past its send buffer", it, sg)
        assert counts.sum() <= size, ("more proposals than listed vertices", it, sg, counts.tolist(), size)
        for r, b in enumerate(self.ranks):
            b.commit(it, sg, torch.cat([send[q, :words] for q in gather_order(self.order, self.world, r)]))

    def rounds(self):
        """ShardedLP._iterations: the moves per round"""
        nsub = {b.num_subrounds() for b in self.ranks}
        assert len(nsub) == 1, nsub
        nsub = nsub.pop()
        moved_per_round = []
        max_it = self.num_iterations if self.num_iterations > 0 else (1 << 62)
        it = 0
        while it < max_it:
            for b in self.ranks:
                b.begin_iteration()
            for sg in range(nsub):
                self.subround(it, sg)
            moved = [b.end_iteration() for b in self.ranks]
            assert len(set(moved)) == 1, ("ranks disagree on the moves", it, moved)
            moved_per_round.append(moved[0])
            it += 1
            if moved[0] == 0:
                break
        return moved_per_round

    def finish(self, moved, k=None):
        out = [b.finish(self.n, k=k) for b in self.ranks]
        return Result([o[0] for o in out], [o[1] for o in out], [o[2] for o in out], moved)

    def cluster(self, mcw, communities=None):
        torch = self.torch
        for b in self.ranks:
            b.begin_cluster(mcw, communities)
        moved = self.rounds()
        if self.world > 1:
            bufs = torch.empty((self.world, self.n), dtype=torch.int32, device=self.dev)
            for r, b in enumerate(self.ranks):
                b.favored_export(bufs[r])
            top = (bufs.to(torch.int64) & UINT32_MAX).max(dim=0).values  # ncclMax over ncclUint32
            fav = torch.where(top >= 1 << 31, top - (1 << 32), top).to(torch.int32)
            for b in self.ranks:
                b.favored_import(fav)
        return self.finish(moved)

    def refine(self, k, mbw, part, min_bw=None, communities=None):
        for b in self.ranks:
            b.begin_refine(k, mbw, min_bw, communities, part)
        return self.finish(self.rounds(), k)


def assert_same(got, want, what):
    if not np.array_equal(got, want):
        bad = np.nonzero(np.asarray(got) != np.asarray(want))[0]
        raise AssertionError(f"{what}: {bad.size} entries differ, first at {bad[:8].tolist()}: "
                             f"{np.asarray(got)[bad[:8]].tolist()} != {np.asarray(want)[bad[:8]].tolist()}")


def check(res, want, world, call):
    labels, bw, st = want
    for r in range(world):
        assert_same(res.labels[r], labels, f"call {call}, labels of rank {r}")
        if bw is not None:
            assert_same(res.block_weights[r], bw, f"call {call}, block weights of rank {r}")
    assert res.moved == list(st.moved[: st.iterations]), (call, res.moved, list(st.moved[: st.iterations]))
    assert sum(s.edges_scanned for s in res.stats) == st.edges_scanned, call
    assert sum(s.nodes_visited for s in res.stats) == st.nodes_visited, call
    if bw is None:
        assert all(s.num_clusters == st.num_clusters and s.two_hop_ran == st.two_hop_ran for s in res.stats), call


def run(case, world, order):
    """The case on `world` emulated ranks, checked against the oracle. Returns the visited vertices per kernel
    tier of every call (summed over the ranks) and the number of sub-rounds with 0 < size < world."""
    g = graph(case.graph)
    sh = Shards(g, config(case), world, order)
    try:
        results = []
        if case.mode == 0:
            mcw, comm = inputs(case)
            for _ in range(case.calls):
                results.append(sh.cluster(mcw, comm))
        else:
            k, mbw, min_bw, part, comm = inputs(case)
            results.append(sh.refine(k, mbw, part, min_bw, comm))
    finally:
        sh.close()
    tiers = []
    for call, (res, want) in enumerate(zip(results, expected(case))):
        check(res, want, world, call)
        tiers.append([sum(s.group_nodes[t] for s in res.stats) for t in range(len(res.stats[0].group_nodes))])
    return tiers, sh.small_subrounds


@functools.lru_cache(maxsize=None)
def world1_tiers(case):
    tiers, _ = run(case, 1, "rank")
    for t in tiers:  # every kernel tier of the input ran
        assert [i for i, x in enumerate(t) if x > 0] == H.tiers_present(graph(case.graph), case.thr), t
    return tiers


def run_sharded(case, world, order):
    """run() at `world` ranks, and at one rank for the per-tier counts it must reproduce"""
    tiers, small = run(case, world, order)
    assert tiers == world1_tiers(case), (tiers, world1_tiers(case))
    return small


# ------------------------------------------------------------------------------------------------
# Clustering and refinement over graphs x worlds
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", WORLDS, ids=[f"W{w}" for w in WORLDS])
@pytest.mark.parametrize("name", GRAPHS)
def test_sharded_clustering(name, world):
    """Two clusterings on the same handles (call indices 0 and 1) per seed; the seeds take different gather
    orders."""
    small = 0
    for i, seed in enumerate(CLUSTER_SEEDS):
        small += run_sharded(Case(name, 0, seed, calls=2), world, ORDERS[(i + world) % 3])
    if world >= EMPTY_SLICES_FROM.get(name, UINT32_MAX):
        assert small > 0


def test_sharded_clustering_rmat16_world2():
    """R-MAT 16 (every kernel tier) at seed 2 on two ranks, the input of the first emulated test of the sharded
    path"""
    run_sharded(Case("rmat16", 0, 2, calls=2), 2, "rank")


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("name", GRAPHS)
def test_sharded_refinement(name, world):
    """k = 2, 64 and 600 blocks, each in another gather order: with 600 blocks the commit's level histograms are
    global, not per CTA."""
    small = 0
    for i, k in enumerate(REFINE_KS):
        small += run_sharded(Case(name, 1, REFINE_SEED, k=k), world, ORDERS[(i + world) % 3])
    if world >= EMPTY_SLICES_FROM.get(name, UINT32_MAX):
        assert small > 0


def test_sharded_refinement_k20000():
    """k = 20000: neither the level histograms nor the block-weight deltas of the commit are per CTA"""
    run_sharded(Case("rmat16_hubs", 1, REFINE_SEED, k=20000), 3, "rotated")


@pytest.mark.parametrize("name,world", [("walshaw_unsorted", 2), ("walshaw_unsorted", 5), ("rmat15_hubs_w", 3)])
def test_sharded_refinement_min_block_weights(name, world):
    """An unbalanced start (contiguous blocks) with minimum block weights 3 % below the start's"""
    run_sharded(Case(name, 1, 4, k=8, start="min"), world, "rotated")


@pytest.mark.parametrize("name,world", [("rmat15_hubs_w", 3), ("walshaw_unsorted", 5)])
def test_sharded_communities(name, world):
    run_sharded(Case(name, 0, 9, communities=True), world, "rotated")
    run_sharded(Case(name, 1, 9, k=16, communities=True), world, "reversed")


@pytest.mark.parametrize("world", WORLDS)
def test_sharded_handles_cluster_twice_then_refine(world):
    """One set of handles: two clusterings (call indices 0, 1), then a refinement hashed with call index 2. The
    handles are clusterer handles, so the refinement commits in one pass."""
    name, seed, k = "rmat15_hubs_w", 7, 16
    g = graph(name)
    case = Case(name, 0, seed)
    cfg = config(case)
    mcw, _ = inputs(case)
    params = B.oracle_params(B.default_cluster_params(), commit_passes=1)
    want_c, st_c = B.oracle_lp_cluster(g, seed, mcw, schedule=B.SYNC, params=params, num_calls=2, return_stats=True)
    ctx = engine_ctx(Case(name, 1, seed, k=k))
    mbw = ctx.partition.max_block_weights()
    part = np.random.default_rng(1).integers(0, k, g.n).astype(np.uint32)
    want_r = B.oracle_lp_refine(g, seed, k, mbw, part, schedule=B.SYNC, params=params, return_stats=True,
                                call_index=2)
    sh = Shards(g, cfg, world, "reversed")
    try:
        for call in range(2):
            check(sh.cluster(mcw), (want_c[call], None, st_c[call]), world, call)
        check(sh.refine(k, mbw, part), want_r, world, 2)
    finally:
        sh.close()


def test_sharded_clustering_of_an_empty_graph_counts_as_a_call():
    """A stepping clustering of an empty graph is a completed clustering, as in kmp_lp_cluster: the next one, on
    the same handles and another graph, hashes with call index 1 (DESIGN.md, "parity across levels and calls")."""
    name, seed, world = "rmat16_hubs", 6, 3
    g = graph(name)
    case = Case(name, 0, seed)
    mcw, _ = inputs(case)
    want, st = B.oracle_lp_cluster(g, seed, mcw, schedule=B.SYNC, params=oracle_params(case), return_stats=True,
                                   call_index=1)
    sh = Shards(H.empty_graph(0), config(case), world, "rotated")
    try:
        for b in sh.ranks:  # no vertices: no sub-round to sweep and no favored entry to exchange
            b.begin_cluster(mcw, None)
        res = sh.finish(sh.rounds())
        assert all(len(labels) == 0 for labels in res.labels)
        for h in sh.handles:
            h.set_graph(g)
        sh.n = g.n
        check(sh.cluster(mcw), (want, None, st[0]), world, 1)
    finally:
        sh.close()


# ------------------------------------------------------------------------------------------------
# Knobs at world 3 (each read once, when a handle is created)
# ------------------------------------------------------------------------------------------------
KNOBS = {
    "p64": ({"KMP_FORCE_P64": "1"}, {}),
    "grid1": ({"KMP_GRID_CAP": "1"}, {}),
    "grid3": ({"KMP_GRID_CAP": "3"}, {}),
    "push": ({"KMP_ACTIVATION": "push"}, {}),
    "pull": ({"KMP_ACTIVATION": "pull"}, {}),
    # the refiner's hub entries through the overflow list, its hub selection in several passes
    "hub_overflow": ({"KMP_HUB_BUCKET_CAP": "8", "KMP_HUB_SEL_LIMIT": "0"}, {}),
    # a capped neighbourhood scan turns pull activation off; hubs above the threshold are not visited
    "neighbour_limits": ({}, {"mnn": 6, "thr": 300}),
    "S31": ({}, {"subrounds": 31}),  # more and smaller lists
}


@pytest.mark.parametrize("knob", list(KNOBS))
@pytest.mark.parametrize("name", ["rmat16_hubs", "rmat15_hubs_w"])
def test_sharded_knobs(name, knob, monkeypatch):
    env, fields = KNOBS[knob]
    for key, value in env.items():
        monkeypatch.setenv(key, value)
    run_sharded(Case(name, 0, 3, calls=2, **fields), 3, "rotated")
    run_sharded(Case(name, 1, 3, k=64, **fields), 3, "rotated")


# ------------------------------------------------------------------------------------------------
# Post passes after the favored MAX exchange
# ------------------------------------------------------------------------------------------------
POST_PASSES = [(4, 3), (4, 4), (2, 2), (4, 2), (2, 1)]  # (two_hop_strategy, isolated_nodes_strategy)


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("name", ["star30000", "star_hub", "with_isolated"])
def test_sharded_post_pass_variants(name, world):
    for i, (ths, iso) in enumerate(POST_PASSES):
        run_sharded(Case(name, 0, 13, two_hop=ths, isolated=iso), world, ORDERS[i % 3])


# ------------------------------------------------------------------------------------------------
# Refusals of the sharding entry points, each followed by a valid call that matches the oracle
# ------------------------------------------------------------------------------------------------
def refused(code, call):
    with pytest.raises(RuntimeError, match=f"error {code}:"):
        lp._check(call())


def test_shard_and_step_refusals():
    import torch

    lib = lp.load_library()
    dev = torch.device("cuda", 0)
    case = Case("grid20", 0, 3)
    g = graph(case.graph)
    mcw, _ = inputs(case)
    buf = torch.zeros(4 * g.n + 64, dtype=torch.int32, device=dev)
    p = C.c_void_p(buf.data_ptr())
    moved = C.c_uint32(0)

    sh = Shards(g, config(case), 1, "rank")
    h = sh.handles[0]._h
    try:
        for rank, world in ((0, 0), (2, 2), (5, 3)):
            refused(-1, lambda: lib.kmp_lp_set_shard(h, C.c_uint32(rank), C.c_uint32(world)))
        # the stepping calls before any step_begin_*
        refused(-1, lambda: lib.kmp_lp_step_begin_iteration(h))
        refused(-1, lambda: lib.kmp_lp_step_sweep(h, C.c_uint32(0), C.c_uint32(0), p))
        refused(-1, lambda: lib.kmp_lp_step_commit(h, C.c_uint32(0), C.c_uint32(0), p))
        refused(-1, lambda: lib.kmp_lp_step_end_iteration(h, C.byref(moved)))
        refused(-1, lambda: lib.kmp_lp_step_favored_export(h, p))
        refused(-1, lambda: lib.kmp_lp_step_favored_import(h, p))
        refused(-1, lambda: lib.kmp_lp_step_finish(h, None, None, None))
        # a sharded sync handle without a communicator
        sh.ranks[0].set_shard(1, 2)
        refused(-1, lambda: lib.kmp_lp_cluster(h, C.c_int32(mcw), C.c_uint32(0), None, None, None))
        part = (np.arange(g.n) % 8).astype(np.uint32)
        mbw = engine_ctx(Case("grid20", 1, 3)).partition.max_block_weights()
        refused(-1, lambda: lib.kmp_lp_refine(h, C.c_uint32(8), lp._ptr(mbw), None, None, lp._ptr(part), None, None))
        # valid: world 1 again, through the library and then the stepping API (call indices 0 and 1)
        sh.ranks[0].set_shard(0, 1)
        c, _ = sh.handles[0].cluster(mcw)
        want = expected(Case("grid20", 0, 3, calls=2))
        assert_same(c, want[0][0], "clustering after the refusals")
        res = sh.cluster(mcw)
        check(res, want[1], 1, 1)
        # after step_finish the run is over
        refused(-1, lambda: lib.kmp_lp_step_sweep(h, C.c_uint32(0), C.c_uint32(0), p))
        refused(-1, lambda: lib.kmp_lp_step_favored_export(h, p))
    finally:
        sh.close()

    # a refinement: sub-rounds out of range, favored export / import; then the same run continues
    rcase = Case("grid20", 1, 3, k=8)
    k, mbw, _, part, _ = inputs(rcase)
    sh = Shards(g, config(rcase), 1, "rank")
    h = sh.handles[0]._h
    try:
        b = sh.ranks[0]
        b.begin_refine(k, mbw, None, None, part)
        nsub = b.num_subrounds()
        assert nsub == 4 * 8
        cap, size = C.c_uint32(0), C.c_uint32(0)
        refused(-1, lambda: lib.kmp_lp_subround_cap(h, C.c_uint32(nsub), C.byref(cap), C.byref(size)))
        refused(-1, lambda: lib.kmp_lp_step_sweep(h, C.c_uint32(0), C.c_uint32(nsub), p))
        refused(-1, lambda: lib.kmp_lp_step_commit(h, C.c_uint32(0), C.c_uint32(nsub), p))
        refused(-1, lambda: lib.kmp_lp_step_favored_export(h, p))
        refused(-1, lambda: lib.kmp_lp_step_favored_import(h, p))
        check(sh.finish(sh.rounds(), k), expected(rcase)[0], 1, 0)
    finally:
        sh.close()


def test_stepping_refusals_by_configuration():
    """seq_strict handles cannot step; a clusterer asking for more than one commit pass is refused as
    kmp_lp_cluster refuses it. Each is followed by a valid call: the seq_strict clustering of BASELINE config 1
    equals the unmodified reference's (tests/golden/ref_rgg2d_k4.npz)."""
    lib = lp.load_library()
    gold = np.load(os.path.join(H.GOLDEN, "ref_rgg2d_k4.npz"))
    gs = CSRGraph(gold["xadj"], gold["adjncy"], sorted=True)
    ctx = lp.create_default_context()
    ctx.engine.schedule = "seq_strict"
    part = gold["part_in_s0"].astype(np.uint32)
    mbw = B.oracle_max_block_weights(gs, 4)
    mcw = int(gold["max_cluster_weight"][0])
    h = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
    try:
        h.set_graph(gs)
        refused(-4, lambda: lib.kmp_lp_step_begin_cluster(h._h, C.c_int32(mcw), None))
        refused(-4, lambda: lib.kmp_lp_step_begin_refine(h._h, C.c_uint32(4), lp._ptr(mbw), None, None,
                                                          lp._ptr(part)))
        c, _ = h.cluster(mcw)
        assert_same(c, gold["clustering_s0"], "seq_strict clustering after the refusals")
    finally:
        h.close()

    case = Case("grid20", 0, 3)
    mcw, _ = inputs(case)
    cfg = config(case)
    cfg.sync_commit_passes = 4
    h = lp.LPHandle(cfg)
    try:
        h.set_graph(graph(case.graph))
        refused(-4, lambda: lib.kmp_lp_step_begin_cluster(h._h, C.c_int32(mcw), None))
    finally:
        h.close()
    run_sharded(case, 2, "rank")
