"""Stepping / sharded path on real GPUs: world = 1 always (pack -> unpack -> accumulate -> commit
through the stepping C ABI), world = 2 over NCCL when the box has two GPUs. Result must equal the
oracle's `sync` schedule bit for bit, i.e. be independent of the number of GPUs. Worlds of 2, 3 and 5
ranks emulated on one GPU: tests/test_gpu_shards.py."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu


def _run_rank(rank, world, port, out):
    import torch
    import torch.distributed as dist

    from kaminpar_b200 import lp
    from kaminpar_b200.dist import CudaBackend, ShardedLP
    from kaminpar_b200.graph import rmat
    from oracle import bindings as B

    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    if world > 1:
        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ["MASTER_PORT"] = str(port)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        g = B.oracle_rearrange(rmat(14, 16, 3))[0]
        ctx = lp.create_default_context()
        ctx.engine.seed = 6
        ctx.engine.device = rank
        ctx.partition.setup(g, 8, 0.03)
        mcw = lp.compute_max_cluster_weight(ctx.coarsening, ctx.partition, g.n, g.total_node_weight())
        h = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
        h.set_graph(g)
        drv = ShardedLP(CudaBackend(h, dev), g.n, 5, rank, world)
        c, moved, st = drv.compute_clustering(mcw)
        c2, moved_b, _ = drv.compute_clustering(mcw)  # second call: call counter advances
        k = 8
        part = (np.arange(g.n) % k).astype(np.uint32)
        h2 = lp.LPHandle(lp._refine_config(ctx.refinement.lp, ctx.engine))
        h2.set_graph(g)
        drv2 = ShardedLP(CudaBackend(h2, dev), g.n, 5, rank, world)
        p, bw, moved2, _ = drv2.refine(k, ctx.partition.max_block_weights(), part)
        np.savez(out + f".{rank}.npz", c=c, c2=c2, p=p, bw=bw, moved=np.array(moved), moved2=np.array(moved2),
                 edges=np.array([st.edges_scanned]))
    finally:
        if world > 1:
            dist.destroy_process_group()


def _run_rank_library(rank, world, port, out):
    """the same job through the library's own NCCL path: kmp_lp_dist_init, then plain cluster() / refine()"""
    import torch
    import torch.distributed as dist

    from kaminpar_b200 import lp
    from kaminpar_b200.graph import rmat
    from oracle import bindings as B

    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    if world > 1:
        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ["MASTER_PORT"] = str(port)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        g = B.oracle_rearrange(rmat(14, 16, 3))[0]
        ctx = lp.create_default_context()
        ctx.engine.seed = 6
        ctx.engine.device = rank
        ctx.partition.setup(g, 8, 0.03)
        mcw = lp.compute_max_cluster_weight(ctx.coarsening, ctx.partition, g.n, g.total_node_weight())
        h = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
        h.dist_init(rank, world)
        h.set_graph(g)
        c, st = h.cluster(mcw)
        c = c.copy()
        c2, _ = h.cluster(mcw)
        k = 8
        part = (np.arange(g.n) % k).astype(np.uint32)
        h2 = lp.LPHandle(lp._refine_config(ctx.refinement.lp, ctx.engine))
        h2.dist_init(rank, world)
        h2.set_graph(g)
        p, bw, st2 = h2.refine(k, ctx.partition.max_block_weights(), part.copy())
        # every rank reports the whole job's counters: divide so that _check's sum over ranks is the total
        np.savez(out + f".{rank}.npz", c=c, c2=c2, p=p, bw=bw, moved=np.array(st.moved_list()),
                 moved2=np.array(st2.moved_list()), edges=np.array([st.edges_scanned // world]),
                 edges_rem=np.array([st.edges_scanned % world]))
    finally:
        if world > 1:
            dist.destroy_process_group()


def _check(world, out):
    from kaminpar_b200 import lp
    from kaminpar_b200.graph import rmat
    from oracle import bindings as B

    g = B.oracle_rearrange(rmat(14, 16, 3))[0]
    ctx = lp.create_default_context()
    ctx.partition.setup(g, 8, 0.03)
    mcw = lp.compute_max_cluster_weight(ctx.coarsening, ctx.partition, g.n, g.total_node_weight())
    expect, st = B.oracle_lp_cluster(g, 6, mcw, schedule=B.SYNC, num_calls=2, return_stats=True)
    k = 8
    part = (np.arange(g.n) % k).astype(np.uint32)
    rp = B.oracle_params(B.default_refine_params(), commit_passes=4)
    ep, ebw, st2 = B.oracle_lp_refine(g, 6, k, ctx.partition.max_block_weights(), part, schedule=B.SYNC, params=rp,
                                      return_stats=True)
    total_edges = 0
    for rank in range(world):
        d = np.load(out + f".{rank}.npz")
        assert np.array_equal(d["c"], expect[0]) and np.array_equal(d["c2"], expect[1])
        assert np.array_equal(d["p"], ep) and np.array_equal(d["bw"], ebw)
        assert list(d["moved"]) == list(st[0].moved[: st[0].iterations])
        assert list(d["moved2"]) == list(st2.moved[: st2.iterations])
        total_edges += int(d["edges"][0]) + (int(d["edges_rem"][0]) if "edges_rem" in d and rank == 0 else 0)
    assert total_edges == st[0].edges_scanned  # the frontier is partitioned, nothing scanned twice


def test_stepping_api_single_gpu(tmp_path):
    out = str(tmp_path / "r")
    _run_rank(0, 1, 0, out)
    _check(1, out)


def test_sharded_two_gpus_nccl(tmp_path):
    import torch
    import torch.multiprocessing as mp

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = str(tmp_path / "r")
    mp.spawn(_run_rank, args=(2, 29731, out), nprocs=2, join=True)
    _check(2, out)


def test_library_dist_path_world1(tmp_path):
    out = str(tmp_path / "r")
    _run_rank_library(0, 1, 0, out)
    _check(1, out)


def test_library_nccl_two_gpus(tmp_path):
    """kmp_lp_dist_init + kmp_lp_cluster / kmp_lp_refine: ncclAllGather inside the library, results identical to 1 GPU"""
    import torch
    import torch.multiprocessing as mp

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = str(tmp_path / "r")
    mp.spawn(_run_rank_library, args=(2, 29741, out), nprocs=2, join=True)
    _check(2, out)
