"""Overload and underload balancers on the device: call time and effect on the two refinement workloads of bench.py.

Overload input: bench.py's refinement partition (hash-of-id blocks, seed 0) with a seeded 10 % of the vertices moved
into block 0, max block weights (1 + 0.03) * ceil(n / k). Underload input: the same partition with a seeded 10 % of
block 0's vertices moved to hashed other blocks (block 0 underloaded, no block overloaded), minimum block weights
ceil((1 - 0.03) * perfectly balanced weight). Per workload and balancer: the device time of kmp_overload_balance /
kmp_underload_balance (CUDA events, after warm-up; median and range over repeated calls, each on a fresh upload of
the same input), rounds, candidates, overload or underload and cut before / after, and the host cost of the
operator's refine on an input that needs nothing (no device work). The card's name and power limit are read in the
same run.

    python scripts/bench_balance.py [--reps 7] [--warmup 2] [--which both|overload|underload] [--out DIR]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = ("rmat22", "grid256")  # k = 16 and k = 64 (bench.py WORKLOADS)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], check=True,
                             capture_output=True, text=True).stdout.strip().splitlines()[0]
        name, power = (x.strip() for x in out.split(","))
        return name, power
    except Exception as e:  # the numbers are still reported, without the card
        return f"unknown ({e})", "unknown"


def workload(name):
    import torch

    import bench
    from kaminpar_b200.graph import CSRGraph

    dev = torch.device("cuda:0")
    xadj64, adj64, k = bench.generate(name, dev)
    d_xadj, d_adj = xadj64.to(torch.int32), adj64.to(torch.int32)
    g = CSRGraph.__new__(CSRGraph)
    g.xadj = d_xadj.cpu().numpy().view(np.uint32)
    g.adjncy = d_adj.cpu().numpy().view(np.uint32)
    g.vwgt = g.adjwgt = None
    g.sorted = True
    g.buckets = None
    return g, d_xadj, d_adj, k


def run(name, reps, warmup):
    import torch

    from kaminpar_b200 import lp

    g, d_xadj, d_adj, k = workload(name)
    n, m = g.n, g.m
    ctx = lp.create_default_context()
    ctx.partition.setup(g, k, 0.03)
    mbw, pbw = ctx.partition.max_block_weights(), ctx.partition.perfectly_balanced_block_weights()
    part0 = np.random.default_rng(0).integers(0, k, n).astype(np.uint32)  # bench.py's refinement partition
    part = part0.copy()
    part[np.random.default_rng(1).random(n) < 0.10] = 0

    h = lp.LPHandle(lp._refine_config(ctx.refinement.lp, ctx.engine))
    h.set_graph_device(n, m, d_xadj.data_ptr(), d_adj.data_ptr())
    h.upload_partition(part)
    cut_before = h.edge_cut()
    times, host_ms, stats = [], [], None
    for i in range(warmup + reps):
        h.upload_partition(part)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        improved, bw, st = h.overload_balance(k, mbw, pbw, None)
        t1 = time.perf_counter()
        if i >= warmup:
            times.append(st.device_ms)
            host_ms.append(1e3 * (t1 - t0))
            stats = st
    cut_after = h.edge_cut()
    out = h.download_labels()
    over_after = int(np.maximum(np.bincount(out, minlength=k) - mbw, 0).sum())

    # the feasible no-op through the operator: host check of the block weights, no upload, no launch
    bal = lp.OverloadBalancer(ctx)
    pg = lp.PartitionedGraph(g, k, part0)
    assert int(np.maximum(pg.block_weights() - mbw, 0).sum()) == 0
    noop = []
    for _ in range(20):
        t0 = time.perf_counter()
        assert not bal.refine(pg, ctx.partition)
        noop.append(1e6 * (time.perf_counter() - t0))
    h.close()
    return dict(
        workload=name, n=n, m=m, k=k,
        device_ms_median=float(np.median(times)), device_ms_min=float(min(times)), device_ms_max=float(max(times)),
        host_ms_median=float(np.median(host_ms)), reps=reps, warmup=warmup,
        rounds=stats.rounds, moved=stats.moved_list(), candidates=int(stats.candidates),
        edges_scanned=int(stats.edges_scanned), kernel_launches=int(stats.kernel_launches),
        overload_before=int(stats.overload_before), overload_after=int(stats.overload_after),
        overload_after_recomputed=over_after, improved=bool(improved), cut_before=int(cut_before),
        cut_after=int(cut_after), noop_us_median=float(np.median(noop)),
        reference_balancer="not measured",
    )


def run_underload(name, reps, warmup, min_eps=0.03):
    import torch

    from kaminpar_b200 import lp

    g, d_xadj, d_adj, k = workload(name)
    n, m = g.n, g.m
    ctx = lp.create_default_context()
    ctx.partition.setup(g, k, 0.03)
    pbw = ctx.partition.perfectly_balanced_block_weights()
    ctx.partition.setup_min_block_weights([math.ceil((1 - min_eps) * int(w)) for w in pbw])
    mbw, mnw = ctx.partition.max_block_weights(), ctx.partition.min_block_weights()
    part0 = np.random.default_rng(0).integers(0, k, n).astype(np.uint32)  # bench.py's refinement partition
    part = part0.copy()
    rng = np.random.default_rng(1)
    pick = np.flatnonzero((part == 0) & (rng.random(n) < 0.10))
    h32 = (pick.astype(np.uint64) * 0x9E3779B1) & 0xFFFFFFFF  # hashed other block
    part[pick] = (1 + (h32 ^ (h32 >> 16)) % (k - 1)).astype(np.uint32)
    W = np.bincount(part, minlength=k)
    assert W[0] < mnw[0] and np.all(W <= mbw)

    h = lp.LPHandle(lp._refine_config(ctx.refinement.lp, ctx.engine))
    h.set_graph_device(n, m, d_xadj.data_ptr(), d_adj.data_ptr())
    h.upload_partition(part)
    cut_before = h.edge_cut()
    times, host_ms, stats = [], [], None
    for i in range(warmup + reps):
        h.upload_partition(part)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        improved, bw, st = h.underload_balance(k, mbw, mnw, None)
        t1 = time.perf_counter()
        if i >= warmup:
            times.append(st.device_ms)
            host_ms.append(1e3 * (t1 - t0))
            stats = st
    cut_after = h.edge_cut()
    out = h.download_labels()
    W1 = np.bincount(out, minlength=k)

    # the no-op through the operator on a min-balanced partition: host check of the block weights, no launch
    bal = lp.UnderloadBalancer(ctx)
    pg = lp.PartitionedGraph(g, k, part0)
    assert np.all(pg.block_weights() >= mnw)
    noop = []
    for _ in range(20):
        t0 = time.perf_counter()
        assert not bal.refine(pg, ctx.partition)
        noop.append(1e6 * (time.perf_counter() - t0))
    h.close()
    return dict(
        workload=name, n=n, m=m, k=k, min_epsilon=min_eps,
        device_ms_median=float(np.median(times)), device_ms_min=float(min(times)), device_ms_max=float(max(times)),
        host_ms_median=float(np.median(host_ms)), reps=reps, warmup=warmup,
        rounds=stats.rounds, moved=stats.moved_list(), candidates=int(stats.candidates),
        edges_scanned=int(stats.edges_scanned), kernel_launches=int(stats.kernel_launches),
        underload_before=int(stats.underload_before), underload_after=int(stats.underload_after),
        underload_after_recomputed=int(np.maximum(mnw - W1, 0).sum()),
        overload_after_recomputed=int(np.maximum(W1 - mbw, 0).sum()), improved=bool(improved),
        cut_before=int(cut_before), cut_after=int(cut_after), noop_us_median=float(np.median(noop)),
        reference_balancer="not measured",
    )


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--which", choices=("both", "overload", "underload"), default="both")
    ap.add_argument("--out", default=None, help="directory for bench_balance.json")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_balance.py needs a CUDA device")
    name, power = card()
    res = dict(card=name, power_limit=power)
    if args.which in ("both", "overload"):
        res["results"] = [run(w, args.reps, args.warmup) for w in WORKLOADS]
    if args.which in ("both", "underload"):
        res["underload"] = [run_underload(w, args.reps, args.warmup) for w in WORKLOADS]
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_balance.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
