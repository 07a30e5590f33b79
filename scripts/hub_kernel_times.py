"""Device time of the hub-tier kernels (sweep_hub_*) per clustering step, one line per kernel, measured with
torch.profiler (CUDA activity) around the same resident clustering call bench.py times.

    python scripts/hub_kernel_times.py [--workload rmat22 rmat24] [--steps 3] [--warmup 2]

Prints one JSON line per workload: total device ms per step of every hub kernel (template arguments folded),
their sum, and the number of launches per step."""
from __future__ import annotations

import argparse
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def short_name(name):
    m = re.search(r"(sweep_hub_[a-z]+)", name)
    return m.group(1) if m else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", nargs="+", default=["rmat22", "rmat24"])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench
    from kaminpar_b200 import lp

    dev = torch.device("cuda", 0)
    for wl in args.workload:
        xadj64, adj64, k = bench.generate(wl, dev)
        n, m = xadj64.numel() - 1, adj64.numel()
        d_xadj, d_adj = xadj64.to(torch.int32), adj64.to(torch.int32)
        del xadj64, adj64
        torch.cuda.synchronize()
        ctx = lp.create_default_context()
        handle = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
        handle.set_graph_device(n, m, d_xadj.data_ptr(), d_adj.data_ptr())
        handle.set_timing(False)
        mcw = bench_mcw(ctx, n, k, lp)
        for _ in range(args.warmup):
            handle.cluster(mcw, fetch=False)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                handle.cluster(mcw, fetch=False)
            torch.cuda.synchronize()
        per = {}
        calls = {}
        for ev in prof.events():
            if ev.device_type != torch.autograd.DeviceType.CUDA:
                continue
            s = short_name(ev.name)
            if s is None:
                continue
            per[s] = per.get(s, 0.0) + ev.device_time / 1000.0
            calls[s] = calls.get(s, 0) + 1
        out = {"workload": wl, "n": n, "m": m, "gpu": torch.cuda.get_device_name(0),
               "hub_ms_per_step": {k_: round(v / args.steps, 4) for k_, v in sorted(per.items())},
               "hub_total_ms_per_step": round(sum(per.values()) / args.steps, 4),
               "launches_per_step": {k_: v // args.steps for k_, v in sorted(calls.items())}}
        print(json.dumps(out), flush=True)
        del handle, d_xadj, d_adj
        torch.cuda.empty_cache()


def bench_mcw(ctx, n, k, lp):
    """bench.py's max cluster weight: partition context of an unweighted n-vertex graph, epsilon 0.03."""
    import numpy as np

    from kaminpar_b200.graph import CSRGraph
    g = CSRGraph.__new__(CSRGraph)
    g.xadj = np.zeros(n + 1, dtype=np.uint32)
    g.adjncy = np.zeros(0, dtype=np.uint32)
    g.vwgt = None
    g.adjwgt = None
    g.sorted = True
    g.buckets = None
    ctx.partition.setup(g, k, 0.03)
    return lp.compute_max_cluster_weight(ctx.coarsening, ctx.partition, n, n)


if __name__ == "__main__":
    main()
