"""Overlay cluster coarsening on the device (DESIGN.md §14) on the first coarsening level of bench.py's graphs.

Per workload and repetition, on one handle with bench.py's clusterer configuration:
  basic    one LP clustering (kmp_lp_cluster), then kmp_contract_clustering from the device labels
  overlay  kmp_lp_cluster_overlay with num_levels = 1 (two LP clusterings intersected), then the same contraction
Reported: the device time (CUDA events; median and range over the repetitions after warm-up) of one LP call, of the
overlay tree (one pairwise overlay at L = 1, including its one host wait), of the contraction after each, and the
coarse vertex counts c_n of basic and overlay. The card's name and power limit are read in the same run.

    python scripts/bench_overlay.py [--reps 5] [--warmup 1] [--workloads rmat22,rmat24,grid256] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], check=True,
                             capture_output=True, text=True).stdout.strip().splitlines()[0]
        name, power = (x.strip() for x in out.split(","))
        return name, power
    except Exception as e:  # the numbers are still reported, without the card
        return f"unknown ({e})", "unknown"


def summary(xs):
    return dict(median=float(np.median(xs)), min=float(min(xs)), max=float(max(xs)))


def run(name, reps, warmup):
    import torch

    import bench
    from kaminpar_b200 import contraction as KC
    from kaminpar_b200 import lp
    from kaminpar_b200.graph import CSRGraph

    dev = torch.device("cuda:0")
    xadj64, adj64, k = bench.generate(name, dev)
    d_xadj, d_adj = xadj64.to(torch.int32).contiguous(), adj64.to(torch.int32).contiguous()
    n, m = d_xadj.numel() - 1, d_adj.numel()
    g = CSRGraph.__new__(CSRGraph)  # the partition context reads n and the node weights only
    g.xadj = d_xadj.cpu().numpy().view(np.uint32)
    g.adjncy = np.zeros(0, np.uint32)
    g.vwgt = g.adjwgt = None
    g.sorted, g.buckets = True, None
    ctx = lp.create_default_context()
    ctx.partition.setup(g, k, 0.03)
    mcw = lp.compute_max_cluster_weight(ctx.coarsening, ctx.partition, n, n)  # as bench.py's clustering line
    h = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
    h.set_graph_device(n, m, d_xadj.data_ptr(), d_adj.data_ptr())
    t = {key: [] for key in ("lp_ms", "overlay_lp_ms_per_call", "overlay_ms", "contract_basic_ms",
                             "contract_overlay_ms", "c_n_basic", "c_n_overlay")}
    row = None
    for it in range(warmup + reps):
        _, ls = h.cluster(mcw, fetch=False)
        cg = KC.contract_on_handle(h, None)
        basic = (ls.device_ms, cg.stats.device_ms, cg.n)
        cg.close()
        _, os_ = h.cluster_overlay(1, mcw, fetch=False)
        cg = KC.contract_on_handle(h, None)
        over = (os_.lp_device_ms / os_.num_clusterings, os_.overlay_device_ms, cg.stats.device_ms, cg.n)
        cg.close()
        if it >= warmup:
            t["lp_ms"].append(basic[0])
            t["contract_basic_ms"].append(basic[1])
            t["c_n_basic"].append(basic[2])
            t["overlay_lp_ms_per_call"].append(over[0])
            t["overlay_ms"].append(over[1])
            t["contract_overlay_ms"].append(over[2])
            t["c_n_overlay"].append(over[3])
        row = dict(workload=name, n=n, m=m, sort_bits=os_.sort_bits, overlay_kernel_launches=os_.kernel_launches)
    row.update({key: summary(v) for key, v in t.items()})
    h.close()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--workloads", default="rmat22,rmat24,grid256")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    name, power = card()
    rows = [run(w, args.reps, args.warmup) for w in args.workloads.split(",")]
    res = dict(card=name, power_limit=power, rows=rows)
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_overlay.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
