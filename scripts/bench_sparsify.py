"""Threshold edge sparsification on the device (DESIGN.md §13) on the first coarsening level of bench.py's graphs.

Per workload: LP clustering on the device (bench.py's clusterer configuration), kmp_contract_clustering, then
kmp_coarse_sparsify. Reported: c_n, c_m before and after, the target of the reference's default factors
(density 0.5, edge 0.5) and whether its laziness factor 4 triggers sparsification, and the device time (CUDA events,
median and range over repeated calls after warm-up) of kmp_coarse_sparsify next to kmp_contract_clustering. Every
repetition contracts afresh and sparsifies to the default target (also when the laziness rule would skip it, so that
the time is measured on every graph). The card's name and power limit are read in the same run.

    python scripts/bench_sparsify.py [--reps 5] [--warmup 1] [--workloads rmat22,rmat24,grid256] [--out DIR]
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


def run(name, reps, warmup):
    import torch

    import bench
    from kaminpar_b200 import contraction as KC
    from kaminpar_b200 import lp

    dev = torch.device("cuda:0")
    xadj64, adj64, k = bench.generate(name, dev)
    d_xadj, d_adj = xadj64.to(torch.int32).contiguous(), adj64.to(torch.int32).contiguous()
    n, m = d_xadj.numel() - 1, d_adj.numel()
    from kaminpar_b200.graph import CSRGraph

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
    h.cluster(mcw, fetch=False)
    s_ctx = KC.SparsificationClusterCoarseningContext()
    contract_ms, sparsify_ms, row = [], [], None
    for it in range(warmup + reps):
        cg = KC.contract_on_handle(h, None)
        target = KC.sparsification_target(m, n, cg.n, s_ctx.density_target_factor, s_ctx.edge_target_factor)
        c_m = cg.m
        triggers = float(c_m) > s_ctx.laziness_factor * target
        st = cg.sparsify(h, min(target, c_m), 0x5EED + it)
        if it >= warmup:
            contract_ms.append(cg.stats.device_ms)
            sparsify_ms.append(st.device_ms)
        row = dict(workload=name, n=n, m=m, c_n=cg.n, c_m_before=c_m, target=target, c_m_after=st.c_m_after,
                   default_laziness_triggers=bool(triggers), threshold=st.threshold, smaller=st.smaller,
                   equal=st.equal, equal_kept=st.equal_kept)
        cg.close()
    row.update(contract_ms=dict(median=float(np.median(contract_ms)), min=min(contract_ms), max=max(contract_ms)),
               sparsify_ms=dict(median=float(np.median(sparsify_ms)), min=min(sparsify_ms), max=max(sparsify_ms)))
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
        with open(os.path.join(args.out, "bench_sparsify.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
