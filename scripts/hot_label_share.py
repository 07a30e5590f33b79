"""Share of each team tier's adjacency entries whose target is among the last K vertex ids (CPU only).

The inputs the facade hands over, and those bench.py generates, are in degree-bucket order, so the last ids are the
highest-degree vertices. Every adjacency entry a sweep scans costs one gather of the target's label; this script
counts, per team tier (tiers 3-5 of lp_sweep.cuh, unit edge weights), which share of those gathers a copy of the
last K labels could serve. DESIGN §5 ("Tried and not kept: a label snapshot") quotes its output. It generates a
bench.py workload on the CPU, with the same generator and seed.

    python scripts/hot_label_share.py [--workload rmat22]

Prints one JSON line."""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

TIERS = {3: (32, 255), 4: (256, 1023), 5: (1024, 4095)}  # team tier -> degrees (unit edge weights)
KS = (1024, 2048, 4096, 8192)


def shares(xadj, adjncy):
    n = len(xadj) - 1
    deg = np.diff(xadj)
    tier = np.zeros(n, np.int8)
    for t, (lo, hi) in TIERS.items():
        tier[(deg >= lo) & (deg <= hi)] = t
    src_tier = np.repeat(tier, deg)  # tier of each adjacency entry's source vertex
    out = {}
    for t in TIERS:
        targets = adjncy[src_tier == t]
        out[f"tier{t}"] = {"vertices": int((tier == t).sum()), "edges": int(targets.size),
                           **{f"K{k}": float((targets >= n - k).mean()) if targets.size else None for k in KS}}
    out["all"] = {f"K{k}": float((adjncy >= n - k).mean()) for k in KS}
    return n, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="rmat22")
    args = ap.parse_args()
    import bench

    xadj, adjncy, _ = bench.generate(args.workload, "cpu")
    n, out = shares(xadj.numpy(), adjncy.numpy())
    print(json.dumps({"workload": args.workload, "n": n, "m_directed": int(adjncy.numel()), **out}))


if __name__ == "__main__":
    main()
