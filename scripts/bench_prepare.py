"""Input preparation on the device (DESIGN.md §15) on bench.py's graphs BEFORE their degree-bucket rearrangement.

Per workload, in one run, with the card's name and power limit read in the same run:
  prepare    kmp_prepare_graph_device on the raw graph in device memory (stats.device_ms: CUDA events around the
             whole call, its two host waits included); median and range over the repetitions after warm-up
  finish     kmp_prepared_finish at k = 64 from a host partition of the n' vertices (host clock around the call: it
             ends in a device synchronise and includes the n'-entry upload and the n-entry download)
  torch      graph.rearrange_by_degree_buckets_torch (what bench.py runs) on the same device, unit weights only
             (CUDA-synchronised host clock)
  bytes      the modelled traffic of the preparation: 12 B per edge (adjncy read, old_to_new gather, new adjncy
             write), 8 B more per edge with edge weights, 40 B per vertex (two xadj passes, old_to_new / new_to_old /
             degree writes, the degree scan, the edge pass's per-vertex lookups), 8 B more with vertex weights; over
             the prepare time, against the HBM peak bench.py uses (MEASURED_PEAKS.json, else the data sheet)
Correctness at the timed sizes: on every unit-weight workload the device's n', xadj, adjncy and old_to_new are compared
with the torch helper's; where they differ, the row counts the vertices the helper's floating-point log2 puts into
another bucket than the reference's integer rule, and checks the device's order against a stable sort by that rule. Where oracle/_ref/libkaminpar_ref.so exists, the reference's own host rearrangement (serial oneTBB
stand-in, one thread) of R-MAT 20 is timed once and reported on a separate line.

    python scripts/bench_prepare.py [--reps 5] [--warmup 1] [--workloads rmat22,...] [--out DIR]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEFAULT = "rmat22,rmat24,rgg24,road,grid512,rmat22_w"


def raw_graph(name, device):
    """bench.generate's graph before its rearrangement: torch int32 (xadj, adjncy[, vwgt, adjwgt]) on `device`."""
    import torch

    import bench
    from kaminpar_b200 import graph as G

    weighted = name.endswith("_w")
    kind, args, _ = bench.WORKLOADS[name[:-2] if weighted else name]
    if kind == "rmat":
        n = 1 << args["scale"]
        src, dst = G.rmat_edges_torch(args["scale"], args["edge_factor"], args["seed"], device)
        xadj, adj = G._csr_from_pairs_torch(n, src, dst, device)
    elif kind == "grid":
        xadj, adj = G.grid3d_torch(args["nx"], device)
    elif kind == "rgg":
        g = G.rgg2d(args["n"], args["seed"], device=device)
        xadj, adj = torch.from_numpy(g.xadj.astype(np.int64)), torch.from_numpy(g.adjncy.astype(np.int64))
    else:
        g = G.road_like(args["side"], args["seed"], args["delete_frac"], args["subdivide_frac"], device=device)
        xadj, adj = torch.from_numpy(g.xadj.astype(np.int64)), torch.from_numpy(g.adjncy.astype(np.int64))
    xadj, adj = xadj.to(device), adj.to(device)
    vw = ew = None
    if weighted:  # symmetric edge weights 1 + (u + v) % 9, vertex weights 1 + u % 5
        n = xadj.numel() - 1
        src = torch.repeat_interleave(torch.arange(n, device=device), xadj[1:] - xadj[:-1])
        ew = (1 + (src + adj) % 9).to(torch.int32)
        vw = (1 + torch.arange(n, device=device) % 5).to(torch.int32)
        del src
    return xadj, adj, vw, ew


def exact_buckets(xadj):
    """floor(log2 d) + 1 in integer arithmetic (d >= 1), 32 for d = 0: the reference's degree_bucket."""
    import torch

    deg = xadj[1:] - xadj[:-1]
    b = torch.zeros_like(deg)
    for j in range(32):
        b += (deg >= (1 << j)).to(deg.dtype)
    return torch.where(deg > 0, b, torch.full_like(b, 32))


def float_buckets(xadj):
    """The bucket rearrange_by_degree_buckets_torch computes (floating-point log2, isolated -> 40)."""
    import torch

    deg = xadj[1:] - xadj[:-1]
    bucket = torch.where(deg > 0, torch.floor(torch.log2(deg.clamp(min=1).double())).long() + 1,
                         torch.full_like(deg, 40))
    return torch.where((deg > 0) & ((1 << (bucket - 1).clamp(min=0, max=62)) > deg), bucket - 1, bucket)


def summary(xs):
    return dict(median=float(np.median(xs)), min=float(min(xs)), max=float(max(xs)))


def run(name, reps, warmup, peak):
    import torch

    from kaminpar_b200 import lp
    from kaminpar_b200 import prepare as PR
    from kaminpar_b200.graph import rearrange_by_degree_buckets_torch

    dev = torch.device("cuda:0")
    xadj64, adj64, vw, ew = raw_graph(name, dev)
    d_xadj, d_adj = xadj64.to(torch.int32).contiguous(), adj64.to(torch.int32).contiguous()
    n, m = d_xadj.numel() - 1, d_adj.numel()
    torch.cuda.synchronize()
    ctx = lp.create_default_context()
    h = lp.LPHandle(lp._refine_config(ctx.refinement.lp, ctx.engine))
    ptr = lambda t: 0 if t is None else t.data_ptr()
    k = 64
    prep_ms, fin_ms, torch_ms = [], [], []
    pg = None
    for it in range(warmup + reps):
        if pg is not None:
            pg.close()
        pg = PR.rearrange_by_degree_buckets_device(h, n, m, ptr(d_xadj), ptr(d_adj), ptr(vw), ptr(ew))
        part = (np.arange(pg.n, dtype=np.int64) * k // max(pg.n, 1)).astype(np.uint32)
        total = int(vw.sum().item()) if vw is not None else n
        mbw = np.full(k, int(1.03 * -(-total // k)), np.int32)
        t0 = time.perf_counter()
        pg.finish(h, k, mbw, part)
        t1 = time.perf_counter()
        if it >= warmup:
            prep_ms.append(pg.stats.device_ms)
            fin_ms.append((t1 - t0) * 1e3)
    row = dict(workload=name, n=n, m=m, n_nonisolated=pg.n, num_isolated=pg.num_isolated,
               weighted=vw is not None, kernel_launches=pg.stats.kernel_launches,
               prepare_ms=summary(prep_ms), finish_k64_ms=summary(fin_ms))
    bytes_ = m * (12 + (8 if ew is not None else 0)) + n * (40 + (8 if vw is not None else 0))
    row["modelled_bytes"] = bytes_
    row["prepare_gbs"] = bytes_ / (row["prepare_ms"]["median"] * 1e-3) / 1e9
    row["share_of_hbm_peak"] = row["prepare_gbs"] / peak
    if vw is None:
        for it in range(warmup + reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            t_xadj, t_adj, t_o2n = rearrange_by_degree_buckets_torch(xadj64, adj64, remove_isolated=True)
            torch.cuda.synchronize()
            if it >= warmup:
                torch_ms.append((time.perf_counter() - t0) * 1e3)
            if it + 1 < warmup + reps:
                del t_xadj, t_adj, t_o2n
        row["torch_helper_ms"] = summary(torch_ms)
        xadj_d, adj_d, _, _, o2n_d = pg._download()
        same = (t_xadj.numel() - 1 == pg.n and np.array_equal(xadj_d[: pg.n + 1], t_xadj.cpu().numpy())
                and np.array_equal(adj_d, t_adj.cpu().numpy()) and np.array_equal(o2n_d, t_o2n.cpu().numpy()))
        row["equals_torch_helper"] = bool(same)
        del t_xadj, t_adj, t_o2n
        # where they differ: vertices the helper's floating-point log2 puts into another bucket than the integer
        # rule, and whether the device's order is exactly the stable sort by the integer rule
        fb, eb = float_buckets(xadj64), exact_buckets(xadj64)
        eb_iso40 = torch.where(eb == 32, torch.full_like(eb, 40), eb)
        row["torch_helper_misbucketed_vertices"] = int((fb != eb_iso40).sum().item())
        new_to_old = torch.argsort(eb, stable=True).cpu().numpy()
        o2n_exact = np.empty(n, np.int64)
        o2n_exact[new_to_old] = np.arange(n)
        row["device_order_equals_integer_bucket_sort"] = bool(np.array_equal(o2n_d, o2n_exact))
    pg.close()
    h.close()
    return row


def reference_line():
    from oracle import bindings as B

    if not B.have_reference():
        return dict(reference="oracle/_ref/libkaminpar_ref.so not present: not measured")
    import torch

    from kaminpar_b200.graph import CSRGraph

    xadj, adj, _, _ = raw_graph("rmat20", torch.device("cpu"))
    g = CSRGraph(xadj.numpy().astype(np.uint32), adj.numpy().astype(np.uint32))
    t0 = time.perf_counter()
    B.ref_rearrange(g)
    return dict(reference="graph::rearrange_by_degree_buckets + remove_isolated_nodes, unmodified reference on the "
                          "serial oneTBB stand-in (one host thread, its heavy assertions compiled in)",
                workload="rmat20", n=g.n, m=g.m, host_ms=(time.perf_counter() - t0) * 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--workloads", default=DEFAULT)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-reference", action="store_true")
    args = ap.parse_args()
    import bench
    from scripts.bench_overlay import card

    name, power = card()
    peak, peak_src = bench.peaks()
    rows = []
    for w in args.workloads.split(","):
        rows.append(run(w, args.reps, args.warmup, peak))
        print(json.dumps(rows[-1]), flush=True)
    res = dict(card=name, power_limit=power, hbm_peak_gbs=peak, hbm_peak_source=peak_src, rows=rows)
    if not args.no_reference:
        res["reference"] = reference_line()
        print(json.dumps(res["reference"]), flush=True)
    print(json.dumps(dict(card=name, power_limit=power, hbm_peak_gbs=peak, hbm_peak_source=peak_src)))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_prepare.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
