"""Graph validation on the device (DESIGN.md §17) on bench.py's graphs, valid, in device memory.

Per workload and edge-weight variant (unit, and random symmetric weights 1..100), in one run, with the card's name and
power limit read in the same run:
  call       kmp_validate_graph_device: report.device_ms (CUDA events on the handle's stream around the whole call, its
             host wait included) and a host clock around the call (it ends in a device synchronise); median and range
             over the repetitions after the warm-up
  phases     device time per phase from torch.profiler in a separate, untimed call: xadj pass (k_val_xadj), segmented
             sort (k_val_iota + CUB's segmented sort), edge probe (k_tile_owners + k_val_edges), duplicates (k_val_dups)
  bytes      modelled traffic, every array access counted once at its element size: 4 B per vertex and 4 B per edge
             (xadj pass), 4 B per edge (positions), 16 B per edge (the sort reads and writes targets and positions),
             20 B per edge (probe: adjncy, xadj[v] and xadj[v+1], the found target and its position; the binary
             search's other probes not counted), 8 B per edge more with weights, 8 B per edge (duplicates: targets and
             the row bound); over report.device_ms, against the HBM peak bench.py uses (MEASURED_PEAKS.json, else the
             data sheet's 3.35 TB/s)
  torch      a torch cross-check on the same device: sort the (u, v) and the (v, u) keys and compare (the multiset of
             edges is symmetric); its time (CUDA-synchronised host clock) and verdict, a sanity figure only

    python scripts/bench_validate.py [--reps 5] [--warmup 1] [--workloads rmat22,rgg24,grid256,road] [--out DIR]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEFAULT = "rmat22,rgg24,grid256,road"
PHASES = (("xadj pass", ("k_val_xadj",)), ("segmented sort", ("k_val_iota", "SegmentedSort", "segmented_sort")),
          ("edge probe", ("k_tile_owners", "k_val_first_bad", "k_val_edges")), ("duplicates", ("k_val_dups",)))


def summary(xs):
    return dict(median=float(np.median(xs)), min=float(min(xs)), max=float(max(xs)))


def symmetric_weights(xadj, adj):
    """1 + a hash of the unordered pair {u, v} mod 100: the same on both directions of an edge."""
    import torch

    n = xadj.numel() - 1
    src = torch.repeat_interleave(torch.arange(n, device=adj.device), xadj[1:] - xadj[:-1])
    lo, hi = torch.minimum(src, adj), torch.maximum(src, adj)
    return (1 + ((lo * 2654435761 + hi * 40503) % 100)).to(torch.int32)


def torch_symmetric(xadj, adj):
    import torch

    n = xadj.numel() - 1
    src = torch.repeat_interleave(torch.arange(n, device=adj.device), xadj[1:] - xadj[:-1])
    fwd = torch.sort(src * n + adj).values
    rev = torch.sort(adj * n + src).values
    return bool(torch.equal(fwd, rev))


def phase_ms(call):
    """Device time per phase of one call, from torch.profiler's kernel records."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
    out = {p: 0.0 for p, _ in PHASES}
    other = 0.0
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        t = ev.cuda_time_total if t is None else t
        for p, keys in PHASES:
            if any(k in ev.key for k in keys):
                out[p] += t / 1e3
                break
        else:
            other += t / 1e3
    out["other"] = other
    return out


def run(name, weighted, reps, warmup, peak):
    import torch

    import bench
    from kaminpar_b200 import lp
    from kaminpar_b200 import validate as VA

    dev = torch.device("cuda:0")
    xadj64, adj64, _ = bench.generate(name, dev)
    ew = symmetric_weights(xadj64, adj64) if weighted else None
    d_xadj, d_adj = xadj64.to(torch.int32).contiguous(), adj64.to(torch.int32).contiguous()
    n, m = d_xadj.numel() - 1, d_adj.numel()
    torch.cuda.synchronize()
    ctx = lp.create_default_context()
    h = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))
    call = lambda: VA.validate_graph_device(h, n, m, d_xadj.data_ptr(), d_adj.data_ptr(),
                                            ew.data_ptr() if ew is not None else 0)
    dev_ms, host_ms = [], []
    for it in range(warmup + reps):
        t0 = time.perf_counter()
        rep = call()
        t1 = time.perf_counter()
        if it >= warmup:
            dev_ms.append(rep.device_ms)
            host_ms.append((t1 - t0) * 1e3)
    row = dict(workload=name, weighted=weighted, n=n, m=m, valid=bool(rep.valid), kind=rep.kind_name,
               duplicates=rep.duplicates, call_device_ms=summary(dev_ms), call_host_ms=summary(host_ms))
    row["phases_ms"] = phase_ms(call)
    bytes_ = 4 * n + m * (4 + 4 + 16 + 20 + 8 + (8 if weighted else 0))
    row["modelled_bytes"] = bytes_
    row["gbs"] = bytes_ / (row["call_device_ms"]["median"] * 1e-3) / 1e9
    row["share_of_hbm_peak"] = row["gbs"] / peak
    if not weighted:
        t_ms = []
        for it in range(warmup + reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sym = torch_symmetric(xadj64, adj64)
            torch.cuda.synchronize()
            if it >= warmup:
                t_ms.append((time.perf_counter() - t0) * 1e3)
        row["torch_cross_check_ms"] = summary(t_ms)
        row["torch_symmetric"] = sym
        row["agrees_with_torch"] = sym == (rep.valid == 1)
    h.close()
    del d_xadj, d_adj, xadj64, adj64, ew
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--workloads", default=DEFAULT)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    import bench
    from scripts.bench_overlay import card

    if not torch.cuda.is_available():
        raise SystemExit("bench_validate: no CUDA device (nothing is measured without one)")
    name, power = card()
    peak, peak_src = bench.peaks()
    rows = []
    for w in args.workloads.split(","):
        for weighted in (False, True):
            rows.append(run(w, weighted, args.reps, args.warmup, peak))
            print(json.dumps(rows[-1]), flush=True)
    res = dict(card=name, power_limit=power, hbm_peak_gbs=peak, hbm_peak_source=peak_src, rows=rows)
    print(json.dumps(dict(card=name, power_limit=power, hbm_peak_gbs=peak, hbm_peak_source=peak_src)))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_validate.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
