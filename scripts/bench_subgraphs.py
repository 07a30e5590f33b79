"""Block-induced subgraph extraction and copy-back on the device (DESIGN.md §16) on bench.py's graphs.

Per workload and k, in one run, with the card's name and power limit read in the same run:
  extract    kmp_extract_subgraphs from the handle's device labels (stats.device_ms: CUDA events around the whole
             call, its two host waits included); median and range over the repetitions after warm-up
  copy_back  kmp_subgraphs_copy_partitions_device at k' = 2k from device sub-partitions, fetch off: CUDA events on the
             handle's stream around the call (the k0 upload, the range check and its host wait, the label copy and the
             k' block weights)
  torch      extract_torch below (stable argsort + masked select) on the same card, CUDA-synchronised host clock
  bytes      the modelled traffic of the extraction (BYTES_* below) over the extract time, as a share of the H100 SXM
             data sheet's 3.35 TB/s
Partitions are contiguous id ranges (block b = the ids [b n / k, (b + 1) n / k)): on the geometric graphs most edges
stay inside a block, on R-MAT most are cut. The torch helper's block_nodes, mapping, local xadj and adjncy are compared
with the device's at every timed size.

    python scripts/bench_subgraphs.py [--reps 5] [--warmup 1] [--workloads rmat22,...] [--ks 2,64,4096] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEFAULT = "rmat22,rgg24,grid256,road"
HBM_GBS = 3350.0  # H100 SXM data sheet, at up to 700 W
# modelled bytes of one extraction (unit weights):
#   per edge: adjncy + part[v] in the count pass, again in the edge pass (8 + 8)
#   per internal edge: mapping[v] gather + adjncy write (4 + 4)
#   per vertex: the label range check (4), xadj in both edge passes (8), the sort's key/value reads and writes per
#   8-bit pass (16 each), node_off / mapping / degree gather and write (16), two degree scans (16), the local xadj
#   kernel (20), delta reads in the edge pass (4)
BYTES_EDGE, BYTES_INTERNAL_EDGE, BYTES_VERTEX, BYTES_VERTEX_SORT_PASS = 16, 8, 68, 16


def card():
    import subprocess

    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [s.strip() for s in out.split(",")]
    return name, power


def extract_torch(xadj, adj, part, k):
    """(block_nodes, mapping, xadj_cat, adjncy) of the one-thread rule with torch ops on the device."""
    import torch

    n = xadj.numel() - 1
    order = torch.argsort(part, stable=True)
    counts = torch.bincount(part, minlength=k)
    node_off = torch.zeros(k + 1, dtype=torch.int64, device=part.device)
    node_off[1:] = torch.cumsum(counts, 0)
    newpos = torch.empty_like(order)
    newpos[order] = torch.arange(n, device=part.device)
    mapping = newpos - node_off[part]
    src = torch.repeat_interleave(torch.arange(n, device=part.device), xadj[1:] - xadj[:-1])
    keep = (part[adj] == part[src]).nonzero().squeeze(1)
    keep = keep[torch.argsort(newpos[src[keep]], stable=True)]
    out_adj = mapping[adj[keep]]
    ideg = torch.bincount(src[keep], minlength=n)[order]
    edge_pos = torch.zeros(n + 1, dtype=torch.int64, device=part.device)
    edge_pos[1:] = torch.cumsum(ideg, 0)
    blk = part[order]
    xcat = torch.zeros(n + k, dtype=torch.int64, device=part.device)
    xcat[torch.arange(n, device=part.device) + blk] = edge_pos[:n] - edge_pos[node_off[blk]]
    xcat[node_off[1:] + torch.arange(k, device=part.device)] = edge_pos[node_off[1:]] - edge_pos[node_off[:-1]]
    return order, mapping, xcat, out_adj


def run(name, ks, reps, warmup):
    import torch

    import bench
    from kaminpar_b200 import lp
    from kaminpar_b200 import subgraphs as SG

    xadj, adj, _ = bench.generate(name, "cuda")
    n, m = xadj.numel() - 1, adj.numel()
    x32, a32 = xadj.to(torch.int32).contiguous(), adj.to(torch.int32).contiguous()
    ctx = lp.create_default_context()
    h = lp.LPHandle(lp._refine_config(ctx.refinement.lp, ctx.engine))
    torch.cuda.synchronize()
    h.set_graph_device(n, m, x32.data_ptr(), a32.data_ptr())
    # the handle works on torch's stream, so that CUDA events on it bracket the copy-back on the device
    stream = torch.cuda.current_stream()
    lp._check(lp.load_library().kmp_lp_set_stream(h._h, C.c_void_p(stream.cuda_stream)))
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    rows = []
    for k in ks:
        part = (torch.arange(n, device="cuda", dtype=torch.int64) * k // n)
        h.upload_partition(part.to(torch.int32).cpu().numpy().view(np.uint32))
        ext, cb = [], []
        sg = None
        for r in range(warmup + reps):
            if sg is not None:
                sg.close()
            sg = SG.extract_subgraphs(h, k)
            no, _ = sg.offsets()
            sub = torch.from_numpy(((np.arange(n, dtype=np.int64) - np.repeat(no[:-1].astype(np.int64), np.diff(
                no.astype(np.int64)))) % 2).astype(np.int32)).cuda()
            torch.cuda.synchronize()
            ev0.record(stream)
            sg.copy_partitions(h, sub.data_ptr(), 2 * k, 2 * k, fetch=False)
            ev1.record(stream)
            torch.cuda.synchronize()
            h.upload_partition(part.to(torch.int32).cpu().numpy().view(np.uint32))
            if r >= warmup:
                ext.append(sg.stats.device_ms)
                cb.append(ev0.elapsed_time(ev1))
        m_int = sg.m
        passes = (max(1, (k - 1).bit_length()) + 7) // 8
        bytes_ = BYTES_EDGE * m + BYTES_INTERNAL_EDGE * m_int + (BYTES_VERTEX + BYTES_VERTEX_SORT_PASS * passes) * n
        med = statistics.median(ext)
        # torch baseline on the same labels, and its output against the device's
        tt = []
        for r in range(warmup + reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = extract_torch(xadj, adj, part, k)
            torch.cuda.synchronize()
            if r >= warmup:
                tt.append((time.perf_counter() - t0) * 1e3)
        order, mapping, xcat, out_adj = [t.cpu().numpy() for t in res]
        del res
        same = (np.array_equal(sg.block_nodes(), order) and np.array_equal(sg.mapping(), mapping)
                and np.array_equal(sg.xadj_cat(), xcat) and np.array_equal(sg._download()[1], out_adj))
        sg.close()
        row = dict(workload=name, n=n, m=m, k=k, m_internal=m_int, internal_share=round(m_int / max(m, 1), 4),
                   extract_ms=round(med, 3), extract_ms_range=[round(min(ext), 3), round(max(ext), 3)],
                   copy_back_ms=round(statistics.median(cb), 3),
                   copy_back_ms_range=[round(min(cb), 3), round(max(cb), 3)],
                   modelled_bytes=bytes_, extract_gbs=round(bytes_ / med / 1e6, 1),
                   share_of_3350_gbs=round(bytes_ / med / 1e6 / HBM_GBS, 3),
                   torch_ms=round(statistics.median(tt), 3), torch_same_output=bool(same))
        rows.append(row)
        print(json.dumps(row), flush=True)
    h.close()
    del x32, a32, xadj, adj
    torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--workloads", default=DEFAULT)
    ap.add_argument("--ks", default="2,64,4096")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_subgraphs.py measures on the GPU: no CUDA device")
    name, power = card()
    ks = [int(x) for x in args.ks.split(",")]
    rows = []
    for w in args.workloads.split(","):
        rows += run(w, ks, args.reps, args.warmup)
    res = dict(card=name, power_limit=power, hbm_datasheet_gbs=HBM_GBS, rows=rows)
    print(json.dumps(dict(card=name, power_limit=power)))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_subgraphs.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
