"""The ParHIP reader on the device (DESIGN.md §19) on bench.py's graphs written as ParHIP files.

Per workload, id / weight width (all 32-bit or all 64-bit) and weight variant (none, or random node weights 1..9 and
edge weights 1..W with W capped so that the edge-weight total fits int32), in one run, with the card's name and power
limit read in the same run; median and range over the repetitions after the warm-up:
  (a) parse    kmp_parse_parhip_device on the file's bytes already in device memory, NATURAL and EXTERNAL orderings:
               report.device_ms (CUDA events on the handle's stream) and a host clock around the call
  (b) read     kmp_read_parhip from a warm page cache (the file was read once before), both orderings: a host clock
               around the call
  (c) floor    the same file read into two pinned 32 MB buffers in turn and copied to the device, nothing else: a host
               clock ending in a device synchronise; the least (b) could take with this read path
  (d) ref      the reference's Release csr_read / csr_read_deg_buckets (oracle/_ref/parhip_read, built by build() from
               oracle/parhip_read.mk where the reference sources exist) on the same warm 32-bit file: ONE thread, its
               tbb::parallel_for loops on the serial oneTBB stand-in, not the reference's TBB build on all cores; the
               program's own host clock around the read; else "not available" (its 32-bit build refuses the 64-bit
               files)
  (e) memory   peak device bytes of the fused EXTERNAL read against a NATURAL read followed by
               kmp_prepare_graph_device, from a file and from resident bytes: the high-water mark of the handle's pool
               (kmp_pool_usage), with the caller's tensor of file bytes added while a path needs it (pool_peaks)
The files are written on the device with torch into a temporary directory and deleted after their workload.

    python scripts/bench_parhip.py [--reps 5] [--warmup 1] [--workloads rmat22,rgg24,grid256,road] [--out DIR]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEFAULT = "rmat22,rgg24,grid256,road"
REF = os.path.join(ROOT, "oracle", "_ref", "parhip_read")


def summary(xs):
    return dict(median=float(np.median(xs)), min=float(min(xs)), max=float(max(xs)))


def parhip_bytes(xadj, adj, vwgt, adjwgt, w64):
    """The ParHIP file of a CSR graph as a uint8 tensor on the arrays' device, at all-64 or all-32 bit widths."""
    import torch

    n, m = xadj.numel() - 1, adj.numel()
    w = 8 if w64 else 4
    dt = torch.int64 if w64 else torch.int32
    version = (0 if adjwgt is not None else 1) | (0 if vwgt is not None else 2) | (0 if w64 else 4 | 8 | 16 | 32)
    parts = [torch.tensor([version, n, m], dtype=torch.int64, device=adj.device).view(torch.uint8),
             (xadj.to(torch.int64) * w + 24 + (n + 1) * w).to(dt).view(torch.uint8), adj.to(dt).view(torch.uint8)]
    for a in (vwgt, adjwgt):
        if a is not None:
            parts.append(a.to(dt).view(torch.uint8))
    return torch.cat(parts)


def pinned_floor(path, d_buf):
    """Read the file through two pinned 32 MB buffers and copy each chunk to d_buf; returns ms."""
    import torch

    chunk = 32 << 20
    size = os.path.getsize(path)
    bufs = [torch.empty(min(chunk, size), dtype=torch.uint8).pin_memory() for _ in range(2)]
    evs = [torch.cuda.Event(), torch.cuda.Event()]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with open(path, "rb", buffering=0) as f:
        off, i = 0, 0
        while off < size:
            b = i & 1
            if i >= 2:
                evs[b].synchronize()
            k = min(chunk, size - off)
            f.readinto(memoryview(bufs[b].numpy())[:k])
            d_buf[off:off + k].copy_(bufs[b][:k], non_blocking=True)
            evs[b].record()
            off += k
            i += 1
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def pool_peaks(h, data, path):
    """Peak device bytes of the fused EXTERNAL read against a NATURAL read followed by kmp_prepare_graph_device (its
    natural graph alive until the prepared one is built), measured on the handle's pool: the high-water mark is reset
    before a step and the use before the first step is subtracted. From a file the bytes are staged in the pool and
    counted there. From resident bytes the caller's tensor is added where it must stay alive: through the whole fused
    parse, but only through the natural parse of the two-step path."""
    from kaminpar_b200 import lp
    from kaminpar_b200 import parhip as PH
    from kaminpar_b200 import prepare as PR

    length = data.numel()
    res = {}
    base, _ = lp.pool_usage(h, reset=True)
    PH.read_parhip_prepared(h, path).close()
    res["read_fused"] = lp.pool_usage(h)[1] - base
    base, _ = lp.pool_usage(h, reset=True)
    g = PH.read_parhip_device(h, path, "natural")
    pg = PR.rearrange_by_degree_buckets_device(h, g.n, g.m, *g.device_arrays()[:4])
    res["read_then_prepare"] = lp.pool_usage(h)[1] - base
    pg.close()
    g.close()
    base, _ = lp.pool_usage(h, reset=True)
    PH.parse_parhip_prepared(h, data).close()
    res["parse_fused"] = lp.pool_usage(h)[1] - base + length
    base, _ = lp.pool_usage(h, reset=True)
    g = PH.parse_parhip_device(h, data, "natural")
    p1 = lp.pool_usage(h, reset=True)[1] - base
    pg = PR.rearrange_by_degree_buckets_device(h, g.n, g.m, *g.device_arrays()[:4])
    p2 = lp.pool_usage(h)[1] - base
    res["parse_then_prepare"] = max(p1 + length, p2)
    pg.close()
    g.close()
    return res


def run(name, w64, weighted, reps, warmup, tmp):
    import torch

    import bench
    from kaminpar_b200 import lp
    from kaminpar_b200 import parhip as PH

    dev = torch.device("cuda:0")
    xadj64, adj64, _ = bench.generate(name, dev)
    n, m = xadj64.numel() - 1, adj64.numel()
    vw = ew = None
    top = 1
    if weighted:
        g = torch.Generator(device=dev).manual_seed(7)
        top = min(100, 2 * ((1 << 31) - 1) // m - 2)  # mean (1 + top) / 2 per entry: the total fits int32
        vw = torch.randint(1, 10, (n,), device=dev, generator=g)
        ew = torch.randint(1, top + 1, (m,), device=dev, generator=g)
    data = parhip_bytes(xadj64, adj64, vw, ew, w64)
    path = os.path.join(tmp, f"{name}_{int(w64)}_{int(weighted)}.parhip")
    data.cpu().numpy().tofile(path)
    del xadj64, adj64, vw, ew
    torch.cuda.synchronize()
    length = data.numel()
    ctx = lp.create_default_context()
    h = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))

    def once(g):
        rep = g.report
        g.close()
        return rep

    calls = {
        "parse_natural": lambda: once(PH.parse_parhip_device(h, data, "natural")),
        "parse_external": lambda: once(PH.parse_parhip_device(h, data, "external_degree_buckets")),
        "read_natural": lambda: once(PH.read_parhip_device(h, path, "natural")),
        "read_external": lambda: once(PH.read_parhip_device(h, path, "external_degree_buckets")),
    }
    row = dict(workload=name, widths=64 if w64 else 32, weighted=weighted, n=n, m=m, file_bytes=length,
               max_edge_weight=top)
    for key, call in calls.items():
        dev_ms, host_ms = [], []
        for it in range(warmup + reps):
            t0 = time.perf_counter()
            rep = call()
            t1 = time.perf_counter()
            if it >= warmup:
                dev_ms.append(rep.device_ms)
                host_ms.append((t1 - t0) * 1e3)
        assert rep.kind == 0 and rep.n == n and rep.m == m, rep
        row[f"{key}_device_ms"] = summary(dev_ms)
        row[f"{key}_host_ms"] = summary(host_ms)
        row[f"{key}_gbs"] = length / (np.median(dev_ms if key.startswith("parse") else host_ms) * 1e-3) / 1e9
    d_buf = torch.empty(length, dtype=torch.uint8, device=dev)
    fl = [pinned_floor(path, d_buf) for _ in range(warmup + reps)][warmup:]
    row["floor_host_ms"] = summary(fl)
    row["floor_gbs"] = length / (np.median(fl) * 1e-3) / 1e9
    del d_buf
    if w64:  # ParHIPHeader::validate: the default build exits on 64-bit widths
        row["reference_ms"] = "refused by the reference's 32-bit build"
    elif os.path.exists(REF):  # its own host clock around the read (process start and exit not counted)
        for key, arg in (("natural", "0"), ("external", "2")):
            rt = []
            for it in range(warmup + reps):
                out = json.loads(subprocess.run([REF, path, arg], check=True, capture_output=True, text=True).stdout)
                assert out["n"] == n and out["m"] == m, out
                if it >= warmup:
                    rt.append(out["ms"])
            row[f"reference_1thread_{key}_ms"] = summary(rt)
            row[f"read_{key}_speedup_over_reference_1thread"] = float(np.median(rt) /
                                                                      row[f"read_{key}_host_ms"]["median"])
    else:
        row["reference_ms"] = "not available"
    for key, val in pool_peaks(h, data, path).items():
        row[f"pool_peak_{key}"] = val
    h.close()
    os.remove(path)
    del data
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

    from scripts.bench_overlay import card

    if not torch.cuda.is_available():
        raise SystemExit("bench_parhip: no CUDA device (nothing is measured without one)")
    name, power = card()
    rows = []
    tmp = tempfile.mkdtemp(prefix="bench_parhip_")
    try:
        for w in args.workloads.split(","):
            for w64 in (False, True):
                for weighted in (False, True):
                    rows.append(run(w, w64, weighted, args.reps, args.warmup, tmp))
                    print(json.dumps(rows[-1]), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    res = dict(card=name, power_limit=power, rows=rows)
    print(json.dumps(dict(card=name, power_limit=power)))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_parhip.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
