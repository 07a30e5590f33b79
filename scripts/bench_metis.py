"""The METIS reader on the device (DESIGN.md §18) on bench.py's graphs written as METIS files.

Per workload and edge-weight variant (unit, and random weights 1..W written after every target, W = 100 or less so
that the total edge weight fits int32, which csr_read asserts), in one run, with
the card's name and power limit read in the same run; median and range over the repetitions after the warm-up:
  (a) parse    kmp_parse_metis_device on the file's bytes already in device memory: report.device_ms (CUDA events on
               the handle's stream around the passes) and a host clock around the call; per-kernel device time from
               torch.profiler in a separate, untimed call
  (b) read     kmp_read_metis from a warm page cache (the file was read once before): a host clock around the call
  (c) floor    the same file read into two pinned 32 MB buffers in turn and copied to the device, no parsing: a host
               clock around it ending in a device synchronise; the least (b) could take with this read path
  (d) ref      the reference's csr_read in its Release build (oracle/_ref/metis_read, built by build() from
               oracle/metis_read.mk where the reference sources exist) on the same warm file: the program's own host
               clock around the read; else "not available"
  bytes        the byte model of (a): the file twice (the summary pass and the write pass; a token's re-read for its
               value is counted once), 4 B per xadj entry, 4 B per adjacency entry per array written, and 3 reads or
               writes of the 88-byte tile summaries; over (a)'s device time, against the data sheet's 3.35 TB/s
The files are written by a vectorised writer on the device (graph.write_metis loops per vertex) into a temporary
directory and deleted after their workload.

    python scripts/bench_metis.py [--reps 5] [--warmup 1] [--workloads rmat22,rgg24,grid256,road] [--out DIR]
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
DATASHEET_GBS = 3350.0
SUMMARY_BYTES = 88  # sizeof(MetisSum<unsigned long long>) in kmp_metis.cuh
TILE = 4096
KERNELS = (("summary", ("k_metis_summary",)), ("scan", ("DeviceScan", "Scan")), ("write", ("k_metis_write",)),
           ("finish", ("k_metis_finish",)))
REF = os.path.join(ROOT, "oracle", "_ref", "metis_read")


def summary(xs):
    return dict(median=float(np.median(xs)), min=float(min(xs)), max=float(max(xs)))


def metis_bytes(xadj, adj, adjwgt=None):
    """The METIS text of a CSR graph as a uint8 tensor on the arrays' device: one line per vertex, targets 1-based,
    each weight after its target, one space between tokens."""
    import torch

    dev = adj.device
    n, m = xadj.numel() - 1, adj.numel()
    ew = int(adjwgt is not None)
    deg = xadj[1:] - xadj[:-1]
    slots = torch.clamp(deg * (1 + ew), min=1)  # an empty row is one token of no digits: its newline
    rs = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    rs[1:] = torch.cumsum(slots, 0)
    T = int(rs[-1])
    val = torch.zeros(T, dtype=torch.int64, device=dev)
    live = torch.zeros(T, dtype=torch.bool, device=dev)
    row = torch.repeat_interleave(torch.arange(n, device=dev), deg)
    pos = rs[:-1][row] + (torch.arange(m, device=dev) - xadj[:-1][row]) * (1 + ew)
    del row
    val[pos] = adj.to(torch.int64) + 1
    live[pos] = True
    if ew:
        val[pos + 1] = adjwgt.to(torch.int64)
        live[pos + 1] = True
    del pos
    nd = live.to(torch.int64)
    p10 = 10
    while bool((val >= p10).any()):
        nd += (val >= p10).to(torch.int64)
        p10 *= 10
    head = f"{n} {m // 2}{' 1' if ew else ''}\n".encode()
    lens = nd + 1
    offs = torch.cumsum(lens, 0) - lens + len(head)
    out = torch.empty(len(head) + int(lens.sum()), dtype=torch.uint8, device=dev)
    out[: len(head)] = torch.tensor(list(head), dtype=torch.uint8, device=dev)
    sep = torch.full((T,), 32, dtype=torch.uint8, device=dev)
    sep[rs[1:] - 1] = 10
    out[offs + nd] = sep
    del sep, lens
    for k in range(int(nd.max())):  # digit k from the right
        sel = torch.nonzero(nd > k).squeeze(1)
        out[offs[sel] + nd[sel] - 1 - k] = (48 + (val[sel] // 10 ** k) % 10).to(torch.uint8)
    return out


def kernel_ms(call, calls=3):
    """Device time per kernel of one call, from torch.profiler over `calls` calls: each kernel's time averaged over the
    launches the profiler recorded (every kernel runs once per call; the first launches of a session can go
    unrecorded, so totals are not divided by `calls`)."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            call()
    out = {k: 0.0 for k, _ in KERNELS}
    other = 0.0
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        t = (ev.cuda_time_total if t is None else t) / max(ev.count, 1)
        for k, keys in KERNELS:
            if any(s in ev.key for s in keys):
                out[k] += t / 1e3
                break
        else:
            other += t / 1e3
    out["other"] = other
    return out


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
            n = min(chunk, size - off)
            f.readinto(memoryview(bufs[b].numpy())[:n])
            d_buf[off:off + n].copy_(bufs[b][:n], non_blocking=True)
            evs[b].record()
            off += n
            i += 1
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def run(name, weighted, reps, warmup, tmp):
    import torch

    import bench
    from kaminpar_b200 import lp
    from kaminpar_b200 import metis as ME

    dev = torch.device("cuda:0")
    xadj64, adj64, _ = bench.generate(name, dev)
    ew = None
    if weighted:
        g = torch.Generator(device=dev).manual_seed(7)
        top = min(100, 2 * ((1 << 31) - 1) // adj64.numel() - 2)  # mean (1 + top) / 2 per entry: the total fits int32
        ew = torch.randint(1, top + 1, (adj64.numel(),), device=dev, generator=g)
    data = metis_bytes(xadj64, adj64, ew)
    n, m = xadj64.numel() - 1, adj64.numel()
    path = os.path.join(tmp, f"{name}_{int(weighted)}.metis")
    data.cpu().numpy().tofile(path)
    del xadj64, adj64, ew
    torch.cuda.synchronize()
    length = data.numel()
    ctx = lp.create_default_context()
    h = lp.LPHandle(lp._cluster_config(ctx.coarsening.clustering.lp, ctx.engine))

    def parse():
        g = ME.parse_metis_device(h, data)
        rep = g.report
        g.close()
        return rep

    def read():
        g = ME.read_metis_device(h, path)
        rep = g.report
        g.close()
        return rep

    row = dict(workload=name, weighted=weighted, n=n, m=m, file_bytes=length, max_edge_weight=top if weighted else 1)
    for key, call in (("parse", parse), ("read", read)):
        dev_ms, host_ms = [], []
        for it in range(warmup + reps):
            t0 = time.perf_counter()
            rep = call()
            t1 = time.perf_counter()
            if it >= warmup:
                dev_ms.append(rep.device_ms)
                host_ms.append((t1 - t0) * 1e3)
        assert rep.kind == 0 and rep.n == n and 2 * rep.m == m, rep
        row[f"{key}_device_ms"] = summary(dev_ms)
        row[f"{key}_host_ms"] = summary(host_ms)
        row[f"{key}_gbs"] = length / (np.median(dev_ms if key == "parse" else host_ms) * 1e-3) / 1e9
    row["parse_kernels_ms"] = kernel_ms(parse)
    d_buf = torch.empty(length, dtype=torch.uint8, device=dev)
    fl = [pinned_floor(path, d_buf) for _ in range(warmup + reps)][warmup:]
    row["floor_host_ms"] = summary(fl)
    row["floor_gbs"] = length / (np.median(fl) * 1e-3) / 1e9
    del d_buf
    if os.path.exists(REF):  # its own host clock around csr_read (process start and exit not counted)
        rt = []
        for it in range(warmup + reps):
            out = json.loads(subprocess.run([REF, path], check=True, capture_output=True, text=True).stdout)
            assert out["n"] == n and out["m"] == m, out
            if it >= warmup:
                rt.append(out["ms"])
        row["reference_ms"] = summary(rt)
        row["reference_gbs"] = length / (np.median(rt) * 1e-3) / 1e9
        row["read_speedup_over_reference"] = float(np.median(rt) / row["read_host_ms"]["median"])
        row["parse_speedup_over_reference"] = float(np.median(rt) / row["parse_host_ms"]["median"])
    else:
        row["reference_ms"] = "not available"
    tiles = (length + TILE - 1) // TILE
    model = 2 * length + 4 * (n + 1) + 4 * m * (2 if weighted else 1) + 3 * tiles * SUMMARY_BYTES
    row["parse_modelled_bytes"] = model
    row["parse_model_gbs"] = model / (row["parse_device_ms"]["median"] * 1e-3) / 1e9
    row["parse_share_of_datasheet"] = row["parse_model_gbs"] / DATASHEET_GBS
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
        raise SystemExit("bench_metis: no CUDA device (nothing is measured without one)")
    name, power = card()
    rows = []
    tmp = tempfile.mkdtemp(prefix="bench_metis_")
    try:
        for w in args.workloads.split(","):
            for weighted in (False, True):
                rows.append(run(w, weighted, args.reps, args.warmup, tmp))
                print(json.dumps(rows[-1]), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    res = dict(card=name, power_limit=power, datasheet_gbs=DATASHEET_GBS, rows=rows)
    print(json.dumps(dict(card=name, power_limit=power)))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_metis.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
