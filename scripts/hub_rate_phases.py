"""Where one item of the clusterer's hub rate kernel (sweep_hub_rate) spends its time: header, stream + insert,
select and clear, from %globaltimer stamps that thread 0 of each CTA takes at the item's barriers.

The stamps exist only in a library built with -DKMP_HUB_PHASE_STAMPS, never in the one bench.py times. This script
builds that library into a temporary directory (or takes one given with --lib) and runs the same resident
clustering call bench.py times.

    python scripts/hub_rate_phases.py [--workload rmat22 rmat24] [--steps 3] [--warmup 2] [--lib PATH]

Prints one JSON line per workload: per rated item, the mean device time of each phase in microseconds; the header
phase is the time from the end of the previous item until the item's header is in shared memory, and `load_us` is
how long the thread that loads a header spends doing it. The stamps add a few atomics per item, so the phase times
add up to somewhat more than the kernel takes without them."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

PHASES = ("header", "stream_insert", "select", "clear")


def build(out_dir):
    import __graft_entry__ as G

    lib = os.path.join(out_dir, "libkaminpar_b200_phases.so")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc] + G.NVCC_FLAGS + ["-DKMP_HUB_PHASE_STAMPS", "-o", lib,
                                                   os.path.join(G.CSRC, "kmp_lp.cu"), "-ldl"], cwd=ROOT)
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", nargs="+", default=["rmat22", "rmat24"])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--lib", help="a library built with -DKMP_HUB_PHASE_STAMPS (default: build one)")
    args = ap.parse_args()

    tmp = tempfile.TemporaryDirectory()
    lib_path = args.lib or build(tmp.name)

    import torch

    import bench
    from hub_kernel_times import bench_mcw
    from kaminpar_b200 import lp

    lp._LIB_PATH = lib_path
    lib = lp.load_library()
    if not hasattr(lib, "kmp_hub_phase_read"):
        raise RuntimeError(f"{lib_path} was not built with -DKMP_HUB_PHASE_STAMPS")
    acc = (C.c_ulonglong * 7)()

    def read(reset):
        if lib.kmp_hub_phase_read(acc, C.c_int(1 if reset else 0)) != 0:
            raise RuntimeError("kmp_hub_phase_read failed")
        return list(acc)

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
        read(reset=True)
        for _ in range(args.steps):
            handle.cluster(mcw, fetch=False)
        v = read(reset=True)
        rated = max(v[4], 1)
        out = {"workload": wl, "gpu": torch.cuda.get_device_name(0), "steps": args.steps,
               "items_rated_per_step": v[4] // args.steps, "items_claimed_per_step": v[5] // args.steps,
               "us_per_rated_item": {p: round(v[i] / rated / 1e3, 3) for i, p in enumerate(PHASES)},
               "load_us": round(v[6] / max(v[5], 1) / 1e3, 3),
               "cta_ms_per_step": {p: round(v[i] / args.steps / 1e6, 3) for i, p in enumerate(PHASES)}}
        print(json.dumps(out), flush=True)
        del handle, d_xadj, d_adj
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
