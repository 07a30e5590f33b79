"""Where a tier-3 vertex (degrees 32..255, one warp per vertex in sweep_team) spends its time: claim wait, header
loads, gather + insert, select and finish, from %globaltimer stamps that lane 0 of each warp takes at the ends of
the phases.

The stamps exist only in a library built with -DKMP_TEAM_PHASE_STAMPS, never in the one bench.py times. This script
builds that library into a temporary directory (or takes one given with --lib) and runs the same resident
clustering call bench.py times.

    python scripts/team_phases.py [--workload rmat22] [--steps 3] [--warmup 2] [--lib PATH]

Prints one JSON line per workload: per claimed vertex, the mean time of each phase in microseconds. The claim wait
is the time from the top of the vertex's iteration until its list index is known, the finish covers the clear,
the `active` write, the proposal and the team barrier. An inactive vertex that is not rated (push rounds) costs a
claim wait and nothing else, so the later phases are also given per rated vertex."""
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

PHASES = ("claim_wait", "header", "gather_insert", "select", "finish")


def build(out_dir):
    import __graft_entry__ as G

    lib = os.path.join(out_dir, "libkaminpar_b200_team_phases.so")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc] + G.NVCC_FLAGS + ["-DKMP_TEAM_PHASE_STAMPS", "-o", lib,
                                                   os.path.join(G.CSRC, "kmp_lp.cu"), "-ldl"], cwd=ROOT)
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", nargs="+", default=["rmat22"])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--lib", help="a library built with -DKMP_TEAM_PHASE_STAMPS (default: build one)")
    args = ap.parse_args()

    tmp = tempfile.TemporaryDirectory()
    lib_path = args.lib or build(tmp.name)

    import torch

    import bench
    from hub_kernel_times import bench_mcw
    from kaminpar_b200 import lp

    lp._LIB_PATH = lib_path
    lib = lp.load_library()
    if not hasattr(lib, "kmp_team_phase_read"):
        raise RuntimeError(f"{lib_path} was not built with -DKMP_TEAM_PHASE_STAMPS")
    acc = (C.c_ulonglong * 7)()

    def read(reset):
        if lib.kmp_team_phase_read(acc, C.c_int(1 if reset else 0)) != 0:
            raise RuntimeError("kmp_team_phase_read failed")
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
        claimed, rated = max(v[5], 1), max(v[6], 1)
        out = {"workload": wl, "gpu": torch.cuda.get_device_name(0), "steps": args.steps,
               "vertices_claimed_per_step": v[5] // args.steps, "vertices_rated_per_step": v[6] // args.steps,
               "us_per_claimed_vertex": {p: round(v[i] / claimed / 1e3, 3) for i, p in enumerate(PHASES)},
               "us_per_rated_vertex": {p: round(v[i] / rated / 1e3, 3) for i, p in enumerate(PHASES) if i > 0},
               "warp_ms_per_step": {p: round(v[i] / args.steps / 1e6, 3) for i, p in enumerate(PHASES)}}
        print(json.dumps(out), flush=True)
        del handle, d_xadj, d_adj
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
