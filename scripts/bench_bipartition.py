"""Block bipartitioning: the device call (kmp_bipartition_subgraphs) against the reference's own initial bipartitioner
(oracle/_ref/bipartition_ref at one thread and bipartition_ref_omp on all cores, built by build() where the reference
sources are present) and the same engine on one host core (the host twin, tests/cpp/ip_host_check.cc under g++ -O2).

Inputs: id-range partitions of R-MAT and 2D random geometric graphs of n = k * block_n vertices, so every block has
block_n vertices (2 048 or 8 192: the deep driver hands over blocks of 2 000-8 000 vertices at contraction limit 2000),
k from 1 to 256, extended to k' = 2k = input_k with the default preset.

Timing. Device: the library's call clock (CUDA events around the whole call, the reduction download included), median
of --reps. Reference: the program's wall clock around the reseed + pool + bipartition calls only. Host twin: the wall
clock around the per-block engine calls only (compiled, blocks extracted and parameters computed before the timer).
PCIe: the download of every block's CSR arrays (kmp_subgraphs_download into host memory), which the host path needs
before it can bipartition. Every row checks the device output equal to the reference's one-thread output and to the
twin's. Prints the card's name and power limit, then one JSON line per row.

    python scripts/bench_bipartition.py [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from kaminpar_b200 import bipartition as BP  # noqa: E402
from kaminpar_b200 import subgraphs as SG  # noqa: E402
from kaminpar_b200.graph import rgg2d, rmat  # noqa: E402
from tests import ip_host as IH  # noqa: E402
from tests import subgraph_oracle as S  # noqa: E402
from tests.test_gpu_subgraphs import _handle  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref", "bipartition_ref")


def write_blocks(path, blocks, k, input_k, mbw, total, seed, eps):
    with open(path, "wb") as f:
        np.array([len(blocks), k, input_k], np.uint32).tofile(f)
        np.array([1, total, seed], np.int32).tofile(f)
        np.array([eps], np.float64).tofile(f)
        np.asarray(mbw, np.int32).tofile(f)
        for b, (bx, ba, bv, be) in blocks:
            np.array([b, len(bx) - 1, len(ba), (bv is not None) | ((be is not None) << 1)], np.uint32).tofile(f)
            bx.tofile(f)
            ba.tofile(f)
            if bv is not None:
                bv.tofile(f)
            if be is not None:
                be.tofile(f)


def run_ref(exe, blocks_path, n):
    out = blocks_path + ".out"
    r = subprocess.run([exe, blocks_path, out, "default"], capture_output=True, text=True, check=True)
    return json.loads(r.stdout.strip().splitlines()[-1])["ms"], np.fromfile(out, np.uint32, n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card, "reference_program": os.path.exists(REF)}), flush=True)
    IH.lib()  # the twin's g++ build, outside every timer
    cfg = BP.IPConfig()
    tmp = tempfile.mkdtemp(prefix="kmp_bench_bip_")
    seed, eps = 1, 0.03
    for block_n, ks in ((8192, (1, 4, 16, 64)), (2048, (1, 4, 16, 64, 256))):
        for name in ("rmat", "rgg2d"):
            for k in ks:
                n = k * block_n
                g = rmat(int(np.log2(n)), 8, seed=1) if name == "rmat" else rgg2d(n, seed=1)
                input_k = 2 * k
                part = (np.arange(g.n, dtype=np.int64) * k // g.n).astype(np.uint32)
                mbw = IH.max_block_weights(g.n, input_k, eps)
                h = _handle()
                h.set_graph(g)
                sg = SG.extract_subgraphs(h, k, part)
                dev = []
                for _ in range(args.reps):
                    out, st = BP.bipartition(sg, h, 2 * k, input_k, mbw, seed=seed, total_node_weight=g.n,
                                             ip_config=cfg, epsilon=eps)
                    dev.append(st.device_ms)
                got = out.cpu().numpy().view(np.uint32)
                t0 = time.perf_counter()
                sg._download()
                pcie_ms = (time.perf_counter() - t0) * 1e3
                # blocks, parameters and the twin's engine calls; only the engine calls are timed
                res = S.lazy_extract_np(g.xadj, g.adjncy, None, None, part, k)
                blocks = [(b, IH.block_arrays(res, b)) for b in range(k)]
                params = [IH.block_params(cfg, input_k, mbw, True, g.n, eps, b, k, *arr) for b, arr in blocks]
                twin = np.zeros(g.n, np.uint32)
                twin_ms = 0.0
                for (b, arr), p in zip(blocks, params):
                    t0 = time.perf_counter()
                    rc, sub, _ = IH.bipartition_block(cfg, p, seed + b, *arr)
                    twin_ms += (time.perf_counter() - t0) * 1e3
                    assert rc == 0
                    twin[int(res["node_off"][b]):int(res["node_off"][b + 1])] = sub
                row = {"graph": name, "n": g.n, "k": k, "block_n": block_n, "device_ms": float(np.median(dev)),
                       "twin_1core_ms": round(twin_ms, 3), "pcie_download_ms": round(pcie_ms, 3),
                       "equal_twin": bool(np.array_equal(got, twin)), "pool_runs": st.pool_runs,
                       "levels": st.coarsening_levels}
                if os.path.exists(REF):
                    path = os.path.join(tmp, "blocks.bin")
                    write_blocks(path, blocks, k, input_k, mbw, g.n, seed, eps)
                    row["ref_1core_ms"], ref_out = run_ref(REF, path, g.n)
                    row["equal_ref"] = bool(np.array_equal(got, ref_out))
                    row["ref_allcores_ms"], omp_out = run_ref(REF + "_omp", path, g.n)
                    row["ref_allcores_threads"] = os.cpu_count()
                else:
                    row["ref_1core_ms"] = row["ref_allcores_ms"] = "not measured"
                print(json.dumps(row), flush=True)
                sg.close()
                h.close()


if __name__ == "__main__":
    main()
