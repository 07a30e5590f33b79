"""The C++ subgraph adapters (kaminpar_b200::extract_subgraphs, Subgraphs, copy_subgraph_partitions in
include/kaminpar_b200_adapters.hpp) are valid C++20, link against the C-ABI library, fail loudly without a GPU (CPU
test) and give the oracle's blocks and copy-back on one (GPU test)."""
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "kaminpar_b200", "csrc")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")


def build(tmp_path):
    exe = str(tmp_path / "subgraph_adapter_smoke")
    cmd = [CXX, "-std=c++20", "-Wall", "-I" + os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "subgraph_adapter_smoke.cc"), "-o", exe, "-L" + LIBDIR,
           "-lkaminpar_b200", "-Wl,-rpath," + LIBDIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_subgraph_adapter_compiles_links_and_has_no_fallback(tmp_path):
    import torch

    exe = build(tmp_path)
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 1 and "no CUDA device" in r.stdout


@pytest.mark.gpu
def test_subgraph_adapter_matches_oracle_on_gpu(tmp_path):
    from tests import subgraph_oracle as S

    exe = build(tmp_path)
    dump = str(tmp_path / "dump.txt")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120, env=dict(os.environ, ADAPTER_DUMP=dump))
    assert r.returncode == 0, r.stdout + r.stderr
    assert "adapter ok" in r.stdout
    lines = open(dump).read().strip().split("\n")
    n, k, k_prime = (int(x) for x in lines[0].split())
    xadj, adj, vw, ew, part, dx, da, dmap, dbn, sub, out = (np.array(lines[i].split(), np.int64) for i in range(1, 12))
    exp = S.lazy_extract(xadj, adj, vw, ew, part, k)
    assert np.array_equal(dx, exp["xadj"]) and np.array_equal(da, exp["adjncy"])
    assert np.array_equal(dmap, exp["mapping"]) and np.array_equal(dbn, exp["block_nodes"])
    want, _ = S.copy_back(part, exp["mapping"], exp["node_off"], sub, k, k_prime, k_prime, vw)
    assert np.array_equal(out, want) and len(np.unique(want)) == k_prime
