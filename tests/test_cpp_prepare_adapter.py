"""The C++ preparation adapters (kaminpar_b200::rearrange_by_degree_buckets, PreparedGraph, assign_isolated_nodes in
include/kaminpar_b200_adapters.hpp) are valid C++20, link against the C-ABI library, fail loudly without a GPU (CPU
test) and give the oracle's rearrangement and finish on one (GPU test)."""
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "kaminpar_b200", "csrc")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")


def build(tmp_path):
    exe = str(tmp_path / "prepare_adapter_smoke")
    cmd = [CXX, "-std=c++20", "-Wall", "-I" + os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "prepare_adapter_smoke.cc"), "-o", exe, "-L" + LIBDIR,
           "-lkaminpar_b200", "-Wl,-rpath," + LIBDIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_prepare_adapter_compiles_links_and_has_no_fallback(tmp_path):
    import torch

    exe = build(tmp_path)
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 1 and "no CUDA device" in r.stdout


@pytest.mark.gpu
def test_prepare_adapter_matches_oracle_on_gpu(tmp_path):
    from tests import prepare_oracle as P

    exe = build(tmp_path)
    dump = str(tmp_path / "dump.txt")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120, env=dict(os.environ, ADAPTER_DUMP=dump))
    assert r.returncode == 0, r.stdout + r.stderr
    assert "adapter ok" in r.stdout
    lines = open(dump).read().strip().split("\n")
    n, m, k = (int(x) for x in lines[0].split())
    xadj, adj, vw, mbw, o2n, part, out, bw = (np.array(lines[i].split(), np.int64) for i in range(1, 9))
    prep = P.rearrange(xadj, adj, vw)
    assert np.array_equal(o2n, prep["old_to_new"]) and len(part) == prep["n_prime"] < n
    exp, exp_bw = P.finish(prep, k, mbw, part)
    assert np.array_equal(out, exp) and np.array_equal(bw, exp_bw)
    assert len(np.unique(exp[prep["new_to_old"][prep["n_prime"]:]])) > 1  # next fit passed a block
