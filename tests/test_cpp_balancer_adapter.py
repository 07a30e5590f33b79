"""The C++ balancer adapters (OverloadBalancer, UnderloadBalancer in include/kaminpar_b200_adapters.hpp) are valid
C++20, link against the C-ABI library, fail loudly without a GPU (CPU test) and give the oracle's results on one
(GPU test)."""
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "kaminpar_b200", "csrc")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")


def build(tmp_path):
    exe = str(tmp_path / "balancer_adapter_smoke")
    cmd = [CXX, "-std=c++20", "-Wall", "-I" + os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "balancer_adapter_smoke.cc"), "-o", exe, "-L" + LIBDIR,
           "-lkaminpar_b200", "-Wl,-rpath," + LIBDIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_balancer_adapters_compile_link_and_have_no_fallback(tmp_path):
    import torch

    exe = build(tmp_path)
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 1 and "no CUDA device" in r.stdout


@pytest.mark.gpu
def test_balancer_adapters_round_trip_on_gpu(tmp_path):
    """Overload then underload balance through the C++ adapters equal the oracle bit for bit."""
    from kaminpar_b200.graph import CSRGraph
    from tests import balance_oracle as O
    from tests import underload_oracle as U

    exe = build(tmp_path)
    dump = str(tmp_path / "dump.txt")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120, env=dict(os.environ, ADAPTER_DUMP=dump))
    assert r.returncode == 0, r.stdout + r.stderr
    assert "adapter ok" in r.stdout
    lines = open(dump).read().strip().split("\n")
    n, m = (int(x) for x in lines[0].split())
    xadj, adj, inp, after_over, under_in, after_under = (np.array(lines[i].split(), np.int64) for i in range(1, 7))
    bw_over, bw_under = (np.array(lines[i].split(), np.int64) for i in (7, 8))
    improved_over, improved_under = (bool(int(x)) for x in lines[9].split())
    g = CSRGraph(xadj.astype(np.uint32), adj.astype(np.uint32))
    assert g.n == n and g.m == m
    k = 4
    maxw, minw, pbw = np.full(k, 37), np.full(k, 35), np.full(k, 36)
    want = O.overload_balance(g, k, inp.astype(np.uint32), maxw, pbw)
    assert improved_over == want["improved"] and improved_over
    assert np.array_equal(after_over, want["labels"]) and np.array_equal(bw_over, want["block_weights"])
    want = U.underload_balance(g, k, under_in.astype(np.uint32), maxw, minw)
    assert improved_under == want["improved"] and improved_under
    assert np.array_equal(after_under, want["labels"]) and np.array_equal(bw_under, want["block_weights"])
    assert want["after"] == 0
