"""The C++ sparsification adapters (kaminpar_b200::sparsification_target, CoarseGraph::sparsify in
include/kaminpar_b200_adapters.hpp) are valid C++20, link against the C-ABI library, fail loudly without a GPU (CPU
test) and give the oracle's coarse graph on one (GPU test)."""
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "kaminpar_b200", "csrc")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")


def build(tmp_path):
    exe = str(tmp_path / "sparsify_adapter_smoke")
    cmd = [CXX, "-std=c++20", "-Wall", "-I" + os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "sparsify_adapter_smoke.cc"), "-o", exe, "-L" + LIBDIR,
           "-lkaminpar_b200", "-Wl,-rpath," + LIBDIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_sparsify_adapter_compiles_links_and_has_no_fallback(tmp_path):
    import torch

    exe = build(tmp_path)
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 1 and "no CUDA device" in r.stdout


@pytest.mark.gpu
def test_sparsify_adapter_matches_oracle_on_gpu(tmp_path):
    """LP clustering -> contract_clustering -> CoarseGraph::sparsify through the adapters equals the oracle; get()
    after sparsify returns the sparsified graph, and sparsification_target equals the C ABI and the oracle."""
    from oracle import contraction_oracle as CO
    from tests import sparsify_oracle as S

    exe = build(tmp_path)
    dump = str(tmp_path / "dump.txt")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120, env=dict(os.environ, ADAPTER_DUMP=dump))
    assert r.returncode == 0, r.stdout + r.stderr
    assert "adapter ok" in r.stdout
    lines = open(dump).read().strip().split("\n")
    n, m, c_n, target, formula = (int(x) for x in lines[0].split())
    xadj, adj, ew, cl = (np.array(lines[i].split(), np.int64) for i in range(1, 5))
    seed = int(lines[5])
    c_xadj, c_adj, c_ew, c_vw = (np.array(lines[i].split() if i < len(lines) else [], np.int64) for i in range(6, 10))
    assert len(xadj) == n + 1 and len(adj) == m
    assert formula == S.sparsification_target(m, n, c_n)
    con = CO.contract(xadj, adj, None, ew, cl)
    assert con["c_n"] == c_n and c_n < n
    o = S.sparsify_contracted(con, target, seed)
    assert len(o["c_adjncy"]) < len(con["c_adjncy"])  # get() cannot have returned the unsparsified copy
    assert np.array_equal(c_xadj, o["c_xadj"]) and np.array_equal(c_adj, o["c_adjncy"])
    assert np.array_equal(c_ew, o["c_adjwgt"]) and np.array_equal(c_vw, o["c_vwgt"])
