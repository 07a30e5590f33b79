"""The C++ validation adapter (kaminpar_b200::validate_graph, GraphReport in include/kaminpar_b200_adapters.hpp) is
valid C++20, links against the C-ABI library, fails loudly without a GPU (CPU test) and gives the oracle's reports
and the reference's warning lines on one (GPU test)."""
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "kaminpar_b200", "csrc")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")


def build(tmp_path):
    exe = str(tmp_path / "validate_adapter_smoke")
    cmd = [CXX, "-std=c++20", "-Wall", "-I" + os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "validate_adapter_smoke.cc"), "-o", exe, "-L" + LIBDIR,
           "-lkaminpar_b200", "-Wl,-rpath," + LIBDIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_validate_adapter_compiles_links_and_has_no_fallback(tmp_path):
    import torch

    exe = build(tmp_path)
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 1 and "no CUDA device" in r.stdout


@pytest.mark.gpu
def test_validate_adapter_matches_oracle_on_gpu(tmp_path):
    from tests import validate_oracle as V

    exe = build(tmp_path)
    dump = str(tmp_path / "dump.txt")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120, env=dict(os.environ, ADAPTER_DUMP=dump))
    assert r.returncode == 0, r.stdout + r.stderr
    assert "adapter ok" in r.stdout
    lines = open(dump).read().split("\n")
    kinds = []
    for i in range(4):
        xadj, adj, w = (np.array(lines[5 * i + j].split(), np.int64) for j in range(3))
        got = [int(x) for x in lines[5 * i + 3].split()]
        exp = V.validate(xadj, adj, w)
        assert got == [exp[f] for f in ("kind", "u", "e", "v", "e_rev", "v_rev", "w", "w_rev", "duplicates")]
        assert lines[5 * i + 4] == V.message(exp)
        kinds.append(exp["kind"])
    assert kinds == [V.VALID, V.MISSING_REVERSE, V.NEIGHBOR_OF_NEIGHBOR_OUT_OF_GRAPH, V.WEIGHT_MISMATCH]
