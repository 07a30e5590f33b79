"""The C++ overlay adapter (kaminpar_b200::LPClustering::compute_overlay_clustering in
include/kaminpar_b200_adapters.hpp) is valid C++20, links against the C-ABI library, fails loudly without a GPU (CPU
test) and gives the overlay oracle's result over the clusterer's own consecutive calls on one (GPU test)."""
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "kaminpar_b200", "csrc")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")


def build(tmp_path):
    exe = str(tmp_path / "overlay_adapter_smoke")
    cmd = [CXX, "-std=c++20", "-Wall", "-I" + os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "overlay_adapter_smoke.cc"), "-o", exe, "-L" + LIBDIR,
           "-lkaminpar_b200", "-Wl,-rpath," + LIBDIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_overlay_adapter_compiles_links_and_has_no_fallback(tmp_path):
    import torch

    exe = build(tmp_path)
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 1 and "no CUDA device" in r.stdout


@pytest.mark.gpu
def test_overlay_adapter_matches_oracle_on_gpu(tmp_path):
    from tests import overlay_oracle as O

    exe = build(tmp_path)
    dump = str(tmp_path / "dump.txt")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120, env=dict(os.environ, ADAPTER_DUMP=dump))
    assert r.returncode == 0, r.stdout + r.stderr
    assert "adapter ok" in r.stdout
    rows = [np.array(x.split(), np.int64) for x in open(dump).read().strip().split("\n")]
    calls, ov = rows[:-1], rows[-1]
    assert len(calls) == 4 and len(ov) == 24 * 24
    assert len({tuple(c) for c in calls}) > 1  # the calls differ: the overlay is not one of them
    assert np.array_equal(ov, O.overlay_tree(calls))
