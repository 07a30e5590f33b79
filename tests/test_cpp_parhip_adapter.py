"""The C++ ParHIP adapter (kaminpar_b200::read_parhip, ParhipGraph, ParhipError in include/kaminpar_b200_adapters.hpp)
is valid C++20, links against the C-ABI library, fails loudly without a GPU (CPU test) and gives the oracle's graphs
and first violations on one (GPU test): a weighted file, a 64-bit file and a refused file."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests import parhip_oracle as PO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "kaminpar_b200", "csrc")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
XADJ, ADJ = [0, 2, 3, 3, 4, 5, 7, 10], [1, 5, 0, 6, 6, 0, 6, 3, 4, 5]


def files():
    bad = bytearray(PO.write(XADJ, ADJ))
    bad[24 + 8 * 4 + 4 * 4: 24 + 8 * 4 + 5 * 4] = (7).to_bytes(4, "little")  # target 7 >= n
    return (PO.write(XADJ, ADJ, [3, 1, 4, 1, 5, 9, 2], list(range(1, 11))),                  # weighted
            PO.write(XADJ, ADJ, None, list(range(11, 21)), PO.version_of(False, True, True, True, True, True)),
            bytes(bad))                                                                       # refused


def build(tmp_path):
    exe = str(tmp_path / "parhip_adapter_smoke")
    cmd = [CXX, "-std=c++20", "-Wall", "-I" + os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "parhip_adapter_smoke.cc"), "-o", exe, "-L" + LIBDIR,
           "-lkaminpar_b200", "-Wl,-rpath," + LIBDIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_parhip_adapter_compiles_links_and_has_no_fallback(tmp_path):
    import torch

    exe = build(tmp_path)
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 1 and "no CUDA device" in r.stdout


@pytest.mark.gpu
def test_parhip_adapter_matches_oracle_on_gpu(tmp_path):
    exe = build(tmp_path)
    paths = []
    for i, data in enumerate(files()):
        p = tmp_path / f"f{i}.parhip"
        p.write_bytes(data)
        paths.append(str(p))
    dump = str(tmp_path / "dump.txt")
    r = subprocess.run([exe] + paths, capture_output=True, text=True, timeout=120,
                       env=dict(os.environ, ADAPTER_DUMP=dump))
    assert r.returncode == 0, r.stdout + r.stderr
    assert "adapter ok" in r.stdout
    lines = open(dump).read().split("\n")
    at = 0
    for data in files():
        exp = PO.read(data, PO.EXTERNAL)
        assert int(lines[at]) == exp["kind"]
        if exp["kind"] == 0:
            got = [np.array(lines[at + 1 + j].split(), np.int64) for j in range(5)]
            for a, f in zip(got, ("xadj", "adjncy", "vwgt", "adjwgt", "old_to_new")):
                want = np.zeros(0, np.int64) if exp[f] is None else np.asarray(exp[f], np.int64)
                assert np.array_equal(a, want), f
            at += 6
        else:
            assert lines[at + 1] == "neighbor out of range at byte %d (adjncy entry %d)" % (exp["offset"], exp["index"])
            at += 2
