"""The C++ METIS adapter (kaminpar_b200::read_metis, MetisGraph, MetisError in include/kaminpar_b200_adapters.hpp) is
valid C++20, links against the C-ABI library, fails loudly without a GPU (CPU test) and gives the oracle's graphs,
dropped weights, extra-lines warning and first violations on one (GPU test)."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests import metis_oracle as MO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "kaminpar_b200", "csrc")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
FILES = (b"3 2 11\n5 2 4 3 1\n1 1 4\n7 1 1\n",       # node and edge weights kept
         b"% c\n3 2 1\n2 1 3 1\n1 1\n1 1\n\n",          # unit edge weights dropped, an extra line
         b"2 1\n2\n2\n")                                 # a self-loop: refused


def build(tmp_path):
    exe = str(tmp_path / "metis_adapter_smoke")
    cmd = [CXX, "-std=c++20", "-Wall", "-I" + os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "metis_adapter_smoke.cc"), "-o", exe, "-L" + LIBDIR,
           "-lkaminpar_b200", "-Wl,-rpath," + LIBDIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_metis_adapter_compiles_links_and_has_no_fallback(tmp_path):
    import torch

    exe = build(tmp_path)
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 1 and "no CUDA device" in r.stdout


@pytest.mark.gpu
def test_metis_adapter_matches_oracle_on_gpu(tmp_path):
    exe = build(tmp_path)
    paths = []
    for i, data in enumerate(FILES):
        p = tmp_path / f"f{i}.metis"
        p.write_bytes(data)
        paths.append(str(p))
    dump = str(tmp_path / "dump.txt")
    r = subprocess.run([exe] + paths, capture_output=True, text=True, timeout=120,
                       env=dict(os.environ, ADAPTER_DUMP=dump))
    assert r.returncode == 0, r.stdout + r.stderr
    assert "adapter ok" in r.stdout
    lines = open(dump).read().split("\n")
    at = 0
    for data in FILES:
        exp = MO.parse(data)
        assert int(lines[at]) == exp["kind"]
        if exp["kind"] == 0:
            got = [np.array(lines[at + 1 + j].split(), np.int64) for j in range(4)]
            for a, f in zip(got, ("xadj", "adjncy", "vwgt", "adjwgt")):
                want = np.zeros(0, np.int64) if exp[f] is None else np.asarray(exp[f], np.int64)
                assert np.array_equal(a, want), f
            assert lines[at + 5] == ("ignorning extra lines in input file" if exp["extra_lines"] else "")
            at += 6
        else:
            rep = MO.report_of(exp)
            assert lines[at + 1] == "self-loop at byte %d (line %d, vertex %d)" % (rep["offset"], rep["line"],
                                                                                   rep["vertex"])
            at += 2
