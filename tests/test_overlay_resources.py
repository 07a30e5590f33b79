"""CPU check of the overlay kernels (kmp_overlay.cuh) in the built library (cuobjdump -res-usage): none of them spills
to local memory or uses a stack frame."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "kaminpar_b200", "csrc", "libkaminpar_b200.so")
KERNELS = ("k_overlay_keys", "k_overlay_heads", "k_overlay_scatter", "k_flag_leaders")


def _usage():
    tool = next((c for c in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump"),
                             shutil.which("cuobjdump")) if c and os.path.exists(c)), None)
    if tool is None:
        pytest.skip("cuobjdump (CUDA toolkit) not found")
    out = subprocess.run([tool, "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    res, name = [], None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        if name and "REG:" in line:
            for k in KERNELS:
                if re.search(r"\d%d%sE" % (len(k), k), name):  # <length><name>E<parameters>, in any namespace
                    res.append((k, name, {a: int(b) for a, b in re.findall(r"([A-Z]+(?:\[\d\])?):(\d+)", line)}))
            name = None
    return res


def test_overlay_kernels_do_not_spill():
    res = _usage()
    assert sorted(k for k, _, _ in res) == sorted(KERNELS)  # one instantiation each
    for k, name, r in res:
        assert r["LOCAL"] == 0 and r["STACK"] == 0, (name, r)
        assert r["SHARED"] <= 48 * 1024, (name, r)
