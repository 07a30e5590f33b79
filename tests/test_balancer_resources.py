"""CPU check of the overload and underload balancers' kernels (kmp_balance.cuh, kmp_underload.cuh) in the built library
(cuobjdump -res-usage): none of them spills to local memory or uses a stack frame, and the shared tables of the
evaluation tiers and every underload kernel fit the 48 KiB of static shared memory."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "kaminpar_b200", "csrc", "libkaminpar_b200.so")
OVERLOAD = ("bal_eval_thread", "bal_eval_warp", "bal_eval_cta", "bal_block_weights", "bal_block_stats",
            "bal_vertex_flags", "bal_iota", "bal_sorted_weights", "bal_propose")
UNDERLOAD = ("ubal_block_stats", "ubal_vertex_flags", "ubal_sort_keys", "ubal_propose", "ubal_keep_sources")
KERNELS = OVERLOAD + UNDERLOAD


def _usage():
    tool = next((c for c in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump"),
                             shutil.which("cuobjdump")) if c and os.path.exists(c)), None)
    if tool is None:
        pytest.skip("cuobjdump (CUDA toolkit) not found")
    out = subprocess.run([tool, "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    res, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        if name and "REG:" in line:
            for k in KERNELS:
                if re.fullmatch(r"_ZN3kmp%d%sE.*" % (len(k), k), name):
                    res[k] = {a: int(b) for a, b in re.findall(r"([A-Z]+(?:\[\d\])?):(\d+)", line)}
            name = None
    return res


def test_balancer_kernels_do_not_spill():
    res = _usage()
    assert sorted(res) == sorted(KERNELS)
    for k, r in res.items():
        assert r["LOCAL"] == 0 and r["STACK"] == 0, (k, r)
    for k in ("bal_eval_warp", "bal_eval_cta") + UNDERLOAD:
        assert res[k]["SHARED"] <= 48 * 1024 + 1024, k
