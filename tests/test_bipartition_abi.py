"""CPU: the block-bipartitioning ABI (include/kaminpar_b200_bipartition.h) compiles as C, the ctypes mirror and the
host twin agree on the default configuration, the host twin's arena re-run gives the same result, and the device
engine's PTX holds no fused multiply-add: every double of the engine is an explicitly rounded add, sub, mul, div or
sqrt. (Its SASS does hold DFMA: ptxas expands the correctly rounded div.rn.f64 and sqrt.rn.f64 into DFMA-based
sequences, whose results are exact IEEE quotients and roots.)"""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from kaminpar_b200.bipartition import IPConfig
from kaminpar_b200.graph import rgg2d
from tests import ip_host as IH
from tests import subgraph_oracle as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def test_header_compiles_as_c(tmp_path):
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "t.c"
    src.write_text('#include "kaminpar_b200_bipartition.h"\nint main(void) { kmp_ip_config c; kmp_bipartition_stats s;'
                   ' (void)c; (void)s; return 0; }\n')
    r = subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), "-c", str(src),
                        "-o", str(tmp_path / "t.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_default_config_matches_host_twin():
    assert bytes(IPConfig()) == bytes(IH.lib().ip_default_config())


def test_arena_rerun_same_result():
    g = rgg2d(3000, seed=4)
    res = S.lazy_extract(g.xadj, g.adjncy, None, None, np.zeros(g.n, np.uint32), 1)
    bx, ba, bv, be = IH.block_arrays(res, 0)
    cfg = IPConfig()
    params = IH.block_params(cfg, 2, IH.max_block_weights(g.n, 2), True, g.n, 0.03, 0, 1, bx, ba, bv, be)
    rc, want, _ = IH.bipartition_block(cfg, params, 5, bx, ba, bv, be)
    assert rc == 0
    size = 4096
    while True:
        rc, got, _ = IH.bipartition_block(cfg, params, 5, bx, ba, bv, be, arena_bytes=size)
        if rc == 0:
            break
        size *= 2
    assert size > 4096 and np.array_equal(got, want)


@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc is not present")
def test_engine_ptx_has_no_fma(tmp_path):
    src = tmp_path / "k.cu"
    src.write_text('#include "%s"\n__global__ void k(const kmp_ip::Config *c, const kmp_ip::BlockParams *bp, '
                   'const uint32_t *x, const uint32_t *a, uint8_t *arena, uint32_t *out, kmp_ip::Counters *cnt) {\n'
                   '  kmp_ip::bipartition_block(x[0], x[1], x + 2, a, nullptr, nullptr, *c, 1, *bp, 1, arena, 1 << 20,'
                   ' out, *cnt);\n}\n' % os.path.join(ROOT, "kaminpar_b200", "csrc", "kmp_bipartition.cuh"))
    ptx = tmp_path / "k.ptx"
    r = subprocess.run([NVCC, "-arch=compute_90a", "-O3", "-std=c++17", "-ptx", "-o", str(ptx), str(src)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    text = ptx.read_text()
    assert "div.rn.f64" in text and "sqrt.rn.f64" in text and "mul.rn.f64" in text  # the engine's doubles
    assert not re.search(r"\bfma\.[a-z.]*f64", text)


def test_ip_kernel_resources():
    """ip_kernel (one engine per warp, lane 0 sequential) keeps no local arrays; its 64-byte stack frame holds
    ptxas's spills of the inlined engine (DESIGN.md §20) and must not grow. ip_reduce neither spills nor uses a
    stack."""
    tool = next((c for c in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump"),
                             shutil.which("cuobjdump")) if c and os.path.exists(c)), None)
    lib = os.path.join(ROOT, "kaminpar_b200", "csrc", "libkaminpar_b200.so")
    if tool is None or not os.path.exists(lib):
        pytest.skip("cuobjdump or the built library not found")
    out = subprocess.run([tool, "-res-usage", lib], check=True, capture_output=True, text=True).stdout
    res, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        if name and "REG:" in line:
            k = re.search(r"\d+(ip_kernel|ip_reduce)E", name)
            if k:
                res[k.group(1)] = {a: int(b) for a, b in re.findall(r"([A-Z]+(?:\[\d\])?):(\d+)", line)}
            name = None
    assert sorted(res) == ["ip_kernel", "ip_reduce"]
    assert res["ip_reduce"]["STACK"] == 0 and res["ip_reduce"]["LOCAL"] == 0
    assert res["ip_kernel"]["LOCAL"] == 0 and res["ip_kernel"]["STACK"] <= 64, res["ip_kernel"]
