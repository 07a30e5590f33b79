"""CPU check of the resources the clusterer's hub kernels were compiled to (cuobjdump -res-usage of the built
library): sweep_hub_rate runs one 1024-thread CTA per SM with a 128 KiB table in dynamic shared memory, and
sweep_hub_gather is launched with 8 CTAs of 256 threads per SM. Neither may spill to local memory, and each must
still fit the CTAs per SM its grid assumes on an H100."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "kaminpar_b200", "csrc", "libkaminpar_b200.so")

# H100 (sm_90) per-SM limits
REGS_PER_SM = 65536
REG_ALLOC_UNIT = 256  # registers are allocated per warp in units of 256
SMEM_PER_SM = 228 * 1024
SMEM_RESERVED_PER_CTA = 1024
THREADS_PER_SM = 2048

# kept in step with lp_sweep.cuh (kRateSlots, kRateListCap, kRateStage, kRateThreads) and the launches in kmp_lp.cu
RATE_THREADS = 1024
RATE_SLOTS = 16384
RATE_LIST_CAP = RATE_SLOTS // 2
RATE_STAGE = 64


def rate_dynamic_smem(ew):
    return RATE_SLOTS * 8 + RATE_LIST_CAP * 2 + (RATE_THREADS // 32) * RATE_STAGE * (8 if ew else 4)


# kernel -> (threads per CTA, CTAs per SM the grid is sized for, dynamic shared memory of the launch)
NAMES = {
    re.compile(r"_ZN3kmp14sweep_hub_rateILb([01])EEEvNS_9SweepArgsENS_7HubArgsE"):
        lambda ew: ("rate", ew, RATE_THREADS, 1, rate_dynamic_smem(ew)),
    re.compile(r"_ZN3kmp16sweep_hub_gatherILb([01])EEEvNS_9SweepArgsENS_7HubArgsE"):
        lambda p64: ("gather", p64, 256, 8, 0),
}


def cuobjdump():
    for cand in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump"),
                 shutil.which("cuobjdump")):
        if cand and os.path.exists(cand):
            return cand
    pytest.skip("cuobjdump (CUDA toolkit) not found")


def hub_kernels():
    out = subprocess.run([cuobjdump(), "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    kernels = {}
    spec = None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            spec = None
            for pat, make in NAMES.items():
                mm = pat.fullmatch(m.group(1))
                if mm:
                    spec = make(int(mm.group(1)))
            continue
        if spec is not None and "REG:" in line:
            res = {k: int(v) for k, v in re.findall(r"([A-Z]+(?:\[\d\])?):(\d+)", line)}
            kernels[spec] = res
            spec = None
    return kernels


def resident_ctas(regs, static_smem, threads, dynamic_smem):
    warps = threads // 32
    per_warp = -(-regs * 32 // REG_ALLOC_UNIT) * REG_ALLOC_UNIT
    by_regs = (REGS_PER_SM // per_warp) // warps
    by_smem = SMEM_PER_SM // (static_smem + dynamic_smem + SMEM_RESERVED_PER_CTA)
    return min(by_regs, by_smem, THREADS_PER_SM // threads, 32)


def test_hub_kernels_fit_their_residency():
    kernels = hub_kernels()
    # rate: edge weights or not; gather: 4- or 8-byte gather word
    assert sorted((k[0], k[1]) for k in kernels) == [("gather", 0), ("gather", 1), ("rate", 0), ("rate", 1)], \
        sorted(kernels)
    for (name, flag, threads, per_sm, dyn), res in sorted(kernels.items()):
        label = f"sweep_hub_{name}<{flag}>"
        got = resident_ctas(res["REG"], res["SHARED"], threads, dyn)
        assert got >= per_sm, f"{label}: {res['REG']} registers, {res['SHARED']} B static + {dyn} B dynamic shared " \
                              f"memory allow {got} CTAs per SM, the grid is sized for {per_sm}"
        assert res["STACK"] == 0 and res["LOCAL"] == 0, f"{label} spills: stack {res['STACK']} B, local {res['LOCAL']} B"


def test_clusterer_has_no_bucket_kernels():
    """The clusterer rates hubs with gather + rate only: no scatter / select instantiation for MODE 0."""
    out = subprocess.run([cuobjdump(), "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    names = re.findall(r"Function (\S+):", out)
    assert not [n for n in names if re.search(r"sweep_hub_(scatter|select)ILi0E", n)]
    assert [n for n in names if re.search(r"sweep_hub_(scatter|select)ILi1E", n)]  # the refiner keeps them


def test_residency_rule_matches_the_h100():
    # the rate table takes most of an SM: one 1024-thread CTA, however few registers it uses
    assert resident_ctas(32, 1552, 1024, rate_dynamic_smem(True)) == 1
    assert resident_ctas(56, 1552, 1024, rate_dynamic_smem(False)) == 1
    # 65 registers would not fit one 1024-thread CTA at all
    assert resident_ctas(65, 1552, 1024, rate_dynamic_smem(False)) == 0
    assert resident_ctas(32, 1024, 256, 0) == 8
