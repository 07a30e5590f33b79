"""CPU check of the resources the sweep_team kernels were compiled to (cuobjdump -res-usage of the built library):
every instantiation still fits the CTAs per SM its launch is built for (team_ctas_per_sm in lp_sweep.cuh) on
an H100, and none of them spills to local memory. A register count that creeps past the budget
would otherwise silently cost a third of the teams of tiers 4 and 5."""
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

# team size T -> CTAs per SM the launch is built for; keep in step with team_ctas_per_sm
CTAS_PER_SM = {32: 6, 128: 3, 512: 3, 1024: 1}

NAME = re.compile(r"_ZN3kmp10sweep_teamILi(\d)ELb([01])ELb([01])ELi(\d+)ELi(\d+)ELi(\d+)ELb([01])EEEvNS_9SweepArgsE")


def cuobjdump():
    for cand in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump"),
                 shutil.which("cuobjdump")):
        if cand and os.path.exists(cand):
            return cand
    pytest.skip("cuobjdump (CUDA toolkit) not found")


def team_kernels():
    out = subprocess.run([cuobjdump(), "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    kernels = {}
    name = None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = NAME.fullmatch(name or "")
        if m and "REG:" in line:
            res = dict(re.findall(r"([A-Z]+(?:\[\d\])?):(\d+)", line))
            mode, ew, p64, t, slots, teams, v16 = (int(x) for x in m.groups())
            kernels[(mode, ew, p64, t, slots, teams, v16)] = {k: int(v) for k, v in res.items()}
            name = None
    return kernels


def resident_ctas(regs, static_smem, t, slots, teams, v16):
    threads = t * teams
    warps = threads // 32
    per_warp = -(-regs * 32 // REG_ALLOC_UNIT) * REG_ALLOC_UNIT
    by_regs = (REGS_PER_SM // per_warp) // warps
    smem = static_smem + slots * teams * (6 if v16 else 8) + SMEM_RESERVED_PER_CTA
    by_smem = SMEM_PER_SM // smem
    return min(by_regs, by_smem, THREADS_PER_SM // threads, 32)


def test_team_kernels_fit_their_residency():
    kernels = team_kernels()
    # 2 modes x edge weights x gather word x 4 team sizes
    assert len(kernels) == 32, sorted(kernels)
    for (mode, ew, p64, t, slots, teams, v16), res in sorted(kernels.items()):
        label = f"sweep_team<{mode},{ew},{p64},{t},{slots},{teams},{v16}>"
        got = resident_ctas(res["REG"], res["SHARED"], t, slots, teams, v16)
        assert got >= CTAS_PER_SM[t], f"{label}: {res['REG']} registers, {res['SHARED']} B static shared memory " \
                                      f"allow {got} CTAs per SM, the launch is built for {CTAS_PER_SM[t]}"
        assert res["STACK"] == 0 and res["LOCAL"] == 0, f"{label} spills: stack {res['STACK']} B, local {res['LOCAL']} B"


def test_residency_rule_matches_the_h100():
    # 40 registers: 3 CTAs of 512 threads; 54 (the count without the launch bounds' minimum) only 2; tier 3's
    # table allows 6 CTAs of 256 threads, not 7, however few registers it uses
    assert resident_ctas(40, 1360, 128, 2048, 4, 0) == 3
    assert resident_ctas(54, 1360, 128, 2048, 4, 0) == 2
    assert resident_ctas(40, 1184, 32, 512, 8, 0) == 6
    assert resident_ctas(32, 1184, 32, 512, 8, 0) == 6
    assert resident_ctas(64, 1568, 1024, 32768, 1, 1) == 1
