"""CPU check of the resources the persistent low-degree clustering kernels (sweep_commit_low, lp_lowgroup.cuh)
were compiled to: each instantiation keeps the CTAs per SM recorded below on an H100 and does not spill. The grid
of a cooperative launch is the co-resident CTA count, so a register count that creeps up shrinks every sub-round's
wave of threads and makes each of its grid barriers wait on fewer, longer CTAs."""
import re
import subprocess

from tests.test_team_resources import LIB, cuobjdump, resident_ctas

NAME = re.compile(r"_ZN3kmp16sweep_commit_lowILb([01])ELb([01])ELi(\d+)ELi(\d+)ELi(\d+)EEEvNS_9SweepArgsENS_10CommitArgs"
                  r"ENS_12LowGroupArgsENS_11GridBarrierE")

# (edge weights, tier A's sort width) -> CTAs of 256 threads per SM (CUDA 12.9, sm_90a): group 0 (N = 8) at
# 40 / 58 registers, group 1 (N = 16 and 32 in one kernel) at 78-80 / 118
CTAS_PER_SM = {(0, 8): 6, (1, 8): 4, (0, 16): 3, (1, 16): 2}


def low_kernels():
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
            kernels[tuple(int(x) for x in m.groups())] = {k: int(v) for k, v in res.items()}
            name = None
    return kernels


def test_low_group_kernels_fit_their_residency():
    kernels = low_kernels()
    # edge weights x gather word x 2 degree groups
    assert sorted(kernels) == sorted((ew, p64, na, nb, lanes) for ew in (0, 1) for p64 in (0, 1)
                                     for na, nb, lanes in ((8, 8, 4), (16, 32, 8))), sorted(kernels)
    for (ew, p64, na, nb, lanes), res in sorted(kernels.items()):
        label = f"sweep_commit_low<{ew},{p64},{na},{nb},{lanes}>"
        got = resident_ctas(res["REG"], res["SHARED"], 256, 0, 1, 0)
        assert got >= CTAS_PER_SM[(ew, na)], f"{label}: {res['REG']} registers allow {got} CTAs per SM, " \
                                             f"recorded {CTAS_PER_SM[(ew, na)]}"
        assert res["STACK"] == 0 and res["LOCAL"] == 0, f"{label} spills: stack {res['STACK']} B, local {res['LOCAL']} B"
