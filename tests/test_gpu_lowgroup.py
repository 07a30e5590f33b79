"""Clustering on one GPU runs degree groups 0 (tier 0) and 1 (tiers 1-2) as one persistent launch per group and
LP round (lp_lowgroup.cuh). On inputs with all four degree groups the result, the per-round move counts and the
scan counters must be the oracle's `sync` schedule, bit for bit, and the launches must be one per group and round."""
import pytest

from tests import helpers as H
from tests.test_gpu_edges import UINT32_MAX, ctx_for, ladder, run_cluster

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["wide_unit", "dense_w"])
def test_low_groups_run_one_launch_per_round(name):
    g = ladder(name)
    present = H.tiers_present(g, UINT32_MAX)
    assert {0, 1, 2, 3} <= set(present) and max(present) >= 4, present  # every degree group has vertices
    _, mcw = ctx_for(g, 8)
    for seed in (0, 5):
        gs = run_cluster(g, seed, mcw)  # labels, moves per round and scan counters against the oracle
        rounds = gs.iterations
        assert rounds > 0
        assert gs.group_launches[0] == rounds and gs.group_launches[1] == rounds, list(gs.group_launches)
        assert gs.group_launches[2] == 0, list(gs.group_launches)  # tier 2 runs inside group 1's launch
        assert gs.group_nodes[1] > 0 and gs.group_nodes[2] > 0  # ... and keeps its own scan counters
