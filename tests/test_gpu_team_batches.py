"""Parity where the team sweep kernels batch their work claims and proposals (-m gpu).

A tier-3 team (one warp per vertex, degrees 32..255) claims TIER3_CLAIM_BATCH consecutive entries of its work list
with one queue atomic, and holds up to 32 proposals before one atomic reserves their slots; the rest go out when
the queue runs dry. The cases put the tier's list at the sizes where a batch is cut
short by the list end, leave teams without any vertex, cap the grid at one CTA so that each warp holds more than 32
proposals, and run sub-rounds in which no vertex or every vertex proposes. All of it is integer work: the GPU must
equal the oracle's `sync` schedule bit for bit (labels, block weights, moves per round, edges scanned).
"""
import functools

import numpy as np
import pytest

from tests import helpers as H
from tests.test_gpu_edges import ctx_for, run_cluster
from tests.test_gpu_waves import TEAMS_PER_CTA, largest_lists, refine_case

pytestmark = pytest.mark.gpu

SEED = 3
TIER3_CLAIM_BATCH = 2  # lp_sweep.cuh, team_claim_batch<32>
STAGED = 32            # proposals a tier-3 warp holds before it reserves their slots


@functools.lru_cache(maxsize=None)
def centres(count, weighted, pool):
    """`count` tier-3 centres of degrees spread over 32..255, neighbours drawn from `pool` vertices of low degree"""
    degs = sorted(32 + (37 * i) % 224 for i in range(count))
    g = H.degree_ladder(degs, pool, weighted=weighted, seed=count)
    tiers = np.array([H.tier_of(int(d), weighted) for d in g.degrees()])
    assert int((tiers == 3).sum()) == count and tiers.max() == 3
    return g


def check(g, S, mcw=None, k=4):
    """clustering and refinement against the oracle, S sub-rounds; returns the clustering's stats"""
    _, default_mcw = ctx_for(g, 8)
    gs = run_cluster(g, SEED, default_mcw if mcw is None else mcw, subrounds=S)
    assert gs.group_nodes[3] > 0
    ctx, _ = ctx_for(g, k)
    part = np.random.default_rng(k).integers(0, k, g.n).astype(np.uint32)
    refine_case(g, SEED, k, part, ctx.partition.max_block_weights(), subrounds=S)
    return gs


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("count", sorted({1, TIER3_CLAIM_BATCH - 1, TIER3_CLAIM_BATCH, TIER3_CLAIM_BATCH + 1,
                                          2 * TIER3_CLAIM_BATCH + 1}))
def test_tier3_list_at_the_claim_batch(count, weighted):
    """One sub-round: the tier-3 list holds exactly `count` vertices, one CTA of 8 teams takes them, and the list
    ends before, at or just after a batch boundary (more teams than vertices in every case)."""
    g = centres(count, weighted, 600)
    assert largest_lists(g, SEED, 1, 4)[3] == count
    check(g, 1)


@pytest.mark.parametrize("weighted", [False, True])
def test_more_teams_than_batches(weighted):
    """100 tier-3 vertices in one list: 13 CTAs of 8 teams and fewer batches than teams, so some teams claim only
    past the end"""
    g = centres(100, weighted, 4000)
    n3 = largest_lists(g, SEED, 1, 4)[3]
    assert n3 == 100 and -(-n3 // TEAMS_PER_CTA[3]) * TEAMS_PER_CTA[3] > -(-n3 // TIER3_CLAIM_BATCH)
    check(g, 1)


@pytest.mark.parametrize("weighted", [False, True])
def test_grid_capped_at_one_cta(weighted, monkeypatch):
    """KMP_GRID_CAP=1: 8 warps take 600 tier-3 vertices, about 75 each; in round 0 every vertex proposes (no
    neighbour carries its singleton label, and the cluster weight limit admits any first merge), so each warp
    reserves slots for 32 staged proposals twice before the queue runs dry."""
    monkeypatch.setenv("KMP_GRID_CAP", "1")
    g = centres(600, weighted, 20000)
    assert largest_lists(g, SEED, 1, 4)[3] > 2 * STAGED * TEAMS_PER_CTA[3]
    gs = check(g, 1, mcw=1 << 20)
    assert gs.moved_list()[0] > 0


@pytest.mark.parametrize("weighted", [False, True])
def test_no_vertex_proposes(weighted):
    """A cluster weight limit below every merge: no vertex proposes in any sub-round, nothing moves"""
    g = centres(40, weighted, 2000)
    gs = run_cluster(g, SEED, 1, subrounds=2)
    assert gs.group_nodes[3] > 0 and not any(gs.moved_list())
