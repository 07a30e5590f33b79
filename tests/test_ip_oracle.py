"""CPU: the host twin of the device initial bipartitioner (tests/ip_host.py) reproduces the reference's pinned
sub-partitions tests/golden/ip_*.npz (tests/golden/make_ip_golden.py) on every case: blocks of misc/rgg2d, walshaw,
R-MAT 13, rgg16 with node and edge weights, a star, 40 components (more than the seed search's 5 attempts), blocks
with n <= 20, n = 1 and n = 2, one vertex heavier than the limit; the presets default, fast, largek, largek-fast and
adaptive FM; uniform and non-uniform block weights; input_k not a power of two and k' = input_k with mixed s_b."""
import numpy as np
import pytest

from kaminpar_b200.bipartition import IPConfig
from tests import ip_golden as G
from tests import ip_host as IH

CASES = [c for f in G.files() for c in G.cases(f)]


def test_goldens_present():
    assert len(CASES) >= 40


def test_recorded_defaults_are_the_config_defaults():
    assert bytes(G.recorded_defaults()) == bytes(IPConfig())


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_host_twin_equals_golden(case):
    _, g, part, k, k_prime, input_k, uniform, eps, seed, mbw, cfg, sub = case
    got = IH.expected_sub_partitions(g, part, k, k_prime, input_k, mbw, seed, cfg, uniform, eps)
    assert np.array_equal(got, sub)
