"""CPU: the validation oracle (tests/validate_oracle.py) against the UNMODIFIED reference's verdicts recorded in
tests/golden/validate_cases.npz (tests/golden/make_validate_golden.py), so that the parity of
tests/test_validate_bridge.py holds where the reference is absent: debug::validate_graph's verdict and warning line,
and validate_undirected_graph's exit status in its domain. The loop and vectorised forms of the oracle agree."""
import os

import numpy as np
import pytest

from tests import test_validate_bridge as TB
from tests import validate_oracle as V

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "validate_cases.npz"))
CASES = TB.CASES


def test_corpus_is_the_recorded_one():
    assert [c[0] for c in CASES] == list(GOLD["names"])
    assert [TB.digest(*c[1:]) for c in CASES] == list(GOLD["digests"])


@pytest.mark.parametrize("i", range(len(CASES)), ids=[c[0] for c in CASES])
def test_oracle_equals_recorded_reference(i):
    _, xadj, adj, w = CASES[i]
    r = V.validate(xadj, adj, w)
    assert V.as_dict(V.validate_loop(xadj, adj, w)) == V.as_dict(r)
    if GOLD["ref_valid"][i] >= 0:
        assert r["valid"] == GOLD["ref_valid"][i]
        assert V.message(r) == str(GOLD["ref_message"][i])
    else:
        assert not TB.shape_ok(xadj, adj) and r["kind"] in (V.XADJ_START, V.XADJ_END)
    if GOLD["ref_undirected"][i] >= 0:
        assert GOLD["ref_undirected"][i] == (0 if r["valid"] and r["duplicates"] == 0 else 1)


def test_every_kind_is_covered():
    kinds = {V.validate(*c[1:])["kind"] for c in CASES}
    assert kinds == set(range(V.NUM_KINDS))
    assert sum(GOLD["ref_undirected"] >= 0) >= 10 and sum(GOLD["ref_undirected"] == 1) >= 1
