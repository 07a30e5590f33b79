"""The oracle's call index (CPU only): the sync schedule keys every tie, favored-cluster and commit hash on the
number of clusterings the device handle computed before, on any graph. One handle reused across the levels of a
hierarchy therefore runs level L with call index L, and `oracle_lp_cluster(call_index=L)` /
`oracle_lp_refine(call_index=c)` state exactly that (DESIGN.md, "parity across levels and calls").

The digests in golden/oracle_sync_digests.json were recorded with the oracle as it was before it took a call
index; `python -m tests.test_oracle_call_index` prints them for the oracle in the tree.
"""
import hashlib
import json
import os

import numpy as np
import pytest

from kaminpar_b200.graph import random_weights, rmat
from oracle import bindings as B
from tests import helpers as H

GOLDEN_CASES = ("rgg2d_k4", "walshaw_k16", "grid12", "road60", "rmat13_w")
NAMES = GOLDEN_CASES + ("rmat14_hubs", "rmat12_hubs_w")
DIGESTS = os.path.join(H.GOLDEN, "oracle_sync_digests.json")
SEED, K = 3, 8


def graph(name):
    if name == "rmat14_hubs":  # degree-sorted, hubs of degree > 4096
        return B.oracle_rearrange(rmat(14, 32, 5))[0]
    if name == "rmat12_hubs_w":  # vertex and edge weights
        return random_weights(B.oracle_rearrange(rmat(12, 48, 11))[0], 5, max_vwgt=3, max_adjwgt=5)
    return H.load_case(name)[0]


def _digest(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes() if isinstance(a, np.ndarray) else bytes(a))
    return h.hexdigest()


def _refine_input(g, k):
    return np.random.default_rng(k).integers(0, k, g.n).astype(np.uint32)


def sync_digests(**kw):
    """sha256 of the sync schedule's labels and stats per graph: two clustering calls, refinements at k = 4, 64."""
    out = {}
    rp = B.oracle_params(B.default_refine_params(), commit_passes=4)
    for name in NAMES:
        g = graph(name)
        mcw = B.oracle_max_cluster_weight(g, K)
        c, st = B.oracle_lp_cluster(g, SEED, mcw, schedule=B.SYNC, num_calls=2, return_stats=True, **kw)
        out[f"{name}/cluster"] = _digest(c, st)
        for k in (4, 64):
            p, bw, rst = B.oracle_lp_refine(g, SEED, k, B.oracle_max_block_weights(g, k), _refine_input(g, k),
                                            schedule=B.SYNC, params=rp, return_stats=True, **kw)
            out[f"{name}/refine{k}"] = _digest(p, bw, rst)
    return out


def test_call_index_zero_is_unchanged():
    with open(DIGESTS) as f:
        want = json.load(f)
    assert sync_digests(call_index=0) == want


@pytest.mark.parametrize("name", NAMES)
def test_call_index_equals_a_later_call_of_a_replay(name):
    g = graph(name)
    mcw = B.oracle_max_cluster_weight(g, K)
    replay, rst = B.oracle_lp_cluster(g, SEED, mcw, schedule=B.SYNC, num_calls=4, return_stats=True)
    for c in (1, 3):
        one, st = B.oracle_lp_cluster(g, SEED, mcw, schedule=B.SYNC, call_index=c, return_stats=True)
        assert np.array_equal(one, replay[c])
        assert bytes(st[0]) == bytes(rst[c])
    # several calls from a start index: calls c, c + 1, ...
    two, st2 = B.oracle_lp_cluster(g, SEED, mcw, schedule=B.SYNC, call_index=2, num_calls=2, return_stats=True)
    assert np.array_equal(two, replay[2:4])
    assert [bytes(s) for s in st2] == [bytes(s) for s in rst[2:4]]


def test_call_index_reaches_every_hash():
    """A refinement or clustering with another call index is another run: at least the move counts differ on
    most inputs (the index is not dropped on the way to the hash keys)."""
    rp = B.oracle_params(B.default_refine_params(), commit_passes=4)
    differ_c = differ_r = 0
    for name in NAMES:
        g = graph(name)
        mcw = B.oracle_max_cluster_weight(g, K)
        a = B.oracle_lp_cluster(g, SEED, mcw, schedule=B.SYNC)
        b = B.oracle_lp_cluster(g, SEED, mcw, schedule=B.SYNC, call_index=5)
        differ_c += not np.array_equal(a, b)
        part = _refine_input(g, 64)
        mbw = B.oracle_max_block_weights(g, 64)
        p0, _ = B.oracle_lp_refine(g, SEED, 64, mbw, part, schedule=B.SYNC, params=rp)
        p1, _ = B.oracle_lp_refine(g, SEED, 64, mbw, part, schedule=B.SYNC, params=rp, call_index=5)
        differ_r += not np.array_equal(p0, p1)
    assert differ_c >= len(NAMES) - 1 and differ_r >= len(NAMES) - 1


def test_refine_call_index_zero_is_the_default():
    g = graph("walshaw_k16")
    rp = B.oracle_params(B.default_refine_params(), commit_passes=4)
    part = _refine_input(g, 16)
    mbw = B.oracle_max_block_weights(g, 16)
    a = B.oracle_lp_refine(g, SEED, 16, mbw, part, schedule=B.SYNC, params=rp, return_stats=True)
    b = B.oracle_lp_refine(g, SEED, 16, mbw, part, schedule=B.SYNC, params=rp, return_stats=True, call_index=0)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and bytes(a[2]) == bytes(b[2])


def test_seq_schedule_takes_no_call_index():
    g = graph("grid12")
    with pytest.raises(ValueError):
        B.oracle_lp_cluster(g, SEED, 10, schedule=B.SEQ, call_index=1)
    with pytest.raises(ValueError):
        B.oracle_lp_refine(g, SEED, 4, B.oracle_max_block_weights(g, 4), _refine_input(g, 4), call_index=1)


if __name__ == "__main__":
    print(json.dumps(sync_digests(), indent=1, sort_keys=True))
