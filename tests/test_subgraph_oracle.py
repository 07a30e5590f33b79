"""CPU checks of the subgraph oracle (tests/subgraph_oracle.py): the reference-shaped loops, the vectorised version
the GPU tests use at large sizes and the non-lazy extraction agree, the blocks are the induced subgraphs, and
compute_final_k / copy-back keep the reference's invariants."""
import os

import numpy as np
import pytest

from kaminpar_b200.graph import CSRGraph, random_weights, rgg2d, rmat
from tests import helpers as H
from tests import subgraph_oracle as S


def cases():
    yield "walshaw_k7", H.load_graph("walshaw_data"), 7, "random"
    yield "rgg16_w_k64", H.load_graph("rgg16_vwgt_adjwgt"), 64, "contiguous"
    yield "rmat12_w_k3", random_weights(rmat(12, 8, seed=4), 2, max_vwgt=5, max_adjwgt=9), 3, "random"
    yield "rgg2d_k1", H.load_graph("rgg2d"), 1, "random"
    yield "empty_blocks", H.path_graph(50), 16, "sparse"
    yield "one_block", rgg2d(2000, seed=3), 8, "one"
    yield "isolated", H.empty_graph(40), 5, "random"
    yield "k_gt_n", H.path_graph(10), 37, "random"
    yield "path_cut", H.path_graph(101), 2, "halves"
    yield "n0", H.empty_graph(0), 3, "random"


def make_part(n, k, how, seed=0):
    rng = np.random.default_rng(seed)
    if how == "random":
        return rng.integers(0, k, n).astype(np.uint32)
    if how == "contiguous" or how == "halves":
        return (np.arange(n, dtype=np.int64) * k // max(n, 1)).astype(np.uint32)
    if how == "sparse":  # every other block empty
        return (2 * rng.integers(0, k // 2, n)).astype(np.uint32)
    return np.full(n, k - 1, np.uint32)


CASES = list(cases())


@pytest.mark.parametrize("name,g,k,how", CASES, ids=[c[0] for c in CASES])
def test_oracles_agree_and_blocks_are_induced_subgraphs(name, g, k, how):
    part = make_part(g.n, k, how)
    a = S.lazy_extract(g.xadj, g.adjncy, g.vwgt, g.adjwgt, part, k)
    b = S.lazy_extract_np(g.xadj, g.adjncy, g.vwgt, g.adjwgt, part, k)
    for key in a:
        assert (a[key] is None) == (b[key] is None), key
        if a[key] is not None:
            assert np.array_equal(a[key], b[key]), key
    blocks, mapping = S.extract_nonlazy(g.xadj, g.adjncy, g.vwgt, g.adjwgt, part, k)
    assert np.array_equal(mapping, a["mapping"])
    assert len(a["xadj"]) == g.n + k
    src = np.repeat(np.arange(g.n), np.diff(g.xadj.astype(np.int64)))
    internal = part[g.adjncy] == part[src] if g.m else np.zeros(0, bool)
    assert a["edge_off"][-1] == int(internal.sum())
    for blk in range(k):
        x, adj, vw, ew = S.block_of(a, blk)
        want = blocks[blk]
        assert np.array_equal(x, want["xadj"]) and np.array_equal(adj, want["adjncy"])
        for got, exp in ((vw, want["vwgt"]), (ew, want["adjwgt"])):
            assert (got is None) == (exp is None)
            if exp is not None:
                assert np.array_equal(got, exp)
        members = a["block_nodes"][a["node_off"][blk]:a["node_off"][blk + 1]]
        assert np.all(part[members] == blk) and np.all(np.diff(members.astype(np.int64)) > 0)
        assert x[0] == 0 and len(x) == len(members) + 1


def test_compute_final_k_sums_to_input_k_on_every_power_of_two_level():
    for input_k in list(range(2, 80)) + [1000, 1023, 1025, 4096, 9999, 10000]:
        current = 1
        while current <= input_k and current <= 4096:
            ks = [S.compute_final_k(b, current, input_k) for b in range(current)]
            assert sum(ks) == input_k, (input_k, current)
            assert max(ks) - min(ks) <= 1
            current *= 2
        assert S.compute_final_k(5, input_k, input_k) == 1


def test_copy_back_matches_a_direct_restatement():
    g = random_weights(rmat(11, 8, seed=2), 1, max_vwgt=4)
    k = 8
    part = make_part(g.n, k, "random", 3)
    a = S.lazy_extract_np(g.xadj, g.adjncy, g.vwgt, g.adjwgt, part, k)
    rng = np.random.default_rng(1)
    for k_prime, input_k in ((16, 100), (11, 11), (37, 37), (8, 8)):
        k0 = S.sub_block_offsets(k, k_prime, input_k)
        counts = k0[1:] - k0[:-1]
        sub = np.zeros(g.n, np.uint32)
        for b in range(k):
            lo, hi = a["node_off"][b], a["node_off"][b + 1]
            sub[lo:hi] = rng.integers(0, counts[b], hi - lo)
        out, bw = S.copy_back(part, a["mapping"], a["node_off"], sub, k, k_prime, input_k, g.vwgt)
        for u in range(0, g.n, 7):
            b = part[u]
            assert out[u] == k0[b] + sub[a["node_off"][b] + a["mapping"][u]]
        assert bw.sum() == g.vwgt.sum() and len(bw) == k_prime


# ---- pinned outputs of the unmodified reference (tests/golden/make_subgraph_golden.py) ---------------------------
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLDENS = sorted(f[len("subgraph_"):-4] for f in os.listdir(GOLDEN_DIR)
                 if f.startswith("subgraph_") and f.endswith(".npz") and f != "subgraph_final_k.npz")


def load_subgraph_golden(name):
    d = np.load(os.path.join(GOLDEN_DIR, f"subgraph_{name}.npz"))
    g = CSRGraph(d["xadj"], d["adjncy"], d["vwgt"] if "vwgt" in d else None, d["adjwgt"] if "adjwgt" in d else None)
    return g, int(d["k"][0]), d["partition"], d


@pytest.mark.parametrize("name", GOLDENS)
def test_oracle_equals_pinned_reference_outputs(name):
    g, k, part, d = load_subgraph_golden(name)
    for res in (S.lazy_extract(g.xadj, g.adjncy, g.vwgt, g.adjwgt, part, k),
                S.lazy_extract_np(g.xadj, g.adjncy, g.vwgt, g.adjwgt, part, k)):
        for key in ("node_off", "edge_off", "block_nodes", "mapping", "xadj", "adjncy", "vwgt", "adjwgt"):
            assert (res[key] is None) == (("ref_" + key) not in d), key
            if res[key] is not None:
                assert np.array_equal(res[key], d["ref_" + key]), key
    for i in range(2):
        k_prime, input_k = (int(x) for x in d[f"copy{i}_args"])
        out, _ = S.copy_back(part, d["ref_mapping"], d["ref_node_off"], d[f"copy{i}_sub"], k, k_prime, input_k)
        assert np.array_equal(out, d[f"copy{i}_out"])


def test_compute_final_k_equals_pinned_reference_outputs():
    d = np.load(os.path.join(GOLDEN_DIR, "subgraph_final_k.npz"))
    assert len(d.files) == 5
    for key in d.files:
        input_k = int(key.split("_")[-1])
        got = [S.compute_final_k(b, 1 << level, input_k) for level in range(13) for b in range(1 << level)]
        assert got == d[key].tolist(), input_k
