"""CPU: the host twin of the device initial bipartitioner (tests/cpp/ip_host_check.cc: kmp_bipartition.cuh and
kmp_ip_params.h under g++) against the UNMODIFIED reference, called through tests/cpp/ref_ip_bridge.cc (compiled here
against the reference headers, linked against oracle/_ref/libkaminpar_ref_full.so; skipped where either is absent).

  - sub-partitions: Random::reseed(seed_b) and a fresh InitialBipartitionerWorkerPool(ctx).bipartition(block, b, k)
    against the engine, block for block, on id-range and random partitions of R-MAT, rgg, a grid, weighted R-MAT, a
    star, many components, blocks with n <= 20, n = 1, n = 2 and one vertex heavier than the limit; the presets
    default, fast, largek, largek-fast and adaptive FM; uniform and non-uniform block weights; input_k not a power
    of two;
  - k is a power of two, as in the reference's extension loop: for other k, create_twoway_context's sub-block
    ranges can run past the input's block weights in the reference itself;
  - parameters: create_twoway_context's max and perfectly balanced block weights and compute_max_cluster_weight
    and the pool's clamped repetition count against kmp_ip_params.h over a grid of (k, input_k, epsilon, uniform or
    not, adaptive epsilon, cluster weight limit, repetition multiplier)."""
import ctypes as C
import os

import numpy as np
import pytest

from kaminpar_b200.bipartition import IPConfig, TWOWAY_ADAPTIVE_FM, preset
from kaminpar_b200.graph import CSRGraph, grid3d, random_weights, rgg2d, rmat
from tests import ip_host as IH
from tests import subgraph_oracle as S
from tests.test_subgraph_bridge import reference_present


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    if not reference_present():
        pytest.skip("the reference sources / oracle/_ref/libkaminpar_ref_full.so are not present")
    so = IH.build_bridge(os.path.join(str(tmp_path_factory.mktemp("ipbridge")), "ref_ip_bridge.so"))
    L = C.CDLL(so)
    args = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_int, C.c_int32, C.c_double, C.c_uint32, C.c_uint32, C.c_uint32,
            C.c_uint32] + [C.c_void_p] * 4
    L.ref_ip_bipartition.argtypes = args + [C.c_int32, C.c_void_p]
    L.ref_ip_params.argtypes = args + [C.c_void_p]
    L.ref_ip_preset_config.argtypes = [C.c_char_p, C.c_void_p]
    return L


P = IH._p


def star(n):
    src = np.concatenate([np.zeros(n - 1, np.int64), np.arange(1, n)])
    dst = np.concatenate([np.arange(1, n), np.zeros(n - 1, np.int64)])
    return _from_pairs(n, src, dst)


def _from_pairs(n, src, dst):
    order = np.lexsort((dst, src))
    src, dst = src[order], dst[order]
    xadj = np.zeros(n + 1, np.uint32)
    np.add.at(xadj, src + 1, 1)
    return CSRGraph(xadj=np.cumsum(xadj).astype(np.uint32), adjncy=dst.astype(np.uint32))


def components(n_comp, size):
    """n_comp paths of `size` vertices: more components than the seed search's 5 attempts."""
    src, dst = [], []
    for c in range(n_comp):
        for i in range(size - 1):
            a, b = c * size + i, c * size + i + 1
            src += [a, b]
            dst += [b, a]
    return _from_pairs(n_comp * size, np.array(src, np.int64), np.array(dst, np.int64))


def heavy(g):
    vw = np.ones(g.n, np.int32)
    vw[0] = 10 * g.n
    return CSRGraph(xadj=g.xadj, adjncy=g.adjncy, vwgt=vw)


GRAPHS = {
    "rmat12": lambda: rmat(12, 8, seed=3),
    "rgg": lambda: rgg2d(4000, seed=2),
    "grid": lambda: grid3d(14),
    "rmat11w": lambda: random_weights(rmat(11, 8, seed=5), 1, max_vwgt=5, max_adjwgt=7),
    "star": lambda: star(3000),
    "components": lambda: components(40, 7),
    "heavy": lambda: heavy(grid3d(8)),
}


def check(ref, g, part, k, input_k, cfg, seed=11, uniform=True, eps=0.03):
    res = S.lazy_extract(g.xadj, g.adjncy, g.vwgt, g.adjwgt, part, k)
    total = int(g.vwgt.sum()) if g.vwgt is not None else g.n
    mbw = IH.max_block_weights(total, input_k, eps, uniform, seed)
    blocks = 0
    for b in range(k):
        bx, ba, bv, be = IH.block_arrays(res, b)
        nb = len(bx) - 1
        if nb == 0:
            continue
        params = IH.block_params(cfg, input_k, mbw, uniform, total, eps, b, k, bx, ba, bv, be)
        want_p = np.zeros(6, np.int32)
        ref.ref_ip_params(C.byref(cfg), input_k, P(mbw), int(uniform), total, eps, b, k, nb, len(ba), P(bx), P(ba),
                          P(bv), P(be), P(want_p))
        assert np.array_equal(params, want_p), (b, params, want_p)
        s = int(np.int32(np.uint32(seed + b)))
        want = np.zeros(nb, np.uint32)
        ref.ref_ip_bipartition(C.byref(cfg), input_k, P(mbw), int(uniform), total, eps, b, k, nb, len(ba), P(bx),
                               P(ba), P(bv), P(be), s, P(want))
        rc, got, _ = IH.bipartition_block(cfg, params, s, bx, ba, bv, be)
        assert rc == 0
        assert np.array_equal(got, want), "block %d of %d (n=%d): %d vertices differ" % (b, k, nb,
                                                                                       int((got != want).sum()))
        blocks += 1
    return blocks


@pytest.mark.parametrize("preset_name", ["default", "fast", "largek", "largek-fast"])
def test_presets_match_reference(ref, preset_name):
    want = IPConfig()
    ref.ref_ip_preset_config(preset_name.encode(), C.byref(want))
    assert bytes(preset(preset_name)) == bytes(want)


@pytest.mark.parametrize("name", sorted(GRAPHS))
@pytest.mark.parametrize("preset_name", ["default", "fast", "largek", "largek-fast", "adaptive"])
def test_engine_equals_reference(ref, name, preset_name):
    g = GRAPHS[name]()
    if preset_name == "adaptive":
        cfg = preset("default")
        cfg.refinement.algorithm = cfg.pool_refinement.algorithm = TWOWAY_ADAPTIVE_FM
    else:
        cfg = preset(preset_name)
    n = 0
    for k, input_k, uniform in [(1, 2, True), (2, 6, False), (4, 12, True), (8, 24, False)]:
        part = (np.arange(g.n) * k // g.n).astype(np.uint32)
        n += check(ref, g, part, k, input_k, cfg, uniform=uniform)
    assert n > 0


def test_small_blocks_equal_reference(ref):
    """blocks with n <= 20 (no coarsening), n = 1 and n = 2, from a random partition with many blocks"""
    g = rmat(10, 4, seed=7)
    rng = np.random.default_rng(3)
    k = 64
    part = rng.integers(0, k, g.n).astype(np.uint32)
    part[:3] = 63  # keep block 63 non-empty
    assert check(ref, g, part, k, 128, preset("default")) > 0
    tiny = _from_pairs(2, np.array([0, 1]), np.array([1, 0]))
    assert check(ref, tiny, np.zeros(2, np.uint32), 1, 2, preset("default")) == 1
    one = CSRGraph(xadj=np.zeros(2, np.uint32), adjncy=np.zeros(0, np.uint32))
    assert check(ref, one, np.zeros(1, np.uint32), 1, 2, preset("default")) == 1


@pytest.mark.parametrize("seed", range(4))
def test_drawn_blocks_equal_reference(ref, seed):
    rng = np.random.default_rng(100 + seed)
    g = random_weights(rmat(11, int(rng.integers(2, 12)), seed=seed), seed, max_vwgt=int(rng.integers(0, 4)),
                       max_adjwgt=int(rng.integers(0, 4)))
    k = 1 << int(rng.integers(0, 4))
    part = rng.integers(0, k, g.n).astype(np.uint32)
    cfg = preset(["default", "fast", "largek", "largek-fast"][seed])
    cfg.num_seed_iterations = int(rng.integers(1, 4))
    check(ref, g, part, k, 2 * k + int(rng.integers(0, 2)), cfg, seed=int(rng.integers(0, 2**31)),
          uniform=bool(seed % 2))


def test_params_grid_equal_reference(ref):
    g = random_weights(rmat(10, 8, seed=1), 1, max_vwgt=4)
    for k, input_k in [(1, 2), (2, 4), (2, 5), (4, 11), (8, 16), (4, 100)]:
        part = (np.arange(g.n) * k // g.n).astype(np.uint32)
        res = S.lazy_extract(g.xadj, g.adjncy, g.vwgt, g.adjwgt, part, k)
        total = int(g.vwgt.sum())
        for eps in (0.01, 0.03, 0.1):
            for uniform in (True, False):
                for adaptive in (0, 1):
                    for cwl in range(4):
                        cfg = IPConfig(use_adaptive_epsilon=adaptive, cluster_weight_limit=cwl,
                                       repetition_multiplier=[1.0, 2.5, 0.3][cwl % 3], min_num_repetitions=1)
                        mbw = IH.max_block_weights(total, input_k, eps, uniform, k)
                        for b in range(k):
                            bx, ba, bv, be = IH.block_arrays(res, b)
                            got = IH.block_params(cfg, input_k, mbw, uniform, total, eps, b, k, bx, ba, bv, be)
                            want = np.zeros(6, np.int32)
                            ref.ref_ip_params(C.byref(cfg), input_k, P(mbw), int(uniform), total, eps, b, k,
                                              len(bx) - 1, len(ba), P(bx), P(ba), P(bv), P(be), P(want))
                            assert np.array_equal(got, want), (k, input_k, eps, uniform, adaptive, cwl, b)
