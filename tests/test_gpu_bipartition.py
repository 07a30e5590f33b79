"""-m gpu: block bipartitioning on the device (kmp_bipartition_subgraphs, DESIGN.md §20).

G0  every pinned reference bipartition (tests/golden/ip_*.npz) reproduced through extract -> bipartition -> copy-back
G1  device == host twin (tests/ip_host.py: the same engine under g++, held to the live reference by
    tests/test_ip_bridge.py and to the goldens by tests/test_ip_oracle.py) block for block on id-range and random
    partitions of R-MAT, rgg, a grid and weighted graphs, k in {1, 2, 64, 1024}, k' = 2k and k' = input_k with mixed
    s_b in {1, 2}, every supported preset; the result goes straight into copy_partitions through its data_ptr()
G2  each refusal leaves the handle's labels and the output buffer untouched, k = 3 (not a power of two) among them
G4  one full extension level, each step held to its oracle: project -> overload -> LP refine -> extract ->
    bipartition -> copy-back -> overload -> LP refine at k'
G3  the arena re-run (KMP_IP_ARENA_CAP) gives the same result
G5  the same seed gives the same output under KMP_GRID_CAP 1..3, another seed a different one
"""
import numpy as np
import pytest
import torch

from kaminpar_b200 import bipartition as BP
from kaminpar_b200 import contraction as KC
from kaminpar_b200 import lp
from kaminpar_b200 import subgraphs as SG
from kaminpar_b200.graph import grid3d, random_weights, rgg2d, rmat
from oracle import bindings as B
from oracle import contraction_oracle as CO
from tests import balance_oracle as O
from tests import ip_golden as G
from tests import ip_host as IH
from tests import subgraph_oracle as S
from tests.test_gpu_subgraphs import REFINE_PARAMS, _handle

pytestmark = pytest.mark.gpu

INVALID, UNSUPPORTED = -1, -4  # KMP_ERR_INVALID, KMP_ERR_UNSUPPORTED

GRAPHS = {
    "rmat13": lambda: rmat(13, 8, seed=2),
    "rgg14": lambda: rgg2d(1 << 14, seed=3),
    "grid24": lambda: grid3d(24),
    "rmat12w": lambda: random_weights(rmat(12, 8, seed=4), 1, max_vwgt=6, max_adjwgt=5),
}
PRESETS = ["default", "fast", "largek", "largek-fast", "adaptive"]
GOLDEN = [c for f in G.files() for c in G.cases(f)]


def _config(name):
    if name == "adaptive":
        cfg = BP.preset("default")
        cfg.refinement.algorithm = cfg.pool_refinement.algorithm = BP.TWOWAY_ADAPTIVE_FM
        return cfg
    return BP.preset(name)


def _run(h, g, part, k, k_prime, input_k, cfg, seed, uniform=True):
    total = int(g.vwgt.sum()) if g.vwgt is not None else g.n
    mbw = IH.max_block_weights(total, input_k, uniform=uniform, seed=k)
    sg = SG.extract_subgraphs(h, k, part)
    out, stats = BP.bipartition(sg, h, k_prime, input_k, mbw, seed=seed, ip_config=cfg, uniform=uniform,
                                total_node_weight=total)
    want = IH.expected_sub_partitions(g, part, k, k_prime, input_k, mbw, seed, cfg, uniform)
    return sg, out, stats, want


@pytest.mark.parametrize("case", GOLDEN, ids=[c[0] for c in GOLDEN])
def test_g0_goldens_through_extract_and_copy_back(case):
    _, g, part, k, k_prime, input_k, uniform, eps, seed, mbw, cfg, sub = case
    h = _handle()
    h.set_graph(g)
    sg = SG.extract_subgraphs(h, k, part)
    total = int(g.vwgt.sum()) if g.vwgt is not None else g.n
    out, _ = BP.bipartition(sg, h, k_prime, input_k, mbw, seed=seed, ip_config=cfg, uniform=uniform,
                            total_node_weight=total, epsilon=eps)
    assert np.array_equal(out.cpu().numpy().view(np.uint32), sub)
    got, bw = sg.copy_partitions(h, out.data_ptr(), k_prime, input_k)
    want, want_bw = S.copy_back(part, sg.mapping(), sg.offsets()[0], sub, k, k_prime, input_k, g.vwgt)
    assert np.array_equal(got, want) and np.array_equal(bw, want_bw)


@pytest.mark.parametrize("preset_name", PRESETS)
@pytest.mark.parametrize("name", sorted(GRAPHS))
@pytest.mark.parametrize("k,k_prime,input_k", [(1, 2, 2), (2, 4, 8), (2, 3, 3), (64, 128, 256), (64, 100, 100),
                                                (1024, 2048, 2048)])
def test_g1_device_equals_host_twin(name, k, k_prime, input_k, preset_name):
    g = GRAPHS[name]()
    h = _handle()
    h.set_graph(g)
    rng = np.random.default_rng(k)
    part = ((np.arange(g.n) * k // g.n) if k != 64 else rng.integers(0, k, g.n)).astype(np.uint32)
    cfg = _config(preset_name)
    sg, out, stats, want = _run(h, g, part, k, k_prime, input_k, cfg, seed=7, uniform=bool(k % 4 != 2))
    assert np.array_equal(out.cpu().numpy().view(np.uint32), want)
    assert stats.blocks_split > 0 and stats.arena_retries == 0
    got, _ = sg.copy_partitions(h, out.data_ptr(), k_prime, input_k)
    mapping, node_off = sg.mapping(), sg.offsets()[0]
    exp, _ = S.copy_back(part, mapping, node_off, want, k, k_prime, input_k, g.vwgt)
    assert np.array_equal(got, exp)


def test_g2_refusals_leave_state_untouched():
    g = rmat(12, 8, seed=1)
    h = _handle()
    h.set_graph(g)
    part = (np.arange(g.n) * 4 // g.n).astype(np.uint32)
    sg = SG.extract_subgraphs(h, 4, part)
    mbw = IH.max_block_weights(g.n, 16)
    buf = torch.full((g.n + 1,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
    ptr = buf.data_ptr()
    labels = h.download_labels().copy()

    def refused(code, k_prime=8, input_k=16, p=ptr, cfg=None):
        with pytest.raises(RuntimeError, match="kaminpar_b200 error %d:" % code):
            BP.bipartition_into(sg, h, k_prime, input_k, mbw if input_k == 16 else IH.max_block_weights(g.n, input_k),
                                p, seed=1, ip_config=cfg if cfg is not None else BP.IPConfig(), total_node_weight=g.n)
        assert np.array_equal(h.download_labels(), labels)
        assert bool((buf == 0x5A5A5A5A).all())

    refused(UNSUPPORTED, k_prime=16)  # s_b = 4
    sg3 = SG.extract_subgraphs(h, 3, (np.arange(g.n) * 3 // g.n).astype(np.uint32))
    labels = h.download_labels().copy()
    with pytest.raises(RuntimeError, match="kaminpar_b200 error %d:" % UNSUPPORTED):  # k = 3: not a power of two
        BP.bipartition_into(sg3, h, 6, 7, IH.max_block_weights(g.n, 7, uniform=False), ptr, seed=1,
                            total_node_weight=g.n, uniform=False)
    assert np.array_equal(h.download_labels(), labels) and bool((buf == 0x5A5A5A5A).all())
    sg3.close()
    sg = SG.extract_subgraphs(h, 4, part)
    labels = h.download_labels().copy()
    long_list = BP.IPConfig()
    long_list.refinement.num_algorithms = 2
    refused(UNSUPPORTED, cfg=long_list)
    flow = BP.IPConfig()
    flow.pool_refinement.algorithm = BP.TWOWAY_FLOW
    refused(UNSUPPORTED, cfg=flow)
    refused(INVALID, p=ptr + 2)
    refused(INVALID, p=0)
    refused(INVALID, k_prime=2)
    h2 = _handle()
    h2.set_graph(g)
    with pytest.raises(RuntimeError, match="kaminpar_b200 error %d:" % INVALID):
        BP.bipartition_into(sg, h2, 8, 16, mbw, ptr, seed=1, total_node_weight=g.n)
    h.set_graph(g)  # a new graph epoch: the subgraphs are stale
    refused(INVALID)


def test_g3_arena_rerun_same_result(monkeypatch):
    g = rgg2d(1 << 14, seed=5)
    h = _handle()
    h.set_graph(g)
    part = (np.arange(g.n) * 8 // g.n).astype(np.uint32)
    _, out, stats, want = _run(h, g, part, 8, 16, 32, BP.IPConfig(), seed=3)
    assert stats.arena_retries == 0 and np.array_equal(out.cpu().numpy().view(np.uint32), want)
    monkeypatch.setenv("KMP_IP_ARENA_CAP", "65536")
    _, out2, stats2, _ = _run(h, g, part, 8, 16, 32, BP.IPConfig(), seed=3)
    assert stats2.arena_retries >= 8 and stats2.kernel_launches >= 3
    assert np.array_equal(out2.cpu().numpy().view(np.uint32), want)


@pytest.mark.parametrize("cap", [1, 2, 3])
def test_g5_determinism_and_seed(cap, monkeypatch):
    monkeypatch.setenv("KMP_GRID_CAP", str(cap))
    g = rmat(13, 8, seed=6)
    h = _handle()
    h.set_graph(g)
    part = (np.arange(g.n) * 16 // g.n).astype(np.uint32)
    total = g.n
    mbw = IH.max_block_weights(total, 32)
    sg = SG.extract_subgraphs(h, 16, part)
    a, _ = BP.bipartition(sg, h, 32, 32, mbw, seed=9, total_node_weight=total)
    b, _ = BP.bipartition(sg, h, 32, 32, mbw, seed=9, total_node_weight=total)
    c, _ = BP.bipartition(sg, h, 32, 32, mbw, seed=10, total_node_weight=total)
    assert torch.equal(a, b)
    assert not torch.equal(a, c)
    want = IH.expected_sub_partitions(g, part, 16, 32, 32, mbw, 9)
    assert np.array_equal(a.cpu().numpy().view(np.uint32), want)


def test_g4_one_extension_level():
    seed, k, input_k = 1, 4, 8
    g = random_weights(rmat(14, 8, seed=21), 6, max_vwgt=4, max_adjwgt=5)
    ctx = lp.create_default_context()
    ctx.engine.seed = seed
    hc = _handle(seed, refine=False)
    hr = _handle(seed)
    hc.set_graph(g)
    p_ctx = ctx.partition.setup(g, k, 0.03)
    mcw = lp.compute_max_cluster_weight(ctx.coarsening, p_ctx, g.n, g.total_node_weight())
    clustering, _ = hc.cluster(mcw)
    assert np.array_equal(clustering, B.oracle_lp_cluster(g, seed, mcw, schedule=B.SYNC)), "clustering"
    cg = KC.contract_on_handle(hc, None)
    con = CO.contract(g.xadj, g.adjncy, g.vwgt, g.adjwgt, clustering)
    cpart = (np.arange(cg.n, dtype=np.int64) * k // max(cg.n, 1)).astype(np.uint32)
    up = cg.project_up(cpart)
    assert np.array_equal(up, CO.project_up(con["mapping"], cpart)), "project_up"
    hr.set_graph(g)
    hr.upload_partition(up)
    mbw, pbw = p_ctx.max_block_weights(), p_ctx.perfectly_balanced_block_weights()
    _, bw, _ = hr.overload_balance(k, mbw, pbw, None)
    ob = O.overload_balance(g, k, up, mbw, pbw, seed=seed, call=0)
    assert np.array_equal(bw, ob["block_weights"]), "overload balance"
    _, bw, _ = hr.refine(k, mbw, None)
    ep, ebw = B.oracle_lp_refine(g, seed, k, mbw, ob["labels"], schedule=B.SYNC, params=REFINE_PARAMS)
    assert np.array_equal(bw, ebw) and np.array_equal(hr.download_labels(), ep), "refinement"
    # extension to k' = 2k: extract from the device labels, bipartition on the device, copy back from the device
    k_prime = 2 * k
    total = int(g.vwgt.sum())
    in_ctx = ctx.partition.setup(g, input_k, 0.03)
    in_mbw = np.asarray(in_ctx.max_block_weights(), np.int32)
    sg = SG.extract_subgraphs(hr, k)
    sub, _ = BP.bipartition(sg, hr, k_prime, input_k, in_mbw, seed=seed, total_node_weight=total, epsilon=0.03)
    want_sub = IH.expected_sub_partitions(g, ep, k, k_prime, input_k, in_mbw, seed, eps=0.03)
    assert np.array_equal(sub.cpu().numpy().view(np.uint32), want_sub), "bipartition"
    sg.copy_partitions(hr, sub.data_ptr(), k_prime, input_k, fetch=False)
    want, _ = S.copy_back(ep, sg.mapping(), sg.offsets()[0], want_sub, k, k_prime, input_k, g.vwgt)
    assert np.array_equal(hr.download_labels(), want), "copy-back"
    p2 = ctx.partition.setup(g, k_prime, 0.03)
    mbw2, pbw2 = p2.max_block_weights(), p2.perfectly_balanced_block_weights()
    _, bw, _ = hr.overload_balance(k_prime, mbw2, pbw2, None)
    ob2 = O.overload_balance(g, k_prime, want, mbw2, pbw2, seed=seed, call=1)
    assert np.array_equal(bw, ob2["block_weights"]), "overload balance at k'"
    _, bw, _ = hr.refine(k_prime, mbw2, None)
    ep2, ebw2 = B.oracle_lp_refine(g, seed, k_prime, mbw2, ob2["labels"], schedule=B.SYNC, params=REFINE_PARAMS)
    assert np.array_equal(bw, ebw2) and np.array_equal(hr.download_labels(), ep2), "refinement at k'"
    sg.close()
    cg.close()
    hr.close()
    hc.close()
