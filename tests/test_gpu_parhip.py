"""GPU: the ParHIP reader on the device (include/kaminpar_b200_parhip.h, kmp_parhip.cuh) against the oracle
(tests/parhip_oracle.py): every report field and every array, through kmp_read_parhip (a file) and
kmp_parse_parhip_device (a torch uint8 tensor), in the natural, implicit and external orderings.
  P0  misc/rgg2d-32bit.parhip and misc/rgg2d-64bit.parhip; all 64 width / weight combinations; n = 0; m = 0;
      isolated vertices; a star whose hub has degree 2^17; KMP_GRID_CAP 1..3; a seq_strict handle
  P1  every refusal kind at the first entry, the last entry and inside the hub row; truncation inside each section;
      competing violations; no graph is returned; the handle works afterwards
  P2  weighted R-MAT 2^20 and rgg 2^20 at 32- and 64-bit widths
  P3  the prepared EXTERNAL read: arrays and permutation == the oracle; set_on -> cluster and -> refine == the LP
      oracle; finish (of a host partition and of the refined device labels) == the preparation oracle's finish, in
      the file's ids; cluster, read, cluster at call indices 0 and 1
  P4  a file becomes a partition without a host CSR: read -> validate -> prepare (NATURAL), and the fused read"""
import functools
import os

import numpy as np
import pytest

from kaminpar_b200 import lp
from kaminpar_b200 import parhip as PH
from kaminpar_b200.graph import random_weights, rgg2d, rmat
from tests import parhip_oracle as PO
from tests import prepare_oracle as PRO
from tests.helpers import big_star

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MISC = os.path.join(ROOT, "tests", "golden", "misc")
ORDERINGS = (PO.NATURAL, PO.IMPLICIT, PO.EXTERNAL)


def _handle(schedule="sync"):
    eng = lp.EngineContext()
    eng.schedule = schedule
    return lp.LPHandle(lp._cluster_config(lp.LabelPropagationCoarseningContext(), eng))


@pytest.fixture(scope="module")
def handle():
    h = _handle()
    yield h
    h.close()


def _tensor(data: bytes):
    import torch

    if not data:
        return torch.empty(0, dtype=torch.uint8, device="cuda")
    return torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()


def _got(call):
    """(report, arrays) of one reader call; a refusal returns no graph."""
    try:
        g = call()
    except PH.ParhipError as e:
        assert e.code == (-4 if e.report.kind == PO.TOO_LARGE else -1)
        return e.report, None
    c = g.get()
    arrays = dict(xadj=c.xadj, adjncy=c.adjncy, vwgt=c.vwgt, adjwgt=c.adjwgt, old_to_new=g.old_to_new())
    assert c.sorted == bool(g.report.sorted)
    rep = g.report
    g.close()
    return rep, arrays


def check(h, data: bytes, tmp_path, orderings=ORDERINGS, name="case", prepared=True):
    """Both entry points == the oracle in every field and array, for each ordering (and the prepared read);
    returns the oracle's natural read."""
    p = tmp_path / f"{name}.parhip"
    p.write_bytes(data)
    t = _tensor(data)
    for o in orderings:
        expect = PO.read(data, o)
        for how, call in (("file", lambda: PH.read_parhip_device(h, str(p), o)),
                          ("device", lambda: PH.parse_parhip_device(h, t, o))):
            rep, arrays = _got(call)
            got = PO.as_dict(rep)
            assert got == PO.report_of(expect), (name, o, how, got, PO.report_of(expect))
            if expect["kind"] != 0:
                assert arrays is None
                continue
            for f in ("xadj", "adjncy", "vwgt", "adjwgt", "old_to_new"):
                assert (arrays[f] is None) == (expect[f] is None), (name, o, how, f)
                if expect[f] is not None:
                    assert np.array_equal(arrays[f].astype(np.int64), np.asarray(expect[f], np.int64)), (name, o, how, f)
    if prepared:
        expect = PO.read(data, PO.EXTERNAL)
        for how, call in (("file", lambda: PH.read_parhip_prepared(h, str(p))),
                          ("device", lambda: PH.parse_parhip_prepared(h, t))):
            try:
                pg = call()
            except PH.ParhipError as e:
                assert PO.as_dict(e.report) == PO.report_of(expect), (name, how)
                continue
            assert expect["kind"] == 0, (name, how)
            xadj, adj, vw, ew, o2n = pg._download()
            n = len(expect["xadj"]) - 1
            assert pg.n + pg.num_isolated == n and pg.num_isolated == int((np.diff(expect["xadj"]) == 0).sum())
            for a, f in ((xadj, "xadj"), (adj, "adjncy"), (vw, "vwgt"), (ew, "adjwgt"), (o2n, "old_to_new")):
                assert (a is None) == (expect[f] is None) and (a is None or np.array_equal(a, expect[f])), (name, how, f)
            pg.close()
    return PO.read(data)


def small(seed=1):
    return random_weights(rmat(7, 4, seed=seed), seed=seed, max_vwgt=9, max_adjwgt=9)


# ---- P0 ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fname", ["rgg2d-32bit.parhip", "rgg2d-64bit.parhip"])
def test_p0_sample_files(handle, tmp_path, fname):
    data = open(os.path.join(MISC, fname), "rb").read()
    r = check(handle, data, tmp_path)
    gold = np.load(os.path.join(ROOT, "tests", "golden", "graph_rgg2d.npz"))
    assert np.array_equal(r["xadj"], gold["xadj"]) and np.array_equal(r["adjncy"], gold["adjncy"])


def test_p0_every_width_and_weight_combination(handle, tmp_path):
    g = small()
    for version in range(64):
        vw, ew = (version & 2) == 0, (version & 1) == 0
        data = PO.write(g.xadj, g.adjncy, g.vwgt if vw else None, g.adjwgt if ew else None, version | (3 << 6))
        r = check(handle, data + b"\x01" * (version % 7), tmp_path, name=f"v{version}", prepared=version % 8 == 0)
        assert r["kind"] == 0


def test_p0_edge_shapes(handle, tmp_path):
    cases = {
        "n0": PO.write([0], []),
        "n0_w": PO.write([0], [], [], []),
        "m0": PO.write([0, 0, 0, 0], [], [3, 1, 2]),
        "isolated": PO.write(*_isolated()),
        "unit_w": PO.write([0, 1, 2], [1, 0], [1, 1], [1, 1]),
        "max_w": PO.write([0, 1, 2], [1, 0], [(1 << 30), (1 << 30) - 1], [(1 << 31) - 2, 1]),
    }
    for name, data in cases.items():
        assert check(handle, data, tmp_path, name=name)["kind"] == 0, name


def _isolated():
    g = small(3)
    xadj = np.concatenate([[0, 0], g.xadj[:50], np.full(5, g.xadj[49]), g.xadj[49:], np.full(9, g.xadj[-1])])
    vw = np.arange(len(xadj) - 1, dtype=np.int64) % 5 + 1
    return xadj, g.adjncy, vw, g.adjwgt  # the reader checks targets against n only


@functools.lru_cache(maxsize=None)
def hub_graph():
    g = random_weights(big_star((1 << 17) + 1), seed=5, max_vwgt=3, max_adjwgt=7)
    return g


def test_p0_hub(handle, tmp_path):
    g = hub_graph()
    assert int(np.diff(g.xadj).max()) >= 1 << 17
    for version in (PO.version_of(True, True), PO.version_of(True, True, True, True, True, True),
                    PO.version_of(False, True, False, True, False, False)):
        data = PO.write(g.xadj, g.adjncy, g.vwgt if (version & 2) == 0 else None,
                        g.adjwgt if (version & 1) == 0 else None, version)
        check(handle, data, tmp_path, name=f"hub{version}")


@pytest.mark.parametrize("cap", [1, 2, 3])
def test_p0_grid_cap(monkeypatch, tmp_path, cap):
    monkeypatch.setenv("KMP_GRID_CAP", str(cap))  # read by kmp_lp_create
    h = _handle()
    g = hub_graph()
    check(h, PO.write(g.xadj, g.adjncy, g.vwgt, g.adjwgt, PO.version_of(True, True, ids64=True)), tmp_path,
          name="hub")
    for name, data in refusals()[:6]:
        check(h, data, tmp_path, name=name, orderings=(PO.NATURAL, PO.EXTERNAL), prepared=False)
    h.close()


def test_p0_seq_strict_handle(tmp_path):
    h = _handle("seq_strict")
    g = small(4)
    check(h, PO.write(g.xadj, g.adjncy, g.vwgt, g.adjwgt), tmp_path)
    h.close()


# ---- P1 ----------------------------------------------------------------------------------------------------------
def _put(data, at, value, width, signed=False):
    data[at:at + width] = int(value).to_bytes(width, "little", signed=signed)


@functools.lru_cache(maxsize=None)
def refusals():
    """(name, bytes): every kind at the first entry, the last entry and inside the hub row, at both widths."""
    out = []
    hub = hub_graph()
    for tag, g in (("small", small(2)), ("hub", hub)):
        for w64 in (False, True):
            version = PO.version_of(True, True, w64, w64, w64, w64)
            d = bytes(PO.write(g.xadj, g.adjncy, g.vwgt, g.adjwgt, version))
            wo, wi, wv, we = PO.widths(version)
            n, m = g.n, g.m
            s_off, s_adj = 24, 24 + (n + 1) * wo
            s_vw = s_adj + m * wi
            s_ew = s_vw + n * wv
            end = s_ew + m * we
            # the hub's row: the middle of it
            u = int(np.argmax(np.diff(g.xadj)))
            mid = int(g.xadj[u] + (g.xadj[u + 1] - g.xadj[u]) // 2)
            name = f"{tag}_{'w64' if w64 else 'w32'}"

            def mut(label, *puts):
                x = bytearray(d)
                for at, val, width, signed in puts:
                    _put(x, at, val, width, signed)
                out.append((f"{name}_{label}", bytes(x)))

            for i, where in ((0, "first"), (m - 1, "last"), (mid, "hub")):
                mut(f"target_{where}", (s_adj + i * wi, n + i % 3, wi, False))
                mut(f"ew_{where}", (s_ew + i * we, -(i % 2), we, True))
            for i, where in ((0, "first"), (n - 1, "last"), (u, "hub")):
                mut(f"vw_{where}", (s_vw + i * wv, 0, wv, True))
            mut("offsets_first", (s_off, s_adj + wi, wo, False))
            mut("offsets_last", (s_off + n * wo, s_adj + (m + 1) * wi, wo, False))
            mut("offsets_hub", (s_off + (u + 1) * wo, s_adj + int(g.xadj[u + 1]) * wi + 1, wo, False))
            mut("offsets_decreasing", (s_off + (u + 1) * wo, s_adj + int(g.xadj[u]) * wi - wi, wo, False))
            mut("total_vw", *[(s_vw + i * wv, 1 << 30, wv, True) for i in range(min(n, 3))])
            mut("total_ew", *[(s_ew + i * we, 1 << 30, we, True) for i in range(3)])
            mut("competing", (s_adj + mid * wi, n, wi, False), (s_adj + (m - 1) * wi, n + 5, wi, False),
                (s_vw, 0, wv, True), (s_off + n * wo, 3, wo, False))
            if w64:
                mut("target_too_large", (s_adj + mid * wi, 1 << 32, wi, False))
                mut("vw_too_large", (s_vw + (n - 1) * wv, 1 << 31, wv, True))
                mut("ew_too_large", (s_ew + mid * we, 1 << 40, we, True))
            mut("n_too_large", (8, 1 << 31, 8, False))
            mut("m_too_large", (16, (1 << 32) + 3, 8, False))
            if tag == "small":
                for cut, where in ((0, "empty"), (7, "header"), (s_off + 3, "offsets"), (s_adj + wi, "adjncy"),
                                   (s_vw + 1, "vwgt"), (s_ew + (m // 2) * we, "adjwgt"), (end - 1, "last_byte")):
                    out.append((f"{name}_truncated_{where}", d[:cut]))
    return out


def test_p1_refusals(handle, tmp_path):
    kinds = set()
    for name, data in refusals():
        r = check(handle, data, tmp_path, name=name, prepared=name.startswith("small"))
        assert r["kind"] != 0, name
        kinds.add(PO.KINDS[r["kind"]])
    assert kinds == set(PO.KINDS[1:])


def test_p1_handle_works_afterwards(handle, tmp_path):
    g = small(5)
    bad = bytearray(PO.write(g.xadj, g.adjncy))
    _put(bad, 24 + (g.n + 1) * 4, g.n, 4)
    p = tmp_path / "bad.parhip"
    p.write_bytes(bytes(bad))
    with pytest.raises(PH.ParhipError) as e:
        PH.read_parhip_device(handle, str(p), "external_degree_buckets")
    assert e.value.report.message() == f"neighbor out of range at byte {24 + (g.n + 1) * 4} (adjncy entry 0)"
    assert check(handle, PO.write(g.xadj, g.adjncy, g.vwgt, g.adjwgt), tmp_path)["kind"] == 0


# ---- P2 ----------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def large(name):
    if name == "rmat20_w":
        return random_weights(rmat(20, 8, seed=3), seed=4, max_vwgt=20, max_adjwgt=100)
    return rgg2d(1 << 20, seed=2)


@pytest.mark.parametrize("name", ["rmat20_w", "rgg20"])
@pytest.mark.parametrize("w64", [False, True])
def test_p2_large(handle, tmp_path, name, w64):
    g = large(name)
    version = PO.version_of(g.vwgt is not None, g.adjwgt is not None, w64, w64, w64, w64)
    r = check(handle, PO.write(g.xadj, g.adjncy, g.vwgt, g.adjwgt, version), tmp_path, name=name,
              orderings=(PO.NATURAL, PO.EXTERNAL))
    assert np.array_equal(r["xadj"], g.xadj) and np.array_equal(r["adjncy"], g.adjncy)


# ---- P3 / P4 -----------------------------------------------------------------------------------------------------
def test_p3_prepared_read_cluster_finish(tmp_path):
    from oracle import bindings as B

    g0 = random_weights(rmat(14, 8, seed=6), seed=2, max_vwgt=4, max_adjwgt=9)
    xadj = np.concatenate([g0.xadj, np.full(17, g0.xadj[-1])])  # 17 isolated vertices at the end of the file
    vw = np.concatenate([g0.vwgt, np.arange(17) % 3 + 1]).astype(np.int32)
    p = tmp_path / "g.parhip"
    p.write_bytes(PO.write(xadj, g0.adjncy, vw, g0.adjwgt, PO.version_of(True, True, ids64=True)))
    expect = PO.read(p.read_bytes(), PO.EXTERNAL)
    h = _handle()
    ctx = lp.create_default_context()
    ctx.partition.setup(g0, 8, 0.03)
    mcw = lp.compute_max_cluster_weight(ctx.coarsening, ctx.partition, g0.n, g0.total_node_weight())
    first, _ = B.oracle_rearrange(g0)
    h.set_graph(first)
    c0, _ = h.cluster(mcw)
    assert np.array_equal(c0, B.oracle_lp_cluster(first, 0, mcw, schedule=B.SYNC, call_index=0))

    pg = PH.read_parhip_prepared(h, str(p))
    assert np.array_equal(pg.old_to_new(), expect["old_to_new"])
    lg = pg.get()
    np_, niso = pg.n, int((np.diff(xadj) == 0).sum())  # R-MAT's own isolated vertices and the 17 appended
    assert niso >= 17 and np_ == len(xadj) - 1 - niso and pg.num_isolated == niso
    assert np.array_equal(lg.xadj, expect["xadj"][:np_ + 1])
    pg.set_on(h)
    c1, _ = h.cluster(mcw)
    assert np.array_equal(c1, B.oracle_lp_cluster(lg, 0, mcw, schedule=B.SYNC, call_index=1))
    k = 8
    mbw = np.full(k, int(vw.sum()) // k + 40, np.int32)
    part = (np.arange(np_) * 7 % k).astype(np.uint32)
    got, bw = pg.finish(h, k, mbw, part)
    prep = dict(xadj=expect["xadj"], vwgt=expect["vwgt"], old_to_new=expect["old_to_new"], n_prime=np_,
                num_isolated=niso, new_to_old=np.argsort(expect["old_to_new"]).astype(np.uint32))
    want, want_bw = PRO.finish(prep, k, mbw, part)
    assert np.array_equal(got, want) and np.array_equal(bw, want_bw)
    # the partition is in the file's ids: a non-isolated file vertex u got the block of its new id
    o2n = expect["old_to_new"].astype(np.int64)
    live = o2n < np_
    assert np.array_equal(got[live], part[o2n[live]])
    # refinement on the forward lists (the preparation's are reversed), then the finish from the device labels
    hr = lp.LPHandle(lp._refine_config(ctx.refinement.lp, ctx.engine))
    pg.set_on(hr)
    rp, rbw, _ = hr.refine(k, mbw, part.copy())
    params = B.oracle_params(B.default_refine_params(), commit_passes=4)
    ep, ebw = B.oracle_lp_refine(lg, 0, k, mbw, part, schedule=B.SYNC, params=params)
    assert np.array_equal(rp, ep) and np.array_equal(rbw, ebw)
    got, bw = pg.finish(hr, k, mbw)
    want, want_bw = PRO.finish(prep, k, mbw, ep)
    assert np.array_equal(got, want) and np.array_equal(bw, want_bw)
    hr.close()
    pg.close()
    h.close()


def test_p4_file_to_partition_without_host_csr(tmp_path):
    from kaminpar_b200 import prepare as PR
    from kaminpar_b200 import validate as VA

    g0 = random_weights(rmat(13, 8, seed=9), seed=1, max_adjwgt=5)
    p = tmp_path / "g.parhip"
    p.write_bytes(PO.write(g0.xadj, g0.adjncy, adjwgt=g0.adjwgt, version=PO.version_of(False, True, True, True)))
    h = _handle()
    g = PH.read_parhip_device(h, str(p))
    d = g.device_arrays()
    rep = VA.validate_graph_device(h, g.n, g.m, d[0], d[1], d[3])
    assert rep.valid == 1
    natural = PR.rearrange_by_degree_buckets_device(h, g.n, g.m, *d[:4])
    fused = PH.read_parhip_prepared(h, str(p))
    assert np.array_equal(natural.old_to_new(), fused.old_to_new()) and natural.n == fused.n
    a, b = natural.get(), fused.get()
    assert np.array_equal(a.xadj, b.xadj)
    for u in range(0, a.n, 97):  # the same rows, reversed in the preparation, forward in the read
        s, e = a.xadj[u], a.xadj[u + 1]
        assert np.array_equal(a.adjncy[s:e][::-1], b.adjncy[s:e]) and np.array_equal(a.adjwgt[s:e][::-1], b.adjwgt[s:e])
    k = 4
    mbw = np.full(k, g.n // k + 10, np.int32)
    outs = []
    for pg in (natural, fused):
        pg.set_on(h)
        h.cluster(50)
        part = (np.arange(pg.n) % k).astype(np.uint32)
        outs.append(pg.finish(h, k, mbw, part)[0])
        pg.close()
    assert np.array_equal(outs[0], outs[1])
    g.close()
    h.close()
