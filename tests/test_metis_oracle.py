"""The METIS reader's oracle (tests/metis_oracle.py), CPU only: its byte-loop and vectorised forms agree on every case
of the corpus, the corpus covers every kind, and on valid files both agree with the host fixture reader
graph.read_metis (which keeps explicit unit weights)."""
import os

import numpy as np
import pytest

from kaminpar_b200.graph import read_metis
from tests import metis_corpus as MC
from tests import metis_oracle as MO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("name,data", MC.cases(), ids=[c[0] for c in MC.cases()])
def test_loop_and_vectorised_forms_agree(name, data):
    if len(data) > 1 << 16:
        data = data[: 1 << 16]  # the byte loop is slow: its prefix (a refusal or a graph, both forms must agree)
    a, b = MO.parse_loop(data), MO.parse(data)
    assert MO.equal(a, b), (name, MO.report_of(a), MO.report_of(b))


def test_refusal_kinds():
    seen = set()
    for name, data, kind in MC.refusal_cases():
        r = MO.parse(data)
        assert MO.KINDS[r["kind"]] == kind, (name, MO.report_of(r))
        assert r["xadj"] is None
        seen.add(kind)
    assert seen == set(MO.KINDS[1:])


def test_valid_cases_are_graphs():
    for name, data in MC.valid_cases():
        r = MO.parse(data)
        assert r["kind"] == 0, (name, MO.report_of(r))


def test_rgg2d_fixture(tmp_path):
    data = open(os.path.join(ROOT, "tests", "golden", "misc", "rgg2d.metis"), "rb").read()
    r = MO.parse(data)
    gold = np.load(os.path.join(ROOT, "tests", "golden", "graph_rgg2d.npz"))
    assert r["kind"] == 0 and r["vwgt"] is None and r["adjwgt"] is None
    assert np.array_equal(r["xadj"], gold["xadj"]) and np.array_equal(r["adjncy"], gold["adjncy"])


def test_agrees_with_host_fixture_reader(tmp_path):
    for name, data in MC.valid_cases():
        if name.startswith(("garbage", "space_only_last", "no_final", "crlf")):
            continue  # graph.read_metis strips '\t' / '\r' and reads a last line of spaces differently
        r = MO.parse(data)
        p = tmp_path / f"{name}.metis"
        p.write_bytes(data)
        g = read_metis(str(p))
        assert np.array_equal(g.xadj, r["xadj"]) and np.array_equal(g.adjncy, r["adjncy"]), name
        for got, mine, dropped in ((g.vwgt, r["vwgt"], r["node_weights_dropped"]),
                                   (g.adjwgt, r["adjwgt"], r["edge_weights_dropped"])):
            if dropped:
                assert np.all(got == 1), name
            else:
                assert (got is None) == (mine is None) and (got is None or np.array_equal(got, mine)), name


def test_writer_round_trip():
    rng = np.random.default_rng(1)
    from kaminpar_b200.graph import rmat

    g = rmat(10, 8, seed=4)
    ew = rng.integers(1, 100, g.m)
    vw = rng.integers(1, 50, g.n)
    r = MO.parse(MO.write_metis(g.xadj, g.adjncy, vwgt=vw, adjwgt=ew))
    assert r["kind"] == 0
    assert np.array_equal(r["xadj"], g.xadj) and np.array_equal(r["adjncy"], g.adjncy)
    assert np.array_equal(r["vwgt"], vw) and np.array_equal(r["adjwgt"], ew)
