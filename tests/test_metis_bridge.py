"""CPU: the METIS oracle (tests/metis_oracle.py) held to the UNMODIFIED reference's reader, csr_read
(kaminpar-io/metis_parser.cc), on every file of tests/metis_corpus.py, through tests/cpp/ref_metis_bridge.cc:
  - in the parity domain (no assertion fires with assertions on), the Release build's arrays, dropped weights and the
    "ignorning extra lines" warning equal the oracle's;
  - for every refused kind, the reference's own assertion fires, at a source line that belongs to that kind (below);
    except EMPTY, where the reference returns nullopt, FORMAT, where it warns (and for 1xx reads the node sizes as
    weights, with or without a later assertion), and TOO_FEW_LINES, where it reads past its mapping (not run).
Live where the reference and oracle/_ref/libkaminpar_ref_full.so exist; everywhere against the reference's verdicts
pinned in tests/golden/metis_cases.npz (tests/golden/make_metis_golden.py)."""
import os
import tempfile

import numpy as np
import pytest

from tests import metis_bridge as MB
from tests import metis_corpus as MC
from tests import metis_oracle as MO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "metis_cases.npz")

# the reference assertions (file:line) that may fire first for a file whose first violation is of each kind
ASSERTIONS = {
    "HEADER": {"file_toker.h:90", "file_toker.h:127", "metis_parser.cc:69"},  # scan_uint, consume_char, m > n(n-1)/2
    "TOO_LARGE": {"metis_parser.cc:61", "metis_parser.cc:65", "file_toker.h:127"},  # n, m; a later 4th token
    "BAD_BYTE": {"file_toker.h:90", "file_toker.h:127"},
    "MISSING_NODE_WEIGHT": {"file_toker.h:90"},
    "MISSING_EDGE_WEIGHT": {"file_toker.h:90"},
    "ZERO_WEIGHT": {"metis_parser.cc:109", "metis_parser.cc:131"},
    "WEIGHT_TOO_LARGE": {"metis_parser.cc:105", "metis_parser.cc:127"},
    "NEIGHBOR_OUT_OF_RANGE": {"metis_parser.cc:134"},
    "SELF_LOOP": {"metis_parser.cc:135"},
    "EDGE_COUNT": {"metis_parser.cc:208", "static_array.h:219"},  # too many entries overrun the edge array first
    "TOTAL_WEIGHT": {"metis_parser.cc:224", "metis_parser.cc:228"},
}
FORMAT_WARNINGS = ("ignoring node sizes", "invalid or unsupported graph format")
CASES = MC.cases()


def check(name, data, v):
    o = MO.parse(data)
    kind = MO.KINDS[o["kind"]]
    if MB.skipped(name, kind):
        return kind
    if kind == "OK":
        assert v["where"] == "" and v["graph"] == 1, (name, v)
        assert v["digest"] == MB.digest(o), name
        assert v["warnings"] == ("ignorning extra lines in input file" if o["extra_lines"] else ""), (name, v)
    elif kind == "EMPTY":
        assert v["where"] == "" and v["graph"] == 0, (name, v)
    elif kind == "FORMAT":
        assert any(w in v["warnings"] for w in FORMAT_WARNINGS), (name, v)
    else:
        assert v["where"] in ASSERTIONS[kind], (name, kind, v)
    return kind


def golden():
    z = np.load(GOLDEN)
    return {str(n): dict(case=str(c), where=str(w), graph=int(g), digest=str(d), warnings=str(s))
            for n, c, w, g, d, s in zip(z["name"], z["case"], z["where"], z["graph"], z["digest"], z["warnings"])}


def test_golden_verdicts():
    gold = golden()
    assert sorted(gold) == sorted(name for name, _ in CASES)
    kinds = set()
    for name, data in CASES:
        g = gold[name]
        assert g["case"] == MB.case_digest(data), f"{name}: the corpus changed; regenerate the goldens"
        kinds.add(check(name, data, g))
    assert kinds == set(MO.KINDS)


@pytest.mark.skipif(not MB.available(), reason="the reference or oracle/_ref/libkaminpar_ref_full.so is absent")
def test_live_reference():
    tmp = tempfile.mkdtemp(prefix="metis_bridge_")
    rel, asr = MB.compile_bridge(tmp, True), MB.compile_bridge(tmp, False)
    gold = golden()
    for name, data in CASES:
        p = os.path.join(tmp, "case.metis")
        with open(p, "wb") as f:
            f.write(data)
        v = MB.verdict(rel, asr, p, name, MO.KINDS[MO.parse(data)["kind"]])
        check(name, data, v)
        assert v == {k: gold[name][k] for k in v}, (name, v, gold[name])
