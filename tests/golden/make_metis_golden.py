"""Writes tests/golden/metis_cases.npz: the unmodified reference's verdict on every file of tests/metis_corpus.py,
through tests/cpp/ref_metis_bridge.cc (needs the reference sources and oracle/_ref/libkaminpar_ref_full.so). Per case:
its name and content digest, the assertion that fires with assertions on ("file:line", "" for none), and in the
Release build whether a graph came back, its arrays' digest and the warnings printed. tests/test_metis_bridge.py holds
the oracle to these where the reference is absent.

    python tests/golden/make_metis_golden.py
"""
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests import metis_bridge as MB  # noqa: E402
from tests import metis_corpus as MC  # noqa: E402
from tests import metis_oracle as MO  # noqa: E402


def main():
    if not MB.available():
        raise SystemExit("make_metis_golden: the reference or oracle/_ref/libkaminpar_ref_full.so is missing")
    tmp = tempfile.mkdtemp(prefix="metis_golden_")
    rel, asr = MB.compile_bridge(tmp, True), MB.compile_bridge(tmp, False)
    cols = {k: [] for k in ("name", "case", "where", "graph", "digest", "warnings")}
    for name, data in MC.cases():
        p = os.path.join(tmp, "case.metis")
        with open(p, "wb") as f:
            f.write(data)
        v = MB.verdict(rel, asr, p, name, MO.KINDS[MO.parse(data)["kind"]])
        cols["name"].append(name)
        cols["case"].append(MB.case_digest(data))
        for k in ("where", "graph", "digest", "warnings"):
            cols[k].append(v[k])
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "metis_cases.npz"),
                        **{k: np.asarray(v) for k, v in cols.items()})


if __name__ == "__main__":
    main()
