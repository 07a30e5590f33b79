"""Writes tests/golden/validate_cases.npz: the UNMODIFIED reference's verdicts on the small validation corpus
(tests/test_validate_bridge.py: corpus(), built from tests/validate_oracle.py), through tests/cpp/ref_validate_bridge.cc.
The corpus is generated, not stored: per case the file holds its name, a digest of its arrays and:
  - ref_valid, ref_message: debug::validate_graph's verdict and its warning line (colour and "[Warning] " stripped),
    for every case whose shape passes (xadj[0] == 0, xadj[n] == m: the reference reads m from xadj[n]), else -1, "";
  - ref_undirected: validate_undirected_graph's exit status on the cases in its parity domain, else -2.
Run from the repository root after the build left oracle/_ref/libkaminpar_ref_full.so:
    python tests/golden/make_validate_golden.py"""
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests import test_validate_bridge as TB  # noqa: E402
from tests import validate_oracle as V  # noqa: E402


def main():
    with tempfile.TemporaryDirectory() as d:
        bridge = TB.compile_bridge(d)
        names, digests, valid, messages, undirected = [], [], [], [], []
        for name, xadj, adj, w in TB.corpus():
            names.append(name)
            digests.append(TB.digest(xadj, adj, w))
            ok, msg = TB.reference_validate(bridge, xadj, adj, w) if TB.shape_ok(xadj, adj) else (-1, "")
            valid.append(ok)
            messages.append(msg)
            undirected.append(TB.reference_undirected(bridge, xadj, adj, w) if TB.in_undirected_domain(xadj, adj) else -2)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "validate_cases.npz"), names=np.array(names),
                        digests=np.array(digests), ref_valid=np.array(valid, np.int32), ref_message=np.array(messages),
                        ref_undirected=np.array(undirected, np.int32))
    print(f"{len(names)} cases")


if __name__ == "__main__":
    main()
