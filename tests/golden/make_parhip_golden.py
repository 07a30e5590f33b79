"""Pins the unmodified reference's ParHIP reads of tests/parhip_bridge.py's corpus (all four orderings) in
tests/golden/parhip_cases.npz, so that tests/test_parhip_bridge.py checks the oracle where the reference is absent.
Needs oracle/_ref/parhip_read (built by build() where the reference sources exist).

    python tests/golden/make_parhip_golden.py
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tests import parhip_bridge as PB  # noqa: E402

FIELDS = ("xadj", "adjncy", "vwgt", "adjwgt", "old_to_new")


def main():
    out = {}
    for name, data in PB.corpus():
        for o in range(4):
            r = PB.run(data, o)
            if r is None:
                raise SystemExit(f"{PB.REF} not built")
            key = f"{name}__{o}"
            out[key + "__exit"] = np.array([r["exit"]])
            if r["exit"] != 0:
                out[key + "__log"] = np.array([r["log"]])
            if r["exit"] == 0:
                out[key + "__sorted"] = np.array([r["sorted"]])
                for f in FIELDS:
                    if r[f] is not None:
                        out[key + "__" + f] = r[f]
    np.savez_compressed(PB.GOLDEN, **out)


if __name__ == "__main__":
    main()
