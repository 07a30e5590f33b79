"""Golden fixtures of the contraction row (run in the authoring container only).

For the graphs and reference LP clusterings already stored in tests/golden/ref_<case>.npz, store what the
UNMODIFIED reference's contract_clustering returns (default algorithm UNBUFFERED; raw, i.e. with the
reference's own coarse numbering and adjacency order) -> tests/golden/contract_<case>.npz. The oracle
(oracle/contraction_oracle.py) must reproduce every one of them after canonicalize()
(tests/test_contraction_oracle.py); that is what pins it. For the generated graphs of that test (live_cases,
multigraph_cases) the digests of the reference's canonical results go to tests/golden/contract_live_digests.json.

    python tests/golden/make_contraction_golden.py
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import bindings as B  # noqa: E402
from tests import helpers as H  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
CASES = ["rgg2d_k4", "rgg16_w", "walshaw_k16", "walshaw_unsorted", "rmat13_w", "grid12", "road60", "star30000"]


def main():
    assert B.have_reference(), "build oracle/_ref first: make -C oracle ref"
    for name in CASES:
        g, d = H.load_case(name)
        seed = int(d["seeds"][0])
        cl = d[f"clustering_s{seed}"]
        cl = cl if cl.ndim == 1 else cl[0]
        r = B.ref_contract(g, cl, 1)
        np.savez_compressed(os.path.join(OUT, f"contract_{name}.npz"), clustering=cl.astype(np.uint32),
                            c_n=np.array([r["c_n"]]), c_xadj=r["c_xadj"], c_adjncy=r["c_adjncy"], c_vwgt=r["c_vwgt"],
                            c_adjwgt=r["c_adjwgt"], mapping=r["mapping"])
        print("wrote", name, g.n, g.m, "->", r["c_n"], len(r["c_adjncy"]))
    write_live_digests()


def write_live_digests():
    from oracle import contraction_oracle as CO
    from tests import test_contraction_oracle as T

    def ref_digest(g, cl, algorithm):
        return T.digest(CO.canonicalize(**B.ref_contract(g, cl, algorithm), clustering=cl))

    assert B.have_reference(), "build oracle/_ref first: make -C oracle ref"
    live = {"algorithm": {str(a): [ref_digest(g, cl, a) for g, cl in T.live_cases(a)] for a in (0, 1, 2)},
            "multigraphs": [ref_digest(g, cl, 1) for g, cl in T.multigraph_cases()]}
    with open(os.path.join(OUT, "contract_live_digests.json"), "w") as f:
        json.dump(live, f, indent=1)
    print("wrote contract_live_digests.json")


if __name__ == "__main__":
    main()
