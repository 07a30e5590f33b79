"""Generator of tests/golden/subgraph_*.npz: outputs of the UNMODIFIED reference's subgraph extraction, copy-back and
compute_final_k (through tests/cpp/ref_subgraph_bridge.cc, serial oneTBB stand-in), pinned for machines without the
reference. tests/test_subgraph_oracle.py holds the NumPy oracle to them.

    python tests/golden/make_subgraph_golden.py      (needs the reference and oracle/_ref/libkaminpar_ref_full.so)
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from tests import test_subgraph_bridge as TB  # noqa: E402

PINNED = ("walshaw_k16", "rmat12_w_k8", "empty_blocks", "k_gt_n", "path_cut")
FINAL_K_INPUTS = (3, 11, 37, 1000, 10000)


def main():
    if not TB.reference_present():
        raise SystemExit("the reference and oracle/_ref/libkaminpar_ref_full.so are needed")
    lib = TB.compile_bridge(tempfile.mkdtemp())
    for name, g, k, part in TB.CASES:
        if name not in PINNED:
            continue
        ref = TB.ref_lazy(lib, g, part, k)
        d = dict(xadj=g.xadj, adjncy=g.adjncy, k=np.array([k], np.uint32), partition=part)
        if g.vwgt is not None:
            d["vwgt"] = g.vwgt
        if g.adjwgt is not None:
            d["adjwgt"] = g.adjwgt
        for key in ("node_off", "edge_off", "block_nodes", "mapping", "xadj", "adjncy", "vwgt", "adjwgt"):
            if ref[key] is not None:
                d["ref_" + key] = ref[key]
        for i, (k_prime, input_k) in enumerate(((2 * k, 8 * k), (k, k))):
            sub = TB._subs(ref, k, k_prime, input_k, 100 + i)
            d[f"copy{i}_args"] = np.array([k_prime, input_k], np.uint32)
            d[f"copy{i}_sub"] = sub
            d[f"copy{i}_out"] = TB.ref_copy_back(lib, g, part, k, k_prime, input_k, sub)
        np.savez_compressed(os.path.join(HERE, f"subgraph_{name}.npz"), **d)
        print("wrote", name)
    d = {f"final_k_{ik}": TB.ref_final_k(lib, ik) for ik in FINAL_K_INPUTS}
    np.savez_compressed(os.path.join(HERE, "subgraph_final_k.npz"), **d)
    print("wrote final_k")


if __name__ == "__main__":
    main()
