"""Generate the overlay goldens tests/golden/overlay_*.npz (run in the authoring container only).

Each file holds a graph and four consecutive clusterings that the UNMODIFIED reference's LPClustering computed on one
object (one thread, oracle/_ref/libkaminpar_ref.so, `make -C oracle ref`): the clusterings OverlayClusterCoarsener
intersects with num_levels = 2 (DESIGN.md §14). tests/test_gpu_overlay.py checks the seq_strict overlay against the
overlay oracle of these clusterings. The graphs are read from the reference checkout's data files (graphs, not source
code) and sorted by degree buckets as the reference's partitioner feeds its finest level.

    python tests/golden/make_overlay_golden.py
"""
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from kaminpar_b200.graph import CSRGraph, read_metis  # noqa: E402
from oracle import bindings as B  # noqa: E402

REF = "/root/reference"
OUT = os.path.dirname(os.path.abspath(__file__))
NUM_CALLS = 4


def walshaw_data() -> CSRGraph:
    xs = open(f"{REF}/tests/endtoend/data.graph.xadj").read()
    ad = open(f"{REF}/tests/endtoend/data.graph.adjncy").read()
    return CSRGraph(np.array([int(t) for t in re.findall(r"\d+", xs)], np.uint32),
                    np.array([int(t) for t in re.findall(r"\d+", ad)], np.uint32))


def main():
    assert B.have_reference(), "build oracle/_ref first: make -C oracle ref"
    cases = [("walshaw", walshaw_data(), 16, 7),  # (name, graph, k of the max cluster weight, seed)
             ("rgg2d", read_metis(f"{REF}/misc/rgg2d.metis"), 8, 3)]
    for name, g0, k, seed in cases:
        g, _ = B.ref_rearrange(g0)
        mcw = B.ref_max_cluster_weight(g, k)
        out = {"xadj": g.xadj, "adjncy": g.adjncy, "buckets": g.buckets, "seed": np.array([seed]),
               "max_cluster_weight": np.array([mcw]),
               "clusterings": B.ref_lp_cluster(g, seed, mcw, num_calls=NUM_CALLS)}
        np.savez_compressed(os.path.join(OUT, f"overlay_{name}.npz"), **out)
        print("wrote", name, g.n, g.m)


if __name__ == "__main__":
    main()
