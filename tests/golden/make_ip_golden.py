"""Generator of tests/golden/ip_*.npz: the UNMODIFIED reference's initial bipartitions of extracted blocks (called
through tests/cpp/ref_ip_bridge.cc), pinned for machines without the reference (tests/test_ip_oracle.py on the CPU,
tests/test_gpu_bipartition.py G0 on the GPU). Needs the reference and oracle/_ref/libkaminpar_ref_full.so.

Each file holds the graph (xadj, adjncy, optional vwgt / adjwgt; per case as c<i>_xadj ... where the cases differ in
it) and cases c0, c1, ...: the partition, k, k', input_k,
uniform, epsilon, seed, the input's maximum block weights, the kmp_ip_config bytes, and the reference's block-major
sub-partitions under DESIGN.md §20's rule (block b: Random::reseed(seed + b), a fresh pool, bipartition(b, k)).
`defaults` holds the default preset's kmp_ip_config bytes as the reference reports them.

    python tests/golden/make_ip_golden.py
"""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from kaminpar_b200.bipartition import TWOWAY_ADAPTIVE_FM, IPConfig, preset  # noqa: E402
from kaminpar_b200.graph import CSRGraph, random_weights, rmat  # noqa: E402
from tests import ip_host as IH  # noqa: E402
from tests import subgraph_oracle as S  # noqa: E402
from tests.test_ip_bridge import components, heavy, star  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
P = IH._p


def bridge():
    L = C.CDLL(IH.build_bridge())
    args = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_int, C.c_int32, C.c_double, C.c_uint32, C.c_uint32, C.c_uint32,
            C.c_uint32] + [C.c_void_p] * 4
    L.ref_ip_bipartition.argtypes = args + [C.c_int32, C.c_void_p]
    L.ref_ip_preset_config.argtypes = [C.c_char_p, C.c_void_p]
    return L


def config(name):
    if name == "adaptive":
        c = preset("default")
        c.refinement.algorithm = c.pool_refinement.algorithm = TWOWAY_ADAPTIVE_FM
        return c
    return preset(name)


def ref_sub(L, g, part, k, k_prime, input_k, mbw, seed, cfg, uniform, eps):
    res = S.lazy_extract(g.xadj, g.adjncy, g.vwgt, g.adjwgt, part, k)
    total = int(g.vwgt.sum()) if g.vwgt is not None else g.n
    sub = np.zeros(g.n, np.uint32)
    for b in range(k):
        s_b = IH.lib().ip_compute_final_k(b, k, input_k) if k_prime == input_k else k_prime // k
        bx, ba, bv, be = IH.block_arrays(res, b)
        nb = len(bx) - 1
        if s_b != 2 or nb == 0:
            continue
        out = np.zeros(nb, np.uint32)
        L.ref_ip_bipartition(C.byref(cfg), input_k, P(mbw), int(uniform), total, eps, b, k, nb, len(ba), P(bx),
                             P(ba), P(bv), P(be), int(np.int32(np.uint32(seed + b))), P(out))
        sub[int(res["node_off"][b]):int(res["node_off"][b + 1])] = out
    return sub


def golden_graph(name):
    d = np.load(os.path.join(OUT, name + ".npz"))
    return CSRGraph(xadj=d["xadj"], adjncy=d["adjncy"], vwgt=d["vwgt"] if "vwgt" in d.files else None,
                    adjwgt=d["adjwgt"] if "adjwgt" in d.files else None)


# (file, graph, [(k, k_prime, input_k, partition kind, preset, uniform)])
def cases():
    presets = ["default", "fast", "largek", "largek-fast", "adaptive"]
    big = [(1, 2, 2, "range", "default", True), (2, 4, 8, "range", "fast", False), (4, 8, 8, "random", "largek", True),
           (4, 7, 7, "range", "largek-fast", False), (8, 16, 48, "random", "adaptive", True),
           (2, 3, 3, "range", "default", False), (8, 12, 12, "range", "largek", True)]
    yield "ip_rgg2d", golden_graph("graph_rgg2d"), big
    yield "ip_walshaw", golden_graph("graph_walshaw_data"), big
    yield "ip_rmat13", random_weights(rmat(13, 8, seed=3), 3, max_vwgt=0, max_adjwgt=0), big[:5]
    yield "ip_rgg16w", golden_graph("graph_rgg16_vwgt_adjwgt"), [(1, 2, 2, "range", p, u) for p in presets
                                                                 for u in (True, False)]
    small = [(1, 2, 2, "range", p, True) for p in presets]
    yield "ip_star", star(3000), small + [(2, 4, 6, "range", "default", False)]
    yield "ip_components", components(40, 7), small
    yield "ip_heavy", heavy(rmat(10, 8, seed=5)), small + [(2, 4, 4, "range", "default", False)]
    tiny2 = CSRGraph(xadj=np.array([0, 1, 2], np.uint32), adjncy=np.array([1, 0], np.uint32))
    tiny1 = CSRGraph(xadj=np.zeros(2, np.uint32), adjncy=np.zeros(0, np.uint32))
    yield "ip_tiny", None, [("n2", tiny2), ("n1", tiny1)]
    yield "ip_manyblocks", rmat(10, 4, seed=7), [(64, 128, 128, "random", "default", True),
                                                 (64, 100, 100, "random", "fast", False)]


def main():
    L = bridge()
    defaults = IPConfig()
    L.ref_ip_preset_config(b"default", C.byref(defaults))
    for fname, g0, specs in cases():
        out = {"defaults": np.frombuffer(bytes(defaults), np.uint8)}
        for i, spec in enumerate(specs):
            if g0 is None:
                g, (k, k_prime, input_k, kind, pname, uniform) = spec[1], (1, 2, 2, "range", "default", True)
            else:
                g, (k, k_prime, input_k, kind, pname, uniform) = g0, spec
            rng = np.random.default_rng(i)
            part = ((np.arange(g.n, dtype=np.int64) * k // g.n) if kind == "range" else
                    rng.integers(0, k, g.n)).astype(np.uint32)
            eps, seed = 0.03, 1000 + i
            total = int(g.vwgt.sum()) if g.vwgt is not None else g.n
            mbw = IH.max_block_weights(total, input_k, eps, uniform, i)
            cfg = config(pname)
            sub = ref_sub(L, g, part, k, k_prime, input_k, mbw, seed, cfg, uniform, eps)
            c = "c%d_" % i
            out.update({c + "part": part, c + "mbw": mbw, c + "sub": sub,
                        c + "cfg": np.frombuffer(bytes(cfg), np.uint8),
                        c + "ints": np.array([k, k_prime, input_k, int(uniform), seed], np.int64),
                        c + "eps": np.array([eps])})
            if g0 is None or i == 0:  # the graph: once per file, or per case where the cases differ in it
                gk = c if g0 is None else ""
                out.update({gk + "xadj": g.xadj, gk + "adjncy": g.adjncy})
                if g.vwgt is not None:
                    out[gk + "vwgt"] = g.vwgt
                if g.adjwgt is not None:
                    out[gk + "adjwgt"] = g.adjwgt
        np.savez_compressed(os.path.join(OUT, fname + ".npz"), **out)
        print(fname, len(specs), "cases")


if __name__ == "__main__":
    main()
