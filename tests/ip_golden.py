"""The pinned reference bipartitions tests/golden/ip_*.npz (tests/golden/make_ip_golden.py) as cases."""
import glob
import os

import numpy as np

from kaminpar_b200.bipartition import IPConfig
from kaminpar_b200.graph import CSRGraph

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def files():
    return sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(GOLDEN, "ip_*.npz")))


def cases(name):
    """[(case id, graph, part, k, k_prime, input_k, uniform, eps, seed, mbw, IPConfig, sub)] of one file."""
    d = np.load(os.path.join(GOLDEN, name + ".npz"))
    out, i = [], 0
    while "c%d_sub" % i in d.files:
        c = "c%d_" % i
        gk = c if c + "xadj" in d.files else ""
        g = CSRGraph(xadj=d[gk + "xadj"], adjncy=d[gk + "adjncy"],
                     vwgt=d[gk + "vwgt"] if gk + "vwgt" in d.files else None,
                     adjwgt=d[gk + "adjwgt"] if gk + "adjwgt" in d.files else None)
        k, k_prime, input_k, uniform, seed = (int(x) for x in d[c + "ints"])
        cfg = IPConfig.from_buffer_copy(d[c + "cfg"].tobytes())
        out.append(("%s-c%d" % (name, i), g, d[c + "part"], k, k_prime, input_k, bool(uniform), float(d[c + "eps"][0]),
                    seed, d[c + "mbw"], cfg, d[c + "sub"]))
        i += 1
    return out


def recorded_defaults():
    return IPConfig.from_buffer_copy(np.load(os.path.join(GOLDEN, "ip_rgg2d.npz"))["defaults"].tobytes())
