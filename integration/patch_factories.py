#!/usr/bin/env python
"""Generate the ONE change a maintainer makes to the reference: kaminpar-shm/factories.cc with the two
LABEL_PROPAGATION cases (factories.cc:66-67, :108-109) returning the GPU glue classes. The patched copy is
written to a build directory (never committed; the reference source is read where it lies).

    python integration/patch_factories.py /root/reference/kaminpar-shm/factories.cc oracle/_ref/gen/factories_b200.cc
"""
import sys


def main(src, dst):
    s = open(src).read()
    a = "return std::make_unique<LPClustering>(ctx.coarsening);"
    b = "return std::make_unique<LabelPropagationRefiner>(ctx);"
    assert s.count(a) == 1 and s.count(b) == 1, "factories.cc does not look like v3.7.3"
    s = s.replace(a, "return std::make_unique<B200LPClustering>(ctx.coarsening);")
    s = s.replace(b, "return std::make_unique<B200LabelPropagationRefiner>(ctx);")
    inc = '#include "kaminpar-shm/factories.h"\n'
    assert s.count(inc) == 1
    s = s.replace(inc, inc + '\n#include "b200_lp_clusterer.h"\n#include "b200_lp_refiner.h"\n')
    open(dst, "w").write(s)


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
