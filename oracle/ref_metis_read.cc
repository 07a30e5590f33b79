// The unmodified reference's METIS reader (kaminpar-io/metis_parser.cc: io::metis::read_graph, i.e. csr_read,
// unsorted) as a program, for scripts/bench_metis.py: reads the file given, then prints one JSON line with the time of
// the read on a host clock and the graph's size. Built by metis_read.mk into _ref/metis_read in the Release build
// users run (-O3 -DNDEBUG).
#include <chrono>
#include <cstdio>

#include "kaminpar-io/metis_parser.h"
#include "kaminpar-shm/datastructures/graph.h"

#include "kaminpar-common/logger.h"

int main(int argc, char **argv) {
  if (argc != 2) {
    std::fprintf(stderr, "usage: %s FILE.metis\n", argv[0]);
    return 2;
  }
  kaminpar::Logger::set_quiet_mode(true);
  const auto t0 = std::chrono::steady_clock::now();
  const auto graph = kaminpar::shm::io::metis::read_graph(argv[1], false, kaminpar::shm::NodeOrdering::NATURAL);
  const auto t1 = std::chrono::steady_clock::now();
  if (!graph) {
    std::fprintf(stderr, "cannot read %s\n", argv[1]);
    return 1;
  }
  std::printf("{\"ms\": %.3f, \"n\": %llu, \"m\": %llu}\n", std::chrono::duration<double, std::milli>(t1 - t0).count(),
              static_cast<unsigned long long>(graph->n()), static_cast<unsigned long long>(graph->m()));
  return 0;
}
