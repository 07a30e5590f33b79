// The unmodified reference's ParHIP reader (kaminpar-io/parhip_parser.cc: io::parhip::read_graph without compression)
// as a program, for scripts/bench_parhip.py: reads the file given in the NodeOrdering given (0 NATURAL: csr_read,
// 2 EXTERNAL_DEGREE_BUCKETS: csr_read_deg_buckets), then prints one JSON line with the time of the read on a host
// clock and the graph's size. With a third argument it also writes the graph there for tests/test_parhip_bridge.py:
// six u64 (n, m, sorted, node weights kept, edge weights kept, permuted), then xadj, adjncy, vwgt, adjwgt and the permutation
// (map_original_node of every vertex) as 32-bit words, the absent ones left out; the reference's log lines go to its
// output as they do in the application. Built by parhip_read.mk into
// _ref/parhip_read in the Release build users run (-O3 -DNDEBUG).
#include <chrono>
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <vector>

#include "kaminpar-io/parhip_parser.h"
#include "kaminpar-shm/datastructures/graph.h"

#include "kaminpar-common/logger.h"

int main(int argc, char **argv) {
  if (argc != 3 && argc != 4) {
    std::fprintf(stderr, "usage: %s FILE.parhip ORDERING [DUMP]\n", argv[0]);
    return 2;
  }
  kaminpar::Logger::set_quiet_mode(argc == 3); // with a dump, its log lines (e.g. a refusal) are kept
  const auto ordering = static_cast<kaminpar::shm::NodeOrdering>(std::atoi(argv[2]));
  const auto t0 = std::chrono::steady_clock::now();
  const auto graph = kaminpar::shm::io::parhip::read_graph(argv[1], false, ordering);
  const auto t1 = std::chrono::steady_clock::now();
  if (!graph) {
    std::fprintf(stderr, "cannot read %s\n", argv[1]);
    return 1;
  }
  if (argc == 4) {
    const auto &g = kaminpar::shm::concretize<kaminpar::shm::CSRGraph>(*graph);
    std::FILE *f = std::fopen(argv[3], "wb");
    // the arrays as read: is_node_weighted() would say false for all-unit weights, which the reader keeps
    const bool vw = !g.raw_node_weights().empty(), ew = !g.raw_edge_weights().empty();
    const std::uint64_t head[6] = {g.n(), g.m(), g.sorted(), vw, ew, g.permuted()};
    std::fwrite(head, 8, 6, f);
    auto put = [f](const auto &a) { std::fwrite(a.data(), sizeof(a[0]), a.size(), f); };
    put(g.raw_nodes());
    put(g.raw_edges());
    if (vw) {
      put(g.raw_node_weights());
    }
    if (ew) {
      put(g.raw_edge_weights());
    }
    if (g.permuted()) {
      std::vector<std::uint32_t> perm(g.n());
      for (std::uint32_t u = 0; u < g.n(); ++u) {
        perm[u] = g.map_original_node(u);
      }
      put(perm);
    }
    std::fclose(f);
  }
  std::printf("{\"ms\": %.3f, \"n\": %llu, \"m\": %llu}\n", std::chrono::duration<double, std::milli>(t1 - t0).count(),
              static_cast<unsigned long long>(graph->n()), static_cast<unsigned long long>(graph->m()));
  return 0;
}
