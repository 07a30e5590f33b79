// Compiles against the C++ adapters + C ABI; used by tests/test_cpp_sparsify_adapter.py to check that
// kaminpar_b200::sparsification_target and CoarseGraph::sparsify are valid C++20 and link, and (with a GPU) that a
// level clustered, contracted and sparsified through them gives the oracle's coarse graph, with get() returning the
// sparsified graph rather than the copy it cached before. Without a device it exits with status 1 and the adapter's
// error message.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "kaminpar_b200_adapters.hpp"

using namespace kaminpar_b200;

int main() {
  // 16x16 grid, symmetric edge weights 1 + (u + v) % 5
  const int R = 16, C = 16;
  std::vector<EdgeID> xadj{0};
  std::vector<NodeID> adj;
  std::vector<EdgeWeight> ew;
  auto add = [&](NodeID u, NodeID v) {
    adj.push_back(v);
    ew.push_back(1 + static_cast<EdgeWeight>((u + v) % 5));
  };
  for (int r = 0; r < R; ++r) {
    for (int c = 0; c < C; ++c) {
      const NodeID u = r * C + c;
      if (r > 0) add(u, u - C);
      if (c > 0) add(u, u - 1);
      if (c + 1 < C) add(u, u + 1);
      if (r + 1 < R) add(u, u + C);
      xadj.push_back(static_cast<EdgeID>(adj.size()));
    }
  }
  CSRGraphView g{xadj, adj, {}, ew};
  const std::uint64_t seed = 0x9E3779B97F4A7C15ull;
  try {
    LPClustering clusterer(LabelPropagationCoarseningContext{});
    clusterer.set_max_cluster_weight(4);
    std::vector<NodeID> clustering(g.n());
    clusterer.compute_clustering(clustering, g, false);
    auto coarse = contract_clustering(clusterer.handle(), {}); // the clustering left on the device
    const auto before = coarse->get();                        // cached host copy of the contracted graph
    const EdgeID formula = sparsification_target(g.m(), g.n(), coarse->n(), 0.5, 0.5);
    if (formula != kmp_sparsification_target(g.m(), g.n(), coarse->n(), 0.5, 0.5)) return 2;
    const EdgeID target = formula < coarse->m() ? formula : coarse->m();
    const kmp_sparsify_stats st = coarse->sparsify(clusterer.handle(), target, seed);
    const auto &after = coarse->get();
    if (st.c_m_after != coarse->m() || after.edges.size() != st.c_m_after || after.nodes.back() != st.c_m_after) {
      return 3;
    }
    std::printf("adapter ok: n=%u c_n=%u c_m %zu -> %u (target %u, T %d)\n", g.n(), coarse->n(), before.edges.size(),
                st.c_m_after, target, st.threshold);
    // ADAPTER_DUMP=<file>: "n m c_n target formula, xadj, adjncy, adjwgt, clustering, seed, then the sparsified coarse
    // xadj, adjncy, adjwgt, vwgt" as text, for the comparison with the oracle
    if (const char *path = std::getenv("ADAPTER_DUMP")) {
      if (std::FILE *f = std::fopen(path, "w")) {
        auto line = [f](const auto &v) {
          for (auto x : v) std::fprintf(f, "%lld ", static_cast<long long>(x));
          std::fprintf(f, "\n");
        };
        std::fprintf(f, "%u %u %u %u %u\n", g.n(), g.m(), coarse->n(), target, formula);
        line(xadj);
        line(adj);
        line(ew);
        line(clustering);
        std::fprintf(f, "%llu\n", static_cast<unsigned long long>(seed));
        line(after.nodes);
        line(after.edges);
        line(after.edge_weights);
        line(after.node_weights);
        std::fclose(f);
      }
    }
  } catch (const std::exception &e) {
    std::printf("exception: %s\n", e.what());
    return 1;
  }
  return 0;
}
