// Compiles against the C++ adapters + C ABI; used by tests/test_cpp_overlay_adapter.py to check that
// kaminpar_b200::LPClustering::compute_overlay_clustering is valid C++20 and links, and (with a GPU) that it returns the
// overlay of the clusterer's consecutive calls, left on the device for contract_clustering. Without a device it exits
// with status 1 and the adapter's error message.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "kaminpar_b200_adapters.hpp"

using namespace kaminpar_b200;

int main() {
  // 24x24 grid with unit weights
  const int R = 24, C = 24;
  std::vector<EdgeID> xadj{0};
  std::vector<NodeID> adj;
  for (int r = 0; r < R; ++r) {
    for (int c = 0; c < C; ++c) {
      const NodeID u = r * C + c;
      if (r > 0) adj.push_back(u - C);
      if (c > 0) adj.push_back(u - 1);
      if (c + 1 < C) adj.push_back(u + 1);
      if (r + 1 < R) adj.push_back(u + C);
      xadj.push_back(static_cast<EdgeID>(adj.size()));
    }
  }
  CSRGraphView g{xadj, adj, {}, {}};
  try {
    // the same configuration twice: `plain` computes the calls one by one, `overlay` intersects them on the device
    LPClustering plain(LabelPropagationCoarseningContext{}), overlay(LabelPropagationCoarseningContext{});
    plain.set_max_cluster_weight(6);
    overlay.set_max_cluster_weight(6);
    const int levels = 2;
    std::vector<std::vector<NodeID>> calls(1 << levels, std::vector<NodeID>(g.n()));
    for (auto &c : calls) {
      plain.compute_clustering(c, g, false);
    }
    std::vector<NodeID> ov(g.n());
    overlay.compute_overlay_clustering(ov, g, levels, false);
    const kmp_overlay_stats st = overlay.last_overlay_stats();
    auto coarse = contract_clustering(overlay.handle(), {}); // the overlay left on the device
    if (st.num_clusterings != (1u << levels) || coarse->n() != st.num_clusters) {
      return 2;
    }
    std::printf("adapter ok: n=%u clusterings=%u overlay classes=%u sort bits=%u\n", g.n(), st.num_clusterings,
                st.num_clusters, st.sort_bits);
    // ADAPTER_DUMP=<file>: one line per LP call, then the overlay, as text
    if (const char *path = std::getenv("ADAPTER_DUMP")) {
      if (std::FILE *f = std::fopen(path, "w")) {
        auto line = [f](const auto &v) {
          for (auto x : v) std::fprintf(f, "%lld ", static_cast<long long>(x));
          std::fprintf(f, "\n");
        };
        for (const auto &c : calls) line(c);
        line(ov);
        std::fclose(f);
      }
    }
  } catch (const std::exception &e) {
    std::printf("exception: %s\n", e.what());
    return 1;
  }
  return 0;
}
