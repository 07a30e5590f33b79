// Compiles against the C++ adapters + C ABI; used by tests/test_cpp_validate_adapter.py to check that
// kaminpar_b200::validate_graph and GraphReport are valid C++20 and link, and (with a GPU) that a weighted grid and
// three broken copies of it come back with the oracle's reports. Without a device it exits with status 1 and the
// adapter's error message.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "kaminpar_b200_adapters.hpp"

using namespace kaminpar_b200;

int main() {
  // 10x10 grid, edge weight 1 + (u + v) % 4 (symmetric)
  const int R = 10, C = 10;
  std::vector<EdgeID> xadj{0};
  std::vector<NodeID> adj;
  std::vector<EdgeWeight> ew;
  for (int r = 0; r < R; ++r) {
    for (int c = 0; c < C; ++c) {
      const NodeID u = r * C + c;
      const int dr[4] = {-1, 0, 0, 1}, dc[4] = {0, -1, 1, 0};
      for (int d = 0; d < 4; ++d) {
        const int rr = r + dr[d], cc = c + dc[d];
        if (rr >= 0 && rr < R && cc >= 0 && cc < C) {
          const NodeID v = rr * C + cc;
          adj.push_back(v);
          ew.push_back(1 + static_cast<EdgeWeight>((u + v) % 4));
        }
      }
      xadj.push_back(static_cast<EdgeID>(adj.size()));
    }
  }
  std::vector<std::vector<NodeID>> adjs{adj, adj, adj};
  std::vector<std::vector<EdgeWeight>> ews{ew, ew, ew};
  ews.push_back(ew);
  adjs.push_back(adj);
  adjs[1][37] = 99;                      // a missing reverse edge (and its partner's)
  adjs[2][adj.size() - 1] = R * C;        // a target out of range
  ews[3][50] += 3;                        // a weight that differs from its reverse edge's
  std::FILE *dump = nullptr;
  if (const char *path = std::getenv("ADAPTER_DUMP")) {
    dump = std::fopen(path, "w");
  }
  try {
    detail::Handle h(detail::balancer_config(EngineContext{}));
    for (std::size_t i = 0; i < adjs.size(); ++i) {
      const GraphReport r = validate_graph(h.get(), CSRGraphView{xadj, adjs[i], {}, ews[i]});
      if (r.is_valid() != (i == 0)) {
        return 2;
      }
      std::printf("graph %zu: %s\n", i, r.is_valid() ? "valid" : r.message().c_str());
      // ADAPTER_DUMP=<file>: per graph "xadj / adjncy / adjwgt / kind u e v e_rev v_rev w w_rev duplicates" and the
      // message, as text for the comparison with the oracle
      if (dump != nullptr) {
        auto line = [dump](const auto &v) {
          for (auto x : v) std::fprintf(dump, "%lld ", static_cast<long long>(x));
          std::fprintf(dump, "\n");
        };
        line(xadj);
        line(adjs[i]);
        line(ews[i]);
        std::fprintf(dump, "%d %u %u %u %u %u %d %d %u\n%s\n", r.kind, r.u, r.e, r.v, r.e_rev, r.v_rev, r.w, r.w_rev,
                     r.duplicates, r.message().c_str());
      }
    }
    std::printf("adapter ok\n");
  } catch (const std::exception &e) {
    std::printf("exception: %s\n", e.what());
    return 1;
  }
  if (dump != nullptr) {
    std::fclose(dump);
  }
  return 0;
}
