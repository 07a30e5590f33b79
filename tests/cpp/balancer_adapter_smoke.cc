// Compiles against the C++ balancer adapters + C ABI; used by tests/test_cpp_balancer_adapter.py to check that the
// header is valid C++20, that the library links, and (with a GPU) that OverloadBalancer and UnderloadBalancer give
// the oracle's results. Without a device it exits with status 1 and the adapter's error message.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "kaminpar_b200_adapters.hpp"

using namespace kaminpar_b200;

int main() {
  // 12x12 grid, k = 4, unit weights: total 144, perfectly balanced 36
  const int R = 12, C = 12;
  const BlockID k = 4;
  std::vector<EdgeID> xadj{0};
  std::vector<NodeID> adj;
  for (int r = 0; r < R; ++r) {
    for (int c = 0; c < C; ++c) {
      if (r > 0) adj.push_back((r - 1) * C + c);
      if (c > 0) adj.push_back(r * C + c - 1);
      if (c + 1 < C) adj.push_back(r * C + c + 1);
      if (r + 1 < R) adj.push_back((r + 1) * C + c);
      xadj.push_back(static_cast<EdgeID>(adj.size()));
    }
  }
  CSRGraphView g{xadj, adj, {}, {}};
  std::vector<BlockWeight> maxw(k, 37), minw(k, 35), pbw(k, 36);
  // quadrants, then the first 12 vertices of quadrant 1 moved into quadrant 0: block 0 overloaded, block 1 underloaded
  std::vector<BlockID> part(g.n()), input(g.n());
  for (NodeID u = 0; u < g.n(); ++u) {
    const int r = static_cast<int>(u) / C, c = static_cast<int>(u) % C;
    part[u] = (r < R / 2 ? 0 : 2) + (c < C / 2 ? 0 : 1);
  }
  for (NodeID u = 0, moved = 0; u < g.n() && moved < 12; ++u) {
    if (part[u] == 1) {
      part[u] = 0;
      ++moved;
    }
  }
  input = part;
  std::vector<BlockWeight> bw(k, 0);
  for (BlockID b : part) ++bw[b];
  try {
    PartitionedGraphView pg{g, k, part, bw};
    OverloadBalancer over;
    if (over.name() != "Overload Balancer") return 2;
    over.initialize(pg);
    const bool improved_over = over.refine(pg, PartitionContextView{k, maxw, {}, pbw});
    std::vector<BlockID> after_over = part;
    std::vector<BlockWeight> bw_over = bw;
    // then make block 3 underloaded by moving 6 of its vertices into block 2, and restore the minimum weights
    for (NodeID u = 0, moved = 0; u < g.n() && moved < 6; ++u) {
      if (part[u] == 3) {
        part[u] = 2;
        --bw[3];
        ++bw[2];
        ++moved;
      }
    }
    std::vector<BlockID> under_in = part;
    UnderloadBalancer under;
    if (under.name() != "Underload Balancer") return 3;
    under.initialize(pg);
    if (under.refine(pg, PartitionContextView{k, maxw, {}, pbw})) return 4; // no minimum weights: nothing to do
    const bool improved_under = under.refine(pg, PartitionContextView{k, maxw, minw, pbw});
    std::printf("adapter ok: overload %d, underload %d, block weights %d/%d/%d/%d\n", improved_over, improved_under,
                bw[0], bw[1], bw[2], bw[3]);
    // ADAPTER_DUMP=<file>: "n m, xadj, adjncy, overload input, its result, underload input, its result, block weights
    // after each, the two return values" as text, for the comparison with the oracle
    if (const char *path = std::getenv("ADAPTER_DUMP")) {
      if (std::FILE *f = std::fopen(path, "w")) {
        auto line = [f](const auto &v) {
          for (auto x : v) std::fprintf(f, "%lld ", static_cast<long long>(x));
          std::fprintf(f, "\n");
        };
        std::fprintf(f, "%u %u\n", g.n(), g.m());
        line(xadj);
        line(adj);
        line(input);
        line(after_over);
        line(under_in);
        line(part);
        line(bw_over);
        line(bw);
        std::fprintf(f, "%d %d\n", improved_over ? 1 : 0, improved_under ? 1 : 0);
        std::fclose(f);
      }
    }
  } catch (const std::exception &e) {
    std::printf("exception: %s\n", e.what());
    return 1;
  }
  return 0;
}
