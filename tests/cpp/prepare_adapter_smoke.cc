// Compiles against the C++ adapters + C ABI; used by tests/test_cpp_prepare_adapter.py to check that
// kaminpar_b200::rearrange_by_degree_buckets, PreparedGraph and assign_isolated_nodes are valid C++20 and link, and
// (with a GPU) that a weighted grid with isolated vertices spread through its ids comes back from the device with the
// oracle's partition: from the handle's device labels and from a host partition alike. Without a device it exits with
// status 1 and the adapter's error message.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "kaminpar_b200_adapters.hpp"

using namespace kaminpar_b200;

int main() {
  // 12x12 grid; after every 5th grid vertex an isolated vertex; vertex weights 1 + u % 3
  const int R = 12, C = 12;
  std::vector<NodeID> id_of(R * C);
  NodeID n = 0;
  for (int i = 0; i < R * C; ++i) {
    id_of[i] = n++;
    if (i % 5 == 4) {
      ++n;
    }
  }
  std::vector<std::vector<NodeID>> nb(n);
  for (int r = 0; r < R; ++r) {
    for (int c = 0; c < C; ++c) {
      const int i = r * C + c;
      if (c + 1 < C) {
        nb[id_of[i]].push_back(id_of[i + 1]);
        nb[id_of[i + 1]].push_back(id_of[i]);
      }
      if (r + 1 < R) {
        nb[id_of[i]].push_back(id_of[i + C]);
        nb[id_of[i + C]].push_back(id_of[i]);
      }
    }
  }
  std::vector<EdgeID> xadj{0};
  std::vector<NodeID> adj;
  std::vector<NodeWeight> vw;
  for (NodeID u = 0; u < n; ++u) {
    adj.insert(adj.end(), nb[u].begin(), nb[u].end());
    xadj.push_back(static_cast<EdgeID>(adj.size()));
    vw.push_back(1 + static_cast<NodeWeight>(u % 3));
  }
  CSRGraphView g{xadj, adj, vw, {}};
  const BlockID k = 4;
  const std::vector<BlockWeight> mbw{70, 60, 75, 80}; // tight enough that next fit passes blocks
  try {
    detail::Handle h(detail::balancer_config(EngineContext{}));
    auto prepared = rearrange_by_degree_buckets(h.get(), g);
    if (prepared->n() != static_cast<NodeID>(R * C) || prepared->num_isolated() != n - R * C ||
        prepared->m() != g.m()) {
      return 2;
    }
    prepared->set_on(h.get());
    std::vector<BlockID> part(prepared->n());
    for (NodeID u = 0; u < prepared->n(); ++u) {
      part[u] = (u * 7) % k;
    }
    detail::check(kmp_lp_upload_partition(h.get(), part.data())); // the handle's device labels of this graph
    PartitionContextView p_ctx{k, mbw, {}, {}};
    std::vector<BlockWeight> bw(k), bw2(k);
    std::vector<BlockID> out(n), out2(n);
    assign_isolated_nodes(h.get(), *prepared, PartitionedGraphView{{}, k, {}, bw}, prepared->num_isolated(), p_ctx, out);
    assign_isolated_nodes(h.get(), *prepared, PartitionedGraphView{{}, k, part, bw2}, prepared->num_isolated(), p_ctx,
                          out2);
    if (out != out2 || bw != bw2) {
      return 3;
    }
    std::printf("adapter ok: n=%u n'=%u isolated=%u bw %d %d %d %d\n", n, prepared->n(), prepared->num_isolated(), bw[0],
                bw[1], bw[2], bw[3]);
    // ADAPTER_DUMP=<file>: "n m k", xadj, adjncy, vwgt, max block weights, old_to_new, partition of the prepared
    // vertices, the output partition and block weights, as text for the comparison with the oracle
    if (const char *path = std::getenv("ADAPTER_DUMP")) {
      if (std::FILE *f = std::fopen(path, "w")) {
        auto line = [f](const auto &v) {
          for (auto x : v) std::fprintf(f, "%lld ", static_cast<long long>(x));
          std::fprintf(f, "\n");
        };
        std::fprintf(f, "%u %u %u\n", n, g.m(), k);
        line(xadj);
        line(adj);
        line(vw);
        line(mbw);
        line(prepared->old_to_new());
        line(part);
        line(out);
        line(bw);
        std::fclose(f);
      }
    }
  } catch (const std::exception &e) {
    std::printf("exception: %s\n", e.what());
    return 1;
  }
  return 0;
}
