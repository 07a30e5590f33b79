// Compiles against the C++ adapters + C ABI; used by tests/test_cpp_subgraph_adapter.py to check that
// kaminpar_b200::extract_subgraphs, Subgraphs and copy_subgraph_partitions are valid C++20 and link, and (with a GPU)
// that a weighted grid's four blocks and the 8-way copy-back come back from the device: from a host partition and from
// the handle's device labels alike. Without a device it exits with status 1 and the adapter's error message.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "kaminpar_b200_adapters.hpp"

using namespace kaminpar_b200;

int main() {
  const NodeID R = 10, C = 13, n = R * C;
  std::vector<EdgeID> xadj{0};
  std::vector<NodeID> adj;
  std::vector<NodeWeight> vw;
  std::vector<EdgeWeight> ew;
  for (NodeID u = 0; u < n; ++u) {
    const NodeID c = u % C;
    for (const long long v : {(long long)u - C, (long long)u - 1, (long long)u + 1, (long long)u + C}) {
      if (v < 0 || v >= n || (v == u - 1 && c == 0) || (v == u + 1 && c + 1 == C)) {
        continue;
      }
      adj.push_back(static_cast<NodeID>(v));
      ew.push_back(1 + static_cast<EdgeWeight>((u + v) % 4));
    }
    xadj.push_back(static_cast<EdgeID>(adj.size()));
    vw.push_back(1 + static_cast<NodeWeight>(u % 3));
  }
  CSRGraphView g{xadj, adj, vw, ew};
  const BlockID k = 4, k_prime = 8;
  std::vector<BlockID> part(n);
  for (NodeID u = 0; u < n; ++u) {
    part[u] = (u * 5 + u / 7) % k;
  }
  try {
    detail::Handle h(detail::balancer_config(EngineContext{}));
    h.set_graph(g);
    auto sg = extract_subgraphs(h.get(), k, part);
    const auto &host = sg->get();
    if (sg->k() != k || sg->n() != n || host.node_offsets[k] != n || host.edge_offsets[k] != sg->m()) {
      return 2;
    }
    detail::check(kmp_lp_upload_partition(h.get(), part.data()));
    auto sg2 = extract_subgraphs(h.get(), k); // the handle's device labels
    if (sg2->get().edges != host.edges || sg2->get().nodes != host.nodes || sg2->get().mapping != host.mapping) {
      return 3;
    }
    std::vector<BlockID> sub(n), out(n);
    for (BlockID b = 0; b < k; ++b) {
      const CSRGraphView blk = sg->block(b);
      for (NodeID i = 0; i < blk.n(); ++i) {
        sub[host.node_offsets[b] + i] = i < blk.n() / 2 ? 0 : 1;
      }
    }
    copy_subgraph_partitions(h.get(), *sg, sub, k_prime, k_prime, out);
    std::printf("adapter ok: n=%u m_internal=%u blocks %u %u %u %u\n", n, sg->m(), host.node_offsets[1],
                host.node_offsets[2] - host.node_offsets[1], host.node_offsets[3] - host.node_offsets[2],
                n - host.node_offsets[3]);
    // ADAPTER_DUMP=<file>: "n k k'", xadj, adjncy, vwgt, adjwgt, partition, then the device's block xadj (n + k),
    // adjncy, mapping, block_nodes, sub-partitions and the k'-way output, as text for the comparison with the oracle
    if (const char *path = std::getenv("ADAPTER_DUMP")) {
      if (std::FILE *f = std::fopen(path, "w")) {
        auto line = [f](const auto &v) {
          for (auto x : v) std::fprintf(f, "%lld ", static_cast<long long>(x));
          std::fprintf(f, "\n");
        };
        std::fprintf(f, "%u %u %u\n", n, k, k_prime);
        line(xadj);
        line(adj);
        line(vw);
        line(ew);
        line(part);
        line(host.nodes);
        line(host.edges);
        line(host.mapping);
        line(host.block_nodes);
        line(sub);
        line(out);
        std::fclose(f);
      }
    }
  } catch (const std::exception &e) {
    std::printf("exception: %s\n", e.what());
    return 1;
  }
  return 0;
}
