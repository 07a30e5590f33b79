// Bridge to the UNMODIFIED reference's subgraph extraction and copy-back, for the CPU tests of
// tests/test_subgraph_bridge.py and the generator tests/golden/make_subgraph_golden.py. Compiled against the reference
// headers and linked against the reference partitioner the build leaves in oracle/_ref/libkaminpar_ref_full.so (serial
// oneTBB stand-in: one thread, so every parallel_for runs in ascending index order).
#include <cstdint>
#include <cstring>
#include <memory>
#include <vector>

#include "kaminpar-shm/datastructures/csr_graph.h"
#include "kaminpar-shm/datastructures/graph.h"
#include "kaminpar-shm/datastructures/partitioned_graph.h"
#include "kaminpar-shm/graphutils/subgraph_extractor.h"
#include "kaminpar-shm/kaminpar.h"
#include "kaminpar-shm/partitioning/partition_utils.h"

#include "kaminpar-common/datastructures/static_array.h"
#include "kaminpar-common/timer.h"

using namespace kaminpar;
using namespace kaminpar::shm;

namespace {
template <typename T> StaticArray<T> copy_array(const T *src, std::size_t n) {
  StaticArray<T> a(n);
  if (n > 0) {
    std::memcpy(a.data(), src, n * sizeof(T));
  }
  return a;
}

Graph make_graph(std::uint32_t n, std::uint32_t m, const std::uint32_t *xadj, const std::uint32_t *adjncy,
                 const std::int32_t *vwgt, const std::int32_t *adjwgt) {
  return Graph(std::make_unique<CSRGraph>(
      copy_array<EdgeID>(xadj, static_cast<std::size_t>(n) + 1), copy_array<NodeID>(adjncy, m),
      vwgt ? copy_array<NodeWeight>(vwgt, n) : StaticArray<NodeWeight>(),
      adjwgt ? copy_array<EdgeWeight>(adjwgt, m) : StaticArray<EdgeWeight>()
  ));
}

// appends block b's graph to the n + k layout: xadj at node_off[b] + b, adjncy / adjwgt at *edge_cursor
void append_block(const Graph &sub, std::uint32_t node_base, std::uint32_t b, std::uint32_t *edge_cursor,
                  std::uint32_t *xadj_out, std::uint32_t *adjncy_out, std::int32_t *vwgt_out,
                  std::int32_t *adjwgt_out, std::int32_t *weighted_out) {
  const CSRGraph &csr = sub.csr_graph();
  const NodeID nb = csr.n();
  const EdgeID mb = csr.m();
  for (NodeID i = 0; i <= nb; ++i) {
    xadj_out[node_base + b + i] = csr.raw_nodes()[i];
  }
  for (EdgeID e = 0; e < mb; ++e) {
    adjncy_out[*edge_cursor + e] = csr.raw_edges()[e];
    if (csr.is_edge_weighted()) {
      adjwgt_out[*edge_cursor + e] = csr.raw_edge_weights()[e];
    }
  }
  if (csr.is_node_weighted()) {
    for (NodeID i = 0; i < nb; ++i) {
      vwgt_out[node_base + i] = csr.raw_node_weights()[i];
    }
  }
  weighted_out[0] |= csr.is_node_weighted() ? 1 : 0;
  weighted_out[1] |= csr.is_edge_weighted() ? 1 : 0;
  *edge_cursor += mb;
}
} // namespace

extern "C" {

// graph::lazy_extract_subgraphs_preprocessing + graph::extract_subgraph for every block, as
// extend_partition_lazy_extraction calls them (partitioning/helper.cc:254-315). Outputs: node_off[k+1],
// block_nodes[n], mapping[n], edge_off[k+1], xadj[n+k], adjncy[m], vwgt[n], adjwgt[m] and weighted[2] (whether the
// subgraphs carry node / edge weights).
int bridge_lazy_extract(std::uint32_t n, std::uint32_t m, const std::uint32_t *xadj, const std::uint32_t *adjncy,
                        const std::int32_t *vwgt, const std::int32_t *adjwgt, std::uint32_t k,
                        const std::uint32_t *partition, std::uint32_t *node_off, std::uint32_t *block_nodes,
                        std::uint32_t *mapping, std::uint32_t *edge_off, std::uint32_t *xadj_out,
                        std::uint32_t *adjncy_out, std::int32_t *vwgt_out, std::int32_t *adjwgt_out,
                        std::int32_t *weighted_out) {
  DISABLE_TIMERS();
  Graph graph = make_graph(n, m, xadj, adjncy, vwgt, adjwgt);
  PartitionedGraph p_graph(graph, k, copy_array<BlockID>(partition, n));
  auto pre = graph::lazy_extract_subgraphs_preprocessing(p_graph);
  for (std::uint32_t b = 0; b <= k; ++b) {
    node_off[b] = pre.block_nodes_offset[b];
  }
  for (NodeID u = 0; u < n; ++u) {
    block_nodes[u] = pre.block_nodes[u];
    mapping[u] = pre.mapping[u];
  }
  graph::SubgraphMemory memory(p_graph);
  std::uint32_t cursor = 0;
  weighted_out[0] = weighted_out[1] = 0;
  for (BlockID b = 0; b < k; ++b) {
    const NodeID nb = pre.block_nodes_offset[b + 1] - pre.block_nodes_offset[b];
    const StaticArray<NodeID> local(nb, pre.block_nodes.data() + pre.block_nodes_offset[b]);
    const Graph sub = graph::extract_subgraph(p_graph, b, local, pre.mapping, memory);
    if (sub.m() != pre.block_num_edges[b]) {
      return -1;
    }
    edge_off[b] = cursor;
    append_block(sub, pre.block_nodes_offset[b], b, &cursor, xadj_out, adjncy_out, vwgt_out, adjwgt_out,
                 weighted_out);
  }
  edge_off[k] = cursor;
  return 0;
}

// graph::extract_subgraphs (the non-lazy path of RBMultilevelPartitioner): every subgraph and node_mapping, written
// into the same n + k layout (the reference's padding slots between blocks are not part of a block's graph).
// node_off must hold the block offsets (from bridge_lazy_extract).
int bridge_extract_subgraphs(std::uint32_t n, std::uint32_t m, const std::uint32_t *xadj, const std::uint32_t *adjncy,
                             const std::int32_t *vwgt, const std::int32_t *adjwgt, std::uint32_t k,
                             std::uint32_t input_k, const std::uint32_t *partition, const std::uint32_t *node_off,
                             std::uint32_t *mapping, std::uint32_t *xadj_out, std::uint32_t *adjncy_out,
                             std::int32_t *vwgt_out, std::int32_t *adjwgt_out, std::int32_t *weighted_out) {
  DISABLE_TIMERS();
  Graph graph = make_graph(n, m, xadj, adjncy, vwgt, adjwgt);
  PartitionedGraph p_graph(graph, k, copy_array<BlockID>(partition, n));
  // every block is followed by compute_final_k(b, k, input_k) padding slots (subgraph_extractor.cc:376-378), at most
  // 2 input_k + k in all
  graph::SubgraphMemory memory(n, 2 * input_k + k, m, graph.is_node_weighted(), graph.is_edge_weighted());
  auto res = graph::extract_subgraphs(p_graph, input_k, memory);
  if (res.subgraphs.size() != k) {
    return -1;
  }
  for (NodeID u = 0; u < n; ++u) {
    mapping[u] = res.node_mapping[u];
  }
  std::uint32_t cursor = 0;
  weighted_out[0] = weighted_out[1] = 0;
  for (BlockID b = 0; b < k; ++b) {
    if (res.subgraphs[b].n() != node_off[b + 1] - node_off[b]) {
      return -2;
    }
    append_block(res.subgraphs[b], node_off[b], b, &cursor, xadj_out, adjncy_out, vwgt_out, adjwgt_out,
                 weighted_out);
  }
  return 0;
}

// graph::copy_subgraph_partitions with the reference's own mapping (lazy_extract_subgraphs_preprocessing) and the
// sub-partitions given block-major (block b's at node_off[b]). partition_out[n].
int bridge_copy_subgraph_partitions(std::uint32_t n, std::uint32_t m, const std::uint32_t *xadj,
                                    const std::uint32_t *adjncy, std::uint32_t k, const std::uint32_t *partition,
                                    std::uint32_t k_prime, std::uint32_t input_k,
                                    const std::uint32_t *sub_block_major, std::uint32_t *partition_out) {
  DISABLE_TIMERS();
  Graph graph = make_graph(n, m, xadj, adjncy, nullptr, nullptr);
  PartitionedGraph p_graph(graph, k, copy_array<BlockID>(partition, n));
  auto pre = graph::lazy_extract_subgraphs_preprocessing(p_graph);
  ScalableVector<StaticArray<BlockID>> subs;
  for (BlockID b = 0; b < k; ++b) {
    const NodeID nb = pre.block_nodes_offset[b + 1] - pre.block_nodes_offset[b];
    subs.emplace_back(copy_array<BlockID>(sub_block_major + pre.block_nodes_offset[b], nb));
  }
  PartitionedGraph out = graph::copy_subgraph_partitions(std::move(p_graph), subs, k_prime, input_k, pre.mapping);
  for (NodeID u = 0; u < n; ++u) {
    partition_out[u] = out.block(u);
  }
  return 0;
}

// partitioning::compute_final_k for current_k = 2^0 .. 2^(levels-1) and every block: out[level][block] laid out
// level-major, 2^levels - 1 entries.
void bridge_compute_final_k(std::uint32_t input_k, std::uint32_t levels, std::uint32_t *out) {
  std::size_t i = 0;
  for (std::uint32_t l = 0; l < levels; ++l) {
    const BlockID current_k = 1u << l;
    for (BlockID b = 0; b < current_k; ++b) {
      out[i++] = partitioning::compute_final_k(b, current_k, input_k);
    }
  }
}

} // extern "C"
