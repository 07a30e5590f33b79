// Bridge to the UNMODIFIED reference's isolated-vertex re-integration, for the CPU tests of
// tests/test_prepare_bridge.py. Compiled by that test against the reference headers and linked against the reference
// partitioner the build leaves in oracle/_ref/libkaminpar_ref_full.so (serial oneTBB stand-in: one thread).
#include <cstdint>
#include <cstring>
#include <memory>
#include <vector>

#include "kaminpar-shm/datastructures/csr_graph.h"
#include "kaminpar-shm/datastructures/graph.h"
#include "kaminpar-shm/datastructures/partitioned_graph.h"
#include "kaminpar-shm/graphutils/permutator.h"
#include "kaminpar-shm/kaminpar.h"

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
} // namespace

extern "C" {

// The steps of KaMinPar::compute_partition around a partition of a graph whose num_isolated last vertices are
// isolated (a sorted graph, as rearrange_by_degree_buckets leaves it): PartitionContext::setup on the full graph with
// the given max block weights (kaminpar.cc:316), CSRGraph::remove_isolated_nodes (:391), a PartitionedGraph over the
// n' = n - num_isolated vertices with `partition`, integrate_isolated_nodes and graph::assign_isolated_nodes
// (:425-430). partition_out[n] and block_weights_out[k] receive the result, in the graph's own ids.
int bridge_assign_isolated_nodes(std::uint32_t n, std::uint32_t m, const std::uint32_t *xadj,
                                 const std::uint32_t *adjncy, const std::int32_t *vwgt, std::uint32_t num_isolated,
                                 std::uint32_t k, const std::int32_t *max_block_weights,
                                 const std::uint32_t *partition, std::uint32_t *partition_out,
                                 std::int32_t *block_weights_out) {
  DISABLE_TIMERS();
  Graph graph(std::make_unique<CSRGraph>(
      copy_array<EdgeID>(xadj, static_cast<std::size_t>(n) + 1), copy_array<NodeID>(adjncy, m),
      vwgt ? copy_array<NodeWeight>(vwgt, n) : StaticArray<NodeWeight>(), StaticArray<EdgeWeight>(), true
  ));
  Context ctx = create_default_context();
  ctx.parallel.num_threads = 1;
  ctx.partition.setup(graph, std::vector<BlockWeight>(max_block_weights, max_block_weights + k));
  CSRGraph &csr = graph.csr_graph();
  csr.remove_isolated_nodes(num_isolated);
  const NodeID n_prime = n - num_isolated;
  PartitionedGraph p_graph(graph, k, copy_array<BlockID>(partition, n_prime));
  const NodeID integrated = csr.integrate_isolated_nodes();
  if (integrated != num_isolated) {
    return -1;
  }
  PartitionedGraph out = graph::assign_isolated_nodes(std::move(p_graph), integrated, ctx.partition);
  for (NodeID u = 0; u < n; ++u) {
    partition_out[u] = out.block(u);
  }
  for (BlockID b = 0; b < k; ++b) {
    block_weights_out[b] = static_cast<std::int32_t>(out.block_weight(b));
  }
  return 0;
}

} // extern "C"
