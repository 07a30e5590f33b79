// Bridge to the UNMODIFIED reference's UnderloadBalancer, for the CPU tests of tests/test_underload_bridge.py.
// Compiled by that test against the reference headers and linked against the reference partitioner the build leaves
// in oracle/_ref/libkaminpar_ref_full.so (serial oneTBB stand-in: one thread).
#include <cstdint>
#include <cstring>
#include <memory>

#include "kaminpar-shm/datastructures/csr_graph.h"
#include "kaminpar-shm/datastructures/graph.h"
#include "kaminpar-shm/datastructures/partitioned_graph.h"
#include "kaminpar-shm/kaminpar.h"
#include "kaminpar-shm/refinement/balancer/underload_balancer.h"

#include "kaminpar-common/datastructures/static_array.h"
#include "kaminpar-common/random.h"
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

// UnderloadBalancer::refine on (graph, partition) with PartitionContext::setup(graph, k, epsilon) and
// setup_min_block_weights(min_epsilon), one thread. Returns the reference's return value; partition_inout is
// balanced in place; min_block_weights_out[k] (nullable) receives the minimum weights the context computed.
int bridge_underload_balance(std::uint32_t n, std::uint32_t m, const std::uint32_t *xadj,
                             const std::uint32_t *adjncy, const std::int32_t *vwgt, const std::int32_t *adjwgt,
                             std::uint32_t k, double epsilon, double min_epsilon, int seed,
                             std::uint32_t *partition_inout, std::int32_t *min_block_weights_out) {
  Random::reseed(seed);
  DISABLE_TIMERS();
  Graph graph(std::make_unique<CSRGraph>(
      copy_array<EdgeID>(xadj, static_cast<std::size_t>(n) + 1), copy_array<NodeID>(adjncy, m),
      vwgt ? copy_array<NodeWeight>(vwgt, n) : StaticArray<NodeWeight>(),
      adjwgt ? copy_array<EdgeWeight>(adjwgt, m) : StaticArray<EdgeWeight>(), false
  ));
  Context ctx = create_default_context();
  ctx.parallel.num_threads = 1;
  ctx.partition.setup(graph, k, epsilon);
  ctx.partition.setup_min_block_weights(min_epsilon);
  if (min_block_weights_out != nullptr) {
    for (std::uint32_t b = 0; b < k; ++b) {
      min_block_weights_out[b] = ctx.partition.min_block_weight(b);
    }
  }
  PartitionedGraph p_graph(graph, k, copy_array<BlockID>(partition_inout, n));
  UnderloadBalancer balancer(ctx);
  balancer.initialize(p_graph);
  const bool improved = balancer.refine(p_graph, ctx.partition);
  for (std::uint32_t u = 0; u < n; ++u) {
    partition_inout[u] = p_graph.block(u);
  }
  return improved ? 1 : 0;
}

} // extern "C"
