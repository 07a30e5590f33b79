// Bridge to the UNMODIFIED reference's SparsificationClusterCoarsener, for the CPU tests of
// tests/test_sparsify_bridge.py. Compiled by that test against the reference headers and linked against the
// reference partitioner the build leaves in oracle/_ref/libkaminpar_ref_full.so (serial oneTBB stand-in: one thread).
#include <cstdint>
#include <cstring>
#include <limits>
#include <memory>
#include <numeric>
#include <vector>

#include "kaminpar-shm/coarsening/contraction/cluster_contraction.h"
#include "kaminpar-shm/coarsening/sparsification_cluster_coarsener.h"
#include "kaminpar-shm/datastructures/csr_graph.h"
#include "kaminpar-shm/datastructures/graph.h"
#include "kaminpar-shm/datastructures/partitioned_graph.h"
#include "kaminpar-shm/kaminpar.h"

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

Graph make_graph(std::uint32_t n, std::uint32_t m, const std::uint32_t *xadj, const std::uint32_t *adjncy,
                 const std::int32_t *vwgt, const std::int32_t *adjwgt) {
  return Graph(std::make_unique<CSRGraph>(
      copy_array<EdgeID>(xadj, static_cast<std::size_t>(n) + 1), copy_array<NodeID>(adjncy, m),
      vwgt ? copy_array<NodeWeight>(vwgt, n) : StaticArray<NodeWeight>(),
      adjwgt ? copy_array<EdgeWeight>(adjwgt, m) : StaticArray<EdgeWeight>(), false
  ));
}
} // namespace

extern "C" {

// The first Random::instance().random_index(0, SIZE_MAX) after Random::reseed(seed): the seed the coarsener draws
// when nothing else consumed random numbers before it (NOOP clustering).
std::uint64_t bridge_first_draw(int seed) {
  Random::reseed(seed);
  return Random::instance().random_index(0, std::numeric_limits<std::size_t>::max());
}

// The mapping of contract_clustering(graph, clustering) at one thread (the coarsener's first contraction).
void bridge_contract_mapping(std::uint32_t n, std::uint32_t m, const std::uint32_t *xadj, const std::uint32_t *adjncy,
                             const std::int32_t *vwgt, const std::int32_t *adjwgt, const std::uint32_t *clustering,
                             std::uint32_t *mapping_out) {
  DISABLE_TIMERS();
  Graph graph = make_graph(n, m, xadj, adjncy, vwgt, adjwgt);
  Context ctx = create_default_context();
  auto coarse = contract_clustering(graph, copy_array<NodeID>(clustering, n), ctx.coarsening.contraction);
  const NodeID c_n = coarse->get().n();
  std::vector<BlockID> ids(c_n);
  std::iota(ids.begin(), ids.end(), 0);
  coarse->project_up(std::span<const BlockID>(ids), std::span<BlockID>(mapping_out, n));
}

// One SparsificationClusterCoarsener::coarsen() on the graph, one thread, after Random::reseed(seed), with
// PartitionContext::setup(graph, k, epsilon). lp_clustering = 0: NOOP clustering (every vertex its own cluster);
// otherwise the reference's LP clusterer. Outputs (sized for the fine graph): the coarse CSR, its vertex weights and
// the fine -> coarse mapping. Returns the coarse edge count.
std::uint32_t bridge_sparsify_coarsen(std::uint32_t n, std::uint32_t m, const std::uint32_t *xadj,
                                      const std::uint32_t *adjncy, const std::int32_t *vwgt,
                                      const std::int32_t *adjwgt, int lp_clustering, std::uint32_t k, double epsilon,
                                      double density_target_factor, double edge_target_factor,
                                      double laziness_factor, int seed, std::uint32_t *c_n_out,
                                      std::uint32_t *c_xadj, std::uint32_t *c_adjncy, std::int32_t *c_vwgt,
                                      std::int32_t *c_adjwgt, std::uint32_t *mapping_out) {
  DISABLE_TIMERS();
  Graph graph = make_graph(n, m, xadj, adjncy, vwgt, adjwgt);
  Context ctx = create_default_context();
  ctx.parallel.num_threads = 1;
  ctx.coarsening.clustering.algorithm =
      lp_clustering != 0 ? ClusteringAlgorithm::LABEL_PROPAGATION : ClusteringAlgorithm::NOOP;
  ctx.coarsening.sparsification_clustering.density_target_factor = density_target_factor;
  ctx.coarsening.sparsification_clustering.edge_target_factor = edge_target_factor;
  ctx.coarsening.sparsification_clustering.laziness_factor = laziness_factor;
  ctx.partition.setup(graph, k, epsilon);
  Random::reseed(seed);
  SparsificationClusterCoarsener coarsener(ctx, ctx.partition);
  coarsener.initialize(&graph);
  coarsener.coarsen();
  const auto &csr = concretize<CSRGraph>(coarsener.current());
  const NodeID c_n = csr.n();
  const EdgeID c_m = csr.m();
  *c_n_out = c_n;
  for (NodeID u = 0; u <= c_n; ++u) {
    c_xadj[u] = csr.raw_nodes()[u];
  }
  for (NodeID u = 0; u < c_n; ++u) {
    c_vwgt[u] = csr.node_weight(u);
  }
  for (EdgeID e = 0; e < c_m; ++e) {
    c_adjncy[e] = csr.raw_edges()[e];
    c_adjwgt[e] = csr.edge_weight(e);
  }
  // the mapping: project the partition "coarse vertex c in block c" up one level
  StaticArray<BlockID> ids(c_n);
  std::iota(ids.begin(), ids.end(), 0);
  PartitionedGraph p_graph(coarsener.current(), c_n, std::move(ids));
  PartitionedGraph fine = coarsener.uncoarsen(std::move(p_graph));
  for (NodeID u = 0; u < n; ++u) {
    mapping_out[u] = fine.block(u);
  }
  return c_m;
}

} // extern "C"
