// Bridge to the UNMODIFIED reference's OverlayClusterCoarsener, for the CPU tests of tests/test_overlay_bridge.py.
// Compiled by that test against the reference headers and linked against the reference partitioner the build leaves
// in oracle/_ref/libkaminpar_ref_full.so (serial oneTBB stand-in: one thread).
#include <cstdint>
#include <cstring>
#include <memory>
#include <numeric>
#include <vector>

#include "kaminpar-shm/coarsening/clusterer.h"
#include "kaminpar-shm/coarsening/contraction/cluster_contraction.h"
#include "kaminpar-shm/coarsening/max_cluster_weights.h"
#include "kaminpar-shm/coarsening/overlay_cluster_coarsener.h"
#include "kaminpar-shm/datastructures/csr_graph.h"
#include "kaminpar-shm/datastructures/graph.h"
#include "kaminpar-shm/datastructures/partitioned_graph.h"
#include "kaminpar-shm/factories.h"
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

Context one_thread_context(const Graph &graph, std::uint32_t k, double epsilon) {
  Context ctx = create_default_context();
  ctx.parallel.num_threads = 1;
  ctx.partition.setup(graph, k, epsilon);
  return ctx;
}

// coarse CSR, vertex weights and fine -> coarse mapping (the partition "coarse vertex c in block c", projected up)
template <typename Up>
std::uint32_t write_level(const Graph &coarse, std::uint32_t n, Up project_up, std::uint32_t *c_n_out,
                          std::uint32_t *c_xadj, std::uint32_t *c_adjncy, std::int32_t *c_vwgt, std::int32_t *c_adjwgt,
                          std::uint32_t *mapping_out) {
  const auto &csr = concretize<CSRGraph>(coarse);
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
  std::vector<BlockID> ids(c_n);
  std::iota(ids.begin(), ids.end(), 0);
  project_up(ids, std::span<BlockID>(mapping_out, n));
  return c_m;
}
} // namespace

extern "C" {

// After Random::reseed(seed): the reference's LP clusterer (factory::create_clusterer), called `count` times on the
// graph with the max cluster weight and desired cluster count the coarsener sets on its first level
// (AbstractClusterCoarsener::compute_clustering_for_current_graph). clusterings_out: count x n.
void bridge_lp_clusterings(std::uint32_t n, std::uint32_t m, const std::uint32_t *xadj, const std::uint32_t *adjncy,
                           const std::int32_t *vwgt, const std::int32_t *adjwgt, std::uint32_t k, double epsilon,
                           int seed, int count, std::uint32_t *clusterings_out) {
  DISABLE_TIMERS();
  Graph graph = make_graph(n, m, xadj, adjncy, vwgt, adjwgt);
  Context ctx = one_thread_context(graph, k, epsilon);
  Random::reseed(seed);
  auto clusterer = factory::create_clusterer(ctx);
  clusterer->set_max_cluster_weight(
      compute_max_cluster_weight<NodeWeight>(ctx.coarsening, ctx.partition, n, graph.total_node_weight())
  );
  clusterer->set_desired_cluster_count(n / ctx.coarsening.clustering.shrink_factor);
  StaticArray<NodeID> clustering(n);
  for (int i = 0; i < count; ++i) {
    clusterer->compute_clustering(clustering, graph, false);
    std::memcpy(clusterings_out + static_cast<std::size_t>(i) * n, clustering.data(), n * sizeof(NodeID));
  }
}

// The reference's contract_clustering(graph, clustering) at one thread. Returns the coarse edge count.
std::uint32_t bridge_contract(std::uint32_t n, std::uint32_t m, const std::uint32_t *xadj, const std::uint32_t *adjncy,
                              const std::int32_t *vwgt, const std::int32_t *adjwgt, const std::uint32_t *clustering,
                              std::uint32_t *c_n_out, std::uint32_t *c_xadj, std::uint32_t *c_adjncy,
                              std::int32_t *c_vwgt, std::int32_t *c_adjwgt, std::uint32_t *mapping_out) {
  DISABLE_TIMERS();
  Graph graph = make_graph(n, m, xadj, adjncy, vwgt, adjwgt);
  Context ctx = create_default_context();
  auto coarse = contract_clustering(graph, copy_array<NodeID>(clustering, n), ctx.coarsening.contraction);
  return write_level(
      coarse->get(), n,
      [&](const std::vector<BlockID> &ids, std::span<BlockID> fine) {
        coarse->project_up(std::span<const BlockID>(ids), fine);
      },
      c_n_out, c_xadj, c_adjncy, c_vwgt, c_adjwgt, mapping_out
  );
}

// One OverlayClusterCoarsener::coarsen() on the graph, one thread, after Random::reseed(seed), with the reference's LP
// clusterer and PartitionContext::setup(graph, k, epsilon). Outputs sized for the fine graph. Returns the coarse edge
// count.
std::uint32_t bridge_overlay_coarsen(std::uint32_t n, std::uint32_t m, const std::uint32_t *xadj,
                                     const std::uint32_t *adjncy, const std::int32_t *vwgt, const std::int32_t *adjwgt,
                                     std::uint32_t k, double epsilon, int num_levels, int max_level, int seed,
                                     std::uint32_t *c_n_out, std::uint32_t *c_xadj, std::uint32_t *c_adjncy,
                                     std::int32_t *c_vwgt, std::int32_t *c_adjwgt, std::uint32_t *mapping_out) {
  DISABLE_TIMERS();
  Graph graph = make_graph(n, m, xadj, adjncy, vwgt, adjwgt);
  Context ctx = one_thread_context(graph, k, epsilon);
  ctx.coarsening.overlay_clustering.num_levels = num_levels;
  ctx.coarsening.overlay_clustering.max_level = max_level;
  Random::reseed(seed);
  OverlayClusterCoarsener coarsener(ctx, ctx.partition);
  coarsener.initialize(&graph);
  coarsener.coarsen();
  return write_level(
      coarsener.current(), n,
      [&](const std::vector<BlockID> &ids, std::span<BlockID> fine) {
        PartitionedGraph p_graph(coarsener.current(), static_cast<BlockID>(ids.size()),
                                 StaticArray<BlockID>(ids.begin(), ids.end()));
        PartitionedGraph up = coarsener.uncoarsen(std::move(p_graph));
        for (NodeID u = 0; u < fine.size(); ++u) {
          fine[u] = up.block(u);
        }
      },
      c_n_out, c_xadj, c_adjncy, c_vwgt, c_adjwgt, mapping_out
  );
}

} // extern "C"
