// C++ host side above the C ABI: adapter classes with the method names, argument meaning and
// error behaviour of the reference's plugin interfaces, so that
//   kaminpar-shm/factories.cc:66-67   case ClusteringAlgorithm::LABEL_PROPAGATION  -> b200::LPClustering
//   kaminpar-shm/factories.cc:108-109 case RefinementAlgorithm::LABEL_PROPAGATION  -> b200::LabelPropagationRefiner
//   the OVERLOAD_BALANCER / UNDERLOAD_BALANCER cases                                 -> b200::OverloadBalancer /
//                                                                                       b200::UnderloadBalancer
// become one-line swaps (INTEGRATION.md shows the glue that maps kaminpar::shm::Graph /
// PartitionedGraph / PartitionContext onto the views below).
//
// Mirrors:
//   class Clusterer  kaminpar-shm/coarsening/clusterer.h:19-47
//   class Refiner    kaminpar-shm/refinement/refiner.h:18-57
//   LPClustering     kaminpar-shm/coarsening/clustering/lp_clusterer.h:19 / lp_clusterer.cc:376-399
//   LabelPropagationRefiner  kaminpar-shm/refinement/lp/lp_refiner.h:19 / lp_refiner.cc:357-376
//   OverloadBalancer   kaminpar-shm/refinement/balancer/overload_balancer.h / overload_balancer.cc:40-160
//   UnderloadBalancer  kaminpar-shm/refinement/balancer/underload_balancer.h / underload_balancer.cc:27-104
//   CoarseGraph / contract_clustering  kaminpar-shm/coarsening/contraction/cluster_contraction.h:22-56
//   sparsification_target / CoarseGraph::sparsify
//                      kaminpar-shm/coarsening/sparsification_cluster_coarsener.cc:41-228 (DESIGN.md §13)
//   LPClustering::compute_overlay_clustering
//                      kaminpar-shm/coarsening/overlay_cluster_coarsener.cc:34-151 (DESIGN.md §14)
//   PreparedGraph / rearrange_by_degree_buckets / assign_isolated_nodes
//                      kaminpar-shm/graphutils/permutator.cc:66-91, 236-264, kaminpar.cc:368-445 (DESIGN.md §15)
//   Subgraphs / extract_subgraphs / copy_subgraph_partitions
//                      kaminpar-shm/graphutils/subgraph_extractor.cc:181-324, 492-533 (DESIGN.md §16)
//   bipartition_subgraphs
//                      kaminpar-shm/initial_partitioning/ (InitialBipartitionerWorkerPool::bipartition, DESIGN.md §20)
//   MetisGraph / read_metis
//                      kaminpar-io/metis_parser.cc:158-245 (csr_read on the device, DESIGN.md §18)
//   ParhipGraph / read_parhip
//                      kaminpar-io/parhip_parser.cc:179-336 (read_graph without compression, DESIGN.md §19)
//   GraphReport / validate_graph
//                      kaminpar-shm/datastructures/csr_graph.cc:266-356 (debug::validate_graph, DESIGN.md §17)
//
// Error convention: the reference's path has no error codes (KASSERT aborts); here a non-zero
// status of the C ABI becomes std::runtime_error. There is no CPU fallback.
#pragma once

#include <cstdint>
#include <memory>
#include <span>
#include <stdexcept>
#include <string>
#include <vector>

#include "kaminpar_b200_balancer.h"
#include "kaminpar_b200_bipartition.h"
#include "kaminpar_b200_contraction.h"
#include "kaminpar_b200_io.h"
#include "kaminpar_b200_parhip.h"
#include "kaminpar_b200_lp.h"
#include "kaminpar_b200_prepare.h"
#include "kaminpar_b200_subgraph.h"
#include "kaminpar_b200_validate.h"

namespace kaminpar_b200 {

using NodeID = std::uint32_t;     // include/kaminpar-shm/kaminpar.h:32-57 (default build)
using EdgeID = std::uint32_t;
using BlockID = std::uint32_t;
using NodeWeight = std::int32_t;
using EdgeWeight = std::int32_t;
using BlockWeight = std::int32_t;

// Borrowed view of a CSRGraph (csr_graph.h:35-482). Empty weight spans mean unit weights.
struct CSRGraphView {
  std::span<const EdgeID> nodes;           // raw_nodes(),   n + 1
  std::span<const NodeID> edges;           // raw_edges(),   m
  std::span<const NodeWeight> node_weights; // raw_node_weights(), n or empty
  std::span<const EdgeWeight> edge_weights; // raw_edge_weights(), m or empty
  bool sorted = false;                      // CSRGraph::sorted(); read by the seq_strict schedule only
  [[nodiscard]] NodeID n() const { return nodes.empty() ? 0 : static_cast<NodeID>(nodes.size() - 1); }
  [[nodiscard]] EdgeID m() const { return static_cast<EdgeID>(edges.size()); }
  [[nodiscard]] const void *identity() const { return nodes.data(); }
};

// The parts of PartitionedGraph (partitioned_graph.h:50-456) the refiner reads and writes.
struct PartitionedGraphView {
  CSRGraphView graph;
  BlockID k = 0;
  std::span<BlockID> partition;          // raw_partition(), refined in place
  std::span<BlockWeight> block_weights;  // k entries, updated to match the refined partition
};

// The parts of PartitionContext (kaminpar.h:417-531) the refiner reads.
struct PartitionContextView {
  BlockID k = 0;
  std::span<const BlockWeight> max_block_weights; // max_block_weight(b)
  std::span<const BlockWeight> min_block_weights; // min_block_weight(b); empty -> 0
  std::span<const BlockWeight> perfectly_balanced_block_weights; // perfectly_balanced_block_weight(b); OverloadBalancer
};

struct LabelPropagationCoarseningContext { // kaminpar.h:140-154, defaults presets.cc:140-153
  std::size_t num_iterations = 5;
  NodeID large_degree_threshold = 0xFFFFFFFFu;
  NodeID max_num_neighbors = 0xFFFFFFFFu;
  int impl = KMP_LP_TWO_PHASE;
  bool relabel_before_second_phase = false;
  int two_hop_strategy = KMP_TWO_HOP_MATCH_THREADWISE;
  double two_hop_threshold = 0.5;
  int isolated_nodes_strategy = KMP_ISOLATED_MATCH_DURING_TWO_HOP;
  int tie_breaking_strategy = KMP_TIE_UNIFORM;
};

struct LabelPropagationRefinementContext { // kaminpar.h:221-228, defaults presets.cc:339-347
  std::size_t num_iterations = 5;
  NodeID large_degree_threshold = 0xFFFFFFFFu;
  NodeID max_num_neighbors = 0xFFFFFFFFu;
  int impl = KMP_LP_SINGLE_PHASE;
  int tie_breaking_strategy = KMP_TIE_UNIFORM;
};

struct EngineContext { // engine knobs without a reference counterpart
  int seed = 0;        // Random::reseed analogue
  unsigned sync_subrounds = 8;
  unsigned sync_granule_log2 = 4;
  int device = -1;
  int schedule = KMP_SCHEDULE_SYNC; // KMP_SCHEDULE_SEQ_STRICT: the reference's one-thread order, bit-identical, small inputs
};

namespace detail {
inline void check(int rc) {
  if (rc != KMP_OK) {
    throw std::runtime_error(std::string("kaminpar_b200: ") + kmp_last_error());
  }
}
class Handle {
public:
  explicit Handle(const kmp_lp_config &cfg) {
    // struct layouts (kmp_lp_config / kmp_lp_stats) are part of the ABI: refuse a library built from another header
    if (kmp_lp_abi_version() != KMP_LP_ABI_VERSION) {
      throw std::runtime_error("kaminpar_b200: library ABI version " + std::to_string(kmp_lp_abi_version()) +
                               " != header ABI version " + std::to_string(KMP_LP_ABI_VERSION));
    }
    check(kmp_lp_create(&cfg, &_h));
  }
  Handle(const Handle &) = delete;
  Handle &operator=(const Handle &) = delete;
  ~Handle() { kmp_lp_destroy(_h); }
  void set_graph(const CSRGraphView &g) {
    if (g.identity() == _graph_id && g.n() == _n && g.m() == _m) {
      return; // same borrowed graph as in the previous call
    }
    check(kmp_lp_set_graph(_h, g.n(), g.m(), g.nodes.data(), g.edges.data(),
                           g.node_weights.empty() ? nullptr : g.node_weights.data(),
                           g.edge_weights.empty() ? nullptr : g.edge_weights.data()));
    if (g.sorted) {
      check(kmp_lp_set_graph_sorted(_h, 1));
    }
    _graph_id = g.identity();
    _n = g.n();
    _m = g.m();
  }
  [[nodiscard]] kmp_lp_handle *get() const { return _h; }
  // The borrowed graph is recognised by (address, n, m): call this when its arrays were rewritten in place (or
  // freed and reallocated at the same address) so that the next call uploads it again.
  void invalidate_graph() { _graph_id = nullptr; }

private:
  kmp_lp_handle *_h = nullptr;
  const void *_graph_id = nullptr;
  NodeID _n = 0;
  EdgeID _m = 0;
};
} // namespace detail

// Same surface as kaminpar::shm::Clusterer (clusterer.h:35-46).
class LPClustering {
public:
  explicit LPClustering(const LabelPropagationCoarseningContext &lp_ctx, const EngineContext &engine = {})
      : _handle(make_config(lp_ctx, engine)) {}

  void set_max_cluster_weight(const NodeWeight weight) { _max_cluster_weight = weight; }
  void set_desired_cluster_count(const NodeID count) { _desired = count; }
  void set_communities(std::span<const NodeID> communities) { _communities = communities; }

  // clustering: caller-allocated, size graph.n(), fully overwritten with ids of cluster leaders in
  // [0, n), not compacted (basic_cluster_coarsener.cc:29, cluster_contraction_preprocessing.cc:17-51).
  void compute_clustering(std::span<NodeID> clustering, const CSRGraphView &graph, const bool free_memory_afterwards) {
    _handle.set_graph(graph);
    detail::check(kmp_lp_cluster(_handle.get(), _max_cluster_weight, _desired,
                                 _communities.empty() ? nullptr : _communities.data(), clustering.data(), &_stats));
    if (free_memory_afterwards) { // lp_clusterer.cc:330-333
      detail::check(kmp_lp_free_scratch(_handle.get()));
    }
  }
  // The clustering step of OverlayClusterCoarsener::coarsen(): 2^num_levels compute_clustering calls on this
  // clusterer, intersected in the reference's tree order on the device (kmp_lp_cluster_overlay). The overlay is
  // written to `clustering` (ids in [0, n), not dense) and stays on the device for contract_clustering(handle(), {}).
  // num_levels = 0 is one compute_clustering. Its stats: last_overlay_stats().
  void compute_overlay_clustering(std::span<NodeID> clustering, const CSRGraphView &graph, const int num_levels,
                                  const bool free_memory_afterwards) {
    _handle.set_graph(graph);
    detail::check(kmp_lp_cluster_overlay(_handle.get(), num_levels, _max_cluster_weight, _desired,
                                         _communities.empty() ? nullptr : _communities.data(),
                                         clustering.empty() ? nullptr : clustering.data(), &_overlay_stats));
    if (free_memory_afterwards) {
      detail::check(kmp_lp_free_scratch(_handle.get()));
    }
  }
  [[nodiscard]] const kmp_lp_stats &last_stats() const { return _stats; }
  [[nodiscard]] const kmp_overlay_stats &last_overlay_stats() const { return _overlay_stats; }
  [[nodiscard]] kmp_lp_handle *handle() const { return _handle.get(); } // graph holder for contract_clustering
  void invalidate_graph() { _handle.invalidate_graph(); }                // the borrowed graph changed in place

private:
  static kmp_lp_config make_config(const LabelPropagationCoarseningContext &c, const EngineContext &e) {
    kmp_lp_config cfg;
    kmp_lp_default_config(0, &cfg);
    cfg.num_iterations = static_cast<std::uint32_t>(c.num_iterations);
    cfg.large_degree_threshold = c.large_degree_threshold;
    cfg.max_num_neighbors = c.max_num_neighbors;
    cfg.impl = c.impl;
    cfg.relabel_before_second_phase = c.relabel_before_second_phase;
    cfg.two_hop_strategy = c.two_hop_strategy;
    cfg.two_hop_threshold = c.two_hop_threshold;
    cfg.isolated_nodes_strategy = c.isolated_nodes_strategy;
    cfg.tie_breaking_strategy = c.tie_breaking_strategy;
    cfg.seed = e.seed;
    cfg.sync_subrounds = e.sync_subrounds;
    cfg.sync_granule_log2 = e.sync_granule_log2;
    cfg.device = e.device;
    cfg.schedule = e.schedule;
    return cfg;
  }
  detail::Handle _handle;
  NodeWeight _max_cluster_weight = 0;
  NodeID _desired = 0;
  std::span<const NodeID> _communities;
  kmp_lp_stats _stats{};
  kmp_overlay_stats _overlay_stats{};
};

// Same surface as kaminpar::shm::Refiner (refiner.h:34-56).
class LabelPropagationRefiner {
public:
  explicit LabelPropagationRefiner(const LabelPropagationRefinementContext &lp_ctx, const EngineContext &engine = {})
      : _handle(make_config(lp_ctx, engine)) {}

  [[nodiscard]] std::string name() const { return "Label Propagation"; }
  void set_communities(std::span<const NodeID> communities) { _communities = communities; }

  void initialize(const PartitionedGraphView &p_graph) { _handle.set_graph(p_graph.graph); }

  // Mutates p_graph in place (labels and block weights stay consistent,
  // partitioned_graph.h:117-135); always returns true like lp_refiner.cc:88.
  bool refine(PartitionedGraphView &p_graph, const PartitionContextView &p_ctx) {
    if (p_graph.k > p_ctx.k || p_ctx.max_block_weights.size() != p_ctx.k) {
      throw std::invalid_argument("kaminpar_b200: inconsistent k / max_block_weights");
    }
    _handle.set_graph(p_graph.graph);
    detail::check(kmp_lp_refine(_handle.get(), p_ctx.k, p_ctx.max_block_weights.data(),
                                p_ctx.min_block_weights.empty() ? nullptr : p_ctx.min_block_weights.data(),
                                _communities.empty() ? nullptr : _communities.data(), p_graph.partition.data(),
                                p_graph.block_weights.empty() ? nullptr : p_graph.block_weights.data(), &_stats));
    return true;
  }
  [[nodiscard]] const kmp_lp_stats &last_stats() const { return _stats; }
  [[nodiscard]] kmp_lp_handle *handle() const { return _handle.get(); } // e.g. for kmp_lp_dist_init
  void invalidate_graph() { _handle.invalidate_graph(); }

private:
  static kmp_lp_config make_config(const LabelPropagationRefinementContext &c, const EngineContext &e) {
    kmp_lp_config cfg;
    kmp_lp_default_config(1, &cfg);
    cfg.num_iterations = static_cast<std::uint32_t>(c.num_iterations);
    cfg.large_degree_threshold = c.large_degree_threshold;
    cfg.max_num_neighbors = c.max_num_neighbors;
    cfg.impl = c.impl;
    cfg.tie_breaking_strategy = c.tie_breaking_strategy;
    cfg.seed = e.seed;
    cfg.sync_subrounds = e.sync_subrounds;
    cfg.sync_granule_log2 = e.sync_granule_log2;
    cfg.device = e.device;
    cfg.schedule = e.schedule;
    return cfg;
  }
  detail::Handle _handle;
  std::span<const NodeID> _communities;
  kmp_lp_stats _stats{};
};

namespace detail {
inline kmp_lp_config balancer_config(const EngineContext &e) {
  kmp_lp_config cfg;
  kmp_lp_default_config(1, &cfg);
  cfg.seed = e.seed;
  cfg.sync_subrounds = e.sync_subrounds;
  cfg.sync_granule_log2 = e.sync_granule_log2;
  cfg.device = e.device;
  cfg.schedule = e.schedule;
  return cfg;
}
inline void check_balancer_args(const PartitionedGraphView &p_graph, const PartitionContextView &p_ctx) {
  if (p_graph.k > p_ctx.k || p_ctx.max_block_weights.size() != p_ctx.k ||
      (!p_graph.block_weights.empty() && p_graph.block_weights.size() != p_ctx.k)) {
    throw std::invalid_argument("kaminpar_b200: inconsistent k / max_block_weights / block_weights");
  }
}
} // namespace detail

// Same surface as kaminpar::shm::Refiner (refiner.h:34-56), OverloadBalancer::refine on the device (DESIGN.md §11).
// Reads p_ctx.perfectly_balanced_block_weights (k entries). Returns false without device work when the block
// weights (if given) show no overloaded block, like overload_balancer.cc:58-60.
class OverloadBalancer {
public:
  explicit OverloadBalancer(const EngineContext &engine = {}) : _handle(detail::balancer_config(engine)) {}

  [[nodiscard]] std::string name() const { return "Overload Balancer"; }
  void initialize(const PartitionedGraphView &) {} // overload_balancer.cc:40-43

  bool refine(PartitionedGraphView &p_graph, const PartitionContextView &p_ctx) {
    detail::check_balancer_args(p_graph, p_ctx);
    if (p_ctx.perfectly_balanced_block_weights.size() != p_ctx.k) {
      throw std::invalid_argument("kaminpar_b200: perfectly_balanced_block_weights needs k entries");
    }
    if (!p_graph.block_weights.empty()) {
      bool overloaded = false;
      for (BlockID b = 0; b < p_ctx.k; ++b) {
        overloaded = overloaded || p_graph.block_weights[b] > p_ctx.max_block_weights[b];
      }
      if (!overloaded) {
        return false;
      }
    }
    _handle.set_graph(p_graph.graph);
    int improved = 0;
    detail::check(kmp_overload_balance(_handle.get(), p_ctx.k, p_ctx.max_block_weights.data(),
                                       p_ctx.perfectly_balanced_block_weights.data(), p_graph.partition.data(),
                                       p_graph.block_weights.empty() ? nullptr : p_graph.block_weights.data(),
                                       &improved, &_stats));
    return improved != 0;
  }
  [[nodiscard]] const kmp_balance_stats &last_stats() const { return _stats; }
  [[nodiscard]] kmp_lp_handle *handle() const { return _handle.get(); }
  void invalidate_graph() { _handle.invalidate_graph(); }

private:
  detail::Handle _handle;
  kmp_balance_stats _stats{};
};

// Same surface as kaminpar::shm::Refiner (refiner.h:34-56), UnderloadBalancer::refine on the device (DESIGN.md §12).
// Returns false without device work when p_ctx has no minimum weights or the block weights (if given) are at or
// above them, like underload_balancer.cc:47-50.
class UnderloadBalancer {
public:
  explicit UnderloadBalancer(const EngineContext &engine = {}) : _handle(detail::balancer_config(engine)) {}

  [[nodiscard]] std::string name() const { return "Underload Balancer"; }
  void initialize(const PartitionedGraphView &) {} // underload_balancer.cc:35-37

  bool refine(PartitionedGraphView &p_graph, const PartitionContextView &p_ctx) {
    detail::check_balancer_args(p_graph, p_ctx);
    if (p_ctx.min_block_weights.empty()) {
      return false;
    }
    if (p_ctx.min_block_weights.size() != p_ctx.k) {
      throw std::invalid_argument("kaminpar_b200: min_block_weights needs k entries");
    }
    if (!p_graph.block_weights.empty()) {
      bool underloaded = false;
      for (BlockID b = 0; b < p_ctx.k; ++b) {
        underloaded = underloaded || p_graph.block_weights[b] < p_ctx.min_block_weights[b];
      }
      if (!underloaded) {
        return false;
      }
    }
    _handle.set_graph(p_graph.graph);
    int improved = 0;
    detail::check(kmp_underload_balance(_handle.get(), p_ctx.k, p_ctx.max_block_weights.data(),
                                        p_ctx.min_block_weights.data(), p_graph.partition.data(),
                                        p_graph.block_weights.empty() ? nullptr : p_graph.block_weights.data(),
                                        &improved, &_stats));
    return improved != 0;
  }
  [[nodiscard]] const kmp_underload_stats &last_stats() const { return _stats; }
  [[nodiscard]] kmp_lp_handle *handle() const { return _handle.get(); }
  void invalidate_graph() { _handle.invalidate_graph(); }

private:
  detail::Handle _handle;
  kmp_underload_stats _stats{};
};

// Same surface as kaminpar::shm::CoarseGraph (cluster_contraction.h:22-32). The coarse graph lives on the
// device; get() copies it into host vectors once (a maintainer's glue wraps them into a CSRGraph).
class CoarseGraph {
public:
  struct HostCSR {
    std::vector<EdgeID> nodes;
    std::vector<NodeID> edges;
    std::vector<NodeWeight> node_weights;
    std::vector<EdgeWeight> edge_weights;
  };
  explicit CoarseGraph(kmp_coarse_graph *g, const kmp_contraction_stats &stats) : _g(g), _stats(stats) {}
  CoarseGraph(const CoarseGraph &) = delete;
  CoarseGraph &operator=(const CoarseGraph &) = delete;
  ~CoarseGraph() { kmp_coarse_destroy(_g); }

  [[nodiscard]] NodeID n() const { return kmp_coarse_n(_g); }
  [[nodiscard]] EdgeID m() const { return kmp_coarse_m(_g); }
  const HostCSR &get() {
    if (_host.nodes.empty()) {
      _host.nodes.resize(static_cast<std::size_t>(n()) + 1);
      _host.edges.resize(m());
      _host.node_weights.resize(n());
      _host.edge_weights.resize(m());
      detail::check(kmp_coarse_download(_g, _host.nodes.data(), _host.edges.data(), _host.node_weights.data(),
                                        _host.edge_weights.data(), nullptr));
    }
    return _host;
  }
  // fine[u] = coarse[mapping[u]] (cluster_contraction_preprocessing.h:36-40)
  void project_up(std::span<const BlockID> coarse, std::span<BlockID> fine) const {
    if (coarse.size() != n() || fine.size() != kmp_coarse_fine_n(_g)) {
      throw std::invalid_argument("project_up: wrong span size");
    }
    detail::check(kmp_coarse_project_up(_g, coarse.data(), fine.data()));
  }
  // coarse[mapping[u]] = fine[u] (:42-46)
  void project_down(std::span<const BlockID> fine, std::span<BlockID> coarse) const {
    if (coarse.size() != n() || fine.size() != kmp_coarse_fine_n(_g)) {
      throw std::invalid_argument("project_down: wrong span size");
    }
    detail::check(kmp_coarse_project_down(_g, fine.data(), coarse.data()));
  }
  // Threshold sparsification in place (kmp_coarse_sparsify) on the handle that contracted this graph: vertices,
  // weights and mapping stay, the edges are replaced. Drops the host copy get() made and invalidates device pointers
  // taken earlier. The caller applies the laziness rule and draws the seed (INTEGRATION.md §2e).
  kmp_sparsify_stats sparsify(kmp_lp_handle *graph_holder, EdgeID target_m, std::uint64_t seed) {
    kmp_sparsify_stats st{};
    detail::check(kmp_coarse_sparsify(graph_holder, _g, target_m, seed, &st));
    _host = HostCSR{};
    return st;
  }
  [[nodiscard]] const kmp_contraction_stats &stats() const { return _stats; }
  [[nodiscard]] const kmp_coarse_graph *device() const { return _g; } // kmp_coarse_device_arrays for the next level

private:
  kmp_coarse_graph *_g;
  kmp_contraction_stats _stats;
  HostCSR _host;
};

// SparsificationClusterCoarsener::sparsification_target (sparsification_cluster_coarsener.cc:41-48): the edge count
// a coarse graph of c_n vertices is sparsified to, from the previous level's (or the input graph's) prev_m / prev_n.
inline EdgeID sparsification_target(EdgeID prev_m, NodeID prev_n, NodeID c_n, double density_target_factor = 0.5,
                                    double edge_target_factor = 0.5) {
  return kmp_sparsification_target(prev_m, prev_n, c_n, density_target_factor, edge_target_factor);
}

// contract_clustering(graph, clustering, con_ctx) (cluster_contraction.h:47-50). `clusterer` is the LP
// clusterer that already holds `graph` on the device (no second H2D copy); an empty `clustering` span
// contracts by the clustering its last compute_clustering() left on the device.
inline std::unique_ptr<CoarseGraph> contract_clustering(kmp_lp_handle *graph_holder, std::span<const NodeID> clustering) {
  kmp_coarse_graph *g = nullptr;
  kmp_contraction_stats stats{};
  detail::check(kmp_contract_clustering(graph_holder, clustering.empty() ? nullptr : clustering.data(), &g, &stats));
  return std::make_unique<CoarseGraph>(g, stats);
}

// The caller's graph rearranged by degree bucket on the device, its isolated vertices cut off the end
// (graph::rearrange_by_degree_buckets + CSRGraph::remove_isolated_nodes, kaminpar.cc:368-402). set_on() hands the
// n() non-isolated vertices to a handle (sorted); assign_isolated_nodes() below brings the isolated ones back.
// Owns device memory of the preparing handle's pool: destroy it before that handle.
class PreparedGraph {
public:
  explicit PreparedGraph(kmp_prepared_graph *g, const kmp_prepare_stats &stats) : _g(g), _stats(stats) {}
  PreparedGraph(const PreparedGraph &) = delete;
  PreparedGraph &operator=(const PreparedGraph &) = delete;
  ~PreparedGraph() { kmp_prepared_destroy(_g); }

  [[nodiscard]] NodeID n() const { return kmp_prepared_n(_g); } // n': the vertices the LP sees
  [[nodiscard]] NodeID num_isolated() const { return kmp_prepared_num_isolated(_g); }
  [[nodiscard]] EdgeID m() const { return kmp_prepared_m(_g); }
  // kmp_lp_set_graph_prepared: the handle's graph becomes the n() prepared vertices, marked sorted
  void set_on(kmp_lp_handle *h) const { detail::check(kmp_lp_set_graph_prepared(h, _g)); }
  // original id -> prepared id (CSRGraph::map_original_node), all n() + num_isolated() vertices
  [[nodiscard]] std::vector<NodeID> old_to_new() const {
    std::vector<NodeID> o2n(static_cast<std::size_t>(n()) + num_isolated());
    detail::check(kmp_prepared_download(_g, nullptr, nullptr, nullptr, nullptr, o2n.data()));
    return o2n;
  }
  [[nodiscard]] const kmp_prepare_stats &stats() const { return _stats; }
  [[nodiscard]] const kmp_prepared_graph *device() const { return _g; } // kmp_prepared_device_arrays

private:
  kmp_prepared_graph *_g;
  kmp_prepare_stats _stats;
};

// graph::rearrange_by_degree_buckets(graph) (permutator.cc:66-91) + the isolated-vertex cut, on the device, stream
// and pool of `h`. Set the PartitionContext up on `graph` before this, as compute_partition does (kaminpar.cc:316):
// its max block weights count the isolated vertices.
inline std::unique_ptr<PreparedGraph> rearrange_by_degree_buckets(kmp_lp_handle *h, const CSRGraphView &graph) {
  kmp_prepared_graph *g = nullptr;
  kmp_prepare_stats stats{};
  detail::check(kmp_prepare_graph(h, graph.n(), graph.m(), graph.nodes.data(), graph.edges.data(),
                                  graph.node_weights.empty() ? nullptr : graph.node_weights.data(),
                                  graph.edge_weights.empty() ? nullptr : graph.edge_weights.data(), &g, &stats));
  return std::make_unique<PreparedGraph>(g, stats);
}

// graph::assign_isolated_nodes(p_graph, num_isolated_nodes, p_ctx) (permutator.cc:236-264) and the map back to the
// caller's ids (kaminpar.cc:434-440): p_graph partitions the prepared graph's n() vertices (an empty partition span
// takes the labels `h` holds on the device for `graph`); its block_weights (k entries, or empty) receive the weights
// including the isolated vertices; partition_out gets one block per original vertex, in the caller's ids.
inline void assign_isolated_nodes(kmp_lp_handle *h, const PreparedGraph &graph, const PartitionedGraphView &p_graph,
                                  NodeID num_isolated_nodes, const PartitionContextView &p_ctx,
                                  std::span<BlockID> partition_out) {
  if (num_isolated_nodes != graph.num_isolated() || partition_out.size() != graph.n() + graph.num_isolated() ||
      (!p_graph.partition.empty() && p_graph.partition.size() != graph.n()) ||
      p_ctx.max_block_weights.size() < p_graph.k ||
      (!p_graph.block_weights.empty() && p_graph.block_weights.size() != p_graph.k)) {
    throw std::invalid_argument("assign_isolated_nodes: wrong span size or isolated vertex count");
  }
  detail::check(kmp_prepared_finish(h, graph.device(), p_graph.k, p_ctx.max_block_weights.data(),
                                    p_graph.partition.empty() ? nullptr : p_graph.partition.data(), partition_out.data(),
                                    p_graph.block_weights.empty() ? nullptr : p_graph.block_weights.data()));
}

// The k block-induced subgraphs of the graph `h` holds (graph::lazy_extract_subgraphs_preprocessing +
// graph::extract_subgraph for every block, subgraph_extractor.cc:181-324), on the device in the reference's
// SubgraphMemory shape: one xadj of n + k entries, block b's local xadj at node_offsets()[b] + b. get() copies them to
// host vectors once; block_nodes() / mapping() are the preprocessing's arrays. Owns device memory of the extracting
// handle's pool: destroy it before that handle.
class Subgraphs {
public:
  struct HostBlocks {
    std::vector<NodeID> node_offsets, edge_offsets; // k + 1 each
    std::vector<EdgeID> nodes;                      // n + k
    std::vector<NodeID> edges;
    std::vector<NodeWeight> node_weights; // empty for unit weights
    std::vector<EdgeWeight> edge_weights; // empty for unit weights
    std::vector<NodeID> mapping, block_nodes;
  };
  explicit Subgraphs(kmp_subgraphs *g, const kmp_subgraph_stats &stats) : _g(g), _stats(stats) {}
  Subgraphs(const Subgraphs &) = delete;
  Subgraphs &operator=(const Subgraphs &) = delete;
  ~Subgraphs() { kmp_subgraphs_destroy(_g); }

  [[nodiscard]] BlockID k() const { return kmp_subgraphs_k(_g); }
  [[nodiscard]] NodeID n() const { return kmp_subgraphs_n(_g); }
  [[nodiscard]] EdgeID m() const { return kmp_subgraphs_m(_g); } // internal directed edges of all blocks
  const HostBlocks &get() {
    if (_host.nodes.empty()) {
      const DeviceArrays d = device_arrays();
      _host.node_offsets.resize(static_cast<std::size_t>(k()) + 1);
      _host.edge_offsets.resize(static_cast<std::size_t>(k()) + 1);
      detail::check(kmp_subgraphs_offsets(_g, _host.node_offsets.data(), _host.edge_offsets.data()));
      _host.nodes.resize(static_cast<std::size_t>(n()) + k());
      _host.edges.resize(m());
      _host.node_weights.resize(d.node_weights != nullptr ? n() : 0);
      _host.edge_weights.resize(d.edge_weights != nullptr ? m() : 0);
      _host.mapping.resize(n());
      _host.block_nodes.resize(n());
      detail::check(kmp_subgraphs_download(_g, _host.nodes.data(), _host.edges.data(), _host.node_weights.data(),
                                           _host.edge_weights.data(), _host.mapping.data(), _host.block_nodes.data()));
    }
    return _host;
  }
  // Block b of get() as a borrowed CSR view (valid while this object and its host copy live).
  CSRGraphView block(BlockID b) {
    const HostBlocks &h = get();
    const NodeID n0 = h.node_offsets[b], n1 = h.node_offsets[b + 1];
    const EdgeID e0 = h.edge_offsets[b], e1 = h.edge_offsets[b + 1];
    return CSRGraphView{std::span<const EdgeID>(h.nodes.data() + n0 + b, n1 - n0 + 1),
                        std::span<const NodeID>(h.edges.data() + e0, e1 - e0),
                        h.node_weights.empty() ? std::span<const NodeWeight>()
                                               : std::span<const NodeWeight>(h.node_weights.data() + n0, n1 - n0),
                        h.edge_weights.empty() ? std::span<const EdgeWeight>()
                                               : std::span<const EdgeWeight>(h.edge_weights.data() + e0, e1 - e0)};
  }
  struct DeviceArrays {
    const std::uint32_t *nodes = nullptr, *edges = nullptr;
    const std::int32_t *node_weights = nullptr, *edge_weights = nullptr;
  };
  [[nodiscard]] DeviceArrays device_arrays() const {
    DeviceArrays d;
    detail::check(kmp_subgraphs_device_arrays(_g, &d.nodes, &d.edges, &d.node_weights, &d.edge_weights, nullptr,
                                              nullptr, nullptr, nullptr));
    return d;
  }
  [[nodiscard]] const kmp_subgraph_stats &stats() const { return _stats; }
  [[nodiscard]] const kmp_subgraphs *device() const { return _g; }

private:
  kmp_subgraphs *_g;
  kmp_subgraph_stats _stats;
  HostBlocks _host;
};

// The block-induced subgraphs of the k-way partition of the graph `h` holds: `partition` (n block ids, loaded as h's
// labels), or, when empty, the labels h holds on the device (e.g. left by the last LP refinement).
inline std::unique_ptr<Subgraphs> extract_subgraphs(kmp_lp_handle *h, BlockID k, std::span<const BlockID> partition = {}) {
  kmp_subgraphs *g = nullptr;
  kmp_subgraph_stats stats{};
  detail::check(kmp_extract_subgraphs(h, k, partition.empty() ? nullptr : partition.data(), &g, &stats));
  return std::make_unique<Subgraphs>(g, stats);
}

// graph::copy_subgraph_partitions(p_graph, subgraph_partitions, k_prime, input_k, mapping) (subgraph_extractor.cc:
// 492-533) on the handle that extracted `subgraphs`: sub_partitions holds every block's sub-partition block-major
// (block b's at node_offsets()[b]; a block that was not split holds zeros). The k'-way result becomes h's labels and
// block weights; `out` (n entries, or empty) receives a host copy.
inline void copy_subgraph_partitions(kmp_lp_handle *h, const Subgraphs &subgraphs,
                                     std::span<const BlockID> sub_partitions, BlockID k_prime, BlockID input_k,
                                     std::span<BlockID> out = {}) {
  if (sub_partitions.size() != subgraphs.n() || (!out.empty() && out.size() != subgraphs.n())) {
    throw std::invalid_argument("copy_subgraph_partitions: wrong span size");
  }
  detail::check(kmp_subgraphs_copy_partitions(h, subgraphs.device(), k_prime, input_k, sub_partitions.data(),
                                              out.empty() ? nullptr : out.data(), nullptr));
}

// InitialBipartitionerWorkerPool::bipartition on every block of `subgraphs` that is split in two, on the device
// (kmp_bipartition_subgraphs): d_sub_partitions (n entries of device memory) receives the block-major sub-partitions
// that copy_subgraph_partitions' device form takes. input_max_block_weights: the input partition context's input_k
// maximum block weights.
inline kmp_bipartition_stats bipartition_subgraphs(kmp_lp_handle *h, const Subgraphs &subgraphs, BlockID k_prime,
                                                   BlockID input_k, std::span<const BlockWeight> input_max_block_weights,
                                                   bool uniform_block_weights, std::int64_t input_total_node_weight,
                                                   double input_epsilon, const kmp_ip_config &cfg, std::int32_t seed,
                                                   std::uint32_t *d_sub_partitions) {
  if (input_max_block_weights.size() != input_k) {
    throw std::invalid_argument("bipartition_subgraphs: input_max_block_weights needs input_k entries");
  }
  kmp_bipartition_stats stats{};
  detail::check(kmp_bipartition_subgraphs(h, subgraphs.device(), k_prime, input_k, input_max_block_weights.data(),
                                          uniform_block_weights ? 1 : 0, input_total_node_weight, input_epsilon, &cfg,
                                          seed, d_sub_partitions, &stats));
  return stats;
}

namespace detail {
// message() of a report: the length query of its kmp_*_report_message, then the text
template <typename R> std::string report_message(int (*format)(const R *, char *, std::size_t), const R *r) {
  const int len = format(r, nullptr, 0);
  std::string out(static_cast<std::size_t>(len > 0 ? len : 0) + 1, '\0');
  format(r, out.data(), out.size());
  out.resize(out.size() - 1);
  return out;
}

// A refused input file: what() is the report's line, report() its first violation.
template <typename Report> class ReadError : public std::runtime_error {
public:
  explicit ReadError(const Report &r) : std::runtime_error("kaminpar_b200: " + r.message()), _report(r) {}
  [[nodiscard]] const Report &report() const { return _report; }

private:
  Report _report;
};

// The status of a read: a refused file (a violation in its report) throws ReadError, any other refusal
// std::runtime_error.
template <typename Report> void check_read(int rc, const Report &r) {
  if (rc != KMP_OK && r.kind != 0) {
    throw ReadError<Report>(r);
  }
  check(rc);
}

// What MetisGraph and ParhipGraph share: the owned result G of a read on the device of the handle that read it, in
// that handle's pool (destroy it before the handle), its report, its four device arrays and their host copy.
template <typename G, typename Report> class ReadGraph {
public:
  struct Host {
    std::vector<EdgeID> xadj;
    std::vector<NodeID> adjncy;
    std::vector<NodeWeight> vwgt;   // empty: unit weights
    std::vector<EdgeWeight> adjwgt; // empty: unit weights
  };

  [[nodiscard]] NodeID n() const { return _n; }
  [[nodiscard]] EdgeID m() const { return _m; }
  [[nodiscard]] const Report &report() const { return _report; }
  [[nodiscard]] const EdgeID *device_xadj() const { return _xadj; }
  [[nodiscard]] const NodeID *device_adjncy() const { return _adjncy; }
  [[nodiscard]] const NodeWeight *device_vwgt() const { return _vwgt; } // null: unit weights
  [[nodiscard]] const EdgeWeight *device_adjwgt() const { return _adjwgt; }

protected:
  ReadGraph(G *g, const Report &r, void (*destroy)(G *), NodeID n, EdgeID m)
      : _g(g, destroy), _report(r), _n(n), _m(m) {}
  // out's arrays sized for this graph and filled by download(g, xadj, adjncy, vwgt, adjwgt, extra...)
  template <typename... Extra>
  void download_into(Host &out, int (*download)(const G *, EdgeID *, NodeID *, NodeWeight *, EdgeWeight *, Extra...),
                     Extra... extra) const {
    out.xadj.resize(static_cast<std::size_t>(_n) + 1);
    out.adjncy.resize(_m);
    out.vwgt.resize(_vwgt != nullptr ? _n : 0);
    out.adjwgt.resize(_adjwgt != nullptr ? _m : 0);
    check(download(_g.get(), out.xadj.data(), out.adjncy.data(), out.vwgt.empty() ? nullptr : out.vwgt.data(),
                   out.adjwgt.empty() ? nullptr : out.adjwgt.data(), extra...));
  }

  std::unique_ptr<G, void (*)(G *)> _g;
  Report _report;
  NodeID _n;
  EdgeID _m;
  const EdgeID *_xadj = nullptr;
  const NodeID *_adjncy = nullptr;
  const NodeWeight *_vwgt = nullptr;
  const EdgeWeight *_adjwgt = nullptr;
};
} // namespace detail

// The report of debug::validate_graph(graph) (csr_graph.cc:266-356) with every edge counted under its first violation
// and the duplicate neighbours beside it (include/kaminpar_b200_validate.h). valid() is the reference's verdict and
// message() its warning line for the first violation.
struct GraphReport : kmp_graph_report {
  [[nodiscard]] bool is_valid() const { return valid != 0; }
  [[nodiscard]] std::string message() const {
    return detail::report_message<kmp_graph_report>(&kmp_graph_report_message, this);
  }
};

// Validates `graph` on the device, stream and pool of `h` (its graph, labels and call counter are not touched). A
// malformed graph is a report, not an exception: only a refused call throws.
inline GraphReport validate_graph(kmp_lp_handle *h, const CSRGraphView &graph) {
  GraphReport r{};
  detail::check(kmp_validate_graph(h, graph.n(), graph.m(), graph.nodes.data(), graph.edges.data(),
                                   graph.edge_weights.empty() ? nullptr : graph.edge_weights.data(), &r));
  return r;
}

// The report of a METIS read (include/kaminpar_b200_io.h): for a graph, the dropped weights and the reference's
// "ignorning extra lines" warning; for a refused file, its first violation.
struct MetisReport : kmp_metis_report {
  [[nodiscard]] std::string message() const {
    return detail::report_message<kmp_metis_report>(&kmp_metis_report_message, this);
  }
};

// A refused METIS file: what() is the report's line, report() its first violation.
using MetisError = detail::ReadError<MetisReport>;

// A METIS file parsed on the device of the handle that read it, in that handle's pool: destroy it before the handle.
// device_*() go straight to kmp_lp_set_graph_device or kmp_prepare_graph_device; download() copies to host arrays
// (the CPU parts of KaMinPar: INTEGRATION.md §2h).
class MetisGraph : public detail::ReadGraph<kmp_metis_graph, MetisReport> {
public:
  MetisGraph(kmp_metis_graph *g, const MetisReport &r)
      : ReadGraph(g, r, &kmp_metis_destroy, kmp_metis_n(g), kmp_metis_m(g)) {
    detail::check(kmp_metis_device_arrays(g, &_xadj, &_adjncy, &_vwgt, &_adjwgt));
  }
  [[nodiscard]] Host download() const {
    Host out;
    download_into(out, &kmp_metis_download);
    return out;
  }
};

// io::metis::read_graph(path) (csr_read, kaminpar-io/metis_parser.cc:158-245) on the device, stream and pool of `h`
// (its graph, labels and call counter are not touched). A malformed file throws MetisError with its first violation;
// any other refusal std::runtime_error.
inline MetisGraph read_metis(kmp_lp_handle *h, const std::string &path) {
  MetisReport r{};
  kmp_metis_graph *g = nullptr;
  detail::check_read(kmp_read_metis(h, path.c_str(), &g, &r), r);
  return MetisGraph(g, r);
}

// The report of a ParHIP read (include/kaminpar_b200_parhip.h): for a refused file, its first violation.
struct ParhipReport : kmp_parhip_report {
  [[nodiscard]] std::string message() const {
    return detail::report_message<kmp_parhip_report>(&kmp_parhip_report_message, this);
  }
};

// A refused ParHIP file: what() is the report's line, report() its first violation.
using ParhipError = detail::ReadError<ParhipReport>;

// The node orderings of read_graph (kaminpar::shm::NodeOrdering, kaminpar.h:66-71)
enum class ParhipOrdering : int {
  NATURAL = KMP_PARHIP_NATURAL,
  DEGREE_BUCKETS = KMP_PARHIP_DEGREE_BUCKETS,
  EXTERNAL_DEGREE_BUCKETS = KMP_PARHIP_EXTERNAL_DEGREE_BUCKETS,
  IMPLICIT_DEGREE_BUCKETS = KMP_PARHIP_IMPLICIT_DEGREE_BUCKETS
};

// A ParHIP file read on the device of the handle that read it, in that handle's pool: destroy it before the handle.
// device_*() go straight to kmp_lp_set_graph_device, kmp_validate_graph_device or kmp_prepare_graph_device;
// download() copies to host arrays (INTEGRATION.md §2i). sorted() and old_to_new are those of the ordering.
class ParhipGraph : public detail::ReadGraph<kmp_parhip_graph, ParhipReport> {
public:
  struct Host : ReadGraph::Host {
    std::vector<NodeID> old_to_new; // empty unless EXTERNAL_DEGREE_BUCKETS
  };

  ParhipGraph(kmp_parhip_graph *g, const ParhipReport &r)
      : ReadGraph(g, r, &kmp_parhip_destroy, kmp_parhip_n(g), kmp_parhip_m(g)) {
    detail::check(kmp_parhip_device_arrays(g, &_xadj, &_adjncy, &_vwgt, &_adjwgt, &_old_to_new));
  }
  [[nodiscard]] bool sorted() const { return kmp_parhip_sorted(_g.get()) != 0; }
  [[nodiscard]] const NodeID *device_old_to_new() const { return _old_to_new; }
  [[nodiscard]] Host download() const {
    Host out;
    out.old_to_new.resize(_old_to_new != nullptr ? n() : 0);
    download_into(out, &kmp_parhip_download, out.old_to_new.empty() ? nullptr : out.old_to_new.data());
    return out;
  }

private:
  const NodeID *_old_to_new = nullptr;
};

// io::parhip::read_graph(path, false, ordering) (kaminpar-io/parhip_parser.cc:580-587) on the device, stream and pool
// of `h` (its graph, labels and call counter are not touched). A malformed file throws ParhipError with its first
// violation; any other refusal std::runtime_error.
inline ParhipGraph read_parhip(kmp_lp_handle *h, const std::string &path,
                               ParhipOrdering ordering = ParhipOrdering::NATURAL) {
  ParhipReport r{};
  kmp_parhip_graph *g = nullptr;
  detail::check_read(kmp_read_parhip(h, path.c_str(), static_cast<int>(ordering), &g, &r), r);
  return ParhipGraph(g, r);
}

} // namespace kaminpar_b200
