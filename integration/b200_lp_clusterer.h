// Glue a KaMinPar maintainer adds to the reference tree (kaminpar-shm/coarsening/clustering/): a Clusterer
// (coarsening/clusterer.h:35-46) that forwards to the GPU engine through include/kaminpar_b200_adapters.hpp.
// This file is OURS (not a copy of reference code); oracle/Makefile target `ref_b200` compiles it together with
// the unmodified reference sources and a generated copy of factories.cc whose LABEL_PROPAGATION case returns it.
#pragma once

#include <span>

#include "kaminpar-shm/coarsening/clusterer.h"
#include "kaminpar-shm/datastructures/csr_graph.h"
#include "kaminpar-shm/datastructures/graph.h"
#include "kaminpar-shm/kaminpar.h"

#include "kaminpar-common/random.h"

#include "kaminpar_b200_adapters.hpp"

namespace kaminpar::shm {

class B200LPClustering final : public Clusterer {
public:
  explicit B200LPClustering(const CoarseningContext &c_ctx)
      : _impl(to_b200(c_ctx.clustering.lp), kaminpar_b200::EngineContext{.seed = Random::get_seed()}) {}

  void set_max_cluster_weight(const NodeWeight weight) final { _impl.set_max_cluster_weight(weight); }
  void set_desired_cluster_count(const NodeID count) final { _impl.set_desired_cluster_count(count); }
  void set_communities(std::span<const NodeID> communities) final { _impl.set_communities(communities); }

  void compute_clustering(StaticArray<NodeID> &clustering, const Graph &graph, const bool free_memory_afterwards) final {
    // compressed graphs are not supported (default preset: compression off, presets.cc:111-114)
    const CSRGraph &csr = concretize<CSRGraph>(graph);
    const kaminpar_b200::CSRGraphView view{
        {csr.raw_nodes().data(), csr.raw_nodes().size()},
        {csr.raw_edges().data(), csr.raw_edges().size()},
        {csr.raw_node_weights().data(), csr.raw_node_weights().size()}, // empty => unit weights
        {csr.raw_edge_weights().data(), csr.raw_edge_weights().size()}};
    if (csr.n() == 0) {
      return;
    }
    _impl.compute_clustering({clustering.data(), clustering.size()}, view, free_memory_afterwards);
  }

private:
  static kaminpar_b200::LabelPropagationCoarseningContext to_b200(const LabelPropagationCoarseningContext &c) {
    kaminpar_b200::LabelPropagationCoarseningContext out;
    out.num_iterations = static_cast<std::size_t>(c.num_iterations);
    out.large_degree_threshold = c.large_degree_threshold;
    out.max_num_neighbors = c.max_num_neighbors;
    out.impl = static_cast<int>(c.impl);
    out.relabel_before_second_phase = c.relabel_before_second_phase;
    out.two_hop_strategy = static_cast<int>(c.two_hop_strategy);
    out.two_hop_threshold = c.two_hop_threshold;
    out.isolated_nodes_strategy = static_cast<int>(c.isolated_nodes_strategy);
    out.tie_breaking_strategy = static_cast<int>(c.tie_breaking_strategy);
    return out;
  }

  kaminpar_b200::LPClustering _impl;
};

} // namespace kaminpar::shm
