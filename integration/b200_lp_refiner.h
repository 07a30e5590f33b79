// Glue a KaMinPar maintainer adds to the reference tree (kaminpar-shm/refinement/lp/): a Refiner
// (refinement/refiner.h:34-56) that forwards to the GPU engine. OUR file; compiled by `make -C oracle ref_b200`.
//
// Labels and block weights of the PartitionedGraph must stay consistent (partitioned_graph.h:117-135). The class
// has no block-weight setter, so the engine refines a COPY of the partition and the changed vertices are
// written back through PartitionedGraph::set_block (partitioned_graph.h:194-214), which maintains the block
// weights itself.
#pragma once

#include <span>
#include <string>
#include <vector>

#include "kaminpar-shm/datastructures/csr_graph.h"
#include "kaminpar-shm/datastructures/graph.h"
#include "kaminpar-shm/datastructures/partitioned_graph.h"
#include "kaminpar-shm/kaminpar.h"
#include "kaminpar-shm/refinement/refiner.h"

#include "kaminpar-common/random.h"

#include "kaminpar_b200_adapters.hpp"

namespace kaminpar::shm {

class B200LabelPropagationRefiner final : public Refiner {
public:
  explicit B200LabelPropagationRefiner(const Context &ctx)
      : _impl(to_b200(ctx.refinement.lp), kaminpar_b200::EngineContext{.seed = Random::get_seed()}) {}

  [[nodiscard]] std::string name() const final { return "Label Propagation (B200)"; }

  void set_communities(std::span<const NodeID> communities) final { _impl.set_communities(communities); }

  void initialize(const PartitionedGraph &p_graph) final {
    if (p_graph.graph().n() != 0) {
      _impl.initialize(view_of(p_graph, {}, {}));
    }
  }

  bool refine(PartitionedGraph &p_graph, const PartitionContext &p_ctx) final {
    const NodeID n = p_graph.graph().n();
    if (n == 0) {
      return true;
    }
    _partition.assign(p_graph.raw_partition().data(), p_graph.raw_partition().data() + n);
    _block_weights.assign(p_ctx.k, 0);
    auto pg = view_of(p_graph, _partition, _block_weights);
    std::vector<BlockWeight> min_w;
    if (p_ctx.has_min_block_weights()) {
      for (BlockID b = 0; b < p_ctx.k; ++b) {
        min_w.push_back(p_ctx.min_block_weight(b));
      }
    }
    const kaminpar_b200::PartitionContextView pc{p_ctx.k, p_ctx.max_block_weights(), min_w};
    const bool result = _impl.refine(pg, pc);
    for (NodeID u = 0; u < n; ++u) {
      if (_partition[u] != p_graph.block(u)) {
        p_graph.set_block(u, _partition[u]); // keeps the block weights consistent
      }
    }
    return result;
  }

private:
  static kaminpar_b200::LabelPropagationRefinementContext to_b200(const LabelPropagationRefinementContext &c) {
    kaminpar_b200::LabelPropagationRefinementContext out;
    out.num_iterations = static_cast<std::size_t>(c.num_iterations);
    out.large_degree_threshold = c.large_degree_threshold;
    out.max_num_neighbors = c.max_num_neighbors;
    out.impl = static_cast<int>(c.impl);
    out.tie_breaking_strategy = static_cast<int>(c.tie_breaking_strategy);
    return out;
  }

  static kaminpar_b200::PartitionedGraphView
  view_of(const PartitionedGraph &p, std::span<BlockID> partition, std::span<BlockWeight> block_weights) {
    const CSRGraph &csr = concretize<CSRGraph>(p.graph());
    return {{{csr.raw_nodes().data(), csr.raw_nodes().size()},
             {csr.raw_edges().data(), csr.raw_edges().size()},
             {csr.raw_node_weights().data(), csr.raw_node_weights().size()},
             {csr.raw_edge_weights().data(), csr.raw_edge_weights().size()}},
            p.k(),
            partition,
            block_weights};
  }

  kaminpar_b200::LabelPropagationRefiner _impl;
  std::vector<BlockID> _partition;
  std::vector<BlockWeight> _block_weights;
};

} // namespace kaminpar::shm
