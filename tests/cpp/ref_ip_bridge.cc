// Bridge to the UNMODIFIED reference's initial bipartitioner, for tests/test_ip_bridge.py and the generator
// tests/golden/make_ip_golden.py. Compiled against the reference headers and linked against
// oracle/_ref/libkaminpar_ref_full.so (serial oneTBB stand-in: one thread, thread index 0).
//
// ref_ip_bipartition: a Context from a named preset with the kmp_ip_config fields written over it, the input
// partition context at input_k, the block as a CSRGraph; then Random::reseed(seed) and a fresh
// InitialBipartitionerWorkerPool(ctx).bipartition(&block, block_id, current_k, false).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "kaminpar-shm/coarsening/max_cluster_weights.h"
#include "kaminpar-shm/datastructures/csr_graph.h"
#include "kaminpar-shm/datastructures/graph.h"
#include "kaminpar-shm/initial_partitioning/initial_bipartitioner_worker_pool.h"
#include "kaminpar-shm/kaminpar.h"
#include "kaminpar-shm/partitioning/helper.h"
#include "kaminpar-shm/partitioning/partition_utils.h"

#include "kaminpar-common/math.h"

#include "kaminpar-common/datastructures/static_array.h"
#include "kaminpar-common/random.h"

#include "../../include/kaminpar_b200_bipartition.h"

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

void apply_refinement(InitialRefinementContext &r, const kmp_ip_refinement &k) {
  r.algorithms.clear();
  if (k.num_algorithms > 0) {
    r.algorithms.push_back(static_cast<InitialRefinementAlgorithm>(k.algorithm));
  }
  r.fm.num_fruitless_moves = k.num_fruitless_moves;
  r.fm.alpha = k.alpha;
  r.fm.num_iterations = k.num_iterations;
  r.fm.improvement_abortion_threshold = k.improvement_abortion_threshold;
}

struct Setup {
  Context ctx;
  std::unique_ptr<Graph> input; // one vertex carrying the input's total node weight: setup() only reads totals
};

std::unique_ptr<Setup> make_setup(const char *preset, const kmp_ip_config *cfg, uint32_t input_k,
                                  const int32_t *input_max_bw, int uniform, int32_t input_total, double epsilon) {
  auto s = std::make_unique<Setup>();
  s->ctx = create_context_by_preset_name(preset);
  InitialPartitioningContext &ip = s->ctx.initial_partitioning;
  if (cfg != nullptr) {
    ip.coarsening.contraction_limit = cfg->contraction_limit;
    ip.coarsening.convergence_threshold = cfg->convergence_threshold;
    ip.coarsening.large_degree_threshold = cfg->large_degree_threshold;
    ip.coarsening.cluster_weight_limit = static_cast<ClusterWeightLimit>(cfg->cluster_weight_limit);
    ip.coarsening.cluster_weight_multiplier = cfg->cluster_weight_multiplier;
    apply_refinement(ip.pool.refinement, cfg->pool_refinement);
    ip.pool.repetition_multiplier = cfg->repetition_multiplier;
    ip.pool.min_num_repetitions = cfg->min_num_repetitions;
    ip.pool.min_num_non_adaptive_repetitions = cfg->min_num_non_adaptive_repetitions;
    ip.pool.max_num_repetitions = cfg->max_num_repetitions;
    ip.pool.num_seed_iterations = cfg->num_seed_iterations;
    ip.pool.use_adaptive_bipartitioner_selection = cfg->use_adaptive_bipartitioner_selection != 0;
    ip.pool.enable_bfs_bipartitioner = cfg->enable_bfs_bipartitioner != 0;
    ip.pool.enable_ggg_bipartitioner = cfg->enable_ggg_bipartitioner != 0;
    ip.pool.enable_random_bipartitioner = cfg->enable_random_bipartitioner != 0;
    apply_refinement(ip.refinement, cfg->refinement);
    ip.refine_pool_partition = cfg->refine_pool_partition != 0;
    ip.use_adaptive_epsilon = cfg->use_adaptive_epsilon != 0;
  }
  StaticArray<EdgeID> nodes(2);
  nodes[0] = nodes[1] = 0;
  StaticArray<NodeWeight> w(1);
  w[0] = input_total;
  s->input = std::make_unique<Graph>(std::make_unique<CSRGraph>(std::move(nodes), StaticArray<NodeID>(0),
                                                                 std::move(w), StaticArray<EdgeWeight>()));
  if (uniform) {
    s->ctx.partition.setup(*s->input, input_k, epsilon);
  } else {
    s->ctx.partition.setup(*s->input, std::vector<BlockWeight>(input_max_bw, input_max_bw + input_k), false);
  }
  return s;
}

Graph make_block(uint32_t n, uint32_t m, const uint32_t *xadj, const uint32_t *adj, const int32_t *vwgt,
                 const int32_t *adjwgt) {
  return Graph(std::make_unique<CSRGraph>(
      copy_array<EdgeID>(xadj, static_cast<std::size_t>(n) + 1), copy_array<NodeID>(adj, m),
      vwgt ? copy_array<NodeWeight>(vwgt, n) : StaticArray<NodeWeight>(),
      adjwgt ? copy_array<EdgeWeight>(adjwgt, m) : StaticArray<EdgeWeight>()
  ));
}
} // namespace

extern "C" {

// the preset's values as a kmp_ip_config (the multilevel refinement list and the pool's)
int ref_ip_preset_config(const char *preset, kmp_ip_config *out) {
  const Context ctx = create_context_by_preset_name(preset);
  const InitialPartitioningContext &ip = ctx.initial_partitioning;
  auto fill = [](const InitialRefinementContext &r, kmp_ip_refinement &k) {
    k.num_algorithms = static_cast<uint32_t>(r.algorithms.size());
    k.algorithm = r.algorithms.empty() ? 0 : static_cast<int32_t>(r.algorithms.front());
    k.num_fruitless_moves = r.fm.num_fruitless_moves;
    k.alpha = r.fm.alpha;
    k.num_iterations = r.fm.num_iterations;
    k.improvement_abortion_threshold = r.fm.improvement_abortion_threshold;
  };
  out->contraction_limit = ip.coarsening.contraction_limit;
  out->convergence_threshold = ip.coarsening.convergence_threshold;
  out->large_degree_threshold = ip.coarsening.large_degree_threshold;
  out->cluster_weight_limit = static_cast<int32_t>(ip.coarsening.cluster_weight_limit);
  out->cluster_weight_multiplier = ip.coarsening.cluster_weight_multiplier;
  fill(ip.pool.refinement, out->pool_refinement);
  out->repetition_multiplier = ip.pool.repetition_multiplier;
  out->min_num_repetitions = ip.pool.min_num_repetitions;
  out->min_num_non_adaptive_repetitions = ip.pool.min_num_non_adaptive_repetitions;
  out->max_num_repetitions = ip.pool.max_num_repetitions;
  out->num_seed_iterations = ip.pool.num_seed_iterations;
  out->use_adaptive_bipartitioner_selection = ip.pool.use_adaptive_bipartitioner_selection;
  out->enable_bfs_bipartitioner = ip.pool.enable_bfs_bipartitioner;
  out->enable_ggg_bipartitioner = ip.pool.enable_ggg_bipartitioner;
  out->enable_random_bipartitioner = ip.pool.enable_random_bipartitioner;
  fill(ip.refinement, out->refinement);
  out->refine_pool_partition = ip.refine_pool_partition;
  out->use_adaptive_epsilon = ip.use_adaptive_epsilon;
  return static_cast<int>(ip.coarsening.cluster_weight_limit);
}

// params[6]: create_twoway_context's max_block_weight(0, 1), perfectly_balanced_block_weight(0, 1),
// compute_max_cluster_weight and the pool's repetition count: InitialMultilevelBipartitioner::initialize's expression
// (initial_multilevel_bipartitioner.cc:67-72) over the reference's compute_final_k and ceil_log2, clamped as
// InitialPoolBipartitioner::bipartition does (initial_pool_bipartitioner.cc:121-122)
void ref_ip_params(const kmp_ip_config *cfg, uint32_t input_k, const int32_t *input_max_bw, int uniform,
                   int32_t input_total, double epsilon, uint32_t block, uint32_t current_k, uint32_t n, uint32_t m,
                   const uint32_t *xadj, const uint32_t *adj, const int32_t *vwgt, const int32_t *adjwgt,
                   int32_t *params) {
  auto s = make_setup("default", cfg, input_k, input_max_bw, uniform, input_total, epsilon);
  Graph g = make_block(n, m, xadj, adj, vwgt, adjwgt);
  const PartitionContext p = partitioning::create_twoway_context(s->ctx, block, current_k, g);
  params[0] = p.max_block_weight(0);
  params[1] = p.max_block_weight(1);
  params[2] = p.perfectly_balanced_block_weight(0);
  params[3] = p.perfectly_balanced_block_weight(1);
  params[4] = compute_max_cluster_weight<NodeWeight>(s->ctx.initial_partitioning.coarsening, p, g.n(),
                                                     g.total_node_weight());
  const InitialPoolPartitionerContext &pool = s->ctx.initial_partitioning.pool;
  const BlockID num_sub_blocks = partitioning::compute_final_k(block, current_k, s->ctx.partition.k);
  const int reps = std::ceil(pool.repetition_multiplier * num_sub_blocks / math::ceil_log2(s->ctx.partition.k));
  params[5] = std::clamp(reps, pool.min_num_repetitions, pool.max_num_repetitions);
}

void ref_ip_bipartition(const kmp_ip_config *cfg, uint32_t input_k, const int32_t *input_max_bw, int uniform,
                        int32_t input_total, double epsilon, uint32_t block, uint32_t current_k, uint32_t n, uint32_t m,
                        const uint32_t *xadj, const uint32_t *adj, const int32_t *vwgt, const int32_t *adjwgt,
                        int32_t seed, uint32_t *out) {
  auto s = make_setup("default", cfg, input_k, input_max_bw, uniform, input_total, epsilon);
  Graph g = make_block(n, m, xadj, adj, vwgt, adjwgt);
  Random::reseed(seed);
  InitialBipartitionerWorkerPool pool(s->ctx);
  PartitionedGraph pg = pool.bipartition(&g, block, current_k, false);
  for (uint32_t u = 0; u < n; ++u) {
    out[u] = pg.block(u);
  }
}

} // extern "C"
