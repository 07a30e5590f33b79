// Host twin of the device initial bipartitioner (DESIGN.md §20): the engine of kaminpar_b200/csrc/kmp_bipartition.cuh
// and the parameter code of kaminpar_b200/csrc/kmp_ip_params.h, compiled with g++ (no FMA contraction:
// -ffp-contract=off) and called from tests/test_ip_oracle.py and tests/test_ip_bridge.py through ctypes.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../kaminpar_b200/csrc/kmp_bipartition.cuh"
#include "../../kaminpar_b200/csrc/kmp_ip_params.h"

namespace {
kmp_ip::FmParams fm_params(const kmp_ip_refinement &r) {
  kmp_ip::FmParams f;
  f.algorithm = r.num_algorithms == 0 ? kmp_ip::kRefineNoop : static_cast<uint32_t>(r.algorithm);
  f.num_fruitless_moves = r.num_fruitless_moves;
  f.alpha = r.alpha;
  f.num_iterations = r.num_iterations;
  f.improvement_abortion_threshold = r.improvement_abortion_threshold;
  return f;
}
} // namespace

extern "C" {

kmp_ip_config ip_default_config() { return kmp_ip_params::default_config(); }

// params[6]: max_bw[2], perfect_bw[2], max_cluster_weight, clamped repetitions; 0 when the block's sub-block range
// runs past input_k (params untouched)
int ip_block_params(uint32_t input_k, const int32_t *input_max_bw, int uniform, int32_t input_total, double epsilon,
                     const kmp_ip_config *cfg, uint32_t block, uint32_t current_k, uint32_t n, uint32_t m,
                     int32_t total_nw, int32_t max_nw, int32_t total_ew, int32_t *params) {
  const kmp_ip_params::InputContext in{input_k, input_max_bw, uniform != 0, input_total, epsilon};
  const kmp_ip_params::BlockStats g{n, m, total_nw, max_nw, total_ew};
  return kmp_ip_params::block_params(in, *cfg, block, current_k, g, params) ? 1 : 0;
}

uint32_t ip_compute_final_k(uint32_t block, uint32_t current_k, uint32_t input_k) {
  return kmp_ip_params::compute_final_k(block, current_k, input_k);
}

// one block; returns 0 ok, 1 arena overflow. counters[2]: pool runs, coarsening levels
int ip_host_bipartition(uint32_t n, uint32_t m, const uint32_t *xadj, const uint32_t *adj, const int32_t *vwgt,
                        const int32_t *adjwgt, const kmp_ip_config *cfg, const int32_t *params, int32_t seed,
                        uint64_t arena_bytes, uint32_t *out, uint32_t *counters) {
  kmp_ip::Config c{};
  c.contraction_limit = cfg->contraction_limit;
  c.convergence_threshold = cfg->convergence_threshold;
  c.large_degree_threshold = cfg->large_degree_threshold;
  c.pool_fm = fm_params(cfg->pool_refinement);
  c.fm = fm_params(cfg->refinement);
  c.min_num_non_adaptive_repetitions = cfg->min_num_non_adaptive_repetitions;
  c.use_adaptive_bipartitioner_selection = cfg->use_adaptive_bipartitioner_selection;
  c.enable_bfs = cfg->enable_bfs_bipartitioner;
  c.enable_ggg = cfg->enable_ggg_bipartitioner;
  c.enable_random = cfg->enable_random_bipartitioner;
  c.refine_pool_partition = cfg->refine_pool_partition;
  kmp_ip::BlockParams bp{{params[0], params[1]}, {params[2], params[3]}, params[4], params[5]};
  if (arena_bytes == 0) {
    arena_bytes = kmp_ip::arena_bound(n, m);
  }
  std::vector<uint8_t> mem(arena_bytes, 0);
  kmp_ip::Counters cnt{0, 0};
  const bool ok = kmp_ip::bipartition_block(n, m, xadj, adj, vwgt, adjwgt, c, cfg->num_seed_iterations, bp, seed,
                                            mem.data(), arena_bytes, out, cnt);
  counters[0] = cnt.pool_runs;
  counters[1] = cnt.levels;
  return ok ? 0 : 1;
}

} // extern "C"
