// Per-block parameters of the initial bipartitioner (DESIGN.md §20), computed on the host in the reference's double
// code and expression order, from per-block reductions. Host-only C++: the library (kmp_lp.cu) and the CPU test
// harness (tests/cpp/ip_host_check.cc) include the same code. std::pow and std::ceil here are the host libm's, as in
// the reference; CUDA's pow is not correctly rounded and is never used for these values.
//
//   partitioning::create_twoway_context      partitioning/helper.cc:63-141
//   PartitionContext::setup (relaxation)     context.cc:41-70, kaminpar.h:436-491
//   compute_max_cluster_weight               coarsening/max_cluster_weights.h (InitialCoarseningContext overload)
//   repetition count                         initial_multilevel_bipartitioner.cc:67-72, pool clamp :121-122
//   compute_final_k / split_integral         partitioning/partition_utils.cc, kaminpar-common/math.h
#pragma once

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <vector>

#include "../../include/kaminpar_b200_bipartition.h"

namespace kmp_ip_params {

inline uint32_t floor_log2(uint32_t x) { return x == 0 ? 0 : 31u - static_cast<uint32_t>(__builtin_clz(x)); }
inline uint32_t ceil_log2(uint32_t x) { return floor_log2(x) + 1 - ((x & (x - 1)) == 0); }

inline uint32_t compute_final_k(uint32_t block, uint32_t current_k, uint32_t input_k) {
  if (current_k == input_k) {
    return 1;
  }
  const uint32_t level = floor_log2(current_k);
  const uint32_t base = input_k >> level;
  const uint32_t num_plus_one_blocks = input_k & ((1u << level) - 1);
  uint32_t rev = 0;
  for (int i = 0; i < 32; ++i) {
    rev |= ((block >> i) & 1u) << (31 - i);
  }
  const int64_t reversed_block = level == 0 ? 0 : static_cast<int64_t>(rev) >> (32 - level);
  return base + (reversed_block < num_plus_one_blocks);
}

inline void split_integral(uint32_t value, uint32_t &lhs, uint32_t &rhs) {
  lhs = static_cast<uint32_t>(std::ceil(value * 0.5));
  rhs = static_cast<uint32_t>(std::floor(value * (1.0 - 0.5)));
}

inline uint32_t compute_first_sub_block(uint32_t block, uint32_t current_k, uint32_t input_k) {
  if (current_k == 1) {
    return 0;
  }
  const int level = static_cast<int>(ceil_log2(current_k));
  int mask = 1 << (level - 1);
  uint32_t width = 1, current_value = input_k, ans = 0;
  while (width <= current_k) {
    width *= 2;
    uint32_t lhs, rhs;
    split_integral(current_value, lhs, rhs);
    if (block & mask) {
      current_value = rhs;
      ans += lhs;
    } else {
      current_value = lhs;
    }
    mask >>= 1;
  }
  return ans;
}

// the input graph's PartitionContext at input_k
struct InputContext {
  uint32_t k;
  const int32_t *max_block_weights; // [k]
  bool uniform;
  int32_t total_node_weight;
  double epsilon; // read only when uniform
  double inferred_epsilon() const {
    if (total_node_weight == 0) {
      return 0.0;
    }
    if (uniform) {
      const double max = (1.0 + epsilon) * std::ceil(1.0 * total_node_weight / k);
      return max / std::ceil(1.0 * total_node_weight / k) - 1.0;
    }
    int32_t total_max = 0;
    for (uint32_t b = 0; b < k; ++b) {
      total_max += max_block_weights[b];
    }
    return 1.0 * total_max / total_node_weight - 1.0;
  }
  int32_t total_max_block_weights(uint32_t begin, uint32_t end) const {
    if (uniform) {
      return max_block_weights[begin] * static_cast<int32_t>(end - begin);
    }
    int32_t s = 0;
    for (uint32_t b = begin; b < end; ++b) {
      s += max_block_weights[b];
    }
    return s;
  }
};

// the reductions of one block graph (CSRGraph's totals: a missing weight array counts every weight as 1)
struct BlockStats {
  uint32_t n, m;
  int32_t total_node_weight, max_node_weight, total_edge_weight;
};

// the two-way PartitionContext of one block (create_twoway_context + setup(graph, max_block_weights, true))
struct TwowayContext {
  int32_t unrelaxed[2];
  int32_t max_bw[2];
  int32_t total_node_weight;
  double inferred_epsilon() const {
    if (total_node_weight == 0) {
      return 0.0;
    }
    return 1.0 * (unrelaxed[0] + unrelaxed[1]) / total_node_weight - 1.0;
  }
  int32_t perfectly_balanced_block_weight(int b) const {
    return static_cast<int32_t>(std::ceil(1.0 * unrelaxed[b] / (1 + inferred_epsilon())));
  }
};

inline TwowayContext create_twoway_context(const InputContext &in, bool use_adaptive_epsilon, uint32_t block,
                                           uint32_t current_k, const BlockStats &g) {
  const uint32_t first_sub_block = compute_first_sub_block(block, current_k, in.k);
  const uint32_t first_invalid_sub_block = first_sub_block + compute_final_k(block, current_k, in.k);
  const uint32_t num_sub_blocks = compute_final_k(block, current_k, in.k);
  uint32_t b0, b1;
  split_integral(num_sub_blocks, b0, b1);
  int32_t mbw[2] = {in.total_max_block_weights(first_sub_block, first_sub_block + b0),
                    in.total_max_block_weights(first_sub_block + b0, first_invalid_sub_block)};
  if (in.uniform && use_adaptive_epsilon) {
    const double base = (1.0 + in.inferred_epsilon()) * num_sub_blocks * in.total_node_weight / in.k /
                        g.total_node_weight;
    const double exponent = 1.0 / ceil_log2(num_sub_blocks);
    const double epsilon_prime = std::pow(base, exponent) - 1.0;
    const double adapted_eps = std::max(epsilon_prime, 0.0001);
    const int32_t total_max_weight = mbw[0] + mbw[1];
    const double ratios[2] = {1.0 * mbw[0] / total_max_weight, 1.0 * mbw[1] / total_max_weight};
    for (int b = 0; b < 2; ++b) {
      mbw[b] = static_cast<int32_t>((1.0 + adapted_eps) * g.total_node_weight * ratios[b]);
    }
  }
  TwowayContext t;
  t.unrelaxed[0] = t.max_bw[0] = mbw[0];
  t.unrelaxed[1] = t.max_bw[1] = mbw[1];
  t.total_node_weight = g.total_node_weight;
  const double eps = t.inferred_epsilon();
  for (int b = 0; b < 2; ++b) {
    t.max_bw[b] = std::max<int32_t>(t.max_bw[b], std::ceil(1.0 * t.max_bw[b] / (1.0 + eps)) + g.max_node_weight);
  }
  return t;
}

inline int32_t compute_max_cluster_weight(const kmp_ip_config &cfg, const TwowayContext &t, uint32_t n,
                                          int64_t total_node_weight) {
  double w = 0.0;
  switch (cfg.cluster_weight_limit) {
  case KMP_IP_CWL_EPSILON_BLOCK_WEIGHT:
    w = (t.inferred_epsilon() * total_node_weight) / std::clamp<uint32_t>(n / cfg.contraction_limit, 2, 2);
    break;
  case KMP_IP_CWL_BLOCK_WEIGHT:
    w = (1.0 + t.inferred_epsilon()) * total_node_weight / 2u;
    break;
  case KMP_IP_CWL_ONE:
    w = 1.0;
    break;
  default:
    w = 0.0;
    break;
  }
  return static_cast<int32_t>(w * cfg.cluster_weight_multiplier);
}

// repetitions before the pool's clamp
inline int32_t num_repetitions(const kmp_ip_config &cfg, uint32_t block, uint32_t current_k, uint32_t input_k) {
  const uint32_t num_sub_blocks = compute_final_k(block, current_k, input_k);
  return static_cast<int32_t>(std::ceil(cfg.repetition_multiplier * num_sub_blocks / ceil_log2(input_k)));
}

// the block's sub-block range [first, first + compute_final_k) lies inside the input's input_k blocks; it always
// does for power-of-two current_k, the only k the reference's extension uses
inline bool sub_block_range_valid(uint32_t block, uint32_t current_k, uint32_t input_k) {
  return static_cast<uint64_t>(compute_first_sub_block(block, current_k, input_k)) +
             compute_final_k(block, current_k, input_k) <=
         input_k;
}

// everything the engine needs for one block: {max_bw[2], perfect_bw[2], max_cluster_weight, clamped repetitions};
// false (out untouched) when the block's sub-block range runs past input_k
inline bool block_params(const InputContext &in, const kmp_ip_config &cfg, uint32_t block, uint32_t current_k,
                         const BlockStats &g, int32_t out[6]) {
  if (!sub_block_range_valid(block, current_k, in.k)) {
    return false;
  }
  const TwowayContext t = create_twoway_context(in, cfg.use_adaptive_epsilon != 0, block, current_k, g);
  out[0] = t.max_bw[0];
  out[1] = t.max_bw[1];
  out[2] = t.perfectly_balanced_block_weight(0);
  out[3] = t.perfectly_balanced_block_weight(1);
  out[4] = compute_max_cluster_weight(cfg, t, g.n, g.total_node_weight);
  out[5] = std::clamp(num_repetitions(cfg, block, current_k, in.k), cfg.min_num_repetitions, cfg.max_num_repetitions);
  return true;
}

inline kmp_ip_config default_config() {
  kmp_ip_config c{};
  c.contraction_limit = 20;
  c.convergence_threshold = 0.05;
  c.large_degree_threshold = 1000000;
  c.cluster_weight_limit = KMP_IP_CWL_BLOCK_WEIGHT;
  c.cluster_weight_multiplier = 1.0 / 12.0;
  c.pool_refinement = {1, KMP_IP_TWOWAY_SIMPLE_FM, 100, 1.0, 5, 0.0001};
  c.repetition_multiplier = 1.0;
  c.min_num_repetitions = 10;
  c.min_num_non_adaptive_repetitions = 5;
  c.max_num_repetitions = 50;
  c.num_seed_iterations = 1;
  c.use_adaptive_bipartitioner_selection = 1;
  c.enable_bfs_bipartitioner = 1;
  c.enable_ggg_bipartitioner = 1;
  c.enable_random_bipartitioner = 1;
  c.refinement = {1, KMP_IP_TWOWAY_SIMPLE_FM, 100, 1.0, 5, 0.0001};
  c.refine_pool_partition = 0;
  c.use_adaptive_epsilon = 1;
  return c;
}

} // namespace kmp_ip_params
