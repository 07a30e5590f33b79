/* kaminpar_b200 -- C ABI of block bipartitioning on the device (DESIGN.md §20): KaMinPar's multilevel initial
 * bipartitioner (InitialBipartitionerWorkerPool::bipartition -> InitialMultilevelBipartitioner, initial_partitioning/)
 * on every block of a kmp_subgraphs in one launch, the step between kmp_extract_subgraphs and
 * kmp_subgraphs_copy_partitions_device.
 *
 * The rule, for block b of subgraphs extracted at k blocks and extended to k' blocks:
 *   - s_b = compute_final_k(b, k, input_k) when k' == input_k, else k' / k (the copy-back's rule);
 *   - s_b <= 1 or n_b == 0: the block's sub-partition is all zeros;
 *   - s_b == 2: what the unmodified reference computes at one thread after Random::reseed(seed_b) with a fresh
 *     InitialBipartitionerWorkerPool(ctx).bipartition(&block, b, k, false), seed_b = (int32_t)((uint32_t)seed + b).
 *     "Fresh" includes the construction-time RandomPermutations draws (coarsener, pool refiner, multilevel refiner).
 *     The reference at one thread shares one random stream across blocks and reuses pooled objects; a fresh stream
 *     per block is this library's restatement, and the form that lets one launch cover every block;
 *   - s_b > 2: the whole call is refused (KMP_ERR_UNSUPPORTED); extend in doubling steps instead.
 * With k = 1 and k' = 2 the call bipartitions the whole graph.
 *
 * The input partition context (the reference's ctx.partition at input_k) is given by input_max_block_weights[input_k]
 * (HOST), uniform_block_weights (PartitionContext::setup(graph, k, epsilon) was used), input_total_node_weight and
 * input_epsilon. The epsilon is only read with uniform block weights: the reference's inferred epsilon then derives
 * from it, and the integer block weights do not determine it to the last bit.
 *
 * Same error convention as kaminpar_b200_lp.h (0 = ok, kmp_last_error()). No CPU fallback. */
#ifndef KAMINPAR_B200_BIPARTITION_H
#define KAMINPAR_B200_BIPARTITION_H

#include <stdint.h>

#include "kaminpar_b200_lp.h"
#include "kaminpar_b200_subgraph.h"

#ifdef __cplusplus
extern "C" {
#endif

/* InitialRefinementAlgorithm */
enum { KMP_IP_NOOP = 0, KMP_IP_TWOWAY_SIMPLE_FM = 1, KMP_IP_TWOWAY_ADAPTIVE_FM = 2, KMP_IP_TWOWAY_FLOW = 3 };
/* ClusterWeightLimit */
enum { KMP_IP_CWL_EPSILON_BLOCK_WEIGHT = 0, KMP_IP_CWL_BLOCK_WEIGHT = 1, KMP_IP_CWL_ONE = 2, KMP_IP_CWL_ZERO = 3 };

/* InitialRefinementContext: a list of at most one algorithm (0 entries = NOOP) and its FM settings */
typedef struct kmp_ip_refinement {
  uint32_t num_algorithms;
  int32_t algorithm;
  uint32_t num_fruitless_moves;
  double alpha;
  uint64_t num_iterations;
  double improvement_abortion_threshold;
} kmp_ip_refinement;

/* The fields of InitialPartitioningContext the call supports */
typedef struct kmp_ip_config {
  /* coarsening */
  uint32_t contraction_limit;
  double convergence_threshold;
  uint32_t large_degree_threshold;
  int32_t cluster_weight_limit;
  double cluster_weight_multiplier;
  /* pool */
  kmp_ip_refinement pool_refinement;
  double repetition_multiplier;
  int32_t min_num_repetitions;
  int32_t min_num_non_adaptive_repetitions;
  int32_t max_num_repetitions;
  int32_t num_seed_iterations;
  int32_t use_adaptive_bipartitioner_selection;
  int32_t enable_bfs_bipartitioner;
  int32_t enable_ggg_bipartitioner;
  int32_t enable_random_bipartitioner;
  /* multilevel */
  kmp_ip_refinement refinement;
  int32_t refine_pool_partition;
  int32_t use_adaptive_epsilon;
} kmp_ip_config;

/* The default preset's values (presets.cc:188-327). */
kmp_ip_config kmp_ip_default_config(void);

typedef struct kmp_bipartition_stats {
  uint32_t blocks_split;      /* blocks with s_b == 2 and n_b > 0 */
  uint32_t pool_runs;         /* flat bipartitioner runs, summed over the blocks */
  uint32_t coarsening_levels; /* summed over the blocks */
  uint32_t arena_retries;     /* blocks run again with a doubled arena */
  uint32_t kernel_launches;
  float device_ms;
} kmp_bipartition_stats;

/* The sub-partitions of every block of g into d_sub_partitions (n entries, device, 4-byte aligned, block-major:
 * block b's at node_off[b]), exactly what kmp_subgraphs_copy_partitions_device takes. Refused before anything is
 * written, the handle's labels and weights untouched:
 *   KMP_ERR_INVALID: a NULL argument, a NULL or misaligned d_sub_partitions, h inside a stepping call, g not extracted
 *     on h or h given a graph since, k' < k, k' neither input_k nor a multiple of k, input_k == 0 or input_k < k',
 *     a configuration value out of range;
 *   KMP_ERR_UNSUPPORTED: k not a power of two (the reference's extension runs at power-of-two k; for other k its
 *     sub-block ranges can run past input_k), some s_b > 2, a refinement list longer than one, TWOWAY_FLOW, every
 *     bipartitioner disabled. stats may be NULL. */
/* The CUDA device ordinal h runs on, where d_sub_partitions must lie; -1 for a NULL handle. */
int kmp_lp_handle_device(const kmp_lp_handle *h);

int kmp_bipartition_subgraphs(kmp_lp_handle *h, const kmp_subgraphs *g, uint32_t k_prime, uint32_t input_k,
                              const int32_t *input_max_block_weights, int uniform_block_weights,
                              int64_t input_total_node_weight, double input_epsilon, const kmp_ip_config *cfg,
                              int32_t seed, uint32_t *d_sub_partitions, kmp_bipartition_stats *stats);

#ifdef __cplusplus
}
#endif
#endif
