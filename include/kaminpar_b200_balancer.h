/* kaminpar_b200 -- C ABI of the overload and underload balancers on the device (H100, sm_90a).
 *
 *   kmp_overload_balance  <->  OverloadBalancer::refine(PartitionedGraph&, const PartitionContext&)
 *                              kaminpar-shm/refinement/balancer/overload_balancer.cc:51-160
 *
 * It works on the graph a kmp_lp_handle holds (kmp_lp_set_graph / kmp_lp_set_graph_device), so that a
 * refinement level can balance and run LP on the device without a host round trip in between:
 *   kmp_lp_upload_partition -> kmp_overload_balance(partition_inout = NULL) -> kmp_lp_refine(partition_inout = NULL)
 *   -> kmp_lp_download_labels.
 *
 * The selection rule is the reference's, restated without thread order (DESIGN.md §11): synchronous rounds
 * against the block weights frozen at the start of the round; per overloaded block the candidates are taken by
 * (relative gain desc, vertex id asc) until the overload is covered; the moves are committed by the order-free
 * ladder of the LP refiner (one pass), so no block ever ends above its maximum by a move of this call. Rounds stop
 * when no block is overloaded, when a round proposes no move, or after KMP_BALANCE_MAX_ROUNDS.
 *
 * Refused: handles created with schedule KMP_SCHEDULE_SEQ_STRICT, sharded handles (kmp_lp_set_shard,
 * kmp_lp_dist_init) and handles in use by the stepping API (KMP_ERR_UNSUPPORTED); labels >= k, e.g. a clustering
 * left on the device by kmp_lp_cluster (KMP_ERR_INVALID; checked before any label indexes a [k] array). Labels are
 * only checked against k: a clustering whose ids all happen to be < k is indistinguishable from a partition.
 */
#ifndef KAMINPAR_B200_BALANCER_H
#define KAMINPAR_B200_BALANCER_H

#include <stdint.h>

#include "kaminpar_b200_lp.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Rounds of one kmp_overload_balance call stop at this many (each round that moves a vertex lowers the total
 * overload, so the cap only bounds pathological inputs). */
#define KMP_BALANCE_MAX_ROUNDS 64

typedef struct kmp_balance_stats {
  uint32_t rounds;           /* rounds executed (the last one may have accepted no move) */
  uint32_t moved[64];        /* accepted moves per round */
  int64_t overload_before;   /* metrics::total_overload before / after the call */
  int64_t overload_after;
  uint64_t candidates;       /* sum over the rounds of the vertices in overloaded blocks */
  uint64_t edges_scanned;    /* their adjacency entries */
  uint64_t kernel_launches;
  float device_ms;           /* CUDA-event time of the whole call on the handle's stream */
} kmp_balance_stats;

/* OverloadBalancer::refine on the graph the handle holds. partition_inout: HOST buffer of n BlockIDs, balanced in
 * place, or NULL = the labels left on the device by kmp_lp_upload_partition / kmp_lp_refine (they stay there;
 * KMP_ERR_INVALID when the device holds no labels of the current graph, or labels >= k).
 * max_block_weights[k] (PartitionContext::max_block_weight), perfectly_balanced_block_weights[k]
 * (PartitionContext::perfectly_balanced_block_weight; the floating-point part stays with the caller).
 * block_weights_out[k] nullable, stats nullable. *improved_out = the reference's return value: 0 when the input
 * had no overloaded block (nothing is touched then), else 1. */
int kmp_overload_balance(kmp_lp_handle *h, uint32_t k, const int32_t *max_block_weights,
                         const int32_t *perfectly_balanced_block_weights, uint32_t *partition_inout,
                         int32_t *block_weights_out, int *improved_out, kmp_balance_stats *stats);

/* T0 parity hook: target and key (the reference's float relative gain) of EVERY vertex against frozen labels /
 * block weights, as round `round` of call `call_index` would compute them; no moves. target_out[u] = labels[u]
 * (key from gain INT32_MIN) when no adjacent block other than labels[u] has room for u. HOST buffers.
 * It loads `labels`, `block_weights` and `max_block_weights` into the handle's device state: labels left on the
 * device by kmp_lp_upload_partition / kmp_lp_refine / kmp_overload_balance are overwritten. */
int kmp_balance_select_all(kmp_lp_handle *h, uint32_t k, const uint32_t *labels, const int32_t *block_weights,
                           const int32_t *max_block_weights, uint32_t call_index, uint32_t round,
                           uint32_t *target_out, float *key_out);

/* ---- underload balancer -------------------------------------------------------------------------------------
 *
 *   kmp_underload_balance  <->  UnderloadBalancer::refine(PartitionedGraph&, const PartitionContext&)
 *                               kaminpar-shm/refinement/balancer/underload_balancer.cc:39-104
 *
 * The last stage of the default refinement chain: it moves vertices into blocks below their minimum weight
 * (PartitionContext::min_block_weight), so that upload -> kmp_overload_balance -> kmp_lp_refine ->
 * kmp_underload_balance -> download runs without a host copy between the stages.
 *
 * The rule is the reference's, restated without thread order (DESIGN.md §12): synchronous rounds against the block
 * weights and underloaded flags frozen at the start of the round; a vertex may leave its block b iff b is not
 * underloaded and W[b] - w(u) >= min[b]; its target is the best adjacent underloaded block with room; per target
 * block the candidates are taken by (relative gain desc, vertex id asc) until its deficit min - W is covered; the
 * moves are committed by the LP refiner's ladder with the minimum weights (one pass), so no block ends above its
 * maximum and no block ends below its minimum because a vertex left it. Rounds stop when every block is at or above
 * its minimum, when a round proposes no move, or after KMP_BALANCE_MAX_ROUNDS.
 *
 * Refused like kmp_overload_balance: seq_strict, sharded, NCCL and stepping handles (KMP_ERR_UNSUPPORTED); labels
 * >= k (KMP_ERR_INVALID; checked before any label indexes a [k] array). */
typedef struct kmp_underload_stats {
  uint32_t rounds;           /* rounds executed (the last one may have accepted no move) */
  uint32_t moved[64];        /* accepted moves per round */
  int64_t underload_before;  /* sum over the blocks of max(0, min[b] - W[b]) before / after the call */
  int64_t underload_after;
  uint64_t candidates;       /* sum over the rounds of the vertices that may leave their block */
  uint64_t edges_scanned;    /* their adjacency entries */
  uint64_t kernel_launches;
  float device_ms;           /* CUDA-event time of the whole call on the handle's stream */
} kmp_underload_stats;

/* UnderloadBalancer::refine on the graph the handle holds. partition_inout: HOST buffer of n BlockIDs, balanced in
 * place, or NULL = the labels on the device (they stay there; refused as by kmp_overload_balance). max_block_weights[k], min_block_weights[k]
 * (PartitionContext::min_block_weight). min_block_weights = NULL means the context has no minimum weights: then
 * *improved_out = 0 and nothing runs on the device (block_weights_out is not written). block_weights_out[k]
 * nullable, stats nullable. *improved_out = the reference's return value: 0 when every block is at or above its
 * minimum (nothing is touched then), else 1. */
int kmp_underload_balance(kmp_lp_handle *h, uint32_t k, const int32_t *max_block_weights,
                          const int32_t *min_block_weights, uint32_t *partition_inout, int32_t *block_weights_out,
                          int *improved_out, kmp_underload_stats *stats);

/* T0 parity hook: target and key of EVERY vertex against frozen labels / block weights, as round `round` of call
 * `call_index` would compute them; no moves. target_out[u] = labels[u] (key from gain INT32_MIN) when u may not
 * leave its block or no adjacent underloaded block has room for it. HOST buffers. Like kmp_balance_select_all it
 * overwrites the labels, block weights and maximum weights held on the device. */
int kmp_underload_select_all(kmp_lp_handle *h, uint32_t k, const uint32_t *labels, const int32_t *block_weights,
                             const int32_t *max_block_weights, const int32_t *min_block_weights, uint32_t call_index,
                             uint32_t round, uint32_t *target_out, float *key_out);

#ifdef __cplusplus
}
#endif
#endif
