/* kaminpar_b200 -- C ABI of the partition extension's device steps (DESIGN.md §16): the block-induced subgraphs of a
 * k-way partition and the copy-back of their sub-partitions as a k'-way partition, the two graph passes of
 * extend_partition (partitioning/helper.cc:220-347, rb/rb_multilevel.cc:90-115).
 *
 * Restates, for CSR graphs with 32-bit ids / weights (the default build types, kaminpar.h:32-57):
 *
 *   graph::lazy_extract_subgraphs_preprocessing + graph::extract_subgraph   graphutils/subgraph_extractor.cc:181-324
 *   graph::extract_subgraphs (per block, without its padding slots)         subgraph_extractor.cc:334-490
 *   graph::copy_subgraph_partitions                                         subgraph_extractor.cc:492-533
 *   partitioning::compute_final_k                                           partitioning/partition_utils.cc:21-49
 *
 * The rule (bit for bit the reference's at one thread, where every parallel_for runs in ascending index order and
 * the atomic bucket positions come out in id order; under real TBB that order depends on thread timing and nothing
 * downstream relies on it, so the one-thread order is the canonical form):
 *   - block b's vertices in ascending old id are block_nodes[node_off[b] .. node_off[b+1]); mapping[u] is the rank
 *     of u within its block;
 *   - for each vertex in that order, its neighbours v with part[v] == part[u] in adjacency order, written as
 *     mapping[v] with the edge weight alongside; cut edges are dropped;
 *   - node weights are copied only if the graph has them, likewise edge weights (a NULL array stays NULL);
 *   - an empty block is a graph with n_b = 0 and xadj = [0]; k > n is legal.
 *
 * Layout (the reference's SubgraphMemory shape, nodes.resize(n + k)): one xadj of n + k entries, block b's local
 * xadj (n_b + 1 entries, starting at 0) at xadj + node_off[b] + b, its adjncy / adjwgt at + edge_off[b] and its vwgt at
 * + node_off[b]. A block is therefore a CSR graph in place: kmp_lp_set_graph_device can take it as a view.
 *
 * Extraction is a pure function of the graph and the labels: it changes no LP state and hashes nothing, so it runs
 * on seq_strict and on sharded handles alike (each rank extracts the whole graph it holds). Only a handle inside a
 * stepping call (kmp_lp_step_begin_* .. kmp_lp_step_finish) is refused.
 *
 * The subgraphs own their device arrays (memory of the handle's device pool, like kmp_coarse_graph), so they outlive
 * the handle moving on to another graph. Same error convention as kaminpar_b200_lp.h (0 = ok, kmp_last_error()). No
 * CPU fallback: every call fails without a GPU.
 */
#ifndef KAMINPAR_B200_SUBGRAPH_H
#define KAMINPAR_B200_SUBGRAPH_H

#include <stdint.h>

#include "kaminpar_b200_lp.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct kmp_subgraphs kmp_subgraphs;

typedef struct kmp_subgraph_stats {
  uint32_t n;               /* vertices of the graph */
  uint32_t k;               /* blocks */
  uint32_t m;               /* directed edges of the graph */
  uint32_t m_internal;      /* directed edges kept (both ends in one block) */
  uint32_t kernel_launches; /* hand-written kernels (not CUB's sort and scans) */
  float device_ms;          /* whole call on the device (H2D of a host partition included) */
} kmp_subgraph_stats;

/* The k block-induced subgraphs of the graph h holds, on h's device and stream. partition: HOST array of n block
 * ids, loaded as h's labels (as kmp_lp_upload_partition does), or NULL for h's labels on the device. The caller owns
 * *out (kmp_subgraphs_destroy). stats may be NULL. Refused before any [k] array is indexed by a label:
 *   no graph, or NULL partition without valid labels, k == 0, a label >= k: KMP_ERR_INVALID;
 *   n + k >= 2^32: KMP_ERR_UNSUPPORTED; a handle inside a stepping call: KMP_ERR_INVALID.
 * h's block weights and LP state are not changed. A host partition refused for a label >= k has already been loaded:
 * h's labels are then marked invalid (a NULL partition is refused until new labels are set). */
int kmp_extract_subgraphs(kmp_lp_handle *h, uint32_t k, const uint32_t *partition, kmp_subgraphs **out,
                          kmp_subgraph_stats *stats);

uint32_t kmp_subgraphs_k(const kmp_subgraphs *g);
uint32_t kmp_subgraphs_n(const kmp_subgraphs *g);
uint32_t kmp_subgraphs_m(const kmp_subgraphs *g); /* internal directed edges of all blocks */

/* HOST copies (each nullable) of node_off[k+1] and edge_off[k+1]. */
int kmp_subgraphs_offsets(const kmp_subgraphs *g, uint32_t *node_off, uint32_t *edge_off);
/* HOST copies (each nullable): xadj[n+k], adjncy[m], vwgt[n], adjwgt[m], mapping[n], block_nodes[n]. A weight array
 * is left untouched when the graph had none. */
int kmp_subgraphs_download(const kmp_subgraphs *g, uint32_t *xadj, uint32_t *adjncy, int32_t *vwgt, int32_t *adjwgt,
                           uint32_t *mapping, uint32_t *block_nodes);
/* Borrowed device pointers (valid until kmp_subgraphs_destroy); each out-pointer nullable. vwgt / adjwgt are NULL
 * for unit weights. node_off / edge_off are device copies of the offsets. */
int kmp_subgraphs_device_arrays(const kmp_subgraphs *g, const uint32_t **d_xadj, const uint32_t **d_adjncy,
                                const int32_t **d_vwgt, const int32_t **d_adjwgt, const uint32_t **d_mapping,
                                const uint32_t **d_block_nodes, const uint32_t **d_node_off,
                                const uint32_t **d_edge_off);

/* The k'-way partition from the blocks' sub-partitions (copy_subgraph_partitions):
 *   out[u] = k0[b] + sub[b][mapping[u]],  b = the block of u at extraction,
 * k0 the exclusive prefix sum of the sub-block counts: k_prime / k for every block while k_prime != input_k, and
 * compute_final_k(b, k, input_k) when k_prime == input_k. sub_partitions: HOST array of n sub-block ids in
 * block-major order (block b's subgraph partition at sub_partitions + node_off[b]); a block that was not split holds
 * zeros. Reads only g and the sub-partitions, not h's old labels. The result becomes h's labels (labels_valid) and
 * its k' block weights (h's weight array), so kmp_overload_balance / kmp_lp_refine with a NULL partition follow
 * without a copy; partition_out[n] and block_weights_out[k'] (HOST) are nullable copies.
 * Refused with KMP_ERR_INVALID, h's labels untouched: h is inside a stepping call; h is not the handle g was
 * extracted on, or it has been given a graph since (any kmp_lp_set_graph* call, even of the same arrays);
 * k_prime < k; k_prime != input_k and k_prime % k != 0; sub-block counts that do not add up to k_prime; a sub label
 * >= its block's sub-block count (checked on the device before any label is written). */
int kmp_subgraphs_copy_partitions(kmp_lp_handle *h, const kmp_subgraphs *g, uint32_t k_prime, uint32_t input_k,
                                  const uint32_t *sub_partitions, uint32_t *partition_out,
                                  int32_t *block_weights_out);
/* The same with sub_partitions in device memory on h's device (4-byte aligned; only read). */
int kmp_subgraphs_copy_partitions_device(kmp_lp_handle *h, const kmp_subgraphs *g, uint32_t k_prime,
                                         uint32_t input_k, const uint32_t *d_sub_partitions,
                                         uint32_t *partition_out, int32_t *block_weights_out);

/* Frees the arrays stream-ordered on the stream of the handle that extracted them: call it before kmp_lp_destroy of
 * that handle, and after any handle that holds a block as its graph is done with it. */
void kmp_subgraphs_destroy(kmp_subgraphs *g);

#ifdef __cplusplus
}
#endif
#endif
