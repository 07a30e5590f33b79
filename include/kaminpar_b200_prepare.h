/* kaminpar_b200 -- C ABI of the input preparation on the device (DESIGN.md §15): what KaMinPar::compute_partition
 * does with the caller's graph before the first and after the last partitioning step.
 *
 * Restates, for CSR graphs with 32-bit ids / weights (the default build types, kaminpar.h:32-57):
 *
 *   graph::rearrange_by_degree_buckets   kaminpar-shm/graphutils/permutator.cc:19-91, permutator.h:28-209
 *   count_isolated_nodes / CSRGraph::remove_isolated_nodes
 *                                        permutator.cc:266-282, datastructures/csr_graph.cc:150-174
 *   CSRGraph::integrate_isolated_nodes / graph::assign_isolated_nodes / map_original_node
 *                                        csr_graph.cc:176-197, permutator.cc:236-264, kaminpar.cc:419-445
 *
 * Rearrangement (bit for bit the reference's): bucket(u) = floor(log2 deg(u)) + 1, and 32 for a degree-0 vertex,
 * so isolated vertices come last. The new ids are a STABLE sort by bucket (old id order within a bucket). new_xadj
 * is the prefix sum of the degrees in the new order; every adjacency list is written in REVERSE (the reference's
 * p_e = --new_nodes[u]) with its targets relabelled through old_to_new; vertex and edge weights travel with their
 * vertex and edge, and a NULL weight array stays NULL (unit weights).
 *
 * The graph the LP sees has the n' = n - #isolated first vertices and all m edges. The isolated vertices keep their
 * weights on the prepared graph for kmp_prepared_finish. The max block weights a caller passes there are the ones
 * it set up on the FULL graph (compute_partition sets up its PartitionContext, kaminpar.cc:316, before it removes
 * the isolated vertices, :391).
 *
 * The prepared graph owns its device arrays (memory of the handle's device pool, like kmp_coarse_graph), so it
 * outlives a handle's kmp_lp_set_graph_device on coarser levels. The reference's "input already sorted" path and
 * EdgeOrdering::COMPRESSION are not taken: a caller with a sorted graph keeps using kmp_lp_set_graph +
 * kmp_lp_set_graph_sorted. Same error convention as kaminpar_b200_lp.h (0 = ok, kmp_last_error()). No CPU
 * fallback: every call fails without a GPU.
 */
#ifndef KAMINPAR_B200_PREPARE_H
#define KAMINPAR_B200_PREPARE_H

#include <stdint.h>

#include "kaminpar_b200_lp.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct kmp_prepared_graph kmp_prepared_graph;

typedef struct kmp_prepare_stats {
  uint32_t n;               /* vertices of the input */
  uint32_t n_nonisolated;   /* n': vertices the LP sees */
  uint32_t num_isolated;    /* n - n' */
  uint32_t m;               /* directed edges */
  uint32_t kernel_launches; /* hand-written kernels (not CUB's scans) */
  float device_ms;          /* whole call on the device (H2D of host input excluded) */
} kmp_prepare_stats;

/* Rearranges the graph (host arrays: xadj[n+1], adjncy[m], vwgt[n] or NULL, adjwgt[m] or NULL) on the device,
 * stream and memory pool of h. h's own graph, labels and state are not touched. The caller owns *out
 * (kmp_prepared_destroy). stats may be NULL. Refused with KMP_ERR_INVALID before any kernel indexes by them:
 * xadj[0] != 0, a decreasing xadj, xadj[n] != m and a target >= n; n or m >= 2^31 is KMP_ERR_UNSUPPORTED. */
int kmp_prepare_graph(kmp_lp_handle *h, uint32_t n, uint32_t m, const uint32_t *xadj, const uint32_t *adjncy,
                      const int32_t *vwgt, const int32_t *adjwgt, kmp_prepared_graph **out, kmp_prepare_stats *stats);
/* The same from device arrays on h's device (4-byte aligned, as for kmp_lp_set_graph_device). They are only read. */
int kmp_prepare_graph_device(kmp_lp_handle *h, uint32_t n, uint32_t m, const uint32_t *d_xadj,
                             const uint32_t *d_adjncy, const int32_t *d_vwgt, const int32_t *d_adjwgt,
                             kmp_prepared_graph **out, kmp_prepare_stats *stats);

uint32_t kmp_prepared_n(const kmp_prepared_graph *g);            /* n' (non-isolated vertices) */
uint32_t kmp_prepared_num_isolated(const kmp_prepared_graph *g); /* n - n' */
uint32_t kmp_prepared_m(const kmp_prepared_graph *g);

/* Borrowed device pointers (valid until kmp_prepared_destroy); each out-pointer nullable. xadj has n + 1 entries
 * (the n' + 1 first describe the LP's graph; the isolated tail repeats m), vwgt n (NULL for unit weights), adjncy /
 * adjwgt m (adjwgt NULL for unit weights), old_to_new and new_to_old n. */
int kmp_prepared_device_arrays(const kmp_prepared_graph *g, const uint32_t **d_xadj, const uint32_t **d_adjncy,
                               const int32_t **d_vwgt, const int32_t **d_adjwgt, const uint32_t **d_old_to_new,
                               const uint32_t **d_new_to_old);
/* Copy to host arrays (each nullable): xadj[n+1], adjncy[m], vwgt[n], adjwgt[m], old_to_new[n]. A weight array is
 * left untouched when the input had none. */
int kmp_prepared_download(const kmp_prepared_graph *g, uint32_t *xadj, uint32_t *adjncy, int32_t *vwgt,
                          int32_t *adjwgt, uint32_t *old_to_new);

/* kmp_lp_set_graph_device(h, n', m, ...) on the prepared arrays + kmp_lp_set_graph_sorted(h, 1). */
int kmp_lp_set_graph_prepared(kmp_lp_handle *h, const kmp_prepared_graph *g);

/* The partition of the caller's graph from a partition of the n' prepared vertices:
 *   1. bw = block weights of the n' vertices' partition;
 *   2. next fit over the isolated vertices in new-id order (permutator.cc:255-261):
 *        while (b + 1 < k && bw[b] + w(u) > max_block_weights[b]) ++b;  p[u] = b;  bw[b] += w(u)
 *      (b starts at 0; the last block takes whatever is left);
 *   3. partition_out[u] = p[old_to_new[u]] for every original u (HOST array of n entries);
 *   4. block_weights_out[k] (HOST, nullable) = bw including the isolated vertices.
 * partition: HOST array of n' block ids, or NULL for the labels h holds on the device for this prepared graph (set
 * by kmp_lp_set_graph_prepared and a clustering / refinement / balancer / upload since); refused when h's labels
 * belong to another graph. Labels >= k are refused (KMP_ERR_INVALID) before any [k] array is indexed by them. Runs
 * on h's stream; h's labels and block weights are not changed. */
int kmp_prepared_finish(kmp_lp_handle *h, const kmp_prepared_graph *g, uint32_t k, const int32_t *max_block_weights,
                        const uint32_t *partition, uint32_t *partition_out, int32_t *block_weights_out);

/* Frees the arrays stream-ordered on the stream of the handle that prepared the graph: call it before kmp_lp_destroy
 * of that handle, and after any handle that holds the graph (kmp_lp_set_graph_prepared) is done with it. */
void kmp_prepared_destroy(kmp_prepared_graph *g);

#ifdef __cplusplus
}
#endif
#endif
