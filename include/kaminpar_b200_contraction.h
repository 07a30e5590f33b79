/* kaminpar_b200 -- C ABI of the device-side cluster contraction (SURVEY.md §8f rank 1: the step that
 * follows LP clustering on every coarsening level).
 *
 * Replaces, for CSR graphs with 32-bit ids / weights (the default build types, kaminpar.h:32-57):
 *
 *   contract_clustering(graph, clustering, con_ctx[, m_ctx]) -> std::unique_ptr<CoarseGraph>
 *       kaminpar-shm/coarsening/contraction/cluster_contraction.h:47-56
 *       (default algorithm UNBUFFERED, presets.cc:181-183;
 *        kaminpar-shm/coarsening/contraction/unbuffered_cluster_contraction.cc:127-606)
 *   CoarseGraph::get() / project_up() / project_down()
 *       kaminpar-shm/coarsening/contraction/cluster_contraction.h:22-32,
 *       cluster_contraction_preprocessing.h:18-51
 *
 * Result: the coarse CSR graph (summed node and edge weights, no self-loops, no parallel edges) and
 * the fine -> coarse mapping. Coarse ids are the ranks of the used cluster (leader) ids
 * (cluster_contraction_preprocessing.cc:17-51) and every adjacency list is sorted by target. The
 * reference additionally renumbers the coarse vertices in the order its threads finish them and
 * emits adjacency lists in hash-map insertion order; both are scheduling artefacts of its
 * implementation (they change from run to run with more than one thread), so parity is defined up
 * to that relabelling -- oracle/contraction_oracle.py: canonicalize().
 *
 * The graph is the one the kmp_lp_handle holds (kmp_lp_set_graph / kmp_lp_set_graph_device), so a
 * coarsening level is: kmp_lp_cluster -> kmp_contract_clustering(h, NULL, ...) (the clustering
 * stays on the device) -> kmp_coarse_device_arrays -> kmp_lp_set_graph_device on the next level's
 * handle. Same error convention as kaminpar_b200_lp.h (0 = ok, kmp_last_error()). No CPU fallback.
 */
#ifndef KAMINPAR_B200_CONTRACTION_H
#define KAMINPAR_B200_CONTRACTION_H

#include <stdint.h>

#include "kaminpar_b200_lp.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct kmp_coarse_graph kmp_coarse_graph;

typedef struct kmp_contraction_stats {
  uint32_t c_n;            /* coarse vertices */
  uint32_t c_m;            /* coarse directed edges */
  uint64_t cut_edges;      /* fine directed edges between different clusters (the sorted items) */
  uint32_t sort_bits;      /* key bits the radix sort ran over */
  uint32_t kernel_launches;
  float device_ms;         /* whole call on the device (H2D of the clustering excluded) */
} kmp_contraction_stats;

/* clustering: host array of n cluster (leader) ids in [0, n) -- what kmp_lp_cluster returns -- or
 * NULL to contract by the labels the last kmp_lp_cluster / kmp_lp_upload_partition left on the device
 * for the current graph (KMP_ERR_INVALID when there are none since the last set_graph / free_scratch).
 * The caller owns *out (kmp_coarse_destroy). stats may be NULL. */
int kmp_contract_clustering(kmp_lp_handle *h, const uint32_t *clustering, kmp_coarse_graph **out,
                            kmp_contraction_stats *stats);

uint32_t kmp_coarse_n(const kmp_coarse_graph *g);
uint32_t kmp_coarse_m(const kmp_coarse_graph *g);
uint32_t kmp_coarse_fine_n(const kmp_coarse_graph *g);

/* Copy to host arrays (each nullable): xadj[c_n+1], adjncy[c_m], vwgt[c_n], adjwgt[c_m], mapping[fine n]. */
int kmp_coarse_download(const kmp_coarse_graph *g, uint32_t *xadj, uint32_t *adjncy, int32_t *vwgt, int32_t *adjwgt,
                        uint32_t *mapping);
/* Borrowed device pointers (valid until kmp_coarse_destroy), e.g. for kmp_lp_set_graph_device. */
int kmp_coarse_device_arrays(const kmp_coarse_graph *g, const uint32_t **d_xadj, const uint32_t **d_adjncy,
                             const int32_t **d_vwgt, const int32_t **d_adjwgt, const uint32_t **d_mapping);

/* CoarseGraph::project_up: fine[u] = coarse[mapping[u]] (host arrays: coarse[c_n] -> fine[n]). */
int kmp_coarse_project_up(const kmp_coarse_graph *g, const uint32_t *coarse, uint32_t *fine);
/* CoarseGraph::project_down: coarse[mapping[u]] = fine[u] (any member's value when they differ). */
int kmp_coarse_project_down(const kmp_coarse_graph *g, const uint32_t *fine, uint32_t *coarse);

/* Frees the arrays stream-ordered on the stream of the handle that contracted the graph: call it before
 * kmp_lp_destroy of that handle. */
void kmp_coarse_destroy(kmp_coarse_graph *g);

/* ---- threshold edge sparsification (SparsificationClusterCoarsener, DESIGN.md §13) --------------------------
 *
 *   SparsificationClusterCoarsener::sparsification_target / recontract_with_threshold_sparsification
 *       kaminpar-shm/coarsening/sparsification_cluster_coarsener.cc:41-48, 158-228
 *
 * The number of edges the coarse graph of a level is cut down to:
 *   target = min(edge_target_factor * prev_m, density_target_factor * prev_m / prev_n * c_n)   (in double)
 * truncated to an edge count if it is below prev_m, else prev_m. prev_m / prev_n belong to the previous level's
 * graph (the input graph on the first level). Host function: no device work. */
uint32_t kmp_sparsification_target(uint32_t prev_m, uint32_t prev_n, uint32_t c_n, double density_target_factor,
                                   double edge_target_factor);

typedef struct kmp_sparsify_stats {
  uint32_t c_m_before;      /* directed edges before */
  uint32_t c_m_after;       /* directed edges kept */
  uint32_t target_m;
  int32_t threshold;        /* T: the (c_m_before - target_m + 1)-th smallest edge weight (0 when target_m < 2) */
  uint32_t smaller;         /* edges with w < T */
  uint32_t equal;           /* edges with w == T */
  uint32_t equal_kept;      /* of those, kept by the hash (c_m_after = c_m_before - smaller - equal + equal_kept) */
  uint32_t kernel_launches;
  float device_ms;          /* whole call on the device, including the one wait for the selection's read-back
                               (the host computes p between the selection and the keep pass) */
} kmp_sparsify_stats;

/* Sparsifies g in place on the device, on the stream of h (the handle that contracted g). An edge (u, v, w) is
 * kept iff w > T, or w == T and dice(u, v) < p, with p = (target_m - #{w > T}) / #{w == T} in double and
 *   dice(u, v) = lo32(fmix64(((max(u, v) << 32) | min(u, v)) + seed)) / (2^32 - 1)
 * (murmur3's 64-bit finaliser). Both tests are symmetric in u and v, so the graph stays undirected; adjacency lists
 * stay sorted by target. target_m < 2 drops every edge (seed unused). Vertices, vertex weights and the mapping are
 * unchanged; xadj / adjncy / adjwgt are replaced, so device pointers taken earlier by kmp_coarse_device_arrays
 * are INVALID afterwards (the old arrays are freed). The caller applies the laziness rule and draws the seed, as
 * the reference's coarsen() does. Refused (KMP_ERR_INVALID): null arguments, target_m > kmp_coarse_m(g), and a
 * graph that lives on another device than h. stats may be NULL. */
int kmp_coarse_sparsify(kmp_lp_handle *h, kmp_coarse_graph *g, uint32_t target_m, uint64_t seed,
                        kmp_sparsify_stats *stats);

#ifdef __cplusplus
}
#endif
#endif
