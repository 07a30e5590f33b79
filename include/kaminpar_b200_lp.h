/* kaminpar_b200 -- C ABI of the CUDA label-propagation engine (H100, sm_90a).
 *
 * This is the drop-in boundary (SURVEY.md §8b). The reference has no FFI below its C++ plugin
 * interfaces; the entry points here are what a binding for those interfaces would call:
 *
 *   kmp_lp_cluster  <->  Clusterer::compute_clustering(StaticArray<NodeID>&, const Graph&, bool)
 *                        kaminpar-shm/coarsening/clusterer.h:35-46, implemented by LPClustering
 *                        (kaminpar-shm/coarsening/clustering/lp_clusterer.cc:376-399)
 *   kmp_lp_refine   <->  Refiner::initialize(const PartitionedGraph&) + Refiner::refine(
 *                        PartitionedGraph&, const PartitionContext&)
 *                        kaminpar-shm/refinement/refiner.h:34-56, implemented by
 *                        LabelPropagationRefiner (kaminpar-shm/refinement/lp/lp_refiner.cc:357-376)
 *   kmp_lp_config   <->  LabelPropagationCoarseningContext / LabelPropagationRefinementContext
 *                        include/kaminpar-shm/kaminpar.h:140-154, :221-228 (same field names)
 *   kmp_lp_set_graph<->  the CSRGraph the reference hands to both (xadj/adjncy/vwgt/adjwgt,
 *                        kaminpar-shm/datastructures/csr_graph.h:35-482); empty weight arrays mean
 *                        unit weights (csr_graph.cc:82-97) -> NULL here
 *
 * Type widths are the reference's default build (kaminpar.h:32-57): NodeID = EdgeID = BlockID =
 * uint32_t, NodeWeight = EdgeWeight = BlockWeight = int32_t. All arithmetic on the path is integer.
 *
 * Error convention: every call returns 0 on success or a negative kmp_status; kmp_last_error()
 * returns a description for the calling thread. There is no CPU fallback: without a CUDA device
 * every compute entry point fails with KMP_ERR_CUDA.
 */
#ifndef KAMINPAR_B200_LP_H
#define KAMINPAR_B200_LP_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KMP_LP_ABI_VERSION 3

typedef enum {
  KMP_OK = 0,
  KMP_ERR_INVALID = -1,     /* bad argument / call order */
  KMP_ERR_CUDA = -2,        /* CUDA runtime failure (incl. no device) */
  KMP_ERR_ALLOC = -3,       /* device or host allocation failed */
  KMP_ERR_UNSUPPORTED = -4, /* e.g. compressed graphs, 64-bit ids */
  KMP_ERR_NCCL = -5
} kmp_status;

/* enums mirror include/kaminpar-shm/kaminpar.h:100-126 */
enum { KMP_LP_SINGLE_PHASE = 0, KMP_LP_TWO_PHASE = 1, KMP_LP_GROWING_HASH_TABLES = 2 };
enum { KMP_TIE_GEOMETRIC = 0, KMP_TIE_UNIFORM = 1 };
enum { KMP_TWO_HOP_DISABLE = 0, KMP_TWO_HOP_MATCH = 1, KMP_TWO_HOP_MATCH_THREADWISE = 2,
       KMP_TWO_HOP_CLUSTER = 3, KMP_TWO_HOP_CLUSTER_THREADWISE = 4 };
enum { KMP_ISOLATED_KEEP = 0, KMP_ISOLATED_MATCH = 1, KMP_ISOLATED_CLUSTER = 2,
       KMP_ISOLATED_MATCH_DURING_TWO_HOP = 3, KMP_ISOLATED_CLUSTER_DURING_TWO_HOP = 4 };

typedef struct {
  /* fields of LabelPropagation{Coarsening,Refinement}Context, same names and defaults
   * (kaminpar-shm/presets.cc:140-153, :339-347) */
  uint32_t num_iterations;         /* 5; refiner: 0 = until no vertex moves */
  uint32_t large_degree_threshold; /* UINT32_MAX: vertices with degree >= this are never moved */
  uint32_t max_num_neighbors;      /* UINT32_MAX: scan at most this many neighbours per vertex */
  int32_t impl;                    /* accepted for API compatibility; every implementation choice of
                                      the reference has the same observable selection rule */
  int32_t tie_breaking_strategy;   /* KMP_TIE_UNIFORM. KMP_TIE_GEOMETRIC (sequential coin flips in rating-map
                                      insertion order, lp_clusterer.cc:252-278) has no order-free restatement:
                                      KMP_ERR_UNSUPPORTED under schedule KMP_SCHEDULE_SYNC, implemented by
                                      KMP_SCHEDULE_SEQ_STRICT */
  int32_t two_hop_strategy;        /* clusterer only. SYNC: DISABLE, MATCH_THREADWISE (default) and CLUSTER_THREADWISE
                                      (the one-thread outcome: pairs / next-fit packing of the singletons that favor the
                                      same cluster, in id order, label_propagation.h:977-1002); the global MATCH /
                                      CLUSTER variants (:1030-1191, an id-ordered chain of CAS hand-offs) are
                                      KMP_ERR_UNSUPPORTED under SYNC and implemented by SEQ_STRICT */
  double two_hop_threshold;        /* 0.5 */
  int32_t isolated_nodes_strategy; /* clusterer only; all five values (CLUSTER = next-fit packing in id order) */
  int32_t relabel_before_second_phase; /* must be 0 (the default, presets.cc:147); the cluster-id compaction of
                                      label_propagation.h:272-319 is not implemented: non-zero = KMP_ERR_UNSUPPORTED */
  /* engine */
  int32_t seed;                /* Random::reseed() analogue; enters every hash key */
  uint32_t sync_subrounds;     /* S: hashed sub-rounds per degree group and iteration (8; 0 = 8, at most 31) */
  uint32_t sync_granule_log2;  /* vertices u >> g share a sub-round (4) */
  uint32_t sync_commit_passes; /* commit passes crediting departures: 1 clusterer, 4 refiner. The clusterer's
                                  commit is single-pass: kmp_lp_cluster refuses > 1 with KMP_ERR_UNSUPPORTED */
  int32_t device;              /* CUDA device ordinal, -1 = current */
  int32_t schedule;            /* KMP_SCHEDULE_SYNC (default) or KMP_SCHEDULE_SEQ_STRICT */
} kmp_lp_config;

/* Visit schedules (SURVEY.md §8b). SYNC: deterministic synchronous sub-rounds, any size, any number of GPUs
 * (DESIGN.md §3). SEQ_STRICT: the reference's own one-thread visit order, rating-map insertion order and
 * libstdc++ mt19937 draws, executed by ONE thread block -- bit-identical to the unmodified reference at one
 * thread (label_propagation.h:1863-1937, kaminpar-common/random.h:64-147); meant for small inputs
 * (n <= KMP_SEQ_STRICT_MAX_N), e.g. BASELINE config 1. */
enum { KMP_SCHEDULE_SYNC = 0, KMP_SCHEDULE_SEQ_STRICT = 1 };
#define KMP_SEQ_STRICT_MAX_N (1u << 20)

typedef struct {
  uint32_t iterations;       /* LP rounds executed */
  uint32_t moved[64];        /* accepted moves per round */
  uint64_t edges_scanned;    /* sum of scanned adjacency entries of visited active vertices */
  uint64_t nodes_visited;
  uint64_t proposals;        /* vertices that wanted to move */
  uint32_t num_clusters;     /* clusterer: non-empty clusters after the rounds (before post passes) */
  uint32_t two_hop_ran;
  float device_ms;           /* CUDA-event time of the whole call on the handle's stream */
  float sweep_ms;            /* CUDA-event time spent in the sweep kernels only (if timing enabled) */
  uint64_t sweep_launches;   /* number of sweep-kernel launches */
  uint64_t kernel_launches;  /* all kernel launches of the call */
  /* per kernel tier (8 in use: 0: deg<=7 sweep_thread<8>, 1: deg<=16 sweep_thread<16>, 2: deg<=31 sweep_thread<32>,
   * 3: deg<256 sweep_team<32>, 4: deg<1024 sweep_team<128>, 5: deg<4096 sweep_team<512>, 6: deg<8192 / 16384
   * sweep_team<1024>, 7: above: sweep_hub_scatter+select+final; slots 8..11 are reserved) */
  uint64_t group_edges[12];
  uint64_t group_nodes[12];
  uint64_t group_launches[12];
  float group_sweep_ms[16];  /* only when timing is enabled: [0..11] sweep tiers, [12] commits,
                              * [13] reserved (0), [14] push activation, [15] stamp ageing */
  uint32_t pull_rounds;      /* LP rounds whose sweeps derived the active flags from the move stamps */
  uint32_t push_rounds;      /* LP rounds in which movers flagged their neighbours */
} kmp_lp_stats;

typedef struct kmp_lp_handle kmp_lp_handle;

int kmp_lp_abi_version(void);
const char *kmp_last_error(void);

/* Fill cfg with the default-preset values for the clusterer (mode 0) or refiner (mode 1). */
void kmp_lp_default_config(int mode, kmp_lp_config *cfg);

/* Environment knobs (experiments / tests only; results never depend on them). Read once per handle in
 * kmp_lp_create: KMP_HUB_WAVE_SLOTS = 8-byte bucket entries one wave of high-degree vertices may use (default 2^28 =
 * 2 GiB; smaller values process a sub-round's hubs in more waves), KMP_HUB_BUCKET_CAP / KMP_HUB_SEL_LIMIT = smaller
 * bucket capacity / claim limit of the hub tier (force its overflow list and multi-pass selection),
 * KMP_FORCE_P64=1 (8-byte gather words at any label count),
 * KMP_GRID_CAP = N caps the CTA count of every launch inside an LP round at N (small inputs then take every
 * grid-stride loop and work-queue refill several times).
 * Read per call: KMP_ACTIVATION=push|pull, KMP_TRACE=1 (set_graph stage times on stderr). */
int kmp_lp_create(const kmp_lp_config *cfg, kmp_lp_handle **out);
int kmp_lp_destroy(kmp_lp_handle *h);

/* Borrow a CSR graph from HOST memory: copies it to the device (pinned staging when the buffers
 * are pageable). vwgt / adjwgt may be NULL (unit weights). The handle keeps device copies until the
 * next set_graph / destroy. */
int kmp_lp_set_graph(kmp_lp_handle *h, uint32_t n, uint32_t m, const uint32_t *xadj,
                     const uint32_t *adjncy, const int32_t *vwgt, const int32_t *adjwgt);
/* Same, but the arrays already live in device memory of the handle's device and stay owned by the
 * caller (must outlive their use by the handle). Every pointer must be 4-byte aligned (KMP_ERR_INVALID
 * otherwise); views into a larger allocation are fine. When d_adjncy is also 16-byte aligned the
 * high-degree tier stages adjacency chunks into shared memory with bulk copies; otherwise it reads them
 * from global memory (same results, somewhat slower on hubs). */
int kmp_lp_set_graph_device(kmp_lp_handle *h, uint32_t n, uint32_t m, const uint32_t *d_xadj,
                            const uint32_t *d_adjncy, const int32_t *d_vwgt, const int32_t *d_adjwgt);

/* CSRGraph::sorted() of the graph just set (csr_graph.h: degree-bucket sorted, as KaMinPar::compute_partition
 * feeds the finest level, kaminpar.cc:369-396; coarse graphs are unsorted = one bucket, csr_graph.cc:242-245).
 * Only KMP_SCHEDULE_SEQ_STRICT reads it -- the reference's chunk order depends on the bucket array
 * (label_propagation.h:1736-1854); set_graph resets it to 0. */
int kmp_lp_set_graph_sorted(kmp_lp_handle *h, int sorted);

/* LPClustering::set_max_cluster_weight / set_desired_cluster_count / set_communities +
 * compute_clustering. clustering_out: HOST buffer of n NodeIDs (cluster = id of a vertex in
 * [0,n), not compacted) or NULL to leave the result on the device (kmp_lp_labels_device).
 * communities: HOST, nullable. Every call advances the handle's call counter (overlay coarsener:
 * same graph, different clustering, overlay_cluster_coarsener.cc:52-54). */
int kmp_lp_cluster(kmp_lp_handle *h, int32_t max_cluster_weight, uint32_t desired_num_clusters,
                   const uint32_t *communities, uint32_t *clustering_out, kmp_lp_stats *stats);

/* LabelPropagationRefiner::refine. partition_inout: HOST buffer of n BlockIDs, refined in place
 * (NULL: operate on the labels already on the device for the current graph, e.g. from
 * kmp_lp_upload_partition; refused with KMP_ERR_INVALID when there are none since the last
 * set_graph / kmp_lp_free_scratch). Labels >= k on either path are refused with KMP_ERR_INVALID
 * before any kernel indexes a [k] array by them (a clustering is not a k-way partition).
 * max_block_weights[k] (PartitionContext::max_block_weight, per block), min_block_weights[k]
 * nullable (PartitionContext::min_block_weight). block_weights_out[k] nullable. The sync hashes
 * use the number of kmp_lp_cluster calls the handle completed before (0 if it only refines). */
int kmp_lp_refine(kmp_lp_handle *h, uint32_t k, const int32_t *max_block_weights,
                  const int32_t *min_block_weights, const uint32_t *communities,
                  uint32_t *partition_inout, int32_t *block_weights_out, kmp_lp_stats *stats);

/* Device-resident variants used when the caller keeps state on the GPU between calls. */
int kmp_lp_upload_partition(kmp_lp_handle *h, const uint32_t *partition);
int kmp_lp_download_labels(kmp_lp_handle *h, uint32_t *labels_out);
const uint32_t *kmp_lp_labels_device(kmp_lp_handle *h);

/* T0 parity hook: evaluate the per-vertex selection rule for EVERY vertex against frozen labels
 * and weights (no moves). mode 0: clusterer (weights[n], scalar max), mode 1: refiner (weights[k],
 * max_weights[k]). Outputs HOST buffers: target[n]; favored[n] (mode 0; UINT32_MAX where the
 * vertex would not store a favored cluster). */
int kmp_lp_select_all(kmp_lp_handle *h, int mode, const uint32_t *labels, const int32_t *weights,
                      uint32_t num_labels, const int32_t *max_weights, int32_t max_cluster_weight,
                      const int32_t *min_weights, uint32_t call_index, uint32_t iteration,
                      uint32_t *target_out, uint32_t *favored_out);

/* free_memory_afterwards analogue (lp_clusterer.cc:330-333): release device scratch; the graph
 * stays. */
int kmp_lp_free_scratch(kmp_lp_handle *h);

/* Enable per-kernel CUDA-event timing of the sweep kernels (serialises nothing, adds events). */
int kmp_lp_set_timing(kmp_lp_handle *h, int enabled);

/* Metrics on the device (metrics.cc:36-53): edge cut of the labels currently on the device
 * (KMP_ERR_INVALID when they do not belong to the current graph). */
int kmp_lp_edge_cut(kmp_lp_handle *h, int64_t *cut_out);

/* ---- Stepping API: one LP sub-round at a time (sharded multi-GPU driver) ----------------------
 * One process per GPU; every rank holds a replica of the graph and of the label / weight state,
 * the vertex frontier (work lists) is sharded. Per sub-round: kmp_lp_step_sweep on the rank's share
 * -> all-gather of the packed proposal buffers (NCCL) -> kmp_lp_step_commit on every rank (the
 * commit rule is order-independent, so all replicas stay bit-identical). This is the role of the
 * reference's distributed twin (kaminpar-dist/refinement/lp/lp_refiner.cc:119-222: local
 * perform_iteration per chunk, then label exchange) with NCCL instead of MPI. */
int kmp_lp_set_shard(kmp_lp_handle *h, uint32_t rank, uint32_t world);

/* NCCL inside the library (what the C++ adapters / the reference's factories use with N GPUs): rank 0 obtains an
 * id with kmp_lp_dist_unique_id and hands its KMP_DIST_ID_BYTES bytes to the other ranks by any means (MPI, a
 * file, torch.distributed ...); every rank then calls kmp_lp_dist_init on its handle (= ncclCommInitRank + the
 * shard of kmp_lp_set_shard). From then on kmp_lp_cluster / kmp_lp_refine run the sharded schedule themselves:
 * per sub-round the rank sweeps its slice of the work lists, ncclAllGather moves the proposal buffers over
 * NVLink on the handle's stream, every rank commits. Results equal the single-GPU run bit for bit. libnccl.so.2 is
 * loaded on demand (KMP_ERR_NCCL if absent). The reference's counterpart is the label exchange of
 * kaminpar-dist/refinement/lp/lp_refiner.cc:119-222. */
#define KMP_DIST_ID_BYTES 128
int kmp_lp_dist_unique_id(void *id_out);
int kmp_lp_dist_init(kmp_lp_handle *h, const void *id, uint32_t rank, uint32_t world);
int kmp_lp_dist_shutdown(kmp_lp_handle *h);
/* Issue all work on the caller's stream (so that it is ordered with the caller's NCCL collectives).
 * 0 = the legacy default stream; (void*)-1 = back to the handle's own stream. */
int kmp_lp_set_stream(kmp_lp_handle *h, void *cuda_stream);
uint32_t kmp_lp_num_subrounds(kmp_lp_handle *h);
/* cap: proposals one rank can emit in sub-round sg (buffer = 4 + 2*cap words); size: vertices in it */
int kmp_lp_subround_cap(kmp_lp_handle *h, uint32_t sg, uint32_t *cap_out, uint32_t *size_out);
int kmp_lp_step_begin_cluster(kmp_lp_handle *h, int32_t max_cluster_weight, const uint32_t *communities);
int kmp_lp_step_begin_refine(kmp_lp_handle *h, uint32_t k, const int32_t *max_block_weights,
                             const int32_t *min_block_weights, const uint32_t *communities,
                             const uint32_t *partition);
int kmp_lp_step_begin_iteration(kmp_lp_handle *h);
/* iter counts the LP rounds of this call from 0 */
int kmp_lp_step_sweep(kmp_lp_handle *h, uint32_t iter, uint32_t sg, void *d_send);
int kmp_lp_step_commit(kmp_lp_handle *h, uint32_t iter, uint32_t sg, const void *d_gathered);
int kmp_lp_step_end_iteration(kmp_lp_handle *h, uint32_t *moved);
int kmp_lp_step_favored_export(kmp_lp_handle *h, void *d_buf);
int kmp_lp_step_favored_import(kmp_lp_handle *h, const void *d_buf);
int kmp_lp_step_finish(kmp_lp_handle *h, uint32_t *labels_out, int32_t *block_weights_out,
                       kmp_lp_stats *stats);

#ifdef __cplusplus
}
#endif
#endif
