/* CPU oracle for the label-propagation hot path -- C ABI.
 *
 * TEST INFRASTRUCTURE ONLY. Nothing under kaminpar_b200/ may include, link or load this; only
 * tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs do.
 *
 * Two schedules are provided:
 *   seq  : restatement of the reference's LP at ONE thread (the only configuration in which the
 *          reference itself is deterministic, tests/endtoend/shm_endtoend_test.cc:152), including
 *          its libstdc++ mt19937 / std::shuffle / uniform_int_distribution draws, chunk order,
 *          insertion-ordered rating maps and two-phase handling. Pinned bit-for-bit against the
 *          unmodified reference built in oracle/_ref (tests/golden/ref_*.npz).
 *   sync : the deterministic synchronous sub-round schedule the CUDA path implements (DESIGN.md
 *          "sync schedule"): identical per-vertex rating / feasibility / arg-max rules, ties
 *          broken by a counter-based hash instead of rating-map insertion order, moves committed
 *          per sub-round in a fixed priority order under the same weight constraints.
 */
#ifndef LP_ORACLE_H
#define LP_ORACLE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Mirrors LabelPropagationCoarseningContext / LabelPropagationRefinementContext
 * (include/kaminpar-shm/kaminpar.h:140-154, 221-228) + the knobs of the sync schedule. */
typedef struct {
  uint32_t num_iterations;         /* 5 (presets.cc:143, :342); refiner: 0 = until convergence */
  uint32_t large_degree_threshold; /* UINT32_MAX */
  uint32_t max_num_neighbors;      /* UINT32_MAX */
  int32_t impl;                    /* 0 SINGLE_PHASE, 1 TWO_PHASE, 2 GROWING_HASH_TABLES */
  int32_t tie_breaking;            /* 0 GEOMETRIC, 1 UNIFORM */
  int32_t two_hop_strategy;        /* 0 DISABLE 1 MATCH 2 MATCH_THREADWISE 3 CLUSTER 4 CLUSTER_THREADWISE */
  double two_hop_threshold;        /* 0.5 */
  int32_t isolated_nodes_strategy; /* 0 KEEP 1 MATCH 2 CLUSTER 3 MATCH_DURING_TWO_HOP 4 CLUSTER_DURING_TWO_HOP */
  /* sync schedule only */
  uint32_t sync_subrounds;    /* S >= 1 */
  uint32_t sync_granule_log2; /* vertices u>>g share a sub-round */
  uint32_t sync_commit_passes; /* commit passes crediting departures (>=1) */
} lpo_params;

typedef struct {
  uint32_t iterations;     /* rounds executed */
  uint32_t moved[64];      /* moved vertices per round */
  uint64_t edges_scanned;  /* sum of deg(u) over visited active vertices */
  uint64_t nodes_visited;
  uint32_t num_clusters;   /* non-empty clusters tracked by the LP (clusterer) */
  uint32_t two_hop_ran;
} lpo_stats;

int lpo_abi_version(void);

/* ---- graph utilities (callers of the path; restated for test inputs) --------------------- */
/* degree_bucket(d) = 0 if d==0 else floor(log2 d)+1 (kaminpar-common/degree_buckets.h:17-26);
 * stable sort by bucket with isolated nodes last, adjacency lists reversed
 * (graphutils/permutator.h:28-208), optional isolated-node removal (csr_graph.cc:150-174).
 * Outputs must be caller-allocated with the input sizes. Returns the LP-visible node count. */
uint32_t lpo_rearrange_by_degree_buckets(
    uint32_t n, uint32_t m, const uint32_t *xadj, const uint32_t *adjncy, const int32_t *vwgt,
    const int32_t *adjwgt, int remove_isolated, uint32_t *out_xadj, uint32_t *out_adjncy,
    int32_t *out_vwgt, int32_t *out_adjwgt, uint32_t *out_old_to_new, uint32_t *out_buckets /*34*/,
    uint32_t *out_num_buckets);

/* Bucket prefix array of a CSR as the reference's CSRGraph ctor computes it
 * (csr_graph.cc:199-248): sorted -> per-degree-bucket counts, else one bucket. */
void lpo_degree_buckets(uint32_t n, const uint32_t *xadj, int sorted, uint32_t *out_buckets /*34*/,
                        uint32_t *out_num_buckets);

int64_t lpo_edge_cut(uint32_t n, const uint32_t *xadj, const uint32_t *adjncy, const int32_t *adjwgt,
                     const uint32_t *partition);
void lpo_block_weights(uint32_t n, const int32_t *vwgt, uint32_t k, const uint32_t *partition,
                       int32_t *out /*k*/);
/* compute_max_cluster_weight, EPSILON_BLOCK_WEIGHT (coarsening/max_cluster_weights.h:17-46) with
 * PartitionContext::setup(graph,k,eps) (context.cc:27-39) and contraction_limit 2000. */
int32_t lpo_max_cluster_weight(uint32_t n, int64_t total_node_weight, uint32_t k, double epsilon);
/* (1+eps)*ceil(W/k), truncated (context.cc:33-36). */
int32_t lpo_max_block_weight(int64_t total_node_weight, uint32_t k, double epsilon);

/* ---- the path ---------------------------------------------------------------------------- */
/* schedule: 0 = seq, 1 = sync. buckets/num_buckets as produced above. Runs num_calls calls on the same
 * graph. first_call (sync only; seq returns -1 unless it is 0): the call index of the first of them,
 * i.e. how many kmp_lp_cluster calls the device handle ran before, on any graph -- it enters the
 * hash keys of the sync schedule. seq: the caller replays earlier calls itself with num_calls. */
int lpo_lp_cluster(int schedule, uint32_t n, uint32_t m, const uint32_t *xadj, const uint32_t *adjncy,
                   const int32_t *vwgt, const int32_t *adjwgt, const uint32_t *buckets,
                   uint32_t num_buckets, int seed, int32_t max_cluster_weight,
                   uint32_t desired_num_clusters, const uint32_t *communities /*nullable*/,
                   const lpo_params *params, int num_calls, uint32_t *out_clustering /* n*num_calls */,
                   lpo_stats *stats /* num_calls, nullable */, uint32_t first_call);

/* call_index (sync only; seq returns -1 unless it is 0): the number of kmp_lp_cluster calls the device
 * handle ran before this refinement (0 for a handle that only refines). */
int lpo_lp_refine(int schedule, uint32_t n, uint32_t m, const uint32_t *xadj, const uint32_t *adjncy,
                  const int32_t *vwgt, const int32_t *adjwgt, const uint32_t *buckets,
                  uint32_t num_buckets, int seed, uint32_t k, const int32_t *max_block_weights,
                  const int32_t *min_block_weights /*nullable*/, const uint32_t *communities /*nullable*/,
                  const lpo_params *params, uint32_t *partition_inout, int32_t *block_weights_out /*k*/,
                  lpo_stats *stats /*nullable*/, uint32_t call_index);

/* ---- T0: per-vertex decision on frozen state (sync rules), for unit parity tests ---------- */
/* For every vertex u (regardless of active flags) compute the target the sync selection rule picks
 * against the given frozen labels / weights: out_target[u] (== label[u] if it stays) and, for the
 * clusterer (mode 0), out_favored[u]. mode 1 = refiner (weights = block weights, max = per block).
 * params (nullable): max_num_neighbors caps the scanned prefix of every adjacency, and a vertex of degree
 * >= large_degree_threshold is not visited (out_target[u] = label[u], out_favored[u] = UINT32_MAX). */
int lpo_sync_select_all(int mode, uint32_t n, const uint32_t *xadj, const uint32_t *adjncy,
                        const int32_t *vwgt, const int32_t *adjwgt, const uint32_t *labels,
                        const int32_t *weights, uint32_t num_labels, const int32_t *max_weights,
                        int32_t max_cluster_weight, const int32_t *min_weights, int seed,
                        uint32_t call_index, uint32_t iteration, uint32_t *out_target,
                        uint32_t *out_favored, const lpo_params *params /*nullable*/);

/* ---- bridge: the reference-pinned `seq` selection code (ClusterPolicy / RefinePolicy::select_best_cluster,
 * the code checked bit-for-bit against the unmodified reference) on the same frozen state. Outputs the
 * reference's choice, the size of the tie set it draws from (UNIFORM) and whether check_target[u] /
 * check_favored[u] lie in that set; see tests/test_bridge_sync_to_reference.py. */
int lpo_seq_select_all(int mode, uint32_t n, const uint32_t *xadj, const uint32_t *adjncy, const int32_t *vwgt,
                       const int32_t *adjwgt, const uint32_t *labels, const int32_t *weights, uint32_t num_labels,
                       const int32_t *max_weights, int32_t max_cluster_weight, const int32_t *min_weights,
                       const uint32_t *check_target /*nullable*/, const uint32_t *check_favored /*nullable*/,
                       uint32_t *out_target, uint32_t *out_favored /*nullable*/, uint32_t *out_num_ties,
                       uint32_t *out_num_fav_ties /*nullable*/, uint8_t *out_check_in_ties /*nullable*/,
                       uint8_t *out_check_fav_in_ties /*nullable*/);

#ifdef __cplusplus
}
#endif
#endif
