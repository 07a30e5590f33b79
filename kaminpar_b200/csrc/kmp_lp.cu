// kaminpar_b200: host side of the CUDA label-propagation engine (H100, sm_90a) + its C ABI
// (include/kaminpar_b200_lp.h). One handle = one CUDA stream on one device; everything between
// the H2D copy of the inputs and the D2H copy of the result runs on the device.
//
// Drivers restated (control flow only; the per-vertex work is in lp_sweep.cuh / lp_commit.cuh):
//   LPClusteringImpl::compute_clustering   kaminpar-shm/coarsening/clustering/lp_clusterer.cc:89-109
//   LPRefinerImpl::refine                  kaminpar-shm/refinement/lp/lp_refiner.cc:68-89
//   ChunkRandomLabelPropagation::perform_iteration  kaminpar-shm/label_propagation.h:1681-1733
// The visit schedule is the "sync" schedule of DESIGN.md instead of the reference's asynchronous
// chunk-random order (which is only deterministic at one thread).
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include <cstdlib>
#include <dlfcn.h>
#include <nccl.h> // types only: the library is dlopen()ed in kmp_lp_dist_init (no link-time dependency)
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "../../include/kaminpar_b200_contraction.h"
#include "../../include/kaminpar_b200_lp.h"
#include "lp_commit.cuh"
#include "lp_device.cuh"
#include "lp_lowgroup.cuh"
#include "lp_strict.cuh"
#include "lp_sweep.cuh"

using namespace kmp;

namespace {

thread_local std::string g_last_error;

int fail(int code, const std::string &msg) {
  g_last_error = msg;
  return code;
}

#define KMP_CUDA(expr)                                                                                     \
  do {                                                                                                     \
    cudaError_t _e = (expr);                                                                               \
    if (_e != cudaSuccess) {                                                                               \
      return fail(_e == cudaErrorMemoryAllocation ? KMP_ERR_ALLOC : KMP_ERR_CUDA,                          \
                  std::string(#expr) + ": " + cudaGetErrorString(_e));                                     \
    }                                                                                                      \
  } while (0)

constexpr int kNumGroups = 4; // degree groups of the schedule
constexpr int kNumTiers = 8;  // kernel tiers: group 1 is split in two, group 3 (deg >= 256) in four
// sync_subrounds: the work-list keys (tier * S + sub-round, plus one key for unvisited vertices) are 8 bits wide
constexpr uint32_t kMaxSubrounds = (255 - 1) / kNumTiers;
constexpr int kHubTier = 7;   // deg >= kHubMinDegree: label-partitioned hub kernels (lp_sweep.cuh)
constexpr int kStatTiers = 12; // tier slots of kmp_lp_stats / ctr64 (edges at [tier], nodes at [kCtrNodes + tier])
constexpr int kCtrNodes = 16, kCtrScratch = 40, kCtrSize = 48;
constexpr uint32_t kHubMinDegree = 8192;       // graphs with edge weights (32-bit ratings in the team tables)
constexpr uint32_t kHubMinDegreeUnit = 16384;  // unit edge weights: 16-bit ratings, twice the slots
constexpr int kSMs = 132; // H100 SXM: caps the grid-stride launches at a few waves of the device
constexpr uint32_t kMaxHubWaves = 448; // work-queue cursors ctr32[64 .. 512), overflow counters ctr32[512 .. 960)
constexpr uint32_t kCtr32Size = 1024;
constexpr int kTagCommit = 12, kTagPush = 14, kTagMisc = 15; // timing slots besides the tiers; 13 is reserved

// kernel tier of a vertex of degree d >= 1
__host__ __device__ inline uint32_t tier_of(uint32_t d, uint32_t hub_min) {
  return d < 8 ? 0u : d <= 16 ? 1u : d < 32 ? 2u : d < 256 ? 3u : d < 1024 ? 4u : d < 4096 ? 5u : d < hub_min ? 6u : 7u;
}
// degree groups of the schedule {<8} {<32} {<256} {>=256} and their kernel tiers
inline int group_of_tier(int tier) { return tier == 0 ? 0 : tier <= 2 ? 1 : tier == 3 ? 2 : 3; }
inline int first_tier_of_group(int g) { return g == 0 ? 0 : g == 1 ? 1 : g == 2 ? 3 : 4; }
inline int last_tier_of_group(int g) { return g == 0 ? 0 : g == 1 ? 2 : g == 2 ? 3 : kNumTiers - 1; }

template <typename T> struct DevBuf {
  T *p = nullptr;
  size_t cap = 0; // elements
  DevBuf() = default;
  DevBuf(const DevBuf &) = delete;
  DevBuf &operator=(const DevBuf &) = delete;
  ~DevBuf() { release(); }
  cudaError_t ensure(size_t n) {
    if (n <= cap) {
      return cudaSuccess;
    }
    release();
    cudaError_t e = cudaMalloc(reinterpret_cast<void **>(&p), std::max<size_t>(n, 1) * sizeof(T));
    if (e == cudaSuccess) {
      cap = std::max<size_t>(n, 1);
    } else {
      p = nullptr;
    }
    return e;
  }
  void release() {
    if (p != nullptr) {
      cudaFree(p);
    }
    p = nullptr;
    cap = 0;
  }
};

} // namespace

cudaMemPool_t kmp_private_pool(int device); // kmp_contract.cuh

struct kmp_lp_handle {
  kmp_lp_config cfg{};
  int device = 0;
  cudaStream_t stream = nullptr;       // stream all work is issued on
  cudaStream_t owned_stream = nullptr; // the stream this handle created (destroyed with it)
  // The kernel tiers of one sub-round of degree group 3 are independent of each other: they are launched on
  // side streams (fork / join by events) so that their tails and latency-bound phases overlap.
  cudaStream_t sweep_stream = nullptr; // stream the running sweep launch goes to
  cudaStream_t side_stream[3] = {nullptr, nullptr, nullptr};
  cudaEvent_t ev_fork = nullptr, ev_join[3] = {nullptr, nullptr, nullptr};
  cudaEvent_t ev_begin = nullptr, ev_end = nullptr;
  cudaEvent_t ev_ct0 = nullptr, ev_ct1 = nullptr; // contraction timing (kmp_contract.cuh), created on first use
  bool timing = false;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> sweep_events;
  std::vector<int> sweep_event_group;
  uint64_t group_launches[kStatTiers] = {};
  uint32_t grid_cap = 0;        // KMP_GRID_CAP: most CTAs of any launch inside an LP round (0: no cap)
  // packed (label, stamp) gather array of the sweeps (lp_device.cuh): 4 B per vertex while labels fit 24 bits
  // (n <= 2^24 clusterer / k <= 2^24 refiner), else 8 B
  DevBuf<unsigned char> labg;
  bool p64 = false;
  bool force_p64 = false;
  bool stamps_ok = false;        // 4 * S sub-rounds fit the stamp code (else push activation only)
  bool pull_this = true, pull_next = true; // activation mode of the running / the next LP round
  uint32_t moved_hist[2] = {0xFFFFFFFFu, 0xFFFFFFFFu}; // accepted moves of the two previous rounds
  uint32_t visited_total = 0;    // vertices on the work lists
  DevBuf<uint32_t> queue;        // work-queue cursors of the team kernels: [tier][sub-round], zeroed per round
  DevBuf<uint32_t> t4_hit;       // hub tier: per list entry "a neighbour moved since the last visit"
  DevBuf<uint32_t> t4_tmp_deg, t4_tmp_beg, t4_tmp_ids; // list building scratch
  size_t sweep_events_used = 0;

  // graph
  uint32_t n = 0, m = 0;
  const uint32_t *xadj = nullptr;
  const uint32_t *adjncy = nullptr;
  const int32_t *vwgt = nullptr;
  const int32_t *adjwgt = nullptr;
  bool adjncy_16b = true; // adjncy starts on a 16-byte boundary: the hub tier may stage it with bulk copies
  DevBuf<uint32_t> own_xadj, own_adjncy;
  DevBuf<int32_t> own_vwgt, own_adjwgt;
  bool have_graph = false;
  uint32_t max_degree = 0;
  uint32_t num_isolated = 0;

  // work lists: order[] holds the vertices of (group g, sub-round s) contiguously
  DevBuf<uint32_t> order;
  std::vector<uint32_t> list_off; // kNumGroups*S + 1 (+1 tail bucket for unvisited vertices)
  uint32_t max_list = 0;
  uint32_t lists_S = 0, lists_G = 0, lists_thr = 0;
  int lists_seed = 0;
  bool lists_valid = false;

  // state
  DevBuf<uint32_t> label, favored, communities;
  // label[] belongs to the current graph: set by a completed clustering, kmp_lp_upload_partition and a refine or
  // balancer call given a partition; cleared by a new graph and by kmp_lp_free_scratch. The calls that read the
  // labels on the device (a NULL partition or clustering) refuse while it is clear.
  bool labels_valid = false;
  DevBuf<int32_t> weight, maxw, minw;
  DevBuf<uint8_t> active;
  // scratch
  DevBuf<uint32_t> mv_u, mv_t, cslot, slotmap;
  DevBuf<uint8_t> acc;
  DevBuf<int32_t> incoming, chist, hist, jmin, out_cur, out_delta, ohist, ojmin;
  DevBuf<uint32_t> ctr32; // [0] mover_count [1] moved_count (per iteration) [2] misc
  DevBuf<unsigned long long> ctr64; // [0] edges [1] nodes [2] proposals
  // hub tier ("t4" in these names is historical): per list entry its first bucket (wave-relative), the
  // (entry, chunk) work items of the scatter pass and the (entry, bucket) items of the select pass; all per sub-round
  DevBuf<uint32_t> t4_table_off, t4_item_entry, t4_item_chunk, t4_sel_entry, t4_sel_piece, t4_sel_begin;
  DevBuf<uint32_t> t4_item_u, t4_item_beg, t4_item_deg; // static per item: vertex, xadj[u], degree
  std::vector<uint32_t> t4_item_off, t4_sel_off; // S + 1
  // A sub-round's hubs are processed in waves whose bucket regions together stay below hub_wave_slots entries
  // (a memory bound: every wave reuses the same regions, cursors and overflow list).
  struct HubWave {
    uint32_t item_lo, item_hi, sel_lo, sel_hi; // absolute ranges in the t4_item_* / t4_sel_* arrays
  };
  std::vector<HubWave> t4_waves;
  std::vector<uint32_t> t4_wave_off; // S + 1
  uint64_t hub_wave_slots = 1ull << 28; // 2 GiB of packed entries (KMP_HUB_WAVE_SLOTS overrides, for experiments)
  DevBuf<Cand> t4_part_best, t4_part_fav;
  uint64_t t4_max_slots = 0;
  uint64_t t4_max_wave_edges = 0; // largest adjacency volume of a wave = capacity of the overflow list
  uint32_t hub_bucket_cap = kBucketCap, hub_sel_limit = 0; // KMP_HUB_BUCKET_CAP / KMP_HUB_SEL_LIMIT (tests: force the overflow paths)
  DevBuf<unsigned long long> hub_tab; // bucket regions: kBucketCap packed (key << 32 | rating) entries each
  DevBuf<uint32_t> hub_cursor;        // per bucket: entries appended in the running sub-round
  DevBuf<HubOverflow> hub_ovf;
  // clusterer hub path (gather + rate): per list entry the start of its row in hub_lab (sub-round-relative) and its
  // first rate item result; the (entry, hash class) rate items of each sub-round, largest degree first
  DevBuf<uint32_t> t4_lab_off, t4_rate_begin, t4_rate_entry, t4_rate_cls;
  std::vector<uint32_t> t4_rate_off; // S + 1
  uint64_t t4_max_subround_edges = 0;
  DevBuf<uint32_t> hub_lab; // staged neighbour labels of the running sub-round's hubs (4 B per edge)
  uint32_t mover_cap = 0;
  uint32_t cur_subround = 0; // hashed class of the running sub-round
  uint32_t cur_sg = 0;       // running sub-round index in [0, 4 * S): queue cursor and stamp code
  DevBuf<uint8_t> sort_keys_in, sort_keys_out;
  DevBuf<uint32_t> sort_vals_in;
  DevBuf<unsigned char> cub_tmp;
  DevBuf<unsigned long long> pairs_a, pairs_b; // two-hop sort; contraction: edge keys (double buffer)
  // contraction scratch (kmp_contract.cuh), grow-only like the rest
  DevBuf<int32_t> ct_vals_a, ct_vals_b;
  DevBuf<uint32_t> ct_flags, ct_rank, ct_cl;
  DevBuf<unsigned long long> ct_counter;
  DevBuf<uint32_t> sp_ctl; // sparsification (kmp_sparsify.cuh): radix-select bins, select state, kept counter
  bool slot_state_clean = false; // incoming/slotmap/chist zeroed for current n

  // schedule KMP_SCHEDULE_SEQ_STRICT (lp_strict.cuh): sequential engine state
  bool graph_sorted = false; // CSRGraph::sorted() of the current graph (kmp_lp_set_graph_sorted)
  bool strict_seeded = false;
  DevBuf<int32_t> st_slot, st_ent_val, st_slot2, st_ent2_val, st_concurrent;
  DevBuf<uint32_t> st_ent_key, st_ent2_key, st_used, st_second, st_tie_best, st_tie_fav, st_chunks, st_sub_perm,
      st_match, st_buckets;
  DevBuf<kmp_strict::Rng> st_rng;
  DevBuf<kmp_strict::Stats> st_stats;

  uint32_t call_counter = 0;
  uint64_t kernel_launches = 0, sweep_launches = 0;
  uint32_t pull_rounds = 0, push_rounds = 0;
  // frontier sharding (one process per GPU): this rank sweeps slice `rank` of `world` of every list
  uint32_t rank = 0, world = 1;
  // NCCL communicator of the sharded run (kmp_lp_dist_init): proposals are all-gathered per sub-round on
  // the handle's stream, inside kmp_lp_cluster / kmp_lp_refine
  ncclComm_t comm = nullptr;
  DevBuf<uint32_t> dist_send, dist_recv;
  uint32_t *direct_send = nullptr; // set while the sweeps of a sharded sub-round write into the send buffer
  uint32_t direct_cap = 0;
  // cooperative single-launch commit of a sub-round (lp_commit.cuh commit_cluster_fused / commit_refine_fused)
  DevBuf<unsigned> grid_bar; // [0] arrivals, [1] generation
  int fused_blocks = 0;      // co-resident CTAs of the clusterer's kernel
  int fused_blocks_refine = 0; // of the refiner's kernel with its largest dynamic shared memory
  // co-resident CTAs of the persistent kernels of degree groups 0 and 1 (lp_lowgroup.cuh), [group][EW][P64]
  uint32_t low_blocks[2][2][2] = {};
  // resident CTAs of each sweep_team instantiation on the device, [MODE][EW][P64][team size 32 / 128 / 512 / 1024]:
  // a larger grid only adds CTAs that start after the work queue is drained
  uint32_t team_grid[2][2][2][4] = {};
  // stepping API state
  int step_mode = -1;
  uint32_t step_iter = 0; // LP round of the stepping API
  uint32_t step_labels = 0;
  int32_t step_mcw = 0;
  bool step_has_min = false, step_has_comm = false;
  uint32_t mover_parity = 0; // proposal counter in use: ctr32[0] (parity 0) or ctr32[3] (parity 1)
  bool stepping = false; // proposals are accumulated by kmp_lp_step_commit, not by the sweep kernels
  // overload balancer (kmp_balance.cuh): its own call counter, so that LP calls hash the same with or without it
  uint32_t bal_calls = 0;
  DevBuf<uint32_t> bal_cand, bal_under, bal_ctr32, bal_target, bal_lists, bal_sv_a, bal_sv_b, bal_blk;
  DevBuf<int32_t> bal_over, bal_pbw, bal_wt, bal_prefix;
  DevBuf<uint8_t> bal_flag;
  DevBuf<float> bal_key;
  DevBuf<unsigned long long> bal_ctrl, bal_sk_a, bal_sk_b;
  // underload balancer (kmp_underload.cuh): its own call counter; shares the overload balancer's scratch
  uint32_t ubal_calls = 0;
  DevBuf<int32_t> ubal_deficit;
  DevBuf<uint8_t> ubal_tmask;
};

namespace kmp {
// block weights from labels; counts labels >= k (a clustering is not a partition) into *bad. The one range check
// of the refiner and both balancers (checked_block_weights).
__global__ void bal_block_weights(uint32_t n, uint32_t k, const int32_t *vwgt, const uint32_t *label, int32_t *weight,
                                  unsigned long long *bad) {
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += gridDim.x * blockDim.x) {
    const uint32_t b = label[u];
    if (b < k) {
      atomicAdd(&weight[b], vwgt != nullptr ? vwgt[u] : 1);
    } else {
      atomicAdd(bad, 1ull);
    }
  }
}
} // namespace kmp

namespace {

// ---- small kernels --------------------------------------------------------------------------
// vertices per degree group of the schedule (hist[0..3]) among the visited ones
__global__ void k_group_counts(uint32_t n, const uint32_t *xadj, uint32_t large_degree_threshold, uint32_t *hist) {
  uint32_t c[4] = {0, 0, 0, 0};
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += gridDim.x * blockDim.x) {
    const uint32_t d = xadj[u + 1] - xadj[u];
    if (d != 0 && d < large_degree_threshold) {
      ++c[degree_group(d)];
    }
  }
  for (int q = 0; q < 4; ++q) {
    uint32_t v = c[q];
    for (int o = 16; o > 0; o >>= 1) {
      v += __shfl_xor_sync(kFull, v, o);
    }
    if ((threadIdx.x & 31) == 0 && v != 0) {
      atomicAdd(&hist[q], v);
    }
  }
}

struct GroupSubrounds {
  uint32_t s[4]; // hashed sub-rounds used by each degree group (<= S)
};

__global__ void k_list_keys(uint32_t n, const uint32_t *xadj, uint32_t S, GroupSubrounds gs, uint32_t granule_log2,
                            uint32_t base_sr, uint32_t large_degree_threshold, uint32_t hub_min, uint8_t *keys,
                            uint32_t *vals, uint32_t *hist, uint32_t *max_deg) {
  // list-size histogram privatised per CTA: n global atomics on < 64 addresses serialise in L2
  // (the cost grows with n: the 512^3 grid has 1.3e8 vertices)
  __shared__ uint32_t s_hist[256];
  s_hist[threadIdx.x & 255] = 0;
  __syncthreads();
  uint32_t local_max = 0;
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += gridDim.x * blockDim.x) {
    const uint32_t d = xadj[u + 1] - xadj[u];
    uint32_t key;
    if (d == 0 || !(d < large_degree_threshold)) {
      key = kNumTiers * S; // never visited (label_propagation.h:1795, :1914-1915)
    } else {
      key = tier_of(d, hub_min) * S + subround_of(u, granule_log2, base_sr, gs.s[degree_group(d)]);
    }
    keys[u] = static_cast<uint8_t>(key);
    vals[u] = u;
    atomicAdd(&s_hist[key], 1u);
    local_max = d > local_max ? d : local_max;
  }
  __syncthreads();
  if (s_hist[threadIdx.x & 255] != 0 && threadIdx.x < 256) {
    atomicAdd(&hist[threadIdx.x], s_hist[threadIdx.x]);
  }
  for (int o = 16; o > 0; o >>= 1) {
    const uint32_t other = __shfl_xor_sync(kFull, local_max, o);
    local_max = other > local_max ? other : local_max;
  }
  if ((threadIdx.x & 31) == 0) {
    atomicMax(max_deg, local_max);
  }
}

__global__ void k_gather_degrees(uint32_t cnt, const uint32_t *list, const uint32_t *xadj, uint32_t *deg, uint32_t *beg,
                                 uint32_t *ids) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < cnt; i += gridDim.x * blockDim.x) {
    const uint32_t u = list[i];
    deg[i] = xadj[u + 1] - xadj[u];
    beg[i] = xadj[u];
    ids[i] = u;
  }
}

template <bool P64>
__global__ void k_init_cluster(uint32_t n, const int32_t *vwgt, uint32_t *label, void *labg, int32_t *weight,
                               uint32_t *favored, uint8_t *active) {
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += gridDim.x * blockDim.x) {
    label[u] = u; // reset_state, label_propagation.h:1194-1220 with initial_cluster(u) = u
    static_cast<typename LabG<P64>::word *>(labg)[u] = LabG<P64>::pack(u, 0);
    favored[u] = u;
    weight[u] = vwgt != nullptr ? vwgt[u] : 1;
    active[u] = 1;
  }
}
// packed gather words from plain labels, stamp 0 (refiner start, T0 hook)
template <bool P64> __global__ void k_pack_labels(uint32_t n, const uint32_t *label, void *labg) {
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += gridDim.x * blockDim.x) {
    static_cast<typename LabG<P64>::word *>(labg)[u] = LabG<P64>::pack(label[u], 0);
  }
}
// start of round r >= 2: forget the moves of round r - 2 (their stamps carry the parity of round r)
template <bool P64> __global__ void k_age_stamps(uint32_t n, void *labg, uint32_t parity) {
  typename LabG<P64>::word *g = static_cast<typename LabG<P64>::word *>(labg);
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += gridDim.x * blockDim.x) {
    const typename LabG<P64>::word w = g[u];
    const uint32_t st = LabG<P64>::stamp(w);
    if (st != 0 && ((st - 1u) >> kStampBits) == parity) {
      g[u] = LabG<P64>::pack(LabG<P64>::label(w), 0);
    }
  }
}
__global__ void k_fill_u8(uint32_t n, uint8_t *p, uint8_t v) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    p[i] = v;
  }
}
__global__ void k_count_nonzero(uint32_t n, const int32_t *w, uint32_t *out) {
  uint32_t c = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    c += w[i] != 0;
  }
  for (int o = 16; o > 0; o >>= 1) {
    c += __shfl_xor_sync(kFull, c, o);
  }
  if ((threadIdx.x & 31) == 0 && c != 0) {
    atomicAdd(out, c);
  }
}
__global__ void k_edge_cut(uint32_t n, const uint32_t *xadj, const uint32_t *adjncy, const int32_t *adjwgt,
                           const uint32_t *label, unsigned long long *out) {
  unsigned long long c = 0;
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t u = warp; u < n; u += nwarps) {
    const uint32_t lu = label[u];
    for (uint32_t e = xadj[u] + lane; e < xadj[u + 1]; e += 32) {
      if (label[adjncy[e]] != lu) {
        c += adjwgt != nullptr ? adjwgt[e] : 1;
      }
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    c += __shfl_xor_sync(kFull, c, o);
  }
  if (lane == 0 && c != 0) {
    atomicAdd(out, c);
  }
}

// warp-aggregated append: one atomic per warp instead of one per element (a single cursor serialises in L2)
__device__ __forceinline__ uint32_t warp_append_slot(uint32_t *count, bool pred) {
  const unsigned ballot = __ballot_sync(kFull, pred);
  if (ballot == 0) {
    return 0;
  }
  const int lane = threadIdx.x & 31;
  uint32_t base = 0;
  if (lane == __ffs(ballot) - 1) {
    base = atomicAdd(count, static_cast<uint32_t>(__popc(ballot)));
  }
  base = __shfl_sync(kFull, base, __ffs(ballot) - 1);
  return base + __popc(ballot & ((1u << lane) - 1u));
}

// ---- post passes of the clusterer (sync definitions, DESIGN.md) ---------------------------------
// isolated nodes: the i-th and (i+1)-th isolated vertex (i even, id order) are matched if they fit
// isolated vertices as (0, u) pairs: one group of the pair-based post passes below
__global__ void k_collect_isolated(uint32_t n, const uint32_t *xadj, unsigned long long *pairs, uint32_t *count) {
  const uint32_t bound = (n + 31u) & ~31u; // whole warps reach the ballot
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < bound; u += gridDim.x * blockDim.x) {
    const bool iso = u < n && xadj[u + 1] == xadj[u];
    const uint32_t slot = warp_append_slot(count, iso);
    if (iso) {
      pairs[slot] = u;
    }
  }
}
__global__ void k_match_isolated(uint32_t cnt, const unsigned long long *sorted_iso, uint32_t *label, int32_t *weight,
                                 int32_t max_w) {
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; 2 * p + 1 < cnt; p += gridDim.x * blockDim.x) {
    const uint32_t a = static_cast<uint32_t>(sorted_iso[2 * p]), b = static_cast<uint32_t>(sorted_iso[2 * p + 1]);
    const uint32_t ca = label[a], cb = label[b];
    if (ca != cb && weight[ca] + weight[cb] <= max_w) {
      weight[ca] += weight[cb];
      weight[cb] = 0;
      label[b] = ca;
    }
  }
}
// two-hop: eligible singletons keyed by (favored, u)
__global__ void k_collect_two_hop(uint32_t n, const uint32_t *xadj, const int32_t *vwgt, const uint32_t *label,
                                  const int32_t *weight, const uint32_t *favored, int32_t max_w,
                                  unsigned long long *pairs, uint32_t *count) {
  const uint32_t bound = (n + 31u) & ~31u;
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < bound; u += gridDim.x * blockDim.x) {
    bool eligible = u < n && xadj[u + 1] != xadj[u] && label[u] == u;
    if (eligible) {
      const int32_t w = weight[u];
      const int32_t nw = vwgt != nullptr ? vwgt[u] : 1;
      eligible = !(w > max_w / 2 || w != nw);
    }
    const uint32_t slot = warp_append_slot(count, eligible);
    if (eligible) {
      pairs[slot] = (static_cast<unsigned long long>(favored[u]) << 32) | u;
    }
  }
}
// head[p] = index of the first element of p's group (equal favored); computed as an inclusive max-scan
// over (is_head ? p : 0)
__global__ void k_two_hop_heads(uint32_t cnt, const unsigned long long *sorted, uint32_t *head) {
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < cnt; p += gridDim.x * blockDim.x) {
    const bool is_head = p == 0 || static_cast<uint32_t>(sorted[p - 1] >> 32) != static_cast<uint32_t>(sorted[p] >> 32);
    head[p] = is_head ? p : 0u;
  }
}
// CLUSTER post passes (next fit in id order = the reference at one thread: label_propagation.h:884-917 for isolated
// vertices, :977-1002 with match = false for two-hop): within a group of equal key (sorted by vertex id) a vertex
// joins the waiting representative while it has room, else becomes the representative. One warp per group;
// 32 members per step, with a prefix sum of their weights and a restart at every vertex that does not fit.
__global__ void __launch_bounds__(256) k_next_fit(uint32_t cnt, const unsigned long long *sorted, uint32_t *label,
                                                   int32_t *weight, int32_t max_w) {
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t p = warp; p < cnt; p += nwarps) {
    const uint32_t key = static_cast<uint32_t>(sorted[p] >> 32);
    if (p != 0 && static_cast<uint32_t>(sorted[p - 1] >> 32) == key) {
      continue; // not a group head (warp-uniform)
    }
    uint32_t rep = static_cast<uint32_t>(sorted[p]);
    int32_t repw = weight[rep];
    for (uint32_t i = p + 1; i < cnt; i += 32) {
      const uint32_t idx = i + lane;
      const bool valid = idx < cnt && static_cast<uint32_t>(sorted[idx] >> 32) == key;
      const int nvalid = __popc(__ballot_sync(kFull, valid)); // members are contiguous: a prefix of the lanes
      if (nvalid == 0) {
        break;
      }
      const uint32_t u = valid ? static_cast<uint32_t>(sorted[idx]) : 0u;
      const int32_t w = valid ? weight[u] : 0;
      int start = 0;
      while (start < nvalid) {
        int32_t pre = (lane >= start && lane < nvalid) ? w : 0; // inclusive prefix over lanes >= start
        for (int o = 1; o < 32; o <<= 1) {
          const int32_t t = __shfl_up_sync(kFull, pre, o);
          if (lane >= o) {
            pre += t;
          }
        }
        const bool over = lane >= start && lane < nvalid && (repw + pre > max_w);
        const unsigned nf = __ballot_sync(kFull, over);
        const int f = nf != 0 ? __ffs(nf) - 1 : nvalid; // first member that does not fit
        if (lane >= start && lane < f) {
          label[u] = rep;
          weight[u] = 0;
        }
        if (f > start) {
          repw += __shfl_sync(kFull, pre, f - 1);
        }
        if (f < nvalid) { // lane f starts a new cluster
          if (lane == 0) {
            weight[rep] = repw;
          }
          rep = __shfl_sync(kFull, u, f);
          repw = __shfl_sync(kFull, w, f);
          start = f + 1;
        } else {
          start = nvalid;
        }
      }
      if (nvalid < 32) {
        break;
      }
    }
    if (lane == 0) {
      weight[rep] = repw;
    }
  }
}

struct MaxOp {
  __host__ __device__ __forceinline__ uint32_t operator()(uint32_t a, uint32_t b) const { return a > b ? a : b; }
};
// the (2i+1)-th member of a group joins the (2i)-th (label_propagation.h:977-1002 at one thread)
__global__ void k_match_two_hop(uint32_t cnt, const unsigned long long *sorted, const uint32_t *head, uint32_t *label,
                                int32_t *weight) {
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < cnt; p += gridDim.x * blockDim.x) {
    const uint32_t rank = p - head[p];
    if (rank & 1u) {
      const uint32_t rep = static_cast<uint32_t>(sorted[p - 1]);
      const uint32_t u = static_cast<uint32_t>(sorted[p]);
      weight[rep] += weight[u];
      weight[u] = 0;
      label[u] = rep;
    }
  }
}

// ---- exchange helpers of the sharded (multi-GPU) path -------------------------------------------
// pack this rank's proposals: buf = [count, pad, pad, pad, u[cap], t[cap]]
__global__ void k_pack_movers(const uint32_t *mv_u, const uint32_t *mv_t, const uint32_t *count, uint32_t cap,
                              uint32_t *buf) {
  const uint32_t cnt = *count;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    buf[0] = cnt;
  }
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < cnt; i += gridDim.x * blockDim.x) {
    buf[4 + i] = mv_u[i];
    buf[4 + cap + i] = mv_t[i];
  }
}
// favored fix-up across ranks: only the owner of u ever writes favored[u] (initially u)
__global__ void k_xor_iota(uint32_t n, const uint32_t *in, uint32_t *out) {
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += gridDim.x * blockDim.x) {
    out[u] = in[u] ^ u;
  }
}

// ---- launch helpers -----------------------------------------------------------------------------
inline uint32_t grid_for(uint64_t threads_needed, uint32_t block, uint32_t max_blocks = kSMs * 16) {
  const uint64_t b = (threads_needed + block - 1) / block;
  return static_cast<uint32_t>(std::max<uint64_t>(1, std::min<uint64_t>(b, max_blocks)));
}
// CTA count of a launch inside an LP round under KMP_GRID_CAP (tests): with a tiny grid, small inputs take every
// grid-stride loop, work-queue refill and persistent-kernel iteration many times. A capped cooperative grid stays
// co-resident.
inline uint32_t capped(const kmp_lp_handle *h, uint32_t blocks) {
  return h->grid_cap != 0 && blocks > h->grid_cap ? h->grid_cap : blocks;
}

constexpr int team_size_index(int T) { return T == 32 ? 0 : T == 128 ? 1 : T == 512 ? 2 : 3; }
template <int SLOTS, int TEAMS, bool V16> constexpr size_t team_smem() {
  return static_cast<size_t>(SLOTS) * TEAMS * (V16 ? 6 : 8);
}

template <int MODE, bool EW, bool P64, int T, int SLOTS, int TEAMS, bool V16 = false>
void launch_team(kmp_lp_handle *h, const SweepArgs &a) {
  const uint32_t want = (a.list_size + TEAMS - 1) / TEAMS;
  const uint32_t blocks = capped(h, std::max<uint32_t>(1, std::min<uint32_t>(want, h->team_grid[MODE][EW][P64][team_size_index(T)])));
  sweep_team<MODE, EW, P64, T, SLOTS, TEAMS, V16><<<blocks, T * TEAMS, team_smem<SLOTS, TEAMS, V16>(), h->sweep_stream>>>(a);
}

// dynamic shared memory opt-in of one team kernel and its resident grid (CTAs per SM from the occupancy calculator)
template <int MODE, bool EW, bool P64, int T, int SLOTS, int TEAMS, bool V16 = false>
bool configure_team(kmp_lp_handle *h, int sms) {
  const auto kernel = sweep_team<MODE, EW, P64, T, SLOTS, TEAMS, V16>;
  constexpr size_t smem = team_smem<SLOTS, TEAMS, V16>();
  int per_sm = 0;
  if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)) != cudaSuccess ||
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, T * TEAMS, smem) != cudaSuccess || per_sm < 1) {
    return false;
  }
  h->team_grid[MODE][EW][P64][team_size_index(T)] = static_cast<uint32_t>(sms * per_sm);
  return true;
}

// per device; called from kmp_lp_create
template <int MODE, bool EW, bool P64> bool configure_team_kernels(kmp_lp_handle *h, int sms) {
  if constexpr (MODE == 0) {
    if (cudaFuncSetAttribute(sweep_hub_rate<EW>, cudaFuncAttributeMaxDynamicSharedMemorySize, rate_smem<EW>()) != cudaSuccess) {
      return false;
    }
  } else {
    cudaFuncSetAttribute(sweep_hub_scatter<MODE, EW, P64>, cudaFuncAttributeMaxDynamicSharedMemorySize, kHubScatterSmem);
  }
  bool ok = configure_team<MODE, EW, P64, 32, 512, 8, !EW>(h, sms) && configure_team<MODE, EW, P64, 128, 2048, 4>(h, sms) &&
            configure_team<MODE, EW, P64, 512, 8192, 1>(h, sms);
  if constexpr (EW) {
    ok = ok && configure_team<MODE, EW, P64, 1024, 16384, 1>(h, sms);
  } else {
    ok = ok && configure_team<MODE, EW, P64, 1024, 32768, 1, true>(h, sms);
  }
  return ok;
}

template <int MODE, bool EW, bool P64> cudaError_t launch_sweep_t(kmp_lp_handle *h, int tier, const SweepArgs &a) {
  if (a.list_size == 0) {
    return cudaSuccess;
  }
  const uint32_t tgrid = capped(h, grid_for(a.list_size, 256));
  switch (tier) {
  case 0: // deg <= 7: thread per vertex, labels sorted in registers
    sweep_thread<MODE, EW, P64, 8><<<tgrid, 256, 0, h->sweep_stream>>>(a);
    break;
  case 1: // deg 8..16
    sweep_thread<MODE, EW, P64, 16><<<tgrid, 256, 0, h->sweep_stream>>>(a);
    break;
  case 2: // deg 17..31
    sweep_thread<MODE, EW, P64, 32><<<tgrid, 256, 0, h->sweep_stream>>>(a);
    break;
  case 3: // deg 32..255: one warp per vertex, 512 slots (a 64-register sort was slower here: 230 registers, one CTA per SM);
          // 16-bit ratings with unit edge weights (a rating is at most the degree), which leaves room for the claim lists
    launch_team<MODE, EW, P64, 32, 512, 8, !EW>(h, a);
    break;
  case 4: // deg < 1024: 128 threads per vertex, 2048 slots
    launch_team<MODE, EW, P64, 128, 2048, 4>(h, a);
    break;
  case 5: // deg < 4096: 512 threads per vertex, 8192 slots
    launch_team<MODE, EW, P64, 512, 8192, 1>(h, a);
    break;
  case 6: // 1024 threads per vertex; deg < 8192: 16384 slots, or (unit edge weights) deg < 16384: 32768 slots
    if constexpr (EW) {
      launch_team<MODE, EW, P64, 1024, 16384, 1>(h, a);
    } else {
      launch_team<MODE, EW, P64, 1024, 32768, 1, true>(h, a);
    }
    break;
  default: {
    HubArgs hb{};
    const uint32_t s_idx = h->cur_subround;
    const uint32_t S = h->lists_S;
    const uint32_t first = h->list_off[kHubTier * S + s_idx] - h->list_off[kHubTier * S];
    hb.sel_limit = h->hub_sel_limit;
    hb.rank = h->rank;
    hb.world = h->world;
    hb.hit = h->t4_hit.p + first;
    if constexpr (MODE == 0) {
      // gather the labels of the sub-round's hub edges once, then rate every (hub, hash class) item in one CTA
      const uint32_t ilo = h->t4_item_off[s_idx], ihi = h->t4_item_off[s_idx + 1];
      hb.item_entry = h->t4_item_entry.p + ilo;
      hb.item_chunk = h->t4_item_chunk.p + ilo;
      hb.item_u = h->t4_item_u.p + ilo;
      hb.item_beg = h->t4_item_beg.p + ilo;
      hb.item_deg = h->t4_item_deg.p + ilo;
      hb.num_items = ihi - ilo;
      hb.lab = h->hub_lab.p;
      hb.lab_off = h->t4_lab_off.p + first;
      sweep_hub_gather<P64><<<capped(h, std::min<uint32_t>(hb.num_items, kSMs * 8)), 256, 0, h->sweep_stream>>>(a, hb);
      const uint32_t rlo = h->t4_rate_off[s_idx], rhi = h->t4_rate_off[s_idx + 1];
      hb.item_entry = h->t4_rate_entry.p + rlo;
      hb.item_cls = h->t4_rate_cls.p + rlo;
      hb.num_items = rhi - rlo;
      hb.sel_begin = h->t4_rate_begin.p + first;
      hb.part_best = h->t4_part_best.p;
      hb.part_fav = h->t4_part_fav.p;
      hb.queue = h->ctr32.p + 64 + s_idx; // zeroed with the other per-round counters
      sweep_hub_rate<EW><<<capped(h, std::min<uint32_t>(hb.num_items, kSMs)), kRateThreads, rate_smem<EW>(), h->sweep_stream>>>(a, hb);
      h->kernel_launches += 2;
    } else {
      hb.table_off = h->t4_table_off.p + first;
      hb.g_tab = h->hub_tab.p;
      hb.cursor = h->hub_cursor.p;
      hb.ovf = h->hub_ovf.p;
      hb.ovf_cap = static_cast<uint32_t>(std::min<uint64_t>(h->t4_max_wave_edges, 0xFFFFFFFFull));
      hb.bucket_cap = h->hub_bucket_cap;
      hb.stage_adjncy = h->adjncy_16b ? 1u : 0u;
      hb.sel_begin = h->t4_sel_begin.p + first;
      // one scatter + select pair per wave; all waves share the bucket memory (cursors reset by the select)
      for (uint32_t w = h->t4_wave_off[s_idx]; w < h->t4_wave_off[s_idx + 1]; ++w) {
        const kmp_lp_handle::HubWave &wv = h->t4_waves[w];
        hb.item_entry = h->t4_item_entry.p + wv.item_lo;
        hb.item_chunk = h->t4_item_chunk.p + wv.item_lo;
        hb.item_u = h->t4_item_u.p + wv.item_lo;
        hb.item_beg = h->t4_item_beg.p + wv.item_lo;
        hb.item_deg = h->t4_item_deg.p + wv.item_lo;
        hb.num_items = wv.item_hi - wv.item_lo;
        hb.queue = h->ctr32.p + 64 + w; // zeroed with the other per-round counters
        hb.ovf_count = h->ctr32.p + 512 + w;
        sweep_hub_scatter<MODE, EW, P64><<<capped(h, std::min<uint32_t>(hb.num_items, kSMs * 4)), kHubThreads, kHubScatterSmem, h->sweep_stream>>>(a, hb, h->m);
        hb.sel_entry = h->t4_sel_entry.p + wv.sel_lo;
        hb.sel_piece = h->t4_sel_piece.p + wv.sel_lo;
        hb.num_sel_items = wv.sel_hi - wv.sel_lo;
        hb.part_best = h->t4_part_best.p + (wv.sel_lo - h->t4_sel_off[s_idx]);
        hb.part_fav = h->t4_part_fav.p + (wv.sel_lo - h->t4_sel_off[s_idx]);
        sweep_hub_select<MODE><<<capped(h, std::min<uint32_t>((hb.num_sel_items + kSelWarps - 1) / kSelWarps, kSMs * 6)), kSelWarps * 32, 0, h->sweep_stream>>>(a, hb);
        h->kernel_launches += 2;
      }
    }
    hb.part_best = h->t4_part_best.p;
    hb.part_fav = h->t4_part_fav.p;
    sweep_hub_final<MODE><<<capped(h, grid_for(static_cast<uint64_t>(a.list_size) * 32, 256)), 256, 0, h->sweep_stream>>>(a, hb);
    break;
  }
  }
  return cudaGetLastError();
}

// timing mode: bracket a section of the stream with an event pair tagged with a stats slot
// (0..7 sweep tiers, kTagCommit commits, kTagPush push activation, kTagMisc stamp ageing)
int timed_begin(kmp_lp_handle *h, int tag, cudaStream_t st = nullptr) {
  if (!h->timing) {
    return -1;
  }
  if (st == nullptr) {
    st = h->stream;
  }
  if (h->sweep_events_used == h->sweep_events.size()) {
    cudaEvent_t x, y;
    cudaEventCreate(&x);
    cudaEventCreate(&y);
    h->sweep_events.emplace_back(x, y);
    h->sweep_event_group.push_back(0);
  }
  const int idx = static_cast<int>(h->sweep_events_used++);
  h->sweep_event_group[idx] = tag;
  cudaEventRecord(h->sweep_events[idx].first, st);
  return idx;
}
void timed_end(kmp_lp_handle *h, int idx, cudaStream_t st = nullptr) {
  if (idx >= 0) {
    cudaEventRecord(h->sweep_events[idx].second, st == nullptr ? h->stream : st);
  }
}

// tier: kernel tier 0..kNumTiers-1 of the list in `a_in`
cudaError_t launch_sweep(kmp_lp_handle *h, int mode, int tier, const SweepArgs &a_in) {
  if (a_in.list_size == 0) {
    return cudaSuccess;
  }
  SweepArgs a = a_in;
  a.counters = h->ctr64.p + tier;
  a.queue = h->queue.p + static_cast<size_t>(tier) * kNumGroups * h->lists_S + h->cur_sg;
  if (h->sweep_stream == nullptr) {
    h->sweep_stream = h->stream;
  }
  const int ev = timed_begin(h, tier, h->sweep_stream);
  const bool ew = h->adjwgt != nullptr;
  const int variant = (mode << 2) | (ew ? 2 : 0) | (h->p64 ? 1 : 0);
  cudaError_t e;
  switch (variant) {
  case 0: e = launch_sweep_t<0, false, false>(h, tier, a); break;
  case 1: e = launch_sweep_t<0, false, true>(h, tier, a); break;
  case 2: e = launch_sweep_t<0, true, false>(h, tier, a); break;
  case 3: e = launch_sweep_t<0, true, true>(h, tier, a); break;
  case 4: e = launch_sweep_t<1, false, false>(h, tier, a); break;
  case 5: e = launch_sweep_t<1, false, true>(h, tier, a); break;
  case 6: e = launch_sweep_t<1, true, false>(h, tier, a); break;
  default: e = launch_sweep_t<1, true, true>(h, tier, a); break;
  }
  timed_end(h, ev, h->sweep_stream);
  ++h->kernel_launches;
  ++h->sweep_launches;
  ++h->group_launches[tier];
  return e;
}

struct TraceClock { // KMP_TRACE=1: wall-clock stages of set_graph on stderr (diagnostics only)
  bool on = std::getenv("KMP_TRACE") != nullptr;
  std::chrono::steady_clock::time_point t = std::chrono::steady_clock::now();
  void lap(const char *what) {
    if (on) {
      const auto now = std::chrono::steady_clock::now();
      std::fprintf(stderr, "[kmp trace] %-28s %8.3f ms\n", what, std::chrono::duration<double, std::milli>(now - t).count());
      t = now;
    }
  }
};

int ensure_lists(kmp_lp_handle *h) {
  TraceClock tc;
  const uint32_t S = std::max<uint32_t>(1, h->cfg.sync_subrounds);
  if (h->lists_valid && h->lists_S == S && h->lists_G == h->cfg.sync_granule_log2 &&
      h->lists_thr == h->cfg.large_degree_threshold && h->lists_seed == h->cfg.seed) {
    return KMP_OK;
  }
  if (S > kMaxSubrounds) {
    return fail(KMP_ERR_INVALID, "sync_subrounds too large (max " + std::to_string(kMaxSubrounds) + ")");
  }
  h->stamps_ok = kNumGroups * S <= kMaxStampSubrounds; // else: push activation only
  const uint32_t n = h->n;
  const uint32_t nkeys = kNumTiers * S + 1;
  KMP_CUDA(h->sort_keys_in.ensure(n));
  KMP_CUDA(h->sort_keys_out.ensure(n));
  KMP_CUDA(h->sort_vals_in.ensure(n));
  KMP_CUDA(h->order.ensure(n));
  KMP_CUDA(h->ctr32.ensure(kCtr32Size));
  KMP_CUDA(cudaMemsetAsync(h->ctr32.p, 0, kCtr32Size * sizeof(uint32_t), h->stream));
  tc.lap("lists: buffers");
  const uint32_t base_sr = sync_base(h->cfg.seed, 0, 0, SALT_SUBROUND);
  // Sub-rounds per degree group: S for a group holding >= 1/16 of the visited vertices, S/4 otherwise
  // (a small group has few same-sub-round neighbours; its launches become 4x larger). DESIGN.md §3.
  GroupSubrounds gs{};
  {
    k_group_counts<<<grid_for(n, 256), 256, 0, h->stream>>>(n, h->xadj, h->cfg.large_degree_threshold, h->ctr32.p);
    uint32_t cnt[4] = {0, 0, 0, 0};
    KMP_CUDA(cudaMemcpyAsync(cnt, h->ctr32.p, sizeof(cnt), cudaMemcpyDeviceToHost, h->stream));
    KMP_CUDA(cudaStreamSynchronize(h->stream));
    const uint64_t visited = static_cast<uint64_t>(cnt[0]) + cnt[1] + cnt[2] + cnt[3];
    h->visited_total = static_cast<uint32_t>(visited);
    for (int q = 0; q < 4; ++q) {
      gs.s[q] = (16ull * cnt[q] >= visited) ? S : std::max<uint32_t>(1, S / 4);
    }
    KMP_CUDA(cudaMemsetAsync(h->ctr32.p, 0, kCtr32Size * sizeof(uint32_t), h->stream));
  }
  tc.lap("lists: group counts (sync)");
  k_list_keys<<<grid_for(n, 256), 256, 0, h->stream>>>(n, h->xadj, S, gs, h->cfg.sync_granule_log2, base_sr,
                                                        h->cfg.large_degree_threshold,
                                                        h->adjwgt != nullptr ? kHubMinDegree : kHubMinDegreeUnit,
                                                        h->sort_keys_in.p, h->sort_vals_in.p, h->ctr32.p, h->ctr32.p + 300);
  KMP_CUDA(cudaGetLastError());
  size_t tmp_bytes = 0;
  KMP_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, h->sort_keys_in.p, h->sort_keys_out.p,
                                           h->sort_vals_in.p, h->order.p, static_cast<int>(n), 0, 8, h->stream));
  KMP_CUDA(h->cub_tmp.ensure(tmp_bytes));
  if (n > 0) {
    KMP_CUDA(cub::DeviceRadixSort::SortPairs(h->cub_tmp.p, tmp_bytes, h->sort_keys_in.p, h->sort_keys_out.p,
                                             h->sort_vals_in.p, h->order.p, static_cast<int>(n), 0, 8, h->stream));
  }
  std::vector<uint32_t> hist(512);
  KMP_CUDA(cudaMemcpyAsync(hist.data(), h->ctr32.p, 512 * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
  KMP_CUDA(cudaStreamSynchronize(h->stream));
  tc.lap("lists: keys + sort (sync)");
  h->list_off.assign(nkeys + 1, 0);
  for (uint32_t kx = 0; kx < nkeys; ++kx) {
    h->list_off[kx + 1] = h->list_off[kx] + hist[kx];
  }
  auto lsize = [&](uint32_t tier, uint32_t sr) { return hist[tier * S + sr]; };
  h->max_list = 0;
  h->mover_cap = 1;
  for (uint32_t sr = 0; sr < S; ++sr) {
    for (int g = 0; g < kNumGroups; ++g) { // the tiers of a degree group share a sub-round
      uint32_t tot = 0;
      for (int t = first_tier_of_group(g); t <= last_tier_of_group(g); ++t) {
        tot += lsize(static_cast<uint32_t>(t), sr);
      }
      h->mover_cap = std::max(h->mover_cap, tot);
    }
  }
  KMP_CUDA(h->queue.ensure(static_cast<size_t>(kNumTiers) * kNumGroups * S));
  h->max_list = h->mover_cap;
  h->max_degree = hist[300];
  // ---- hub tier metadata: bucket regions, chunk work items and (entry, bucket) selection items per sub-round --
  {
    const uint32_t t4_begin = h->list_off[kHubTier * S], t4_end = h->list_off[(kHubTier + 1) * S];
    const uint32_t t4_cnt = t4_end - t4_begin;
    h->t4_item_off.assign(S + 1, 0);
    h->t4_wave_off.assign(S + 1, 0);
    h->t4_waves.clear();
    h->t4_max_slots = 0;
    h->t4_max_wave_edges = 0;
    h->t4_max_subround_edges = 0;
    if (t4_cnt > 0) {
      DevBuf<uint32_t> &d_deg = h->t4_tmp_deg, &d_beg = h->t4_tmp_beg, &d_ids = h->t4_tmp_ids; // grow-only
      KMP_CUDA(d_deg.ensure(t4_cnt));
      KMP_CUDA(d_beg.ensure(t4_cnt));
      KMP_CUDA(d_ids.ensure(t4_cnt));
      k_gather_degrees<<<grid_for(t4_cnt, 256), 256, 0, h->stream>>>(t4_cnt, h->order.p + t4_begin, h->xadj, d_deg.p,
                                                                      d_beg.p, d_ids.p);
      std::vector<uint32_t> vbeg(t4_cnt), vids(t4_cnt), iu, ibeg, ideg;
      KMP_CUDA(cudaMemcpyAsync(vbeg.data(), d_beg.p, t4_cnt * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
      KMP_CUDA(cudaMemcpyAsync(vids.data(), d_ids.p, t4_cnt * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
      std::vector<uint32_t> deg(t4_cnt), toff(t4_cnt), sbeg(t4_cnt), ient, ichk, sent, spiece;
      h->t4_sel_off.assign(S + 1, 0);
      size_t max_sel = 0;
      KMP_CUDA(cudaMemcpyAsync(deg.data(), d_deg.p, t4_cnt * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
      KMP_CUDA(cudaStreamSynchronize(h->stream));
      // at most kMaxHubWaves work-queue cursors exist per LP round: coarsen the waves if necessary
      // (the degrees must be on the host before this sum -- ADVICE r1)
      uint64_t wave_slots = h->hub_wave_slots;
      {
        uint64_t total = 0;
        for (uint32_t i = 0; i < t4_cnt; ++i) {
          total += static_cast<uint64_t>(hub_buckets(deg[i])) * kBucketCap;
        }
        wave_slots = std::max<uint64_t>(wave_slots, total / (kMaxHubWaves / 2 - S) + 1);
      }
      for (uint32_t sr = 0; sr < S; ++sr) {
        const uint32_t lo = h->list_off[kHubTier * S + sr] - t4_begin, hi = h->list_off[kHubTier * S + sr + 1] - t4_begin;
        uint64_t slots = 0, wave_edges = 0;
        kmp_lp_handle::HubWave wave{static_cast<uint32_t>(ient.size()), 0, static_cast<uint32_t>(sent.size()), 0};
        auto close_wave = [&]() {
          wave.item_hi = static_cast<uint32_t>(ient.size());
          wave.sel_hi = static_cast<uint32_t>(sent.size());
          if (wave.item_hi > wave.item_lo) {
            h->t4_waves.push_back(wave);
          }
          wave.item_lo = wave.item_hi;
          wave.sel_lo = wave.sel_hi;
          h->t4_max_slots = std::max(h->t4_max_slots, slots);
          h->t4_max_wave_edges = std::max(h->t4_max_wave_edges, wave_edges);
          slots = 0;
          wave_edges = 0;
        };
        for (uint32_t i = lo; i < hi; ++i) {
          const uint32_t buckets = hub_buckets(deg[i]);
          const uint64_t cap = static_cast<uint64_t>(buckets) * kBucketCap;
          if (slots > 0 && slots + cap > wave_slots) {
            close_wave();
          }
          if ((slots + cap) / kBucketCap > 0xFFFFFFFFull) {
            return fail(KMP_ERR_UNSUPPORTED, "high-degree buckets of one wave exceed 2^32");
          }
          toff[i] = static_cast<uint32_t>(slots / kBucketCap); // first bucket of the entry, wave-relative
          slots += cap;
          wave_edges += deg[i];
          const uint32_t chunks = (deg[i] + kChunkEdges - 1) / kChunkEdges;
          for (uint32_t c = 0; c < chunks; ++c) {
            ient.push_back(i - lo);
            ichk.push_back(c);
            iu.push_back(vids[i]);
            ibeg.push_back(vbeg[i]);
            ideg.push_back(deg[i]);
          }
          sbeg[i] = static_cast<uint32_t>(sent.size() - h->t4_sel_off[sr]);
          for (uint32_t c = 0; c < buckets; ++c) { // one selection item per bucket
            sent.push_back(i - lo);
            spiece.push_back(c);
          }
        }
        close_wave();
        h->t4_wave_off[sr + 1] = static_cast<uint32_t>(h->t4_waves.size());
        h->t4_sel_off[sr + 1] = static_cast<uint32_t>(sent.size());
        max_sel = std::max<size_t>(max_sel, sent.size() - h->t4_sel_off[sr]);
        h->t4_item_off[sr + 1] = static_cast<uint32_t>(ient.size());
      }
      if (h->t4_waves.size() > kMaxHubWaves) {
        return fail(KMP_ERR_UNSUPPORTED, "too many high-degree table waves (raise KMP_HUB_WAVE_SLOTS)");
      }
      // clusterer: per entry its row in the staged labels and its first result slot, and the (entry, hash class)
      // rate items of every sub-round, largest degree first (the longest items start first)
      std::vector<uint32_t> loff(t4_cnt), rbeg(t4_cnt), rent, rcls, ord;
      h->t4_rate_off.assign(S + 1, 0);
      size_t max_rate = 0;
      for (uint32_t sr = 0; sr < S; ++sr) {
        const uint32_t lo = h->list_off[kHubTier * S + sr] - t4_begin, hi = h->list_off[kHubTier * S + sr + 1] - t4_begin;
        uint64_t edges = 0; // <= m < 2^32
        uint32_t res = 0;
        ord.clear();
        for (uint32_t i = lo; i < hi; ++i) {
          loff[i] = static_cast<uint32_t>(edges);
          edges += deg[i];
          rbeg[i] = res;
          res += hub_classes(deg[i]);
          ord.push_back(i);
        }
        std::stable_sort(ord.begin(), ord.end(), [&](uint32_t x, uint32_t y) { return deg[x] > deg[y]; });
        for (const uint32_t i : ord) {
          for (uint32_t c = 0; c < hub_classes(deg[i]); ++c) {
            rent.push_back(i - lo);
            rcls.push_back(c);
          }
        }
        h->t4_rate_off[sr + 1] = static_cast<uint32_t>(rent.size());
        max_rate = std::max<size_t>(max_rate, res);
        h->t4_max_subround_edges = std::max(h->t4_max_subround_edges, edges);
      }
      max_sel = std::max(max_sel, max_rate);
      KMP_CUDA(h->t4_lab_off.ensure(t4_cnt));
      KMP_CUDA(h->t4_rate_begin.ensure(t4_cnt));
      KMP_CUDA(h->t4_rate_entry.ensure(rent.size()));
      KMP_CUDA(h->t4_rate_cls.ensure(rcls.size()));
      KMP_CUDA(cudaMemcpyAsync(h->t4_lab_off.p, loff.data(), t4_cnt * 4, cudaMemcpyHostToDevice, h->stream));
      KMP_CUDA(cudaMemcpyAsync(h->t4_rate_begin.p, rbeg.data(), t4_cnt * 4, cudaMemcpyHostToDevice, h->stream));
      KMP_CUDA(cudaMemcpyAsync(h->t4_rate_entry.p, rent.data(), rent.size() * 4, cudaMemcpyHostToDevice, h->stream));
      KMP_CUDA(cudaMemcpyAsync(h->t4_rate_cls.p, rcls.data(), rcls.size() * 4, cudaMemcpyHostToDevice, h->stream));
      KMP_CUDA(h->t4_table_off.ensure(t4_cnt));
      KMP_CUDA(h->t4_hit.ensure(t4_cnt));
      KMP_CUDA(cudaMemsetAsync(h->t4_hit.p, 0, static_cast<size_t>(t4_cnt) * 4, h->stream));
      KMP_CUDA(h->t4_item_entry.ensure(ient.size()));
      KMP_CUDA(h->t4_item_chunk.ensure(ichk.size()));
      KMP_CUDA(cudaMemcpyAsync(h->t4_table_off.p, toff.data(), t4_cnt * 4, cudaMemcpyHostToDevice, h->stream));
      KMP_CUDA(cudaMemcpyAsync(h->t4_item_entry.p, ient.data(), ient.size() * 4, cudaMemcpyHostToDevice, h->stream));
      KMP_CUDA(cudaMemcpyAsync(h->t4_item_chunk.p, ichk.data(), ichk.size() * 4, cudaMemcpyHostToDevice, h->stream));
      KMP_CUDA(h->t4_item_u.ensure(iu.size()));
      KMP_CUDA(h->t4_item_beg.ensure(iu.size()));
      KMP_CUDA(h->t4_item_deg.ensure(iu.size()));
      KMP_CUDA(cudaMemcpyAsync(h->t4_item_u.p, iu.data(), iu.size() * 4, cudaMemcpyHostToDevice, h->stream));
      KMP_CUDA(cudaMemcpyAsync(h->t4_item_beg.p, ibeg.data(), iu.size() * 4, cudaMemcpyHostToDevice, h->stream));
      KMP_CUDA(cudaMemcpyAsync(h->t4_item_deg.p, ideg.data(), iu.size() * 4, cudaMemcpyHostToDevice, h->stream));
      KMP_CUDA(h->t4_sel_entry.ensure(sent.size()));
      KMP_CUDA(h->t4_sel_piece.ensure(spiece.size()));
      KMP_CUDA(h->t4_sel_begin.ensure(t4_cnt));
      KMP_CUDA(h->t4_part_best.ensure(max_sel));
      KMP_CUDA(h->t4_part_fav.ensure(max_sel));
      KMP_CUDA(cudaMemcpyAsync(h->t4_sel_entry.p, sent.data(), sent.size() * 4, cudaMemcpyHostToDevice, h->stream));
      KMP_CUDA(cudaMemcpyAsync(h->t4_sel_piece.p, spiece.data(), spiece.size() * 4, cudaMemcpyHostToDevice, h->stream));
      KMP_CUDA(cudaMemcpyAsync(h->t4_sel_begin.p, sbeg.data(), t4_cnt * 4, cudaMemcpyHostToDevice, h->stream));
      KMP_CUDA(cudaStreamSynchronize(h->stream));
    }
  }
  tc.lap("lists: hub metadata");
  h->lists_S = S;
  h->lists_G = h->cfg.sync_granule_log2;
  h->lists_thr = h->cfg.large_degree_threshold;
  h->lists_seed = h->cfg.seed;
  h->lists_valid = true;
  // the sort buffers are only needed here
  // The sort buffers stay allocated (grow-only, released by kmp_lp_free_scratch): a cudaFree / cudaMalloc pair per
  // set_graph synchronises the whole device, and waits for the graph upload in flight (scripts/e2e_probe.py).
  tc.lap("lists: done");
  return KMP_OK;
}

// scratch shared by both modes
int ensure_scratch(kmp_lp_handle *h, int mode, uint32_t num_labels) {
  const size_t cap = std::max<uint32_t>(h->mover_cap, 1);
  KMP_CUDA(h->mv_u.ensure(cap));
  KMP_CUDA(h->mv_t.ensure(cap));
  KMP_CUDA(h->acc.ensure(cap));
  KMP_CUDA(h->ctr32.ensure(kCtr32Size));
  KMP_CUDA(h->ctr64.ensure(kCtrSize));
  KMP_CUDA(h->active.ensure(h->n));
  if (mode == 0) {
    KMP_CUDA(h->cslot.ensure(cap));
    const bool fresh = h->incoming.cap < h->n || h->slotmap.cap < h->n || h->chist.cap < cap * kLadderLevels;
    KMP_CUDA(h->incoming.ensure(h->n));
    KMP_CUDA(h->slotmap.ensure(h->n));
    KMP_CUDA(h->chist.ensure(cap * kLadderLevels));
    if (fresh || !h->slot_state_clean) {
      KMP_CUDA(cudaMemsetAsync(h->incoming.p, 0, h->incoming.cap * sizeof(int32_t), h->stream));
      KMP_CUDA(cudaMemsetAsync(h->slotmap.p, 0xFF, h->slotmap.cap * sizeof(uint32_t), h->stream));
      KMP_CUDA(cudaMemsetAsync(h->chist.p, 0, h->chist.cap * sizeof(int32_t), h->stream));
      h->slot_state_clean = true;
    }
  } else {
    const size_t kk = std::max<uint32_t>(num_labels, 1);
    KMP_CUDA(h->hist.ensure(kk * kLadderLevels));
    KMP_CUDA(h->ohist.ensure(kk * kLadderLevels));
    KMP_CUDA(h->jmin.ensure(kk));
    KMP_CUDA(h->ojmin.ensure(kk));
    KMP_CUDA(h->out_cur.ensure(kk));
    KMP_CUDA(h->out_delta.ensure(kk));
    KMP_CUDA(cudaMemsetAsync(h->hist.p, 0, kk * kLadderLevels * sizeof(int32_t), h->stream));
    KMP_CUDA(cudaMemsetAsync(h->ohist.p, 0, kk * kLadderLevels * sizeof(int32_t), h->stream));
  }
  // hub tier scratch: the clusterer stages 4 B per hub edge of the largest sub-round; the refiner has bucket
  // regions, cursors and an overflow list
  if (mode == 0 && h->t4_max_subround_edges > 0) {
    KMP_CUDA(h->hub_lab.ensure(h->t4_max_subround_edges));
  }
  if (mode == 1 && h->t4_max_slots > 0) {
    KMP_CUDA(h->hub_tab.ensure(h->t4_max_slots)); // no initialisation: the cursors say how much of a region is valid
    KMP_CUDA(h->hub_cursor.ensure(h->t4_max_slots / kBucketCap));
    KMP_CUDA(h->hub_ovf.ensure(std::max<uint64_t>(h->t4_max_wave_edges, 1)));
    KMP_CUDA(cudaGetLastError());
  }
  (void)num_labels;
  return KMP_OK;
}

struct RunCtx {
  int mode;
  uint32_t num_labels;
  int32_t max_cluster_weight;
  bool has_min;
  bool has_comm;
};

SweepArgs make_sweep_args(kmp_lp_handle *h, const RunCtx &rc) {
  SweepArgs a{};
  a.xadj = h->xadj;
  a.adjncy = h->adjncy;
  a.vwgt = h->vwgt;
  a.adjwgt = h->adjwgt;
  a.label = h->label.p;
  a.labg = h->labg.p;
  a.pull = false;
  a.window = make_window(0, 0);
  a.queue = h->queue.p;
  a.weight = h->weight.p;
  a.max_w = rc.mode == 1 ? h->maxw.p : nullptr;
  a.min_w = rc.has_min ? h->minw.p : nullptr;
  a.communities = rc.has_comm ? h->communities.p : nullptr;
  a.active = h->active.p;
  a.favored = h->favored.p;
  a.max_cluster_weight = rc.max_cluster_weight;
  a.num_labels = rc.num_labels;
  a.max_num_neighbors = h->cfg.max_num_neighbors;
  a.mv_u = h->mv_u.p;
  a.mv_t = h->mv_t.p;
  a.mover_count = h->ctr32.p + (h->mover_parity ? 3 : 0);
  if (h->direct_send != nullptr) { // sharded library path: [count, -, -, -, u[cap], t[cap]]
    a.mover_count = h->direct_send;
    a.mv_u = h->direct_send + 4;
    a.mv_t = h->direct_send + 4 + h->direct_cap;
  }
  a.incoming = h->incoming.p;
  a.hist = h->hist.p;
  a.counters = h->ctr64.p;
  a.sel_target = nullptr;
  a.sel_favored = nullptr;
  return a;
}

CommitArgs make_commit_args(kmp_lp_handle *h, const RunCtx &rc) {
  CommitArgs c{};
  c.xadj = h->xadj;
  c.adjncy = h->adjncy;
  c.vwgt = h->vwgt;
  c.label = h->label.p;
  c.labg = h->labg.p;
  c.stamp = 0;
  c.weight = h->weight.p;
  c.max_w = rc.mode == 1 ? h->maxw.p : nullptr;
  c.min_w = rc.has_min ? h->minw.p : nullptr;
  c.active = h->active.p;
  c.max_cluster_weight = rc.max_cluster_weight;
  c.k = rc.num_labels;
  c.mv_u = h->mv_u.p;
  c.mv_t = h->mv_t.p;
  c.acc = h->acc.p;
  c.mover_count = h->ctr32.p + (h->mover_parity ? 3 : 0);
  c.next_mover_count = h->ctr32.p + (h->mover_parity ? 0 : 3);
  c.also_zero = (h->world > 1 && h->comm != nullptr) ? h->dist_send.p : nullptr;
  c.incoming = h->incoming.p;
  c.slotmap = h->slotmap.p;
  c.cslot = h->cslot.p;
  c.chist = h->chist.p;
  c.hist = h->hist.p;
  c.jmin = h->jmin.p;
  c.out_cur = h->out_cur.p;
  c.out_delta = h->out_delta.p;
  c.ohist = h->ohist.p;
  c.ojmin = h->ojmin.p;
  c.moved_count = h->ctr32.p + 1;
  return c;
}

// A sub-round sg in [0, 4 * S) = (degree group, hashed class). Groups 0 and 2 have one work list (tiers 0 and 3),
// group 1 has the lists of tiers 1-2, group 3 those of tiers 4..7 (tier 7 = hubs, sharded round-robin instead of by
// range).
struct SubRound {
  int group;
  uint32_t sr;
  int first_tier, last_tier;  // inclusive
  uint32_t size[kNumTiers];   // full list sizes of the tiers of this sub-round (0 elsewhere)
  uint32_t lo[kNumTiers], hi[kNumTiers]; // this rank's slice (range-sharded tiers)
  uint32_t total;
};

SubRound subround_of_sg(const kmp_lp_handle *h, uint32_t sg) {
  const uint32_t S = h->lists_S;
  SubRound q{};
  q.group = static_cast<int>(sg / S);
  q.sr = sg % S;
  q.first_tier = first_tier_of_group(q.group);
  q.last_tier = last_tier_of_group(q.group);
  for (int t = q.first_tier; t <= q.last_tier; ++t) {
    const uint32_t sz = h->list_off[t * S + q.sr + 1] - h->list_off[t * S + q.sr];
    q.size[t] = sz;
    q.total += sz;
    if (t == kHubTier) { // every rank sees the whole hub list and takes entries i % world == rank
      q.lo[t] = 0;
      q.hi[t] = sz;
    } else {
      q.lo[t] = static_cast<uint32_t>(static_cast<uint64_t>(sz) * h->rank / h->world);
      q.hi[t] = static_cast<uint32_t>(static_cast<uint64_t>(sz) * (h->rank + 1) / h->world);
    }
  }
  return q;
}

// capacity of one rank's proposal buffer for sub-round sg (identical on every rank)
uint32_t subround_cap(const kmp_lp_handle *h, const SubRound &q) {
  uint32_t cap = 1;
  for (int t = q.first_tier; t <= q.last_tier; ++t) {
    cap += (q.size[t] + h->world - 1) / h->world;
  }
  return cap;
}

// sweep kernels of one sub-round over this rank's share of the lists
int sweep_subround(kmp_lp_handle *h, const RunCtx &rc, uint32_t iter, uint32_t sg, const SubRound &q) {
  const uint32_t S = h->lists_S;
  SweepArgs sa = make_sweep_args(h, rc);
  sa.base_tie = sync_base(h->cfg.seed, h->call_counter, iter, SALT_TIE);
  sa.base_fav = sync_base(h->cfg.seed, h->call_counter, iter, SALT_FAV);
  sa.base_commit = sync_base(h->cfg.seed, h->call_counter, iter * 4096 + sg, SALT_COMMIT);
  sa.accumulate = !h->stepping && rc.mode == 0; // refiner: commit_refine_fused builds the level histograms
  sa.pull = h->pull_this;
  sa.window = make_window(iter, sg);
  h->cur_subround = q.sr;
  h->cur_sg = sg;
  int live = 0;
  for (int t = q.first_tier; t <= q.last_tier; ++t) {
    live += q.size[t] != 0;
  }
  // several tiers in this sub-round: fork them onto side streams (per-tier timing mode keeps them serial so
  // that every tier's CUDA-event time is its own)
  const bool fork = live > 1 && !h->timing;
  if (fork) {
    KMP_CUDA(cudaEventRecord(h->ev_fork, h->stream));
  }
  int side = 0;
  bool used[3] = {false, false, false};
  for (int t = q.last_tier; t >= q.first_tier; --t) { // largest degrees first: the longest tails start earliest
    if (q.size[t] == 0) {
      continue;
    }
    sa.list = h->order.p + h->list_off[t * S + q.sr] + q.lo[t];
    sa.list_size = q.hi[t] - q.lo[t];
    h->sweep_stream = h->stream;
    if (fork && side < 3 && t != q.first_tier) {
      h->sweep_stream = h->side_stream[side];
      used[side] = true;
      KMP_CUDA(cudaStreamWaitEvent(h->sweep_stream, h->ev_fork, 0));
    }
    const cudaError_t e = launch_sweep(h, rc.mode, t, sa);
    if (h->sweep_stream != h->stream) {
      KMP_CUDA(cudaEventRecord(h->ev_join[side], h->sweep_stream));
      ++side;
    }
    h->sweep_stream = h->stream;
    KMP_CUDA(e);
  }
  for (int i = 0; i < 3; ++i) {
    if (used[i]) {
      KMP_CUDA(cudaStreamWaitEvent(h->stream, h->ev_join[i], 0));
    }
  }
  return KMP_OK;
}

// push activation (rounds with few movers): flags for the neighbours of the accepted movers; reads acc[] / mv_u[]
void launch_push_activation(kmp_lp_handle *h, const CommitArgs &ca, const SubRound &q) {
  const uint32_t size = q.total;
  const int ev = timed_begin(h, kTagPush);
  switch (q.group) {
  case 0: commit_activate<4><<<capped(h, grid_for(static_cast<uint64_t>(size) * 4, 256, kSMs * 6)), 256, 0, h->stream>>>(ca); break;
  case 1: commit_activate<8><<<capped(h, grid_for(static_cast<uint64_t>(size) * 8, 256, kSMs * 6)), 256, 0, h->stream>>>(ca); break;
  case 2: commit_activate<32><<<capped(h, grid_for(static_cast<uint64_t>(size) * 32, 256, kSMs * 6)), 256, 0, h->stream>>>(ca); break;
  default: commit_activate<256><<<capped(h, grid_for(static_cast<uint64_t>(size) * 256, 256, kSMs * 6)), 256, 0, h->stream>>>(ca); break;
  }
  timed_end(h, ev);
  ++h->kernel_launches;
}
// The whole commit of sub-round sg in one cooperative launch, over the proposals in mv_u / mv_t -- or, with
// gathered != nullptr, over the all-gathered proposal buffers (world * (4 + 2 * cap) words) of a sharded run or of
// the stepping API, which the same launch unpacks and accumulates first. Every rank runs the same
// order-independent commit on the same proposals, so the replicas stay bit-identical.
int commit_subround(kmp_lp_handle *h, const RunCtx &rc, uint32_t iter, uint32_t sg, const SubRound &q,
                    const uint32_t *gathered) {
  CommitArgs ca = make_commit_args(h, rc);
  ca.base_commit = sync_base(h->cfg.seed, h->call_counter, iter * 4096 + sg, SALT_COMMIT);
  ca.stamp = h->stamps_ok ? make_stamp(iter, sg) : 0;
  GatheredArgs ga{gathered, h->world, gathered != nullptr ? subround_cap(h, q) : 0u,
                  h->ctr32.p + (h->mover_parity ? 3 : 0)};
  GridBarrier bar{h->grid_bar.p, h->grid_bar.p + 1};
  const int ev = timed_begin(h, kTagCommit);
  if (rc.mode == 1) {
    uint32_t passes = std::max<uint32_t>(1, h->cfg.sync_commit_passes);
    const uint32_t k = rc.num_labels;
    const size_t smem = 4 * std::max<size_t>(k * kLadderLevels <= kSmemPrivLimit ? static_cast<size_t>(k) * kLadderLevels : 0,
                                             k <= kSmemPrivLimit ? k : 0);
    const uint32_t blocks = capped(h, std::min<uint32_t>(grid_for(std::max<uint32_t>(q.total, k), 256),
                                                         static_cast<uint32_t>(h->fused_blocks_refine)));
    void *rargs[] = {&ca, &ga, &bar, &passes};
    if (h->p64) {
      KMP_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void *>(commit_refine_fused<true>), dim3(blocks), dim3(256), rargs,
                                           smem, h->stream));
    } else {
      KMP_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void *>(commit_refine_fused<false>), dim3(blocks), dim3(256), rargs,
                                           smem, h->stream));
    }
  } else {
    const uint32_t blocks = capped(h, std::min<uint32_t>(grid_for(q.total, 256), static_cast<uint32_t>(h->fused_blocks)));
    void *args[] = {&ca, &ga, &bar};
    if (h->p64) {
      KMP_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void *>(commit_cluster_fused<true>), dim3(blocks), dim3(256), args, 0,
                                           h->stream));
    } else {
      KMP_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void *>(commit_cluster_fused<false>), dim3(blocks), dim3(256), args,
                                           0, h->stream));
    }
  }
  timed_end(h, ev);
  ++h->kernel_launches;
  if (!h->pull_this || !h->pull_next) {
    launch_push_activation(h, ca, q); // acc[] / mv_u[] still hold this sub-round's verdicts
  }
  h->mover_parity ^= 1u;
  return KMP_OK;
}

// Activation mode of LP round `iter` (lp_device.cuh): in PULL rounds the sweeps scan every listed vertex
// and read the moves of their neighbours from the stamps next to the labels -- free when most vertices
// are active anyway (all of a fresh clustering, the first rounds of a refinement); in PUSH rounds movers
// flag their neighbours (a second walk over their adjacency) and the sweeps skip inactive vertices
// without touching their adjacency -- cheaper once few vertices move. Round r + 1 pulls iff at least
// 1/16 of the listed vertices moved in round r - 1 (rounds 0 and 1 always pull); movers push whenever the
// running or the next round reads flags. Both modes give the same active set as the reference's flags.
void choose_activation(kmp_lp_handle *h, uint32_t iter) {
  // a capped neighbourhood scan cannot see all neighbours' stamps
  const bool can_pull = h->stamps_ok && h->cfg.max_num_neighbors >= h->max_degree;
  auto heavy = [&](uint32_t moved) { return moved == 0xFFFFFFFFu || 16ull * moved >= h->visited_total; };
  if (iter == 0) {
    h->moved_hist[0] = h->moved_hist[1] = 0xFFFFFFFFu; // [0]: round iter - 1, [1]: round iter - 2
    h->pull_this = can_pull;
  } else {
    h->pull_this = h->pull_next;
  }
  h->pull_next = can_pull && heavy(h->moved_hist[0]);
  if (const char *e = std::getenv("KMP_ACTIVATION")) { // experiments / tests: force one mode
    if (e[0] == 'p' && e[1] == 'u' && e[2] == 's') {
      h->pull_this = h->pull_next = false;
    } else if (e[0] == 'p' && e[1] == 'u' && e[2] == 'l' && can_pull) {
      h->pull_this = h->pull_next = true;
    }
  }
}

int begin_iteration(kmp_lp_handle *h, uint32_t iter) {
  KMP_CUDA(cudaMemsetAsync(h->ctr32.p, 0, kCtr32Size * sizeof(uint32_t), h->stream)); // proposal counters, moved, hub queues
  KMP_CUDA(cudaMemsetAsync(h->queue.p, 0, h->queue.cap * sizeof(uint32_t), h->stream));
  if (h->hub_cursor.p != nullptr) { // normally already zero (sweep_hub_select resets what it reads)
    KMP_CUDA(cudaMemsetAsync(h->hub_cursor.p, 0, h->hub_cursor.cap * sizeof(uint32_t), h->stream));
  }
  if (h->world > 1 && h->comm != nullptr && h->dist_send.p != nullptr) {
    KMP_CUDA(cudaMemsetAsync(h->dist_send.p, 0, sizeof(uint32_t), h->stream)); // proposal counter of the send buffer
  }
  h->mover_parity = 0;
  choose_activation(h, iter);
  h->pull_rounds += h->pull_this ? 1 : 0;
  h->push_rounds += (!h->pull_this || !h->pull_next) ? 1 : 0;
  if (iter >= 2 && h->stamps_ok && h->n > 0) {
    const int ev = timed_begin(h, kTagMisc);
    if (h->p64) {
      k_age_stamps<true><<<grid_for(h->n, 256), 256, 0, h->stream>>>(h->n, h->labg.p, iter & 1u);
    } else {
      k_age_stamps<false><<<grid_for(h->n, 256), 256, 0, h->stream>>>(h->n, h->labg.p, iter & 1u);
    }
    timed_end(h, ev);
    ++h->kernel_launches;
  }
  return KMP_OK;
}

void end_iteration(kmp_lp_handle *h, uint32_t moved) {
  h->moved_hist[1] = h->moved_hist[0];
  h->moved_hist[0] = moved;
}

// ---- NCCL, loaded on demand ----------------------------------------------------------------------------
struct NcclApi {
  void *lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllReduce)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  const char *(*GetErrorString)(ncclResult_t) = nullptr;
};
NcclApi g_nccl;

int load_nccl() {
  if (g_nccl.lib != nullptr) {
    return KMP_OK;
  }
  // an already loaded libnccl.so.2 (e.g. the one torch ships) is reused by the loader; else the system one
  void *lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (lib == nullptr) {
    lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  }
  if (lib == nullptr) {
    return fail(KMP_ERR_NCCL, std::string("cannot load libnccl.so.2: ") + dlerror());
  }
  NcclApi a;
  a.lib = lib;
  a.GetUniqueId = reinterpret_cast<decltype(a.GetUniqueId)>(dlsym(lib, "ncclGetUniqueId"));
  a.CommInitRank = reinterpret_cast<decltype(a.CommInitRank)>(dlsym(lib, "ncclCommInitRank"));
  a.CommDestroy = reinterpret_cast<decltype(a.CommDestroy)>(dlsym(lib, "ncclCommDestroy"));
  a.AllGather = reinterpret_cast<decltype(a.AllGather)>(dlsym(lib, "ncclAllGather"));
  a.AllReduce = reinterpret_cast<decltype(a.AllReduce)>(dlsym(lib, "ncclAllReduce"));
  a.GetErrorString = reinterpret_cast<decltype(a.GetErrorString)>(dlsym(lib, "ncclGetErrorString"));
  if (!a.GetUniqueId || !a.CommInitRank || !a.CommDestroy || !a.AllGather || !a.AllReduce || !a.GetErrorString) {
    return fail(KMP_ERR_NCCL, "libnccl.so.2 lacks a required symbol");
  }
  g_nccl = a;
  return KMP_OK;
}

#define KMP_NCCL(expr)                                                                                     \
  do {                                                                                                     \
    ncclResult_t _r = (expr);                                                                              \
    if (_r != ncclSuccess) {                                                                               \
      return fail(KMP_ERR_NCCL, std::string(#expr) + ": " + g_nccl.GetErrorString(_r));                    \
    }                                                                                                      \
  } while (0)

// Sweep this rank's share of sub-round sg and pack its proposals into d_send (4 + 2 * cap words:
// [count, -, -, -, u[cap], t[cap]]).
int dist_sweep_pack(kmp_lp_handle *h, const RunCtx &rc, uint32_t iter, uint32_t sg, const SubRound &q, uint32_t *d_send) {
  const uint32_t cap = subround_cap(h, q);
  // library path: the sweeps write their proposals straight into the send buffer (count in word 0, zeroed by the
  // previous commit / begin_iteration) -- no pack kernel
  h->direct_send = (d_send == h->dist_send.p && h->comm != nullptr) ? d_send : nullptr;
  h->direct_cap = cap;
  h->stepping = true;
  const int r = sweep_subround(h, rc, iter, sg, q);
  h->stepping = false;
  const bool direct = h->direct_send != nullptr;
  h->direct_send = nullptr;
  if (r != KMP_OK) {
    return r;
  }
  if (direct) {
    return KMP_OK;
  }
  k_pack_movers<<<capped(h, grid_for(cap, 256, kSMs * 4)), 256, 0, h->stream>>>(h->mv_u.p, h->mv_t.p,
                                                                      h->ctr32.p + (h->mover_parity ? 3 : 0), cap, d_send);
  ++h->kernel_launches;
  KMP_CUDA(cudaGetLastError());
  return KMP_OK;
}

// ---- degree groups 0 and 1 of a clustering round: one persistent cooperative launch each (lp_lowgroup.cuh) ----
template <bool EW, bool P64> const void *low_group_kernel_t(int group) {
  return group == 0 ? reinterpret_cast<const void *>(sweep_commit_low<EW, P64, 8, 8, 4>)
                    : reinterpret_cast<const void *>(sweep_commit_low<EW, P64, 16, 32, 8>);
}
const void *low_group_kernel(bool ew, bool p64, int group) {
  return ew ? (p64 ? low_group_kernel_t<true, true>(group) : low_group_kernel_t<true, false>(group))
            : (p64 ? low_group_kernel_t<false, true>(group) : low_group_kernel_t<false, false>(group));
}
// per device, from kmp_lp_create: false if a kernel cannot be resident
bool configure_low_groups(kmp_lp_handle *h, int sms) {
  for (int g = 0; g < 2; ++g) {
    for (int ew = 0; ew < 2; ++ew) {
      for (int p64 = 0; p64 < 2; ++p64) {
        int per_sm = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, low_group_kernel(ew, p64, g), 256, 0) != cudaSuccess ||
            per_sm < 1) {
          return false;
        }
        h->low_blocks[g][ew][p64] = static_cast<uint32_t>(sms * per_sm);
      }
    }
  }
  return true;
}
// The clusterer on one GPU; the sharded run, the refiner and the stepping API keep the per-sub-round path (a sweep
// launch and a commit launch per sub-round).
bool can_run_low_groups(const kmp_lp_handle *h, const RunCtx &rc) {
  return rc.mode == 0 && h->world == 1 && !h->stepping;
}
static_assert(kMaxSubrounds <= kLowMaxSubrounds, "ensure_lists admits more sub-rounds than LowGroupArgs holds");
// All sub-rounds of degree group `group` (0: tier 0, 1: tiers 1-2) of LP round `iter`, in sub-round order, with the
// hashes, stamp windows, move stamps and proposal-counter parities the per-sub-round path uses.
int run_low_group(kmp_lp_handle *h, const RunCtx &rc, uint32_t iter, int group) {
  const uint32_t S = h->lists_S;
  const int ta = first_tier_of_group(group), tb = last_tier_of_group(group);
  SweepArgs sa = make_sweep_args(h, rc);
  sa.base_tie = sync_base(h->cfg.seed, h->call_counter, iter, SALT_TIE);
  sa.base_fav = sync_base(h->cfg.seed, h->call_counter, iter, SALT_FAV);
  sa.accumulate = true;
  sa.pull = h->pull_this;
  sa.list = h->order.p;
  CommitArgs ca = make_commit_args(h, rc);
  LowGroupArgs g{};
  g.push = !h->pull_this || !h->pull_next;
  g.ctr32 = h->ctr32.p;
  g.counters[0] = h->ctr64.p + ta;
  g.counters[1] = h->ctr64.p + tb;
  uint32_t max_total = 0;
  for (uint32_t s = 0; s < S; ++s) {
    const uint32_t sg = static_cast<uint32_t>(group) * S + s;
    const SubRound q = subround_of_sg(h, sg);
    if (q.total == 0) {
      continue;
    }
    LowSubround &x = g.sub[g.num_sub++];
    x.off[0] = h->list_off[ta * S + s];
    x.size[0] = q.size[ta];
    x.off[1] = h->list_off[tb * S + s];
    x.size[1] = tb != ta ? q.size[tb] : 0u;
    const StampWindow w = make_window(iter, sg);
    x.window_start = w.start;
    x.window_len = w.len;
    x.base_commit = sync_base(h->cfg.seed, h->call_counter, iter * 4096 + sg, SALT_COMMIT);
    x.stamp = h->stamps_ok ? make_stamp(iter, sg) : 0u;
    x.parity = h->mover_parity;
    h->mover_parity ^= 1u;
    max_total = std::max(max_total, q.total);
  }
  if (g.num_sub == 0) {
    return KMP_OK;
  }
  const bool ew = h->adjwgt != nullptr;
  const uint32_t blocks = capped(h, std::min<uint32_t>(grid_for(max_total, 256), h->low_blocks[group][ew][h->p64]));
  GridBarrier bar{h->grid_bar.p, h->grid_bar.p + 1};
  void *args[] = {&sa, &ca, &g, &bar};
  // timing mode: the group's sweeps AND commits are this one event pair, under the group's first tier
  const int ev = timed_begin(h, ta);
  KMP_CUDA(cudaLaunchCooperativeKernel(low_group_kernel(ew, h->p64, group), dim3(blocks), dim3(256), args, 0, h->stream));
  timed_end(h, ev);
  ++h->kernel_launches;
  ++h->sweep_launches;
  ++h->group_launches[ta];
  return KMP_OK;
}

// One LP round over all (group, sub-round) lists. Returns via *moved the accepted moves.
int run_iteration(kmp_lp_handle *h, const RunCtx &rc, uint32_t iter, uint32_t *moved, uint32_t *proposals) {
  const uint32_t S = h->lists_S;
  int rc0 = begin_iteration(h, iter);
  if (rc0 != KMP_OK) {
    return rc0;
  }
  if (h->world > 1) { // exchange buffers for the largest sub-round, allocated once
    size_t max_words = 4;
    for (uint32_t sg = 0; sg < kNumGroups * S; ++sg) {
      max_words = std::max<size_t>(max_words, 4 + 2 * static_cast<size_t>(subround_cap(h, subround_of_sg(h, sg))));
    }
    KMP_CUDA(h->dist_send.ensure(max_words));
    KMP_CUDA(h->dist_recv.ensure(std::max<size_t>(max_words * h->world, h->n)));
  }
  for (uint32_t sg = 0; sg < kNumGroups * S; ++sg) {
    const SubRound q = subround_of_sg(h, sg);
    if (q.total == 0) {
      continue;
    }
    int rc2;
    if (h->world > 1) { // sharded: sweep the own slice, all-gather the proposals (NVLink), replicated commit
      const size_t words = 4 + 2 * static_cast<size_t>(subround_cap(h, q));
      rc2 = dist_sweep_pack(h, rc, iter, sg, q, h->dist_send.p);
      if (rc2 != KMP_OK) {
        return rc2;
      }
      KMP_NCCL(g_nccl.AllGather(h->dist_send.p, h->dist_recv.p, words, ncclUint32, h->comm, h->stream));
      rc2 = commit_subround(h, rc, iter, sg, q, h->dist_recv.p);
      if (rc2 != KMP_OK) {
        return rc2;
      }
      continue;
    }
    if (q.group <= 1 && can_run_low_groups(h, rc)) { // every sub-round of the group in one launch
      rc2 = run_low_group(h, rc, iter, q.group);
      if (rc2 != KMP_OK) {
        return rc2;
      }
      sg = static_cast<uint32_t>(q.group + 1) * S - 1;
      continue;
    }
    rc2 = sweep_subround(h, rc, iter, sg, q);
    if (rc2 != KMP_OK) {
      return rc2;
    }
    rc2 = commit_subround(h, rc, iter, sg, q, nullptr);
    if (rc2 != KMP_OK) {
      return rc2;
    }
  }
  uint32_t host[2] = {0, 0};
  KMP_CUDA(cudaMemcpyAsync(host, h->ctr32.p, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
  KMP_CUDA(cudaStreamSynchronize(h->stream));
  *moved = host[1];
  end_iteration(h, host[1]);
  (void)proposals;
  return KMP_OK;
}

// packed gather array: word width by the label range; (re)allocated grow-only
int prepare_labg(kmp_lp_handle *h, uint32_t num_labels) {
  h->p64 = num_labels > (1u << 24) || h->force_p64; // KMP_FORCE_P64=1: the 8-byte gather words on small test inputs
  KMP_CUDA(h->labg.ensure(static_cast<size_t>(std::max<uint32_t>(h->n, 1)) * (h->p64 ? 8 : 4)));
  return KMP_OK;
}
void launch_init_cluster(kmp_lp_handle *h) {
  if (h->p64) {
    k_init_cluster<true><<<grid_for(h->n, 256), 256, 0, h->stream>>>(h->n, h->vwgt, h->label.p, h->labg.p, h->weight.p,
                                                                       h->favored.p, h->active.p);
  } else {
    k_init_cluster<false><<<grid_for(h->n, 256), 256, 0, h->stream>>>(h->n, h->vwgt, h->label.p, h->labg.p, h->weight.p,
                                                                        h->favored.p, h->active.p);
  }
}
void launch_pack_labels(kmp_lp_handle *h) {
  if (h->p64) {
    k_pack_labels<true><<<grid_for(h->n, 256), 256, 0, h->stream>>>(h->n, h->label.p, h->labg.p);
  } else {
    k_pack_labels<false><<<grid_for(h->n, 256), 256, 0, h->stream>>>(h->n, h->label.p, h->labg.p);
  }
}

// The labels on the device as a k-way partition: weight[0, k) (zeroed by the caller) += their block weights, and
// labels >= k (e.g. a clustering left on the device, or a host partition with an id >= k) are refused before any
// kernel indexes a [k] array by a label. bad: a zeroed device counter. One n-sized read and one host wait.
int checked_block_weights(kmp_lp_handle *h, uint32_t k, unsigned long long *bad) {
  const uint32_t n = h->n;
  if (n > 0) {
    bal_block_weights<<<capped(h, grid_for(n, 256)), 256, 0, h->stream>>>(n, k, h->vwgt, h->label.p, h->weight.p, bad);
    ++h->kernel_launches;
  }
  unsigned long long b = 0;
  KMP_CUDA(cudaMemcpyAsync(&b, bad, sizeof(b), cudaMemcpyDeviceToHost, h->stream));
  KMP_CUDA(cudaStreamSynchronize(h->stream));
  if (b != 0) {
    return fail(KMP_ERR_INVALID, "labels >= k on the device: a clustering is not a k-way partition");
  }
  return KMP_OK;
}

int refuse_without_labels(const kmp_lp_handle *h) {
  if (!h->labels_valid) {
    return fail(KMP_ERR_INVALID, "no labels of the current graph on the device: cluster, pass a partition or call "
                                 "kmp_lp_upload_partition first");
  }
  return KMP_OK;
}

int begin_call(kmp_lp_handle *h, kmp_lp_stats *stats) {
  if (h == nullptr || !h->have_graph) {
    return fail(KMP_ERR_INVALID, "no graph set");
  }
  KMP_CUDA(cudaSetDevice(h->device));
  if (stats != nullptr) {
    std::memset(stats, 0, sizeof(*stats));
  }
  h->kernel_launches = 0;
  h->sweep_launches = 0;
  h->pull_rounds = h->push_rounds = 0;
  h->sweep_events_used = 0;
  for (int g = 0; g < kStatTiers; ++g) {
    h->group_launches[g] = 0;
  }
  KMP_CUDA(cudaEventRecord(h->ev_begin, h->stream));
  return KMP_OK;
}

int end_call(kmp_lp_handle *h, kmp_lp_stats *stats) {
  if (h->world > 1 && h->comm != nullptr && stats != nullptr) { // every rank reports the whole job's scan counters
    KMP_NCCL(g_nccl.AllReduce(h->ctr64.p, h->ctr64.p, kCtrNodes + kStatTiers, ncclUint64, ncclSum, h->comm, h->stream));
  }
  KMP_CUDA(cudaEventRecord(h->ev_end, h->stream));
  KMP_CUDA(cudaStreamSynchronize(h->stream));
  if (stats != nullptr) {
    unsigned long long c[kCtrNodes + kStatTiers] = {0};
    KMP_CUDA(cudaMemcpy(c, h->ctr64.p, sizeof(c), cudaMemcpyDeviceToHost));
    for (int g = 0; g < kStatTiers; ++g) {
      stats->group_edges[g] = c[g];
      stats->group_nodes[g] = c[kCtrNodes + g];
      stats->group_launches[g] = h->group_launches[g];
      stats->edges_scanned += c[g];
      stats->nodes_visited += c[kCtrNodes + g];
    }
    float ms = 0.f;
    cudaEventElapsedTime(&ms, h->ev_begin, h->ev_end);
    stats->device_ms = ms;
    float sweep = 0.f;
    for (size_t i = 0; i < h->sweep_events_used; ++i) {
      float t = 0.f;
      cudaEventElapsedTime(&t, h->sweep_events[i].first, h->sweep_events[i].second);
      if (h->sweep_event_group[i] < kNumTiers) {
        sweep += t;
      }
      stats->group_sweep_ms[h->sweep_event_group[i]] += t;
      (void)kTagPush;
    }
    stats->sweep_ms = sweep;
    stats->sweep_launches = h->sweep_launches;
    stats->kernel_launches = h->kernel_launches;
    stats->pull_rounds = h->pull_rounds;
    stats->push_rounds = h->push_rounds;
  }
  return KMP_OK;
}

int upload_optional_u32(kmp_lp_handle *h, DevBuf<uint32_t> &buf, const uint32_t *host, size_t n) {
  if (host == nullptr) {
    return KMP_OK;
  }
  KMP_CUDA(buf.ensure(n));
  KMP_CUDA(cudaMemcpyAsync(buf.p, host, n * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
  return KMP_OK;
}

int cluster_post_passes(kmp_lp_handle *h, int32_t max_w, uint32_t num_clusters, kmp_lp_stats *stats) {
  const uint32_t n = h->n;
  const bool two_hop = (1.0 - 1.0 * num_clusters / n) <= h->cfg.two_hop_threshold; // lp_clusterer.cc:164-166
  const int iso = h->cfg.isolated_nodes_strategy;
  const bool iso_match = iso == KMP_ISOLATED_MATCH || (iso == KMP_ISOLATED_MATCH_DURING_TWO_HOP && two_hop);
  const bool iso_cluster = iso == KMP_ISOLATED_CLUSTER || (iso == KMP_ISOLATED_CLUSTER_DURING_TWO_HOP && two_hop);
  auto sort_pairs = [&](uint32_t cnt, int bits) -> int { // pairs_a -> pairs_b, ascending
    size_t tmp = 0;
    KMP_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tmp, h->pairs_a.p, h->pairs_b.p, static_cast<int>(cnt), 0, bits, h->stream));
    KMP_CUDA(h->cub_tmp.ensure(tmp));
    KMP_CUDA(cub::DeviceRadixSort::SortKeys(h->cub_tmp.p, tmp, h->pairs_a.p, h->pairs_b.p, static_cast<int>(cnt), 0, bits,
                                            h->stream));
    return KMP_OK;
  };
  if ((iso_match || iso_cluster) && h->num_isolated > 1) {
    KMP_CUDA(h->pairs_a.ensure(h->num_isolated));
    KMP_CUDA(h->pairs_b.ensure(h->num_isolated));
    reset_u32<<<1, 1, 0, h->stream>>>(h->ctr32.p + 2);
    k_collect_isolated<<<grid_for(n, 256), 256, 0, h->stream>>>(n, h->xadj, h->pairs_a.p, h->ctr32.p + 2);
    uint32_t iso_cnt = 0;
    KMP_CUDA(cudaMemcpyAsync(&iso_cnt, h->ctr32.p + 2, sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
    KMP_CUDA(cudaStreamSynchronize(h->stream));
    if (iso_cnt > 1) {
      const int rc = sort_pairs(iso_cnt, 32); // key 0: ascending vertex id
      if (rc != KMP_OK) {
        return rc;
      }
      if (iso_match) {
        k_match_isolated<<<grid_for(iso_cnt / 2 + 1, 256), 256, 0, h->stream>>>(iso_cnt, h->pairs_b.p, h->label.p, h->weight.p, max_w);
      } else {
        k_next_fit<<<1, 256, 0, h->stream>>>(iso_cnt, h->pairs_b.p, h->label.p, h->weight.p, max_w); // one group
      }
      h->kernel_launches += 3;
      KMP_CUDA(cudaGetLastError());
    }
  }
  if (!two_hop || h->cfg.two_hop_strategy == KMP_TWO_HOP_DISABLE) {
    return KMP_OK;
  }
  if (stats != nullptr) {
    stats->two_hop_ran = 1;
  }
  KMP_CUDA(h->pairs_a.ensure(n));
  KMP_CUDA(h->pairs_b.ensure(n));
  reset_u32<<<1, 1, 0, h->stream>>>(h->ctr32.p + 2);
  k_collect_two_hop<<<grid_for(n, 256), 256, 0, h->stream>>>(n, h->xadj, h->vwgt, h->label.p, h->weight.p,
                                                              h->favored.p, max_w, h->pairs_a.p, h->ctr32.p + 2);
  uint32_t cnt = 0;
  KMP_CUDA(cudaMemcpyAsync(&cnt, h->ctr32.p + 2, sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
  KMP_CUDA(cudaStreamSynchronize(h->stream));
  if (cnt > 1) {
    const int rc = sort_pairs(cnt, 64);
    if (rc != KMP_OK) {
      return rc;
    }
    if (h->cfg.two_hop_strategy == KMP_TWO_HOP_CLUSTER_THREADWISE) {
      k_next_fit<<<grid_for(static_cast<uint64_t>(cnt) * 32, 256, kSMs * 8), 256, 0, h->stream>>>(cnt, h->pairs_b.p, h->label.p,
                                                                                                 h->weight.p, max_w);
      h->kernel_launches += 3;
    } else {
      // group heads: reuse mv-independent scratch (pairs_a is free after the sort)
      uint32_t *head_in = reinterpret_cast<uint32_t *>(h->pairs_a.p);
      uint32_t *head_out = head_in + cnt;
      k_two_hop_heads<<<grid_for(cnt, 256), 256, 0, h->stream>>>(cnt, h->pairs_b.p, head_in);
      size_t tmp2 = 0;
      KMP_CUDA(cub::DeviceScan::InclusiveScan(nullptr, tmp2, head_in, head_out, MaxOp(), static_cast<int>(cnt), h->stream));
      KMP_CUDA(h->cub_tmp.ensure(tmp2));
      KMP_CUDA(cub::DeviceScan::InclusiveScan(h->cub_tmp.p, tmp2, head_in, head_out, MaxOp(), static_cast<int>(cnt), h->stream));
      k_match_two_hop<<<grid_for(cnt, 256), 256, 0, h->stream>>>(cnt, h->pairs_b.p, head_out, h->label.p, h->weight.p);
      h->kernel_launches += 5;
    }
    KMP_CUDA(cudaGetLastError());
  }
  return KMP_OK;
}

// ---- schedule KMP_SCHEDULE_SEQ_STRICT ----------------------------------------------------------------
// mode 0: labels are (re)initialised by the engine; mode 1: h->label holds the partition. Results stay in
// h->label / h->weight; iteration statistics go to *stats, the scan counters to the last tier slot of ctr64.
int run_strict(kmp_lp_handle *h, int mode, uint32_t num_keys, int32_t max_cluster_weight, uint32_t desired,
               uint32_t k, bool has_min, bool has_comm, kmp_lp_stats *stats) {
  const size_t n = std::max<uint32_t>(h->n, 1);
  const size_t keys = std::max<size_t>(std::max<size_t>(num_keys, n), 1);
  KMP_CUDA(h->favored.ensure(n));
  KMP_CUDA(h->active.ensure(n));
  KMP_CUDA(h->st_slot.ensure(keys));
  KMP_CUDA(h->st_slot2.ensure(keys));
  KMP_CUDA(h->st_concurrent.ensure(keys));
  KMP_CUDA(h->st_used.ensure(keys));
  KMP_CUDA(h->st_ent_key.ensure(keys + 1));
  KMP_CUDA(h->st_ent_val.ensure(keys + 1));
  KMP_CUDA(h->st_ent2_key.ensure(keys + 1));
  KMP_CUDA(h->st_ent2_val.ensure(keys + 1));
  KMP_CUDA(h->st_tie_best.ensure(keys + 1));
  KMP_CUDA(h->st_tie_fav.ensure(keys + 1));
  KMP_CUDA(h->st_second.ensure(n));
  KMP_CUDA(h->st_chunks.ensure(2 * (n + 64)));
  KMP_CUDA(h->st_sub_perm.ensure(n / 64 + 2));
  KMP_CUDA(h->st_match.ensure(n));
  KMP_CUDA(h->st_buckets.ensure(36));
  KMP_CUDA(h->st_rng.ensure(1));
  KMP_CUDA(h->st_stats.ensure(1));
  if (!h->strict_seeded) { // Random::reseed + the RandomPermutations member of the LP object, once per object
    kmp_strict::strict_seed_kernel<<<1, 32, 0, h->stream>>>(h->st_rng.p, h->cfg.seed);
    h->strict_seeded = true;
    ++h->kernel_launches;
  }
  kmp_strict::Args a{};
  a.n = h->n;
  a.m = h->m;
  a.xadj = h->xadj;
  a.adjncy = h->adjncy;
  a.vwgt = h->vwgt;
  a.adjwgt = h->adjwgt;
  a.sorted = h->graph_sorted ? 1 : 0;
  a.buckets = h->st_buckets.p;
  a.num_iterations = h->cfg.num_iterations;
  a.large_degree_threshold = h->cfg.large_degree_threshold;
  a.max_num_neighbors = h->cfg.max_num_neighbors;
  a.impl = h->cfg.impl;
  a.tie_uniform = h->cfg.tie_breaking_strategy == KMP_TIE_UNIFORM ? 1 : 0;
  a.two_hop_strategy = h->cfg.two_hop_strategy;
  a.isolated_nodes_strategy = h->cfg.isolated_nodes_strategy;
  a.two_hop_threshold = h->cfg.two_hop_threshold;
  a.mode = mode;
  a.max_cluster_weight = max_cluster_weight;
  a.desired_num_clusters = desired;
  a.k = k;
  a.max_bw = mode == 1 ? h->maxw.p : nullptr;
  a.min_bw = has_min ? h->minw.p : nullptr;
  a.communities = has_comm ? h->communities.p : nullptr;
  a.label = h->label.p;
  a.weight = h->weight.p;
  a.favored = h->favored.p;
  a.active = h->active.p;
  a.slot = h->st_slot.p;
  a.ent_key = h->st_ent_key.p;
  a.ent_val = h->st_ent_val.p;
  a.slot2 = h->st_slot2.p;
  a.ent2_key = h->st_ent2_key.p;
  a.ent2_val = h->st_ent2_val.p;
  a.concurrent = h->st_concurrent.p;
  a.used_entries = h->st_used.p;
  a.second_phase_nodes = h->st_second.p;
  a.tie_best = h->st_tie_best.p;
  a.tie_fav = h->st_tie_fav.p;
  a.chunks = h->st_chunks.p;
  a.sub_perm = h->st_sub_perm.p;
  a.match_map = h->st_match.p;
  a.rng = h->st_rng.p;
  a.stats = h->st_stats.p;
  kmp_strict::strict_kernel<<<1, 32, 0, h->stream>>>(a);
  ++h->kernel_launches;
  KMP_CUDA(cudaGetLastError());
  kmp_strict::Stats hs{};
  KMP_CUDA(cudaMemcpyAsync(&hs, h->st_stats.p, sizeof(hs), cudaMemcpyDeviceToHost, h->stream));
  KMP_CUDA(cudaStreamSynchronize(h->stream));
  if (stats != nullptr) {
    stats->iterations = hs.iterations;
    for (uint32_t i = 0; i < 64; ++i) {
      stats->moved[i] = hs.moved[i];
    }
    stats->num_clusters = hs.num_clusters;
    stats->two_hop_ran = hs.two_hop_ran;
  }
  // end_call sums the per-tier scan counters: park the engine's totals in tier slot 7
  unsigned long long c[2] = {hs.edges_scanned, hs.nodes_visited};
  KMP_CUDA(cudaMemcpy(h->ctr64.p + (kStatTiers - 1), &c[0], 8, cudaMemcpyHostToDevice));
  KMP_CUDA(cudaMemcpy(h->ctr64.p + kCtrNodes + (kStatTiers - 1), &c[1], 8, cudaMemcpyHostToDevice));
  return KMP_OK;
}

int end_call(kmp_lp_handle *h, kmp_lp_stats *stats);

int strict_cluster(kmp_lp_handle *h, int32_t max_cluster_weight, uint32_t desired_num_clusters,
                   const uint32_t *communities, uint32_t *clustering_out, kmp_lp_stats *stats) {
  const uint32_t n = h->n;
  KMP_CUDA(h->label.ensure(std::max<uint32_t>(n, 1)));
  KMP_CUDA(h->weight.ensure(std::max<uint32_t>(n, 1)));
  KMP_CUDA(h->ctr64.ensure(kCtrSize));
  KMP_CUDA(cudaMemsetAsync(h->ctr64.p, 0, kCtrSize * sizeof(unsigned long long), h->stream));
  if (communities != nullptr) {
    KMP_CUDA(h->communities.ensure(n));
    KMP_CUDA(cudaMemcpyAsync(h->communities.p, communities, static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, h->stream));
  }
  int rc = run_strict(h, 0, n, max_cluster_weight, desired_num_clusters, 0, false, communities != nullptr, stats);
  if (rc != KMP_OK) {
    return rc;
  }
  if (clustering_out != nullptr && n > 0) {
    KMP_CUDA(cudaMemcpyAsync(clustering_out, h->label.p, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost, h->stream));
  }
  ++h->call_counter;
  h->labels_valid = true;
  const kmp_lp_stats keep = stats != nullptr ? *stats : kmp_lp_stats{};
  rc = end_call(h, stats);
  if (stats != nullptr) { // end_call fills the timing / counter fields only
    stats->iterations = keep.iterations;
    std::memcpy(stats->moved, keep.moved, sizeof(keep.moved));
    stats->num_clusters = keep.num_clusters;
    stats->two_hop_ran = keep.two_hop_ran;
  }
  return rc;
}

int strict_refine(kmp_lp_handle *h, uint32_t k, const int32_t *max_block_weights, const int32_t *min_block_weights,
                  const uint32_t *communities, uint32_t *partition_inout, int32_t *block_weights_out,
                  kmp_lp_stats *stats) {
  const uint32_t n = h->n;
  KMP_CUDA(h->label.ensure(std::max<uint32_t>(n, 1)));
  KMP_CUDA(h->weight.ensure(std::max<uint32_t>(std::max(n, k), 1)));
  KMP_CUDA(h->maxw.ensure(k));
  KMP_CUDA(h->ctr64.ensure(kCtrSize));
  KMP_CUDA(cudaMemsetAsync(h->ctr64.p, 0, kCtrSize * sizeof(unsigned long long), h->stream));
  if (partition_inout != nullptr && n > 0) {
    KMP_CUDA(cudaMemcpyAsync(h->label.p, partition_inout, static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, h->stream));
  }
  if (partition_inout != nullptr) {
    h->labels_valid = true;
  }
  KMP_CUDA(cudaMemsetAsync(h->weight.p, 0, static_cast<size_t>(k) * 4, h->stream));
  int rc = checked_block_weights(h, k, h->ctr64.p + kCtrScratch); // the engine recomputes the weights itself
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(cudaMemcpyAsync(h->maxw.p, max_block_weights, static_cast<size_t>(k) * 4, cudaMemcpyHostToDevice, h->stream));
  if (min_block_weights != nullptr) {
    KMP_CUDA(h->minw.ensure(k));
    KMP_CUDA(cudaMemcpyAsync(h->minw.p, min_block_weights, static_cast<size_t>(k) * 4, cudaMemcpyHostToDevice, h->stream));
  }
  if (communities != nullptr) {
    KMP_CUDA(h->communities.ensure(n));
    KMP_CUDA(cudaMemcpyAsync(h->communities.p, communities, static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, h->stream));
  }
  rc = run_strict(h, 1, k, 0, 0, k, min_block_weights != nullptr, communities != nullptr, stats);
  if (rc != KMP_OK) {
    return rc;
  }
  if (partition_inout != nullptr && n > 0) {
    KMP_CUDA(cudaMemcpyAsync(partition_inout, h->label.p, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost, h->stream));
  }
  if (block_weights_out != nullptr) {
    KMP_CUDA(cudaMemcpyAsync(block_weights_out, h->weight.p, static_cast<size_t>(k) * 4, cudaMemcpyDeviceToHost, h->stream));
  }
  const kmp_lp_stats keep = stats != nullptr ? *stats : kmp_lp_stats{};
  rc = end_call(h, stats);
  if (stats != nullptr) {
    stats->iterations = keep.iterations;
    std::memcpy(stats->moved, keep.moved, sizeof(keep.moved));
  }
  return rc;
}

} // namespace

// ================================================================================================
// C ABI
// ================================================================================================
extern "C" {

int kmp_lp_abi_version(void) { return KMP_LP_ABI_VERSION; }

const char *kmp_last_error(void) { return g_last_error.c_str(); }

void kmp_lp_default_config(int mode, kmp_lp_config *cfg) {
  if (cfg == nullptr) {
    return;
  }
  std::memset(cfg, 0, sizeof(*cfg));
  cfg->num_iterations = 5;                   // presets.cc:143 / :342
  cfg->large_degree_threshold = 0xFFFFFFFFu; // :144 / :343
  cfg->max_num_neighbors = 0xFFFFFFFFu;      // :145 / :344
  cfg->tie_breaking_strategy = KMP_TIE_UNIFORM;
  cfg->two_hop_threshold = 0.5;
  cfg->seed = 0;
  cfg->sync_subrounds = 8;
  cfg->sync_granule_log2 = 4;
  cfg->device = -1;
  if (mode == 0) {
    cfg->impl = KMP_LP_TWO_PHASE;                                     // :146
    cfg->two_hop_strategy = KMP_TWO_HOP_MATCH_THREADWISE;             // :148
    cfg->isolated_nodes_strategy = KMP_ISOLATED_MATCH_DURING_TWO_HOP; // :150-151
    cfg->sync_commit_passes = 1;
  } else {
    cfg->impl = KMP_LP_SINGLE_PHASE; // :345
    cfg->two_hop_strategy = KMP_TWO_HOP_DISABLE;
    cfg->isolated_nodes_strategy = KMP_ISOLATED_KEEP;
    cfg->sync_commit_passes = 4;
  }
}

int kmp_lp_create(const kmp_lp_config *cfg, kmp_lp_handle **out) {
  if (cfg == nullptr || out == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) {
    return fail(KMP_ERR_CUDA, std::string("no CUDA device available (there is no CPU fallback): ") +
                                  cudaGetErrorString(e));
  }
  // options the sync schedule cannot honour are refused, never silently mapped to something else
  if (cfg->schedule != KMP_SCHEDULE_SYNC && cfg->schedule != KMP_SCHEDULE_SEQ_STRICT) {
    return fail(KMP_ERR_INVALID, "unknown schedule");
  }
  if (cfg->schedule == KMP_SCHEDULE_SYNC) {
    if (cfg->tie_breaking_strategy == KMP_TIE_GEOMETRIC) {
      return fail(KMP_ERR_UNSUPPORTED, "tie_breaking_strategy GEOMETRIC is order-dependent (lp_clusterer.cc:252-278): "
                                       "use KMP_SCHEDULE_SEQ_STRICT or UNIFORM");
    }
    if (cfg->tie_breaking_strategy != KMP_TIE_UNIFORM) {
      return fail(KMP_ERR_INVALID, "unknown tie_breaking_strategy");
    }
    if (cfg->two_hop_strategy == KMP_TWO_HOP_MATCH || cfg->two_hop_strategy == KMP_TWO_HOP_CLUSTER) {
      return fail(KMP_ERR_UNSUPPORTED, "global two-hop MATCH / CLUSTER (label_propagation.h:1030-1191) is an id-ordered "
                                       "chain: use MATCH_THREADWISE or KMP_SCHEDULE_SEQ_STRICT");
    }

  }
  if (cfg->relabel_before_second_phase != 0) { // default false (presets.cc:147)
    return fail(KMP_ERR_UNSUPPORTED, "relabel_before_second_phase (label_propagation.h:272-319) is not implemented");
  }
  if (cfg->two_hop_strategy < KMP_TWO_HOP_DISABLE || cfg->two_hop_strategy > KMP_TWO_HOP_CLUSTER_THREADWISE ||
      cfg->isolated_nodes_strategy < KMP_ISOLATED_KEEP || cfg->isolated_nodes_strategy > KMP_ISOLATED_CLUSTER_DURING_TWO_HOP ||
      cfg->impl < KMP_LP_SINGLE_PHASE || cfg->impl > KMP_LP_GROWING_HASH_TABLES) {
    return fail(KMP_ERR_INVALID, "unknown two_hop_strategy / isolated_nodes_strategy / impl");
  }
  kmp_lp_handle *h = new (std::nothrow) kmp_lp_handle();
  if (h == nullptr) {
    return fail(KMP_ERR_ALLOC, "out of host memory");
  }
  h->cfg = *cfg;
  if (const char *e = std::getenv("KMP_HUB_BUCKET_CAP")) { // experiment / test knobs; results do not depend on them
    h->hub_bucket_cap = static_cast<uint32_t>(std::min<long>(kBucketCap, std::max(1, std::atoi(e))));
  }
  if (const char *e = std::getenv("KMP_HUB_SEL_LIMIT")) {
    h->hub_sel_limit = static_cast<uint32_t>(std::max(0, std::atoi(e)));
  }
  if (const char *e = std::getenv("KMP_HUB_WAVE_SLOTS")) {
    h->hub_wave_slots = static_cast<uint64_t>(std::max(32ll, std::atoll(e)));
  }
  if (const char *e = std::getenv("KMP_GRID_CAP")) {
    h->grid_cap = static_cast<uint32_t>(std::max(1, std::atoi(e)));
  }
  if (h->cfg.sync_subrounds == 0) {
    h->cfg.sync_subrounds = 8;
  }
  if (h->cfg.sync_commit_passes == 0) {
    h->cfg.sync_commit_passes = 1;
  }
  int dev = cfg->device;
  if (dev < 0) {
    cudaGetDevice(&dev);
  }
  h->device = dev;
  if (cudaSetDevice(dev) != cudaSuccess || cudaStreamCreateWithFlags(&h->owned_stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreate(&h->ev_begin) != cudaSuccess || cudaEventCreate(&h->ev_end) != cudaSuccess) {
    delete h;
    return fail(KMP_ERR_CUDA, "failed to create stream/events");
  }
  h->stream = h->owned_stream;
  h->sweep_stream = h->stream;
  for (int i = 0; i < 3; ++i) {
    if (cudaStreamCreateWithFlags(&h->side_stream[i], cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&h->ev_join[i], cudaEventDisableTiming) != cudaSuccess) {
      delete h;
      return fail(KMP_ERR_CUDA, "failed to create side streams");
    }
  }
  if (cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming) != cudaSuccess) {
    delete h;
    return fail(KMP_ERR_CUDA, "failed to create events");
  }
  if (const char *e = std::getenv("KMP_FORCE_P64")) {
    h->force_p64 = std::atoi(e) != 0;
  }
  int sms = kSMs;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  // every commit is a cooperative launch (grid barriers between its phases)
  int coop = 0, per_sm = 0, per_sm_r = 0;
  cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
  if (coop == 0) {
    delete h;
    return fail(KMP_ERR_CUDA, "this device does not support cooperative launches");
  }
  // co-resident CTAs of both commit kernels, the refiner's with its largest dynamic shared memory (kSmemPrivLimit ints)
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, commit_cluster_fused<false>, 256, 0) != cudaSuccess ||
      per_sm < 1 ||
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_r, commit_refine_fused<false>, 256, kSmemPrivLimit * 4) !=
          cudaSuccess ||
      per_sm_r < 1) {
    delete h;
    return fail(KMP_ERR_CUDA, "a fused commit kernel cannot be resident on this device");
  }
  if (h->grid_bar.ensure(2) != cudaSuccess || cudaMemset(h->grid_bar.p, 0, 2 * sizeof(unsigned)) != cudaSuccess) {
    delete h;
    return fail(KMP_ERR_CUDA, "failed to allocate the grid barrier");
  }
  // all co-resident CTAs: a sub-round of a 10^8-vertex graph commits 10^7 proposals, each a short chain of
  // dependent random accesses -- the grid is sized by the proposal count up to this limit
  h->fused_blocks = sms * per_sm;
  h->fused_blocks_refine = sms * per_sm_r;
  if (!configure_low_groups(h, sms)) {
    delete h;
    return fail(KMP_ERR_CUDA, "a persistent low-degree clustering kernel cannot be resident on this device");
  }
  if (!(configure_team_kernels<0, false, false>(h, sms) && configure_team_kernels<0, false, true>(h, sms) &&
        configure_team_kernels<0, true, false>(h, sms) && configure_team_kernels<0, true, true>(h, sms) &&
        configure_team_kernels<1, false, false>(h, sms) && configure_team_kernels<1, false, true>(h, sms) &&
        configure_team_kernels<1, true, false>(h, sms) && configure_team_kernels<1, true, true>(h, sms))) {
    delete h;
    return fail(KMP_ERR_CUDA, "a sweep_team kernel cannot be resident on this device");
  }
  *out = h;
  return KMP_OK;
}

int kmp_lp_destroy(kmp_lp_handle *h) {
  if (h == nullptr) {
    return KMP_OK;
  }
  cudaSetDevice(h->device);
  cudaStreamSynchronize(h->stream);
  if (h->comm != nullptr) {
    g_nccl.CommDestroy(h->comm);
    h->comm = nullptr;
  }
  kmp_lp_free_scratch(h);
  h->own_xadj.release();
  h->own_adjncy.release();
  h->own_vwgt.release();
  h->own_adjwgt.release();
  h->order.release();
  for (auto &p : h->sweep_events) {
    cudaEventDestroy(p.first);
    cudaEventDestroy(p.second);
  }
  cudaEventDestroy(h->ev_begin);
  cudaEventDestroy(h->ev_end);
  if (h->ev_ct0 != nullptr) {
    cudaEventDestroy(h->ev_ct0);
    cudaEventDestroy(h->ev_ct1);
  }
  cudaEventDestroy(h->ev_fork);
  for (int i = 0; i < 3; ++i) {
    cudaEventDestroy(h->ev_join[i]);
    cudaStreamDestroy(h->side_stream[i]);
  }
  cudaStreamDestroy(h->owned_stream);
  delete h;
  return KMP_OK;
}

int kmp_lp_set_timing(kmp_lp_handle *h, int enabled) {
  if (h == nullptr) {
    return fail(KMP_ERR_INVALID, "null handle");
  }
  h->timing = enabled != 0;
  return KMP_OK;
}

static int set_graph_common(kmp_lp_handle *h, uint32_t n, uint32_t m) {
  if (n > 0x7FFFFFFFu || m > 0x7FFFFFFFu) { // CUB scans / sorts take int counts; 32-bit EdgeID build of the reference
    return fail(KMP_ERR_UNSUPPORTED, "n and m must be below 2^31");
  }
  h->n = n;
  h->m = m;
  h->have_graph = true;
  h->labels_valid = false;
  h->lists_valid = false;
  h->slot_state_clean = false;
  h->graph_sorted = false;
  if (h->cfg.schedule == KMP_SCHEDULE_SEQ_STRICT) {
    if (n > KMP_SEQ_STRICT_MAX_N) {
      return fail(KMP_ERR_UNSUPPORTED, "KMP_SCHEDULE_SEQ_STRICT is a one-thread-block schedule for n <= KMP_SEQ_STRICT_MAX_N");
    }
    return KMP_OK; // no work lists: the engine walks the reference's chunk order
  }
  int rc = ensure_lists(h);
  if (rc != KMP_OK) {
    return rc;
  }
  h->num_isolated = 0;
  {
    // vertices in the tail bucket are either isolated or above the degree threshold; count isolated
    // ones exactly only when a post pass needs them (cheap: tail bucket size is an upper bound)
    const uint32_t S = h->lists_S;
    h->num_isolated = h->list_off[kNumTiers * S + 1] - h->list_off[kNumTiers * S];
  }
  return KMP_OK;
}

int kmp_lp_set_graph(kmp_lp_handle *h, uint32_t n, uint32_t m, const uint32_t *xadj, const uint32_t *adjncy,
                     const int32_t *vwgt, const int32_t *adjwgt) {
  if (h == nullptr || xadj == nullptr || (m > 0 && adjncy == nullptr)) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  KMP_CUDA(cudaSetDevice(h->device));
  KMP_CUDA(h->own_xadj.ensure(static_cast<size_t>(n) + 1));
  KMP_CUDA(h->own_adjncy.ensure(m));
  // xadj first, on the handle's stream: the work lists only need the degrees and are built (kernels, a radix
  // pass, three small host round trips) while the m-sized arrays are still crossing PCIe on a side stream
  KMP_CUDA(cudaStreamSynchronize(h->stream)); // earlier work may still read the old arrays
  KMP_CUDA(cudaMemcpyAsync(h->own_xadj.p, xadj, (static_cast<size_t>(n) + 1) * 4, cudaMemcpyHostToDevice, h->stream));
  const cudaStream_t big = h->side_stream[0];
  if (m > 0) {
    KMP_CUDA(cudaMemcpyAsync(h->own_adjncy.p, adjncy, static_cast<size_t>(m) * 4, cudaMemcpyHostToDevice, big));
  }
  h->xadj = h->own_xadj.p;
  h->adjncy = h->own_adjncy.p;
  h->adjncy_16b = true; // cudaMalloc: 256-byte aligned
  h->vwgt = nullptr;
  h->adjwgt = nullptr;
  if (vwgt != nullptr) {
    KMP_CUDA(h->own_vwgt.ensure(n));
    KMP_CUDA(cudaMemcpyAsync(h->own_vwgt.p, vwgt, static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, h->stream));
    h->vwgt = h->own_vwgt.p;
  }
  if (adjwgt != nullptr) {
    KMP_CUDA(h->own_adjwgt.ensure(m));
    KMP_CUDA(cudaMemcpyAsync(h->own_adjwgt.p, adjwgt, static_cast<size_t>(m) * 4, cudaMemcpyHostToDevice, big));
    h->adjwgt = h->own_adjwgt.p;
  }
  KMP_CUDA(cudaEventRecord(h->ev_join[0], big));
  const int rc = set_graph_common(h, n, m);
  KMP_CUDA(cudaStreamWaitEvent(h->stream, h->ev_join[0], 0)); // later work on the handle's stream sees the whole graph
  return rc;
}

int kmp_lp_set_graph_device(kmp_lp_handle *h, uint32_t n, uint32_t m, const uint32_t *d_xadj, const uint32_t *d_adjncy,
                            const int32_t *d_vwgt, const int32_t *d_adjwgt) {
  if (h == nullptr || d_xadj == nullptr || (m > 0 && d_adjncy == nullptr)) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  auto misaligned4 = [](const void *p) { return (reinterpret_cast<uintptr_t>(p) & 3u) != 0; };
  if (misaligned4(d_xadj) || misaligned4(d_adjncy) || misaligned4(d_vwgt) || misaligned4(d_adjwgt)) {
    return fail(KMP_ERR_INVALID, "device graph arrays must be 4-byte aligned");
  }
  KMP_CUDA(cudaSetDevice(h->device));
  h->xadj = d_xadj;
  h->adjncy = d_adjncy;
  // a view into a larger buffer may start anywhere: the hub tier then reads adjncy from global memory
  h->adjncy_16b = (reinterpret_cast<uintptr_t>(d_adjncy) & 15u) == 0;
  h->vwgt = d_vwgt;
  h->adjwgt = d_adjwgt;
  return set_graph_common(h, n, m);
}

int kmp_lp_set_graph_sorted(kmp_lp_handle *h, int sorted) {
  if (h == nullptr || !h->have_graph) {
    return fail(KMP_ERR_INVALID, "no graph set");
  }
  h->graph_sorted = sorted != 0;
  return KMP_OK;
}

int kmp_lp_cluster(kmp_lp_handle *h, int32_t max_cluster_weight, uint32_t desired_num_clusters,
                   const uint32_t *communities, uint32_t *clustering_out, kmp_lp_stats *stats) {
  int rc = begin_call(h, stats);
  if (rc != KMP_OK) {
    return rc;
  }
  if (h->cfg.schedule == KMP_SCHEDULE_SEQ_STRICT) {
    return strict_cluster(h, max_cluster_weight, desired_num_clusters, communities, clustering_out, stats);
  }
  if (h->cfg.sync_commit_passes > 1) { // the cluster commit kernels decide in one pass: no departure credit
    return fail(KMP_ERR_UNSUPPORTED, "the clusterer's sync commit is single-pass (sync_commit_passes must be 1)");
  }
  if (h->world > 1 && h->comm == nullptr) {
    return fail(KMP_ERR_INVALID, "sharded handle without a communicator: call kmp_lp_dist_init (or drive the "
                                 "stepping API yourself)");
  }
  const uint32_t n = h->n;
  rc = ensure_lists(h);
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(h->label.ensure(n));
  KMP_CUDA(h->favored.ensure(n));
  KMP_CUDA(h->weight.ensure(n));
  rc = ensure_scratch(h, 0, n);
  if (rc != KMP_OK) {
    return rc;
  }
  rc = prepare_labg(h, n);
  if (rc != KMP_OK) {
    return rc;
  }
  rc = upload_optional_u32(h, h->communities, communities, n);
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(cudaMemsetAsync(h->ctr64.p, 0, kCtrSize * sizeof(unsigned long long), h->stream));
  if (n > 0) {
    launch_init_cluster(h);
    ++h->kernel_launches;
  }
  RunCtx ctx{0, n, max_cluster_weight, false, communities != nullptr};
  uint32_t num_clusters = n;
  for (uint32_t it = 0; it < h->cfg.num_iterations && n > 0; ++it) { // lp_clusterer.cc:94-105
    uint32_t moved = 0;
    rc = run_iteration(h, ctx, it, &moved, nullptr);
    if (rc != KMP_OK) {
      return rc;
    }
    if (stats != nullptr && it < 64) {
      stats->moved[it] = moved;
      stats->iterations = it + 1;
    }
    if (moved == 0) {
      break;
    }
    if (desired_num_clusters > 0) { // should_stop(), label_propagation.h:260-265
      reset_u32<<<1, 1, 0, h->stream>>>(h->ctr32.p + 2);
      k_count_nonzero<<<grid_for(n, 256), 256, 0, h->stream>>>(n, h->weight.p, h->ctr32.p + 2);
      KMP_CUDA(cudaMemcpyAsync(&num_clusters, h->ctr32.p + 2, 4, cudaMemcpyDeviceToHost, h->stream));
      KMP_CUDA(cudaStreamSynchronize(h->stream));
      if (num_clusters <= desired_num_clusters) {
        break;
      }
    }
  }
  if (n > 0) {
    reset_u32<<<1, 1, 0, h->stream>>>(h->ctr32.p + 2);
    k_count_nonzero<<<grid_for(n, 256), 256, 0, h->stream>>>(n, h->weight.p, h->ctr32.p + 2);
    KMP_CUDA(cudaMemcpyAsync(&num_clusters, h->ctr32.p + 2, 4, cudaMemcpyDeviceToHost, h->stream));
    KMP_CUDA(cudaStreamSynchronize(h->stream));
    h->kernel_launches += 2;
    if (stats != nullptr) {
      stats->num_clusters = num_clusters;
    }
    if (h->world > 1) { // favored[u] is only written by the rank that swept u: MAX over (favored ^ u), 0 elsewhere
      KMP_CUDA(h->dist_recv.ensure(n));
      k_xor_iota<<<grid_for(n, 256), 256, 0, h->stream>>>(n, h->favored.p, h->dist_recv.p);
      KMP_NCCL(g_nccl.AllReduce(h->dist_recv.p, h->dist_recv.p, n, ncclUint32, ncclMax, h->comm, h->stream));
      k_xor_iota<<<grid_for(n, 256), 256, 0, h->stream>>>(n, h->dist_recv.p, h->favored.p);
    }
    rc = cluster_post_passes(h, max_cluster_weight, num_clusters, stats); // lp_clusterer.cc:107-108
    if (rc != KMP_OK) {
      return rc;
    }
  }
  if (clustering_out != nullptr && n > 0) {
    KMP_CUDA(cudaMemcpyAsync(clustering_out, h->label.p, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost, h->stream));
  }
  ++h->call_counter;
  h->labels_valid = true;
  return end_call(h, stats);
}

int kmp_lp_upload_partition(kmp_lp_handle *h, const uint32_t *partition) {
  if (h == nullptr || !h->have_graph || partition == nullptr) {
    return fail(KMP_ERR_INVALID, "bad argument");
  }
  KMP_CUDA(cudaSetDevice(h->device));
  KMP_CUDA(h->label.ensure(h->n));
  KMP_CUDA(cudaMemcpyAsync(h->label.p, partition, static_cast<size_t>(h->n) * 4, cudaMemcpyHostToDevice, h->stream));
  KMP_CUDA(cudaStreamSynchronize(h->stream));
  h->labels_valid = true;
  return KMP_OK;
}

int kmp_lp_download_labels(kmp_lp_handle *h, uint32_t *labels_out) {
  if (h == nullptr || !h->have_graph || labels_out == nullptr || h->label.p == nullptr) {
    return fail(KMP_ERR_INVALID, "bad argument");
  }
  KMP_CUDA(cudaSetDevice(h->device));
  KMP_CUDA(cudaMemcpyAsync(labels_out, h->label.p, static_cast<size_t>(h->n) * 4, cudaMemcpyDeviceToHost, h->stream));
  KMP_CUDA(cudaStreamSynchronize(h->stream));
  return KMP_OK;
}

const uint32_t *kmp_lp_labels_device(kmp_lp_handle *h) { return h != nullptr ? h->label.p : nullptr; }

int kmp_lp_refine(kmp_lp_handle *h, uint32_t k, const int32_t *max_block_weights, const int32_t *min_block_weights,
                  const uint32_t *communities, uint32_t *partition_inout, int32_t *block_weights_out,
                  kmp_lp_stats *stats) {
  if (max_block_weights == nullptr || k == 0) {
    return fail(KMP_ERR_INVALID, "max_block_weights / k missing");
  }
  int rc = begin_call(h, stats);
  if (rc != KMP_OK) {
    return rc;
  }
  if (partition_inout == nullptr && (rc = refuse_without_labels(h)) != KMP_OK) {
    return rc;
  }
  if (h->cfg.schedule == KMP_SCHEDULE_SEQ_STRICT) {
    return strict_refine(h, k, max_block_weights, min_block_weights, communities, partition_inout, block_weights_out, stats);
  }
  if (h->world > 1 && h->comm == nullptr) {
    return fail(KMP_ERR_INVALID, "sharded handle without a communicator: call kmp_lp_dist_init (or drive the "
                                 "stepping API yourself)");
  }
  const uint32_t n = h->n;
  rc = ensure_lists(h);
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(h->label.ensure(n));
  KMP_CUDA(h->weight.ensure(k));
  KMP_CUDA(h->maxw.ensure(k));
  rc = ensure_scratch(h, 1, k);
  if (rc != KMP_OK) {
    return rc;
  }
  rc = prepare_labg(h, k);
  if (rc != KMP_OK) {
    return rc;
  }
  if (partition_inout != nullptr && n > 0) {
    KMP_CUDA(cudaMemcpyAsync(h->label.p, partition_inout, static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, h->stream));
  }
  if (partition_inout != nullptr) {
    h->labels_valid = true;
  }
  KMP_CUDA(cudaMemcpyAsync(h->maxw.p, max_block_weights, static_cast<size_t>(k) * 4, cudaMemcpyHostToDevice, h->stream));
  if (min_block_weights != nullptr) {
    KMP_CUDA(h->minw.ensure(k));
    KMP_CUDA(cudaMemcpyAsync(h->minw.p, min_block_weights, static_cast<size_t>(k) * 4, cudaMemcpyHostToDevice, h->stream));
  }
  rc = upload_optional_u32(h, h->communities, communities, n);
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(cudaMemsetAsync(h->ctr64.p, 0, kCtrSize * sizeof(unsigned long long), h->stream));
  KMP_CUDA(cudaMemsetAsync(h->weight.p, 0, static_cast<size_t>(k) * 4, h->stream));
  if (n > 0) {
    k_fill_u8<<<grid_for(n, 256), 256, 0, h->stream>>>(n, h->active.p, 1); // Base::initialize: all active
    launch_pack_labels(h); // reads the labels without indexing by them
    h->kernel_launches += 2;
  }
  rc = checked_block_weights(h, k, h->ctr64.p + kCtrScratch); // last: its wait covers the set-up above
  if (rc != KMP_OK) {
    return rc;
  }
  RunCtx ctx{1, k, 0, min_block_weights != nullptr, communities != nullptr};
  const uint64_t max_it = h->cfg.num_iterations == 0 ? ~0ull : h->cfg.num_iterations; // lp_refiner.cc:78-79
  for (uint64_t it = 0; it < max_it && n > 0; ++it) {
    uint32_t moved = 0;
    rc = run_iteration(h, ctx, static_cast<uint32_t>(it), &moved, nullptr);
    if (rc != KMP_OK) {
      return rc;
    }
    if (stats != nullptr && it < 64) {
      stats->moved[it] = moved;
      stats->iterations = static_cast<uint32_t>(it + 1);
    }
    if (moved == 0) {
      break;
    }
  }
  if (partition_inout != nullptr && n > 0) {
    KMP_CUDA(cudaMemcpyAsync(partition_inout, h->label.p, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost, h->stream));
  }
  if (block_weights_out != nullptr) {
    KMP_CUDA(cudaMemcpyAsync(block_weights_out, h->weight.p, static_cast<size_t>(k) * 4, cudaMemcpyDeviceToHost, h->stream));
  }
  return end_call(h, stats);
}

int kmp_lp_select_all(kmp_lp_handle *h, int mode, const uint32_t *labels, const int32_t *weights, uint32_t num_labels,
                      const int32_t *max_weights, int32_t max_cluster_weight, const int32_t *min_weights,
                      uint32_t call_index, uint32_t iteration, uint32_t *target_out, uint32_t *favored_out) {
  int rc = begin_call(h, nullptr);
  if (rc != KMP_OK) {
    return rc;
  }
  if (labels == nullptr || weights == nullptr || target_out == nullptr || (mode == 1 && max_weights == nullptr)) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  if (h->cfg.schedule != KMP_SCHEDULE_SYNC) {
    return fail(KMP_ERR_UNSUPPORTED, "kmp_lp_select_all evaluates the sync selection rule");
  }
  const uint32_t n = h->n;
  rc = ensure_lists(h);
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(h->label.ensure(n));
  KMP_CUDA(h->weight.ensure(num_labels));
  rc = ensure_scratch(h, mode, num_labels);
  if (rc != KMP_OK) {
    return rc;
  }
  rc = prepare_labg(h, mode == 0 ? std::max(n, num_labels) : num_labels);
  if (rc != KMP_OK) {
    return rc;
  }
  DevBuf<uint32_t> d_target, d_fav;
  KMP_CUDA(d_target.ensure(n));
  KMP_CUDA(d_fav.ensure(n));
  KMP_CUDA(cudaMemcpyAsync(h->label.p, labels, static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, h->stream));
  KMP_CUDA(cudaMemcpyAsync(d_target.p, labels, static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, h->stream));
  KMP_CUDA(cudaMemsetAsync(d_fav.p, 0xFF, static_cast<size_t>(n) * 4, h->stream));
  KMP_CUDA(cudaMemcpyAsync(h->weight.p, weights, static_cast<size_t>(num_labels) * 4, cudaMemcpyHostToDevice, h->stream));
  if (mode == 1) {
    KMP_CUDA(h->maxw.ensure(num_labels));
    KMP_CUDA(cudaMemcpyAsync(h->maxw.p, max_weights, static_cast<size_t>(num_labels) * 4, cudaMemcpyHostToDevice, h->stream));
    if (min_weights != nullptr) {
      KMP_CUDA(h->minw.ensure(num_labels));
      KMP_CUDA(cudaMemcpyAsync(h->minw.p, min_weights, static_cast<size_t>(num_labels) * 4, cudaMemcpyHostToDevice, h->stream));
    }
  }
  KMP_CUDA(cudaMemsetAsync(h->ctr64.p, 0, kCtrSize * sizeof(unsigned long long), h->stream));
  if (n > 0) {
    launch_pack_labels(h);
  }
  RunCtx ctx{mode, num_labels, max_cluster_weight, mode == 1 && min_weights != nullptr, false};
  SweepArgs sa = make_sweep_args(h, ctx);
  sa.active = nullptr;
  KMP_CUDA(cudaMemsetAsync(h->ctr32.p, 0, kCtr32Size * sizeof(uint32_t), h->stream)); // hub work-queue cursors
  KMP_CUDA(cudaMemsetAsync(h->queue.p, 0, h->queue.cap * sizeof(uint32_t), h->stream));
  if (h->hub_cursor.p != nullptr) {
    KMP_CUDA(cudaMemsetAsync(h->hub_cursor.p, 0, h->hub_cursor.cap * sizeof(uint32_t), h->stream));
  }
  sa.sel_target = d_target.p;
  sa.sel_favored = mode == 0 ? d_fav.p : nullptr;
  sa.base_tie = sync_base(h->cfg.seed, call_index, iteration, SALT_TIE);
  sa.base_fav = sync_base(h->cfg.seed, call_index, iteration, SALT_FAV);
  const uint32_t S = h->lists_S;
  for (uint32_t ts = 0; ts < kNumTiers * S; ++ts) { // every (tier, class) list once
    const uint32_t off = h->list_off[ts];
    const uint32_t size = h->list_off[ts + 1] - off;
    const int tier = static_cast<int>(ts / S);
    sa.list = h->order.p + off;
    sa.list_size = size;
    h->cur_subround = ts % S;
    h->cur_sg = group_of_tier(tier) * S + ts % S; // one queue cursor per (tier, sub-round)
    KMP_CUDA(launch_sweep(h, mode, tier, sa));
  }
  KMP_CUDA(cudaMemcpyAsync(target_out, d_target.p, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost, h->stream));
  if (favored_out != nullptr) {
    KMP_CUDA(cudaMemcpyAsync(favored_out, d_fav.p, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost, h->stream));
  }
  KMP_CUDA(cudaStreamSynchronize(h->stream));
  return KMP_OK;
}

int kmp_lp_free_scratch(kmp_lp_handle *h) {
  if (h == nullptr) {
    return KMP_OK;
  }
  cudaSetDevice(h->device);
  cudaStreamSynchronize(h->stream);
  h->label.release();
  h->labels_valid = false;
  h->favored.release();
  h->communities.release();
  h->weight.release();
  h->maxw.release();
  h->minw.release();
  h->active.release();
  h->mv_u.release();
  h->mv_t.release();
  h->cslot.release();
  h->slotmap.release();
  h->acc.release();
  h->incoming.release();
  h->chist.release();
  h->hist.release();
  h->jmin.release();
  h->out_cur.release();
  h->out_delta.release();
  h->ohist.release();
  h->ojmin.release();
  h->ctr32.release();
  h->ctr64.release();
  h->hub_tab.release();
  h->hub_cursor.release();
  h->hub_ovf.release();
  h->hub_lab.release();
  h->labg.release();
  h->sort_keys_in.release();
  h->sort_keys_out.release();
  h->sort_vals_in.release();
  h->t4_tmp_deg.release();
  h->t4_tmp_beg.release();
  h->t4_tmp_ids.release();
  h->cub_tmp.release();
  h->pairs_a.release();
  h->pairs_b.release();
  h->ct_vals_a.release();
  h->ct_vals_b.release();
  h->ct_flags.release();
  h->ct_rank.release();
  h->ct_cl.release();
  h->ct_counter.release();
  h->sp_ctl.release();
  for (DevBuf<uint32_t> *b : {&h->bal_cand, &h->bal_under, &h->bal_ctr32, &h->bal_target, &h->bal_lists, &h->bal_sv_a,
                              &h->bal_sv_b, &h->bal_blk}) {
    b->release();
  }
  for (DevBuf<int32_t> *b : {&h->bal_over, &h->bal_pbw, &h->bal_wt, &h->bal_prefix}) {
    b->release();
  }
  h->bal_flag.release();
  h->bal_key.release();
  h->bal_ctrl.release();
  h->bal_sk_a.release();
  h->bal_sk_b.release();
  h->ubal_deficit.release();
  h->ubal_tmask.release();
  {
    cudaMemPool_t pool = kmp_private_pool(h->device); // blocks cached for coarse graphs (kmp_contract.cuh)
    if (pool != nullptr) {
      cudaMemPoolTrimTo(pool, 0);
    }
  }
  h->slot_state_clean = false;
  return KMP_OK;
}

int kmp_lp_edge_cut(kmp_lp_handle *h, int64_t *cut_out) {
  if (h == nullptr || !h->have_graph || cut_out == nullptr || h->label.p == nullptr) {
    return fail(KMP_ERR_INVALID, "bad argument");
  }
  const int rc = refuse_without_labels(h);
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(cudaSetDevice(h->device));
  KMP_CUDA(h->ctr64.ensure(kCtrSize));
  KMP_CUDA(cudaMemsetAsync(h->ctr64.p + kCtrScratch, 0, sizeof(unsigned long long), h->stream));
  k_edge_cut<<<grid_for(static_cast<uint64_t>(h->n) * 32, 256), 256, 0, h->stream>>>(h->n, h->xadj, h->adjncy, h->adjwgt,
                                                                                      h->label.p, h->ctr64.p + kCtrScratch);
  unsigned long long c = 0;
  KMP_CUDA(cudaMemcpyAsync(&c, h->ctr64.p + kCtrScratch, sizeof(c), cudaMemcpyDeviceToHost, h->stream));
  KMP_CUDA(cudaStreamSynchronize(h->stream));
  *cut_out = static_cast<int64_t>(c / 2); // metrics.cc:51-52
  return KMP_OK;
}


// ================================================================================================
// Stepping API: one LP sub-round at a time, for the sharded multi-GPU driver (kaminpar_b200/dist.py).
// Every rank owns a full replica of the graph and of the label / weight / active state; the vertex
// frontier (the work lists) is sharded across ranks. Per sub-round each rank sweeps its share,
// the proposals are all-gathered, and every rank runs the same deterministic commit.
// ================================================================================================
int kmp_lp_set_shard(kmp_lp_handle *h, uint32_t rank, uint32_t world) {
  if (h == nullptr || world == 0 || rank >= world) {
    return fail(KMP_ERR_INVALID, "bad rank/world");
  }
  h->rank = rank;
  h->world = world;
  return KMP_OK;
}

// ---- NCCL inside the library: one process per GPU, every rank calls the same entry points ------------------
int kmp_lp_dist_unique_id(void *id_out) {
  if (id_out == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  const int rc = load_nccl();
  if (rc != KMP_OK) {
    return rc;
  }
  ncclUniqueId id;
  KMP_NCCL(g_nccl.GetUniqueId(&id));
  static_assert(sizeof(ncclUniqueId) == KMP_DIST_ID_BYTES, "ncclUniqueId size");
  std::memcpy(id_out, &id, sizeof(id));
  return KMP_OK;
}

int kmp_lp_dist_init(kmp_lp_handle *h, const void *id, uint32_t rank, uint32_t world) {
  if (h == nullptr || id == nullptr || world == 0 || rank >= world) {
    return fail(KMP_ERR_INVALID, "bad argument");
  }
  if (h->cfg.schedule != KMP_SCHEDULE_SYNC) {
    return fail(KMP_ERR_UNSUPPORTED, "only the sync schedule shards across GPUs");
  }
  const int rc = load_nccl();
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(cudaSetDevice(h->device));
  if (h->comm != nullptr) {
    g_nccl.CommDestroy(h->comm);
    h->comm = nullptr;
  }
  ncclUniqueId nid;
  std::memcpy(&nid, id, sizeof(nid));
  if (world > 1) {
    KMP_NCCL(g_nccl.CommInitRank(&h->comm, static_cast<int>(world), nid, static_cast<int>(rank)));
  }
  h->rank = rank;
  h->world = world;
  return KMP_OK;
}

int kmp_lp_dist_shutdown(kmp_lp_handle *h) {
  if (h == nullptr) {
    return KMP_OK;
  }
  if (h->comm != nullptr) {
    cudaStreamSynchronize(h->stream);
    g_nccl.CommDestroy(h->comm);
    h->comm = nullptr;
  }
  h->rank = 0;
  h->world = 1;
  return KMP_OK;
}

int kmp_lp_set_stream(kmp_lp_handle *h, void *cuda_stream) {
  if (h == nullptr) {
    return fail(KMP_ERR_INVALID, "null handle");
  }
  KMP_CUDA(cudaStreamSynchronize(h->stream));
  // 0 is a valid handle (the legacy default stream, which is what torch uses unless told otherwise);
  // (void*)-1 switches back to the handle's own stream
  h->stream = cuda_stream == reinterpret_cast<void *>(-1) ? h->owned_stream : static_cast<cudaStream_t>(cuda_stream);
  h->sweep_stream = h->stream;
  return KMP_OK;
}

uint32_t kmp_lp_num_subrounds(kmp_lp_handle *h) {
  return h != nullptr && h->lists_valid ? kNumGroups * h->lists_S : 0;
}

int kmp_lp_subround_cap(kmp_lp_handle *h, uint32_t sg, uint32_t *cap_out, uint32_t *size_out) {
  if (h == nullptr || !h->lists_valid || sg >= kNumGroups * h->lists_S) {
    return fail(KMP_ERR_INVALID, "bad sub-round");
  }
  const SubRound q = subround_of_sg(h, sg);
  if (cap_out != nullptr) {
    *cap_out = subround_cap(h, q);
  }
  if (size_out != nullptr) {
    *size_out = q.total;
  }
  return KMP_OK;
}

int kmp_lp_step_begin_cluster(kmp_lp_handle *h, int32_t max_cluster_weight, const uint32_t *communities) {
  int rc = begin_call(h, nullptr);
  if (rc != KMP_OK) {
    return rc;
  }
  if (h->cfg.schedule != KMP_SCHEDULE_SYNC) {
    return fail(KMP_ERR_UNSUPPORTED, "the stepping API drives the sync schedule");
  }
  const uint32_t n = h->n;
  rc = ensure_lists(h);
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(h->label.ensure(n));
  KMP_CUDA(h->favored.ensure(n));
  KMP_CUDA(h->weight.ensure(n));
  rc = ensure_scratch(h, 0, n);
  if (rc != KMP_OK) {
    return rc;
  }
  rc = upload_optional_u32(h, h->communities, communities, n);
  if (rc != KMP_OK) {
    return rc;
  }
  rc = prepare_labg(h, n);
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(cudaMemsetAsync(h->ctr64.p, 0, kCtrSize * sizeof(unsigned long long), h->stream));
  if (n > 0) {
    launch_init_cluster(h);
  }
  h->step_iter = 0;
  h->step_mode = 0;
  h->step_labels = n;
  h->step_mcw = max_cluster_weight;
  h->step_has_min = false;
  h->step_has_comm = communities != nullptr;
  return KMP_OK;
}

int kmp_lp_step_begin_refine(kmp_lp_handle *h, uint32_t k, const int32_t *max_block_weights,
                             const int32_t *min_block_weights, const uint32_t *communities, const uint32_t *partition) {
  if (max_block_weights == nullptr || partition == nullptr || k == 0) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  int rc = begin_call(h, nullptr);
  if (rc != KMP_OK) {
    return rc;
  }
  if (h->cfg.schedule != KMP_SCHEDULE_SYNC) {
    return fail(KMP_ERR_UNSUPPORTED, "the stepping API drives the sync schedule");
  }
  const uint32_t n = h->n;
  rc = ensure_lists(h);
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(h->label.ensure(n));
  KMP_CUDA(h->weight.ensure(k));
  KMP_CUDA(h->maxw.ensure(k));
  rc = ensure_scratch(h, 1, k);
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(cudaMemcpyAsync(h->label.p, partition, static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, h->stream));
  h->labels_valid = true;
  KMP_CUDA(cudaMemcpyAsync(h->maxw.p, max_block_weights, static_cast<size_t>(k) * 4, cudaMemcpyHostToDevice, h->stream));
  if (min_block_weights != nullptr) {
    KMP_CUDA(h->minw.ensure(k));
    KMP_CUDA(cudaMemcpyAsync(h->minw.p, min_block_weights, static_cast<size_t>(k) * 4, cudaMemcpyHostToDevice, h->stream));
  }
  rc = upload_optional_u32(h, h->communities, communities, n);
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(cudaMemsetAsync(h->ctr64.p, 0, kCtrSize * sizeof(unsigned long long), h->stream));
  KMP_CUDA(cudaMemsetAsync(h->weight.p, 0, static_cast<size_t>(k) * 4, h->stream));
  rc = prepare_labg(h, k);
  if (rc != KMP_OK) {
    return rc;
  }
  rc = checked_block_weights(h, k, h->ctr64.p + kCtrScratch);
  if (rc != KMP_OK) {
    return rc;
  }
  if (n > 0) {
    k_fill_u8<<<grid_for(n, 256), 256, 0, h->stream>>>(n, h->active.p, 1);
    launch_pack_labels(h);
  }
  h->step_iter = 0;
  h->step_mode = 1;
  h->step_labels = k;
  h->step_mcw = 0;
  h->step_has_min = min_block_weights != nullptr;
  h->step_has_comm = communities != nullptr;
  return KMP_OK;
}

int kmp_lp_step_begin_iteration(kmp_lp_handle *h) {
  if (h == nullptr || h->step_mode < 0) {
    return fail(KMP_ERR_INVALID, "step_begin_* not called");
  }
  return begin_iteration(h, h->step_iter);
}

// Sweep this rank's share of sub-round sg and pack its proposals into d_send (device memory,
// 4 + 2 * cap words: [count, -, -, -, u[cap], t[cap]]).
int kmp_lp_step_sweep(kmp_lp_handle *h, uint32_t iter, uint32_t sg, void *d_send) {
  if (h == nullptr || h->step_mode < 0 || d_send == nullptr) {
    return fail(KMP_ERR_INVALID, "bad argument");
  }
  const RunCtx rc{h->step_mode, h->step_labels, h->step_mcw, h->step_has_min, h->step_has_comm};
  return dist_sweep_pack(h, rc, iter, sg, subround_of_sg(h, sg), static_cast<uint32_t *>(d_send));
}

// Commit sub-round sg from the all-gathered proposal buffers (world * (4 + 2 * cap) words).
int kmp_lp_step_commit(kmp_lp_handle *h, uint32_t iter, uint32_t sg, const void *d_gathered) {
  if (h == nullptr || h->step_mode < 0 || d_gathered == nullptr) {
    return fail(KMP_ERR_INVALID, "bad argument");
  }
  const RunCtx rc{h->step_mode, h->step_labels, h->step_mcw, h->step_has_min, h->step_has_comm};
  return commit_subround(h, rc, iter, sg, subround_of_sg(h, sg), static_cast<const uint32_t *>(d_gathered));
}

int kmp_lp_step_end_iteration(kmp_lp_handle *h, uint32_t *moved) {
  if (h == nullptr || moved == nullptr) {
    return fail(KMP_ERR_INVALID, "bad argument");
  }
  uint32_t host[2] = {0, 0};
  KMP_CUDA(cudaMemcpyAsync(host, h->ctr32.p, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
  KMP_CUDA(cudaStreamSynchronize(h->stream));
  *moved = host[1];
  end_iteration(h, host[1]);
  ++h->step_iter;
  return KMP_OK;
}

// favored[u] ^ u into / out of a caller-provided device buffer of n words (for a MAX all-reduce:
// only the rank that owns u ever writes favored[u]; everybody else still holds u, i.e. 0 here).
int kmp_lp_step_favored_export(kmp_lp_handle *h, void *d_buf) {
  if (h == nullptr || d_buf == nullptr || h->step_mode != 0) {
    return fail(KMP_ERR_INVALID, "bad argument");
  }
  k_xor_iota<<<grid_for(h->n, 256), 256, 0, h->stream>>>(h->n, h->favored.p, static_cast<uint32_t *>(d_buf));
  KMP_CUDA(cudaGetLastError());
  return KMP_OK;
}
int kmp_lp_step_favored_import(kmp_lp_handle *h, const void *d_buf) {
  if (h == nullptr || d_buf == nullptr || h->step_mode != 0) {
    return fail(KMP_ERR_INVALID, "bad argument");
  }
  k_xor_iota<<<grid_for(h->n, 256), 256, 0, h->stream>>>(h->n, static_cast<const uint32_t *>(d_buf), h->favored.p);
  KMP_CUDA(cudaGetLastError());
  return KMP_OK;
}

// Post passes (clusterer) and result download; stats hold THIS rank's share of the scan counters.
int kmp_lp_step_finish(kmp_lp_handle *h, uint32_t *labels_out, int32_t *block_weights_out, kmp_lp_stats *stats) {
  if (h == nullptr || h->step_mode < 0) {
    return fail(KMP_ERR_INVALID, "step_begin_* not called");
  }
  const uint32_t n = h->n;
  if (stats != nullptr) {
    std::memset(stats, 0, sizeof(*stats));
  }
  if (h->step_mode == 0 && n > 0) {
    uint32_t num_clusters = 0;
    reset_u32<<<1, 1, 0, h->stream>>>(h->ctr32.p + 2);
    k_count_nonzero<<<grid_for(n, 256), 256, 0, h->stream>>>(n, h->weight.p, h->ctr32.p + 2);
    KMP_CUDA(cudaMemcpyAsync(&num_clusters, h->ctr32.p + 2, 4, cudaMemcpyDeviceToHost, h->stream));
    KMP_CUDA(cudaStreamSynchronize(h->stream));
    if (stats != nullptr) {
      stats->num_clusters = num_clusters;
    }
    int rc = cluster_post_passes(h, h->step_mcw, num_clusters, stats);
    if (rc != KMP_OK) {
      return rc;
    }
    ++h->call_counter;
    h->labels_valid = true;
  }
  if (labels_out != nullptr && n > 0) {
    KMP_CUDA(cudaMemcpyAsync(labels_out, h->label.p, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost, h->stream));
  }
  if (block_weights_out != nullptr && h->step_mode == 1) {
    KMP_CUDA(cudaMemcpyAsync(block_weights_out, h->weight.p, static_cast<size_t>(h->step_labels) * 4,
                             cudaMemcpyDeviceToHost, h->stream));
  }
  h->step_mode = -1;
  return end_call(h, stats);
}

} // extern "C"

#include "kmp_contract.cuh"
#include "kmp_sparsify.cuh"
#include "kmp_balance.cuh"
#include "kmp_underload.cuh"
