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
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <utility>
#include <vector>

#include <cstdlib>
#include <dlfcn.h>
#include <nccl.h> // types only: the library is dlopen()ed in kmp_lp_dist_init (no link-time dependency)
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_sort.cuh>

#include "../../include/kaminpar_b200_contraction.h"
#include "../../include/kaminpar_b200_lp.h"
#include "../../include/kaminpar_b200_prepare.h"
#include "../../include/kaminpar_b200_subgraph.h"
#include "../../include/kaminpar_b200_validate.h"
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
  DevBuf(DevBuf &&o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
  DevBuf &operator=(DevBuf &&o) noexcept {
    if (this != &o) {
      release();
      p = std::exchange(o.p, nullptr);
      cap = std::exchange(o.cap, 0);
    }
    return *this;
  }
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

// The result objects of the graph operations (coarse, prepared and subgraph arrays) and their per-call scratch come
// from the device's stream-ordered memory pool (cudaMallocAsync): a coarsening loop allocates and frees coarse graphs
// of hundreds of MB per level, and cudaMalloc / cudaFree of that size cost milliseconds and serialise the device. The
// pool keeps freed blocks (its release threshold is unbounded), so after the first level an allocation is a pointer
// bump. A PRIVATE pool per device (never the device's default pool, which the host application or torch's
// cudaMallocAsync backend may share): freed blocks stay in it until kmp_lp_free_scratch trims it.
inline cudaMemPool_t kmp_private_pool(int device) {
  static std::mutex mu;
  static cudaMemPool_t pools[64] = {};
  std::lock_guard<std::mutex> lock(mu);
  if (device < 0 || device >= 64) {
    return nullptr;
  }
  if (pools[device] == nullptr) {
    cudaMemPoolProps props{};
    props.allocType = cudaMemAllocationTypePinned;
    props.handleTypes = cudaMemHandleTypeNone;
    props.location.type = cudaMemLocationTypeDevice;
    props.location.id = device;
    cudaMemPool_t pool = nullptr;
    if (cudaMemPoolCreate(&pool, &props) == cudaSuccess) {
      unsigned long long keep = ~0ull;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
      pools[device] = pool;
    }
  }
  return pools[device];
}

// An owned block of kmp_private_pool. It is freed stream-ordered, on the stream it was allocated on, when the owner is
// destroyed, reallocated or assigned another block: a later user of the arrays on another stream (e.g. the next
// level's LP handle) must have synchronised with `stream` before then (kmp_coarse_destroy documents it).
template <typename T> struct PoolBuf {
  T *p = nullptr;
  size_t cap = 0;
  cudaStream_t stream = nullptr;
  PoolBuf() = default;
  PoolBuf(const PoolBuf &) = delete;
  PoolBuf &operator=(const PoolBuf &) = delete;
  PoolBuf(PoolBuf &&o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)), stream(o.stream) {}
  PoolBuf &operator=(PoolBuf &&o) noexcept {
    if (this != &o) {
      release();
      p = std::exchange(o.p, nullptr);
      cap = std::exchange(o.cap, 0);
      stream = o.stream;
    }
    return *this;
  }
  ~PoolBuf() { release(); }
  cudaError_t alloc(size_t n, cudaStream_t st, int device) {
    release();
    cudaMemPool_t pool = kmp_private_pool(device);
    if (pool == nullptr) {
      return cudaErrorMemoryAllocation;
    }
    cudaError_t e = cudaMallocFromPoolAsync(reinterpret_cast<void **>(&p), std::max<size_t>(n, 1) * sizeof(T), pool, st);
    if (e == cudaSuccess) {
      cap = std::max<size_t>(n, 1);
      stream = st;
    } else {
      p = nullptr;
    }
    return e;
  }
  void release() {
    if (p != nullptr) {
      cudaFreeAsync(p, stream);
    }
    p = nullptr;
    cap = 0;
  }
};

namespace {
// D2H copy of the first `count` elements of a result array; a null destination, an unallocated array (unit weights)
// or count 0 copies nothing
template <typename T> cudaError_t copy_out(T *dst, const PoolBuf<T> &buf, size_t count) {
  if (dst == nullptr || buf.p == nullptr || count == 0) {
    return cudaSuccess;
  }
  return cudaMemcpy(dst, buf.p, count * sizeof(T), cudaMemcpyDeviceToHost);
}

// H2D copy of a caller's host array into a new block of the pool on `st` (count 0: a one-element block, no copy)
template <typename T> cudaError_t upload(PoolBuf<T> &buf, const T *src, size_t count, cudaStream_t st, int device) {
  cudaError_t e = buf.alloc(count, st, device);
  if (e == cudaSuccess && count > 0) {
    e = cudaMemcpyAsync(buf.p, src, count * sizeof(T), cudaMemcpyHostToDevice, st);
  }
  return e;
}

// the device pointer of a result array (null: unallocated) to a caller's non-null slot
template <typename T> void hand_out(const T **dst, const PoolBuf<T> &buf) {
  if (dst != nullptr) {
    *dst = buf.p;
  }
}

// kmp_*_destroy of a result object: its arrays free themselves on its device's pool
template <typename T> void destroy_result(T *g) {
  if (g == nullptr) {
    return;
  }
  cudaSetDevice(g->device);
  delete g;
}

// The buffer protocol of the *_report_message calls: the message is formatted into buf (a null or zero-size buffer
// formats into a one-byte dummy), and its full length is returned
template <typename... A> int format_report(char *buf, size_t size, const char *fmt, A... args) {
  char dummy = 0;
  if (buf == nullptr || size == 0) {
    buf = &dummy;
    size = 1;
  }
  return std::snprintf(buf, size, fmt, args...);
}

// The overlay's state on the handle (kmp_overlay.cuh): the stashed clusterings of the last overlay call (pool blocks,
// kept between calls) and the sort's values
struct OverlayState {
  std::vector<PoolBuf<uint32_t>> stash;
  DevBuf<uint32_t> vals_a, vals_b;
};

// What one LP run (a clustering or a refinement) passes to its sweeps and commits.
struct RunCtx {
  int mode;
  uint32_t num_labels;
  int32_t max_cluster_weight;
  bool has_min;
  bool has_comm;
};
} // namespace

// The CSR arrays of a graph result (kmp_metis_graph, kmp_parhip_graph, kmp_prepared_graph, kmp_coarse_graph) on
// `device`'s pool; vwgt / adjwgt are unallocated for unit weights.
struct DeviceCsr {
  int device = 0;
  PoolBuf<uint32_t> xadj, adjncy;
  PoolBuf<int32_t> vwgt, adjwgt;

  DeviceCsr() = default;
  DeviceCsr(DeviceCsr &&) = default;
  DeviceCsr &operator=(DeviceCsr &&) = default;
  // always inlined into the result types' destructors: an out-of-line instance of one of those would be a new
  // exported symbol of the library
  [[gnu::always_inline]] ~DeviceCsr() = default;
};

namespace {
// D2H copy of the arrays of g the caller asks for: xadj_len entries of xadj, n of vwgt and m of adjncy / adjwgt
int download_csr(const DeviceCsr &g, uint32_t *x, uint32_t *a, int32_t *vw, int32_t *aw, size_t xadj_len, size_t n,
                 size_t m) {
  KMP_CUDA(cudaSetDevice(g.device));
  KMP_CUDA(copy_out(x, g.xadj, xadj_len));
  KMP_CUDA(copy_out(a, g.adjncy, m));
  KMP_CUDA(copy_out(vw, g.vwgt, n));
  KMP_CUDA(copy_out(aw, g.adjwgt, m));
  return KMP_OK;
}
void hand_out_csr(const DeviceCsr &g, const uint32_t **x, const uint32_t **a, const int32_t **vw, const int32_t **aw) {
  hand_out(x, g.xadj);
  hand_out(a, g.adjncy);
  hand_out(vw, g.vwgt);
  hand_out(aw, g.adjwgt);
}
} // namespace

// The handle's buffers are grouped by owner. kmp_lp_free_scratch resets the groups marked "released" (the next call
// that needs a grow-only buffer allocates it again); it keeps the groups marked "kept" and everything outside the
// groups, the call counters included.
struct kmp_lp_handle {
  kmp_lp_config cfg{};
  int device = 0;
  cudaStream_t stream = nullptr;       // stream all work is issued on
  // The kernel tiers of one sub-round of degree group 3 are independent of each other: they are launched on
  // side streams (fork / join by events) so that their tails and latency-bound phases overlap.
  cudaStream_t sweep_stream = nullptr; // stream the running sweep launch goes to
  // the streams and events this handle created, destroyed with it
  struct Streams {
    cudaStream_t owned = nullptr; // the handle's stream unless kmp_lp_set_stream replaced it
    cudaStream_t side[3] = {nullptr, nullptr, nullptr};
    cudaEvent_t ev_fork = nullptr, ev_join[3] = {nullptr, nullptr, nullptr};
    cudaEvent_t ev_begin = nullptr, ev_end = nullptr;
    cudaEvent_t ev_ct0 = nullptr, ev_ct1 = nullptr; // graph-operation timing (call_clock_start), created on first use
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> sweep_events; // timing mode (timed_begin), created on first use
    std::vector<int> sweep_event_group;
    Streams() = default;
    Streams(const Streams &) = delete;
    Streams &operator=(const Streams &) = delete;
    ~Streams() {
      for (cudaEvent_t e : {ev_fork, ev_join[0], ev_join[1], ev_join[2], ev_begin, ev_end, ev_ct0, ev_ct1}) {
        if (e != nullptr) {
          cudaEventDestroy(e);
        }
      }
      for (auto &p : sweep_events) {
        cudaEventDestroy(p.first);
        cudaEventDestroy(p.second);
      }
      for (cudaStream_t s : {side[0], side[1], side[2], owned}) {
        if (s != nullptr) {
          cudaStreamDestroy(s);
        }
      }
    }
  } streams;
  bool timing = false;
  uint32_t grid_cap = 0;        // KMP_GRID_CAP: most CTAs of any launch inside an LP round (0: no cap)
  bool force_p64 = false;
  uint64_t hub_wave_slots = 1ull << 28; // 2 GiB of packed entries (KMP_HUB_WAVE_SLOTS overrides, for experiments)
  uint32_t hub_bucket_cap = kBucketCap, hub_sel_limit = 0; // KMP_HUB_BUCKET_CAP / KMP_HUB_SEL_LIMIT (tests: force the overflow paths)
  // cooperative single-launch commit of a sub-round (lp_commit.cuh commit_cluster_fused / commit_refine_fused)
  DevBuf<unsigned> grid_bar; // [0] arrivals, [1] generation
  int fused_blocks = 0;      // co-resident CTAs of the clusterer's kernel
  int fused_blocks_refine = 0; // of the refiner's kernel with its largest dynamic shared memory
  // co-resident CTAs of the persistent kernels of degree groups 0 and 1 (lp_lowgroup.cuh), [group][EW][P64]
  uint32_t low_blocks[2][2][2] = {};
  // resident CTAs of each sweep_team instantiation on the device, [MODE][EW][P64][team size 32 / 128 / 512 / 1024]:
  // a larger grid only adds CTAs that start after the work queue is drained
  uint32_t team_grid[2][2][2][4] = {};

  uint32_t call_counter = 0; // clusterings computed on this handle: the sync schedule's call index
  // overload and underload balancers (kmp_balance.cuh, kmp_underload.cuh): one call counter each, so that LP calls
  // and either balancer hash the same with or without the other
  uint32_t bal_calls = 0, ubal_calls = 0;

  // per-call counters of kmp_lp_stats, reset by begin_call
  struct CallCounters {
    uint64_t kernel_launches = 0, sweep_launches = 0;
    uint32_t pull_rounds = 0, push_rounds = 0;
    size_t sweep_events_used = 0;
    uint64_t group_launches[kStatTiers] = {};
  } counts;

  // the graph: the caller's device arrays or the handle's own copies (own_*); kept
  struct Graph {
    uint32_t n = 0, m = 0;
    const uint32_t *xadj = nullptr;
    const uint32_t *adjncy = nullptr;
    const int32_t *vwgt = nullptr;
    const int32_t *adjwgt = nullptr;
    bool adjncy_16b = true; // adjncy starts on a 16-byte boundary: the hub tier may stage it with bulk copies
    DevBuf<uint32_t> own_xadj, own_adjncy;
    DevBuf<int32_t> own_vwgt, own_adjwgt;
    bool present = false;
    uint64_t epoch = 0; // counts set_graph calls: a kmp_subgraphs knows which graph it was extracted from
    uint32_t max_degree = 0;
    uint32_t num_isolated = 0;
    bool sorted = false; // CSRGraph::sorted() of the current graph (kmp_lp_set_graph_sorted)
  } graph;

  // the graph's work lists (ensure_lists): order[] holds the vertices of (group g, sub-round s) contiguously; kept
  struct WorkLists {
    DevBuf<uint32_t> order;
    std::vector<uint32_t> off; // kNumGroups*S + 1 (+1 tail bucket for unvisited vertices)
    DevBuf<uint32_t> queue;    // work-queue cursors of the team kernels: [tier][sub-round], zeroed per round
    uint32_t max_list = 0;
    uint32_t mover_cap = 0;
    uint32_t visited_total = 0; // vertices on the work lists
    bool stamps_ok = false;     // 4 * S sub-rounds fit the stamp code (else push activation only)
    // the sync_subrounds, sync_granule_log2, large_degree_threshold and seed they were built for
    uint32_t S = 0, G = 0, thr = 0;
    int seed = 0;
    bool valid = false;
  } lists;

  // temporaries of ensure_lists: the list-key sort and the hub degrees; released
  struct ListScratch {
    DevBuf<uint8_t> sort_keys_in, sort_keys_out;
    DevBuf<uint32_t> sort_vals_in;
    DevBuf<uint32_t> hub_deg, hub_beg, hub_ids;
  } list_tmp;

  // hub tier metadata of the work lists (build_hub_meta): per list entry its first bucket (wave-relative), the
  // (entry, chunk) work items of the scatter pass and the (entry, bucket) items of the select pass; all per sub-round.
  // Kept.
  struct HubMeta {
    DevBuf<uint32_t> hit; // per list entry "a neighbour moved since the last visit"
    DevBuf<uint32_t> table_off, item_entry, item_chunk, sel_entry, sel_piece, sel_begin;
    DevBuf<uint32_t> item_u, item_beg, item_deg; // static per item: vertex, xadj[u], degree
    std::vector<uint32_t> item_off, sel_off;     // S + 1
    // A sub-round's hubs are processed in waves whose bucket regions together stay below hub_wave_slots entries
    // (a memory bound: every wave reuses the same regions, cursors and overflow list).
    struct Wave {
      uint32_t item_lo, item_hi, sel_lo, sel_hi; // absolute ranges in the item_* / sel_* arrays
    };
    std::vector<Wave> waves;
    std::vector<uint32_t> wave_off; // S + 1
    DevBuf<Cand> part_best, part_fav;
    uint64_t max_slots = 0;
    uint64_t max_wave_edges = 0; // largest adjacency volume of a wave = capacity of the overflow list
    // clusterer hub path (gather + rate): per list entry the start of its row in hub_tmp.lab (sub-round-relative) and
    // its first rate item result; the (entry, hash class) rate items of each sub-round, largest degree first
    DevBuf<uint32_t> lab_off, rate_begin, rate_entry, rate_cls;
    // unit edge weights: per list entry the start of its chunks' class offsets in hub_tmp.cls (sub-round-relative)
    DevBuf<uint32_t> cls_off;
    uint64_t max_subround_cls = 0;
    std::vector<uint32_t> rate_off; // S + 1
    uint64_t max_subround_edges = 0;
  } hub;

  // hub tier scratch of the running sub-round; released
  struct HubScratch {
    DevBuf<unsigned long long> tab; // bucket regions: kBucketCap packed (key << 32 | rating) entries each
    DevBuf<uint32_t> cursor;        // per bucket: entries appended in the running sub-round
    DevBuf<HubOverflow> ovf;
    DevBuf<uint16_t> cls; // class offsets of the running sub-round's staged chunks (hub_sort_classes + 1 each)
    DevBuf<uint32_t> lab; // staged neighbour labels of the running sub-round's hubs (4 B per edge)
  } hub_tmp;

  // LP labels and weights; released
  struct LpState {
    DevBuf<uint32_t> label, favored, communities;
    // label[] belongs to the current graph: set by a completed clustering, kmp_lp_upload_partition and a refine or
    // balancer call given a partition; cleared by a new graph and by kmp_lp_free_scratch. The calls that read the
    // labels on the device (a NULL partition or clustering) refuse while it is clear.
    bool labels_valid = false;
    DevBuf<int32_t> weight, maxw, minw;
    DevBuf<uint8_t> active;
    // packed (label, stamp) gather array of the sweeps (lp_device.cuh): 4 B per vertex while labels fit 24 bits
    // (n <= 2^24 clusterer / k <= 2^24 refiner), else 8 B (round.p64)
    DevBuf<unsigned char> labg;
  } lp;

  // LP commit scratch, and the temporary storage of every CUB call (cub_call); released
  struct CommitScratch {
    DevBuf<uint32_t> mv_u, mv_t, cslot, slotmap;
    DevBuf<uint8_t> acc;
    DevBuf<int32_t> incoming, chist, hist, jmin, out_cur, out_delta, ohist, ojmin;
    DevBuf<uint32_t> ctr32; // [0] mover_count [1] moved_count (per iteration) [2] misc
    DevBuf<unsigned long long> ctr64; // [0] edges [1] nodes [2] proposals
    DevBuf<unsigned char> cub_tmp;
    bool slot_state_clean = false; // incoming/slotmap/chist zeroed for current n
  } commit;

  // the running LP round; kept
  struct Round {
    bool p64 = false;
    bool pull_this = true, pull_next = true; // activation mode of the running / the next LP round
    uint32_t moved_hist[2] = {0xFFFFFFFFu, 0xFFFFFFFFu}; // accepted moves of the two previous rounds
    uint32_t cur_subround = 0; // hashed class of the running sub-round
    uint32_t cur_sg = 0;       // running sub-round index in [0, 4 * S): queue cursor and stamp code
    uint32_t mover_parity = 0; // proposal counter in use: ctr32[0] (parity 0) or ctr32[3] (parity 1)
    bool stepping = false; // proposals are accumulated by kmp_lp_step_commit, not by the sweep kernels
  } round;

  // scratch of the graph operations (contraction, sparsification, overlay; pairs_a/b also the two-hop sort); released
  struct OpScratch {
    DevBuf<unsigned long long> pairs_a, pairs_b; // two-hop sort; contraction: edge keys (double buffer)
    DevBuf<int32_t> ct_vals_a, ct_vals_b; // contraction (kmp_contract.cuh)
    DevBuf<uint32_t> ct_flags, ct_rank, ct_cl;
    DevBuf<unsigned long long> ct_counter;
    DevBuf<uint32_t> sp_ctl; // sparsification (kmp_sparsify.cuh): radix-select bins, select state, kept counter
    OverlayState ov;         // set_graph releases its stash, which belongs to the previous graph
  } ops;

  // scratch of both balancers (kmp_balance.cuh, kmp_underload.cuh); released
  struct BalScratch {
    DevBuf<uint32_t> cand, under, ctr32, target, lists, sv_a, sv_b, blk;
    // over[b]: the quota a block's segment of sorted candidates is selected against (overload of b, or the
    // underload balancer's deficit of target b)
    DevBuf<int32_t> over, pbw, wt, prefix;
    DevBuf<uint8_t> flag, tmask; // tmask: the underload balancer's allowed targets
    DevBuf<float> key;
    // ctrl: [0] total over- / underload [1] candidates [2] |U| (underloaded blocks) [3] bad labels [4] edges
    //       [5] candidates with a target
    // ctr32: [0] movers [1] scratch [2..3] tier counts [4 + r] moved in round r
    DevBuf<unsigned long long> ctrl, sk_a, sk_b;
  } bal;

  // schedule KMP_SCHEDULE_SEQ_STRICT (lp_strict.cuh): sequential engine state and its per-object RNG; kept
  struct Strict {
    bool seeded = false;
    DevBuf<int32_t> slot, ent_val, slot2, ent2_val, concurrent;
    DevBuf<uint32_t> ent_key, ent2_key, used, second, tie_best, tie_fav, chunks, sub_perm, match, buckets;
    DevBuf<kmp_strict::Rng> rng;
    DevBuf<kmp_strict::Stats> stats;
  } strict;

  // frontier sharding (one process per GPU): this rank sweeps slice `rank` of `world` of every list. The NCCL
  // communicator of the sharded run (kmp_lp_dist_init) all-gathers the proposals per sub-round on the handle's
  // stream, inside kmp_lp_cluster / kmp_lp_refine. Kept.
  struct Dist {
    uint32_t rank = 0, world = 1;
    ncclComm_t comm = nullptr;
    DevBuf<uint32_t> send, recv;
    uint32_t *direct_send = nullptr; // set while the sweeps of a sharded sub-round write into the send buffer
    uint32_t direct_cap = 0;
  } dist;

  // stepping API: the open run (between kmp_lp_step_begin_* and kmp_lp_step_finish) and its LP round
  struct Stepping {
    RunCtx run{};
    bool open = false;
    uint32_t iter = 0;
  } step;
};

namespace {

// A CUB device-wide call in its two phases: call(nullptr, bytes) asks for the temporary storage, call(tmp, bytes) runs
// on h->commit.cub_tmp grown to it (CUB never asks for 0 bytes, so tmp is never null and the second call is never a query).
template <typename Fn> cudaError_t cub_call(kmp_lp_handle *h, Fn &&call) {
  size_t bytes = 0;
  cudaError_t e = call(static_cast<void *>(nullptr), bytes);
  if (e == cudaSuccess) {
    e = h->commit.cub_tmp.ensure(bytes);
  }
  return e != cudaSuccess ? e : call(static_cast<void *>(h->commit.cub_tmp.p), bytes);
}

// Device time of one graph-operation call (contraction, sparsification, overlay, preparation, subgraph extraction) on
// the handle's event pair ev_ct0 / ev_ct1, created on first use. None of these calls runs inside another, and the pair
// is not ev_begin / ev_end, which may bracket an open stepping call.
cudaError_t call_clock_start(kmp_lp_handle *h, cudaStream_t st) {
  if (h->streams.ev_ct0 == nullptr) {
    cudaError_t e = cudaEventCreate(&h->streams.ev_ct0);
    if (e == cudaSuccess) {
      e = cudaEventCreate(&h->streams.ev_ct1);
    }
    if (e != cudaSuccess) {
      return e;
    }
  }
  return cudaEventRecord(h->streams.ev_ct0, st);
}
cudaError_t call_clock_stop(kmp_lp_handle *h, cudaStream_t st) { return cudaEventRecord(h->streams.ev_ct1, st); }
// after the caller has waited for the stop event (on the event or on its stream)
float call_clock_ms(const kmp_lp_handle *h) {
  float ms = 0.f;
  cudaEventElapsedTime(&ms, h->streams.ev_ct0, h->streams.ev_ct1);
  return ms;
}

// A new result object T of a call on h (kmp_coarse_graph, kmp_prepared_graph, kmp_subgraphs), filled by impl(obj) and
// handed to *out only if impl succeeds. A refused call leaves *out untouched and frees what impl allocated; obj->device
// is set before impl allocates anything.
template <typename T, typename Impl> int make_result(const kmp_lp_handle *h, T **out, Impl &&impl) {
  std::unique_ptr<T> obj(new (std::nothrow) T());
  if (obj == nullptr) {
    return fail(KMP_ERR_ALLOC, "out of host memory");
  }
  obj->device = h->device;
  const int rc = impl(obj.get());
  if (rc == KMP_OK) {
    *out = obj.release();
  }
  return rc;
}
} // namespace

namespace kmp {
// block weights from labels; counts labels >= k (a clustering is not a partition) into *bad. The one range check
// of the refiner and both balancers (checked_block_weights). Warp-aggregated: the lanes of a warp that share a block
// add their weights first and one lane issues the atomic, so that with few blocks (k = 2 on 10^7 vertices) the
// atomics do not serialise on a handful of addresses. Integer sums: the result is the per-vertex atomics' result.
// blockDim.x must be a multiple of 32 (the loop bound is warp-uniform).
__global__ void bal_block_weights(uint32_t n, uint32_t k, const int32_t *vwgt, const uint32_t *label, int32_t *weight,
                                  unsigned long long *bad) {
  const uint32_t lane = threadIdx.x & 31;
  for (uint32_t base = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < n; base += gridDim.x * blockDim.x) {
    const uint32_t u = base + lane;
    const bool live = u < n;
    const uint32_t b = live ? label[u] : 0xFFFFFFFFu;
    const bool ok = live && b < k;
    const int32_t w = ok ? (vwgt != nullptr ? vwgt[u] : 1) : 0;
    const unsigned out_of_range = __ballot_sync(kFull, live && !ok);
    if (lane == 0 && out_of_range != 0) {
      atomicAdd(bad, static_cast<unsigned long long>(__popc(out_of_range)));
    }
    const unsigned peers = __match_any_sync(kFull, ok ? b : 0xFFFFFFFFu);
    int32_t sum = 0;
    for (int j = 0; j < 32; ++j) {
      const int32_t x = __shfl_sync(kFull, w, j);
      sum += ((peers >> j) & 1u) ? x : 0;
    }
    if (ok && lane == static_cast<uint32_t>(__ffs(peers) - 1)) {
      atomicAdd(&weight[b], sum);
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
  bool ok = configure_team<MODE, EW, P64, 32, 512, 8, !EW>(h, sms) && configure_team<MODE, EW, P64, 128, 2048, 4, !EW>(h, sms) &&
            configure_team<MODE, EW, P64, 512, 8192, 1, !EW>(h, sms);
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
  case 4: // deg < 1024: 128 threads per vertex, 2048 slots; 16-bit ratings with unit edge weights
    launch_team<MODE, EW, P64, 128, 2048, 4, !EW>(h, a);
    break;
  case 5: // deg < 4096: 512 threads per vertex, 8192 slots; 16-bit ratings with unit edge weights
    launch_team<MODE, EW, P64, 512, 8192, 1, !EW>(h, a);
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
    const uint32_t s_idx = h->round.cur_subround;
    const uint32_t S = h->lists.S;
    const uint32_t first = h->lists.off[kHubTier * S + s_idx] - h->lists.off[kHubTier * S];
    hb.sel_limit = h->hub_sel_limit;
    hb.rank = h->dist.rank;
    hb.world = h->dist.world;
    hb.hit = h->hub.hit.p + first;
    if constexpr (MODE == 0) {
      // gather the labels of the sub-round's hub edges once, then rate every (hub, hash class) item in one CTA
      const uint32_t ilo = h->hub.item_off[s_idx], ihi = h->hub.item_off[s_idx + 1];
      hb.item_entry = h->hub.item_entry.p + ilo;
      hb.item_chunk = h->hub.item_chunk.p + ilo;
      hb.item_u = h->hub.item_u.p + ilo;
      hb.item_beg = h->hub.item_beg.p + ilo;
      hb.item_deg = h->hub.item_deg.p + ilo;
      hb.num_items = ihi - ilo;
      hb.lab = h->hub_tmp.lab.p;
      hb.lab_off = h->hub.lab_off.p + first;
      if constexpr (!EW) {
        hb.cls = h->hub_tmp.cls.p;
        hb.cls_off = h->hub.cls_off.p + first;
      }
      sweep_hub_gather<P64><<<capped(h, std::min<uint32_t>(hb.num_items, kSMs * 8)), 256, 0, h->sweep_stream>>>(a, hb);
      const uint32_t rlo = h->hub.rate_off[s_idx], rhi = h->hub.rate_off[s_idx + 1];
      hb.item_entry = h->hub.rate_entry.p + rlo;
      hb.item_cls = h->hub.rate_cls.p + rlo;
      hb.num_items = rhi - rlo;
      hb.sel_begin = h->hub.rate_begin.p + first;
      hb.part_best = h->hub.part_best.p;
      hb.part_fav = h->hub.part_fav.p;
      hb.queue = h->commit.ctr32.p + 64 + s_idx; // zeroed with the other per-round counters
      sweep_hub_rate<EW><<<capped(h, std::min<uint32_t>(hb.num_items, kSMs)), kRateThreads, rate_smem<EW>(), h->sweep_stream>>>(a, hb);
      h->counts.kernel_launches += 2;
    } else {
      hb.table_off = h->hub.table_off.p + first;
      hb.g_tab = h->hub_tmp.tab.p;
      hb.cursor = h->hub_tmp.cursor.p;
      hb.ovf = h->hub_tmp.ovf.p;
      hb.ovf_cap = static_cast<uint32_t>(std::min<uint64_t>(h->hub.max_wave_edges, 0xFFFFFFFFull));
      hb.bucket_cap = h->hub_bucket_cap;
      hb.stage_adjncy = h->graph.adjncy_16b ? 1u : 0u;
      hb.sel_begin = h->hub.sel_begin.p + first;
      // one scatter + select pair per wave; all waves share the bucket memory (cursors reset by the select)
      for (uint32_t w = h->hub.wave_off[s_idx]; w < h->hub.wave_off[s_idx + 1]; ++w) {
        const kmp_lp_handle::HubMeta::Wave &wv = h->hub.waves[w];
        hb.item_entry = h->hub.item_entry.p + wv.item_lo;
        hb.item_chunk = h->hub.item_chunk.p + wv.item_lo;
        hb.item_u = h->hub.item_u.p + wv.item_lo;
        hb.item_beg = h->hub.item_beg.p + wv.item_lo;
        hb.item_deg = h->hub.item_deg.p + wv.item_lo;
        hb.num_items = wv.item_hi - wv.item_lo;
        hb.queue = h->commit.ctr32.p + 64 + w; // zeroed with the other per-round counters
        hb.ovf_count = h->commit.ctr32.p + 512 + w;
        sweep_hub_scatter<MODE, EW, P64><<<capped(h, std::min<uint32_t>(hb.num_items, kSMs * 4)), kHubThreads, kHubScatterSmem, h->sweep_stream>>>(a, hb, h->graph.m);
        hb.sel_entry = h->hub.sel_entry.p + wv.sel_lo;
        hb.sel_piece = h->hub.sel_piece.p + wv.sel_lo;
        hb.num_sel_items = wv.sel_hi - wv.sel_lo;
        hb.part_best = h->hub.part_best.p + (wv.sel_lo - h->hub.sel_off[s_idx]);
        hb.part_fav = h->hub.part_fav.p + (wv.sel_lo - h->hub.sel_off[s_idx]);
        sweep_hub_select<MODE><<<capped(h, std::min<uint32_t>((hb.num_sel_items + kSelWarps - 1) / kSelWarps, kSMs * 6)), kSelWarps * 32, 0, h->sweep_stream>>>(a, hb);
        h->counts.kernel_launches += 2;
      }
    }
    hb.part_best = h->hub.part_best.p;
    hb.part_fav = h->hub.part_fav.p;
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
  if (h->counts.sweep_events_used == h->streams.sweep_events.size()) {
    cudaEvent_t x, y;
    cudaEventCreate(&x);
    cudaEventCreate(&y);
    h->streams.sweep_events.emplace_back(x, y);
    h->streams.sweep_event_group.push_back(0);
  }
  const int idx = static_cast<int>(h->counts.sweep_events_used++);
  h->streams.sweep_event_group[idx] = tag;
  cudaEventRecord(h->streams.sweep_events[idx].first, st);
  return idx;
}
void timed_end(kmp_lp_handle *h, int idx, cudaStream_t st = nullptr) {
  if (idx >= 0) {
    cudaEventRecord(h->streams.sweep_events[idx].second, st == nullptr ? h->stream : st);
  }
}

// tier: kernel tier 0..kNumTiers-1 of the list in `a_in`
cudaError_t launch_sweep(kmp_lp_handle *h, int mode, int tier, const SweepArgs &a_in) {
  if (a_in.list_size == 0) {
    return cudaSuccess;
  }
  SweepArgs a = a_in;
  a.counters = h->commit.ctr64.p + tier;
  a.queue = h->lists.queue.p + static_cast<size_t>(tier) * kNumGroups * h->lists.S + h->round.cur_sg;
  if (h->sweep_stream == nullptr) {
    h->sweep_stream = h->stream;
  }
  const int ev = timed_begin(h, tier, h->sweep_stream);
  const bool ew = h->graph.adjwgt != nullptr;
  const int variant = (mode << 2) | (ew ? 2 : 0) | (h->round.p64 ? 1 : 0);
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
  ++h->counts.kernel_launches;
  ++h->counts.sweep_launches;
  ++h->counts.group_launches[tier];
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

// The hub tier metadata of the work lists just built with S sub-rounds (kmp_lp_handle::HubMeta): bucket regions, chunk
// work items and (entry, bucket) selection items per sub-round.
int build_hub_meta(kmp_lp_handle *h, uint32_t S) {
  const uint32_t hub_begin = h->lists.off[kHubTier * S], hub_end = h->lists.off[(kHubTier + 1) * S];
  const uint32_t hub_cnt = hub_end - hub_begin;
  h->hub.item_off.assign(S + 1, 0);
  h->hub.wave_off.assign(S + 1, 0);
  h->hub.waves.clear();
  h->hub.max_slots = 0;
  h->hub.max_wave_edges = 0;
  h->hub.max_subround_edges = 0;
  h->hub.max_subround_cls = 0;
  if (hub_cnt > 0) {
    DevBuf<uint32_t> &d_deg = h->list_tmp.hub_deg, &d_beg = h->list_tmp.hub_beg, &d_ids = h->list_tmp.hub_ids; // grow-only
    KMP_CUDA(d_deg.ensure(hub_cnt));
    KMP_CUDA(d_beg.ensure(hub_cnt));
    KMP_CUDA(d_ids.ensure(hub_cnt));
    k_gather_degrees<<<grid_for(hub_cnt, 256), 256, 0, h->stream>>>(hub_cnt, h->lists.order.p + hub_begin, h->graph.xadj, d_deg.p,
                                                                    d_beg.p, d_ids.p);
    std::vector<uint32_t> vbeg(hub_cnt), vids(hub_cnt), iu, ibeg, ideg;
    KMP_CUDA(cudaMemcpyAsync(vbeg.data(), d_beg.p, hub_cnt * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
    KMP_CUDA(cudaMemcpyAsync(vids.data(), d_ids.p, hub_cnt * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
    std::vector<uint32_t> deg(hub_cnt), toff(hub_cnt), sbeg(hub_cnt), ient, ichk, sent, spiece;
    h->hub.sel_off.assign(S + 1, 0);
    size_t max_sel = 0;
    KMP_CUDA(cudaMemcpyAsync(deg.data(), d_deg.p, hub_cnt * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
    KMP_CUDA(cudaStreamSynchronize(h->stream));
    // at most kMaxHubWaves work-queue cursors exist per LP round: coarsen the waves if necessary
    // (the degrees must be on the host before this sum -- ADVICE r1)
    uint64_t wave_slots = h->hub_wave_slots;
    {
      uint64_t total = 0;
      for (uint32_t i = 0; i < hub_cnt; ++i) {
        total += static_cast<uint64_t>(hub_buckets(deg[i])) * kBucketCap;
      }
      wave_slots = std::max<uint64_t>(wave_slots, total / (kMaxHubWaves / 2 - S) + 1);
    }
    for (uint32_t sr = 0; sr < S; ++sr) {
      const uint32_t lo = h->lists.off[kHubTier * S + sr] - hub_begin, hi = h->lists.off[kHubTier * S + sr + 1] - hub_begin;
      uint64_t slots = 0, wave_edges = 0;
      kmp_lp_handle::HubMeta::Wave wave{static_cast<uint32_t>(ient.size()), 0, static_cast<uint32_t>(sent.size()), 0};
      auto close_wave = [&]() {
        wave.item_hi = static_cast<uint32_t>(ient.size());
        wave.sel_hi = static_cast<uint32_t>(sent.size());
        if (wave.item_hi > wave.item_lo) {
          h->hub.waves.push_back(wave);
        }
        wave.item_lo = wave.item_hi;
        wave.sel_lo = wave.sel_hi;
        h->hub.max_slots = std::max(h->hub.max_slots, slots);
        h->hub.max_wave_edges = std::max(h->hub.max_wave_edges, wave_edges);
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
        sbeg[i] = static_cast<uint32_t>(sent.size() - h->hub.sel_off[sr]);
        for (uint32_t c = 0; c < buckets; ++c) { // one selection item per bucket
          sent.push_back(i - lo);
          spiece.push_back(c);
        }
      }
      close_wave();
      h->hub.wave_off[sr + 1] = static_cast<uint32_t>(h->hub.waves.size());
      h->hub.sel_off[sr + 1] = static_cast<uint32_t>(sent.size());
      max_sel = std::max<size_t>(max_sel, sent.size() - h->hub.sel_off[sr]);
      h->hub.item_off[sr + 1] = static_cast<uint32_t>(ient.size());
    }
    if (h->hub.waves.size() > kMaxHubWaves) {
      return fail(KMP_ERR_UNSUPPORTED, "too many high-degree table waves (raise KMP_HUB_WAVE_SLOTS)");
    }
    // clusterer: per entry its row in the staged labels and its first result slot, and the (entry, hash class)
    // rate items of every sub-round, largest degree first (the longest items start first)
    std::vector<uint32_t> loff(hub_cnt), coff(hub_cnt), rbeg(hub_cnt), rent, rcls, ord;
    h->hub.rate_off.assign(S + 1, 0);
    size_t max_rate = 0;
    for (uint32_t sr = 0; sr < S; ++sr) {
      const uint32_t lo = h->lists.off[kHubTier * S + sr] - hub_begin, hi = h->lists.off[kHubTier * S + sr + 1] - hub_begin;
      // edges <= m < 2^32; cls <= (m / 2048 + hubs) * 257 < 2^31 (hubs <= m / 8192)
      uint64_t edges = 0, cls = 0;
      uint32_t res = 0;
      ord.clear();
      for (uint32_t i = lo; i < hi; ++i) {
        loff[i] = static_cast<uint32_t>(edges);
        edges += deg[i];
        coff[i] = static_cast<uint32_t>(cls);
        if (h->graph.adjwgt == nullptr) {
          cls += static_cast<uint64_t>((deg[i] + kChunkEdges - 1) / kChunkEdges) * (hub_sort_classes(deg[i]) + 1);
        }
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
      h->hub.rate_off[sr + 1] = static_cast<uint32_t>(rent.size());
      max_rate = std::max<size_t>(max_rate, res);
      h->hub.max_subround_edges = std::max(h->hub.max_subround_edges, edges);
      h->hub.max_subround_cls = std::max(h->hub.max_subround_cls, cls);
    }
    max_sel = std::max(max_sel, max_rate);
    KMP_CUDA(h->hub.lab_off.ensure(hub_cnt));
    KMP_CUDA(h->hub.rate_begin.ensure(hub_cnt));
    KMP_CUDA(h->hub.rate_entry.ensure(rent.size()));
    KMP_CUDA(h->hub.rate_cls.ensure(rcls.size()));
    KMP_CUDA(cudaMemcpyAsync(h->hub.lab_off.p, loff.data(), hub_cnt * 4, cudaMemcpyHostToDevice, h->stream));
    KMP_CUDA(h->hub.cls_off.ensure(hub_cnt));
    KMP_CUDA(cudaMemcpyAsync(h->hub.cls_off.p, coff.data(), hub_cnt * 4, cudaMemcpyHostToDevice, h->stream));
    KMP_CUDA(cudaMemcpyAsync(h->hub.rate_begin.p, rbeg.data(), hub_cnt * 4, cudaMemcpyHostToDevice, h->stream));
    KMP_CUDA(cudaMemcpyAsync(h->hub.rate_entry.p, rent.data(), rent.size() * 4, cudaMemcpyHostToDevice, h->stream));
    KMP_CUDA(cudaMemcpyAsync(h->hub.rate_cls.p, rcls.data(), rcls.size() * 4, cudaMemcpyHostToDevice, h->stream));
    KMP_CUDA(h->hub.table_off.ensure(hub_cnt));
    KMP_CUDA(h->hub.hit.ensure(hub_cnt));
    KMP_CUDA(cudaMemsetAsync(h->hub.hit.p, 0, static_cast<size_t>(hub_cnt) * 4, h->stream));
    KMP_CUDA(h->hub.item_entry.ensure(ient.size()));
    KMP_CUDA(h->hub.item_chunk.ensure(ichk.size()));
    KMP_CUDA(cudaMemcpyAsync(h->hub.table_off.p, toff.data(), hub_cnt * 4, cudaMemcpyHostToDevice, h->stream));
    KMP_CUDA(cudaMemcpyAsync(h->hub.item_entry.p, ient.data(), ient.size() * 4, cudaMemcpyHostToDevice, h->stream));
    KMP_CUDA(cudaMemcpyAsync(h->hub.item_chunk.p, ichk.data(), ichk.size() * 4, cudaMemcpyHostToDevice, h->stream));
    KMP_CUDA(h->hub.item_u.ensure(iu.size()));
    KMP_CUDA(h->hub.item_beg.ensure(iu.size()));
    KMP_CUDA(h->hub.item_deg.ensure(iu.size()));
    KMP_CUDA(cudaMemcpyAsync(h->hub.item_u.p, iu.data(), iu.size() * 4, cudaMemcpyHostToDevice, h->stream));
    KMP_CUDA(cudaMemcpyAsync(h->hub.item_beg.p, ibeg.data(), iu.size() * 4, cudaMemcpyHostToDevice, h->stream));
    KMP_CUDA(cudaMemcpyAsync(h->hub.item_deg.p, ideg.data(), iu.size() * 4, cudaMemcpyHostToDevice, h->stream));
    KMP_CUDA(h->hub.sel_entry.ensure(sent.size()));
    KMP_CUDA(h->hub.sel_piece.ensure(spiece.size()));
    KMP_CUDA(h->hub.sel_begin.ensure(hub_cnt));
    KMP_CUDA(h->hub.part_best.ensure(max_sel));
    KMP_CUDA(h->hub.part_fav.ensure(max_sel));
    KMP_CUDA(cudaMemcpyAsync(h->hub.sel_entry.p, sent.data(), sent.size() * 4, cudaMemcpyHostToDevice, h->stream));
    KMP_CUDA(cudaMemcpyAsync(h->hub.sel_piece.p, spiece.data(), spiece.size() * 4, cudaMemcpyHostToDevice, h->stream));
    KMP_CUDA(cudaMemcpyAsync(h->hub.sel_begin.p, sbeg.data(), hub_cnt * 4, cudaMemcpyHostToDevice, h->stream));
    KMP_CUDA(cudaStreamSynchronize(h->stream));
  }
  return KMP_OK;
}

int ensure_lists(kmp_lp_handle *h) {
  TraceClock tc;
  const uint32_t S = std::max<uint32_t>(1, h->cfg.sync_subrounds);
  if (h->lists.valid && h->lists.S == S && h->lists.G == h->cfg.sync_granule_log2 &&
      h->lists.thr == h->cfg.large_degree_threshold && h->lists.seed == h->cfg.seed) {
    return KMP_OK;
  }
  if (S > kMaxSubrounds) {
    return fail(KMP_ERR_INVALID, "sync_subrounds too large (max " + std::to_string(kMaxSubrounds) + ")");
  }
  h->lists.stamps_ok = kNumGroups * S <= kMaxStampSubrounds; // else: push activation only
  const uint32_t n = h->graph.n;
  const uint32_t nkeys = kNumTiers * S + 1;
  KMP_CUDA(h->list_tmp.sort_keys_in.ensure(n));
  KMP_CUDA(h->list_tmp.sort_keys_out.ensure(n));
  KMP_CUDA(h->list_tmp.sort_vals_in.ensure(n));
  KMP_CUDA(h->lists.order.ensure(n));
  KMP_CUDA(h->commit.ctr32.ensure(kCtr32Size));
  KMP_CUDA(cudaMemsetAsync(h->commit.ctr32.p, 0, kCtr32Size * sizeof(uint32_t), h->stream));
  tc.lap("lists: buffers");
  const uint32_t base_sr = sync_base(h->cfg.seed, 0, 0, SALT_SUBROUND);
  // Sub-rounds per degree group: S for a group holding >= 1/16 of the visited vertices, S/4 otherwise
  // (a small group has few same-sub-round neighbours; its launches become 4x larger). DESIGN.md §3.
  GroupSubrounds gs{};
  {
    k_group_counts<<<grid_for(n, 256), 256, 0, h->stream>>>(n, h->graph.xadj, h->cfg.large_degree_threshold, h->commit.ctr32.p);
    uint32_t cnt[4] = {0, 0, 0, 0};
    KMP_CUDA(cudaMemcpyAsync(cnt, h->commit.ctr32.p, sizeof(cnt), cudaMemcpyDeviceToHost, h->stream));
    KMP_CUDA(cudaStreamSynchronize(h->stream));
    const uint64_t visited = static_cast<uint64_t>(cnt[0]) + cnt[1] + cnt[2] + cnt[3];
    h->lists.visited_total = static_cast<uint32_t>(visited);
    for (int q = 0; q < 4; ++q) {
      gs.s[q] = (16ull * cnt[q] >= visited) ? S : std::max<uint32_t>(1, S / 4);
    }
    KMP_CUDA(cudaMemsetAsync(h->commit.ctr32.p, 0, kCtr32Size * sizeof(uint32_t), h->stream));
  }
  tc.lap("lists: group counts (sync)");
  k_list_keys<<<grid_for(n, 256), 256, 0, h->stream>>>(n, h->graph.xadj, S, gs, h->cfg.sync_granule_log2, base_sr,
                                                        h->cfg.large_degree_threshold,
                                                        h->graph.adjwgt != nullptr ? kHubMinDegree : kHubMinDegreeUnit,
                                                        h->list_tmp.sort_keys_in.p, h->list_tmp.sort_vals_in.p, h->commit.ctr32.p,
                                                        h->commit.ctr32.p + 300);
  KMP_CUDA(cudaGetLastError());
  if (n > 0) {
    KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
      return cub::DeviceRadixSort::SortPairs(tmp, bytes, h->list_tmp.sort_keys_in.p, h->list_tmp.sort_keys_out.p,
                                             h->list_tmp.sort_vals_in.p, h->lists.order.p, static_cast<int>(n), 0, 8,
                                             h->stream);
    }));
  }
  std::vector<uint32_t> hist(512);
  KMP_CUDA(cudaMemcpyAsync(hist.data(), h->commit.ctr32.p, 512 * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
  KMP_CUDA(cudaStreamSynchronize(h->stream));
  tc.lap("lists: keys + sort (sync)");
  h->lists.off.assign(nkeys + 1, 0);
  for (uint32_t kx = 0; kx < nkeys; ++kx) {
    h->lists.off[kx + 1] = h->lists.off[kx] + hist[kx];
  }
  auto lsize = [&](uint32_t tier, uint32_t sr) { return hist[tier * S + sr]; };
  h->lists.max_list = 0;
  h->lists.mover_cap = 1;
  for (uint32_t sr = 0; sr < S; ++sr) {
    for (int g = 0; g < kNumGroups; ++g) { // the tiers of a degree group share a sub-round
      uint32_t tot = 0;
      for (int t = first_tier_of_group(g); t <= last_tier_of_group(g); ++t) {
        tot += lsize(static_cast<uint32_t>(t), sr);
      }
      h->lists.mover_cap = std::max(h->lists.mover_cap, tot);
    }
  }
  KMP_CUDA(h->lists.queue.ensure(static_cast<size_t>(kNumTiers) * kNumGroups * S));
  h->lists.max_list = h->lists.mover_cap;
  h->graph.max_degree = hist[300];
  const int rc = build_hub_meta(h, S);
  if (rc != KMP_OK) {
    return rc;
  }
  tc.lap("lists: hub metadata");
  h->lists.S = S;
  h->lists.G = h->cfg.sync_granule_log2;
  h->lists.thr = h->cfg.large_degree_threshold;
  h->lists.seed = h->cfg.seed;
  h->lists.valid = true;
  // the sort buffers are only needed here
  // The sort buffers stay allocated (grow-only, released by kmp_lp_free_scratch): a cudaFree / cudaMalloc pair per
  // set_graph synchronises the whole device, and waits for the graph upload in flight (scripts/e2e_probe.py).
  tc.lap("lists: done");
  return KMP_OK;
}

// scratch shared by both modes
int ensure_scratch(kmp_lp_handle *h, int mode, uint32_t num_labels) {
  const size_t cap = std::max<uint32_t>(h->lists.mover_cap, 1);
  KMP_CUDA(h->commit.mv_u.ensure(cap));
  KMP_CUDA(h->commit.mv_t.ensure(cap));
  KMP_CUDA(h->commit.acc.ensure(cap));
  KMP_CUDA(h->commit.ctr32.ensure(kCtr32Size));
  KMP_CUDA(h->commit.ctr64.ensure(kCtrSize));
  KMP_CUDA(h->lp.active.ensure(h->graph.n));
  if (mode == 0) {
    KMP_CUDA(h->commit.cslot.ensure(cap));
    const bool fresh = h->commit.incoming.cap < h->graph.n || h->commit.slotmap.cap < h->graph.n ||
                       h->commit.chist.cap < cap * kLadderLevels;
    KMP_CUDA(h->commit.incoming.ensure(h->graph.n));
    KMP_CUDA(h->commit.slotmap.ensure(h->graph.n));
    KMP_CUDA(h->commit.chist.ensure(cap * kLadderLevels));
    if (fresh || !h->commit.slot_state_clean) {
      KMP_CUDA(cudaMemsetAsync(h->commit.incoming.p, 0, h->commit.incoming.cap * sizeof(int32_t), h->stream));
      KMP_CUDA(cudaMemsetAsync(h->commit.slotmap.p, 0xFF, h->commit.slotmap.cap * sizeof(uint32_t), h->stream));
      KMP_CUDA(cudaMemsetAsync(h->commit.chist.p, 0, h->commit.chist.cap * sizeof(int32_t), h->stream));
      h->commit.slot_state_clean = true;
    }
  } else {
    const size_t kk = std::max<uint32_t>(num_labels, 1);
    KMP_CUDA(h->commit.hist.ensure(kk * kLadderLevels));
    KMP_CUDA(h->commit.ohist.ensure(kk * kLadderLevels));
    KMP_CUDA(h->commit.jmin.ensure(kk));
    KMP_CUDA(h->commit.ojmin.ensure(kk));
    KMP_CUDA(h->commit.out_cur.ensure(kk));
    KMP_CUDA(h->commit.out_delta.ensure(kk));
    KMP_CUDA(cudaMemsetAsync(h->commit.hist.p, 0, kk * kLadderLevels * sizeof(int32_t), h->stream));
    KMP_CUDA(cudaMemsetAsync(h->commit.ohist.p, 0, kk * kLadderLevels * sizeof(int32_t), h->stream));
  }
  // hub tier scratch: the clusterer stages 4 B per hub edge of the largest sub-round; the refiner has bucket
  // regions, cursors and an overflow list
  if (mode == 0 && h->hub.max_subround_edges > 0) {
    KMP_CUDA(h->hub_tmp.lab.ensure(h->hub.max_subround_edges));
    KMP_CUDA(h->hub_tmp.cls.ensure(h->hub.max_subround_cls));
  }
  if (mode == 1 && h->hub.max_slots > 0) {
    KMP_CUDA(h->hub_tmp.tab.ensure(h->hub.max_slots)); // no initialisation: the cursors say how much of a region is valid
    KMP_CUDA(h->hub_tmp.cursor.ensure(h->hub.max_slots / kBucketCap));
    KMP_CUDA(h->hub_tmp.ovf.ensure(std::max<uint64_t>(h->hub.max_wave_edges, 1)));
    KMP_CUDA(cudaGetLastError());
  }
  (void)num_labels;
  return KMP_OK;
}

SweepArgs make_sweep_args(kmp_lp_handle *h, const RunCtx &rc) {
  SweepArgs a{};
  a.xadj = h->graph.xadj;
  a.adjncy = h->graph.adjncy;
  a.vwgt = h->graph.vwgt;
  a.adjwgt = h->graph.adjwgt;
  a.label = h->lp.label.p;
  a.labg = h->lp.labg.p;
  a.pull = false;
  a.window = make_window(0, 0);
  a.queue = h->lists.queue.p;
  a.weight = h->lp.weight.p;
  a.max_w = rc.mode == 1 ? h->lp.maxw.p : nullptr;
  a.min_w = rc.has_min ? h->lp.minw.p : nullptr;
  a.communities = rc.has_comm ? h->lp.communities.p : nullptr;
  a.active = h->lp.active.p;
  a.favored = h->lp.favored.p;
  a.max_cluster_weight = rc.max_cluster_weight;
  a.num_labels = rc.num_labels;
  a.max_num_neighbors = h->cfg.max_num_neighbors;
  a.mv_u = h->commit.mv_u.p;
  a.mv_t = h->commit.mv_t.p;
  a.mover_count = h->commit.ctr32.p + (h->round.mover_parity ? 3 : 0);
  if (h->dist.direct_send != nullptr) { // sharded library path: [count, -, -, -, u[cap], t[cap]]
    a.mover_count = h->dist.direct_send;
    a.mv_u = h->dist.direct_send + 4;
    a.mv_t = h->dist.direct_send + 4 + h->dist.direct_cap;
  }
  a.incoming = h->commit.incoming.p;
  a.hist = h->commit.hist.p;
  a.counters = h->commit.ctr64.p;
  a.sel_target = nullptr;
  a.sel_favored = nullptr;
  return a;
}

CommitArgs make_commit_args(kmp_lp_handle *h, const RunCtx &rc) {
  CommitArgs c{};
  c.xadj = h->graph.xadj;
  c.adjncy = h->graph.adjncy;
  c.vwgt = h->graph.vwgt;
  c.label = h->lp.label.p;
  c.labg = h->lp.labg.p;
  c.stamp = 0;
  c.weight = h->lp.weight.p;
  c.max_w = rc.mode == 1 ? h->lp.maxw.p : nullptr;
  c.min_w = rc.has_min ? h->lp.minw.p : nullptr;
  c.active = h->lp.active.p;
  c.max_cluster_weight = rc.max_cluster_weight;
  c.k = rc.num_labels;
  c.mv_u = h->commit.mv_u.p;
  c.mv_t = h->commit.mv_t.p;
  c.acc = h->commit.acc.p;
  c.mover_count = h->commit.ctr32.p + (h->round.mover_parity ? 3 : 0);
  c.next_mover_count = h->commit.ctr32.p + (h->round.mover_parity ? 0 : 3);
  c.also_zero = (h->dist.world > 1 && h->dist.comm != nullptr) ? h->dist.send.p : nullptr;
  c.incoming = h->commit.incoming.p;
  c.slotmap = h->commit.slotmap.p;
  c.cslot = h->commit.cslot.p;
  c.chist = h->commit.chist.p;
  c.hist = h->commit.hist.p;
  c.jmin = h->commit.jmin.p;
  c.out_cur = h->commit.out_cur.p;
  c.out_delta = h->commit.out_delta.p;
  c.ohist = h->commit.ohist.p;
  c.ojmin = h->commit.ojmin.p;
  c.moved_count = h->commit.ctr32.p + 1;
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
  const uint32_t S = h->lists.S;
  SubRound q{};
  q.group = static_cast<int>(sg / S);
  q.sr = sg % S;
  q.first_tier = first_tier_of_group(q.group);
  q.last_tier = last_tier_of_group(q.group);
  for (int t = q.first_tier; t <= q.last_tier; ++t) {
    const uint32_t sz = h->lists.off[t * S + q.sr + 1] - h->lists.off[t * S + q.sr];
    q.size[t] = sz;
    q.total += sz;
    if (t == kHubTier) { // every rank sees the whole hub list and takes entries i % world == rank
      q.lo[t] = 0;
      q.hi[t] = sz;
    } else {
      q.lo[t] = static_cast<uint32_t>(static_cast<uint64_t>(sz) * h->dist.rank / h->dist.world);
      q.hi[t] = static_cast<uint32_t>(static_cast<uint64_t>(sz) * (h->dist.rank + 1) / h->dist.world);
    }
  }
  return q;
}

// capacity of one rank's proposal buffer for sub-round sg (identical on every rank)
uint32_t subround_cap(const kmp_lp_handle *h, const SubRound &q) {
  uint32_t cap = 1;
  for (int t = q.first_tier; t <= q.last_tier; ++t) {
    cap += (q.size[t] + h->dist.world - 1) / h->dist.world;
  }
  return cap;
}

// sweep kernels of one sub-round over this rank's share of the lists
int sweep_subround(kmp_lp_handle *h, const RunCtx &rc, uint32_t iter, uint32_t sg, const SubRound &q) {
  const uint32_t S = h->lists.S;
  SweepArgs sa = make_sweep_args(h, rc);
  sa.base_tie = sync_base(h->cfg.seed, h->call_counter, iter, SALT_TIE);
  sa.base_fav = sync_base(h->cfg.seed, h->call_counter, iter, SALT_FAV);
  sa.base_commit = sync_base(h->cfg.seed, h->call_counter, iter * 4096 + sg, SALT_COMMIT);
  sa.accumulate = !h->round.stepping && rc.mode == 0; // refiner: commit_refine_fused builds the level histograms
  sa.pull = h->round.pull_this;
  sa.window = make_window(iter, sg);
  h->round.cur_subround = q.sr;
  h->round.cur_sg = sg;
  int live = 0;
  for (int t = q.first_tier; t <= q.last_tier; ++t) {
    live += q.size[t] != 0;
  }
  // several tiers in this sub-round: fork them onto side streams (per-tier timing mode keeps them serial so
  // that every tier's CUDA-event time is its own)
  const bool fork = live > 1 && !h->timing;
  if (fork) {
    KMP_CUDA(cudaEventRecord(h->streams.ev_fork, h->stream));
  }
  int side = 0;
  bool used[3] = {false, false, false};
  for (int t = q.last_tier; t >= q.first_tier; --t) { // largest degrees first: the longest tails start earliest
    if (q.size[t] == 0) {
      continue;
    }
    sa.list = h->lists.order.p + h->lists.off[t * S + q.sr] + q.lo[t];
    sa.list_size = q.hi[t] - q.lo[t];
    h->sweep_stream = h->stream;
    if (fork && side < 3 && t != q.first_tier) {
      h->sweep_stream = h->streams.side[side];
      used[side] = true;
      KMP_CUDA(cudaStreamWaitEvent(h->sweep_stream, h->streams.ev_fork, 0));
    }
    const cudaError_t e = launch_sweep(h, rc.mode, t, sa);
    if (h->sweep_stream != h->stream) {
      KMP_CUDA(cudaEventRecord(h->streams.ev_join[side], h->sweep_stream));
      ++side;
    }
    h->sweep_stream = h->stream;
    KMP_CUDA(e);
  }
  for (int i = 0; i < 3; ++i) {
    if (used[i]) {
      KMP_CUDA(cudaStreamWaitEvent(h->stream, h->streams.ev_join[i], 0));
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
  ++h->counts.kernel_launches;
}
// The refiner's ladder commit (lp_commit.cuh commit_refine_fused) in one cooperative launch, for the LP refiner and
// both balancers. Its dynamic shared memory follows the kernel's choice of CTA-private level histograms (priv_h) and
// block-weight deltas (priv_k) for k = ca.k; work: the proposals the launch handles (grid before the clamp).
int launch_commit_refine(kmp_lp_handle *h, CommitArgs ca, GatheredArgs ga, uint32_t passes, uint32_t work) {
  const uint32_t k = ca.k;
  const size_t smem = 4 * std::max<size_t>(k * kLadderLevels <= kSmemPrivLimit ? static_cast<size_t>(k) * kLadderLevels : 0,
                                           k <= kSmemPrivLimit ? k : 0);
  const uint32_t blocks = capped(h, std::min<uint32_t>(grid_for(std::max<uint32_t>(work, k), 256),
                                                       static_cast<uint32_t>(h->fused_blocks_refine)));
  GridBarrier bar{h->grid_bar.p, h->grid_bar.p + 1};
  void *args[] = {&ca, &ga, &bar, &passes};
  if (h->round.p64) {
    KMP_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void *>(commit_refine_fused<true>), dim3(blocks), dim3(256), args,
                                         smem, h->stream));
  } else {
    KMP_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void *>(commit_refine_fused<false>), dim3(blocks), dim3(256), args,
                                         smem, h->stream));
  }
  return KMP_OK;
}
// The whole commit of sub-round sg in one cooperative launch, over the proposals in mv_u / mv_t -- or, with
// gathered != nullptr, over the all-gathered proposal buffers (world * (4 + 2 * cap) words) of a sharded run or of
// the stepping API, which the same launch unpacks and accumulates first. Every rank runs the same
// order-independent commit on the same proposals, so the replicas stay bit-identical.
int commit_subround(kmp_lp_handle *h, const RunCtx &rc, uint32_t iter, uint32_t sg, const SubRound &q,
                    const uint32_t *gathered) {
  CommitArgs ca = make_commit_args(h, rc);
  ca.base_commit = sync_base(h->cfg.seed, h->call_counter, iter * 4096 + sg, SALT_COMMIT);
  ca.stamp = h->lists.stamps_ok ? make_stamp(iter, sg) : 0;
  GatheredArgs ga{gathered, h->dist.world, gathered != nullptr ? subround_cap(h, q) : 0u,
                  h->commit.ctr32.p + (h->round.mover_parity ? 3 : 0)};
  const int ev = timed_begin(h, kTagCommit);
  if (rc.mode == 1) {
    const int r = launch_commit_refine(h, ca, ga, std::max<uint32_t>(1, h->cfg.sync_commit_passes), q.total);
    if (r != KMP_OK) {
      return r;
    }
  } else {
    GridBarrier bar{h->grid_bar.p, h->grid_bar.p + 1};
    const uint32_t blocks = capped(h, std::min<uint32_t>(grid_for(q.total, 256), static_cast<uint32_t>(h->fused_blocks)));
    void *args[] = {&ca, &ga, &bar};
    if (h->round.p64) {
      KMP_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void *>(commit_cluster_fused<true>), dim3(blocks), dim3(256), args, 0,
                                           h->stream));
    } else {
      KMP_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void *>(commit_cluster_fused<false>), dim3(blocks), dim3(256), args,
                                           0, h->stream));
    }
  }
  timed_end(h, ev);
  ++h->counts.kernel_launches;
  if (!h->round.pull_this || !h->round.pull_next) {
    launch_push_activation(h, ca, q); // acc[] / mv_u[] still hold this sub-round's verdicts
  }
  h->round.mover_parity ^= 1u;
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
  const bool can_pull = h->lists.stamps_ok && h->cfg.max_num_neighbors >= h->graph.max_degree;
  auto heavy = [&](uint32_t moved) { return moved == 0xFFFFFFFFu || 16ull * moved >= h->lists.visited_total; };
  if (iter == 0) {
    h->round.moved_hist[0] = h->round.moved_hist[1] = 0xFFFFFFFFu; // [0]: round iter - 1, [1]: round iter - 2
    h->round.pull_this = can_pull;
  } else {
    h->round.pull_this = h->round.pull_next;
  }
  h->round.pull_next = can_pull && heavy(h->round.moved_hist[0]);
  if (const char *e = std::getenv("KMP_ACTIVATION")) { // experiments / tests: force one mode
    if (e[0] == 'p' && e[1] == 'u' && e[2] == 's') {
      h->round.pull_this = h->round.pull_next = false;
    } else if (e[0] == 'p' && e[1] == 'u' && e[2] == 'l' && can_pull) {
      h->round.pull_this = h->round.pull_next = true;
    }
  }
}

int begin_iteration(kmp_lp_handle *h, uint32_t iter) {
  KMP_CUDA(cudaMemsetAsync(h->commit.ctr32.p, 0, kCtr32Size * sizeof(uint32_t), h->stream)); // proposal counters, moved, hub queues
  KMP_CUDA(cudaMemsetAsync(h->lists.queue.p, 0, h->lists.queue.cap * sizeof(uint32_t), h->stream));
  if (h->hub_tmp.cursor.p != nullptr) { // normally already zero (sweep_hub_select resets what it reads)
    KMP_CUDA(cudaMemsetAsync(h->hub_tmp.cursor.p, 0, h->hub_tmp.cursor.cap * sizeof(uint32_t), h->stream));
  }
  if (h->dist.world > 1 && h->dist.comm != nullptr && h->dist.send.p != nullptr) {
    KMP_CUDA(cudaMemsetAsync(h->dist.send.p, 0, sizeof(uint32_t), h->stream)); // proposal counter of the send buffer
  }
  h->round.mover_parity = 0;
  choose_activation(h, iter);
  h->counts.pull_rounds += h->round.pull_this ? 1 : 0;
  h->counts.push_rounds += (!h->round.pull_this || !h->round.pull_next) ? 1 : 0;
  if (iter >= 2 && h->lists.stamps_ok && h->graph.n > 0) {
    const int ev = timed_begin(h, kTagMisc);
    if (h->round.p64) {
      k_age_stamps<true><<<grid_for(h->graph.n, 256), 256, 0, h->stream>>>(h->graph.n, h->lp.labg.p, iter & 1u);
    } else {
      k_age_stamps<false><<<grid_for(h->graph.n, 256), 256, 0, h->stream>>>(h->graph.n, h->lp.labg.p, iter & 1u);
    }
    timed_end(h, ev);
    ++h->counts.kernel_launches;
  }
  return KMP_OK;
}

// The accepted moves of the round into *moved (one host wait), and into the history choose_activation reads.
int end_iteration(kmp_lp_handle *h, uint32_t *moved) {
  uint32_t host[2] = {0, 0};
  KMP_CUDA(cudaMemcpyAsync(host, h->commit.ctr32.p, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
  KMP_CUDA(cudaStreamSynchronize(h->stream));
  *moved = host[1];
  h->round.moved_hist[1] = h->round.moved_hist[0];
  h->round.moved_hist[0] = host[1];
  return KMP_OK;
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
  h->dist.direct_send = (d_send == h->dist.send.p && h->dist.comm != nullptr) ? d_send : nullptr;
  h->dist.direct_cap = cap;
  h->round.stepping = true;
  const int r = sweep_subround(h, rc, iter, sg, q);
  h->round.stepping = false;
  const bool direct = h->dist.direct_send != nullptr;
  h->dist.direct_send = nullptr;
  if (r != KMP_OK) {
    return r;
  }
  if (direct) {
    return KMP_OK;
  }
  k_pack_movers<<<capped(h, grid_for(cap, 256, kSMs * 4)), 256, 0, h->stream>>>(h->commit.mv_u.p, h->commit.mv_t.p,
                                                                      h->commit.ctr32.p + (h->round.mover_parity ? 3 : 0), cap, d_send);
  ++h->counts.kernel_launches;
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
  return rc.mode == 0 && h->dist.world == 1 && !h->round.stepping;
}
static_assert(kMaxSubrounds <= kLowMaxSubrounds, "ensure_lists admits more sub-rounds than LowGroupArgs holds");
// All sub-rounds of degree group `group` (0: tier 0, 1: tiers 1-2) of LP round `iter`, in sub-round order, with the
// hashes, stamp windows, move stamps and proposal-counter parities the per-sub-round path uses.
int run_low_group(kmp_lp_handle *h, const RunCtx &rc, uint32_t iter, int group) {
  const uint32_t S = h->lists.S;
  const int ta = first_tier_of_group(group), tb = last_tier_of_group(group);
  SweepArgs sa = make_sweep_args(h, rc);
  sa.base_tie = sync_base(h->cfg.seed, h->call_counter, iter, SALT_TIE);
  sa.base_fav = sync_base(h->cfg.seed, h->call_counter, iter, SALT_FAV);
  sa.accumulate = true;
  sa.pull = h->round.pull_this;
  sa.list = h->lists.order.p;
  CommitArgs ca = make_commit_args(h, rc);
  LowGroupArgs g{};
  g.push = !h->round.pull_this || !h->round.pull_next;
  g.ctr32 = h->commit.ctr32.p;
  g.counters[0] = h->commit.ctr64.p + ta;
  g.counters[1] = h->commit.ctr64.p + tb;
  uint32_t max_total = 0;
  for (uint32_t s = 0; s < S; ++s) {
    const uint32_t sg = static_cast<uint32_t>(group) * S + s;
    const SubRound q = subround_of_sg(h, sg);
    if (q.total == 0) {
      continue;
    }
    LowSubround &x = g.sub[g.num_sub++];
    x.off[0] = h->lists.off[ta * S + s];
    x.size[0] = q.size[ta];
    x.off[1] = h->lists.off[tb * S + s];
    x.size[1] = tb != ta ? q.size[tb] : 0u;
    const StampWindow w = make_window(iter, sg);
    x.window_start = w.start;
    x.window_len = w.len;
    x.base_commit = sync_base(h->cfg.seed, h->call_counter, iter * 4096 + sg, SALT_COMMIT);
    x.stamp = h->lists.stamps_ok ? make_stamp(iter, sg) : 0u;
    x.parity = h->round.mover_parity;
    h->round.mover_parity ^= 1u;
    max_total = std::max(max_total, q.total);
  }
  if (g.num_sub == 0) {
    return KMP_OK;
  }
  const bool ew = h->graph.adjwgt != nullptr;
  const uint32_t blocks = capped(h, std::min<uint32_t>(grid_for(max_total, 256), h->low_blocks[group][ew][h->round.p64]));
  GridBarrier bar{h->grid_bar.p, h->grid_bar.p + 1};
  void *args[] = {&sa, &ca, &g, &bar};
  // timing mode: the group's sweeps AND commits are this one event pair, under the group's first tier
  const int ev = timed_begin(h, ta);
  KMP_CUDA(cudaLaunchCooperativeKernel(low_group_kernel(ew, h->round.p64, group), dim3(blocks), dim3(256), args, 0, h->stream));
  timed_end(h, ev);
  ++h->counts.kernel_launches;
  ++h->counts.sweep_launches;
  ++h->counts.group_launches[ta];
  return KMP_OK;
}

// One LP round over all (group, sub-round) lists. Returns via *moved the accepted moves.
int run_iteration(kmp_lp_handle *h, const RunCtx &rc, uint32_t iter, uint32_t *moved) {
  const uint32_t S = h->lists.S;
  int rc0 = begin_iteration(h, iter);
  if (rc0 != KMP_OK) {
    return rc0;
  }
  if (h->dist.world > 1) { // exchange buffers for the largest sub-round, allocated once
    size_t max_words = 4;
    for (uint32_t sg = 0; sg < kNumGroups * S; ++sg) {
      max_words = std::max<size_t>(max_words, 4 + 2 * static_cast<size_t>(subround_cap(h, subround_of_sg(h, sg))));
    }
    KMP_CUDA(h->dist.send.ensure(max_words));
    KMP_CUDA(h->dist.recv.ensure(std::max<size_t>(max_words * h->dist.world, h->graph.n)));
  }
  for (uint32_t sg = 0; sg < kNumGroups * S; ++sg) {
    const SubRound q = subround_of_sg(h, sg);
    if (q.total == 0) {
      continue;
    }
    int rc2;
    if (h->dist.world > 1) { // sharded: sweep the own slice, all-gather the proposals (NVLink), replicated commit
      const size_t words = 4 + 2 * static_cast<size_t>(subround_cap(h, q));
      rc2 = dist_sweep_pack(h, rc, iter, sg, q, h->dist.send.p);
      if (rc2 != KMP_OK) {
        return rc2;
      }
      KMP_NCCL(g_nccl.AllGather(h->dist.send.p, h->dist.recv.p, words, ncclUint32, h->dist.comm, h->stream));
      rc2 = commit_subround(h, rc, iter, sg, q, h->dist.recv.p);
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
  return end_iteration(h, moved);
}

// packed gather array: word width by the label range; (re)allocated grow-only
int prepare_labg(kmp_lp_handle *h, uint32_t num_labels) {
  h->round.p64 = num_labels > (1u << 24) || h->force_p64; // KMP_FORCE_P64=1: the 8-byte gather words on small test inputs
  KMP_CUDA(h->lp.labg.ensure(static_cast<size_t>(std::max<uint32_t>(h->graph.n, 1)) * (h->round.p64 ? 8 : 4)));
  return KMP_OK;
}
void launch_init_cluster(kmp_lp_handle *h) {
  if (h->round.p64) {
    k_init_cluster<true><<<grid_for(h->graph.n, 256), 256, 0, h->stream>>>(h->graph.n, h->graph.vwgt, h->lp.label.p,
                                                                             h->lp.labg.p, h->lp.weight.p,
                                                                             h->lp.favored.p, h->lp.active.p);
  } else {
    k_init_cluster<false><<<grid_for(h->graph.n, 256), 256, 0, h->stream>>>(h->graph.n, h->graph.vwgt, h->lp.label.p,
                                                                              h->lp.labg.p, h->lp.weight.p,
                                                                              h->lp.favored.p, h->lp.active.p);
  }
}
void launch_pack_labels(kmp_lp_handle *h) {
  if (h->round.p64) {
    k_pack_labels<true><<<grid_for(h->graph.n, 256), 256, 0, h->stream>>>(h->graph.n, h->lp.label.p, h->lp.labg.p);
  } else {
    k_pack_labels<false><<<grid_for(h->graph.n, 256), 256, 0, h->stream>>>(h->graph.n, h->lp.label.p, h->lp.labg.p);
  }
}

// The labels on the device as a k-way partition: weight[0, k) (zeroed by the caller) += their block weights, and
// labels >= k (e.g. a clustering left on the device, or a host partition with an id >= k) are refused before any
// kernel indexes a [k] array by a label. bad: a zeroed device counter. One n-sized read and one host wait.
int checked_block_weights(kmp_lp_handle *h, uint32_t k, unsigned long long *bad) {
  const uint32_t n = h->graph.n;
  if (n > 0) {
    bal_block_weights<<<capped(h, grid_for(n, 256)), 256, 0, h->stream>>>(n, k, h->graph.vwgt, h->lp.label.p, h->lp.weight.p, bad);
    ++h->counts.kernel_launches;
  }
  unsigned long long b = 0;
  KMP_CUDA(cudaMemcpyAsync(&b, bad, sizeof(b), cudaMemcpyDeviceToHost, h->stream));
  KMP_CUDA(cudaStreamSynchronize(h->stream));
  if (b != 0) {
    return fail(KMP_ERR_INVALID, "labels >= k on the device: a clustering is not a k-way partition");
  }
  return KMP_OK;
}

// A k-way partition onto the handle: the labels (uploaded from partition when non-null, else the device labels
// stay), the max (and, when given, min) block weights, weight[0, k) zeroed for checked_block_weights, which the
// caller runs last so that its host wait covers this set-up.
int load_partition(kmp_lp_handle *h, uint32_t k, const uint32_t *partition, const int32_t *max_block_weights,
                   const int32_t *min_block_weights) {
  const uint32_t n = h->graph.n;
  KMP_CUDA(h->lp.label.ensure(n));
  KMP_CUDA(h->lp.weight.ensure(k));
  KMP_CUDA(h->lp.maxw.ensure(k));
  if (partition != nullptr) {
    KMP_CUDA(cudaMemcpyAsync(h->lp.label.p, partition, static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, h->stream));
    h->lp.labels_valid = true;
  }
  KMP_CUDA(cudaMemcpyAsync(h->lp.maxw.p, max_block_weights, static_cast<size_t>(k) * 4, cudaMemcpyHostToDevice, h->stream));
  if (min_block_weights != nullptr) {
    KMP_CUDA(h->lp.minw.ensure(k));
    KMP_CUDA(cudaMemcpyAsync(h->lp.minw.p, min_block_weights, static_cast<size_t>(k) * 4, cudaMemcpyHostToDevice, h->stream));
  }
  KMP_CUDA(cudaMemsetAsync(h->lp.weight.p, 0, static_cast<size_t>(k) * 4, h->stream));
  return KMP_OK;
}

int refuse_without_labels(const kmp_lp_handle *h) {
  if (!h->lp.labels_valid) {
    return fail(KMP_ERR_INVALID, "no labels of the current graph on the device: cluster, pass a partition or call "
                                 "kmp_lp_upload_partition first");
  }
  return KMP_OK;
}

// The calls that run on one GPU only (the balancers, the overlay) refuse sharded, NCCL and open stepping handles.
int refuse_multi_gpu(const kmp_lp_handle *h, const char *what) {
  if (h->dist.world > 1 || h->dist.comm != nullptr || h->step.open) {
    return fail(KMP_ERR_UNSUPPORTED,
                std::string(what) + " runs on one GPU: sharded, NCCL and stepping handles are refused");
  }
  return KMP_OK;
}

int begin_call(kmp_lp_handle *h, kmp_lp_stats *stats) {
  if (h == nullptr || !h->graph.present) {
    return fail(KMP_ERR_INVALID, "no graph set");
  }
  KMP_CUDA(cudaSetDevice(h->device));
  if (stats != nullptr) {
    std::memset(stats, 0, sizeof(*stats));
  }
  h->counts = {};
  KMP_CUDA(cudaEventRecord(h->streams.ev_begin, h->stream));
  return KMP_OK;
}

int end_call(kmp_lp_handle *h, kmp_lp_stats *stats) {
  if (h->dist.world > 1 && h->dist.comm != nullptr && stats != nullptr) { // every rank reports the whole job's scan counters
    KMP_NCCL(g_nccl.AllReduce(h->commit.ctr64.p, h->commit.ctr64.p, kCtrNodes + kStatTiers, ncclUint64, ncclSum, h->dist.comm, h->stream));
  }
  KMP_CUDA(cudaEventRecord(h->streams.ev_end, h->stream));
  KMP_CUDA(cudaStreamSynchronize(h->stream));
  if (stats != nullptr) {
    unsigned long long c[kCtrNodes + kStatTiers] = {0};
    KMP_CUDA(cudaMemcpy(c, h->commit.ctr64.p, sizeof(c), cudaMemcpyDeviceToHost));
    for (int g = 0; g < kStatTiers; ++g) {
      stats->group_edges[g] = c[g];
      stats->group_nodes[g] = c[kCtrNodes + g];
      stats->group_launches[g] = h->counts.group_launches[g];
      stats->edges_scanned += c[g];
      stats->nodes_visited += c[kCtrNodes + g];
    }
    float ms = 0.f;
    cudaEventElapsedTime(&ms, h->streams.ev_begin, h->streams.ev_end);
    stats->device_ms = ms;
    float sweep = 0.f;
    for (size_t i = 0; i < h->counts.sweep_events_used; ++i) {
      float t = 0.f;
      cudaEventElapsedTime(&t, h->streams.sweep_events[i].first, h->streams.sweep_events[i].second);
      if (h->streams.sweep_event_group[i] < kNumTiers) {
        sweep += t;
      }
      stats->group_sweep_ms[h->streams.sweep_event_group[i]] += t;
      (void)kTagPush;
    }
    stats->sweep_ms = sweep;
    stats->sweep_launches = h->counts.sweep_launches;
    stats->kernel_launches = h->counts.kernel_launches;
    stats->pull_rounds = h->counts.pull_rounds;
    stats->push_rounds = h->counts.push_rounds;
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
  const uint32_t n = h->graph.n;
  const bool two_hop = (1.0 - 1.0 * num_clusters / n) <= h->cfg.two_hop_threshold; // lp_clusterer.cc:164-166
  const int iso = h->cfg.isolated_nodes_strategy;
  const bool iso_match = iso == KMP_ISOLATED_MATCH || (iso == KMP_ISOLATED_MATCH_DURING_TWO_HOP && two_hop);
  const bool iso_cluster = iso == KMP_ISOLATED_CLUSTER || (iso == KMP_ISOLATED_CLUSTER_DURING_TWO_HOP && two_hop);
  auto sort_pairs = [&](uint32_t cnt, int bits) { // pairs_a -> pairs_b, ascending
    return cub_call(h, [&](void *tmp, size_t &bytes) {
      return cub::DeviceRadixSort::SortKeys(tmp, bytes, h->ops.pairs_a.p, h->ops.pairs_b.p, static_cast<int>(cnt), 0, bits,
                                            h->stream);
    });
  };
  if ((iso_match || iso_cluster) && h->graph.num_isolated > 1) {
    KMP_CUDA(h->ops.pairs_a.ensure(h->graph.num_isolated));
    KMP_CUDA(h->ops.pairs_b.ensure(h->graph.num_isolated));
    reset_u32<<<1, 1, 0, h->stream>>>(h->commit.ctr32.p + 2);
    k_collect_isolated<<<grid_for(n, 256), 256, 0, h->stream>>>(n, h->graph.xadj, h->ops.pairs_a.p, h->commit.ctr32.p + 2);
    uint32_t iso_cnt = 0;
    KMP_CUDA(cudaMemcpyAsync(&iso_cnt, h->commit.ctr32.p + 2, sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
    KMP_CUDA(cudaStreamSynchronize(h->stream));
    if (iso_cnt > 1) {
      KMP_CUDA(sort_pairs(iso_cnt, 32)); // key 0: ascending vertex id
      if (iso_match) {
        k_match_isolated<<<grid_for(iso_cnt / 2 + 1, 256), 256, 0, h->stream>>>(iso_cnt, h->ops.pairs_b.p, h->lp.label.p,
                                                                                h->lp.weight.p, max_w);
      } else {
        k_next_fit<<<1, 256, 0, h->stream>>>(iso_cnt, h->ops.pairs_b.p, h->lp.label.p, h->lp.weight.p, max_w); // one group
      }
      h->counts.kernel_launches += 3;
      KMP_CUDA(cudaGetLastError());
    }
  }
  if (!two_hop || h->cfg.two_hop_strategy == KMP_TWO_HOP_DISABLE) {
    return KMP_OK;
  }
  if (stats != nullptr) {
    stats->two_hop_ran = 1;
  }
  KMP_CUDA(h->ops.pairs_a.ensure(n));
  KMP_CUDA(h->ops.pairs_b.ensure(n));
  reset_u32<<<1, 1, 0, h->stream>>>(h->commit.ctr32.p + 2);
  k_collect_two_hop<<<grid_for(n, 256), 256, 0, h->stream>>>(n, h->graph.xadj, h->graph.vwgt, h->lp.label.p, h->lp.weight.p,
                                                              h->lp.favored.p, max_w, h->ops.pairs_a.p, h->commit.ctr32.p + 2);
  uint32_t cnt = 0;
  KMP_CUDA(cudaMemcpyAsync(&cnt, h->commit.ctr32.p + 2, sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
  KMP_CUDA(cudaStreamSynchronize(h->stream));
  if (cnt > 1) {
    KMP_CUDA(sort_pairs(cnt, 64));
    if (h->cfg.two_hop_strategy == KMP_TWO_HOP_CLUSTER_THREADWISE) {
      k_next_fit<<<grid_for(static_cast<uint64_t>(cnt) * 32, 256, kSMs * 8), 256, 0, h->stream>>>(cnt, h->ops.pairs_b.p, h->lp.label.p,
                                                                                                 h->lp.weight.p, max_w);
      h->counts.kernel_launches += 3;
    } else {
      // group heads: reuse mv-independent scratch (pairs_a is free after the sort)
      uint32_t *head_in = reinterpret_cast<uint32_t *>(h->ops.pairs_a.p);
      uint32_t *head_out = head_in + cnt;
      k_two_hop_heads<<<grid_for(cnt, 256), 256, 0, h->stream>>>(cnt, h->ops.pairs_b.p, head_in);
      KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
        return cub::DeviceScan::InclusiveScan(tmp, bytes, head_in, head_out, MaxOp(), static_cast<int>(cnt), h->stream);
      }));
      k_match_two_hop<<<grid_for(cnt, 256), 256, 0, h->stream>>>(cnt, h->ops.pairs_b.p, head_out, h->lp.label.p, h->lp.weight.p);
      h->counts.kernel_launches += 5;
    }
    KMP_CUDA(cudaGetLastError());
  }
  return KMP_OK;
}

// ---- one LP run of the sync schedule: set-up and finish of kmp_lp_cluster / kmp_lp_refine and the stepping API ----
// Clustering set-up: every vertex its own cluster. *ctx is written only when the set-up succeeds.
int begin_cluster_run(kmp_lp_handle *h, int32_t max_cluster_weight, const uint32_t *communities, RunCtx *ctx) {
  if (h->cfg.sync_commit_passes > 1) { // the cluster commit kernels decide in one pass: no departure credit
    return fail(KMP_ERR_UNSUPPORTED, "the clusterer's sync commit is single-pass (sync_commit_passes must be 1)");
  }
  const uint32_t n = h->graph.n;
  int rc = ensure_lists(h);
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(h->lp.label.ensure(n));
  KMP_CUDA(h->lp.favored.ensure(n));
  KMP_CUDA(h->lp.weight.ensure(n));
  rc = ensure_scratch(h, 0, n);
  if (rc == KMP_OK) {
    rc = prepare_labg(h, n);
  }
  if (rc == KMP_OK) {
    rc = upload_optional_u32(h, h->lp.communities, communities, n);
  }
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(cudaMemsetAsync(h->commit.ctr64.p, 0, kCtrSize * sizeof(unsigned long long), h->stream));
  if (n > 0) {
    launch_init_cluster(h);
    ++h->counts.kernel_launches;
  }
  *ctx = RunCtx{0, n, max_cluster_weight, false, communities != nullptr};
  return KMP_OK;
}

// Refinement set-up: the partition (uploaded when non-null, else the device labels), all vertices active. *ctx is
// written only when the set-up succeeds.
int begin_refine_run(kmp_lp_handle *h, uint32_t k, const int32_t *max_block_weights, const int32_t *min_block_weights,
                     const uint32_t *communities, const uint32_t *partition, RunCtx *ctx) {
  const uint32_t n = h->graph.n;
  int rc = ensure_lists(h);
  if (rc == KMP_OK) {
    rc = ensure_scratch(h, 1, k);
  }
  if (rc == KMP_OK) {
    rc = prepare_labg(h, k);
  }
  if (rc == KMP_OK) {
    rc = load_partition(h, k, partition, max_block_weights, min_block_weights);
  }
  if (rc == KMP_OK) {
    rc = upload_optional_u32(h, h->lp.communities, communities, n);
  }
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(cudaMemsetAsync(h->commit.ctr64.p, 0, kCtrSize * sizeof(unsigned long long), h->stream));
  if (n > 0) {
    k_fill_u8<<<grid_for(n, 256), 256, 0, h->stream>>>(n, h->lp.active.p, 1); // Base::initialize: all active
    launch_pack_labels(h); // reads the labels without indexing by them
    h->counts.kernel_launches += 2;
  }
  rc = checked_block_weights(h, k, h->commit.ctr64.p + kCtrScratch); // last: its wait covers the set-up above
  if (rc != KMP_OK) {
    return rc;
  }
  *ctx = RunCtx{1, k, 0, min_block_weights != nullptr, communities != nullptr};
  return KMP_OK;
}

// The clusters (labels of nonzero weight) of a non-empty graph: two launches, which the caller counts, and a host wait.
int count_clusters(kmp_lp_handle *h, uint32_t *num_clusters) {
  reset_u32<<<1, 1, 0, h->stream>>>(h->commit.ctr32.p + 2);
  k_count_nonzero<<<grid_for(h->graph.n, 256), 256, 0, h->stream>>>(h->graph.n, h->lp.weight.p, h->commit.ctr32.p + 2);
  KMP_CUDA(cudaMemcpyAsync(num_clusters, h->commit.ctr32.p + 2, 4, cudaMemcpyDeviceToHost, h->stream));
  KMP_CUDA(cudaStreamSynchronize(h->stream));
  return KMP_OK;
}

// Clustering finish: the cluster count and the post passes. Every completed clustering, of an empty graph too,
// advances the call index of the sync hashes.
int finish_cluster_run(kmp_lp_handle *h, int32_t max_cluster_weight, kmp_lp_stats *stats) {
  if (h->graph.n > 0) {
    uint32_t num_clusters = 0;
    int rc = count_clusters(h, &num_clusters);
    if (rc != KMP_OK) {
      return rc;
    }
    h->counts.kernel_launches += 2;
    if (stats != nullptr) {
      stats->num_clusters = num_clusters;
    }
    rc = cluster_post_passes(h, max_cluster_weight, num_clusters, stats); // lp_clusterer.cc:107-108
    if (rc != KMP_OK) {
      return rc;
    }
  }
  ++h->call_counter;
  h->lp.labels_valid = true;
  return KMP_OK;
}

// n labels into labels_out and k block weights into block_weights_out, each when non-null.
int download_results(kmp_lp_handle *h, uint32_t *labels_out, int32_t *block_weights_out, uint32_t k) {
  if (labels_out != nullptr && h->graph.n > 0) {
    KMP_CUDA(cudaMemcpyAsync(labels_out, h->lp.label.p, static_cast<size_t>(h->graph.n) * 4, cudaMemcpyDeviceToHost, h->stream));
  }
  if (block_weights_out != nullptr) {
    KMP_CUDA(cudaMemcpyAsync(block_weights_out, h->lp.weight.p, static_cast<size_t>(k) * 4, cudaMemcpyDeviceToHost, h->stream));
  }
  return KMP_OK;
}

// ---- schedule KMP_SCHEDULE_SEQ_STRICT ----------------------------------------------------------------
// mode 0: labels are (re)initialised by the engine; mode 1: h->lp.label holds the partition. Results stay in
// h->lp.label / h->lp.weight; iteration statistics go to *stats, the scan counters to the last tier slot of ctr64.
int run_strict(kmp_lp_handle *h, int mode, uint32_t num_keys, int32_t max_cluster_weight, uint32_t desired,
               uint32_t k, bool has_min, bool has_comm, kmp_lp_stats *stats) {
  const size_t n = std::max<uint32_t>(h->graph.n, 1);
  const size_t keys = std::max<size_t>(std::max<size_t>(num_keys, n), 1);
  KMP_CUDA(h->lp.favored.ensure(n));
  KMP_CUDA(h->lp.active.ensure(n));
  KMP_CUDA(h->strict.slot.ensure(keys));
  KMP_CUDA(h->strict.slot2.ensure(keys));
  KMP_CUDA(h->strict.concurrent.ensure(keys));
  KMP_CUDA(h->strict.used.ensure(keys));
  KMP_CUDA(h->strict.ent_key.ensure(keys + 1));
  KMP_CUDA(h->strict.ent_val.ensure(keys + 1));
  KMP_CUDA(h->strict.ent2_key.ensure(keys + 1));
  KMP_CUDA(h->strict.ent2_val.ensure(keys + 1));
  KMP_CUDA(h->strict.tie_best.ensure(keys + 1));
  KMP_CUDA(h->strict.tie_fav.ensure(keys + 1));
  KMP_CUDA(h->strict.second.ensure(n));
  KMP_CUDA(h->strict.chunks.ensure(2 * (n + 64)));
  KMP_CUDA(h->strict.sub_perm.ensure(n / 64 + 2));
  KMP_CUDA(h->strict.match.ensure(n));
  KMP_CUDA(h->strict.buckets.ensure(36));
  KMP_CUDA(h->strict.rng.ensure(1));
  KMP_CUDA(h->strict.stats.ensure(1));
  if (!h->strict.seeded) { // Random::reseed + the RandomPermutations member of the LP object, once per object
    kmp_strict::strict_seed_kernel<<<1, 32, 0, h->stream>>>(h->strict.rng.p, h->cfg.seed);
    h->strict.seeded = true;
    ++h->counts.kernel_launches;
  }
  kmp_strict::Args a{};
  a.n = h->graph.n;
  a.m = h->graph.m;
  a.xadj = h->graph.xadj;
  a.adjncy = h->graph.adjncy;
  a.vwgt = h->graph.vwgt;
  a.adjwgt = h->graph.adjwgt;
  a.sorted = h->graph.sorted ? 1 : 0;
  a.buckets = h->strict.buckets.p;
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
  a.max_bw = mode == 1 ? h->lp.maxw.p : nullptr;
  a.min_bw = has_min ? h->lp.minw.p : nullptr;
  a.communities = has_comm ? h->lp.communities.p : nullptr;
  a.label = h->lp.label.p;
  a.weight = h->lp.weight.p;
  a.favored = h->lp.favored.p;
  a.active = h->lp.active.p;
  a.slot = h->strict.slot.p;
  a.ent_key = h->strict.ent_key.p;
  a.ent_val = h->strict.ent_val.p;
  a.slot2 = h->strict.slot2.p;
  a.ent2_key = h->strict.ent2_key.p;
  a.ent2_val = h->strict.ent2_val.p;
  a.concurrent = h->strict.concurrent.p;
  a.used_entries = h->strict.used.p;
  a.second_phase_nodes = h->strict.second.p;
  a.tie_best = h->strict.tie_best.p;
  a.tie_fav = h->strict.tie_fav.p;
  a.chunks = h->strict.chunks.p;
  a.sub_perm = h->strict.sub_perm.p;
  a.match_map = h->strict.match.p;
  a.rng = h->strict.rng.p;
  a.stats = h->strict.stats.p;
  kmp_strict::strict_kernel<<<1, 32, 0, h->stream>>>(a);
  ++h->counts.kernel_launches;
  KMP_CUDA(cudaGetLastError());
  kmp_strict::Stats hs{};
  KMP_CUDA(cudaMemcpyAsync(&hs, h->strict.stats.p, sizeof(hs), cudaMemcpyDeviceToHost, h->stream));
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
  KMP_CUDA(cudaMemcpy(h->commit.ctr64.p + (kStatTiers - 1), &c[0], 8, cudaMemcpyHostToDevice));
  KMP_CUDA(cudaMemcpy(h->commit.ctr64.p + kCtrNodes + (kStatTiers - 1), &c[1], 8, cudaMemcpyHostToDevice));
  return KMP_OK;
}

int strict_cluster(kmp_lp_handle *h, int32_t max_cluster_weight, uint32_t desired_num_clusters,
                   const uint32_t *communities, uint32_t *clustering_out, kmp_lp_stats *stats) {
  const uint32_t n = h->graph.n;
  KMP_CUDA(h->lp.label.ensure(std::max<uint32_t>(n, 1)));
  KMP_CUDA(h->lp.weight.ensure(std::max<uint32_t>(n, 1)));
  KMP_CUDA(h->commit.ctr64.ensure(kCtrSize));
  KMP_CUDA(cudaMemsetAsync(h->commit.ctr64.p, 0, kCtrSize * sizeof(unsigned long long), h->stream));
  int rc = upload_optional_u32(h, h->lp.communities, communities, n);
  if (rc == KMP_OK) {
    rc = run_strict(h, 0, n, max_cluster_weight, desired_num_clusters, 0, false, communities != nullptr, stats);
  }
  if (rc == KMP_OK) {
    rc = download_results(h, clustering_out, nullptr, 0);
  }
  if (rc != KMP_OK) {
    return rc;
  }
  ++h->call_counter;
  h->lp.labels_valid = true;
  return end_call(h, stats);
}

int strict_refine(kmp_lp_handle *h, uint32_t k, const int32_t *max_block_weights, const int32_t *min_block_weights,
                  const uint32_t *communities, uint32_t *partition_inout, int32_t *block_weights_out,
                  kmp_lp_stats *stats) {
  const uint32_t n = h->graph.n;
  // the engine's sizes, above the n labels and k weights load_partition ensures
  KMP_CUDA(h->lp.label.ensure(std::max<uint32_t>(n, 1)));
  KMP_CUDA(h->lp.weight.ensure(std::max<uint32_t>(std::max(n, k), 1)));
  KMP_CUDA(h->commit.ctr64.ensure(kCtrSize));
  KMP_CUDA(cudaMemsetAsync(h->commit.ctr64.p, 0, kCtrSize * sizeof(unsigned long long), h->stream));
  int rc = load_partition(h, k, partition_inout, max_block_weights, min_block_weights);
  if (rc == KMP_OK) {
    rc = upload_optional_u32(h, h->lp.communities, communities, n);
  }
  if (rc == KMP_OK) {
    rc = checked_block_weights(h, k, h->commit.ctr64.p + kCtrScratch); // the engine recomputes the weights itself
  }
  if (rc == KMP_OK) {
    rc = run_strict(h, 1, k, 0, 0, k, min_block_weights != nullptr, communities != nullptr, stats);
  }
  if (rc == KMP_OK) {
    rc = download_results(h, partition_inout, block_weights_out, k);
  }
  if (rc != KMP_OK) {
    return rc;
  }
  return end_call(h, stats);
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
  // a refused call frees what was already created: the handle's members own their streams, events and buffers
  std::unique_ptr<kmp_lp_handle> owner(new (std::nothrow) kmp_lp_handle());
  kmp_lp_handle *h = owner.get();
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
  if (cudaSetDevice(dev) != cudaSuccess || cudaStreamCreateWithFlags(&h->streams.owned, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreate(&h->streams.ev_begin) != cudaSuccess || cudaEventCreate(&h->streams.ev_end) != cudaSuccess) {
    return fail(KMP_ERR_CUDA, "failed to create stream/events");
  }
  h->stream = h->streams.owned;
  h->sweep_stream = h->stream;
  for (int i = 0; i < 3; ++i) {
    if (cudaStreamCreateWithFlags(&h->streams.side[i], cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&h->streams.ev_join[i], cudaEventDisableTiming) != cudaSuccess) {
        return fail(KMP_ERR_CUDA, "failed to create side streams");
    }
  }
  if (cudaEventCreateWithFlags(&h->streams.ev_fork, cudaEventDisableTiming) != cudaSuccess) {
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
    return fail(KMP_ERR_CUDA, "this device does not support cooperative launches");
  }
  // co-resident CTAs of both commit kernels, the refiner's with its largest dynamic shared memory (kSmemPrivLimit ints)
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, commit_cluster_fused<false>, 256, 0) != cudaSuccess ||
      per_sm < 1 ||
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_r, commit_refine_fused<false>, 256, kSmemPrivLimit * 4) !=
          cudaSuccess ||
      per_sm_r < 1) {
    return fail(KMP_ERR_CUDA, "a fused commit kernel cannot be resident on this device");
  }
  if (h->grid_bar.ensure(2) != cudaSuccess || cudaMemset(h->grid_bar.p, 0, 2 * sizeof(unsigned)) != cudaSuccess) {
    return fail(KMP_ERR_CUDA, "failed to allocate the grid barrier");
  }
  // all co-resident CTAs: a sub-round of a 10^8-vertex graph commits 10^7 proposals, each a short chain of
  // dependent random accesses -- the grid is sized by the proposal count up to this limit
  h->fused_blocks = sms * per_sm;
  h->fused_blocks_refine = sms * per_sm_r;
  if (!configure_low_groups(h, sms)) {
    return fail(KMP_ERR_CUDA, "a persistent low-degree clustering kernel cannot be resident on this device");
  }
  if (!(configure_team_kernels<0, false, false>(h, sms) && configure_team_kernels<0, false, true>(h, sms) &&
        configure_team_kernels<0, true, false>(h, sms) && configure_team_kernels<0, true, true>(h, sms) &&
        configure_team_kernels<1, false, false>(h, sms) && configure_team_kernels<1, false, true>(h, sms) &&
        configure_team_kernels<1, true, false>(h, sms) && configure_team_kernels<1, true, true>(h, sms))) {
    return fail(KMP_ERR_CUDA, "a sweep_team kernel cannot be resident on this device");
  }
  *out = owner.release();
  return KMP_OK;
}

int kmp_lp_destroy(kmp_lp_handle *h) {
  if (h == nullptr) {
    return KMP_OK;
  }
  cudaSetDevice(h->device);
  cudaStreamSynchronize(h->stream);
  if (h->dist.comm != nullptr) {
    g_nccl.CommDestroy(h->dist.comm);
  }
  kmp_lp_free_scratch(h); // trims the pool
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
  h->graph.n = n;
  h->graph.m = m;
  h->graph.present = true;
  ++h->graph.epoch;
  h->lp.labels_valid = false;
  h->ops.ov.stash.clear(); // the stash belongs to the previous graph; freed stream-ordered, after the work that reads it
  h->lists.valid = false;
  h->commit.slot_state_clean = false;
  h->graph.sorted = false;
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
  h->graph.num_isolated = 0;
  {
    // vertices in the tail bucket are either isolated or above the degree threshold; count isolated
    // ones exactly only when a post pass needs them (cheap: tail bucket size is an upper bound)
    const uint32_t S = h->lists.S;
    h->graph.num_isolated = h->lists.off[kNumTiers * S + 1] - h->lists.off[kNumTiers * S];
  }
  return KMP_OK;
}

int kmp_lp_set_graph(kmp_lp_handle *h, uint32_t n, uint32_t m, const uint32_t *xadj, const uint32_t *adjncy,
                     const int32_t *vwgt, const int32_t *adjwgt) {
  if (h == nullptr || xadj == nullptr || (m > 0 && adjncy == nullptr)) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  KMP_CUDA(cudaSetDevice(h->device));
  KMP_CUDA(h->graph.own_xadj.ensure(static_cast<size_t>(n) + 1));
  KMP_CUDA(h->graph.own_adjncy.ensure(m));
  // xadj first, on the handle's stream: the work lists only need the degrees and are built (kernels, a radix
  // pass, three small host round trips) while the m-sized arrays are still crossing PCIe on a side stream
  KMP_CUDA(cudaStreamSynchronize(h->stream)); // earlier work may still read the old arrays
  KMP_CUDA(cudaMemcpyAsync(h->graph.own_xadj.p, xadj, (static_cast<size_t>(n) + 1) * 4, cudaMemcpyHostToDevice, h->stream));
  const cudaStream_t big = h->streams.side[0];
  if (m > 0) {
    KMP_CUDA(cudaMemcpyAsync(h->graph.own_adjncy.p, adjncy, static_cast<size_t>(m) * 4, cudaMemcpyHostToDevice, big));
  }
  h->graph.xadj = h->graph.own_xadj.p;
  h->graph.adjncy = h->graph.own_adjncy.p;
  h->graph.adjncy_16b = true; // cudaMalloc: 256-byte aligned
  h->graph.vwgt = nullptr;
  h->graph.adjwgt = nullptr;
  if (vwgt != nullptr) {
    KMP_CUDA(h->graph.own_vwgt.ensure(n));
    KMP_CUDA(cudaMemcpyAsync(h->graph.own_vwgt.p, vwgt, static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, h->stream));
    h->graph.vwgt = h->graph.own_vwgt.p;
  }
  if (adjwgt != nullptr) {
    KMP_CUDA(h->graph.own_adjwgt.ensure(m));
    KMP_CUDA(cudaMemcpyAsync(h->graph.own_adjwgt.p, adjwgt, static_cast<size_t>(m) * 4, cudaMemcpyHostToDevice, big));
    h->graph.adjwgt = h->graph.own_adjwgt.p;
  }
  KMP_CUDA(cudaEventRecord(h->streams.ev_join[0], big));
  const int rc = set_graph_common(h, n, m);
  KMP_CUDA(cudaStreamWaitEvent(h->stream, h->streams.ev_join[0], 0)); // later work on the handle's stream sees the whole graph
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
  h->graph.xadj = d_xadj;
  h->graph.adjncy = d_adjncy;
  // a view into a larger buffer may start anywhere: the hub tier then reads adjncy from global memory
  h->graph.adjncy_16b = (reinterpret_cast<uintptr_t>(d_adjncy) & 15u) == 0;
  h->graph.vwgt = d_vwgt;
  h->graph.adjwgt = d_adjwgt;
  return set_graph_common(h, n, m);
}

int kmp_lp_set_graph_sorted(kmp_lp_handle *h, int sorted) {
  if (h == nullptr || !h->graph.present) {
    return fail(KMP_ERR_INVALID, "no graph set");
  }
  h->graph.sorted = sorted != 0;
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
  if (h->dist.world > 1 && h->dist.comm == nullptr) {
    return fail(KMP_ERR_INVALID, "sharded handle without a communicator: call kmp_lp_dist_init (or drive the "
                                 "stepping API yourself)");
  }
  const uint32_t n = h->graph.n;
  RunCtx ctx;
  rc = begin_cluster_run(h, max_cluster_weight, communities, &ctx);
  if (rc != KMP_OK) {
    return rc;
  }
  for (uint32_t it = 0; it < h->cfg.num_iterations && n > 0; ++it) { // lp_clusterer.cc:94-105
    uint32_t moved = 0;
    rc = run_iteration(h, ctx, it, &moved);
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
      uint32_t num_clusters = 0;
      rc = count_clusters(h, &num_clusters);
      if (rc != KMP_OK) {
        return rc;
      }
      if (num_clusters <= desired_num_clusters) {
        break;
      }
    }
  }
  if (h->dist.world > 1 && n > 0) { // favored[u] is only written by the rank that swept u: MAX over (favored ^ u), 0 elsewhere
    KMP_CUDA(h->dist.recv.ensure(n));
    k_xor_iota<<<grid_for(n, 256), 256, 0, h->stream>>>(n, h->lp.favored.p, h->dist.recv.p);
    KMP_NCCL(g_nccl.AllReduce(h->dist.recv.p, h->dist.recv.p, n, ncclUint32, ncclMax, h->dist.comm, h->stream));
    k_xor_iota<<<grid_for(n, 256), 256, 0, h->stream>>>(n, h->dist.recv.p, h->lp.favored.p);
  }
  rc = finish_cluster_run(h, max_cluster_weight, stats);
  if (rc == KMP_OK) {
    rc = download_results(h, clustering_out, nullptr, 0);
  }
  if (rc != KMP_OK) {
    return rc;
  }
  return end_call(h, stats);
}

int kmp_lp_upload_partition(kmp_lp_handle *h, const uint32_t *partition) {
  if (h == nullptr || !h->graph.present || partition == nullptr) {
    return fail(KMP_ERR_INVALID, "bad argument");
  }
  KMP_CUDA(cudaSetDevice(h->device));
  KMP_CUDA(h->lp.label.ensure(h->graph.n));
  KMP_CUDA(cudaMemcpyAsync(h->lp.label.p, partition, static_cast<size_t>(h->graph.n) * 4, cudaMemcpyHostToDevice, h->stream));
  KMP_CUDA(cudaStreamSynchronize(h->stream));
  h->lp.labels_valid = true;
  return KMP_OK;
}

int kmp_lp_download_labels(kmp_lp_handle *h, uint32_t *labels_out) {
  if (h == nullptr || !h->graph.present || labels_out == nullptr || h->lp.label.p == nullptr) {
    return fail(KMP_ERR_INVALID, "bad argument");
  }
  KMP_CUDA(cudaSetDevice(h->device));
  KMP_CUDA(cudaMemcpyAsync(labels_out, h->lp.label.p, static_cast<size_t>(h->graph.n) * 4, cudaMemcpyDeviceToHost, h->stream));
  KMP_CUDA(cudaStreamSynchronize(h->stream));
  return KMP_OK;
}

const uint32_t *kmp_lp_labels_device(kmp_lp_handle *h) { return h != nullptr ? h->lp.label.p : nullptr; }

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
  if (h->dist.world > 1 && h->dist.comm == nullptr) {
    return fail(KMP_ERR_INVALID, "sharded handle without a communicator: call kmp_lp_dist_init (or drive the "
                                 "stepping API yourself)");
  }
  const uint32_t n = h->graph.n;
  RunCtx ctx;
  rc = begin_refine_run(h, k, max_block_weights, min_block_weights, communities, partition_inout, &ctx);
  if (rc != KMP_OK) {
    return rc;
  }
  const uint64_t max_it = h->cfg.num_iterations == 0 ? ~0ull : h->cfg.num_iterations; // lp_refiner.cc:78-79
  for (uint64_t it = 0; it < max_it && n > 0; ++it) {
    uint32_t moved = 0;
    rc = run_iteration(h, ctx, static_cast<uint32_t>(it), &moved);
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
  rc = download_results(h, partition_inout, block_weights_out, k);
  if (rc != KMP_OK) {
    return rc;
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
  const uint32_t n = h->graph.n;
  rc = ensure_lists(h);
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(h->lp.label.ensure(n));
  KMP_CUDA(h->lp.weight.ensure(num_labels));
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
  KMP_CUDA(cudaMemcpyAsync(h->lp.label.p, labels, static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, h->stream));
  KMP_CUDA(cudaMemcpyAsync(d_target.p, labels, static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, h->stream));
  KMP_CUDA(cudaMemsetAsync(d_fav.p, 0xFF, static_cast<size_t>(n) * 4, h->stream));
  KMP_CUDA(cudaMemcpyAsync(h->lp.weight.p, weights, static_cast<size_t>(num_labels) * 4, cudaMemcpyHostToDevice, h->stream));
  if (mode == 1) {
    KMP_CUDA(h->lp.maxw.ensure(num_labels));
    KMP_CUDA(cudaMemcpyAsync(h->lp.maxw.p, max_weights, static_cast<size_t>(num_labels) * 4, cudaMemcpyHostToDevice, h->stream));
    if (min_weights != nullptr) {
      KMP_CUDA(h->lp.minw.ensure(num_labels));
      KMP_CUDA(cudaMemcpyAsync(h->lp.minw.p, min_weights, static_cast<size_t>(num_labels) * 4, cudaMemcpyHostToDevice, h->stream));
    }
  }
  KMP_CUDA(cudaMemsetAsync(h->commit.ctr64.p, 0, kCtrSize * sizeof(unsigned long long), h->stream));
  if (n > 0) {
    launch_pack_labels(h);
  }
  RunCtx ctx{mode, num_labels, max_cluster_weight, mode == 1 && min_weights != nullptr, false};
  SweepArgs sa = make_sweep_args(h, ctx);
  sa.active = nullptr;
  KMP_CUDA(cudaMemsetAsync(h->commit.ctr32.p, 0, kCtr32Size * sizeof(uint32_t), h->stream)); // hub work-queue cursors
  KMP_CUDA(cudaMemsetAsync(h->lists.queue.p, 0, h->lists.queue.cap * sizeof(uint32_t), h->stream));
  if (h->hub_tmp.cursor.p != nullptr) {
    KMP_CUDA(cudaMemsetAsync(h->hub_tmp.cursor.p, 0, h->hub_tmp.cursor.cap * sizeof(uint32_t), h->stream));
  }
  sa.sel_target = d_target.p;
  sa.sel_favored = mode == 0 ? d_fav.p : nullptr;
  sa.base_tie = sync_base(h->cfg.seed, call_index, iteration, SALT_TIE);
  sa.base_fav = sync_base(h->cfg.seed, call_index, iteration, SALT_FAV);
  const uint32_t S = h->lists.S;
  for (uint32_t ts = 0; ts < kNumTiers * S; ++ts) { // every (tier, class) list once
    const uint32_t off = h->lists.off[ts];
    const uint32_t size = h->lists.off[ts + 1] - off;
    const int tier = static_cast<int>(ts / S);
    sa.list = h->lists.order.p + off;
    sa.list_size = size;
    h->round.cur_subround = ts % S;
    h->round.cur_sg = group_of_tier(tier) * S + ts % S; // one queue cursor per (tier, sub-round)
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
  h->lp = {};
  h->commit = {};
  h->hub_tmp = {};
  h->list_tmp = {};
  h->ops = {};
  h->bal = {};
  cudaMemPool_t pool = kmp_private_pool(h->device); // blocks cached for coarse graphs (kmp_contract.cuh)
  if (pool != nullptr) {
    cudaMemPoolTrimTo(pool, 0);
  }
  return KMP_OK;
}

int kmp_pool_usage(kmp_lp_handle *h, int reset, uint64_t *used, uint64_t *used_high) {
  if (h == nullptr || used == nullptr || used_high == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  KMP_CUDA(cudaSetDevice(h->device));
  cudaMemPool_t pool = kmp_private_pool(h->device);
  if (pool == nullptr) {
    return fail(KMP_ERR_CUDA, "no device memory pool");
  }
  KMP_CUDA(cudaStreamSynchronize(h->stream)); // the stream-ordered frees of h's calls have happened
  uint64_t cur = 0, high = 0;
  KMP_CUDA(cudaMemPoolGetAttribute(pool, cudaMemPoolAttrUsedMemCurrent, &cur));
  KMP_CUDA(cudaMemPoolGetAttribute(pool, cudaMemPoolAttrUsedMemHigh, &high));
  *used = cur;
  *used_high = high;
  if (reset != 0) {
    uint64_t zero = 0; // the only value the attribute accepts: the mark restarts at the current use
    KMP_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrUsedMemHigh, &zero));
  }
  return KMP_OK;
}

int kmp_lp_edge_cut(kmp_lp_handle *h, int64_t *cut_out) {
  if (h == nullptr || !h->graph.present || cut_out == nullptr || h->lp.label.p == nullptr) {
    return fail(KMP_ERR_INVALID, "bad argument");
  }
  const int rc = refuse_without_labels(h);
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(cudaSetDevice(h->device));
  KMP_CUDA(h->commit.ctr64.ensure(kCtrSize));
  KMP_CUDA(cudaMemsetAsync(h->commit.ctr64.p + kCtrScratch, 0, sizeof(unsigned long long), h->stream));
  k_edge_cut<<<grid_for(static_cast<uint64_t>(h->graph.n) * 32, 256), 256, 0, h->stream>>>(
      h->graph.n, h->graph.xadj, h->graph.adjncy, h->graph.adjwgt, h->lp.label.p, h->commit.ctr64.p + kCtrScratch);
  unsigned long long c = 0;
  KMP_CUDA(cudaMemcpyAsync(&c, h->commit.ctr64.p + kCtrScratch, sizeof(c), cudaMemcpyDeviceToHost, h->stream));
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
  h->dist.rank = rank;
  h->dist.world = world;
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
  if (h->dist.comm != nullptr) {
    g_nccl.CommDestroy(h->dist.comm);
    h->dist.comm = nullptr;
  }
  ncclUniqueId nid;
  std::memcpy(&nid, id, sizeof(nid));
  if (world > 1) {
    KMP_NCCL(g_nccl.CommInitRank(&h->dist.comm, static_cast<int>(world), nid, static_cast<int>(rank)));
  }
  h->dist.rank = rank;
  h->dist.world = world;
  return KMP_OK;
}

int kmp_lp_dist_shutdown(kmp_lp_handle *h) {
  if (h == nullptr) {
    return KMP_OK;
  }
  if (h->dist.comm != nullptr) {
    cudaStreamSynchronize(h->stream);
    g_nccl.CommDestroy(h->dist.comm);
    h->dist.comm = nullptr;
  }
  h->dist.rank = 0;
  h->dist.world = 1;
  return KMP_OK;
}

int kmp_lp_set_stream(kmp_lp_handle *h, void *cuda_stream) {
  if (h == nullptr) {
    return fail(KMP_ERR_INVALID, "null handle");
  }
  KMP_CUDA(cudaStreamSynchronize(h->stream));
  // 0 is a valid handle (the legacy default stream, which is what torch uses unless told otherwise);
  // (void*)-1 switches back to the handle's own stream
  h->stream = cuda_stream == reinterpret_cast<void *>(-1) ? h->streams.owned : static_cast<cudaStream_t>(cuda_stream);
  h->sweep_stream = h->stream;
  return KMP_OK;
}

uint32_t kmp_lp_num_subrounds(kmp_lp_handle *h) {
  return h != nullptr && h->lists.valid ? kNumGroups * h->lists.S : 0;
}

int kmp_lp_subround_cap(kmp_lp_handle *h, uint32_t sg, uint32_t *cap_out, uint32_t *size_out) {
  if (h == nullptr || !h->lists.valid || sg >= kNumGroups * h->lists.S) {
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
  rc = begin_cluster_run(h, max_cluster_weight, communities, &h->step.run);
  if (rc != KMP_OK) {
    return rc;
  }
  h->step.open = true;
  h->step.iter = 0;
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
  rc = begin_refine_run(h, k, max_block_weights, min_block_weights, communities, partition, &h->step.run);
  if (rc != KMP_OK) {
    return rc;
  }
  h->step.open = true;
  h->step.iter = 0;
  return KMP_OK;
}

int kmp_lp_step_begin_iteration(kmp_lp_handle *h) {
  if (h == nullptr || !h->step.open) {
    return fail(KMP_ERR_INVALID, "step_begin_* not called");
  }
  return begin_iteration(h, h->step.iter);
}

// Sweep this rank's share of sub-round sg and pack its proposals into d_send (device memory,
// 4 + 2 * cap words: [count, -, -, -, u[cap], t[cap]]).
int kmp_lp_step_sweep(kmp_lp_handle *h, uint32_t iter, uint32_t sg, void *d_send) {
  if (h == nullptr || !h->step.open || d_send == nullptr) {
    return fail(KMP_ERR_INVALID, "bad argument");
  }
  if (sg >= kNumGroups * h->lists.S) { // subround_of_sg indexes lists.off by sg
    return fail(KMP_ERR_INVALID, "bad sub-round");
  }
  return dist_sweep_pack(h, h->step.run, iter, sg, subround_of_sg(h, sg), static_cast<uint32_t *>(d_send));
}

// Commit sub-round sg from the all-gathered proposal buffers (world * (4 + 2 * cap) words).
int kmp_lp_step_commit(kmp_lp_handle *h, uint32_t iter, uint32_t sg, const void *d_gathered) {
  if (h == nullptr || !h->step.open || d_gathered == nullptr) {
    return fail(KMP_ERR_INVALID, "bad argument");
  }
  if (sg >= kNumGroups * h->lists.S) {
    return fail(KMP_ERR_INVALID, "bad sub-round");
  }
  return commit_subround(h, h->step.run, iter, sg, subround_of_sg(h, sg), static_cast<const uint32_t *>(d_gathered));
}

int kmp_lp_step_end_iteration(kmp_lp_handle *h, uint32_t *moved) {
  if (h == nullptr || !h->step.open || moved == nullptr) {
    return fail(KMP_ERR_INVALID, "bad argument");
  }
  const int rc = end_iteration(h, moved);
  if (rc != KMP_OK) {
    return rc;
  }
  ++h->step.iter;
  return KMP_OK;
}

// favored[u] ^ u into / out of a caller-provided device buffer of n words (for a MAX all-reduce:
// only the rank that owns u ever writes favored[u]; everybody else still holds u, i.e. 0 here).
int kmp_lp_step_favored_export(kmp_lp_handle *h, void *d_buf) {
  if (h == nullptr || d_buf == nullptr || !h->step.open || h->step.run.mode != 0) {
    return fail(KMP_ERR_INVALID, "bad argument");
  }
  k_xor_iota<<<grid_for(h->graph.n, 256), 256, 0, h->stream>>>(h->graph.n, h->lp.favored.p, static_cast<uint32_t *>(d_buf));
  KMP_CUDA(cudaGetLastError());
  return KMP_OK;
}
int kmp_lp_step_favored_import(kmp_lp_handle *h, const void *d_buf) {
  if (h == nullptr || d_buf == nullptr || !h->step.open || h->step.run.mode != 0) {
    return fail(KMP_ERR_INVALID, "bad argument");
  }
  k_xor_iota<<<grid_for(h->graph.n, 256), 256, 0, h->stream>>>(h->graph.n, static_cast<const uint32_t *>(d_buf), h->lp.favored.p);
  KMP_CUDA(cudaGetLastError());
  return KMP_OK;
}

// Post passes (clusterer) and result download; stats hold THIS rank's share of the scan counters.
int kmp_lp_step_finish(kmp_lp_handle *h, uint32_t *labels_out, int32_t *block_weights_out, kmp_lp_stats *stats) {
  if (h == nullptr || !h->step.open) {
    return fail(KMP_ERR_INVALID, "step_begin_* not called");
  }
  if (stats != nullptr) {
    std::memset(stats, 0, sizeof(*stats));
  }
  const bool cluster = h->step.run.mode == 0;
  int rc = cluster ? finish_cluster_run(h, h->step.run.max_cluster_weight, stats) : KMP_OK;
  if (rc == KMP_OK) {
    rc = download_results(h, labels_out, cluster ? nullptr : block_weights_out, h->step.run.num_labels);
  }
  if (rc != KMP_OK) {
    return rc;
  }
  h->step.open = false;
  return end_call(h, stats);
}

} // extern "C"

#include "kmp_contract.cuh"
#include "kmp_sparsify.cuh"
#include "kmp_overlay.cuh"
#include "kmp_balance.cuh"
#include "kmp_underload.cuh"
#include "kmp_prepare.cuh"
#include "kmp_subgraph.cuh"
#include "kmp_bipartition_dev.cuh"
#include "kmp_validate.cuh"
#include "kmp_read.cuh"
#include "kmp_metis.cuh"
#include "kmp_parhip.cuh"

#ifdef KMP_HUB_PHASE_STAMPS
// scripts/hub_rate_phases.py: reads (and with reset != 0 zeroes) the rate kernel's 7 phase accumulators
// (lp_sweep.cuh, g_hub_phase). Only in a library built with -DKMP_HUB_PHASE_STAMPS.
extern "C" int kmp_hub_phase_read(unsigned long long *out, int reset) {
  if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpyFromSymbol(out, kmp::g_hub_phase, sizeof(kmp::g_hub_phase)) != cudaSuccess) {
    return 1;
  }
  if (reset != 0) {
    const unsigned long long zero[7] = {};
    if (cudaMemcpyToSymbol(kmp::g_hub_phase, zero, sizeof(zero)) != cudaSuccess) {
      return 1;
    }
  }
  return 0;
}
#endif

#ifdef KMP_TEAM_PHASE_STAMPS
// scripts/team_phases.py: reads (and with reset != 0 zeroes) tier 3's 7 phase accumulators (lp_sweep.cuh,
// g_team_phase). Only in a library built with -DKMP_TEAM_PHASE_STAMPS.
extern "C" int kmp_team_phase_read(unsigned long long *out, int reset) {
  if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpyFromSymbol(out, kmp::g_team_phase, 7 * sizeof(unsigned long long)) != cudaSuccess) {
    return 1;
  }
  if (reset != 0) {
    const unsigned long long zero[7] = {};
    if (cudaMemcpyToSymbol(kmp::g_team_phase, zero, sizeof(zero)) != cudaSuccess) {
      return 1;
    }
  }
  return 0;
}
#endif
