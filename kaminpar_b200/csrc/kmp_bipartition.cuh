// KaMinPar's multilevel initial bipartitioner (InitialBipartitionerWorkerPool::bipartition ->
// InitialMultilevelBipartitioner) at one thread, restated as one sequential engine (DESIGN.md §20). Every function is
// plain sequential code marked KMP_HD, so that tests/cpp/ip_host_check.cc compiles the same engine with g++; the
// library runs it in ip_kernel (kmp_bipartition_dev.cuh, kmp_bipartition_subgraphs), lane 0 of one warp per block.
//
// What is restated:
//   InitialMultilevelBipartitioner::partition / coarsen / uncoarsen      initial_multilevel_bipartitioner.cc:81-193
//   InitialCoarsener (LP with chunk shuffles and permutations, rating    coarsening/initial_coarsener.cc:24-454
//     maps in first-insertion order, random_bool ties, locked leaders,
//     contraction with the interleaved LP of the next level)
//   SequentialGraphHierarchy::pop (projection)                           util/sequential_graph_hierarchy.cc:53-103
//   InitialPoolBipartitioner (registration order, adaptive selection,   bipartitioning/initial_pool_bipartitioner.cc
//     best-partition rule with the imbalance tie-break, RunningVariance)
//   BFS (5 block-selection strategies), GGG, random bipartitioners       bipartitioning/initial_*_bipartitioner.cc
//   find_far_away_nodes                                                  util/seed_node_utils.cc
//   InitialFMRefiner (MaxOverload selection, BalancedMinCut acceptance, refinement/initial_fm_refiner.cc
//     simple / adaptive stopping, chunked PQ init, rollback)
//   BinaryMinHeap (4-ary), Marker, Queue, FastResetArray                 kaminpar-common/datastructures/
//   metrics::edge_cut_seq / imbalance / is_feasible / total_overload     metrics.cc, metrics.h
//
// The few doubles left in the engine go through d_add / d_sub / d_mul / d_div / d_sqrt: the correctly rounded
// intrinsics on the device, plain operators on the host, so no contraction into FMA can happen on either side and
// the results are IEEE-identical to g++'s x86-64 SSE code. The doubles of the per-block parameters (pow, ceil of
// quotients) are computed on the host (kmp_ip_params.h).
//
// State lives in one arena per block (Arena, zero-filled before the run): a bump allocator that sets `overflow` and
// makes the run stop instead of writing past its end.
#pragma once

#include <cstdint>

#include "kmp_rng.cuh"

namespace kmp_ip {

using namespace kmp_rng;

// every engine function is inlined into the kernel: out-of-line device calls would need a stack frame
#if defined(__CUDACC__)
#define KMP_IPF __host__ __device__ __forceinline__
#else
#define KMP_IPF inline
#endif

#if defined(__CUDA_ARCH__)
KMP_IPF double d_add(double a, double b) { return __dadd_rn(a, b); }
KMP_IPF double d_sub(double a, double b) { return __dsub_rn(a, b); }
KMP_IPF double d_mul(double a, double b) { return __dmul_rn(a, b); }
KMP_IPF double d_div(double a, double b) { return __ddiv_rn(a, b); }
KMP_IPF double d_sqrt(double a) { return __dsqrt_rn(a); }
KMP_IPF double d_ceil(double a) { return ceil(a); }
#else
inline double d_add(double a, double b) { return a + b; }
inline double d_sub(double a, double b) { return a - b; }
inline double d_mul(double a, double b) { return a * b; }
inline double d_div(double a, double b) { return a / b; }
inline double d_sqrt(double a) { return __builtin_sqrt(a); }
inline double d_ceil(double a) { return __builtin_ceil(a); }
#endif

constexpr uint32_t kCoarsenChunk = 256, kCoarsenPerms = 16; // InitialCoarsener: RandomPermutations<NodeID, 256, 16>
constexpr uint32_t kFmChunk = 64, kFmPerms = 32;             // InitialFMRefiner: RandomPermutations<NodeID, 64, 32>
constexpr int32_t kMaxWeight = 0x7FFFFFFF;

enum : uint32_t { kRefineNoop = 0, kRefineSimpleFm = 1, kRefineAdaptiveFm = 2 };

struct FmParams {
  uint32_t algorithm; // kRefine*
  uint32_t num_fruitless_moves;
  double alpha;
  uint64_t num_iterations;
  double improvement_abortion_threshold;
};

// the call's settings (the same for every block)
struct Config {
  uint32_t contraction_limit;
  double convergence_threshold;
  uint32_t large_degree_threshold;
  FmParams pool_fm, fm;
  int32_t min_num_non_adaptive_repetitions;
  int32_t use_adaptive_bipartitioner_selection;
  int32_t enable_bfs, enable_ggg, enable_random;
  int32_t refine_pool_partition;
};

// one block's parameters, from the reference's double code on the host (kmp_ip_params.h)
struct BlockParams {
  int32_t max_bw[2];      // PartitionContext::max_block_weight after the relaxation
  int32_t perfect_bw[2];  // PartitionContext::perfectly_balanced_block_weight
  int32_t max_cluster_weight;
  int32_t num_repetitions; // already clamped to [min_num_repetitions, max_num_repetitions]
};

struct Counters {
  uint32_t pool_runs;
  uint32_t levels;
};

struct Arena {
  uint8_t *base;
  uint64_t cap, top;
  bool overflow;
  template <typename T> KMP_IPF T *alloc(uint64_t count) {
    const uint64_t bytes = (count * sizeof(T) + 7) & ~7ull;
    if (overflow || top + bytes > cap) {
      overflow = true;
      return nullptr;
    }
    T *p = reinterpret_cast<T *>(base + top);
    top += bytes;
    return p;
  }
};

// One level of the hierarchy. CSRGraph's weight rule: a graph is node (edge) weighted iff n (m) differs from the
// total weight, else every weight reads as 1 (csr_graph.h:92-113).
struct Level {
  uint32_t n, m;
  const uint32_t *xadj, *adj;
  const int32_t *vwgt, *adjwgt;
  int32_t total_nw;
  bool nweighted, eweighted;
  uint32_t *mapping; // [finer level's n] -> vertex of this level; nullptr on the finest level
  Level *finer;
  KMP_IPF int32_t nw(uint32_t u) const { return nweighted ? vwgt[u] : 1; }
  KMP_IPF int32_t ew(uint32_t e) const { return eweighted ? adjwgt[e] : 1; }
};

KMP_IPF void level_weights(Level &L) {
  uint32_t tn = L.n, te = L.m;
  if (L.vwgt != nullptr) {
    tn = 0;
    for (uint32_t u = 0; u < L.n; ++u) {
      tn += static_cast<uint32_t>(L.vwgt[u]);
    }
  }
  if (L.adjwgt != nullptr) {
    te = 0;
    for (uint32_t e = 0; e < L.m; ++e) {
      te += static_cast<uint32_t>(L.adjwgt[e]);
    }
  }
  L.total_nw = static_cast<int32_t>(tn);
  L.nweighted = static_cast<int32_t>(L.n) != L.total_nw;
  L.eweighted = static_cast<int32_t>(L.m) != static_cast<int32_t>(te);
}

// InitialCoarsener::Cluster keeps the weight in a 30-bit signed bit field
KMP_IPF int32_t wrap30(int32_t x) { return static_cast<int32_t>(static_cast<uint32_t>(x) << 2) >> 2; }

KMP_IPF uint32_t floor_log2(uint32_t x) {
  uint32_t r = 0;
  while (x >>= 1) {
    ++r;
  }
  return r;
}

// Marker<K> (marker.h): timestamped bit sets. The reference's 64-bit stamp never wraps; this 32-bit one clears its
// data when it would, which gives the same get() answers.
struct Marker {
  uint32_t *data;
  uint32_t size, id, mask;
  uint32_t first[3];
  KMP_IPF void init(uint32_t *d, uint32_t sz, uint32_t k) {
    data = d;
    size = sz;
    id = 0;
    mask = (1u << k) - 1u;
    first[0] = first[1] = first[2] = 0;
  }
  KMP_IPF bool get(uint32_t e, uint32_t m = 0) const { return (data[e] & ~mask) == id && (data[e] & (1u << m)) != 0; }
  // track: set<true>; bound is the marker's capacity, which is the graph's n wherever it is read
  KMP_IPF void set(uint32_t e, uint32_t m, bool track, uint32_t bound) {
    data[e] = ((data[e] & ~mask) == id) ? (data[e] | (1u << m)) : (id | (1u << m));
    if (track) {
      while (first[m] < bound && get(first[m], m)) {
        ++first[m];
      }
    }
  }
  KMP_IPF void reset() {
    id |= mask;
    id += 1u;
    first[0] = first[1] = first[2] = 0;
    if ((id | mask) == 0xFFFFFFFFu) {
      id = 0;
      for (uint32_t i = 0; i < size; ++i) {
        data[i] = 0;
      }
    }
  }
};

// BinaryMinHeap<EdgeWeight> (binary_heap.h): 4-ary, sift_up always walks to the root. pos1 = position + 1, 0 = absent.
struct Heap {
  uint32_t *id;
  int32_t *key;
  uint32_t *pos1;
  uint32_t size;
  KMP_IPF bool contains(uint32_t v) const { return pos1[v] != 0; }
  KMP_IPF int32_t key_of(uint32_t v) const { return key[pos1[v] - 1]; }
  KMP_IPF void swap_at(uint32_t a, uint32_t b) {
    const uint32_t ti = id[a];
    const int32_t tk = key[a];
    id[a] = id[b];
    key[a] = key[b];
    id[b] = ti;
    key[b] = tk;
    pos1[id[a]] = a + 1;
    pos1[id[b]] = b + 1;
  }
  KMP_IPF void sift_up(uint32_t pos) {
    while (pos != 0) {
      const uint32_t parent = (pos - 1) / 4;
      if (key[parent] > key[pos]) {
        swap_at(pos, parent);
      }
      pos = parent;
    }
  }
  KMP_IPF void sift_down(uint32_t pos) {
    while (true) {
      const uint32_t first_child = 4 * pos + 1;
      if (first_child >= size) {
        return;
      }
      uint32_t smallest = first_child;
      const uint32_t end = (4 * pos + 5 < size) ? 4 * pos + 5 : size;
      for (uint32_t c = first_child + 1; c < end; ++c) {
        if (key[smallest] > key[c]) {
          smallest = c;
        }
      }
      if (key[smallest] >= key[pos]) {
        return;
      }
      swap_at(pos, smallest);
      pos = smallest;
    }
  }
  KMP_IPF void push(uint32_t v, int32_t k) {
    const uint32_t p = size++;
    id[p] = v;
    key[p] = k;
    pos1[v] = p + 1;
    sift_up(p);
  }
  KMP_IPF void pop() {
    --size;
    const uint32_t ti = id[0];
    const int32_t tk = key[0];
    id[0] = id[size];
    key[0] = key[size];
    id[size] = ti;
    key[size] = tk;
    pos1[id[0]] = 1;
    pos1[id[size]] = 0;
    sift_down(0);
  }
  KMP_IPF void decrease_to(uint32_t v, int32_t k) {
    key[pos1[v] - 1] = k;
    sift_up(pos1[v] - 1);
  }
  KMP_IPF void increase_to(uint32_t v, int32_t k) {
    key[pos1[v] - 1] = k;
    sift_down(pos1[v] - 1);
  }
  KMP_IPF void remove(uint32_t v) {
    decrease_to(v, static_cast<int32_t>(0x80000000u));
    pop();
  }
  KMP_IPF void change_priority(uint32_t v, int32_t k) {
    const int32_t old = key_of(v);
    if (k > old) {
      increase_to(v, k);
    } else if (old > k) {
      decrease_to(v, k);
    }
  }
  KMP_IPF void clear() {
    for (uint32_t i = 0; i < size; ++i) {
      pos1[id[i]] = 0;
    }
    size = 0;
  }
};

// a partition of one level with its two block weights
struct Part {
  uint32_t *p;
  int32_t bw[2];
};

// The engine object itself lives at the start of the block's arena, with every array it allocates after it: the
// kernel keeps no per-block state in local memory.
struct Engine {
  Config c;
  BlockParams bp;
  Arena ar;
  Counters cnt;
  RngCore *rng;
  uint32_t *coarsen_perms, *pool_fm_perms, *fm_perms;
  uint32_t n0;

  // InitialCoarsener
  uint32_t *leader;
  int32_t *cweight;
  uint8_t *locked;
  int32_t *rating, *ewc;
  uint32_t *rating_used, *ewc_used;
  uint32_t rating_size = 0, ewc_size = 0;
  uint32_t *cluster_sizes, *lnm, *cluster_nodes, *chunks;
  uint32_t num_moves = 0;
  bool precomputed = false, ilocked = false;
  int32_t imcw = 0;

  // flat bipartitioners and the FM refiners (every structure is empty or reset before each use, so the pool's and
  // the multilevel bipartitioner's objects can share one)
  Marker seed_marker, bfs_marker, ggg_marker, fm_marker;
  uint32_t *queue[2];
  uint32_t qhead[2], qtail[2];
  Heap heap[2];
  int32_t *wdeg;
  uint32_t *moves;
  uint32_t num_moves_fm = 0;
  // AdaptiveStoppingPolicy / SimpleStoppingPolicy
  uint64_t steps = 0;
  double beta = 0.0, variance = 0.0, Mk = 0.0, Mk1 = 0.0, Sk = 0.0, Sk1 = 0.0;
  // the pool's statistics (RunningVariance) and partitions, the partition being projected
  uint32_t kinds[7];
  uint64_t run_count[7];
  double run_mean[7], run_m2[7];
  Part cur, best, proj;
  Level fine;

  // ---- construction: Random::reseed, then the RandomPermutations in member-initialisation order ----------------
  KMP_IPF void draw_perms(uint32_t *t, uint32_t count, uint32_t size) {
    for (uint32_t p = 0; p < count; ++p) {
      for (uint32_t i = 0; i < size; ++i) {
        t[p * size + i] = i;
      }
      shuffle(*rng, t + p * size, size);
    }
  }
  KMP_IPF bool construct(int seed, uint32_t n) {
    n0 = n;
    rng = ar.alloc<RngCore>(1);
    coarsen_perms = ar.alloc<uint32_t>(kCoarsenChunk * kCoarsenPerms);
    pool_fm_perms = ar.alloc<uint32_t>(kFmChunk * kFmPerms);
    fm_perms = ar.alloc<uint32_t>(kFmChunk * kFmPerms);
    leader = ar.alloc<uint32_t>(n + 1);
    cweight = ar.alloc<int32_t>(n + 1);
    locked = ar.alloc<uint8_t>(n + 1);
    rating = ar.alloc<int32_t>(n);
    ewc = ar.alloc<int32_t>(n);
    rating_used = ar.alloc<uint32_t>(n);
    ewc_used = ar.alloc<uint32_t>(n);
    cluster_sizes = ar.alloc<uint32_t>(n);
    lnm = ar.alloc<uint32_t>(n);
    cluster_nodes = ar.alloc<uint32_t>(n);
    chunks = ar.alloc<uint32_t>(n / kFmChunk + 2);
    uint32_t *md0 = ar.alloc<uint32_t>(n), *md1 = ar.alloc<uint32_t>(n), *md2 = ar.alloc<uint32_t>(n),
             *md3 = ar.alloc<uint32_t>(n);
    for (int i = 0; i < 2; ++i) {
      queue[i] = ar.alloc<uint32_t>(n);
      heap[i].id = ar.alloc<uint32_t>(n);
      heap[i].key = ar.alloc<int32_t>(n);
      heap[i].pos1 = ar.alloc<uint32_t>(n);
      heap[i].size = 0;
    }
    wdeg = ar.alloc<int32_t>(n);
    moves = ar.alloc<uint32_t>(n);
    if (ar.overflow) {
      return false;
    }
    seed_marker.init(md0, n, 1);
    bfs_marker.init(md1, n, 3);
    ggg_marker.init(md2, n, 1);
    fm_marker.init(md3, n, 1);
    rng_seed(*rng, seed);
    draw_perms(coarsen_perms, kCoarsenPerms, kCoarsenChunk);
    if (c.pool_fm.algorithm != kRefineNoop) {
      draw_perms(pool_fm_perms, kFmPerms, kFmChunk);
    }
    if (c.fm.algorithm != kRefineNoop) {
      draw_perms(fm_perms, kFmPerms, kFmChunk);
    }
    return true;
  }

  // ---- FastResetArray --------------------------------------------------------------------------------------------
  KMP_IPF void rating_add(uint32_t key, int32_t w) {
    if (rating[key] == 0) {
      rating_used[rating_size++] = key;
    }
    rating[key] += w;
  }
  KMP_IPF void ewc_add(uint32_t key, int32_t w) {
    if (ewc[key] == 0) {
      ewc_used[ewc_size++] = key;
    }
    ewc[key] += w;
  }

  // ---- InitialCoarsener ------------------------------------------------------------------------------------------
  KMP_IPF uint32_t pick_from_rating_map(uint32_t u, int32_t u_weight, int32_t mcw) {
    uint32_t best = u;
    int32_t best_gain = 0;
    for (uint32_t i = 0; i < rating_size; ++i) {
      const uint32_t cluster = rating_used[i];
      const int32_t gain = rating[cluster];
      rating[cluster] = 0;
      const int32_t weight = cweight[cluster];
      if ((gain > best_gain || (gain == best_gain && random_bool(*rng))) && (weight + u_weight <= mcw)) {
        best = cluster;
        best_gain = gain;
      }
    }
    rating_size = 0;
    return best;
  }
  KMP_IPF void handle_node(const Level &L, uint32_t u, int32_t mcw) {
    if (locked[u]) {
      return;
    }
    const int32_t u_weight = L.nw(u);
    for (uint32_t e = L.xadj[u]; e < L.xadj[u + 1]; ++e) {
      rating_add(leader[L.adj[e]], L.ew(e));
    }
    const uint32_t best = pick_from_rating_map(u, u_weight, mcw);
    if (best != u) {
      leader[u] = best;
      locked[best] = 1;
      cweight[best] = wrap30(cweight[best] + u_weight);
      ++num_moves;
    }
  }
  KMP_IPF void reset_clustering(const Level &L) {
    num_moves = 0;
    const int32_t unit = L.nweighted ? 0 : static_cast<int32_t>(L.total_nw / static_cast<int32_t>(L.n));
    for (uint32_t u = 0; u < L.n; ++u) {
      locked[u] = 0;
      leader[u] = u;
      cweight[u] = wrap30(L.nweighted ? L.vwgt[u] : unit);
    }
  }
  KMP_IPF void perform_label_propagation(const Level &L, int32_t mcw) {
    reset_clustering(L);
    // the blocks are unsorted CSR graphs: one degree bucket holding every vertex
    if (floor_log2(c.large_degree_threshold) >= 1 && L.n > 0) {
      const uint32_t num_chunks = L.n / kCoarsenChunk;
      for (uint32_t i = 0; i < num_chunks; ++i) {
        chunks[i] = i * kCoarsenChunk;
      }
      shuffle(*rng, chunks, num_chunks);
      for (uint32_t i = 0; i < num_chunks; ++i) {
        const uint32_t *perm = coarsen_perms + random_index(*rng, 0, kCoarsenPerms) * kCoarsenChunk;
        for (uint32_t j = 0; j < kCoarsenChunk; ++j) {
          handle_node(L, chunks[i] + perm[j], mcw);
        }
      }
      const uint32_t last = L.n % kCoarsenChunk;
      for (uint32_t j = 0; j < last; ++j) {
        handle_node(L, L.n - last + j, mcw);
      }
    }
    precomputed = true;
  }
  KMP_IPF void interleaved_handle_node(uint32_t cu, int32_t cu_weight) {
    if (!ilocked) {
      const uint32_t best = pick_from_rating_map(cu, cu_weight, imcw);
      if (best != cu) {
        ++num_moves;
        leader[cu] = best;
        cweight[best] = wrap30(cweight[best] + cu_weight);
        locked[best] = 1;
      }
    }
    ilocked = locked[cu + 1] != 0; // may read the stale entry c_n, as the reference does
  }
  KMP_IPF void finish_coarse_node(uint32_t &cu, uint32_t &cm, uint32_t *cxadj, uint32_t *cadj, int32_t *cadjwgt,
                                 const int32_t *cvwgt) {
    interleaved_handle_node(cu, cvwgt[cu]);
    for (uint32_t i = 0; i < ewc_size; ++i) {
      const uint32_t cv = ewc_used[i];
      cadj[cm] = cv;
      cadjwgt[cm] = ewc[cv];
      ++cm;
    }
    for (uint32_t i = 0; i < ewc_size; ++i) {
      ewc[ewc_used[i]] = 0;
    }
    ewc_size = 0;
    cxadj[++cu] = cm;
  }
  // contract_current_clustering (initial_coarsener.cc:186-406); nullptr on arena overflow
  KMP_IPF Level *contract(Level &L) {
    const uint32_t n = L.n;
    const uint32_t cn = n - num_moves;
    Level *C = ar.alloc<Level>(1);
    uint32_t *mapping = ar.alloc<uint32_t>(n);
    uint32_t *cxadj = ar.alloc<uint32_t>(cn + 1);
    int32_t *cvwgt = ar.alloc<int32_t>(cn);
    // the reference overcommits m entries for the edges; the weights are moved down behind them at the end
    uint32_t *cadj = ar.alloc<uint32_t>(2ull * L.m);
    if (ar.overflow) {
      return nullptr;
    }
    int32_t *cadjwgt = reinterpret_cast<int32_t *>(cadj + L.m);
    for (uint32_t u = 0; u < n; ++u) {
      cluster_sizes[u] = 0;
      lnm[u] = 0;
    }
    uint32_t current = 0;
    for (uint32_t u = 0; u < n; ++u) {
      const uint32_t ld = leader[u];
      if (lnm[ld] == 0) {
        cvwgt[current] = cweight[ld];
        lnm[ld] = ++current;
      }
      const uint32_t cluster = lnm[ld] - 1;
      mapping[u] = cluster;
      ++cluster_sizes[cluster];
    }
    uint32_t counter = 0;
    for (uint32_t u = 0; u < n; ++u) {
      const uint32_t s = cluster_sizes[u];
      cluster_sizes[u] = counter;
      counter += s;
    }
    for (uint32_t u = 0; u < n; ++u) {
      cluster_nodes[cluster_sizes[mapping[u]]++] = u;
    }
    num_moves = 0; // reset_current_clustering(c_n, c_node_weights)
    for (uint32_t u = 0; u < cn; ++u) {
      locked[u] = 0;
      leader[u] = u;
      cweight[u] = wrap30(cvwgt[u]);
    }
    uint32_t cu = 0, cm = 0;
    cxadj[0] = 0;
    for (uint32_t i = 0; i < n; ++i) {
      const uint32_t u = cluster_nodes[i];
      if (mapping[u] != cu) {
        finish_coarse_node(cu, cm, cxadj, cadj, cadjwgt, cvwgt);
      }
      for (uint32_t e = L.xadj[u]; e < L.xadj[u + 1]; ++e) {
        const uint32_t cv = mapping[L.adj[e]];
        const int32_t w = L.ew(e);
        if (cu != cv) {
          ewc_add(cv, w);
          if (!ilocked) {
            rating_add(leader[cv], w);
          }
        }
      }
    }
    finish_coarse_node(cu, cm, cxadj, cadj, cadjwgt, cvwgt);
    for (uint32_t e = 0; e < cm; ++e) {
      cadj[cm + e] = static_cast<uint32_t>(cadjwgt[e]);
    }
    ar.top -= ((2ull * L.m * 4 + 7) & ~7ull) - ((2ull * cm * 4 + 7) & ~7ull); // give back the unused overcommit
    C->n = cn;
    C->m = cm;
    C->xadj = cxadj;
    C->adj = cadj;
    C->vwgt = cvwgt;
    C->adjwgt = reinterpret_cast<int32_t *>(cadj + cm);
    C->mapping = mapping;
    C->finer = &L;
    level_weights(*C);
    return C;
  }
  // InitialCoarsener::coarsen: the same level when it converged, nullptr on arena overflow
  KMP_IPF Level *coarsen(Level *L, int32_t mcw) {
    if (!precomputed) {
      perform_label_propagation(*L, mcw);
    }
    const uint32_t cn = L->n - num_moves;
    const bool converged =
        d_sub(1.0, d_div(static_cast<double>(cn), static_cast<double>(L->n))) <= c.convergence_threshold;
    if (!converged) {
      imcw = mcw;
      return contract(*L);
    }
    return L;
  }

  // ---- metrics ---------------------------------------------------------------------------------------------------
  KMP_IPF int32_t edge_cut(const Level &L, const uint32_t *p) const {
    int64_t cut = 0;
    for (uint32_t u = 0; u < L.n; ++u) {
      for (uint32_t e = L.xadj[u]; e < L.xadj[u + 1]; ++e) {
        cut += (p[u] != p[L.adj[e]]) ? L.ew(e) : 0;
      }
    }
    return static_cast<int32_t>(cut / 2);
  }
  KMP_IPF double imbalance(const Level &L, const Part &P) const {
    const double perfect = d_ceil(d_div(static_cast<double>(L.total_nw), 2.0));
    double mx = 0.0;
    for (int b = 0; b < 2; ++b) {
      const double x = d_sub(d_div(static_cast<double>(P.bw[b]), perfect), 1.0);
      mx = (mx < x) ? x : mx;
    }
    return mx;
  }
  KMP_IPF bool is_feasible(const Part &P) const { return P.bw[0] <= bp.max_bw[0] && P.bw[1] <= bp.max_bw[1]; }
  KMP_IPF int32_t total_overload(const Part &P) const {
    int32_t o = 0;
    for (int b = 0; b < 2; ++b) {
      const int32_t d = P.bw[b] - bp.max_bw[b];
      o += d > 0 ? d : 0;
    }
    return o;
  }
  KMP_IPF void set_block(const Level &L, Part &P, uint32_t u, uint32_t to) {
    const int32_t w = L.nw(u);
    P.bw[P.p[u]] -= w;
    P.bw[to] += w;
    P.p[u] = to;
  }

  // ---- InitialFMRefiner ------------------------------------------------------------------------------------------
  KMP_IPF void fm_init(const Level &L, const FmParams &f) {
    if (f.algorithm == kRefineNoop) {
      return;
    }
    beta = d_sqrt(static_cast<double>(L.n));
    steps = 0;
    variance = 0.0;
    for (uint32_t u = 0; u < L.n; ++u) {
      int32_t d = 0;
      for (uint32_t e = L.xadj[u]; e < L.xadj[u + 1]; ++e) {
        d += L.ew(e);
      }
      wdeg[u] = d;
    }
  }
  KMP_IPF bool should_stop(const FmParams &f) const {
    if (f.algorithm == kRefineSimpleFm) {
      return steps > f.num_fruitless_moves;
    }
    const double factor = d_sub(d_div(f.alpha, 2.0), 0.25);
    const double s = static_cast<double>(steps);
    return (s > beta) && ((Mk == 0) || (s >= d_mul(d_div(variance, d_mul(Mk, Mk)), factor)));
  }
  KMP_IPF void stop_update(const FmParams &f, int32_t gain) {
    ++steps;
    if (f.algorithm != kRefineAdaptiveFm) {
      return;
    }
    const double g = static_cast<double>(gain);
    if (steps == 1) {
      Mk1 = g;
      Mk = Mk1;
      Sk1 = 0.0;
    } else {
      Mk = d_add(Mk1, d_div(d_sub(g, Mk1), static_cast<double>(steps)));
      Sk = d_add(Sk1, d_mul(d_sub(g, Mk1), d_sub(g, Mk)));
      variance = d_div(Sk, d_sub(static_cast<double>(steps), 1.0));
      Mk1 = Mk;
      Sk1 = Sk;
    }
  }
  KMP_IPF void stop_reset() {
    steps = 0;
    variance = 0.0;
  }
  // MaxOverloadSelectionPolicy -> MaxGainSelectionPolicy -> MaxWeightSelectionPolicy
  KMP_IPF uint32_t select_queue(const Part &P) {
    const int32_t d0 = P.bw[0] - bp.max_bw[0], d1 = P.bw[1] - bp.max_bw[1];
    const int32_t o0 = d0 > 0 ? d0 : 0, o1 = d1 > 0 ? d1 : 0;
    if (o0 == 0 && o1 == 0) {
      const int32_t l0 = heap[0].size == 0 ? kMaxWeight : heap[0].key[0];
      const int32_t l1 = heap[1].size == 0 ? kMaxWeight : heap[1].key[0];
      if (l0 == l1) {
        const int32_t w0 = P.bw[0] - bp.perfect_bw[0], w1 = P.bw[1] - bp.perfect_bw[1];
        return w1 > w0 || (w0 == w1 && random_bool(*rng));
      }
      return l1 < l0;
    }
    return o1 > o0 || (o1 == o0 && random_bool(*rng));
  }
  KMP_IPF void init_pq(const Level &L, const Part &P, const uint32_t *perms) {
    const uint32_t num_chunks = L.n / kFmChunk + 1;
    for (uint32_t i = 0; i < num_chunks; ++i) {
      chunks[i] = i * kFmChunk;
    }
    shuffle(*rng, chunks, num_chunks);
    for (uint32_t i = 0; i < num_chunks; ++i) {
      const uint32_t *perm = perms + random_index(*rng, 0, kFmPerms) * kFmChunk;
      for (uint32_t j = 0; j < kFmChunk; ++j) {
        const uint32_t u = chunks[i] + perm[j];
        if (u < L.n) {
          int32_t ext = 0;
          for (uint32_t e = L.xadj[u]; e < L.xadj[u + 1]; ++e) {
            ext += (P.p[L.adj[e]] != P.p[u]) * L.ew(e);
          }
          const int32_t gain = (wdeg[u] - ext) - ext;
          if (wdeg[u] != gain) {
            heap[P.p[u]].push(u, gain);
          }
        }
      }
    }
  }
  KMP_IPF int32_t fm_round(const Level &L, Part &P, const FmParams &f, const uint32_t *perms) {
    stop_reset();
    init_pq(L, P, perms);
    int32_t current_overload = total_overload(P);
    int32_t accepted_overload = current_overload;
    int32_t current_delta = 0, accepted_delta = 0;
    while ((heap[0].size != 0 || heap[1].size != 0) && !should_stop(f)) {
      uint32_t active = select_queue(P);
      if (heap[active].size == 0) {
        active = 1 - active;
      }
      Heap &q = heap[active];
      const uint32_t u = q.id[0];
      const int32_t delta = q.key[0];
      const uint32_t to = 1 - active;
      fm_marker.set(u, 0, false, 0);
      q.pop();
      set_block(L, P, u, to);
      current_delta += delta;
      moves[num_moves_fm++] = u;
      stop_update(f, -delta);
      current_overload = total_overload(P);
      for (uint32_t e = L.xadj[u]; e < L.xadj[u + 1]; ++e) {
        const uint32_t v = L.adj[e];
        if (fm_marker.get(v)) {
          continue;
        }
        const uint32_t vb = P.p[v];
        const int32_t loss_delta = 2 * L.ew(e) * ((to == vb) ? 1 : -1);
        if (heap[vb].contains(v)) {
          const int32_t new_loss = heap[vb].key_of(v) + loss_delta;
          if (!(new_loss < wdeg[v])) {
            heap[vb].remove(v);
          } else {
            heap[vb].change_priority(v, new_loss);
          }
        } else {
          heap[vb].push(v, wdeg[v] + loss_delta);
        }
      }
      if (current_overload <= accepted_overload && current_delta < accepted_delta) {
        stop_reset();
        accepted_delta = current_delta;
        accepted_overload = current_overload;
        num_moves_fm = 0;
      }
    }
    for (uint32_t i = 0; i < num_moves_fm; ++i) {
      set_block(L, P, moves[i], 1 - P.p[moves[i]]);
    }
    heap[0].clear();
    heap[1].clear();
    fm_marker.reset();
    num_moves_fm = 0;
    return accepted_delta;
  }
  KMP_IPF void fm_refine(const Level &L, Part &P, const FmParams &f, const uint32_t *perms) {
    if (f.algorithm == kRefineNoop) {
      return;
    }
    if (f.num_iterations == 1) {
      fm_round(L, P, f, perms);
      return;
    }
    const int32_t initial = edge_cut(L, P.p);
    if (initial == 0) {
      return;
    }
    int32_t prev = initial, cur = initial;
    cur += fm_round(L, P, f, perms);
    for (uint64_t it = 1; 0 < cur && it < f.num_iterations &&
                          !(d_sub(1.0, d_div(static_cast<double>(cur), static_cast<double>(prev))) <
                            f.improvement_abortion_threshold);
         ++it) {
      prev = cur;
      cur += fm_round(L, P, f, perms);
    }
  }

  // ---- flat bipartitioners ---------------------------------------------------------------------------------------
  KMP_IPF void flat_set(const Level &L, Part &P, uint32_t u, uint32_t b) {
    P.p[u] = b;
    P.bw[b] += L.nw(u);
  }
  // find_furthest_away_node (seed_node_utils.cc:21-68); queue 0 doubles as the BFS queue
  KMP_IPF void furthest(const Level &L, uint32_t start, uint32_t &last, uint32_t &dist) {
    uint32_t *q = queue[0];
    uint32_t head = 0, tail = 0;
    q[tail++] = start;
    seed_marker.set(start, 0, true, L.n);
    uint32_t current_distance = 0, remaining = 1, next = 0;
    last = start;
    while (head != tail) {
      const uint32_t u = q[head++];
      last = u;
      for (uint32_t e = L.xadj[u]; e < L.xadj[u + 1]; ++e) {
        const uint32_t v = L.adj[e];
        if (seed_marker.get(v)) {
          continue;
        }
        q[tail++] = v;
        seed_marker.set(v, 0, true, L.n);
        ++next;
      }
      if (--remaining == 0) {
        ++current_distance;
        remaining = next;
        next = 0;
      }
    }
    --current_distance;
    if (seed_marker.first[0] < L.n) {
      last = seed_marker.first[0];
      current_distance = 0xFFFFFFFFu;
    }
    seed_marker.reset();
    dist = current_distance;
  }
  KMP_IPF void bfs_fill(const Level &L, Part &P, int32_t num_seed_iterations, uint32_t strategy) {
    seed_marker.reset();
    uint32_t best_distance = 0, start_a = 0, start_b = 0;
    for (int32_t i = 0; i < num_seed_iterations; ++i) {
      const uint32_t u = random_index(*rng, 0, L.n);
      uint32_t v, d;
      furthest(L, u, v, d);
      if (d > best_distance || (d == best_distance && random_bool(*rng))) {
        best_distance = d;
        start_a = u;
        start_b = v;
      }
    }
    Marker &mk = bfs_marker;
    mk.reset();
    qhead[0] = qtail[0] = qhead[1] = qtail[1] = 0;
    queue[0][qtail[0]++] = start_a;
    queue[1][qtail[1]++] = start_b;
    mk.set(start_a, 0, true, L.n);
    mk.set(start_b, 1, true, L.n);
    uint32_t active = 0;
    while (mk.first[2] < L.n) {
      if (qhead[active] == qtail[active]) {
        const uint32_t f = mk.first[2];
        if (mk.get(f, active)) {
          active = 1 - active;
          continue;
        }
        queue[active][qtail[active]++] = f;
        mk.set(f, active, false, L.n);
      }
      const uint32_t u = queue[active][qhead[active]++];
      if (!mk.get(u, 2)) {
        const bool allowed = P.bw[active] + L.nw(u) <= bp.max_bw[active];
        active = allowed ? active : 1 - active;
        flat_set(L, P, u, active);
        mk.set(u, 2, true, L.n);
        for (uint32_t e = L.xadj[u]; e < L.xadj[u + 1]; ++e) {
          const uint32_t v = L.adj[e];
          if (mk.get(v, 2) || mk.get(v, active)) {
            continue;
          }
          queue[active][qtail[active]++] = v;
          mk.set(v, active, false, L.n);
        }
      }
      const uint32_t s0 = qtail[0] - qhead[0], s1 = qtail[1] - qhead[1];
      switch (strategy) {
      case 0: active = 1 - active; break;                                  // alternating
      case 1: active = (P.bw[0] < P.bw[1]) ? 0 : 1; break;                 // lighter
      case 2: active = (s0 < s1) ? 1 : 0; break;                           // longer_queue
      case 3: active = (s0 < s1) ? 0 : 1; break;                           // shorter_queue
      default: active = (P.bw[0] < bp.perfect_bw[0]) ? 0 : 1; break;       // sequential
      }
    }
  }
  // InitialGGGBipartitioner::fill_bipartition: its neighbour lambda tests _partition[u] == V2 right after
  // change_block(u, V2) and returns, so no neighbour is ever queued and the queue only ever holds the start node.
  KMP_IPF void ggg_fill(const Level &L, Part &P) {
    ggg_marker.reset();
    for (uint32_t u = 0; u < L.n; ++u) {
      P.p[u] = 0;
    }
    P.bw[0] = L.total_nw;
    do {
      uint32_t start = 0, counter = 0;
      do {
        start = random_index(*rng, 0, L.n);
        ++counter;
      } while (ggg_marker.get(start) && counter < 5);
      if (ggg_marker.get(start)) {
        start = ggg_marker.first[0];
      }
      if (start >= L.n) {
        break;
      }
      ggg_marker.set(start, 0, true, L.n);
      const int32_t w = L.nw(start);
      P.p[start] = 1;
      P.bw[1] += w;
      P.bw[0] -= w;
    } while (P.bw[1] < bp.perfect_bw[1]);
  }
  KMP_IPF void random_fill(const Level &L, Part &P) {
    for (uint32_t u = 0; u < L.n; ++u) {
      const uint32_t b = random_index(*rng, 0, 2);
      if (P.bw[b] + L.nw(u) < bp.perfect_bw[b]) {
        flat_set(L, P, u, b);
      } else {
        const int32_t d1 = P.bw[0] - bp.perfect_bw[0], d2 = P.bw[1] - bp.perfect_bw[1];
        flat_set(L, P, u, d1 < d2 ? 0 : 1);
      }
    }
  }

  // ---- InitialPoolBipartitioner ----------------------------------------------------------------------------------
  // the pool's result is left in `best`
  KMP_IPF bool pool(const Level &L, int32_t num_seed_iterations) {
    uint32_t num = 0;
    if (c.enable_bfs) { // alternating, lighter, longer queue, shorter queue, sequential
      for (uint32_t i = 0; i < 5; ++i) {
        kinds[num++] = i;
      }
    }
    if (c.enable_ggg) {
      kinds[num++] = 5;
    }
    if (c.enable_random) {
      kinds[num++] = 6;
    }
    for (uint32_t i = 0; i < 7; ++i) {
      run_count[i] = 0;
      run_mean[i] = run_m2[i] = 0.0;
    }
    cur.p = ar.alloc<uint32_t>(L.n);
    best.p = ar.alloc<uint32_t>(L.n);
    if (ar.overflow) {
      return false;
    }
    best.bw[0] = best.bw[1] = 0;
    fm_init(L, c.pool_fm);
    bool best_feasible = false;
    int32_t best_cut = kMaxWeight;
    double best_imbalance = 0.0;
    for (int32_t rep = 0; rep < bp.num_repetitions; ++rep) {
      for (uint32_t i = 0; i < num; ++i) {
        if (rep >= c.min_num_non_adaptive_repetitions && c.use_adaptive_bipartitioner_selection) {
          // likely_to_improve: RunningVariance::get
          double mn, var;
          if (run_count[i] == 0) {
            mn = 1.7976931348623157e308;
            var = 0.0;
          } else if (run_count[i] < 2) {
            mn = run_mean[i];
            var = 0.0;
          } else {
            mn = run_mean[i];
            var = d_div(run_m2[i], static_cast<double>(run_count[i]));
          }
          const double rhs = d_div(d_sub(mn, static_cast<double>(best_cut)), 2.0);
          if (!(var > d_mul(rhs, rhs))) {
            continue;
          }
        }
        cur.bw[0] = cur.bw[1] = 0;
        if (kinds[i] < 5) {
          bfs_fill(L, cur, num_seed_iterations, kinds[i]);
        } else if (kinds[i] == 5) {
          ggg_fill(L, cur);
        } else {
          random_fill(L, cur);
        }
        fm_refine(L, cur, c.pool_fm, pool_fm_perms);
        ++cnt.pool_runs;
        const int32_t cut = edge_cut(L, cur.p);
        const double imb = imbalance(L, cur);
        const bool feasible = is_feasible(cur);
        if (feasible) {
          ++run_count[i];
          const double value = static_cast<double>(cut);
          const double delta = d_sub(value, run_mean[i]);
          run_mean[i] = d_add(run_mean[i], d_div(delta, static_cast<double>(run_count[i])));
          run_m2[i] = d_add(run_m2[i], d_mul(delta, d_sub(value, run_mean[i])));
        }
        if (best_feasible <= feasible &&
            (best_feasible < feasible || cut < best_cut || (cut == best_cut && imb < best_imbalance))) {
          best_cut = cut;
          best_imbalance = imb;
          best_feasible = feasible;
          uint32_t *const tp = cur.p;
          cur.p = best.p;
          best.p = tp;
          const int32_t t0 = cur.bw[0], t1 = cur.bw[1];
          cur.bw[0] = best.bw[0];
          cur.bw[1] = best.bw[1];
          best.bw[0] = t0;
          best.bw[1] = t1;
        }
      }
    }
    return true;
  }

  // ---- InitialMultilevelBipartitioner::partition ------------------------------------------------------------------
  // writes the finest partition to out[0, n); false on arena overflow
  KMP_IPF bool run(int32_t num_seed_iterations, uint32_t *out) {
    fm_init(fine, c.fm); // _refiner->init(graph) in initialize()
    Level *cg = &fine;
    bool shrunk = true;
    while (shrunk && cg->n > c.contraction_limit) {
      Level *ng = coarsen(cg, bp.max_cluster_weight);
      if (ng == nullptr) {
        return false;
      }
      shrunk = ng != cg;
      if (shrunk) {
        cg = ng;
        ++cnt.levels;
      }
    }
    if (!pool(*cg, num_seed_iterations)) {
      return false;
    }
    if (c.refine_pool_partition) {
      fm_init(*cg, c.fm);
      fm_refine(*cg, best, c.fm, fm_perms);
    }
    proj = best;
    while (cg != &fine) {
      Level *fg = cg->finer;
      uint32_t *fp = (fg == &fine) ? out : ar.alloc<uint32_t>(fg->n);
      if (ar.overflow) {
        return false;
      }
      const uint32_t *cp = proj.p;
      proj.p = fp;
      proj.bw[0] = proj.bw[1] = 0;
      for (uint32_t u = 0; u < fg->n; ++u) {
        fp[u] = cp[cg->mapping[u]];
        proj.bw[fp[u]] += fg->nw(u);
      }
      cg = fg;
      fm_init(*cg, c.fm);
      fm_refine(*cg, proj, c.fm, fm_perms);
    }
    if (proj.p != out) {
      for (uint32_t u = 0; u < fine.n; ++u) {
        out[u] = proj.p[u];
      }
    }
    return true;
  }
};

// One block from its CSR arrays (vwgt / adjwgt nullable), in the zero-filled arena [base, base + cap) (8-byte
// aligned). Returns false when the arena is too small; out is then incomplete and the block must be run again with a
// larger arena. cnt receives the block's pool runs and coarsening levels.
KMP_IPF bool bipartition_block(uint32_t n, uint32_t m, const uint32_t *xadj, const uint32_t *adj,
                                     const int32_t *vwgt, const int32_t *adjwgt, const Config &c,
                                     int32_t num_seed_iterations, const BlockParams &bp, int seed, uint8_t *base,
                                     uint64_t cap, uint32_t *out, Counters &cnt) {
  const uint64_t self = (sizeof(Engine) + 7) & ~7ull;
  if (cap < self) {
    return false;
  }
  Engine *e = reinterpret_cast<Engine *>(base); // zero-filled: every member starts at 0 / false / nullptr
  e->c = c;
  e->bp = bp;
  e->ar.base = base;
  e->ar.cap = cap;
  e->ar.top = self;
  e->ar.overflow = false;
  bool ok = e->construct(seed, n);
  if (ok) {
    Level &f = e->fine;
    f.n = n;
    f.m = m;
    f.xadj = xadj;
    f.adj = adj;
    f.vwgt = vwgt;
    f.adjwgt = adjwgt;
    f.mapping = nullptr;
    f.finer = nullptr;
    level_weights(f);
    ok = e->run(num_seed_iterations, out);
  }
  cnt = e->cnt;
  return ok;
}

// A first arena bound in bytes for a block of n vertices and m directed edges. The coarse levels usually take a
// fraction of it; a block that needs more is run again with a doubled bound.
KMP_IPF uint64_t arena_bound(uint32_t n, uint32_t m) {
  return 65536ull + 160ull * (static_cast<uint64_t>(n) + 8) + 24ull * m;
}

} // namespace kmp_ip
