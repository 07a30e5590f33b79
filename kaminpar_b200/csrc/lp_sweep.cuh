// The LP sweep kernels: one kernel family per degree group of the sync schedule.
//
//   tier 0 (deg 1..7)      sweep_thread<N=8>  : one thread per vertex, neighbour labels sorted in registers
//   tier 1 (deg 8..16)     sweep_thread<N=16>
//   tier 2 (deg 17..31)    sweep_thread<N=32>
//   tier 3 (deg 32..255)   sweep_team<T=32>   : one warp per vertex, 512-slot shared-memory hash map
//   tier 4 (deg 256..1023) sweep_team<T=128>  : 128 threads per vertex, 2048 slots
//   tier 5 (deg 1024..4095) sweep_team<T=512> : one 512-thread CTA per vertex, 8192 slots
//   tier 6 (deg 4096..8191, or ..16383 with unit edge weights: 16-bit ratings) sweep_team<T=1024>: one
//                          1024-thread CTA per vertex, 16384 / 32768 slots
//   tier 7 (deg >= 8192 / 16384) sweep_hub_*  : clusterer: staged labels rated per hash class, one CTA per class;
//                          refiner: edge-parallel chunks, label-partitioned bucket appends (see below)
//   (tiers 1-2 are degree group 1 of the schedule, tiers 4..7 group 3)
//
// Each of them restates label_propagation.h:460-541 (find_best_cluster): accumulate
// rating[label[v]] += w(u,v) over adj(u) (:487-505), clear active[u] (:507-508), select
// (lp_clusterer.cc:181-250 / lp_refiner.cc:151-245) and -- instead of moving immediately
// (try_node_move :817-841) -- emit a proposal (u, target) that the commit kernels resolve.
#pragma once

#include "lp_device.cuh"
#include "lp_sortnet.cuh"

namespace kmp {

// ---- proposal emission --------------------------------------------------------------------------
template <int MODE>
__device__ __forceinline__ void emit_proposal(const SweepArgs &a, uint32_t idx, uint32_t u, uint32_t target,
                                              int32_t uw) {
  a.mv_u[idx] = u;
  a.mv_t[idx] = target;
  if (!a.accumulate) {
    return; // sharded run: incoming[] / hist[] are accumulated over the gathered proposals
  }
  if (MODE == 0) {
    atomicAdd(&a.incoming[target], uw);
  } else {
    const uint32_t lvl = ladder_level(bijective32(u, a.base_commit));
    atomicAdd(&a.hist[target * kLadderLevels + lvl], uw);
  }
}

__device__ __forceinline__ void block_count_flush(const SweepArgs &a, unsigned long long edges,
                                                  unsigned long long nodes) {
  // warp-level then one atomic per warp
  for (int o = 16; o > 0; o >>= 1) {
    edges += __shfl_xor_sync(kFull, edges, o);
    nodes += __shfl_xor_sync(kFull, nodes, o);
  }
  if ((threadIdx.x & 31) == 0 && nodes != 0) {
    atomicAdd(&a.counters[0], edges); // counters points at this degree group's slot
    atomicAdd(&a.counters[kCounterNodesOffset], nodes);
  }
}

// ---- neighbour access ---------------------------------------------------------------------------
template <bool P64>
__device__ __forceinline__ typename LabG<P64>::word load_labg(const SweepArgs &a, uint32_t v) {
  return static_cast<const typename LabG<P64>::word *>(a.labg)[v];
}

// ================================================================================================
// tiers 0..2: thread per vertex, deg <= N (N = 8, 16, 32). The neighbour labels are gathered into N
// registers (N independent gathers in flight per thread), sorted there with Batcher's odd-even merge network
// (fully unrolled: 19 / 63 / 191 compare-exchanges of two instructions each, no divergence -- empty slots
// hold 0xFFFFFFFF and sort to the end), and the ratings are the run lengths of the sorted sequence. Per vertex this
// costs a few hundred to ~1500 thread instructions (20-50 per edge) where a warp-wide hash-map kernel spends
// ~250 per edge (N = 64 was tried too: 230 registers, slower than the warp kernel on deg 32..64), and consecutive list entries have consecutive adjacency rows, so the per-thread row reads share
// sectors across the warp.
// ================================================================================================
// The static inputs of one list entry: vertex, CSR row and (R > 0) its first R neighbour ids. None of them
// depends on the labels, so the persistent low-degree kernel (lp_lowgroup.cuh) loads them ahead, across the
// commit of the running sub-round. sweep_thread uses R = 0 and reads the ids in its gather loop.
template <int R> struct ThreadRow {
  uint32_t u, beg, deg;
  uint32_t v[R > 0 ? R : 1];
};
template <int R> __device__ __forceinline__ void load_row(const SweepArgs &a, ThreadRow<R> &r) {
  r.beg = a.xadj[r.u];
  const uint32_t deg = a.xadj[r.u + 1] - r.beg;
  r.deg = deg > a.max_num_neighbors ? a.max_num_neighbors : deg;
#pragma unroll
  for (int j = 0; j < R; ++j) {
    r.v[j] = j < static_cast<int>(r.deg) ? a.adjncy[r.beg + j] : 0u;
  }
}

// Rating, selection and final action of one vertex of degree <= N whose row is loaded (R = 0 or R >= N); `flag`
// is its active flag. Returns whether it proposes the move u -> target.
template <int MODE, bool EW, bool P64, int N, int R>
__device__ __forceinline__ bool sweep_thread_vertex(const SweepArgs &a, const ThreadRow<R> &r, bool flag,
                                                    unsigned long long &edges, unsigned long long &nodes,
                                                    uint32_t &target, int32_t &uw) {
  const uint32_t u = r.u;
  const uint32_t own = a.label[u];
  uw = a.vwgt != nullptr ? a.vwgt[u] : 1;
  const int32_t own_w = a.weight[own];
  uint32_t keys[N];
  int32_t ws[N];
  bool hit = false;
#pragma unroll
  for (int j = 0; j < N; ++j) {
    keys[j] = kEmpty;
    ws[j] = 0;
    if (j < static_cast<int>(r.deg)) {
      const uint32_t v = R > 0 ? r.v[j] : a.adjncy[r.beg + j];
      const typename LabG<P64>::word g = load_labg<P64>(a, v);
      hit = hit || stamp_hit(LabG<P64>::stamp(g), a.window);
      bool ok = true;
      if (MODE == 1 && a.communities != nullptr) {
        ok = a.communities[u] == a.communities[v];
      }
      if (ok) {
        keys[j] = LabG<P64>::label(g);
        ws[j] = EW ? a.adjwgt[r.beg + j] : 1;
      }
    }
  }
  if (!(flag || hit)) {
    return false;
  }
  edges += r.deg;
  nodes += 1;
  if (a.active != nullptr && flag) {
    a.active[u] = 0;
  }
  bool skip = false;
  if (MODE == 1) {
    const int32_t mn = a.min_w != nullptr ? a.min_w[own] : 0;
    skip = (own_w - uw) < mn; // lp_refiner.cc:160-162
  }
  const bool store_fav = (MODE == 0) && (uw == own_w) && (own_w <= a.max_cluster_weight / 2);
  Cand best = cand_none(), fav = cand_none();
  if (!skip) {
    sort_registers<N, EW>(keys, ws);
    bool lazy_done = false;
    if (MODE == 0) {
      // Clusterer: rank the candidates WITHOUT their cluster weights (one random gather each, DRAM-resident
      // on large graphs); only the top one is checked. If it is full, fall through to the full evaluation.
      // A run rated below the running maximum cannot win: its tie hashes are never computed.
      Cand top = cand_none();
      int32_t run = 0;
#pragma unroll
      for (int j = 0; j < N; ++j) {
        run += EW ? ws[j] : 1;
        const bool last = (j == N - 1) || (keys[j + 1 < N ? j + 1 : j] != keys[j]);
        if (last) {
          const int32_t rating = run;
          run = 0;
          if (keys[j] != kEmpty && rating > 0) {
            if (rating >= top.gain) {
              const Cand x{rating, 0, tie_hash(a.base_tie, u, keys[j]), keys[j]};
              if (cand_better<0>(x, top)) {
                top = x;
              }
            }
            if (store_fav && rating >= fav.gain) {
              const Cand y{rating, 0, tie_hash(a.base_fav, u, keys[j]), keys[j]};
              if (cand_better<0>(y, fav)) {
                fav = y;
              }
            }
          }
        }
      }
      bool top_ok = true;
      if (top.gain > 0) {
        top_ok = (a.weight[top.key] + uw <= a.max_cluster_weight) || (top.key == own);
        if (a.communities != nullptr) {
          top_ok = top_ok && (a.communities[top.key] == a.communities[own]);
        }
      }
      if (top_ok) {
        best = top;
        lazy_done = true;
      }
    }
    if (!lazy_done) {
      int32_t run = 0;
#pragma unroll
      for (int j = 0; j < N; ++j) {
        run += EW ? ws[j] : 1;
        const bool last = (j == N - 1) || (keys[j + 1 < N ? j + 1 : j] != keys[j]);
        if (last) {
          const int32_t rating = run;
          run = 0;
          if (keys[j] != kEmpty) {
            Cand f;
            const Cand c = eval_candidate<MODE>(a, u, own, uw, own_w, keys[j], rating, MODE == 0 ? false : store_fav, f);
            if (cand_better<MODE>(c, best)) {
              best = c;
            }
          }
        }
      }
    }
  }
  return finish_vertex<MODE>(a, u, own, store_fav, best, fav, target);
}

// ONE atomic on the proposal counter per CTA iteration (256 vertices): on graphs that live in the thread tiers
// (grid, road) nearly every vertex proposes in round 0 and the single address serialises in L2. Every thread of
// the 256-thread CTA calls it once per iteration `it`; s_cnt / s_base are double-buffered by its parity.
template <int MODE>
__device__ __forceinline__ void emit_cta_iteration(const SweepArgs &a, bool proposes, uint32_t u, uint32_t target,
                                                   int32_t uw, uint32_t it, uint32_t (&s_cnt)[2][8],
                                                   uint32_t (&s_base)[2]) {
  const unsigned ballot = __ballot_sync(kFull, proposes);
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int par = it & 1;
  if (lane == 0) {
    s_cnt[par][wib] = static_cast<uint32_t>(__popc(ballot));
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t total = 0;
    for (int w = 0; w < 8; ++w) {
      total += s_cnt[par][w];
    }
    s_base[par] = total != 0 ? atomicAdd(a.mover_count, total) : 0u;
  }
  __syncthreads();
  if (proposes) {
    uint32_t idx = s_base[par] + __popc(ballot & ((1u << lane) - 1u));
    for (int w = 0; w < wib; ++w) {
      idx += s_cnt[par][w];
    }
    emit_proposal<MODE>(a, idx, u, target, uw);
  }
}

template <int MODE, bool EW, bool P64, int N> __global__ void __launch_bounds__(256) sweep_thread(const SweepArgs a) {
  __shared__ uint32_t s_cnt[2][8]; // proposals per warp of the running CTA iteration (parity-double-buffered)
  __shared__ uint32_t s_base[2];
  unsigned long long edges = 0, nodes = 0;
  const uint32_t stride = gridDim.x * blockDim.x;
  // the loop bound is rounded up to a full CTA so that all threads reach the barriers
  const uint32_t bound = (a.list_size + 255u) & ~255u;
  uint32_t it = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < bound; i += stride, ++it) {
    bool proposes = false;
    uint32_t target = 0;
    int32_t uw = 1;
    ThreadRow<0> r;
    r.u = 0;
    if (i < a.list_size) {
      r.u = a.list[i];
      const bool flag = a.active == nullptr || a.active[r.u] != 0;
      if (flag || a.pull) {
        load_row<0>(a, r);
        proposes = sweep_thread_vertex<MODE, EW, P64, N>(a, r, flag, edges, nodes, target, uw);
      }
    }
    emit_cta_iteration<MODE>(a, proposes, r.u, target, uw, it, s_cnt, s_base);
  }
  block_count_flush(a, edges, nodes);
}

// ================================================================================================
// shared helpers for the hash-map kernels
// ================================================================================================
__device__ __forceinline__ uint32_t pow2_ceil(uint32_t x) { // x >= 1
  return x <= 1 ? 1u : (1u << (32 - __clz(static_cast<int>(x - 1))));
}

// open addressing, linear probing in shared memory
__device__ __forceinline__ void table_add(uint32_t *keys, int32_t *vals, uint32_t mask, bool direct, uint32_t key,
                                          int32_t w) {
  uint32_t slot = direct ? key : (lowbias32(key) & mask);
  while (true) {
    const uint32_t prev = atomicCAS(&keys[slot], kEmpty, key);
    if (prev == kEmpty || prev == key) {
      atomicAdd(&vals[slot], w);
      return;
    }
    slot = (slot + 1) & mask;
  }
}

// ================================================================================================
// tiers 3..6: a TEAM of T threads (one warp, 128, 512 or 1024 threads) per vertex, rating map = an
// open-addressing table in shared memory sized for the tier's largest degree (load <= 0.5), used whole.
//
//   1. gather : every thread loads its neighbours (coalesced adjncy stream), gathers the packed
//               (label, stamp) word of each -- B independent gathers in flight per thread -- and inserts the
//               label into the table (one shared-memory CAS + one add per edge; the FixedSizeSparseMap role,
//               kaminpar-common/datastructures/fixed_size_sparse_map.h). A CAS that claims an empty slot appends
//               the slot to the team's CLAIM LIST (16-bit slot indices, appends aggregated per warp). The stamps
//               decide whether the vertex is active at all (pull activation, see lp_device.cuh); an inactive
//               vertex stops here.
//   2. select : the listed slots -- the distinct labels, not the whole table -- are scanned once WITHOUT touching
//               the cluster-weight array: the team arg-max of (rating, tie hash) over all entries is the favored
//               cluster, and -- if that cluster is feasible, one broadcast load -- also the move target
//               (lp_clusterer.cc:199-250). Only when the top entry is infeasible the entries are evaluated in full
//               (one weight gather per distinct label). The refiner (k blocks, weights cached) always evaluates in
//               full. The selection is a total order, so the order of the list does not matter.
//   3. every thread clears the listed slots it scanned; vertices are claimed from a work queue.
// ================================================================================================
template <int T> struct TeamSync {
  // id: named barrier of the team (1..15); teams of a CTA use distinct ids
  static __device__ __forceinline__ void sync(int id) {
    if (T == 32) {
      __syncwarp();
    } else {
      asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(T) : "memory");
    }
  }
  // also a barrier: shared-memory stores before it are visible to the whole team after it
  static __device__ __forceinline__ bool any(int id, bool p) {
    if (T == 32) {
      __syncwarp(); // the vote alone does not order memory
      return __any_sync(kFull, p);
    } else {
      int r;
      asm volatile(
          "{\n"
          ".reg .pred q, r;\n"
          "setp.ne.s32 q, %3, 0;\n"
          "bar.red.or.pred r, %1, %2, q;\n"
          "selp.s32 %0, 1, 0, r;\n"
          "}\n"
          : "=r"(r)
          : "r"(id), "r"(T), "r"(static_cast<int>(p))
          : "memory");
      return r != 0;
    }
  }
};

// arg-max over a team: warp_argmax, then (T > 32) the warp results through shared memory
template <int MODE, int T>
__device__ __forceinline__ Cand team_argmax(int id, int tid, Cand c, Cand *s_red) {
  Cand r = warp_argmax<MODE>(kFull, c);
  if (T == 32) {
    return r;
  }
  TeamSync<T>::sync(id); // s_red free (previous use consumed)
  if ((tid & 31) == 0) {
    s_red[tid >> 5] = r;
  }
  TeamSync<T>::sync(id);
  Cand x = cand_none();
  if ((tid & 31) < T / 32) {
    x = s_red[tid & 31];
  }
  return warp_argmax<MODE>(kFull, x);
}

// Ratings of a team table: 32-bit, or -- V16, unit edge weights only, where a rating is at most the degree
// < 2^16 -- two 16-bit counters per word (a 32768-slot table then fits one SM's shared memory: 192 KiB).
template <bool V16> struct TeamVals;
template <> struct TeamVals<false> {
  using word = int32_t;
  static constexpr int kBytesPerSlot = 4;
  static __device__ __forceinline__ void add(word *v, uint32_t slot, int32_t w) { atomicAdd(&v[slot], w); }
  static __device__ __forceinline__ int32_t get(const word *v, uint32_t slot) { return v[slot]; }
  static __device__ __forceinline__ void clear(word *v, uint32_t slot) { v[slot] = 0; }
};
template <> struct TeamVals<true> {
  using word = uint32_t;
  static constexpr int kBytesPerSlot = 2;
  static __device__ __forceinline__ void add(word *v, uint32_t slot, int32_t w) {
    atomicAdd(&v[slot >> 1], static_cast<uint32_t>(w) << ((slot & 1u) * 16u)); // halves never carry: rating < 2^16
  }
  static __device__ __forceinline__ int32_t get(const word *v, uint32_t slot) {
    return static_cast<int32_t>((v[slot >> 1] >> ((slot & 1u) * 16u)) & 0xFFFFu);
  }
  static __device__ __forceinline__ void clear(word *v, uint32_t slot) { reinterpret_cast<uint16_t *>(v)[slot] = 0; }
};

// With unit edge weights (EW = false) the thread whose CAS claims a slot does NOT add its 1: the stored count is
// "occurrences beyond the first" and readers add 1 (team_rating). Neighbourhoods are mostly label-distinct, so
// this halves the shared-memory atomics per edge. Returns whether this call claimed `slot` (the key's first insert).
template <bool V16, bool EW>
__device__ __forceinline__ bool team_table_add(uint32_t *keys, typename TeamVals<V16>::word *vals, uint32_t mask,
                                               bool direct, uint32_t key, int32_t w, uint32_t &slot) {
  slot = direct ? key : (lowbias32(key) & mask);
  while (true) {
    const uint32_t prev = atomicCAS(&keys[slot], kEmpty, key);
    if (!EW && prev == kEmpty) {
      return true;
    }
    if (prev == kEmpty || prev == key) {
      TeamVals<V16>::add(vals, slot, w);
      return prev == kEmpty;
    }
    slot = (slot + 1) & mask;
  }
}
template <bool V16, bool EW>
__device__ __forceinline__ int32_t team_rating(const typename TeamVals<V16>::word *vals, uint32_t slot) {
  return TeamVals<V16>::get(vals, slot) + (EW ? 0 : 1);
}

// CTAs per SM a team tier is built for. __launch_bounds__ caps the registers so that this many fit
// (65536 / (threads * CTAs), allocated in steps of 8): tier 3 (256 threads) fits 6 with <= 40 registers, and with
// edge weights it is held to 6 by shared memory too (32 KiB table + 4 KiB claim lists + the 1 KiB cuobjdump counts
// as static + 1 KiB reserved per CTA: exactly 228 KiB for 6), tiers 4 and 5 (512 threads, 64 KiB table + 8 KiB
// lists) fit 3 with <= 40 registers, tier 6 takes a whole SM. tests/test_team_resources.py checks the build.
template <int T> constexpr int team_ctas_per_sm() { return T == 32 ? 6 : T == 1024 ? 1 : 3; }

template <int MODE, bool EW, bool P64, int T, int SLOTS, int TEAMS, bool V16 = false>
__global__ void __launch_bounds__(T *TEAMS, team_ctas_per_sm<T>()) sweep_team(const SweepArgs a) {
  static_assert((SLOTS & (SLOTS - 1)) == 0, "table size must be a power of two");
  static_assert(SLOTS <= 65536, "claim lists hold 16-bit slot indices");
  static_assert(!(V16 && EW), "16-bit ratings need unit edge weights");
  using TV = TeamVals<V16>;
  // a vertex claims one slot per distinct label, and the degrees of its tier are below SLOTS / 2 (tier_of)
  constexpr int kListCap = SLOTS / 2;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ Cand s_red_all[TEAMS][T > 32 ? T / 32 : 1];
  __shared__ uint16_t s_list_all[TEAMS][kListCap];
  // T > 32 only (a one-warp team keeps them in registers, and tier 3 with edge weights has no shared memory left):
  // the next list index, the running vertex's claim count, and the scan counters, which are written by the team's
  // thread 0 only -- kept here, not in four registers of every thread
  __shared__ uint32_t s_next[TEAMS], s_claims[TEAMS];
  __shared__ unsigned long long s_edges[TEAMS], s_nodes[TEAMS];
  const int team = threadIdx.x / T;
  const int tid = threadIdx.x % T;
  const int lane = threadIdx.x & 31;
  const int bar = 1 + team;
  uint32_t *keys = reinterpret_cast<uint32_t *>(smem_raw) + static_cast<size_t>(team) * SLOTS;
  typename TV::word *vals = reinterpret_cast<typename TV::word *>(
      smem_raw + sizeof(uint32_t) * SLOTS * TEAMS + static_cast<size_t>(team) * SLOTS * TV::kBytesPerSlot);
  Cand *s_red = s_red_all[team];
  uint16_t *list = s_list_all[team];
  for (int s = tid; s < SLOTS; s += T) {
    keys[s] = kEmpty;
    TV::clear(vals, s);
  }
  // work queue: the next list index is claimed one vertex ahead (by thread 0; its result is needed a vertex later)
  uint32_t next = 0;
  unsigned long long edges = 0, nodes = 0; // T == 32
  if (tid == 0) {
    next = atomicAdd(a.queue, 1u);
    if (T > 32) {
      s_edges[team] = 0;
      s_nodes[team] = 0;
    }
  }
  TeamSync<T>::sync(bar); // the table is clear before the first inserts
  while (true) {
    uint32_t i;
    if (T == 32) {
      i = __shfl_sync(kFull, next, 0);
    } else {
      if (tid == 0) {
        s_next[team] = next;
        s_claims[team] = 0; // the previous vertex's count was read before its last barrier
      }
      TeamSync<T>::sync(bar);
      i = s_next[team];
    }
    if (i >= a.list_size) {
      break;
    }
    if (tid == 0) {
      next = atomicAdd(a.queue, 1u);
    }
    const uint32_t u = a.list[i];
    const bool flag = a.active == nullptr || a.active[u] != 0;
    if (!flag && !a.pull) {
      TeamSync<T>::sync(bar);
      continue;
    }
    const uint32_t beg = a.xadj[u];
    uint32_t deg = a.xadj[u + 1] - beg;
    if (deg > a.max_num_neighbors) {
      deg = a.max_num_neighbors;
    }
    const uint32_t own = a.label[u];
    const int32_t uw = a.vwgt != nullptr ? a.vwgt[u] : 1;
    const int32_t own_w = a.weight[own];
    bool skip = false;
    if (MODE == 1) {
      const int32_t mn = a.min_w != nullptr ? a.min_w[own] : 0;
      skip = (own_w - uw) < mn; // lp_refiner.cc:160-162
    }
    // direct: slot = label; hashed: the whole table (the scans below cost the claims, not the table size)
    const bool direct = a.num_labels <= static_cast<uint32_t>(SLOTS);
    // ---- 1. gather + insert --------------------------------------------------------------------
    bool hit = false;
    uint32_t claims = 0; // T == 32: slots the team has claimed so far (the same in every lane)
    constexpr int B = 4;
    for (uint32_t e0 = 0; e0 < deg; e0 += T * B) {
      uint32_t kb[B];
      int32_t wb[B];
      uint32_t vb[B];
#pragma unroll
      for (int j = 0; j < B; ++j) {
        const uint32_t e = e0 + j * T + tid;
        vb[j] = e < deg ? a.adjncy[beg + e] : kEmpty;
        wb[j] = (EW && e < deg) ? a.adjwgt[beg + e] : 1;
      }
#pragma unroll
      for (int j = 0; j < B; ++j) {
        kb[j] = kEmpty;
        if (vb[j] != kEmpty) {
          const typename LabG<P64>::word g = load_labg<P64>(a, vb[j]);
          hit = hit || stamp_hit(LabG<P64>::stamp(g), a.window);
          bool ok = !skip;
          if (MODE == 1 && a.communities != nullptr) {
            ok = ok && a.communities[u] == a.communities[vb[j]];
          }
          if (ok) {
            kb[j] = LabG<P64>::label(g);
          }
        }
      }
      uint32_t sl[B];
      unsigned claimed[B];
#pragma unroll
      for (int j = 0; j < B; ++j) {
        sl[j] = 0;
        claimed[j] = __ballot_sync(kFull, kb[j] != kEmpty && team_table_add<V16, EW>(keys, vals, SLOTS - 1, direct,
                                                                                     kb[j], wb[j], sl[j]));
      }
      // append the claimed slots to the list: one shared atomic per warp and step (none in a one-warp team)
      uint32_t n = 0;
#pragma unroll
      for (int j = 0; j < B; ++j) {
        n += __popc(claimed[j]);
      }
      if (n != 0) {
        uint32_t base = claims;
        if (T == 32) {
          claims += n;
        } else {
          if (lane == 0) {
            base = atomicAdd(&s_claims[team], n);
          }
          base = __shfl_sync(kFull, base, 0);
        }
        const unsigned below = (1u << lane) - 1u;
#pragma unroll
        for (int j = 0; j < B; ++j) {
          if ((claimed[j] >> lane) & 1u) {
            list[base + __popc(claimed[j] & below)] = static_cast<uint16_t>(sl[j]);
          }
          base += __popc(claimed[j]);
        }
      }
    }
    const bool any_hit = TeamSync<T>::any(bar, hit); // also the barrier after the inserts
    const bool act = flag || any_hit;
    const uint32_t nc = T == 32 ? claims : s_claims[team];
    // ---- 2. select over the listed slots: thread tid takes entries tid, tid + T, ... --------------
    const bool store_fav = (MODE == 0) && (uw == own_w) && (own_w <= a.max_cluster_weight / 2);
    Cand best = cand_none(), fav = cand_none();
    if (act) {
      Cand c = cand_none(), f = cand_none();
      if (MODE == 0) {
        // pass A: no weight gathers
        for (uint32_t l = tid; l < nc; l += T) {
          const uint32_t s = list[l];
          const uint32_t k = keys[s];
          const int32_t r = team_rating<V16, EW>(vals, s);
          // an entry rated below the thread's running maximum cannot win: its tie hashes are never computed
          // (most entries of a late-round neighbourhood have rating 1 next to a few heavy clusters)
          if (r >= c.gain) {
            Cand x{r, 0, tie_hash(a.base_tie, u, k), k};
            if (cand_better<0>(x, c)) {
              c = x;
            }
          }
          if (store_fav && r >= f.gain) {
            Cand y{r, 0, tie_hash(a.base_fav, u, k), k};
            if (cand_better<0>(y, f)) {
              f = y;
            }
          }
        }
        const Cand top = team_argmax<0, T>(bar, tid, c, s_red);
        if (store_fav) {
          fav = team_argmax<0, T>(bar, tid, f, s_red);
        }
        bool top_ok = true;
        if (top.gain > 0) {
          top_ok = (a.weight[top.key] + uw <= a.max_cluster_weight) || (top.key == own);
          if (a.communities != nullptr) {
            top_ok = top_ok && (a.communities[top.key] == a.communities[own]);
          }
        }
        if (top_ok) {
          best = top;
        } else {
          // pass B: the top entry is full -- evaluate every entry with its cluster weight
          Cand cb = cand_none();
          for (uint32_t l0 = 0; l0 < nc; l0 += T * 4) {
            uint32_t kk[4];
            int32_t rr[4], ww[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const uint32_t l = l0 + j * T + tid;
              const uint32_t s = l < nc ? list[l] : 0u;
              kk[j] = l < nc ? keys[s] : kEmpty;
              rr[j] = l < nc ? team_rating<V16, EW>(vals, s) : 0;
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              ww[j] = kk[j] != kEmpty ? a.weight[kk[j]] : 0;
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              if (kk[j] != kEmpty) {
                Cand ff;
                const Cand cc = eval_candidate_w<0>(a, u, own, uw, own_w, kk[j], rr[j], ww[j], false, ff);
                if (cand_better<0>(cc, cb)) {
                  cb = cc;
                }
              }
            }
          }
          best = team_argmax<0, T>(bar, tid, cb, s_red);
        }
      } else {
        for (uint32_t l = tid; l < nc; l += T) {
          const uint32_t s = list[l];
          const uint32_t k = keys[s];
          Cand ff;
          const Cand cc = eval_candidate_w<1>(a, u, own, uw, own_w, k, team_rating<V16, EW>(vals, s), a.weight[k], false, ff);
          if (cand_better<1>(cc, c)) {
            c = cc;
          }
        }
        best = team_argmax<1, T>(bar, tid, c, s_red);
      }
    }
    // ---- 3. clear the listed slots, finish the vertex ---------------------------------------------
    // no barrier first: every thread clears exactly the entries it scanned
    for (uint32_t l = tid; l < nc; l += T) {
      const uint32_t s = list[l];
      keys[s] = kEmpty;
      TV::clear(vals, s);
    }
    if (act && tid == 0) {
      if (T == 32) {
        edges += deg;
        nodes += 1;
      } else {
        s_edges[team] += deg;
        s_nodes[team] += 1;
      }
      if (a.active != nullptr && flag) {
        a.active[u] = 0;
      }
      uint32_t target;
      if (finish_vertex<MODE>(a, u, own, store_fav, best, fav, target)) {
        const uint32_t idx = atomicAdd(a.mover_count, 1u);
        emit_proposal<MODE>(a, idx, u, target, uw);
      }
    }
    TeamSync<T>::sync(bar); // table clean
  }
  if (T > 32 && tid == 0) {
    edges = s_edges[team];
    nodes = s_nodes[team];
  }
  if (tid == 0 && nodes != 0) {
    atomicAdd(&a.counters[0], edges);
    atomicAdd(&a.counters[kCounterNodesOffset], nodes);
  }
}

// ================================================================================================
// tier 7 (deg >= 8192 / 16384), clusterer (MODE 0): label-partitioned rating with final results per CTA.
//   gather : edge-parallel over the 2048-edge chunks of the sub-round's hubs: every neighbour label is gathered
//            once and written, coalesced, to a scratch row per hub (4 B per edge); the stamps mark pull activation.
//            With unit edge weights each chunk is counting-sorted by class (lowbias32(label) & (Ks - 1), Ks =
//            hub_sort_classes(deg)) in shared memory before it is written back, and its Ks + 1 class offsets are
//            stored beside the row.
//   rate   : one 1024-thread CTA per work item (hub u, hash class c of K_u = hub_classes(deg) classes, taken from a
//            queue in order of decreasing degree). Its warps claim (chunk, part) pieces from a shared counter and
//            read only class c's range of each sorted chunk, inserting every label into a 16384-slot shared-memory
//            table with a claim list; then it selects as the team kernels do. Classes of a hub hold disjoint labels,
//            so each result is final for its class: no merge. Where a chunk's range holds more than class c
//            (edge weights: unsorted chunks; K_u > Ks; a split class) the labels are filtered by their hash and
//            compacted per warp first. A class that claims more than the list holds is split by the next hash bit
//            and read again, until every sub-class fits (lowbias32 is a bijection, so this terminates). While an
//            item streams, one warp claims the next item and loads its header, so the CTA does not wait on that
//            chain of dependent loads between items.
//   final  : as below: the arg-max over the K_u class results of each hub.
// tier 7, refiner (MODE 1): edge-parallel, label-partitioned two-pass aggregation (a refiner hub sees at most k
// labels, so the slice maps compress 256 edges to <= k appends). No random access ever touches a table outside
// shared memory, and after the chunk is staged every warp works on its own:
//   scatter : a CTA takes 2048-edge chunks of hub adjacencies from a work queue. The producer warp stages each
//             chunk with one 1-D bulk TMA copy; each of the 8 consumer warps gathers the labels of its 256-edge
//             slice, aggregates them in its private 512-slot shared-memory hash map (slice-local ratings: a label
//             that dominates the neighbourhood costs one entry per slice, not one per edge) and appends every
//             distinct (label, rating) to the BUCKET lowbias32(label) & (P-1) of the vertex -- P = hub_buckets(deg)
//             buckets of kBucketCap packed 8-byte entries each, filled through one atomic cursor per bucket
//             (streaming writes). An append beyond a bucket's capacity (possible only with skewed label hashes: the
//             expected fill is <= 256 of 512) goes to a shared overflow list, so nothing is ever dropped.
//   select  : one WARP per (vertex, bucket) streams the bucket's entries into its private 1024-slot hash map,
//             ranks the distinct labels and writes the bucket's best / favored candidate. Labels of different
//             buckets are disjoint, so the vertex's decision is the arg-max over its buckets (final). A bucket
//             that also has overflow entries may exceed the map: it is then processed in K = 2, 4, ... passes over
//             disjoint hash classes (lowbias32 is a bijection, so the classes eventually separate all labels).
//   final   : one warp per vertex reduces its buckets' candidates and proposes / stores the favored cluster.
// ================================================================================================
constexpr int kChunkEdges = 2048;
constexpr int kSliceEdges = 256;        // edges per consumer warp and chunk
constexpr int kSliceTableSlots = 512;   // warp-private map of the scatter pass: <= 256 distinct labels, load <= 0.5
constexpr int kChunkThreads = 256;
constexpr uint32_t kBucketCap = 512;       // entries per bucket region
constexpr uint32_t kBucketTargetFill = 256;
constexpr uint32_t kSelTableSlots = 1024;  // warp-private map of the select pass
constexpr int kSelWarps = 4;               // warps (= buckets in flight) per select CTA: 32 KiB of shared memory

struct HubOverflow { // an entry that did not fit its bucket region
  uint32_t bucket;   // wave-relative bucket index
  uint32_t key;
  int32_t rating;
  uint32_t pad;
};

struct HubArgs {
  const uint32_t *__restrict__ item_entry; // index into the hub list of this sub-round
  const uint32_t *__restrict__ item_chunk;
  const uint32_t *__restrict__ item_u;   // static per item: vertex id, xadj[u], degree
  const uint32_t *__restrict__ item_beg;
  const uint32_t *__restrict__ item_deg;
  uint32_t num_items;
  const uint32_t *__restrict__ table_off;  // per list entry: its first bucket (wave-relative)
  unsigned long long *__restrict__ g_tab;  // bucket regions: kBucketCap packed (key << 32 | rating) entries each
  uint32_t *__restrict__ cursor;           // per bucket: entries appended (zero between sub-rounds: select resets it)
  HubOverflow *__restrict__ ovf;           // overflow list of the running wave
  uint32_t *__restrict__ ovf_count;        // its length (per wave; zeroed with the per-round counters)
  uint32_t ovf_cap;
  uint32_t bucket_cap;                     // entries a region takes (kBucketCap; smaller only in tests: KMP_HUB_BUCKET_CAP)
  uint32_t sel_limit;                      // 0, or a smaller claim limit of the select map (tests: KMP_HUB_SEL_LIMIT)
  uint32_t stage_adjncy;                   // adjncy is 16-byte aligned: chunks are staged with bulk copies
  // select: one item per (list entry, bucket)
  const uint32_t *__restrict__ sel_entry;
  const uint32_t *__restrict__ sel_piece;
  uint32_t num_sel_items;
  const uint32_t *__restrict__ sel_begin; // per list entry: its first selection item
  Cand *__restrict__ part_best;           // per selection item
  Cand *__restrict__ part_fav;
  uint32_t rank, world;                   // hub entry i is owned by rank i % world
  uint32_t *__restrict__ queue;           // work-queue cursor of this launch (zeroed per LP round)
  uint32_t *__restrict__ hit;             // per list entry: a neighbour moved since the last visit (pull); reset by final
  // clusterer (gather + rate): the staged neighbour labels of the sub-round and, per list entry, where its row
  // starts in them; rate items are (item_entry, item_cls) pairs, their results go to part_*[sel_begin[entry] + cls]
  uint32_t *__restrict__ lab;
  const uint32_t *__restrict__ lab_off;
  const uint32_t *__restrict__ item_cls;
  // unit edge weights: each staged chunk is sorted by class; its hub_sort_classes + 1 class offsets start at
  // cls[cls_off[entry] + chunk * (Ks + 1)]. nullptr with edge weights (chunks stay in edge order)
  uint16_t *__restrict__ cls;
  const uint32_t *__restrict__ cls_off;
};

// buckets of a hub: a power of two with <= kBucketTargetFill expected distinct labels per bucket
__host__ __device__ __forceinline__ uint32_t hub_buckets(uint32_t full_degree) {
  const uint32_t need = (full_degree + kBucketTargetFill - 1) / kBucketTargetFill;
  uint32_t p = 1;
  while (p < need) {
    p <<= 1;
  }
  return p;
}

// ---- 1-D bulk TMA (cp.async.bulk) + mbarrier helpers -----------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// global -> shared bulk copy; dst/src 16-byte aligned, bytes a multiple of 16
__device__ __forceinline__ void tma_load_1d(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

struct HubItem {
  uint32_t valid;   // 0: nothing to do for this item
  uint32_t u;
  uint32_t entry;
  uint32_t full_deg;
  uint32_t gbeg, gend; // edge range of the chunk (indices into adjncy)
  uint32_t a0;         // first staged element (gbeg rounded down to a 16-byte boundary)
  uint32_t staged;     // number of staged elements (multiple of 4), may stop short of gend at the array end;
                       // 0 when adjncy itself is not 16-byte aligned
};

__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

constexpr int kHubStages = 2;
constexpr int kHubConsumerWarps = kChunkThreads / 32;          // 8 consumer warps
constexpr int kHubThreads = kChunkThreads + 32;                // + 1 producer warp
constexpr int kHubScatterSmem = kHubConsumerWarps * kSliceTableSlots * 8; // dynamic: 8 warp maps (keys + ratings)

template <int MODE, bool EW, bool P64>
__global__ void __launch_bounds__(kHubThreads, 4) sweep_hub_scatter(const SweepArgs a, const HubArgs hb, uint32_t m_total) {
  // warp-specialised producer / consumer pipeline:
  //   producer warp : claims the next work item (2048-edge chunk of a hub's adjacency), publishes its descriptor
  //                   and stages the chunk with ONE bulk TMA copy (cp.async.bulk, completion on the stage's `full`
  //                   mbarrier);
  //   consumer warps: wait on `full`; each warp gathers the neighbour labels of its 256-edge slice (4 independent
  //                   gathers per lane) into its private map, releases the stage (`empty` mbarrier), then appends
  //                   the map's entries to the vertex's buckets and clears it. No barrier between warps.
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int kAllSlots = kHubConsumerWarps * kSliceTableSlots;
  uint32_t *all_keys = reinterpret_cast<uint32_t *>(smem_raw);
  int32_t *all_vals = reinterpret_cast<int32_t *>(smem_raw + sizeof(uint32_t) * kAllSlots);
  __shared__ __align__(16) uint32_t s_adj[kHubStages][kChunkEdges + 8];
  __shared__ __align__(8) uint64_t s_full[kHubStages];
  __shared__ __align__(8) uint64_t s_empty[kHubStages];
  __shared__ HubItem s_item[kHubStages];
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kHubStages; ++s) {
      mbar_init(&s_full[s], 1);
      mbar_init(&s_empty[s], kHubConsumerWarps);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int s = threadIdx.x; s < kAllSlots; s += kHubThreads) {
    all_keys[s] = kEmpty;
    all_vals[s] = 0;
  }
  __syncthreads();

  if (wib == kHubConsumerWarps) {
    // ------------------------------- producer warp -------------------------------------------
    if (lane == 0) {
      // items are claimed from a global cursor (dynamic load balancing: chunks of inactive hubs cost
      // nothing, full chunks cost ~2048 gathers); valid = 2 tells the consumers to stop
      for (uint32_t k = 0;; ++k) {
        const int stage = static_cast<int>(k % kHubStages);
        const uint32_t round = k / kHubStages;
        mbar_wait(&s_empty[stage], (round & 1u) ^ 1u); // passes immediately in the first round
        const uint32_t it = atomicAdd(hb.queue, 1u);
        HubItem d{};
        d.valid = 0;
        if (it >= hb.num_items) {
          d.valid = 2;
          s_item[stage] = d;
          mbar_arrive(&s_full[stage]);
          break;
        }
        const uint32_t entry = hb.item_entry[it]; // the descriptor loads are independent
        const uint32_t u = hb.item_u[it];
        const uint32_t beg0 = hb.item_beg[it];
        const uint32_t full_deg = hb.item_deg[it];
        const uint32_t chunk = hb.item_chunk[it];
        if (entry % hb.world == hb.rank && (a.active == nullptr || a.pull || a.active[u] != 0)) {
          uint32_t deg = full_deg;
          if (deg > a.max_num_neighbors) {
            deg = a.max_num_neighbors;
          }
          const uint32_t cbeg = chunk * kChunkEdges;
          bool ok = cbeg < deg;
          if (ok && MODE == 1) {
            const uint32_t own = a.label[u];
            const int32_t uw = a.vwgt != nullptr ? a.vwgt[u] : 1;
            const int32_t mn = a.min_w != nullptr ? a.min_w[own] : 0;
            ok = !((a.weight[own] - uw) < mn); // lp_refiner.cc:160-162: no ratings needed
          }
          if (ok) {
            const uint32_t cend = (cbeg + kChunkEdges < deg) ? cbeg + kChunkEdges : deg;
            d.valid = 1;
            d.u = u;
            d.entry = entry;
            d.full_deg = full_deg;
            d.gbeg = beg0 + cbeg;
            d.gend = beg0 + cend;
            d.a0 = d.gbeg & ~3u;
            d.staged = 0;
            if (hb.stage_adjncy) { // cp.async.bulk needs a 16-byte aligned source; else the consumers read adjncy
              uint32_t a1 = (d.gend + 3u) & ~3u;
              const uint32_t m4 = m_total & ~3u; // last 16-byte block that lies fully inside adjncy
              if (a1 > m4) {
                a1 = m4;
              }
              d.staged = a1 > d.a0 ? a1 - d.a0 : 0;
            }
          }
        }
        s_item[stage] = d;
        if (d.valid && d.staged > 0) {
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          mbar_arrive_expect_tx(&s_full[stage], d.staged * 4);
          tma_load_1d(&s_adj[stage][0], a.adjncy + d.a0, d.staged * 4, &s_full[stage]);
        } else {
          mbar_arrive(&s_full[stage]); // nothing staged: publish the descriptor only
        }
      }
    }
    return;
  }

  // --------------------------------- consumer warps ----------------------------------------------
  uint32_t *keys = all_keys + wib * kSliceTableSlots;
  int32_t *vals = all_vals + wib * kSliceTableSlots;
  for (uint32_t k = 0;; ++k) {
    const int stage = static_cast<int>(k % kHubStages);
    const uint32_t round = k / kHubStages;
    mbar_wait(&s_full[stage], round & 1u);
    const HubItem d = s_item[stage];
    if (d.valid == 2) {
      break; // queue exhausted
    }
    const uint32_t wbeg = d.gbeg + wib * kSliceEdges;
    const bool mine = d.valid && wbeg < d.gend;
    if (mine) {
      const uint32_t wend = wbeg + kSliceEdges < d.gend ? wbeg + kSliceEdges : d.gend;
      const uint32_t staged_end = d.a0 + d.staged;
      bool hit = false;
      // ---- gather + slice-local aggregation
      for (uint32_t e0 = wbeg; e0 < wend; e0 += 128) {
        uint32_t k4[4];
        int32_t w4[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) { // 4 independent label gathers per lane in flight
          const uint32_t e = e0 + j * 32 + lane;
          k4[j] = kEmpty;
          w4[j] = 0;
          if (e < wend) {
            const uint32_t v = e < staged_end ? s_adj[stage][e - d.a0] : a.adjncy[e];
            bool ok = true;
            if (MODE == 1 && a.communities != nullptr) {
              ok = a.communities[d.u] == a.communities[v];
            }
            const typename LabG<P64>::word g = load_labg<P64>(a, v);
            hit = hit || stamp_hit(LabG<P64>::stamp(g), a.window);
            if (ok) {
              k4[j] = LabG<P64>::label(g);
              w4[j] = EW ? a.adjwgt[e] : 1;
            }
          }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (k4[j] != kEmpty) {
            table_add(keys, vals, kSliceTableSlots - 1, false, k4[j], w4[j]);
          }
        }
      }
      if (a.pull && __any_sync(kFull, hit) && lane == 0) {
        atomicOr(&hb.hit[d.entry], 1u);
      }
    }
    __syncwarp(); // the warp's map is complete, its reads of the staged adjacency are done
    if (lane == 0) {
      mbar_arrive(&s_empty[stage]);
    }
    if (mine) {
      // ---- append the distinct (label, rating) pairs to the vertex's buckets, clear the map
      const uint32_t pmask = hub_buckets(d.full_deg) - 1;
      const uint32_t bucket0 = hb.table_off[d.entry];
      constexpr int B = 4; // B independent cursor atomics in flight per lane
      for (uint32_t s0 = lane; s0 < kSliceTableSlots; s0 += 32 * B) {
        uint32_t kk[B], bb[B], pos[B];
        int32_t rr[B];
#pragma unroll
        for (int j = 0; j < B; ++j) {
          const uint32_t s = s0 + j * 32;
          kk[j] = keys[s];
          rr[j] = vals[s];
          if (kk[j] != kEmpty) {
            keys[s] = kEmpty;
            vals[s] = 0;
          }
        }
#pragma unroll
        for (int j = 0; j < B; ++j) {
          bb[j] = bucket0 + (lowbias32(kk[j]) & pmask);
          pos[j] = kk[j] != kEmpty ? atomicAdd(&hb.cursor[bb[j]], 1u) : 0u;
        }
#pragma unroll
        for (int j = 0; j < B; ++j) {
          if (kk[j] != kEmpty) {
            if (pos[j] < hb.bucket_cap) {
              hb.g_tab[static_cast<size_t>(bb[j]) * kBucketCap + pos[j]] =
                  (static_cast<unsigned long long>(kk[j]) << 32) | static_cast<uint32_t>(rr[j]);
            } else {
              const uint32_t o = atomicAdd(hb.ovf_count, 1u); // < ovf_cap: at most one entry per edge of the wave
              if (o < hb.ovf_cap) {
                hb.ovf[o] = HubOverflow{bb[j], kk[j], rr[j], 0u};
              }
            }
          }
        }
      }
      __syncwarp(); // map clean before the warp's next slice
    }
  }
}

// select (refiner): one warp per (hub, bucket): best candidate of the bucket's labels
template <int MODE> __global__ void __launch_bounds__(kSelWarps * 32) sweep_hub_select(const SweepArgs a, const HubArgs hb) {
  static_assert(MODE == 1, "the clusterer rates its hubs with sweep_hub_rate");
  __shared__ uint32_t s_keys[kSelWarps][kSelTableSlots];
  __shared__ int32_t s_vals[kSelWarps][kSelTableSlots];
  __shared__ uint32_t s_claims_all[kSelWarps];
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  uint32_t *keys = s_keys[wib];
  int32_t *vals = s_vals[wib];
  uint32_t *s_claims = &s_claims_all[wib];
  for (uint32_t s = lane; s < kSelTableSlots; s += 32) {
    keys[s] = kEmpty;
    vals[s] = 0;
  }
  if (lane == 0) {
    *s_claims = 0;
  }
  __syncwarp();
  const uint32_t nwarps = gridDim.x * kSelWarps;
  for (uint32_t it = blockIdx.x * kSelWarps + wib; it < hb.num_sel_items; it += nwarps) {
    const uint32_t entry = hb.sel_entry[it];
    const uint32_t u = a.list[entry];
    Cand c = cand_none();
    // a bucket is read (and its cursor reset) whenever the scatter pass may have filled it; activity is decided
    // by sweep_hub_final
    const bool act = (entry % hb.world == hb.rank) && (a.active == nullptr || a.pull || a.active[u] != 0);
    const uint32_t b = hb.table_off[entry] + hb.sel_piece[it];
    const uint32_t appended = act ? __ldcg(&hb.cursor[b]) : 0u;
    if (appended != 0) {
      const uint32_t full_deg = a.xadj[u + 1] - a.xadj[u];
      const uint32_t pbits = 31 - __clz(static_cast<int>(hub_buckets(full_deg)));
      const uint32_t own = a.label[u];
      const int32_t uw = a.vwgt != nullptr ? a.vwgt[u] : 1;
      const int32_t own_w = a.weight[own];
      const uint32_t n_reg = appended < hb.bucket_cap ? appended : hb.bucket_cap;
      const uint32_t n_ovf = appended > hb.bucket_cap ? min(__ldcg(hb.ovf_count), hb.ovf_cap) : 0u;
      // The map is sized for the entries at hand. A bucket without overflow entries holds <= kBucketCap =
      // kSelTableSlots / 2 labels: it can never fill the map. K > 1 only when overflow entries push the distinct
      // labels of this bucket beyond 5/8 of the map (checked after every batch of <= 128 inserts, so the map
      // holds at most 640 + 128 < 1024 labels).
      uint32_t tcap = pow2_ceil(2 * appended);
      tcap = tcap < 64 ? 64u : tcap > kSelTableSlots ? kSelTableSlots : tcap;
      const uint32_t tmask = tcap - 1;
      const uint32_t full_limit = tcap / 2 + tcap / 8;
      const uint32_t limit = (hb.sel_limit != 0 && hb.sel_limit < full_limit) ? hb.sel_limit : full_limit;
      const unsigned long long *reg = hb.g_tab + static_cast<size_t>(b) * kBucketCap;
      auto insert = [&](uint32_t key, int32_t r) {
        uint32_t slot = lowbias32(key ^ 0x9E3779B9u) & tmask;
        while (true) {
          const uint32_t prev = atomicCAS(&keys[slot], kEmpty, key);
          if (prev == kEmpty) {
            atomicAdd(s_claims, 1u);
          }
          if (prev == kEmpty || prev == key) {
            atomicAdd(&vals[slot], r);
            return;
          }
          slot = (slot + 1) & tmask;
        }
      };
      uint32_t K = 1;
      while (true) {
        c = cand_none();
        bool overflowed = false;
        for (uint32_t cls = 0; cls < K && !overflowed; ++cls) {
          // ---- insert the entries of hash class `cls`
          constexpr int B = 4;
          for (uint32_t i0 = 0; i0 < n_reg && !overflowed; i0 += 32 * B) {
            unsigned long long e[B];
#pragma unroll
            for (int j = 0; j < B; ++j) {
              const uint32_t i = i0 + j * 32 + lane;
              e[j] = i < n_reg ? __ldcs(reg + i) : ~0ull;
            }
#pragma unroll
            for (int j = 0; j < B; ++j) {
              const uint32_t key = static_cast<uint32_t>(e[j] >> 32);
              if (key != kEmpty && ((lowbias32(key) >> pbits) & (K - 1)) == cls) {
                insert(key, static_cast<int32_t>(static_cast<uint32_t>(e[j])));
              }
            }
            if (n_ovf != 0) { // with overflow entries (appended > bucket_cap, hence the full map): check the claims
              __syncwarp();
              overflowed = *s_claims > limit;
              __syncwarp();
            }
          }
          for (uint32_t i0 = 0; i0 < n_ovf && !overflowed; i0 += 32 * B) {
#pragma unroll
            for (int j = 0; j < B; ++j) {
              const uint32_t i = i0 + j * 32 + lane;
              if (i < n_ovf) {
                const HubOverflow o = hb.ovf[i];
                if (o.bucket == b && ((lowbias32(o.key) >> pbits) & (K - 1)) == cls) {
                  insert(o.key, o.rating);
                }
              }
            }
            __syncwarp();
            overflowed = *s_claims > limit;
            __syncwarp();
          }
          __syncwarp(); // the class is inserted (or abandoned)
          // ---- evaluate + clear
          const bool evaluate = !overflowed;
          for (uint32_t s0 = 0; s0 < tcap; s0 += 32 * B) {
            uint32_t kk[B];
            int32_t rr[B], ww[B];
#pragma unroll
            for (int j = 0; j < B; ++j) {
              const uint32_t s = s0 + j * 32 + lane;
              kk[j] = s < tcap ? keys[s] : kEmpty;
              rr[j] = kk[j] != kEmpty ? vals[s] : 0;
            }
#pragma unroll
            for (int j = 0; j < B; ++j) {
              ww[j] = (kk[j] != kEmpty && evaluate) ? a.weight[kk[j]] : 0;
            }
#pragma unroll
            for (int j = 0; j < B; ++j) {
              if (kk[j] != kEmpty) {
                const uint32_t s = s0 + j * 32 + lane;
                keys[s] = kEmpty;
                vals[s] = 0;
                if (evaluate) {
                  Cand ff;
                  const Cand cc = eval_candidate_w<1>(a, u, own, uw, own_w, kk[j], rr[j], ww[j], false, ff);
                  if (cand_better<1>(cc, c)) {
                    c = cc;
                  }
                }
              }
            }
          }
          __syncwarp();
          if (lane == 0) {
            *s_claims = 0;
          }
          __syncwarp();
        }
        if (!overflowed) {
          break;
        }
        K <<= 1; // too many distinct labels for the map: split into more hash classes and start over
      }
      if (lane == 0) {
        hb.cursor[b] = 0;
      }
    }
    const Cand best = warp_argmax<1>(kFull, c);
    if (lane == 0) {
      hb.part_best[it] = best;
    }
  }
}

// ---- clusterer: gather + rate ---------------------------------------------------------------------------------
constexpr int kRateThreads = 1024;
constexpr uint32_t kRateSlots = 16384;            // table of the rate kernel: 128 KiB of keys + 32-bit ratings
constexpr uint32_t kRateListCap = kRateSlots / 2; // claim list (16-bit slot indices); the table load stays <= 0.5
constexpr uint32_t kHubClassEdges = 8192;         // edges per hash class: a class fits the list even if all distinct
constexpr uint32_t kRateStage = 64;               // per-warp staging ring: < 32 pending + 32 new labels
// dynamic shared memory of the rate kernel: keys + ratings, the claim list, the staging buffers (labels, weights)
template <bool EW> constexpr int rate_smem() {
  return static_cast<int>(kRateSlots * 8 + kRateListCap * 2 + (kRateThreads / 32) * kRateStage * (EW ? 8 : 4));
}

// hash classes of a hub: a power of two with <= kHubClassEdges edges per class (the low bits of lowbias32(label),
// the same bits as the bucket index of the refiner's path)
__host__ __device__ __forceinline__ uint32_t hub_classes(uint32_t full_degree) {
  const uint32_t need = (full_degree + kHubClassEdges - 1) / kHubClassEdges;
  uint32_t p = 1;
  while (p < need) {
    p <<= 1;
  }
  return p;
}

// classes a staged chunk is sorted by: the hub's hash classes, at most kHubSortClasses of them (a hub with more
// classes reads the range of its class's low bits and filters by the rest); 1 (unsorted) with edge weights, whose
// rate items read each label's weight by its edge index
constexpr uint32_t kHubSortClasses = 256;
static_assert(kHubSortClasses <= 256, "sweep_hub_gather scans the class counts with one class per thread");
__host__ __device__ __forceinline__ uint32_t hub_sort_classes(uint32_t full_degree) {
  const uint32_t k = hub_classes(full_degree);
  return k < kHubSortClasses ? k : kHubSortClasses;
}

// gather: one 256-thread CTA per (hub, 2048-edge chunk) item, 8 independent label gathers per thread. With
// hb.cls_off set (unit edge weights), the chunk is counting-sorted by sort class in shared memory, written back to
// its own range of the row, and its Ks + 1 class offsets go to hb.cls. Order inside a class is free: ratings are
// sums and the selection is a total order.
template <bool P64> __global__ void __launch_bounds__(256, 8) sweep_hub_gather(const SweepArgs a, const HubArgs hb) {
  constexpr int B = kChunkEdges / 256;
  __shared__ uint32_t s_lab[kChunkEdges], s_sorted[kChunkEdges];
  __shared__ uint16_t s_rank[kChunkEdges]; // a label's rank within its class in the chunk
  __shared__ uint32_t s_cnt[kHubSortClasses + 1];
  __shared__ uint32_t s_wsum[256 / 32];
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  for (uint32_t it = blockIdx.x; it < hb.num_items; it += gridDim.x) {
    const uint32_t entry = hb.item_entry[it];
    const uint32_t u = hb.item_u[it];
    if (entry % hb.world != hb.rank || !(a.active == nullptr || a.pull || a.active[u] != 0)) {
      continue;
    }
    const uint32_t deg = min(hb.item_deg[it], a.max_num_neighbors);
    const uint32_t cbeg = hb.item_chunk[it] * kChunkEdges;
    if (cbeg >= deg) {
      continue;
    }
    const uint32_t cend = min(cbeg + kChunkEdges, deg);
    const uint32_t *adj = a.adjncy + hb.item_beg[it];
    uint32_t *out = hb.lab + hb.lab_off[entry];
    uint32_t v[B];
#pragma unroll
    for (int j = 0; j < B; ++j) {
      const uint32_t e = cbeg + j * 256 + threadIdx.x;
      v[j] = e < cend ? adj[e] : kEmpty;
    }
    const uint32_t Ks = hb.cls_off != nullptr ? hub_sort_classes(hb.item_deg[it]) : 1u;
    bool hit = false;
#pragma unroll
    for (int j = 0; j < B; ++j) {
      if (v[j] != kEmpty) {
        const typename LabG<P64>::word g = load_labg<P64>(a, v[j]);
        hit = hit || stamp_hit(LabG<P64>::stamp(g), a.window);
        if (Ks == 1) {
          out[cbeg + j * 256 + threadIdx.x] = LabG<P64>::label(g);
        } else {
          s_lab[j * 256 + threadIdx.x] = LabG<P64>::label(g);
        }
      }
    }
    if (a.pull && __any_sync(kFull, hit) && lane == 0) {
      atomicOr(&hb.hit[entry], 1u);
    }
    if (Ks == 1) {
      continue;
    }
    // ---- counting sort by class: per-class counts (warp-aggregated: one atomic per class and warp), an
    // exclusive scan of the counts, the scatter into s_sorted and a coalesced copy back to the row
    for (uint32_t t = threadIdx.x; t <= Ks; t += 256) {
      s_cnt[t] = 0;
    }
    __syncthreads();
#pragma unroll 1
    for (int j = 0; j < B; ++j) {
      const uint32_t e = j * 256 + threadIdx.x;
      const uint32_t cls = cbeg + e < cend ? lowbias32(s_lab[e]) & (Ks - 1) : kEmpty;
      const unsigned peers = __match_any_sync(kFull, cls);
      const int leader = __ffs(peers) - 1;
      uint32_t base = 0;
      if (cls != kEmpty && lane == leader) {
        base = atomicAdd(&s_cnt[cls], static_cast<uint32_t>(__popc(peers)));
      }
      s_rank[e] =
          static_cast<uint16_t>(__shfl_sync(kFull, base, leader) + __popc(peers & ((1u << lane) - 1u)));
    }
    __syncthreads();
    {
      const uint32_t c = threadIdx.x < Ks ? s_cnt[threadIdx.x] : 0u;
      uint32_t x = c;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(kFull, x, o);
        x += lane >= o ? y : 0u;
      }
      if (lane == 31) {
        s_wsum[wib] = x;
      }
      __syncthreads();
      for (int w = 0; w < wib; ++w) {
        x += s_wsum[w];
      }
      if (threadIdx.x < Ks) {
        s_cnt[threadIdx.x] = x - c; // only this thread reads or writes entry threadIdx.x
      }
      if (threadIdx.x == 0) {
        s_cnt[Ks] = cend - cbeg;
      }
    }
    __syncthreads();
#pragma unroll 1
    for (int j = 0; j < B; ++j) {
      const uint32_t e = j * 256 + threadIdx.x;
      if (cbeg + e < cend) {
        const uint32_t l = s_lab[e];
        s_sorted[s_cnt[lowbias32(l) & (Ks - 1)] + s_rank[e]] = l;
      }
    }
    uint16_t *off = hb.cls + hb.cls_off[entry] + hb.item_chunk[it] * (Ks + 1);
    for (uint32_t t = threadIdx.x; t <= Ks; t += 256) {
      off[t] = static_cast<uint16_t>(s_cnt[t]);
    }
    __syncthreads();
#pragma unroll 1
    for (int j = 0; j < B; ++j) {
      const uint32_t e = j * 256 + threadIdx.x;
      if (cbeg + e < cend) {
        out[cbeg + e] = s_sorted[e];
      }
    }
    __syncthreads(); // s_sorted and s_cnt are free for the next item
  }
}

// One warp inserts up to 32 staged labels (one per lane where `valid`) into the rate table and appends the slots
// it claims to the list. With unit edge weights the claimer does not add its 1 (see team_table_add). Returns, in
// every lane, whether the claims of the running class have passed `limit`.
template <bool EW>
__device__ __forceinline__ bool rate_insert(uint32_t *keys, int32_t *vals, uint16_t *list, uint32_t *s_claims,
                                            uint32_t limit, uint32_t key, int32_t w, bool valid, int lane) {
  uint32_t slot = 0;
  bool claimed = false;
  if (valid) {
    // the class fixes the low bits of lowbias32(key): the slot comes from another hash of the key
    slot = lowbias32(key ^ 0x9E3779B9u) & (kRateSlots - 1);
    while (true) {
      const uint32_t prev = atomicCAS(&keys[slot], kEmpty, key);
      if (prev == kEmpty || prev == key) {
        claimed = prev == kEmpty;
        if (EW || !claimed) {
          atomicAdd(&vals[slot], w);
        }
        break;
      }
      slot = (slot + 1) & (kRateSlots - 1);
    }
  }
  const unsigned mask = __ballot_sync(kFull, claimed);
  if (mask == 0) {
    return false;
  }
  const uint32_t n = __popc(mask);
  uint32_t base = 0;
  if (lane == 0) {
    base = atomicAdd(s_claims, n);
  }
  base = __shfl_sync(kFull, base, 0);
  const uint32_t idx = base + __popc(mask & ((1u << lane) - 1u));
  if (claimed && idx < kRateListCap) {
    list[idx] = static_cast<uint16_t>(slot);
  }
  return base + n > limit;
}

// header of a rate item in shared memory, loaded by one thread
struct RateHead {
  uint32_t it;  // item index; >= num_items once the queue is drained
  uint32_t go;  // the item's hub is this rank's and active
  uint32_t c0, u, beg, full_deg, own, row, coff, res;
  int32_t uw, own_w;
};

__device__ __forceinline__ void rate_load_head(const SweepArgs &a, const HubArgs &hb, RateHead *h) {
  const uint32_t it = atomicAdd(hb.queue, 1u);
  h->it = it;
  h->go = 0;
  if (it >= hb.num_items) {
    return;
  }
  const uint32_t entry = hb.item_entry[it];
  const uint32_t u = a.list[entry];
  if (entry % hb.world != hb.rank || !(a.active == nullptr || a.pull || a.active[u] != 0)) {
    return;
  }
  const uint32_t beg = a.xadj[u];
  const uint32_t own = a.label[u];
  h->go = 1;
  h->c0 = hb.item_cls[it];
  h->u = u;
  h->beg = beg;
  h->full_deg = a.xadj[u + 1] - beg;
  h->own = own;
  h->row = hb.lab_off[entry];
  h->coff = hb.cls_off != nullptr ? hb.cls_off[entry] : 0u;
  h->res = hb.sel_begin[entry];
  h->uw = a.vwgt != nullptr ? a.vwgt[u] : 1;
  h->own_w = a.weight[own];
}

// Per-phase device time of the rate kernel's items, for scripts/hub_rate_phases.py: only a library built with
// -DKMP_HUB_PHASE_STAMPS takes %globaltimer stamps; otherwise the stamps compile to nothing. Thread 0 adds, in ns:
// [0] waiting for the item's header (from the end of the previous item to the barrier after which it is read),
// [1] stream + insert, [2] select, [3] clear (also the full clear of a split), [4] items rated, [5] items claimed,
// [6] time the loading thread spends in rate_load_head (for the next item).
#ifdef KMP_HUB_PHASE_STAMPS
constexpr bool kHubPhaseStamps = true;
#else
constexpr bool kHubPhaseStamps = false;
#endif
__device__ unsigned long long g_hub_phase[7];
__device__ __forceinline__ unsigned long long phase_clock() {
  unsigned long long t = 0;
  if constexpr (kHubPhaseStamps) {
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  }
  return t;
}
// adds now - t0 (or 1 when count) to slot i and returns now
__device__ __forceinline__ unsigned long long phase_add(int i, unsigned long long t0, bool count = false) {
  const unsigned long long t = phase_clock();
  if constexpr (kHubPhaseStamps) {
    atomicAdd(&g_hub_phase[i], count ? 1ull : t - t0);
  }
  return t;
}
__device__ __forceinline__ void rate_load_head_timed(const SweepArgs &a, const HubArgs &hb, RateHead *h) {
  const unsigned long long t0 = phase_clock();
  rate_load_head(a, hb, h);
  phase_add(6, t0);
}

// rate: one CTA per (hub, hash class) item; writes the class's best and favored candidates
template <bool EW> __global__ void __launch_bounds__(kRateThreads, 1) sweep_hub_rate(const SweepArgs a, const HubArgs hb) {
  constexpr int T = kRateThreads;
  constexpr int kWarps = T / 32;
  constexpr int B = 8; // independent label loads in flight per lane
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint32_t *keys = reinterpret_cast<uint32_t *>(smem_raw);
  int32_t *vals = reinterpret_cast<int32_t *>(smem_raw + sizeof(uint32_t) * kRateSlots);
  uint32_t *stage_k = reinterpret_cast<uint32_t *>(smem_raw + 8 * kRateSlots);
  int32_t *stage_w = reinterpret_cast<int32_t *>(stage_k + kWarps * kRateStage); // EW only
  uint16_t *list = reinterpret_cast<uint16_t *>(stage_k + (EW ? 2 : 1) * kWarps * kRateStage);
  __shared__ Cand s_red[kWarps];
  __shared__ RateHead s_head[2];
  __shared__ uint32_t s_claims, s_piece;
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int wib = tid >> 5;
  const unsigned below = (1u << lane) - 1u;
  uint32_t *stk = stage_k + wib * kRateStage;
  int32_t *stw = stage_w + wib * kRateStage;
  for (uint32_t s = tid; s < kRateSlots; s += T) {
    keys[s] = kEmpty;
    vals[s] = 0;
  }
  // a class with one label never splits, one with two may: the limit is >= 2 so that K stays below 2^32
  const uint32_t limit = (hb.sel_limit != 0 && hb.sel_limit < kRateListCap) ? max(hb.sel_limit, 2u) : kRateListCap;
  if (tid == 0) {
    rate_load_head_timed(a, hb, &s_head[0]);
  }
  unsigned long long t_ph = phase_clock(); // thread 0: the last phase stamp
  for (uint32_t b = 0;; b ^= 1) {
    __syncthreads(); // s_head[b] is loaded, the table is clean, s_head[b ^ 1] is no longer read
    if (tid == 0) {
      t_ph = phase_add(0, t_ph);
    }
    if (s_head[b].it >= hb.num_items) {
      break;
    }
    if (tid == 0) {
      phase_add(5, 0, true);
    }
    // lane 0 of the last warp loads the next item's header while this item streams
    bool next = tid == (kWarps - 1) * 32;
    if (s_head[b].go != 0) {
      const uint32_t c0 = s_head[b].c0, u = s_head[b].u, beg = s_head[b].beg, full_deg = s_head[b].full_deg;
      const uint32_t own = s_head[b].own;
      const int32_t uw = s_head[b].uw, own_w = s_head[b].own_w;
      const uint32_t deg = min(full_deg, a.max_num_neighbors);
      const uint32_t K0 = hub_classes(full_deg);
      const uint32_t Ks = EW ? 1u : hub_sort_classes(full_deg);
      // a chunk is read in P parts of about 256 labels of the class each: (chunk, part) pieces go to the warps
      const uint32_t pshift = Ks >= 8 ? 0u : 3u - (31 - __clz(Ks));
      const uint32_t pieces = ((deg + kChunkEdges - 1) / kChunkEdges) << pshift;
      const bool store_fav = (uw == own_w) && (own_w <= a.max_cluster_weight / 2);
      const uint32_t *lab = hb.lab + s_head[b].row;
      const uint16_t *coff = hb.cls + s_head[b].coff;
      Cand best = cand_none(), fav = cand_none();
      uint32_t cls = c0, K = K0;
      while (true) {
        if (tid == 0) {
          s_claims = 0;
          s_piece = 0;
        }
        __syncthreads();
        if (tid == 0) {
          t_ph = phase_clock();
        }
        if (next) {
          rate_load_head_timed(a, hb, &s_head[b ^ 1]);
          next = false;
        }
        // ---- read class `cls` (mod K): the range of its sort class in each chunk. Only where that range may
        // hold other classes (K > Ks) are the labels filtered and compacted in the warp's 64-entry ring, then
        // inserted 32 at a time. No barrier inside: a warp stops once the claims have passed the limit, after at
        // most one more batch of 32 claims, so the table stays below 3/4 full.
        const bool filter = K > Ks;
        const uint32_t scls = cls & (Ks - 1);
        bool wover = false;
        uint32_t head = 0, pend = 0; // ring index of the oldest staged label, labels staged (warp-uniform)
        while (!wover) {
          uint32_t p = 0;
          if (lane == 0) {
            p = atomicAdd(&s_piece, 1u);
          }
          p = __shfl_sync(kFull, p, 0);
          if (p >= pieces) {
            break;
          }
          const uint32_t ch = p >> pshift;
          const uint32_t step = 32u << pshift; // lane stride within the range
          uint32_t lo = 0, hi = min(deg - ch * kChunkEdges, static_cast<uint32_t>(kChunkEdges));
          if (Ks > 1) {
            const uint16_t *o = coff + ch * (Ks + 1) + scls;
            lo = o[0];
            hi = o[1];
          }
          const uint32_t *cl = lab + ch * kChunkEdges;
          const uint32_t wbase = beg + ch * kChunkEdges; // edge index of the chunk's first label (EW: unsorted)
          for (uint32_t i0 = lo + (p & ((1u << pshift) - 1)) * 32; i0 < hi && !wover; i0 += step * B) {
            uint32_t kb[B];
#pragma unroll
            for (int j = 0; j < B; ++j) {
              const uint32_t i = i0 + j * step + lane;
              kb[j] = i < hi ? __ldcg(cl + i) : kEmpty;
            }
#pragma unroll
            for (int j = 0; j < B; ++j) {
              if (!wover) {
                const uint32_t i = i0 + j * step + lane;
                if (!filter) {
                  const bool v = kb[j] != kEmpty;
                  wover = rate_insert<EW>(keys, vals, list, &s_claims, limit, kb[j], (EW && v) ? a.adjwgt[wbase + i] : 1,
                                          v, lane);
                  continue;
                }
                const bool in = kb[j] != kEmpty && (lowbias32(kb[j]) & (K - 1)) == cls;
                const unsigned m = __ballot_sync(kFull, in);
                if (in) {
                  const uint32_t pos = (head + pend + __popc(m & below)) & (kRateStage - 1);
                  stk[pos] = kb[j];
                  if (EW) {
                    stw[pos] = a.adjwgt[wbase + i];
                  }
                }
                pend += __popc(m);
                if (pend >= 32) {
                  __syncwarp();
                  const uint32_t sl = (head + lane) & (kRateStage - 1);
                  wover = rate_insert<EW>(keys, vals, list, &s_claims, limit, stk[sl], EW ? stw[sl] : 1, true, lane);
                  __syncwarp(); // the ring slots are read before they are staged again
                  head = (head + 32) & (kRateStage - 1);
                  pend -= 32;
                }
              }
            }
          }
        }
        if (!wover) { // insert the rest
          __syncwarp();
          const bool v = lane < pend;
          const uint32_t sl = (head + lane) & (kRateStage - 1);
          wover = rate_insert<EW>(keys, vals, list, &s_claims, limit, v ? stk[sl] : 0u, (EW && v) ? stw[sl] : 1, v, lane);
        }
        const bool over = __syncthreads_or(wover);
        if (tid == 0) {
          t_ph = phase_add(1, t_ph);
        }
        if (over) {
          // more labels than the list takes: clear the whole table (not every claim is listed), split the class
          // by the next hash bit and stream again
          for (uint32_t s = tid; s < kRateSlots; s += T) {
            keys[s] = kEmpty;
            vals[s] = 0;
          }
          K <<= 1;
          __syncthreads();
          if (tid == 0) {
            t_ph = phase_add(3, t_ph);
          }
          continue;
        }
        const uint32_t nc = s_claims;
        // ---- select (as the team kernels): pass A without weights, pass B only if the top entry is full
        Cand c = cand_none(), f = cand_none();
        for (uint32_t l = tid; l < nc; l += T) {
          const uint32_t s = list[l];
          const uint32_t k = keys[s];
          const int32_t r = vals[s] + (EW ? 0 : 1);
          if (r > 0 && r >= c.gain) {
            const Cand x{r, 0, tie_hash(a.base_tie, u, k), k};
            if (cand_better<0>(x, c)) {
              c = x;
            }
          }
          if (store_fav && r > 0 && r >= f.gain) {
            const Cand y{r, 0, tie_hash(a.base_fav, u, k), k};
            if (cand_better<0>(y, f)) {
              f = y;
            }
          }
        }
        Cand cb = team_argmax<0, T>(1, tid, c, s_red);
        if (store_fav) {
          const Cand cf = team_argmax<0, T>(1, tid, f, s_red);
          if (cand_better<0>(cf, fav)) {
            fav = cf;
          }
        }
        bool top_ok = true;
        if (cb.gain > 0) {
          top_ok = (a.weight[cb.key] + uw <= a.max_cluster_weight) || (cb.key == own);
          if (a.communities != nullptr) {
            top_ok = top_ok && (a.communities[cb.key] == a.communities[own]);
          }
        }
        if (!top_ok) {
          Cand ce = cand_none();
          for (uint32_t l0 = 0; l0 < nc; l0 += T * 4) {
            uint32_t kk[4];
            int32_t rr[4], ww[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const uint32_t l = l0 + j * T + tid;
              const uint32_t s = l < nc ? list[l] : 0u;
              kk[j] = l < nc ? keys[s] : kEmpty;
              rr[j] = l < nc ? vals[s] + (EW ? 0 : 1) : 0;
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              ww[j] = kk[j] != kEmpty ? a.weight[kk[j]] : 0;
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              if (kk[j] != kEmpty) {
                Cand ff;
                const Cand cc = eval_candidate_w<0>(a, u, own, uw, own_w, kk[j], rr[j], ww[j], false, ff);
                if (cand_better<0>(cc, ce)) {
                  ce = cc;
                }
              }
            }
          }
          cb = team_argmax<0, T>(1, tid, ce, s_red);
        }
        if (cand_better<0>(cb, best)) {
          best = cb;
        }
        if (tid == 0) {
          t_ph = phase_add(2, t_ph);
        }
        // every thread clears the listed slots it scanned
        for (uint32_t l = tid; l < nc; l += T) {
          const uint32_t s = list[l];
          keys[s] = kEmpty;
          vals[s] = 0;
        }
        __syncthreads(); // table clean, s_claims read
        if (tid == 0) {
          t_ph = phase_add(3, t_ph);
        }
        // next class: the second half of the deepest split whose first half is done, up to the item's own class
        bool done = true;
        while (K > K0) {
          const uint32_t half = K >> 1;
          if ((cls & half) == 0) {
            cls |= half;
            done = false;
            break;
          }
          cls &= ~half;
          K = half;
        }
        if (done) {
          break;
        }
      }
      if (tid == 0) {
        hb.part_best[s_head[b].res + c0] = best;
        hb.part_fav[s_head[b].res + c0] = fav;
        phase_add(4, 0, true);
      }
    }
    if (next) { // an item with nothing to do
      rate_load_head_timed(a, hb, &s_head[b ^ 1]);
    }
    if (tid == 0) {
      t_ph = phase_clock();
    }
  }
}

// final: one warp per hub: reduce its buckets' (clusterer: hash classes') candidates, then propose / store the
// favored cluster.
template <int MODE> __global__ void __launch_bounds__(256) sweep_hub_final(const SweepArgs a, const HubArgs hb) {
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  unsigned long long edges = 0, nodes = 0;
  for (uint32_t i = warp; i < a.list_size; i += nwarps) {
    if (i % hb.world != hb.rank) {
      continue;
    }
    const uint32_t u = a.list[i];
    bool flag = true;
    if (a.active != nullptr) {
      int fl = 0, ht = 0;
      if (lane == 0) {
        fl = static_cast<int>(a.active[u]);
        if (a.pull) {
          ht = static_cast<int>(hb.hit[i]);
          hb.hit[i] = 0;
        }
      }
      fl = __shfl_sync(kFull, fl, 0);
      ht = __shfl_sync(kFull, ht, 0);
      flag = fl != 0;
      if (fl == 0 && ht == 0) {
        continue;
      }
    }
    const uint32_t full_deg = a.xadj[u + 1] - a.xadj[u];
    uint32_t deg = full_deg;
    if (deg > a.max_num_neighbors) {
      deg = a.max_num_neighbors;
    }
    const uint32_t own = a.label[u];
    const int32_t uw = a.vwgt != nullptr ? a.vwgt[u] : 1;
    const int32_t own_w = a.weight[own];
    const uint32_t pieces = MODE == 0 ? hub_classes(full_deg) : hub_buckets(full_deg);
    const uint32_t first = hb.sel_begin[i];
    const bool store_fav = (MODE == 0) && (uw == own_w) && (own_w <= a.max_cluster_weight / 2);
    Cand c = cand_none(), f = cand_none();
    for (uint32_t q = lane; q < pieces; q += 32) {
      const Cand pb = hb.part_best[first + q];
      if (cand_better<MODE>(pb, c)) {
        c = pb;
      }
      if (MODE == 0) {
        const Cand pf = hb.part_fav[first + q];
        if (cand_better<0>(pf, f)) {
          f = pf;
        }
      }
    }
    const Cand best = warp_argmax<MODE>(kFull, c);
    const Cand fav = (MODE == 0) ? warp_argmax<0>(kFull, f) : cand_none();
    if (lane == 0) {
      edges += deg;
      nodes += 1;
      if (a.active != nullptr && flag) {
        a.active[u] = 0;
      }
      uint32_t target;
      if (finish_vertex<MODE>(a, u, own, store_fav, best, fav, target)) {
        const uint32_t idx = atomicAdd(a.mover_count, 1u);
        emit_proposal<MODE>(a, idx, u, target, uw);
      }
    }
  }
  block_count_flush(a, edges, nodes);
}

} // namespace kmp
