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
//   tier 7 (deg >= 8192 / 16384) sweep_hub_*  : edge-parallel chunks, label-partitioned bucket appends (see below)
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
    uint32_t u = 0, target = 0;
    int32_t uw = 1;
    if (i < a.list_size) {
      u = a.list[i];
      const bool flag = a.active == nullptr || a.active[u] != 0;
      if (flag || a.pull) {
        const uint32_t beg = a.xadj[u];
        uint32_t deg = a.xadj[u + 1] - beg;
        if (deg > a.max_num_neighbors) {
          deg = a.max_num_neighbors;
        }
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
          if (j < static_cast<int>(deg)) {
            const uint32_t v = a.adjncy[beg + j];
            const typename LabG<P64>::word g = load_labg<P64>(a, v);
            hit = hit || stamp_hit(LabG<P64>::stamp(g), a.window);
            bool ok = true;
            if (MODE == 1 && a.communities != nullptr) {
              ok = a.communities[u] == a.communities[v];
            }
            if (ok) {
              keys[j] = LabG<P64>::label(g);
              ws[j] = EW ? a.adjwgt[beg + j] : 1;
            }
          }
        }
        if (flag || hit) {
          edges += deg;
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
          proposes = finish_vertex<MODE>(a, u, own, store_fav, best, fav, target);
        }
      }
    }
    // ONE atomic on the proposal counter per CTA iteration (256 vertices): on graphs that live in this tier
    // (grid, road) nearly every vertex proposes in round 0 and the single address serialises in L2
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
// tiers 2..5: a TEAM of T threads (one warp, 128, 512 or 1024 threads) per vertex, rating map = an
// open-addressing table in shared memory sized for the tier's largest degree (load <= 0.5).
//
//   1. gather : every thread loads its neighbours (coalesced adjncy stream), gathers the packed
//               (label, stamp) word of each -- B independent gathers in flight per thread -- and inserts the
//               label into the table (one shared-memory CAS + one add per edge; the FixedSizeSparseMap role,
//               kaminpar-common/datastructures/fixed_size_sparse_map.h). The stamps decide whether the vertex
//               is active at all (pull activation, see lp_device.cuh); an inactive vertex stops here.
//   2. select : the table is scanned once WITHOUT touching the cluster-weight array: the team arg-max of
//               (rating, tie hash) over all entries is the favored cluster, and -- if that cluster is feasible,
//               one broadcast load -- also the move target (lp_clusterer.cc:199-250). Only when the top entry is
//               infeasible the entries are evaluated in full (one weight gather per distinct label).
//               The refiner (k blocks, weights cached) always evaluates in full.
//   3. the scan clears the slots it visited; vertices are claimed from a work queue.
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
  static __device__ __forceinline__ bool any(int id, bool p) {
    if (T == 32) {
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
// this halves the shared-memory atomics per edge.
template <bool V16, bool EW>
__device__ __forceinline__ void team_table_add(uint32_t *keys, typename TeamVals<V16>::word *vals, uint32_t mask,
                                               bool direct, uint32_t key, int32_t w) {
  uint32_t slot = direct ? key : (lowbias32(key) & mask);
  while (true) {
    const uint32_t prev = atomicCAS(&keys[slot], kEmpty, key);
    if (!EW && prev == kEmpty) {
      return;
    }
    if (prev == kEmpty || prev == key) {
      TeamVals<V16>::add(vals, slot, w);
      return;
    }
    slot = (slot + 1) & mask;
  }
}
template <bool V16, bool EW>
__device__ __forceinline__ int32_t team_rating(const typename TeamVals<V16>::word *vals, uint32_t slot) {
  return TeamVals<V16>::get(vals, slot) + (EW ? 0 : 1);
}

template <int MODE, bool EW, bool P64, int T, int SLOTS, int TEAMS, bool V16 = false>
__global__ void __launch_bounds__(T *TEAMS) sweep_team(const SweepArgs a) {
  static_assert((SLOTS & (SLOTS - 1)) == 0, "table size must be a power of two");
  static_assert(!(V16 && EW), "16-bit ratings need unit edge weights");
  using TV = TeamVals<V16>;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ Cand s_red_all[TEAMS][T > 32 ? T / 32 : 1];
  __shared__ uint32_t s_next[TEAMS];
  const int team = threadIdx.x / T;
  const int tid = threadIdx.x % T;
  const int bar = 1 + team;
  uint32_t *keys = reinterpret_cast<uint32_t *>(smem_raw) + static_cast<size_t>(team) * SLOTS;
  typename TV::word *vals = reinterpret_cast<typename TV::word *>(
      smem_raw + sizeof(uint32_t) * SLOTS * TEAMS + static_cast<size_t>(team) * SLOTS * TV::kBytesPerSlot);
  Cand *s_red = s_red_all[team];
  for (int s = tid; s < SLOTS; s += T) {
    keys[s] = kEmpty;
    TV::clear(vals, s);
  }
  unsigned long long edges = 0, nodes = 0;
  // work queue: the next list index is claimed one vertex ahead
  if (tid == 0) {
    s_next[team] = atomicAdd(a.queue, 1u);
  }
  TeamSync<T>::sync(bar);
  while (true) {
    const uint32_t i = s_next[team];
    TeamSync<T>::sync(bar); // everybody has read s_next
    if (i >= a.list_size) {
      break;
    }
    if (tid == 0) {
      s_next[team] = atomicAdd(a.queue, 1u);
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
    const uint32_t distinct = deg < a.num_labels ? deg : a.num_labels;
    const bool direct = a.num_labels <= static_cast<uint32_t>(SLOTS);
    uint32_t cap = direct ? pow2_ceil(a.num_labels) : pow2_ceil(2 * distinct);
    if (cap < 32) {
      cap = 32;
    }
    const uint32_t mask = cap - 1;
    // ---- 1. gather + insert --------------------------------------------------------------------
    bool hit = false;
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
#pragma unroll
      for (int j = 0; j < B; ++j) {
        if (kb[j] != kEmpty) {
          team_table_add<V16, EW>(keys, vals, mask, direct, kb[j], wb[j]);
        }
      }
    }
    const bool any_hit = TeamSync<T>::any(bar, hit); // also the barrier after the inserts
    const bool act = flag || any_hit;
    // ---- 2. select ---------------------------------------------------------------------------------
    const bool store_fav = (MODE == 0) && (uw == own_w) && (own_w <= a.max_cluster_weight / 2);
    Cand best = cand_none(), fav = cand_none();
    if (act) {
      Cand c = cand_none(), f = cand_none();
      if (MODE == 0) {
        // pass A: no weight gathers
        for (uint32_t s = tid; s < cap; s += T) {
          const uint32_t k = keys[s];
          if (k != kEmpty) {
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
          for (uint32_t s0 = 0; s0 < cap; s0 += T * 4) {
            uint32_t kk[4];
            int32_t rr[4], ww[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const uint32_t s = s0 + j * T + tid;
              kk[j] = s < cap ? keys[s] : kEmpty;
              rr[j] = kk[j] != kEmpty ? team_rating<V16, EW>(vals, s) : 0;
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
        for (uint32_t s = tid; s < cap; s += T) {
          const uint32_t k = keys[s];
          if (k != kEmpty) {
            Cand ff;
            const Cand cc = eval_candidate_w<1>(a, u, own, uw, own_w, k, team_rating<V16, EW>(vals, s), a.weight[k], false, ff);
            if (cand_better<1>(cc, c)) {
              c = cc;
            }
          }
        }
        best = team_argmax<1, T>(bar, tid, c, s_red);
      }
    }
    // ---- 3. clear the table, finish the vertex ---------------------------------------------------
    TeamSync<T>::sync(bar); // all scans done before the slots are cleared
    for (uint32_t s = tid; s < cap; s += T) {
      keys[s] = kEmpty;
      TV::clear(vals, s);
    }
    if (act && tid == 0) {
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
    TeamSync<T>::sync(bar); // table clean, s_next written
  }
  block_count_flush(a, edges, nodes);
}

// ================================================================================================
// tier 7 (deg >= 8192 / 16384): edge-parallel, label-partitioned two-pass aggregation. No random access ever
// touches a table outside shared memory, and after the chunk is staged every warp works on its own:
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

// select: one warp per (hub, bucket): best candidates of the bucket's labels
template <int MODE> __global__ void __launch_bounds__(kSelWarps * 32) sweep_hub_select(const SweepArgs a, const HubArgs hb) {
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
    Cand c = cand_none(), f = cand_none();
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
      const bool store_fav = (MODE == 0) && (uw == own_w) && (own_w <= a.max_cluster_weight / 2);
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
        f = cand_none();
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
          bool lazy_done = false;
          if (MODE == 0 && K == 1 && !overflowed) {
            // Clusterer, single class: rank the labels WITHOUT their cluster weights (the team kernels do the
            // same): if the bucket's top label is feasible it is the bucket's best; the favored label never needs
            // weights. Only a full top label costs the second scan with one weight gather per label.
            Cand ct = cand_none();
            for (uint32_t s = lane; s < tcap; s += 32) {
              const uint32_t kx = keys[s];
              if (kx != kEmpty) {
                const int32_t r = vals[s];
                if (r >= ct.gain && r > 0) {
                  const Cand x{r, 0, tie_hash(a.base_tie, u, kx), kx};
                  if (cand_better<0>(x, ct)) {
                    ct = x;
                  }
                }
                if (store_fav && r >= f.gain && r > 0) {
                  const Cand y{r, 0, tie_hash(a.base_fav, u, kx), kx};
                  if (cand_better<0>(y, f)) {
                    f = y;
                  }
                }
              }
            }
            const Cand top = warp_argmax<0>(kFull, ct);
            bool top_ok = true;
            if (top.gain > 0) {
              top_ok = (a.weight[top.key] + uw <= a.max_cluster_weight) || (top.key == own);
              if (a.communities != nullptr) {
                top_ok = top_ok && (a.communities[top.key] == a.communities[own]);
              }
            }
            if (top_ok) {
              c = top;
              lazy_done = true;
            }
          }
          const bool evaluate = !overflowed && !lazy_done;
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
                  // (the favored candidate of the lazy pass is final: no second evaluation)
                  const Cand cc = eval_candidate_w<MODE>(a, u, own, uw, own_w, kk[j], rr[j], ww[j],
                                                         store_fav && !(MODE == 0 && K == 1), ff);
                  if (cand_better<MODE>(cc, c)) {
                    c = cc;
                  }
                  if (MODE == 0 && cand_better<0>(ff, f)) {
                    f = ff;
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
    const Cand best = warp_argmax<MODE>(kFull, c);
    const Cand fav = (MODE == 0) ? warp_argmax<0>(kFull, f) : cand_none();
    if (lane == 0) {
      hb.part_best[it] = best;
      hb.part_fav[it] = fav;
    }
  }
}

// final: one warp per hub: reduce its buckets' candidates, then propose / store the favored cluster.
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
    const uint32_t pieces = hub_buckets(full_deg);
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
