// Commit kernels: resolve the proposals of one sub-round deterministically (DESIGN.md "commit
// rule"), apply the accepted moves and re-activate neighbourhoods.
//
// They replace the reference's immediate, racy move (label_propagation.h:817-841 try_node_move,
// :2139-2152 move_cluster_weight, partitioned_graph.h:397-428 move_block_weight) by an
// order-independent rule: proposals into a target are accepted by ladder level
// lvl(u) = min(clz(prio(u)), 15) from the top level downwards as long as the target's weight limit
// holds; with several passes the weight of accepted departures is credited.
#pragma once

#include "lp_device.cuh"

namespace kmp {

struct CommitArgs {
  // graph
  const uint32_t *__restrict__ xadj;
  const uint32_t *__restrict__ adjncy;
  const int32_t *__restrict__ vwgt; // nullable
  // state
  uint32_t *__restrict__ label;
  int32_t *__restrict__ weight;       // [n] or [k]
  const int32_t *__restrict__ max_w;  // refiner [k]
  const int32_t *__restrict__ min_w;  // refiner [k], nullable
  uint8_t *__restrict__ active;
  int32_t max_cluster_weight;
  uint32_t k;
  // proposals
  const uint32_t *__restrict__ mv_u;
  const uint32_t *__restrict__ mv_t;
  uint8_t *__restrict__ acc; // 0 rejected/pending, 1 accepted, 2 contended-pending (clusterer)
  const uint32_t *__restrict__ mover_count;
  uint32_t *__restrict__ next_mover_count; // zeroed for the following sub-round
  uint32_t *__restrict__ also_zero;        // nullable: a second proposal counter to zero (sharded run: send buffer)
  uint32_t base_commit;
  // clusterer
  int32_t *__restrict__ incoming; // [n]
  uint32_t *__restrict__ slotmap; // [n], kEmpty when unused
  uint32_t *__restrict__ cslot;   // [movers]
  int32_t *__restrict__ chist;    // [movers][16], zero when unused
  // refiner
  int32_t *__restrict__ hist;  // [k][16]  weight per (target, level); becomes suffix sums (cum)
  int32_t *__restrict__ jmin;  // [k]
  int32_t *__restrict__ out_cur;   // [k] credited departures (complete)
  int32_t *__restrict__ out_delta; // [k] departures accepted in the running pass
  int32_t *__restrict__ ohist; // [k][16] source-side ladder (min weights)
  int32_t *__restrict__ ojmin; // [k]
  // results
  uint32_t *__restrict__ moved_count;
  // packed (label, stamp) gather array of the sweeps (lp_device.cuh) and the stamp of this sub-round
  void *__restrict__ labg;
  uint32_t stamp;
};

__device__ __forceinline__ int32_t node_weight(const CommitArgs &a, uint32_t u) {
  return a.vwgt != nullptr ? a.vwgt[u] : 1;
}

// ---- clusterer: the whole commit of a sub-round in ONE cooperative launch -------------------------
// (unpack + accumulate the all-gathered proposals when sharded) -> classify -> decide -> apply, separated by
// grid-wide barriers instead of kernel boundaries: a sub-round's commit is a few microseconds of work, so
// three to five launches with their drain / fill gaps cost more than the work itself.
struct GridBarrier {
  unsigned *count;        // arrivals of the running barrier (returns to 0)
  volatile unsigned *gen; // generation, only ever incremented
};
// Thread 0 of each CTA arrives with a release-acquire add (its CTA's writes are ordered before it by the first
// __syncthreads) and the last arrival publishes the next generation with a release store; the others wait for
// it with acquire loads. Release / acquire at GPU scope instead of sequentially consistent fences: the barrier
// runs up to four times per sub-round.
__device__ __forceinline__ void grid_sync(const GridBarrier &b) {
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned g = *b.gen; // before the arrival: the release add keeps it there
    unsigned prev;
    asm volatile("atom.add.acq_rel.gpu.u32 %0, [%1], 1;" : "=r"(prev) : "l"(b.count) : "memory");
    if (prev == gridDim.x - 1) {
      *b.count = 0;
      asm volatile("st.release.gpu.u32 [%0], %1;" ::"l"(b.gen), "r"(g + 1) : "memory");
    } else {
      unsigned cur;
      do {
        asm volatile("ld.acquire.gpu.u32 %0, [%1];" : "=r"(cur) : "l"(b.gen) : "memory");
      } while (cur == g);
    }
  }
  __syncthreads();
}

struct GatheredArgs {              // sharded run: proposal buffers of all ranks, [count, -, -, -, u[cap], t[cap]] each
  const uint32_t *gathered;        // nullptr: mv_u / mv_t / *mover_count already hold the proposals
  uint32_t world, cap;
  uint32_t *mover_count_w;         // writable alias of CommitArgs::mover_count
};

// The phases of a grid-wide clusterer commit over the `cnt` proposals (grid_sync between them). Thread `tid` of
// `nth` takes proposals tid, tid + nth, ... in every phase, so acc[i] / cslot[i] are read back by the thread that
// wrote them; what other threads accumulated in an earlier phase is read through L2 (__ldcg).
// (1) classify: uncontended targets accept everything; contended ones get a slot and a level histogram
__device__ __forceinline__ void cluster_classify(const CommitArgs &a, uint32_t cnt, uint32_t tid, uint32_t nth) {
  for (uint32_t i = tid; i < cnt; i += nth) {
    const uint32_t u = a.mv_u[i];
    const uint32_t t = a.mv_t[i];
    if (a.weight[t] + __ldcg(&a.incoming[t]) <= a.max_cluster_weight) {
      a.acc[i] = 1;
    } else {
      const uint32_t prev = atomicCAS(&a.slotmap[t], kEmpty, i);
      const uint32_t slot = prev == kEmpty ? i : prev;
      a.cslot[i] = slot;
      const uint32_t lvl = ladder_level(bijective32(u, a.base_commit));
      atomicAdd(&a.chist[static_cast<size_t>(slot) * kLadderLevels + lvl], node_weight(a, u));
      a.acc[i] = 2;
    }
  }
}
// (2) decide (contended proposals): accept iff level >= jmin(target); weights are still the frozen ones
__device__ __forceinline__ void cluster_decide(const CommitArgs &a, uint32_t cnt, uint32_t tid, uint32_t nth) {
  for (uint32_t i = tid; i < cnt; i += nth) {
    if (a.acc[i] != 2) {
      continue;
    }
    const uint32_t u = a.mv_u[i];
    const uint32_t t = a.mv_t[i];
    const int32_t *h = a.chist + static_cast<size_t>(a.cslot[i]) * kLadderLevels;
    const int32_t w_t = a.weight[t];
    int32_t cum = 0;
    int jm = kLadderLevels; // none
#pragma unroll
    for (int j = kLadderLevels - 1; j >= 0; --j) {
      cum += __ldcg(&h[j]);
      if (w_t + cum <= a.max_cluster_weight) {
        jm = j; // feasible at level j; keep lowering while it still fits (cum is monotone)
      }
    }
    const uint32_t lvl = ladder_level(bijective32(u, a.base_commit));
    a.acc[i] = static_cast<int>(lvl) >= jm ? 1 : 0;
  }
}
// (3) apply the accepted moves, clean the contended-target scratch, zero the next sub-round's proposal counter
template <bool P64>
__device__ __forceinline__ void cluster_apply(const CommitArgs &a, uint32_t cnt, uint32_t tid, uint32_t nth) {
  if (tid == 0) {
    *a.next_mover_count = 0;
    if (a.also_zero != nullptr) {
      *a.also_zero = 0;
    }
  }
  uint32_t moved = 0;
  for (uint32_t i = tid; i < cnt; i += nth) {
    const uint32_t u = a.mv_u[i];
    const uint32_t t = a.mv_t[i];
    a.incoming[t] = 0;
    if (__ldcg(&a.slotmap[t]) == i) {
      int32_t *h = a.chist + static_cast<size_t>(i) * kLadderLevels;
#pragma unroll
      for (int j = 0; j < kLadderLevels; ++j) {
        h[j] = 0;
      }
      a.slotmap[t] = kEmpty;
    }
    if (a.acc[i] == 1) {
      const uint32_t from = a.label[u];
      const int32_t w = node_weight(a, u);
      atomicAdd(&a.weight[t], w);
      atomicSub(&a.weight[from], w);
      a.label[u] = t;
      static_cast<typename LabG<P64>::word *>(a.labg)[u] = LabG<P64>::pack(t, a.stamp);
      ++moved;
    } else {
      a.active[u] = 1;
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    moved += __shfl_xor_sync(kFull, moved, o);
  }
  if ((threadIdx.x & 31) == 0 && moved != 0) {
    atomicAdd(a.moved_count, moved);
  }
}

template <bool P64>
__global__ void __launch_bounds__(256) commit_cluster_fused(const CommitArgs a, const GatheredArgs ga, const GridBarrier bar) {
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t nth = gridDim.x * blockDim.x;
  uint32_t cnt;
  if (ga.gathered != nullptr) {
    // ---- unpack (rank order) + accumulate incoming[] over ALL proposals
    const size_t stride = 4 + 2 * static_cast<size_t>(ga.cap);
    uint32_t total = 0;
    uint32_t *mv_u = const_cast<uint32_t *>(a.mv_u), *mv_t = const_cast<uint32_t *>(a.mv_t);
    for (uint32_t r = 0; r < ga.world; ++r) {
      const uint32_t c = ga.gathered[r * stride];
      for (uint32_t i = tid; i < c; i += nth) {
        const uint32_t u = ga.gathered[r * stride + 4 + i];
        const uint32_t t = ga.gathered[r * stride + 4 + ga.cap + i];
        mv_u[total + i] = u;
        mv_t[total + i] = t;
        atomicAdd(&a.incoming[t], node_weight(a, u));
      }
      total += c;
    }
    cnt = total;
    if (tid == 0) {
      *ga.mover_count_w = total;
    }
    grid_sync(bar);
  } else {
    cnt = *a.mover_count;
  }
  cluster_classify(a, cnt, tid, nth);
  grid_sync(bar);
  cluster_decide(a, cnt, tid, nth);
  grid_sync(bar);
  cluster_apply<P64>(a, cnt, tid, nth);
}

// ---- refiner: the whole commit of a sub-round in ONE cooperative launch -----------------------------
// (unpack) -> level histograms -> suffix sums -> passes x (jmin, decide) -> [min-weight ladder] -> apply + reset.
// Block-weight style accumulators are privatised per CTA in shared memory when k is small: millions of
// proposals hitting k <= a few hundred global addresses serialise in the L2 atomic units.
constexpr uint32_t kSmemPrivLimit = 8192; // ints of dynamic shared memory a commit kernel may use

template <bool P64>
__global__ void __launch_bounds__(256) commit_refine_fused(const CommitArgs a, const GatheredArgs ga, const GridBarrier bar,
                                                            const uint32_t passes) {
  extern __shared__ int32_t s_priv[]; // k * 16 ints (level histograms), later k ints (departure / weight deltas)
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t nth = gridDim.x * blockDim.x;
  const bool priv_h = a.k * kLadderLevels <= kSmemPrivLimit;
  const bool priv_k = a.k <= kSmemPrivLimit;
  uint32_t cnt;
  // ---- proposals (unpacked from the all-gathered buffers when sharded), acc = 0, level histograms
  if (priv_h) {
    for (uint32_t b = threadIdx.x; b < a.k * kLadderLevels; b += blockDim.x) {
      s_priv[b] = 0;
    }
    __syncthreads();
  }
  if (ga.gathered != nullptr) {
    const size_t stride = 4 + 2 * static_cast<size_t>(ga.cap);
    uint32_t total = 0;
    uint32_t *mv_u = const_cast<uint32_t *>(a.mv_u), *mv_t = const_cast<uint32_t *>(a.mv_t);
    for (uint32_t r = 0; r < ga.world; ++r) {
      const uint32_t c = ga.gathered[r * stride];
      for (uint32_t i = tid; i < c; i += nth) {
        const uint32_t u = ga.gathered[r * stride + 4 + i];
        const uint32_t t = ga.gathered[r * stride + 4 + ga.cap + i];
        mv_u[total + i] = u;
        mv_t[total + i] = t;
        a.acc[total + i] = 0;
        const uint32_t slot = t * kLadderLevels + ladder_level(bijective32(u, a.base_commit));
        atomicAdd(priv_h ? &s_priv[slot] : &a.hist[slot], node_weight(a, u));
      }
      total += c;
    }
    cnt = total;
    if (tid == 0) {
      *ga.mover_count_w = total;
    }
  } else {
    cnt = *a.mover_count;
    for (uint32_t i = tid; i < cnt; i += nth) {
      const uint32_t u = a.mv_u[i];
      a.acc[i] = 0;
      const uint32_t slot = a.mv_t[i] * kLadderLevels + ladder_level(bijective32(u, a.base_commit));
      atomicAdd(priv_h ? &s_priv[slot] : &a.hist[slot], node_weight(a, u));
    }
  }
  if (priv_h) {
    __syncthreads();
    for (uint32_t b = threadIdx.x; b < a.k * kLadderLevels; b += blockDim.x) {
      if (s_priv[b] != 0) {
        atomicAdd(&a.hist[b], s_priv[b]);
      }
    }
  }
  grid_sync(bar);
  // ---- suffix sums of the level histograms, pass state
  for (uint32_t b = tid; b < a.k; b += nth) {
    int32_t cum = 0;
    for (int j = kLadderLevels - 1; j >= 0; --j) {
      cum += __ldcg(&a.hist[b * kLadderLevels + j]);
      a.hist[b * kLadderLevels + j] = cum;
    }
    a.out_cur[b] = 0;
    a.out_delta[b] = 0;
  }
  for (uint32_t p = 0; p < passes; ++p) {
    grid_sync(bar);
    // ---- jmin per block; folds the previous pass' departures into out_cur
    for (uint32_t b = tid; b < a.k; b += nth) {
      const int32_t credit = a.out_cur[b] + __ldcg(&a.out_delta[b]);
      a.out_cur[b] = credit;
      a.out_delta[b] = 0;
      int jm = kLadderLevels;
      for (int j = 0; j < kLadderLevels; ++j) {
        if (a.weight[b] + __ldcg(&a.hist[b * kLadderLevels + j]) - credit <= a.max_w[b]) {
          jm = j;
          break;
        }
      }
      a.jmin[b] = jm;
    }
    if (priv_k) {
      for (uint32_t b = threadIdx.x; b < a.k; b += blockDim.x) {
        s_priv[b] = 0;
      }
    }
    grid_sync(bar);
    // ---- decide
    for (uint32_t i = tid; i < cnt; i += nth) {
      if (a.acc[i] != 0) {
        continue;
      }
      const uint32_t u = a.mv_u[i];
      const uint32_t t = a.mv_t[i];
      const uint32_t lvl = ladder_level(bijective32(u, a.base_commit));
      if (static_cast<int>(lvl) >= __ldcg(&a.jmin[t])) {
        a.acc[i] = 1;
        const uint32_t from = a.label[u];
        // no credit for departures from a block with a min-weight constraint: the min-weight ladder below may
        // still revoke them, and arrivals accepted on that credit would overshoot the block's maximum
        if (a.min_w == nullptr || a.min_w[from] <= 0) {
          atomicAdd(priv_k ? &s_priv[from] : &a.out_delta[from], node_weight(a, u));
        }
      }
    }
    if (priv_k) {
      __syncthreads();
      for (uint32_t b = threadIdx.x; b < a.k; b += blockDim.x) {
        if (s_priv[b] != 0) {
          atomicAdd(&a.out_delta[b], s_priv[b]);
        }
      }
    }
  }
  if (a.min_w != nullptr) { // source-side ladder for min block weights
    grid_sync(bar);
    for (uint32_t i = tid; i < cnt; i += nth) {
      if (a.acc[i] == 1) {
        const uint32_t u = a.mv_u[i];
        atomicAdd(&a.ohist[a.label[u] * kLadderLevels + ladder_level(bijective32(u, a.base_commit))], node_weight(a, u));
      }
    }
    grid_sync(bar);
    for (uint32_t b = tid; b < a.k; b += nth) {
      int32_t cum[kLadderLevels];
      int32_t c = 0;
      for (int j = kLadderLevels - 1; j >= 0; --j) {
        c += __ldcg(&a.ohist[b * kLadderLevels + j]);
        cum[j] = c;
        a.ohist[b * kLadderLevels + j] = 0;
      }
      int jm = kLadderLevels;
      for (int j = 0; j < kLadderLevels; ++j) {
        if (a.weight[b] - cum[j] >= a.min_w[b]) {
          jm = j;
          break;
        }
      }
      a.ojmin[b] = jm;
    }
    grid_sync(bar);
    for (uint32_t i = tid; i < cnt; i += nth) {
      if (a.acc[i] == 1) {
        const uint32_t u = a.mv_u[i];
        if (static_cast<int>(ladder_level(bijective32(u, a.base_commit))) < __ldcg(&a.ojmin[a.label[u]])) {
          a.acc[i] = 0;
        }
      }
    }
  }
  grid_sync(bar);
  // ---- apply + reset of the histograms
  if (priv_k) {
    for (uint32_t b = threadIdx.x; b < a.k; b += blockDim.x) {
      s_priv[b] = 0;
    }
    __syncthreads();
  }
  if (tid == 0) {
    *a.next_mover_count = 0;
    if (a.also_zero != nullptr) {
      *a.also_zero = 0;
    }
  }
  for (uint32_t b = tid; b < a.k * kLadderLevels; b += nth) {
    a.hist[b] = 0;
  }
  uint32_t moved = 0;
  for (uint32_t i = tid; i < cnt; i += nth) {
    const uint32_t u = a.mv_u[i];
    if (a.acc[i] == 1) {
      const uint32_t t = a.mv_t[i];
      const uint32_t from = a.label[u];
      const int32_t w = node_weight(a, u);
      if (priv_k) {
        atomicAdd(&s_priv[t], w);
        atomicSub(&s_priv[from], w);
      } else {
        atomicAdd(&a.weight[t], w);
        atomicSub(&a.weight[from], w);
      }
      a.label[u] = t;
      static_cast<typename LabG<P64>::word *>(a.labg)[u] = LabG<P64>::pack(t, a.stamp);
      ++moved;
    } else {
      a.active[u] = 1;
    }
  }
  if (priv_k) {
    __syncthreads();
    for (uint32_t b = threadIdx.x; b < a.k; b += blockDim.x) {
      if (s_priv[b] != 0) {
        atomicAdd(&a.weight[b], s_priv[b]);
      }
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    moved += __shfl_xor_sync(kFull, moved, o);
  }
  if ((threadIdx.x & 31) == 0 && moved != 0) {
    atomicAdd(a.moved_count, moved);
  }
}

// ---- push activation (only in rounds with few movers, see kmp_lp.cu choose_activation) ---------
// A team of LANES threads (by the degree group of the sub-round) flags the neighbours of one accepted
// mover as active (label_propagation.h:848-870).
template <int LANES>
__device__ __forceinline__ void activate_neighbours(const CommitArgs &a, uint32_t cnt, uint32_t tid, uint32_t nth) {
  const uint32_t sub = tid % LANES;
  const uint32_t nteams = nth / LANES;
  for (uint32_t i = tid / LANES; i < cnt; i += nteams) {
    if (a.acc[i] != 1) {
      continue;
    }
    const uint32_t u = a.mv_u[i];
    const uint32_t end = a.xadj[u + 1];
    for (uint32_t e = a.xadj[u] + sub; e < end; e += LANES * 4) {
      uint32_t v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        v[j] = e + j * LANES < end ? a.adjncy[e + j * LANES] : kEmpty;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (v[j] != kEmpty) {
          a.active[v[j]] = 1;
        }
      }
    }
  }
}
template <int LANES> __global__ void __launch_bounds__(256) commit_activate(const CommitArgs a) {
  activate_neighbours<LANES>(a, *a.mover_count, blockIdx.x * blockDim.x + threadIdx.x, gridDim.x * blockDim.x);
}
__global__ void reset_u32(uint32_t *p) { *p = 0; }

} // namespace kmp
