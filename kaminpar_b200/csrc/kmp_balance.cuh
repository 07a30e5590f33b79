// kaminpar_b200: overload balancer on the device + its C ABI (include/kaminpar_b200_balancer.h).
// Included at the end of kmp_lp.cu (same translation unit: it balances the partition a kmp_lp_handle holds and
// commits through the refiner's cooperative ladder kernel, lp_commit.cuh commit_refine_fused). The round driver, the
// round tail and the select_all body here serve the underload balancer (kmp_underload.cuh) too.
//
// What it restates: OverloadBalancer::refine (refinement/balancer/overload_balancer.cc:51-326) as synchronous
// rounds (DESIGN.md §11). One round:
//   1. block stats against the frozen weights: over[b] = max(0, W[b] - max[b]), the total overload, the blocks
//      below their perfectly balanced weight (targets of internal vertices); the vertices of overloaded blocks
//      and those blocks are compacted in id order (one small read-back per round: total, counts)
//   2. candidate evaluation, degree-tiered (conn(u, .) over the blocks adjacent to u, exactly, for any k):
//      deg <= 8 one thread with the (block, weight) pairs in registers, deg <= 256 one warp with a 512-slot
//      shared hash table (never full: at most deg keys), above one CTA with a direct shared table over block-id
//      ranges of 8192 (ceil(k / 8192) passes over the adjacency)
//   3. per-block selection: stable radix sort by (block, key desc) of the candidates in id order, exclusive
//      weight scan per block, selected iff the weight before a candidate is < over[b]
//   4. proposals (border: the target; internal: a hashed draw among the underloaded blocks), then the ladder
//      commit of the LP refiner with one pass and no minimum weights, which applies the accepted moves
#pragma once

#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>

#include "../../include/kaminpar_b200_balancer.h"

namespace kmp {

enum : uint32_t { SALT_BAL_TIE = 5, SALT_BAL_DRAW = 6, SALT_BAL_COMMIT = 7, SALT_UBAL_TIE = 8, SALT_UBAL_COMMIT = 9 };
constexpr uint32_t kBalMaxRounds = KMP_BALANCE_MAX_ROUNDS;
constexpr uint32_t kBalThreadDeg = 8;    // deg <= 8: one thread per vertex
constexpr uint32_t kBalWarpDeg = 256;    // deg <= 256: one warp per vertex
constexpr uint32_t kBalWarpSlots = 512;  // > kBalWarpDeg: the warp's table never fills
constexpr int kBalWarpsPerCta = 8;
constexpr uint32_t kBalRange = 8192;     // deg > 256: direct table over block ids [r, r + kBalRange)
constexpr int kBalCtaThreads = 256;

// compute_relative_gain (refinement/balancer/relative_gain.h:14-16), rounded exactly as the host's float code
__host__ __device__ __forceinline__ float bal_relative_gain(int32_t gain, int32_t weight) {
#ifdef __CUDA_ARCH__
  const float g = __int2float_rn(gain), w = __int2float_rn(weight);
  return gain > 0 ? __fmul_rn(g, w) : __fdiv_rn(g, w);
#else
  return gain > 0 ? 1.0f * gain * weight : 1.0f * gain / weight;
#endif
}
// descending-key sort word: the float's order as an unsigned integer, complemented
__device__ __forceinline__ uint32_t bal_desc_bits(float f) {
  const uint32_t b = __float_as_uint(f);
  return ~(b ^ ((b >> 31) ? 0xFFFFFFFFu : 0x80000000u));
}
__host__ __device__ __forceinline__ uint32_t bal_draw(uint32_t base, uint32_t u) { return lowbias32((u * 0x9E3779B1u) ^ base); }

struct BalArgs {
  const uint32_t *__restrict__ xadj;
  const uint32_t *__restrict__ adjncy;
  const int32_t *__restrict__ vwgt;   // nullable
  const int32_t *__restrict__ adjwgt; // nullable
  const uint32_t *__restrict__ label;
  const int32_t *__restrict__ weight; // [k], frozen
  const int32_t *__restrict__ max_w;  // [k]
  const uint8_t *__restrict__ tmask;  // nullable: [k] the blocks a vertex may move to (underload balancer: W < min)
  uint32_t k;
  uint32_t base_tie;
  const uint32_t *__restrict__ cand;  // candidate i is vertex cand[i]
  uint32_t num_cand;
  uint32_t *__restrict__ warp_list;   // candidate indices of the warp / CTA tiers, filled by the thread tier
  uint32_t *__restrict__ cta_list;
  uint32_t *__restrict__ tier_count;  // [0] warp tier, [1] CTA tier
  unsigned long long *__restrict__ edges;
  // outputs per candidate index
  uint32_t *__restrict__ target;
  float *__restrict__ key;
  unsigned long long *__restrict__ sort_key; // nullable: (block << 32 | desc key bits)
  uint32_t *__restrict__ sort_val;           // candidate index
};

// best feasible target so far: (gain desc, tie_hash asc, block asc)
struct BalBest {
  int32_t gain;
  uint32_t hash, c;
};
__device__ __forceinline__ BalBest bal_none() { return BalBest{INT32_MIN, kEmpty, kEmpty}; }
__device__ __forceinline__ bool bal_better(const BalBest &a, const BalBest &b) {
  if (a.c == kEmpty) {
    return false;
  }
  if (b.c == kEmpty || a.gain != b.gain) {
    return b.c == kEmpty || a.gain > b.gain;
  }
  return a.hash != b.hash ? a.hash < b.hash : a.c < b.c;
}
__device__ __forceinline__ void bal_offer(const BalArgs &a, uint32_t u, uint32_t own, int32_t uw, int32_t conn_own,
                                          uint32_t c, int32_t conn, BalBest &best) {
  if (c == own || a.weight[c] + uw > a.max_w[c] || (a.tmask != nullptr && a.tmask[c] == 0)) {
    return;
  }
  const BalBest x{conn - conn_own, tie_hash(a.base_tie, u, c), c};
  if (bal_better(x, best)) {
    best = x;
  }
}
__device__ __forceinline__ BalBest bal_warp_best(BalBest b) {
  const bool have = __any_sync(kFull, b.c != kEmpty);
  if (!have) {
    return bal_none();
  }
  const int32_t g = __reduce_max_sync(kFull, b.c != kEmpty ? b.gain : INT32_MIN);
  bool in = b.c != kEmpty && b.gain == g;
  const uint32_t hmin = __reduce_min_sync(kFull, in ? b.hash : kEmpty);
  in = in && b.hash == hmin;
  const uint32_t cmin = __reduce_min_sync(kFull, in ? b.c : kEmpty);
  return BalBest{g, hmin, cmin};
}
__device__ __forceinline__ void bal_write(const BalArgs &a, uint32_t i, uint32_t own, int32_t uw, const BalBest &best) {
  const uint32_t t = best.c == kEmpty ? own : best.c;
  const float key = bal_relative_gain(best.c == kEmpty ? INT32_MIN : best.gain, uw);
  a.target[i] = t;
  a.key[i] = key;
  if (a.sort_key != nullptr) {
    a.sort_key[i] = (static_cast<unsigned long long>(own) << 32) | bal_desc_bits(key);
    a.sort_val[i] = i;
  }
}

// ---- tier 0: one thread per candidate (deg <= 8); hands higher degrees to the other tiers -------------------
__global__ void __launch_bounds__(256) bal_eval_thread(const BalArgs a) {
  unsigned long long edges = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.num_cand; i += gridDim.x * blockDim.x) {
    const uint32_t u = a.cand[i];
    const uint32_t beg = a.xadj[u], deg = a.xadj[u + 1] - beg;
    edges += deg;
    if (deg > kBalWarpDeg) {
      a.cta_list[atomicAdd(&a.tier_count[1], 1u)] = i;
      continue;
    }
    if (deg > kBalThreadDeg) {
      a.warp_list[atomicAdd(&a.tier_count[0], 1u)] = i;
      continue;
    }
    const uint32_t own = a.label[u];
    const int32_t uw = a.vwgt != nullptr ? a.vwgt[u] : 1;
    uint32_t c[kBalThreadDeg];
    int32_t w[kBalThreadDeg];
#pragma unroll
    for (uint32_t j = 0; j < kBalThreadDeg; ++j) {
      c[j] = j < deg ? a.label[a.adjncy[beg + j]] : kEmpty;
      w[j] = j < deg ? (a.adjwgt != nullptr ? a.adjwgt[beg + j] : 1) : 0;
    }
    int32_t conn_own = 0;
#pragma unroll
    for (uint32_t j = 0; j < kBalThreadDeg; ++j) {
      conn_own += c[j] == own ? w[j] : 0;
    }
    BalBest best = bal_none();
#pragma unroll
    for (uint32_t j = 0; j < kBalThreadDeg; ++j) {
      bool first = c[j] != kEmpty;
      int32_t conn = w[j];
#pragma unroll
      for (uint32_t q = 0; q < kBalThreadDeg; ++q) {
        if (q < j && c[q] == c[j]) {
          first = false;
        }
        if (q > j && c[q] == c[j]) {
          conn += w[q];
        }
      }
      if (first) {
        bal_offer(a, u, own, uw, conn_own, c[j], conn, best);
      }
    }
    bal_write(a, i, own, uw, best);
  }
  for (int o = 16; o > 0; o >>= 1) {
    edges += __shfl_xor_sync(kFull, edges, o);
  }
  if ((threadIdx.x & 31) == 0 && edges != 0) {
    atomicAdd(a.edges, edges);
  }
}

// ---- tier 1: one warp per candidate (8 < deg <= 256), open-addressing table in shared memory ---------------
__global__ void __launch_bounds__(kBalWarpsPerCta * 32) bal_eval_warp(const BalArgs a) {
  __shared__ uint32_t s_key[kBalWarpsPerCta][kBalWarpSlots];
  __shared__ int32_t s_val[kBalWarpsPerCta][kBalWarpSlots];
  const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  uint32_t *keys = s_key[wib];
  int32_t *vals = s_val[wib];
  const uint32_t cnt = a.tier_count[0];
  for (uint32_t e = blockIdx.x * kBalWarpsPerCta + wib; e < cnt; e += gridDim.x * kBalWarpsPerCta) {
    const uint32_t i = a.warp_list[e];
    const uint32_t u = a.cand[i];
    const uint32_t beg = a.xadj[u], end = a.xadj[u + 1];
    const uint32_t own = a.label[u];
    const int32_t uw = a.vwgt != nullptr ? a.vwgt[u] : 1;
    for (uint32_t s = lane; s < kBalWarpSlots; s += 32) {
      keys[s] = kEmpty;
      vals[s] = 0;
    }
    __syncwarp();
    for (uint32_t x = beg + lane; x < end; x += 32) {
      const uint32_t c = a.label[a.adjncy[x]];
      const int32_t w = a.adjwgt != nullptr ? a.adjwgt[x] : 1;
      uint32_t s = (c * 0x9E3779B1u) >> 23; // log2(kBalWarpSlots) = 9 bits
      while (true) {
        const uint32_t prev = atomicCAS(&keys[s], kEmpty, c);
        if (prev == kEmpty || prev == c) {
          atomicAdd(&vals[s], w);
          break;
        }
        s = (s + 1) & (kBalWarpSlots - 1);
      }
    }
    __syncwarp();
    int32_t own_part = 0;
    for (uint32_t s = lane; s < kBalWarpSlots; s += 32) {
      own_part += keys[s] == own ? vals[s] : 0;
    }
    const int32_t conn_own = __reduce_add_sync(kFull, own_part);
    BalBest best = bal_none();
    for (uint32_t s = lane; s < kBalWarpSlots; s += 32) {
      if (keys[s] != kEmpty) {
        bal_offer(a, u, own, uw, conn_own, keys[s], vals[s], best);
      }
    }
    best = bal_warp_best(best);
    if (lane == 0) {
      bal_write(a, i, own, uw, best);
    }
    __syncwarp();
  }
}

// ---- tier 2: one CTA per candidate (deg > 256), direct table over block-id ranges --------------------------
// The range holding the own block goes first, so conn(u, own) is known before any other block is offered.
__global__ void __launch_bounds__(kBalCtaThreads) bal_eval_cta(const BalArgs a) {
  __shared__ int32_t s_conn[kBalRange];
  __shared__ uint32_t s_seen[kBalRange / 32];
  __shared__ BalBest s_best[kBalCtaThreads / 32];
  __shared__ int32_t s_own;
  const uint32_t cnt = a.tier_count[1];
  const uint32_t ranges = (a.k + kBalRange - 1) / kBalRange;
  for (uint32_t e = blockIdx.x; e < cnt; e += gridDim.x) {
    const uint32_t i = a.cta_list[e];
    const uint32_t u = a.cand[i];
    const uint32_t beg = a.xadj[u], end = a.xadj[u + 1];
    const uint32_t own = a.label[u];
    const int32_t uw = a.vwgt != nullptr ? a.vwgt[u] : 1;
    BalBest best = bal_none(); // per thread, across the ranges
    for (uint32_t rr = 0; rr < ranges; ++rr) {
      const uint32_t lo = ((own / kBalRange + rr) % ranges) * kBalRange;
      const uint32_t len = min(kBalRange, a.k - lo);
      for (uint32_t s = threadIdx.x; s < len; s += blockDim.x) {
        s_conn[s] = 0;
      }
      for (uint32_t s = threadIdx.x; s < kBalRange / 32; s += blockDim.x) {
        s_seen[s] = 0;
      }
      __syncthreads();
      for (uint32_t x = beg + threadIdx.x; x < end; x += blockDim.x) {
        const uint32_t c = a.label[a.adjncy[x]];
        if (c - lo < len) {
          atomicAdd(&s_conn[c - lo], a.adjwgt != nullptr ? a.adjwgt[x] : 1);
          atomicOr(&s_seen[(c - lo) >> 5], 1u << ((c - lo) & 31));
        }
      }
      __syncthreads();
      if (rr == 0 && threadIdx.x == 0) {
        s_own = s_conn[own - lo];
      }
      __syncthreads();
      const int32_t conn_own = s_own;
      for (uint32_t s = threadIdx.x; s < len; s += blockDim.x) {
        if ((s_seen[s >> 5] >> (s & 31)) & 1u) {
          bal_offer(a, u, own, uw, conn_own, lo + s, s_conn[s], best);
        }
      }
      __syncthreads(); // the table is cleared for the next range
    }
    const BalBest wb = bal_warp_best(best);
    if ((threadIdx.x & 31) == 0) {
      s_best[threadIdx.x >> 5] = wb;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      BalBest b = s_best[0];
      for (int q = 1; q < kBalCtaThreads / 32; ++q) {
        if (bal_better(s_best[q], b)) {
          b = s_best[q];
        }
      }
      bal_write(a, i, own, uw, b);
    }
    __syncthreads();
  }
}

// ---- round set-up and selection ----------------------------------------------------------------------------
// over[b], the total overload (ctrl[0]) and the flags of the underloaded blocks (targets of internal vertices)
__global__ void bal_block_stats(uint32_t k, const int32_t *weight, const int32_t *max_w, const int32_t *pbw, int32_t *over,
                                uint8_t *under, unsigned long long *ctrl) {
  unsigned long long total = 0;
  for (uint32_t b = blockIdx.x * blockDim.x + threadIdx.x; b < k; b += gridDim.x * blockDim.x) {
    const int32_t o = max(0, weight[b] - max_w[b]);
    over[b] = o;
    under[b] = pbw != nullptr && weight[b] < pbw[b];
    total += static_cast<unsigned long long>(o);
  }
  for (int off = 16; off > 0; off >>= 1) {
    total += __shfl_xor_sync(kFull, total, off);
  }
  if ((threadIdx.x & 31) == 0 && total != 0) {
    atomicAdd(&ctrl[0], total);
  }
}
__global__ void bal_vertex_flags(uint32_t n, const uint32_t *label, const int32_t *over, uint8_t *flag) {
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += gridDim.x * blockDim.x) {
    flag[u] = over[label[u]] > 0;
  }
}
__global__ void bal_iota(uint32_t n, uint32_t *p) {
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += gridDim.x * blockDim.x) {
    p[u] = u;
  }
}
// sorted position p -> block and weight of the candidate there
__global__ void bal_sorted_weights(uint32_t nc, const unsigned long long *sort_key, const uint32_t *sort_val,
                                   const uint32_t *cand, const int32_t *vwgt, uint32_t *blk, int32_t *wt) {
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < nc; p += gridDim.x * blockDim.x) {
    blk[p] = static_cast<uint32_t>(sort_key[p] >> 32);
    wt[p] = vwgt != nullptr ? vwgt[cand[sort_val[p]]] : 1;
  }
}
// selected iff the weight of the candidates before it in its block is < over[b]; an internal vertex takes the first
// underloaded block (ctrl[2] of them, in under_list) with room for it, scanning cyclically from a hashed start
// (the reference retries random blocks of its list until one fits, overload_balancer.cc:290-316)
__global__ void bal_propose(uint32_t nc, const uint32_t *blk, const int32_t *prefix, const int32_t *over,
                            const uint32_t *sort_val, const uint32_t *cand, const uint32_t *target, const int32_t *vwgt,
                            const int32_t *weight, const int32_t *max_w, const uint32_t *under_list,
                            const unsigned long long *ctrl, uint32_t base_draw, uint32_t *mv_u, uint32_t *mv_t,
                            uint32_t *mover_count) {
  const uint32_t nu = static_cast<uint32_t>(ctrl[2]);
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < nc; p += gridDim.x * blockDim.x) {
    const uint32_t b = blk[p];
    if (prefix[p] >= over[b]) {
      continue;
    }
    const uint32_t i = sort_val[p];
    const uint32_t u = cand[i];
    uint32_t t = target[i];
    if (t == b && nu > 0) {
      const int32_t uw = vwgt != nullptr ? vwgt[u] : 1;
      const uint32_t start = bal_draw(base_draw, u) % nu;
      for (uint32_t q = 0; q < nu; ++q) {
        const uint32_t c = under_list[start + q < nu ? start + q : start + q - nu];
        if (weight[c] + uw <= max_w[c]) {
          t = c;
          break;
        }
      }
    }
    if (t != b) {
      const uint32_t slot = atomicAdd(mover_count, 1u);
      mv_u[slot] = u;
      mv_t[slot] = t;
    }
  }
}
// underload balancer: selected iff the weight of the candidates before it in its target's segment is < deficit[target]
__global__ void ubal_propose(uint32_t nt, const uint32_t *blk, const int32_t *prefix, const int32_t *deficit,
                             const uint32_t *sort_val, const uint32_t *cand, uint32_t *mv_u, uint32_t *mv_t,
                             uint32_t *mover_count) {
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < nt; p += gridDim.x * blockDim.x) {
    const uint32_t t = blk[p];
    if (prefix[p] < deficit[t]) {
      const uint32_t slot = atomicAdd(mover_count, 1u);
      mv_u[slot] = cand[sort_val[p]];
      mv_t[slot] = t;
    }
  }
}

// the underload balancer's kernels of select_all (kmp_underload.cuh)
__global__ void ubal_block_stats(uint32_t k, const int32_t *weight, const int32_t *min_w, int32_t *deficit,
                                 uint8_t *tmask, unsigned long long *ctrl);
__global__ void ubal_vertex_flags(uint32_t n, const uint32_t *label, const int32_t *vwgt, const int32_t *weight,
                                  const int32_t *min_w, const uint8_t *tmask, uint8_t *flag);
__global__ void ubal_keep_sources(uint32_t n, const uint8_t *flag, const uint32_t *label, const int32_t *vwgt,
                                  uint32_t *target, float *key);

} // namespace kmp

namespace {

using namespace kmp;

enum class BalKind { Overload, Underload };

int bal_refuse(kmp_lp_handle *h, BalKind kind) {
  const bool under = kind == BalKind::Underload;
  const char *what = under ? "the underload balancer" : "the overload balancer";
  const char *section = under ? "§12" : "§11";
  if (h == nullptr || !h->graph.present) {
    return fail(KMP_ERR_INVALID, "no graph set");
  }
  if (h->cfg.schedule == KMP_SCHEDULE_SEQ_STRICT) {
    return fail(KMP_ERR_UNSUPPORTED, std::string(what) + " has no seq_strict schedule (DESIGN.md " + section + ")");
  }
  return refuse_multi_gpu(h, what);
}

// Scratch of both balancers, grow-only in the handle (kmp_lp_free_scratch releases it).
int bal_ensure(kmp_lp_handle *h, uint32_t k, uint32_t nc) {
  const size_t n = std::max<uint32_t>(h->graph.n, 1), kk = std::max<uint32_t>(k, 1), c = std::max<uint32_t>(nc, 1);
  KMP_CUDA(h->bal.cand.ensure(n));
  KMP_CUDA(h->bal.flag.ensure(std::max(n, kk)));
  KMP_CUDA(h->bal.tmask.ensure(kk));
  KMP_CUDA(h->bal.over.ensure(kk));
  KMP_CUDA(h->bal.pbw.ensure(kk));
  KMP_CUDA(h->bal.under.ensure(kk));
  KMP_CUDA(h->bal.ctrl.ensure(8));
  KMP_CUDA(h->bal.ctr32.ensure(4 + kBalMaxRounds));
  KMP_CUDA(h->bal.target.ensure(c));
  KMP_CUDA(h->bal.key.ensure(c));
  KMP_CUDA(h->bal.lists.ensure(2 * c));
  KMP_CUDA(h->bal.sk_a.ensure(c));
  KMP_CUDA(h->bal.sk_b.ensure(c));
  KMP_CUDA(h->bal.sv_a.ensure(c));
  KMP_CUDA(h->bal.sv_b.ensure(c));
  KMP_CUDA(h->bal.blk.ensure(c));
  KMP_CUDA(h->bal.wt.ensure(c));
  KMP_CUDA(h->bal.prefix.ensure(c));
  return KMP_OK;
}

// Target and key of candidates cand[0 .. nc) against the frozen labels / weights on the device: three launches,
// the thread tier hands the higher degrees to the warp and CTA tiers. tmask (nullable, [k]): the allowed targets.
int bal_evaluate(kmp_lp_handle *h, uint32_t k, uint32_t nc, uint32_t base_tie, bool sort_keys,
                 const uint8_t *tmask = nullptr) {
  BalArgs a{};
  a.xadj = h->graph.xadj;
  a.adjncy = h->graph.adjncy;
  a.vwgt = h->graph.vwgt;
  a.adjwgt = h->graph.adjwgt;
  a.label = h->lp.label.p;
  a.weight = h->lp.weight.p;
  a.max_w = h->lp.maxw.p;
  a.tmask = tmask;
  a.k = k;
  a.base_tie = base_tie;
  a.cand = h->bal.cand.p;
  a.num_cand = nc;
  a.warp_list = h->bal.lists.p;
  a.cta_list = h->bal.lists.p + std::max<uint32_t>(nc, 1);
  a.tier_count = h->bal.ctr32.p + 2;
  a.edges = h->bal.ctrl.p + 4;
  a.target = h->bal.target.p;
  a.key = h->bal.key.p;
  a.sort_key = sort_keys ? h->bal.sk_a.p : nullptr;
  a.sort_val = h->bal.sv_a.p;
  KMP_CUDA(cudaMemsetAsync(h->bal.ctr32.p + 2, 0, 2 * sizeof(uint32_t), h->stream));
  bal_eval_thread<<<capped(h, grid_for(nc, 256)), 256, 0, h->stream>>>(a);
  bal_eval_warp<<<capped(h, grid_for(static_cast<uint64_t>(nc) * 32, kBalWarpsPerCta * 32)), kBalWarpsPerCta * 32, 0,
                  h->stream>>>(a);
  bal_eval_cta<<<capped(h, grid_for(static_cast<uint64_t>(nc) * kBalCtaThreads, kBalCtaThreads, kSMs * 8)), kBalCtaThreads,
                 0, h->stream>>>(a);
  h->counts.kernel_launches += 3;
  KMP_CUDA(cudaGetLastError());
  return KMP_OK;
}

// The end of a round of either balancer, after its selection left ns sort words (block << 32 | desc key bits) and
// candidate indices in bal.sk_a / bal.sv_a: sort them by (block, key desc), scan the weights per block, propose the
// candidates whose preceding weight in their block is below the block's quota bal.over[b], and commit the proposals
// with the refiner's ladder, one pass (moves land in bal.ctr32[4 + r]). The overload balancer commits without
// minimum weights: accepted moves never push a target above its maximum. The underload balancer commits with them:
// the target side keeps every block <= max, the source side keeps every source >= min (targets are underloaded and
// sources are not, so no block is both).
int bal_round_tail(kmp_lp_handle *h, BalKind kind, uint32_t k, uint32_t ns, uint32_t call, uint32_t r) {
  uint32_t end_bit = 32;
  while (end_bit < 64 && (static_cast<uint64_t>(k - 1) >> (end_bit - 32)) != 0) {
    ++end_bit;
  }
  cudaStream_t st = h->stream;
  KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
    return cub::DeviceRadixSort::SortPairs(tmp, bytes, h->bal.sk_a.p, h->bal.sk_b.p, h->bal.sv_a.p, h->bal.sv_b.p,
                                           static_cast<int>(ns), 0, static_cast<int>(end_bit), st);
  }));
  bal_sorted_weights<<<capped(h, grid_for(ns, 256)), 256, 0, st>>>(ns, h->bal.sk_b.p, h->bal.sv_b.p, h->bal.cand.p, h->graph.vwgt,
                                                                   h->bal.blk.p, h->bal.wt.p);
  KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
    return cub::DeviceScan::ExclusiveSumByKey(tmp, bytes, h->bal.blk.p, h->bal.wt.p, h->bal.prefix.p,
                                              static_cast<int>(ns), cub::Equality(), st);
  }));
  const bool under = kind == BalKind::Underload;
  uint32_t *mover_count = h->bal.ctr32.p;
  if (under) {
    ubal_propose<<<capped(h, grid_for(ns, 256)), 256, 0, st>>>(ns, h->bal.blk.p, h->bal.prefix.p, h->bal.over.p,
                                                               h->bal.sv_b.p, h->bal.cand.p, h->commit.mv_u.p, h->commit.mv_t.p,
                                                               mover_count);
  } else {
    bal_propose<<<capped(h, grid_for(ns, 256)), 256, 0, st>>>(ns, h->bal.blk.p, h->bal.prefix.p, h->bal.over.p,
                                                              h->bal.sv_b.p, h->bal.cand.p, h->bal.target.p, h->graph.vwgt,
                                                              h->lp.weight.p, h->lp.maxw.p, h->bal.under.p, h->bal.ctrl.p,
                                                              sync_base(h->cfg.seed, call, r, SALT_BAL_DRAW), h->commit.mv_u.p,
                                                              h->commit.mv_t.p, mover_count);
  }
  CommitArgs ca = make_commit_args(h, RunCtx{1, k, 0, under, false});
  ca.mover_count = mover_count;
  ca.next_mover_count = h->bal.ctr32.p + 1; // scratch: nothing reads it
  ca.also_zero = nullptr;
  ca.moved_count = h->bal.ctr32.p + 4 + r;
  ca.base_commit = sync_base(h->cfg.seed, call, r, under ? SALT_UBAL_COMMIT : SALT_BAL_COMMIT);
  ca.stamp = 0;
  const int rc = launch_commit_refine(h, ca, GatheredArgs{nullptr, 1, 0, nullptr}, 1, ns);
  if (rc != KMP_OK) {
    return rc;
  }
  h->counts.kernel_launches += 5;
  KMP_CUDA(cudaGetLastError());
  return KMP_OK;
}

// Round start: over[], underloaded blocks, candidates; read back {total overload, #candidates, #underloaded} and the
// number of proposals of the previous round.
int bal_round_begin(kmp_lp_handle *h, uint32_t k, unsigned long long *host_ctrl, uint32_t *host_proposals) {
  cudaStream_t st = h->stream;
  const uint32_t n = h->graph.n;
  KMP_CUDA(cudaMemsetAsync(h->bal.ctrl.p, 0, 3 * sizeof(unsigned long long), st));
  bal_block_stats<<<capped(h, grid_for(k, 256)), 256, 0, st>>>(k, h->lp.weight.p, h->lp.maxw.p, h->bal.pbw.p, h->bal.over.p,
                                                               h->bal.flag.p, h->bal.ctrl.p);
  KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
    return cub::DeviceSelect::Flagged(tmp, bytes, thrust::counting_iterator<uint32_t>(0), h->bal.flag.p, h->bal.under.p,
                                      h->bal.ctrl.p + 2, static_cast<int>(k), st);
  }));
  bal_vertex_flags<<<capped(h, grid_for(n, 256)), 256, 0, st>>>(n, h->lp.label.p, h->bal.over.p, h->bal.flag.p);
  KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
    return cub::DeviceSelect::Flagged(tmp, bytes, thrust::counting_iterator<uint32_t>(0), h->bal.flag.p, h->bal.cand.p,
                                      h->bal.ctrl.p + 1, static_cast<int>(n), st);
  }));
  h->counts.kernel_launches += 4;
  KMP_CUDA(cudaMemcpyAsync(host_ctrl, h->bal.ctrl.p, 4 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaMemcpyAsync(host_proposals, h->bal.ctr32.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaStreamSynchronize(st));
  return KMP_OK;
}

// the underload balancer's round steps (kmp_underload.cuh)
int ubal_round_begin(kmp_lp_handle *h, uint32_t k, unsigned long long *host_ctrl, uint32_t *host_proposals);
int ubal_select(kmp_lp_handle *h, uint32_t k, uint32_t nc, uint32_t call, uint32_t r, uint32_t *nt);

struct BalResult {
  uint32_t rounds = 0;
  uint32_t moved[kBalMaxRounds] = {};
  unsigned long long before = 0, after = 0; // total overload / underload
  unsigned long long candidates = 0, edges = 0;
  float device_ms = 0.f;
};

// One balancer call after its entry point's checks: load the partition (pbw: the overload balancer's perfectly
// balanced weights, min_w: the underload balancer's minimum weights), run rounds until the stop rule, download.
int bal_run(kmp_lp_handle *h, BalKind kind, uint32_t k, const int32_t *max_w, const int32_t *min_w, const int32_t *pbw,
            uint32_t *partition_inout, int32_t *block_weights_out, BalResult &res) {
  const uint32_t n = h->graph.n;
  KMP_CUDA(cudaSetDevice(h->device));
  h->counts.kernel_launches = 0;
  cudaStream_t st = h->stream;
  KMP_CUDA(cudaEventRecord(h->streams.ev_begin, st));
  int rc = ensure_scratch(h, 1, k); // the commit's ladder histograms (zeroed), counters, active flags
  if (rc == KMP_OK) {
    rc = prepare_labg(h, k); // the commit writes the packed labels (kmp_lp_refine repacks them on entry)
  }
  if (rc == KMP_OK) {
    rc = bal_ensure(h, k, 0);
  }
  if (rc == KMP_OK) {
    rc = load_partition(h, k, partition_inout, max_w, min_w);
  }
  if (rc != KMP_OK) {
    return rc;
  }
  if (pbw != nullptr) {
    KMP_CUDA(cudaMemcpyAsync(h->bal.pbw.p, pbw, static_cast<size_t>(k) * 4, cudaMemcpyHostToDevice, st));
  }
  KMP_CUDA(cudaMemsetAsync(h->bal.ctrl.p, 0, 8 * sizeof(unsigned long long), st));
  KMP_CUDA(cudaMemsetAsync(h->bal.ctr32.p, 0, (4 + kBalMaxRounds) * sizeof(uint32_t), st));
  rc = checked_block_weights(h, k, h->bal.ctrl.p + 3);
  if (rc != KMP_OK) {
    return rc;
  }
  const bool under = kind == BalKind::Underload;
  const uint32_t call = under ? h->ubal_calls++ : h->bal_calls++;
  unsigned long long ctrl[4] = {0, 0, 0, 0};
  uint32_t proposals = 0;
  for (;; ++res.rounds) {
    const uint32_t r = res.rounds;
    rc = under ? ubal_round_begin(h, k, ctrl, &proposals) : bal_round_begin(h, k, ctrl, &proposals);
    if (rc != KMP_OK) {
      return rc;
    }
    if (r == 0) {
      res.before = ctrl[0];
    }
    // stop: balanced, or the last round proposed no move (then no round would: without moves the next round selects
    // the same candidates with the same targets and quotas), or the cap. A round whose proposals the ladder
    // rejected is retried: its commit priorities, ties and draws are hashed with the round.
    if (ctrl[0] == 0 || (r > 0 && proposals == 0) || r == kBalMaxRounds) {
      break;
    }
    const uint32_t nc = static_cast<uint32_t>(ctrl[1]);
    res.candidates += nc;
    rc = bal_ensure(h, k, nc);
    if (rc == KMP_OK && h->commit.mv_u.cap < nc) {
      KMP_CUDA(h->commit.mv_u.ensure(nc));
      KMP_CUDA(h->commit.mv_t.ensure(nc));
      KMP_CUDA(h->commit.acc.ensure(nc));
    }
    if (rc != KMP_OK) {
      return rc;
    }
    KMP_CUDA(cudaMemsetAsync(h->bal.ctr32.p, 0, sizeof(uint32_t), st)); // this round's proposals
    uint32_t ns = nc; // sort words the selection left
    rc = under ? ubal_select(h, k, nc, call, r, &ns)
               : bal_evaluate(h, k, nc, sync_base(h->cfg.seed, call, r, SALT_BAL_TIE), true);
    // an underload round without a candidate that has a target ends here; an overload round always commits
    if (rc == KMP_OK && (ns > 0 || !under)) {
      rc = bal_round_tail(h, kind, k, ns, call, r);
    }
    if (rc != KMP_OK) {
      return rc;
    }
  }
  res.after = ctrl[0];
  if (partition_inout != nullptr && res.before != 0 && n > 0) {
    KMP_CUDA(cudaMemcpyAsync(partition_inout, h->lp.label.p, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost, st));
  }
  if (block_weights_out != nullptr) {
    KMP_CUDA(cudaMemcpyAsync(block_weights_out, h->lp.weight.p, static_cast<size_t>(k) * 4, cudaMemcpyDeviceToHost, st));
  }
  KMP_CUDA(cudaMemcpyAsync(res.moved, h->bal.ctr32.p + 4, sizeof(res.moved), cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaMemcpyAsync(&res.edges, h->bal.ctrl.p + 4, sizeof(res.edges), cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaEventRecord(h->streams.ev_end, st));
  KMP_CUDA(cudaStreamSynchronize(st));
  cudaEventElapsedTime(&res.device_ms, h->streams.ev_begin, h->streams.ev_end);
  return KMP_OK;
}

// Target and key of every vertex against host labels and block weights, for one (call, round) of either balancer's
// hash schedule (min_w: the underload balancer's minimum weights, required for it).
int bal_select_all(kmp_lp_handle *h, BalKind kind, uint32_t k, const uint32_t *labels, const int32_t *block_weights,
                   const int32_t *max_w, const int32_t *min_w, uint32_t call_index, uint32_t round, uint32_t *target_out,
                   float *key_out) {
  int rc = bal_refuse(h, kind);
  if (rc != KMP_OK) {
    return rc;
  }
  const bool under = kind == BalKind::Underload;
  if (k == 0 || labels == nullptr || block_weights == nullptr || max_w == nullptr || (under && min_w == nullptr) ||
      target_out == nullptr || key_out == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  const uint32_t n = h->graph.n;
  for (uint32_t u = 0; u < n; ++u) {
    if (labels[u] >= k) {
      return fail(KMP_ERR_INVALID, "labels >= k: not a k-way partition");
    }
  }
  KMP_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = h->stream;
  rc = bal_ensure(h, k, n);
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(h->lp.label.ensure(n));
  KMP_CUDA(h->lp.weight.ensure(k));
  KMP_CUDA(h->lp.maxw.ensure(k));
  if (n > 0) {
    KMP_CUDA(cudaMemcpyAsync(h->lp.label.p, labels, static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, st));
  }
  KMP_CUDA(cudaMemcpyAsync(h->lp.weight.p, block_weights, static_cast<size_t>(k) * 4, cudaMemcpyHostToDevice, st));
  KMP_CUDA(cudaMemcpyAsync(h->lp.maxw.p, max_w, static_cast<size_t>(k) * 4, cudaMemcpyHostToDevice, st));
  KMP_CUDA(cudaMemsetAsync(h->bal.ctrl.p, 0, 8 * sizeof(unsigned long long), st));
  if (under) { // the target mask
    KMP_CUDA(h->lp.minw.ensure(k));
    KMP_CUDA(cudaMemcpyAsync(h->lp.minw.p, min_w, static_cast<size_t>(k) * 4, cudaMemcpyHostToDevice, st));
    ubal_block_stats<<<capped(h, grid_for(k, 256)), 256, 0, st>>>(k, h->lp.weight.p, h->lp.minw.p, h->bal.over.p,
                                                                  h->bal.tmask.p, h->bal.ctrl.p);
  }
  if (n > 0) {
    bal_iota<<<capped(h, grid_for(n, 256)), 256, 0, st>>>(n, h->bal.cand.p);
    rc = bal_evaluate(h, k, n, sync_base(h->cfg.seed, call_index, round, under ? SALT_UBAL_TIE : SALT_BAL_TIE), false,
                      under ? h->bal.tmask.p : nullptr);
    if (rc != KMP_OK) {
      return rc;
    }
    if (under) { // a vertex that may not leave its block keeps it
      ubal_vertex_flags<<<capped(h, grid_for(n, 256)), 256, 0, st>>>(n, h->lp.label.p, h->graph.vwgt, h->lp.weight.p, h->lp.minw.p,
                                                                     h->bal.tmask.p, h->bal.flag.p);
      ubal_keep_sources<<<capped(h, grid_for(n, 256)), 256, 0, st>>>(n, h->bal.flag.p, h->lp.label.p, h->graph.vwgt,
                                                                     h->bal.target.p, h->bal.key.p);
      KMP_CUDA(cudaGetLastError());
    }
    KMP_CUDA(cudaMemcpyAsync(target_out, h->bal.target.p, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost, st));
    KMP_CUDA(cudaMemcpyAsync(key_out, h->bal.key.p, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost, st));
  }
  KMP_CUDA(cudaStreamSynchronize(st));
  return KMP_OK;
}

} // namespace

extern "C" {

int kmp_overload_balance(kmp_lp_handle *h, uint32_t k, const int32_t *max_block_weights,
                         const int32_t *perfectly_balanced_block_weights, uint32_t *partition_inout,
                         int32_t *block_weights_out, int *improved_out, kmp_balance_stats *stats) {
  int rc = bal_refuse(h, BalKind::Overload);
  if (rc != KMP_OK) {
    return rc;
  }
  if (k == 0 || max_block_weights == nullptr || perfectly_balanced_block_weights == nullptr) {
    return fail(KMP_ERR_INVALID, "k / max_block_weights / perfectly_balanced_block_weights missing");
  }
  if (partition_inout == nullptr && (rc = refuse_without_labels(h)) != KMP_OK) {
    return rc;
  }
  if (stats != nullptr) {
    std::memset(stats, 0, sizeof(*stats));
  }
  BalResult res;
  rc = bal_run(h, BalKind::Overload, k, max_block_weights, nullptr, perfectly_balanced_block_weights, partition_inout,
               block_weights_out, res);
  if (rc != KMP_OK) {
    return rc;
  }
  if (improved_out != nullptr) {
    *improved_out = res.before != 0 ? 1 : 0;
  }
  if (stats != nullptr) {
    stats->rounds = res.rounds;
    std::memcpy(stats->moved, res.moved, sizeof(res.moved));
    stats->overload_before = static_cast<int64_t>(res.before);
    stats->overload_after = static_cast<int64_t>(res.after);
    stats->candidates = res.candidates;
    stats->edges_scanned = res.edges;
    stats->kernel_launches = h->counts.kernel_launches;
    stats->device_ms = res.device_ms;
  }
  return KMP_OK;
}

int kmp_balance_select_all(kmp_lp_handle *h, uint32_t k, const uint32_t *labels, const int32_t *block_weights,
                           const int32_t *max_block_weights, uint32_t call_index, uint32_t round, uint32_t *target_out,
                           float *key_out) {
  return bal_select_all(h, BalKind::Overload, k, labels, block_weights, max_block_weights, nullptr, call_index, round,
                        target_out, key_out);
}

} // extern "C"
