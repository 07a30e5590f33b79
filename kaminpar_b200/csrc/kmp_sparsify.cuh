// kaminpar_b200: threshold edge sparsification of a contracted graph on the device + its C ABI
// (include/kaminpar_b200_contraction.h). Included at the end of kmp_lp.cu after kmp_contract.cuh: it rewrites a
// kmp_coarse_graph in place on the stream of the handle that contracted it, and finds the source vertex of an edge
// with the contraction's tile owners (k_tile_owners, owner_of_edge).
//
// What it restates (DESIGN.md §13): SparsificationClusterCoarsener::recontract_with_threshold_sparsification
// (coarsening/sparsification_cluster_coarsener.cc:158-228) with quickselect_k_smallest
// (kaminpar-common/parallel/quickselect.h) and sparsification_target (:41-48).
//   1. radix select of the k-th smallest edge weight, k = c_m - target + 1, over the order-preserving key
//      w ^ 0x80000000 in three histogram passes of 11 / 11 / 10 bits (shared-memory bins, warp-aggregated
//      increments). After each pass one CTA finds the bin that holds rank k and narrows the prefix on the device;
//      the last pass yields T and the exact counts smaller / equal. One read-back: the host computes p in double
//      as the reference does. The only other read-back (kept counts) rides on the call's final synchronisation.
//   2. keep flags, one thread per edge: w > T, or w == T and dice(u, v) < p (IEEE double, no FMA)
//   3. exclusive scan of the flags in place -> the new position of every kept edge; new xadj[c] = pos[xadj[c]]
//      (the kept edges before vertex c, i.e. the scan of the per-vertex kept counts); an order-preserving
//      scatter writes adjncy / adjwgt, so every adjacency list stays sorted by target (the canonical form of §9).
#pragma once

namespace kmp {

constexpr uint32_t kSpHistWords = 2048 + 2048 + 1024; // the bins of the three passes, side by side
constexpr uint32_t kSpState = kSpHistWords;            // SpSelect, then the equal_kept counter
constexpr uint32_t kSpEqualKept = kSpState + 4;
constexpr uint32_t kSpCtlWords = kSpEqualKept + 1;

// the radix select's state between passes: the key prefix fixed so far, the rank of the wanted key among the keys
// with that prefix (1-based), the keys below the prefix, and (after a pass) the keys in the chosen bin
struct SpSelect {
  uint32_t prefix, k, smaller, equal;
};

template <int PASS> struct SpPass {
  static constexpr int kBits = PASS == 2 ? 10 : 11;
  static constexpr int kShift = PASS == 0 ? 21 : PASS == 1 ? 10 : 0; // lowest key bit of this pass's digit
  static constexpr uint32_t kBins = 1u << kBits;
  static constexpr uint32_t kOffset = PASS == 0 ? 0 : PASS == 1 ? 2048 : 4096; // into the control words
};

// histogram of this pass's digit over the keys whose higher digits equal the prefix chosen so far
template <int PASS>
__global__ void __launch_bounds__(256) sp_radix_hist(uint32_t m, const int32_t *__restrict__ w, const uint32_t *ctl,
                                                     uint32_t *hist) {
  using P = SpPass<PASS>;
  __shared__ uint32_t s_hist[P::kBins];
  for (uint32_t i = threadIdx.x; i < P::kBins; i += blockDim.x) {
    s_hist[i] = 0;
  }
  __syncthreads();
  const uint32_t prefix = PASS == 0 ? 0u : reinterpret_cast<const SpSelect *>(ctl + kSpState)->prefix;
  // every thread of a CTA runs the same trip count: the warp-wide ballot / match below see whole warps
  for (uint64_t base = static_cast<uint64_t>(blockIdx.x) * blockDim.x; base < m;
       base += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    const uint64_t e = base + threadIdx.x;
    uint32_t key = 0;
    bool in = false;
    if (e < m) {
      key = static_cast<uint32_t>(w[e]) ^ 0x80000000u;
      if constexpr (PASS == 0) {
        in = true;
      } else {
        in = (key >> (P::kShift + P::kBits)) == prefix;
      }
    }
    const unsigned active = __ballot_sync(kFull, in);
    if (in) {
      const uint32_t bin = (key >> P::kShift) & (P::kBins - 1);
      const unsigned peers = __match_any_sync(active, bin);
      if ((threadIdx.x & 31) == static_cast<unsigned>(__ffs(peers) - 1)) {
        atomicAdd(&s_hist[bin], static_cast<uint32_t>(__popc(peers)));
      }
    }
  }
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < P::kBins; i += blockDim.x) {
    if (s_hist[i] != 0) {
      atomicAdd(&hist[i], s_hist[i]);
    }
  }
}

// one CTA: the bin that holds rank k; narrows the prefix and the rank for the next pass. k0: the rank of pass 0.
template <int PASS> __global__ void __launch_bounds__(1024) sp_radix_pick(const uint32_t *hist, uint32_t *ctl, uint32_t k0) {
  using P = SpPass<PASS>;
  constexpr uint32_t kPer = P::kBins / 1024;
  using BlockScan = cub::BlockScan<uint32_t, 1024>;
  __shared__ typename BlockScan::TempStorage scan_tmp;
  SpSelect *s = reinterpret_cast<SpSelect *>(ctl + kSpState);
  const uint32_t k = PASS == 0 ? k0 : s->k;
  const uint32_t prefix = PASS == 0 ? 0u : s->prefix;
  const uint32_t smaller = PASS == 0 ? 0u : s->smaller;
  uint32_t c[kPer];
  uint32_t sum = 0;
#pragma unroll
  for (uint32_t j = 0; j < kPer; ++j) {
    c[j] = hist[threadIdx.x * kPer + j];
    sum += c[j];
  }
  uint32_t before = 0;
  BlockScan(scan_tmp).ExclusiveSum(sum, before); // its barriers order every read of *s before the write below
  if (before < k && k <= before + sum) {         // exactly one thread
#pragma unroll
    for (uint32_t j = 0; j < kPer; ++j) {
      if (k <= before + c[j]) {
        s->prefix = (prefix << P::kBits) | (threadIdx.x * kPer + j);
        s->k = k - before;
        s->smaller = smaller + before;
        s->equal = c[j];
        break;
      }
      before += c[j];
    }
  }
}

// dice(u, v) < p (sparsification_cluster_coarsener.cc:201-214): murmur3's fmix64 of the ordered pair plus the seed,
// low 32 bits scaled to [0, 1] by a correctly rounded double division
__device__ __forceinline__ bool sp_dice_below(uint32_t u, uint32_t v, unsigned long long seed, double p) {
  unsigned long long x = ((static_cast<unsigned long long>(max(u, v)) << 32) | min(u, v)) + seed;
  x ^= x >> 33;
  x *= 0xff51afd7ed558ccdull;
  x ^= x >> 33;
  x *= 0xc4ceb9fe1a85ec53ull;
  x ^= x >> 33;
  return __ddiv_rn(static_cast<double>(static_cast<uint32_t>(x)), 4294967295.0) < p;
}

// flag[e] = keep(e); tiles of kTileEdges edges, grid-stride over the tiles. The source vertex is searched only for
// edges at the threshold weight, in the tile's slice of xadj staged in shared memory as in k_contract_edge_keys.
__global__ void __launch_bounds__(256) sp_keep_flags(uint32_t m, const uint32_t *__restrict__ xadj,
                                                     const uint32_t *__restrict__ tile_lo, uint32_t tiles,
                                                     const uint32_t *__restrict__ adjncy,
                                                     const int32_t *__restrict__ adjwgt, int32_t threshold, double p,
                                                     unsigned long long seed, uint32_t *__restrict__ flag,
                                                     uint32_t *equal_kept) {
  __shared__ uint32_t s_x[kTileVerts + 1];
  uint32_t kept_equal = 0;
  for (uint32_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    const uint32_t e0 = t * kTileEdges;
    const uint32_t e1 = e0 + kTileEdges < m ? e0 + kTileEdges : m;
    const uint32_t u_lo = tile_lo[t], u_hi = tile_lo[t + 1];
    const bool staged = u_hi - u_lo + 1 <= kTileVerts;
    __syncthreads(); // the previous tile's searches are done
    if (staged) {
      for (uint32_t i = threadIdx.x; i <= u_hi - u_lo; i += blockDim.x) {
        s_x[i] = xadj[u_lo + i];
      }
    }
    __syncthreads();
#pragma unroll 4
    for (int j = 0; j < kTileEdges / 256; ++j) {
      const uint32_t e = e0 + j * 256 + threadIdx.x;
      if (e < e1) {
        const int32_t w = adjwgt[e];
        bool keep = w > threshold;
        if (w == threshold) {
          const uint32_t u = staged ? u_lo + owner_of_edge(s_x, 0, u_hi - u_lo, e) : owner_of_edge(xadj, u_lo, u_hi, e);
          keep = sp_dice_below(u, adjncy[e], seed, p);
          kept_equal += keep;
        }
        flag[e] = keep;
      }
    }
  }
  for (int off = 16; off > 0; off >>= 1) {
    kept_equal += __shfl_xor_sync(kFull, kept_equal, off);
  }
  if ((threadIdx.x & 31) == 0 && kept_equal != 0) {
    atomicAdd(equal_kept, kept_equal);
  }
}

// new xadj[c] = kept edges before the first edge of c
__global__ void sp_offsets(uint32_t c_n, const uint32_t *xadj, const uint32_t *pos, uint32_t *out_xadj) {
  for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c <= c_n; c += gridDim.x * blockDim.x) {
    out_xadj[c] = pos[xadj[c]];
  }
}
// order-preserving compaction: edge e is kept iff the exclusive scan of the flags steps after it
__global__ void sp_scatter(uint32_t m, const uint32_t *__restrict__ pos, const uint32_t *__restrict__ adjncy,
                           const int32_t *__restrict__ adjwgt, uint32_t *__restrict__ out_adjncy,
                           int32_t *__restrict__ out_adjwgt) {
  for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < m; e += gridDim.x * blockDim.x) {
    const uint32_t o = pos[e];
    if (pos[e + 1] != o) {
      out_adjncy[o] = adjncy[e];
      out_adjwgt[o] = adjwgt[e];
    }
  }
}

} // namespace kmp

namespace {

// The new arrays go to `out` (they free themselves if this fails); g is not modified here.
int sparsify_impl(kmp_lp_handle *h, const kmp_coarse_graph *g, uint32_t target_m, uint64_t seed, kmp_coarse_graph *out,
                  kmp_sparsify_stats *stats) {
  using namespace kmp;
  const uint32_t c_n = g->c_n, m = g->c_m;
  cudaStream_t st = h->stream;
  uint32_t launches = 0;
  KMP_CUDA(call_clock_start(h, st));
  KMP_CUDA(out->xadj.alloc(static_cast<size_t>(c_n) + 1, st, h->device));
  int32_t threshold = 0;
  uint32_t smaller = 0, equal = 0, kept = 0, equal_kept = 0;
  uint32_t counts[2] = {0, 0}; // kept edges, kept edges at T: read with the final synchronisation
  if (target_m < 2) { // sparsification_cluster_coarsener.cc:166-175: no edge survives, no seed is drawn
    KMP_CUDA(cudaMemsetAsync(out->xadj.p, 0, (static_cast<size_t>(c_n) + 1) * 4, st));
    KMP_CUDA(out->adjncy.alloc(1, st, h->device));
    KMP_CUDA(out->adjwgt.alloc(1, st, h->device));
  } else {
    // ---- 1. radix select of the k-th smallest weight (quickselect_k_smallest(c_m - target_m + 1, ...)) ----------
    const uint32_t k = m - target_m + 1;
    DevBuf<uint32_t> &ctl = h->ops.sp_ctl;
    KMP_CUDA(ctl.ensure(kSpCtlWords));
    KMP_CUDA(cudaMemsetAsync(ctl.p, 0, kSpCtlWords * 4, st));
    const int32_t *w = g->adjwgt.p;
    const uint32_t hist_grid = capped(h, grid_for(m, 256, kSMs * 4));
    sp_radix_hist<0><<<hist_grid, 256, 0, st>>>(m, w, ctl.p, ctl.p + SpPass<0>::kOffset);
    sp_radix_pick<0><<<1, 1024, 0, st>>>(ctl.p + SpPass<0>::kOffset, ctl.p, k);
    sp_radix_hist<1><<<hist_grid, 256, 0, st>>>(m, w, ctl.p, ctl.p + SpPass<1>::kOffset);
    sp_radix_pick<1><<<1, 1024, 0, st>>>(ctl.p + SpPass<1>::kOffset, ctl.p, 0);
    sp_radix_hist<2><<<hist_grid, 256, 0, st>>>(m, w, ctl.p, ctl.p + SpPass<2>::kOffset);
    sp_radix_pick<2><<<1, 1024, 0, st>>>(ctl.p + SpPass<2>::kOffset, ctl.p, 0);
    launches += 6;
    KMP_CUDA(cudaGetLastError());
    SpSelect sel{};
    KMP_CUDA(cudaMemcpyAsync(&sel, ctl.p + kSpState, sizeof(sel), cudaMemcpyDeviceToHost, st));
    KMP_CUDA(cudaStreamSynchronize(st));
    threshold = static_cast<int32_t>(sel.prefix ^ 0x80000000u);
    smaller = sel.smaller;
    equal = sel.equal;
    const uint32_t larger = m - smaller - equal;
    if (equal == 0 || larger > target_m) {
      return fail(KMP_ERR_CUDA, "radix select returned an inconsistent threshold");
    }
    // :191-193, in double as there
    const double p = 1.0 * static_cast<double>(target_m - larger) / static_cast<double>(equal);
    // ---- 2. keep flags -----------------------------------------------------------------------------------------
    const uint32_t tiles = (m + kTileEdges - 1) / kTileEdges;
    DevBuf<uint32_t> &tile_lo = h->ops.ct_flags, &pos = h->ops.ct_rank;
    KMP_CUDA(tile_lo.ensure(static_cast<size_t>(tiles) + 1));
    KMP_CUDA(pos.ensure(static_cast<size_t>(m) + 1));
    KMP_CUDA(cudaMemsetAsync(pos.p + m, 0, 4, st));
    k_tile_owners<<<capped(h, grid_for(static_cast<uint64_t>(tiles) + 1, 256)), 256, 0, st>>>(c_n, m, g->xadj.p, tiles,
                                                                                              tile_lo.p);
    sp_keep_flags<<<capped(h, std::min<uint32_t>(tiles, kSMs * 8)), 256, 0, st>>>(
        m, g->xadj.p, tile_lo.p, tiles, g->adjncy.p, w, threshold, p, static_cast<unsigned long long>(seed), pos.p,
        ctl.p + kSpEqualKept);
    launches += 2;
    KMP_CUDA(cudaGetLastError());
    // ---- 3. compaction -----------------------------------------------------------------------------------------
    // The new arrays are sized by the bound larger + equal = c_m - smaller on the kept edges, known since the
    // selection's read-back, so that the kept count is read only with the call's final synchronisation.
    KMP_CUDA(out->adjncy.alloc(m - smaller, st, h->device));
    KMP_CUDA(out->adjwgt.alloc(m - smaller, st, h->device));
    KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
      return cub::DeviceScan::ExclusiveSum(tmp, bytes, pos.p, m + 1, st);
    }));
    sp_offsets<<<capped(h, grid_for(static_cast<uint64_t>(c_n) + 1, 256)), 256, 0, st>>>(c_n, g->xadj.p, pos.p,
                                                                                         out->xadj.p);
    sp_scatter<<<capped(h, grid_for(m, 256)), 256, 0, st>>>(m, pos.p, g->adjncy.p, w, out->adjncy.p, out->adjwgt.p);
    launches += 3; // + the scan inside CUB
    KMP_CUDA(cudaGetLastError());
  }
  KMP_CUDA(call_clock_stop(h, st));
  if (target_m >= 2) {
    KMP_CUDA(cudaMemcpyAsync(&counts[0], h->ops.ct_rank.p + m, 4, cudaMemcpyDeviceToHost, st));
    KMP_CUDA(cudaMemcpyAsync(&counts[1], h->ops.sp_ctl.p + kSpEqualKept, 4, cudaMemcpyDeviceToHost, st));
  }
  KMP_CUDA(cudaStreamSynchronize(st));
  kept = counts[0];
  equal_kept = counts[1];
  const float ms = call_clock_ms(h);
  out->c_m = kept;
  if (stats != nullptr) {
    stats->c_m_before = m;
    stats->c_m_after = kept;
    stats->target_m = target_m;
    stats->threshold = threshold;
    stats->smaller = smaller;
    stats->equal = equal;
    stats->equal_kept = equal_kept;
    stats->kernel_launches = launches;
    stats->device_ms = ms;
  }
  return KMP_OK;
}

} // namespace

extern "C" {

uint32_t kmp_sparsification_target(uint32_t prev_m, uint32_t prev_n, uint32_t c_n, double density_target_factor,
                                   double edge_target_factor) {
  // sparsification_cluster_coarsener.cc:41-48, operand for operand
  const double target = std::min(edge_target_factor * prev_m, density_target_factor * prev_m / prev_n * c_n);
  return target < prev_m ? static_cast<uint32_t>(target) : prev_m;
}

int kmp_coarse_sparsify(kmp_lp_handle *h, kmp_coarse_graph *g, uint32_t target_m, uint64_t seed,
                        kmp_sparsify_stats *stats) {
  if (h == nullptr || g == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  if (g->device != h->device) {
    return fail(KMP_ERR_INVALID, "the coarse graph lives on another device than the handle");
  }
  if (target_m > g->c_m) {
    return fail(KMP_ERR_INVALID, "target_m exceeds the coarse graph's edge count");
  }
  KMP_CUDA(cudaSetDevice(h->device));
  if (stats != nullptr) {
    std::memset(stats, 0, sizeof(*stats));
  }
  kmp_coarse_graph out;
  const int rc = sparsify_impl(h, g, target_m, seed, &out, stats);
  if (rc != KMP_OK) {
    return rc;
  }
  // the stream is idle (sparsify_impl synchronised it): the old arrays are unused when they are freed
  g->xadj = std::move(out.xadj);
  g->adjncy = std::move(out.adjncy);
  g->adjwgt = std::move(out.adjwgt);
  g->c_m = out.c_m;
  return KMP_OK;
}

} // extern "C"
