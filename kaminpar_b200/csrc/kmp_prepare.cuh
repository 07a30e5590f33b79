// kaminpar_b200: input preparation on the device + its C ABI (include/kaminpar_b200_prepare.h, DESIGN.md §15).
// Included at the end of kmp_lp.cu after kmp_contract.cuh: the edge copy finds the vertex that owns a new-edge
// position with the contraction's tile owners (k_tile_owners, owner_of_edge), and the finish counts block weights
// and labels >= k with the refiner's bal_block_weights.
//
// What it restates (see the header): graph::rearrange_by_degree_buckets (graphutils/permutator.h:28-209), the
// isolated-vertex cut (csr_graph.cc:150-174) and graph::assign_isolated_nodes (permutator.cc:236-264).
//   1. vertex tiles of kPrepTileVerts: validate xadj, bucket every vertex, a per-tile 33-bucket histogram
//      (bucket-major: hist[b * tiles + t]); an exclusive scan gives each (bucket, tile) its first new id, and the
//      start of bucket 32 is n'. One host wait: the validation flag and n'.
//   2. the stable scatter over the same tiles: a vertex's rank within its tile is the count of its bucket in the
//      earlier rounds of the tile, in the earlier warps of its round and in the lower lanes of its warp
//      (__match_any_sync + popc) -- no atomics, so the order is the old id order. Writes old_to_new, new_to_old,
//      the new degrees and vwgt; a scan of the degrees gives new_xadj.
//   3. the edge copy (the hot path, 12 B per edge + 8 B with edge weights): CTAs over tiles of kTileEdges new-edge
//      positions; a thread finds the new vertex u owning position p, reads e = xadj[old_u] + (new_xadj[u+1] - 1 - p)
//      (the reversed list) and writes new_adjncy[p] = old_to_new[adjncy[e]] coalesced. A target >= n is flagged,
//      never used as an index. A hub spreads over as many tiles as it needs.
//   4. finish: block weights of the n' part (bal_block_weights), a 64-bit inclusive scan S of the isolated weights,
//      the next-fit chain as k dependent warp-wide searches (block b takes the isolated vertices [s_b, e_b) with
//      e_b the first i >= s_b where bw[b] + S[i+1] - S[s_b] > max(b); weights >= 0 keep S monotone) and a map-back
//      pass over the original ids.
#pragma once

namespace {

constexpr uint32_t kPrepTileVerts = 4096; // vertices per CTA of passes 1 and 2 (256 threads x 16 rounds)
constexpr uint32_t kPrepBuckets = 33;     // kNumberOfDegreeBuckets<uint32_t> (degree_buckets.h:17)
constexpr uint32_t kPrepIsolated = 32;    // the bucket of a degree-0 vertex

__device__ __forceinline__ uint32_t prep_bucket(uint32_t d) { // degree_buckets.h:24-26, permutator.h:105-107
  return d == 0 ? kPrepIsolated : 32u - __clz(d);
}

// bad[0]: xadj checks (xadj[0] != 0, decreasing, xadj[n] != m); bad[1]: targets >= n
__global__ void __launch_bounds__(256) k_prep_count(uint32_t n, uint32_t m, const uint32_t *__restrict__ xadj,
                                                    uint32_t tiles, uint32_t *__restrict__ hist,
                                                    uint32_t *__restrict__ bad) {
  __shared__ uint32_t s_hist[kPrepBuckets];
  for (uint32_t i = threadIdx.x; i < kPrepBuckets; i += blockDim.x) {
    s_hist[i] = 0;
  }
  __syncthreads();
  const uint32_t t0 = blockIdx.x * kPrepTileVerts;
  bool ok = true;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    ok = xadj[0] == 0 && (n != 0 || m == 0);
  }
  for (uint32_t r = 0; r < kPrepTileVerts / 256; ++r) {
    const uint32_t u = t0 + r * 256 + threadIdx.x;
    if (u < n) {
      const uint32_t x0 = xadj[u], x1 = xadj[u + 1];
      ok = ok && x1 >= x0 && (u + 1 != n || x1 == m);
      atomicAdd(&s_hist[prep_bucket(x1 - x0)], 1u);
    }
  }
  if (!ok) {
    bad[0] = 1;
  }
  __syncthreads();
  for (uint32_t b = threadIdx.x; b < kPrepBuckets; b += blockDim.x) {
    hist[b * tiles + blockIdx.x] = s_hist[b];
  }
}

// base[b * tiles + t]: the first new id of bucket b's vertices in tile t
__global__ void __launch_bounds__(256) k_prep_scatter(uint32_t n, const uint32_t *__restrict__ xadj,
                                                      const int32_t *__restrict__ vwgt, uint32_t tiles,
                                                      const uint32_t *__restrict__ base, uint32_t *__restrict__ old_to_new,
                                                      uint32_t *__restrict__ new_to_old, uint32_t *__restrict__ new_deg,
                                                      int32_t *__restrict__ new_vwgt) {
  constexpr uint32_t kWarps = 8;
  __shared__ uint32_t s_base[kPrepBuckets];
  __shared__ uint32_t s_run[kPrepBuckets];           // vertices of each bucket in the tile's earlier rounds
  __shared__ uint32_t s_warp[kWarps][kPrepBuckets];  // this round: vertices of each bucket per warp
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (uint32_t b = threadIdx.x; b < kPrepBuckets; b += blockDim.x) {
    s_base[b] = base[b * tiles + blockIdx.x];
    s_run[b] = 0;
  }
  for (uint32_t i = threadIdx.x; i < kWarps * kPrepBuckets; i += blockDim.x) {
    (&s_warp[0][0])[i] = 0;
  }
  __syncthreads();
  const uint32_t t0 = blockIdx.x * kPrepTileVerts;
  for (uint32_t r = 0; r < kPrepTileVerts / 256 && t0 + r * 256 < n; ++r) { // CTA-uniform bound
    const uint32_t u = t0 + r * 256 + threadIdx.x;
    const bool live = u < n;
    const uint32_t d = live ? xadj[u + 1] - xadj[u] : 0u;
    const uint32_t b = live ? prep_bucket(d) : kPrepBuckets; // past-the-end vertices form a class of their own
    const unsigned peers = __match_any_sync(kFull, b);
    if (live && lane == static_cast<uint32_t>(__ffs(peers) - 1)) {
      s_warp[warp][b] = __popc(peers);
    }
    __syncthreads();
    if (live) {
      uint32_t id = s_base[b] + s_run[b] + __popc(peers & ((1u << lane) - 1u));
      for (uint32_t w = 0; w < warp; ++w) {
        id += s_warp[w][b];
      }
      old_to_new[u] = id;
      new_to_old[id] = u;
      new_deg[id] = d;
      if (vwgt != nullptr) {
        new_vwgt[id] = vwgt[u];
      }
    }
    __syncthreads();
    if (threadIdx.x < kPrepBuckets) {
      uint32_t add = 0;
      for (uint32_t w = 0; w < kWarps; ++w) {
        add += s_warp[w][threadIdx.x];
        s_warp[w][threadIdx.x] = 0;
      }
      s_run[threadIdx.x] += add;
    }
    __syncthreads();
  }
}

// new_adjncy[p] = old_to_new[adjncy[e]], e = xadj[old_u] + (new_xadj[u + 1] - 1 - p) for the new vertex u owning p
template <bool EW>
__global__ void __launch_bounds__(256) k_prep_edges(uint32_t n, uint32_t m, const uint32_t *__restrict__ xadj,
                                                    const uint32_t *__restrict__ adjncy,
                                                    const int32_t *__restrict__ adjwgt,
                                                    const uint32_t *__restrict__ new_xadj,
                                                    const uint32_t *__restrict__ tile_lo,
                                                    const uint32_t *__restrict__ new_to_old,
                                                    const uint32_t *__restrict__ old_to_new,
                                                    uint32_t *__restrict__ new_adjncy, int32_t *__restrict__ new_adjwgt,
                                                    uint32_t *__restrict__ bad) {
  __shared__ uint32_t s_x[kTileVerts + 1];
  const uint32_t p0 = blockIdx.x * kTileEdges;
  const uint32_t p1 = p0 + kTileEdges < m ? p0 + kTileEdges : m; // p0 < m by the grid size
  const uint32_t u_lo = tile_lo[blockIdx.x], u_hi = tile_lo[blockIdx.x + 1];
  // u_hi owns an edge, so u_hi + 1 <= n' <= n: the staged range [u_lo, u_hi + 1] includes every end the tile reads
  const bool staged = u_hi - u_lo + 2 <= kTileVerts + 1;
  if (staged) {
    for (uint32_t i = threadIdx.x; i <= u_hi - u_lo + 1; i += blockDim.x) {
      s_x[i] = new_xadj[u_lo + i];
    }
  }
  __syncthreads();
  uint32_t e[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { // the owner searches of the eight positions are independent
    const uint32_t p = p0 + j * 256 + threadIdx.x;
    e[j] = 0;
    if (p < p1) {
      uint32_t u, end;
      if (staged) {
        const uint32_t i = owner_of_edge(s_x, 0, u_hi - u_lo, p);
        u = u_lo + i;
        end = s_x[i + 1];
      } else {
        u = owner_of_edge(new_xadj, u_lo, u_hi, p);
        end = new_xadj[u + 1];
      }
      e[j] = xadj[new_to_old[u]] + (end - 1 - p);
    }
  }
  uint32_t v[8];
  int32_t w[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const uint32_t p = p0 + j * 256 + threadIdx.x;
    v[j] = p < p1 ? adjncy[e[j]] : 0u;
    w[j] = (EW && p < p1) ? adjwgt[e[j]] : 0;
  }
  bool ok = true;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const uint32_t p = p0 + j * 256 + threadIdx.x;
    if (p < p1) {
      ok = ok && v[j] < n;
      new_adjncy[p] = v[j] < n ? old_to_new[v[j]] : v[j];
      if (EW) {
        new_adjwgt[p] = w[j];
      }
    }
  }
  if (!ok) {
    bad[1] = 1;
  }
}

// ---- finish ---------------------------------------------------------------------------------------------------
__global__ void k_prep_iso_weights(uint32_t ni, const int32_t *vwgt, long long *w) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < ni; i += gridDim.x * blockDim.x) {
    w[i] = vwgt[i];
  }
}

// S[i] = total weight of the isolated vertices [0, i) (unit weights: S == nullptr, S[i] = i)
__device__ __forceinline__ long long prep_prefix(const long long *S, uint32_t i) {
  return S != nullptr ? S[i] : static_cast<long long>(i);
}

// The next-fit chain of permutator.cc:255-261 in one warp. start[b] = s_b (start[k] = ni), bw_out[b] = bw[b] plus
// the isolated weight block b takes. Block b (b + 1 < k) ends at the first i >= s_b with
// bw[b] + S[i + 1] - S[s_b] > max(b), found by a 32-way search over the monotone S; the last block takes the rest.
__global__ void __launch_bounds__(32) k_prep_next_fit(uint32_t k, uint32_t ni, const long long *S, const int32_t *bw,
                                                      const int32_t *maxw, uint32_t *start, int32_t *bw_out) {
  const uint32_t lane = threadIdx.x;
  uint32_t s = 0;
  for (uint32_t b = 0; b < k; ++b) {
    uint32_t lo = s, hi = ni; // the answer is the first true in [lo, hi), else hi
    if (b + 1 < k) {
      const long long thr = static_cast<long long>(maxw[b]) - bw[b] + prep_prefix(S, s); // pred(i): S[i+1] > thr
      while (lo < hi) {
        const uint32_t step = static_cast<uint32_t>((static_cast<uint64_t>(hi - lo) + 31) >> 5);
        const uint64_t a = lo + static_cast<uint64_t>(lane) * step; // lane's chunk [a, min(a + step, hi))
        const uint64_t last = (a + step < hi ? a + step : hi) - 1;
        const bool t = a >= hi || prep_prefix(S, static_cast<uint32_t>(last) + 1) > thr; // an empty chunk counts as true
        const unsigned bal = __ballot_sync(kFull, t);
        if (bal == 0) {
          lo = hi;
          break;
        }
        const uint64_t af = lo + static_cast<uint64_t>(__ffs(bal) - 1) * step;
        if (af >= hi) {
          lo = hi;
          break;
        }
        // the last element of chunk f is true: the answer lies in [af, last_f]
        hi = static_cast<uint32_t>((af + step < hi ? af + step : hi) - 1);
        lo = static_cast<uint32_t>(af);
      }
    }
    const uint32_t e = b + 1 < k ? hi : ni;
    if (lane == 0) {
      start[b] = s;
      bw_out[b] = static_cast<int32_t>(bw[b] + (prep_prefix(S, e) - prep_prefix(S, s)));
    }
    s = e;
  }
  if (lane == 0) {
    start[k] = ni;
  }
}

// out[u] = p[old_to_new[u]]: the given partition for the n' vertices, the next-fit block for the isolated ones
__global__ void k_prep_map_back(uint32_t n, uint32_t np, uint32_t k, const uint32_t *old_to_new, const uint32_t *part,
                                const uint32_t *start, uint32_t *out) {
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += gridDim.x * blockDim.x) {
    const uint32_t nu = old_to_new[u];
    uint32_t b;
    if (nu < np) {
      b = part[nu];
    } else {
      const uint32_t i = nu - np;
      uint32_t lo = 0, hi = k - 1; // the largest b with start[b] <= i (start[0] = 0)
      while (lo < hi) {
        const uint32_t mid = lo + (hi - lo + 1) / 2;
        if (start[mid] <= i) {
          lo = mid;
        } else {
          hi = mid - 1;
        }
      }
      b = lo;
    }
    out[u] = b;
  }
}

} // namespace

struct kmp_prepared_graph {
  int device = 0;
  uint32_t n = 0, np = 0, m = 0;
  PoolBuf<uint32_t> xadj, adjncy, old_to_new, new_to_old;
  PoolBuf<int32_t> vwgt, adjwgt; // unallocated for unit weights
};

namespace {

int prepare_impl(kmp_lp_handle *h, uint32_t n, uint32_t m, const uint32_t *xadj, const uint32_t *adjncy,
                 const int32_t *vwgt, const int32_t *adjwgt, kmp_prepared_graph *g, kmp_prepare_stats *stats) {
  const cudaStream_t st = h->stream;
  const int dev = h->device;
  uint32_t launches = 0;
  KMP_CUDA(call_clock_start(h, st));
  g->n = n;
  g->m = m;
  KMP_CUDA(g->xadj.alloc(static_cast<size_t>(n) + 1, st, dev));
  KMP_CUDA(g->adjncy.alloc(m, st, dev));
  KMP_CUDA(g->old_to_new.alloc(n, st, dev));
  KMP_CUDA(g->new_to_old.alloc(n, st, dev));
  if (vwgt != nullptr) {
    KMP_CUDA(g->vwgt.alloc(n, st, dev));
  }
  if (adjwgt != nullptr) {
    KMP_CUDA(g->adjwgt.alloc(m, st, dev));
  }
  // ---- 1. validate, bucket, histogram -----------------------------------------------------------------------
  const uint32_t tiles = std::max<uint32_t>(1, (n + kPrepTileVerts - 1) / kPrepTileVerts);
  const size_t cells = static_cast<size_t>(kPrepBuckets) * tiles;
  PoolBuf<uint32_t> hist, base, deg, bad; // scratch of this call
  KMP_CUDA(hist.alloc(cells, st, dev));
  KMP_CUDA(base.alloc(cells, st, dev));
  KMP_CUDA(bad.alloc(2, st, dev));
  KMP_CUDA(cudaMemsetAsync(bad.p, 0, 8, st));
  k_prep_count<<<tiles, 256, 0, st>>>(n, m, xadj, tiles, hist.p, bad.p);
  ++launches;
  KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
    return cub::DeviceScan::ExclusiveSum(tmp, bytes, hist.p, base.p, static_cast<int>(cells), st);
  }));
  uint32_t host[2] = {0, 0};
  KMP_CUDA(cudaMemcpyAsync(&host[0], bad.p, 4, cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaMemcpyAsync(&host[1], base.p + static_cast<size_t>(kPrepIsolated) * tiles, 4, cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaStreamSynchronize(st));
  if (host[0] != 0) {
    return fail(KMP_ERR_INVALID, "malformed xadj: xadj[0] != 0, a decreasing entry or xadj[n] != m");
  }
  g->np = host[1];
  // ---- 2. stable scatter, new xadj --------------------------------------------------------------------------
  KMP_CUDA(deg.alloc(static_cast<size_t>(n) + 1, st, dev));
  KMP_CUDA(cudaMemsetAsync(g->xadj.p, 0, 4, st));
  if (n > 0) {
    k_prep_scatter<<<tiles, 256, 0, st>>>(n, xadj, vwgt, tiles, base.p, g->old_to_new.p, g->new_to_old.p, deg.p,
                                          g->vwgt.p);
    ++launches;
    KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
      return cub::DeviceScan::InclusiveSum(tmp, bytes, deg.p, g->xadj.p + 1, static_cast<int>(n), st);
    }));
  }
  // ---- 3. edge copy -----------------------------------------------------------------------------------------
  if (m > 0) {
    const uint32_t etiles = (m + kTileEdges - 1) / kTileEdges;
    KMP_CUDA(hist.alloc(static_cast<size_t>(etiles) + 1, st, dev)); // the histogram is dead: tile owners
    k_tile_owners<<<grid_for(static_cast<uint64_t>(etiles) + 1, 256), 256, 0, st>>>(n, m, g->xadj.p, etiles, hist.p);
    if (adjwgt != nullptr) {
      k_prep_edges<true><<<etiles, 256, 0, st>>>(n, m, xadj, adjncy, adjwgt, g->xadj.p, hist.p, g->new_to_old.p,
                                                 g->old_to_new.p, g->adjncy.p, g->adjwgt.p, bad.p);
    } else {
      k_prep_edges<false><<<etiles, 256, 0, st>>>(n, m, xadj, adjncy, nullptr, g->xadj.p, hist.p, g->new_to_old.p,
                                                  g->old_to_new.p, g->adjncy.p, nullptr, bad.p);
    }
    launches += 2;
  }
  KMP_CUDA(cudaGetLastError());
  KMP_CUDA(cudaMemcpyAsync(&host[0], bad.p + 1, 4, cudaMemcpyDeviceToHost, st));
  KMP_CUDA(call_clock_stop(h, st));
  KMP_CUDA(cudaStreamSynchronize(st));
  if (host[0] != 0) {
    return fail(KMP_ERR_INVALID, "adjncy holds a target >= n");
  }
  if (stats != nullptr) {
    stats->n = n;
    stats->n_nonisolated = g->np;
    stats->num_isolated = n - g->np;
    stats->m = m;
    stats->kernel_launches = launches;
    stats->device_ms = call_clock_ms(h);
  }
  return KMP_OK;
}

int prepare_checked(kmp_lp_handle *h, uint32_t n, uint32_t m, const uint32_t *xadj, const uint32_t *adjncy,
                    const int32_t *vwgt, const int32_t *adjwgt, bool host_input, kmp_prepared_graph **out,
                    kmp_prepare_stats *stats) {
  if (h == nullptr || out == nullptr || xadj == nullptr || (m > 0 && adjncy == nullptr)) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  if (n > 0x7FFFFFFFu || m > 0x7FFFFFFFu) {
    return fail(KMP_ERR_UNSUPPORTED, "n and m must be below 2^31");
  }
  auto misaligned4 = [](const void *p) { return (reinterpret_cast<uintptr_t>(p) & 3u) != 0; };
  if (!host_input && (misaligned4(xadj) || misaligned4(adjncy) || misaligned4(vwgt) || misaligned4(adjwgt))) {
    return fail(KMP_ERR_INVALID, "device graph arrays must be 4-byte aligned");
  }
  KMP_CUDA(cudaSetDevice(h->device));
  if (stats != nullptr) {
    std::memset(stats, 0, sizeof(*stats));
  }
  return make_result(h, out, [&](kmp_prepared_graph *g) {
    PoolBuf<uint32_t> d_xadj, d_adj;
    PoolBuf<int32_t> d_vw, d_ew;
    if (host_input) { // copies on the handle's stream, freed stream-ordered behind the kernels that read them
      const cudaStream_t st = h->stream;
      cudaError_t e = upload(d_xadj, xadj, static_cast<size_t>(n) + 1, st, h->device);
      if (e == cudaSuccess) {
        e = upload(d_adj, adjncy, m, st, h->device);
      }
      if (e == cudaSuccess && vwgt != nullptr) {
        e = upload(d_vw, vwgt, n, st, h->device);
      }
      if (e == cudaSuccess && adjwgt != nullptr) {
        e = upload(d_ew, adjwgt, m, st, h->device);
      }
      if (e != cudaSuccess) {
        return fail(e == cudaErrorMemoryAllocation ? KMP_ERR_ALLOC : KMP_ERR_CUDA,
                    std::string("uploading the graph: ") + cudaGetErrorString(e));
      }
      xadj = d_xadj.p;
      adjncy = d_adj.p;
      vwgt = vwgt != nullptr ? d_vw.p : nullptr;
      adjwgt = adjwgt != nullptr ? d_ew.p : nullptr;
    }
    return prepare_impl(h, n, m, xadj, adjncy, vwgt, adjwgt, g, stats);
  });
}

int finish_impl(kmp_lp_handle *h, const kmp_prepared_graph *g, uint32_t k, const int32_t *max_block_weights,
                const uint32_t *partition, uint32_t *partition_out, int32_t *block_weights_out) {
  const cudaStream_t st = h->stream;
  const int dev = h->device;
  const uint32_t n = g->n, np = g->np, ni = n - np;
  PoolBuf<uint32_t> d_part, start, out; // scratch of this call
  PoolBuf<int32_t> bw, maxw, bw_out;
  PoolBuf<unsigned long long> bad;
  PoolBuf<long long> w, S;
  const uint32_t *part = h->lp.label.p;
  if (partition != nullptr) {
    KMP_CUDA(d_part.alloc(np, st, dev));
    if (np > 0) {
      KMP_CUDA(cudaMemcpyAsync(d_part.p, partition, static_cast<size_t>(np) * 4, cudaMemcpyHostToDevice, st));
    }
    part = d_part.p;
  }
  // ---- block weights of the n' part; labels >= k are counted, never used as an index ----------------------------
  KMP_CUDA(bw.alloc(k, st, dev));
  KMP_CUDA(bad.alloc(1, st, dev));
  KMP_CUDA(cudaMemsetAsync(bw.p, 0, static_cast<size_t>(k) * 4, st));
  KMP_CUDA(cudaMemsetAsync(bad.p, 0, 8, st));
  if (np > 0) {
    bal_block_weights<<<grid_for(np, 256), 256, 0, st>>>(np, k, g->vwgt.p, part, bw.p, bad.p);
  }
  unsigned long long nbad = 0;
  KMP_CUDA(cudaMemcpyAsync(&nbad, bad.p, sizeof(nbad), cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaStreamSynchronize(st));
  if (nbad != 0) {
    return fail(KMP_ERR_INVALID, "partition holds a block id >= k");
  }
  // ---- next fit over the isolated vertices ------------------------------------------------------------------
  const long long *s_ptr = nullptr; // unit weights: S[i] = i
  if (g->vwgt.p != nullptr && ni > 0) {
    KMP_CUDA(w.alloc(ni, st, dev));
    KMP_CUDA(S.alloc(static_cast<size_t>(ni) + 1, st, dev));
    KMP_CUDA(cudaMemsetAsync(S.p, 0, 8, st));
    k_prep_iso_weights<<<grid_for(ni, 256), 256, 0, st>>>(ni, g->vwgt.p + np, w.p);
    KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
      return cub::DeviceScan::InclusiveSum(tmp, bytes, w.p, S.p + 1, static_cast<int>(ni), st);
    }));
    s_ptr = S.p;
  }
  KMP_CUDA(maxw.alloc(k, st, dev));
  KMP_CUDA(start.alloc(static_cast<size_t>(k) + 1, st, dev));
  KMP_CUDA(bw_out.alloc(k, st, dev));
  KMP_CUDA(cudaMemcpyAsync(maxw.p, max_block_weights, static_cast<size_t>(k) * 4, cudaMemcpyHostToDevice, st));
  k_prep_next_fit<<<1, 32, 0, st>>>(k, ni, s_ptr, bw.p, maxw.p, start.p, bw_out.p);
  // ---- map back to the caller's ids -------------------------------------------------------------------------
  if (n > 0) {
    KMP_CUDA(out.alloc(n, st, dev));
    k_prep_map_back<<<grid_for(n, 256), 256, 0, st>>>(n, np, k, g->old_to_new.p, part, start.p, out.p);
    KMP_CUDA(cudaMemcpyAsync(partition_out, out.p, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost, st));
  }
  KMP_CUDA(cudaGetLastError());
  if (block_weights_out != nullptr) {
    KMP_CUDA(cudaMemcpyAsync(block_weights_out, bw_out.p, static_cast<size_t>(k) * 4, cudaMemcpyDeviceToHost, st));
  }
  KMP_CUDA(cudaStreamSynchronize(st));
  return KMP_OK;
}

} // namespace

extern "C" {

int kmp_prepare_graph(kmp_lp_handle *h, uint32_t n, uint32_t m, const uint32_t *xadj, const uint32_t *adjncy,
                      const int32_t *vwgt, const int32_t *adjwgt, kmp_prepared_graph **out, kmp_prepare_stats *stats) {
  return prepare_checked(h, n, m, xadj, adjncy, vwgt, adjwgt, true, out, stats);
}

int kmp_prepare_graph_device(kmp_lp_handle *h, uint32_t n, uint32_t m, const uint32_t *d_xadj,
                             const uint32_t *d_adjncy, const int32_t *d_vwgt, const int32_t *d_adjwgt,
                             kmp_prepared_graph **out, kmp_prepare_stats *stats) {
  return prepare_checked(h, n, m, d_xadj, d_adjncy, d_vwgt, d_adjwgt, false, out, stats);
}

uint32_t kmp_prepared_n(const kmp_prepared_graph *g) { return g != nullptr ? g->np : 0; }
uint32_t kmp_prepared_num_isolated(const kmp_prepared_graph *g) { return g != nullptr ? g->n - g->np : 0; }
uint32_t kmp_prepared_m(const kmp_prepared_graph *g) { return g != nullptr ? g->m : 0; }

int kmp_prepared_device_arrays(const kmp_prepared_graph *g, const uint32_t **d_xadj, const uint32_t **d_adjncy,
                               const int32_t **d_vwgt, const int32_t **d_adjwgt, const uint32_t **d_old_to_new,
                               const uint32_t **d_new_to_old) {
  if (g == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  hand_out(d_xadj, g->xadj);
  hand_out(d_adjncy, g->adjncy);
  hand_out(d_vwgt, g->vwgt);
  hand_out(d_adjwgt, g->adjwgt);
  hand_out(d_old_to_new, g->old_to_new);
  hand_out(d_new_to_old, g->new_to_old);
  return KMP_OK;
}

int kmp_prepared_download(const kmp_prepared_graph *g, uint32_t *xadj, uint32_t *adjncy, int32_t *vwgt,
                          int32_t *adjwgt, uint32_t *old_to_new) {
  if (g == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  KMP_CUDA(cudaSetDevice(g->device));
  KMP_CUDA(copy_out(xadj, g->xadj, static_cast<size_t>(g->n) + 1));
  KMP_CUDA(copy_out(adjncy, g->adjncy, g->m));
  KMP_CUDA(copy_out(vwgt, g->vwgt, g->n));
  KMP_CUDA(copy_out(adjwgt, g->adjwgt, g->m));
  KMP_CUDA(copy_out(old_to_new, g->old_to_new, g->n));
  return KMP_OK;
}

int kmp_lp_set_graph_prepared(kmp_lp_handle *h, const kmp_prepared_graph *g) {
  if (h == nullptr || g == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  if (g->device != h->device) {
    return fail(KMP_ERR_INVALID, "the prepared graph lives on another device than the handle");
  }
  const int rc = kmp_lp_set_graph_device(h, g->np, g->m, g->xadj.p, g->adjncy.p, g->vwgt.p, g->adjwgt.p);
  return rc != KMP_OK ? rc : kmp_lp_set_graph_sorted(h, 1);
}

int kmp_prepared_finish(kmp_lp_handle *h, const kmp_prepared_graph *g, uint32_t k, const int32_t *max_block_weights,
                        const uint32_t *partition, uint32_t *partition_out, int32_t *block_weights_out) {
  if (h == nullptr || g == nullptr || max_block_weights == nullptr || (partition_out == nullptr && g->n > 0)) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  if (k == 0) {
    return fail(KMP_ERR_INVALID, "k must be at least 1");
  }
  if (g->device != h->device) {
    return fail(KMP_ERR_INVALID, "the prepared graph lives on another device than the handle");
  }
  if (partition == nullptr) {
    // the device labels must be the handle's labels of exactly this prepared graph
    const bool holds_g = h->graph.present && h->graph.xadj == g->xadj.p && h->graph.adjncy == g->adjncy.p && h->graph.n == g->np &&
                         h->graph.m == g->m;
    if (!holds_g) {
      return fail(KMP_ERR_INVALID, "the handle holds another graph than this prepared graph: pass the partition");
    }
    const int rc = refuse_without_labels(h);
    if (rc != KMP_OK) {
      return rc;
    }
  }
  KMP_CUDA(cudaSetDevice(h->device));
  return finish_impl(h, g, k, max_block_weights, partition, partition_out, block_weights_out);
}

void kmp_prepared_destroy(kmp_prepared_graph *g) {
  if (g == nullptr) {
    return;
  }
  cudaSetDevice(g->device); // the arrays free themselves on this device's pool
  delete g;
}

} // extern "C"
