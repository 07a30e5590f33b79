// kaminpar_b200: device-side cluster contraction + its C ABI (include/kaminpar_b200_contraction.h).
// Included at the end of kmp_lp.cu (same translation unit: it contracts the graph a kmp_lp_handle holds).
//
// What it restates (see the header for the parity definition):
//   fill_leader_mapping / compute_mapping   coarsening/contraction/cluster_contraction_preprocessing.cc:17-51
//   contract_clustering_unbuffered          coarsening/contraction/unbuffered_cluster_contraction.cc:127-606
//   CoarseGraphImpl::project_up/down        coarsening/contraction/cluster_contraction_preprocessing.h:36-46
//
// How: the reference aggregates, per coarse vertex, the neighbourhoods of its members in a hash map.
// On the GPU the natural formulation is a segmented reduction over the whole edge stream:
//   1. leader flags -> inclusive scan -> mapping[u] = rank(clustering[u])            (3 streaming passes over n)
//   2. coarse node weights: atomicAdd per fine vertex
//   3. one pass over the m fine edges: key = (mapping[u] << b | mapping[v]), value = w(u,v); edges inside
//      a cluster are dropped at the source (block-level compaction, one atomic per 2048 edges). The source
//      vertex of an edge is found by a binary search in the tile's slice of xadj staged in shared memory.
//   4. LSD radix sort of the surviving (key, value) pairs over exactly 2·ceil(log2 c_n) key bits; with unit
//      edge weights (the finest level) the keys alone are sorted
//   5. reduce-by-key (run-length encode when unweighted) -> unique coarse edges with summed weights;
//      c_xadj by binary search per coarse vertex
// Steps 4-5 use CUB (library sort / segmented reduce, like cuBLAS for a plain GEMM); 1-3 and the
// CSR assembly are hand-written. Everything is HBM-streaming integer work: algorithmic bytes per fine
// edge = 4 (adjncy) + 4 (mapping gather) [+ 4 weight] read, and per surviving edge 12 B written, then
// ceil(2b/8) radix passes of 24 B each.
#pragma once

#include <cub/block/block_scan.cuh>
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_run_length_encode.cuh>

struct kmp_coarse_graph : DeviceCsr {
  uint32_t fine_n = 0, c_n = 0, c_m = 0;
  PoolBuf<uint32_t> mapping;
};

namespace {

constexpr int kTileEdges = 2048;  // fine edges per CTA in the key pass (256 threads x 8)
constexpr int kTileVerts = 2304;  // xadj entries of a tile staged in shared memory (else: global search)

__global__ void k_flag_leaders(uint32_t n, const uint32_t *cl, uint32_t *flags, uint32_t *bad) {
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += gridDim.x * blockDim.x) {
    const uint32_t c = cl[u];
    if (c < n) {
      flags[c] = 1; // cluster_contraction_preprocessing.cc:28-30
    } else {
      *bad = 1;
    }
  }
}
// mapping[u] = leader_mapping[clustering[u]] - 1 (:44-46) and the coarse node weights
__global__ void k_map_and_weigh(uint32_t n, const uint32_t *cl, const uint32_t *rank, const int32_t *vwgt,
                                uint32_t *mapping, int32_t *c_vwgt) {
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += gridDim.x * blockDim.x) {
    const uint32_t c = rank[cl[u]] - 1;
    mapping[u] = c;
    atomicAdd(&c_vwgt[c], vwgt != nullptr ? vwgt[u] : 1);
  }
}

// largest u in [lo, hi] with x[u] <= e (x non-decreasing, x[lo] <= e)
__device__ __forceinline__ uint32_t owner_of_edge(const uint32_t *x, uint32_t lo, uint32_t hi, uint32_t e) {
  while (lo < hi) {
    const uint32_t mid = lo + (hi - lo + 1) / 2;
    if (x[mid] <= e) {
      lo = mid;
    } else {
      hi = mid - 1;
    }
  }
  return lo;
}

// tile_lo[t] = owner of the first edge of tile t (t < tiles); tile_lo[tiles] = owner of the last edge.
// One thread per tile, so that the CTAs of the key pass do not start with a serial 2 x log2(n) search.
__global__ void k_tile_owners(uint32_t n, uint32_t m, const uint32_t *xadj, uint32_t tiles, uint32_t *tile_lo) {
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t <= tiles; t += gridDim.x * blockDim.x) {
    const uint32_t e = t < tiles ? t * kTileEdges : m - 1;
    tile_lo[t] = owner_of_edge(xadj, 0, n, e);
  }
}

template <bool EW>
__global__ void __launch_bounds__(256) k_contract_edge_keys(uint32_t n, uint32_t m, const uint32_t *__restrict__ xadj,
                                                            const uint32_t *__restrict__ tile_lo,
                                                            const uint32_t *__restrict__ adjncy,
                                                            const int32_t *__restrict__ adjwgt,
                                                            const uint32_t *__restrict__ mapping, uint32_t shift,
                                                            unsigned long long *__restrict__ keys,
                                                            int32_t *__restrict__ vals, unsigned long long *counter) {
  using BlockScan = cub::BlockScan<uint32_t, 256>;
  __shared__ typename BlockScan::TempStorage scan_tmp;
  __shared__ uint32_t s_x[kTileVerts + 1];
  __shared__ unsigned long long s_base;
  const uint32_t e0 = blockIdx.x * kTileEdges;
  const uint32_t e1 = e0 + kTileEdges < m ? e0 + kTileEdges : m; // e0 < m by the grid size
  // the owners of this tile's edges lie in [u_lo, u_hi] (u_hi: owner of the next tile's first edge)
  const uint32_t u_lo = tile_lo[blockIdx.x], u_hi = tile_lo[blockIdx.x + 1];
  const bool staged = u_hi - u_lo + 1 <= kTileVerts;
  if (staged) {
    for (uint32_t i = threadIdx.x; i <= u_hi - u_lo; i += blockDim.x) {
      s_x[i] = xadj[u_lo + i];
    }
  }
  __syncthreads();
  unsigned long long key[8];
  int32_t val[8];
  uint32_t mine = 0;
  uint32_t v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { // independent, coalesced
    const uint32_t e = e0 + j * 256 + threadIdx.x;
    v[j] = e < e1 ? adjncy[e] : 0u;
    val[j] = (EW && e < e1) ? adjwgt[e] : 1;
  }
  uint32_t cv[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { // independent gathers
    const uint32_t e = e0 + j * 256 + threadIdx.x;
    cv[j] = e < e1 ? mapping[v[j]] : 0u;
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const uint32_t e = e0 + j * 256 + threadIdx.x;
    key[j] = ~0ull;
    if (e < e1) {
      const uint32_t u = staged ? u_lo + owner_of_edge(s_x, 0, u_hi - u_lo, e) : owner_of_edge(xadj, u_lo, u_hi, e);
      const uint32_t cu = mapping[u];
      if (cu != cv[j]) { // unbuffered_cluster_contraction.cc:282
        key[j] = (static_cast<unsigned long long>(cu) << shift) | cv[j];
        ++mine;
      }
    }
  }
  uint32_t off = 0, total = 0;
  BlockScan(scan_tmp).ExclusiveSum(mine, off, total);
  if (total == 0) {
    return;
  }
  if (threadIdx.x == 0) {
    s_base = atomicAdd(counter, static_cast<unsigned long long>(total));
  }
  __syncthreads();
  unsigned long long o = s_base + off;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    if (key[j] != ~0ull) {
      keys[o] = key[j];
      if (EW) {
        vals[o] = val[j];
      }
      ++o;
    }
  }
}

// c_xadj[c] = first unique edge whose source is >= c; c_adjncy = low key bits
__global__ void k_coarse_offsets(uint32_t c_n, uint32_t c_m, const unsigned long long *ukeys, uint32_t shift,
                                 uint32_t *c_xadj) {
  for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c <= c_n; c += gridDim.x * blockDim.x) {
    const unsigned long long target = static_cast<unsigned long long>(c) << shift;
    uint32_t lo = 0, hi = c_m;
    while (lo < hi) {
      const uint32_t mid = lo + (hi - lo) / 2;
      if (ukeys[mid] < target) {
        lo = mid + 1;
      } else {
        hi = mid;
      }
    }
    c_xadj[c] = lo;
  }
}
__global__ void k_coarse_targets(uint32_t c_m, const unsigned long long *ukeys, uint32_t shift, uint32_t *c_adjncy) {
  const unsigned long long mask = (1ull << shift) - 1;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < c_m; i += gridDim.x * blockDim.x) {
    c_adjncy[i] = static_cast<uint32_t>(ukeys[i] & mask);
  }
}
__global__ void k_project_up(uint32_t n, const uint32_t *mapping, const uint32_t *coarse, uint32_t *fine) {
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += gridDim.x * blockDim.x) {
    fine[u] = coarse[mapping[u]];
  }
}
__global__ void k_project_down(uint32_t n, const uint32_t *mapping, const uint32_t *fine, uint32_t *coarse) {
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += gridDim.x * blockDim.x) {
    coarse[mapping[u]] = fine[u];
  }
}

uint32_t ceil_log2_u32(uint32_t x) { // smallest b with 2^b >= x (x >= 1)
  uint32_t b = 0;
  while ((1ull << b) < x) {
    ++b;
  }
  return b;
}

int contract_impl(kmp_lp_handle *h, const uint32_t *clustering, kmp_coarse_graph *cg, kmp_contraction_stats *stats) {
  const uint32_t n = h->graph.n, m = h->graph.m;
  cudaStream_t st = h->stream;
  uint32_t launches = 0;
  cg->fine_n = n;
  KMP_CUDA(cg->mapping.alloc(n, st, h->device));
  if (n == 0) {
    KMP_CUDA(cg->xadj.alloc(1, st, h->device));
    KMP_CUDA(cudaMemsetAsync(cg->xadj.p, 0, sizeof(uint32_t), st));
    KMP_CUDA(cudaStreamSynchronize(st));
    return KMP_OK;
  }
  // scratch lives in the handle (grow-only): no cudaMalloc / cudaFree on the timed path after the first call
  DevBuf<uint32_t> &d_cl = h->ops.ct_cl, &flags = h->ops.ct_flags, &rank = h->ops.ct_rank;
  const uint32_t *cl = nullptr;
  if (clustering != nullptr) {
    KMP_CUDA(d_cl.ensure(n));
    KMP_CUDA(cudaMemcpyAsync(d_cl.p, clustering, static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, st));
    cl = d_cl.p;
  } else {
    cl = h->lp.label.p; // kmp_contract_clustering refused labels of another graph
  }
  KMP_CUDA(call_clock_start(h, st));
  // ---- 1. mapping ------------------------------------------------------------------------------
  KMP_CUDA(flags.ensure(static_cast<size_t>(n) + 1)); // flags[n]: out-of-range marker
  KMP_CUDA(rank.ensure(n));
  KMP_CUDA(cudaMemsetAsync(flags.p, 0, (static_cast<size_t>(n) + 1) * 4, st));
  k_flag_leaders<<<grid_for(n, 256), 256, 0, st>>>(n, cl, flags.p, flags.p + n);
  KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
    return cub::DeviceScan::InclusiveSum(tmp, bytes, flags.p, rank.p, static_cast<int>(n), st);
  }));
  uint32_t host2[2] = {0, 0};
  KMP_CUDA(cudaMemcpyAsync(&host2[0], rank.p + (n - 1), 4, cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaMemcpyAsync(&host2[1], flags.p + n, 4, cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaStreamSynchronize(st));
  if (host2[1] != 0) {
    return fail(KMP_ERR_INVALID, "clustering holds an id >= n");
  }
  const uint32_t c_n = host2[0];
  cg->c_n = c_n;
  KMP_CUDA(cg->vwgt.alloc(c_n, st, h->device));
  KMP_CUDA(cudaMemsetAsync(cg->vwgt.p, 0, static_cast<size_t>(c_n) * 4, st));
  k_map_and_weigh<<<grid_for(n, 256), 256, 0, st>>>(n, cl, rank.p, h->graph.vwgt, cg->mapping.p, cg->vwgt.p);
  launches += 4;
  // ---- 2. edge keys ----------------------------------------------------------------------------
  const uint32_t shift = std::max<uint32_t>(1, ceil_log2_u32(c_n));
  const uint32_t bits = shift + std::max<uint32_t>(1, ceil_log2_u32(c_n));
  unsigned long long cut = 0;
  DevBuf<unsigned long long> &keys_a = h->ops.pairs_a, &keys_b = h->ops.pairs_b, &counter = h->ops.ct_counter;
  DevBuf<int32_t> &vals_a = h->ops.ct_vals_a, &vals_b = h->ops.ct_vals_b;
  KMP_CUDA(counter.ensure(2));
  KMP_CUDA(cudaMemsetAsync(counter.p, 0, 16, st));
  if (m > 0) {
    KMP_CUDA(keys_a.ensure(m));
    if (h->graph.adjwgt != nullptr) {
      KMP_CUDA(vals_a.ensure(m));
    }
    const uint32_t tiles = (m + kTileEdges - 1) / kTileEdges;
    KMP_CUDA(flags.ensure(static_cast<size_t>(tiles) + 1)); // the leader flags are dead: reuse as tile_lo
    k_tile_owners<<<grid_for(static_cast<uint64_t>(tiles) + 1, 256), 256, 0, st>>>(n, m, h->graph.xadj, tiles, flags.p);
    if (h->graph.adjwgt != nullptr) {
      k_contract_edge_keys<true><<<tiles, 256, 0, st>>>(n, m, h->graph.xadj, flags.p, h->graph.adjncy, h->graph.adjwgt, cg->mapping.p,
                                                        shift, keys_a.p, vals_a.p, counter.p);
    } else {
      k_contract_edge_keys<false><<<tiles, 256, 0, st>>>(n, m, h->graph.xadj, flags.p, h->graph.adjncy, nullptr, cg->mapping.p,
                                                         shift, keys_a.p, vals_a.p, counter.p);
    }
    launches += 2;
    KMP_CUDA(cudaGetLastError());
    KMP_CUDA(cudaMemcpyAsync(&cut, counter.p, 8, cudaMemcpyDeviceToHost, st));
    KMP_CUDA(cudaStreamSynchronize(st));
  }
  if (cut > 0x7FFFFFFFull) {
    return fail(KMP_ERR_UNSUPPORTED, "more than 2^31 - 1 inter-cluster edges");
  }
  // ---- 3. sort + reduce by key -----------------------------------------------------------------
  uint32_t c_m = 0;
  KMP_CUDA(cg->xadj.alloc(static_cast<size_t>(c_n) + 1, st, h->device));
  if (cut > 0) {
    const int items = static_cast<int>(cut);
    KMP_CUDA(keys_b.ensure(cut));
    KMP_CUDA(vals_b.ensure(cut));
    cub::DoubleBuffer<unsigned long long> dk(keys_a.p, keys_b.p);
    uint32_t *num_runs = reinterpret_cast<uint32_t *>(counter.p + 1);
    unsigned long long *uk = nullptr; // unique keys: the idle half of the key double buffer
    int32_t *uw = nullptr;            // their weights
    if (h->graph.adjwgt != nullptr) {
      cub::DoubleBuffer<int32_t> dv(vals_a.p, vals_b.p);
      KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
        return cub::DeviceRadixSort::SortPairs(tmp, bytes, dk, dv, items, 0, static_cast<int>(bits), st);
      }));
      uk = dk.Alternate();
      uw = dv.Alternate();
      KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
        return cub::DeviceReduce::ReduceByKey(tmp, bytes, dk.Current(), uk, dv.Current(), uw, num_runs, cub::Sum(),
                                              items, st);
      }));
    } else {
      // unit edge weights (the finest, i.e. largest, level): sort the keys alone (8 instead of 12 bytes per
      // item and pass); the weight of a coarse edge is the length of its run
      KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
        return cub::DeviceRadixSort::SortKeys(tmp, bytes, dk, items, 0, static_cast<int>(bits), st);
      }));
      uk = dk.Alternate();
      uw = vals_b.p;
      KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
        return cub::DeviceRunLengthEncode::Encode(tmp, bytes, dk.Current(), uk, uw, num_runs, items, st);
      }));
    }
    KMP_CUDA(cudaMemcpyAsync(&c_m, num_runs, 4, cudaMemcpyDeviceToHost, st));
    KMP_CUDA(cudaStreamSynchronize(st));
    // ---- 4. CSR assembly -------------------------------------------------------------------------
    KMP_CUDA(cg->adjncy.alloc(c_m, st, h->device));
    KMP_CUDA(cg->adjwgt.alloc(c_m, st, h->device));
    KMP_CUDA(cudaMemcpyAsync(cg->adjwgt.p, uw, static_cast<size_t>(c_m) * 4, cudaMemcpyDeviceToDevice, st));
    k_coarse_offsets<<<grid_for(static_cast<uint64_t>(c_n) + 1, 256), 256, 0, st>>>(c_n, c_m, uk, shift, cg->xadj.p);
    k_coarse_targets<<<grid_for(c_m, 256), 256, 0, st>>>(c_m, uk, shift, cg->adjncy.p);
    launches += 4; // + the radix passes and the reduce inside CUB
    KMP_CUDA(cudaGetLastError());
  } else {
    KMP_CUDA(cudaMemsetAsync(cg->xadj.p, 0, (static_cast<size_t>(c_n) + 1) * 4, st));
    KMP_CUDA(cg->adjncy.alloc(1, st, h->device));
    KMP_CUDA(cg->adjwgt.alloc(1, st, h->device));
  }
  cg->c_m = c_m;
  KMP_CUDA(call_clock_stop(h, st));
  KMP_CUDA(cudaStreamSynchronize(st));
  const float ms = call_clock_ms(h);
  if (stats != nullptr) {
    stats->c_n = c_n;
    stats->c_m = c_m;
    stats->cut_edges = cut;
    stats->sort_bits = bits;
    stats->kernel_launches = launches;
    stats->device_ms = ms;
  }
  return KMP_OK;
}

} // namespace

extern "C" {

int kmp_contract_clustering(kmp_lp_handle *h, const uint32_t *clustering, kmp_coarse_graph **out,
                            kmp_contraction_stats *stats) {
  if (h == nullptr || out == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  if (!h->graph.present) {
    return fail(KMP_ERR_INVALID, "no graph set");
  }
  int rc = clustering == nullptr ? refuse_without_labels(h) : KMP_OK;
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(cudaSetDevice(h->device));
  if (stats != nullptr) {
    std::memset(stats, 0, sizeof(*stats));
  }
  return make_result(h, out, [&](kmp_coarse_graph *cg) { return contract_impl(h, clustering, cg, stats); });
}

uint32_t kmp_coarse_n(const kmp_coarse_graph *g) { return g != nullptr ? g->c_n : 0; }
uint32_t kmp_coarse_m(const kmp_coarse_graph *g) { return g != nullptr ? g->c_m : 0; }
uint32_t kmp_coarse_fine_n(const kmp_coarse_graph *g) { return g != nullptr ? g->fine_n : 0; }

int kmp_coarse_download(const kmp_coarse_graph *g, uint32_t *xadj, uint32_t *adjncy, int32_t *vwgt, int32_t *adjwgt,
                        uint32_t *mapping) {
  if (g == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  const int rc = download_csr(*g, xadj, adjncy, vwgt, adjwgt, static_cast<size_t>(g->c_n) + 1, g->c_n, g->c_m);
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(copy_out(mapping, g->mapping, g->fine_n));
  return KMP_OK;
}

int kmp_coarse_device_arrays(const kmp_coarse_graph *g, const uint32_t **d_xadj, const uint32_t **d_adjncy,
                             const int32_t **d_vwgt, const int32_t **d_adjwgt, const uint32_t **d_mapping) {
  if (g == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  hand_out_csr(*g, d_xadj, d_adjncy, d_vwgt, d_adjwgt);
  hand_out(d_mapping, g->mapping);
  return KMP_OK;
}

int kmp_coarse_project_up(const kmp_coarse_graph *g, const uint32_t *coarse, uint32_t *fine) {
  if (g == nullptr || coarse == nullptr || fine == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  if (g->fine_n == 0) {
    return KMP_OK;
  }
  KMP_CUDA(cudaSetDevice(g->device));
  DevBuf<uint32_t> d_c, d_f;
  KMP_CUDA(d_c.ensure(g->c_n));
  KMP_CUDA(d_f.ensure(g->fine_n));
  KMP_CUDA(cudaMemcpy(d_c.p, coarse, static_cast<size_t>(g->c_n) * 4, cudaMemcpyHostToDevice));
  k_project_up<<<grid_for(g->fine_n, 256), 256>>>(g->fine_n, g->mapping.p, d_c.p, d_f.p);
  KMP_CUDA(cudaGetLastError());
  KMP_CUDA(cudaMemcpy(fine, d_f.p, static_cast<size_t>(g->fine_n) * 4, cudaMemcpyDeviceToHost));
  return KMP_OK;
}

int kmp_coarse_project_down(const kmp_coarse_graph *g, const uint32_t *fine, uint32_t *coarse) {
  if (g == nullptr || coarse == nullptr || fine == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  if (g->fine_n == 0) {
    return KMP_OK;
  }
  KMP_CUDA(cudaSetDevice(g->device));
  DevBuf<uint32_t> d_c, d_f;
  KMP_CUDA(d_c.ensure(g->c_n));
  KMP_CUDA(d_f.ensure(g->fine_n));
  KMP_CUDA(cudaMemcpy(d_f.p, fine, static_cast<size_t>(g->fine_n) * 4, cudaMemcpyHostToDevice));
  KMP_CUDA(cudaMemset(d_c.p, 0, static_cast<size_t>(g->c_n) * 4));
  k_project_down<<<grid_for(g->fine_n, 256), 256>>>(g->fine_n, g->mapping.p, d_f.p, d_c.p);
  KMP_CUDA(cudaGetLastError());
  KMP_CUDA(cudaMemcpy(coarse, d_c.p, static_cast<size_t>(g->c_n) * 4, cudaMemcpyDeviceToHost));
  return KMP_OK;
}

void kmp_coarse_destroy(kmp_coarse_graph *g) { destroy_result(g); }

} // extern "C"
