// kaminpar_b200: block-induced subgraph extraction and the copy-back of sub-partitions on the device + their C ABI
// (include/kaminpar_b200_subgraph.h, DESIGN.md §16). Included at the end of kmp_lp.cu after kmp_prepare.cuh: the
// edge passes find the vertex that owns an edge with the contraction's tile owners (k_tile_owners, owner_of_edge),
// labels >= k and the k' block weights go through the refiner's bal_block_weights, scratch is PoolBuf.
//
// What it restates (see the header): graph::lazy_extract_subgraphs_preprocessing + graph::extract_subgraph
// (graphutils/subgraph_extractor.cc:181-324) and graph::copy_subgraph_partitions (:492-533).
//   1. count (edge tiles of kTileEdges, grid-stride): flag(e) = part[adjncy[e]] == part[u]; per tile the number of
//      internal edges, per vertex its internal degree (shared-memory counts, a plain store for a vertex whose edges
//      lie in the tile, a global atomic only for one that spans tiles).
//   2. vertex order: a stable CUB radix sort of (part[u], u) over ceil(log2 k) bits gives block_nodes and the block
//      per position; node_off by a lower bound per block; mapping, node weights and the internal degrees in the new order
//      by one gather; a scan of those degrees gives the global edge offsets, and one kernel the per-block local xadj
//      (n + k entries) and per vertex delta[u] = (its first new edge) - (internal edges before it in fine order).
//      One host wait reads the internal edge count for the allocation.
//   3. edges (the hot path): the flag again; an in-tile exclusive scan (warp ballots) plus the tile prefix gives each
//      internal edge its fine-order rank r, and it lands at delta[u] + r as mapping[v] (+ its weight). No m-sized
//      flag or scan array.
//   4. copy-back: out[block_nodes[p]] = k0[blk[p]] + sub[p], range-checked on the device before h's labels change.
#pragma once

namespace {

// the in-tile edge ranks of k_sub_edges: one counter per (round, warp) of a 256-thread CTA
constexpr int kSubWarps = 8;
constexpr int kSubRounds = kTileEdges / 256;
static_assert(kSubWarps * kSubRounds == 64, "the tile scan of k_sub_edges covers 64 counters with one warp");

// Stage xadj[u_lo .. u_hi + 1] (u_hi owns an edge, so u_hi + 1 <= n). Returns false where the range does not fit.
__device__ __forceinline__ bool sub_stage(const uint32_t *__restrict__ xadj, uint32_t u_lo, uint32_t u_hi,
                                          uint32_t *s_x) {
  const bool staged = u_hi - u_lo + 2 <= kTileVerts + 1;
  if (staged) {
    for (uint32_t i = threadIdx.x; i <= u_hi - u_lo + 1; i += blockDim.x) {
      s_x[i] = xadj[u_lo + i];
    }
  }
  return staged;
}

// tile_cnt[t] = internal edges of tile t; deg[u] (zeroed) = internal degree of u
__global__ void __launch_bounds__(256) k_sub_count(uint32_t m, const uint32_t *__restrict__ xadj,
                                                   const uint32_t *__restrict__ adjncy,
                                                   const uint32_t *__restrict__ tile_lo, uint32_t tiles,
                                                   const uint32_t *__restrict__ part, uint32_t *__restrict__ tile_cnt,
                                                   uint32_t *__restrict__ deg) {
  __shared__ uint32_t s_x[kTileVerts + 1];
  __shared__ uint32_t s_deg[kTileVerts + 1];
  __shared__ uint32_t s_red[kSubWarps];
  for (uint32_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    const uint32_t e0 = t * kTileEdges;
    const uint32_t e1 = e0 + kTileEdges < m ? e0 + kTileEdges : m;
    const uint32_t u_lo = tile_lo[t], u_hi = tile_lo[t + 1];
    __syncthreads(); // the previous tile is done with s_x, s_deg and s_red
    const bool staged = sub_stage(xadj, u_lo, u_hi, s_x);
    if (staged) {
      for (uint32_t i = threadIdx.x; i <= u_hi - u_lo; i += blockDim.x) {
        s_deg[i] = 0;
      }
    }
    __syncthreads();
    uint32_t v[kSubRounds];
#pragma unroll
    for (int j = 0; j < kSubRounds; ++j) { // independent, coalesced
      const uint32_t e = e0 + j * 256 + threadIdx.x;
      v[j] = e < e1 ? adjncy[e] : 0u;
    }
    uint32_t mine = 0;
#pragma unroll
    for (int j = 0; j < kSubRounds; ++j) {
      const uint32_t e = e0 + j * 256 + threadIdx.x;
      if (e < e1) {
        const uint32_t i = staged ? owner_of_edge(s_x, 0, u_hi - u_lo, e) : owner_of_edge(xadj, u_lo, u_hi, e) - u_lo;
        if (part[v[j]] == part[u_lo + i]) {
          ++mine;
          if (staged) {
            atomicAdd(&s_deg[i], 1u);
          } else {
            atomicAdd(&deg[u_lo + i], 1u);
          }
        }
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      mine += __shfl_xor_sync(kFull, mine, o);
    }
    if ((threadIdx.x & 31) == 0) {
      s_red[threadIdx.x >> 5] = mine;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t c = 0;
      for (int w = 0; w < kSubWarps; ++w) {
        c += s_red[w];
      }
      tile_cnt[t] = c;
    }
    if (staged) {
      for (uint32_t i = threadIdx.x; i <= u_hi - u_lo; i += blockDim.x) {
        const uint32_t d = s_deg[i];
        if (d != 0) {
          if (s_x[i] >= e0 && s_x[i + 1] <= e1) {
            deg[u_lo + i] = d; // all of u's edges lie in this tile
          } else {
            atomicAdd(&deg[u_lo + i], d);
          }
        }
      }
    }
  }
}

// node_off[b] = first position of block b in the sorted blk (node_off[k] = n): a lower bound per block, so that
// empty blocks cost what non-empty ones do even when k is much larger than n
__global__ void k_sub_node_off(uint32_t n, uint32_t k, const uint32_t *__restrict__ blk, uint32_t *__restrict__ node_off) {
  for (uint32_t b = blockIdx.x * blockDim.x + threadIdx.x; b <= k; b += gridDim.x * blockDim.x) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
      const uint32_t mid = lo + (hi - lo) / 2;
      if (blk[mid] < b) {
        lo = mid + 1;
      } else {
        hi = mid;
      }
    }
    node_off[b] = lo;
  }
}

// position p of the sorted order: mapping[u], the node weight and the internal degree of u = block_nodes[p]
__global__ void k_sub_map(uint32_t n, const uint32_t *__restrict__ blk, const uint32_t *__restrict__ block_nodes,
                          const uint32_t *__restrict__ node_off, const int32_t *__restrict__ vwgt,
                          const uint32_t *__restrict__ deg, uint32_t *__restrict__ mapping,
                          int32_t *__restrict__ sub_vwgt, uint32_t *__restrict__ deg_new) {
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
    const uint32_t u = block_nodes[p];
    mapping[u] = p - node_off[blk[p]];
    if (vwgt != nullptr) {
      sub_vwgt[p] = vwgt[u];
    }
    deg_new[p] = deg[u];
  }
}

// items [0, n): the local xadj entry of position p and delta[u]; items [n, n + k]: edge_off[b] and, for b < k, the
// closing entry of block b's local xadj. edge_pos: exclusive scan of the internal degrees in the new order (n + 1).
__global__ void k_sub_xadj(uint32_t n, uint32_t k, const uint32_t *__restrict__ blk,
                           const uint32_t *__restrict__ block_nodes, const uint32_t *__restrict__ node_off,
                           const uint32_t *__restrict__ edge_pos, const uint32_t *__restrict__ first_rank,
                           uint32_t *__restrict__ xadj_cat, uint32_t *__restrict__ edge_off,
                           uint32_t *__restrict__ delta) {
  const uint64_t items = static_cast<uint64_t>(n) + k + 1;
  for (uint64_t i = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; i < items;
       i += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    if (i < n) {
      const uint32_t p = static_cast<uint32_t>(i), b = blk[p], u = block_nodes[p];
      xadj_cat[p + b] = edge_pos[p] - edge_pos[node_off[b]];
      delta[u] = edge_pos[p] - first_rank[u];
    } else {
      const uint32_t b = static_cast<uint32_t>(i - n);
      const uint32_t lo = edge_pos[node_off[b]];
      edge_off[b] = lo;
      if (b < k) {
        xadj_cat[node_off[b + 1] + b] = edge_pos[node_off[b + 1]] - lo;
      }
    }
  }
}

// internal edge e of u, fine-order rank r (tile_base[t] + its rank in the tile): adjncy_out[delta[u] + r] = mapping[v]
template <bool EW>
__global__ void __launch_bounds__(256) k_sub_edges(uint32_t m, const uint32_t *__restrict__ xadj,
                                                   const uint32_t *__restrict__ adjncy,
                                                   const int32_t *__restrict__ adjwgt,
                                                   const uint32_t *__restrict__ tile_lo, uint32_t tiles,
                                                   const uint32_t *__restrict__ tile_base,
                                                   const uint32_t *__restrict__ part,
                                                   const uint32_t *__restrict__ mapping,
                                                   const uint32_t *__restrict__ delta, uint32_t *__restrict__ adjncy_out,
                                                   int32_t *__restrict__ adjwgt_out) {
  __shared__ uint32_t s_x[kTileVerts + 1];
  __shared__ uint32_t s_off[kSubRounds * kSubWarps];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned below = (1u << lane) - 1u;
  for (uint32_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    const uint32_t e0 = t * kTileEdges;
    const uint32_t e1 = e0 + kTileEdges < m ? e0 + kTileEdges : m;
    const uint32_t u_lo = tile_lo[t], u_hi = tile_lo[t + 1];
    __syncthreads(); // the previous tile is done with s_x and s_off
    const bool staged = sub_stage(xadj, u_lo, u_hi, s_x);
    __syncthreads();
    uint32_t v[kSubRounds], u[kSubRounds];
    unsigned bal[kSubRounds];
#pragma unroll
    for (int j = 0; j < kSubRounds; ++j) {
      const uint32_t e = e0 + j * 256 + threadIdx.x;
      v[j] = e < e1 ? adjncy[e] : 0u;
    }
#pragma unroll
    for (int j = 0; j < kSubRounds; ++j) {
      const uint32_t e = e0 + j * 256 + threadIdx.x;
      bool in = false;
      u[j] = 0;
      if (e < e1) {
        u[j] = staged ? u_lo + owner_of_edge(s_x, 0, u_hi - u_lo, e) : owner_of_edge(xadj, u_lo, u_hi, e);
        in = part[v[j]] == part[u[j]];
      }
      bal[j] = __ballot_sync(kFull, in);
      if (lane == 0) {
        s_off[j * kSubWarps + warp] = __popc(bal[j]);
      }
    }
    __syncthreads();
    if (warp == 0) { // exclusive scan of the 64 (round, warp) counts in edge order, two per lane
      const uint32_t a = s_off[2 * lane], b = s_off[2 * lane + 1];
      uint32_t incl = a + b;
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t x = __shfl_up_sync(kFull, incl, o);
        incl += lane >= static_cast<uint32_t>(o) ? x : 0u;
      }
      const uint32_t excl = incl - a - b;
      s_off[2 * lane] = excl;
      s_off[2 * lane + 1] = excl + a;
    }
    __syncthreads();
    const uint32_t base = tile_base[t];
#pragma unroll
    for (int j = 0; j < kSubRounds; ++j) {
      if ((bal[j] >> lane) & 1u) {
        const uint32_t e = e0 + j * 256 + threadIdx.x;
        const uint32_t r = base + s_off[j * kSubWarps + warp] + __popc(bal[j] & below);
        const uint32_t dst = delta[u[j]] + r;
        adjncy_out[dst] = mapping[v[j]];
        if (EW) {
          adjwgt_out[dst] = adjwgt[e];
        }
      }
    }
  }
}

// out[block_nodes[p]] = k0[blk[p]] + sub[p]; a sub label >= its block's sub-block count is counted, not written
__global__ void k_sub_copy_back(uint32_t n, const uint32_t *__restrict__ blk, const uint32_t *__restrict__ block_nodes,
                                const uint32_t *__restrict__ k0, const uint32_t *__restrict__ sub,
                                uint32_t *__restrict__ out, unsigned long long *bad) {
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
    const uint32_t b = blk[p], s = sub[p], lo = k0[b];
    if (s < k0[b + 1] - lo) {
      out[block_nodes[p]] = lo + s;
    } else {
      atomicAdd(bad, 1ull);
    }
  }
}

inline uint32_t sub_ceil_log2(uint32_t k) {
  uint32_t b = 0;
  while (b < 32 && (1ull << b) < k) {
    ++b;
  }
  return b;
}

} // namespace

struct kmp_subgraphs {
  int device = 0;
  uint32_t n = 0, k = 0, m = 0;
  uint64_t graph_epoch = 0; // the handle's graph this was extracted from
  const kmp_lp_handle *source = nullptr;
  PoolBuf<uint32_t> xadj, adjncy, mapping, block_nodes, blk, node_off, edge_off;
  PoolBuf<int32_t> vwgt, adjwgt; // unallocated for unit weights
};

namespace {

// compute_final_k (partitioning/partition_utils.cc:21-49): block's number of final blocks at current_k on the way
// to input_k (base, or base + 1 for the blocks whose bit-reversed id is below input_k mod 2^level)
uint32_t sub_final_k(uint32_t block, uint32_t current_k, uint32_t input_k) {
  if (current_k == input_k) {
    return 1;
  }
  uint32_t level = 0;
  while ((current_k >> (level + 1)) != 0) { // floor_log2
    ++level;
  }
  const uint32_t base = input_k >> level;
  const uint32_t plus_one = input_k & ((1u << level) - 1u);
  uint32_t rev = 0;
  for (int i = 0; i < 32; ++i) {
    rev |= ((block >> i) & 1u) << (31 - i);
  }
  const int64_t reversed = static_cast<int64_t>(rev) >> (32 - level);
  return base + (reversed < static_cast<int64_t>(plus_one) ? 1u : 0u);
}

int extract_impl(kmp_lp_handle *h, uint32_t k, kmp_subgraphs *g, kmp_subgraph_stats *stats) {
  const cudaStream_t st = h->stream;
  const int dev = h->device;
  const uint32_t n = h->graph.n, m = h->graph.m;
  const uint32_t *part = h->lp.label.p;
  uint32_t launches = 0;
  // ---- labels >= k are refused before any [k] array is indexed by one ---------------------------------------
  {
    PoolBuf<int32_t> bw;
    PoolBuf<unsigned long long> bad;
    KMP_CUDA(bw.alloc(k, st, dev));
    KMP_CUDA(bad.alloc(1, st, dev));
    KMP_CUDA(cudaMemsetAsync(bw.p, 0, static_cast<size_t>(k) * 4, st));
    KMP_CUDA(cudaMemsetAsync(bad.p, 0, 8, st));
    if (n > 0) {
      bal_block_weights<<<capped(h, grid_for(n, 256)), 256, 0, st>>>(n, k, nullptr, part, bw.p, bad.p);
      ++launches;
    }
    unsigned long long nbad = 0;
    KMP_CUDA(cudaMemcpyAsync(&nbad, bad.p, sizeof(nbad), cudaMemcpyDeviceToHost, st));
    KMP_CUDA(cudaStreamSynchronize(st));
    if (nbad != 0) {
      h->lp.labels_valid = false; // a host partition was loaded as the labels: they are not a k-way partition
      return fail(KMP_ERR_INVALID, "partition holds a block id >= k");
    }
  }
  g->n = n;
  g->k = k;
  g->graph_epoch = h->graph.epoch;
  g->source = h;
  KMP_CUDA(g->xadj.alloc(static_cast<size_t>(n) + k, st, dev));
  KMP_CUDA(g->mapping.alloc(n, st, dev));
  KMP_CUDA(g->block_nodes.alloc(n, st, dev));
  KMP_CUDA(g->blk.alloc(n, st, dev));
  KMP_CUDA(g->node_off.alloc(static_cast<size_t>(k) + 1, st, dev));
  KMP_CUDA(g->edge_off.alloc(static_cast<size_t>(k) + 1, st, dev));
  if (h->graph.vwgt != nullptr) {
    KMP_CUDA(g->vwgt.alloc(n, st, dev));
  }
  const uint32_t tiles = (m + kTileEdges - 1) / kTileEdges;
  PoolBuf<uint32_t> tile_lo, tile_cnt, tile_base, deg, first_rank, iota, deg_new, edge_pos, delta;
  // ---- 1. count ---------------------------------------------------------------------------------------------
  KMP_CUDA(deg.alloc(n, st, dev));
  KMP_CUDA(cudaMemsetAsync(deg.p, 0, static_cast<size_t>(n) * 4, st));
  KMP_CUDA(tile_lo.alloc(static_cast<size_t>(tiles) + 1, st, dev));
  KMP_CUDA(tile_cnt.alloc(static_cast<size_t>(tiles) + 1, st, dev));
  KMP_CUDA(tile_base.alloc(static_cast<size_t>(tiles) + 1, st, dev));
  if (m > 0) {
    k_tile_owners<<<capped(h, grid_for(static_cast<uint64_t>(tiles) + 1, 256)), 256, 0, st>>>(n, m, h->graph.xadj, tiles,
                                                                                              tile_lo.p);
    k_sub_count<<<capped(h, std::min<uint32_t>(tiles, kSMs * 8)), 256, 0, st>>>(m, h->graph.xadj, h->graph.adjncy, tile_lo.p, tiles,
                                                                                part, tile_cnt.p, deg.p);
    launches += 2;
    KMP_CUDA(cudaMemsetAsync(tile_cnt.p + tiles, 0, 4, st));
    KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
      return cub::DeviceScan::ExclusiveSum(tmp, bytes, tile_cnt.p, tile_base.p, static_cast<int>(tiles) + 1, st);
    }));
  }
  // ---- 2. vertex order, offsets, local xadj -----------------------------------------------------------------
  KMP_CUDA(deg_new.alloc(static_cast<size_t>(n) + 1, st, dev));
  KMP_CUDA(edge_pos.alloc(static_cast<size_t>(n) + 1, st, dev));
  KMP_CUDA(cudaMemsetAsync(edge_pos.p, 0, 4, st)); // n == 0: edge_pos = [0]
  if (n > 0) {
    KMP_CUDA(iota.alloc(n, st, dev));
    bal_iota<<<capped(h, grid_for(n, 256)), 256, 0, st>>>(n, iota.p);
    const int bits = static_cast<int>(std::max<uint32_t>(1, sub_ceil_log2(k)));
    KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
      return cub::DeviceRadixSort::SortPairs(tmp, bytes, part, g->blk.p, iota.p, g->block_nodes.p, static_cast<int>(n),
                                             0, bits, st);
    }));
    k_sub_node_off<<<capped(h, grid_for(static_cast<uint64_t>(k) + 1, 256)), 256, 0, st>>>(n, k, g->blk.p,
                                                                                            g->node_off.p);
    k_sub_map<<<capped(h, grid_for(n, 256)), 256, 0, st>>>(n, g->blk.p, g->block_nodes.p, g->node_off.p, h->graph.vwgt, deg.p,
                                                           g->mapping.p, g->vwgt.p, deg_new.p);
    launches += 3;
    KMP_CUDA(cudaMemsetAsync(deg_new.p + n, 0, 4, st));
    KMP_CUDA(first_rank.alloc(n, st, dev));
    KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
      return cub::DeviceScan::ExclusiveSum(tmp, bytes, deg.p, first_rank.p, static_cast<int>(n), st);
    }));
    KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
      return cub::DeviceScan::ExclusiveSum(tmp, bytes, deg_new.p, edge_pos.p, static_cast<int>(n) + 1, st);
    }));
  } else {
    KMP_CUDA(cudaMemsetAsync(g->node_off.p, 0, (static_cast<size_t>(k) + 1) * 4, st));
  }
  KMP_CUDA(delta.alloc(n, st, dev));
  k_sub_xadj<<<capped(h, grid_for(static_cast<uint64_t>(n) + k + 1, 256)), 256, 0, st>>>(
      n, k, g->blk.p, g->block_nodes.p, g->node_off.p, edge_pos.p, first_rank.p, g->xadj.p, g->edge_off.p, delta.p);
  ++launches;
  uint32_t m_int = 0;
  KMP_CUDA(cudaMemcpyAsync(&m_int, edge_pos.p + n, 4, cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaStreamSynchronize(st));
  g->m = m_int;
  // ---- 3. edges ---------------------------------------------------------------------------------------------
  KMP_CUDA(g->adjncy.alloc(m_int, st, dev));
  if (h->graph.adjwgt != nullptr) {
    KMP_CUDA(g->adjwgt.alloc(m_int, st, dev));
  }
  if (m_int > 0) {
    const uint32_t grid = capped(h, std::min<uint32_t>(tiles, kSMs * 8));
    if (h->graph.adjwgt != nullptr) {
      k_sub_edges<true><<<grid, 256, 0, st>>>(m, h->graph.xadj, h->graph.adjncy, h->graph.adjwgt, tile_lo.p, tiles, tile_base.p, part,
                                              g->mapping.p, delta.p, g->adjncy.p, g->adjwgt.p);
    } else {
      k_sub_edges<false><<<grid, 256, 0, st>>>(m, h->graph.xadj, h->graph.adjncy, nullptr, tile_lo.p, tiles, tile_base.p, part,
                                               g->mapping.p, delta.p, g->adjncy.p, nullptr);
    }
    ++launches;
  }
  KMP_CUDA(cudaGetLastError());
  KMP_CUDA(call_clock_stop(h, st));
  KMP_CUDA(cudaStreamSynchronize(st));
  if (stats != nullptr) {
    stats->n = n;
    stats->k = k;
    stats->m = m;
    stats->m_internal = m_int;
    stats->kernel_launches = launches;
    stats->device_ms = call_clock_ms(h);
  }
  return KMP_OK;
}

int copy_back_impl(kmp_lp_handle *h, const kmp_subgraphs *g, uint32_t k_prime, uint32_t input_k,
                   const uint32_t *sub, bool host_sub, uint32_t *partition_out, int32_t *block_weights_out) {
  const cudaStream_t st = h->stream;
  const int dev = h->device;
  const uint32_t n = g->n, k = g->k;
  // k0: copy_subgraph_partitions's offsets (subgraph_extractor.cc:507-515)
  std::vector<uint32_t> k0(static_cast<size_t>(k) + 1, k_prime / k);
  if (k_prime == input_k) {
    for (uint32_t b = 0; b < k; ++b) {
      k0[b + 1] = sub_final_k(b, k, input_k);
    }
  }
  k0[0] = 0;
  uint64_t sum = 0;
  for (uint32_t b = 0; b <= k; ++b) {
    sum += k0[b];
    k0[b] = static_cast<uint32_t>(sum);
  }
  if (sum != k_prime) {
    return fail(KMP_ERR_INVALID, "the sub-block counts do not add up to k_prime (k must be a power of two when "
                                 "k_prime == input_k)");
  }
  PoolBuf<uint32_t> d_k0, d_sub, out; // scratch of this call
  PoolBuf<unsigned long long> bad;
  KMP_CUDA(d_k0.alloc(k0.size(), st, dev));
  KMP_CUDA(cudaMemcpyAsync(d_k0.p, k0.data(), k0.size() * 4, cudaMemcpyHostToDevice, st));
  if (host_sub) {
    KMP_CUDA(d_sub.alloc(n, st, dev));
    KMP_CUDA(cudaMemcpyAsync(d_sub.p, sub, static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, st));
    sub = d_sub.p;
  }
  KMP_CUDA(out.alloc(n, st, dev));
  KMP_CUDA(bad.alloc(1, st, dev));
  KMP_CUDA(cudaMemsetAsync(bad.p, 0, 8, st));
  if (n > 0) {
    k_sub_copy_back<<<capped(h, grid_for(n, 256)), 256, 0, st>>>(n, g->blk.p, g->block_nodes.p, d_k0.p, sub, out.p,
                                                                 bad.p);
  }
  KMP_CUDA(cudaGetLastError());
  unsigned long long nbad = 0;
  KMP_CUDA(cudaMemcpyAsync(&nbad, bad.p, sizeof(nbad), cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaStreamSynchronize(st));
  if (nbad != 0) {
    return fail(KMP_ERR_INVALID, "a sub-partition label is >= its block's sub-block count");
  }
  // ---- the k'-way partition becomes h's labels and block weights ---------------------------------------------
  KMP_CUDA(h->lp.label.ensure(n));
  KMP_CUDA(h->lp.weight.ensure(k_prime));
  KMP_CUDA(cudaMemcpyAsync(h->lp.label.p, out.p, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToDevice, st));
  h->lp.labels_valid = true;
  KMP_CUDA(cudaMemsetAsync(h->lp.weight.p, 0, static_cast<size_t>(k_prime) * 4, st));
  KMP_CUDA(cudaMemsetAsync(bad.p, 0, 8, st));
  if (n > 0) {
    bal_block_weights<<<capped(h, grid_for(n, 256)), 256, 0, st>>>(n, k_prime, h->graph.vwgt, h->lp.label.p, h->lp.weight.p,
                                                                   bad.p);
  }
  KMP_CUDA(cudaGetLastError());
  if (partition_out != nullptr && n > 0) {
    KMP_CUDA(cudaMemcpyAsync(partition_out, h->lp.label.p, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost, st));
  }
  if (block_weights_out != nullptr) {
    KMP_CUDA(cudaMemcpyAsync(block_weights_out, h->lp.weight.p, static_cast<size_t>(k_prime) * 4, cudaMemcpyDeviceToHost,
                             st));
  }
  KMP_CUDA(cudaStreamSynchronize(st));
  return KMP_OK;
}

int copy_back_checked(kmp_lp_handle *h, const kmp_subgraphs *g, uint32_t k_prime, uint32_t input_k,
                      const uint32_t *sub, bool host_sub, uint32_t *partition_out, int32_t *block_weights_out) {
  if (h == nullptr || g == nullptr || (sub == nullptr && g->n > 0)) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  if (!host_sub && (reinterpret_cast<uintptr_t>(sub) & 3u) != 0) {
    return fail(KMP_ERR_INVALID, "device sub-partitions must be 4-byte aligned");
  }
  if (h->step.open) {
    return fail(KMP_ERR_INVALID, "the handle is inside a stepping call");
  }
  if (g->source != h || !h->graph.present || h->graph.epoch != g->graph_epoch) {
    return fail(KMP_ERR_INVALID, "the handle holds another graph than the one the subgraphs were extracted from");
  }
  if (k_prime < g->k) {
    return fail(KMP_ERR_INVALID, "k_prime must be at least k");
  }
  if (k_prime != input_k && k_prime % g->k != 0) {
    return fail(KMP_ERR_INVALID, "k_prime must be a multiple of k unless it is input_k");
  }
  KMP_CUDA(cudaSetDevice(h->device));
  return copy_back_impl(h, g, k_prime, input_k, sub, host_sub, partition_out, block_weights_out);
}

} // namespace

extern "C" {

int kmp_extract_subgraphs(kmp_lp_handle *h, uint32_t k, const uint32_t *partition, kmp_subgraphs **out,
                          kmp_subgraph_stats *stats) {
  if (h == nullptr || out == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  if (!h->graph.present) {
    return fail(KMP_ERR_INVALID, "no graph set");
  }
  if (h->step.open) {
    return fail(KMP_ERR_INVALID, "the handle is inside a stepping call");
  }
  if (k == 0) {
    return fail(KMP_ERR_INVALID, "k must be at least 1");
  }
  if (static_cast<uint64_t>(h->graph.n) + k >= (1ull << 32)) {
    return fail(KMP_ERR_UNSUPPORTED, "n + k must be below 2^32");
  }
  if (partition == nullptr) {
    const int rc = refuse_without_labels(h);
    if (rc != KMP_OK) {
      return rc;
    }
  }
  KMP_CUDA(cudaSetDevice(h->device));
  if (stats != nullptr) {
    std::memset(stats, 0, sizeof(*stats));
  }
  KMP_CUDA(call_clock_start(h, h->stream));
  if (partition != nullptr) { // loaded as the handle's labels, as load_partition does
    KMP_CUDA(h->lp.label.ensure(h->graph.n));
    KMP_CUDA(cudaMemcpyAsync(h->lp.label.p, partition, static_cast<size_t>(h->graph.n) * 4, cudaMemcpyHostToDevice, h->stream));
    h->lp.labels_valid = true;
  }
  return make_result(h, out, [&](kmp_subgraphs *g) { return extract_impl(h, k, g, stats); });
}

uint32_t kmp_subgraphs_k(const kmp_subgraphs *g) { return g != nullptr ? g->k : 0; }
uint32_t kmp_subgraphs_n(const kmp_subgraphs *g) { return g != nullptr ? g->n : 0; }
uint32_t kmp_subgraphs_m(const kmp_subgraphs *g) { return g != nullptr ? g->m : 0; }

int kmp_subgraphs_offsets(const kmp_subgraphs *g, uint32_t *node_off, uint32_t *edge_off) {
  if (g == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  KMP_CUDA(cudaSetDevice(g->device));
  KMP_CUDA(copy_out(node_off, g->node_off, static_cast<size_t>(g->k) + 1));
  KMP_CUDA(copy_out(edge_off, g->edge_off, static_cast<size_t>(g->k) + 1));
  return KMP_OK;
}

int kmp_subgraphs_download(const kmp_subgraphs *g, uint32_t *xadj, uint32_t *adjncy, int32_t *vwgt, int32_t *adjwgt,
                           uint32_t *mapping, uint32_t *block_nodes) {
  if (g == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  KMP_CUDA(cudaSetDevice(g->device));
  KMP_CUDA(copy_out(xadj, g->xadj, static_cast<size_t>(g->n) + g->k));
  KMP_CUDA(copy_out(adjncy, g->adjncy, g->m));
  KMP_CUDA(copy_out(vwgt, g->vwgt, g->n));
  KMP_CUDA(copy_out(adjwgt, g->adjwgt, g->m));
  KMP_CUDA(copy_out(mapping, g->mapping, g->n));
  KMP_CUDA(copy_out(block_nodes, g->block_nodes, g->n));
  return KMP_OK;
}

int kmp_subgraphs_device_arrays(const kmp_subgraphs *g, const uint32_t **d_xadj, const uint32_t **d_adjncy,
                                const int32_t **d_vwgt, const int32_t **d_adjwgt, const uint32_t **d_mapping,
                                const uint32_t **d_block_nodes, const uint32_t **d_node_off,
                                const uint32_t **d_edge_off) {
  if (g == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  hand_out(d_xadj, g->xadj);
  hand_out(d_adjncy, g->adjncy);
  hand_out(d_vwgt, g->vwgt);
  hand_out(d_adjwgt, g->adjwgt);
  hand_out(d_mapping, g->mapping);
  hand_out(d_block_nodes, g->block_nodes);
  hand_out(d_node_off, g->node_off);
  hand_out(d_edge_off, g->edge_off);
  return KMP_OK;
}

int kmp_subgraphs_copy_partitions(kmp_lp_handle *h, const kmp_subgraphs *g, uint32_t k_prime, uint32_t input_k,
                                  const uint32_t *sub_partitions, uint32_t *partition_out,
                                  int32_t *block_weights_out) {
  return copy_back_checked(h, g, k_prime, input_k, sub_partitions, true, partition_out, block_weights_out);
}

int kmp_subgraphs_copy_partitions_device(kmp_lp_handle *h, const kmp_subgraphs *g, uint32_t k_prime,
                                         uint32_t input_k, const uint32_t *d_sub_partitions,
                                         uint32_t *partition_out, int32_t *block_weights_out) {
  return copy_back_checked(h, g, k_prime, input_k, d_sub_partitions, false, partition_out, block_weights_out);
}

void kmp_subgraphs_destroy(kmp_subgraphs *g) {
  if (g == nullptr) {
    return;
  }
  cudaSetDevice(g->device); // the arrays free themselves on this device's pool
  delete g;
}

} // extern "C"
