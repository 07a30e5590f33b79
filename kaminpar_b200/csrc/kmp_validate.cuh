// kaminpar_b200: graph validation on the device + its C ABI (include/kaminpar_b200_validate.h, DESIGN.md §17).
// Included at the end of kmp_lp.cu after kmp_subgraph.cuh: the edge passes find the vertex that owns an edge with the
// contraction's tile owners (k_tile_owners, owner_of_edge) and stage a tile's xadj with sub_stage; scratch is PoolBuf.
//
// What it restates (see the header): debug::validate_graph (csr_graph.cc:266-356) and the multi-edge check of
// validate_undirected_graph (graph_validator.cc:33-85), without the reference's per-edge scan of the neighbour's row.
//   1. k_val_xadj: the shape flags, the first decreasing u and their count, and the count of targets >= n. One host
//      wait: nothing below indexes a row unless xadj is well formed.
//   2. a STABLE segmented sort of each row's (target, position): the first of a run of equal targets is the first
//      occurrence p of that target in input order.
//   3. only when a target >= n exists: q[v] = the first such position in v's row (atomicMin on the tile owners).
//   4. k_val_edges over edge tiles in input order: range, self-loop, a binary search of u in v's sorted row for p, the
//      q < p test and the weight test; a violation takes one 64-bit atomicMin of (e << 8) | kind and one counter
//      atomic. A valid graph issues no atomics.
//   5. k_val_dups over the sorted rows: equal neighbours next to each other, counted, and the min of (u, position).
//   6. k_val_detail gathers the first violation's fields; one copy of the control block to the host.
#pragma once

namespace {

// device control block of one validation; zeroed except for the min-reduced fields
struct ValCtl {
  unsigned long long first;     // min over the edge violations of (e << 8) | kind
  unsigned long long dup_first; // min over the duplicates of (u << 32) | position
  uint32_t first_dec;           // smallest u with xadj[u] > xadj[u + 1]
  uint32_t shape;               // bit 0: xadj[0] != 0, bit 1: xadj[n] != m
  uint32_t x0, xn;              // xadj[0], xadj[n]
  uint32_t bad_targets;         // edges with a target >= n
  uint32_t duplicates;
  uint32_t count[KMP_GRAPH_NUM_KINDS];
  uint32_t u, e, v, e_rev, v_rev; // the first violation (k_val_detail)
  int32_t w, w_rev;
};
constexpr uint32_t kValNone = 0xFFFFFFFFu;

__global__ void __launch_bounds__(256) k_val_xadj(uint32_t n, uint32_t m, const uint32_t *__restrict__ xadj,
                                                  const uint32_t *__restrict__ adjncy, ValCtl *ctl) {
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
  if (tid == 0) {
    ctl->x0 = xadj[0];
    ctl->xn = xadj[n];
    ctl->shape = (xadj[0] != 0 ? 1u : 0u) | (xadj[n] != m ? 2u : 0u);
  }
  for (uint32_t u = tid; u < n; u += stride) { // n, m < 2^31: u + stride does not wrap
    if (xadj[u] > xadj[u + 1]) {
      atomicMin(&ctl->first_dec, u);
      atomicAdd(&ctl->count[KMP_GRAPH_XADJ_DECREASING], 1u);
    }
  }
  for (uint32_t e = tid; e < m; e += stride) {
    if (adjncy[e] >= n) {
      atomicAdd(&ctl->bad_targets, 1u);
    }
  }
}

__global__ void k_val_iota(uint32_t m, uint32_t *out) {
  for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < m; e += gridDim.x * blockDim.x) {
    out[e] = e;
  }
}

// q[u] = first position in u's row with a target >= n (q preset to kValNone)
__global__ void __launch_bounds__(256) k_val_first_bad(uint32_t n, uint32_t m, const uint32_t *__restrict__ xadj,
                                                       const uint32_t *__restrict__ adjncy,
                                                       const uint32_t *__restrict__ tile_lo, uint32_t tiles,
                                                       uint32_t *__restrict__ q) {
  for (uint32_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    const uint32_t e0 = t * kTileEdges;
    const uint32_t e1 = e0 + kTileEdges < m ? e0 + kTileEdges : m;
    for (uint32_t e = e0 + threadIdx.x; e < e1; e += blockDim.x) {
      if (adjncy[e] >= n) {
        atomicMin(&q[owner_of_edge(xadj, tile_lo[t], tile_lo[t + 1], e)], e);
      }
    }
  }
}

// the first sorted index in [lo, hi) whose key is >= u
__device__ __forceinline__ uint32_t val_lower_bound(const uint32_t *__restrict__ keys, uint32_t lo, uint32_t hi,
                                                    uint32_t u) {
  while (lo < hi) {
    const uint32_t mid = lo + (hi - lo) / 2;
    if (keys[mid] < u) {
      lo = mid + 1;
    } else {
      hi = mid;
    }
  }
  return lo;
}

// p: the first position of u in v's row (v < n), kValNone if u is absent
__device__ __forceinline__ uint32_t val_first_of(const uint32_t *__restrict__ xadj, const uint32_t *__restrict__ keys,
                                                 const uint32_t *__restrict__ pos, uint32_t v, uint32_t u) {
  const uint32_t end = xadj[v + 1];
  const uint32_t i = val_lower_bound(keys, xadj[v], end, u);
  return i < end && keys[i] == u ? pos[i] : kValNone;
}

// the first kind of every edge (q == nullptr: no target >= n anywhere)
template <bool EW>
__global__ void __launch_bounds__(256) k_val_edges(uint32_t n, uint32_t m, const uint32_t *__restrict__ xadj,
                                                   const uint32_t *__restrict__ adjncy,
                                                   const int32_t *__restrict__ adjwgt,
                                                   const uint32_t *__restrict__ tile_lo, uint32_t tiles,
                                                   const uint32_t *__restrict__ keys, const uint32_t *__restrict__ pos,
                                                   const uint32_t *__restrict__ q, ValCtl *ctl) {
  __shared__ uint32_t s_x[kTileVerts + 1];
  for (uint32_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    const uint32_t e0 = t * kTileEdges;
    const uint32_t e1 = e0 + kTileEdges < m ? e0 + kTileEdges : m;
    const uint32_t u_lo = tile_lo[t], u_hi = tile_lo[t + 1];
    __syncthreads(); // the previous tile is done with s_x
    const bool staged = sub_stage(xadj, u_lo, u_hi, s_x);
    __syncthreads();
    for (uint32_t e = e0 + threadIdx.x; e < e1; e += blockDim.x) {
      const uint32_t u = staged ? u_lo + owner_of_edge(s_x, 0, u_hi - u_lo, e) : owner_of_edge(xadj, u_lo, u_hi, e);
      const uint32_t v = adjncy[e];
      uint32_t kind = KMP_GRAPH_VALID;
      if (v >= n) {
        kind = KMP_GRAPH_NEIGHBOR_OUT_OF_GRAPH;
      } else if (v == u) {
        kind = KMP_GRAPH_SELF_LOOP;
      } else {
        const uint32_t p = val_first_of(xadj, keys, pos, v, u);
        const uint32_t qv = q != nullptr ? q[v] : kValNone;
        if (qv < p) { // also when u is absent (p == kValNone) and v's row holds a target >= n
          kind = KMP_GRAPH_NEIGHBOR_OF_NEIGHBOR_OUT_OF_GRAPH;
        } else if (p == kValNone) {
          kind = KMP_GRAPH_MISSING_REVERSE;
        } else if (EW && adjwgt[e] != adjwgt[p]) {
          kind = KMP_GRAPH_WEIGHT_MISMATCH;
        }
      }
      if (kind != KMP_GRAPH_VALID) {
        atomicMin(&ctl->first, (static_cast<unsigned long long>(e) << 8) | kind);
        atomicAdd(&ctl->count[kind], 1u);
      }
    }
  }
}

// duplicates: sorted index i of row u with keys[i] == keys[i - 1] (i > xadj[u]) is the later occurrence pos[i]
__global__ void __launch_bounds__(256) k_val_dups(uint32_t m, const uint32_t *__restrict__ xadj,
                                                  const uint32_t *__restrict__ tile_lo, uint32_t tiles,
                                                  const uint32_t *__restrict__ keys, const uint32_t *__restrict__ pos,
                                                  ValCtl *ctl) {
  __shared__ uint32_t s_x[kTileVerts + 1];
  for (uint32_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    const uint32_t e0 = t * kTileEdges;
    const uint32_t e1 = e0 + kTileEdges < m ? e0 + kTileEdges : m;
    const uint32_t u_lo = tile_lo[t], u_hi = tile_lo[t + 1];
    __syncthreads();
    const bool staged = sub_stage(xadj, u_lo, u_hi, s_x);
    __syncthreads();
    uint32_t cnt = 0;
    unsigned long long first = ~0ull;
    for (uint32_t i = e0 + threadIdx.x; i < e1; i += blockDim.x) {
      uint32_t u, begin;
      if (staged) {
        const uint32_t j = owner_of_edge(s_x, 0, u_hi - u_lo, i);
        u = u_lo + j;
        begin = s_x[j];
      } else {
        u = owner_of_edge(xadj, u_lo, u_hi, i);
        begin = xadj[u];
      }
      if (i > begin && keys[i] == keys[i - 1]) {
        ++cnt;
        first = min(first, (static_cast<unsigned long long>(u) << 32) | pos[i]);
      }
    }
    cnt = __reduce_add_sync(kFull, cnt);
    for (int o = 16; o > 0; o >>= 1) {
      first = min(first, __shfl_xor_sync(kFull, first, o));
    }
    if ((threadIdx.x & 31) == 0 && cnt != 0) {
      atomicAdd(&ctl->duplicates, cnt);
      atomicMin(&ctl->dup_first, first);
    }
  }
}

// the fields of the first edge violation (one thread)
__global__ void k_val_detail(uint32_t n, const uint32_t *__restrict__ xadj, const uint32_t *__restrict__ adjncy,
                             const int32_t *__restrict__ adjwgt, const uint32_t *__restrict__ keys,
                             const uint32_t *__restrict__ pos, const uint32_t *__restrict__ q, ValCtl *ctl) {
  if (blockIdx.x != 0 || threadIdx.x != 0 || ctl->first == ~0ull) {
    return;
  }
  const uint32_t e = static_cast<uint32_t>(ctl->first >> 8);
  const uint32_t kind = static_cast<uint32_t>(ctl->first & 0xFFu);
  const uint32_t u = owner_of_edge(xadj, 0, n, e); // xadj[n] = m > e: u < n
  const uint32_t v = adjncy[e];
  ctl->u = u;
  ctl->e = e;
  ctl->v = v;
  if (kind == KMP_GRAPH_NEIGHBOR_OF_NEIGHBOR_OUT_OF_GRAPH) { // v < n, and q[v] exists
    ctl->e_rev = q[v];
    ctl->v_rev = adjncy[q[v]];
  } else if (kind == KMP_GRAPH_WEIGHT_MISMATCH) { // v < n, p exists, edge weights present
    const uint32_t p = val_first_of(xadj, keys, pos, v, u);
    ctl->e_rev = p;
    ctl->v_rev = u;
    ctl->w = adjwgt[e];
    ctl->w_rev = adjwgt[p];
  }
}

int validate_impl(kmp_lp_handle *h, uint32_t n, uint32_t m, const uint32_t *xadj, const uint32_t *adjncy,
                  const int32_t *adjwgt, kmp_graph_report *out) {
  const cudaStream_t st = h->stream;
  const int dev = h->device;
  const uint32_t tiles = (m + kTileEdges - 1) / kTileEdges;
  // ---- every allocation before the first kernel ------------------------------------------------------------
  PoolBuf<ValCtl> ctl;
  PoolBuf<uint32_t> keys, iota, pos, owners, q;
  KMP_CUDA(ctl.alloc(1, st, dev));
  if (m > 0) {
    KMP_CUDA(keys.alloc(m, st, dev));
    KMP_CUDA(iota.alloc(m, st, dev));
    KMP_CUDA(pos.alloc(m, st, dev));
    KMP_CUDA(owners.alloc(static_cast<size_t>(tiles) + 1, st, dev));
    KMP_CUDA(q.alloc(n, st, dev));
  }
  auto sort = [&](void *tmp, size_t &bytes) {
    return cub::DeviceSegmentedSort::StableSortPairs(tmp, bytes, adjncy, keys.p, iota.p, pos.p, static_cast<int>(m),
                                                     static_cast<int>(n), xadj, xadj + 1, st);
  };
  if (m > 0) { // CUB's temporary, grown now (the query reads no data) so that the sort below allocates nothing
    size_t bytes = 0;
    KMP_CUDA(sort(nullptr, bytes));
    KMP_CUDA(h->commit.cub_tmp.ensure(bytes));
  }
  KMP_CUDA(call_clock_start(h, st));
  ValCtl init{};
  init.first = ~0ull;
  init.dup_first = ~0ull;
  init.first_dec = kValNone;
  KMP_CUDA(cudaMemcpyAsync(ctl.p, &init, sizeof(init), cudaMemcpyHostToDevice, st));
  // ---- 1. shape, monotonicity, targets >= n ------------------------------------------------------------------
  k_val_xadj<<<capped(h, grid_for(std::max(n, m), 256)), 256, 0, st>>>(n, m, xadj, adjncy, ctl.p);
  ValCtl c{};
  KMP_CUDA(cudaGetLastError());
  KMP_CUDA(cudaMemcpyAsync(&c, ctl.p, sizeof(c), cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaStreamSynchronize(st));
  const bool shape_ok = c.shape == 0 && c.first_dec == kValNone;
  if (shape_ok && m > 0) {
    // ---- 2. stable segmented sort of (target, position) per row -------------------------------------------
    k_val_iota<<<capped(h, grid_for(m, 256)), 256, 0, st>>>(m, iota.p);
    KMP_CUDA(cub_call(h, sort));
    k_tile_owners<<<capped(h, grid_for(static_cast<uint64_t>(tiles) + 1, 256)), 256, 0, st>>>(n, m, xadj, tiles,
                                                                                              owners.p);
    // ---- 3. the first target >= n per row -----------------------------------------------------------------
    const uint32_t *qp = nullptr;
    if (c.bad_targets > 0) {
      KMP_CUDA(cudaMemsetAsync(q.p, 0xFF, static_cast<size_t>(n) * 4, st));
      k_val_first_bad<<<capped(h, std::min<uint32_t>(tiles, kSMs * 16)), 256, 0, st>>>(n, m, xadj, adjncy, owners.p,
                                                                                     tiles, q.p);
      qp = q.p;
    }
    // ---- 4. edge probe, 5. duplicates, 6. details -----------------------------------------------------------
    const uint32_t grid = capped(h, std::min<uint32_t>(tiles, kSMs * 16));
    if (adjwgt != nullptr) {
      k_val_edges<true><<<grid, 256, 0, st>>>(n, m, xadj, adjncy, adjwgt, owners.p, tiles, keys.p, pos.p, qp, ctl.p);
    } else {
      k_val_edges<false><<<grid, 256, 0, st>>>(n, m, xadj, adjncy, nullptr, owners.p, tiles, keys.p, pos.p, qp, ctl.p);
    }
    k_val_dups<<<grid, 256, 0, st>>>(m, xadj, owners.p, tiles, keys.p, pos.p, ctl.p);
    k_val_detail<<<capped(h, 1), 32, 0, st>>>(n, xadj, adjncy, adjwgt, keys.p, pos.p, qp, ctl.p);
    KMP_CUDA(cudaGetLastError());
    KMP_CUDA(cudaMemcpyAsync(&c, ctl.p, sizeof(c), cudaMemcpyDeviceToHost, st));
  }
  KMP_CUDA(call_clock_stop(h, st));
  KMP_CUDA(cudaStreamSynchronize(st));
  // ---- the report ---------------------------------------------------------------------------------------------
  kmp_graph_report r{};
  r.n = n;
  r.m = m;
  r.count[KMP_GRAPH_XADJ_START] = c.shape & 1u;
  r.count[KMP_GRAPH_XADJ_END] = (c.shape >> 1) & 1u;
  r.count[KMP_GRAPH_XADJ_DECREASING] = c.count[KMP_GRAPH_XADJ_DECREASING];
  if (c.shape & 1u) {
    r.kind = KMP_GRAPH_XADJ_START;
    r.e = c.x0;
  } else if (c.shape & 2u) {
    r.kind = KMP_GRAPH_XADJ_END;
    r.u = n;
    r.e = c.xn;
  } else if (c.first_dec != kValNone) {
    r.kind = KMP_GRAPH_XADJ_DECREASING;
    r.u = c.first_dec;
  } else {
    for (int k = KMP_GRAPH_NEIGHBOR_OUT_OF_GRAPH; k < KMP_GRAPH_NUM_KINDS; ++k) {
      r.count[k] = c.count[k];
    }
    r.duplicates = c.duplicates;
    if (c.duplicates > 0) {
      r.dup_u = static_cast<uint32_t>(c.dup_first >> 32);
      r.dup_e = static_cast<uint32_t>(c.dup_first);
    }
    if (c.first != ~0ull) {
      r.kind = static_cast<int32_t>(c.first & 0xFFu);
      r.u = c.u;
      r.e = c.e;
      r.v = c.v;
      r.e_rev = c.e_rev;
      r.v_rev = c.v_rev;
      r.w = c.w;
      r.w_rev = c.w_rev;
    }
  }
  r.valid = r.kind == KMP_GRAPH_VALID ? 1 : 0;
  r.device_ms = call_clock_ms(h);
  *out = r;
  return KMP_OK;
}

int validate_checked(kmp_lp_handle *h, uint32_t n, uint32_t m, const uint32_t *xadj, const uint32_t *adjncy,
                     const int32_t *adjwgt, bool host_input, kmp_graph_report *out) {
  if (h == nullptr || out == nullptr || xadj == nullptr || (m > 0 && adjncy == nullptr)) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  if (h->step.open) {
    return fail(KMP_ERR_INVALID, "the handle is inside a stepping call");
  }
  if (n > 0x7FFFFFFFu || m > 0x7FFFFFFFu) {
    return fail(KMP_ERR_UNSUPPORTED, "n and m must be below 2^31");
  }
  auto misaligned4 = [](const void *p) { return (reinterpret_cast<uintptr_t>(p) & 3u) != 0; };
  if (!host_input && (misaligned4(xadj) || misaligned4(adjncy) || misaligned4(adjwgt))) {
    return fail(KMP_ERR_INVALID, "device graph arrays must be 4-byte aligned");
  }
  KMP_CUDA(cudaSetDevice(h->device));
  PoolBuf<uint32_t> d_xadj, d_adj;
  PoolBuf<int32_t> d_ew;
  if (host_input) { // copies on the handle's stream, freed stream-ordered behind the kernels that read them
    const cudaStream_t st = h->stream;
    KMP_CUDA(upload(d_xadj, xadj, static_cast<size_t>(n) + 1, st, h->device));
    KMP_CUDA(upload(d_adj, adjncy, m, st, h->device));
    if (adjwgt != nullptr) {
      KMP_CUDA(upload(d_ew, adjwgt, m, st, h->device));
    }
    xadj = d_xadj.p;
    adjncy = d_adj.p;
    adjwgt = adjwgt != nullptr ? d_ew.p : nullptr;
  }
  return validate_impl(h, n, m, xadj, adjncy, adjwgt, out);
}

} // namespace

extern "C" {

int kmp_validate_graph(kmp_lp_handle *h, uint32_t n, uint32_t m, const uint32_t *xadj, const uint32_t *adjncy,
                       const int32_t *adjwgt, kmp_graph_report *out) {
  return validate_checked(h, n, m, xadj, adjncy, adjwgt, true, out);
}

int kmp_validate_graph_device(kmp_lp_handle *h, uint32_t n, uint32_t m, const uint32_t *d_xadj,
                              const uint32_t *d_adjncy, const int32_t *d_adjwgt, kmp_graph_report *out) {
  return validate_checked(h, n, m, d_xadj, d_adjncy, d_adjwgt, false, out);
}

int kmp_graph_report_message(const kmp_graph_report *r, char *buf, size_t size) {
  if (r == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  switch (r->kind) { // csr_graph.cc:276-350, word for word
  case KMP_GRAPH_XADJ_START:
    return format_report(buf, size, "xadj[0] is %u, not 0", r->e);
  case KMP_GRAPH_XADJ_END:
    return format_report(buf, size, "xadj[%u] is %u, not the number of edges %u", r->u, r->e, r->m);
  case KMP_GRAPH_XADJ_DECREASING:
    return format_report(buf, size, "Bad node array at position %u", r->u);
  case KMP_GRAPH_NEIGHBOR_OUT_OF_GRAPH:
    return format_report(buf, size, "Neighbor %u of %u is out-of-graph", r->v, r->u);
  case KMP_GRAPH_SELF_LOOP:
    return format_report(buf, size, "Self-loop at %u: %u --> %u", r->u, r->e, r->v);
  case KMP_GRAPH_NEIGHBOR_OF_NEIGHBOR_OUT_OF_GRAPH:
    return format_report(buf, size, "Neighbor %u of neighbor %u of %u is out-of-graph", r->v_rev, r->v, r->u);
  case KMP_GRAPH_MISSING_REVERSE:
    return format_report(buf, size, "Edge %u --> %u exists with edge %u, but the reverse edges does not exist", r->u,
                         r->v, r->e);
  case KMP_GRAPH_WEIGHT_MISMATCH:
    return format_report(buf, size, "Weight of edge %u (%d) differs from the weight of its reverse edge %u (%d)", r->e,
                         r->w, r->e_rev, r->w_rev);
  default:
    return format_report(buf, size, "%s", "");
  }
}

} // extern "C"
