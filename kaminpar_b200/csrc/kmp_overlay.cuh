// kaminpar_b200: overlay of clusterings on the device + its C ABI (include/kaminpar_b200_contraction.h).
// Included at the end of kmp_lp.cu after kmp_contract.cuh: it reuses the contraction's leader flags (k_flag_leaders),
// its scratch and the stream of the kmp_lp_handle whose graph the clusterings belong to.
//
// What it restates (DESIGN.md §14): OverlayClusterCoarsener::coarsen (coarsening/overlay_cluster_coarsener.cc:34-80)
// and overlay (:82-151) with fill_leader_mapping / compute_mapping / fill_cluster_buckets
// (coarsening/contraction/cluster_contraction_preprocessing.cc). Let ra(x) be the rank of x among the distinct values
// of a and index(c) the number of vertices u with ra(a[u]) < c. The reference's overlay is
//   out[u] = index(ra(a[u])) + |{distinct b[v] : a[v] == a[u], b[v] < b[u]}|,
// independent of thread order (its sort by b only permutes equal keys). One pairwise overlay:
//   1. leader flags of a -> inclusive scan -> ra(a[u]) = rank[a[u]] - 1, c_a = rank[n - 1]   (as in the contraction)
//   2. key[u] = (ra(a[u]) << ceil(log2 n)) | b[u], value u; a label >= n of either input is refused
//   3. LSD radix sort of the pairs over exactly ceil(log2 n) + ceil(log2 c_a) key bits (CUB, like §9's sort)
//   4. pair heads (first of equal keys) and, at the first key of each cluster c of a, seg[c] = its sorted position
//      (= index(c)); inclusive scan of the pair heads -> P
//   5. out[value[i]] = seg[c] + P[i] - P[seg[c]]
// One host wait per pair (after step 2: c_a sizes the sort, and a bad label stops the call before any output is
// written). The 2^L clusterings are reduced in the reference's tree order (:61-67): for level = L .. 1, h = 2^(level-1),
// C[p] = overlay(C[p], C[h + p]) for p < h; every overlay but the last writes in place over C[p] (its inputs are
// consumed by step 2, before step 5 writes), the last one writes the handle's labels.
#pragma once

namespace {

// key[u] = (ra(a[u]) << nb) | b[u], value u (step 2); a label >= n of either input sets *bad
__global__ void k_overlay_keys(uint32_t n, const uint32_t *__restrict__ a, const uint32_t *__restrict__ b,
                               const uint32_t *__restrict__ rank, uint32_t nb, unsigned long long *__restrict__ keys,
                               uint32_t *__restrict__ vals, uint32_t *bad) {
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += gridDim.x * blockDim.x) {
    const uint32_t ca = a[u], cb = b[u];
    unsigned long long key = 0;
    if (ca < n && cb < n) {
      key = (static_cast<unsigned long long>(rank[ca] - 1) << nb) | cb;
    } else {
      *bad = 1;
    }
    keys[u] = key;
    vals[u] = u;
  }
}

// over the sorted keys: head[i] = first of its equal keys; seg[c] = i at the first key of cluster c = key >> nb
__global__ void k_overlay_heads(uint32_t n, const unsigned long long *__restrict__ keys, uint32_t nb,
                                uint32_t *__restrict__ head, uint32_t *__restrict__ seg) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned long long k = keys[i];
    const bool first = i == 0;
    const unsigned long long prev = first ? 0ull : keys[i - 1];
    head[i] = first || k != prev;
    if (first || (k >> nb) != (prev >> nb)) {
      seg[k >> nb] = i;
    }
  }
}

// out[u] = index(c) + (distinct b of cluster c below b[u]), with P the inclusive scan of the pair heads
__global__ void k_overlay_scatter(uint32_t n, const unsigned long long *__restrict__ keys,
                                  const uint32_t *__restrict__ vals, const uint32_t *__restrict__ P,
                                  const uint32_t *__restrict__ seg, uint32_t nb, uint32_t *__restrict__ out) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t s = seg[keys[i] >> nb];
    out[vals[i]] = s + P[i] - P[s];
  }
}

struct OverlayCounts {
  uint32_t launches = 0, sort_bits = 0, num_clusters = 0;
};

// leader flags + inclusive scan of labels (n >= 1) into h->ops.ct_flags / h->ops.ct_rank; then one wait for the number of
// distinct labels and the out-of-range flag. `then` may enqueue more work before the wait (it sees the ranks).
template <typename Then> int overlay_ranks(kmp_lp_handle *h, const uint32_t *labels, uint32_t *distinct, Then then) {
  const uint32_t n = h->graph.n;
  cudaStream_t st = h->stream;
  DevBuf<uint32_t> &flags = h->ops.ct_flags, &rank = h->ops.ct_rank;
  KMP_CUDA(flags.ensure(static_cast<size_t>(n) + 1)); // flags[n]: out-of-range marker
  KMP_CUDA(rank.ensure(n));
  KMP_CUDA(cudaMemsetAsync(flags.p, 0, (static_cast<size_t>(n) + 1) * 4, st));
  k_flag_leaders<<<capped(h, grid_for(n, 256)), 256, 0, st>>>(n, labels, flags.p, flags.p + n);
  KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
    return cub::DeviceScan::InclusiveSum(tmp, bytes, flags.p, rank.p, static_cast<int>(n), st);
  }));
  int rc = then(rank.p, flags.p + n);
  if (rc != KMP_OK) {
    return rc;
  }
  uint32_t host2[2] = {0, 0};
  KMP_CUDA(cudaMemcpyAsync(&host2[0], rank.p + (n - 1), 4, cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaMemcpyAsync(&host2[1], flags.p + n, 4, cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaStreamSynchronize(st));
  if (host2[1] != 0) {
    return fail(KMP_ERR_INVALID, "clustering holds an id >= n");
  }
  *distinct = host2[0];
  return KMP_OK;
}

// out = overlay(a, b) on the handle's graph (n >= 1); out may alias a or b. Leaves P in h->ops.ct_flags.
int overlay_pair(kmp_lp_handle *h, const uint32_t *a, const uint32_t *b, uint32_t *out, OverlayCounts *cnt) {
  const uint32_t n = h->graph.n;
  cudaStream_t st = h->stream;
  OverlayState &ov = h->ops.ov;
  DevBuf<unsigned long long> &keys_a = h->ops.pairs_a, &keys_b = h->ops.pairs_b;
  KMP_CUDA(keys_a.ensure(n));
  KMP_CUDA(keys_b.ensure(n));
  KMP_CUDA(ov.vals_a.ensure(n));
  KMP_CUDA(ov.vals_b.ensure(n));
  const uint32_t nb = ceil_log2_u32(n);
  uint32_t c_a = 0;
  int rc = overlay_ranks(h, a, &c_a, [&](const uint32_t *rank, uint32_t *bad) -> int {
    k_overlay_keys<<<capped(h, grid_for(n, 256)), 256, 0, st>>>(n, a, b, rank, nb, keys_a.p, ov.vals_a.p, bad);
    KMP_CUDA(cudaGetLastError());
    return KMP_OK;
  });
  cnt->launches += 2;
  if (rc != KMP_OK) {
    return rc;
  }
  // ---- 3. sort the (key, vertex) pairs -----------------------------------------------------------------------------
  const uint32_t bits = nb + ceil_log2_u32(c_a);
  cnt->sort_bits = std::max(cnt->sort_bits, bits);
  cub::DoubleBuffer<unsigned long long> dk(keys_a.p, keys_b.p);
  cub::DoubleBuffer<uint32_t> dv(ov.vals_a.p, ov.vals_b.p);
  if (bits > 0) { // bits == 0 only for n == 1: one pair is sorted
    KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
      return cub::DeviceRadixSort::SortPairs(tmp, bytes, dk, dv, static_cast<int>(n), 0, static_cast<int>(bits), st);
    }));
  }
  // ---- 4. heads + scan; 5. scatter. The leader flags and ranks are dead: P reuses the flags, seg the ranks ------------
  uint32_t *P = h->ops.ct_flags.p, *seg = h->ops.ct_rank.p;
  k_overlay_heads<<<capped(h, grid_for(n, 256)), 256, 0, st>>>(n, dk.Current(), nb, P, seg);
  KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
    return cub::DeviceScan::InclusiveSum(tmp, bytes, P, P, static_cast<int>(n), st);
  }));
  k_overlay_scatter<<<capped(h, grid_for(n, 256)), 256, 0, st>>>(n, dk.Current(), dv.Current(), P, seg, nb, out);
  cnt->launches += 2; // + the sort and the scans inside CUB
  KMP_CUDA(cudaGetLastError());
  return KMP_OK;
}

// Reduces the first `count` (a power of two) stashed clusterings in the reference's tree order into dst (n >= 1).
// count == 1 checks and copies C[0].
int overlay_tree(kmp_lp_handle *h, uint32_t count, uint32_t *dst, OverlayCounts *cnt) {
  const uint32_t n = h->graph.n;
  cudaStream_t st = h->stream;
  std::vector<PoolBuf<uint32_t>> &c = h->ops.ov.stash;
  if (count == 1) {
    int rc = overlay_ranks(h, c[0].p, &cnt->num_clusters, [](const uint32_t *, uint32_t *) { return KMP_OK; });
    cnt->launches += 1;
    if (rc != KMP_OK) {
      return rc;
    }
    KMP_CUDA(cudaMemcpyAsync(dst, c[0].p, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToDevice, st));
    KMP_CUDA(cudaStreamSynchronize(st));
    return KMP_OK;
  }
  for (uint32_t half = count / 2; half >= 1; half /= 2) { // overlay_cluster_coarsener.cc:61-67
    for (uint32_t p = 0; p < half; ++p) {
      const int rc = overlay_pair(h, c[p].p, c[half + p].p, half == 1 ? dst : c[p].p, cnt);
      if (rc != KMP_OK) {
        return rc;
      }
    }
  }
  KMP_CUDA(cudaMemcpyAsync(&cnt->num_clusters, h->ops.ct_flags.p + (n - 1), 4, cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaStreamSynchronize(st));
  return KMP_OK;
}

// the stash holds at least `count` blocks of n labels
int overlay_stash(kmp_lp_handle *h, uint32_t count) {
  std::vector<PoolBuf<uint32_t>> &c = h->ops.ov.stash;
  if (c.size() < count) {
    c.resize(count);
  }
  for (uint32_t i = 0; i < count; ++i) {
    if (c[i].p == nullptr || c[i].cap < h->graph.n) {
      KMP_CUDA(c[i].alloc(h->graph.n, h->stream, h->device));
    }
  }
  return KMP_OK;
}

int overlay_checks(kmp_lp_handle *h) {
  if (h == nullptr) {
    return fail(KMP_ERR_INVALID, "null handle");
  }
  if (!h->graph.present) {
    return fail(KMP_ERR_INVALID, "no graph set");
  }
  return refuse_multi_gpu(h, "the overlay");
}

// reduce the stash's first `count` clusterings into the handle's labels; timing and stats
int overlay_finish(kmp_lp_handle *h, uint32_t count, uint32_t *clustering_out, kmp_overlay_stats *stats) {
  const uint32_t n = h->graph.n;
  cudaStream_t st = h->stream;
  OverlayCounts cnt;
  float ms = 0.f;
  if (n > 0) {
    KMP_CUDA(h->lp.label.ensure(n));
    KMP_CUDA(call_clock_start(h, st));
    const int rc = overlay_tree(h, count, h->lp.label.p, &cnt);
    if (rc != KMP_OK) {
      return rc;
    }
    KMP_CUDA(call_clock_stop(h, st));
    KMP_CUDA(cudaEventSynchronize(h->streams.ev_ct1));
    ms = call_clock_ms(h);
    if (clustering_out != nullptr) {
      KMP_CUDA(cudaMemcpyAsync(clustering_out, h->lp.label.p, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost, st));
      KMP_CUDA(cudaStreamSynchronize(st));
    }
  }
  h->lp.labels_valid = true;
  if (stats != nullptr) {
    stats->num_clusterings = count;
    stats->num_clusters = cnt.num_clusters;
    stats->sort_bits = cnt.sort_bits;
    stats->kernel_launches = cnt.launches;
    stats->overlay_device_ms = ms;
  }
  return KMP_OK;
}

} // namespace

extern "C" {

int kmp_lp_cluster_overlay(kmp_lp_handle *h, int num_levels, int32_t max_cluster_weight, uint32_t desired_num_clusters,
                           const uint32_t *communities, uint32_t *clustering_out, kmp_overlay_stats *stats) {
  int rc = overlay_checks(h);
  if (rc != KMP_OK) {
    return rc;
  }
  if (num_levels < 0 || num_levels > KMP_OVERLAY_MAX_LEVELS) {
    return fail(KMP_ERR_INVALID, "num_levels must lie in [0, KMP_OVERLAY_MAX_LEVELS]");
  }
  KMP_CUDA(cudaSetDevice(h->device));
  if (stats != nullptr) {
    std::memset(stats, 0, sizeof(*stats));
  }
  const uint32_t count = 1u << num_levels;
  float lp_ms = 0.f;
  if (num_levels == 0) { // exactly one clustering
    kmp_lp_stats ls{};
    rc = kmp_lp_cluster(h, max_cluster_weight, desired_num_clusters, communities, clustering_out, &ls);
    if (rc != KMP_OK) {
      return rc;
    }
    OverlayCounts cnt;
    if (h->graph.n > 0) {
      rc = overlay_ranks(h, h->lp.label.p, &cnt.num_clusters, [](const uint32_t *, uint32_t *) { return KMP_OK; });
      if (rc != KMP_OK) {
        return rc;
      }
      cnt.launches = 1;
    }
    if (stats != nullptr) {
      stats->num_clusterings = 1;
      stats->num_clusters = cnt.num_clusters;
      stats->kernel_launches = cnt.launches;
      stats->lp_device_ms = ls.device_ms;
    }
    return KMP_OK;
  }
  rc = overlay_stash(h, count);
  if (rc != KMP_OK) {
    return rc;
  }
  // compute_clustering_for_current_graph 2^L times on the same clusterer (:52-54): each call advances the call
  // counter (sync) or continues the random stream (seq_strict), so the clusterings differ
  for (uint32_t i = 0; i < count; ++i) {
    kmp_lp_stats ls{};
    rc = kmp_lp_cluster(h, max_cluster_weight, desired_num_clusters, communities, nullptr, &ls);
    if (rc != KMP_OK) {
      return rc;
    }
    lp_ms += ls.device_ms;
    if (h->graph.n > 0) {
      KMP_CUDA(cudaMemcpyAsync(h->ops.ov.stash[i].p, h->lp.label.p, static_cast<size_t>(h->graph.n) * 4,
                               cudaMemcpyDeviceToDevice, h->stream));
    }
  }
  h->lp.labels_valid = false; // until the overlay below replaces the last call's labels
  rc = overlay_finish(h, count, clustering_out, stats);
  if (stats != nullptr) {
    stats->lp_device_ms = lp_ms;
  }
  return rc;
}

int kmp_overlay_clusterings(kmp_lp_handle *h, uint32_t count, const uint32_t *clusterings, uint32_t *out,
                            kmp_overlay_stats *stats) {
  int rc = overlay_checks(h);
  if (rc != KMP_OK) {
    return rc;
  }
  if (count == 0 || (count & (count - 1)) != 0 || count > (1u << KMP_OVERLAY_MAX_LEVELS)) {
    return fail(KMP_ERR_INVALID, "count must be a power of two in [1, 2^KMP_OVERLAY_MAX_LEVELS]");
  }
  if (clusterings == nullptr && h->graph.n > 0) {
    return fail(KMP_ERR_INVALID, "null clusterings");
  }
  KMP_CUDA(cudaSetDevice(h->device));
  if (stats != nullptr) {
    std::memset(stats, 0, sizeof(*stats));
  }
  const uint32_t n = h->graph.n;
  if (n > 0) {
    rc = overlay_stash(h, count);
    if (rc != KMP_OK) {
      return rc;
    }
    for (uint32_t i = 0; i < count; ++i) {
      KMP_CUDA(cudaMemcpyAsync(h->ops.ov.stash[i].p, clusterings + static_cast<size_t>(i) * n, static_cast<size_t>(n) * 4,
                               cudaMemcpyHostToDevice, h->stream));
    }
  }
  // a refused call leaves the labels as they were: the tree checks every input before the last pair writes them
  return overlay_finish(h, count, out, stats);
}

} // extern "C"
