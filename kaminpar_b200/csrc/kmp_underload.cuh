// kaminpar_b200: underload balancer on the device + its C ABI (include/kaminpar_b200_balancer.h).
// Included at the end of kmp_lp.cu after kmp_balance.cuh: it evaluates candidates with the overload balancer's
// degree tiers (bal_eval_thread / _warp / _cta, with a target mask) and commits through the refiner's cooperative
// ladder kernel with the minimum block weights (lp_commit.cuh commit_refine_fused).
//
// What it restates: UnderloadBalancer::refine (refinement/balancer/underload_balancer.cc:39-244) as synchronous
// rounds (DESIGN.md §12). One round:
//   1. block stats against the frozen weights: deficit[b] = max(0, min[b] - W[b]), the total underload, the
//      underloaded flags (the target mask); the vertices that may leave their block (block not underloaded,
//      W[b] - w(u) >= min[b]) are compacted in id order (one small read-back per round: total, count)
//   2. candidate evaluation by the overload balancer's tiers, targets restricted to underloaded blocks
//   3. the candidates with a target are compacted in id order (a second read-back: their count) and sorted by
//      (target, key desc); exclusive weight scan per target, selected iff the weight before a candidate is
//      < deficit[target]
//   4. the ladder commit of the LP refiner with one pass and the minimum weights: targets stay <= max, sources >= min
#pragma once

namespace kmp {

enum : uint32_t { SALT_UBAL_TIE = 8, SALT_UBAL_COMMIT = 9 };

// deficit[b], the total underload (ctrl[0]) and the underloaded flags (the allowed targets)
__global__ void ubal_block_stats(uint32_t k, const int32_t *weight, const int32_t *min_w, int32_t *deficit,
                                 uint8_t *tmask, unsigned long long *ctrl) {
  unsigned long long total = 0;
  for (uint32_t b = blockIdx.x * blockDim.x + threadIdx.x; b < k; b += gridDim.x * blockDim.x) {
    const int32_t d = max(0, min_w[b] - weight[b]);
    deficit[b] = d;
    tmask[b] = d > 0;
    total += static_cast<unsigned long long>(d);
  }
  for (int off = 16; off > 0; off >>= 1) {
    total += __shfl_xor_sync(kFull, total, off);
  }
  if ((threadIdx.x & 31) == 0 && total != 0) {
    atomicAdd(&ctrl[0], total);
  }
}
// movable from (underload_balancer.cc:241-244): the own block is not underloaded and stays at or above its minimum
__global__ void ubal_vertex_flags(uint32_t n, const uint32_t *label, const int32_t *vwgt, const int32_t *weight,
                                  const int32_t *min_w, const uint8_t *tmask, uint8_t *flag) {
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += gridDim.x * blockDim.x) {
    const uint32_t b = label[u];
    flag[u] = tmask[b] == 0 && weight[b] - (vwgt != nullptr ? vwgt[u] : 1) >= min_w[b];
  }
}
// candidate index i has a target (the evaluation wrote its own block otherwise)
struct UbalHasTarget {
  const uint32_t *cand, *label, *target;
  __device__ __forceinline__ bool operator()(uint32_t i) const { return target[i] != label[cand[i]]; }
};
// sort words of the candidates with a target: (target << 32 | desc key bits), value = candidate index
__global__ void ubal_sort_keys(uint32_t nt, const uint32_t *list, const uint32_t *target, const float *key,
                               unsigned long long *sort_key, uint32_t *sort_val) {
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < nt; j += gridDim.x * blockDim.x) {
    const uint32_t i = list[j];
    sort_key[j] = (static_cast<unsigned long long>(target[i]) << 32) | bal_desc_bits(key[i]);
    sort_val[j] = i;
  }
}
// selected iff the weight of the candidates before it in its target's segment is < deficit[target]
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
// T0 hook: a vertex that may not leave its block keeps it, with the key of "no target"
__global__ void ubal_keep_sources(uint32_t n, const uint8_t *flag, const uint32_t *label, const int32_t *vwgt,
                                  uint32_t *target, float *key) {
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < n; u += gridDim.x * blockDim.x) {
    if (flag[u] == 0) {
      target[u] = label[u];
      key[u] = bal_relative_gain(INT32_MIN, vwgt != nullptr ? vwgt[u] : 1);
    }
  }
}

} // namespace kmp

namespace {

using namespace kmp;

constexpr const char *kUbalName = "the underload balancer";

int ubal_ensure(kmp_lp_handle *h, uint32_t k, uint32_t nc) {
  const size_t kk = std::max<uint32_t>(k, 1);
  KMP_CUDA(h->ubal_deficit.ensure(kk));
  KMP_CUDA(h->ubal_tmask.ensure(kk));
  return bal_ensure(h, k, nc);
}

// Round start: deficit[], target mask, candidates; read back {total underload, #candidates} and the number of
// proposals of the previous round.
int ubal_round_begin(kmp_lp_handle *h, uint32_t k, unsigned long long *host_ctrl, uint32_t *host_proposals) {
  cudaStream_t st = h->stream;
  const uint32_t n = h->n;
  KMP_CUDA(cudaMemsetAsync(h->bal_ctrl.p, 0, 2 * sizeof(unsigned long long), st));
  ubal_block_stats<<<capped(h, grid_for(k, 256)), 256, 0, st>>>(k, h->weight.p, h->minw.p, h->ubal_deficit.p,
                                                                h->ubal_tmask.p, h->bal_ctrl.p);
  ubal_vertex_flags<<<capped(h, grid_for(n, 256)), 256, 0, st>>>(n, h->label.p, h->vwgt, h->weight.p, h->minw.p,
                                                                 h->ubal_tmask.p, h->bal_flag.p);
  int rc = bal_cub(h, [&](void *tmp, size_t &bytes) {
    return cub::DeviceSelect::Flagged(tmp, bytes, thrust::counting_iterator<uint32_t>(0), h->bal_flag.p, h->bal_cand.p,
                                      h->bal_ctrl.p + 1, static_cast<int>(n), st);
  });
  if (rc != KMP_OK) {
    return rc;
  }
  h->kernel_launches += 3;
  KMP_CUDA(cudaMemcpyAsync(host_ctrl, h->bal_ctrl.p, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaMemcpyAsync(host_proposals, h->bal_ctr32.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaStreamSynchronize(st));
  return KMP_OK;
}

// One round after its read-back: evaluate, compact the candidates with a target, select per target, commit (moves
// land in bal_ctr32[4 + r], proposals in bal_ctr32[0]).
int ubal_round(kmp_lp_handle *h, uint32_t k, uint32_t nc, uint32_t call, uint32_t r) {
  cudaStream_t st = h->stream;
  uint32_t *mover_count = h->bal_ctr32.p;
  KMP_CUDA(cudaMemsetAsync(mover_count, 0, sizeof(uint32_t), st));
  if (nc == 0) {
    return KMP_OK;
  }
  int rc = bal_evaluate(h, k, nc, sync_base(h->cfg.seed, call, r, SALT_UBAL_TIE), false, h->ubal_tmask.p);
  if (rc != KMP_OK) {
    return rc;
  }
  // Most candidates have no underloaded neighbour block (typically few blocks are underloaded): compacting them
  // away costs one select and a read-back, where sorting them into a zero-deficit segment would cost radix passes
  // over nearly every vertex.
  uint32_t *list = h->bal_lists.p; // free again after the evaluation
  rc = bal_cub(h, [&](void *tmp, size_t &bytes) {
    return cub::DeviceSelect::If(tmp, bytes, thrust::counting_iterator<uint32_t>(0), list, h->bal_ctrl.p + 5,
                                 static_cast<int>(nc), UbalHasTarget{h->bal_cand.p, h->label.p, h->bal_target.p}, st);
  });
  if (rc != KMP_OK) {
    return rc;
  }
  unsigned long long nt64 = 0;
  KMP_CUDA(cudaMemcpyAsync(&nt64, h->bal_ctrl.p + 5, sizeof(nt64), cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaStreamSynchronize(st));
  const uint32_t nt = static_cast<uint32_t>(nt64);
  if (nt == 0) {
    return KMP_OK;
  }
  ubal_sort_keys<<<capped(h, grid_for(nt, 256)), 256, 0, st>>>(nt, list, h->bal_target.p, h->bal_key.p, h->bal_sk_a.p,
                                                               h->bal_sv_a.p);
  uint32_t end_bit = 32;
  while (end_bit < 64 && (static_cast<uint64_t>(k - 1) >> (end_bit - 32)) != 0) {
    ++end_bit;
  }
  rc = bal_cub(h, [&](void *tmp, size_t &bytes) {
    return cub::DeviceRadixSort::SortPairs(tmp, bytes, h->bal_sk_a.p, h->bal_sk_b.p, h->bal_sv_a.p, h->bal_sv_b.p,
                                           static_cast<int>(nt), 0, static_cast<int>(end_bit), st);
  });
  if (rc != KMP_OK) {
    return rc;
  }
  bal_sorted_weights<<<capped(h, grid_for(nt, 256)), 256, 0, st>>>(nt, h->bal_sk_b.p, h->bal_sv_b.p, h->bal_cand.p,
                                                                   h->vwgt, h->bal_blk.p, h->bal_wt.p);
  rc = bal_cub(h, [&](void *tmp, size_t &bytes) {
    return cub::DeviceScan::ExclusiveSumByKey(tmp, bytes, h->bal_blk.p, h->bal_wt.p, h->bal_prefix.p,
                                              static_cast<int>(nt), cub::Equality(), st);
  });
  if (rc != KMP_OK) {
    return rc;
  }
  ubal_propose<<<capped(h, grid_for(nt, 256)), 256, 0, st>>>(nt, h->bal_blk.p, h->bal_prefix.p, h->ubal_deficit.p,
                                                             h->bal_sv_b.p, h->bal_cand.p, h->mv_u.p, h->mv_t.p,
                                                             mover_count);
  // the refiner's commit, one pass, with the minimum weights: the target side keeps every block <= max, the source
  // side keeps every source >= min (targets are underloaded and sources are not, so no block is both)
  CommitArgs ca = make_commit_args(h, RunCtx{1, k, 0, true, false});
  ca.mover_count = mover_count;
  ca.next_mover_count = h->bal_ctr32.p + 1; // scratch: nothing reads it
  ca.also_zero = nullptr;
  ca.moved_count = h->bal_ctr32.p + 4 + r;
  ca.base_commit = sync_base(h->cfg.seed, call, r, SALT_UBAL_COMMIT);
  ca.stamp = 0;
  GatheredArgs ga{nullptr, 1, 0, nullptr};
  GridBarrier bar{h->grid_bar.p, h->grid_bar.p + 1};
  uint32_t passes = 1;
  const size_t smem = 4 * std::max<size_t>(k * kLadderLevels <= kSmemPrivLimit ? static_cast<size_t>(k) * kLadderLevels : 0,
                                           k <= kSmemPrivLimit ? k : 0);
  const uint32_t blocks = capped(h, std::min<uint32_t>(grid_for(std::max<uint32_t>(nt, k), 256),
                                                       static_cast<uint32_t>(h->fused_blocks_refine)));
  void *args[] = {&ca, &ga, &bar, &passes};
  if (h->p64) {
    KMP_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void *>(commit_refine_fused<true>), dim3(blocks), dim3(256), args,
                                         smem, st));
  } else {
    KMP_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void *>(commit_refine_fused<false>), dim3(blocks), dim3(256), args,
                                         smem, st));
  }
  h->kernel_launches += 7;
  KMP_CUDA(cudaGetLastError());
  return KMP_OK;
}

} // namespace

extern "C" {

int kmp_underload_balance(kmp_lp_handle *h, uint32_t k, const int32_t *max_block_weights,
                          const int32_t *min_block_weights, uint32_t *partition_inout, int32_t *block_weights_out,
                          int *improved_out, kmp_underload_stats *stats) {
  int rc = bal_refuse(h, kUbalName, "§12");
  if (rc != KMP_OK) {
    return rc;
  }
  if (k == 0 || max_block_weights == nullptr) {
    return fail(KMP_ERR_INVALID, "k / max_block_weights missing");
  }
  if (partition_inout == nullptr && (rc = refuse_without_labels(h)) != KMP_OK) {
    return rc;
  }
  if (stats != nullptr) {
    std::memset(stats, 0, sizeof(*stats));
  }
  if (min_block_weights == nullptr) { // underload_balancer.cc:47: no minimum weights, nothing to do
    if (improved_out != nullptr) {
      *improved_out = 0;
    }
    return KMP_OK;
  }
  const uint32_t n = h->n;
  KMP_CUDA(cudaSetDevice(h->device));
  h->kernel_launches = 0;
  cudaStream_t st = h->stream;
  KMP_CUDA(cudaEventRecord(h->ev_begin, st));
  rc = ensure_scratch(h, 1, k); // the commit's ladder histograms (zeroed), counters, active flags
  if (rc == KMP_OK) {
    rc = prepare_labg(h, k); // the commit writes the packed labels (kmp_lp_refine repacks them on entry)
  }
  if (rc == KMP_OK) {
    rc = ubal_ensure(h, k, 0);
  }
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(h->label.ensure(n));
  KMP_CUDA(h->weight.ensure(k));
  KMP_CUDA(h->maxw.ensure(k));
  KMP_CUDA(h->minw.ensure(k));
  if (partition_inout != nullptr && n > 0) {
    KMP_CUDA(cudaMemcpyAsync(h->label.p, partition_inout, static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, st));
  }
  if (partition_inout != nullptr) {
    h->labels_valid = true;
  }
  KMP_CUDA(cudaMemcpyAsync(h->maxw.p, max_block_weights, static_cast<size_t>(k) * 4, cudaMemcpyHostToDevice, st));
  KMP_CUDA(cudaMemcpyAsync(h->minw.p, min_block_weights, static_cast<size_t>(k) * 4, cudaMemcpyHostToDevice, st));
  KMP_CUDA(cudaMemsetAsync(h->weight.p, 0, static_cast<size_t>(k) * 4, st));
  KMP_CUDA(cudaMemsetAsync(h->bal_ctrl.p, 0, 8 * sizeof(unsigned long long), st));
  KMP_CUDA(cudaMemsetAsync(h->bal_ctr32.p, 0, (4 + kBalMaxRounds) * sizeof(uint32_t), st));
  rc = checked_block_weights(h, k, h->bal_ctrl.p + 3);
  if (rc != KMP_OK) {
    return rc;
  }
  const uint32_t call = h->ubal_calls++;
  unsigned long long ctrl[2] = {0, 0};
  unsigned long long before = 0, candidates = 0;
  uint32_t proposals = 0;
  uint32_t rounds = 0;
  for (;; ++rounds) {
    rc = ubal_round_begin(h, k, ctrl, &proposals);
    if (rc != KMP_OK) {
      return rc;
    }
    if (rounds == 0) {
      before = ctrl[0];
    }
    // stop: min-balanced, or the last round proposed no move (then no round would: without moves the next round
    // has the same candidates, targets and deficits), or the cap. A round whose proposals the ladder rejected is
    // retried: its commit priorities and ties are hashed with the round.
    if (ctrl[0] == 0 || (rounds > 0 && proposals == 0) || rounds == kBalMaxRounds) {
      break;
    }
    const uint32_t nc = static_cast<uint32_t>(ctrl[1]);
    candidates += nc;
    rc = ubal_ensure(h, k, nc);
    if (rc == KMP_OK && h->mv_u.cap < nc) {
      KMP_CUDA(h->mv_u.ensure(nc));
      KMP_CUDA(h->mv_t.ensure(nc));
      KMP_CUDA(h->acc.ensure(nc));
    }
    if (rc == KMP_OK) {
      rc = ubal_round(h, k, nc, call, rounds);
    }
    if (rc != KMP_OK) {
      return rc;
    }
  }
  if (partition_inout != nullptr && before != 0 && n > 0) {
    KMP_CUDA(cudaMemcpyAsync(partition_inout, h->label.p, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost, st));
  }
  if (block_weights_out != nullptr) {
    KMP_CUDA(cudaMemcpyAsync(block_weights_out, h->weight.p, static_cast<size_t>(k) * 4, cudaMemcpyDeviceToHost, st));
  }
  uint32_t moved[kBalMaxRounds] = {};
  unsigned long long edges = 0;
  KMP_CUDA(cudaMemcpyAsync(moved, h->bal_ctr32.p + 4, sizeof(moved), cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaMemcpyAsync(&edges, h->bal_ctrl.p + 4, sizeof(edges), cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaEventRecord(h->ev_end, st));
  KMP_CUDA(cudaStreamSynchronize(st));
  if (improved_out != nullptr) {
    *improved_out = before != 0 ? 1 : 0;
  }
  if (stats != nullptr) {
    stats->rounds = rounds;
    std::memcpy(stats->moved, moved, sizeof(moved));
    stats->underload_before = static_cast<int64_t>(before);
    stats->underload_after = static_cast<int64_t>(ctrl[0]);
    stats->candidates = candidates;
    stats->edges_scanned = edges;
    stats->kernel_launches = h->kernel_launches;
    float ms = 0.f;
    cudaEventElapsedTime(&ms, h->ev_begin, h->ev_end);
    stats->device_ms = ms;
  }
  return KMP_OK;
}

int kmp_underload_select_all(kmp_lp_handle *h, uint32_t k, const uint32_t *labels, const int32_t *block_weights,
                             const int32_t *max_block_weights, const int32_t *min_block_weights, uint32_t call_index,
                             uint32_t round, uint32_t *target_out, float *key_out) {
  int rc = bal_refuse(h, kUbalName, "§12");
  if (rc != KMP_OK) {
    return rc;
  }
  if (k == 0 || labels == nullptr || block_weights == nullptr || max_block_weights == nullptr ||
      min_block_weights == nullptr || target_out == nullptr || key_out == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  const uint32_t n = h->n;
  for (uint32_t u = 0; u < n; ++u) {
    if (labels[u] >= k) {
      return fail(KMP_ERR_INVALID, "labels >= k: not a k-way partition");
    }
  }
  KMP_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = h->stream;
  rc = ubal_ensure(h, k, n);
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(h->label.ensure(n));
  KMP_CUDA(h->weight.ensure(k));
  KMP_CUDA(h->maxw.ensure(k));
  KMP_CUDA(h->minw.ensure(k));
  if (n > 0) {
    KMP_CUDA(cudaMemcpyAsync(h->label.p, labels, static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, st));
  }
  KMP_CUDA(cudaMemcpyAsync(h->weight.p, block_weights, static_cast<size_t>(k) * 4, cudaMemcpyHostToDevice, st));
  KMP_CUDA(cudaMemcpyAsync(h->maxw.p, max_block_weights, static_cast<size_t>(k) * 4, cudaMemcpyHostToDevice, st));
  KMP_CUDA(cudaMemcpyAsync(h->minw.p, min_block_weights, static_cast<size_t>(k) * 4, cudaMemcpyHostToDevice, st));
  KMP_CUDA(cudaMemsetAsync(h->bal_ctrl.p, 0, 8 * sizeof(unsigned long long), st));
  ubal_block_stats<<<capped(h, grid_for(k, 256)), 256, 0, st>>>(k, h->weight.p, h->minw.p, h->ubal_deficit.p,
                                                                h->ubal_tmask.p, h->bal_ctrl.p);
  if (n > 0) {
    bal_iota<<<capped(h, grid_for(n, 256)), 256, 0, st>>>(n, h->bal_cand.p);
    rc = bal_evaluate(h, k, n, sync_base(h->cfg.seed, call_index, round, SALT_UBAL_TIE), false, h->ubal_tmask.p);
    if (rc != KMP_OK) {
      return rc;
    }
    ubal_vertex_flags<<<capped(h, grid_for(n, 256)), 256, 0, st>>>(n, h->label.p, h->vwgt, h->weight.p, h->minw.p,
                                                                   h->ubal_tmask.p, h->bal_flag.p);
    ubal_keep_sources<<<capped(h, grid_for(n, 256)), 256, 0, st>>>(n, h->bal_flag.p, h->label.p, h->vwgt,
                                                                   h->bal_target.p, h->bal_key.p);
    KMP_CUDA(cudaGetLastError());
    KMP_CUDA(cudaMemcpyAsync(target_out, h->bal_target.p, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost, st));
    KMP_CUDA(cudaMemcpyAsync(key_out, h->bal_key.p, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost, st));
  }
  KMP_CUDA(cudaStreamSynchronize(st));
  return KMP_OK;
}

} // extern "C"
