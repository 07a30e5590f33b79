// kaminpar_b200: underload balancer on the device + its C ABI (include/kaminpar_b200_balancer.h).
// Included at the end of kmp_lp.cu after kmp_balance.cuh, which holds what the two balancers share: the degree-tiered
// candidate evaluation (bal_eval_thread / _warp / _cta, here with a target mask), the scratch on the handle, the round
// driver (bal_run) with its stop rule, the round tail (sort, per-block weight scan, ubal_propose, the refiner's
// cooperative ladder commit, here with the minimum block weights) and the body of select_all. This file holds the
// underload balancer's own steps: the round start and the selection before the sort.
//
// What it restates: UnderloadBalancer::refine (refinement/balancer/underload_balancer.cc:39-244) as synchronous
// rounds (DESIGN.md §12). One round:
//   1. block stats against the frozen weights: deficit[b] = max(0, min[b] - W[b]) (kept in bal.over), the total
//      underload, the underloaded flags (the target mask); the vertices that may leave their block (block not
//      underloaded, W[b] - w(u) >= min[b]) are compacted in id order (one small read-back per round: total, count)
//   2. candidate evaluation by the overload balancer's tiers, targets restricted to underloaded blocks
//   3. the candidates with a target are compacted in id order (a second read-back: their count) and sorted by
//      (target, key desc); exclusive weight scan per target, selected iff the weight before a candidate is
//      < deficit[target]
//   4. the ladder commit of the LP refiner with one pass and the minimum weights: targets stay <= max, sources >= min
#pragma once

namespace kmp {

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

// Round start: deficit[] (in bal.over), target mask, candidates; read back {total underload, #candidates} and the
// number of proposals of the previous round.
int ubal_round_begin(kmp_lp_handle *h, uint32_t k, unsigned long long *host_ctrl, uint32_t *host_proposals) {
  cudaStream_t st = h->stream;
  const uint32_t n = h->graph.n;
  KMP_CUDA(cudaMemsetAsync(h->bal.ctrl.p, 0, 2 * sizeof(unsigned long long), st));
  ubal_block_stats<<<capped(h, grid_for(k, 256)), 256, 0, st>>>(k, h->lp.weight.p, h->lp.minw.p, h->bal.over.p,
                                                                h->bal.tmask.p, h->bal.ctrl.p);
  ubal_vertex_flags<<<capped(h, grid_for(n, 256)), 256, 0, st>>>(n, h->lp.label.p, h->graph.vwgt, h->lp.weight.p, h->lp.minw.p,
                                                                 h->bal.tmask.p, h->bal.flag.p);
  KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
    return cub::DeviceSelect::Flagged(tmp, bytes, thrust::counting_iterator<uint32_t>(0), h->bal.flag.p, h->bal.cand.p,
                                      h->bal.ctrl.p + 1, static_cast<int>(n), st);
  }));
  h->counts.kernel_launches += 3;
  KMP_CUDA(cudaMemcpyAsync(host_ctrl, h->bal.ctrl.p, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaMemcpyAsync(host_proposals, h->bal.ctr32.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaStreamSynchronize(st));
  return KMP_OK;
}

// Selection of a round after its read-back: evaluate the nc candidates, compact those with a target and write their
// sort words (target << 32 | desc key bits) into bal.sk_a / bal.sv_a; *nt: their count (0: the round proposes nothing).
int ubal_select(kmp_lp_handle *h, uint32_t k, uint32_t nc, uint32_t call, uint32_t r, uint32_t *nt) {
  *nt = 0;
  if (nc == 0) {
    return KMP_OK;
  }
  cudaStream_t st = h->stream;
  int rc = bal_evaluate(h, k, nc, sync_base(h->cfg.seed, call, r, SALT_UBAL_TIE), false, h->bal.tmask.p);
  if (rc != KMP_OK) {
    return rc;
  }
  // Most candidates have no underloaded neighbour block (typically few blocks are underloaded): compacting them
  // away costs one select and a read-back, where sorting them into a zero-deficit segment would cost radix passes
  // over nearly every vertex.
  uint32_t *list = h->bal.lists.p; // free again after the evaluation
  KMP_CUDA(cub_call(h, [&](void *tmp, size_t &bytes) {
    return cub::DeviceSelect::If(tmp, bytes, thrust::counting_iterator<uint32_t>(0), list, h->bal.ctrl.p + 5,
                                 static_cast<int>(nc), UbalHasTarget{h->bal.cand.p, h->lp.label.p, h->bal.target.p}, st);
  }));
  unsigned long long nt64 = 0;
  KMP_CUDA(cudaMemcpyAsync(&nt64, h->bal.ctrl.p + 5, sizeof(nt64), cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaStreamSynchronize(st));
  *nt = static_cast<uint32_t>(nt64);
  if (*nt == 0) {
    return KMP_OK;
  }
  ubal_sort_keys<<<capped(h, grid_for(*nt, 256)), 256, 0, st>>>(*nt, list, h->bal.target.p, h->bal.key.p, h->bal.sk_a.p,
                                                                h->bal.sv_a.p);
  h->counts.kernel_launches += 2;
  KMP_CUDA(cudaGetLastError());
  return KMP_OK;
}

} // namespace

extern "C" {

int kmp_underload_balance(kmp_lp_handle *h, uint32_t k, const int32_t *max_block_weights,
                          const int32_t *min_block_weights, uint32_t *partition_inout, int32_t *block_weights_out,
                          int *improved_out, kmp_underload_stats *stats) {
  int rc = bal_refuse(h, BalKind::Underload);
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
  BalResult res;
  rc = bal_run(h, BalKind::Underload, k, max_block_weights, min_block_weights, nullptr, partition_inout,
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
    stats->underload_before = static_cast<int64_t>(res.before);
    stats->underload_after = static_cast<int64_t>(res.after);
    stats->candidates = res.candidates;
    stats->edges_scanned = res.edges;
    stats->kernel_launches = h->counts.kernel_launches;
    stats->device_ms = res.device_ms;
  }
  return KMP_OK;
}

int kmp_underload_select_all(kmp_lp_handle *h, uint32_t k, const uint32_t *labels, const int32_t *block_weights,
                             const int32_t *max_block_weights, const int32_t *min_block_weights, uint32_t call_index,
                             uint32_t round, uint32_t *target_out, float *key_out) {
  return bal_select_all(h, BalKind::Underload, k, labels, block_weights, max_block_weights, min_block_weights,
                        call_index, round, target_out, key_out);
}

} // extern "C"
