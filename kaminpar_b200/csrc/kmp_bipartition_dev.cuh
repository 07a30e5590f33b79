// kmp_bipartition_subgraphs (include/kaminpar_b200_bipartition.h, DESIGN.md §20): the multilevel initial bipartitioner
// of kmp_bipartition.cuh on every block of a kmp_subgraphs that is split in two, one warp per block in one launch.
//
//   1. ip_reduce: per block, the reductions the parameters need (total / max node weight, total edge weight), one
//      warp per block; downloaded in one copy with nothing else.
//   2. host: s_b per block and the refusals, then the parameters in the reference's double code (kmp_ip_params.h),
//      a work list in descending block size and each block's arena bound (kmp_ip::arena_bound, or the test-only
//      KMP_IP_ARENA_CAP when it is lower).
//   3. ip_kernel: warps claim list entries from a counter, so the largest blocks start first; the warp zero-fills
//      the block's arena and lane 0 runs the engine. A block whose arena is too small stops and sets its flag.
//   4. the flagged blocks run again, alone, with doubled arenas. The engine is deterministic, so the result of a
//      block does not depend on which launch ran it.
#include "kmp_bipartition.cuh"
#include "kmp_ip_params.h"
#include "../../include/kaminpar_b200_bipartition.h"

namespace {

__global__ void ip_reduce(uint32_t k, const uint32_t *node_off, const uint32_t *edge_off, const int32_t *vwgt,
                          const int32_t *adjwgt, int32_t *red) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t warps = gridDim.x * (blockDim.x / 32);
  for (uint32_t b = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32; b < k; b += warps) {
    const uint32_t n0 = node_off[b], n1 = node_off[b + 1], e0 = edge_off[b], e1 = edge_off[b + 1];
    uint32_t tn = 0, te = 0;
    int32_t mx = 1;
    if (vwgt != nullptr) {
      mx = n1 > n0 ? static_cast<int32_t>(0x80000000u) : 1;
      for (uint32_t u = n0 + lane; u < n1; u += 32) {
        tn += static_cast<uint32_t>(vwgt[u]);
        mx = max(mx, vwgt[u]);
      }
    } else {
      tn = lane == 0 ? n1 - n0 : 0;
    }
    if (adjwgt != nullptr) {
      for (uint32_t e = e0 + lane; e < e1; e += 32) {
        te += static_cast<uint32_t>(adjwgt[e]);
      }
    } else {
      te = lane == 0 ? e1 - e0 : 0;
    }
    for (int o = 16; o > 0; o >>= 1) {
      tn += __shfl_xor_sync(0xFFFFFFFFu, tn, o);
      te += __shfl_xor_sync(0xFFFFFFFFu, te, o);
      mx = max(mx, __shfl_xor_sync(0xFFFFFFFFu, mx, o));
    }
    if (lane == 0) {
      red[3 * b] = static_cast<int32_t>(tn);
      red[3 * b + 1] = mx;
      red[3 * b + 2] = static_cast<int32_t>(te);
    }
  }
}

struct IpLaunch {
  const kmp_ip::Config *cfg; // device memory: a reference into the kernel's parameters would copy them to the stack
  int32_t num_seed_iterations;
  int32_t seed;
  uint32_t num;                 // list entries
  const uint32_t *list;         // block ids, descending n
  const kmp_ip::BlockParams *bp; // [num]
  const unsigned long long *arena_off, *arena_size; // [num] bytes
  uint8_t *arena;
  const uint32_t *xadj, *adjncy, *node_off, *edge_off;
  const int32_t *vwgt, *adjwgt;
  uint32_t *out;
  uint32_t *overflow; // [num]
  uint32_t *counter;
  uint32_t *counters; // [2]: pool runs, coarsening levels
};

__global__ void __launch_bounds__(128) ip_kernel(const IpLaunch a) {
  const uint32_t lane = threadIdx.x & 31u;
  while (true) {
    uint32_t i = 0;
    if (lane == 0) {
      i = atomicAdd(a.counter, 1u);
    }
    i = __shfl_sync(0xFFFFFFFFu, i, 0);
    if (i >= a.num) {
      return;
    }
    uint8_t *base = a.arena + a.arena_off[i];
    const uint64_t size = a.arena_size[i];
    for (uint64_t w = lane; w < size / 8; w += 32) {
      reinterpret_cast<unsigned long long *>(base)[w] = 0ull;
    }
    __syncwarp();
    if (lane == 0) {
      const uint32_t b = a.list[i];
      const uint32_t n0 = a.node_off[b], n = a.node_off[b + 1] - n0;
      const uint32_t e0 = a.edge_off[b], m = a.edge_off[b + 1] - e0;
      kmp_ip::Counters cnt{0, 0};
      const bool ok = kmp_ip::bipartition_block(
          n, m, a.xadj + n0 + b, a.adjncy + e0, a.vwgt != nullptr ? a.vwgt + n0 : nullptr,
          a.adjwgt != nullptr ? a.adjwgt + e0 : nullptr, *a.cfg, a.num_seed_iterations, a.bp[i],
          static_cast<int32_t>(static_cast<uint32_t>(a.seed) + b), base, size, a.out + n0, cnt);
      a.overflow[i] = ok ? 0u : 1u;
      if (ok) {
        atomicAdd(a.counters, cnt.pool_runs);
        atomicAdd(a.counters + 1, cnt.levels);
      }
    }
    __syncwarp();
  }
}

kmp_ip::FmParams ip_fm(const kmp_ip_refinement &r) {
  kmp_ip::FmParams f;
  f.algorithm = r.num_algorithms == 0 ? kmp_ip::kRefineNoop : static_cast<uint32_t>(r.algorithm);
  f.num_fruitless_moves = r.num_fruitless_moves;
  f.alpha = r.alpha;
  f.num_iterations = r.num_iterations;
  f.improvement_abortion_threshold = r.improvement_abortion_threshold;
  return f;
}

int ip_check_refinement(const kmp_ip_refinement &r) {
  if (r.num_algorithms > 1) {
    return fail(KMP_ERR_UNSUPPORTED, "a refinement algorithm list longer than one is not supported");
  }
  if (r.num_algorithms == 1) {
    if (r.algorithm == KMP_IP_TWOWAY_FLOW) {
      return fail(KMP_ERR_UNSUPPORTED, "TWOWAY_FLOW initial refinement is not supported");
    }
    if (r.algorithm < KMP_IP_NOOP || r.algorithm > KMP_IP_TWOWAY_FLOW) {
      return fail(KMP_ERR_INVALID, "unknown initial refinement algorithm");
    }
  }
  return KMP_OK;
}

uint64_t ip_arena_first_bound(uint32_t n, uint32_t m) {
  uint64_t bound = kmp_ip::arena_bound(n, m);
  if (const char *e = std::getenv("KMP_IP_ARENA_CAP")) { // tests: reach the re-run path with small blocks
    const uint64_t cap = std::strtoull(e, nullptr, 10);
    if (cap >= 8 && cap < bound) {
      bound = cap & ~7ull;
    }
  }
  return (bound + 7) & ~7ull;
}

} // namespace

extern "C" {

kmp_ip_config kmp_ip_default_config(void) { return kmp_ip_params::default_config(); }

int kmp_lp_handle_device(const kmp_lp_handle *h) { return h != nullptr ? h->device : -1; }

int kmp_bipartition_subgraphs(kmp_lp_handle *h, const kmp_subgraphs *g, uint32_t k_prime, uint32_t input_k,
                              const int32_t *input_max_block_weights, int uniform_block_weights,
                              int64_t input_total_node_weight, double input_epsilon, const kmp_ip_config *cfg,
                              int32_t seed, uint32_t *d_sub_partitions, kmp_bipartition_stats *stats) {
  if (h == nullptr || g == nullptr || cfg == nullptr || input_max_block_weights == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  if (d_sub_partitions == nullptr || (reinterpret_cast<uintptr_t>(d_sub_partitions) & 3u) != 0) {
    return fail(KMP_ERR_INVALID, "d_sub_partitions must be a 4-byte aligned device pointer");
  }
  if (h->step.open) {
    return fail(KMP_ERR_INVALID, "the handle is inside a stepping call");
  }
  if (g->source != h || !h->graph.present || h->graph.epoch != g->graph_epoch) {
    return fail(KMP_ERR_INVALID, "the handle holds another graph than the one the subgraphs were extracted from");
  }
  const uint32_t k = g->k;
  if (k_prime < k || input_k == 0 || k_prime > input_k || (k_prime != input_k && k_prime % k != 0)) {
    return fail(KMP_ERR_INVALID, "k_prime must lie in [k, input_k] and be input_k or a multiple of k");
  }
  if ((k & (k - 1)) != 0) {
    // the reference's extension runs at power-of-two k only: for other k, create_twoway_context's sub-block ranges
    // (compute_first_sub_block + compute_final_k) can run past input_k
    return fail(KMP_ERR_UNSUPPORTED, "k must be a power of two");
  }
  if (input_total_node_weight < 0 || input_total_node_weight > 0x7FFFFFFF) {
    return fail(KMP_ERR_INVALID, "input_total_node_weight must fit a 32-bit node weight");
  }
  for (const kmp_ip_refinement *r : {&cfg->pool_refinement, &cfg->refinement}) {
    const int rc = ip_check_refinement(*r);
    if (rc != KMP_OK) {
      return rc;
    }
  }
  if (cfg->contraction_limit == 0 || cfg->cluster_weight_limit < KMP_IP_CWL_EPSILON_BLOCK_WEIGHT ||
      cfg->cluster_weight_limit > KMP_IP_CWL_ZERO || cfg->min_num_repetitions > cfg->max_num_repetitions) {
    return fail(KMP_ERR_INVALID, "initial partitioning configuration out of range");
  }
  if (!cfg->enable_bfs_bipartitioner && !cfg->enable_ggg_bipartitioner && !cfg->enable_random_bipartitioner) {
    return fail(KMP_ERR_UNSUPPORTED, "every initial bipartitioner is disabled");
  }
  std::vector<uint32_t> split(k, k_prime / k);
  if (k_prime == input_k) {
    for (uint32_t b = 0; b < k; ++b) {
      split[b] = kmp_ip_params::compute_final_k(b, k, input_k);
    }
  }
  for (uint32_t b = 0; b < k; ++b) {
    if (split[b] > 2) {
      return fail(KMP_ERR_UNSUPPORTED, "a block would be split into more than two sub-blocks: extend in doubling "
                                       "steps");
    }
  }
  KMP_CUDA(cudaSetDevice(h->device));
  if (stats != nullptr) {
    std::memset(stats, 0, sizeof(*stats));
  }
  const cudaStream_t st = h->stream;
  const int dev = h->device;
  const uint32_t n = g->n;
  uint32_t launches = 0, retries = 0;
  KMP_CUDA(call_clock_start(h, st));
  std::vector<uint32_t> node_off(static_cast<size_t>(k) + 1), edge_off(static_cast<size_t>(k) + 1);
  KMP_CUDA(cudaMemcpyAsync(node_off.data(), g->node_off.p, node_off.size() * 4, cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaMemcpyAsync(edge_off.data(), g->edge_off.p, edge_off.size() * 4, cudaMemcpyDeviceToHost, st));
  KMP_CUDA(cudaStreamSynchronize(st));
  std::vector<uint32_t> list;
  for (uint32_t b = 0; b < k; ++b) {
    if (split[b] == 2 && node_off[b + 1] > node_off[b]) {
      list.push_back(b);
    }
  }
  kmp_bipartition_stats s{};
  s.blocks_split = static_cast<uint32_t>(list.size());
  if (!list.empty()) {
    PoolBuf<int32_t> red;
    KMP_CUDA(red.alloc(static_cast<size_t>(k) * 3, st, dev));
    ip_reduce<<<capped(h, grid_for(static_cast<uint64_t>(k) * 32, 256)), 256, 0, st>>>(
        k, g->node_off.p, g->edge_off.p, g->vwgt.p, g->adjwgt.p, red.p);
    ++launches;
    std::vector<int32_t> hred(static_cast<size_t>(k) * 3);
    KMP_CUDA(cudaMemcpyAsync(hred.data(), red.p, hred.size() * 4, cudaMemcpyDeviceToHost, st));
    KMP_CUDA(cudaStreamSynchronize(st));
    std::stable_sort(list.begin(), list.end(), [&](uint32_t a, uint32_t b) {
      return node_off[a + 1] - node_off[a] > node_off[b + 1] - node_off[b];
    });
    const kmp_ip_params::InputContext in{input_k, input_max_block_weights, uniform_block_weights != 0,
                                         static_cast<int32_t>(input_total_node_weight), input_epsilon};
    const size_t num = list.size();
    std::vector<kmp_ip::BlockParams> bp(num);
    std::vector<unsigned long long> size(num), off(num);
    for (size_t i = 0; i < num; ++i) {
      const uint32_t b = list[i];
      const kmp_ip_params::BlockStats bs{node_off[b + 1] - node_off[b], edge_off[b + 1] - edge_off[b], hred[3 * b],
                                         hred[3 * b + 1], hred[3 * b + 2]};
      int32_t p[6];
      if (!kmp_ip_params::block_params(in, *cfg, b, k, bs, p)) {
        return fail(KMP_ERR_UNSUPPORTED, "a block's sub-block range runs past input_k");
      }
      bp[i] = kmp_ip::BlockParams{{p[0], p[1]}, {p[2], p[3]}, p[4], p[5]};
      size[i] = ip_arena_first_bound(bs.n, bs.m);
    }
    KMP_CUDA(cudaMemsetAsync(d_sub_partitions, 0, static_cast<size_t>(n) * 4, st));
    kmp_ip::Config hc{};
    hc.contraction_limit = cfg->contraction_limit;
    hc.convergence_threshold = cfg->convergence_threshold;
    hc.large_degree_threshold = cfg->large_degree_threshold;
    hc.pool_fm = ip_fm(cfg->pool_refinement);
    hc.fm = ip_fm(cfg->refinement);
    hc.min_num_non_adaptive_repetitions = cfg->min_num_non_adaptive_repetitions;
    hc.use_adaptive_bipartitioner_selection = cfg->use_adaptive_bipartitioner_selection;
    hc.enable_bfs = cfg->enable_bfs_bipartitioner;
    hc.enable_ggg = cfg->enable_ggg_bipartitioner;
    hc.enable_random = cfg->enable_random_bipartitioner;
    hc.refine_pool_partition = cfg->refine_pool_partition;
    IpLaunch a{};
    a.num_seed_iterations = cfg->num_seed_iterations;
    a.seed = seed;
    a.xadj = g->xadj.p;
    a.adjncy = g->adjncy.p;
    a.vwgt = g->vwgt.p;
    a.adjwgt = g->adjwgt.p;
    a.node_off = g->node_off.p;
    a.edge_off = g->edge_off.p;
    a.out = d_sub_partitions;
    PoolBuf<uint32_t> d_list, d_flag, d_counter;
    PoolBuf<kmp_ip::BlockParams> d_bp;
    PoolBuf<kmp_ip::Config> d_cfg;
    KMP_CUDA(d_cfg.alloc(1, st, dev));
    KMP_CUDA(cudaMemcpyAsync(d_cfg.p, &hc, sizeof(hc), cudaMemcpyHostToDevice, st));
    a.cfg = d_cfg.p;
    PoolBuf<unsigned long long> d_off, d_size;
    KMP_CUDA(d_list.alloc(num, st, dev));
    KMP_CUDA(d_flag.alloc(num, st, dev));
    KMP_CUDA(d_counter.alloc(3, st, dev));
    KMP_CUDA(d_bp.alloc(num, st, dev));
    KMP_CUDA(d_off.alloc(num, st, dev));
    KMP_CUDA(d_size.alloc(num, st, dev));
    KMP_CUDA(cudaMemsetAsync(d_counter.p, 0, 12, st));
    std::vector<uint32_t> flag(num);
    for (int attempt = 0; !list.empty(); ++attempt) {
      if (attempt > 40) {
        return fail(KMP_ERR_ALLOC, "a block's initial bipartitioning arena did not fit after 40 doublings");
      }
      const size_t cnt = list.size();
      unsigned long long total = 0;
      for (size_t i = 0; i < cnt; ++i) {
        off[i] = total;
        total += size[i];
      }
      PoolBuf<uint8_t> arena;
      KMP_CUDA(arena.alloc(total, st, dev));
      KMP_CUDA(cudaMemcpyAsync(d_list.p, list.data(), cnt * 4, cudaMemcpyHostToDevice, st));
      KMP_CUDA(cudaMemcpyAsync(d_bp.p, bp.data(), cnt * sizeof(kmp_ip::BlockParams), cudaMemcpyHostToDevice, st));
      KMP_CUDA(cudaMemcpyAsync(d_off.p, off.data(), cnt * 8, cudaMemcpyHostToDevice, st));
      KMP_CUDA(cudaMemcpyAsync(d_size.p, size.data(), cnt * 8, cudaMemcpyHostToDevice, st));
      KMP_CUDA(cudaMemsetAsync(d_counter.p, 0, 4, st));
      a.num = static_cast<uint32_t>(cnt);
      a.list = d_list.p;
      a.bp = d_bp.p;
      a.arena_off = d_off.p;
      a.arena_size = d_size.p;
      a.arena = arena.p;
      a.overflow = d_flag.p;
      a.counter = d_counter.p;
      a.counters = d_counter.p + 1;
      ip_kernel<<<capped(h, grid_for(static_cast<uint64_t>(cnt) * 32, 128)), 128, 0, st>>>(a);
      ++launches;
      KMP_CUDA(cudaGetLastError());
      KMP_CUDA(cudaMemcpyAsync(flag.data(), d_flag.p, cnt * 4, cudaMemcpyDeviceToHost, st));
      KMP_CUDA(cudaStreamSynchronize(st));
      size_t kept = 0;
      for (size_t i = 0; i < cnt; ++i) {
        if (flag[i] != 0) {
          list[kept] = list[i];
          bp[kept] = bp[i];
          size[kept] = size[i] * 2;
          ++kept;
        }
      }
      retries += static_cast<uint32_t>(kept);
      list.resize(kept);
    }
    uint32_t counters[2];
    KMP_CUDA(cudaMemcpyAsync(counters, d_counter.p + 1, 8, cudaMemcpyDeviceToHost, st));
    KMP_CUDA(cudaStreamSynchronize(st));
    s.pool_runs = counters[0];
    s.coarsening_levels = counters[1];
  }
  if (s.blocks_split == 0) {
    KMP_CUDA(cudaMemsetAsync(d_sub_partitions, 0, static_cast<size_t>(n) * 4, st));
  }
  KMP_CUDA(call_clock_stop(h, st));
  KMP_CUDA(cudaStreamSynchronize(st));
  s.arena_retries = retries;
  s.kernel_launches = launches;
  s.device_ms = call_clock_ms(h);
  if (stats != nullptr) {
    *stats = s;
  }
  return KMP_OK;
}

} // extern "C"
