// Degree groups 0 and 1 of a clustering round in ONE cooperative launch per group.
//
// A sub-round of these groups is one wave of thread-per-vertex sweeps (tiers 0..2, deg < 32) over a few
// million edges at most: a few microseconds of gathers behind a launch, a chain of dependent loads per thread
// (list entry -> CSR row -> neighbour ids -> packed labels -> sort -> weights -> proposal) and a commit of three
// grid-barrier phases. Here the group's sub-rounds run back to back in one persistent kernel:
//
//   for each non-empty sub-round s of the group:
//     sweep   (sweep_thread_vertex of lp_sweep.cuh over the tier lists of s, proposals as in sweep_thread)
//     prefetch the static row (list entry, xadj pair, neighbour ids) of this thread's first entry of s + 1
//     | classify | decide | apply (+ push activation)      -- lp_commit.cuh cluster_*, grid_sync between phases
//
// The prefetched row does not depend on the commit, so its loads are in flight across the commit's barriers;
// only the label, weight and active reads of s + 1 wait for them. The result is the per-sub-round path's: the
// same proposals, counters, window / stamp / commit base per sub-round, the same mover-counter parity.
#pragma once

#include "lp_commit.cuh"
#include "lp_sweep.cuh"

namespace kmp {

constexpr uint32_t kLowMaxSubrounds = 32; // >= the largest sync_subrounds (kmp_lp.cu ensure_lists)

struct LowSubround {
  uint32_t off[2];      // first entry of the tier lists (tier A, tier B) in SweepArgs::list
  uint32_t size[2];     // list sizes; tier B is empty in group 0
  uint32_t window_start, window_len; // StampWindow of the sweep
  uint32_t base_commit; // commit priorities of the sweep's proposals and of the commit
  uint32_t stamp;       // move stamp written by the apply (0: push activation only)
  uint32_t parity;      // proposal counter: ctr32[0] (0) or ctr32[3] (1); the other one is zeroed for s + 1
};

struct LowGroupArgs {
  uint32_t num_sub;                       // non-empty sub-rounds of the group in this round
  bool push;                              // movers flag their neighbours (push rounds)
  uint32_t *ctr32;                        // proposal counters at [0] and [3]
  unsigned long long *counters[2];        // scan counters of tier A and tier B (ctr64 + tier)
  LowSubround sub[kLowMaxSubrounds];
};

// Entry i of the concatenated lists (tier A, then tier B) of sub-round q
__device__ __forceinline__ uint32_t low_entry(const SweepArgs &a, const LowSubround &q, uint32_t i) {
  return a.list[i < q.size[0] ? q.off[0] + i : q.off[1] + (i - q.size[0])];
}

// NA / NB: register-sort width of tier A / tier B (group 0: 8 / 8 with an empty tier B; group 1: 16 / 32).
// LANES: push-activation team size of the group (commit_activate).
template <bool EW, bool P64, int NA, int NB, int LANES>
__global__ void __launch_bounds__(256) sweep_commit_low(const SweepArgs a0, const CommitArgs c0, const LowGroupArgs g,
                                                         const GridBarrier bar) {
  __shared__ uint32_t s_cnt[2][8];
  __shared__ uint32_t s_base[2];
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t nth = gridDim.x * blockDim.x;
  SweepArgs a = a0;
  CommitArgs c = c0;
  unsigned long long edges[2] = {0, 0}, nodes[2] = {0, 0};
  // static row of this thread's coming entry: loaded one entry ahead, in the sub-round and across the commit
  // (assigned on every path, so that the old row is dead while the current vertex sorts)
  ThreadRow<NB> r;
  auto fetch = [&](const LowSubround &q, uint32_t i) {
    if (i < q.size[0] + q.size[1]) {
      r.u = low_entry(a, q, i);
      load_row<NB>(a, r);
    } else {
      r = ThreadRow<NB>{};
    }
  };
  fetch(g.sub[0], tid);
  uint32_t it = 0;
  for (uint32_t s = 0; s < g.num_sub; ++s) {
    const LowSubround &q = g.sub[s];
    a.window = StampWindow{q.window_start, q.window_len};
    a.base_commit = q.base_commit;
    a.mover_count = g.ctr32 + (q.parity ? 3 : 0);
    // ---- sweep (the bound is rounded up to a full CTA so that all threads reach emit_cta_iteration's barriers)
    const uint32_t total = q.size[0] + q.size[1];
    const uint32_t bound = (total + 255u) & ~255u;
    for (uint32_t i = tid; i < bound; i += nth, ++it) {
      bool proposes = false;
      uint32_t target = 0;
      int32_t uw = 1;
      const uint32_t u = r.u;
      if (i < total) {
        const bool flag = a.active == nullptr || a.active[u] != 0;
        if (flag || a.pull) {
          if (NA == NB || i < q.size[0]) {
            proposes = sweep_thread_vertex<0, EW, P64, NA>(a, r, flag, edges[0], nodes[0], target, uw);
          } else {
            proposes = sweep_thread_vertex<0, EW, P64, NB>(a, r, flag, edges[1], nodes[1], target, uw);
          }
        }
      }
      fetch(q, i + nth);
      emit_cta_iteration<0>(a, proposes, u, target, uw, it, s_cnt, s_base);
    }
    if (s + 1 < g.num_sub) {
      fetch(g.sub[s + 1], tid);
    }
    // ---- commit (commit_cluster_fused's phases; the proposal count was written by this launch's atomics)
    grid_sync(bar);
    c.mover_count = a.mover_count;
    c.next_mover_count = g.ctr32 + (q.parity ? 0 : 3);
    c.base_commit = q.base_commit;
    c.stamp = q.stamp;
    const uint32_t cnt = __ldcg(c.mover_count);
    cluster_classify(c, cnt, tid, nth);
    grid_sync(bar);
    cluster_decide(c, cnt, tid, nth);
    grid_sync(bar);
    cluster_apply<P64>(c, cnt, tid, nth);
    if (g.push) { // only sets flags, as the apply does, and reads nothing the apply writes: no barrier between them
      activate_neighbours<LANES>(c, cnt, tid, nth);
    }
    if (s + 1 < g.num_sub) {
      grid_sync(bar);
    }
  }
  a.counters = g.counters[0];
  block_count_flush(a, edges[0], nodes[0]);
  if (NA != NB) {
    a.counters = g.counters[1];
    block_count_flush(a, edges[1], nodes[1]);
  }
}

} // namespace kmp
