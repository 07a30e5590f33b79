// Schedule KMP_SCHEDULE_SEQ_STRICT: the reference's label propagation at ONE thread, restated for one GPU
// thread block -- same visit order, same rating-map insertion order, same random draws -- so that the
// label vector is bit-identical to the unmodified reference (SURVEY.md §7 "strict mode", §8b).
//
// What is restated (all of it runs on the device, sequentially; the graph sits in L1/L2):
//   Random / RandomPermutations        kaminpar-common/random.h:27-147, random.cc:18-56
//     std::mt19937                     ISO C++ [rand.eng.mers] (32-bit Mersenne twister)
//     std::uniform_int_distribution    libstdc++ 13 <bits/uniform_int_dist.h>: Lemire's nearly divisionless
//                                      method on a 32-bit generator (_S_nd)
//     std::shuffle                     libstdc++ 13 <bits/stl_algo.h>: two swap positions per draw
//                                      (__gen_two_uniform_ints) while size^2 fits the generator range
//     -- libstdc++-specific; tests/cpp/strict_rng_check.cc pins these restatements against the real
//        std:: facilities on the host.
//   init_chunks / shuffle_chunks       label_propagation.h:1736-1861
//   perform / perform_first_phase      label_propagation.h:1863-2020
//   handle_node -> find_best_cluster   label_propagation.h:330-368, :460-638 (two-phase deferral at 10 000 keys)
//   second phase                       label_propagation.h:640-815, :2022-2051
//   select_best_cluster                lp_clusterer.cc:181-280, lp_refiner.cc:151-285 (UNIFORM and GEOMETRIC)
//   try_node_move / activate_neighbors label_propagation.h:817-870, :2139-2152; partitioned_graph.h:397-428
//   isolated nodes / two-hop           label_propagation.h:884-1191, gating lp_clusterer.cc:112-166
//
// Every function is plain sequential integer code marked KMP_HD so that tests/cpp can also compile it with
// g++ and step through it next to the oracle; the PRODUCT only ever runs it inside strict_kernel below.
#pragma once

#include <cstdint>

#include "kmp_rng.cuh"

namespace kmp_strict {

using namespace kmp_rng;

constexpr uint32_t kInvalid = 0xFFFFFFFFu;
constexpr uint32_t kRatingMapThreshold = 10000; // label_propagation.h:62
constexpr uint32_t kPermSize = 64, kNumPerms = 64; // RandomPermutations<NodeID, 64, 64>

// ---- Random / RandomPermutations<NodeID, 64, 64> -------------------------------------------------
struct Rng : RngCore {
  uint32_t perms[kNumPerms][kPermSize];
};

// Random::reseed (random.cc:45-56) with thread index 0 + RandomPermutations ctor (random.h:138-143)
KMP_HD inline void rng_init(Rng &r, int seed) {
  rng_seed(r, seed);
  for (uint32_t p = 0; p < kNumPerms; ++p) {
    for (uint32_t i = 0; i < kPermSize; ++i) {
      r.perms[p][i] = i;
    }
    shuffle(r, r.perms[p], kPermSize);
  }
}

// ---- engine state (device memory, owned by the handle) ----------------------------------------
struct Stats {
  uint32_t iterations;
  uint32_t moved[64];
  unsigned long long edges_scanned, nodes_visited;
  uint32_t num_clusters, two_hop_ran;
};

struct Args {
  // graph
  uint32_t n, m;
  const uint32_t *xadj, *adjncy;
  const int32_t *vwgt, *adjwgt; // nullable
  int sorted;                   // CSRGraph::sorted(): the vertices are ordered by degree bucket
  uint32_t *buckets;            // [34] degree-bucket prefix array, filled by init_buckets
  // configuration (kmp_lp_config)
  uint32_t num_iterations, large_degree_threshold, max_num_neighbors;
  int impl, tie_uniform, two_hop_strategy, isolated_nodes_strategy;
  double two_hop_threshold;
  int mode; // 0 clusterer, 1 refiner
  int32_t max_cluster_weight;
  uint32_t desired_num_clusters;
  uint32_t k;
  const int32_t *max_bw, *min_bw; // refiner; min nullable
  const uint32_t *communities;    // nullable
  // state
  uint32_t *label;
  int32_t *weight;   // [n] cluster weights / [k] block weights
  uint32_t *favored; // clusterer
  uint8_t *active;
  // rating map: insertion-ordered accumulator (all reference back-ends enumerate in first-insertion order)
  int32_t *slot;     // [num_keys] 0 = absent, else index + 1 into the entry arrays
  uint32_t *ent_key; // [max distinct keys of one vertex]
  int32_t *ent_val;
  int32_t *slot2;    // second phase: thread-local small map
  uint32_t *ent2_key;
  int32_t *ent2_val;
  int32_t *concurrent;     // [num_keys] ConcurrentFastResetArray data
  uint32_t *used_entries;  // [num_keys]
  uint32_t *second_phase_nodes; // [n]
  uint32_t *tie_best, *tie_fav; // [max distinct keys]
  uint32_t *chunks;        // {start, end} pairs, [2 * (n + 64)]
  uint32_t *sub_perm;      // [n / 64 + 2]
  uint32_t *match_map;     // [n] two-hop threadwise: favored cluster -> waiting vertex + 1
  Rng *rng;
  Stats *stats;
};

struct Engine {
  const Args &a;
  Rng &rand;
  uint32_t map_size = 0, map2_size = 0, used_size = 0;
  uint32_t num_chunks = 0, num_bucket_ranges = 0;
  uint32_t bucket_start[40], bucket_end[40];
  uint32_t num_second = 0;
  uint32_t num_buckets = 0;
  uint32_t initial_num_clusters = 0;
  long long current_num_clusters = 0;
  uint32_t next_chunk = 0;

  KMP_HD Engine(const Args &a_) : a(a_), rand(*a_.rng) {}

  KMP_HD int32_t nw(uint32_t u) const { return a.vwgt ? a.vwgt[u] : 1; }
  KMP_HD int32_t ew(uint32_t e) const { return a.adjwgt ? a.adjwgt[e] : 1; }
  KMP_HD uint32_t deg(uint32_t u) const { return a.xadj[u + 1] - a.xadj[u]; }
  KMP_HD int32_t max_w(uint32_t c) const { return a.mode == 0 ? a.max_cluster_weight : a.max_bw[c]; }
  KMP_HD int32_t min_w(uint32_t c) const { return (a.mode == 1 && a.min_bw) ? a.min_bw[c] : 0; }
  KMP_HD bool accept_neighbor(uint32_t u, uint32_t v) const {
    return a.mode == 0 || !a.communities || a.communities[u] == a.communities[v];
  }

  // ---- rating map ------------------------------------------------------------------------------
  KMP_HD void map_add(uint32_t key, int32_t w) {
    int32_t &s = a.slot[key];
    if (s == 0) {
      a.ent_key[map_size] = key;
      a.ent_val[map_size] = w;
      s = static_cast<int32_t>(++map_size);
    } else {
      a.ent_val[s - 1] += w;
    }
  }
  KMP_HD void map_clear() {
    for (uint32_t i = 0; i < map_size; ++i) {
      a.slot[a.ent_key[i]] = 0;
    }
    map_size = 0;
  }
  KMP_HD void map2_add(uint32_t key, int32_t w) {
    int32_t &s = a.slot2[key];
    if (s == 0) {
      a.ent2_key[map2_size] = key;
      a.ent2_val[map2_size] = w;
      s = static_cast<int32_t>(++map2_size);
    } else {
      a.ent2_val[s - 1] += w;
    }
  }

  // ---- weights ---------------------------------------------------------------------------------
  // clusterer: label_propagation.h:2139-2152; refiner: partitioned_graph.h:397-428
  KMP_HD bool move_cluster_weight(uint32_t from, uint32_t to, int32_t d, int32_t mx) {
    if (a.weight[to] + d <= mx) {
      a.weight[to] += d;
      a.weight[from] -= d;
      if (a.mode == 0 || a.weight[from] >= min_w(from)) {
        return true;
      }
      a.weight[from] += d;
      a.weight[to] -= d;
    }
    return false;
  }

  // ---- selection -------------------------------------------------------------------------------
  struct Sel {
    uint32_t u;
    int32_t u_weight;
    uint32_t initial_cluster;
    int32_t initial_cluster_weight;
    uint32_t best_cluster;
    int32_t best_gain;
    int32_t best_cluster_weight;
    int32_t overall_best_gain;
  };

  // lp_clusterer.cc:181-280 over entries (keys[i], vals[i]), i < cnt; returns the favored cluster
  KMP_HD uint32_t select_cluster(bool store_favored, Sel &st, const uint32_t *keys, const int32_t *vals, uint32_t cnt) {
    uint32_t favored_cluster = st.initial_cluster;
    const int32_t mx = a.max_cluster_weight;
    if (a.tie_uniform) {
      uint32_t ntb = 0, ntf = 0;
      for (uint32_t i = 0; i < cnt; ++i) {
        const uint32_t c = keys[i];
        const int32_t gain = vals[i];
        const int32_t cw = a.weight[c];
        const bool comm_ok = !a.communities || a.communities[c] == a.communities[st.initial_cluster];
        const bool accept = (cw + st.u_weight <= mx || c == st.initial_cluster) && comm_ok;
        if (store_favored) {
          if (gain > st.overall_best_gain) {
            st.overall_best_gain = gain;
            favored_cluster = c;
            ntf = 0;
            a.tie_fav[ntf++] = c;
          } else if (gain == st.overall_best_gain) {
            a.tie_fav[ntf++] = c;
          }
        }
        if (gain > st.best_gain) {
          if (accept) {
            ntb = 0;
            a.tie_best[ntb++] = c;
            st.best_cluster = c;
            st.best_gain = gain;
          }
        } else if (gain == st.best_gain) {
          if (accept) {
            a.tie_best[ntb++] = c;
          }
        }
      }
      if (ntb > 1) {
        st.best_cluster = a.tie_best[random_index(rand, 0, ntb)];
      }
      if (ntf > 1) {
        favored_cluster = a.tie_fav[random_index(rand, 0, ntf)];
      }
      return favored_cluster;
    }
    for (uint32_t i = 0; i < cnt; ++i) { // GEOMETRIC (:252-278)
      const uint32_t c = keys[i];
      const int32_t gain = vals[i];
      const int32_t cw = a.weight[c];
      if (store_favored && gain > st.overall_best_gain) {
        st.overall_best_gain = gain;
        favored_cluster = c;
      }
      const bool comm_ok = !a.communities || a.communities[c] == a.communities[st.initial_cluster];
      const bool acc = (gain > st.best_gain || (gain == st.best_gain && random_bool(rand))) &&
                       (cw + st.u_weight <= mx || c == st.initial_cluster) && comm_ok;
      if (acc) {
        st.best_cluster = c;
        st.best_cluster_weight = cw;
        st.best_gain = gain;
      }
    }
    return favored_cluster;
  }

  // lp_refiner.cc:151-285
  KMP_HD uint32_t select_refine(Sel &st, const uint32_t *keys, const int32_t *vals, uint32_t cnt) {
    if (st.initial_cluster_weight - st.u_weight < min_w(st.initial_cluster)) { // :160-162
      return st.initial_cluster;
    }
    const int32_t initial_overload = st.initial_cluster_weight - a.max_bw[st.initial_cluster];
    if (a.tie_uniform) {
      uint32_t ntb = 0;
      for (uint32_t i = 0; i < cnt; ++i) {
        const uint32_t c = keys[i];
        const int32_t gain = vals[i];
        const int32_t cw = a.weight[c];
        const int32_t cmax = a.max_bw[c];
        const int32_t cover = cw - cmax;
        const bool feasible = (cw + st.u_weight <= cmax) || cover < initial_overload || c == st.initial_cluster;
        if (gain > st.best_gain) {
          if (feasible) {
            ntb = 0;
            a.tie_best[ntb++] = c;
            st.best_cluster = c;
            st.best_cluster_weight = cw;
            st.best_gain = gain;
          }
        } else if (gain == st.best_gain) {
          const int32_t best_over = st.best_cluster_weight - a.max_bw[st.best_cluster];
          if (cover < best_over) {
            if (feasible) {
              ntb = 0;
              a.tie_best[ntb++] = c;
              st.best_cluster = c;
              st.best_cluster_weight = cw;
            }
          } else if (cover == best_over) {
            if (feasible) {
              a.tie_best[ntb++] = c;
            }
          }
        }
      }
      if (ntb > 1) {
        st.best_cluster = a.tie_best[random_index(rand, 0, ntb)];
      }
      return st.initial_cluster;
    }
    for (uint32_t i = 0; i < cnt; ++i) { // GEOMETRIC (:246-284)
      const uint32_t c = keys[i];
      const int32_t gain = vals[i];
      const int32_t cw = a.weight[c];
      const int32_t cmax = a.max_bw[c];
      const int32_t best_over = st.best_cluster_weight - a.max_bw[st.best_cluster];
      const int32_t cover = cw - cmax;
      const bool acc =
          (gain > st.best_gain || (gain == st.best_gain && (cover < best_over || (cover == best_over && random_bool(rand))))) &&
          ((cw + st.u_weight <= cmax) || cover < initial_overload || c == st.initial_cluster);
      if (acc) {
        st.best_cluster = c;
        st.best_cluster_weight = cw;
        st.best_gain = gain;
      }
    }
    return st.initial_cluster;
  }

  KMP_HD uint32_t select(bool store_favored, Sel &st, const uint32_t *keys, const int32_t *vals, uint32_t cnt) {
    return a.mode == 0 ? select_cluster(store_favored, st, keys, vals, cnt) : select_refine(st, keys, vals, cnt);
  }

  // try_node_move (:817-841) + activate_neighbors (:848-870); returns moved, sets emptied
  KMP_HD bool try_node_move(uint32_t u, int32_t u_weight, uint32_t u_cluster, uint32_t new_cluster, bool &emptied) {
    emptied = false;
    if (a.label[u] != new_cluster) {
      if (move_cluster_weight(u_cluster, new_cluster, u_weight, max_w(new_cluster))) {
        a.label[u] = new_cluster;
        for (uint32_t e = a.xadj[u]; e < a.xadj[u + 1]; ++e) {
          a.active[a.adjncy[e]] = 1;
        }
        emptied = a.weight[u_cluster] == 0;
        return true;
      }
    }
    return false;
  }

  KMP_HD bool store_favored_for(int32_t u_weight, uint32_t u_cluster, int32_t icw) const {
    return a.mode == 0 && u_weight == icw && icw <= max_w(u_cluster) / 2; // :520-522 (kUseTwoHopClustering)
  }

  // handle_node -> find_best_cluster (:330-368, :460-541); first-phase variant (:543-638)
  KMP_HD bool handle_node(uint32_t u, bool first_phase, bool &emptied) {
    emptied = false;
    const int32_t u_weight = nw(u);
    const uint32_t u_cluster = a.label[u];
    const int32_t icw = a.weight[u_cluster];
    Sel st{u, u_weight, u_cluster, icw, u_cluster, 0, icw, 0};
    const uint32_t begin = a.xadj[u];
    uint32_t end = a.xadj[u + 1];
    if (a.max_num_neighbors != kInvalid && end - begin > a.max_num_neighbors) { // csr_graph.h:220-263
      end = begin + a.max_num_neighbors;
    }
    bool deferred = false;
    for (uint32_t e = begin; e < end; ++e) {
      const uint32_t v = a.adjncy[e];
      if (accept_neighbor(u, v)) {
        map_add(a.label[v], ew(e));
        if (first_phase && map_size >= kRatingMapThreshold) { // :576-579
          deferred = true;
          break;
        }
      }
    }
    a.stats->edges_scanned += end - begin;
    a.stats->nodes_visited += 1;
    if (deferred) { // :598-602 -- the active flag is NOT cleared
      map_clear();
      a.second_phase_nodes[num_second++] = u;
      return false;
    }
    a.active[u] = 0; // :507-508
    const bool store_favored = store_favored_for(u_weight, u_cluster, icw);
    const uint32_t favored = select(store_favored, st, a.ent_key, a.ent_val, map_size);
    if (store_favored && st.best_cluster == st.initial_cluster) {
      a.favored[u] = favored;
    }
    map_clear();
    return try_node_move(u, u_weight, u_cluster, st.best_cluster, emptied);
  }

  // handle_second_phase_node -> find_best_cluster_second_phase (:424-436, :640-815) at one thread
  KMP_HD bool handle_second_phase_node(uint32_t u, bool &emptied) {
    const int32_t u_weight = nw(u);
    const uint32_t u_cluster = a.label[u];
    const int32_t icw = a.weight[u_cluster];
    const uint32_t begin = a.xadj[u];
    uint32_t end = a.xadj[u + 1];
    if (a.max_num_neighbors != kInvalid && end - begin > a.max_num_neighbors) {
      end = begin + a.max_num_neighbors;
    }
    for (uint32_t e = begin; e < end; ++e) {
      const uint32_t v = a.adjncy[e];
      if (accept_neighbor(u, v)) {
        map2_add(a.label[v], ew(e));
        if (map2_size >= kRatingMapThreshold) {
          flush_small_map();
        }
      }
    }
    flush_small_map(); // :682-688
    a.stats->edges_scanned += end - begin;
    a.stats->nodes_visited += 1;
    a.active[u] = 0; // :690-691
    const bool store_favored = store_favored_for(u_weight, u_cluster, icw);
    uint32_t favored_cluster = u_cluster, best_cluster = u_cluster;
    int32_t best_gain = 0;
    int32_t l_best_gain = -1, l_fav_gain = -1;
    uint32_t l_best = 0, l_fav = 0;
    if (used_size != 0) {
      // entries in first-touch order; the first-phase map's entry arrays are free here
      for (uint32_t i = 0; i < used_size; ++i) {
        a.ent_key[i] = a.used_entries[i];
        a.ent_val[i] = a.concurrent[a.used_entries[i]];
      }
      Sel st{u, u_weight, u_cluster, icw, u_cluster, 0, icw, 0};
      const uint32_t lf = select(store_favored, st, a.ent_key, a.ent_val, used_size);
      l_best_gain = st.best_gain;
      l_best = st.best_cluster;
      l_fav_gain = a.concurrent[lf];
      l_fav = lf;
      for (uint32_t i = 0; i < used_size; ++i) {
        a.concurrent[a.used_entries[i]] = 0;
      }
      used_size = 0;
    }
    int32_t fav_gain = 0; // global reduction over one thread-local state (:742-806)
    if (l_best_gain > best_gain) {
      best_gain = l_best_gain;
      best_cluster = l_best;
    }
    if (store_favored && l_fav_gain > fav_gain) {
      fav_gain = l_fav_gain;
      favored_cluster = l_fav;
    }
    if (store_favored && best_cluster == u_cluster) {
      a.favored[u] = favored_cluster;
    }
    return try_node_move(u, u_weight, u_cluster, best_cluster, emptied);
  }
  KMP_HD void flush_small_map() { // :649-659
    for (uint32_t i = 0; i < map2_size; ++i) {
      const uint32_t c = a.ent2_key[i];
      const int32_t prev = a.concurrent[c];
      a.concurrent[c] += a.ent2_val[i];
      if (prev == 0) {
        a.used_entries[used_size++] = c;
      }
      a.slot2[c] = 0;
    }
    map2_size = 0;
  }

  // ---- schedule ----------------------------------------------------------------------------------
  KMP_HD static uint32_t floor_log2(uint32_t x) { // x >= 1
    uint32_t r = 0;
    while (x >>= 1) {
      ++r;
    }
    return r;
  }
  KMP_HD static uint32_t isqrt_trunc(uint32_t x) { // static_cast<T>(std::sqrt(double(x))): exact floor
    uint32_t r = 0;
    for (uint32_t bit = 1u << 15; bit != 0; bit >>= 1) {
      const uint32_t t = r | bit;
      if (static_cast<uint64_t>(t) * t <= x) {
        r = t;
      }
    }
    return r;
  }
  // CSRGraph::init_degree_buckets (csr_graph.cc:199-248); degree_bucket(d) = 0 if d == 0 else floor(log2 d) + 1
  // (kaminpar-common/degree_buckets.h:17-26)
  KMP_HD void init_buckets() {
    constexpr int kSlots = 34; // kNumberOfDegreeBuckets<uint32_t> + 1
    for (int i = 0; i < kSlots; ++i) {
      a.buckets[i] = 0;
    }
    if (a.sorted) {
      for (uint32_t u = 0; u < a.n; ++u) {
        const uint32_t d = deg(u);
        ++a.buckets[(d == 0 ? 0 : floor_log2(d) + 1) + 1];
      }
      int last = kSlots - 1;
      while (last >= 0 && a.buckets[last] == 0) {
        --last;
      }
      num_buckets = last < 0 ? 0 : static_cast<uint32_t>(last);
    } else {
      a.buckets[1] = a.n;
      num_buckets = 1;
    }
    for (int i = 1; i < kSlots; ++i) {
      a.buckets[i] += a.buckets[i - 1];
    }
  }

  // init_chunks (:1736-1854) at one thread, from = 0, to = n
  KMP_HD void init_chunks() {
    num_chunks = 0;
    num_bucket_ranges = 0;
    const uint32_t to = a.n;
    const uint32_t max_degree = a.large_degree_threshold;
    uint32_t max_bucket = floor_log2(max_degree == 0 ? 1 : max_degree);
    if (max_bucket > num_buckets) {
      max_bucket = num_buckets;
    }
    const uint32_t sm = isqrt_trunc(a.m), sn = isqrt_trunc(a.n);
    const uint32_t max_chunk_size = sm > 1024 ? sm : 1024;
    const uint32_t max_node_chunk_size = sn > 1024 ? sn : 1024;
    uint32_t position = 0;
    for (uint32_t bucket = 0; bucket < max_bucket; ++bucket) {
      const uint32_t bsz = a.buckets[bucket + 1] - a.buckets[bucket];
      if (bsz == 0) {
        continue;
      }
      if (position >= to) {
        break;
      }
      uint32_t bsize = bsz;
      if (to - position < bsize) {
        bsize = to - position;
      }
      const uint32_t bstart = a.buckets[bucket];
      const uint32_t chunks_start = num_chunks;
      uint32_t offset = 0;
      while (offset < bsize) {
        const uint32_t begin = offset;
        offset += max_node_chunk_size;
        const uint32_t end = begin + max_node_chunk_size < bsize ? begin + max_node_chunk_size : bsize;
        uint32_t cur = 0;
        uint32_t chunk_start = bstart + begin;
        for (uint32_t i = begin; i < end; ++i) {
          const uint32_t u = bstart + i;
          cur += deg(u);
          if (cur >= max_chunk_size) {
            a.chunks[2 * num_chunks] = chunk_start;
            a.chunks[2 * num_chunks + 1] = u + 1;
            ++num_chunks;
            chunk_start = u + 1;
            cur = 0;
          }
        }
        if (cur > 0) {
          a.chunks[2 * num_chunks] = chunk_start;
          a.chunks[2 * num_chunks + 1] = bstart + end;
          ++num_chunks;
        }
      }
      bucket_start[num_bucket_ranges] = chunks_start;
      bucket_end[num_bucket_ranges] = num_chunks;
      ++num_bucket_ranges;
      position += bsz;
    }
  }

  KMP_HD bool should_stop() const { return current_num_clusters <= static_cast<long long>(a.desired_num_clusters); } // :260-265

  // perform / perform_first_phase (:1863-2020) at one thread
  KMP_HD uint32_t perform(bool first_phase) {
    uint32_t moved = 0;
    for (uint32_t chunk_id = 0; chunk_id < num_chunks; ++chunk_id) {
      if (should_stop()) {
        continue; // the task returns before claiming a chunk (:1868-1870, :1880)
      }
      uint32_t removed = 0;
      const uint32_t cstart = a.chunks[2 * next_chunk], cend = a.chunks[2 * next_chunk + 1];
      ++next_chunk;
      const uint32_t *perm = rand.perms[random_index(rand, 0, kNumPerms)];
      const uint32_t num_sub = (cend - cstart + 63) / 64; // ceil(1.0 * size / 64)
      for (uint32_t i = 0; i < num_sub; ++i) {
        a.sub_perm[i] = i;
      }
      shuffle(rand, a.sub_perm, num_sub);
      for (uint32_t sc = 0; sc < num_sub; ++sc) {
        for (uint32_t i = 0; i < 64; ++i) {
          const uint32_t u = cstart + 64 * a.sub_perm[sc] + perm[i % 64];
          if (u >= cend || !a.active[u]) {
            continue;
          }
          if (deg(u) < a.large_degree_threshold) {
            bool emptied;
            moved += handle_node(u, first_phase, emptied) ? 1 : 0;
            removed += emptied ? 1 : 0;
          }
        }
      }
      current_num_clusters -= removed;
    }
    return moved;
  }

  // perform_iteration (:1681-1733)
  KMP_HD uint32_t perform_iteration() {
    if (num_chunks == 0) {
      init_chunks();
    }
    for (uint32_t b = 0; b < num_bucket_ranges; ++b) { // shuffle_chunks (:1856-1861)
      shuffle(rand, a.chunks + 2 * static_cast<uint64_t>(bucket_start[b]), bucket_end[b] - bucket_start[b], 2);
    }
    next_chunk = 0;
    uint32_t moved = 0;
    if (a.impl == 1) { // TWO_PHASE
      moved += perform(true);
      if (num_second != 0) { // perform_second_phase (:2022-2051)
        for (uint32_t i = 0; i < num_second; ++i) {
          bool emptied;
          moved += handle_second_phase_node(a.second_phase_nodes[i], emptied) ? 1 : 0;
          if (emptied) {
            --current_num_clusters;
          }
        }
        num_second = 0;
      }
    } else { // SINGLE_PHASE; GROWING_HASH_TABLES has the same observable semantics (insertion order)
      moved += perform(false);
    }
    return moved;
  }

  // ---- clusterer post passes ---------------------------------------------------------------------
  KMP_HD void isolated_nodes(bool match) { // :884-917
    uint32_t cluster = kInvalid;
    for (uint32_t u = 0; u < a.n; ++u) {
      if (deg(u) == 0) {
        const uint32_t cu = a.label[u];
        if (cluster != kInvalid && move_cluster_weight(cu, cluster, a.weight[cu], a.max_cluster_weight)) {
          a.label[u] = cluster;
          if (match) {
            cluster = kInvalid;
          }
        } else {
          cluster = cu;
        }
      }
    }
  }
  KMP_HD bool considered(uint32_t u) const { // :939-975 with _relabeled == false / :1038-1058
    if (deg(u) == 0 || u != a.label[u]) {
      return false;
    }
    const int32_t cw = a.weight[u];
    return !(cw > a.max_cluster_weight / 2 || cw != nw(u));
  }
  KMP_HD void two_hop_threadwise(bool match) { // :931-1016
    for (uint32_t u = 0; u < a.n; ++u) {
      a.match_map[u] = 0;
    }
    for (uint32_t u = 0; u < a.n; ++u) {
      if (!considered(u)) {
        continue;
      }
      const uint32_t c_u = a.label[u];
      uint32_t &rep_key = a.match_map[a.favored[u]];
      if (rep_key == 0) {
        rep_key = c_u + 1;
      } else {
        const uint32_t rep = rep_key - 1;
        const bool could = move_cluster_weight(c_u, rep, a.weight[c_u], a.max_cluster_weight);
        if (match) {
          a.label[u] = rep;
          rep_key = 0;
        } else if (could) {
          a.label[u] = rep;
        } else {
          rep_key = c_u + 1;
        }
      }
    }
  }
  KMP_HD void two_hop_global(bool match) { // :1030-1191
    for (uint32_t u = 0; u < a.n; ++u) { // :1064-1077
      if (considered(u)) {
        const uint32_t c = a.favored[u];
        if (considered(c) && move_cluster_weight(u, c, a.weight[u], a.max_cluster_weight)) {
          a.label[u] = c;
          --current_num_clusters;
        }
      } else {
        a.favored[u] = u;
      }
    }
    for (uint32_t u = 0; u < a.n; ++u) { // :1107-1190
      if (should_stop() || !considered(u)) {
        continue;
      }
      const uint32_t C = a.favored[u];
      uint32_t &sync = a.favored[C];
      const uint32_t cluster = sync;
      if (cluster == C) {
        sync = u;
        continue;
      }
      if (match) {
        sync = C;
        move_cluster_weight(u, cluster, a.weight[u], a.max_cluster_weight);
        a.label[u] = cluster;
        --current_num_clusters;
      } else if (move_cluster_weight(u, cluster, a.weight[u], a.max_cluster_weight)) {
        a.label[u] = cluster;
        --current_num_clusters;
      } else {
        sync = C;
      }
    }
  }
  KMP_HD void post_passes() { // lp_clusterer.cc:107-166
    const bool two_hop = (1.0 - 1.0 * static_cast<double>(current_num_clusters) / a.n) <= a.two_hop_threshold;
    switch (a.isolated_nodes_strategy) {
    case 1: isolated_nodes(true); break;
    case 2: isolated_nodes(false); break;
    case 3: if (two_hop) { isolated_nodes(true); } break;
    case 4: if (two_hop) { isolated_nodes(false); } break;
    default: break;
    }
    if (!two_hop) {
      return;
    }
    a.stats->two_hop_ran = 1;
    switch (a.two_hop_strategy) {
    case 1: two_hop_global(true); break;
    case 2: two_hop_threadwise(true); break;
    case 3: two_hop_global(false); break;
    case 4: two_hop_threadwise(false); break;
    default: break;
    }
  }

  // ---- drivers -----------------------------------------------------------------------------------
  // LPClusteringImpl::compute_clustering (lp_clusterer.cc:89-109) / LPRefinerImpl::refine (lp_refiner.cc:68-89)
  KMP_HD void run() {
    Stats &st = *a.stats;
    st.iterations = 0;
    st.edges_scanned = st.nodes_visited = 0;
    st.num_clusters = st.two_hop_ran = 0;
    const uint32_t num_keys = a.mode == 0 ? a.n : a.k;
    initial_num_clusters = num_keys;
    current_num_clusters = num_keys;
    for (uint32_t u = 0; u < a.n; ++u) { // initialize (:242-253, :1194-1220)
      a.active[u] = 1;
    }
    if (a.mode == 0) {
      for (uint32_t u = 0; u < a.n; ++u) {
        a.label[u] = u;
        a.favored[u] = u;
        a.weight[u] = nw(u);
      }
    } else {
      for (uint32_t b = 0; b < a.k; ++b) {
        a.weight[b] = 0;
      }
      for (uint32_t u = 0; u < a.n; ++u) {
        a.weight[a.label[u]] += nw(u);
      }
    }
    for (uint32_t c = 0; c < num_keys; ++c) {
      a.slot[c] = 0;
      a.slot2[c] = 0;
      a.concurrent[c] = 0;
    }
    num_chunks = 0;
    init_buckets();
    const unsigned long long max_it = (a.mode == 1 && a.num_iterations == 0) ? ~0ull : a.num_iterations;
    for (unsigned long long it = 0; it < max_it; ++it) {
      const uint32_t moved = perform_iteration();
      if (it < 64) {
        st.moved[it] = moved;
        st.iterations = static_cast<uint32_t>(it + 1);
      }
      if (moved == 0) {
        break;
      }
    }
    if (a.mode == 0) {
      if (a.n > 0) {
        post_passes();
      }
      st.num_clusters = static_cast<uint32_t>(current_num_clusters > 0 ? current_num_clusters : 0);
    }
  }
};

#if defined(__CUDACC__)
__global__ void strict_seed_kernel(Rng *rng, int seed) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    rng_init(*rng, seed);
  }
}
// ONE thread walks the reference's sequential schedule; the other lanes of its warp idle (the algorithm is
// a dependency chain by definition -- every decision reads the weights all earlier moves left behind).
__global__ void strict_kernel(const Args a) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    Engine e(a);
    e.run();
  }
}
#endif

} // namespace kmp_strict
