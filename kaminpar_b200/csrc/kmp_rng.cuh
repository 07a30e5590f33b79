// The reference's thread-local Random (kaminpar-common/random.h:27-125, random.cc:18-56) at thread index 0, restated
// as KMP_HD code: std::mt19937, libstdc++ 13's uniform_int_distribution and std::shuffle, and the 1024 precomputed
// random bools. Shared by the seq_strict LP engine (lp_strict.cuh) and the initial bipartitioner
// (kmp_bipartition.cuh); each keeps its own RandomPermutations tables, whose sizes differ.
// tests/cpp/strict_host_check.cc pins these restatements against the real std:: facilities on the host.
#pragma once

#include <cstdint>

#if defined(__CUDACC__)
#define KMP_HD __host__ __device__
#else
#define KMP_HD
#endif

namespace kmp_rng {

constexpr uint32_t kBools = 1024;

struct RngCore {
  uint32_t mt[624];
  uint32_t idx;
  uint8_t bools[kBools];
  uint32_t next_bool;
};

KMP_HD inline void mt_seed(RngCore &r, uint32_t seed) {
  r.mt[0] = seed;
  for (uint32_t i = 1; i < 624; ++i) {
    r.mt[i] = 1812433253u * (r.mt[i - 1] ^ (r.mt[i - 1] >> 30)) + i;
  }
  r.idx = 624;
}
KMP_HD inline uint32_t mt_next(RngCore &r) {
  if (r.idx >= 624) {
    for (uint32_t i = 0; i < 624; ++i) {
      const uint32_t y = (r.mt[i] & 0x80000000u) | (r.mt[(i + 1) % 624] & 0x7FFFFFFFu);
      r.mt[i] = r.mt[(i + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908B0DFu : 0u);
    }
    r.idx = 0;
  }
  uint32_t y = r.mt[r.idx++];
  y ^= y >> 11;
  y ^= (y << 7) & 0x9D2C5680u;
  y ^= (y << 15) & 0xEFC60000u;
  y ^= y >> 18;
  return y;
}
// uniform_int_distribution<T>(0, range - 1) on a 32-bit generator, 1 <= range <= 2^32 - 1 (_S_nd<uint64_t>)
KMP_HD inline uint32_t uniform_below(RngCore &r, uint32_t range) {
  uint64_t product = static_cast<uint64_t>(mt_next(r)) * range;
  uint32_t low = static_cast<uint32_t>(product);
  if (low < range) {
    const uint32_t threshold = (0u - range) % range;
    while (low < threshold) {
      product = static_cast<uint64_t>(mt_next(r)) * range;
      low = static_cast<uint32_t>(product);
    }
  }
  return static_cast<uint32_t>(product >> 32);
}
// std::shuffle(first, first + size, gen) over 32-bit elements; stride: elements are `stride` words wide
// (chunks are {start, end} pairs) -- the index sequence does not depend on the element type
KMP_HD inline void swap_elems(uint32_t *a, uint64_t i, uint64_t j, uint32_t stride) {
  for (uint32_t q = 0; q < stride; ++q) {
    const uint32_t t = a[i * stride + q];
    a[i * stride + q] = a[j * stride + q];
    a[j * stride + q] = t;
  }
}
KMP_HD inline void shuffle(RngCore &r, uint32_t *a, uint64_t size, uint32_t stride = 1) {
  if (size == 0) {
    return;
  }
  const uint64_t urngrange = 0xFFFFFFFFull;
  if (urngrange / size >= size) {
    uint64_t i = 1;
    if ((size % 2) == 0) {
      swap_elems(a, i, uniform_below(r, 2), stride);
      ++i;
    }
    while (i != size) {
      const uint64_t swap_range = i + 1;
      const uint32_t x = uniform_below(r, static_cast<uint32_t>(swap_range * (swap_range + 1)));
      const uint64_t p0 = x / (swap_range + 1), p1 = x % (swap_range + 1);
      swap_elems(a, i, p0, stride);
      ++i;
      swap_elems(a, i, p1, stride);
      ++i;
    }
    return;
  }
  for (uint64_t i = 1; i != size; ++i) {
    swap_elems(a, i, uniform_below(r, static_cast<uint32_t>(i + 1)), stride);
  }
}
// Random::reseed (random.cc:45-56) with thread index 0: the generator and the precomputed bools
KMP_HD inline void rng_seed(RngCore &r, int seed) {
  mt_seed(r, static_cast<uint32_t>(seed));
  r.next_bool = 0;
  for (uint32_t i = 0; i < kBools; ++i) {
    r.bools[i] = static_cast<uint8_t>(uniform_below(r, 2));
  }
}
KMP_HD inline uint32_t random_index(RngCore &r, uint32_t lo, uint32_t hi) { return lo + uniform_below(r, hi - lo); } // random.h:64-68
KMP_HD inline bool random_bool(RngCore &r) { return r.bools[r.next_bool++ % kBools] != 0; }                          // random.h:70-72

} // namespace kmp_rng
