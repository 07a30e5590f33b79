// Micro-benchmarks behind DESIGN.md's "what bounds the LP sweep": the rate of the memory operations a
// label-propagation sweep is made of, measured on the box the bench runs on.
//   gather4 / gather8 : v = adj[e] (coalesced), x = table[v] (random 4 B / 8 B element of an L2-resident table)
//   smem_cas_add      : per edge one atomicCAS + one atomicAdd on a shared-memory hash table
//   smem_plain        : per edge plain ld/st claims on a shared-memory table (optimistic insertion)
//   redg / atomg      : per edge one RED / one ATOM.EXCH on a random word of an L2-resident table
//   atom_same         : atomicAdd with return on ONE address, from lane 0 of every warp of the grid, at the tier-3
//                       team kernel's launch shape (6 x 256-thread CTAs per SM): the work-queue claim / proposal slot
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -o microbench_lsu microbench_lsu.cu
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

constexpr int kSMs = 132; // H100 SXM

#define CK(x)                                                                                              \
  do {                                                                                                     \
    cudaError_t e = (x);                                                                                   \
    if (e != cudaSuccess) {                                                                                \
      printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__);                                    \
      return 1;                                                                                            \
    }                                                                                                      \
  } while (0)

__host__ __device__ inline uint32_t mix(uint32_t x) {
  x ^= x >> 16;
  x *= 0x7FEB352Du;
  x ^= x >> 15;
  x *= 0x846CA68Bu;
  x ^= x >> 16;
  return x;
}

__global__ void k_fill_adj(uint32_t *adj, uint64_t m, uint32_t n) {
  for (uint64_t e = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; e < m; e += (uint64_t)gridDim.x * blockDim.x) {
    adj[e] = mix((uint32_t)e * 2654435761u + 12345u) % n;
  }
}
template <typename T> __global__ void k_fill_tab(T *t, uint32_t n) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    t[i] = (T)i;
  }
}

template <typename T, int B> __global__ void __launch_bounds__(256) k_gather(const uint32_t *__restrict__ adj, const T *__restrict__ tab, uint64_t m,
                                                     unsigned long long *out) {
  unsigned long long acc = 0;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x * B;
  for (uint64_t e0 = (uint64_t)blockIdx.x * blockDim.x * B + threadIdx.x; e0 < m; e0 += stride) {
    uint32_t v[B];
    T x[B];
#pragma unroll
    for (int j = 0; j < B; ++j) {
      const uint64_t e = e0 + (uint64_t)j * blockDim.x;
      v[j] = e < m ? adj[e] : 0;
    }
#pragma unroll
    for (int j = 0; j < B; ++j) {
      x[j] = tab[v[j]];
    }
#pragma unroll
    for (int j = 0; j < B; ++j) {
      acc += (unsigned long long)x[j];
    }
  }
  if (acc == 0x1234567ull) {
    out[0] = acc;
  }
}

// stream only (no gather): the coalesced part
template <int B> __global__ void __launch_bounds__(256) k_stream(const uint32_t *__restrict__ adj, uint64_t m, unsigned long long *out) {
  unsigned long long acc = 0;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x * B;
  for (uint64_t e0 = (uint64_t)blockIdx.x * blockDim.x * B + threadIdx.x; e0 < m; e0 += stride) {
#pragma unroll
    for (int j = 0; j < B; ++j) {
      const uint64_t e = e0 + (uint64_t)j * blockDim.x;
      acc += e < m ? adj[e] : 0;
    }
  }
  if (acc == 0x1234567ull) {
    out[0] = acc;
  }
}

// per CTA: E edges per "vertex" into a shared table of C slots, CAS + add; then clear
template <int T, int EPT, int C> __global__ void __launch_bounds__(T) k_smem_cas_add(const uint32_t *__restrict__ adj, uint64_t m, unsigned long long *out) {
  extern __shared__ uint32_t sm[];
  uint32_t *keys = sm;
  int *vals = (int *)(sm + C);
  for (int s = threadIdx.x; s < C; s += T) {
    keys[s] = 0xFFFFFFFFu;
    vals[s] = 0;
  }
  __syncthreads();
  unsigned long long acc = 0;
  const uint64_t per = (uint64_t)T * EPT;
  for (uint64_t base = blockIdx.x * per; base + per <= m; base += gridDim.x * per) {
    uint32_t c[EPT];
    uint32_t slot[EPT];
#pragma unroll
    for (int j = 0; j < EPT; ++j) {
      c[j] = adj[base + j * T + threadIdx.x]; // "labels": mostly distinct
    }
#pragma unroll
    for (int j = 0; j < EPT; ++j) {
      uint32_t s = mix(c[j]) & (C - 1);
      while (true) {
        const uint32_t prev = atomicCAS(&keys[s], 0xFFFFFFFFu, c[j]);
        if (prev == 0xFFFFFFFFu || prev == c[j]) {
          atomicAdd(&vals[s], 1);
          break;
        }
        s = (s + 1) & (C - 1);
      }
      slot[j] = s;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < EPT; ++j) {
      acc += vals[slot[j]];
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < EPT; ++j) {
      keys[slot[j]] = 0xFFFFFFFFu;
      vals[slot[j]] = 0;
    }
    __syncthreads();
  }
  if (acc == 0x1234567ull) {
    out[0] = acc;
  }
}

// optimistic: tags table (u32), labels in smem, plain stores + checks, stragglers by CAS, dups by atomicAdd
template <int T, int EPT, int C> __global__ void __launch_bounds__(T) k_smem_plain(const uint32_t *__restrict__ adj, uint64_t m, unsigned long long *out) {
  extern __shared__ uint32_t sm[];
  uint32_t *tag = sm;                  // C
  uint32_t *lab = sm + C;              // T*EPT
  int *accw = (int *)(sm + C + T * EPT); // T*EPT
  for (int s = threadIdx.x; s < C; s += T) {
    tag[s] = 0xFFFFFFFFu;
  }
  __syncthreads();
  unsigned long long acc = 0;
  const uint64_t per = (uint64_t)T * EPT;
  for (uint64_t base = blockIdx.x * per; base + per <= m; base += gridDim.x * per) {
    uint32_t pos[EPT];
    uint32_t rep[EPT];
    uint32_t pending = 0;
#pragma unroll
    for (int j = 0; j < EPT; ++j) {
      const uint32_t e = j * T + threadIdx.x;
      const uint32_t c = adj[base + e];
      lab[e] = c;
      accw[e] = 0;
      pos[j] = mix(c) & (C - 1);
      rep[j] = 0xFFFFFFFFu;
      pending |= 1u << j;
    }
    __syncthreads();
    for (int round = 0; round < 3 && __syncthreads_or(pending != 0); ++round) {
#pragma unroll
      for (int j = 0; j < EPT; ++j) {
        if ((pending >> j) & 1u) {
          if (tag[pos[j]] == 0xFFFFFFFFu) {
            tag[pos[j]] = j * T + threadIdx.x;
          }
        }
      }
      __syncthreads();
#pragma unroll
      for (int j = 0; j < EPT; ++j) {
        if ((pending >> j) & 1u) {
          const uint32_t e = j * T + threadIdx.x;
          const uint32_t t = tag[pos[j]];
          if (t == e) {
            rep[j] = e;
            pending &= ~(1u << j);
          } else if (lab[t] == lab[e]) {
            rep[j] = t;
            pending &= ~(1u << j);
          } else {
            pos[j] = (pos[j] + 1) & (C - 1);
          }
        }
      }
    }
    // stragglers
#pragma unroll
    for (int j = 0; j < EPT; ++j) {
      if ((pending >> j) & 1u) {
        const uint32_t e = j * T + threadIdx.x;
        while (true) {
          const uint32_t t = atomicCAS(&tag[pos[j]], 0xFFFFFFFFu, e);
          if (t == 0xFFFFFFFFu) {
            rep[j] = e;
            break;
          }
          if (lab[t] == lab[e]) {
            rep[j] = t;
            break;
          }
          pos[j] = (pos[j] + 1) & (C - 1);
        }
      }
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < EPT; ++j) {
      const uint32_t e = j * T + threadIdx.x;
      if (rep[j] != e) {
        atomicAdd(&accw[rep[j]], 1);
      }
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < EPT; ++j) {
      const uint32_t e = j * T + threadIdx.x;
      if (rep[j] == e) {
        acc += 1 + accw[e];
        tag[pos[j]] = 0xFFFFFFFFu;
      }
    }
    __syncthreads();
  }
  if (acc == 0x1234567ull) {
    out[0] = acc;
  }
}

template <int B, bool RET> __global__ void __launch_bounds__(256) k_gatom(const uint32_t *__restrict__ adj, int *tab, uint64_t m, unsigned long long *out) {
  unsigned long long acc = 0;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x * B;
  for (uint64_t e0 = (uint64_t)blockIdx.x * blockDim.x * B + threadIdx.x; e0 < m; e0 += stride) {
    uint32_t v[B];
#pragma unroll
    for (int j = 0; j < B; ++j) {
      const uint64_t e = e0 + (uint64_t)j * blockDim.x;
      v[j] = e < m ? adj[e] : 0;
    }
#pragma unroll
    for (int j = 0; j < B; ++j) {
      if (RET) {
        acc += atomicExch(&tab[v[j]], 0);
      } else {
        atomicAdd(&tab[v[j]], 1);
      }
    }
  }
  if (acc == 0x1234567ull) {
    out[0] = acc;
  }
}

// lane 0 of every warp: R atomicAdds with return on one word (the team kernels' queue claim and proposal slot)
template <int R> __global__ void __launch_bounds__(256) k_atom_same(uint32_t *ctr, unsigned long long *out) {
  if ((threadIdx.x & 31) != 0) {
    return;
  }
  uint32_t acc = 0;
  for (int r = 0; r < R; ++r) {
    acc += atomicAdd(ctr, 1u);
  }
  if (acc == 0x1234567u) {
    out[0] = acc;
  }
}

template <typename F> float time_ms(F f, int reps) {
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  f();
  f();
  cudaDeviceSynchronize();
  cudaEventRecord(a);
  for (int i = 0; i < reps; ++i) {
    f();
  }
  cudaEventRecord(b);
  cudaEventSynchronize(b);
  float ms = 0;
  cudaEventElapsedTime(&ms, a, b);
  return ms / reps;
}

int main() {
  const uint64_t m = 128ull << 20;
  uint32_t *adj;
  unsigned long long *out;
  CK(cudaMalloc(&adj, m * 4));
  CK(cudaMalloc(&out, 64));
  k_fill_adj<<<kSMs * 8, 256>>>(adj, m, 1u << 31);
  CK(cudaDeviceSynchronize());
  printf("{\"m\": %llu", (unsigned long long)m);
  {
    const float ms = time_ms([&] { k_stream<8><<<kSMs * 8, 256>>>(adj, m, out); }, 5);
    printf(", \"stream_Gedges_s\": %.1f", m / ms * 1e-6);
  }
  for (uint32_t n : {2400000u, 9000000u, 64000000u}) {
    uint32_t *t4;
    unsigned long long *t8;
    CK(cudaMalloc(&t4, (size_t)n * 4));
    CK(cudaMalloc(&t8, (size_t)n * 8));
    k_fill_adj<<<kSMs * 8, 256>>>(adj, m, n);
    k_fill_tab<<<kSMs * 8, 256>>>(t4, n);
    k_fill_tab<<<kSMs * 8, 256>>>(t8, n);
    CK(cudaDeviceSynchronize());
    float ms = time_ms([&] { k_gather<uint32_t, 8><<<kSMs * 8, 256>>>(adj, t4, m, out); }, 5);
    printf(", \"gather4_n%u_G_s\": %.1f", n, m / ms * 1e-6);
    ms = time_ms([&] { k_gather<unsigned long long, 8><<<kSMs * 8, 256>>>(adj, t8, m, out); }, 5);
    printf(", \"gather8_n%u_G_s\": %.1f", n, m / ms * 1e-6);
    ms = time_ms([&] { k_gather<uint32_t, 4><<<kSMs * 16, 256>>>(adj, t4, m, out); }, 5);
    printf(", \"gather4_b4_n%u_G_s\": %.1f", n, m / ms * 1e-6);
    ms = time_ms([&] { k_gather<uint32_t, 16><<<kSMs * 4, 256>>>(adj, t4, m, out); }, 5);
    printf(", \"gather4_b16_n%u_G_s\": %.1f", n, m / ms * 1e-6);
    if (n == 2400000u) {
      ms = time_ms([&] { k_gatom<8, false><<<kSMs * 8, 256>>>(adj, (int *)t4, m, out); }, 3);
      printf(", \"redg_G_s\": %.1f", m / ms * 1e-6);
      ms = time_ms([&] { k_gatom<8, true><<<kSMs * 8, 256>>>(adj, (int *)t4, m, out); }, 3);
      printf(", \"atomg_exch_G_s\": %.1f", m / ms * 1e-6);
    }
    cudaFree(t4);
    cudaFree(t8);
  }
  // shared-memory aggregation: labels drawn from 2^22 values (mostly distinct within 8192)
  k_fill_adj<<<kSMs * 8, 256>>>(adj, m, 1u << 22);
  CK(cudaDeviceSynchronize());
  {
    constexpr int T = 512, EPT = 16, C = 16384;
    const size_t smem = C * 8;
    CK(cudaFuncSetAttribute(k_smem_cas_add<T, EPT, C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    float ms = time_ms([&] { k_smem_cas_add<T, EPT, C><<<kSMs * 1, T, smem>>>(adj, m, out); }, 3);
    printf(", \"smem_cas_add_1cta_G_s\": %.1f", m / ms * 1e-6);
    ms = time_ms([&] { k_smem_cas_add<T, EPT, C><<<kSMs * 2, T, smem>>>(adj, m, out); }, 3);
    printf(", \"smem_cas_add_2cta_G_s\": %.1f", m / ms * 1e-6);
    const size_t smem2 = (C + 2 * T * EPT) * 4;
    CK(cudaFuncSetAttribute(k_smem_plain<T, EPT, C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
    ms = time_ms([&] { k_smem_plain<T, EPT, C><<<kSMs * 1, T, smem2>>>(adj, m, out); }, 3);
    printf(", \"smem_plain_1cta_G_s\": %.1f", m / ms * 1e-6);
    ms = time_ms([&] { k_smem_plain<T, EPT, C><<<kSMs * 2, T, smem2>>>(adj, m, out); }, 3);
    printf(", \"smem_plain_2cta_G_s\": %.1f", m / ms * 1e-6);
  }
  {
    constexpr int T = 128, EPT = 8, C = 2048;
    const size_t smem = C * 8;
    float ms = time_ms([&] { k_smem_cas_add<T, EPT, C><<<kSMs * 8, T, smem>>>(adj, m, out); }, 3);
    printf(", \"smem_cas_add_t128_G_s\": %.1f", m / ms * 1e-6);
    const size_t smem2 = (C + 2 * T * EPT) * 4;
    ms = time_ms([&] { k_smem_plain<T, EPT, C><<<kSMs * 8, T, smem2>>>(adj, m, out); }, 3);
    printf(", \"smem_plain_t128_G_s\": %.1f", m / ms * 1e-6);
  }
  {
    constexpr int R = 256;
    const uint32_t blocks = kSMs * 6;
    uint32_t *ctr;
    CK(cudaMalloc(&ctr, 4));
    CK(cudaMemset(ctr, 0, 4));
    const float ms = time_ms([&] { k_atom_same<R><<<blocks, 256>>>(ctr, out); }, 5);
    printf(", \"atom_same_addr_per_ns\": %.3f", (double)blocks * 8 * R / (ms * 1e6));
    cudaFree(ctr);
  }
  printf("}\n");
  return 0;
}
