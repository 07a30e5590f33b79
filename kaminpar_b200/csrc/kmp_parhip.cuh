// kaminpar_b200: the ParHIP reader on the device + its C ABI (include/kaminpar_b200_parhip.h, DESIGN.md §19).
// Included at the end of kmp_lp.cu after kmp_prepare.cuh and kmp_metis.cuh: the EXTERNAL ordering reuses the
// preparation's tile histogram and stable scatter (k_prep_count, k_prep_scatter) and the contraction's tile owners
// (k_tile_owners, owner_of_edge); kmp_read_parhip streams the file with kmp_read.cuh's stream_file.
//
// What it restates (see the header): csr_read and csr_read_deg_buckets (parhip_parser.cc:179-336).
//   The 24-byte header is read on the host, which lays out the sections and refuses n or m >= 2^31.
//   k_parhip_pass<SEC, W8>: one thread per 16-byte-aligned group of a section's bytes (4 entries at 32 bits, 2 at 64),
//     one 16-byte load (four 4-byte loads where 8-byte entries are not 8-byte aligned, or at the file's end); every
//     complete entry is checked and narrowed, and written where the call has an output for it. kmp_read_parhip launches it on the entries of each chunk as soon
//     as the chunk's copy is queued.
//   EXTERNAL: the offsets pass writes the file's xadj into scratch (n + 1 words) and the node-weight pass the file's
//     weights; k_prep_count buckets the degrees into per-tile histograms, a scan gives every (bucket, tile) its first
//     new id, k_prep_scatter writes old_to_new / new_to_old / the new degrees / vwgt stably, a scan of the degrees is
//     new_xadj. k_parhip_edges then copies the edges over tiles of kTileEdges NEW positions (a hub row spreads over
//     many CTAs), reading each target and edge weight at the file's width, checking it (the adjacency and edge-weight
//     passes are not run) and relabelling it through old_to_new. It does nothing when the offsets were refused,
//     since its owner search needs them valid; an offsets violation precedes every edge in file order.
//   A violation is one atomicMin of (offset << 8) | kind. The host adds the section totals and the truncation.
#pragma once

#include "../../include/kaminpar_b200_parhip.h"

struct kmp_parhip_graph : DeviceCsr { // vwgt / adjwgt: unallocated for absent weights
  uint32_t n = 0, m = 0;
  int sorted = 0;
  PoolBuf<uint32_t> old_to_new; // EXTERNAL only
};

namespace {

constexpr int kPhOffsets = KMP_PARHIP_SECTION_OFFSETS, kPhAdjncy = KMP_PARHIP_SECTION_ADJNCY,
              kPhVwgt = KMP_PARHIP_SECTION_VWGT, kPhAdjwgt = KMP_PARHIP_SECTION_ADJWGT;
constexpr unsigned long long kPhNone = ~0ull;

// device control block of one read; zeroed except for `first`
struct ParhipCtl {
  unsigned long long first;  // min over the violations of (offset << 8) | kind
  unsigned long long sum[2]; // node / edge weight totals of the accepted weights
};

struct ParhipArgs {
  const uint8_t *bytes;
  unsigned long long len;
  unsigned long long n, m, base; // base = the first byte of adjncy
  unsigned long long sec[5];     // first byte of each section (KMP_PARHIP_SECTION_*)
  uint32_t w[5];                 // entry width of each section (4 or 8)
  uint32_t *xadj, *adjncy;       // outputs; NULL: check only
  int32_t *vwgt, *adjwgt;
  ParhipCtl *ctl;
};

__device__ __forceinline__ void ph_violate(ParhipCtl *ctl, unsigned long long at, uint32_t kind) {
  atomicMin(&ctl->first, (at << 8) | kind);
}

__device__ __forceinline__ uint32_t ph_word(const uint8_t *b, unsigned long long at) {
  return __ldg(reinterpret_cast<const uint32_t *>(b + at));
}

// the entry at byte `at` (4-byte aligned) of width 8 or 4
__device__ __forceinline__ unsigned long long ph_entry(const uint8_t *b, unsigned long long at, bool w8) {
  return w8 ? (ph_word(b, at) | (static_cast<unsigned long long>(ph_word(b, at + 4)) << 32)) : ph_word(b, at);
}

// the 16 bytes [at, at + 16) as four words (at is 4-byte aligned; words past `len` are 0)
__device__ __forceinline__ void ph_load16(const uint8_t *b, unsigned long long at, unsigned long long len,
                                          uint32_t (&q)[4]) {
  if (at + 16 <= len && (at & 15u) == 0) {
    const uint4 v = __ldg(reinterpret_cast<const uint4 *>(b + at));
    q[0] = v.x;
    q[1] = v.y;
    q[2] = v.z;
    q[3] = v.w;
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      q[j] = at + 4 * j + 4 <= len ? ph_word(b, at + 4 * j) : 0u;
    }
  }
}

// a weight at its width, sign-extended
template <bool W8> __device__ __forceinline__ long long ph_signed(unsigned long long v) {
  return W8 ? static_cast<long long>(v) : static_cast<long long>(static_cast<int32_t>(static_cast<uint32_t>(v)));
}

// checks one weight; true if it is accepted
__device__ __forceinline__ bool ph_weight(ParhipCtl *ctl, unsigned long long at, long long s) {
  if (s < 1) {
    ph_violate(ctl, at, KMP_PARHIP_WEIGHT);
    return false;
  }
  if (s > 0x7FFFFFFFll) {
    ph_violate(ctl, at, KMP_PARHIP_TOO_LARGE);
    return false;
  }
  return true;
}

// checks one target; true if it is accepted
__device__ __forceinline__ bool ph_target(ParhipCtl *ctl, unsigned long long at, unsigned long long v,
                                          unsigned long long n) {
  if ((v >> 32) != 0) {
    ph_violate(ctl, at, KMP_PARHIP_TOO_LARGE);
    return false;
  }
  if (v >= n) {
    ph_violate(ctl, at, KMP_PARHIP_NEIGHBOR_OUT_OF_RANGE);
    return false;
  }
  return true;
}

// one atomic per warp for the weight total of section `which` (0 node, 1 edge); blockDim.x is a multiple of 32
__device__ __forceinline__ void ph_add_sum(ParhipCtl *ctl, int which, unsigned long long sum) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sum += __shfl_xor_sync(kFull, sum, o);
  }
  if ((threadIdx.x & 31u) == 0 && sum != 0) {
    atomicAdd(&ctl->sum[which], sum);
  }
}

// entries [i0, i1) of section SEC at width 8 (W8) or 4
template <int SEC, bool W8>
__global__ void __launch_bounds__(256) k_parhip_pass(ParhipArgs a, unsigned long long i0, unsigned long long i1) {
  constexpr uint32_t kW = W8 ? 8 : 4, kPer = 16 / kW;
  const unsigned long long start = a.sec[SEC];
  // groups of 16 bytes at absolute 16-byte boundaries, so that each is one 16-byte load; only 8-byte entries that
  // start 4 bytes off an 8-byte boundary (32-bit offsets, 64-bit ids, n even) would straddle them: those groups
  // start at the section and take four 4-byte loads
  const unsigned long long org = (start & (kW - 1)) == 0 ? start & ~15ull : start;
  const unsigned long long g0 = (start + i0 * kW - org) / 16, g1 = (start + i1 * kW - org + 15) / 16;
  const unsigned long long shift = a.w[kPhAdjncy] == 8 ? 3 : 2; // offsets count bytes of ids
  unsigned long long sum = 0;
  // warp-uniform trip count, so that every lane reaches the shuffles of ph_add_sum
  for (unsigned long long gb = g0 + static_cast<unsigned long long>(blockIdx.x) * blockDim.x; gb < g1;
       gb += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
    const unsigned long long g = gb + threadIdx.x;
    if (g >= g1) {
      continue;
    }
    uint32_t q[4];
    ph_load16(a.bytes, org + g * 16, a.len, q);
#pragma unroll
    for (uint32_t j = 0; j < kPer; ++j) {
      const unsigned long long at = org + g * 16 + j * kW;
      if (at < start) { // before the section: another section's bytes
        continue;
      }
      const unsigned long long i = (at - start) / kW;
      if (i < i0 || i >= i1 || at + kW > a.len) { // an incomplete entry: TRUNCATED, judged on the host
        continue;
      }
      const unsigned long long v = W8 ? (q[2 * j] | (static_cast<unsigned long long>(q[2 * j + 1]) << 32)) : q[j];
      if (SEC == kPhOffsets) {
        unsigned long long prev = 0;
        if (i > 0) {
          prev = j > 0 ? (W8 ? (q[2 * j - 2] | (static_cast<unsigned long long>(q[2 * j - 1]) << 32)) : q[j - 1])
                       : ph_entry(a.bytes, at - kW, W8);
        }
        const unsigned long long rel = v - a.base;
        const bool bad = (i == 0 && v != a.base) || (i > 0 && v < prev) || (rel & ((1ull << shift) - 1)) != 0 ||
                         (i == a.n && v != a.base + (a.m << shift));
        if (bad) {
          ph_violate(a.ctl, at, KMP_PARHIP_OFFSETS);
        } else if (a.xadj != nullptr) {
          a.xadj[i] = static_cast<uint32_t>(rel >> shift);
        }
      } else if (SEC == kPhAdjncy) {
        if (ph_target(a.ctl, at, v, a.n) && a.adjncy != nullptr) {
          a.adjncy[i] = static_cast<uint32_t>(v);
        }
      } else {
        const long long s = ph_signed<W8>(v);
        if (ph_weight(a.ctl, at, s)) {
          sum += static_cast<unsigned long long>(s);
          int32_t *out = SEC == kPhVwgt ? a.vwgt : a.adjwgt;
          if (out != nullptr) {
            out[i] = static_cast<int32_t>(s);
          }
        }
      }
    }
  }
  if (SEC == kPhVwgt || SEC == kPhAdjwgt) {
    ph_add_sum(a.ctl, SEC == kPhVwgt ? 0 : 1, sum);
  }
}

// EXTERNAL: new_adjncy[p] = old_to_new[target of file edge e], e = xadj_file[new_to_old[u]] + (p - new_xadj[u]) for
// the new vertex u owning p (forward order), with the edge weight; each file edge is read and checked once here.
__global__ void __launch_bounds__(256) k_parhip_edges(ParhipArgs a, uint32_t etiles, const uint32_t *__restrict__ file_xadj,
                                                      const uint32_t *__restrict__ new_xadj,
                                                      const uint32_t *__restrict__ tile_lo,
                                                      const uint32_t *__restrict__ new_to_old,
                                                      const uint32_t *__restrict__ old_to_new) {
  __shared__ uint32_t s_x[kTileVerts + 1];
  if (a.ctl->first < (a.sec[kPhAdjncy] << 8)) { // the offsets were refused: the owner search would index by them
    return;
  }
  const uint32_t m = static_cast<uint32_t>(a.m);
  const bool w8 = a.w[kPhAdjncy] == 8, ew = a.adjwgt != nullptr, ew8 = a.w[kPhAdjwgt] == 8;
  unsigned long long sum = 0;
  for (uint32_t t = blockIdx.x; t < etiles; t += gridDim.x) {
    const uint32_t p0 = t * kTileEdges;
    const uint32_t p1 = p0 + kTileEdges < m ? p0 + kTileEdges : m;
    const uint32_t u_lo = tile_lo[t], u_hi = tile_lo[t + 1];
    const bool staged = u_hi - u_lo + 2 <= kTileVerts + 1; // [u_lo, u_hi + 1]: every start and end the tile reads
    __syncthreads(); // the previous tile is done with s_x
    if (staged) {
      for (uint32_t i = threadIdx.x; i <= u_hi - u_lo + 1; i += blockDim.x) {
        s_x[i] = new_xadj[u_lo + i];
      }
    }
    __syncthreads();
    uint32_t e[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { // the owner searches of the eight positions are independent
      const uint32_t p = p0 + j * 256 + threadIdx.x;
      e[j] = 0;
      if (p < p1) {
        uint32_t u, begin;
        if (staged) {
          const uint32_t i = owner_of_edge(s_x, 0, u_hi - u_lo, p);
          u = u_lo + i;
          begin = s_x[i];
        } else {
          u = owner_of_edge(new_xadj, u_lo, u_hi, p);
          begin = new_xadj[u];
        }
        e[j] = file_xadj[new_to_old[u]] + (p - begin);
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t p = p0 + j * 256 + threadIdx.x;
      if (p < p1) {
        const unsigned long long at = a.sec[kPhAdjncy] + static_cast<unsigned long long>(e[j]) * (w8 ? 8 : 4);
        const unsigned long long v = ph_entry(a.bytes, at, w8);
        a.adjncy[p] = ph_target(a.ctl, at, v, a.n) ? old_to_new[v] : 0u;
        if (ew) {
          const unsigned long long wat = a.sec[kPhAdjwgt] + static_cast<unsigned long long>(e[j]) * (ew8 ? 8 : 4);
          const unsigned long long raw = ph_entry(a.bytes, wat, ew8);
          const long long s = ew8 ? static_cast<long long>(raw) : static_cast<long long>(static_cast<int32_t>(raw));
          if (ph_weight(a.ctl, wat, s)) {
            sum += static_cast<unsigned long long>(s);
            a.adjwgt[p] = static_cast<int32_t>(s);
          }
        }
      }
    }
  }
  ph_add_sum(a.ctl, 1, sum);
}

// ---- host ---------------------------------------------------------------------------------------------------------

const char *const kParhipSectionNames[5] = {"header", "offsets", "adjncy", "vwgt", "adjwgt"};
const char *const kParhipKindNames[KMP_PARHIP_NUM_KINDS] = {
    "ok", "truncated", "too large", "bad offsets", "neighbor out of range", "weight below 1", "total weight too large"};

struct ParhipLayout {
  unsigned long long len = 0, n = 0, m = 0, version = 0;
  bool vw = false, ew = false;
  unsigned long long sec[6] = {};   // first byte of each section; sec[5] = the end of the last one
  unsigned long long count[5] = {}; // entries of each section (0 for an absent one)
  uint32_t w[5] = {};
};

void parhip_refuse(kmp_parhip_report &r, uint32_t kind, unsigned long long offset, int section, long long index) {
  r.kind = static_cast<int32_t>(kind);
  r.offset = offset;
  r.section = section;
  r.index = index;
}

// The layout from the header (the file's first min(len, 24) bytes in p). false: a refusal in r (the header ends the
// file, or n / m >= 2^31).
bool parhip_layout(const uint8_t *p, uint64_t len, ParhipLayout &L, kmp_parhip_report &r) {
  auto u64 = [&](int at) {
    unsigned long long v = 0;
    std::memcpy(&v, p + at, 8); // little-endian host
    return v;
  };
  L.len = len;
  if (len >= 8) {
    L.version = r.version = u64(0);
    L.ew = (L.version & 1u) == 0;
    L.vw = (L.version & 2u) == 0;
    r.has_edge_weights = L.ew ? 1 : 0;
    r.has_node_weights = L.vw ? 1 : 0;
    L.w[kPhOffsets] = (L.version & 4u) == 0 ? 8 : 4;
    L.w[kPhAdjncy] = (L.version & 8u) == 0 ? 8 : 4;
    L.w[kPhVwgt] = (L.version & 16u) == 0 ? 8 : 4;
    L.w[kPhAdjwgt] = (L.version & 32u) == 0 ? 8 : 4;
    r.widths = L.w[1] | (L.w[2] << 8) | (L.w[3] << 16) | (L.w[4] << 24);
  }
  if (len >= 16) {
    L.n = r.n = u64(8);
    if (L.n >= (1ull << 31)) {
      parhip_refuse(r, KMP_PARHIP_TOO_LARGE, 8, KMP_PARHIP_SECTION_HEADER, -1);
      return false;
    }
  }
  if (len >= 24) {
    L.m = r.m = u64(16);
    if (L.m >= (1ull << 31)) {
      parhip_refuse(r, KMP_PARHIP_TOO_LARGE, 16, KMP_PARHIP_SECTION_HEADER, -1);
      return false;
    }
  } else {
    parhip_refuse(r, KMP_PARHIP_TRUNCATED, len, KMP_PARHIP_SECTION_HEADER, -1);
    return false;
  }
  L.count[kPhOffsets] = L.n + 1;
  L.count[kPhAdjncy] = L.m;
  L.count[kPhVwgt] = L.vw ? L.n : 0;
  L.count[kPhAdjwgt] = L.ew ? L.m : 0;
  L.sec[KMP_PARHIP_SECTION_HEADER] = 0;
  L.sec[kPhOffsets] = 24;
  for (int s = kPhOffsets; s <= kPhAdjwgt; ++s) {
    L.sec[s + 1] = L.sec[s] + L.count[s] * L.w[s];
  }
  return true;
}

// the section holding byte `at` (at < the end of the last section) and the entry there
void parhip_locate(const ParhipLayout &L, unsigned long long at, int &section, long long &index) {
  section = KMP_PARHIP_SECTION_HEADER;
  index = -1;
  for (int s = kPhOffsets; s <= kPhAdjwgt; ++s) {
    if (L.count[s] > 0 && at >= L.sec[s] && at < L.sec[s + 1]) {
      section = s;
      index = static_cast<long long>((at - L.sec[s]) / L.w[s]);
    }
  }
}

int parhip_fail(const kmp_parhip_report &r) {
  char buf[160];
  kmp_parhip_report_message(&r, buf, sizeof(buf));
  return fail(r.kind == KMP_PARHIP_TOO_LARGE ? KMP_ERR_UNSUPPORTED : KMP_ERR_INVALID,
              std::string("malformed ParHIP input: ") + buf);
}

// One read after the header. prepare() allocates the outputs, the scratch and CUB's temporaries before any kernel
// runs; ready(end) runs the passes on the entries whose bytes lie in [0, end); finish() runs the EXTERNAL rebuild
// and fills the report.
struct ParhipJob {
  kmp_lp_handle *h;
  ParhipLayout L;
  bool ext = false;   // EXTERNAL_DEGREE_BUCKETS, on a complete file
  bool check = false; // the file ends before its last section: check what is there, write nothing
  ParhipArgs a{};
  unsigned long long done[5] = {};
  uint32_t tiles = 0, etiles = 0;
  PoolBuf<ParhipCtl> ctl;
  PoolBuf<uint32_t> file_xadj, hist, base, deg, owners, bad; // EXTERNAL scratch
  PoolBuf<int32_t> file_vwgt;

  int prepare(const uint8_t *d_bytes, kmp_parhip_graph *g, kmp_prepared_graph *pg);
  int ready(unsigned long long end);
  int finish(kmp_parhip_report &r, kmp_prepared_graph *pg);
  auto hist_scan() {
    return [this](void *tmp, size_t &bytes) {
      return cub::DeviceScan::ExclusiveSum(tmp, bytes, hist.p, base.p, static_cast<int>(kPrepBuckets * tiles), h->stream);
    };
  }
  auto deg_scan(uint32_t *xadj) {
    return [this, xadj](void *tmp, size_t &bytes) {
      return cub::DeviceScan::InclusiveSum(tmp, bytes, deg.p, xadj + 1, static_cast<int>(L.n), h->stream);
    };
  }
};

int ParhipJob::prepare(const uint8_t *d_bytes, kmp_parhip_graph *g, kmp_prepared_graph *pg) {
  const cudaStream_t st = h->stream;
  const int dev = h->device;
  const size_t n = L.n, m = L.m;
  check = L.len < L.sec[5];
  ext = ext && !check;
  KMP_CUDA(ctl.alloc(1, st, dev));
  a.bytes = d_bytes;
  a.len = L.len;
  a.n = L.n;
  a.m = L.m;
  a.base = L.sec[kPhAdjncy];
  for (int s = 0; s < 5; ++s) {
    a.sec[s] = L.sec[s];
    a.w[s] = L.w[s];
  }
  a.ctl = ctl.p;
  if (ext) {
    pg->n = static_cast<uint32_t>(n);
    pg->m = static_cast<uint32_t>(m);
    KMP_CUDA(pg->xadj.alloc(n + 1, st, dev));
    KMP_CUDA(pg->adjncy.alloc(m, st, dev));
    KMP_CUDA(pg->old_to_new.alloc(n, st, dev));
    KMP_CUDA(pg->new_to_old.alloc(n, st, dev));
    if (L.vw) {
      KMP_CUDA(pg->vwgt.alloc(n, st, dev));
      KMP_CUDA(file_vwgt.alloc(n, st, dev));
    }
    if (L.ew) {
      KMP_CUDA(pg->adjwgt.alloc(m, st, dev));
    }
    tiles = static_cast<uint32_t>(std::max<size_t>(1, (n + kPrepTileVerts - 1) / kPrepTileVerts));
    etiles = static_cast<uint32_t>((m + kTileEdges - 1) / kTileEdges);
    KMP_CUDA(file_xadj.alloc(n + 1, st, dev));
    KMP_CUDA(hist.alloc(static_cast<size_t>(kPrepBuckets) * tiles, st, dev));
    KMP_CUDA(base.alloc(static_cast<size_t>(kPrepBuckets) * tiles, st, dev));
    KMP_CUDA(deg.alloc(n + 1, st, dev));
    KMP_CUDA(owners.alloc(static_cast<size_t>(etiles) + 1, st, dev));
    KMP_CUDA(bad.alloc(2, st, dev));
    size_t b1 = 0, b2 = 0; // CUB's temporaries, grown now (the queries read no data)
    KMP_CUDA(hist_scan()(nullptr, b1));
    KMP_CUDA(deg_scan(pg->xadj.p)(nullptr, b2));
    KMP_CUDA(h->commit.cub_tmp.ensure(std::max(b1, b2)));
    a.xadj = file_xadj.p;
    a.vwgt = file_vwgt.p;
    a.adjncy = pg->adjncy.p; // written by k_parhip_edges in the new layout
    a.adjwgt = pg->adjwgt.p;
  } else if (!check) {
    KMP_CUDA(g->xadj.alloc(n + 1, st, dev));
    KMP_CUDA(g->adjncy.alloc(m, st, dev));
    if (L.vw) {
      KMP_CUDA(g->vwgt.alloc(n, st, dev));
    }
    if (L.ew) {
      KMP_CUDA(g->adjwgt.alloc(m, st, dev));
    }
    a.xadj = g->xadj.p;
    a.adjncy = g->adjncy.p;
    a.vwgt = g->vwgt.p;
    a.adjwgt = g->adjwgt.p;
  }
  ParhipCtl init{};
  init.first = kPhNone;
  KMP_CUDA(cudaMemcpyAsync(ctl.p, &init, sizeof(init), cudaMemcpyHostToDevice, st));
  return KMP_OK;
}

template <int SEC> void parhip_launch(kmp_lp_handle *h, const ParhipArgs &a, unsigned long long i0,
                                      unsigned long long i1) {
  const unsigned long long groups = (i1 - i0) / (16 / a.w[SEC]) + 2;
  const uint32_t blocks = capped(h, grid_for(groups, 256));
  if (a.w[SEC] == 8) {
    k_parhip_pass<SEC, true><<<blocks, 256, 0, h->stream>>>(a, i0, i1);
  } else {
    k_parhip_pass<SEC, false><<<blocks, 256, 0, h->stream>>>(a, i0, i1);
  }
}

int ParhipJob::ready(unsigned long long end) {
  for (int s = kPhOffsets; s <= kPhAdjwgt; ++s) {
    if (ext && (s == kPhAdjncy || s == kPhAdjwgt)) { // k_parhip_edges reads and checks them
      continue;
    }
    const unsigned long long c = L.count[s], e = std::min<unsigned long long>(end, L.len);
    const unsigned long long r = e <= L.sec[s] ? 0 : std::min(c, (e - L.sec[s]) / L.w[s]); // entries wholly in [0, e)
    if (r > done[s]) {
      switch (s) {
      case kPhOffsets: parhip_launch<kPhOffsets>(h, a, done[s], r); break;
      case kPhAdjncy: parhip_launch<kPhAdjncy>(h, a, done[s], r); break;
      case kPhVwgt: parhip_launch<kPhVwgt>(h, a, done[s], r); break;
      default: parhip_launch<kPhAdjwgt>(h, a, done[s], r); break;
      }
      done[s] = r;
    }
  }
  KMP_CUDA(cudaGetLastError());
  return KMP_OK;
}

int ParhipJob::finish(kmp_parhip_report &r, kmp_prepared_graph *pg) {
  const cudaStream_t st = h->stream;
  const uint32_t n = static_cast<uint32_t>(L.n), m = static_cast<uint32_t>(L.m);
  uint32_t np = 0;
  if (ext) {
    // the reused preparation kernels index one CTA per tile and so take the full grid
    KMP_CUDA(cudaMemsetAsync(bad.p, 0, 8, st));
    k_prep_count<<<tiles, 256, 0, st>>>(n, m, file_xadj.p, tiles, hist.p, bad.p);
    KMP_CUDA(cub_call(h, hist_scan()));
    KMP_CUDA(cudaMemsetAsync(pg->xadj.p, 0, 4, st));
    if (n > 0) {
      k_prep_scatter<<<tiles, 256, 0, st>>>(n, file_xadj.p, file_vwgt.p, tiles, base.p, pg->old_to_new.p,
                                            pg->new_to_old.p, deg.p, pg->vwgt.p);
      KMP_CUDA(cub_call(h, deg_scan(pg->xadj.p)));
    }
    if (m > 0) {
      k_tile_owners<<<capped(h, grid_for(static_cast<uint64_t>(etiles) + 1, 256)), 256, 0, st>>>(n, m, pg->xadj.p, etiles,
                                                                                               owners.p);
      k_parhip_edges<<<capped(h, std::min<uint32_t>(etiles, kSMs * 8)), 256, 0, st>>>(
          a, etiles, file_xadj.p, pg->xadj.p, owners.p, pg->new_to_old.p, pg->old_to_new.p);
    }
    KMP_CUDA(cudaGetLastError());
    KMP_CUDA(cudaMemcpyAsync(&np, base.p + static_cast<size_t>(kPrepIsolated) * tiles, 4, cudaMemcpyDeviceToHost, st));
  }
  ParhipCtl c{};
  KMP_CUDA(cudaMemcpyAsync(&c, ctl.p, sizeof(c), cudaMemcpyDeviceToHost, st));
  KMP_CUDA(call_clock_stop(h, st));
  KMP_CUDA(cudaStreamSynchronize(st));
  r.device_ms = call_clock_ms(h);
  // the host's candidates: the weight totals of complete sections at their last byte, the truncation at the end
  unsigned long long first = c.first;
  int which = -1; // the weight section whose total wins
  for (int t = 0; t < 2; ++t) {
    const int s = t == 0 ? kPhVwgt : kPhAdjwgt;
    if (L.count[s] > 0 && L.sec[s + 1] <= L.len && c.sum[t] > 0x7FFFFFFFull) {
      const unsigned long long key = ((L.sec[s + 1] - 1) << 8) | KMP_PARHIP_TOTAL_WEIGHT;
      if (key < first) {
        first = key;
        which = s;
      }
    }
  }
  if (check && ((L.len << 8) | KMP_PARHIP_TRUNCATED) < first) {
    first = (L.len << 8) | KMP_PARHIP_TRUNCATED;
    which = -2;
  }
  if (first == kPhNone) {
    if (ext) {
      pg->np = np;
    }
    return KMP_OK;
  }
  const unsigned long long off = first >> 8;
  if (which >= 0) {
    parhip_refuse(r, KMP_PARHIP_TOTAL_WEIGHT, off, which, static_cast<long long>(L.count[which]));
  } else if (which == -2) {
    int s = kPhOffsets;
    while (L.sec[s + 1] <= L.len) { // the section the file ends in (one exists: the file is short)
      ++s;
    }
    parhip_refuse(r, KMP_PARHIP_TRUNCATED, off, s, static_cast<long long>((L.len - L.sec[s]) / L.w[s]));
  } else {
    int s;
    long long idx;
    parhip_locate(L, off, s, idx);
    parhip_refuse(r, static_cast<uint32_t>(first & 0xFFu), off, s, idx);
  }
  return parhip_fail(r);
}

int parhip_begin(kmp_lp_handle *h, int ordering, bool prepared, void *out, kmp_parhip_report *report) {
  return reader_begin(h, out, report, [&](kmp_parhip_report &r) { r.ordering = ordering; }, [&]() -> int {
    if ((ordering & KMP_PARHIP_COMPRESS) != 0 && (ordering & ~KMP_PARHIP_COMPRESS) >= 0 &&
        (ordering & ~KMP_PARHIP_COMPRESS) <= KMP_PARHIP_IMPLICIT_DEGREE_BUCKETS) {
      return fail(KMP_ERR_UNSUPPORTED, "the compressed ParHIP read is not supported");
    }
    if (ordering < KMP_PARHIP_NATURAL || ordering > KMP_PARHIP_IMPLICIT_DEGREE_BUCKETS) {
      return fail(KMP_ERR_INVALID, "unknown node ordering");
    }
    if (prepared && ordering != KMP_PARHIP_EXTERNAL_DEGREE_BUCKETS) {
      return fail(KMP_ERR_INVALID, "a prepared read takes the external degree-bucket ordering");
    }
    report->sorted = ordering == KMP_PARHIP_IMPLICIT_DEGREE_BUCKETS || ordering == KMP_PARHIP_EXTERNAL_DEGREE_BUCKETS;
    return KMP_OK;
  });
}

// The read of one file into g (NATURAL / IMPLICIT) or pg (EXTERNAL). head: the file's first min(len, 24) bytes;
// load(job) puts the bytes on the device and runs job.ready on them, and returns the device bytes in *d_bytes.
template <typename Load>
int parhip_run(kmp_lp_handle *h, const uint8_t *head, uint64_t len, int ordering, kmp_parhip_graph *g,
               kmp_prepared_graph *pg, kmp_parhip_report &r, Load &&load) {
  r.bytes = len;
  ParhipJob job{h};
  if (!parhip_layout(head, len, job.L, r)) {
    return parhip_fail(r);
  }
  job.ext = ordering == KMP_PARHIP_EXTERNAL_DEGREE_BUCKETS;
  int rc = load(job);
  if (rc != KMP_OK) {
    return rc;
  }
  rc = job.finish(r, pg);
  if (rc != KMP_OK) {
    return rc;
  }
  if (g != nullptr) {
    g->n = static_cast<uint32_t>(job.L.n);
    g->m = static_cast<uint32_t>(job.L.m);
    g->sorted = r.sorted;
    if (job.ext) { // the prepared arrays become the graph's; new_to_old is freed with pg
      static_cast<DeviceCsr &>(*g) = std::move(*pg);
      g->old_to_new = std::move(pg->old_to_new);
    }
  }
  return KMP_OK;
}

int read_parhip_impl(kmp_lp_handle *h, const char *path, int ordering, kmp_parhip_graph *g, kmp_prepared_graph *pg,
                     kmp_parhip_report &r) {
  InputFile f;
  int rc = f.open(path);
  const uint64_t len = f.len;
  uint8_t head[24] = {};
  if (rc == KMP_OK) {
    rc = f.read(head, std::min<uint64_t>(len, 24), 0);
  }
  if (rc != KMP_OK) {
    return rc;
  }
  PoolBuf<uint8_t> bytes; // released stream-ordered when the read ends
  FileStaging stage;
  return parhip_run(h, head, len, ordering, g, pg, r, [&](ParhipJob &job) {
    KMP_CUDA(bytes.alloc(len, h->stream, h->device));
    int rc = job.prepare(bytes.p, g, pg);
    if (rc != KMP_OK) {
      return rc;
    }
    return stream_file(h, stage, f, bytes.p, [&](uint64_t end) { return job.ready(end); });
  });
}

int parse_parhip_impl(kmp_lp_handle *h, const uint8_t *d_bytes, uint64_t len, int ordering, kmp_parhip_graph *g,
                      kmp_prepared_graph *pg, kmp_parhip_report &r) {
  uint8_t head[24] = {};
  if (len > 0) {
    const int rc = fetch_device_prefix(h, head, d_bytes, std::min<uint64_t>(len, 24));
    if (rc != KMP_OK) {
      return rc;
    }
  }
  return parhip_run(h, head, len, ordering, g, pg, r, [&](ParhipJob &job) {
    int rc = job.prepare(d_bytes, g, pg);
    if (rc != KMP_OK) {
      return rc;
    }
    KMP_CUDA(call_clock_start(h, h->stream));
    return job.ready(len);
  });
}

// the graph result of either entry point: EXTERNAL goes through a prepared graph whose arrays it takes over
template <typename Impl> int parhip_graph_result(kmp_lp_handle *h, kmp_parhip_graph **out, Impl &&impl) {
  return make_result(h, out, [&](kmp_parhip_graph *g) {
    kmp_prepared_graph pg;
    pg.device = h->device;
    return impl(g, &pg);
  });
}

} // namespace

extern "C" {

int kmp_read_parhip(kmp_lp_handle *h, const char *path, int ordering, kmp_parhip_graph **out,
                    kmp_parhip_report *report) {
  int rc = parhip_begin(h, ordering, false, out, report);
  if (rc == KMP_OK && path == nullptr) {
    rc = fail(KMP_ERR_INVALID, "null argument");
  }
  if (rc != KMP_OK) {
    return rc;
  }
  return parhip_graph_result(h, out, [&](kmp_parhip_graph *g, kmp_prepared_graph *pg) {
    return read_parhip_impl(h, path, ordering, g, pg, *report);
  });
}

int kmp_parse_parhip_device(kmp_lp_handle *h, const void *d_bytes, uint64_t len, int ordering,
                            kmp_parhip_graph **out, kmp_parhip_report *report) {
  int rc = parhip_begin(h, ordering, false, out, report);
  if (rc == KMP_OK) {
    rc = check_device_bytes(h, d_bytes, len);
  }
  if (rc != KMP_OK) {
    return rc;
  }
  return parhip_graph_result(h, out, [&](kmp_parhip_graph *g, kmp_prepared_graph *pg) {
    return parse_parhip_impl(h, static_cast<const uint8_t *>(d_bytes), len, ordering, g, pg, *report);
  });
}

int kmp_read_parhip_prepared(kmp_lp_handle *h, const char *path, kmp_prepared_graph **out,
                             kmp_parhip_report *report) {
  int rc = parhip_begin(h, KMP_PARHIP_EXTERNAL_DEGREE_BUCKETS, true, out, report);
  if (rc == KMP_OK && path == nullptr) {
    rc = fail(KMP_ERR_INVALID, "null argument");
  }
  if (rc != KMP_OK) {
    return rc;
  }
  return make_result(h, out, [&](kmp_prepared_graph *pg) {
    return read_parhip_impl(h, path, KMP_PARHIP_EXTERNAL_DEGREE_BUCKETS, nullptr, pg, *report);
  });
}

int kmp_parse_parhip_device_prepared(kmp_lp_handle *h, const void *d_bytes, uint64_t len, kmp_prepared_graph **out,
                                     kmp_parhip_report *report) {
  int rc = parhip_begin(h, KMP_PARHIP_EXTERNAL_DEGREE_BUCKETS, true, out, report);
  if (rc == KMP_OK) {
    rc = check_device_bytes(h, d_bytes, len);
  }
  if (rc != KMP_OK) {
    return rc;
  }
  return make_result(h, out, [&](kmp_prepared_graph *pg) {
    return parse_parhip_impl(h, static_cast<const uint8_t *>(d_bytes), len, KMP_PARHIP_EXTERNAL_DEGREE_BUCKETS,
                             nullptr, pg, *report);
  });
}

uint32_t kmp_parhip_n(const kmp_parhip_graph *g) { return g != nullptr ? g->n : 0; }
uint32_t kmp_parhip_m(const kmp_parhip_graph *g) { return g != nullptr ? g->m : 0; }
int kmp_parhip_sorted(const kmp_parhip_graph *g) { return g != nullptr ? g->sorted : 0; }

int kmp_parhip_device_arrays(const kmp_parhip_graph *g, const uint32_t **d_xadj, const uint32_t **d_adjncy,
                             const int32_t **d_vwgt, const int32_t **d_adjwgt, const uint32_t **d_old_to_new) {
  if (g == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  hand_out_csr(*g, d_xadj, d_adjncy, d_vwgt, d_adjwgt);
  hand_out(d_old_to_new, g->old_to_new);
  return KMP_OK;
}

int kmp_parhip_download(const kmp_parhip_graph *g, uint32_t *xadj, uint32_t *adjncy, int32_t *vwgt, int32_t *adjwgt,
                        uint32_t *old_to_new) {
  if (g == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  const int rc = download_csr(*g, xadj, adjncy, vwgt, adjwgt, static_cast<size_t>(g->n) + 1, g->n, g->m);
  if (rc != KMP_OK) {
    return rc;
  }
  KMP_CUDA(copy_out(old_to_new, g->old_to_new, g->n));
  return KMP_OK;
}

void kmp_parhip_destroy(kmp_parhip_graph *g) { destroy_result(g); }

int kmp_parhip_report_message(const kmp_parhip_report *r, char *buf, size_t size) {
  if (r == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  if (r->kind <= KMP_PARHIP_OK || r->kind >= KMP_PARHIP_NUM_KINDS) {
    return format_report(buf, size, "%s", "");
  }
  const int s = r->section >= 0 && r->section <= KMP_PARHIP_SECTION_ADJWGT ? r->section : 0;
  return format_report(buf, size, "%s at byte %llu (%s entry %lld)", kParhipKindNames[r->kind],
                       static_cast<unsigned long long>(r->offset), kParhipSectionNames[s],
                       static_cast<long long>(r->index));
}

} // extern "C"
