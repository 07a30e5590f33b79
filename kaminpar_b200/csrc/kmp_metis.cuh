// kaminpar_b200: the METIS reader on the device + its C ABI (include/kaminpar_b200_io.h, DESIGN.md §18).
// Included at the end of kmp_lp.cu: scratch and results are PoolBuf, CUB calls go through cub_call, every launch
// through capped().
//
// What it restates (see the header): csr_read (metis_parser.cc:158-245), parallel over the file's bytes.
//   The header is parsed on the host (metis_header). The data section is a line-state machine over three states:
//   line start (only spaces so far), comment, data. A data line begins at the first byte of a line that is neither
//   ' ' nor '%' (its '\n' for an empty line); a token begins at a digit of a data line after a non-digit.
//   (a) k_metis_summary: per tile of KMP_METIS_TILE_BYTES and per entry state, the exit state and the counts of data
//       lines, tokens, tokens of the open line and newlines; composing two summaries is composing two functions.
//   (b) an inclusive CUB scan of the tile summaries with that composition gives every tile its entry state, vertex,
//       token index (64-bit) and line number.
//   (c) k_metis_write: each tile re-reads its bytes, writes xadj[v] = (T[v] - v*vw) >> ew at each data-line start and
//       scatters each token t of line v by closed form: the node weight (first token, vw), or the target / weight of
//       edge (t - (v+1)*vw) >> ew. A token that starts in the tile may end past it. A violation is one atomicMin of
//       (offset << 8) | kind; the weight totals are one atomicAdd per CTA.
//   k_metis_finish closes the last line at the end of the file; on a refusal, k_metis_write<true> re-runs the one
//   tile that holds the first violation to fill in its vertex and line.
#pragma once

#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <cub/block/block_scan.cuh>

#include "../../include/kaminpar_b200_io.h"

struct kmp_metis_graph {
  int device = 0;
  uint32_t n = 0, m = 0;
  PoolBuf<uint32_t> xadj, adjncy;
  PoolBuf<int32_t> vwgt, adjwgt; // unallocated for absent or dropped weights
  PoolBuf<uint8_t> bytes;        // the file's bytes (kmp_read_metis), released when the read ends
};

namespace {

constexpr uint32_t kMetisThreads = 256;
constexpr uint32_t kMetisBytesPerThread = KMP_METIS_TILE_BYTES / kMetisThreads;
static_assert(kMetisBytesPerThread == 16, "one uint4 per thread");
constexpr uint32_t kMLineStart = 0, kMComment = 1, kMData = 2; // line states
constexpr unsigned long long kMetisCap = 1ull << 40;           // saturation of a token's value: above every id / weight
constexpr unsigned long long kMetisNone = ~0ull;
constexpr uint64_t kMetisChunk = 32ull << 20; // bytes per pinned staging buffer of kmp_read_metis

// The line-state machine over a run of bytes, for each entry state s: the exit state (2 bits at 2s), the data lines
// and tokens that begin, the tokens of the line open at the end (all tokens of the run if no data line begins), and
// the newlines (the same for every entry state).
template <typename C> struct MetisSum {
  uint32_t exit;
  C lines[3], toks[3], tail[3];
  C nl;
};

template <typename C> __host__ __device__ __forceinline__ MetisSum<C> metis_identity() {
  MetisSum<C> s{};
  s.exit = kMLineStart | (kMComment << 2) | (kMData << 4);
  return s;
}

// a[s] for a state s known only at run time, as selects (an indexed load would put the array in local memory)
template <typename C> __host__ __device__ __forceinline__ C metis_at(const C (&a)[3], uint32_t s) {
  return s == 0 ? a[0] : s == 1 ? a[1] : a[2];
}

// f then g
struct MetisCompose {
  template <typename C> __host__ __device__ __forceinline__ MetisSum<C> operator()(const MetisSum<C> &f,
                                                                                     const MetisSum<C> &g) const {
    MetisSum<C> o;
    o.exit = 0;
#pragma unroll
    for (uint32_t s = 0; s < 3; ++s) {
      const uint32_t s1 = (f.exit >> (2 * s)) & 3u;
      o.exit |= ((g.exit >> (2 * s1)) & 3u) << (2 * s);
      const C g_lines = metis_at(g.lines, s1), g_toks = metis_at(g.toks, s1);
      o.lines[s] = f.lines[s] + g_lines;
      o.toks[s] = f.toks[s] + g_toks;
      o.tail[s] = g_lines != 0 ? metis_at(g.tail, s1) : f.tail[s] + g_toks;
    }
    o.nl = f.nl + g.nl;
    return o;
  }
};

struct MetisArgs {
  const uint8_t *bytes;
  unsigned long long len, data; // file length, first byte after the header
  unsigned long long n, m2;     // vertices, adjacency entries (2m)
  uint32_t vw, ew;              // 0 / 1
  uint32_t *xadj, *adjncy;
  int32_t *vwgt, *adjwgt;
};

// device control block of one read; zeroed except for `first`
struct MetisCtl {
  unsigned long long first;  // min over the violations of (offset << 8) | kind
  unsigned long long t_end;  // token index at the start of data line n (all tokens if there is none)
  unsigned long long lines;  // data lines in the file
  unsigned long long nl;     // newlines in the file
  unsigned long long sum_vw, sum_ew;
  unsigned long long line;   // the first violation's line and vertex (k_metis_write<true>, k_metis_finish)
  long long vertex;
  uint32_t extra;            // a line after vertex n-1's line that does not start with '%'
};

__device__ __forceinline__ bool metis_digit(uint32_t b) { return b - '0' < 10u; }

__device__ __forceinline__ uint32_t metis_byte(const uint32_t (&w)[4], uint32_t k) {
  const uint32_t word = k < 4 ? w[0] : k < 8 ? w[1] : k < 12 ? w[2] : w[3];
  return (word >> (8 * (k & 3u))) & 0xFFu;
}

// the thread's 16 bytes [i0, i0 + 16) (zero past the end); `bytes` is 16-byte aligned and i0 a multiple of 16
__device__ __forceinline__ void metis_load(const uint8_t *__restrict__ bytes, unsigned long long len,
                                           unsigned long long i0, uint32_t (&w)[4]) {
  if (i0 + kMetisBytesPerThread <= len) {
    const uint4 q = __ldg(reinterpret_cast<const uint4 *>(bytes + i0));
    w[0] = q.x;
    w[1] = q.y;
    w[2] = q.z;
    w[3] = q.w;
  } else {
#pragma unroll
    for (uint32_t j = 0; j < 4; ++j) {
      uint32_t x = 0;
#pragma unroll
      for (uint32_t k = 0; k < 4; ++k) {
        const unsigned long long i = i0 + 4 * j + k;
        x |= (i < len ? static_cast<uint32_t>(bytes[i]) : 0u) << (8 * k);
      }
      w[j] = x;
    }
  }
}

// one byte of the machine in state s; `prev` is the byte before
__device__ __forceinline__ void metis_step(uint32_t &s, uint32_t &lines, uint32_t &toks, uint32_t &tail, uint32_t b,
                                           uint32_t prev) {
  if (s == kMComment) {
    s = b == '\n' ? kMLineStart : kMComment;
    return;
  }
  if (s == kMLineStart) {
    if (b == ' ') {
      return;
    }
    if (b == '%') {
      s = kMComment;
      return;
    }
    ++lines; // a data line begins; this byte is its first non-space byte
    tail = 0;
  }
  if (b == '\n') {
    s = kMLineStart;
  } else {
    s = kMData;
    if (metis_digit(b) && !metis_digit(prev)) {
      ++toks;
      ++tail;
    }
  }
}

// the summary of the thread's bytes (bytes before the data section are the identity)
__device__ __forceinline__ MetisSum<uint32_t> metis_thread_sum(const MetisArgs &a, unsigned long long i0,
                                                                const uint32_t (&w)[4], uint32_t prev) {
  MetisSum<uint32_t> r = metis_identity<uint32_t>();
  uint32_t st[3] = {kMLineStart, kMComment, kMData};
#pragma unroll
  for (uint32_t k = 0; k < kMetisBytesPerThread; ++k) {
    const unsigned long long i = i0 + k;
    const uint32_t b = metis_byte(w, k);
    if (i >= a.data && i < a.len) {
#pragma unroll
      for (uint32_t s = 0; s < 3; ++s) {
        metis_step(st[s], r.lines[s], r.toks[s], r.tail[s], b, prev);
      }
      r.nl += b == '\n' ? 1u : 0u;
    }
    prev = b;
  }
  r.exit = st[0] | (st[1] << 2) | (st[2] << 4);
  return r;
}

using MetisBlockScan = cub::BlockScan<MetisSum<uint32_t>, kMetisThreads>;

// (a) the summary of tiles [t0, t1)
__global__ void __launch_bounds__(kMetisThreads) k_metis_summary(MetisArgs a, uint32_t t0, uint32_t t1,
                                                                 MetisSum<unsigned long long> *__restrict__ sums) {
  __shared__ typename MetisBlockScan::TempStorage tmp;
  for (uint32_t t = t0 + blockIdx.x; t < t1; t += gridDim.x) {
    const unsigned long long i0 = static_cast<unsigned long long>(t) * KMP_METIS_TILE_BYTES + threadIdx.x * kMetisBytesPerThread;
    uint32_t w[4];
    metis_load(a.bytes, a.len, i0, w);
    const uint32_t prev = i0 > 0 && i0 <= a.len ? a.bytes[i0 - 1] : '\n';
    MetisSum<uint32_t> s = metis_thread_sum(a, i0, w, prev);
    __syncthreads(); // the previous tile is done with tmp
    MetisBlockScan(tmp).InclusiveScan(s, s, MetisCompose());
    if (threadIdx.x == kMetisThreads - 1) {
      MetisSum<unsigned long long> o;
      o.exit = s.exit;
#pragma unroll
      for (uint32_t k = 0; k < 3; ++k) {
        o.lines[k] = s.lines[k];
        o.toks[k] = s.toks[k];
        o.tail[k] = s.tail[k];
      }
      o.nl = s.nl;
      sums[t] = o;
    }
  }
}

// (c) the write pass over tiles [t0, t1) given the scanned summaries. DETAIL: nothing is written; the violation whose
// key is ctl->first records its vertex and line.
template <bool DETAIL>
__global__ void __launch_bounds__(kMetisThreads) k_metis_write(MetisArgs a, uint32_t t0, uint32_t t1,
                                                               const MetisSum<unsigned long long> *__restrict__ incl,
                                                               MetisCtl *ctl) {
  __shared__ typename MetisBlockScan::TempStorage tmp;
  unsigned long long sum_vw = 0, sum_ew = 0;
  for (uint32_t t = t0 + blockIdx.x; t < t1; t += gridDim.x) {
    const unsigned long long i0 = static_cast<unsigned long long>(t) * KMP_METIS_TILE_BYTES + threadIdx.x * kMetisBytesPerThread;
    uint32_t w[4];
    metis_load(a.bytes, a.len, i0, w);
    uint32_t prev = i0 > 0 && i0 <= a.len ? a.bytes[i0 - 1] : '\n';
    MetisSum<uint32_t> p = metis_thread_sum(a, i0, w, prev);
    __syncthreads();
    MetisBlockScan(tmp).ExclusiveScan(p, p, metis_identity<uint32_t>(), MetisCompose());
    const MetisSum<unsigned long long> P = t > 0 ? incl[t - 1] : metis_identity<unsigned long long>();
    const uint32_t es = P.exit & 3u; // the tile's entry state (the data section begins at a line start)
    uint32_t s = (p.exit >> (2 * es)) & 3u;
    const uint32_t p_lines = metis_at(p.lines, es), p_toks = metis_at(p.toks, es);
    unsigned long long v = P.lines[0] + p_lines;
    unsigned long long tok = P.toks[0] + p_toks;
    unsigned long long tail = p_lines != 0 ? metis_at(p.tail, es) : P.tail[0] + p_toks;
    unsigned long long nl = P.nl + p.nl;
    auto violate = [&](unsigned long long off, uint32_t kind, unsigned long long vtx) {
      const unsigned long long key = (off << 8) | kind;
      if (DETAIL) {
        if (key == ctl->first) {
          ctl->vertex = static_cast<long long>(vtx);
          ctl->line = nl + 1;
        }
      } else {
        atomicMin(&ctl->first, key);
      }
    };
    // the end of data line vc at byte `off` ('\n'): its token count
    auto terminate = [&](unsigned long long off, unsigned long long vc) {
      if (vc < a.n) {
        if (a.vw && tail == 0) {
          violate(off, KMP_METIS_MISSING_NODE_WEIGHT, vc);
        } else if (a.ew && ((tail - a.vw) & 1ull)) {
          violate(off, KMP_METIS_MISSING_EDGE_WEIGHT, vc);
        }
      }
    };
    for (uint32_t k = 0; k < kMetisBytesPerThread; ++k) {
      const unsigned long long i = i0 + k;
      if (i >= a.len) {
        break;
      }
      const uint32_t b = metis_byte(w, k);
      if (i < a.data) {
        prev = b;
        continue;
      }
      if (s == kMComment) {
        if (b == '\n') {
          s = kMLineStart;
          ++nl;
        }
        prev = b;
        continue;
      }
      if (s == kMLineStart) {
        if (!DETAIL && prev == '\n' && v >= a.n && b != '%') { // a line after vertex n-1's line
          ctl->extra = 1u;
        }
        if (b == ' ') {
          prev = b;
          continue;
        }
        if (b == '%') {
          s = kMComment;
          prev = b;
          continue;
        }
        if (!DETAIL) { // data line v begins
          if (v < a.n) {
            a.xadj[v] = static_cast<uint32_t>((tok - v * a.vw) >> a.ew);
          } else if (v == a.n) {
            ctl->t_end = tok;
          }
        }
        ++v;
        tail = 0;
      }
      const unsigned long long vc = v - 1; // the line's vertex
      if (b == '\n') {
        terminate(i, vc);
        s = kMLineStart;
        ++nl;
      } else {
        s = kMData;
        if (metis_digit(b)) {
          if (!metis_digit(prev)) { // a token begins: parse it to its end, which may lie past the tile
            if (vc < a.n) {
              unsigned long long val = 0;
              for (unsigned long long j = i; j < a.len; ++j) {
                const uint32_t d = static_cast<uint32_t>(a.bytes[j]) - '0';
                if (d > 9u) {
                  break;
                }
                val = min(val * 10 + d, kMetisCap);
              }
              if (a.vw && tail == 0) { // the node weight
                if (val == 0) {
                  violate(i, KMP_METIS_ZERO_WEIGHT, vc);
                } else if (val > 0x7FFFFFFFull) {
                  violate(i, KMP_METIS_WEIGHT_TOO_LARGE, vc);
                } else if (!DETAIL) {
                  a.vwgt[vc] = static_cast<int32_t>(val);
                  sum_vw += val;
                }
              } else {
                const unsigned long long base = (vc + 1) * a.vw;
                const unsigned long long e = tok >= base ? (tok - base) >> a.ew : kMetisNone;
                if (!a.ew || ((tail - a.vw) & 1ull) == 0) { // a target
                  if (val == 0 || val > a.n) {
                    violate(i, KMP_METIS_NEIGHBOR_OUT_OF_RANGE, vc);
                  } else if (val - 1 == vc) {
                    violate(i, KMP_METIS_SELF_LOOP, vc);
                  } else if (!DETAIL && e < a.m2) {
                    a.adjncy[e] = static_cast<uint32_t>(val - 1);
                  }
                } else { // an edge weight
                  if (val == 0) {
                    violate(i, KMP_METIS_ZERO_WEIGHT, vc);
                  } else if (val > 0x7FFFFFFFull) {
                    violate(i, KMP_METIS_WEIGHT_TOO_LARGE, vc);
                  } else if (!DETAIL) {
                    sum_ew += val;
                    if (e < a.m2) {
                      a.adjwgt[e] = static_cast<int32_t>(val);
                    }
                  }
                }
              }
            }
            ++tok;
            ++tail;
          }
        } else if (b != ' ' && vc < a.n) {
          violate(i, KMP_METIS_BAD_BYTE, vc);
        }
      }
      prev = b;
    }
  }
  if (!DETAIL) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      sum_vw += __shfl_xor_sync(kFull, sum_vw, o);
      sum_ew += __shfl_xor_sync(kFull, sum_ew, o);
    }
    if ((threadIdx.x & 31u) == 0) {
      if (sum_vw != 0) {
        atomicAdd(&ctl->sum_vw, sum_vw);
      }
      if (sum_ew != 0) {
        atomicAdd(&ctl->sum_ew, sum_ew);
      }
    }
  }
}

// the end of the file (one thread): a last line of spaces only, the checks of an open last line at offset len, the
// token index after vertex n-1's line, xadj[n]
__global__ void k_metis_finish(MetisArgs a, uint32_t tiles, const MetisSum<unsigned long long> *__restrict__ incl,
                               MetisCtl *ctl) {
  if (blockIdx.x != 0 || threadIdx.x != 0) {
    return;
  }
  const MetisSum<unsigned long long> T = tiles > 0 ? incl[tiles - 1] : metis_identity<unsigned long long>();
  const uint32_t s = T.exit & 3u;
  unsigned long long lines = T.lines[0], tail = T.tail[0];
  bool open = s == kMData;
  if (s == kMLineStart && a.len > a.data && a.bytes[a.len - 1] == ' ') { // data line `lines` is spaces up to the end
    if (lines < a.n) {
      a.xadj[lines] = static_cast<uint32_t>((T.toks[0] - lines * a.vw) >> a.ew);
    } else if (lines == a.n) {
      ctl->t_end = T.toks[0];
    }
    ++lines;
    tail = 0;
    open = true;
  }
  if (open && lines - 1 < a.n) {
    uint32_t kind = KMP_METIS_OK;
    if (a.vw && tail == 0) {
      kind = KMP_METIS_MISSING_NODE_WEIGHT;
    } else if (a.ew && ((tail - a.vw) & 1ull)) {
      kind = KMP_METIS_MISSING_EDGE_WEIGHT;
    }
    const unsigned long long key = (a.len << 8) | kind;
    if (kind != KMP_METIS_OK && key < ctl->first) {
      ctl->first = key;
      ctl->vertex = static_cast<long long>(lines - 1);
      ctl->line = T.nl + 1;
    }
  }
  if (lines <= a.n) {
    ctl->t_end = T.toks[0];
  }
  ctl->lines = lines;
  ctl->nl = T.nl;
  a.xadj[a.n] = static_cast<uint32_t>((ctl->t_end - a.n * a.vw) >> a.ew);
}

struct MetisHeader {
  unsigned long long n = 0, m = 0, fmt = 0, data = 0;
  unsigned long long n_at = 0, m_at = 0, fmt_at = 0;
  unsigned long long nl = 0; // newlines before `data` (the device passes count the data section's)
  bool vw = false, ew = false;
};

void metis_refuse(kmp_metis_report &r, uint32_t kind, unsigned long long offset, unsigned long long line,
                  long long vertex) {
  r.kind = static_cast<int32_t>(kind);
  r.offset = offset;
  r.line = line;
  r.vertex = vertex;
}

// The header from the file's first `avail` of `len` bytes. 0: parsed into hd; 1: more bytes are needed; 2: a violation
// (in r, in file order: the value checks of the tokens read before a malformed byte come first).
int metis_header(const uint8_t *p, uint64_t avail, uint64_t len, MetisHeader &hd, kmp_metis_report &r) {
  uint64_t i = 0;
  int tokens = 0; // header tokens read
  auto line_of = [&](uint64_t off) {
    unsigned long long nl = 0;
    for (uint64_t j = 0; j < off && j < avail; ++j) {
      nl += p[j] == '\n';
    }
    return nl + 1;
  };
  // the value checks of the tokens read so far, in file order; true if one fires
  auto values = [&]() {
    if (tokens >= 1 && hd.n >= (1ull << 32)) {
      metis_refuse(r, KMP_METIS_TOO_LARGE, hd.n_at, line_of(hd.n_at), -1);
    } else if (tokens >= 2 && 2 * hd.m >= (1ull << 32)) {
      metis_refuse(r, KMP_METIS_TOO_LARGE, hd.m_at, line_of(hd.m_at), -1);
    } else if (tokens >= 2 && hd.m > hd.n * (hd.n - 1) / 2) {
      metis_refuse(r, KMP_METIS_HEADER, hd.m_at, line_of(hd.m_at), -1);
    } else if (tokens >= 3 && hd.fmt != 0 && hd.fmt != 1 && hd.fmt != 10 && hd.fmt != 11) {
      metis_refuse(r, KMP_METIS_FORMAT, hd.fmt_at, line_of(hd.fmt_at), -1);
    } else {
      return false;
    }
    return true;
  };
  auto malformed = [&](uint64_t off) {
    if (!values()) {
      metis_refuse(r, KMP_METIS_HEADER, off, line_of(off), -1);
    }
    return 2;
  };
  auto need = [&]() { return i >= avail && avail < len; };
  auto skip_spaces = [&]() {
    while (!need() && i < len && p[i] == ' ') {
      ++i;
    }
    return need();
  };
  // scan_uint: digits, then spaces; 1 / 2 as above
  auto scan = [&](unsigned long long &val, unsigned long long &at) {
    at = i;
    if (need()) {
      return 1;
    }
    if (i >= len || p[i] - '0' > 9u) {
      return malformed(i);
    }
    val = 0;
    while (!need() && i < len && p[i] - '0' <= 9u) {
      val = std::min<unsigned long long>(val * 10 + (p[i] - '0'), kMetisCap);
      ++i;
    }
    ++tokens;
    return skip_spaces() ? 1 : 0;
  };
  for (;;) { // comment lines before the header
    if (skip_spaces()) {
      return 1;
    }
    if (i < len && p[i] == '%') {
      while (!need() && i < len && p[i] != '\n') {
        ++i;
      }
      if (need()) {
        return 1;
      }
      i += i < len ? 1 : 0;
      continue;
    }
    break;
  }
  int rc = scan(hd.n, hd.n_at);
  if (rc == 0) {
    rc = scan(hd.m, hd.m_at);
  }
  if (rc == 0 && i < len && p[i] != '\n') {
    rc = scan(hd.fmt, hd.fmt_at);
  }
  if (rc != 0) {
    return rc;
  }
  if (i >= len || p[i] != '\n') {
    return malformed(i);
  }
  hd.data = i + 1;
  hd.nl = line_of(hd.data) - 1;
  if (values()) {
    return 2;
  }
  hd.vw = (hd.fmt % 100) / 10 != 0;
  hd.ew = hd.fmt % 10 != 0;
  return 0;
}

// One read after the header: the output arrays, the scratch and CUB's temporary are allocated by prepare() before any
// kernel runs; summarise() runs (a) on the tiles whose bytes are on the device; finish() runs (b), (c) and the report.
struct MetisJob {
  kmp_lp_handle *h;
  MetisArgs a{};
  unsigned long long header_nl = 0;
  uint32_t tiles = 0;
  PoolBuf<MetisSum<unsigned long long>> sums, incl;
  PoolBuf<MetisCtl> ctl;

  int prepare(const MetisHeader &hd, const uint8_t *d_bytes, uint64_t len, kmp_metis_graph *g);
  int summarise(uint32_t t0, uint32_t t1) {
    if (t1 > t0) {
      k_metis_summary<<<capped(h, std::min<uint32_t>(t1 - t0, kSMs * 8)), kMetisThreads, 0, h->stream>>>(a, t0, t1, sums.p);
    }
    KMP_CUDA(cudaGetLastError());
    return KMP_OK;
  }
  int finish(kmp_metis_graph *g, kmp_metis_report &r);
  auto scan() {
    return [this](void *tmp, size_t &bytes) {
      return cub::DeviceScan::InclusiveScan(tmp, bytes, sums.p, incl.p, MetisCompose(), static_cast<int>(tiles), h->stream);
    };
  }
};

int MetisJob::prepare(const MetisHeader &hd, const uint8_t *d_bytes, uint64_t len, kmp_metis_graph *g) {
  const cudaStream_t st = h->stream;
  const int dev = h->device;
  tiles = static_cast<uint32_t>((len + KMP_METIS_TILE_BYTES - 1) / KMP_METIS_TILE_BYTES);
  KMP_CUDA(g->xadj.alloc(hd.n + 1, st, dev));
  KMP_CUDA(g->adjncy.alloc(2 * hd.m, st, dev));
  if (hd.vw) {
    KMP_CUDA(g->vwgt.alloc(hd.n, st, dev));
  }
  if (hd.ew) {
    KMP_CUDA(g->adjwgt.alloc(2 * hd.m, st, dev));
  }
  KMP_CUDA(sums.alloc(tiles, st, dev));
  KMP_CUDA(incl.alloc(tiles, st, dev));
  KMP_CUDA(ctl.alloc(1, st, dev));
  size_t bytes = 0; // CUB's temporary, grown now (the query reads no data) so that the scan below allocates nothing
  auto sc = scan();
  KMP_CUDA(sc(nullptr, bytes));
  KMP_CUDA(h->commit.cub_tmp.ensure(bytes));
  MetisCtl init{};
  init.first = kMetisNone;
  KMP_CUDA(cudaMemcpyAsync(ctl.p, &init, sizeof(init), cudaMemcpyHostToDevice, st));
  header_nl = hd.nl;
  a.bytes = d_bytes;
  a.len = len;
  a.data = hd.data;
  a.n = hd.n;
  a.m2 = 2 * hd.m;
  a.vw = hd.vw ? 1u : 0u;
  a.ew = hd.ew ? 1u : 0u;
  a.xadj = g->xadj.p;
  a.adjncy = g->adjncy.p;
  a.vwgt = g->vwgt.p;
  a.adjwgt = g->adjwgt.p;
  return KMP_OK;
}

int MetisJob::finish(kmp_metis_graph *g, kmp_metis_report &r) {
  const cudaStream_t st = h->stream;
  KMP_CUDA(cub_call(h, scan()));
  k_metis_write<false><<<capped(h, std::min<uint32_t>(tiles, kSMs * 8)), kMetisThreads, 0, st>>>(a, 0, tiles, incl.p, ctl.p);
  k_metis_finish<<<capped(h, 1), 32, 0, st>>>(a, tiles, incl.p, ctl.p);
  KMP_CUDA(cudaGetLastError());
  MetisCtl c{};
  KMP_CUDA(cudaMemcpyAsync(&c, ctl.p, sizeof(c), cudaMemcpyDeviceToHost, st));
  KMP_CUDA(call_clock_stop(h, st));
  KMP_CUDA(cudaStreamSynchronize(st));
  r.device_ms = call_clock_ms(h);
  const unsigned long long off = c.first >> 8;
  if (c.first != kMetisNone && off < a.len) { // the vertex and line of the first violation
    const uint32_t t = static_cast<uint32_t>(off / KMP_METIS_TILE_BYTES);
    k_metis_write<true><<<capped(h, 1), kMetisThreads, 0, st>>>(a, t, t + 1, incl.p, ctl.p);
    KMP_CUDA(cudaGetLastError());
    KMP_CUDA(cudaMemcpyAsync(&c, ctl.p, sizeof(c), cudaMemcpyDeviceToHost, st));
    KMP_CUDA(cudaStreamSynchronize(st));
  }
  r.extra_lines = c.extra != 0 ? 1 : 0;
  const unsigned long long eof_line = header_nl + c.nl + 1;
  const unsigned long long edges = (c.t_end - a.n * a.vw) >> a.ew;
  if (c.first != kMetisNone) {
    metis_refuse(r, static_cast<uint32_t>(c.first & 0xFFu), off, header_nl + c.line, c.vertex);
  } else if (c.lines < a.n) {
    metis_refuse(r, KMP_METIS_TOO_FEW_LINES, a.len, eof_line, static_cast<long long>(c.lines));
  } else if (edges != a.m2) {
    metis_refuse(r, KMP_METIS_EDGE_COUNT, a.len, eof_line, static_cast<long long>(a.n));
  } else if (c.sum_vw > 0x7FFFFFFFull || c.sum_ew > 0x7FFFFFFFull) {
    metis_refuse(r, KMP_METIS_TOTAL_WEIGHT, a.len, eof_line, static_cast<long long>(a.n));
  }
  if (r.kind != KMP_METIS_OK) {
    r.extra_lines = 0;
    return KMP_ERR_INVALID;
  }
  g->n = static_cast<uint32_t>(a.n);
  g->m = static_cast<uint32_t>(a.m2);
  if (a.vw && c.sum_vw == a.n) { // all node weights 1 (each is >= 1)
    r.node_weights_dropped = 1;
    g->vwgt.release();
  }
  if (a.ew && c.sum_ew == a.m2) {
    r.edge_weights_dropped = 1;
    g->adjwgt.release();
  }
  return KMP_OK;
}

int metis_code(const kmp_metis_report &r) {
  if (r.kind == KMP_METIS_FORMAT || r.kind == KMP_METIS_TOO_LARGE) {
    return KMP_ERR_UNSUPPORTED;
  }
  return KMP_ERR_INVALID;
}

int metis_fail(const kmp_metis_report &r) {
  char buf[160];
  kmp_metis_report_message(&r, buf, sizeof(buf));
  return fail(metis_code(r), std::string("malformed METIS input: ") + buf);
}

void metis_report_header(kmp_metis_report &r, const MetisHeader &hd) {
  r.n = hd.n;
  r.m = hd.m;
  r.format = static_cast<uint32_t>(std::min<unsigned long long>(hd.fmt, 0xFFFFFFFFull));
  r.has_node_weights = (hd.fmt % 100) / 10 != 0 ? 1 : 0;
  r.has_edge_weights = hd.fmt % 10 != 0 ? 1 : 0;
}

int metis_begin(kmp_lp_handle *h, kmp_metis_graph **out, kmp_metis_report *report) {
  if (h == nullptr || out == nullptr || report == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  std::memset(report, 0, sizeof(*report));
  if (h->step.open) {
    return fail(KMP_ERR_INVALID, "the handle is inside a stepping call");
  }
  KMP_CUDA(cudaSetDevice(h->device));
  return KMP_OK;
}

// pread until `size` bytes are in or the file ends; false on a read error
bool metis_pread(int fd, uint8_t *dst, uint64_t size, uint64_t off) {
  while (size > 0) {
    const ssize_t got = pread(fd, dst, size, static_cast<off_t>(off));
    if (got <= 0) {
      return false;
    }
    dst += got;
    size -= static_cast<uint64_t>(got);
    off += static_cast<uint64_t>(got);
  }
  return true;
}

// the two pinned staging buffers of kmp_read_metis and the events of the copies out of them
struct MetisStaging {
  cudaStream_t st = nullptr;
  uint8_t *buf[2] = {nullptr, nullptr};
  cudaEvent_t ev[2] = {nullptr, nullptr};
  ~MetisStaging() {
    if (st != nullptr) {
      cudaStreamSynchronize(st); // no copy reads a buffer any more
    }
    for (int b = 0; b < 2; ++b) {
      if (buf[b] != nullptr) {
        cudaFreeHost(buf[b]);
      }
      if (ev[b] != nullptr) {
        cudaEventDestroy(ev[b]);
      }
    }
  }
};

struct MetisFile {
  int fd = -1;
  ~MetisFile() {
    if (fd >= 0) {
      close(fd);
    }
  }
};

// The header from the file's first bytes, fetched by fetch(dst, size) in growing prefixes until metis_header has what
// it needs; KMP_OK with hd filled, a refusal with r filled, or fetch's error.
template <typename Fetch> int metis_read_header(uint64_t len, MetisHeader &hd, kmp_metis_report &r, Fetch &&fetch) {
  std::vector<uint8_t> head;
  for (uint64_t size = std::min<uint64_t>(len, 1u << 16);; size = std::min<uint64_t>(len, 2 * size)) {
    head.resize(size);
    const int frc = fetch(head.data(), size);
    if (frc != KMP_OK) {
      return frc;
    }
    const int rc = metis_header(head.data(), size, len, hd, r);
    metis_report_header(r, hd);
    if (rc == 2) {
      return metis_fail(r);
    }
    if (rc == 0) {
      return KMP_OK;
    }
  }
}

int read_metis_impl(kmp_lp_handle *h, const char *path, kmp_metis_graph **out, kmp_metis_report &r) {
  MetisFile f;
  f.fd = open(path, O_RDONLY);
  struct stat info {};
  if (f.fd < 0 || fstat(f.fd, &info) != 0) {
    return fail(KMP_ERR_INVALID, std::string("cannot open ") + path);
  }
  const uint64_t len = static_cast<uint64_t>(info.st_size);
  r.bytes = len;
  if (len == 0) {
    metis_refuse(r, KMP_METIS_EMPTY, 0, 1, -1);
    return metis_fail(r);
  }
  if (len >= (1ull << 56)) {
    return fail(KMP_ERR_UNSUPPORTED, "files of 2^56 bytes or more are not supported");
  }
  MetisHeader hd;
  int rc = metis_read_header(len, hd, r, [&](uint8_t *dst, uint64_t size) -> int {
    return metis_pread(f.fd, dst, size, 0) ? KMP_OK : fail(KMP_ERR_INVALID, std::string("cannot read ") + path);
  });
  if (rc != KMP_OK) {
    return rc;
  }
  return make_result(h, out, [&](kmp_metis_graph *g) {
    const cudaStream_t st = h->stream;
    MetisJob job{h};
    KMP_CUDA(g->bytes.alloc(len, st, h->device));
    rc = job.prepare(hd, g->bytes.p, len, g);
    if (rc != KMP_OK) {
      return rc;
    }
    MetisStaging stage;
    stage.st = st;
    const uint64_t chunk = std::min<uint64_t>(len, kMetisChunk);
    for (int b = 0; b < 2; ++b) {
      KMP_CUDA(cudaHostAlloc(reinterpret_cast<void **>(&stage.buf[b]), chunk, cudaHostAllocDefault));
      KMP_CUDA(cudaEventCreateWithFlags(&stage.ev[b], cudaEventDisableTiming));
    }
    KMP_CUDA(call_clock_start(h, st));
    uint32_t done = 0; // tiles summarised
    for (uint64_t off = 0, idx = 0; off < len; off += chunk, ++idx) {
      const int b = static_cast<int>(idx & 1u);
      const uint64_t size = std::min<uint64_t>(chunk, len - off);
      if (idx >= 2) {
        KMP_CUDA(cudaEventSynchronize(stage.ev[b])); // the copy of chunk idx - 2 is out of this buffer
      }
      if (!metis_pread(f.fd, stage.buf[b], size, off)) {
        return fail(KMP_ERR_INVALID, std::string("cannot read ") + path);
      }
      KMP_CUDA(cudaMemcpyAsync(g->bytes.p + off, stage.buf[b], size, cudaMemcpyHostToDevice, st));
      KMP_CUDA(cudaEventRecord(stage.ev[b], st));
      // tiles whose bytes (and the byte before them) are all on the device
      const uint32_t ready = off + size == len ? job.tiles : static_cast<uint32_t>((off + size) / KMP_METIS_TILE_BYTES);
      rc = job.summarise(done, ready);
      if (rc != KMP_OK) {
        return rc;
      }
      done = ready;
    }
    rc = job.finish(g, r);
    g->bytes.release();
    return rc != KMP_OK && r.kind != KMP_METIS_OK ? metis_fail(r) : rc;
  });
}

int parse_metis_impl(kmp_lp_handle *h, const uint8_t *d_bytes, uint64_t len, kmp_metis_graph **out,
                     kmp_metis_report &r) {
  r.bytes = len;
  if (len == 0) {
    metis_refuse(r, KMP_METIS_EMPTY, 0, 1, -1);
    return metis_fail(r);
  }
  MetisHeader hd;
  const int hrc = metis_read_header(len, hd, r, [&](uint8_t *dst, uint64_t size) -> int {
    KMP_CUDA(cudaMemcpyAsync(dst, d_bytes, size, cudaMemcpyDeviceToHost, h->stream));
    KMP_CUDA(cudaStreamSynchronize(h->stream));
    return KMP_OK;
  });
  if (hrc != KMP_OK) {
    return hrc;
  }
  return make_result(h, out, [&](kmp_metis_graph *g) {
    MetisJob job{h};
    int rc = job.prepare(hd, d_bytes, len, g);
    if (rc != KMP_OK) {
      return rc;
    }
    KMP_CUDA(call_clock_start(h, h->stream));
    rc = job.summarise(0, job.tiles);
    if (rc == KMP_OK) {
      rc = job.finish(g, r);
      if (rc != KMP_OK && r.kind != KMP_METIS_OK) {
        rc = metis_fail(r);
      }
    }
    return rc;
  });
}

const char *const kMetisKindNames[KMP_METIS_NUM_KINDS] = {
    "ok",          "empty file",         "malformed header",    "unsupported format",   "too large",
    "bad byte",    "missing node weight", "missing edge weight", "zero weight",          "weight too large",
    "neighbor out of range", "self-loop", "too few lines",       "wrong edge count",     "total weight too large"};

} // namespace

extern "C" {

int kmp_read_metis(kmp_lp_handle *h, const char *path, kmp_metis_graph **out, kmp_metis_report *report) {
  int rc = metis_begin(h, out, report);
  if (rc == KMP_OK && path == nullptr) {
    rc = fail(KMP_ERR_INVALID, "null argument");
  }
  return rc != KMP_OK ? rc : read_metis_impl(h, path, out, *report);
}

int kmp_parse_metis_device(kmp_lp_handle *h, const void *d_bytes, uint64_t len, kmp_metis_graph **out,
                           kmp_metis_report *report) {
  int rc = metis_begin(h, out, report);
  if (rc != KMP_OK) {
    return rc;
  }
  if (d_bytes == nullptr && len > 0) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  if ((reinterpret_cast<uintptr_t>(d_bytes) & 15u) != 0) {
    return fail(KMP_ERR_INVALID, "the device bytes must be 16-byte aligned");
  }
  if (len >= (1ull << 56)) {
    return fail(KMP_ERR_UNSUPPORTED, "inputs of 2^56 bytes or more are not supported");
  }
  if (len > 0) { // host memory or another device's memory would reach the kernels as a raw pointer
    cudaPointerAttributes attr{};
    const bool on_device = cudaPointerGetAttributes(&attr, d_bytes) == cudaSuccess &&
                           (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged) &&
                           attr.device == h->device;
    cudaGetLastError(); // an unregistered host pointer leaves no sticky error
    if (!on_device) {
      return fail(KMP_ERR_INVALID, "the bytes must be device memory on the handle's device");
    }
  }
  return parse_metis_impl(h, static_cast<const uint8_t *>(d_bytes), len, out, *report);
}

uint32_t kmp_metis_n(const kmp_metis_graph *g) { return g != nullptr ? g->n : 0; }
uint32_t kmp_metis_m(const kmp_metis_graph *g) { return g != nullptr ? g->m : 0; }

int kmp_metis_device_arrays(const kmp_metis_graph *g, const uint32_t **d_xadj, const uint32_t **d_adjncy,
                            const int32_t **d_vwgt, const int32_t **d_adjwgt) {
  if (g == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  hand_out(d_xadj, g->xadj);
  hand_out(d_adjncy, g->adjncy);
  hand_out(d_vwgt, g->vwgt);
  hand_out(d_adjwgt, g->adjwgt);
  return KMP_OK;
}

int kmp_metis_download(const kmp_metis_graph *g, uint32_t *xadj, uint32_t *adjncy, int32_t *vwgt, int32_t *adjwgt) {
  if (g == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  KMP_CUDA(cudaSetDevice(g->device));
  KMP_CUDA(copy_out(xadj, g->xadj, static_cast<size_t>(g->n) + 1));
  KMP_CUDA(copy_out(adjncy, g->adjncy, g->m));
  KMP_CUDA(copy_out(vwgt, g->vwgt, g->n));
  KMP_CUDA(copy_out(adjwgt, g->adjwgt, g->m));
  return KMP_OK;
}

void kmp_metis_destroy(kmp_metis_graph *g) {
  if (g == nullptr) {
    return;
  }
  cudaSetDevice(g->device); // the arrays free themselves on this device's pool
  delete g;
}

int kmp_metis_report_message(const kmp_metis_report *r, char *buf, size_t size) {
  if (r == nullptr) {
    return fail(KMP_ERR_INVALID, "null argument");
  }
  char dummy = 0;
  if (buf == nullptr || size == 0) {
    buf = &dummy;
    size = 1;
  }
  if (r->kind <= KMP_METIS_OK || r->kind >= KMP_METIS_NUM_KINDS) {
    return std::snprintf(buf, size, "%s", r->extra_lines ? "ignorning extra lines in input file" : ""); // :151
  }
  return std::snprintf(buf, size, "%s at byte %llu (line %llu, vertex %lld)", kMetisKindNames[r->kind],
                       static_cast<unsigned long long>(r->offset), static_cast<unsigned long long>(r->line),
                       static_cast<long long>(r->vertex));
}

} // extern "C"
