// The reference's initial bipartitioner as a program (_ref/bipartition_ref, _ref/bipartition_ref_omp), timed by
// scripts/bench_bipartition.py against kmp_bipartition_subgraphs (DESIGN.md §20). Unmodified reference code from
// _ref/libkaminpar_ref_full.so; this file only reads the blocks and calls it.
//
//   bipartition_ref <blocks.bin> <out.bin> <preset>
//
// blocks.bin (little endian): uint32 num_blocks, current_k, input_k; int32 uniform, total_node_weight, seed;
// double epsilon; int32 max_block_weights[input_k]; then per block: uint32 block_id, n, m, flags (1: node weights,
// 2: edge weights), xadj[n + 1], adjncy[m], [vwgt[n]], [adjwgt[m]].
// out.bin: the blocks' sub-partitions, concatenated in input order. stdout: one JSON line with the time.
//
// Each block: Random::reseed(seed + block_id) (the OpenMP build: reinit of the thread's own Random instance) and a
// fresh InitialBipartitionerWorkerPool(ctx).bipartition(&block, block_id, current_k, false) -- the rule of
// DESIGN.md §20. Only those calls are timed; reading the file and building the CSR graphs are not. The OpenMP build
// runs the blocks on all cores, one pool per block, for timing: the reference's own parallel driver shares pools
// per thread and a random stream per thread.
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <memory>
#include <vector>

#ifdef _OPENMP
#include <omp.h>
#endif

#include "kaminpar-shm/datastructures/csr_graph.h"
#include "kaminpar-shm/datastructures/graph.h"
#include "kaminpar-shm/initial_partitioning/initial_bipartitioner_worker_pool.h"
#include "kaminpar-shm/kaminpar.h"

#include "kaminpar-common/datastructures/static_array.h"
#include "kaminpar-common/random.h"

using namespace kaminpar;
using namespace kaminpar::shm;

namespace {
template <typename T> bool read(std::FILE *f, T *dst, std::size_t count) {
  return std::fread(dst, sizeof(T), count, f) == count;
}
template <typename T> StaticArray<T> read_array(std::FILE *f, std::size_t count, bool &ok) {
  StaticArray<T> a(count);
  ok = ok && (count == 0 || read(f, a.data(), count));
  return a;
}
} // namespace

int main(int argc, char **argv) {
  if (argc != 4) {
    std::fprintf(stderr, "usage: %s <blocks.bin> <out.bin> <preset>\n", argv[0]);
    return 2;
  }
  std::FILE *f = std::fopen(argv[1], "rb");
  if (f == nullptr) {
    std::perror(argv[1]);
    return 1;
  }
  std::uint32_t head[3];
  std::int32_t ihead[3];
  double epsilon = 0.0;
  bool ok = read(f, head, 3) && read(f, ihead, 3) && read(f, &epsilon, 1);
  const std::uint32_t num_blocks = head[0], current_k = head[1], input_k = head[2];
  std::vector<BlockWeight> mbw(input_k);
  ok = ok && read(f, mbw.data(), input_k);
  std::vector<std::uint32_t> ids(num_blocks);
  std::vector<std::unique_ptr<Graph>> blocks;
  for (std::uint32_t i = 0; ok && i < num_blocks; ++i) {
    std::uint32_t h[4];
    ok = read(f, h, 4);
    if (!ok) {
      break;
    }
    ids[i] = h[0];
    const std::uint32_t n = h[1], m = h[2];
    auto xadj = read_array<EdgeID>(f, n + 1, ok);
    auto adj = read_array<NodeID>(f, m, ok);
    auto vw = (h[3] & 1u) ? read_array<NodeWeight>(f, n, ok) : StaticArray<NodeWeight>();
    auto ew = (h[3] & 2u) ? read_array<EdgeWeight>(f, m, ok) : StaticArray<EdgeWeight>();
    blocks.push_back(std::make_unique<Graph>(
        std::make_unique<CSRGraph>(std::move(xadj), std::move(adj), std::move(vw), std::move(ew))));
  }
  std::fclose(f);
  if (!ok) {
    std::fprintf(stderr, "%s: truncated input\n", argv[1]);
    return 1;
  }

  Context ctx = create_context_by_preset_name(argv[3]);
  // the input graph's partition context: setup() reads only the totals, so one vertex carries the total weight
  StaticArray<EdgeID> nodes(2);
  nodes[0] = nodes[1] = 0;
  StaticArray<NodeWeight> w(1);
  w[0] = ihead[1];
  Graph input(std::make_unique<CSRGraph>(std::move(nodes), StaticArray<NodeID>(0), std::move(w),
                                         StaticArray<EdgeWeight>()));
  if (ihead[0] != 0) {
    ctx.partition.setup(input, input_k, epsilon);
  } else {
    ctx.partition.setup(input, std::vector<BlockWeight>(mbw), false);
  }

  std::vector<std::vector<BlockID>> out(num_blocks);
  const auto t0 = std::chrono::steady_clock::now();
#ifdef _OPENMP
#pragma omp parallel for schedule(dynamic, 1)
#endif
  for (std::int64_t i = 0; i < static_cast<std::int64_t>(num_blocks); ++i) {
    const std::int32_t seed = static_cast<std::int32_t>(static_cast<std::uint32_t>(ihead[2]) + ids[i]);
#ifdef _OPENMP
    Random::instance().reinit(seed);
#else
    Random::reseed(seed);
#endif
    InitialBipartitionerWorkerPool pool(ctx);
    PartitionedGraph pg = pool.bipartition(blocks[i].get(), ids[i], current_k, false);
    out[i].resize(blocks[i]->n());
    for (NodeID u = 0; u < blocks[i]->n(); ++u) {
      out[i][u] = pg.block(u);
    }
  }
  const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();

  std::FILE *o = std::fopen(argv[2], "wb");
  if (o == nullptr) {
    std::perror(argv[2]);
    return 1;
  }
  for (const auto &p : out) {
    std::fwrite(p.data(), sizeof(BlockID), p.size(), o);
  }
  std::fclose(o);
  int threads = 1;
#ifdef _OPENMP
  threads = omp_get_max_threads();
#endif
  std::printf("{\"blocks\": %u, \"threads\": %d, \"ms\": %.3f}\n", num_blocks, threads, ms);
  return 0;
}
