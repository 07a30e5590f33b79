// Compiles against the C++ adapters + C ABI; used by tests/test_cpp_parhip_adapter.py to check that
// kaminpar_b200::read_parhip, ParhipGraph and ParhipError are valid C++20 and link, and (with a GPU) that the files
// given on the command line come back as the oracle reads them in the external degree-bucket order. Without a device
// it exits with status 1 and the adapter's error message.
#include <cstdio>
#include <cstdlib>

#include "kaminpar_b200_adapters.hpp"

using namespace kaminpar_b200;

int main(int argc, char **argv) {
  std::FILE *dump = nullptr;
  if (const char *path = std::getenv("ADAPTER_DUMP")) {
    dump = std::fopen(path, "w");
  }
  try {
    detail::Handle h(detail::balancer_config(EngineContext{}));
    // ADAPTER_DUMP=<file>: per file "kind", then for a graph "xadj / adjncy / vwgt / adjwgt / old_to_new", else the
    // report's line
    for (int i = 1; i < argc; ++i) {
      auto line = [dump](const auto &v) {
        for (auto x : v) std::fprintf(dump, "%lld ", static_cast<long long>(x));
        std::fprintf(dump, "\n");
      };
      try {
        const ParhipGraph g = read_parhip(h.get(), argv[i], ParhipOrdering::EXTERNAL_DEGREE_BUCKETS);
        const ParhipGraph::Host c = g.download();
        std::printf("%s: n=%u m=%u sorted=%d\n", argv[i], g.n(), g.m(), g.sorted() ? 1 : 0);
        if (dump != nullptr) {
          std::fprintf(dump, "%d\n", g.report().kind);
          line(c.xadj);
          line(c.adjncy);
          line(c.vwgt);
          line(c.adjwgt);
          line(c.old_to_new);
        }
      } catch (const ParhipError &e) {
        std::printf("%s: %s\n", argv[i], e.what());
        if (dump != nullptr) {
          std::fprintf(dump, "%d\n%s\n", e.report().kind, e.report().message().c_str());
        }
      }
    }
    std::printf("adapter ok\n");
  } catch (const std::exception &e) {
    std::printf("exception: %s\n", e.what());
    return 1;
  }
  if (dump != nullptr) {
    std::fclose(dump);
  }
  return 0;
}
