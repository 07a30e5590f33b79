// Compiles against the C++ adapters + C ABI; used by tests/test_cpp_metis_adapter.py to check that
// kaminpar_b200::read_metis, MetisGraph and MetisError are valid C++20 and link, and (with a GPU) that the files given
// on the command line come back as the oracle reads them. Without a device it exits with status 1 and the adapter's
// error message.
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
    // ADAPTER_DUMP=<file>: per file "kind", then for a graph "xadj / adjncy / vwgt / adjwgt" and the report's line
    for (int i = 1; i < argc; ++i) {
      auto line = [dump](const auto &v) {
        for (auto x : v) std::fprintf(dump, "%lld ", static_cast<long long>(x));
        std::fprintf(dump, "\n");
      };
      try {
        const MetisGraph g = read_metis(h.get(), argv[i]);
        const MetisGraph::Host c = g.download();
        std::printf("%s: n=%u m=%u\n", argv[i], g.n(), g.m());
        if (dump != nullptr) {
          std::fprintf(dump, "%d\n", g.report().kind);
          line(c.xadj);
          line(c.adjncy);
          line(c.vwgt);
          line(c.adjwgt);
          std::fprintf(dump, "%s\n", g.report().message().c_str());
        }
      } catch (const MetisError &e) {
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
