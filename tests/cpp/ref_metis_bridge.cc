// Bridge to the UNMODIFIED reference's METIS reader (kaminpar-io/metis_parser.cc, compiled into this library by
// tests/test_metis_bridge.py and tests/golden/make_metis_golden.py against the reference headers, the rest of the
// reference linked from oracle/_ref/libkaminpar_ref_full.so). Built twice from this file:
//   with -DNDEBUG (the Release build users run): bridge_read calls io::metis::read_graph (= csr_read, unsorted) in
//     this process and keeps the graph for bridge_sizes / bridge_copy, with everything the reader printed;
//   without -DNDEBUG (KASSERT is plain assert() without kassert, assert.h:22-28): bridge_assert runs the same read in a
//     forked child whose failed assert() reports its file and line through a pipe instead of aborting.
#include <sys/wait.h>
#include <unistd.h>

#include <cstdint>
#include <cstdio>
#include <cstring>
#include <fcntl.h>
#include <iostream>
#include <optional>
#include <sstream>
#include <string>

#include "kaminpar-io/metis_parser.h"
#include "kaminpar-shm/datastructures/csr_graph.h"
#include "kaminpar-shm/datastructures/graph.h"

#include "kaminpar-common/logger.h"

using namespace kaminpar;
using namespace kaminpar::shm;

namespace {
std::optional<Graph> g_graph;
int g_assert_fd = -1;
} // namespace

extern "C" {

// The child's failed assert(): "file:line" to the parent, then exit status 3 (no abort, no core file).
void __assert_fail(const char *, const char *file, unsigned int line, const char *) noexcept {
  char buf[512];
  const int len = std::snprintf(buf, sizeof(buf), "%s:%u", file, line);
  if (g_assert_fd >= 0 && len > 0) {
    const ssize_t wrote = write(g_assert_fd, buf, static_cast<size_t>(len));
    (void)wrote;
  }
  _exit(3);
}

// 1: a graph (kept for bridge_sizes / bridge_copy), 0: nullopt. msg receives what the reader printed.
int bridge_read(const char *path, char *msg, std::size_t msg_size) {
  std::ostringstream captured;
  const bool quiet = Logger::is_quiet();
  Logger::set_quiet_mode(false);
  std::streambuf *old = std::cout.rdbuf(captured.rdbuf());
  g_graph = io::metis::read_graph(path, false, NodeOrdering::NATURAL);
  std::cout.rdbuf(old);
  Logger::set_quiet_mode(quiet);
  std::snprintf(msg, msg_size, "%s", captured.str().c_str());
  return g_graph.has_value() ? 1 : 0;
}

void bridge_sizes(std::uint64_t *n, std::uint64_t *m, int *node_weighted, int *edge_weighted) {
  const auto &g = concretize<CSRGraph>(*g_graph);
  *n = g.n();
  *m = g.m();
  *node_weighted = g.raw_node_weights().empty() ? 0 : 1;
  *edge_weighted = g.raw_edge_weights().empty() ? 0 : 1;
}

void bridge_copy(std::uint32_t *xadj, std::uint32_t *adjncy, std::int32_t *vwgt, std::int32_t *adjwgt) {
  const auto &g = concretize<CSRGraph>(*g_graph);
  std::memcpy(xadj, g.raw_nodes().data(), (g.n() + 1) * sizeof(std::uint32_t));
  std::memcpy(adjncy, g.raw_edges().data(), g.m() * sizeof(std::uint32_t));
  if (vwgt != nullptr && !g.raw_node_weights().empty()) {
    std::memcpy(vwgt, g.raw_node_weights().data(), g.n() * sizeof(std::int32_t));
  }
  if (adjwgt != nullptr && !g.raw_edge_weights().empty()) {
    std::memcpy(adjwgt, g.raw_edge_weights().data(), g.m() * sizeof(std::int32_t));
  }
  g_graph.reset();
}

// The read in a forked child: 0 if it returned, 3 with where = "file:line" if an assertion fired, -1 otherwise.
int bridge_assert(const char *path, char *where, std::size_t where_size) {
  int fds[2];
  if (pipe(fds) != 0) {
    return -1;
  }
  std::fflush(nullptr);
  const pid_t pid = fork();
  if (pid < 0) {
    return -1;
  }
  if (pid == 0) {
    close(fds[0]);
    g_assert_fd = fds[1];
    const int devnull = open("/dev/null", O_WRONLY);
    if (devnull >= 0) {
      dup2(devnull, 1);
      dup2(devnull, 2);
    }
    const auto graph = io::metis::read_graph(path, false, NodeOrdering::NATURAL);
    _exit(0);
  }
  close(fds[1]);
  std::string got;
  char buf[256];
  ssize_t r;
  while ((r = read(fds[0], buf, sizeof(buf))) > 0) {
    got.append(buf, static_cast<size_t>(r));
  }
  close(fds[0]);
  int status = 0;
  if (waitpid(pid, &status, 0) != pid || !WIFEXITED(status)) {
    return -1;
  }
  std::snprintf(where, where_size, "%s", got.c_str());
  return WEXITSTATUS(status);
}

} // extern "C"
