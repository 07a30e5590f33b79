// Bridge to the UNMODIFIED reference's two graph validators, for the CPU tests of tests/test_validate_bridge.py and
// tests/golden/make_validate_golden.py. Compiled by them against the reference headers and linked against the
// reference partitioner the build leaves in oracle/_ref/libkaminpar_ref_full.so (serial oneTBB stand-in: one thread).
#include <sys/wait.h>
#include <unistd.h>

#include <cstdint>
#include <cstdio>
#include <cstring>
#include <fcntl.h>
#include <iostream>
#include <memory>
#include <sstream>
#include <string>

#include "kaminpar-shm/datastructures/csr_graph.h"
#include "kaminpar-shm/datastructures/graph.h"
#include "kaminpar-shm/graphutils/graph_validator.h"
#include "kaminpar-shm/kaminpar.h"

#include "kaminpar-common/datastructures/static_array.h"
#include "kaminpar-common/logger.h"
#include "kaminpar-common/timer.h"

using namespace kaminpar;
using namespace kaminpar::shm;

namespace {
template <typename T> StaticArray<T> copy_array(const T *src, std::size_t n) {
  StaticArray<T> a(n);
  if (n > 0) {
    std::memcpy(a.data(), src, n * sizeof(T));
  }
  return a;
}
} // namespace

extern "C" {

// debug::validate_graph(n, xadj, adjncy, {}, adjwgt) with check_undirected = true and num_pseudo_nodes = 0, as
// KaMinPar::borrow_and_mutate_graph / copy_graph assert it (kaminpar.cc:174, :215). Returns its verdict (1 valid);
// msg[msg_size] receives everything it printed (its LOG_WARNING line, colour codes included). adjwgt NULL: no weights.
// The caller passes arrays with xadj[n] == m (the reference reads m from xadj[n]).
int bridge_validate_graph(std::uint32_t n, std::uint32_t m, const std::uint32_t *xadj, const std::uint32_t *adjncy,
                          const std::int32_t *adjwgt, char *msg, std::size_t msg_size) {
  std::ostringstream captured;
  const bool quiet = Logger::is_quiet(); // another caller in this process may have silenced the logger
  Logger::set_quiet_mode(false);
  std::streambuf *old = std::cout.rdbuf(captured.rdbuf());
  const bool ok = debug::validate_graph(
      n, copy_array<EdgeID>(xadj, static_cast<std::size_t>(n) + 1), copy_array<NodeID>(adjncy, m),
      StaticArray<NodeWeight>(), adjwgt != nullptr ? copy_array<EdgeWeight>(adjwgt, m) : StaticArray<EdgeWeight>(),
      true, 0
  );
  std::cout.rdbuf(old);
  Logger::set_quiet_mode(quiet);
  std::snprintf(msg, msg_size, "%s", captured.str().c_str());
  return ok ? 1 : 0;
}

// validate_undirected_graph(graph) (graphutils/graph_validator.cc, the CLI's --validate) in a forked child, since it
// ends the process with std::exit(1) on an invalid graph. Returns the child's exit status (0: valid, 1: invalid) or
// -1 when the child did not exit normally. Its message goes to /dev/null.
int bridge_validate_undirected(std::uint32_t n, std::uint32_t m, const std::uint32_t *xadj,
                               const std::uint32_t *adjncy, const std::int32_t *adjwgt) {
  std::fflush(nullptr);
  const pid_t pid = fork();
  if (pid < 0) {
    return -1;
  }
  if (pid == 0) {
    const int devnull = open("/dev/null", O_WRONLY);
    if (devnull >= 0) {
      dup2(devnull, 1);
      dup2(devnull, 2);
    }
    DISABLE_TIMERS();
    Graph graph(std::make_unique<CSRGraph>(
        copy_array<EdgeID>(xadj, static_cast<std::size_t>(n) + 1), copy_array<NodeID>(adjncy, m),
        StaticArray<NodeWeight>(), adjwgt != nullptr ? copy_array<EdgeWeight>(adjwgt, m) : StaticArray<EdgeWeight>(),
        false
    ));
    validate_undirected_graph(graph);
    _exit(0);
  }
  int status = 0;
  if (waitpid(pid, &status, 0) != pid || !WIFEXITED(status)) {
    return -1;
  }
  return WEXITSTATUS(status);
}

} // extern "C"
