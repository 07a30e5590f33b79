"""The C++ adapter kaminpar_b200::bipartition_subgraphs (include/kaminpar_b200_adapters.hpp) is valid C++20 and links
against the C-ABI library, whose kmp_ip_default_config answers without a device."""
import os
import shutil
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "kaminpar_b200", "csrc")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")

SRC = r"""
#include <cstdio>
#include "kaminpar_b200_adapters.hpp"
int main() {
  auto *fn = &kaminpar_b200::bipartition_subgraphs;
  const kmp_ip_config c = kmp_ip_default_config();
  std::printf("%u %d %d %p\n", c.contraction_limit, c.min_num_repetitions, c.refinement.algorithm,
              reinterpret_cast<void *>(fn));
  return 0;
}
"""


def test_bipartition_adapter_compiles_and_links(tmp_path):
    src = tmp_path / "bip.cc"
    src.write_text(SRC)
    exe = str(tmp_path / "bip")
    r = subprocess.run([CXX, "-std=c++20", "-Wall", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe,
                        "-L" + LIBDIR, "-lkaminpar_b200", "-Wl,-rpath," + LIBDIR], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.split()[:3] == ["20", "10", "1"]
