"""The seed kernel of the Gauss-Newton product over several target times
(gcb_output_loss_gn_seed_feedback) compiles for sm_90a without register spills: `-Xptxas -v` reports 0
bytes of stack and spill.  Needs nvcc (CUDA 12), no GPU."""
import os
import re
import shutil
import subprocess

import pytest

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "graphcast_b200", "csrc")
KERNEL = "output_loss_gn_seed_feedback_kernel"


def _nvcc():
  for cand in (shutil.which("nvcc"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"),
                                                  "bin", "nvcc")):
    if cand and os.path.exists(cand):
      return cand
  return None


def test_gn_seed_feedback_kernel_does_not_spill(tmp_path):
  nvcc = _nvcc()
  if nvcc is None:
    pytest.skip("nvcc not found")
  src = tmp_path / "kernels.cu"
  src.write_text('#include "backward_kernels.cuh"\n')
  out = subprocess.run(
      [nvcc, "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-cubin",
       "-I", CSRC, "-o", str(tmp_path / "kernels.cubin"), str(src)],
      capture_output=True, text=True, timeout=600)
  assert out.returncode == 0, out.stderr[-2000:]
  # ptxas prints, per entry function, "Compiling entry function '<name>'" and then its stack / spills
  report = {}
  name = None
  for line in out.stderr.splitlines():
    m = re.search(r"Compiling entry function '([^']+)'", line)
    if m:
      name = m.group(1)
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
    if m and name:
      report[name] = tuple(int(x) for x in m.groups())
  found = [(n, r) for n, r in report.items() if KERNEL in n]
  assert len(found) == 1, (KERNEL, sorted(report))
  assert found[0][1] == (0, 0, 0), found
