"""bench.py host helpers: the algorithmic FLOP model must reproduce SURVEY.md section 8(d)
(29.29 TFLOP per 0.25 degree / 37 level step, 28.81 operational, 4.11 for the 1 degree model),
since `roofline.achieved` and the CPU-sample scaling are defined on it."""
import importlib.util
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def bench():
  spec = importlib.util.spec_from_file_location("bench_module", os.path.join(ROOT, "bench.py"))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod


@pytest.mark.parametrize("workload,tflop", [("graphcast_0.25deg_37lvl", 29.29),
                                            ("graphcast_operational_0.25deg_13lvl", 28.81),
                                            ("graphcast_small_1deg_13lvl", 4.11)])
def test_algorithmic_flops_match_survey(bench, workload, tflop):
  got = bench.algorithmic_flops(*bench.full_workload_sizes(workload)) / 1e12
  assert abs(got - tflop) / tflop < 0.004


def test_thread_candidates(bench):
  assert bench.thread_candidates(128) == [32, 16]        # the oversubscribed 128-thread pass is skipped
  assert bench.thread_candidates(8) == [8]
  assert bench.thread_candidates(48) == [48, 32, 16]


def test_ncu_traffic_reads_a_launch_list(tmp_path, monkeypatch):
  import bench
  assert bench.ncu_traffic(bench.DEFAULT_WORKLOAD, "bf16x3") == (None, None)   # none committed
  # A launch list in the format tools/ncu_launch_list.py writes: kernel names may contain commas.
  (tmp_path / "profiles").mkdir()
  (tmp_path / "profiles" / "r02_launches_ncu.csv").write_text(
      "# one step\n"
      "id,kernel,ms,dram_read,dram_write\n"
      "0,gcb::mlp_chain_tc_kernel<true, true, false>(gcb_chain_desc, int, int),9.5,60e9,40e9\n"
      "1,gcb::segment_sum_kernel<4>(const float *, int),3.2,12e9,5e9\n"
      "2,gcb::mlp_layer_tc_kernel<true, false, true>(gcb_layer_desc),1.1,7e9,3e9\n")
  monkeypatch.setattr(bench, "REPO", str(tmp_path))
  tc, src = bench.ncu_traffic(bench.DEFAULT_WORKLOAD, "bf16x3")
  assert tc == 110e9                                      # tensor-core kernels: DRAM bytes per step
  assert "r02_launches_ncu.csv" in src and "127.0 GB" in src
  assert bench.ncu_traffic("graphcast_small_1deg_13lvl", "bf16x3") == (None, None)


def test_algorithmic_flops_match_the_survey():
  import bench
  f = bench.algorithmic_flops(1038240, 40962, 1618818, 327660, 3114720, 471, 227, 16)
  assert abs(f / 1e12 - 29.29) < 0.01                     # SURVEY.md section 8(d)
