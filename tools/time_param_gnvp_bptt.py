"""Seconds per call and peak device memory of the Gauss-Newton product over several target times
(autoregressive.Predictor(..., gradient_checkpointing=True).loss_and_param_gnvp) against multi-step
loss_and_grads (backprop through time) and multi-step param_jvp.

  python tools/time_param_gnvp_bptt.py [--reps 3] [--configs 1,0.25]

Cases: InputsAndResiduals(GraphCast) in bf16x3, B = 1, random tangents on every parameter and random
targets; at 1 deg / 13 levels (TASK_13, mesh 5) with T = 2 and 4, and at 0.25 deg / 37 levels (TASK,
mesh 6) with T = 2.  After one warm-up of each, the calls alternate in one process, rep by rep, so that
clock drift reaches all of them alike.  Times are CUDA events around one synchronised call: median, min
and max of --reps; the peak is torch.cuda.max_memory_allocated over one more call of each, from an
empty allocator cache.  The card name and power limit are read in the same run, and the SM clock is
sampled while the calls run (bench.ClockSampler; nvidia-smi, read-only).  A call that runs out of
device memory is reported as such with the peak it reached."""
import argparse
import gc
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

from graphcast_b200 import autoregressive, graphcast, normalization, synthetic  # noqa: E402
from test_gpu_loss import _stats  # noqa: E402
from time_input_grads import _card, _peak  # noqa: E402
from time_input_jvp import _random_like  # noqa: E402
from time_param_hvp import _once  # noqa: E402
from bench import ClockSampler  # noqa: E402

CONFIGS = {"1": [(1.0, 5, graphcast.TASK_13, 2), (1.0, 5, graphcast.TASK_13, 4)],
           "0.25": [(0.25, 6, graphcast.TASK, 2)]}


def case(resolution, mesh_size, task, steps, reps):
  gc.collect()
  torch.cuda.empty_cache()
  inputs, template, forcings = synthetic.make_example(task, resolution, batch=1,
                                                      num_target_steps=steps, seed=2)
  rng = np.random.default_rng(3)
  targets = _random_like(template, rng)
  cfg = graphcast.ModelConfig(resolution, mesh_size, 512, 16, 1, 0.6)
  params = graphcast.init_params(cfg, task, synthetic.num_input_channels(task), seed=1)
  v = {n: {f: (rng.standard_normal(np.shape(a)) * (float(np.std(a)) or 0.1)).astype(np.float32)
           for f, a in fs.items()} for n, fs in params.items()}
  model = graphcast.GraphCast(cfg, task, params=params)
  ar = autoregressive.Predictor(normalization.InputsAndResiduals(model, *_stats(task, seed=1)),
                                gradient_checkpointing=True)
  calls = {
      "loss_and_param_gnvp": lambda: ar.loss_and_param_gnvp(inputs, targets, forcings, v),
      "loss_and_grads": lambda: ar.loss_and_grads(inputs, targets, forcings),
      "param_jvp": lambda: ar.param_jvp(inputs, targets, forcings, v),
  }
  tag = f"{resolution} deg / {len(task.pressure_levels)} levels, T = {steps}"
  failed = {}
  for what, fn in calls.items():
    try:
      gc.collect()
      torch.cuda.empty_cache()
      torch.cuda.reset_peak_memory_stats()
      fn()
    except torch.cuda.OutOfMemoryError:
      failed[what] = torch.cuda.max_memory_allocated() / 2**30
      print(f"{tag}: {what} ran out of device memory at a peak of {failed[what]:.1f} GiB",
            flush=True)
  calls = {w: fn for w, fn in calls.items() if w not in failed}
  clocks = ClockSampler()
  clocks.start()
  times = {what: [] for what in calls}
  for _ in range(reps):
    for what, fn in calls.items():
      gc.collect()
      torch.cuda.empty_cache()
      times[what].append(_once(fn))
  clk = clocks.stop()
  peaks = {what: _peak(fn) for what, fn in calls.items()}
  for what, ts in times.items():
    print(f"{tag}: {what}: {np.median(ts):.3f} s [{min(ts):.3f}, {max(ts):.3f}] (median [min, max] "
          f"of {reps}), peak {peaks[what]:.1f} GiB", flush=True)
  if "loss_and_param_gnvp" in times:
    g = np.median(times["loss_and_param_gnvp"])
    ratios = ", ".join(f"/ {w} {g / np.median(times[w]):.2f}" for w in times if w != "loss_and_param_gnvp")
    print(f"{tag}: loss_and_param_gnvp {ratios}; SM clock under load {clk['sm_mhz']} MHz "
          f"({clk.get('samples', 0)} samples, reasons {clk['reasons']})", flush=True)
  del model, ar, calls
  gc.collect()
  torch.cuda.empty_cache()


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=3)
  ap.add_argument("--configs", default="1,0.25")
  args = ap.parse_args()
  print(f"card: {_card()}", flush=True)
  for key in args.configs.split(","):
    for config in CONFIGS[key]:
      case(*config, args.reps)


if __name__ == "__main__":
  main()
