"""Seconds per call and peak device memory of the parameter tangent (param_jvp) against the forecast
(__call__) and the input tangent (input_jvp), and of the Gauss-Newton product (loss_and_param_gnvp)
against the parameter gradient (loss_and_grads) of the same call.

  python tools/time_param_jvp.py [--reps 3] [--skip-full]

Cases: 1 deg / 13 levels (TASK_13) with B = 1 and T = 1 and 4, and 0.25 deg / 37 levels (TASK) with
T = 1, all InputsAndResiduals(GraphCast) in bf16x3 (autoregressive.Predictor for T > 1, where only
param_jvp, input_jvp and __call__ run).  The parameter tangents are random on every parameter, the
input tangents on every input and forcing variable.  Times are CUDA events around one synchronised
call: median, min and max of --reps after one warm-up; the peak is torch.cuda.max_memory_allocated over
one more call.  The card name and power limit are read in the same run, and the SM clock is sampled
while each case's calls run (bench.ClockSampler; nvidia-smi, read-only)."""
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
from time_input_grads import _card, _peak, _timed  # noqa: E402
from time_input_jvp import _random_like  # noqa: E402
from bench import ClockSampler  # noqa: E402


def case(task, resolution, mesh_size, steps, reps):
  inputs, template, forcings = synthetic.make_example(task, resolution, batch=1, num_target_steps=steps,
                                                      seed=2)
  rng = np.random.default_rng(3)
  d_in, d_f, targets = _random_like(inputs, rng), _random_like(forcings, rng), _random_like(template, rng)
  cfg = graphcast.ModelConfig(resolution, mesh_size, 512, 16, 1, 0.6)
  params = graphcast.init_params(cfg, task, synthetic.num_input_channels(task), seed=1)
  v = {n: {f: (rng.standard_normal(np.shape(a)) * (float(np.std(a)) or 0.1)).astype(np.float32)
           for f, a in fs.items()} for n, fs in params.items()}
  model = graphcast.GraphCast(cfg, task, params=params)
  pred = normalization.InputsAndResiduals(model, *_stats(task, seed=1))
  if steps > 1:
    pred = autoregressive.Predictor(pred)
  pred(inputs, template, forcings)
  calls = {"__call__": lambda: pred(inputs, template, forcings),
           "input_jvp": lambda: pred.input_jvp(inputs, template, forcings, d_in, d_f),
           "param_jvp": lambda: pred.param_jvp(inputs, template, forcings, v)}
  if steps == 1:
    calls["loss_and_grads"] = lambda: pred.loss_and_grads(inputs, targets, forcings)
    calls["loss_and_param_gnvp"] = lambda: pred.loss_and_param_gnvp(inputs, targets, forcings, v)
  clocks = ClockSampler()
  clocks.start()
  row = {}
  for what, fn in calls.items():
    gc.collect()
    torch.cuda.empty_cache()
    row[what] = (_timed(fn, reps), _peak(fn))
  clk = clocks.stop()
  fmt = lambda r: f"{r[0][1]:.3f} s [{r[0][0]:.3f}, {r[0][2]:.3f}] (peak {r[1]:.1f} GiB)"
  ratio = lambda a, b: f"{a} / {b} {row[a][0][1] / row[b][0][1]:.2f}"
  ratios = [ratio("param_jvp", "__call__"), ratio("param_jvp", "input_jvp")]
  if steps == 1:
    ratios.append(ratio("loss_and_param_gnvp", "loss_and_grads"))
  print(f"{resolution} deg, {len(task.pressure_levels)} levels, T = {steps} (median [min, max] of "
        f"{reps}): " + "; ".join(f"{what} {fmt(r)}" for what, r in row.items()) + "; " +
        ", ".join(ratios) + f"; SM clock under load {clk['sm_mhz']} MHz ({clk.get('samples', 0)} "
        f"samples, reasons {clk['reasons']})", flush=True)
  del model, pred, calls


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=3)
  ap.add_argument("--skip-full", action="store_true", help="only the 1 degree cases")
  args = ap.parse_args()
  print(f"card: {_card()}", flush=True)
  case(graphcast.TASK_13, 1.0, 5, 1, args.reps)
  case(graphcast.TASK_13, 1.0, 5, 4, args.reps)
  if not args.skip_full:
    case(graphcast.TASK, 0.25, 6, 1, args.reps)


if __name__ == "__main__":
  main()
