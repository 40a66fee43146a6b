"""Seconds per call of the input gradient (loss_and_input_grads) against the parameter gradient
(loss_and_grads) of the same call, their peak device memory, and the GB/s of the two input-gradient
kernels (gcb_output_cotangent_grad_feedback, gcb_broadcast_grad_sum) at the 0.25 degree sizes.

  python tools/time_input_grads.py [--reps 5] [--skip-full]

Cases: 0.25 deg / 37 levels (TASK) with B = 1 and T = 1, 2, and 1 deg / 13 levels (TASK_13) with T = 4,
all InputsAndResiduals(GraphCast) in bf16x3 (autoregressive.Predictor with gradient_checkpointing for
T > 1).  Times are CUDA events around one synchronised call: min / median / max of --reps after one
warm-up.  `loss` (the forward alone) is timed too, to split a gradient call into forward and the rest.
The card name and power limit are read in the same run, and the SM clock is sampled every 100 ms
while each case's calls run (bench.ClockSampler: median of the samples above idle, and the throttle
reasons seen; nvidia-smi, read-only)."""
import argparse
import gc
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

from graphcast_b200 import _native, autoregressive, graphcast, normalization, synthetic  # noqa: E402
from graphcast_b200 import xarray_shim as xs  # noqa: E402
from test_gpu_loss import _stats  # noqa: E402
from bench import ClockSampler  # noqa: E402

DEV = torch.device("cuda:0")


def _card():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                          "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    out = torch.cuda.get_device_name(0) + ", power limit not read"
  return out


def _timed(fn, reps):
  fn()
  times = []
  for _ in range(reps):
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    end.record()
    torch.cuda.synchronize()
    times.append(start.elapsed_time(end) / 1e3)
  return float(np.min(times)), float(np.median(times)), float(np.max(times))


def _peak(fn):
  gc.collect()
  torch.cuda.empty_cache()
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  fn()
  torch.cuda.synchronize()
  return torch.cuda.max_memory_allocated() / 2**30


def case(task, resolution, mesh_size, steps, reps):
  inputs, template, forcings = synthetic.make_example(task, resolution, batch=1, num_target_steps=steps,
                                                      seed=2)
  rng = np.random.default_rng(3)
  targets = xs.Dataset(coords=template.coords)
  for name, v in template.data_vars.items():
    targets[name] = xs.DataArray(rng.standard_normal(v.shape).astype(np.float32), v.dims)
  cfg = graphcast.ModelConfig(resolution, mesh_size, 512, 16, 1, 0.6)
  params = graphcast.init_params(cfg, task, synthetic.num_input_channels(task), seed=1)
  model = graphcast.GraphCast(cfg, task, params=params)
  pred = normalization.InputsAndResiduals(model, *_stats(task, seed=1))
  if steps > 1:
    pred = autoregressive.Predictor(pred, gradient_checkpointing=True)
  pred.loss(inputs, targets, forcings)
  clocks = ClockSampler()
  clocks.start()
  row = {}
  for what in ("loss", "loss_and_grads", "loss_and_input_grads"):
    fn = lambda: getattr(pred, what)(inputs, targets, forcings)
    row[what] = (_timed(fn, reps), _peak(fn))
  clk = clocks.stop()
  fmt = lambda t: f"{t[1]:.3f} s [{t[0]:.3f}, {t[2]:.3f}]"
  (tl, _), (tp, mp), (ti, mi) = row["loss"], row["loss_and_grads"], row["loss_and_input_grads"]
  print(f"{resolution} deg, {len(task.pressure_levels)} levels, T = {steps} (median [min, max] of "
        f"{reps}): loss {fmt(tl)}; loss_and_grads {fmt(tp)} (peak {mp:.1f} GiB); loss_and_input_grads "
        f"{fmt(ti)} (peak {mi:.1f} GiB); ratio of medians {ti[1] / tp[1]:.3f}; SM clock under load "
        f"{clk['sm_mhz']} MHz ({clk.get('samples', 0)} samples, reasons {clk['reasons']})", flush=True)
  del model, pred
  gc.collect()
  torch.cuda.empty_cache()


def kernels(reps):
  """The two kernels at the 0.25 degree / 37 level sizes: 227 outputs, 471 rows, 721 x 1440 nodes."""
  lib = _native.lib()
  n_lat, n_lon, n_out, n_rows = 721, 1440, 227, 471
  n = n_lat * n_lon
  st = lambda: torch.cuda.current_stream().cuda_stream
  cot = torch.randn(n_out, n, device=DEV)
  a_next = torch.randn(n_rows, n, device=DEV)
  a_out = torch.empty(n_rows, n, device=DEV)
  g = torch.empty(n, 256, device=DEV)
  scale = torch.rand(n_out, device=DEV) + 0.5
  dpred = torch.arange(n_out, dtype=torch.int32, device=DEV)
  resid = torch.full([n_rows], -1, dtype=torch.int32, device=DEV)
  resid[:n_out] = dpred
  carry = torch.arange(n_rows, dtype=torch.int32, device=DEV) - 1
  seed = lambda: _native.check(lib.gcb_output_cotangent_grad_feedback(
      n_out, n, scale.data_ptr(), cot.data_ptr(), a_next.data_ptr(), dpred.data_ptr(), n_rows,
      resid.data_ptr(), carry.data_ptr(), a_out.data_ptr(), g.data_ptr(), 256, st()), "seed")
  t = _timed(seed, reps * 10)[1]
  nbytes = 4.0 * n * (3 * n_out + 2 * n_rows)
  print(f"gcb_output_cotangent_grad_feedback: {t * 1e3:.3f} ms, {nbytes / t / 1e9:.0f} GB/s", flush=True)
  for mode, rows, label in ((_native.BCAST_NONE, 2, "copy, 2 static rows"),
                            (_native.BCAST_LAT, 2, "over lat, 2 rows"),
                            (_native.BCAST_LAT_LON, 4, "over lat and lon, 4 rows")):
    width = (n, n_lon, 1)[mode]
    out = torch.zeros(rows, width, device=DEV)
    idx = torch.arange(rows, dtype=torch.int32, device=DEV)
    fn = lambda: _native.check(lib.gcb_broadcast_grad_sum(a_out.data_ptr(), n_lat, n_lon, rows,
                                                          idx.data_ptr(), mode, out.data_ptr(), 1, st()),
                               "sum")
    t = _timed(fn, reps * 10)[1]
    nbytes = 4.0 * rows * (n + 2 * width)
    print(f"gcb_broadcast_grad_sum ({label}): {t * 1e3:.3f} ms, {nbytes / t / 1e9:.0f} GB/s", flush=True)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=5)
  ap.add_argument("--skip-full", action="store_true", help="only the 1 degree case and the kernels")
  args = ap.parse_args()
  print(f"card: {_card()}", flush=True)
  kernels(args.reps)
  case(graphcast.TASK_13, 1.0, 5, 4, args.reps)
  if not args.skip_full:
    case(graphcast.TASK, 0.25, 6, 1, args.reps)
    case(graphcast.TASK, 0.25, 6, 2, args.reps)


if __name__ == "__main__":
  main()
