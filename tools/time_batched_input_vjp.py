"""Seconds per call of input_vjp for K cotangents at once (batched_input_vjp) against K input_vjp calls
with the same cotangents, their peak device memory, and (--profile, a run of its own) a torch.profiler
breakdown of one 1 degree call.

  python tools/time_batched_input_vjp.py [--reps 3] [--skip-full | --skip-1deg] [--profile]

Cases: 1 deg / 13 levels (TASK_13) with K = 1, 4, 8, 16 at T = 1 and 4, and 0.25 deg / 37 levels (TASK)
with K = 2, one direction per pass, at T = 1 and 2 (at T = 2 the one rollout forward and its stash are
all the batched call shares); B = 1, InputsAndResiduals(GraphCast) in bf16x3 (autoregressive.Predictor
with gradient_checkpointing=True for T > 1).  The cotangents are random on every target variable.  In
one process, the two ways alternate: each repetition times one batched call and then the K single
calls, with CUDA events around each synchronised whole; median, min and max of --reps after one
warm-up of each.  The peak is torch.cuda.max_memory_allocated over one more call of each, the cache
emptied before each.  The card name and power limit are read in the same run, and the SM clock is
sampled every 100 ms while each case runs (bench.ClockSampler)."""
import argparse
import gc
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

from graphcast_b200 import autoregressive, graphcast, normalization, synthetic  # noqa: E402
from graphcast_b200 import xarray_shim as xs  # noqa: E402
from test_gpu_loss import _stats  # noqa: E402
from time_input_grads import _card, _peak  # noqa: E402
from bench import ClockSampler  # noqa: E402


def _cotangents(ds, rng, dirs):
  out = xs.Dataset(coords=ds.coords)
  for name, v in ds.data_vars.items():
    out[name] = xs.DataArray(rng.standard_normal((dirs,) + tuple(v.shape)).astype(np.float32),
                             ("direction",) + tuple(v.dims))
  return out


def _problem(task, resolution, mesh_size, steps):
  gc.collect()
  torch.cuda.empty_cache()
  inputs, template, forcings = synthetic.make_example(task, resolution, batch=1, num_target_steps=steps,
                                                      seed=2)
  cfg = graphcast.ModelConfig(resolution, mesh_size, 512, 16, 1, 0.6)
  params = graphcast.init_params(cfg, task, synthetic.num_input_channels(task), seed=1)
  model = graphcast.GraphCast(cfg, task, params=params)
  pred = normalization.InputsAndResiduals(model, *_stats(task, seed=1))
  if steps > 1:
    pred = autoregressive.Predictor(pred, gradient_checkpointing=True)
  pred(inputs, template, forcings)
  return model, pred, inputs, template, forcings


def _elapsed(fn):
  torch.cuda.synchronize()
  start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  fn()
  end.record()
  torch.cuda.synchronize()
  return start.elapsed_time(end) / 1e3


def _stats3(times):
  return float(np.median(times)), float(np.min(times)), float(np.max(times))


def case(pred, inputs, template, forcings, dirs, reps, label, per=None):
  rng = np.random.default_rng(3)
  cot = _cotangents(template, rng, dirs)
  singles = [cot.isel(direction=k) for k in range(dirs)]
  batched = lambda: pred.batched_input_vjp(inputs, template, forcings, cot, directions_per_pass=per)

  def single():
    for c in singles:
      pred.input_vjp(inputs, template, forcings, c)

  clocks = ClockSampler()
  clocks.start()
  times = {"batched": [], "singles": []}
  for r in range(reps + 1):
    tb, ts = _elapsed(batched), _elapsed(single)
    if r:                                    # the first of each is the warm-up
      times["batched"].append(tb)
      times["singles"].append(ts)
  peaks = {"batched": _peak(batched), "singles": _peak(single)}
  clk = clocks.stop()
  b, s = _stats3(times["batched"]), _stats3(times["singles"])
  print(f"{label}, K = {dirs}, directions_per_pass {per or dirs} (median [min, max] of {reps}): "
        f"batched_input_vjp {b[0]:.3f} s [{b[1]:.3f}, {b[2]:.3f}] (peak {peaks['batched']:.2f} GiB); "
        f"{dirs} x input_vjp {s[0]:.3f} s [{s[1]:.3f}, {s[2]:.3f}] (peak {peaks['singles']:.2f} GiB); "
        f"speed-up {s[0] / b[0]:.2f}x; per direction {b[0] / dirs:.3f} s; SM clock under load "
        f"{clk['sm_mhz']} MHz ({clk.get('samples', 0)} samples, reasons {clk['reasons']})", flush=True)
  return peaks["batched"]


def profile(pred, inputs, template, forcings, label, dirs=1):
  """Where one call's time goes: torch.profiler CUDA time per kernel (top 14) and in all, against the
  wall time of the call."""
  cot = _cotangents(template, np.random.default_rng(4), dirs)
  fn = lambda: pred.batched_input_vjp(inputs, template, forcings, cot)
  fn()
  torch.cuda.synchronize()
  acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
  with torch.profiler.profile(activities=acts) as prof:
    wall = _elapsed(fn)
  events = [e for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA]
  total = sum(e.self_device_time_total for e in events) / 1e6
  launches = sum(e.count for e in events)
  print(f"profile {label}, K = {dirs}: wall {wall:.3f} s, GPU busy {total:.3f} s ({100 * total / wall:.0f} %), "
        f"{launches} kernels and copies", flush=True)
  for e in sorted(events, key=lambda e: -e.self_device_time_total)[:14]:
    print(f"  {e.self_device_time_total / 1e6:8.4f} s {e.count:6d}x  {e.key[:100]}", flush=True)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=3)
  ap.add_argument("--skip-full", action="store_true", help="only the 1 degree cases")
  ap.add_argument("--skip-1deg", action="store_true", help="only the 0.25 degree cases")
  ap.add_argument("--profile", action="store_true", help="only the profile of one 1 degree call")
  args = ap.parse_args()
  print(f"card: {_card()}", flush=True)
  if args.profile:
    model, pred, inputs, template, forcings = _problem(graphcast.TASK_13, 1.0, 5, 1)
    for dirs in (1, 8):
      profile(pred, inputs, template, forcings, "1 deg, 13 levels, T = 1", dirs)
    return
  for steps in () if args.skip_1deg else (1, 4):
    model, pred, inputs, template, forcings = _problem(graphcast.TASK_13, 1.0, 5, steps)
    label = f"1 deg, 13 levels, T = {steps}"
    for dirs in (1, 4, 8, 16):
      case(pred, inputs, template, forcings, dirs, args.reps, label)
    del model, pred
  if args.skip_full:
    return
  for steps in (1, 2):
    model, pred, inputs, template, forcings = _problem(graphcast.TASK, 0.25, 6, steps)
    case(pred, inputs, template, forcings, 2, args.reps, f"0.25 deg, 37 levels, T = {steps}", per=1)
    del model, pred


if __name__ == "__main__":
  main()
