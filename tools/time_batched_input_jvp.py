"""Seconds per call of the tangent-linear forecast of K directions at once (batched_input_jvp) against K
input_jvp calls along the same directions, their peak device memory, and a torch.profiler breakdown of
one input_jvp call.

  python tools/time_batched_input_jvp.py [--reps 3] [--skip-full | --skip-1deg] [--no-profile]

Cases: 1 deg / 13 levels (TASK_13) with K = 1, 4, 8, 16 at T = 1 and 4, and 0.25 deg / 37 levels (TASK)
with K = 1, 2 and as many directions as the measured per-direction increment leaves room for on the
card, at T = 1; B = 1, InputsAndResiduals(GraphCast) in bf16x3 (autoregressive.Predictor for T > 1).
The tangents are random on every input and forcing variable.  In one process, the two ways alternate:
each repetition times one batched call and then the K single calls, with CUDA events around each
synchronised whole; median, min and max of --reps after one warm-up of each.  The peak is
torch.cuda.max_memory_allocated over one more call of each.  The card name and power limit are read in
the same run, and the SM clock is sampled every 100 ms while each case runs (bench.ClockSampler)."""
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


def _directions(ds, rng, dirs):
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
    pred = autoregressive.Predictor(pred)
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


def case(pred, inputs, template, forcings, dirs, reps, label):
  rng = np.random.default_rng(3)
  d_in, d_f = _directions(inputs, rng, dirs), _directions(forcings, rng, dirs)
  at = lambda ds, k: ds.isel(direction=k)
  singles = [(at(d_in, k), at(d_f, k)) for k in range(dirs)]
  batched = lambda: pred.batched_input_jvp(inputs, template, forcings, d_in, d_f)

  def single():
    for a, b in singles:
      pred.input_jvp(inputs, template, forcings, a, b)

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
  print(f"{label}, K = {dirs} (median [min, max] of {reps}): batched_input_jvp {b[0]:.3f} s "
        f"[{b[1]:.3f}, {b[2]:.3f}] (peak {peaks['batched']:.2f} GiB); {dirs} x input_jvp {s[0]:.3f} s "
        f"[{s[1]:.3f}, {s[2]:.3f}] (peak {peaks['singles']:.2f} GiB); speed-up {s[0] / b[0]:.2f}x; "
        f"per direction {b[0] / dirs:.3f} s; SM clock under load {clk['sm_mhz']} MHz "
        f"({clk.get('samples', 0)} samples, reasons {clk['reasons']})", flush=True)
  return peaks["batched"]


def profile(pred, inputs, template, forcings, label, dirs=1):
  """Where one call's time goes: torch.profiler CUDA time per kernel (top 12) and in all, against the
  wall time of the call."""
  rng = np.random.default_rng(4)
  d_in, d_f = _directions(inputs, rng, dirs), _directions(forcings, rng, dirs)
  fn = lambda: pred.batched_input_jvp(inputs, template, forcings, d_in, d_f)
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
  for e in sorted(events, key=lambda e: -e.self_device_time_total)[:12]:
    print(f"  {e.self_device_time_total / 1e6:8.4f} s {e.count:6d}x  {e.key[:100]}", flush=True)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=3)
  ap.add_argument("--skip-full", action="store_true", help="only the 1 degree cases")
  ap.add_argument("--skip-1deg", action="store_true", help="only the 0.25 degree cases")
  ap.add_argument("--no-profile", action="store_true")
  args = ap.parse_args()
  print(f"card: {_card()}", flush=True)
  for steps in () if args.skip_1deg else (1, 4):
    model, pred, inputs, template, forcings = _problem(graphcast.TASK_13, 1.0, 5, steps)
    label = f"1 deg, 13 levels, T = {steps}"
    if steps == 1 and not args.no_profile:
      profile(pred, inputs, template, forcings, label, 1)
      profile(pred, inputs, template, forcings, label, 8)
    for dirs in (1, 4, 8, 16):
      case(pred, inputs, template, forcings, dirs, args.reps, label)
    del model, pred
  if args.skip_full:
    return
  model, pred, inputs, template, forcings = _problem(graphcast.TASK, 0.25, 6, 1)
  label = "0.25 deg, 37 levels, T = 1"
  if not args.no_profile:
    profile(pred, inputs, template, forcings, label, 1)
  peak = {dirs: case(pred, inputs, template, forcings, dirs, args.reps, label) for dirs in (1, 2)}
  step = peak[2] - peak[1]
  card = torch.cuda.get_device_properties(0).total_memory / 2**30
  most = 2 + int((card - 2.0 - peak[2]) // step) if step > 0 else 2
  print(f"{label}: peak {peak[1]:.2f} GiB at K = 1, {step:.2f} GiB per further direction; "
        f"{card:.1f} GiB card: at most {most} directions per pass (2 GiB left free)", flush=True)
  if most > 2:
    case(pred, inputs, template, forcings, most, max(args.reps - 1, 1), label)


if __name__ == "__main__":
  main()
