"""Seconds per call of Hessian-vector products along K tangent directions at once
(batched_loss_and_input_hvp) against K loss_and_input_hvp calls with the same tangents, and their peak
device memory.

  python tools/time_batched_input_hvp.py [--reps 3] [--dirs 1 4 8 16] [--steps 1 4]

Cases: 1 deg / 13 levels (TASK_13), B = 1, InputsAndResiduals(GraphCast) in bf16x3, at T = 1 and T = 4
(autoregressive.Predictor with gradient_checkpointing=True), K = 1, 4, 8 and 16 in one pass; a K that
does not fit on the card is reported as such and the larger ones are skipped.  The tangents are random
on every input and forcing variable.  In one process the two ways alternate: each repetition times one
batched call and then the K single calls, with CUDA events around each synchronised whole; median, min
and max of --reps after one warm-up of each.  The peak is torch.cuda.max_memory_allocated over one more
call of each, the cache emptied before each.  The card name and power limit are read in the same run,
and the SM clock is sampled every 100 ms while each case runs (bench.ClockSampler)."""
import argparse
import gc
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

from graphcast_b200 import graphcast  # noqa: E402
from graphcast_b200 import xarray_shim as xs  # noqa: E402
from time_batched_input_vjp import _elapsed, _problem, _stats3  # noqa: E402
from time_input_grads import _card, _peak  # noqa: E402
from bench import ClockSampler  # noqa: E402


def _directions(ds, rng, dirs):
  out = xs.Dataset(coords=ds.coords)
  for name, v in ds.data_vars.items():
    out[name] = xs.DataArray(rng.standard_normal((dirs,) + tuple(v.shape)).astype(np.float32),
                             ("direction",) + tuple(v.dims))
  return out


def case(pred, inputs, targets, forcings, dirs, reps, label):
  rng = np.random.default_rng(3)
  it, ft = _directions(inputs, rng, dirs), _directions(forcings, rng, dirs)
  singles = [(it.isel(direction=k), ft.isel(direction=k)) for k in range(dirs)]
  batched = lambda: pred.batched_loss_and_input_hvp(inputs, targets, forcings, it, ft)

  def single():
    for a, b in singles:
      pred.loss_and_input_hvp(inputs, targets, forcings, a, b)

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
  print(f"{label}, K = {dirs} (median [min, max] of {reps}): batched_loss_and_input_hvp "
        f"{b[0]:.3f} s [{b[1]:.3f}, {b[2]:.3f}] (peak {peaks['batched']:.2f} GiB); {dirs} x "
        f"loss_and_input_hvp {s[0]:.3f} s [{s[1]:.3f}, {s[2]:.3f}] (peak {peaks['singles']:.2f} GiB); "
        f"speed-up {s[0] / b[0]:.2f}x; per direction {b[0] / dirs:.3f} s; SM clock under load "
        f"{clk['sm_mhz']} MHz ({clk.get('samples', 0)} samples, reasons {clk['reasons']})", flush=True)
  return peaks["batched"]


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=3)
  ap.add_argument("--dirs", type=int, nargs="+", default=[1, 4, 8, 16])
  ap.add_argument("--steps", type=int, nargs="+", default=[1, 4])
  args = ap.parse_args()
  print(f"card: {_card()}", flush=True)
  for steps in args.steps:
    model, pred, inputs, template, forcings = _problem(graphcast.TASK_13, 1.0, 5, steps)
    rng = np.random.default_rng(5)
    targets = xs.Dataset(coords=template.coords)
    for name, v in template.data_vars.items():
      targets[name] = xs.DataArray(rng.standard_normal(v.shape).astype(np.float32), v.dims)
    label = f"1 deg, 13 levels, T = {steps}"
    peaks = {}
    for dirs in args.dirs:
      try:
        peaks[dirs] = case(pred, inputs, targets, forcings, dirs, args.reps, label)
      except torch.cuda.OutOfMemoryError:
        print(f"{label}, K = {dirs}: does not fit on the card in one pass", flush=True)
        break
      finally:
        gc.collect()
        torch.cuda.empty_cache()
    ks = sorted(peaks)
    if len(ks) > 1:
      growth = (peaks[ks[-1]] - peaks[ks[0]]) / (ks[-1] - ks[0])
      total = torch.cuda.get_device_properties(0).total_memory / 2**30
      print(f"{label}: peak grows {growth:.2f} GiB per direction from K = {ks[0]} to {ks[-1]}; about "
            f"{int(ks[0] + (total - 2.0 - peaks[ks[0]]) / growth)} directions fit in one pass on this "
            f"{total:.0f} GiB card (2 GiB left for the allocator)", flush=True)
    del model, pred


if __name__ == "__main__":
  main()
