"""Seconds per call of the Hessian-vector product of the loss (loss_and_input_hvp) against
loss_and_input_grads + input_jvp (the gradient and the tangent-linear model, each on its own) and
against two loss_and_input_grads calls (the cost of a central difference), with their peak device
memory.

  python tools/time_input_hvp.py [--reps 3]

Cases: 1 deg / 13 levels (TASK_13), B = 1, InputsAndResiduals(GraphCast) in bf16x3, at T = 1 and T = 4
(autoregressive.Predictor with gradient_checkpointing=True).  The tangents are random on every input
and forcing variable.  In one process the three ways alternate: each repetition times one of each, with
CUDA events around each synchronised whole; median, min and max of --reps after one warm-up of each.
The peak is torch.cuda.max_memory_allocated over one more call of each, the cache emptied before each.
The card name and power limit are read in the same run, and the SM clock is sampled every 100 ms while
each case runs (bench.ClockSampler)."""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

from graphcast_b200 import graphcast  # noqa: E402
from graphcast_b200 import xarray_shim as xs  # noqa: E402
from time_batched_input_vjp import _elapsed, _problem, _stats3  # noqa: E402
from time_input_grads import _card, _peak  # noqa: E402
from bench import ClockSampler  # noqa: E402


def _tangents(ds, rng):
  out = xs.Dataset(coords=ds.coords)
  for name, v in ds.data_vars.items():
    out[name] = xs.DataArray(rng.standard_normal(v.shape).astype(np.float32), v.dims)
  return out


def case(steps, reps):
  model, pred, inputs, targets, forcings = _problem(graphcast.TASK_13, 1.0, 5, steps)
  rng = np.random.default_rng(3)
  it, ft = _tangents(inputs, rng), _tangents(forcings, rng)
  ways = {
      "loss_and_input_hvp": lambda: pred.loss_and_input_hvp(inputs, targets, forcings, it, ft),
      "loss_and_input_grads + input_jvp": lambda: (pred.loss_and_input_grads(inputs, targets, forcings),
                                                   pred.input_jvp(inputs, targets, forcings, it, ft)),
      "2 x loss_and_input_grads": lambda: (pred.loss_and_input_grads(inputs, targets, forcings),
                                           pred.loss_and_input_grads(inputs, targets, forcings)),
  }
  clocks = ClockSampler()
  clocks.start()
  times = {k: [] for k in ways}
  for r in range(reps + 1):
    for k, fn in ways.items():
      t = _elapsed(fn)
      if r:                                  # the first of each is the warm-up
        times[k].append(t)
  peaks = {k: _peak(fn) for k, fn in ways.items()}
  clk = clocks.stop()
  hvp = _stats3(times["loss_and_input_hvp"])[0]
  for k in ways:
    m, lo, hi = _stats3(times[k])
    print(f"1 deg / 13 levels, T = {steps}: {k} {m:.3f} s [{lo:.3f}, {hi:.3f}] (median [min, max] of "
          f"{reps}), peak {peaks[k]:.2f} GiB, {m / hvp:.2f}x the HVP call", flush=True)
  print(f"  SM clock under load {clk['sm_mhz']} MHz ({clk.get('samples', 0)} samples, reasons "
        f"{clk['reasons']})", flush=True)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=3)
  args = ap.parse_args()
  print(f"card: {_card()}", flush=True)
  for steps in (1, 4):
    case(steps, args.reps)


if __name__ == "__main__":
  main()
