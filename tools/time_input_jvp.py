"""Seconds per call of the tangent-linear forecast (input_jvp) against the forecast (__call__) and the
vector-Jacobian product (input_vjp) of the same call, and their peak device memory.

  python tools/time_input_jvp.py [--reps 3] [--skip-full]

Cases: 0.25 deg / 37 levels (TASK) with B = 1 and T = 1, 2, and 1 deg / 13 levels (TASK_13) with T = 4,
all InputsAndResiduals(GraphCast) in bf16x3 (autoregressive.Predictor with gradient_checkpointing for
T > 1, which input_vjp needs and input_jvp does not use).  The tangents are random on every input and
forcing variable, the cotangents random on every prediction.  Times are CUDA events around one
synchronised call: median, min and max of --reps after one warm-up; the peak is
torch.cuda.max_memory_allocated over one more call.  The card name and power limit are read in the same
run, and the SM clock is sampled every 100 ms while each case's calls run (bench.ClockSampler: median
of the samples above idle, and the throttle reasons seen; nvidia-smi, read-only)."""
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
from time_input_grads import _card, _peak, _timed  # noqa: E402
from bench import ClockSampler  # noqa: E402


def _random_like(ds, rng):
  out = xs.Dataset(coords=ds.coords)
  for name, v in ds.data_vars.items():
    out[name] = xs.DataArray(rng.standard_normal(v.shape).astype(np.float32), v.dims)
  return out


def case(task, resolution, mesh_size, steps, reps):
  inputs, template, forcings = synthetic.make_example(task, resolution, batch=1, num_target_steps=steps,
                                                      seed=2)
  rng = np.random.default_rng(3)
  d_in, d_f, cot = _random_like(inputs, rng), _random_like(forcings, rng), _random_like(template, rng)
  cfg = graphcast.ModelConfig(resolution, mesh_size, 512, 16, 1, 0.6)
  params = graphcast.init_params(cfg, task, synthetic.num_input_channels(task), seed=1)
  model = graphcast.GraphCast(cfg, task, params=params)
  pred = normalization.InputsAndResiduals(model, *_stats(task, seed=1))
  if steps > 1:
    pred = autoregressive.Predictor(pred, gradient_checkpointing=True)
  pred(inputs, template, forcings)
  calls = {"__call__": lambda: pred(inputs, template, forcings),
           "input_jvp": lambda: pred.input_jvp(inputs, template, forcings, d_in, d_f),
           "input_vjp": lambda: pred.input_vjp(inputs, template, forcings, cot)}
  clocks = ClockSampler()
  clocks.start()
  row = {}
  for what, fn in calls.items():
    # each method starts from an empty allocator cache: at 0.25 deg input_vjp peaks within a few GiB of
    # the card, and the blocks input_jvp leaves cached are not shaped for it
    gc.collect()
    torch.cuda.empty_cache()
    row[what] = (_timed(fn, reps), _peak(fn))
  clk = clocks.stop()
  fmt = lambda r: f"{r[0][1]:.3f} s [{r[0][0]:.3f}, {r[0][2]:.3f}] (peak {r[1]:.1f} GiB)"
  print(f"{resolution} deg, {len(task.pressure_levels)} levels, T = {steps} (median [min, max] of "
        f"{reps}): " + "; ".join(f"{what} {fmt(r)}" for what, r in row.items()) +
        f"; input_jvp / __call__ {row['input_jvp'][0][1] / row['__call__'][0][1]:.2f}, "
        f"input_jvp / input_vjp {row['input_jvp'][0][1] / row['input_vjp'][0][1]:.2f}; SM clock "
        f"under load {clk['sm_mhz']} MHz ({clk.get('samples', 0)} samples, reasons {clk['reasons']})",
        flush=True)
  del model, pred, calls


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=3)
  ap.add_argument("--skip-full", action="store_true", help="only the 1 degree case")
  args = ap.parse_args()
  print(f"card: {_card()}", flush=True)
  case(graphcast.TASK_13, 1.0, 5, 4, args.reps)
  if not args.skip_full:
    case(graphcast.TASK, 0.25, 6, 1, args.reps)
    case(graphcast.TASK, 0.25, 6, 2, args.reps)


if __name__ == "__main__":
  main()
