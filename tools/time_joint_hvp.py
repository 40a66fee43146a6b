"""Seconds per call and peak device memory of the joint Hessian-vector product (loss_and_joint_hvp)
against the two diagonal products (loss_and_param_hvp + loss_and_input_hvp) and the four gradient
calls of the central difference of the mixed blocks (loss_and_input_grads at params +- eps v_theta,
loss_and_grads at inputs +- eps v_x).

  python tools/time_joint_hvp.py [--reps 3]

Case: InputsAndResiduals(GraphCast) at 1 deg / 13 levels (TASK_13), bf16x3, B = 1, T = 1, random
tangents on every parameter, input and forcing, and random targets.  The central difference's shifted
params are loaded with set_params inside the timed call, as a user would load them.  After one warm-up
of each, the calls alternate in one process, rep by rep, so that clock drift reaches all of them alike.
Times are CUDA events around one synchronised call: median, min and max of --reps; the peak is
torch.cuda.max_memory_allocated over one more call of each.  The card name and power limit are read in
the same run, and the SM clock is sampled while the calls run (bench.ClockSampler; nvidia-smi,
read-only)."""
import argparse
import gc
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

from graphcast_b200 import graphcast, normalization, synthetic  # noqa: E402
from graphcast_b200 import xarray_shim as xs  # noqa: E402
from test_gpu_loss import _stats  # noqa: E402
from time_input_grads import _card, _peak  # noqa: E402
from time_input_jvp import _random_like  # noqa: E402
from time_param_hvp import _once  # noqa: E402
from bench import ClockSampler  # noqa: E402


def _shifted(ds, tan, eps):
  out = xs.Dataset(coords=ds.coords)
  for name, v in ds.data_vars.items():
    x = np.asarray(v.values, np.float32)
    if name in tan.data_vars:
      x = x + np.float32(eps) * np.asarray(tan.data_vars[name].transpose(*v.dims).values)
    out[name] = xs.DataArray(x, v.dims)
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=3)
  args = ap.parse_args()
  print(f"card: {_card()}", flush=True)
  task, resolution, mesh_size = graphcast.TASK_13, 1.0, 5
  inputs, template, forcings = synthetic.make_example(task, resolution, batch=1, num_target_steps=1,
                                                      seed=2)
  rng = np.random.default_rng(3)
  targets = _random_like(template, rng)
  it, ft = _random_like(inputs, rng), _random_like(forcings, rng)
  cfg = graphcast.ModelConfig(resolution, mesh_size, 512, 16, 1, 0.6)
  params = graphcast.init_params(cfg, task, synthetic.num_input_channels(task), seed=1)
  v = {n: {f: (rng.standard_normal(np.shape(a)) * (float(np.std(a)) or 0.1)).astype(np.float32)
           for f, a in fs.items()} for n, fs in params.items()}
  model = graphcast.GraphCast(cfg, task, params=params)
  pred = normalization.InputsAndResiduals(model, *_stats(task, seed=1))
  eps = 1e-2
  shifted = {s: {n: {f: a + np.float32(s * eps) * v[n][f] for f, a in fs.items()}
                 for n, fs in params.items()} for s in (1, -1)}
  plus = (_shifted(inputs, it, eps), _shifted(forcings, ft, eps))
  minus = (_shifted(inputs, it, -eps), _shifted(forcings, ft, -eps))

  def central_difference():
    for s in (1, -1):
      model.set_params(shifted[s])
      pred.loss_and_input_grads(inputs, targets, forcings)
    model.set_params(params)
    for x, f in (plus, minus):
      pred.loss_and_grads(x, targets, f)

  calls = {
      "loss_and_joint_hvp": lambda: pred.loss_and_joint_hvp(inputs, targets, forcings, v, it, ft),
      "loss_and_param_hvp + loss_and_input_hvp": lambda: (
          pred.loss_and_param_hvp(inputs, targets, forcings, v),
          pred.loss_and_input_hvp(inputs, targets, forcings, it, ft)),
      "central difference (4 gradient calls)": central_difference,
  }
  for fn in calls.values():
    fn()
  clocks = ClockSampler()
  clocks.start()
  times = {what: [] for what in calls}
  for _ in range(args.reps):
    for what, fn in calls.items():
      times[what].append(_once(fn))
  clk = clocks.stop()
  peaks = {}
  for what, fn in calls.items():
    gc.collect()
    torch.cuda.empty_cache()
    peaks[what] = _peak(fn)
  for what, ts in times.items():
    print(f"{what}: {np.median(ts):.3f} s [{min(ts):.3f}, {max(ts):.3f}] (median [min, max] of "
          f"{args.reps}), peak {peaks[what]:.1f} GiB", flush=True)
  h = np.median(times["loss_and_joint_hvp"])
  ratios = ", ".join(f"/ {what} {h / np.median(ts):.2f}" for what, ts in times.items()
                     if what != "loss_and_joint_hvp")
  print(f"loss_and_joint_hvp {ratios}; SM clock under load {clk['sm_mhz']} MHz "
        f"({clk.get('samples', 0)} samples, reasons {clk['reasons']})", flush=True)


if __name__ == "__main__":
  main()
