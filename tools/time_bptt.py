"""Times one gradient of the multi-step loss (backprop through time,
autoregressive.Predictor(InputsAndResiduals(GraphCast), gradient_checkpointing=True).loss_and_grads)
at 1 degree / 13 levels (mesh 5) with four target times and at 0.25 degree / 37 levels (mesh 6) with
two, 16 message steps, bf16x3, batch 1, best of --reps after --warmup calls (CUDA events).  Prints:

  * seconds per gradient, and its split into the forward (the rollout of `loss` plus the copies of
    every step's planes to pinned host memory) and the backward pass per step;
  * the plain multi-step `loss` for comparison, and the host-to-device upload of one step's planes;
  * the two kernels of the feedback path on the configuration's shapes: gcb_output_loss_grad_feedback
    (seed + dL/d(inputs) rows) and gcb_input_grad (accumulate), with their algorithmic HBM GB/s;
  * the peak device memory, and the card name, power limit and clocks read in the same run.

Needs a GPU; there is no CPU mode.

  python tools/time_bptt.py [--reps 2] [--warmup 1] [--configs 1,0.25]
"""
import argparse
import gc
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from graphcast_b200 import (_native, autoregressive, feedback, graphcast, normalization,  # noqa: E402
                            synthetic)
from graphcast_b200 import xarray_shim as xs  # noqa: E402

CONFIGS = {"1": (1.0, 5, graphcast.TASK_13, 4), "0.25": (0.25, 6, graphcast.TASK, 2)}


def _card():
  try:
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True,
                          check=True).stdout.strip()
  except (OSError, subprocess.CalledProcessError):
    return torch.cuda.get_device_name(0)


def _stats(task):
  rng = np.random.default_rng(0)
  levels = np.asarray(task.pressure_levels)

  def stats(lo, hi):
    ds = xs.Dataset(coords={"level": levels})
    for name in set(task.input_variables) | set(task.target_variables) | set(task.forcing_variables):
      if name in graphcast.variables.ALL_ATMOSPHERIC_VARS:
        ds[name] = xs.DataArray(rng.uniform(lo, hi, len(levels)).astype(np.float32), ("level",))
      else:
        ds[name] = xs.DataArray(np.float32(rng.uniform(lo, hi)), ())
    return ds
  return stats(0.5, 2.0), stats(-1.0, 1.0), stats(0.5, 2.0)


def _events(fn, reps):
  times = []
  for _ in range(reps):
    beg, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    beg.record()
    fn()
    end.record()
    end.synchronize()
    times.append(beg.elapsed_time(end))
  return times


def _kernels(eng, plan, n_lat, reps):
  """ms and algorithmic GB/s of the two feedback kernels on this engine's shapes."""
  lib = _native.lib()
  dev = eng.device
  ng, n_out, n_rows = eng.num_grid, eng.n_out, plan.n_rows
  gen = torch.Generator(device=dev).manual_seed(0)
  y = torch.randn(ng, 256, device=dev, generator=gen)
  tgt = torch.randn(n_out, ng, device=dev, generator=gen)
  planes = torch.randn(eng.c_in, ng, device=dev, generator=gen)
  scale = torch.rand(max(n_out, eng.c_in), device=dev, generator=gen) + 0.5
  w = torch.ones(n_lat, device=dev)
  coef = torch.full((n_out,), 1e-9, dtype=torch.float64, device=dev)
  add = plan.last_frame_channel()
  i32 = lambda a: torch.as_tensor(np.asarray(a, np.int32)).to(dev)
  add_d, dpred, resid, carry, rows = (i32(add), i32(plan.dpred_row), i32(plan.resid_channel(add)),
                                      i32(plan.carry_row), i32(plan.rows))
  a_next = torch.randn(n_rows, ng, device=dev, generator=gen)
  a_out = torch.empty(n_rows, ng, device=dev)
  g = torch.empty(ng, 256, device=dev)
  dx = torch.randn(ng, 512, device=dev, generator=gen)
  st = lambda: torch.cuda.current_stream().cuda_stream

  def seed():
    _native.check(lib.gcb_output_loss_grad_feedback(
        y.data_ptr(), 256, n_out, n_lat, ng // n_lat, scale.data_ptr(), None, planes.data_ptr(),
        add_d.data_ptr(), tgt.data_ptr(), w.data_ptr(), coef.data_ptr(), a_next.data_ptr(),
        dpred.data_ptr(), n_rows, resid.data_ptr(), carry.data_ptr(), a_out.data_ptr(), g.data_ptr(),
        256, st()), "gcb_output_loss_grad_feedback")

  def input_grad():
    _native.check(lib.gcb_input_grad(dx.data_ptr(), 512, ng, n_rows, rows.data_ptr(), scale.data_ptr(),
                                     a_out.data_ptr(), 1, st()), "gcb_input_grad")

  n_res = int((plan.resid_channel(add) >= 0).sum())
  n_fb = int((plan.dpred_row >= 0).sum())
  n_carry = int((plan.carry_row >= 0).sum())
  # seed: y, targets, add planes, fed-back rows read and g written per output channel; per row the
  # output written, y / targets / add planes / fed-back row read again for residual rows, the carry read
  seed_bytes = 4.0 * ng * (n_out * 4 + n_fb + n_rows + n_res * 4 + n_carry)
  grad_bytes = 4.0 * ng * n_rows * 3
  out = {}
  for name, fn, nbytes in (("feedback_seed", seed, seed_bytes), ("input_grad", input_grad, grad_bytes)):
    fn()
    ms = min(_events(fn, reps + 2))
    out[name] = {"ms": ms, "GB_per_s": nbytes / ms / 1e6}
  return out


def run(res, mesh, task, steps, reps, warmup):
  dev = torch.device("cuda:0")
  inputs, template, forcings = synthetic.make_example(task, res, batch=1, num_target_steps=steps,
                                                      seed=2)
  rng = np.random.default_rng(3)
  targets = xs.Dataset(coords=template.coords)
  for name, v in template.data_vars.items():
    targets[name] = xs.DataArray(rng.standard_normal(v.shape).astype(np.float32), v.dims)
  cfg = graphcast.ModelConfig(res, mesh, 512, 16, 1, 0.6)
  params = graphcast.init_params(cfg, task, synthetic.num_input_channels(task), seed=1)
  model = graphcast.GraphCast(cfg, task, params=params)
  ar = autoregressive.Predictor(normalization.InputsAndResiduals(model, *_stats(task)),
                                gradient_checkpointing=True)
  # split of loss_and_grads: an event when the backward pass starts
  marks = []
  inner = graphcast.GraphCast._bptt_grads

  def marked(self, *a, **k):
    ev = torch.cuda.Event(enable_timing=True)
    ev.record()
    marks.append(ev)
    return inner(self, *a, **k)

  graphcast.GraphCast._bptt_grads = marked
  try:
    for _ in range(warmup):
      ar.loss_and_grads(inputs, targets, forcings)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    totals, fwd = [], []
    for _ in range(reps):
      marks.clear()
      beg, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      torch.cuda.synchronize()
      beg.record()
      ar.loss_and_grads(inputs, targets, forcings)
      end.record()
      end.synchronize()
      totals.append(beg.elapsed_time(end))
      fwd.append(beg.elapsed_time(marks[0]))
    peak = torch.cuda.max_memory_allocated()
  finally:
    graphcast.GraphCast._bptt_grads = inner
  best = int(np.argmin(totals))
  loss_ms = min(_events(lambda: ar.loss(inputs, targets, forcings), reps))
  eng = model.engine
  one = torch.empty((eng.c_in + eng.n_out) * eng.num_grid, dtype=torch.float32, pin_memory=True)
  one_dev = torch.empty_like(one, device=dev)
  upload_ms = min(_events(lambda: one_dev.copy_(one, non_blocking=True), reps + 1))
  del one, one_dev
  plan = feedback.FeedbackPlan(inputs, targets.isel(time=slice(0, 1)),
                               forcings.isel(time=slice(0, 1)))
  kernels = _kernels(eng, plan, inputs.sizes["lat"], reps)
  out = {"grid_nodes": eng.num_grid, "steps": steps, "c_in": eng.c_in,
         "n_out": eng.n_out, "rows": plan.n_rows,
         "s_per_grad": totals[best] / 1e3, "runs_s": [t / 1e3 for t in totals],
         "forward_incl_host_copies_s": fwd[best] / 1e3,
         "backward_per_step_s": (totals[best] - fwd[best]) / 1e3 / steps,
         "loss_s": loss_ms / 1e3, "upload_one_step_s": upload_ms / 1e3, "peak_GiB": peak / 2 ** 30,
         "kernels": kernels}
  del ar, model, eng
  gc.collect()                  # the engine and its gradient workspace reference each other
  torch.cuda.empty_cache()
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=2)
  ap.add_argument("--warmup", type=int, default=1)
  ap.add_argument("--configs", default="1,0.25")
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("time_bptt.py needs a CUDA device")
  card = _card()
  print(f"card (name, power limit, SM clock, max SM clock): {card}")
  out = {"card": card}
  for name in args.configs.split(","):
    r = run(*CONFIGS[name], args.reps, args.warmup)
    out[name] = r
    print(f"{name} deg, T = {r['steps']}: {r['s_per_grad']:.3f} s per gradient (runs "
          + ", ".join(f"{t:.3f}" for t in r["runs_s"]) + f"); forward + host copies "
          f"{r['forward_incl_host_copies_s']:.3f} s (loss alone {r['loss_s']:.3f} s), backward "
          f"{r['backward_per_step_s']:.3f} s per step, upload of one step {r['upload_one_step_s']:.3f} s; "
          f"peak {r['peak_GiB']:.1f} GiB")
    for k, d in r["kernels"].items():
      print(f"  {k:14s} {d['ms']:8.3f} ms  {d['GB_per_s']:7.0f} GB/s")
  print(json.dumps(out))


if __name__ == "__main__":
  main()
