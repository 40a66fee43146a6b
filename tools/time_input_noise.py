"""Times the input noise of the multi-step training loss at GraphCast 0.25 degree / 37 levels (TASK, B = 1):

  noise pass       one gcb_add_gaussian_noise launch over every time-dependent input (the 2 input frames
                   of the 6 surface and 6 x 37 level variables, the solar radiation and the progress
                   features: about 1.9 GB read and 1.9 GB written), CUDA events over --reps launches after
                   --warmup; the rate is the algorithmic HBM traffic over the time, against the H100 SXM
                   data-sheet 3.35 TB/s
  loss_and_grads   autoregressive.Predictor(InputsAndResiduals(GraphCast), gradient_checkpointing=True)
                   at T = 2, without and with noise_level, alternated; min / median / max of --grad-reps
                   synchronised calls after one warm-up each, and the peak device memory of each

The card, its power limit and SM clock limit are printed next to the numbers.  Needs a GPU.

  python tools/time_input_noise.py [--reps 50] [--warmup 5] [--grad-reps 3] [--skip-grads]
"""
import argparse
import gc
import os
import subprocess
import sys
import zlib

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

from graphcast_b200 import _native, autoregressive, graphcast, normalization, synthetic  # noqa: E402
from graphcast_b200 import xarray_shim as xs  # noqa: E402
from test_gpu_loss import _stats  # noqa: E402

DEV = torch.device("cuda:0")
PEAK_BW = 3.35e12


def _card():
  try:
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                           "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                          timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    return torch.cuda.get_device_name(0) + ", power limit not read"


def noise_pass(inputs, targets, forcings, reps, warmup):
  plan = autoregressive.noise_plan(inputs, targets, forcings)
  srcs = [torch.as_tensor(np.ascontiguousarray(inputs.data_vars[n].values, np.float32)).to(DEV)
          for n, _ in plan]
  dsts = [torch.empty_like(s) for s in srcs]
  table = (_native.NoiseSegment * len(plan))()
  for entry, src, dst, (_, stream) in zip(table, srcs, dsts, plan):
    entry.src, entry.dst, entry.n, entry.offset, entry.stream = (src.data_ptr(), dst.data_ptr(),
                                                                 dst.numel(), 0, stream)
  lib = _native.lib()
  st = torch.cuda.current_stream().cuda_stream
  run = lambda: _native.check(lib.gcb_add_gaussian_noise(table, len(plan), 7, 0, 0.1, st), "noise")
  elems = sum(s.numel() for s in srcs)
  nbytes = 8.0 * elems
  runs = []
  for _ in range(3):
    for _ in range(warmup):
      run()
    beg, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    beg.record()
    for _ in range(reps):
      run()
    end.record()
    end.synchronize()
    runs.append(beg.elapsed_time(end) / reps)
  ms = min(runs)
  print(f"noise pass: {len(plan)} variables, {elems / 1e6:.1f} M elements, {nbytes / 1e9:.2f} GB moved: "
        f"{ms:.3f} ms, {nbytes / ms / 1e6:.0f} GB/s = {100 * nbytes / ms / 1e-3 / PEAK_BW:.1f} % of "
        f"3.35 TB/s (runs: {', '.join(f'{r:.3f}' for r in runs)} ms)", flush=True)
  # the same launch without the load (src = NULL): how much of the time the generator itself takes
  for entry in table:
    entry.src = None
  torch.cuda.synchronize()
  beg, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  beg.record()
  for _ in range(reps):
    run()
  end.record()
  end.synchronize()
  ms0 = beg.elapsed_time(end) / reps
  print(f"noise alone (src = NULL, {nbytes / 2e9:.2f} GB written): {ms0:.3f} ms, "
        f"{nbytes / 2 / ms0 / 1e6:.0f} GB/s", flush=True)
  del srcs, dsts


def _peak(fn):
  gc.collect()
  torch.cuda.empty_cache()
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  fn()
  torch.cuda.synchronize()
  return torch.cuda.max_memory_allocated() / 2**30


def grads(inputs, targets, forcings, reps):
  task = graphcast.TASK
  cfg = graphcast.ModelConfig(0.25, 6, 512, 16, 1, 0.6)
  params = graphcast.init_params(cfg, task, synthetic.num_input_channels(task), seed=1)
  model = graphcast.GraphCast(cfg, task, params=params)
  inner = normalization.InputsAndResiduals(model, *_stats(task, seed=1))
  preds = {"noiseless": (autoregressive.Predictor(inner, gradient_checkpointing=True), {}),
           "noisy": (autoregressive.Predictor(inner, noise_level=0.1, gradient_checkpointing=True),
                     {"rng": 7})}
  times = {k: [] for k in preds}
  for name, (p, kw) in preds.items():                   # warm-up
    p.loss_and_grads(inputs, targets, forcings, **kw)
  for _ in range(reps):                                 # alternated
    for name, (p, kw) in preds.items():
      torch.cuda.synchronize()
      beg, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      beg.record()
      p.loss_and_grads(inputs, targets, forcings, **kw)
      end.record()
      torch.cuda.synchronize()
      times[name].append(beg.elapsed_time(end) / 1e3)
  peaks = {name: _peak(lambda: p.loss_and_grads(inputs, targets, forcings, **kw))
           for name, (p, kw) in preds.items()}
  for name in preds:
    t = times[name]
    print(f"loss_and_grads 0.25 deg / 37 levels, T = 2, {name}: median {np.median(t):.3f} s "
          f"[{min(t):.3f}, {max(t):.3f}] over {reps}; peak {peaks[name]:.2f} GiB", flush=True)
  print(f"ratio of medians noisy / noiseless: {np.median(times['noisy']) / np.median(times['noiseless']):.4f}",
        flush=True)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=50)
  ap.add_argument("--warmup", type=int, default=5)
  ap.add_argument("--grad-reps", type=int, default=3)
  ap.add_argument("--skip-grads", action="store_true")
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("time_input_noise.py needs a CUDA device")
  print(f"card: {_card()}", flush=True)
  inputs, template, forcings = synthetic.make_example(graphcast.TASK, 0.25, batch=1, num_target_steps=2,
                                                      seed=2)
  noise_pass(inputs, template, forcings, args.reps, args.warmup)
  if not args.skip_grads:
    rng = np.random.default_rng(3)
    targets = xs.Dataset(coords=template.coords)
    for name, v in template.data_vars.items():
      targets[name] = xs.DataArray(rng.standard_normal(v.shape).astype(np.float32), v.dims)
    grads(inputs, targets, forcings, args.grad_reps)


if __name__ == "__main__":
  main()
