"""In-process A/B of the static-edge cache (Engine.static_cache): milliseconds per device-resident step
with the cache and without it, alternated on ONE engine, with a check that both give the same bits.

  python tools/time_static_cache.py [--resolution 0.25] [--steps 10] [--rounds 3]

GraphCast with 16 message-passing steps and 37 levels (TASK), bf16x3.  Each round times --steps
steps of each arm with CUDA events after three warm-up steps of that arm (the cache is released
before the off arm and rebuilt by the first step of the on arm; the step records a CUDA graph per
state, so the warm-up also runs its capture).  Also prints the cache size, its build
time, the peak device memory of a step with and without it, and the card name and power limit read
in the same run."""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from graphcast_b200 import graphcast, synthetic  # noqa: E402


def _card():
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    q = torch.cuda.get_device_name(0)
  return q


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--resolution", type=float, default=0.25)
  ap.add_argument("--mesh-size", type=int, default=6)
  ap.add_argument("--steps", type=int, default=10)
  ap.add_argument("--rounds", type=int, default=3)
  args = ap.parse_args()
  task = graphcast.TASK
  inputs, template, forcings = synthetic.make_example(task, args.resolution, batch=1, seed=0)
  cfg = graphcast.ModelConfig(args.resolution, args.mesh_size, 512, 16, 1, 0.6)
  params = graphcast.init_params(cfg, task, synthetic.num_input_channels(task), seed=1)
  model = graphcast.GraphCast(cfg, task, params=params)
  model(inputs, template, forcings)
  eng = model.engine
  planes = model._planes_in[0]
  print(f"card: {_card()}")

  def step():
    eng.pack_inputs(planes)
    eng.step()

  def arm(on):
    eng.static_cache = on
    if not on:
      eng.release_static_cache()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    for _ in range(3):          # a new cache state is a new recorded step: run, capture, replay
      step()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    out = eng.grid_out.clone()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
      step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / args.steps, peak, out

  for r in range(args.rounds):
    ms_on, peak_on, y_on = arm(True)
    build = eng.static_cache_build_ms()
    size = sum(t.numel() * t.element_size() for t in eng._static.values())
    ms_off, peak_off, y_off = arm(False)
    same = torch.equal(y_on, y_off)
    print(f"round {r}: cache on {ms_on:.2f} ms/step, off {ms_off:.2f} ms/step ({ms_off - ms_on:+.2f}); "
          f"bitwise equal: {same}; cache {size / 2**30:.2f} GiB built in {build:.1f} ms; step peak "
          f"{peak_on / 2**30:.2f} GiB on, {peak_off / 2**30:.2f} GiB off", flush=True)
    if not same:
      sys.exit(1)


if __name__ == "__main__":
  main()
