"""Times one parameter gradient of the one-step loss (Engine.grads_begin + loss_and_grads_element,
what GraphCast.loss_and_grads runs per batch element) at 0.25 degree / 37 levels (mesh 6) and at
1 degree / 13 levels (mesh 5), 16 message steps, bf16x3, after warm-up calls.  Prints the wall time
per gradient (CUDA events), the per-kernel-kind breakdown of one gradient from gcb_profile_begin/end
(ms, executed TFLOP/s for the tensor-core kinds), the peak device memory, and the card name and
power limit read in the same run.  Needs a GPU; there is no CPU mode.

  python tools/time_grads.py [--reps 3] [--warmup 1] [--configs 0.25,1]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from graphcast_b200 import _native, engine, graph as graph_lib, graphcast, synthetic  # noqa: E402

KINDS = {0: "layer_tc", 1: "segment_sum", 2: "pack", 3: "unpack", 4: "layer_simt", 5: "rows_to_image",
         6: "chain_tc", 7: "gather", 8: "loss", 9: "weight_grad", 10: "rowwise_bwd"}
CONFIGS = {"0.25": (0.25, 6, graphcast.TASK), "1": (1.0, 5, graphcast.TASK_13)}


def _card():
  try:
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True,
                          check=True).stdout.strip()
  except (OSError, subprocess.CalledProcessError):
    return torch.cuda.get_device_name(0)


def run(res, mesh, task, reps, warmup):
  dev = torch.device("cuda:0")
  lat, lon = synthetic.grid_coords(res)
  g = graph_lib.cached_static_graph(grid_lat=lat, grid_lon=lon, mesh_size=mesh,
                                    radius_query_fraction_edge_length=0.6)
  c_in, n_out = synthetic.num_input_channels(task), graphcast.num_outputs(task)
  params = graphcast.init_params(graphcast.ModelConfig(res, mesh, 512, 16, 1, 0.6), task, c_in, seed=1)
  eng = engine.Engine(g, params, c_in=c_in, n_out=n_out, msg_steps=16, precision="bf16x3")
  gen = torch.Generator(device=dev).manual_seed(0)
  planes = torch.randn(c_in, g.num_grid_nodes, device=dev, generator=gen)
  targets = torch.randn(n_out, g.num_grid_nodes, device=dev, generator=gen)
  lat_w = torch.rand(len(lat), device=dev, generator=gen) + 0.5
  coef = torch.full((n_out,), 2.0 / (n_out * g.num_grid_nodes), dtype=torch.float64, device=dev)
  sums = torch.empty(n_out, dtype=torch.float64, device=dev)

  def grad():
    eng.grads_begin()
    eng.pack_inputs(planes)
    eng.loss_and_grads_element(targets, lat_w, coef, channel_sums=sums)

  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  for _ in range(warmup):
    grad()
  times = []
  for _ in range(reps):
    beg, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    beg.record()
    grad()
    end.record()
    end.synchronize()
    times.append(beg.elapsed_time(end))
  peak = torch.cuda.max_memory_allocated()
  lib = _native.lib()
  cap = 1 << 16
  kinds = (C.c_int32 * cap)()
  ms = (C.c_float * cap)()
  flops, nbytes = (C.c_double * cap)(), (C.c_double * cap)()
  count = C.c_int32(0)
  _native.check(lib.gcb_profile_begin(), "gcb_profile_begin")
  grad()
  torch.cuda.synchronize()
  _native.check(lib.gcb_profile_end(cap, kinds, ms, flops, nbytes, C.byref(count)), "gcb_profile_end")
  per = {}
  for i in range(min(count.value, cap)):
    k = KINDS.get(kinds[i], str(kinds[i]))
    d = per.setdefault(k, {"launches": 0, "ms": 0.0, "tflop": 0.0, "gb": 0.0})
    d["launches"] += 1
    d["ms"] += ms[i]
    d["tflop"] += flops[i] / 1e12
    d["gb"] += nbytes[i] / 1e9
  del eng
  torch.cuda.empty_cache()
  return {"grid": [len(lat), len(lon)], "mesh": mesh, "n_out": n_out, "ms_per_grad": min(times),
          "runs_ms": times, "peak_GiB": peak / 2 ** 30, "profiled_launches": count.value,
          "breakdown": per}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=3)
  ap.add_argument("--warmup", type=int, default=1)
  ap.add_argument("--configs", default="0.25,1")
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("time_grads.py needs a CUDA device")
  card = _card()
  print(f"card: {card}")
  out = {"card": card}
  for name in args.configs.split(","):
    r = run(*CONFIGS[name], args.reps, args.warmup)
    out[name] = r
    print(f"{name} deg: {r['ms_per_grad']:.1f} ms per gradient (runs "
          + ", ".join(f"{t:.1f}" for t in r["runs_ms"]) + f"), peak {r['peak_GiB']:.1f} GiB")
    for k, d in sorted(r["breakdown"].items(), key=lambda kv: -kv[1]["ms"]):
      rate = f"{d['tflop'] / d['ms'] * 1e3:7.1f} TFLOP/s" if d["tflop"] else " " * 15
      print(f"  {k:13s} {d['launches']:5d} launches {d['ms']:9.2f} ms {rate} {d['gb']:8.1f} GB")
  print(json.dumps(out))


if __name__ == "__main__":
  main()
