"""Times one fine-tuning iteration two ways, on autoregressive.Predictor(InputsAndResiduals(GraphCast))
with bf16x3, batch 1, 16 message steps, best of --reps after --warmup iterations (CUDA events):

  * device: optim.AdamW.step -- the gradient (loss_and_grads with the gradient copied into the flat
    buffer), gcb_sum_squares + gcb_adamw_step (ms and algorithmic GB/s: 32 B per parameter, p, g, m, v
    read and the norm's second read of g, p, m, v written), and Engine.load_params_device (ms, its
    kernel launches counted by torch.profiler, and the bytes of the weight buffers it writes);
  * host, as INTEGRATION.md described it before the optimiser existed: loss_and_grads (the gradient
    copied to host numpy arrays), AdamW in numpy (fp32), set_params (host packing + upload); with the
    gradient's device-to-host conversion timed on its own;
  * the peak device memory of the device iteration, and the card name, power limit and clocks read in
    the same run.

Configurations: 0.25 degree / 37 levels (mesh 6) with T = 1 and T = 2 target times, 1 degree / 13
levels (mesh 5) with T = 1.  Needs a GPU; there is no CPU mode.

  python tools/time_train.py [--reps 2] [--warmup 1] [--configs 0.25:1,0.25:2,1:1]
"""
import argparse
import gc
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from graphcast_b200 import _native, autoregressive, graphcast, normalization, optim, synthetic  # noqa: E402
from graphcast_b200 import xarray_shim as xs  # noqa: E402
from time_bptt import _card, _events, _stats  # noqa: E402

CONFIGS = {"0.25": (0.25, 6, graphcast.TASK), "1": (1.0, 5, graphcast.TASK_13)}
HBM_TB_S = 3.35                      # H100 SXM peak HBM3 bandwidth


def _setup(res, mesh, task, steps):
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
  return model, ar, inputs, targets, forcings


def _device(model, ar, data, reps, warmup):
  opt = optim.AdamW(ar, learning_rate=1e-5)
  for _ in range(warmup):
    opt.step(*data)
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  step_ms = min(_events(lambda: opt.step(*data), reps))
  peak = torch.cuda.max_memory_allocated()
  lib, b, n = _native.lib(), opt._bufs, opt.layout.size
  st = lambda: torch.cuda.current_stream().cuda_stream

  def update():
    _native.check(lib.gcb_sum_squares(b["g"].data_ptr(), n, b["ws"].data_ptr(), b["ws"].numel(),
                                      b["sumsq"].data_ptr(), st()), "gcb_sum_squares")
    _native.check(lib.gcb_adamw_step(b["p"].data_ptr(), b["g"].data_ptr(), b["m"].data_ptr(),
                                     b["v"].data_ptr(), n, opt.layout.n_decay, 10, 1e-5, 0.9, 0.95,
                                     1e-8, 0.0, 0.1, b["sumsq"].data_ptr(), 32.0, st()),
                  "gcb_adamw_step")
  update()
  update_ms = min(_events(update, reps + 3))
  eng = model.engine
  reload = lambda: eng.load_params_device(opt._p_views)
  reload()
  reload_ms = min(_events(reload, reps + 3))
  with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    reload()
    torch.cuda.synchronize()
  launches = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
  written = sum(t.numel() * t.element_size() for *_, bufs, _, _ in eng._weights.values()
                for t in bufs.values())
  written += sum(t.numel() * t.element_size() for info in eng._backward._all for t in info.t.values())
  return opt, {"params": n, "step_s": step_ms / 1e3, "peak_GiB": peak / 2 ** 30,
               "grad_s": (step_ms - update_ms - reload_ms) / 1e3,
               "norm_adamw_ms": update_ms, "norm_adamw_GB_per_s": 32.0 * n / update_ms / 1e6,
               "reload_ms": reload_ms, "reload_launches": launches, "reload_bytes_written": written}


def _host(model, ar, data, reps, warmup):
  """loss_and_grads -> numpy AdamW -> set_params."""
  params = {k: {f: np.array(a, np.float32) for f, a in v.items()} for k, v in model._params.items()}
  mu = {k: {f: np.zeros_like(a) for f, a in v.items()} for k, v in params.items()}
  nu = {k: {f: np.zeros_like(a) for f, a in v.items()} for k, v in params.items()}
  lr, b1, b2, eps, wd = np.float32(1e-5), np.float32(0.9), np.float32(0.95), np.float32(1e-8), np.float32(0.1)
  count = [0]

  def adamw(grads):
    count[0] += 1
    c1, c2 = np.float32(1 - 0.9 ** count[0]), np.float32(1 - 0.95 ** count[0])
    norm = np.sqrt(sum(float(np.sum(np.square(g, dtype=np.float64))) for v in grads.values()
                       for g in v.values()))
    clip = np.float32(1.0 if norm < 32.0 else 32.0 / norm)
    for k, v in grads.items():
      for f, g in v.items():
        g = g * clip
        m, s, p = mu[k][f], nu[k][f], params[k][f]
        m *= b1
        m += (1 - b1) * g
        s *= b2
        s += (1 - b2) * g * g
        p -= lr * ((m / c1) / (np.sqrt(s / c2) + eps) + wd * p)

  rows = []
  for i in range(warmup + reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    _, _, grads = ar.loss_and_grads(*data)
    t1 = time.perf_counter()
    adamw(grads)
    t2 = time.perf_counter()
    model.set_params(params)
    torch.cuda.synchronize()
    t3 = time.perf_counter()
    rows.append((t3 - t0, t1 - t0, t2 - t1, t3 - t2))
  best = min(rows[warmup:])
  eng = model.engine
  d2h = lambda: {k: {f: t.cpu().numpy() for f, t in v.items()} for k, v in eng.grads().items()}
  d2h()
  times = []
  for _ in range(reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    d2h()
    times.append(time.perf_counter() - t0)
  return {"iteration_s": best[0], "loss_and_grads_s": best[1], "of_which_grad_d2h_s": min(times),
          "numpy_adamw_s": best[2], "set_params_s": best[3]}


def run(name, steps, reps, warmup):
  res, mesh, task = CONFIGS[name]
  model, ar, inputs, targets, forcings = _setup(res, mesh, task, steps)
  data = (inputs, targets, forcings)
  opt, dev = _device(model, ar, data, reps, warmup)
  del opt
  gc.collect()
  torch.cuda.empty_cache()
  host = _host(model, ar, data, reps, warmup)
  out = {"grid_nodes": model.engine.num_grid, "steps": steps, "device": dev, "host": host}
  del ar, model
  gc.collect()
  torch.cuda.empty_cache()
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=2)
  ap.add_argument("--warmup", type=int, default=1)
  ap.add_argument("--configs", default="0.25:1,0.25:2,1:1")
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("time_train.py needs a CUDA device")
  card = _card()
  print(f"card (name, power limit, SM clock, max SM clock): {card}")
  out = {"card": card}
  for spec in args.configs.split(","):
    name, steps = spec.split(":")
    r = run(name, int(steps), args.reps, args.warmup)
    out[spec] = r
    d, h = r["device"], r["host"]
    print(f"{name} deg, T = {steps}, {d['params']} parameters:\n"
          f"  device opt.step {d['step_s']:.3f} s = gradient {d['grad_s']:.3f} s + norm & AdamW "
          f"{d['norm_adamw_ms']:.3f} ms ({d['norm_adamw_GB_per_s']:.0f} GB/s, "
          f"{d['norm_adamw_GB_per_s'] / 1e3 / HBM_TB_S:.0%} of {HBM_TB_S} TB/s) + reload "
          f"{d['reload_ms']:.3f} ms ({d['reload_launches']} launches, "
          f"{d['reload_bytes_written'] / 1e6:.0f} MB written); peak {d['peak_GiB']:.1f} GiB\n"
          f"  host path {h['iteration_s']:.3f} s = loss_and_grads {h['loss_and_grads_s']:.3f} s (grad "
          f"D2H {h['of_which_grad_d2h_s']:.3f} s) + numpy AdamW {h['numpy_adamw_s']:.3f} s + "
          f"set_params {h['set_params_s']:.3f} s")
  print(json.dumps(out))


if __name__ == "__main__":
  main()
