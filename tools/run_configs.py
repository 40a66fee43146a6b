"""Measures the BASELINE.json configs beyond the headline bench (run on an H100):
rollout (config 3), operational 13-level batch-of-4 (config 5), bf16 mode, 1-degree small."""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from graphcast_b200 import graphcast, rollout, synthetic

dev = torch.device("cuda:0")
out = {}

def model_for(task, res, mesh, precision="bf16x3"):
  cfg = graphcast.ModelConfig(res, mesh, 512, 16, 1, 0.6)
  params = graphcast.init_params(cfg, task, synthetic.num_input_channels(task), seed=1)
  return graphcast.GraphCast(cfg, task, params=params, precision=precision, device=dev)

def time_steps(fn, n, warm=2):
  for _ in range(warm): fn()
  torch.cuda.synchronize(); e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
  e0.record()
  for _ in range(n): fn()
  e1.record(); torch.cuda.synchronize()
  return e0.elapsed_time(e1) / n

# config 3: 40-step autoregressive rollout at 0.25 deg, device-resident state, predictions to host
task = graphcast.TASK
inputs, template, forcings = synthetic.make_example(task, 0.25, num_target_steps=40, seed=0, pinned=True)
m = model_for(task, 0.25, 6)
fn = lambda rng, inputs, targets_template, forcings: m(inputs, targets_template, forcings)
first = next(iter(rollout.chunked_prediction_generator(fn, None, inputs, rollout.extend_targets_template(template, 1), 1, forcings.isel(time=slice(0, 1)))))
torch.cuda.synchronize()
t0 = time.perf_counter()
n = 0
for chunk in rollout.chunked_prediction_generator(fn, None, inputs, template, 1, forcings):
  n += 1
  del chunk
torch.cuda.synchronize()
dt = time.perf_counter() - t0
out["config3_rollout_40_steps"] = {"steps": n, "seconds_per_10_day_forecast": dt, "steps_per_s": n / dt,
                                   "note": "chunked_prediction_generator, device-resident state, forcings H2D per step"}
# same rollout with the forcings generated on the device (TISR kernel + progress features): no forcing upload
t_dt = (np.datetime64("2021-03-17T06:00:00") + np.asarray(template.coords["time"][1])).astype("datetime64[ns]")[None, :]
template_dt = template.assign_coords(datetime=(("batch", "time"), t_dt))
gen = list(task.forcing_variables)
next(iter(rollout.chunked_prediction_generator(fn, None, inputs, rollout.extend_targets_template(template_dt, 1), 1, None, generate_forcings=gen)))
torch.cuda.synchronize()
t0 = time.perf_counter()
n = 0
for chunk in rollout.chunked_prediction_generator(fn, None, inputs, template_dt, 1, None, generate_forcings=gen):
  n += 1
  del chunk
torch.cuda.synchronize()
dt = time.perf_counter() - t0
out["config3_rollout_40_steps_device_forcings"] = {
    "steps": n, "seconds_per_10_day_forecast": dt, "steps_per_s": n / dt,
    "note": "forcings generated per step on the device (gcb_toa_incident_solar_radiation + progress features)"}
# bf16 mode at config 2
planes = m._planes_in[0]
eng = m.engine
po = torch.empty([eng.n_out, eng.num_grid], device=dev)
def step():
  eng.pack_inputs(planes); eng.step(); eng.unpack_outputs(po)
for prec in ("bf16x3", "bf16"):
  eng.set_precision(prec)
  out[f"config2_{prec}_ms_per_step"] = time_steps(step, 5)
eng.set_precision("bf16x3")
del m, eng, planes, po, inputs, template, forcings
torch.cuda.empty_cache()

# config 5: operational 13 levels, batch of 4 members on one GPU (the N-GPU run = 1 member per GPU)
task = graphcast.TASK_13_PRECIP_OUT
inputs, template, forcings = synthetic.make_example(task, 0.25, batch=4, seed=0, pinned=True)
m = model_for(task, 0.25, 6)
call = lambda: m(inputs, template, forcings)
ms = time_steps(call, 3, warm=1)
out["config5_operational_13lvl_batch4_1gpu"] = {"ms_per_call": ms, "member_steps_per_s": 4e3 / ms,
                                                "note": "GraphCast.__call__ incl. H2D of inputs, batch=4"}
del m, inputs, template, forcings
torch.cuda.empty_cache()

# config 1 on the GPU: GraphCast_small 1 deg
task = graphcast.TASK_13
inputs, template, forcings = synthetic.make_example(task, 1.0, seed=0, pinned=True)
m = model_for(task, 1.0, 5)
call = lambda: m(inputs, template, forcings)
out["config1_small_1deg_gpu_ms_per_call"] = time_steps(call, 10)
print(json.dumps(out, indent=1))
