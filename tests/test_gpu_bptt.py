"""Backprop through time on the device: the engine's input gradient against torch autograd of the fp64
oracle, and the multi-step gradient of autoregressive.Predictor.loss_and_grads against an independent
autograd unroll of the oracle.  The feedback-seed and input-gradient kernels are checked against fp64
in test_gpu_grid_io_kernels.py."""
import gc

import numpy as np
import pytest
import torch

import _cases
from graphcast_b200 import (_native, autoregressive, casting, engine, graphcast,
                            losses, model_utils, normalization, synthetic)
from graphcast_b200 import xarray_shim as xs
from oracle import gnn as oracle_gnn
from test_gpu_grads import _GradOracle, _compare, _frob
from test_gpu_loss import _HostLoss, _lat_weight, _model_and_data, _stats

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _st():
  return torch.cuda.current_stream().cuda_stream


def _i32(a):
  return torch.as_tensor(np.asarray(a, np.int32)).to(DEV)


# ---- the engine's input gradient ---------------------------------------------------------------------
@pytest.mark.parametrize("prec,tol,c_in", [
    pytest.param("bf16x3", 1e-4, 31, id="bf16x3-0.0001"),
    pytest.param("bf16", 5e-2, 31, id="bf16-0.05"),
    # c_in_pad 304 > 256: the 512-wide transpose of the grid embedder (Backward.input_transposed)
    pytest.param("bf16x3", 1e-4, 300, id="bf16x3-0.0001-c_in300"),
])
def test_engine_input_gradient_against_fp64_autograd(prec, tol, c_in):
  g, params, x = _cases.small_case(c_in=c_in, n_out=23, msg_steps=3, batch=2, randomize_affine=True)
  n_lat = len(g.grid_lat)
  lat_w = _lat_weight(np.linspace(-90, 90, n_lat))
  rng = np.random.default_rng(7)
  targets = rng.standard_normal((g.num_grid_nodes, 2, 23)).astype(np.float32)
  coef = rng.uniform(0.5, 2.0, 23) / (23 * g.num_grid_nodes)
  eng = engine.Engine(g, params, c_in=c_in, n_out=23, msg_steps=3, precision=prec)
  eng.grads_begin()
  none = lambda n: _i32(np.full(n, -1))
  fb = engine.Feedback(_i32(np.arange(c_in)), none(23), none(c_in), none(c_in), None)
  assert eng._backward.input_transposed()[1] == (256 if eng.c_in_pad <= 256 else 512)
  w, c = torch.as_tensor(lat_w).to(DEV), torch.as_tensor(coef).to(DEV)
  sums = torch.empty(2, 23, dtype=torch.float64, device=DEV)
  got = []
  for b in range(2):
    fb.a = None
    eng.pack_inputs(torch.as_tensor(x[:, b, :].T.copy()).to(DEV))
    eng.loss_and_grads_element(torch.as_tensor(targets[:, b, :].T.copy()).to(DEV), w, c,
                               channel_sums=sums[b], feedback=fb, input_grad=True)
    got.append(fb.a.t().cpu())
  got = torch.stack(got, dim=1)                                      # [Ng, B, c_in]
  orc = _GradOracle(params, torch.float64)
  xt = torch.as_tensor(x).double().requires_grad_(True)
  y = orc.forward(g.as_dict(), xt)
  wn = torch.as_tensor(np.repeat(lat_w, g.num_grid_nodes // n_lat)).double()[:, None, None]
  d = y - torch.as_tensor(targets).double()
  (torch.as_tensor(coef) / 2 * wn * d * d).sum().backward()
  err = _frob(got, xt.grad)
  print(f"{prec}, c_in {c_in}: input gradient relative error {err:.3g}")
  assert err <= tol


# ---- backprop through time against an autograd unroll of the oracle -----------------------------------
def _data(task, batch=2, steps=3, seed=5):
  """_model_and_data for any task."""
  inputs, template, forcings = synthetic.make_example(task, 10.0, batch=batch,
                                                      num_target_steps=steps, seed=seed)
  rng = np.random.default_rng(seed)
  targets = xs.Dataset(coords=template.coords)
  for name, v in template.data_vars.items():
    targets[name] = xs.DataArray(rng.standard_normal(v.shape).astype(np.float32), v.dims)
  cfg = graphcast.ModelConfig(10.0, 2, 512, 2, 1, 0.6)
  params = oracle_gnn.init_params(c_in=synthetic.num_input_channels(task),
                                  n_out=graphcast.num_outputs(task), msg_steps=2, seed=4,
                                  randomize_affine=True)
  return graphcast.GraphCast(cfg, task, params=params), inputs, targets, forcings


def _unrolled_reference(model, inputs, targets, forcings, stats, teacher_forced=False):
  """(losses [batch], parameter gradients) of the mean over steps and batch by torch autograd of the
  fp64 oracle, unrolled here by variable name and level: normalisation, residual add, loss and the
  feeding of predictions and forcings into the next inputs (reference autoregressive.py:114-125,
  normalization.py:113-146).  teacher_forced: every step starts from detached inputs."""
  g = model._static_graph
  params = model._params
  orc = _GradOracle(params, torch.float64)
  for fields in orc.p.values():
    for t in fields.values():
      t.requires_grad_(True)
  batch, n_lat, n_lon = inputs.sizes["batch"], inputs.sizes["lat"], inputs.sizes["lon"]
  ng = n_lat * n_lon
  sizes = {"batch": batch, "lat": n_lat, "lon": n_lon}

  def field(ds, name):          # [batch, frames, levels, nodes] fp64 (levels = 1 for surface vars)
    v = ds.data_vars[name]
    p = torch.as_tensor(np.asarray(model_utils.variable_to_planes(v, sizes), np.float64))
    frames = v.sizes["time"] if "time" in v.dims else 1
    return p.reshape(batch, frames, -1, ng)

  def stat(ds, name):
    return torch.as_tensor(np.asarray(ds[name].values, np.float64)).reshape(1, 1, -1, 1)

  std, mean, dstd = stats if stats is not None else (None, None, None)
  state = {name: field(inputs, name) for name in inputs.keys()}
  time_dep = {name for name in inputs.keys() if "time" in inputs.data_vars[name].dims}
  lat_w = torch.as_tensor(np.repeat(_lat_weight(np.asarray(inputs.coords["lat"][1])), n_lon),
                          dtype=torch.float64)
  n_steps = targets.sizes["time"]
  slabs = model_utils.channel_layout(targets.isel(time=slice(0, 1)))
  kappa = torch.as_tensor(losses.channel_kappa(slabs, ng, graphcast.LOSS_PER_VARIABLE_WEIGHTS))
  total = torch.zeros(batch, dtype=torch.float64)
  for t in range(n_steps):
    f_t = forcings.isel(time=slice(t, t + 1))
    if teacher_forced:
      state = {k: v.detach() for k, v in state.items()}
    feats = []
    for src, names in ((state, sorted(inputs.keys())), (None, sorted(f_t.keys()))):
      for name in names:
        v = src[name] if src is not None else field(f_t, name)
        if stats is not None:
          v = (v - stat(mean, name)) / stat(std, name)
        feats.append(v.reshape(batch, -1, ng))
    x = torch.cat(feats, dim=1).permute(2, 0, 1)                    # [Ng, B, c_in]
    y = orc.forward(g.as_dict(), x).permute(1, 2, 0)               # [B, n_out, Ng]
    tgt = targets.isel(time=slice(t, t + 1))
    preds, loss_t = {}, torch.zeros(batch, dtype=torch.float64)
    for s in slabs:
      y_v = y[:, s.start:s.start + s.count].reshape(batch, 1, -1, ng)
      t_v = field(tgt, s.name)
      if stats is None:
        pred, t_norm = y_v, t_v
      elif s.name in state:
        last = state[s.name][:, -1:]
        pred = y_v * stat(dstd, s.name) + last
        t_norm = (t_v - last) / stat(dstd, s.name)
      else:
        pred = y_v * stat(std, s.name) + stat(mean, s.name)
        t_norm = (t_v - stat(mean, s.name)) / stat(std, s.name)
      preds[s.name] = pred
      k = kappa[s.start:s.start + s.count].reshape(1, 1, -1, 1)
      loss_t = loss_t + (k * lat_w * (y_v - t_norm) ** 2).sum(dim=(1, 2, 3))
    total = total + loss_t
    state = {name: (torch.cat([v[:, 1:], preds[name] if name in preds else field(f_t, name)], dim=1)
                    if name in time_dep else v) for name, v in state.items()}
  mean_loss = total / n_steps
  mean_loss.mean().backward()
  grads = {k: {f: t.grad for f, t in v.items()} for k, v in orc.p.items()}
  return mean_loss.detach(), grads


def _as_torch(grads):
  return {k: {f: torch.as_tensor(a) for f, a in v.items()} for k, v in grads.items()}


def _rel_all(a, b):
  num = sum(float(((a[k][f].double() - b[k][f].double()) ** 2).sum()) for k in b for f in b[k]
            if b[k][f] is not None)
  den = sum(float((b[k][f].double() ** 2).sum()) for k in b for f in b[k] if b[k][f] is not None)
  return (num / den) ** 0.5


@pytest.mark.parametrize("task_name,stack,tol", [
    ("TASK_13_PRECIP_OUT", "normalized", 1e-4),
    ("TASK_13", "normalized", 1e-4),
    ("TASK_13_PRECIP_OUT", "plain", 1e-4),
    ("TASK_13", "plain", 1e-4),
    ("TASK_13", "demo", 5e-2),
    # 37 levels: c_in_pad 480, the 512-wide input transpose and the 37-level feedback plan
    ("TASK", "normalized", 1e-4),
])
def test_bptt_against_autograd_unroll(task_name, stack, tol):
  task = getattr(graphcast, task_name)
  model, inputs, targets, forcings = _data(task)
  stats = _stats(task, seed=1) if stack != "plain" else None
  inner = model
  if stack == "demo":
    inner = casting.Bfloat16Cast(model)
  if stats is not None:
    inner = normalization.InputsAndResiduals(inner, *stats)
  ar = autoregressive.Predictor(inner, gradient_checkpointing=True)
  loss, _, grads = ar.loss_and_grads(inputs, targets, forcings)
  ref_loss, ref = _unrolled_reference(model, inputs, targets, forcings, stats)
  assert np.max(np.abs(loss.values - ref_loss.numpy()) / ref_loss.numpy()) <= max(tol, 1e-5)
  got = _as_torch(grads)
  worst = _compare(got, ref, model._params, tol)
  dead = "mesh2grid_gnn/~_networks_builder/processor_nodes_0_mesh_nodes_mlp/~/linear_0"
  assert not grads[dead]["w"].any() and not grads[dead]["b"].any()
  _, forced = _unrolled_reference(model, inputs, targets, forcings, stats, teacher_forced=True)
  sensitivity = _rel_all(forced, ref)
  print(f"{task_name} {stack}: worst per-tensor error {max(worst.values()):.3g}; teacher-forced "
        f"gradient differs by {sensitivity:.3g}")
  assert sensitivity >= 10 * tol


# ---- the public surface ------------------------------------------------------------------------------
def test_loss_and_grads_surface_and_refusals():
  task, model, inputs, targets, forcings = _model_and_data(batch=2, steps=3)
  std, mean, dstd = _stats(task, seed=1)
  ar = autoregressive.Predictor(normalization.InputsAndResiduals(model, std, mean, dstd),
                                gradient_checkpointing=True)
  loss, diag, grads = ar.loss_and_grads(inputs, targets, forcings)
  loss_ref, diag_ref = ar.loss(inputs, targets, forcings)
  assert np.array_equal(loss.values, loss_ref.values)
  assert set(diag.keys()) == set(diag_ref.keys())
  for name in diag_ref.keys():
    assert np.array_equal(diag.data_vars[name].values, diag_ref.data_vars[name].values)
  assert set(grads) == set(model._params)
  _, _, again = ar.loss_and_grads(inputs, targets, forcings)
  for name in grads:
    for f in grads[name]:
      assert grads[name][f].dtype == np.float32 and np.isfinite(grads[name][f]).all()
      assert np.array_equal(grads[name][f], again[name][f]), (name, f)
  # one target time: the inner predictor's gradient
  one = lambda ds: ds.isel(time=slice(0, 1))
  l1, _, g1 = ar.loss_and_grads(inputs, one(targets), one(forcings))
  l1_inner, _, g1_inner = ar._predictor.loss_and_grads(inputs, one(targets), one(forcings))
  assert np.array_equal(l1.values, l1_inner.values)
  for name in g1:
    for f in g1[name]:
      assert np.array_equal(g1[name][f], g1_inner[name][f])
  # refusals
  with pytest.raises(NotImplementedError, match="gradient_checkpointing=True"):
    autoregressive.Predictor(ar._predictor).loss_and_grads(inputs, targets, forcings)
  generic = autoregressive.Predictor(normalization.InputsAndResiduals(_HostLoss(model), std, mean, dstd),
                                     gradient_checkpointing=True)
  with pytest.raises(NotImplementedError):
    generic.loss_and_grads(inputs, targets, forcings)
  model.set_precision("fp32_simt")
  with pytest.raises(NotImplementedError):
    ar.loss_and_grads(inputs, targets, forcings)


# ---- larger grids: directional derivative of the device loss ----------------------------------------------
def _directional_check(task, resolution, mesh_size, steps, tol):
  gc.collect()              # earlier engines (an engine and its gradient workspace refer to each other)
  torch.cuda.empty_cache()  # at 0.25 deg the gradient peaks within a few GiB of an 80 GB card
  inputs, template, forcings = synthetic.make_example(task, resolution, batch=1,
                                                      num_target_steps=steps, seed=2)
  rng = np.random.default_rng(3)
  targets = xs.Dataset(coords=template.coords)
  for name, v in template.data_vars.items():
    targets[name] = xs.DataArray(rng.standard_normal(v.shape).astype(np.float32), v.dims)
  cfg = graphcast.ModelConfig(resolution, mesh_size, 512, 16, 1, 0.6)
  params = graphcast.init_params(cfg, task, synthetic.num_input_channels(task), seed=1)
  model = graphcast.GraphCast(cfg, task, params=params)
  std, mean, dstd = _stats(task, seed=1)
  ar = autoregressive.Predictor(normalization.InputsAndResiduals(model, std, mean, dstd),
                                gradient_checkpointing=True)
  ar.loss(inputs, targets, forcings)                      # builds the engine
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  loss, _, grads = ar.loss_and_grads(inputs, targets, forcings)
  torch.cuda.synchronize()
  peak = torch.cuda.max_memory_allocated()
  loss = float(loss.values[0])
  gnorm = np.sqrt(sum(float((a.astype(np.float64) ** 2).sum()) for v in grads.values()
                      for a in v.values()))
  eps = 1e-2 * loss / gnorm
  shifted = []
  for sign in (1.0, -1.0):
    model.set_params({k: {f: (np.asarray(a, np.float64) + sign * eps * grads[k][f] / gnorm
                              ).astype(np.float32) for f, a in v.items()} for k, v in params.items()})
    gc.collect()                              # the backward pass's cached blocks
    torch.cuda.empty_cache()
    shifted.append(float(np.asarray(ar.loss(inputs, targets, forcings)[0].values, np.float64)[0]))
  fd = (shifted[0] - shifted[1]) / (2 * eps)
  rel = abs(fd - gnorm) / gnorm
  print(f"{resolution} deg, T = {steps}: loss {loss:.6g}, |g| {gnorm:.6g}, central difference "
        f"{fd:.6g} (relative {rel:.3g}); peak device memory {peak / 2**30:.1f} GiB on "
        f"{torch.cuda.get_device_name(0)}")
  assert rel <= tol


def test_full_size_bptt_directional_derivative_and_peak_memory():
  """0.25 deg / 37 levels, two target times, on an 80 GB GPU."""
  if torch.cuda.get_device_properties(0).total_memory < 75e9:
    pytest.skip("needs an 80 GB GPU")
  _directional_check(graphcast.TASK, 0.25, 6, 2, 1e-2)
