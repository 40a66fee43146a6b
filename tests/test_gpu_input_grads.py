"""Gradients with respect to the inputs and forcings on the device (loss_and_input_grads, input_vjp):
every variable's gradient against torch autograd of an fp64 oracle unroll that differentiates the
inputs and forcings, the bit-identity of the parameter-free backward pass, and, at full size, variable
by variable central differences of the device loss.  The seed and broadcast-sum kernels are checked
against fp64 in test_gpu_grid_io_kernels.py."""
import gc

import numpy as np
import pytest
import torch

from graphcast_b200 import (_native, autoregressive, casting, feedback, graphcast, losses,
                            model_utils, normalization, rollout, synthetic)
from graphcast_b200 import xarray_shim as xs
from test_gpu_bptt import _data
from test_gpu_grads import _GradOracle, _frob
from test_gpu_loss import _lat_weight, _stats

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _st():
  return torch.cuda.current_stream().cuda_stream


def _i32(a):
  return torch.as_tensor(np.asarray(a, np.int32)).to(DEV)


# ---- against torch autograd of the fp64 oracle unroll --------------------------------------------------
def _planes_t(x, dims, batch, n_lat, n_lon):
  """variable_to_planes in torch, differentiable: x with `dims` -> [batch, channels, lat * lon]."""
  stack = [d for d in dims if d not in ("batch", "lat", "lon")]
  order = [d for d in ("batch",) if d in dims] + stack + [d for d in ("lat", "lon") if d in dims]
  x = x.permute([dims.index(d) for d in order])
  nch = int(np.prod([x.shape[order.index(d)] for d in stack])) if stack else 1
  shape = [batch if "batch" in dims else 1, nch, n_lat if "lat" in dims else 1,
           n_lon if "lon" in dims else 1]
  return x.reshape(shape).expand(batch, nch, n_lat, n_lon).reshape(batch, nch, n_lat * n_lon)


def _oracle(model, inputs, targets, forcings, stats, cotangents=None):
  """(per-batch losses or J, {("inputs" | "forcings", name): fp64 gradient}) by torch autograd of the
  fp64 oracle, unrolled by variable name: normalisation, residual add, loss (or J = sum cotangents *
  physical predictions) and the feeding of predictions and forcings into the next inputs."""
  g = model._static_graph
  orc = _GradOracle(model._params, torch.float64)
  batch, n_lat, n_lon = inputs.sizes["batch"], inputs.sizes["lat"], inputs.sizes["lon"]
  ng = n_lat * n_lon
  leaves = {}
  for tag, ds in (("inputs", inputs), ("forcings", forcings)):
    for name, v in ds.data_vars.items():
      leaves[(tag, name)] = torch.as_tensor(np.asarray(v.values, np.float64)).requires_grad_(True)

  def field(tag, name, t=None):        # [batch, frames, levels, nodes]
    v = (inputs if tag == "inputs" else forcings).data_vars[name]
    x, dims = leaves[(tag, name)], list(v.dims)
    if t is not None:
      x = x.narrow(dims.index("time"), t, 1)
    frames = x.shape[dims.index("time")] if "time" in dims else 1
    return _planes_t(x, dims, batch, n_lat, n_lon).reshape(batch, frames, -1, ng)

  def plain(ds, name, t):
    v = ds.isel(time=slice(t, t + 1)).data_vars[name]
    p = np.asarray(model_utils.variable_to_planes(v, {"batch": batch, "lat": n_lat, "lon": n_lon}),
                   np.float64)
    return torch.as_tensor(p).reshape(batch, 1, -1, ng)

  def stat(ds, name):
    return torch.as_tensor(np.asarray(ds[name].values, np.float64)).reshape(1, 1, -1, 1)

  std, mean, dstd = stats if stats is not None else (None, None, None)
  state = {name: field("inputs", name) for name in inputs.keys()}
  time_dep = {name for name in inputs.keys() if "time" in inputs.data_vars[name].dims}
  lat_w = torch.as_tensor(np.repeat(_lat_weight(np.asarray(inputs.coords["lat"][1])), n_lon),
                          dtype=torch.float64)
  n_steps = targets.sizes["time"]
  slabs = model_utils.channel_layout(targets.isel(time=slice(0, 1)))
  kappa = torch.as_tensor(losses.channel_kappa(slabs, ng, graphcast.LOSS_PER_VARIABLE_WEIGHTS))
  total = torch.zeros(batch, dtype=torch.float64)
  for t in range(n_steps):
    f_t = {name: field("forcings", name, t) for name in forcings.keys()}
    feats = []
    for src, names in ((state, sorted(inputs.keys())), (f_t, sorted(forcings.keys()))):
      for name in names:
        v = src[name]
        if stats is not None:
          v = (v - stat(mean, name)) / stat(std, name)
        feats.append(v.reshape(batch, -1, ng))
    x = torch.cat(feats, dim=1).permute(2, 0, 1)
    y = orc.forward(g.as_dict(), x).permute(1, 2, 0)
    preds = {}
    for s in slabs:
      y_v = y[:, s.start:s.start + s.count].reshape(batch, 1, -1, ng)
      t_v = plain(targets, s.name, t)
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
      if cotangents is None:
        k = kappa[s.start:s.start + s.count].reshape(1, 1, -1, 1)
        total = total + (k * lat_w * (y_v - t_norm) ** 2).sum(dim=(1, 2, 3)) / n_steps
      else:
        total = total + (plain(cotangents, s.name, t) * pred).sum(dim=(1, 2, 3))
    state = {name: (torch.cat([v[:, 1:], preds[name] if name in preds else f_t[name]], dim=1)
                    if name in time_dep else v) for name, v in state.items()}
  (total.mean() if cotangents is None else total.sum()).backward()
  return total.detach(), {k: v.grad for k, v in leaves.items()}


def _stack(task_name, stack, steps, seed=5):
  task = getattr(graphcast, task_name)
  model, inputs, targets, forcings = _data(task, steps=steps, seed=seed)
  stats = _stats(task, seed=1) if stack != "plain" else None
  inner = casting.Bfloat16Cast(model) if stack == "demo" else model
  if stats is not None:
    inner = normalization.InputsAndResiduals(inner, *stats)
  pred = autoregressive.Predictor(inner, gradient_checkpointing=True) if steps > 1 else inner
  return model, pred, inputs, targets, forcings, stats


def _random_cotangents(targets, seed=9):
  rng = np.random.default_rng(seed)
  out = xs.Dataset(coords=targets.coords)
  for name, v in targets.data_vars.items():
    out[name] = xs.DataArray(rng.standard_normal(v.shape).astype(np.float32), v.dims)
  return out


def _compare_vars(input_grads, forcing_grads, ref, inputs, forcings, tol, tag):
  worst = 0.0
  for key_tag, got_ds, ds in (("inputs", input_grads, inputs), ("forcings", forcing_grads, forcings)):
    assert set(got_ds.keys()) == set(ds.keys())
    for name in ds.keys():
      got, want = got_ds.data_vars[name], ds.data_vars[name]
      assert got.dims == want.dims and tuple(got.shape) == tuple(want.shape)
      assert np.asarray(got.values).dtype == np.float32
      r = ref[(key_tag, name)]
      err = _frob(torch.as_tensor(np.asarray(got.values)), r)
      worst = max(worst, err)
      assert err <= tol, (tag, key_tag, name, err)
  print(f"{tag}: worst per-variable relative error {worst:.3g}")


@pytest.mark.parametrize("task_name,stack,steps,tol", [
    ("TASK_13_PRECIP_OUT", "normalized", 3, 1e-4),
    ("TASK_13", "normalized", 3, 1e-4),
    ("TASK_13", "plain", 3, 1e-4),
    ("TASK_13", "demo", 3, 5e-2),
    ("TASK_13_PRECIP_OUT", "plain", 1, 1e-4),
    ("TASK_13", "normalized", 1, 1e-4),
    ("TASK_13", "demo", 1, 5e-2),
    # 37 levels: c_in_pad 480, the 512-wide input transpose
    ("TASK", "normalized", 3, 1e-4),
])
def test_input_grads_against_autograd_unroll(task_name, stack, steps, tol):
  model, pred, inputs, targets, forcings, stats = _stack(task_name, stack, steps)
  loss, diag, ig, fg = pred.loss_and_input_grads(inputs, targets, forcings)
  ref_loss, ref = _oracle(model, inputs, targets, forcings, stats)
  assert np.max(np.abs(loss.values - ref_loss.numpy()) / ref_loss.numpy()) <= max(tol, 1e-5)
  _compare_vars(ig, fg, ref, inputs, forcings, tol, f"{task_name} {stack} T={steps} loss")
  cot = _random_cotangents(targets)
  predictions, ig, fg = pred.input_vjp(inputs, targets, forcings, cot)
  _, ref = _oracle(model, inputs, targets, forcings, stats, cotangents=cot)
  _compare_vars(ig, fg, ref, inputs, forcings, tol, f"{task_name} {stack} T={steps} vjp")
  again = pred(inputs, targets, forcings)
  for name in again.keys():
    assert np.array_equal(np.asarray(predictions.data_vars[name].values),
                          np.asarray(again.data_vars[name].values))


def test_vjp_of_the_loss_derivative_is_the_loss_gradient():
  """Plain GraphCast over three steps: the loss depends on the inputs only through the predictions,
  so input_vjp with the cotangent dL/d(predictions) gives loss_and_input_grads."""
  model, pred, inputs, targets, forcings, _ = _stack("TASK_13", "plain", 3)
  _, _, ig, fg = pred.loss_and_input_grads(inputs, targets, forcings)
  predictions = pred(inputs, targets, forcings)
  batch, n_lat, n_lon = inputs.sizes["batch"], inputs.sizes["lat"], inputs.sizes["lon"]
  steps = targets.sizes["time"]
  slabs = model_utils.channel_layout(targets.isel(time=slice(0, 1)))
  kappa = losses.channel_kappa(slabs, n_lat * n_lon, graphcast.LOSS_PER_VARIABLE_WEIGHTS)
  w = _lat_weight(np.asarray(inputs.coords["lat"][1]))
  cot = xs.Dataset(coords=targets.coords)
  for s in slabs:
    dims = list(targets.data_vars[s.name].dims)
    p = np.asarray(predictions.data_vars[s.name].transpose(*dims).values, np.float64)
    t = np.asarray(targets.data_vars[s.name].values, np.float64)
    k_shape, w_shape = [1] * len(dims), [1] * len(dims)
    if "level" in dims:
      k_shape[dims.index("level")] = s.count
    w_shape[dims.index("lat")] = n_lat
    k = kappa[s.start:s.start + s.count].reshape(k_shape)
    cot[s.name] = xs.DataArray((2 * k * w.reshape(w_shape) * (p - t) / (batch * steps)
                                ).astype(np.float32), tuple(dims))
  _, ig2, fg2 = pred.input_vjp(inputs, targets, forcings, cot)
  for a, b in ((ig, ig2), (fg, fg2)):
    for name in a.keys():
      err = _frob(torch.as_tensor(np.asarray(b.data_vars[name].values)),
                  torch.as_tensor(np.asarray(a.data_vars[name].values)).double())
      assert err <= 1e-5, (name, err)


def test_parameter_free_rows_are_the_parameter_path_rows():
  model, pred, inputs, targets, forcings, stats = _stack("TASK_13", "normalized", 1)
  pred.loss(inputs, targets, forcings)                         # builds the engine
  eng = model.engine
  norm = pred._fused_constants(inputs, targets, forcings, DEV)
  plan = feedback.FeedbackPlan.all_channels(inputs, targets, forcings)
  eng.grads_begin()
  fb = eng.feedback(plan, norm.add_plane_index, norm.in_scale)
  planes = model._planes_in[0].clone()
  tgt = model._planes_tgt[0].clone()
  lat_w = model._lat_weight(targets, DEV)
  coef = torch.rand(eng.n_out, dtype=torch.float64, device=DEV)
  sums = torch.empty(eng.n_out, dtype=torch.float64, device=DEV)
  affine = dict(scale=norm.out_scale, offset=norm.out_offset, add_planes=planes,
                add_plane_index=norm.add_plane_index)
  rows = []
  for param in (True, False, True, False):
    fb.a = torch.randn(plan.n_rows, eng.num_grid, device=DEV, generator=torch.Generator(
        device=DEV).manual_seed(3))
    eng.pack_inputs(planes, mean=norm.in_mean, scale=norm.in_scale)
    if param:
      eng.loss_and_grads_element(tgt, lat_w, coef, channel_sums=sums, feedback=fb, input_grad=True,
                                 **affine)
    else:
      before = {k: {f: t.clone() for f, t in v.items()} for k, v in eng.grads().items()}
      eng.input_grads_element(fb, dict(affine, targets_planes=tgt), lat_weight=lat_w, coef=coef,
                              channel_sums=sums)
      after = eng.grads()
      assert all(torch.equal(before[k][f], after[k][f]) for k in before for f in before[k])
    rows.append(fb.a.clone())
  assert all(torch.equal(rows[0], r) for r in rows[1:])


def test_surface_determinism_and_no_interference():
  model, pred, inputs, targets, forcings, stats = _stack("TASK_13", "normalized", 1)
  l0, d0 = pred.loss(inputs, targets, forcings)
  g0 = pred.loss_and_grads(inputs, targets, forcings)
  loss, diag, ig, fg = pred.loss_and_input_grads(inputs, targets, forcings)
  assert np.array_equal(loss.values, l0.values)
  for name in d0.keys():
    assert np.array_equal(diag.data_vars[name].values, d0.data_vars[name].values)
  _, _, ig2, fg2 = pred.loss_and_input_grads(inputs, targets, forcings)
  for a, b in ((ig, ig2), (fg, fg2)):
    for name in a.keys():
      assert np.array_equal(a.data_vars[name].values, b.data_vars[name].values), name
  l1, _ = pred.loss(inputs, targets, forcings)
  g1 = pred.loss_and_grads(inputs, targets, forcings)
  assert np.array_equal(l0.values, l1.values)
  for k in g0[2]:
    for f in g0[2][k]:
      assert np.array_equal(g0[2][k][f], g1[2][k][f]), (k, f)
  # coords, dims and dtypes of the inputs and forcings
  for got, ds in ((ig, inputs), (fg, forcings)):
    for name in ds.keys():
      assert got.data_vars[name].dims == ds.data_vars[name].dims
  model.set_precision("fp32_simt")
  with pytest.raises(NotImplementedError, match="tensor-core precisions"):
    pred.loss_and_input_grads(inputs, targets, forcings)
  with pytest.raises(NotImplementedError, match="tensor-core precisions"):
    pred.input_vjp(inputs, targets, forcings, _random_cotangents(targets))
  model.set_precision("bf16x3")
  _, pred3, inputs3, targets3, forcings3, _ = _stack("TASK_13", "normalized", 3)
  with pytest.raises(NotImplementedError, match="gradient_checkpointing=True"):
    autoregressive.Predictor(pred3._predictor).loss_and_input_grads(inputs3, targets3, forcings3)


# ---- full size: variable by variable central differences of the device loss --------------------------------
def _full_problem(task, resolution, mesh_size, steps):
  gc.collect()
  torch.cuda.empty_cache()
  inputs, template, forcings = synthetic.make_example(task, resolution, batch=1,
                                                      num_target_steps=steps, seed=2)
  rng = np.random.default_rng(3)
  targets = xs.Dataset(coords=template.coords)
  for name, v in template.data_vars.items():
    targets[name] = xs.DataArray(rng.standard_normal(v.shape).astype(np.float32), v.dims)
  cfg = graphcast.ModelConfig(resolution, mesh_size, 512, 16, 1, 0.6)
  params = graphcast.init_params(cfg, task, synthetic.num_input_channels(task), seed=1)
  model = graphcast.GraphCast(cfg, task, params=params)
  ar = autoregressive.Predictor(normalization.InputsAndResiduals(model, *_stats(task, seed=1)),
                                gradient_checkpointing=True)
  return model, ar, inputs, targets, forcings


def _loss64(ar, inputs, targets, forcings):
  """The device loss in fp64 from the per-step channel sums (mean over steps and batch)."""
  device_step = ar._device_step()
  sums = []

  def step(rng, inputs, targets_template, forcings):
    _, predictions, s = device_step(inputs, targets_template, forcings)
    sums.append(s)
    return predictions

  for _ in rollout.chunked_prediction_generator(step, rng=None, inputs=inputs, targets_template=targets,
                                                num_steps_per_chunk=1, forcings=forcings):
    pass
  s = torch.stack(sums).cpu().numpy()                     # [steps, batch, n_out]
  slabs = model_utils.channel_layout(targets.isel(time=slice(0, 1)))
  kappa = losses.channel_kappa(slabs, inputs.sizes["lat"] * inputs.sizes["lon"],
                               graphcast.LOSS_PER_VARIABLE_WEIGHTS)
  return float((s * kappa).sum(-1).mean())


def _replace(ds, name, values):
  out = xs.Dataset(coords=ds.coords)
  for k, v in ds.data_vars.items():
    out[k] = xs.DataArray(values, v.dims) if k == name else v
  return out


def _per_variable(ar, inputs, targets, forcings, ig, fg, loss0, tag):
  worst = {}
  print(f"\n{tag}: variable, |g_v|, FD(eps) / predicted, FD(eps/2) / predicted, Richardson |error|")
  for kind, grads, ds in (("inputs", ig, inputs), ("forcings", fg, forcings)):
    for name in sorted(ds.keys()):
      g = np.asarray(grads.data_vars[name].values, np.float64)
      x = np.asarray(ds.data_vars[name].values, np.float64)
      gn = np.sqrt((g * g).sum())
      assert gn > 0, (kind, name)
      eps = 1e-3 * abs(loss0) / gn
      ratios = []
      for e in (eps, eps / 2):
        plus, minus = (x + e * g / gn).astype(np.float32), (x - e * g / gn).astype(np.float32)
        at = lambda v: _loss64(ar, *((_replace(inputs, name, v), targets, forcings) if kind == "inputs"
                                     else (inputs, targets, _replace(forcings, name, v))))
        diff = at(plus) - at(minus)
        predicted = float((g * (plus.astype(np.float64) - minus.astype(np.float64))).sum())
        ratios.append(diff / predicted)
      err = abs((4 * ratios[1] - ratios[0]) / 3 - 1)
      worst[(kind, name)] = err
      print(f"  {kind}/{name:<40s} {gn:10.3e} {ratios[0]:.8f} {ratios[1]:.8f} {err:9.3e}")
  w = max(worst.items(), key=lambda kv: kv[1])
  print(f"{tag}: worst {w[1]:.3g} at {w[0]} on {torch.cuda.get_device_name(0)}")
  for k, err in worst.items():
    assert err <= 1e-2, (k, err)


@pytest.mark.parametrize("task_name,resolution,mesh_size,steps", [
    ("TASK", 0.25, 6, 1), ("TASK_13", 1.0, 5, 4)])
def test_full_size_per_variable_central_differences(task_name, resolution, mesh_size, steps):
  if resolution < 1 and torch.cuda.get_device_properties(0).total_memory < 75e9:
    pytest.skip("needs an 80 GB GPU")
  model, ar, inputs, targets, forcings = _full_problem(getattr(graphcast, task_name), resolution,
                                                       mesh_size, steps)
  loss, _, ig, fg = ar.loss_and_input_grads(inputs, targets, forcings)
  _per_variable(ar, inputs, targets, forcings, ig, fg, float(loss.values[0]),
                f"{resolution} deg, T = {steps}")


def test_full_size_whole_vector_and_peak_memory():
  """0.25 deg / 37 levels, two target times: the peak of loss_and_input_grads does not exceed that of
  loss_and_grads for the same call."""
  if torch.cuda.get_device_properties(0).total_memory < 75e9:
    pytest.skip("needs an 80 GB GPU")
  model, ar, inputs, targets, forcings = _full_problem(graphcast.TASK, 0.25, 6, 2)
  ar.loss(inputs, targets, forcings)
  peaks = {}
  for what in ("loss_and_grads", "loss_and_input_grads"):
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    out = getattr(ar, what)(inputs, targets, forcings)
    torch.cuda.synchronize()
    peaks[what] = torch.cuda.max_memory_allocated()
  _, _, ig, fg = out
  loss0 = _loss64(ar, inputs, targets, forcings)
  keys = [("inputs", n) for n in inputs.keys()] + [("forcings", n) for n in forcings.keys()]
  get = lambda k: np.asarray((ig if k[0] == "inputs" else fg).data_vars[k[1]].values, np.float64)
  gn = np.sqrt(sum((get(k) ** 2).sum() for k in keys))
  eps = 1e-3 * loss0 / gn
  shifted = []
  for sign in (1.0, -1.0):
    new_in, new_f = inputs, forcings
    for kind, name in keys:
      src = inputs if kind == "inputs" else forcings
      v = (np.asarray(src.data_vars[name].values, np.float64) + sign * eps * get((kind, name)) / gn
           ).astype(np.float32)
      if kind == "inputs":
        new_in = _replace(new_in, name, v)
      else:
        new_f = _replace(new_f, name, v)
    shifted.append(_loss64(ar, new_in, targets, new_f))
  fd = (shifted[0] - shifted[1]) / (2 * eps)
  rel = abs(fd - gn) / gn
  print(f"0.25 deg, T = 2: |g| {gn:.6g}, central difference {fd:.6g} (relative {rel:.3g}); peak "
        f"device memory loss_and_grads {peaks['loss_and_grads'] / 2**30:.2f} GiB, "
        f"loss_and_input_grads {peaks['loss_and_input_grads'] / 2**30:.2f} GiB on "
        f"{torch.cuda.get_device_name(0)}")
  assert rel <= 1e-2
  assert peaks["loss_and_input_grads"] <= peaks["loss_and_grads"]
