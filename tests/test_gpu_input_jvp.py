"""The tangent-linear forecast on the device (input_jvp): the LayerNorm tangent kernel against fp64
torch and against the LayerNorm backward, every prediction tangent against forward-mode autodiff of
an fp64 oracle unroll, the adjoint identity with input_vjp, the exact properties (predictions of
__call__, linearity under exact scalings, determinism, no interference), and, at full size, central
differences and the memory plan."""
import gc

import numpy as np
import pytest
import torch
import torch.autograd.forward_ad as fwAD

from graphcast_b200 import _native, graphcast, model_utils
from graphcast_b200 import xarray_shim as xs
from test_gpu_grads import _GradOracle, _frob
from test_gpu_input_grads import _full_problem, _planes_t, _random_cotangents, _replace, _stack

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _st():
  return torch.cuda.current_stream().cuda_stream


# ---- kernel ------------------------------------------------------------------------------------------
def test_layernorm_jvp_kernel_against_fp64_and_the_backward():
  lib = _native.lib()
  gen = torch.Generator(device=DEV).manual_seed(31)
  rows, n = 1003, 512                                   # ragged: not a multiple of the 8-row block
  z = torch.randn(rows, n, generator=gen, device=DEV) * 2 + 0.5
  dz = torch.randn(rows, n, generator=gen, device=DEV)
  scale = torch.rand(n, generator=gen, device=DEV) + 0.5
  res = torch.randn(rows, n, generator=gen, device=DEV)

  def run(residual):
    out = torch.full((rows, n), float("nan"), device=DEV)
    _native.check(lib.gcb_layernorm_jvp(
        z.data_ptr(), n, dz.data_ptr(), n, scale.data_ptr(), rows, n,
        None if residual is None else residual.data_ptr(), n, out.data_ptr(), n, _st()), "jvp")
    return out

  zd, dzd, sd = z.double(), dz.double(), scale.double()
  ln = lambda x: (x - x.mean(-1, keepdim=True)) * torch.rsqrt(x.var(-1, unbiased=False, keepdim=True)
                                                              + 1e-5) * sd
  _, want = torch.func.jvp(ln, (zd,), (dzd,))           # forward-mode autodiff, fp64
  for residual in (None, res):
    out = run(residual)
    ref = want if residual is None else want + residual.double()
    err = _frob(out, ref)
    print(f"gcb_layernorm_jvp (residual: {residual is not None}): relative error {err:.3g}")
    assert err <= 1e-6
    assert torch.equal(run(residual), out)              # deterministic
  # the Jacobian is symmetric: the backward with unit scale applied to dz, times the scale
  ws = torch.empty(lib.gcb_rowwise_workspace_bytes(n), dtype=torch.uint8, device=DEV)
  sums = [torch.empty(n, device=DEV) for _ in range(3)]
  back = torch.empty(rows, n, device=DEV)
  ones = torch.ones(n, device=DEV)
  _native.check(lib.gcb_layernorm_backward(
      dz.data_ptr(), n, z.data_ptr(), n, ones.data_ptr(), rows, n, back.data_ptr(), n, ws.data_ptr(),
      ws.numel(), *(s.data_ptr() for s in sums), 0, _st()), "backward")
  diff = float((run(None) - back * scale).abs().max() / (back * scale).abs().max())
  print(f"gcb_layernorm_jvp against scale * gcb_layernorm_backward(unit scale): {diff:.3g}")
  assert diff <= 1e-6


# ---- against forward-mode autodiff of the fp64 oracle unroll -------------------------------------------
def _host(ds):
  """A Dataset with numpy data (the device results moved to the host)."""
  out = xs.Dataset(coords=ds.coords)
  for name, v in ds.data_vars.items():
    out[name] = xs.DataArray(np.asarray(v.values), v.dims)
  return out


def _oracle_jvp(model, inputs, targets, forcings, stats, d_in, d_f):
  """{name: [batch, steps, channels, nodes] fp64 prediction tangents} by forward-mode autodiff
  (torch.autograd.forward_ad) of the fp64 oracle, unrolled by variable name as
  test_gpu_input_grads._oracle unrolls it: normalisation, residual add and the feeding of predictions
  and forcings into the next inputs.  Variables absent from d_in / d_f have zero tangents."""
  g = model._static_graph
  orc = _GradOracle(model._params, torch.float64)
  batch, n_lat, n_lon = inputs.sizes["batch"], inputs.sizes["lat"], inputs.sizes["lon"]
  ng = n_lat * n_lon
  slabs = model_utils.channel_layout(targets.isel(time=slice(0, 1)))

  def stat(ds, name):
    return torch.as_tensor(np.asarray(ds[name].values, np.float64)).reshape(1, 1, -1, 1)

  std, mean, dstd = stats if stats is not None else (None, None, None)
  out = {s.name: [] for s in slabs}
  with fwAD.dual_level():
    leaves = {}
    for tag, ds, tan in (("inputs", inputs, d_in), ("forcings", forcings, d_f)):
      for name, v in ds.data_vars.items():
        x = torch.as_tensor(np.asarray(v.values, np.float64))
        t = torch.zeros_like(x)
        if tan is not None and name in tan.data_vars:
          t = torch.as_tensor(np.asarray(tan.data_vars[name].transpose(*v.dims).values, np.float64))
        leaves[(tag, name)] = fwAD.make_dual(x, t)

    def field(tag, name, t=None):        # [batch, frames, levels, nodes]
      v = (inputs if tag == "inputs" else forcings).data_vars[name]
      x, dims = leaves[(tag, name)], list(v.dims)
      if t is not None:
        x = x.narrow(dims.index("time"), t, 1)
      frames = x.shape[dims.index("time")] if "time" in dims else 1
      return _planes_t(x, dims, batch, n_lat, n_lon).reshape(batch, frames, -1, ng)

    state = {name: field("inputs", name) for name in inputs.keys()}
    time_dep = {name for name in inputs.keys() if "time" in inputs.data_vars[name].dims}
    for t in range(targets.sizes["time"]):
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
        if stats is None:
          pred = y_v
        elif s.name in state:
          pred = y_v * stat(dstd, s.name) + state[s.name][:, -1:]
        else:
          pred = y_v * stat(std, s.name) + stat(mean, s.name)
        preds[s.name] = pred
        out[s.name].append(fwAD.unpack_dual(pred).tangent.detach().clone())
      state = {name: (torch.cat([v[:, 1:], preds[name] if name in preds else f_t[name]], dim=1)
                      if name in time_dep else v) for name, v in state.items()}
  return {name: torch.cat(ts, dim=1) for name, ts in out.items()}


def _device_planes(ds, name, steps, batch, n_lat, n_lon):
  """[batch, steps, channels, nodes] of a device result variable, packed as the oracle's."""
  sizes = {"batch": batch, "lat": n_lat, "lon": n_lon}
  host = _host(ds)
  per = [np.asarray(model_utils.variable_to_planes(host.isel(time=slice(t, t + 1)).data_vars[name],
                                                   sizes), np.float64).reshape(batch, 1, -1, n_lat * n_lon)
         for t in range(steps)]
  return torch.as_tensor(np.concatenate(per, axis=1))


def _random_tangents(ds, rng, names=None):
  out = xs.Dataset(coords=ds.coords)
  for name, v in ds.data_vars.items():
    if names is None or name in names:
      out[name] = xs.DataArray(rng.standard_normal(v.shape).astype(np.float32), v.dims)
  return out


@pytest.mark.parametrize("task_name,stack,steps,which,tol", [
    ("TASK_13_PRECIP_OUT", "normalized", 3, "all", 1e-4),
    ("TASK_13", "normalized", 3, "all", 1e-4),
    ("TASK_13", "normalized", 3, "single", 1e-4),
    ("TASK_13", "plain", 3, "all", 1e-4),
    ("TASK_13", "demo", 3, "all", 5e-2),
    ("TASK_13_PRECIP_OUT", "plain", 1, "all", 1e-4),
    ("TASK_13", "normalized", 1, "all", 1e-4),
    ("TASK_13", "plain", 1, "single", 1e-4),
    ("TASK_13", "demo", 1, "all", 5e-2),
    ("TASK", "normalized", 3, "all", 1e-4),             # 37 levels: c_in_pad 480
    ("TASK", "normalized", 1, "single", 1e-4),
])
def test_prediction_tangents_against_forward_mode_unroll(task_name, stack, steps, which, tol):
  model, pred, inputs, targets, forcings, stats = _stack(task_name, stack, steps)
  rng = np.random.default_rng(11)
  if which == "all":
    d_in, d_f = _random_tangents(inputs, rng), _random_tangents(forcings, rng)
  else:                                                 # one input variable alone, forcings fixed
    d_in, d_f = _random_tangents(inputs, rng, names=["temperature"]), None
  predictions, tangents = pred.input_jvp(inputs, targets, forcings, d_in, d_f)
  ref = _oracle_jvp(model, inputs, targets, forcings, stats, d_in, d_f)
  batch, n_lat, n_lon = inputs.sizes["batch"], inputs.sizes["lat"], inputs.sizes["lon"]
  worst = 0.0
  assert set(tangents.keys()) == set(targets.keys())
  for name in targets.keys():
    got_v = tangents.data_vars[name]
    assert got_v.dims == predictions.data_vars[name].dims
    assert tuple(got_v.shape) == tuple(predictions.data_vars[name].shape)
    assert np.asarray(got_v.values).dtype == np.float32
    err = _frob(_device_planes(tangents, name, steps, batch, n_lat, n_lon), ref[name])
    worst = max(worst, err)
    assert err <= tol, (name, err)
  print(f"{task_name} {stack} T={steps} {which}: worst per-variable relative error {worst:.3g}")
  again = pred(inputs, targets, forcings)
  for name in again.keys():
    assert np.array_equal(np.asarray(predictions.data_vars[name].values),
                          np.asarray(again.data_vars[name].values))


# ---- the adjoint identity with input_vjp -----------------------------------------------------------------
def _dot(a, b):
  return sum(float((np.asarray(a.data_vars[k].values, np.float64) *
                    np.asarray(b.data_vars[k].transpose(*a.data_vars[k].dims).values, np.float64)).sum())
             for k in a.keys())


def _adjoint_gap(pred, inputs, targets, forcings, seed=12):
  rng = np.random.default_rng(seed)
  d_in, d_f = _random_tangents(inputs, rng), _random_tangents(forcings, rng)
  w = _random_cotangents(targets, seed=seed + 1)
  _, tangents = pred.input_jvp(inputs, targets, forcings, d_in, d_f)
  _, ig, fg = pred.input_vjp(inputs, targets, forcings, w)
  lhs = _dot(w, tangents)
  rhs = _dot(d_in, ig) + _dot(d_f, fg)
  return lhs, rhs, abs(lhs - rhs) / max(abs(lhs), abs(rhs))


@pytest.mark.parametrize("task_name,stack,steps", [
    ("TASK_13", "normalized", 1), ("TASK_13", "normalized", 3), ("TASK_13_PRECIP_OUT", "plain", 3)])
def test_adjoint_identity_with_input_vjp(task_name, stack, steps):
  _, pred, inputs, targets, forcings, _ = _stack(task_name, stack, steps)
  lhs, rhs, rel = _adjoint_gap(pred, inputs, targets, forcings)
  print(f"{task_name} {stack} T={steps}: <w, J v> {lhs:.10g}, <J^T w, v> {rhs:.10g}, relative {rel:.3g}")
  assert rel <= 1e-4


# ---- exact properties ------------------------------------------------------------------------------------
def _values(ds):
  return {k: np.asarray(v.values) for k, v in ds.data_vars.items()}


def _scaled(ds, c):
  out = xs.Dataset(coords=ds.coords)
  for k, v in ds.data_vars.items():
    out[k] = xs.DataArray((np.asarray(v.values) * np.float32(c)).astype(np.float32), v.dims)
  return out


@pytest.mark.parametrize("steps", [1, 3])
def test_exact_properties(steps):
  model, pred, inputs, targets, forcings, _ = _stack("TASK_13", "normalized", steps)
  rng = np.random.default_rng(13)
  d_in, d_f = _random_tangents(inputs, rng), _random_tangents(forcings, rng)
  call = _values(pred(inputs, targets, forcings))
  predictions, base = pred.input_jvp(inputs, targets, forcings, d_in, d_f)
  base = _values(base)
  assert all(np.array_equal(a, call[k]) for k, a in _values(predictions).items())
  # zero tangents (no variables, forcings held fixed) give exactly zero
  _, zero = pred.input_jvp(inputs, targets, forcings, xs.Dataset(coords=inputs.coords))
  assert all(not np.any(a) for a in _values(zero).values())
  # power-of-two scalings and the sign are exact; two calls agree bit for bit
  for c in (-1.0, 2.0, 0.25):
    _, t = pred.input_jvp(inputs, targets, forcings, _scaled(d_in, c), _scaled(d_f, c))
    for k, a in _values(t).items():
      assert np.array_equal(a, (base[k] * np.float32(c)).astype(np.float32)), (c, k)
  _, again = pred.input_jvp(inputs, targets, forcings, d_in, d_f)
  assert all(np.array_equal(a, base[k]) for k, a in _values(again).items())


def test_no_interference_with_the_gradients():
  model, pred, inputs, targets, forcings, _ = _stack("TASK_13", "normalized", 1)
  rng = np.random.default_rng(14)
  d_in, d_f = _random_tangents(inputs, rng), _random_tangents(forcings, rng)
  w = _random_cotangents(targets)
  g0 = pred.loss_and_grads(inputs, targets, forcings)[2]
  v0 = pred.input_vjp(inputs, targets, forcings, w)
  pred.input_jvp(inputs, targets, forcings, d_in, d_f)
  g1 = pred.loss_and_grads(inputs, targets, forcings)[2]
  v1 = pred.input_vjp(inputs, targets, forcings, w)
  for k in g0:
    for f in g0[k]:
      assert np.array_equal(g0[k][f], g1[k][f]), (k, f)
  for a, b in zip(v0, v1):
    for k in a.keys():
      assert np.array_equal(np.asarray(a.data_vars[k].values), np.asarray(b.data_vars[k].values)), k
  # the refusals of input_vjp
  model.set_precision("fp32_simt")
  with pytest.raises(NotImplementedError, match="tensor-core precisions"):
    pred.input_jvp(inputs, targets, forcings, d_in)
  model.set_precision("bf16x3")


# ---- full size -------------------------------------------------------------------------------------------
def _scaled_tangents(ds, rng):
  """A random tangent of every variable, on the scale of the variable's own spread."""
  out = xs.Dataset(coords=ds.coords)
  for name, v in ds.data_vars.items():
    x = np.asarray(v.values, np.float64)
    out[name] = xs.DataArray((rng.standard_normal(x.shape) * (x.std() + 1e-3 * np.abs(x).mean() + 1e-12)
                              ).astype(np.float32), v.dims)
  return out


def _shift(ds, d, e):
  out = ds
  for name in d.keys():
    v = np.asarray(ds.data_vars[name].values, np.float64) + e * np.asarray(
        d.data_vars[name].transpose(*ds.data_vars[name].dims).values, np.float64)
    out = _replace(out, name, v.astype(np.float32))
  return out


@pytest.mark.parametrize("task_name,resolution,mesh_size,steps", [
    ("TASK", 0.25, 6, 1), ("TASK_13", 1.0, 5, 2)])
def test_full_size_per_variable_central_differences(task_name, resolution, mesh_size, steps):
  """F_var = sum w_var * P_var (fp64 from the fp32 predictions) at x +- eps v for two step sizes, with
  Richardson extrapolation, against sum w_var * Pdot_var, variable by variable.  w_var is the device's
  own tangent Pdot_var, a fixed weight: sum w Pdot = |Pdot|^2 has no cancellation, and a tangent wrong
  in size or direction moves the difference quotient away from it (it tends to <Pdot, P'>).  With
  random weights the sum cancels down to the rounding noise of the predictions' differences."""
  if resolution < 1 and torch.cuda.get_device_properties(0).total_memory < 75e9:
    pytest.skip("needs an 80 GB GPU")
  model, ar, inputs, targets, forcings = _full_problem(getattr(graphcast, task_name), resolution,
                                                       mesh_size, steps)
  rng = np.random.default_rng(15)
  d_in, d_f = _scaled_tangents(inputs, rng), _scaled_tangents(forcings, rng)
  _, tangents = ar.input_jvp(inputs, targets, forcings, d_in, d_f)
  w = {k: np.asarray(v.values, np.float64) for k, v in tangents.data_vars.items()}
  predicted = {k: float((w[k] * w[k]).sum()) for k in w}
  del tangents

  def f(e):
    p = ar(_shift(inputs, d_in, e), targets, _shift(forcings, d_f, e))
    return {k: float((w[k] * np.asarray(v.values, np.float64)).sum()) for k, v in p.data_vars.items()}

  eps = 2e-2
  fd = []
  for e in (eps, eps / 2):
    plus, minus = f(e), f(-e)
    fd.append({k: (plus[k] - minus[k]) / (2 * e) for k in plus})
  worst = {}
  print(f"\n{resolution} deg, T = {steps}: variable, sum w Pdot, Richardson FD, relative error")
  for k in sorted(predicted):
    rich = (4 * fd[1][k] - fd[0][k]) / 3
    worst[k] = abs(rich - predicted[k]) / abs(predicted[k])
    print(f"  {k:<40s} {predicted[k]:14.6e} {rich:14.6e} {worst[k]:9.3e}")
  name = max(worst, key=worst.get)
  print(f"{resolution} deg, T = {steps}: worst {worst[name]:.3g} at {name} on "
        f"{torch.cuda.get_device_name(0)}")
  for k, err in worst.items():
    assert err <= 1e-2, (k, err)


def _peak(fn):
  gc.collect()
  torch.cuda.empty_cache()
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  out = fn()
  torch.cuda.synchronize()
  return torch.cuda.max_memory_allocated(), out


def _result_bytes(*datasets):
  """Device bytes of the returned Datasets (the predictions and tangents of every step)."""
  return sum(v.data.numel() * v.data.element_size() for ds in datasets for v in ds.data_vars.values()
             if isinstance(v.data, torch.Tensor) and v.data.is_cuda)


def test_full_size_peak_memory_and_the_adjoint_identity():
  """0.25 deg / 37 levels, one target time: the peak of input_jvp stays at or below that of input_vjp
  in the same process, and <w, J v> = <J^T w, v>.  1 deg / 13 levels: the working memory of input_jvp
  (the peak less the returned Datasets, which hold every step) does not grow from T = 2 to T = 4 by one
  step's input planes."""
  if torch.cuda.get_device_properties(0).total_memory < 75e9:
    pytest.skip("needs an 80 GB GPU")
  model, ar, inputs, targets, forcings = _full_problem(graphcast.TASK, 0.25, 6, 1)
  ar(inputs, targets, forcings)                           # builds the engine
  rng = np.random.default_rng(17)
  d_in, d_f = _random_tangents(inputs, rng), _random_tangents(forcings, rng)
  w = _random_cotangents(targets, seed=18)
  peak_vjp, (_, ig, fg) = _peak(lambda: ar.input_vjp(inputs, targets, forcings, w))
  peak_jvp, (_, tangents) = _peak(lambda: ar.input_jvp(inputs, targets, forcings, d_in, d_f))
  lhs, rhs = _dot(w, tangents), _dot(d_in, ig) + _dot(d_f, fg)
  rel = abs(lhs - rhs) / max(abs(lhs), abs(rhs))
  print(f"0.25 deg, T = 1: <w, J v> {lhs:.10g}, <J^T w, v> {rhs:.10g}, relative {rel:.3g}; peak "
        f"input_vjp {peak_vjp / 2**30:.2f} GiB, input_jvp {peak_jvp / 2**30:.2f} GiB on "
        f"{torch.cuda.get_device_name(0)}")
  assert rel <= 1e-3
  assert peak_jvp <= peak_vjp
  del model, ar, ig, fg, tangents
  working = {}
  for steps in (2, 4):
    model, ar, inputs, targets, forcings = _full_problem(graphcast.TASK_13, 1.0, 5, steps)
    ar(inputs, targets, forcings)
    rng = np.random.default_rng(19)
    d_in, d_f = _random_tangents(inputs, rng), _random_tangents(forcings, rng)
    peak, out = _peak(lambda: ar.input_jvp(inputs, targets, forcings, d_in, d_f))
    working[steps] = peak - _result_bytes(*out)
    one_step = model.engine.c_in * model.engine.num_grid * 4
    del out, model, ar
  print(f"1 deg, T = 2 / 4: input_jvp peak less its results {working[2] / 2**20:.1f} / "
        f"{working[4] / 2**20:.1f} MiB (one step's input planes {one_step / 2**20:.1f} MiB)")
  assert abs(working[4] - working[2]) < one_step
