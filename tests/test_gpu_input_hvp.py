"""Hessian-vector products of the forecast loss on the device (loss_and_input_hvp): the two coupled
backward kernels against the one-direction kernels and fp64 forward-mode autodiff; the loss and
gradients bit for bit those of loss_and_input_grads (T = 1 and 3, with noise at T = 2); H v against the
fp64 oracle (T = 1 and 3); the Gauss-Newton limit against input_jvp + input_vjp; central differences of
loss_and_input_grads at 1 degree / 13 levels (16 message-passing steps); and the exact properties
(scaling, zero tangent, symmetry, determinism, no interference)."""
import numpy as np
import pytest
import torch

from graphcast_b200 import _native, autoregressive, graphcast, losses, model_utils
from graphcast_b200 import xarray_shim as xs
from test_gpu_grads import _frob
from test_gpu_input_grads import _full_problem, _oracle, _stack

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _st():
  return torch.cuda.current_stream().cuda_stream


# ---- kernels ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [1, 77, 1003])
def test_swish_backward_jvp_kernel(rows):
  lib = _native.lib()
  gen = torch.Generator(device=DEV).manual_seed(7)
  n = 512
  stride = (rows + 127) // 128 * 128
  h = torch.randn(rows, n, generator=gen, device=DEV) * 3
  hd = torch.randn(rows, n, generator=gen, device=DEV)
  da = torch.randn(stride + rows, n, generator=gen, device=DEV)

  def run(src):
    out = torch.full_like(src, float("nan"))
    _native.check(lib.gcb_swish_backward_jvp(h.data_ptr(), n, hd.data_ptr(), n, rows, n, src.data_ptr(),
                                             n, stride, out.data_ptr(), n, _st()), "swish_backward_jvp")
    return out

  out = run(da)
  want0 = torch.empty(rows, n, device=DEV)
  _native.check(lib.gcb_swish_jvp(h.data_ptr(), n, rows, n, da.data_ptr(), n, rows, 1, want0.data_ptr(),
                                  n, _st()), "swish_jvp")
  assert torch.equal(out[:rows], want0)
  back = lambda x, d: d * torch.func.grad(lambda u: torch.nn.functional.silu(u).sum())(x)
  _, want1 = torch.func.jvp(lambda x, d: back(x, d), (h.double(), da[:rows].double()),
                            (hd.double(), da[stride:].double()))
  err = _frob(out[stride:], want1)
  print(f"gcb_swish_backward_jvp rows={rows}: direction 1 relative error {err:.3g}")
  assert err <= 1e-6
  again = run(da)                                         # deterministic (the pad rows stay unwritten)
  assert torch.equal(again[:rows], out[:rows]) and torch.equal(again[stride:], out[stride:])
  inplace = da.clone()
  _native.check(lib.gcb_swish_backward_jvp(h.data_ptr(), n, hd.data_ptr(), n, rows, n,
                                           inplace.data_ptr(), n, stride, inplace.data_ptr(), n, _st()),
                "in place")
  assert torch.equal(inplace[:rows], out[:rows]) and torch.equal(inplace[stride:], out[stride:])


@pytest.mark.parametrize("rows", [1, 77, 1003])
def test_layernorm_backward_jvp_kernel(rows):
  lib = _native.lib()
  gen = torch.Generator(device=DEV).manual_seed(11)
  n = 512
  stride = (rows + 127) // 128 * 128
  z = torch.randn(rows, n, generator=gen, device=DEV) * 2 + 0.5
  zd = torch.randn(rows, n, generator=gen, device=DEV)
  dy = torch.randn(stride + rows, n, generator=gen, device=DEV)
  scale = torch.rand(n, generator=gen, device=DEV) + 0.5

  def run():
    out = torch.full_like(dy, float("nan"))
    _native.check(lib.gcb_layernorm_backward_jvp(
        dy.data_ptr(), n, z.data_ptr(), n, zd.data_ptr(), n, scale.data_ptr(), rows, n, stride,
        out.data_ptr(), n, _st()), "layernorm_backward_jvp")
    return out

  out = run()
  want0 = torch.empty(rows, n, device=DEV)
  _native.check(lib.gcb_layernorm_backward_dirs(
      dy.data_ptr(), n, z.data_ptr(), n, scale.data_ptr(), rows, n, rows, 1, want0.data_ptr(), n, _st()),
      "layernorm_backward_dirs")
  assert torch.equal(out[:rows], want0)
  sd = scale.double()

  def back(x, g):                      # the fp64 LayerNorm backward formula
    r = torch.rsqrt(x.var(-1, unbiased=False, keepdim=True) + 1e-5)
    xh = (x - x.mean(-1, keepdim=True)) * r
    gg = g * sd
    return r * (gg - gg.mean(-1, keepdim=True) - xh * (gg * xh).mean(-1, keepdim=True))

  _, want1 = torch.func.jvp(back, (z.double(), dy[:rows].double()), (zd.double(), dy[stride:].double()))
  err = _frob(out[stride:], want1)
  print(f"gcb_layernorm_backward_jvp rows={rows}: direction 1 relative error {err:.3g}")
  assert err <= 1e-5
  again = run()                                           # deterministic (the pad rows stay unwritten)
  assert torch.equal(again[:rows], out[:rows]) and torch.equal(again[stride:], out[stride:])


# ---- the model ---------------------------------------------------------------------------------------
def _random(ds, seed, names=None):
  rng = np.random.default_rng(seed)
  out = xs.Dataset(coords=ds.coords)
  for name, v in ds.data_vars.items():
    if names is None or name in names:
      out[name] = xs.DataArray(rng.standard_normal(v.shape).astype(np.float32), v.dims)
  return out


def _vals(ds):
  return {k: np.asarray(v.values) for k, v in ds.data_vars.items()}


def _same(a, b):
  va, vb = _vals(a), _vals(b)
  assert set(va) == set(vb)
  for k in va:
    assert np.array_equal(va[k], vb[k]), k


def _shifted(ds, tan, eps):
  out = xs.Dataset(coords=ds.coords)
  for name, v in ds.data_vars.items():
    x = np.asarray(v.values, np.float64)
    if tan is not None and name in tan.data_vars:
      x = x + eps * np.asarray(tan.data_vars[name].transpose(*v.dims).values, np.float64)
    out[name] = xs.DataArray(x, v.dims)
  return out


def _oracle_hvp(model, inputs, forcings, targets, stats, it, ft, eps=1e-4):
  """H v of the fp64 oracle: the central difference, in fp64, of its autograd gradients along v
  (truncation O(eps^2), rounding about 1e-16 / eps)."""
  _, gp = _oracle(model, _shifted(inputs, it, eps), targets, _shifted(forcings, ft, eps), stats)
  _, gm = _oracle(model, _shifted(inputs, it, -eps), targets, _shifted(forcings, ft, -eps), stats)
  return {k: (gp[k] - gm[k]) / (2 * eps) for k in gp}


@pytest.mark.parametrize("task_name,stack", [
    ("TASK_13", "plain"), ("TASK_13", "normalized"), ("TASK_13", "demo"), ("TASK", "normalized"),
])
@pytest.mark.parametrize("with_forcings", [False, True])
@pytest.mark.parametrize("steps", [1, 3])
def test_loss_and_gradients_bit_for_bit(task_name, stack, with_forcings, steps):
  model, pred, inputs, targets, forcings, _ = _stack(task_name, stack, steps)
  it = _random(inputs, 3)
  ft = _random(forcings, 4) if with_forcings else None
  loss, diag, ig, fg, ih, fh = pred.loss_and_input_hvp(inputs, targets, forcings, it, ft)
  loss0, diag0, ig0, fg0 = pred.loss_and_input_grads(inputs, targets, forcings)
  assert np.array_equal(np.asarray(loss.values), np.asarray(loss0.values))
  _same(diag, diag0)
  _same(ig, ig0)
  _same(fg, fg0)
  for got, like in ((ih, inputs), (fh, forcings)):
    for name, v in like.data_vars.items():
      g = got.data_vars[name]
      assert g.dims == v.dims and tuple(g.shape) == tuple(v.shape)
      assert np.asarray(g.values).dtype == np.float32 and np.all(np.isfinite(np.asarray(g.values)))
  loss1 = pred.loss(inputs, targets, forcings)[0]
  assert np.array_equal(np.asarray(loss.values), np.asarray(loss1.values))


def test_loss_and_gradients_bit_for_bit_with_noise():
  _, pred, inputs, targets, forcings, _ = _stack("TASK_13", "normalized", 2)
  noisy = autoregressive.Predictor(pred._predictor, noise_level=0.1, gradient_checkpointing=True)
  it, ft = _random(inputs, 15), _random(forcings, 16)
  loss, diag, ig, fg, ih, fh = noisy.loss_and_input_hvp(inputs, targets, forcings, it, ft, rng=7)
  loss0, diag0, ig0, fg0 = noisy.loss_and_input_grads(inputs, targets, forcings, rng=7)
  assert np.array_equal(np.asarray(loss.values), np.asarray(loss0.values))
  _same(diag, diag0)
  _same(ig, ig0)
  _same(fg, fg0)
  for ds in (ih, fh):
    for k, v in _vals(ds).items():
      assert np.all(np.isfinite(v)), k


@pytest.mark.parametrize("task_name,stack,steps,tol", [
    ("TASK_13", "plain", 1, 1e-4), ("TASK_13", "normalized", 1, 1e-4),
    ("TASK_13_PRECIP_OUT", "normalized", 1, 1e-4), ("TASK_13", "plain", 3, 1e-4),
    ("TASK_13", "normalized", 3, 1e-4),
])
def test_hvp_against_fp64_oracle(task_name, stack, steps, tol):
  model, pred, inputs, targets, forcings, stats = _stack(task_name, stack, steps)
  it, ft = _random(inputs, 5), _random(forcings, 6)
  _, _, _, _, ih, fh = pred.loss_and_input_hvp(inputs, targets, forcings, it, ft)
  ref = _oracle_hvp(model, inputs, forcings, targets, stats, it, ft)
  worst = 0.0
  for tag, got_ds, ds in (("inputs", ih, inputs), ("forcings", fh, forcings)):
    for name in ds.keys():
      err = _frob(torch.as_tensor(np.asarray(got_ds.data_vars[name].values)), ref[(tag, name)])
      worst = max(worst, err)
      assert err <= tol, (tag, name, err)
  print(f"{task_name} {stack} T={steps}: worst per-variable relative error of H v {worst:.3g} on "
        f"{torch.cuda.get_device_name(0)}")


def test_exact_properties_and_no_interference():
  model, pred, inputs, targets, forcings, _ = _stack("TASK_13", "normalized", 1)
  it, ft = _random(inputs, 8), _random(forcings, 9)
  before_g = pred.loss_and_input_grads(inputs, targets, forcings)
  before_j = pred.input_jvp(inputs, targets, forcings, it, ft)
  out = pred.loss_and_input_hvp(inputs, targets, forcings, it, ft)
  again = pred.loss_and_input_hvp(inputs, targets, forcings, it, ft)
  for a, b in zip(out[2:], again[2:]):                     # deterministic
    _same(a, b)
  after_g = pred.loss_and_input_grads(inputs, targets, forcings)
  after_j = pred.input_jvp(inputs, targets, forcings, it, ft)
  for a, b in zip(before_g[2:], after_g[2:]):
    _same(a, b)
  for a, b in zip(before_j, after_j):
    _same(a, b)
  # a power-of-two scaling of v scales H v exactly
  def scale(ds, c):
    out = xs.Dataset(coords=ds.coords)
    for k, v in ds.data_vars.items():
      out[k] = xs.DataArray(np.asarray(v.values) * np.float32(c), v.dims)
    return out

  scaled = pred.loss_and_input_hvp(inputs, targets, forcings, scale(it, 4.0), scale(ft, 4.0))
  for a, b in zip(out[4:], scaled[4:]):
    va, vb = _vals(a), _vals(b)
    for k in va:
      assert np.array_equal(va[k] * np.float32(4.0), vb[k]), k
  # a zero tangent gives exact zeros
  zero = pred.loss_and_input_hvp(inputs, targets, forcings, scale(it, 0.0), None)
  for ds in zero[4:]:
    for k, v in _vals(ds).items():
      assert not np.any(v), k
  # symmetry: <w, H v> = <v, H w>
  wi, wf = _random(inputs, 21), _random(forcings, 22)
  hw = pred.loss_and_input_hvp(inputs, targets, forcings, wi, wf)

  def dot(a_in, a_f, b_in, b_f):
    s = 0.0
    for a, b in ((a_in, b_in), (a_f, b_f)):
      for k, v in a.data_vars.items():
        s += float(np.sum(np.asarray(v.values, np.float64) *
                          np.asarray(b.data_vars[k].transpose(*v.dims).values, np.float64)))
    return s

  lhs, rhs = dot(wi, wf, out[4], out[5]), dot(it, ft, hw[4], hw[5])
  print(f"<w, Hv> = {lhs:.9g}, <v, Hw> = {rhs:.9g}")
  assert abs(lhs - rhs) <= 1e-4 * max(abs(lhs), abs(rhs))


# ---- the Gauss-Newton limit ------------------------------------------------------------------------
@pytest.mark.parametrize("steps", [1, 3])
def test_gauss_newton_limit(steps):
  """With the targets set to the predictions of __call__ (plain GraphCast: prediction = decoder output,
  so every residual is exactly zero) H v is J^T W J v: input_vjp with the cotangent
  coef * w_lat * (J v), coef = 2 kappa / (batch * steps), J v from input_jvp."""
  model, pred, inputs, targets, forcings, _ = _stack("TASK_13", "plain", steps)
  preds = pred(inputs, targets, forcings)
  it, ft = _random(inputs, 13), _random(forcings, 14)
  _, _, _, _, ih, fh = pred.loss_and_input_hvp(inputs, preds, forcings, it, ft)
  _, pdot = pred.input_jvp(inputs, preds, forcings, it, ft)
  one = preds.isel(time=slice(0, 1))
  n_lat, n_lon, batch = inputs.sizes["lat"], inputs.sizes["lon"], inputs.sizes["batch"]
  kappa = losses.channel_kappa(model_utils.channel_layout(one), n_lat * n_lon,
                               graphcast.LOSS_PER_VARIABLE_WEIGHTS)
  w_lat = np.asarray(model._lat_weight(one, "cpu").numpy(), np.float64)
  cot = xs.Dataset(coords=preds.coords)
  for s in model_utils.channel_layout(one):
    v = pdot.data_vars[s.name]
    rest = [d for d in v.dims if d not in ("batch", "time", "lat", "lon")]
    x = np.asarray(v.transpose("batch", "time", *rest, "lat", "lon").values, np.float64)
    k = kappa[s.start:s.start + s.count].reshape((1, 1) + tuple(x.shape[2:-2]) + (1, 1))
    c = 2.0 * k / (batch * steps) * w_lat.reshape(n_lat, 1) * x
    cot[s.name] = xs.DataArray(c.astype(np.float32), ("batch", "time", *rest, "lat", "lon"))
  _, ig, fg = pred.input_vjp(inputs, preds, forcings, cot)
  worst = 0.0
  for got_ds, want_ds in ((ih, ig), (fh, fg)):
    for name in want_ds.keys():
      want = torch.as_tensor(np.asarray(want_ds.data_vars[name].values, np.float64))
      err = _frob(torch.as_tensor(np.asarray(got_ds.data_vars[name].values)), want)
      worst = max(worst, err)
      assert err <= 1e-4, (name, err)
  print(f"Gauss-Newton limit T={steps}: worst per-variable relative difference {worst:.3g}")


# ---- central differences at 1 degree / 13 levels ------------------------------------------------------
def test_central_differences_at_one_degree():
  """H v against (g(x + eps v) - g(x - eps v)) / (2 eps) of loss_and_input_grads, variable by variable,
  at 1 degree / 13 levels with 16 message-passing steps (every tangent edge snapshot of the processor
  is read), v scaled per variable by its spread and eps = 1e-3."""
  model, ar, inputs, targets, forcings = _full_problem(graphcast.TASK_13, 1.0, 5, 1)
  pred = ar._predictor
  rng = np.random.default_rng(17)

  def tangents(ds):
    out = xs.Dataset(coords=ds.coords)
    for name, v in ds.data_vars.items():
      x = np.asarray(v.values, np.float64)
      out[name] = xs.DataArray((rng.standard_normal(x.shape) * (x.std() or 1.0)).astype(np.float32),
                               v.dims)
    return out

  it, ft = tangents(inputs), tangents(forcings)
  _, _, _, _, ih, fh = pred.loss_and_input_hvp(inputs, targets, forcings, it, ft)
  eps = 1e-3
  _, _, gp_i, gp_f = pred.loss_and_input_grads(_as_f32(_shifted(inputs, it, eps)), targets,
                                               _as_f32(_shifted(forcings, ft, eps)))
  _, _, gm_i, gm_f = pred.loss_and_input_grads(_as_f32(_shifted(inputs, it, -eps)), targets,
                                               _as_f32(_shifted(forcings, ft, -eps)))
  worst = {}
  for got_ds, p_ds, m_ds in ((ih, gp_i, gm_i), (fh, gp_f, gm_f)):
    for name in got_ds.keys():
      fd = (np.asarray(p_ds.data_vars[name].values, np.float64) -
            np.asarray(m_ds.data_vars[name].values, np.float64)) / (2 * eps)
      got = np.asarray(got_ds.data_vars[name].values, np.float64)
      worst[name] = _frob(torch.as_tensor(got), torch.as_tensor(fd))
  w = max(worst.items(), key=lambda kv: kv[1])
  print(f"1 deg / 13 levels central differences: worst per-variable relative difference {w[1]:.3g} "
        f"at {w[0]} on {torch.cuda.get_device_name(0)}")
  for name, err in worst.items():
    assert err <= 2e-2, (name, err)


def _as_f32(ds):
  out = xs.Dataset(coords=ds.coords)
  for name, v in ds.data_vars.items():
    out[name] = xs.DataArray(np.asarray(v.values, np.float32), v.dims)
  return out
