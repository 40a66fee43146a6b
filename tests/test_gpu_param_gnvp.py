"""Gauss-Newton products of the forecast loss with respect to the parameters on the device
(loss_and_param_gnvp): G v against the fp64 oracle
(forward-mode J v, then reverse mode through the loss Hessian), the exact identities (symmetry, the
quadratic form, linearity, zero tangents, the loss of loss()), and the full-Hessian limit where the
predictions equal the targets."""
import numpy as np
import pytest
import torch
import torch.autograd.forward_ad as fwAD

from graphcast_b200 import _native, graphcast, losses, model_utils
from graphcast_b200 import xarray_shim as xs
from test_gpu_grads import _GradOracle, _frob
from test_gpu_input_grads import _full_problem, _planes_t, _stack
from test_gpu_input_jvp import _host
from test_gpu_param_jvp import M2G_MESH, _host_loss, _pair, _random_param_tangents, _shift, _values

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _st():
  return torch.cuda.current_stream().cuda_stream


# ---- against the fp64 oracle -----------------------------------------------------------------------------
def _features(inputs, forcings, stats):
  """[Ng, batch, c_in] fp64 features of one step, normalised by `stats` (None: plain)."""
  batch, n_lat, n_lon = inputs.sizes["batch"], inputs.sizes["lat"], inputs.sizes["lon"]
  ng = n_lat * n_lon
  std, mean = (None, None) if stats is None else stats[:2]
  feats = []
  for ds in (inputs, forcings.isel(time=slice(0, 1))):
    for name in sorted(ds.keys()):
      v = ds.data_vars[name]
      dims = list(v.dims)
      frames = v.shape[dims.index("time")] if "time" in dims else 1
      x = _planes_t(torch.as_tensor(np.asarray(v.values, np.float64)), dims, batch, n_lat,
                    n_lon).reshape(batch, frames, -1, ng)
      if stats is not None:
        x = (x - torch.as_tensor(np.asarray(mean[name].values, np.float64)).reshape(1, 1, -1, 1)) \
            / torch.as_tensor(np.asarray(std[name].values, np.float64)).reshape(1, 1, -1, 1)
      feats.append(x.reshape(batch, -1, ng))
  return torch.cat(feats, dim=1).permute(2, 0, 1)


def _oracle_gnvp(model, inputs, targets, forcings, stats, v):
  """J^T H J v of the fp64 oracle: J v by forward mode, then reverse mode of <H J v, y>, H = coef w."""
  g = model._static_graph.as_dict()
  x = _features(inputs, forcings, stats)
  batch, n_lat, n_lon = inputs.sizes["batch"], inputs.sizes["lat"], inputs.sizes["lon"]
  slabs = model_utils.channel_layout(targets)
  coef = 2.0 * losses.channel_kappa(slabs, n_lat * n_lon, graphcast.LOSS_PER_VARIABLE_WEIGHTS) / batch
  w = losses.normalized_latitude_weights(targets[sorted(targets.keys())[0]])
  h = torch.as_tensor(np.repeat(np.asarray(w, np.float64), n_lon))[:, None, None] * \
      torch.as_tensor(np.asarray(coef, np.float64))[None, None, :]
  orc = _GradOracle(model._params, torch.float64)
  with fwAD.dual_level():
    for name, fields in v.items():
      for f, t in fields.items():
        orc.p[name][f] = fwAD.make_dual(orc.p[name][f], torch.as_tensor(np.asarray(t, np.float64)))
    ydot = fwAD.unpack_dual(orc.forward(g, x)).tangent.detach().clone()
  orc = _GradOracle(model._params, torch.float64)
  for fields in orc.p.values():
    for t in fields.values():
      t.requires_grad_(True)
  (orc.forward(g, x) * (h * ydot)).sum().backward()
  return {k: {f: (t.grad if t.grad is not None else torch.zeros_like(t)) for f, t in fs.items()}
          for k, fs in orc.p.items()}


@pytest.mark.parametrize("task_name,stack,tol", [
    ("TASK_13", "plain", 1e-4), ("TASK_13", "normalized", 1e-4), ("TASK_13", "demo", 5e-2),
    ("TASK", "normalized", 1e-4)])
def test_gnvp_against_the_fp64_oracle(task_name, stack, tol):
  """Tolerances as for loss_and_grads: the tangent and the backward pass are each within about 1e-5
  of fp64 in bf16x3 (relative to the norm), within 2^-8-driven 5e-2 in bf16; compared tensor by
  tensor relative to each tensor's norm."""
  model, pred, inputs, targets, forcings, stats = _stack(task_name, stack, 1)
  v = _random_param_tangents(model._params, np.random.default_rng(3))
  _, _, gnvp = pred.loss_and_param_gnvp(inputs, targets, forcings, v)
  ref = _oracle_gnvp(model, inputs, targets, forcings, stats, v)
  worst = 0.0
  assert set(gnvp) == set(model._params)
  for name, fields in model._params.items():
    assert set(gnvp[name]) == set(fields)
    for f, a in fields.items():
      got = gnvp[name][f]
      assert got.dtype == np.float32 and got.shape == np.shape(a)
      if name.startswith(M2G_MESH + "_"):
        assert not got.any()                            # the step never reads it: exact zeros
        continue
      err = _frob(torch.as_tensor(got), ref[name][f])
      worst = max(worst, err)
      assert err <= tol, (name, f, err)
  print(f"{task_name} {stack}: worst tensor relative error {worst:.3g}")


# ---- exact identities -------------------------------------------------------------------------------------
def _dot(a, b):
  return sum(float(np.sum(np.asarray(a[n][f], np.float64) * np.asarray(b[n][f], np.float64)))
             for n in a for f in a[n])


@pytest.mark.parametrize("stack", ["plain", "normalized"])
def test_exact_identities(stack):
  model, pred, inputs, targets, forcings, _ = _stack("TASK_13", stack, 1)
  params = model._params
  rng = np.random.default_rng(12)
  u, v = _random_param_tangents(params, rng), _random_param_tangents(params, rng)
  loss0, diag0 = pred.loss(inputs, targets, forcings)
  loss, diag, gv = pred.loss_and_param_gnvp(inputs, targets, forcings, v)
  assert np.array_equal(np.asarray(loss.values), np.asarray(loss0.values))
  for name in diag0.keys():
    assert np.array_equal(np.asarray(diag.data_vars[name].values), np.asarray(diag0.data_vars[name].values))
  _, _, gu = pred.loss_and_param_gnvp(inputs, targets, forcings, u)
  # symmetry: G u and G v are each within 1e-4 of exact relative to their norms (the oracle test), so
  # by Cauchy-Schwarz the two products differ by at most 1e-4 (|v| |Gu| + |u| |Gv|)
  a, b = _dot(gu, v), _dot(gv, u)
  bound = 1e-4 * (_dot(v, v) ** 0.5 * _dot(gu, gu) ** 0.5 + _dot(u, u) ** 0.5 * _dot(gv, gv) ** 0.5)
  print(f"{stack}: <u, Gv> {b:.8g}, <v, Gu> {a:.8g}, difference / bound {abs(a - b) / bound:.3g}")
  assert abs(a - b) <= bound
  # linearity under an exact scaling, determinism
  v2 = {n: {f: 2 * x for f, x in fs.items()} for n, fs in v.items()}
  _, _, g2 = pred.loss_and_param_gnvp(inputs, targets, forcings, v2)
  _, _, g1 = pred.loss_and_param_gnvp(inputs, targets, forcings, v)
  for n in gv:
    for f in gv[n]:
      assert np.array_equal(2 * gv[n][f], g2[n][f]), (n, f)
      assert np.array_equal(gv[n][f], g1[n][f]), (n, f)
  # a zero tangent
  _, _, g0 = pred.loss_and_param_gnvp(inputs, targets, forcings, {})
  for n in g0:
    for f in g0[n]:
      assert not g0[n][f].any(), (n, f)
  # the quadratic form: <v, G v> = 2 L(pred + pdot; targets = pred) (the loss is in physical units on
  # the plain stack only)
  if stack == "plain":
    predictions, tangents = pred.param_jvp(inputs, targets, forcings, v)
    q = 2 * _host_loss(_shift(predictions, tangents, 1.0), _shift(predictions, tangents, 0.0))
    vgv = _pair(gv, v)
    print(f"<v, Gv> {vgv:.8g}, 2 L(pred + pdot; pred) {q:.8g}")
    assert abs(vgv - q) <= 1e-4 * (_dot(v, v) ** 0.5 * _dot(gv, gv) ** 0.5 + abs(q))


# ---- the full Hessian where the predictions equal the targets -------------------------------------------
def test_full_hessian_limit_at_1_degree():
  """With targets = the predictions at p the residual term vanishes and G v is the Hessian times v:
  against [grad L(p + eps v) - grad L(p - eps v)] / 2 eps from loss_and_grads, tensor by tensor.  The
  central difference's truncation error is O(eps^2) relative and its fp32 noise about
  1e-6 |grad| / eps; with eps = 1e-2 of tangents at the parameters' scale, 5e-2 per tensor."""
  model, ar, inputs, template, forcings = _full_problem(graphcast.TASK_13, 1.0, 5, 1)
  pred = ar._predictor
  params = {n: {f: np.asarray(a, np.float32) for f, a in fs.items()} for n, fs in model._params.items()}
  targets = _host(pred(inputs, template, forcings))
  v = _random_param_tangents(params, np.random.default_rng(22))
  torch.cuda.reset_peak_memory_stats()
  _, _, gv = pred.loss_and_param_gnvp(inputs, targets, forcings, v)
  peak = torch.cuda.max_memory_allocated() / 2**30
  eps = 1e-2
  shifted = lambda s: {n: {f: a + s * eps * v[n][f] if n in v and f in v[n] else a
                           for f, a in fs.items()} for n, fs in params.items()}
  model.set_params(shifted(1.0))
  _, _, gp = pred.loss_and_grads(inputs, targets, forcings)
  model.set_params(shifted(-1.0))
  _, _, gm = pred.loss_and_grads(inputs, targets, forcings)
  model.set_params(params)
  worst = 0.0
  for n, fs in gv.items():
    for f, got in fs.items():
      fd = (gp[n][f].astype(np.float64) - gm[n][f]) / (2 * eps)
      if n.startswith(M2G_MESH + "_"):
        assert not got.any()
        continue
      err = float(np.linalg.norm(got - fd) / np.linalg.norm(fd))
      worst = max(worst, err)
      assert err <= 5e-2, (n, f, err)
  print(f"1 deg / 13 levels: worst tensor error against the Hessian central difference {worst:.3g}; "
        f"loss_and_param_gnvp peak {peak:.1f} GiB")
