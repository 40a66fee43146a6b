"""Hessian-vector products of the forecast loss with respect to the parameters on the device
(loss_and_param_hvp): the LayerNorm kernel gcb_layernorm_backward_jvp_params against fp64 and its
one-direction counterparts, the loss / diagnostics / gradients bit for bit those of loss() and
loss_and_grads, H v against double backward of the fp64 oracle, the Gauss-Newton relation, the exact
identities (symmetry, scaling, zero tangents), central differences at 1 degree, and no interference
with the other calls."""
import numpy as np
import pytest
import torch

from graphcast_b200 import _native, graphcast, losses, model_utils
from test_gpu_grads import _GradOracle, _frob
from test_gpu_input_grads import _full_problem, _stack
from test_gpu_input_jvp import _host
from test_gpu_param_gnvp import _dot, _features
from test_gpu_param_jvp import GAMMA, LN_OFFSET, M2G_MESH, _random_param_tangents, _same

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
N = 512


def _st():
  return torch.cuda.current_stream().cuda_stream


# ---- kernel ------------------------------------------------------------------------------------------
def _ln_backward(dy, z, s):
  """dz of hk.LayerNorm's backward in the arithmetic of the input dtype, and its three column sums."""
  mu = z.mean(-1, keepdim=True)
  rstd = torch.rsqrt(z.var(-1, unbiased=False, keepdim=True) + 1e-5)
  zhat = (z - mu) * rstd
  g = dy * s
  dz = rstd * (g - g.mean(-1, keepdim=True) - zhat * (g * zhat).mean(-1, keepdim=True))
  return dz, dz.sum(0), (dy * zhat).sum(0), dy.sum(0)


@pytest.mark.parametrize("rows,pad", [(1, 0), (7, 5), (255, 0), (256, 3), (257, 128), (1003, 21),
                                      (70001, 0)])
def test_layernorm_backward_jvp_params_kernel(rows, pad):
  """Direction 0 and its sums are gcb_layernorm_backward's bits; with scale_dot NULL, direction 1 is
  gcb_layernorm_backward_jvp's bits; against fp64 torch.func.jvp of the LayerNorm backward with
  respect to (dy, z, scale).

  Rounding model (fp32, unit roundoff u = 2^-24): the row statistics, zhat and zhat-dot carry relative
  errors of at most ~2 * 512 u of the magnitudes they are summed from, each of the four row means of
  the tangent another 512 u, and every element at most 12 further roundings.  So per element
  |err| <= 3000 u * m, m = the fp64 magnitude of the tangent formula with every term and mean taken
  in absolute value.  A tangent column sum adds the fp32 partials of 256 row slices in fp64: its error
  is at most the sum of the element bounds plus 2^-24 of the sum of magnitudes per slice fold."""
  lib = _native.lib()
  gen = torch.Generator(device=DEV).manual_seed(rows + pad)
  stride = rows + pad
  z = torch.randn(rows, N, generator=gen, device=DEV) * 2 + 0.5
  zd = torch.randn(rows, N, generator=gen, device=DEV)
  dy = torch.full((stride + rows, N), float("nan"), device=DEV)
  dy[:rows] = torch.randn(rows, N, generator=gen, device=DEV)
  dy[stride:] = torch.randn(rows, N, generator=gen, device=DEV)
  scale = torch.rand(N, generator=gen, device=DEV) + 0.5
  sdot = torch.randn(N, generator=gen, device=DEV)
  base = [torch.randn(N, generator=gen, device=DEV) for _ in range(6)]
  ws = torch.empty(lib.gcb_rowwise_workspace_bytes(N), dtype=torch.uint8, device=DEV)

  def run(sd):
    dz = torch.full((stride + rows, N), float("nan"), device=DEV)
    sums = [b.clone() for b in base]
    _native.check(lib.gcb_layernorm_backward_jvp_params(
        dy.data_ptr(), N, stride, z.data_ptr(), N, zd.data_ptr(), N, scale.data_ptr(),
        None if sd is None else sd.data_ptr(), rows, N, dz.data_ptr(), N, ws.data_ptr(), ws.numel(),
        *[t.data_ptr() for t in sums], 1, _st()), "gcb_layernorm_backward_jvp_params")
    return dz, sums

  dz, sums = run(sdot)
  if pad:
    assert torch.isnan(dz[rows:stride]).all()              # pad rows between directions: not written
  # direction 0: gcb_layernorm_backward's bits
  dz0 = torch.full((rows, N), float("nan"), device=DEV)
  ref = [b.clone() for b in base[:3]]
  _native.check(lib.gcb_layernorm_backward(
      dy.data_ptr(), N, z.data_ptr(), N, scale.data_ptr(), rows, N, dz0.data_ptr(), N, ws.data_ptr(),
      ws.numel(), *[t.data_ptr() for t in ref], 1, _st()), "gcb_layernorm_backward")
  assert _same(dz[:rows], dz0)
  for a, b in zip(sums[:3], ref):
    assert _same(a, b)
  # scale_dot NULL: gcb_layernorm_backward_jvp's direction 1
  dzn, _ = run(None)
  dzj = torch.full((stride + rows, N), float("nan"), device=DEV)
  _native.check(lib.gcb_layernorm_backward_jvp(
      dy.data_ptr(), N, z.data_ptr(), N, zd.data_ptr(), N, scale.data_ptr(), rows, N, stride,
      dzj.data_ptr(), N, _st()), "gcb_layernorm_backward_jvp")
  assert _same(dzn[stride:], dzj[stride:])
  # deterministic
  dz2, sums2 = run(sdot)
  assert _same(dz, dz2) and all(_same(a, b) for a, b in zip(sums, sums2))
  # against fp64
  d = lambda t: t.double()
  prim = (d(dy[:rows]), d(z), d(scale))
  _, tan = torch.func.jvp(_ln_backward, prim, (d(dy[stride:]), d(zd), d(sdot)))
  y0, z64, s64 = prim
  mu = z64.mean(-1, keepdim=True)
  rstd = torch.rsqrt(z64.var(-1, unbiased=False, keepdim=True) + 1e-5)
  zhat = (z64 - mu) * rstd
  zh_d = rstd * (d(zd).abs() + d(zd).abs().mean(-1, keepdim=True)
                 + zhat.abs() * (zhat * d(zd)).abs().mean(-1, keepdim=True))
  g, gd = (y0 * s64).abs(), (d(dy[stride:]) * s64).abs() + (y0 * d(sdot)).abs()
  mean = lambda x: x.mean(-1, keepdim=True)
  rd = rstd * mean((zhat * d(zd)).abs())
  m = (rd * (g + mean(g) + zhat.abs() * mean(g * zhat.abs()))
       + rstd * (gd + mean(gd) + zh_d * mean(g * zhat.abs()) + zhat.abs() * mean(gd * zhat.abs() + g * zh_d)))
  bound = 3000 * GAMMA * m
  err = (d(dz[stride:]) - tan[0]).abs()
  worst = float((err / bound).max())
  assert bool((err <= bound).all()), worst
  # tangent sums: [bias, scale, offset]
  mags = [m, d(dy[stride:]).abs() * zhat.abs() + y0.abs() * zh_d, d(dy[stride:]).abs()]
  for q, (got, want, mag) in enumerate(zip(sums[3:], tan[1:], mags)):
    b = 3000 * GAMMA * (m.sum(0) if q == 0 else mag.sum(0)) + 2 * GAMMA * mag.sum(0) + 2 * GAMMA * \
        base[3 + q].double().abs()
    e = (got.double() - base[3 + q].double() - want).abs()
    worst = max(worst, float((e / b).max()))
    assert bool((e <= b).all()), (q, float((e / b).max()))
  print(f"rows {rows}: largest error / bound {worst:.3g}")


# ---- the primal results ------------------------------------------------------------------------------
def _same_ds(a, b):
  return all(np.array_equal(np.asarray(a.data_vars[k].values), np.asarray(b.data_vars[k].values))
             for k in a.keys())


def _same_grads(a, b):
  assert set(a) == set(b)
  for n in a:
    for f in a[n]:
      assert np.array_equal(a[n][f], b[n][f]), (n, f)


@pytest.mark.parametrize("task_name,stack", [("TASK_13", "plain"), ("TASK_13", "normalized"),
                                             ("TASK_13", "demo"), ("TASK", "normalized")])
def test_loss_and_grads_are_those_of_loss_and_grads(task_name, stack):
  """Batch 2: loss and diagnostics bit for bit loss(), grads bit for bit loss_and_grads."""
  model, pred, inputs, targets, forcings, _ = _stack(task_name, stack, 1)
  assert inputs.sizes["batch"] == 2
  v = _random_param_tangents(model._params, np.random.default_rng(4))
  loss0, diag0 = pred.loss(inputs, targets, forcings)
  _, _, grads0 = pred.loss_and_grads(inputs, targets, forcings)
  loss, diag, grads, hvp = pred.loss_and_param_hvp(inputs, targets, forcings, v)
  assert np.array_equal(np.asarray(loss.values), np.asarray(loss0.values))
  assert _same_ds(diag, diag0)
  _same_grads(grads, grads0)
  assert set(hvp) == set(model._params)
  for n, fs in model._params.items():
    for f, a in fs.items():
      assert hvp[n][f].dtype == np.float32 and hvp[n][f].shape == np.shape(a)
      if n.startswith(M2G_MESH + "_"):
        assert not hvp[n][f].any()


# ---- against the fp64 oracle -------------------------------------------------------------------------
class _NoForcings:
  """No forcings: _features of the targets alone."""

  def isel(self, **kw):
    return {}

  def keys(self):
    return []


def _oracle_hvp(model, inputs, targets, forcings, v):
  """(grad, H v) of the fp64 oracle's loss sum_c coef_c / 2 sum_node w (y - t)^2 (plain stack): double
  backward of _GradOracle."""
  g = model._static_graph.as_dict()
  x = _features(inputs, forcings, None)
  batch, n_lat, n_lon = inputs.sizes["batch"], inputs.sizes["lat"], inputs.sizes["lon"]
  slabs = model_utils.channel_layout(targets)
  coef = 2.0 * losses.channel_kappa(slabs, n_lat * n_lon, graphcast.LOSS_PER_VARIABLE_WEIGHTS) / batch
  w = losses.normalized_latitude_weights(targets[sorted(targets.keys())[0]])
  h = torch.as_tensor(np.repeat(np.asarray(w, np.float64), n_lon))[:, None, None] * \
      torch.as_tensor(np.asarray(coef, np.float64))[None, None, :]
  t = _features(targets, _NoForcings(), None)
  orc = _GradOracle(model._params, torch.float64)
  leaves = [(n, f, p) for n, fs in orc.p.items() for f, p in fs.items()]
  for _, _, p in leaves:
    p.requires_grad_(True)
  y = orc.forward(g, x)
  loss = (h / 2 * (y - t) ** 2).sum()
  grads = torch.autograd.grad(loss, [p for _, _, p in leaves], create_graph=True, allow_unused=True)
  dot = sum((gr * torch.as_tensor(np.asarray(v[n][f], np.float64))).sum()
            for (n, f, _), gr in zip(leaves, grads) if gr is not None and n in v and f in v[n])
  hv = torch.autograd.grad(dot, [p for _, _, p in leaves], allow_unused=True)
  out_g, out_h = {}, {}
  for (n, f, p), gr, hh in zip(leaves, grads, hv):
    out_g.setdefault(n, {})[f] = torch.zeros_like(p) if gr is None else gr.detach()
    out_h.setdefault(n, {})[f] = torch.zeros_like(p) if hh is None else hh.detach()
  return out_g, out_h


LN_SCALE = LN_OFFSET


def _tangents(params, which, rng):
  if which == "ln_scale":
    a = np.asarray(params[LN_SCALE]["scale"], np.float32)
    return {LN_SCALE: {"scale": (rng.standard_normal(a.shape) * (float(np.std(a)) or 0.1))
                       .astype(np.float32)}}
  if which == "mesh_encoder":
    stem = "grid2mesh_gnn/~_networks_builder/encoder_nodes_mesh_nodes"
    return {n: {f: (rng.standard_normal(np.shape(a)) * (float(np.std(a)) or 0.1)).astype(np.float32)
                for f, a in fs.items()} for n, fs in params.items() if n.startswith(stem + "_")}
  return _random_param_tangents(params, rng, which)


@pytest.mark.parametrize("task_name,which,tol", [
    ("TASK_13", "all", 1e-4), ("TASK_13", "ln_scale", 1e-4), ("TASK_13", "g2m_edge_embedder", 1e-4),
    ("TASK_13", "mesh_encoder", 1e-4), ("TASK_13", "processor_edge_mlp", 1e-4),
    ("TASK_13", "decoder", 1e-4), ("TASK", "all", 1e-4)])
def test_hvp_against_the_fp64_oracle(task_name, which, tol):
  """H v tensor by tensor against double backward of the fp64 oracle, relative to each tensor's norm
  (bf16x3: the tangent forward and both directions of the walk are each within about 1e-5 of fp64).
  The gradient is checked first, which also checks the oracle's target planes."""
  model, pred, inputs, targets, forcings, _ = _stack(task_name, "plain", 1)
  v = _tangents(model._params, which, np.random.default_rng(3))
  assert v
  _, _, grads, hvp = pred.loss_and_param_hvp(inputs, targets, forcings, v)
  ref_g, ref_h = _oracle_hvp(model, inputs, targets, forcings, v)
  worst = 0.0
  for name, fields in model._params.items():
    for f in fields:
      if name.startswith(M2G_MESH + "_"):
        assert not hvp[name][f].any()
        continue
      assert _frob(torch.as_tensor(grads[name][f]), ref_g[name][f]) <= 1e-4, (name, f)
      if not float(torch.linalg.norm(ref_h[name][f])):
        assert not hvp[name][f].any(), (name, f)
        continue
      err = _frob(torch.as_tensor(hvp[name][f]), ref_h[name][f])
      worst = max(worst, err)
      assert err <= tol, (name, f, err)
  print(f"{task_name} {which}: worst tensor relative error of H v {worst:.3g}")


def test_hvp_bf16_against_the_fp64_oracle():
  """The bf16 precision, plain stack: 5e-2 per tensor (2^-8 operand rounding)."""
  model, pred, inputs, targets, forcings, _ = _stack("TASK_13", "plain", 1)
  model.set_precision("bf16")
  try:
    v = _random_param_tangents(model._params, np.random.default_rng(5))
    _, _, _, hvp = pred.loss_and_param_hvp(inputs, targets, forcings, v)
  finally:
    model.set_precision("bf16x3")
  _, ref_h = _oracle_hvp(model, inputs, targets, forcings, v)
  worst = 0.0
  for name, fields in model._params.items():
    for f in fields:
      if name.startswith(M2G_MESH + "_") or not float(torch.linalg.norm(ref_h[name][f])):
        continue
      err = _frob(torch.as_tensor(hvp[name][f]), ref_h[name][f])
      worst = max(worst, err)
      assert err <= 5e-2, (name, f, err)
  print(f"bf16: worst tensor relative error of H v {worst:.3g}")


# ---- the Gauss-Newton relation and exact properties ---------------------------------------------------
def _diff(a, b):
  num = sum(float(np.sum((np.asarray(a[n][f], np.float64) - b[n][f]) ** 2)) for n in a for f in a[n])
  return num ** 0.5 / _dot(b, b) ** 0.5


def test_gauss_newton_relation():
  """With targets = the predictions the residual term vanishes and H v = G v: both are within 1e-4 of
  their fp64 values relative to their norms, so they differ by at most 2e-4 relative.  At random
  targets the residual term is present, and the two differ by far more."""
  model, pred, inputs, targets, forcings, _ = _stack("TASK_13", "plain", 1)
  v = _random_param_tangents(model._params, np.random.default_rng(8))
  at = _host(pred(inputs, targets, forcings))
  _, _, _, hv = pred.loss_and_param_hvp(inputs, at, forcings, v)
  _, _, gv = pred.loss_and_param_gnvp(inputs, at, forcings, v)
  near = _diff(hv, gv)
  _, _, _, hv_r = pred.loss_and_param_hvp(inputs, targets, forcings, v)
  _, _, gv_r = pred.loss_and_param_gnvp(inputs, targets, forcings, v)
  far = _diff(hv_r, gv_r)
  print(f"|Hv - Gv| / |Gv|: {near:.3g} at targets = predictions, {far:.3g} at random targets")
  assert near <= 2e-4
  assert far > 2e-4


@pytest.mark.parametrize("stack", ["plain", "normalized"])
def test_exact_properties(stack):
  model, pred, inputs, targets, forcings, _ = _stack("TASK_13", stack, 1)
  rng = np.random.default_rng(12)
  u, v = _random_param_tangents(model._params, rng), _random_param_tangents(model._params, rng)
  _, _, g0, hv = pred.loss_and_param_hvp(inputs, targets, forcings, v)
  _, _, _, hu = pred.loss_and_param_hvp(inputs, targets, forcings, u)
  # symmetry: H u and H v are each within 1e-4 of exact relative to their norms, so by Cauchy-Schwarz
  # <u, Hv> and <v, Hu> differ by at most 1e-4 (|u| |Hv| + |v| |Hu|)
  a, b = _dot(hu, v), _dot(hv, u)
  bound = 1e-4 * (_dot(v, v) ** 0.5 * _dot(hu, hu) ** 0.5 + _dot(u, u) ** 0.5 * _dot(hv, hv) ** 0.5)
  print(f"{stack}: <u, Hv> {b:.8g}, <v, Hu> {a:.8g}, difference / bound {abs(a - b) / bound:.3g}")
  assert abs(a - b) <= bound
  v2 = {n: {f: 2 * x for f, x in fs.items()} for n, fs in v.items()}
  _, _, _, h2 = pred.loss_and_param_hvp(inputs, targets, forcings, v2)
  _, _, g1, h1 = pred.loss_and_param_hvp(inputs, targets, forcings, v)
  _same_grads(g1, g0)
  for n in hv:
    for f in hv[n]:
      assert np.array_equal(2 * hv[n][f], h2[n][f]), (n, f)
      assert np.array_equal(hv[n][f], h1[n][f]), (n, f)
  _, _, gz, hz = pred.loss_and_param_hvp(inputs, targets, forcings, {})
  _same_grads(gz, g0)
  for n in hz:
    for f in hz[n]:
      assert not hz[n][f].any(), (n, f)


def test_no_interference():
  """The other calls give the same bits before and after a parameter HVP; weights_version is kept."""
  model, pred, inputs, targets, forcings, _ = _stack("TASK_13", "normalized", 1)
  v = _random_param_tangents(model._params, np.random.default_rng(6))

  def everything():
    out = [_host(pred(inputs, targets, forcings))]
    out.append(pred.loss_and_grads(inputs, targets, forcings)[2])
    out.append(pred.loss_and_param_gnvp(inputs, targets, forcings, v)[2])
    out.append(pred.param_jvp(inputs, targets, forcings, v)[1])
    out.append(pred.loss_and_input_hvp(inputs, targets, forcings, inputs)[4])
    return out

  before = everything()
  version = model._engine.weights_version
  pred.loss_and_param_hvp(inputs, targets, forcings, v)
  assert model._engine.weights_version == version
  after = everything()
  for a, b in zip(before, after):
    if isinstance(a, dict):
      _same_grads(a, b)
    else:
      assert _same_ds(_host(a), _host(b))


# ---- 1 degree, 13 levels, 16 message-passing steps ----------------------------------------------------
def test_central_differences_at_1_degree():
  """H v against [grad L(p + eps v) - grad L(p - eps v)] / 2 eps from loss_and_grads at random targets,
  tensor by tensor: the central difference's truncation error is O(eps^2) relative and its fp32 noise
  about 1e-6 |grad| / eps; with eps = 1e-2 of tangents at the parameters' scale, 5e-2 per tensor."""
  model, ar, inputs, targets, forcings = _full_problem(graphcast.TASK_13, 1.0, 5, 1)
  pred = ar._predictor
  params = {n: {f: np.asarray(a, np.float32) for f, a in fs.items()} for n, fs in model._params.items()}
  v = _random_param_tangents(params, np.random.default_rng(22))
  torch.cuda.reset_peak_memory_stats()
  _, _, _, hv = pred.loss_and_param_hvp(inputs, targets, forcings, v)
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
  for n, fs in hv.items():
    for f, got in fs.items():
      if n.startswith(M2G_MESH + "_"):
        assert not got.any()
        continue
      fd = (gp[n][f].astype(np.float64) - gm[n][f]) / (2 * eps)
      err = float(np.linalg.norm(got - fd) / np.linalg.norm(fd))
      worst = max(worst, err)
      assert err <= 5e-2, (n, f, err)
  print(f"1 deg / 13 levels: worst tensor error against the central difference {worst:.3g}; "
        f"loss_and_param_hvp peak {peak:.1f} GiB")
