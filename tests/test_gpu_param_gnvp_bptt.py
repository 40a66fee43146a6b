"""Gauss-Newton products of the multi-step forecast loss (autoregressive.Predictor.loss_and_param_gnvp
over several target times) on the device: the seed kernel gcb_output_loss_gn_seed_feedback against its
one-step and loss-seed counterparts bit for bit and against fp64, the loss of loss(), G v against the
fp64 oracle unroll (forward-mode r-dot, then reverse mode of sum_t <Lambda_t r-dot_t, r_t>), the
quadratic form against multi-step param_jvp, the exact properties, the full-Hessian limit against
central differences of multi-step loss_and_grads, and no interference with the other calls."""
import numpy as np
import pytest
import torch
import torch.autograd.forward_ad as fwAD

from graphcast_b200 import _native, autoregressive, graphcast, losses, model_utils, normalization
from graphcast_b200 import xarray_shim as xs
from test_gpu_bptt import _data
from test_gpu_grads import _GradOracle, _frob
from test_gpu_input_grads import _full_problem, _stack
from test_gpu_input_jvp import _host
from test_gpu_loss import _lat_weight, _stats
from test_gpu_param_jvp import M2G_MESH, _random_param_tangents, _values

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
GAMMA = 2.0 ** -24                                      # unit roundoff of fp32


def _st():
  return torch.cuda.current_stream().cuda_stream


def _bits(a):
  return a.contiguous().view(torch.int32)


def _one(ds, t=0):
  return ds.isel(time=slice(t, t + 1)) if "time" in ds.sizes else ds


# ---- seed kernel -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_lat,n_lon,n_out,ld_g,n_rows", [
    (1, 1, 1, 1, 0), (1, 4, 3, 4, 5), (19, 36, 83, 256, 70), (7, 33, 227, 260, 454),
    (181, 360, 227, 256, 454)])
def test_gn_seed_feedback_kernel(n_lat, n_lon, n_out, ld_g, n_rows):
  """Bit for bit gcb_output_loss_grad_feedback with y = pdot^T, zero targets and no offset / add planes
  (scale NULL), and gcb_output_loss_gn_seed without feedback or rows; with a scale, against the fp64
  formula.  d = pdot / scale is one fp32 rounding, g and a_out one more each (the fp64 terms are exact
  to 2^-50), and the carry one fp32 addition: |g - g64| <= 2 g (|coef w d| + |scale dp|), |a_out -
  a64| <= 3 g (|coef w d / scale| + |dp| + |carry|)."""
  lib = _native.lib()
  gen = torch.Generator(device=DEV).manual_seed(n_out + n_rows)
  rng = np.random.default_rng(n_out + n_rows)
  ng = n_lat * n_lon
  n_next = max(n_rows, 1) + 3
  pdot = torch.randn(n_out, ng, generator=gen, device=DEV)
  pdot[0, 0] = -0.0
  scale = torch.rand(n_out, generator=gen, device=DEV) + 0.5
  lat = torch.rand(n_lat, generator=gen, device=DEV) + 0.1
  coef = torch.rand(n_out, generator=gen, device=DEV, dtype=torch.float64)
  a_next = torch.randn(n_next, ng, generator=gen, device=DEV)
  i32 = lambda a: torch.as_tensor(np.asarray(a, np.int32)).to(DEV)
  dpred = i32(rng.integers(-1, n_next, n_out))
  resid = i32(rng.integers(-1, n_out, max(n_rows, 1)))
  carry = i32(rng.integers(-1, n_next, max(n_rows, 1)))
  zeros = torch.zeros(n_out, ng, device=DEV)
  y = torch.full((ng, ld_g), float("nan"), device=DEV)
  y[:, :n_out] = pdot.t()
  ptr = lambda t: None if t is None else t.data_ptr()

  def new(sc, an, rows):
    g = torch.full((ng, ld_g), float("nan"), device=DEV)
    a = torch.full((max(rows, 1), ng), float("nan"), device=DEV)
    _native.check(lib.gcb_output_loss_gn_seed_feedback(
        pdot.data_ptr(), n_out, n_lat, n_lon, ptr(sc), lat.data_ptr(), coef.data_ptr(), ptr(an),
        dpred.data_ptr(), rows, resid.data_ptr(), carry.data_ptr(), a.data_ptr(), g.data_ptr(), ld_g,
        _st()), "gcb_output_loss_gn_seed_feedback")
    return g, a

  for an in (None, a_next):
    g, a = new(None, an, n_rows)
    want_g = torch.full((ng, ld_g), float("nan"), device=DEV)
    want_a = torch.full((max(n_rows, 1), ng), float("nan"), device=DEV)
    _native.check(lib.gcb_output_loss_grad_feedback(
        y.data_ptr(), ld_g, n_out, n_lat, n_lon, None, None, None, None, zeros.data_ptr(),
        lat.data_ptr(), coef.data_ptr(), ptr(an), dpred.data_ptr(), n_rows, resid.data_ptr(),
        carry.data_ptr(), want_a.data_ptr(), want_g.data_ptr(), ld_g, _st()),
        "gcb_output_loss_grad_feedback")
    assert torch.equal(_bits(g), _bits(want_g))          # pad columns included: both NaN
    assert torch.equal(_bits(a), _bits(want_a))
  g, _ = new(None, None, 0)
  want = torch.full((ng, ld_g), float("nan"), device=DEV)
  _native.check(lib.gcb_output_loss_gn_seed(y.data_ptr(), ld_g, n_out, n_lat, n_lon, lat.data_ptr(),
                                            coef.data_ptr(), want.data_ptr(), ld_g, _st()),
                "gcb_output_loss_gn_seed")
  assert torch.equal(_bits(g), _bits(want))
  # with a scale, against fp64
  w = lat.double().repeat_interleave(n_lon)[None, :]
  c = coef[:, None]
  s = scale.double()[:, None]
  d = pdot.double() / s
  for an in (None, a_next):
    g, a = new(scale, an, n_rows)
    assert torch.isnan(g[:, n_out:]).all()                # columns >= n_out are never written
    dp = torch.zeros(n_out, ng, dtype=torch.float64, device=DEV)
    if an is not None:
      ok = dpred >= 0
      dp[ok] = an.double()[dpred[ok].long()]
    g64 = c * w * d + s * dp
    err = (g[:, :n_out].t().double() - g64).abs()
    bound = 2 * GAMMA * ((c * w * d).abs() + (s * dp).abs()) + 1e-300
    assert bool((err <= bound).all()), float((err / bound).max())
    assert torch.equal(_bits(new(scale, an, n_rows)[0]), _bits(g))     # deterministic
    if n_rows == 0:
      assert torch.isnan(a).all()
      continue
    rc = resid.long()
    on = rc >= 0
    a64 = torch.zeros(n_rows, ng, dtype=torch.float64, device=DEV)
    a64[on] = (c * w * d / s + dp)[rc[on]]
    mag = torch.zeros_like(a64)
    mag[on] = ((c * w * d / s).abs() + dp.abs())[rc[on]]
    if an is not None:
      k = carry.long()
      has = k >= 0
      a64[has] += an.double()[k[has]]
      mag[has] += an.double()[k[has]].abs()
    err = (a.double() - a64).abs()
    assert bool((err <= 3 * GAMMA * mag + 1e-300).all())


# ---- the fp64 oracle: forward-mode r-dot of the unroll, then reverse mode of <Lambda r-dot, r> ------------
def _residuals(orc, model, inputs, targets, forcings, stats, teacher_forced):
  """[batch, n_out, Ng] fp64 normalised residuals of every step of the oracle unroll (normalisation,
  residual add, the feeding of predictions and forcings into the next inputs).  teacher_forced: every
  step starts from inputs without derivatives (primal values, detached)."""
  g = model._static_graph
  batch, n_lat, n_lon = inputs.sizes["batch"], inputs.sizes["lat"], inputs.sizes["lon"]
  ng = n_lat * n_lon
  sizes = {"batch": batch, "lat": n_lat, "lon": n_lon}

  def field(ds, name):
    v = ds.data_vars[name]
    p = torch.as_tensor(np.asarray(model_utils.variable_to_planes(v, sizes), np.float64))
    return p.reshape(batch, v.sizes["time"] if "time" in v.dims else 1, -1, ng)

  def stat(ds, name):
    return torch.as_tensor(np.asarray(ds[name].values, np.float64)).reshape(1, 1, -1, 1)

  std, mean, dstd = stats if stats is not None else (None, None, None)
  state = {name: field(inputs, name) for name in inputs.keys()}
  time_dep = {name for name in inputs.keys() if "time" in inputs.data_vars[name].dims}
  slabs = model_utils.channel_layout(_one(targets))
  out = []
  for t in range(targets.sizes["time"]):
    f_t, tgt = _one(forcings, t), _one(targets, t)
    if teacher_forced:
      state = {k: fwAD.unpack_dual(v).primal.detach() for k, v in state.items()}
    feats = []
    for src, names in ((state, sorted(inputs.keys())), (None, sorted(f_t.keys()))):
      for name in names:
        v = src[name] if src is not None else field(f_t, name)
        if stats is not None:
          v = (v - stat(mean, name)) / stat(std, name)
        feats.append(v.reshape(batch, -1, ng))
    x = torch.cat(feats, dim=1).permute(2, 0, 1)
    y = orc.forward(g.as_dict(), x).permute(1, 2, 0)
    preds, r = {}, []
    for s in slabs:
      y_v = y[:, s.start:s.start + s.count].reshape(batch, 1, -1, ng)
      t_v = field(tgt, s.name)
      if stats is None:
        pred, t_norm = y_v, t_v
      elif s.name in state:
        last = state[s.name][:, -1:]
        pred, t_norm = y_v * stat(dstd, s.name) + last, (t_v - last) / stat(dstd, s.name)
      else:
        pred = y_v * stat(std, s.name) + stat(mean, s.name)
        t_norm = (t_v - stat(mean, s.name)) / stat(std, s.name)
      preds[s.name] = pred
      r.append((y_v - t_norm).reshape(batch, -1, ng))
    out.append(torch.cat(r, dim=1))
    state = {name: (torch.cat([v[:, 1:], preds[name] if name in preds else field(f_t, name)], dim=1)
                    if name in time_dep else v) for name, v in state.items()}
  return out


def _oracle_gnvp(model, inputs, targets, forcings, stats, v, teacher_forced=False):
  """sum_t J_t^T Lambda_t J_t v of the fp64 oracle: r-dot_t by forward mode through the unroll, then
  autograd of sum_t <stopgrad(Lambda_t r-dot_t), r_t>, Lambda_t = coef * lat_weight."""
  batch, n_lat, n_lon = inputs.sizes["batch"], inputs.sizes["lat"], inputs.sizes["lon"]
  steps = targets.sizes["time"]
  slabs = model_utils.channel_layout(_one(targets))
  kappa = losses.channel_kappa(slabs, n_lat * n_lon, graphcast.LOSS_PER_VARIABLE_WEIGHTS)
  coef = torch.as_tensor(2.0 * kappa / (batch * steps), dtype=torch.float64)[None, :, None]
  w = torch.as_tensor(np.repeat(_lat_weight(np.asarray(inputs.coords["lat"][1])), n_lon),
                      dtype=torch.float64)[None, None, :]
  orc = _GradOracle(model._params, torch.float64)
  with fwAD.dual_level():
    for name, fields in v.items():
      for f, t in fields.items():
        orc.p[name][f] = fwAD.make_dual(orc.p[name][f], torch.as_tensor(np.asarray(t, np.float64)))
    rdot = []
    for r in _residuals(orc, model, inputs, targets, forcings, stats, teacher_forced):
      tan = fwAD.unpack_dual(r).tangent
      rdot.append(torch.zeros_like(r) if tan is None else tan.detach().clone())
  orc = _GradOracle(model._params, torch.float64)
  for fields in orc.p.values():
    for t in fields.values():
      t.requires_grad_(True)
  rs = _residuals(orc, model, inputs, targets, forcings, stats, teacher_forced)
  sum((coef * w * rd * r).sum() for rd, r in zip(rdot, rs)).backward()
  return {k: {f: (t.grad if t.grad is not None else torch.zeros_like(t)) for f, t in fs.items()}
          for k, fs in orc.p.items()}


def _rel_all(a, b):
  num = sum(float(((torch.as_tensor(a[k][f]).double() - b[k][f]) ** 2).sum()) for k in b for f in b[k])
  den = sum(float((b[k][f] ** 2).sum()) for k in b for f in b[k])
  return (num / den) ** 0.5


def _same_loss(got, want):
  (loss, diag), (loss0, diag0) = got, want
  assert np.array_equal(np.asarray(loss.values), np.asarray(loss0.values))
  assert set(diag.keys()) == set(diag0.keys())
  for name in diag0.keys():
    assert np.array_equal(np.asarray(diag.data_vars[name].values),
                          np.asarray(diag0.data_vars[name].values)), name


@pytest.mark.parametrize("task_name,stack,steps,which,tol", [
    ("TASK_13", "plain", 2, "all", 1e-4),
    ("TASK_13", "normalized", 2, "all", 1e-4),
    ("TASK_13", "normalized", 3, "all", 1e-4),
    ("TASK_13", "plain", 3, "ln_offset", 1e-4),
    ("TASK_13", "normalized", 2, "g2m_edge_embedder", 1e-4),
    ("TASK_13", "normalized", 3, "processor_edge_mlp", 1e-4),
    ("TASK_13", "normalized", 2, "decoder", 1e-4),
    ("TASK_13", "demo", 2, "all", 5e-2),
    ("TASK_13", "demo", 3, "all", 5e-2),
    ("TASK", "normalized", 2, "all", 1e-4),              # 37 levels: c_in_pad 480
    ("TASK", "plain", 3, "all", 1e-4),
])
def test_gnvp_against_the_fp64_oracle(task_name, stack, steps, which, tol):
  """Tolerances as for the one-step call and multi-step loss_and_grads: the tangent rollout and the
  backward pass are each within about 1e-5 of fp64 in bf16x3 relative to the norm, 2^-8-driven 5e-2 in
  bf16; tensor by tensor relative to each tensor's norm.  The loss and diagnostics are loss()'s bits."""
  model, pred, inputs, targets, forcings, stats = _stack(task_name, stack, steps)
  v = _random_param_tangents(model._params, np.random.default_rng(3), which)
  loss, diag, gnvp = pred.loss_and_param_gnvp(inputs, targets, forcings, v)
  _same_loss((loss, diag), pred.loss(inputs, targets, forcings))
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
  forced = _oracle_gnvp(model, inputs, targets, forcings, stats, v, teacher_forced=True)
  sensitivity = _rel_all({k: {f: a for f, a in fs.items()} for k, fs in gnvp.items()}, forced)
  print(f"{task_name} {stack} T={steps} {which}: worst tensor relative error {worst:.3g}; the "
        f"teacher-forced product differs by {sensitivity:.3g}")
  assert sensitivity >= 10 * tol


# ---- noise -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stack", ["plain", "norm"])
def test_noise_is_that_of_loss_and_grads(stack):
  task = graphcast.TASK_13
  model, inputs, targets, forcings = _data(task, steps=2)
  inner = model if stack == "plain" else normalization.InputsAndResiduals(model, *_stats(task, seed=1))
  noisy = autoregressive.Predictor(inner, noise_level=0.1, gradient_checkpointing=True)
  clean = autoregressive.Predictor(inner, gradient_checkpointing=True)
  v = _random_param_tangents(model._params, np.random.default_rng(6))
  loss, diag, gv = noisy.loss_and_param_gnvp(inputs, targets, forcings, v, rng=42)
  _same_loss((loss, diag), noisy.loss(inputs, targets, forcings, rng=42))
  noised = noisy.noisy_inputs(inputs, targets, forcings, 42)
  _, _, want = clean.loss_and_param_gnvp(noised, targets, forcings, v)
  _, _, plain = clean.loss_and_param_gnvp(inputs, targets, forcings, v)
  differs = False
  for n in want:
    for f in want[n]:
      assert np.array_equal(gv[n][f], want[n][f]), (n, f)
      differs |= not np.array_equal(gv[n][f], plain[n][f])
  assert differs                                        # the noise reaches the product


# ---- against multi-step param_jvp ----------------------------------------------------------------------------
def _dot(a, b):
  return sum(float(np.sum(np.asarray(a[n][f], np.float64) * np.asarray(b[n][f], np.float64)))
             for n in a if n in b for f in a[n] if f in b[n])


def _jvp_form(ar, model, inputs, targets, forcings, u, v):
  """sum_b sum_t sum_{c, node} coef_c lat (pdot_t(u) / s_c)(pdot_t(v) / s_c) from param_jvp's
  prediction tangents, s the output scale (1 on the plain stack)."""
  eng = model.engine
  batch, steps = inputs.sizes["batch"], targets.sizes["time"]
  one = _one(targets)
  inner = ar._predictor
  if isinstance(inner, normalization.InputsAndResiduals):
    s = inner._fused_constants(inputs, one, _one(forcings), eng.device).out_scale.double().cpu()
  else:
    s = torch.ones(eng.n_out, dtype=torch.float64)
  slabs = model_utils.channel_layout(one)
  kappa = losses.channel_kappa(slabs, eng.num_grid, graphcast.LOSS_PER_VARIABLE_WEIGHTS)
  coef = torch.as_tensor(2.0 * kappa / (batch * steps), dtype=torch.float64)
  lat = model._lat_weight(one, eng.device).double().cpu()
  w = lat.repeat_interleave(eng.num_grid // lat.shape[0])
  planes = []
  for x in (u, v):
    tangents = _host(ar.param_jvp(inputs, targets, forcings, x)[1])
    planes.append([model._cotangent_planes(_one(tangents, t), one, batch).double() / s[:, None]
                   for t in range(steps)])
  return sum(float((coef[:, None] * w[None, :] * a * b).sum()) for a, b in zip(*planes))


@pytest.mark.parametrize("size", ["small", "1deg"])
def test_quadratic_form_against_param_jvp(size):
  """<u, G v> against the quadratic form of param_jvp's prediction tangents (the tangent rollout is
  shared, the backward through time is not), to 1e-4 of sqrt(Q(u, u) Q(v, v)); symmetry within the
  same bound."""
  if size == "small":
    model, ar, inputs, targets, forcings, _ = _stack("TASK_13", "normalized", 3)
  else:
    model, ar, inputs, targets, forcings = _full_problem(graphcast.TASK_13, 1.0, 5, 2)
  rng = np.random.default_rng(31)
  u, v = _random_param_tangents(model._params, rng), _random_param_tangents(model._params, rng)
  _, _, gv = ar.loss_and_param_gnvp(inputs, targets, forcings, v)
  _, _, gu = ar.loss_and_param_gnvp(inputs, targets, forcings, u)
  quv = _jvp_form(ar, model, inputs, targets, forcings, u, v)
  quu = _jvp_form(ar, model, inputs, targets, forcings, u, u)
  qvv = _jvp_form(ar, model, inputs, targets, forcings, v, v)
  scale = (quu * qvv) ** 0.5
  uv, vu, vv = _dot(u, gv), _dot(v, gu), _dot(v, gv)
  print(f"{size}: <u, Gv> {uv:.8g}, <v, Gu> {vu:.8g}, form {quv:.8g}; <v, Gv> {vv:.8g}, form "
        f"{qvv:.8g}; errors / sqrt(Q(u,u) Q(v,v)) {abs(uv - quv) / scale:.3g}, "
        f"{abs(vv - qvv) / qvv:.3g}, symmetry {abs(uv - vu) / scale:.3g}")
  assert abs(uv - quv) <= 1e-4 * scale
  assert abs(vv - qvv) <= 1e-4 * qvv
  assert abs(uv - vu) <= 1e-4 * scale


# ---- exact properties ------------------------------------------------------------------------------------------
def test_exact_properties():
  model, ar, inputs, targets, forcings, _ = _stack("TASK_13", "normalized", 2)
  v = _random_param_tangents(model._params, np.random.default_rng(12))
  v2 = {n: {f: 2 * x for f, x in fs.items()} for n, fs in v.items()}
  loss, _, g1 = ar.loss_and_param_gnvp(inputs, targets, forcings, v)
  _, _, g2 = ar.loss_and_param_gnvp(inputs, targets, forcings, v2)
  again, _, g1b = ar.loss_and_param_gnvp(inputs, targets, forcings, v)
  zero_loss, _, g0 = ar.loss_and_param_gnvp(inputs, targets, forcings, {})
  assert np.array_equal(loss.values, again.values) and np.array_equal(loss.values, zero_loss.values)
  for n in g1:
    for f in g1[n]:
      assert np.array_equal(2 * g1[n][f], g2[n][f]), (n, f)      # G (2 v) = 2 G v, bit for bit
      assert np.array_equal(g1[n][f], g1b[n][f]), (n, f)         # deterministic
      assert not g0[n][f].any(), (n, f)                          # a zero tangent: exact zeros


# ---- the full Hessian where every step's targets are the rollout's own predictions -----------------------------
def test_full_hessian_limit_at_1_degree():
  """With targets = the rollout's predictions every step's residual vanishes and G v is the Hessian of
  the multi-step loss times v: against [grad L(p + eps v) - grad L(p - eps v)] / 2 eps from multi-step
  loss_and_grads, tensor by tensor.  Truncation O(eps^2) relative, fp32 noise about 1e-6 |grad| / eps;
  with eps = 1e-2 of tangents at the parameters' scale, 5e-2 per tensor."""
  model, ar, inputs, template, forcings = _full_problem(graphcast.TASK_13, 1.0, 5, 2)
  params = {n: {f: np.asarray(a, np.float32) for f, a in fs.items()} for n, fs in model._params.items()}
  targets = _host(ar(inputs, template, forcings))
  v = _random_param_tangents(params, np.random.default_rng(22))
  torch.cuda.reset_peak_memory_stats()
  _, _, gv = ar.loss_and_param_gnvp(inputs, targets, forcings, v)
  peak = torch.cuda.max_memory_allocated() / 2**30
  eps = 1e-2
  shifted = lambda s: {n: {f: a + s * eps * v[n][f] if n in v and f in v[n] else a
                           for f, a in fs.items()} for n, fs in params.items()}
  model.set_params(shifted(1.0))
  _, _, gp = ar.loss_and_grads(inputs, targets, forcings)
  model.set_params(shifted(-1.0))
  _, _, gm = ar.loss_and_grads(inputs, targets, forcings)
  model.set_params(params)
  worst = 0.0
  for n, fs in gv.items():
    for f, got in fs.items():
      if n.startswith(M2G_MESH + "_"):
        assert not got.any()
        continue
      fd = (gp[n][f].astype(np.float64) - gm[n][f]) / (2 * eps)
      err = float(np.linalg.norm(got - fd) / np.linalg.norm(fd))
      worst = max(worst, err)
      assert err <= 5e-2, (n, f, err)
  print(f"1 deg / 13 levels, T = 2: worst tensor error against the Hessian central difference "
        f"{worst:.3g}; peak {peak:.1f} GiB")


# ---- no interference ---------------------------------------------------------------------------------------------
def test_does_not_interfere():
  model, ar, inputs, targets, forcings, _ = _stack("TASK_13", "normalized", 3)
  rng = np.random.default_rng(4)
  v = _random_param_tangents(model._params, rng)
  two = lambda ds: ds.isel(time=slice(0, 2))
  d_in = xs.Dataset(coords=inputs.coords)
  d_in["temperature"] = xs.DataArray(
      rng.standard_normal(inputs.data_vars["temperature"].shape).astype(np.float32),
      inputs.data_vars["temperature"].dims)
  flat = lambda d: {f"{n}:{f}": a for n, fs in d.items() for f, a in fs.items()}

  def observe():
    out = {"call": _values(ar(inputs, targets, forcings))}
    for tag, sl in (("1", _one), ("2", two)):
      loss, _, grads = ar.loss_and_grads(inputs, sl(targets), sl(forcings))
      out["loss" + tag], out["grads" + tag] = {"": np.asarray(loss.values)}, flat(grads)
    out["gnvp1"] = flat(ar.loss_and_param_gnvp(inputs, _one(targets), _one(forcings), v)[2])
    out["param_jvp3"] = _values(ar.param_jvp(inputs, targets, forcings, v)[1])
    hvp = ar.loss_and_input_hvp(inputs, two(targets), two(forcings), d_in)
    out["input_hvp2"] = {**{"g" + k: a for k, a in _values(hvp[2]).items()},
                         **{"h" + k: a for k, a in _values(hvp[4]).items()}}
    return out

  before = observe()
  version = model.engine.weights_version
  ar.loss_and_param_gnvp(inputs, two(targets), two(forcings), v)
  assert model.engine.weights_version == version
  after = observe()
  for key in before:
    for name in before[key]:
      assert np.array_equal(before[key][name], after[key][name]), (key, name)
