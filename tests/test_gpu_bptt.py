"""Backprop through time on the device: the feedback-seed and input-gradient kernels against PyTorch,
the engine's input gradient against torch autograd of the fp64 oracle, and the multi-step gradient of
autoregressive.Predictor.loss_and_grads against an independent autograd unroll of the oracle."""
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


# ---- kernels ---------------------------------------------------------------------------------------
def test_feedback_seed_kernel_against_fp64_formula():
  lib = _native.lib()
  gen = torch.Generator(device=DEV).manual_seed(11)
  rng = np.random.default_rng(11)
  lat = np.linspace(-90, 90, 19)
  n_lat, n_lon, n_out, n_planes, n_next, n_rows = len(lat), 37, 45, 60, 50, 70
  n_nodes = n_lat * n_lon
  w = torch.as_tensor(_lat_weight(lat)).to(DEV)
  y = torch.randn(n_nodes, 256, generator=gen, device=DEV)
  targets = torch.randn(n_out, n_nodes, generator=gen, device=DEV)
  add = torch.randn(n_planes, n_nodes, generator=gen, device=DEV)
  scale = torch.rand(n_out, generator=gen, device=DEV) + 0.5
  offset = torch.randn(n_out, generator=gen, device=DEV)
  idx = torch.arange(n_out, dtype=torch.int32, device=DEV) + 7
  idx[::3] = -1
  coef = torch.rand(n_out, generator=gen, device=DEV, dtype=torch.float64)
  a_next = torch.randn(n_next, n_nodes, generator=gen, device=DEV)
  dpred = rng.integers(0, n_next, n_out)
  dpred[::4] = -1
  resid = rng.integers(0, n_out, n_rows)
  resid[::3] = -1
  carry = rng.integers(0, n_next, n_rows)
  carry[::5] = -1
  dpred_d, resid_d, carry_d = _i32(dpred), _i32(resid), _i32(carry)

  def run(with_next):
    g = torch.zeros(n_nodes, 256, device=DEV)
    a_out = torch.full((n_rows, n_nodes), float("nan"), device=DEV)
    _native.check(lib.gcb_output_loss_grad_feedback(
        y.data_ptr(), 256, n_out, n_lat, n_lon, scale.data_ptr(), offset.data_ptr(), add.data_ptr(),
        idx.data_ptr(), targets.data_ptr(), w.data_ptr(), coef.data_ptr(),
        a_next.data_ptr() if with_next else None, dpred_d.data_ptr(), n_rows, resid_d.data_ptr(),
        carry_d.data_ptr(), a_out.data_ptr(), g.data_ptr(), 256, _st()), "feedback")
    return g, a_out

  g, a_out = run(True)
  a = add[idx.clamp(min=0).long()] * (idx >= 0)[:, None]
  t_norm = ((targets - a) - offset[:, None]) / scale[:, None]
  wn = w.double().repeat_interleave(n_lon)
  g_loss = coef[None] * wn[:, None] * (y[:, :n_out] - t_norm.t()).double()        # [nodes, n_out]
  dp = torch.where(torch.as_tensor(dpred >= 0, device=DEV)[None],
                   a_next.double()[torch.as_tensor(np.maximum(dpred, 0), device=DEV)].t(), 0.0)
  want_g = g_loss + scale.double()[None] * dp
  assert _frob(g[:, :n_out], want_g) <= 1e-6
  assert torch.all(g[:, n_out:] == 0)
  want_a = torch.zeros(n_rows, n_nodes, dtype=torch.float64, device=DEV)
  for r in range(n_rows):
    c = resid[r]
    if c >= 0:
      want_a[r] = g_loss[:, c] / scale[c].double() + dp[:, c]
    if carry[r] >= 0:
      want_a[r] += a_next[carry[r]].double()
  assert _frob(a_out, want_a) <= 1e-6
  assert torch.equal(a_out[torch.as_tensor((resid < 0) & (carry < 0), device=DEV)],
                     torch.zeros_like(a_out[torch.as_tensor((resid < 0) & (carry < 0), device=DEV)]))
  g2, a2 = run(True)
  assert torch.equal(g, g2) and torch.equal(a_out, a2)
  # without the following step: g is gcb_output_loss_grad bit for bit
  g_plain = torch.zeros(n_nodes, 256, device=DEV)
  _native.check(lib.gcb_output_loss_grad(
      y.data_ptr(), 256, n_out, n_lat, n_lon, scale.data_ptr(), offset.data_ptr(), add.data_ptr(),
      idx.data_ptr(), targets.data_ptr(), w.data_ptr(), coef.data_ptr(), g_plain.data_ptr(), 256,
      _st()), "g")
  g_null, a_null = run(False)
  assert torch.equal(g_null, g_plain)
  want_null = torch.zeros_like(want_a)
  for r in range(n_rows):
    if resid[r] >= 0:
      want_null[r] = g_loss[:, resid[r]] / scale[resid[r]].double()
  assert _frob(a_null, want_null) <= 1e-6


@pytest.mark.parametrize("with_scale", [True, False])
def test_input_grad_kernel_is_the_same_order_expression(with_scale):
  lib = _native.lib()
  gen = torch.Generator(device=DEV).manual_seed(12)
  n_nodes, ld, n_ch = 19 * 37 + 5, 64, 50
  dx = torch.randn(n_nodes, ld, generator=gen, device=DEV)
  ch = np.random.default_rng(12).integers(0, n_ch, 77)
  ch_d = _i32(ch)
  scale = torch.rand(n_ch, generator=gen, device=DEV) + 0.3
  base = torch.randn(len(ch), n_nodes, generator=gen, device=DEV)
  sel = dx[:, torch.as_tensor(ch, device=DEV)].t()
  term = sel / scale[torch.as_tensor(ch, device=DEV)][:, None] if with_scale else sel

  def run(acc):
    a = base.clone() if acc else torch.full_like(base, float("nan"))
    _native.check(lib.gcb_input_grad(dx.data_ptr(), ld, n_nodes, len(ch), ch_d.data_ptr(),
                                      scale.data_ptr() if with_scale else None, a.data_ptr(), acc,
                                      _st()), "gcb_input_grad")
    return a

  assert torch.equal(run(0), term)
  got = run(1)
  assert torch.equal(got, base + term)
  assert torch.equal(got, run(1))


# ---- the engine's input gradient ---------------------------------------------------------------------
@pytest.mark.parametrize("prec,tol", [("bf16x3", 1e-4), ("bf16", 5e-2)])
def test_engine_input_gradient_against_fp64_autograd(prec, tol):
  g, params, x = _cases.small_case(c_in=31, n_out=23, msg_steps=3, batch=2, randomize_affine=True)
  n_lat = 46
  lat_w = _lat_weight(np.linspace(-90, 90, n_lat))
  rng = np.random.default_rng(7)
  targets = rng.standard_normal((g.num_grid_nodes, 2, 23)).astype(np.float32)
  coef = rng.uniform(0.5, 2.0, 23) / (23 * g.num_grid_nodes)
  eng = engine.Engine(g, params, c_in=31, n_out=23, msg_steps=3, precision=prec)
  eng.grads_begin()
  none = lambda n: _i32(np.full(n, -1))
  fb = engine.Feedback(_i32(np.arange(31)), none(23), none(31), none(31), None)
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
  print(f"{prec}: input gradient relative error {err:.3g}")
  assert err <= tol


# ---- backprop through time against an autograd unroll of the oracle -----------------------------------
def _data(task, batch=2, steps=3, seed=5):
  """_model_and_data for any of the 13-level tasks."""
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
    gc.collect()                              # the dropped engine and its gradient workspace
    torch.cuda.empty_cache()
    shifted.append(float(np.asarray(ar.loss(inputs, targets, forcings)[0].values, np.float64)[0]))
  fd = (shifted[0] - shifted[1]) / (2 * eps)
  rel = abs(fd - gnorm) / gnorm
  print(f"{resolution} deg, T = {steps}: loss {loss:.6g}, |g| {gnorm:.6g}, central difference "
        f"{fd:.6g} (relative {rel:.3g}); peak device memory {peak / 2**30:.1f} GiB on "
        f"{torch.cuda.get_device_name(0)}")
  assert rel <= tol


def test_config1_bptt_directional_derivative():
  """BASELINE config 1 (1 deg, mesh 5, 13 levels, 16 steps), four target times."""
  _directional_check(graphcast.TASK_13, 1.0, 5, 4, 1e-2)


def test_full_size_bptt_directional_derivative_and_peak_memory():
  """0.25 deg / 37 levels, two target times, on an 80 GB GPU."""
  if torch.cuda.get_device_properties(0).total_memory < 75e9:
    pytest.skip("needs an 80 GB GPU")
  _directional_check(graphcast.TASK, 0.25, 6, 2, 1e-2)
