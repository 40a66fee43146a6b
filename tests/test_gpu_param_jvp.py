"""Forward-mode derivatives with respect to the parameters on the device (param_jvp): the LayerNorm
tangent kernel with parameter terms against fp64 torch.func.jvp, every prediction tangent against
forward-mode autodiff of the fp64 oracle unroll with the params as primals, the exact properties
(predictions of __call__, zero tangents, linearity under an exact scaling), the directional derivative
of the loss against loss_and_grads, central differences through set_params, and no interference with
the other calls."""
import gc

import numpy as np
import pytest
import torch
import torch.autograd.forward_ad as fwAD

from graphcast_b200 import _native, graphcast, losses, model_utils
from graphcast_b200 import xarray_shim as xs
from test_gpu_grads import _GradOracle, _frob
from test_gpu_input_grads import _full_problem, _planes_t, _stack
from test_gpu_input_jvp import _device_planes

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
GAMMA = 2.0 ** -24                                      # unit roundoff of fp32


def _st():
  return torch.cuda.current_stream().cuda_stream


def _same(a, b):
  """Bit for bit, NaNs included."""
  return torch.equal(a.view(torch.int32), b.view(torch.int32))


# ---- kernel ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [0, 1, 7, 8, 9, 1003])
@pytest.mark.parametrize("ld", [512, 516])
def test_layernorm_jvp_params_kernel_against_fp64(rows, ld):
  """out = residual + scale * rstd * (dz - mean dz - zhat mean(zhat dz)) + dscale * zhat + doffset
  against torch.func.jvp in fp64 of layer_norm with respect to (z, scale, offset).

  Rounding model (fp32, unit roundoff g = 2^-24): the row statistics are sums of 512 terms, each with a
  relative error of at most 512 g of the sum of the magnitudes; mu, rstd and zhat inherit that (the
  variance sum and its rsqrt: <= 2 * 512 g + 4 g).  The tangent's two row means add 2 * 512 g of
  |scale| rstd (mean|dz| + |zhat| mean|zhat dz|), and every element takes at most 8 further roundings.
  So per element |err| <= 1100 g * (|scale| rstd (|dz| + mean|dz| + |zhat| mean|zhat dz|) + |dscale
  zhat|) + 4 g (|residual| + |doffset|), with rstd and zhat taken from fp64."""
  lib = _native.lib()
  n = 512
  gen = torch.Generator(device=DEV).manual_seed(rows + ld)
  z = torch.randn(max(rows, 1), ld, generator=gen, device=DEV) * 2 + 0.5
  dz = torch.randn(max(rows, 1), ld, generator=gen, device=DEV)
  scale = torch.rand(n, generator=gen, device=DEV) + 0.5
  offset = torch.randn(n, generator=gen, device=DEV)
  dscale, doffset = torch.randn(n, generator=gen, device=DEV), torch.randn(n, generator=gen, device=DEV)
  res = torch.randn(max(rows, 1), ld, generator=gen, device=DEV)

  def run(residual, ds, do, entry="params"):
    out = torch.full((max(rows, 1), ld), float("nan"), device=DEV)
    rp = None if residual is None else residual.data_ptr()
    if entry == "params":
      _native.check(lib.gcb_layernorm_jvp_params(
          z.data_ptr(), ld, dz.data_ptr(), ld, scale.data_ptr(), rows, n, rp, ld,
          None if ds is None else ds.data_ptr(), None if do is None else do.data_ptr(),
          out.data_ptr(), ld, _st()), "gcb_layernorm_jvp_params")
    else:
      _native.check(lib.gcb_layernorm_jvp(z.data_ptr(), ld, dz.data_ptr(), ld, scale.data_ptr(), rows,
                                          n, rp, ld, out.data_ptr(), ld, _st()), "gcb_layernorm_jvp")
    return out

  zd, dzd = z[:rows, :n].double(), dz[:rows, :n].double()

  def ln(x, s, o):
    return (x - x.mean(-1, keepdim=True)) * torch.rsqrt(x.var(-1, unbiased=False, keepdim=True)
                                                        + 1e-5) * s + o
  rstd = torch.rsqrt(zd.var(-1, unbiased=False, keepdim=True) + 1e-5)
  zhat = (zd - zd.mean(-1, keepdim=True)) * rstd
  worst = 0.0
  for residual in (None, res):
    for ds, do in ((dscale, doffset), (dscale, None), (None, doffset), (None, None)):
      out = run(residual, ds, do)
      if rows == 0:
        assert torch.isnan(out).all()                     # nothing written
        continue
      zero = torch.zeros(n, dtype=torch.float64, device=DEV)
      sd = zero if ds is None else ds.double()
      od = zero if do is None else do.double()
      _, want = torch.func.jvp(ln, (zd, scale.double(), offset.double()), (dzd, sd, od))
      r = torch.zeros_like(want) if residual is None else residual[:rows, :n].double()
      want = want + r
      mag = (scale.double().abs() * rstd * (dzd.abs() + dzd.abs().mean(-1, keepdim=True)
                                           + zhat.abs() * (zhat * dzd).abs().mean(-1, keepdim=True))
             + (sd * zhat).abs())
      bound = 1100 * GAMMA * mag + 4 * GAMMA * (r.abs() + od.abs())
      err = (out[:rows, :n].double() - want).abs()
      worst = max(worst, float((err / bound).max()))
      assert bool((err <= bound).all()), float((err / bound).max())
      if ld > n:
        assert torch.isnan(out[:rows, n:]).all()          # the columns past n are not written
      assert _same(run(residual, ds, do), out)            # deterministic
    # without parameter tangents: bit for bit gcb_layernorm_jvp
    assert _same(run(residual, None, None), run(residual, None, None, entry="jvp"))
  print(f"rows {rows}, ld {ld}: largest error / bound {worst:.3g}")


# ---- against forward-mode autodiff of the fp64 oracle unroll -------------------------------------------
def _oracle_param_jvp(model, inputs, targets, forcings, stats, tangents):
  """{name: [batch, steps, channels, nodes] fp64 prediction tangents} by forward-mode autodiff of the
  fp64 oracle unroll (normalisation, residual add, the feeding of predictions and forcings into the next
  inputs), the params the primals and `tangents` ({module: {field: array}}) their tangents."""
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
    for name, fields in tangents.items():
      for f, t in fields.items():
        orc.p[name][f] = fwAD.make_dual(orc.p[name][f], torch.as_tensor(np.asarray(t, np.float64)))

    def field(ds, name, t=None):
      v = ds.data_vars[name]
      x, dims = torch.as_tensor(np.asarray(v.values, np.float64)), list(v.dims)
      if t is not None:
        x = x.narrow(dims.index("time"), t, 1)
      frames = x.shape[dims.index("time")] if "time" in dims else 1
      return _planes_t(x, dims, batch, n_lat, n_lon).reshape(batch, frames, -1, ng)

    state = {name: field(inputs, name) for name in inputs.keys()}
    time_dep = {name for name in inputs.keys() if "time" in inputs.data_vars[name].dims}
    for t in range(targets.sizes["time"]):
      f_t = {name: field(forcings, name, t) for name in forcings.keys()}
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
        tan = fwAD.unpack_dual(pred).tangent
        out[s.name].append(torch.zeros_like(pred) if tan is None else tan.detach().clone())
      state = {name: (torch.cat([v[:, 1:], preds[name] if name in preds else f_t[name]], dim=1)
                      if name in time_dep else v) for name, v in state.items()}
  return {name: torch.cat(ts, dim=1) for name, ts in out.items()}


STEMS = {
    "g2m_edge_embedder": "grid2mesh_gnn/~_networks_builder/encoder_edges_grid2mesh",
    "processor_edge_mlp": "mesh_gnn/~_networks_builder/processor_edges_1_mesh",
    "decoder": "mesh2grid_gnn/~_networks_builder/decoder_nodes_grid_nodes",
}
LN_OFFSET = "mesh_gnn/~_networks_builder/processor_nodes_0_mesh_nodes_layer_norm"
M2G_MESH = "mesh2grid_gnn/~_networks_builder/processor_nodes_0_mesh_nodes"


def _random_param_tangents(params, rng, which="all"):
  """Random tangents shaped like the params, each entry of about its parameter's scale."""
  out = {}
  for name, fields in params.items():
    if which == "all":
      keep = True
    elif which == "ln_offset":
      keep = name == LN_OFFSET
    else:
      keep = name.startswith(STEMS[which] + "_")
    if not keep:
      continue
    for f, a in fields.items():
      if which == "ln_offset" and f != "offset":
        continue
      a = np.asarray(a, np.float32)
      s = float(np.std(a)) or 0.1
      out.setdefault(name, {})[f] = (rng.standard_normal(a.shape) * s).astype(np.float32)
  return out


@pytest.mark.parametrize("task_name,stack,steps,which,tol", [
    ("TASK_13", "plain", 1, "all", 1e-4),
    ("TASK_13", "normalized", 1, "all", 1e-4),
    ("TASK_13", "normalized", 3, "all", 1e-4),
    ("TASK_13", "plain", 3, "g2m_edge_embedder", 1e-4),
    ("TASK_13", "normalized", 1, "processor_edge_mlp", 1e-4),
    ("TASK_13", "normalized", 3, "ln_offset", 1e-4),
    ("TASK_13", "plain", 1, "decoder", 1e-4),
    ("TASK_13", "demo", 1, "all", 5e-2),
    ("TASK_13", "demo", 3, "all", 5e-2),
    ("TASK", "normalized", 1, "all", 1e-4),             # 37 levels: c_in_pad 480
    ("TASK", "normalized", 3, "g2m_edge_embedder", 1e-4),
])
def test_prediction_tangents_against_forward_mode_unroll(task_name, stack, steps, which, tol):
  """Tolerances as test_gpu_input_jvp derives them: bf16x3 GEMMs carry about 1e-6 relative error per
  product and the tangent is linear in them, so the fp32 tangent stays within 1e-4 of fp64 relative
  to its norm; bf16 operands (the demo stack) carry 2^-8 per product, hence 5e-2."""
  model, pred, inputs, targets, forcings, stats = _stack(task_name, stack, steps)
  rng = np.random.default_rng(17)
  v = _random_param_tangents(model._params, rng, which)
  predictions, tangents = pred.param_jvp(inputs, targets, forcings, v)
  ref = _oracle_param_jvp(model, inputs, targets, forcings, stats, v)
  batch, n_lat, n_lon = inputs.sizes["batch"], inputs.sizes["lat"], inputs.sizes["lon"]
  worst = 0.0
  assert set(tangents.keys()) == set(targets.keys())
  for name in targets.keys():
    got_v = tangents.data_vars[name]
    assert got_v.dims == predictions.data_vars[name].dims
    assert tuple(got_v.shape) == tuple(predictions.data_vars[name].shape)
    assert np.asarray(got_v.values).dtype == np.float32
    want = ref[name]
    if float(torch.linalg.norm(want)) == 0.0:
      assert not np.asarray(got_v.values).any(), name
      continue
    err = _frob(_device_planes(tangents, name, steps, batch, n_lat, n_lon), want)
    worst = max(worst, err)
    assert err <= tol, (name, err)
  print(f"{task_name} {stack} T={steps} {which}: worst per-variable relative error {worst:.3g}")
  again = pred(inputs, targets, forcings)
  for name in again.keys():
    assert np.array_equal(np.asarray(predictions.data_vars[name].values),
                          np.asarray(again.data_vars[name].values))


# ---- exact properties ----------------------------------------------------------------------------------
def _values(ds):
  return {k: np.asarray(ds.data_vars[k].values) for k in ds.keys()}


@pytest.mark.parametrize("stack,steps", [("normalized", 1), ("normalized", 3), ("plain", 1)])
def test_zero_tangents_and_exact_scaling(stack, steps):
  model, pred, inputs, targets, forcings, _ = _stack("TASK_13", stack, steps)
  params = model._params
  zero = {name: {f: np.zeros(np.shape(a), np.float32) for f, a in fields.items()}
          for name, fields in params.items()}
  m2g_mesh = {name: {f: np.ones(np.shape(a), np.float32) for f, a in fields.items()}
              for name, fields in params.items() if name.startswith(M2G_MESH + "_")}
  assert m2g_mesh
  for v in (zero, {}, m2g_mesh):
    _, t = pred.param_jvp(inputs, targets, forcings, v)
    for name, a in _values(t).items():
      assert not a.any(), name
  v = _random_param_tangents(params, np.random.default_rng(5))
  v2 = {n: {f: 2 * a for f, a in fs.items()} for n, fs in v.items()}
  _, t1 = pred.param_jvp(inputs, targets, forcings, v)
  _, t2 = pred.param_jvp(inputs, targets, forcings, v2)
  _, t1b = pred.param_jvp(inputs, targets, forcings, v)
  for name in t1.keys():
    a1, a2 = np.asarray(t1.data_vars[name].values), np.asarray(t2.data_vars[name].values)
    assert np.array_equal(2 * a1, a2), name
    assert np.array_equal(a1, np.asarray(t1b.data_vars[name].values)), name   # deterministic


# ---- the directional derivative of the loss ---------------------------------------------------------------
def _host_loss(predictions, targets):
  loss, _ = losses.weighted_mse_per_level(predictions, targets,
                                          per_variable_weights=graphcast.LOSS_PER_VARIABLE_WEIGHTS)
  return float(np.mean(np.asarray(loss.values, np.float64)))


def _shift(ds, tangents, s):
  out = xs.Dataset(coords=ds.coords)
  for k in ds.keys():
    out[k] = xs.DataArray(np.asarray(ds.data_vars[k].values, np.float64)
                          + s * np.asarray(tangents.data_vars[k].transpose(*ds.data_vars[k].dims).values,
                                           np.float64), ds.data_vars[k].dims)
  return out


def _pair(grads, v):
  return sum(float(np.sum(np.asarray(grads[n][f], np.float64) * np.asarray(a, np.float64)))
             for n, fs in v.items() for f, a in fs.items())


@pytest.mark.parametrize("stack", ["plain"])
def test_directional_derivative_matches_loss_and_grads(stack):
  """sum over tensors of <grad, v> = dL/d eps along v, the latter from param_jvp's outputs as
  [L(pred + pdot) - L(pred - pdot)] / 2, exact for the quadratic loss.  L is losses.weighted_mse_per_level
  of the physical predictions, the model's loss on the plain stack (the normalised stack's loss is on
  normalised residuals)."""
  model, pred, inputs, targets, forcings, _ = _stack("TASK_13", stack, 1)
  v = _random_param_tangents(model._params, np.random.default_rng(8))
  _, _, grads = pred.loss_and_grads(inputs, targets, forcings)
  predictions, tangents = pred.param_jvp(inputs, targets, forcings, v)
  fd = (_host_loss(_shift(predictions, tangents, 1.0), targets)
        - _host_loss(_shift(predictions, tangents, -1.0), targets)) / 2
  got = _pair(grads, v)
  print(f"{stack}: <grad, v> {got:.6g}, loss derivative from param_jvp {fd:.6g}")
  assert abs(got - fd) <= 1e-4 * abs(fd)


# ---- central differences through set_params ----------------------------------------------------------------
@pytest.mark.parametrize("resolution,mesh_size,task_name", [(1.0, 5, "TASK_13")])
def test_central_differences(resolution, mesh_size, task_name):
  """Per variable against (f(p + eps v) - f(p - eps v)) / 2 eps with in-place set_params, eps = 1e-3
  of tangents at the parameters' scale: the truncation error is O(eps^2) relative and the fp32
  cancellation about 1e-7 / eps, so 1e-2 per variable."""
  model, ar, inputs, targets, forcings = _full_problem(getattr(graphcast, task_name), resolution,
                                                       mesh_size, 1)
  pred = ar._predictor
  params = {n: {f: np.asarray(a, np.float32) for f, a in fs.items()} for n, fs in model._params.items()}
  v = _random_param_tangents(params, np.random.default_rng(21))
  _, tangents = pred.param_jvp(inputs, targets, forcings, v)
  eps = 1e-3
  shifted = lambda s: {n: {f: a + s * eps * v[n][f] if n in v and f in v[n] else a
                           for f, a in fs.items()} for n, fs in params.items()}
  model.set_params(shifted(1.0))
  plus = _values(pred(inputs, targets, forcings))
  model.set_params(shifted(-1.0))
  minus = _values(pred(inputs, targets, forcings))
  model.set_params(params)
  worst = 0.0
  for name, t in _values(tangents).items():
    fd = (plus[name].astype(np.float64) - minus[name]) / (2 * eps)
    err = float(np.linalg.norm(t - fd) / np.linalg.norm(fd))
    worst = max(worst, err)
    assert err <= 1e-2, (name, err)
  print(f"{resolution} deg: worst per-variable central-difference error {worst:.3g}; "
        f"param_jvp peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")


# ---- no interference ------------------------------------------------------------------------------------
def test_param_jvp_does_not_interfere():
  model, pred, inputs, targets, forcings, _ = _stack("TASK_13", "normalized", 1)
  rng = np.random.default_rng(4)
  v = _random_param_tangents(model._params, rng)
  d_in = xs.Dataset(coords=inputs.coords)
  d_in["temperature"] = xs.DataArray(
      rng.standard_normal(inputs.data_vars["temperature"].shape).astype(np.float32),
      inputs.data_vars["temperature"].dims)

  def observe():
    out = {"call": _values(pred(inputs, targets, forcings))}
    loss, _, grads = pred.loss_and_grads(inputs, targets, forcings)
    out["loss"] = np.asarray(loss.values)
    out["grads"] = {f"{n}:{f}": a for n, fs in grads.items() for f, a in fs.items()}
    _, t = pred.input_jvp(inputs, targets, forcings, d_in)
    out["input_jvp"] = _values(t)
    return out

  before = observe()
  version = model.engine.weights_version
  pred.param_jvp(inputs, targets, forcings, v)
  assert model.engine.weights_version == version
  after = observe()
  for key in before:
    if isinstance(before[key], dict):
      for name in before[key]:
        assert np.array_equal(before[key][name], after[key][name]), (key, name)
    else:
      assert np.array_equal(before[key], after[key]), key
  # the static-edge cache comes back for inference once the derivative workspace is released
  model.engine.release_gradient_workspace()
  builds = model.engine.static_cache_builds
  again = _values(pred(inputs, targets, forcings))
  assert model.engine.static_cache_builds == builds + 1
  for name in again:
    assert np.array_equal(again[name], before["call"][name]), name
  gc.collect()
