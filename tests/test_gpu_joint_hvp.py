"""Hessian-vector products of the forecast loss jointly in the parameters and the inputs on the device
(loss_and_joint_hvp): both sides against double backward of the fp64 oracle with respect to the params
and the input and forcing variables (each new coupling term in isolation too); the loss, diagnostics
and gradients bit for bit those of loss(), loss_and_grads and loss_and_input_grads; exact scaling and
zero tangents; agreement with the diagonal calls; symmetry of the mixed blocks; central differences at
1 degree / 13 levels; and no interference with the other calls."""
import numpy as np
import pytest
import torch

from graphcast_b200 import graphcast, losses, model_utils
from graphcast_b200 import xarray_shim as xs
from test_gpu_grads import _GradOracle, _frob
from test_gpu_input_grads import _full_problem, _planes_t, _stack
from test_gpu_input_hvp import _as_f32, _random, _same, _shifted, _vals
from test_gpu_input_jvp import _host
from test_gpu_loss import _lat_weight
from test_gpu_param_hvp import _same_ds, _same_grads
from test_gpu_param_jvp import M2G_MESH, _random_param_tangents

pytestmark = pytest.mark.gpu

GRID_EMBEDDER = "grid2mesh_gnn/~_networks_builder/encoder_nodes_grid_nodes"


# ---- against the fp64 oracle -------------------------------------------------------------------------
def _oracle_joint(model, inputs, targets, forcings, stats, vp, it, ft):
  """(parameter gradients, {param: H v}, {("inputs" | "forcings", name): H v}) of the fp64 oracle's
  one-step loss (that of loss_and_grads, through the normalisation and the residual add when `stats`
  are given): double backward with respect to the params and the input and forcing variables, along
  v = (vp, it, ft) (None: zero)."""
  g = model._static_graph.as_dict()
  orc = _GradOracle(model._params, torch.float64)
  batch, n_lat, n_lon = inputs.sizes["batch"], inputs.sizes["lat"], inputs.sizes["lon"]
  ng = n_lat * n_lon
  params = [(n, f, p) for n, fs in orc.p.items() for f, p in fs.items()]
  data, planes = {}, {}
  for tag, ds in (("inputs", inputs), ("forcings", forcings)):
    for name, v in ds.data_vars.items():
      data[(tag, name)] = torch.as_tensor(np.asarray(v.values, np.float64))
  leaves = [p for _, _, p in params] + list(data.values())
  for t in leaves:
    t.requires_grad_(True)

  def field(tag, name):                # [batch, frames, levels, nodes]
    v = (inputs if tag == "inputs" else forcings).data_vars[name]
    dims = list(v.dims)
    frames = v.shape[dims.index("time")] if "time" in dims else 1
    planes[(tag, name)] = _planes_t(data[(tag, name)], dims, batch, n_lat, n_lon).reshape(
        batch, frames, -1, ng)
    return planes[(tag, name)]

  def stat(ds, name):
    return torch.as_tensor(np.asarray(ds[name].values, np.float64)).reshape(1, 1, -1, 1)

  std, mean, dstd = stats if stats is not None else (None, None, None)
  state = {name: field("inputs", name) for name in inputs.keys()}
  feats = []
  for tag, names in (("inputs", sorted(inputs.keys())), ("forcings", sorted(forcings.keys()))):
    for name in names:
      x = state[name] if tag == "inputs" else field(tag, name)
      if stats is not None:
        x = (x - stat(mean, name)) / stat(std, name)
      feats.append(x.reshape(batch, -1, ng))
  y = orc.forward(g, torch.cat(feats, dim=1).permute(2, 0, 1)).permute(1, 2, 0)
  lat_w = torch.as_tensor(np.repeat(_lat_weight(np.asarray(inputs.coords["lat"][1])), n_lon),
                          dtype=torch.float64)
  slabs = model_utils.channel_layout(targets)
  kappa = torch.as_tensor(losses.channel_kappa(slabs, ng, graphcast.LOSS_PER_VARIABLE_WEIGHTS))
  total = torch.zeros(batch, dtype=torch.float64)
  for s in slabs:
    y_v = y[:, s.start:s.start + s.count].reshape(batch, 1, -1, ng)
    t_v = torch.as_tensor(np.asarray(model_utils.variable_to_planes(
        targets.data_vars[s.name], {"batch": batch, "lat": n_lat, "lon": n_lon}), np.float64))
    t_v = t_v.reshape(batch, 1, -1, ng)
    if stats is None:
      t_norm = t_v
    elif s.name in state:
      t_norm = (t_v - state[s.name][:, -1:]) / stat(dstd, s.name)
    else:
      t_norm = (t_v - stat(mean, s.name)) / stat(std, s.name)
    k = kappa[s.start:s.start + s.count].reshape(1, 1, -1, 1)
    total = total + (k * lat_w * (y_v - t_norm) ** 2).sum(dim=(1, 2, 3))
  grads = torch.autograd.grad(total.mean(), leaves, create_graph=True, allow_unused=True)

  tangents = []
  for n, f, _ in params:
    tangents.append(None if vp is None or f not in vp.get(n, {}) else
                    torch.as_tensor(np.asarray(vp[n][f], np.float64)))
  for tag, name in data:
    ds = it if tag == "inputs" else ft
    dims = (inputs if tag == "inputs" else forcings).data_vars[name].dims
    tangents.append(None if ds is None or name not in ds.data_vars else torch.as_tensor(
        np.asarray(ds.data_vars[name].transpose(*dims).values, np.float64)))
  dot = sum((gr * t).sum() for gr, t in zip(grads, tangents) if gr is not None and t is not None)
  hv = torch.autograd.grad(dot, leaves + list(planes.values()), retain_graph=True,
                           allow_unused=True)
  zero = lambda h, leaf: torch.zeros_like(leaf) if h is None else h.detach()
  ref_g, ref_p, ref_x, mag_x = {}, {}, {}, {}
  for (n, f, p), gr, h in zip(params, grads, hv):
    ref_g.setdefault(n, {})[f] = zero(gr, p)
    ref_p.setdefault(n, {})[f] = zero(h, p)
  for key, h in zip(data, hv[len(params):len(leaves)]):
    ref_x[key] = zero(h, data[key])
  # the magnitudes the packing's transpose sums: for a variable broadcast over the grid, the sum of
  # |H v| over its plane's nodes (else |H v| itself)
  for (key, plane), h in zip(planes.items(), hv[len(leaves):]):
    mag_x[key] = torch.autograd.grad(plane, data[key], grad_outputs=zero(h, plane).abs(),
                                     retain_graph=True)[0]
  return ref_g, ref_p, ref_x, mag_x


def _tangents(model, inputs, forcings, which, seed):
  """(v_theta, input tangents, forcing tangents) of one case: "params" (v_x = 0), "inputs"
  (v_theta = 0), "both", or "grid_embedder" (v_theta on the grid embedder alone, v_x = 0)."""
  rng = np.random.default_rng(seed)
  vp = it = ft = None
  if which in ("params", "both"):
    vp = _random_param_tangents(model._params, rng)
  if which == "grid_embedder":
    vp = {n: v for n, v in _random_param_tangents(model._params, rng).items()
          if n.startswith(GRID_EMBEDDER + "_")}
    assert vp
  if which in ("inputs", "both"):
    it, ft = _random(inputs, seed + 1), _random(forcings, seed + 2)
  return vp, it, ft


@pytest.mark.parametrize("task_name,stack,which,precision,tol", [
    ("TASK_13", "plain", "both", "bf16x3", 1e-4),
    ("TASK_13", "plain", "grid_embedder", "bf16x3", 1e-4),
    ("TASK_13", "normalized", "params", "bf16x3", 1e-4),
    ("TASK_13", "normalized", "inputs", "bf16x3", 1e-4),
    ("TASK_13", "normalized", "both", "bf16x3", 1e-4),
    ("TASK_13", "normalized", "grid_embedder", "bf16x3", 1e-4),
    ("TASK", "normalized", "both", "bf16x3", 1e-4),     # 37 levels: c_in_pad 480, n = 512 transposes
    ("TASK_13", "normalized", "both", "bf16", 5e-2),
])
def test_against_the_fp64_oracle(task_name, stack, which, precision, tol):
  """Every parameter tensor of param_hvp and every variable of input_hvp / forcing_hvp against double
  backward of the fp64 oracle.  A parameter tensor's error is relative to its norm.  A variable's is
  relative to the norm of the magnitudes its value sums: |H v| per element, or for a variable the
  packing broadcast (over the grid or the batch) the sum of |H v| over the plane elements it feeds,
  whose fp32 terms carry the error and may cancel in the sum (by 115x for the forcing
  year_progress_sin with v_x alone; for the other variables the two norms are equal).  "inputs" exercises the grid embedder's X-dot^T dh term of the parameter side,
  "grid_embedder" its dh W0-dot^T term of the input side, each without the other.  The gradient is
  checked first, which also checks the oracle's loss."""
  model, pred, inputs, targets, forcings, stats = _stack(task_name, stack, 1)
  vp, it, ft = _tangents(model, inputs, forcings, which, 3)
  model.set_precision(precision)
  try:
    _, _, grads, _, _, ph, ih, fh = pred.loss_and_joint_hvp(inputs, targets, forcings, vp, it, ft)
  finally:
    model.set_precision("bf16x3")
  ref_g, ref_p, ref_x, mag_x = _oracle_joint(model, inputs, targets, forcings, stats, vp, it, ft)
  worst = {"params": 0.0, "inputs": 0.0}
  for name, fields in model._params.items():
    for f in fields:
      if name.startswith(M2G_MESH + "_"):
        assert not ph[name][f].any()
        continue
      if precision == "bf16x3":
        assert _frob(torch.as_tensor(grads[name][f]), ref_g[name][f]) <= 1e-4, (name, f)
      if not float(torch.linalg.norm(ref_p[name][f])):
        assert not ph[name][f].any(), (name, f)
        continue
      err = _frob(torch.as_tensor(ph[name][f]), ref_p[name][f])
      worst["params"] = max(worst["params"], err)
      assert err <= tol, (name, f, err)
  for tag, got_ds, ds in (("inputs", ih, inputs), ("forcings", fh, forcings)):
    for name, v in ds.data_vars.items():
      got = got_ds.data_vars[name]
      assert got.dims == v.dims and np.asarray(got.values).dtype == np.float32
      ref, mag = ref_x[(tag, name)], mag_x[(tag, name)]
      err = float(torch.linalg.norm(torch.as_tensor(np.asarray(got.values)).double() - ref)
                  / torch.linalg.norm(mag))
      worst["inputs"] = max(worst["inputs"], err)
      assert err <= tol, (tag, name, err, _frob(torch.as_tensor(np.asarray(got.values)), ref))
  print(f"{task_name} {stack} {which} {precision}: worst relative error of the parameter side "
        f"{worst['params']:.3g}, of the input side {worst['inputs']:.3g}")


# ---- the primal results and exact properties ---------------------------------------------------------
@pytest.mark.parametrize("task_name,stack", [("TASK_13", "plain"), ("TASK_13", "normalized"),
                                             ("TASK_13", "demo"), ("TASK", "normalized")])
def test_loss_and_gradients_bit_for_bit(task_name, stack):
  """Batch 2: loss and diagnostics bit for bit loss(), grads loss_and_grads, input_grads and
  forcing_grads loss_and_input_grads; the products are shaped like what they differentiate."""
  model, pred, inputs, targets, forcings, _ = _stack(task_name, stack, 1)
  assert inputs.sizes["batch"] == 2
  vp, it, ft = _tangents(model, inputs, forcings, "both", 4)
  loss0, diag0 = pred.loss(inputs, targets, forcings)
  _, _, g0 = pred.loss_and_grads(inputs, targets, forcings)
  _, _, ig0, fg0 = pred.loss_and_input_grads(inputs, targets, forcings)
  loss, diag, g, ig, fg, ph, ih, fh = pred.loss_and_joint_hvp(inputs, targets, forcings, vp, it, ft)
  assert np.array_equal(np.asarray(loss.values), np.asarray(loss0.values))
  assert _same_ds(diag, diag0)
  _same_grads(g, g0)
  _same(ig, ig0)
  _same(fg, fg0)
  assert set(ph) == set(model._params)
  for n, fs in model._params.items():
    for f, a in fs.items():
      assert ph[n][f].dtype == np.float32 and ph[n][f].shape == np.shape(a)
      if n.startswith(M2G_MESH + "_"):
        assert not ph[n][f].any()
  for got, like in ((ih, inputs), (fh, forcings)):
    for name, v in like.data_vars.items():
      h = got.data_vars[name]
      assert h.dims == v.dims and tuple(h.shape) == tuple(v.shape)
      assert np.asarray(h.values).dtype == np.float32 and np.all(np.isfinite(np.asarray(h.values)))


def _scaled(ds, c):
  out = xs.Dataset(coords=ds.coords)
  for k, v in ds.data_vars.items():
    out[k] = xs.DataArray(np.asarray(v.values) * np.float32(c), v.dims)
  return out


def test_scaling_and_zero_tangents():
  """Doubling both tangents doubles every product bit for bit; the same call again gives the same
  bits; no tangents (None) give exact zeros and the same loss and gradients."""
  model, pred, inputs, targets, forcings, _ = _stack("TASK_13", "normalized", 1)
  vp, it, ft = _tangents(model, inputs, forcings, "both", 5)
  out = pred.loss_and_joint_hvp(inputs, targets, forcings, vp, it, ft)
  again = pred.loss_and_joint_hvp(inputs, targets, forcings, vp, it, ft)
  _same_grads(out[5], again[5])
  _same(out[6], again[6])
  _same(out[7], again[7])
  vp2 = {n: {f: 2 * a for f, a in fs.items()} for n, fs in vp.items()}
  two = pred.loss_and_joint_hvp(inputs, targets, forcings, vp2, _scaled(it, 2), _scaled(ft, 2))
  for n, fs in out[5].items():
    for f, a in fs.items():
      assert np.array_equal(2 * a, two[5][n][f]), (n, f)
  for a, b in zip(out[6:], two[6:]):
    va, vb = _vals(a), _vals(b)
    for k in va:
      assert np.array_equal(va[k] * np.float32(2), vb[k]), k
  zero = pred.loss_and_joint_hvp(inputs, targets, forcings)
  assert np.array_equal(np.asarray(zero[0].values), np.asarray(out[0].values))
  _same_grads(zero[2], out[2])
  _same(zero[3], out[3])
  _same(zero[4], out[4])
  for fs in zero[5].values():
    for a in fs.values():
      assert not a.any()
  for ds in zero[6:]:
    for k, a in _vals(ds).items():
      assert not np.any(a), k


def _rel(a, b):
  """Worst relative difference of matching tensors (dicts of dicts) or variables (Datasets)."""
  if isinstance(a, dict):
    pairs = [(a[n][f], b[n][f]) for n in a for f in a[n]]
  else:
    va, vb = _vals(a), _vals(b)
    pairs = [(va[k], vb[k]) for k in va]
  worst = 0.0
  for x, y in pairs:
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    den = np.linalg.norm(y)
    worst = max(worst, float(np.linalg.norm(x - y) / den) if den else float(np.linalg.norm(x)))
  return worst


@pytest.mark.parametrize("stack", ["plain", "normalized"])
def test_the_diagonal_calls(stack):
  """v_x = 0: param_hvp is loss_and_param_hvp's; v_theta = 0: input_hvp and forcing_hvp are
  loss_and_input_hvp's.  The walks differ only in launches that do not form those products (or add
  exact zeros), so they agree to the last bits or within 1e-5."""
  model, pred, inputs, targets, forcings, _ = _stack("TASK_13", stack, 1)
  vp, it, ft = _tangents(model, inputs, forcings, "both", 6)
  ph = pred.loss_and_joint_hvp(inputs, targets, forcings, vp)[5]
  ph0 = pred.loss_and_param_hvp(inputs, targets, forcings, vp)[3]
  ih, fh = pred.loss_and_joint_hvp(inputs, targets, forcings, None, it, ft)[6:]
  ih0, fh0 = pred.loss_and_input_hvp(inputs, targets, forcings, it, ft)[4:]
  d = {"param_hvp": _rel(ph, ph0), "input_hvp": _rel(ih, ih0), "forcing_hvp": _rel(fh, fh0)}
  print(f"{stack}: worst relative difference to the diagonal calls " +
        ", ".join(f"{k} {x:.3g}" for k, x in d.items()))
  for k, x in d.items():
    assert x <= 1e-5, (k, x)


def _joint_dot(a, b):
  """<a, b> of joint vectors (params, input Dataset, forcing Dataset); None parts are zero."""
  s = 0.0
  if a[0] is not None and b[0] is not None:
    s += sum(float(np.sum(np.asarray(x, np.float64) * np.asarray(b[0][n][f], np.float64)))
             for n, fs in a[0].items() for f, x in fs.items() if f in b[0].get(n, {}))
  for x, y in zip(a[1:], b[1:]):
    if x is None or y is None:
      continue
    for k, v in x.data_vars.items():
      s += float(np.sum(np.asarray(v.values, np.float64) *
                        np.asarray(y.data_vars[k].transpose(*v.dims).values, np.float64)))
  return s


def test_symmetry_of_the_mixed_blocks():
  """<u, H v> = <v, H u> for joint tangents u, v, within the Cauchy-Schwarz bound of loss_and_param_hvp's
  test (each product within 1e-4 of exact relative to its norm); and the mixed blocks alone:
  <u_theta, H_theta,x v_x> = <v_x, H_x,theta u_theta>."""
  model, pred, inputs, targets, forcings, _ = _stack("TASK_13", "normalized", 1)
  u = _tangents(model, inputs, forcings, "both", 11)
  v = _tangents(model, inputs, forcings, "both", 21)
  norm = lambda w: _joint_dot(w, w) ** 0.5
  hu = tuple(pred.loss_and_joint_hvp(inputs, targets, forcings, *u)[5:])
  hv = tuple(pred.loss_and_joint_hvp(inputs, targets, forcings, *v)[5:])
  a, b = _joint_dot(u, hv), _joint_dot(v, hu)
  bound = 1e-4 * (norm(u) * norm(hv) + norm(v) * norm(hu))
  print(f"<u, Hv> {a:.9g}, <v, Hu> {b:.9g}, difference / bound {abs(a - b) / bound:.3g}")
  assert abs(a - b) <= bound
  u_p = (u[0], None, None)
  v_x = (None,) + v[1:]
  h_xp = tuple(pred.loss_and_joint_hvp(inputs, targets, forcings, u[0])[5:])   # (H_th,th u, H_x,th u)
  h_px = tuple(pred.loss_and_joint_hvp(inputs, targets, forcings, None, *v[1:])[5:])
  a, b = _joint_dot(u_p, h_px), _joint_dot(v_x, h_xp)
  bound = 1e-4 * (norm(u_p) * norm((h_px[0], None, None)) + norm(v_x) * norm((None,) + h_xp[1:]))
  print(f"<u_th, H_th,x v_x> {a:.9g}, <v_x, H_x,th u_th> {b:.9g}, difference / bound "
        f"{abs(a - b) / bound:.3g}")
  assert abs(a - b) <= bound


def test_no_interference():
  """The other calls give the same bits before and after a joint HVP; weights_version is kept."""
  model, pred, inputs, targets, forcings, _ = _stack("TASK_13", "normalized", 1)
  vp, it, ft = _tangents(model, inputs, forcings, "both", 7)

  def everything():
    out = [_host(pred(inputs, targets, forcings))]
    out.append(pred.loss_and_grads(inputs, targets, forcings)[2])
    out += list(pred.loss_and_input_grads(inputs, targets, forcings)[2:])
    out.append(pred.loss_and_param_hvp(inputs, targets, forcings, vp)[3])
    out += list(pred.loss_and_input_hvp(inputs, targets, forcings, it, ft)[4:])
    out.append(pred.param_jvp(inputs, targets, forcings, vp)[1])
    return out

  before = everything()
  version = model._engine.weights_version
  pred.loss_and_joint_hvp(inputs, targets, forcings, vp, it, ft)
  assert model._engine.weights_version == version
  after = everything()
  for a, b in zip(before, after):
    if isinstance(a, dict):
      _same_grads(a, b)
    else:
      assert _same_ds(_host(a), _host(b))


# ---- 1 degree, 13 levels, 16 message-passing steps ----------------------------------------------------
def test_central_differences_at_1_degree():
  """The mixed blocks against central differences of the gradient calls at random targets:
  H_x,theta v_theta against [loss_and_input_grads(params +- eps v_theta)] / 2 eps, variable by
  variable, and H_theta,x v_x against [loss_and_grads(inputs +- eps v_x)] / 2 eps, tensor by tensor,
  v_x scaled per variable by its spread.  eps = 1e-2: truncation O(eps^2) relative, fp32 noise about
  1e-6 |grad| / eps; 5e-2 per tensor or variable."""
  model, ar, inputs, targets, forcings = _full_problem(graphcast.TASK_13, 1.0, 5, 1)
  pred = ar._predictor
  params = {n: {f: np.asarray(a, np.float32) for f, a in fs.items()} for n, fs in model._params.items()}
  rng = np.random.default_rng(23)
  vp = _random_param_tangents(params, rng)

  def spread_tangents(ds):
    out = xs.Dataset(coords=ds.coords)
    for name, v in ds.data_vars.items():
      x = np.asarray(v.values, np.float64)
      out[name] = xs.DataArray((rng.standard_normal(x.shape) * (x.std() or 1.0)).astype(np.float32),
                               v.dims)
    return out

  it, ft = spread_tangents(inputs), spread_tangents(forcings)
  torch.cuda.reset_peak_memory_stats()
  h_xp = pred.loss_and_joint_hvp(inputs, targets, forcings, vp)[6:]
  peak = torch.cuda.max_memory_allocated() / 2**30
  h_px = pred.loss_and_joint_hvp(inputs, targets, forcings, None, it, ft)[5]
  eps = 1e-2
  shifted = lambda s: {n: {f: a + s * eps * vp[n][f] if n in vp and f in vp[n] else a
                           for f, a in fs.items()} for n, fs in params.items()}
  model.set_params(shifted(1.0))
  _, _, gp_i, gp_f = pred.loss_and_input_grads(inputs, targets, forcings)
  model.set_params(shifted(-1.0))
  _, _, gm_i, gm_f = pred.loss_and_input_grads(inputs, targets, forcings)
  model.set_params(params)
  _, _, gp = pred.loss_and_grads(_as_f32(_shifted(inputs, it, eps)), targets,
                                 _as_f32(_shifted(forcings, ft, eps)))
  _, _, gm = pred.loss_and_grads(_as_f32(_shifted(inputs, it, -eps)), targets,
                                 _as_f32(_shifted(forcings, ft, -eps)))
  worst = {}
  for got_ds, p_ds, m_ds in ((h_xp[0], gp_i, gm_i), (h_xp[1], gp_f, gm_f)):
    for name in got_ds.keys():
      fd = (np.asarray(p_ds.data_vars[name].values, np.float64) -
            np.asarray(m_ds.data_vars[name].values, np.float64)) / (2 * eps)
      worst[("x", name)] = _frob(torch.as_tensor(np.asarray(got_ds.data_vars[name].values)),
                                 torch.as_tensor(fd))
  for n, fs in h_px.items():
    for f, got in fs.items():
      if n.startswith(M2G_MESH + "_"):
        assert not got.any()
        continue
      fd = (gp[n][f].astype(np.float64) - gm[n][f]) / (2 * eps)
      worst[("theta", n, f)] = _frob(torch.as_tensor(got), torch.as_tensor(fd))
  for side in ("x", "theta"):
    w = max(((k, e) for k, e in worst.items() if k[0] == side), key=lambda kv: kv[1])
    print(f"1 deg / 13 levels: worst relative difference of H_{side},other against the central "
          f"difference {w[1]:.3g} at {w[0][1:]}")
  print(f"loss_and_joint_hvp peak {peak:.1f} GiB on {torch.cuda.get_device_name(0)}")
  for k, err in worst.items():
    assert err <= 5e-2, (k, err)
