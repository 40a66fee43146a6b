"""The forecast loss on the device: the argument checks of gcb_output_loss (its arithmetic is checked
against fp64 in test_gpu_grid_io_kernels.py), and GraphCast.loss / loss_and_predictions, InputsAndResiduals and the autoregressive loss against the host mirror of the
reference's losses (graphcast_b200.losses, itself pinned to the executed reference in
tests/test_reference_losses_golden.py)."""
import numpy as np
import pytest
import torch

from graphcast_b200 import (_native, autoregressive, casting, engine, graph as graph_lib, graphcast,
                            losses, model_utils, normalization, rollout, synthetic)
from graphcast_b200 import xarray_shim as xs
from oracle import gnn as oracle_gnn

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _lat_weight(lat):
  da = xs.DataArray(np.zeros(len(lat), np.float32), ("lat",), coords={"lat": lat})
  return losses.normalized_latitude_weights(da).astype(np.float32)


def test_output_loss_argument_checks():
  lib = _native.lib()
  st = torch.cuda.current_stream().cuda_stream
  n_out, n_lat, n_lon = 5, 3, 4
  y = torch.zeros(12, 8, device=DEV)
  t = torch.zeros(n_out, 12, device=DEV)
  w = torch.ones(n_lat, device=DEV)
  sums = torch.zeros(n_out, dtype=torch.float64, device=DEV)
  nbytes = lib.gcb_output_loss_workspace_bytes(n_out)
  assert nbytes > 0 and lib.gcb_output_loss_workspace_bytes(0) == -1
  ws = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
  idx = torch.zeros(n_out, dtype=torch.int32, device=DEV)

  def call(y_=y.data_ptr(), ld=8, n=n_out, lat=n_lat, lon=n_lon, add=None, index=None,
           targets=t.data_ptr(), ws_bytes=nbytes, ws_ptr=ws.data_ptr(), out=sums.data_ptr()):
    return lib.gcb_output_loss(y_, ld, n, lat, lon, None, None, add, index, targets, w.data_ptr(),
                               None, ws_ptr, ws_bytes, out, st)

  assert call() == 0
  assert call(targets=None) != 0
  assert call(y_=None) != 0
  assert call(out=None) != 0
  assert call(ld=4) != 0                                     # ld_y < n_out
  assert call(lat=0) != 0
  assert call(index=idx.data_ptr()) != 0                     # add planes / index mismatch
  assert call(ws_bytes=nbytes - 8) != 0
  assert call(ws_ptr=ws.data_ptr() + 4) != 0                 # fp64 partials unaligned
  torch.cuda.synchronize()


# ---- the Python surface --------------------------------------------------------------------------
def _model_and_data(batch=2, steps=1, seed=5):
  task = graphcast.TASK_13_PRECIP_OUT
  inputs, template, forcings = synthetic.make_example(task, 10.0, batch=batch,
                                                      num_target_steps=steps, seed=seed)
  rng = np.random.default_rng(seed)
  targets = xs.Dataset(coords=template.coords)
  for name, v in template.data_vars.items():
    targets[name] = xs.DataArray(rng.standard_normal(v.shape).astype(np.float32), v.dims)
  cfg = graphcast.ModelConfig(10.0, 2, 512, 2, 1, 0.6)
  params = oracle_gnn.init_params(c_in=synthetic.num_input_channels(task), n_out=83, msg_steps=2,
                                  seed=4, randomize_affine=True)
  return task, graphcast.GraphCast(cfg, task, params=params), inputs, targets, forcings


def _rel(a, b):
  a, b = np.asarray(a.values, np.float64), np.asarray(b.values, np.float64)
  return float(np.max(np.abs(a - b) / np.abs(b)))


def _assert_loss_close(got, want, tol):
  (gl, gd), (wl, wd) = got, want
  assert gl.dims == ("batch",) and gl.values.dtype == np.float32
  assert _rel(gl, wl) <= tol
  assert set(gd.keys()) == set(wd.keys())
  for name in wd.keys():
    assert _rel(gd.data_vars[name], wd.data_vars[name]) <= tol, name


def _stats(task, seed=0):
  rng = np.random.default_rng(seed)
  levels = np.asarray(task.pressure_levels)

  def stats(lo, hi):
    ds = xs.Dataset(coords={"level": levels})
    # sorted: the draws go to the same variables in every process (set order follows string hashing)
    for name in sorted(set(task.input_variables) | set(task.target_variables) | set(task.forcing_variables)):
      if name in graphcast.variables.ALL_ATMOSPHERIC_VARS:
        ds[name] = xs.DataArray(rng.uniform(lo, hi, len(levels)).astype(np.float32), ("level",))
      else:
        ds[name] = xs.DataArray(np.float32(rng.uniform(lo, hi)), ())
    return ds
  return stats(0.5, 2.0), stats(-1.0, 1.0), stats(0.5, 2.0)


class _HostLoss(graphcast.Predictor):
  """Hides the GraphCast type: predictions from the device, the loss from the host mirror."""

  def __init__(self, model):
    self._model = model

  def __call__(self, inputs, targets_template, forcings, **kw):
    out = self._model(inputs, targets_template, forcings)
    return xs.Dataset({k: xs.DataArray(v.values, v.dims) for k, v in out.data_vars.items()}, out.coords)

  def loss_and_predictions(self, inputs, targets, forcings, **kw):
    predictions = self(inputs, targets, forcings)
    return losses.weighted_mse_per_level(predictions, targets,
                                         per_variable_weights=graphcast.LOSS_PER_VARIABLE_WEIGHTS), predictions

  def loss(self, inputs, targets, forcings, **kw):
    return self.loss_and_predictions(inputs, targets, forcings)[0]


def test_graphcast_loss_and_predictions():
  task, model, inputs, targets, forcings = _model_and_data()
  (loss, diag), pred = model.loss_and_predictions(inputs, targets, forcings)
  plain = model(inputs, targets, forcings)
  for name in targets.keys():
    assert torch.equal(pred.data_vars[name].data, plain.data_vars[name].data), name
  want = losses.weighted_mse_per_level(pred, targets,
                                       per_variable_weights=graphcast.LOSS_PER_VARIABLE_WEIGHTS)
  _assert_loss_close((loss, diag), want, 1e-6)
  loss2, diag2 = model.loss(inputs, targets, forcings)
  assert np.array_equal(loss2.values, loss.values)
  # a weight for a variable the targets lack is refused (reference losses.py:146-149)
  few = xs.Dataset({k: targets.data_vars[k] for k in targets.keys() if k != "2m_temperature"},
                   targets.coords)
  with pytest.raises(ValueError, match="does not correspond"):
    losses.sum_per_variable_losses(diag, {"2m_temperature": 1.0, "nope": 1.0})
  with pytest.raises(ValueError, match="Expected 82 channels"):   # targets must match the outputs
    model.loss(inputs, few, forcings)


def test_fused_inputs_and_residuals_loss_matches_generic_path():
  task, model, inputs, targets, forcings = _model_and_data(batch=1)
  std, mean, dstd = _stats(task)
  fused = normalization.InputsAndResiduals(model, std, mean, dstd)
  generic = normalization.InputsAndResiduals(_HostLoss(model), std, mean, dstd)
  (fl, fd), fpred = fused.loss_and_predictions(inputs, targets, forcings)
  (gl, gd), gpred = generic.loss_and_predictions(inputs, targets, forcings)
  _assert_loss_close((fl, fd), (gl, gd), 1e-5)
  _assert_loss_close(fused.loss(inputs, targets, forcings), (gl, gd), 1e-5)
  call = fused(inputs, targets, forcings)
  for name in targets.keys():
    assert torch.equal(fpred.data_vars[name].data, call.data_vars[name].data), name
    np.testing.assert_allclose(fpred.data_vars[name].values, gpred.data_vars[name].values,
                               rtol=2e-4, atol=2e-4)


def test_autoregressive_loss_is_the_mean_of_the_rollout_step_losses():
  task, model, inputs, targets, forcings = _model_and_data(batch=2, steps=3)
  ar = autoregressive.Predictor(model)
  loss, diag = ar.loss(inputs, targets, forcings)
  fn = lambda rng, inputs, targets_template, forcings: model(inputs, targets_template, forcings)
  steps = []
  for k, chunk in enumerate(rollout.chunked_prediction_generator(fn, None, inputs, targets, 1, forcings)):
    t_k = targets.isel(time=slice(k, k + 1))
    steps.append(losses.weighted_mse_per_level(
        chunk, t_k, per_variable_weights=graphcast.LOSS_PER_VARIABLE_WEIGHTS))
  mean = lambda arrays: np.mean([np.asarray(a.values, np.float64) for a in arrays], axis=0)
  assert np.max(np.abs(loss.values - mean([l for l, _ in steps])) / mean([l for l, _ in steps])) <= 1e-6
  for name in diag.keys():
    want = mean([d.data_vars[name] for _, d in steps])
    assert np.max(np.abs(diag.data_vars[name].values - want) / want) <= 1e-6, name
  # one target time: the inner loss itself
  one = lambda ds: ds.isel(time=slice(0, 1))
  l1, _ = ar.loss(inputs, one(targets), one(forcings))
  l1_inner, _ = model.loss(inputs, one(targets), one(forcings))
  assert np.array_equal(l1.values, l1_inner.values)


def test_demo_wrapper_stack_loss():
  """autoregressive.Predictor(InputsAndResiduals(Bfloat16Cast(GraphCast))).loss, as the reference
  demo calls it: the fused device path equals the generic path (host losses) on the same model."""
  task, model, inputs, targets, forcings = _model_and_data(batch=1, steps=2)
  std, mean, dstd = _stats(task, seed=1)
  cast = casting.Bfloat16Cast(model)
  assert cast is model and model._precision == "bf16"
  demo = autoregressive.Predictor(normalization.InputsAndResiduals(cast, std, mean, dstd))
  loss, diag = demo.loss(inputs, targets, forcings)
  assert loss.dims == ("batch",) and loss.shape == (1,) and np.isfinite(loss.values).all()
  generic = autoregressive.Predictor(normalization.InputsAndResiduals(
      casting.Bfloat16Cast(_HostLoss(model)), std, mean, dstd))
  _assert_loss_close((loss, diag), generic.loss(inputs, targets, forcings), 1e-5)


# ---- full size ----------------------------------------------------------------------------------
def test_full_size_loss_matches_host_mirror():
  if torch.cuda.get_device_properties(0).total_memory < 75e9:
    pytest.skip("needs an 80 GB GPU")
  task = graphcast.TASK
  lat, lon = synthetic.grid_coords(0.25)
  g = graph_lib.cached_static_graph(grid_lat=lat, grid_lon=lon, mesh_size=6,
                                    radius_query_fraction_edge_length=0.6)
  c_in = synthetic.num_input_channels(task)
  params = graphcast.init_params(graphcast.ModelConfig(0.25, 6, 512, 16, 1, 0.6), task, c_in, seed=1)
  n_out = graphcast.num_outputs(task)
  eng = engine.Engine(g, params, c_in=c_in, n_out=n_out, msg_steps=16, precision="bf16x3")
  gen = torch.Generator(device=DEV).manual_seed(0)
  planes = torch.randn(c_in, g.num_grid_nodes, device=DEV, generator=gen)
  targets = torch.randn(n_out, g.num_grid_nodes, device=DEV, generator=gen)
  eng.pack_inputs(planes)
  eng.step()
  w = _lat_weight(lat)
  assert w[0] > 0 and w[-1] > 0 and w[0] == w[-1]           # both pole rows carry weight
  sums = torch.empty(1, n_out, dtype=torch.float64, device=DEV)
  pred = torch.empty(n_out, g.num_grid_nodes, device=DEV)
  eng.output_loss(targets, torch.as_tensor(w).to(DEV), channel_sums=sums[0], planes_out=pred)
  # Datasets of the TASK targets from the channel planes
  coords = {"lat": lat, "lon": lon, "level": np.asarray(task.pressure_levels, np.int32),
            "time": np.array([np.timedelta64(6, "h")])}
  template = xs.Dataset(coords=coords)
  for name in task.target_variables:
    dims = synthetic._var_dims(name, True)
    shape = [1 if d in ("batch", "time") else len(coords[d]) for d in dims]
    template[name] = xs.DataArray(np.broadcast_to(np.float32(0), shape), dims)
  slabs = model_utils.channel_layout(template)

  def to_ds(p):
    host = p.cpu().numpy()
    out = xs.Dataset(coords=coords)
    for s in slabs:
      piece = host[s.start:s.start + s.count].reshape((1,) + s.stack_sizes + (len(lat), len(lon)))
      out[s.name] = xs.DataArray(piece, ("batch",) + s.stack_dims + ("lat", "lon")).transpose(*s.var_dims)
    return out
  got = losses.losses_from_channel_sums(sums.cpu().numpy(), slabs, g.num_grid_nodes,
                                        graphcast.LOSS_PER_VARIABLE_WEIGHTS)
  want = losses.weighted_mse_per_level(to_ds(pred), to_ds(targets),
                                       per_variable_weights=graphcast.LOSS_PER_VARIABLE_WEIGHTS)
  _assert_loss_close(got, want, 1e-6)
  assert torch.equal(pred, eng.grid_out[:, :n_out].t())
