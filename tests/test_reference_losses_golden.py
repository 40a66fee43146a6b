"""graphcast_b200.losses, the GraphCast loss weights, InputsAndResiduals.loss (generic path) and
autoregressive.Predictor.loss against the reference executed on numpy stand-ins
(tests/golden/make_golden_losses.py -> reference_losses.npz): utils/losses.py, GraphCast.loss_and_predictions,
normalization.InputsAndResiduals.loss / loss_and_predictions and autoregressive.Predictor.loss."""
import os

import numpy as np
import pytest

from graphcast_b200 import autoregressive, graphcast, losses, model_utils, normalization
from graphcast_b200 import xarray_shim as xs

Z = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_losses.npz"))
LEVELS = Z["levels"]
LON = np.arange(8) * 45.0
HOUR = np.timedelta64(6, "h")


def _names(prefix):
  return sorted(k[len(prefix) + 1:] for k in Z.files if k.startswith(prefix + ":"))


def _ds(prefix, lat, time=None):
  coords = {"lat": lat, "lon": LON, "level": LEVELS}
  if time is not None:
    coords["time"] = np.asarray(time) * HOUR
  return xs.Dataset({k: xs.DataArray(Z[f"{prefix}:{k}"], tuple(Z[f"{prefix}_dims:{k}"]))
                     for k in _names(prefix)}, coords)


def _close(got, want, rtol):
  got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
  assert got.shape == want.shape
  assert np.array_equal(np.isnan(got), np.isnan(want))
  ok = ~np.isnan(want)
  np.testing.assert_allclose(got[ok], want[ok], rtol=rtol, atol=0)


def _check(prefix, loss_and_diag, rtol=1e-6):
  total, per_var = loss_and_diag
  assert total.dims == ("batch",) and np.asarray(total.values).dtype == np.float32
  _close(total.values, Z[f"{prefix}:total"], rtol)
  assert sorted(per_var.keys()) == _names(f"{prefix}:var")
  for k in per_var.keys():
    _close(per_var.data_vars[k].values, Z[f"{prefix}:var:{k}"], rtol)


@pytest.mark.parametrize("grid", ["poles", "nopoles"])
def test_weighted_losses_match_reference(grid):
  lat = Z[f"{grid}:lat"]
  pred, tgt = _ds(f"{grid}:pred", lat), _ds(f"{grid}:tgt", lat)
  w = {"2m_temperature": 1.0, "total_precipitation_6hr": 0.1}
  _check(f"{grid}:mse", losses.weighted_mse_per_level(pred, tgt, per_variable_weights=w))
  _check(f"{grid}:mae", losses.weighted_mae_per_level(pred, tgt))
  _check(f"{grid}:mse_nan", losses.weighted_mse_per_level(
      pred, tgt, per_variable_weights=w, vars_with_nan_targets=("total_precipitation_6hr",),
      loss_for_nan_targets=0.5))
  assert np.isnan(Z[f"{grid}:mse:total"][1])                 # the NaN target propagates


@pytest.mark.parametrize("grid", ["poles", "nopoles"])
def test_latitude_and_level_weights_match_reference(grid):
  lat = Z[f"{grid}:lat"]
  tgt = _ds(f"{grid}:tgt", lat)
  np.testing.assert_allclose(losses.normalized_latitude_weights(tgt["geopotential"]),
                             Z[f"{grid}:lat_weights"], rtol=1e-7, atol=0)
  np.testing.assert_allclose(losses.normalized_level_weights(tgt["geopotential"]),
                             Z[f"{grid}:level_weights"], rtol=1e-7, atol=0)


def test_latitude_weight_errors_match_reference():
  for name in ("nonuniform", "no_pole_wrong_ends", "one_pole"):
    lat = Z[f"bad_lat:{name}"]
    da = xs.DataArray(np.zeros(len(lat), np.float32), ("lat",), coords={"lat": lat})
    assert bool(Z[f"bad_lat_raises:{name}"])
    with pytest.raises(ValueError):
      losses.normalized_latitude_weights(da)
  assert bool(Z["unknown_weight_raises"])
  with pytest.raises(ValueError, match="does not correspond to any variable"):
    losses.sum_per_variable_losses(xs.Dataset({"a": xs.DataArray(np.ones(2), ("batch",))}), {"b": 1.0})


def test_graphcast_loss_weights_and_channel_sum_path_match_reference():
  lat = Z["poles:lat"]
  pred, tgt = _ds("gc:pred", lat), _ds("gc:tgt", lat)
  w = graphcast.LOSS_PER_VARIABLE_WEIGHTS
  _check("gc", losses.weighted_mse_per_level(pred, tgt, per_variable_weights=w))
  _check("gc_loss", losses.weighted_mse_per_level(pred, tgt, per_variable_weights=w))
  # The GraphCast path forms the same losses from per-channel sums (what gcb_output_loss returns):
  # here the sums are taken on the host in fp64 from the same data.
  slabs = model_utils.channel_layout(tgt)
  lw = losses.normalized_latitude_weights(tgt["geopotential"]).astype(np.float32).astype(np.float64)
  b = tgt.sizes["batch"]
  sums = np.zeros([b, sum(s.count for s in slabs)])
  for s in slabs:
    d = (np.asarray(pred.data_vars[s.name].values) - np.asarray(tgt.data_vars[s.name].values))
    d2 = d.astype(np.float64) ** 2 * lw[:, None]
    sums[:, s.start:s.start + s.count] = d2.reshape(b, s.count, -1).sum(-1)
  _check("gc", losses.losses_from_channel_sums(sums, slabs, len(lat) * len(LON), w))
  assert bool(Z["gc:missing_weighted_var_raises"])
  few = xs.Dataset({k: tgt.data_vars[k] for k in tgt.keys() if k != "mean_sea_level_pressure"}, tgt.coords)
  with pytest.raises(ValueError):
    losses.weighted_mse_per_level(few, few, per_variable_weights=w)


class _Recording(graphcast.Predictor):
  """The golden's recording predictor: predictions a fixed function of the normalised inputs, the
  loss the MSE against the (normalised) targets it is given."""

  def __init__(self):
    self.seen = []

  def __call__(self, inputs, targets_template, forcings, **kw):
    raise AssertionError("not used by the loss")

  def loss_and_predictions(self, inputs, targets, forcings, **kw):
    self.seen.append(targets)
    out = xs.Dataset(coords=targets.coords)
    for name in sorted(targets.keys()):
      t = targets[name]
      if name in inputs:
        x = inputs[name]                                     # (batch, time, [level], lat, lon)
        out[name] = xs.DataArray(0.5 * np.asarray(x.values)[:, -1:] + 0.25, x.dims)
      else:
        out[name] = xs.DataArray(np.full(t.shape, 0.125, np.float32), t.dims)
    return losses.weighted_mse_per_level(out, targets), out

  def loss(self, inputs, targets, forcings, **kw):
    return self.loss_and_predictions(inputs, targets, forcings)[0]


def _stats(name):
  ds = xs.Dataset(coords={"level": LEVELS})
  for k in _names(f"iar:{name}"):
    v = Z[f"iar:{name}:{k}"]
    ds[k] = xs.DataArray(v, ("level",) if v.ndim else ())
  return ds


def test_inputs_and_residuals_loss_matches_reference():
  lat = Z["poles:lat"]
  inner = _Recording()
  iar = normalization.InputsAndResiduals(inner, _stats("std"), _stats("mean"), _stats("diffs_std"))
  inputs, forcings = _ds("iar:in", lat, [-1, 0]), _ds("iar:forcing", lat, [1])
  targets = _ds("iar:tgt", lat, [1])
  _check("iar_loss", iar.loss(inputs, targets, forcings))
  (loss, diag), pred = iar.loss_and_predictions(inputs, targets, forcings)
  _check("iar", (loss, diag))
  for k in targets.keys():
    np.testing.assert_allclose(inner.seen[-1].data_vars[k].transpose(*targets.data_vars[k].dims).values,
                               Z[f"iar:norm_target:{k}"], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(pred.data_vars[k].transpose(*targets.data_vars[k].dims).values,
                               Z[f"iar:pred:{k}"], rtol=1e-6, atol=1e-6)


class _Feedback(graphcast.Predictor):
  """The golden's feedback predictor: both input frames, the step's forcing and a constant input."""

  def __call__(self, inputs, targets_template, forcings, **kw):
    raise AssertionError("not used by the loss")

  def loss_and_predictions(self, inputs, targets, forcings, **kw):
    f = np.asarray(forcings["toa_incident_solar_radiation"].transpose("batch", "time", "lat", "lon").values)
    out = xs.Dataset(coords=targets.coords)
    for name in sorted(targets.keys()):
      dims = inputs[name].dims                               # (batch, time, [level], lat, lon)
      x = np.asarray(inputs[name].values)
      fb = f.reshape(f.shape[:2] + (1,) * (x.ndim - 4) + f.shape[2:])
      lsm = np.asarray(inputs["land_sea_mask"].values)
      out[name] = xs.DataArray(0.9 * x[:, 1:] + 0.1 * x[:, :1] + 0.05 * fb + 0.01 * lsm, dims)
    return losses.weighted_mse_per_level(out, targets, per_variable_weights={"2m_temperature": 0.5}), out

  def loss(self, inputs, targets, forcings, **kw):
    return self.loss_and_predictions(inputs, targets, forcings)[0]


def test_autoregressive_loss_matches_reference():
  lat = Z["poles:lat"]
  ar = autoregressive.Predictor(_Feedback())
  inputs = _ds("ar:in", lat, [-1, 0])
  targets, forcings = _ds("ar:tgt", lat, [1, 2, 3]), _ds("ar:forcing", lat, [1, 2, 3])
  _check("ar3", ar.loss(inputs, targets, forcings))
  one = lambda ds: ds.isel(time=slice(0, 1))
  _check("ar1", ar.loss(inputs, one(targets), one(forcings)))
