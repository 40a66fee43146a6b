"""Forecast losses -- host mirror of `weathernext/utils/losses.py` on `xarray_shim` Datasets.

Public surface kept: `weighted_mse_per_level`, `weighted_mae_per_level`, `weighted_loss_per_level`
(:67-128, incl. `vars_with_nan_targets` / `loss_for_nan_targets`), `sum_per_variable_losses`
(:135-158), `normalized_level_weights` (:161-164), `normalized_latitude_weights` (:167-243), with the
reference's errors.  A loss is a `(batch,)` DataArray, the diagnostics a Dataset of the per-variable
`(batch,)` losses.

Semantics: per variable, l = loss_fn(prediction, target) * latitude weight * level weight (the
level weight only for variables with a `level` dim), both weights cast to the data's dtype and
normalised to mean 1; l is averaged over every dim except `batch` with NaNs propagating
(skipna=False), and the total is the weighted sum of the per-variable losses (default weight 1).
The element-wise terms are evaluated in the data's dtype (float32) as in the reference; the means
and the weighted sum are accumulated in float64 and returned as float32.

This module runs on the host.  It scores predictors that are not this package's `GraphCast` and is
the CPU-side check of the fused device loss (`gcb_output_loss`), whose per-channel sums are turned
into the same per-variable losses by `losses_from_channel_sums`.
"""

from __future__ import annotations

import logging
from typing import Callable, Mapping, Optional, Sequence, Tuple

import numpy as np

from graphcast_b200 import xarray_shim as xs

LossAndDiagnostics = Tuple[xs.DataArray, xs.Dataset]

DEFAULT_PER_VARIABLE_WEIGHT = 1.0


def _abs_diff(prediction, target):
  return np.abs(prediction - target)


def _squared_diff(prediction, target):
  return (prediction - target) ** 2


def weighted_mae_per_level(*args, **kwargs) -> LossAndDiagnostics:
  """Latitude- and pressure-level-weighted MAE loss."""
  return weighted_loss_per_level(*args, loss_fn=_abs_diff, **kwargs)


def weighted_mse_per_level(*args, **kwargs) -> LossAndDiagnostics:
  """Latitude- and pressure-level-weighted MSE loss."""
  return weighted_loss_per_level(*args, loss_fn=_squared_diff, **kwargs)


def _coord(da: xs.DataArray, name: str) -> np.ndarray:
  if name not in da.coords:
    raise KeyError(name)
  return np.asarray(da.coords[name][1])


def _along(weights: np.ndarray, dim: str, dims: Sequence[str]) -> np.ndarray:
  """1-d `weights` shaped to broadcast along `dim` of an array with `dims`."""
  shape = [1] * len(dims)
  shape[list(dims).index(dim)] = weights.shape[0]
  return weights.reshape(shape)


def _mean_preserving_batch(x: np.ndarray, dims: Sequence[str]) -> xs.DataArray:
  axes = tuple(i for i, d in enumerate(dims) if d != "batch")
  out = np.mean(x.astype(np.float64), axis=axes) if axes else x.astype(np.float64)
  return xs.DataArray(out.astype(np.float32), tuple(d for d in dims if d == "batch"))


def weighted_loss_per_level(
    predictions, targets, loss_fn: Callable[..., np.ndarray],
    per_variable_weights: Optional[Mapping[str, float]] = None,
    vars_with_nan_targets: Sequence[str] = (),
    loss_for_nan_targets: float = 0.0) -> LossAndDiagnostics:
  """Latitude- and pressure-level-weighted loss, parameterised by `loss_fn(prediction=, target=)`."""
  predictions, targets = xs.from_xarray(predictions), xs.from_xarray(targets)
  per_variable = xs.Dataset()
  for name in predictions.keys():
    target = targets[name]
    dims = target.dims
    t = np.asarray(target.values)
    p = np.asarray(predictions[name].transpose(*dims).values)
    mask = None
    if name in vars_with_nan_targets:
      mask = ~np.isnan(t)
      t = np.where(mask, t, np.array(0.0, dtype=t.dtype))
    l = loss_fn(prediction=p, target=t)
    l = l * _along(normalized_latitude_weights(target).astype(l.dtype), "lat", dims)
    if "level" in dims:
      l = l * _along(normalized_level_weights(target).astype(l.dtype), "level", dims)
    if mask is not None:
      l = np.where(mask, l, np.array(loss_for_nan_targets, dtype=l.dtype))
    per_variable[name] = _mean_preserving_batch(l, dims)
  return sum_per_variable_losses(per_variable, per_variable_weights or {})


def sum_per_variable_losses(per_variable_losses: xs.Dataset,
                            weights: Optional[Mapping[str, float]] = None) -> LossAndDiagnostics:
  """Optionally-weighted sum of per-variable losses; NaNs propagate."""
  if weights is None:
    weights = {}
  if weights:
    logging.info("Weighting variables in loss as %s (any others weighted as 1)", weights)
  if not set(weights.keys()).issubset(set(per_variable_losses.keys())):
    raise ValueError("Passing a weight that does not correspond to any variable "
                     f"{set(weights.keys()) - set(per_variable_losses.keys())}")
  total, dims = None, None
  for name in per_variable_losses.keys():
    v = per_variable_losses.data_vars[name]
    if dims is not None and v.dims != dims:
      raise ValueError(f"per-variable losses have different dims: {dims} vs {v.dims}")
    dims = v.dims
    term = np.asarray(v.values, np.float64) * weights.get(name, DEFAULT_PER_VARIABLE_WEIGHT)
    total = term if total is None else total + term
  if total is None:
    raise ValueError("no per-variable losses to sum")
  return xs.DataArray(total.astype(np.float32), dims), per_variable_losses


def normalized_level_weights(data: xs.DataArray) -> np.ndarray:
  """Weights proportional to the pressure of each level, mean 1 (float64, along `level`)."""
  level = _coord(data, "level")
  return level / level.mean()


def normalized_latitude_weights(data: xs.DataArray) -> np.ndarray:
  """Weights roughly proportional to the area of each latitude row, mean 1 (along `lat`).

  Two equispaced grids are supported: with rows at the poles (pole rows get sin^2(d/4), the others
  cos(lat) sin(d/2): the area of their bands) and without (rows at +-(90 - d/2), weight cos(lat)).
  Anything else raises ValueError.  Computed in the dtype of the `lat` coordinate."""
  latitude = _coord(data, "lat")
  if np.any(np.isclose(np.abs(latitude), 90.)):
    weights = _weight_for_latitude_vector_with_poles(latitude)
  else:
    weights = _weight_for_latitude_vector_without_poles(latitude)
  return weights / weights.mean()


def _weight_for_latitude_vector_without_poles(latitude: np.ndarray) -> np.ndarray:
  delta = np.abs(_check_uniform_spacing_and_get_delta(latitude))
  if (not np.isclose(np.max(latitude), 90 - delta / 2)
      or not np.isclose(np.min(latitude), -90 + delta / 2)):
    raise ValueError(f"Latitude vector {latitude} does not start/end at "
                     "+- (90 - delta_latitude/2) degrees.")
  return np.cos(np.deg2rad(latitude))


def _weight_for_latitude_vector_with_poles(latitude: np.ndarray) -> np.ndarray:
  delta = np.abs(_check_uniform_spacing_and_get_delta(latitude))
  if not np.isclose(np.max(latitude), 90.) or not np.isclose(np.min(latitude), -90.):
    raise ValueError(f"Latitude vector {latitude} does not start/end at +- 90 degrees.")
  weights = np.cos(np.deg2rad(latitude)) * np.sin(np.deg2rad(delta / 2))
  # uniform spacing and both poles present: the first and last rows are the poles
  weights[[0, -1]] = np.sin(np.deg2rad(delta / 4)) ** 2
  return weights


def _check_uniform_spacing_and_get_delta(vector: np.ndarray):
  diff = np.diff(vector)
  if not np.all(np.isclose(diff[0], diff)):
    raise ValueError(f"Vector {diff} is not uniformly spaced.")
  return diff[0]


def channel_level_weights(slab, dtype=np.float32) -> np.ndarray:
  """[slab.count] level weight of every channel of a packed variable (1 without a `level` dim),
  cast to `dtype` as the per-element loss does (model_utils.channel_layout order)."""
  if "level" not in slab.stack_dims:
    return np.ones([slab.count], np.float64)
  if "level" not in slab.stack_labels:
    raise KeyError("level")
  level = np.asarray(slab.stack_labels["level"])
  w = (level / level.mean()).astype(dtype).astype(np.float64)
  shape = [1] * len(slab.stack_dims)
  shape[slab.stack_dims.index("level")] = w.shape[0]
  return np.broadcast_to(w.reshape(shape), slab.stack_sizes).reshape(-1)


def losses_from_channel_sums(channel_sums: np.ndarray, slabs, num_nodes: int,
                             per_variable_weights: Optional[Mapping[str, float]] = None
                             ) -> LossAndDiagnostics:
  """(total, per-variable losses) from the [batch, channels] latitude-weighted squared-error sums of
  `gcb_output_loss`: per variable, sum over its channels of level weight * sum, divided by
  (channels x nodes) -- the mean of `weighted_mse_per_level` -- then `sum_per_variable_losses`."""
  sums = np.asarray(channel_sums, np.float64)
  per_variable = xs.Dataset()
  for s in slabs:
    w = channel_level_weights(s)
    loss = (sums[:, s.start:s.start + s.count] * w).sum(axis=1) / (float(s.count) * num_nodes)
    per_variable[s.name] = xs.DataArray(loss.astype(np.float32), ("batch",))
  return sum_per_variable_losses(per_variable, per_variable_weights or {})
