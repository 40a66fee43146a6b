"""Input normalisation / residual un-normalisation wrapper -- mirror of
`weathernext/utils/normalization.py` (`normalize` :29-48, `unnormalize` :51-70,
`InputsAndResiduals` :73-160).

Semantics kept:
  model input      = (x - mean) / std                 for every input / forcing
  prediction       = y * diffs_std + last input frame for targets present in inputs
  prediction       = y * std + mean                   for targets not in inputs
  only single-step targets are supported (ValueError otherwise, :114-117).

When the wrapped predictor is this package's `GraphCast`, the affine maps are not
applied to the Datasets at all: they are folded into per-channel vectors and
executed inside the pack / unpack kernels (`gcb_pack_grid_features`,
`gcb_unpack_grid_outputs`), which removes three full passes over the 0.25 degree
state per step.  Any other predictor gets the generic Dataset arithmetic.

`loss` / `loss_and_predictions` (reference :134-146, :162-196) score the inner predictor in normalised
space: targets that are also inputs become (target - last input frame) / diffs_std, the others
(target - mean) / std, and the inner predictor's raw output is compared with them;
`loss_and_predictions` returns un-normalised predictions.  Around `GraphCast` the same per-channel
vectors normalise the targets inside the loss kernel (`gcb_output_loss`), so the normalised targets
are never built as Datasets.
"""

from __future__ import annotations

import logging
from typing import Optional

import numpy as np
import torch

from graphcast_b200 import graphcast
from graphcast_b200 import model_utils
from graphcast_b200 import xarray_shim as xs


def normalize(values: xs.Dataset, scales: xs.Dataset, locations: Optional[xs.Dataset]
              ) -> xs.Dataset:
  def one(array: xs.DataArray) -> xs.DataArray:
    if array.name is None:
      raise ValueError("Can't look up normalization constants because array has no name.")
    if locations is not None:
      if array.name in locations:
        array = array - locations[array.name].astype(array.dtype)
      else:
        logging.warning("No normalization location found for %s", array.name)
    if array.name in scales:
      array = array / scales[array.name].astype(array.dtype)
    else:
      logging.warning("No normalization scale found for %s", array.name)
    return array
  return values.map(one)


def unnormalize(values: xs.Dataset, scales: xs.Dataset, locations: Optional[xs.Dataset]
                ) -> xs.Dataset:
  def one(array: xs.DataArray) -> xs.DataArray:
    if array.name is None:
      raise ValueError("Can't look up normalization constants because array has no name.")
    if array.name in scales:
      array = array * scales[array.name].astype(array.dtype)
    else:
      logging.warning("No normalization scale found for %s", array.name)
    if locations is not None:
      if array.name in locations:
        array = array + locations[array.name].astype(array.dtype)
      else:
        logging.warning("No normalization location found for %s", array.name)
    return array
  return values.map(one)


_warned_missing = set()


def _warn_missing_once(kind: str, name: str) -> None:
  if (kind, name) not in _warned_missing:
    _warned_missing.add((kind, name))
    logging.warning("No normalization %s found for %s", kind, name)


def _per_channel(slab: model_utils.ChannelSlab, stats: Optional[xs.Dataset], default: float,
                 kind: str = "scale") -> np.ndarray:
  """Per-channel constant of one variable: stats[var] may be a scalar or vary
  along stacked dims (e.g. "level"); it is broadcast over the slab's stack dims.

  Statistics are selected by LABEL along every labelled dim they share with the variable
  (xarray's alignment, which the reference relies on: the released 37-level `*_by_level`
  files serve 13-level models); a label of the variable that the statistics lack raises.
  A variable without statistics keeps `default` and logs the reference's warning once."""
  out = np.full(slab.stack_sizes if slab.stack_sizes else (1,), default, np.float64)
  if stats is None:
    return out.reshape(-1)
  if slab.name not in stats:
    _warn_missing_once(kind, slab.name)
    return out.reshape(-1)
  v = stats[slab.name]                # with the statistics' coordinates attached
  bad = [d for d in v.dims if d not in slab.stack_dims]
  if bad:
    raise ValueError(f"normalisation statistics of {slab.name!r} vary along {bad}, "
                     "which is not a channel dimension")
  for d in v.dims:
    want, have = slab.stack_labels.get(d), v.index_labels(d)
    size = slab.stack_sizes[slab.stack_dims.index(d)]
    if want is not None and have is not None:
      pos = {x.item(): i for i, x in enumerate(have)}
      missing = [x.item() for x in want if x.item() not in pos]
      if missing:
        raise ValueError(f"normalisation statistics of {slab.name!r} lack {d} = {missing}")
      v = v.isel({d: np.asarray([pos[x.item()] for x in want], np.int64)})
    elif v.sizes[d] != size:
      raise ValueError(f"normalisation statistics of {slab.name!r} have {v.sizes[d]} entries "
                       f"along {d!r}, the data {size}, and no labels to align them by")
  arr = np.asarray(v.values, np.float64)
  shape = [v.sizes[d] if d in v.dims else 1 for d in slab.stack_dims] or [1]
  arr = np.transpose(arr, [v.dims.index(d) for d in slab.stack_dims if d in v.dims]) \
      if v.dims else arr
  out = out * 0 + arr.reshape(shape)
  return out.reshape(-1)


class InputsAndResiduals(graphcast.Predictor):
  """Normalises inputs and predicts normalised residuals (reference :73-160)."""

  def __init__(self, predictor: graphcast.Predictor, stddev_by_level: xs.Dataset,
               mean_by_level: xs.Dataset, diffs_stddev_by_level: xs.Dataset):
    self._predictor = predictor
    self._scales = xs.from_xarray(stddev_by_level)
    self._locations = xs.from_xarray(mean_by_level)
    self._residual_scales = xs.from_xarray(diffs_stddev_by_level)
    self._residual_locations = None
    self._fused_cache = None

  def _unnormalize_prediction_and_add_input(self, inputs, norm_prediction):
    if norm_prediction.sizes.get("time") != 1:
      raise ValueError("normalization.InputsAndResiduals only supports predicting a "
                       "single timestep.")
    if norm_prediction.name in inputs:
      prediction = unnormalize(xs.Dataset({norm_prediction.name: norm_prediction}),
                               self._residual_scales, self._residual_locations
                               )[norm_prediction.name]
      # isel(time=-1) drops the time dim (reference :128-129), so the add broadcasts over the
      # prediction's single time step instead of aligning two different time labels.
      last_input = inputs[norm_prediction.name].isel(time=-1)
      return prediction + last_input
    return unnormalize(xs.Dataset({norm_prediction.name: norm_prediction}),
                       self._scales, self._locations)[norm_prediction.name]

  # -- fused path --------------------------------------------------------------------
  def _fused_constants(self, inputs, targets_template, forcings, device):
    in_slabs = model_utils.channel_layout(inputs)
    n_in = sum(s.count for s in in_slabs)
    f_slabs = model_utils.channel_layout(forcings, start=n_in)
    t_slabs = model_utils.channel_layout(targets_template)
    sig = lambda s: (s.name, s.stack_dims, s.stack_sizes,
                     tuple((d, v.tobytes()) for d, v in sorted(s.stack_labels.items())))
    key = (tuple(sig(s) for s in in_slabs + f_slabs), tuple(sig(s) for s in t_slabs), str(device))
    if self._fused_cache is not None and self._fused_cache[0] == key:
      return self._fused_cache[1]
    mean = np.concatenate([_per_channel(s, self._locations, 0.0, "location")
                           for s in in_slabs + f_slabs])
    scale = np.concatenate([_per_channel(s, self._scales, 1.0) for s in in_slabs + f_slabs])
    out_scale, out_offset, add_idx = [], [], []
    in_by_name = {s.name: s for s in in_slabs}
    for s in t_slabs:
      # reference :114-117: `norm_prediction.sizes.get("time") != 1` raises (also without a time dim)
      if "time" not in s.stack_dims or s.stack_sizes[s.stack_dims.index("time")] != 1:
        raise ValueError("normalization.InputsAndResiduals only supports predicting a "
                         "single timestep.")
      if s.name in in_by_name:
        src = in_by_name[s.name]
        # channel of the LAST input frame with the same non-time indices
        n_time = src.stack_sizes[src.stack_dims.index("time")] if "time" in src.stack_dims else 1
        per_frame = src.count // n_time
        if "time" in src.stack_dims and src.stack_dims[0] != "time":
          raise ValueError(f"{s.name}: time must be the leading stacked dim of the inputs")
        if per_frame != s.count:
          raise ValueError(f"{s.name}: target has {s.count} channels per frame, input {per_frame}")
        out_scale.append(_per_channel(s, self._residual_scales, 1.0))
        out_offset.append(np.zeros([s.count]))
        add_idx.append(src.start + (n_time - 1) * per_frame + np.arange(s.count))
      else:
        out_scale.append(_per_channel(s, self._scales, 1.0))
        out_offset.append(_per_channel(s, self._locations, 0.0, "location"))
        add_idx.append(np.full([s.count], -1))
    t = lambda a, dt: torch.as_tensor(np.concatenate(a) if isinstance(a, list) else a).to(dt).to(device)
    consts = graphcast.FusedNormalization(
        in_mean=t(mean, torch.float32), in_scale=t(scale, torch.float32),
        out_scale=t(out_scale, torch.float32), out_offset=t(out_offset, torch.float32),
        add_plane_index=t(add_idx, torch.int32))
    self._fused_cache = (key, consts)
    return consts

  def __call__(self, inputs, targets_template, forcings, **kwargs):
    inputs, forcings = xs.from_xarray(inputs), xs.from_xarray(forcings)
    targets_template = xs.from_xarray(targets_template)
    if isinstance(self._predictor, graphcast.GraphCast):
      consts = self._norm_of()(inputs, targets_template, forcings)
      return self._predictor._call(inputs, targets_template, forcings, norm=consts)
    norm_inputs = normalize(inputs, self._scales, self._locations)
    norm_forcings = normalize(forcings, self._scales, self._locations)
    norm_predictions = self._predictor(norm_inputs, targets_template, forcings=norm_forcings,
                                       **kwargs)
    return norm_predictions.map(
        lambda pred: self._unnormalize_prediction_and_add_input(inputs, pred))

  # -- the loss, in normalised space (reference :134-146, :162-196) -------------------
  def _subtract_input_and_normalize_target(self, inputs, target):
    if target.sizes.get("time") != 1:
      raise ValueError("normalization.InputsAndResiduals only supports wrapping predictors"
                       "that predict a single timestep.")
    if target.name in inputs:
      residual = target - inputs[target.name].isel(time=-1)
      return normalize(xs.Dataset({target.name: residual}), self._residual_scales,
                       self._residual_locations)[target.name]
    return normalize(xs.Dataset({target.name: target}), self._scales, self._locations)[target.name]

  def _normalized(self, inputs, targets, forcings):
    return (normalize(inputs, self._scales, self._locations),
            targets.map(lambda t: self._subtract_input_and_normalize_target(inputs, t)),
            normalize(forcings, self._scales, self._locations))

  def _fuses(self) -> bool:
    return isinstance(self._predictor, graphcast.GraphCast)

  def _norm_of(self, what: str = "fused calls"):
    """norm_of(inputs, targets, forcings) -> their FusedNormalization, its constants on the device the
    wrapped GraphCast runs on (GraphCast.compute_device).  A wrapped predictor that is not a GraphCast
    raises NotImplementedError here, `what` naming the call, so a call that refuses it before its
    other checks asks for norm_of first."""
    if not self._fuses():
      raise NotImplementedError(f"{what} need a GraphCast predictor directly inside "
                                "InputsAndResiduals (the fused normalisation)")
    return lambda inputs, targets, forcings: self._fused_constants(
        xs.from_xarray(inputs), xs.from_xarray(targets), xs.from_xarray(forcings),
        self._predictor.compute_device())

  def _device_loss(self, inputs, targets, forcings, predictions: bool):
    """GraphCast only: the step with the fused loss (graphcast.GraphCast._device_loss), the
    target normalisation applied inside the kernel from the fused constants."""
    norm = self._norm_of()(inputs, targets, forcings)
    return self._predictor._device_loss(inputs, targets, forcings, norm, predictions)

  def loss_and_grads(self, inputs, targets, forcings, **kwargs):
    """(loss, diagnostics, grads) of `loss` and its parameter gradients (GraphCast.loss_and_grads),
    with the normalisation fused into the kernels as in `loss`.  GraphCast only."""
    norm = self._norm_of("parameter gradients")(inputs, targets, forcings)
    return self._predictor._loss_and_grads(inputs, targets, forcings, norm=norm)

  def loss_and_input_grads(self, inputs, targets, forcings, **kwargs):
    """(loss, diagnostics, input_grads, forcing_grads) of `loss` (GraphCast.loss_and_input_grads):
    the gradients are in the physical units of the inputs and forcings, through the normalisation of
    the inputs, the residual add and the target normalisation.  GraphCast only."""
    norm = self._norm_of("input gradients")(inputs, targets, forcings)
    return self._predictor._loss_and_input_grads(inputs, targets, forcings, norm=norm)

  def loss_and_input_hvp(self, inputs, targets, forcings, input_tangents, forcing_tangents=None,
                         **kwargs):
    """loss_and_input_grads and the Hessian-vector product of its loss (GraphCast.loss_and_input_hvp),
    with respect to the inputs and forcings in their physical units.  GraphCast only."""
    norm = self._norm_of("input gradients")(inputs, targets, forcings)
    return self._predictor._loss_and_input_grads(inputs, targets, forcings, norm=norm,
                                                 tangents=(input_tangents, forcing_tangents))

  def batched_loss_and_input_hvp(self, inputs, targets, forcings, input_tangents, forcing_tangents=None,
                                 *, directions_per_pass=None, **kwargs):
    """loss_and_input_hvp along K tangent directions at once (GraphCast.batched_loss_and_input_hvp),
    with respect to the inputs and forcings in their physical units.  GraphCast only."""
    def one_pass(it, ft):
      norm = self._norm_of("input gradients")(inputs, targets, forcings)
      return self._predictor._loss_and_input_grads(inputs, targets, forcings, norm=norm,
                                                   tangents=(it, ft), directions=True)
    return graphcast.batched_hvp(one_pass, inputs, forcings, input_tangents, forcing_tangents,
                                 directions_per_pass)

  def input_vjp(self, inputs, targets_template, forcings, cotangents, **kwargs):
    """(predictions, input_grads, forcing_grads) of the un-normalised predictions of __call__
    (GraphCast.input_vjp).  GraphCast only."""
    norm = self._norm_of("input gradients")(inputs, targets_template, forcings)
    return self._predictor._input_vjp(inputs, targets_template, forcings, cotangents, norm=norm)

  def batched_input_vjp(self, inputs, targets_template, forcings, cotangents, *,
                        directions_per_pass=None, **kwargs):
    """input_vjp of K cotangents at once (GraphCast.batched_input_vjp), of the un-normalised
    predictions.  GraphCast only."""
    def one_pass(cot, first):
      norm = self._norm_of("input gradients")(inputs, targets_template, forcings)
      return self._predictor._input_vjp(inputs, targets_template, forcings, cot, norm=norm,
                                        directions=True, predictions=first)
    return graphcast.batched_vjp(one_pass, targets_template, cotangents, directions_per_pass)

  def input_jvp(self, inputs, targets_template, forcings, input_tangents, forcing_tangents=None,
                **kwargs):
    """(predictions, prediction_tangents) of the un-normalised predictions of __call__
    (GraphCast.input_jvp): the tangents are in physical units, through the normalisation of the inputs
    and the residual add.  GraphCast only."""
    run = graphcast.GraphCast._one_step_tangents(inputs, targets_template, forcings, input_tangents,
                                                 forcing_tangents)
    norm = self._norm_of("input gradients")(inputs, targets_template, forcings)
    return self._predictor._input_jvp(inputs, targets_template, forcings, run, norm=norm)

  def batched_input_jvp(self, inputs, targets_template, forcings, input_tangents,
                        forcing_tangents=None, *, directions_per_pass=None, **kwargs):
    """input_jvp along K tangent directions at once (GraphCast.batched_input_jvp), through the
    normalisation of the inputs and the residual add.  GraphCast only."""
    def one_pass(it, ft):
      run = graphcast.GraphCast._one_step_tangents(inputs, targets_template, forcings, it, ft,
                                                   directions=True)
      norm = self._norm_of("input gradients")(inputs, targets_template, forcings)
      return self._predictor._input_jvp(inputs, targets_template, forcings, run, norm=norm)
    return graphcast.batched_jvp(one_pass, inputs, forcings, input_tangents, forcing_tangents,
                                 directions_per_pass)

  def param_jvp(self, inputs, targets_template, forcings, param_tangents, **kwargs):
    """(predictions, prediction_tangents) of the un-normalised predictions of __call__ along
    param_tangents (GraphCast.param_jvp): the tangents are in physical units, through the
    un-normalisation of the outputs.  GraphCast only."""
    norm_of = self._norm_of("parameter gradients")
    run = self._predictor._param_tangent_run(inputs, targets_template, forcings, param_tangents,
                                             num_steps=1)
    return self._predictor._input_jvp(inputs, targets_template, forcings, run,
                                      norm=norm_of(inputs, targets_template, forcings))

  def loss_and_param_gnvp(self, inputs, targets, forcings, param_tangents, **kwargs):
    """(loss, diagnostics, gnvp) of `loss` (GraphCast.loss_and_param_gnvp), with the normalisation
    fused into the kernels as in `loss`.  GraphCast only."""
    norm_of = self._norm_of("parameter gradients")
    if xs.from_xarray(targets).sizes.get("time", 1) != 1:
      raise NotImplementedError("Gauss-Newton products cover one target time (several are not "
                                "provided)")
    self._predictor._checked_param_tangents(param_tangents)
    return self._predictor._loss_and_param_gnvp(inputs, targets, forcings, param_tangents,
                                                norm=norm_of(inputs, targets, forcings))

  def loss_and_param_hvp(self, inputs, targets, forcings, param_tangents, **kwargs):
    """(loss, diagnostics, grads, hvp) of `loss` (GraphCast.loss_and_param_hvp), with the
    normalisation fused into the kernels as in `loss`.  GraphCast only."""
    norm_of = self._norm_of("parameter gradients")
    if xs.from_xarray(targets).sizes.get("time", 1) != 1:
      raise NotImplementedError("parameter Hessian-vector products cover one target time (several "
                                "are not provided)")
    self._predictor._checked_param_tangents(param_tangents)
    return self._predictor._loss_and_param_hvp(inputs, targets, forcings, param_tangents,
                                               norm=norm_of(inputs, targets, forcings))

  def loss(self, inputs, targets, forcings, **kwargs):
    """The loss computed on normalised inputs and targets (targets that are also inputs as
    normalised residuals against the last input frame)."""
    if self._fuses():
      finish, _, sums = self._device_loss(inputs, targets, forcings, predictions=False)
      return finish(sums.cpu().numpy())
    inputs, forcings = xs.from_xarray(inputs), xs.from_xarray(forcings)
    norm_inputs, norm_targets, norm_forcings = self._normalized(inputs, xs.from_xarray(targets),
                                                                forcings)
    return self._predictor.loss(norm_inputs, norm_targets, forcings=norm_forcings, **kwargs)

  def loss_and_predictions(self, inputs, targets, forcings, **kwargs):
    """The loss computed on normalised data, with un-normalised predictions."""
    if self._fuses():
      finish, predictions, sums = self._device_loss(inputs, targets, forcings, predictions=True)
      return finish(sums.cpu().numpy()), predictions
    inputs, forcings = xs.from_xarray(inputs), xs.from_xarray(forcings)
    norm_inputs, norm_targets, norm_forcings = self._normalized(inputs, xs.from_xarray(targets),
                                                                forcings)
    (loss, diagnostics), norm_predictions = self._predictor.loss_and_predictions(
        norm_inputs, norm_targets, forcings=norm_forcings, **kwargs)
    predictions = norm_predictions.map(
        lambda pred: self._unnormalize_prediction_and_add_input(inputs, pred))
    return (loss, diagnostics), predictions
