"""Inference mirror of `autoregressive.Predictor` (weathernext/utils/autoregressive.py:36-312).

The reference wrapper turns a one-step predictor into a multi-step one: a call with a
`targets_template` of T time steps unrolls the inner predictor T times (`hk.scan`), feeding
the predictions - and the forcings of the step - back as the next inputs, with the time
coordinates of every inner call reset to those of the first step.  That feeding logic is the
one of `rollout.chunked_prediction_generator` (pinned against the reference's generator in
tests/test_reference_rollout_golden.py), so this mirror unrolls through it and concatenates the
per-step predictions on the device.  Kept from the reference: the validation errors
(:88-116), constant inputs passed through unchanged, predictions carrying the template's time
coordinate.

`loss` (:224-312) is the mean over the target times of the inner predictor's per-step losses:
with one target time it delegates to the inner `loss`; otherwise it unrolls the same way, calling
the inner `loss_and_predictions` with the targets of each step and feeding its predictions back.
When the inner predictor is this package's `GraphCast` (directly or under a fused
`normalization.InputsAndResiduals`), every step's loss stays on the device as per-channel sums of
`gcb_output_loss` and all of them are read back once, after the last step.

Not provided: input noise and gradient checkpointing (training-side features)."""

from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from graphcast_b200 import graphcast
from graphcast_b200 import normalization
from graphcast_b200 import rollout
from graphcast_b200 import xarray_shim as xs


class Predictor(graphcast.Predictor):
  """Wraps a one-step predictor to make multi-step predictions auto-regressively."""

  def __init__(self, predictor: graphcast.Predictor, noise_level: Optional[float] = None,
               gradient_checkpointing: bool = False):
    if noise_level:
      raise NotImplementedError("input noise is a training-time feature")
    del gradient_checkpointing            # no backward pass here
    self._predictor = predictor

  @staticmethod
  def _validate(inputs: xs.Dataset, targets: xs.Dataset, forcings: xs.Dataset) -> None:
    for name in inputs.keys():
      if name in targets or name in forcings:
        continue
      if "time" in inputs.data_vars[name].dims:
        raise ValueError(
            f"Time-dependent input variable {name} must either be a forcing "
            "variable, or a target variable to allow for auto-regressive feedback.")
    for name in targets.keys():
      if "time" not in targets.data_vars[name].dims:
        raise ValueError(f"Target variable {name} must be time-dependent.")
    for name in forcings.keys():
      if "time" not in forcings.data_vars[name].dims:
        raise ValueError(f"Forcing variable {name} must be time-dependent.")
    overlap = set(forcings.keys()) & set(targets.keys())
    if overlap:
      raise ValueError("The following were specified as both targets and "
                       f"forcings, which isn't allowed: {overlap}")

  def __call__(self, inputs, targets_template, forcings, **kwargs) -> xs.Dataset:
    inputs = xs.from_xarray(inputs)
    targets_template = xs.from_xarray(targets_template)
    forcings = xs.from_xarray(forcings)
    self._validate(inputs, targets_template, forcings)
    step = lambda rng, inputs, targets_template, forcings: self._predictor(
        inputs, targets_template, forcings, **kwargs)
    chunks = list(rollout.chunked_prediction_generator(
        step, rng=None, inputs=inputs, targets_template=targets_template,
        num_steps_per_chunk=1, forcings=forcings))
    return xs.concat_time(chunks)

  def _device_step(self):
    """(inputs, targets, forcings) -> (finish, predictions, device channel sums) when the inner
    predictor reduces its loss on the device, else None."""
    p = self._predictor
    if isinstance(p, graphcast.GraphCast):
      return lambda i, t, f: p._device_loss(i, t, f, None, True)
    if isinstance(p, normalization.InputsAndResiduals) and p._fuses():
      return lambda i, t, f: p._device_loss(i, t, f, True)
    return None

  def loss(self, inputs, targets, forcings, **kwargs):
    """The mean over target times of the per-step losses of the underlying predictor."""
    inputs, targets = xs.from_xarray(inputs), xs.from_xarray(targets)
    forcings = xs.from_xarray(forcings)
    if targets.sizes["time"] == 1:
      return self._predictor.loss(inputs, targets, forcings, **kwargs)
    self._validate(inputs, targets, forcings)
    device_step = self._device_step()
    records = []

    def step(rng, inputs, targets_template, forcings):
      if device_step is not None:
        finish, predictions, sums = device_step(inputs, targets_template, forcings)
        records.append((finish, sums))
      else:
        loss_and_diagnostics, predictions = self._predictor.loss_and_predictions(
            inputs, targets_template, forcings, **kwargs)
        records.append(loss_and_diagnostics)
      return predictions

    for _ in rollout.chunked_prediction_generator(
        step, rng=None, inputs=inputs, targets_template=targets, num_steps_per_chunk=1,
        forcings=forcings):
      pass
    if device_step is not None:
      sums = torch.stack([s for _, s in records]).cpu().numpy()      # the one read-back
      records = [finish(sums[t]) for t, (finish, _) in enumerate(records)]
    return _mean_over_time([l for l, _ in records], [d for _, d in records])


def _mean_over_time(step_losses, step_diagnostics):
  """Mean over the steps of `(batch,)` losses and diagnostics (NaNs propagate)."""
  mean = lambda arrays: xs.DataArray(
      np.mean(np.stack([np.asarray(a.values, np.float64) for a in arrays]), axis=0
              ).astype(np.float32), step_losses[0].dims)
  diagnostics = xs.Dataset()
  for name in step_diagnostics[0].keys():
    diagnostics[name] = mean([d.data_vars[name] for d in step_diagnostics])
  return mean(step_losses), diagnostics
