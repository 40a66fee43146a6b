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

`loss_and_grads` (the reference demo's `jax.value_and_grad` of `loss` with
`gradient_checkpointing=True`, :262-310) differentiates that mean through the fed-back predictions:
backprop through time.  Every step is recomputed from its saved input planes in the backward pass,
which is what the reference's per-step `hk.remat` asks for; without `gradient_checkpointing` only one
target time is supported.  The gradient reaches a step's inputs through the residual add and the
target normalisation of InputsAndResiduals, the frame shift and the grid embedder; see
graphcast_b200/feedback.py and DESIGN.md section 3.5.

Not provided: input noise (a training-side feature)."""

from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from graphcast_b200 import feedback
from graphcast_b200 import graphcast
from graphcast_b200 import losses
from graphcast_b200 import model_utils
from graphcast_b200 import normalization
from graphcast_b200 import rollout
from graphcast_b200 import xarray_shim as xs


class Predictor(graphcast.Predictor):
  """Wraps a one-step predictor to make multi-step predictions auto-regressively."""

  def __init__(self, predictor: graphcast.Predictor, noise_level: Optional[float] = None,
               gradient_checkpointing: bool = False):
    if noise_level:
      raise NotImplementedError("input noise is a training-time feature")
    # The multi-step gradient recomputes every step from its saved inputs (the reference's hk.remat
    # per step); without checkpointing it would hold every step's activations, which is not offered.
    self._gradient_checkpointing = bool(gradient_checkpointing)
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

  def _device_parts(self):
    """(GraphCast, norm_of) when the inner predictor's loss runs on the device, else None;
    norm_of(inputs, targets, forcings) -> the FusedNormalization of a step or None."""
    p = self._predictor
    if isinstance(p, graphcast.GraphCast):
      return p, lambda i, t, f: None
    if isinstance(p, normalization.InputsAndResiduals) and p._fuses():
      def norm_of(i, t, f):
        device = p._predictor._device or f"cuda:{torch.cuda.current_device()}"
        return p._fused_constants(i, t, f, torch.device(device))
      return p._predictor, norm_of
    return None

  def loss_and_grads(self, inputs, targets, forcings, **kwargs):
    """(loss, diagnostics, grads): `loss` and `diagnostics` exactly as `loss` returns them, `grads`
    the gradient of loss.mean() (the mean over the batch) with respect to the parameters.

    One target time delegates to the inner predictor.  Several target times differentiate through the
    fed-back predictions (backprop through time, the reference demo's gradient cell): this needs
    gradient_checkpointing=True, and GraphCast directly or under a fused InputsAndResiduals.  The
    forward is the device path of `loss`, which also keeps every step's input and target planes in
    pinned host memory; the backward pass then recomputes each step from them, last step first, and
    carries dL/d(inputs) from step to step (feedback.FeedbackPlan, gcb_output_loss_grad_feedback,
    gcb_input_grad)."""
    inputs, targets = xs.from_xarray(inputs), xs.from_xarray(targets)
    forcings = xs.from_xarray(forcings)
    if targets.sizes["time"] == 1:
      return self._predictor.loss_and_grads(inputs, targets, forcings, **kwargs)
    if not self._gradient_checkpointing:
      raise NotImplementedError(
          "loss_and_grads over several target times (backprop through time) recomputes every step "
          "from its saved inputs: construct autoregressive.Predictor with gradient_checkpointing=True")
    parts = self._device_parts()
    if parts is None:
      raise NotImplementedError("backprop through time needs a GraphCast predictor, directly or inside "
                                "InputsAndResiduals (the fused normalisation)")
    model, norm_of = parts
    self._validate(inputs, targets, forcings)
    records, first = [], {}
    stash = None

    def step(rng, inputs, targets_template, forcings):
      nonlocal stash
      norm = norm_of(inputs, targets_template, forcings)
      finish, predictions, sums = model._device_loss(inputs, targets_template, forcings, norm, True)
      records.append((finish, sums))
      if stash is None:
        stash = graphcast.StepStash(model.engine.device)
        first.update(inputs=inputs, targets=targets_template, forcings=forcings, norm=norm)
      model._stash_step(stash)
      return predictions

    for _ in rollout.chunked_prediction_generator(
        step, rng=None, inputs=inputs, targets_template=targets, num_steps_per_chunk=1,
        forcings=forcings):
      pass
    sums = torch.stack([s for _, s in records]).cpu().numpy()      # the one read-back
    records = [finish(sums[t]) for t, (finish, _) in enumerate(records)]
    loss, diagnostics = _mean_over_time([l for l, _ in records], [d for _, d in records])

    plan = feedback.FeedbackPlan(first["inputs"], first["targets"], first["forcings"])
    num_steps, batch = len(records), stash.batch
    slabs = model_utils.channel_layout(first["targets"])
    kappa = losses.channel_kappa(slabs, model.engine.num_grid, graphcast.LOSS_PER_VARIABLE_WEIGHTS)
    lat_weight = model._lat_weight(first["targets"], model.engine.device)
    grads = model._bptt_grads(stash, plan, first["norm"], lat_weight,
                              2.0 * kappa / (batch * num_steps))
    return loss, diagnostics, grads


def _mean_over_time(step_losses, step_diagnostics):
  """Mean over the steps of `(batch,)` losses and diagnostics (NaNs propagate)."""
  mean = lambda arrays: xs.DataArray(
      np.mean(np.stack([np.asarray(a.values, np.float64) for a in arrays]), axis=0
              ).astype(np.float32), step_losses[0].dims)
  diagnostics = xs.Dataset()
  for name in step_diagnostics[0].keys():
    diagnostics[name] = mean([d.data_vars[name] for d in step_diagnostics])
  return mean(step_losses), diagnostics
