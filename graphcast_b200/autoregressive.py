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

`input_jvp` (the tangent-linear forecast, `jax.jvp` of the unroll) runs forward with the rollout: each
step's tangent planes are fed on the device from the step before, so it needs no checkpointing.
`param_jvp` (its derivative with respect to the parameters) runs the same rollout from zero input
tangents, every step adding its weight-tangent terms.

Input noise (`noise_level`, :63-86 and :238-249) applies where the reference applies it: in `loss`,
`loss_and_grads` and `loss_and_input_grads` with several target times, once, to the time-dependent
inputs (those that are targets or forcings) before the unroll, each variable with noise of its own
shape, in physical units.  `__call__`, `input_vjp`, `input_jvp` and every one-step call are
noise-free.  The noise is drawn on the device by gcb_add_gaussian_noise, a counter-based generator
(Philox4x32-10 and Box-Muller) keyed by `rng` (an int seed, or a uint32 [2] array laid out as
jax.random.PRNGKey's key), and a variable's noise depends only on the key, the variable's name and the
element index.  JAX's threefry draws are not reproduced.  `noisy_inputs` returns the noised Dataset, and
the loss and its gradients are exactly those of the noiseless path on it; the input gradients are
returned with respect to the caller's inputs (the derivative of x + noise with respect to x is 1)."""

from __future__ import annotations

import zlib
from typing import List, Optional, Tuple

import numpy as np
import torch

from graphcast_b200 import _native
from graphcast_b200 import feedback
from graphcast_b200 import graphcast
from graphcast_b200 import normalization
from graphcast_b200 import rollout
from graphcast_b200 import xarray_shim as xs


class Predictor(graphcast.Predictor):
  """Wraps a one-step predictor to make multi-step predictions auto-regressively."""

  def __init__(self, predictor: graphcast.Predictor, noise_level: Optional[float] = None,
               gradient_checkpointing: bool = False):
    if noise_level is not None:
      noise_level = float(noise_level)
      if not np.isfinite(noise_level):
        raise ValueError(f"noise_level must be finite, not {noise_level}")
    # None and 0 turn the noise off (the reference's `if self._noise_level:`)
    self._noise_level = noise_level or None
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

  def noisy_inputs(self, inputs, targets, forcings, rng, *, _noise_fold: int = 0) -> xs.Dataset:
    """The inputs the multi-step loss unrolls from: with noise and several target times, the constant
    inputs unchanged and every time-dependent input (noise_plan) as a new float32 tensor x + noise on
    the device of the GraphCast at the bottom of the stack; otherwise `inputs` itself.  The caller's
    arrays are not modified."""
    inputs, targets = xs.from_xarray(inputs), xs.from_xarray(targets)
    forcings = xs.from_xarray(forcings)
    if targets.sizes["time"] == 1 or not self._noise_level:
      return inputs
    self._validate(inputs, targets, forcings)
    return self._noised(inputs, targets, forcings, rng, _noise_fold)

  def _noised(self, inputs: xs.Dataset, targets: xs.Dataset, forcings: xs.Dataset, rng,
              fold: int) -> xs.Dataset:
    """noisy_inputs after its checks (several target times); `inputs` itself without noise."""
    if not self._noise_level:
      return inputs
    if rng is None:
      raise ValueError("input noise needs an rng: pass rng= (an int seed, or a uint32 [2] key)")
    seed = rng_seed(rng)
    if not 0 <= int(fold) < 2**32:
      raise ValueError(f"the noise fold must lie in [0, 2**32), not {fold}")
    plan = noise_plan(inputs, targets, forcings)
    model = graphcast.innermost_graphcast(self)
    if model is None:
      raise NotImplementedError("input noise is drawn on the device of the GraphCast at the bottom of "
                                f"the predictor stack; {type(self._predictor).__name__} holds none")
    dev = model.compute_device()
    out = inputs.copy()
    segments = []
    with torch.cuda.device(dev):
      for name, stream in plan:
        v = inputs.data_vars[name]
        if isinstance(v.data, torch.Tensor):
          caller = v.data.detach()
          src = caller.to(device=dev, dtype=torch.float32).contiguous()
          # noised in place when that made a copy, else into a new tensor
          copied = src.untyped_storage().data_ptr() != caller.untyped_storage().data_ptr()
          dst = src if copied else torch.empty_like(src)
        else:                                     # uploaded once, then noised in place
          src = torch.from_numpy(np.ascontiguousarray(v.data, np.float32)).to(dev)
          dst = src
        segments.append((src, dst, stream))
        out[name] = v.copy(dst)
      lib = _native.lib()
      st = torch.cuda.current_stream(dev).cuda_stream
      for k in range(0, len(segments), _native.GCB_NOISE_MAX_SEGMENTS):
        chunk = segments[k:k + _native.GCB_NOISE_MAX_SEGMENTS]
        table = (_native.NoiseSegment * len(chunk))()
        for entry, (src, dst, stream) in zip(table, chunk):
          entry.src, entry.dst, entry.n, entry.offset, entry.stream = (
              src.data_ptr(), dst.data_ptr(), dst.numel(), 0, stream)
        _native.check(lib.gcb_add_gaussian_noise(table, len(chunk), seed, int(fold),
                                                 float(self._noise_level), st),
                      "gcb_add_gaussian_noise")
    return out

  def loss(self, inputs, targets, forcings, rng=None, *, _noise_fold: int = 0, **kwargs):
    """The mean over target times of the per-step losses of the underlying predictor; with noise,
    those of the inputs noised by `rng` (noisy_inputs)."""
    inputs, targets = xs.from_xarray(inputs), xs.from_xarray(targets)
    forcings = xs.from_xarray(forcings)
    if targets.sizes["time"] == 1:
      return self._predictor.loss(inputs, targets, forcings, **kwargs)
    self._validate(inputs, targets, forcings)
    inputs = self._noised(inputs, targets, forcings, rng, _noise_fold)
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
      return p._predictor, p._norm_of()
    return None

  def loss_and_grads(self, inputs, targets, forcings, rng=None, *, _noise_fold: int = 0, **kwargs):
    """(loss, diagnostics, grads): `loss` and `diagnostics` exactly as `loss` returns them, `grads`
    the gradient of loss.mean() (the mean over the batch) with respect to the parameters.

    One target time delegates to the inner predictor.  Several target times differentiate through the
    fed-back predictions (backprop through time, the reference demo's gradient cell): this needs
    gradient_checkpointing=True, and GraphCast directly or under a fused InputsAndResiduals.  The
    forward is the device path of `loss`, which also keeps every step's input and target planes in
    pinned host memory; the backward pass then recomputes each step from them, last step first, and
    carries dL/d(inputs) from step to step (feedback.FeedbackPlan, gcb_output_loss_grad_feedback,
    gcb_input_grad).  With noise, all of this runs on noisy_inputs(inputs, targets, forcings, rng),
    whose tensors are released before the backward pass."""
    inputs, targets = xs.from_xarray(inputs), xs.from_xarray(targets)
    forcings = xs.from_xarray(forcings)
    if targets.sizes["time"] == 1:
      return self._predictor.loss_and_grads(inputs, targets, forcings, **kwargs)
    model, norm_of = self._checkpointed_parts(inputs, targets, forcings, "loss_and_grads")
    loss, diagnostics, stash, first, lat_weight, coef = self._checkpointed_loss(
        model, norm_of, self._noised(inputs, targets, forcings, rng, _noise_fold), targets, forcings)
    plan = feedback.FeedbackPlan(first["inputs"], first["targets"], first["forcings"])
    grads = model._bptt_grads(stash, plan, first["norm"], lat_weight, coef)
    return loss, diagnostics, grads

  def _checkpointed_parts(self, inputs, targets, forcings, what: str):
    """(GraphCast, norm_of) for a gradient over several target times, with its refusals."""
    if not self._gradient_checkpointing:
      raise NotImplementedError(
          f"{what} over several target times (backprop through time) recomputes every step "
          "from its saved inputs: construct autoregressive.Predictor with gradient_checkpointing=True")
    parts = self._device_parts()
    if parts is None:
      raise NotImplementedError("backprop through time needs a GraphCast predictor, directly or inside "
                                "InputsAndResiduals (the fused normalisation)")
    self._validate(inputs, targets, forcings)
    return parts

  @staticmethod
  def _checkpointed_loss(model, norm_of, inputs, targets, forcings, tangent_run=None,
                         keep_predictions: bool = False):
    """The forward of a gradient over several target times: the device path of `loss`, which also
    keeps every step's input and target planes in pinned host memory (graphcast.StepStash).  Returns
    (loss, diagnostics, stash, first step's {inputs, targets, forcings, norm}, latitude weights,
    loss-derivative coefficients 2 kappa / (batch * steps)).  first["inputs"] is the layout of step 0's
    inputs only (_layout): the stash holds their values, and the tensors of noised inputs (1.9 GB at
    0.25 degree) must not outlive the forward.

    With tangent_run (a graphcast._TangentRun of one direction: loss_and_input_hvp; of K directions:
    a pass of batched_loss_and_input_hvp), every step also carries the input tangent planes of every
    direction on the device (GraphCast._device_loss_tangent) and keeps them in pinned host memory too:
    first["tangents"] is that StepStash.  keep_predictions (a run of one direction along parameter
    tangents: loss_and_param_gnvp): it keeps each step's prediction tangents [batch, n_out, Ng]
    instead."""
    records, first = [], {}
    stash = None

    def step(rng, inputs, targets_template, forcings):
      nonlocal stash
      norm = norm_of(inputs, targets_template, forcings)
      if tangent_run is None:
        finish, predictions, sums = model._device_loss(inputs, targets_template, forcings, norm, True)
      else:
        finish, predictions, sums, tangent = model._device_loss_tangent(
            inputs, targets_template, forcings, norm, tangent_run, keep_predictions)
      records.append((finish, sums))
      if stash is None:
        stash = graphcast.StepStash(model.engine.device)
        first.update(inputs=_layout(inputs), targets=targets_template, forcings=forcings, norm=norm)
        if tangent_run is not None:
          first["tangents"] = graphcast.StepStash(model.engine.device)
      model._stash_step(stash)
      if tangent_run is not None:
        first["tangents"].save(tangent)
      return predictions

    for _ in rollout.chunked_prediction_generator(
        step, rng=None, inputs=inputs, targets_template=targets, num_steps_per_chunk=1,
        forcings=forcings):
      pass
    sums = torch.stack([s for _, s in records]).cpu().numpy()      # the one read-back
    records = [finish(sums[t]) for t, (finish, _) in enumerate(records)]
    loss, diagnostics = _mean_over_time([l for l, _ in records], [d for _, d in records])
    _, coef = graphcast.loss_coefficients(first["targets"], model.engine.num_grid, stash.batch,
                                          len(records))
    lat_weight = model._lat_weight(first["targets"], model.engine.device)
    return loss, diagnostics, stash, first, lat_weight, coef

  def loss_and_input_grads(self, inputs, targets, forcings, rng=None, *, _noise_fold: int = 0,
                           **kwargs):
    """(loss, diagnostics, input_grads, forcing_grads): `loss` and `diagnostics` exactly as `loss`
    returns them, the gradients of loss.mean() with respect to every variable of `inputs` and
    `forcings` (GraphCast.loss_and_input_grads).  One target time delegates to the inner predictor;
    several differentiate through the fed-back predictions and forcings as loss_and_grads does
    (gradient_checkpointing=True), over every input channel (feedback.FeedbackPlan.all_channels): the
    inputs collect every step's contributions, the forcings of target time t those of step t and of
    the last input frame of step t + 1.  With noise, the gradients are taken at noisy_inputs(inputs,
    targets, forcings, rng) and returned with respect to `inputs`."""
    inputs, targets = xs.from_xarray(inputs), xs.from_xarray(targets)
    forcings = xs.from_xarray(forcings)
    if targets.sizes["time"] == 1:
      return self._predictor.loss_and_input_grads(inputs, targets, forcings, **kwargs)
    model, norm_of = self._checkpointed_parts(inputs, targets, forcings, "input gradients")
    loss, diagnostics, stash, first, lat_weight, coef = self._checkpointed_loss(
        model, norm_of, self._noised(inputs, targets, forcings, rng, _noise_fold), targets, forcings)
    plan = feedback.FeedbackPlan.all_channels(first["inputs"], first["targets"], first["forcings"])
    input_grads, forcing_grads = model._input_grads(stash, plan, first["norm"], inputs, forcings,
                                                    lat_weight=lat_weight, coef=coef)
    return loss, diagnostics, input_grads, forcing_grads

  def loss_and_input_hvp(self, inputs, targets, forcings, input_tangents, forcing_tangents=None,
                         rng=None, *, _noise_fold: int = 0, **kwargs):
    """(loss, diagnostics, input_grads, forcing_grads, input_hvp, forcing_hvp): those of
    loss_and_input_grads, bit for bit, and H v, H the Hessian of loss.mean() with respect to every
    variable of `inputs` and `forcings` and v the tangents (GraphCast.loss_and_input_hvp; the forcing
    tangents cover every target time).  One target time delegates to the inner predictor.  Several
    need gradient_checkpointing=True: one rollout computes the loss of `loss`, keeps every step's input
    and target planes and carries the input tangent planes on the device (as input_jvp does), keeping
    them too; then, last step first, each step is recomputed with its tangent and differentiated with
    the gradient and its tangent stacked (Engine.input_hvp_element), the pair carried from step to step
    over every input channel.  With noise, everything is taken at noisy_inputs(inputs, targets,
    forcings, rng)."""
    inputs, targets = xs.from_xarray(inputs), xs.from_xarray(targets)
    forcings = xs.from_xarray(forcings)
    if targets.sizes["time"] == 1:
      return self._predictor.loss_and_input_hvp(inputs, targets, forcings, input_tangents,
                                                forcing_tangents, **kwargs)
    model, norm_of = self._checkpointed_parts(inputs, targets, forcings, "input gradients")
    one = lambda ds: ds.isel(time=slice(0, 1))
    run = graphcast._TangentRun(inputs, forcings, input_tangents, forcing_tangents,
                                targets.sizes["time"],
                                feedback.FeedbackPlan(inputs, one(targets), one(forcings)))
    loss, diagnostics, stash, first, lat_weight, coef = self._checkpointed_loss(
        model, norm_of, self._noised(inputs, targets, forcings, rng, _noise_fold), targets, forcings,
        tangent_run=run)
    del run
    plan = feedback.FeedbackPlan.all_channels(first["inputs"], first["targets"], first["forcings"])
    return (loss, diagnostics) + model._input_grads(stash, plan, first["norm"], inputs, forcings,
                                                    lat_weight=lat_weight, coef=coef,
                                                    tangents=first["tangents"])

  def batched_loss_and_input_hvp(self, inputs, targets, forcings, input_tangents,
                                 forcing_tangents=None, rng=None, *, directions_per_pass=None,
                                 _noise_fold: int = 0, **kwargs):
    """loss_and_input_hvp along K tangent directions at once (GraphCast.batched_loss_and_input_hvp),
    over every target time: the tangent Datasets carry a leading "direction" dim (the forcing tangents
    cover every target time), and so do input_hvp and forcing_hvp; the loss, diagnostics and gradients
    are bit for bit those of loss_and_input_grads.  One target time delegates to the inner predictor.
    Several need gradient_checkpointing=True: each pass of directions_per_pass directions (None: all)
    is what loss_and_input_hvp runs, with every step's K tangents carried on the device and stashed
    together, and each step's recompute and backward walk shared by the gradient and its K tangents.
    With noise, everything is taken at noisy_inputs(inputs, targets, forcings, rng), the same noise in
    every pass."""
    inputs, targets = xs.from_xarray(inputs), xs.from_xarray(targets)
    forcings = xs.from_xarray(forcings)
    if targets.sizes["time"] == 1:
      return self._predictor.batched_loss_and_input_hvp(inputs, targets, forcings, input_tangents,
                                                        forcing_tangents,
                                                        directions_per_pass=directions_per_pass,
                                                        **kwargs)
    model, norm_of = self._checkpointed_parts(inputs, targets, forcings, "input gradients")
    one = lambda ds: ds.isel(time=slice(0, 1))

    def one_pass(it, ft):
      run = graphcast._TangentRun(inputs, forcings, it, ft, targets.sizes["time"],
                                  feedback.FeedbackPlan(inputs, one(targets), one(forcings)),
                                  directions=True)
      loss, diagnostics, stash, first, lat_weight, coef = self._checkpointed_loss(
          model, norm_of, self._noised(inputs, targets, forcings, rng, _noise_fold), targets,
          forcings, tangent_run=run)
      del run
      plan = feedback.FeedbackPlan.all_channels(first["inputs"], first["targets"], first["forcings"])
      return (loss, diagnostics) + model._input_grads(stash, plan, first["norm"], inputs, forcings,
                                                      lat_weight=lat_weight, coef=coef,
                                                      tangents=first["tangents"])
    return graphcast.batched_hvp(one_pass, inputs, forcings, input_tangents, forcing_tangents,
                                 directions_per_pass)

  def input_vjp(self, inputs, targets_template, forcings, cotangents, **kwargs):
    """(predictions, input_grads, forcing_grads): `predictions` as __call__ returns them, the gradients
    of sum(cotangents * predictions) over all target times with respect to every variable of `inputs`
    and `forcings` (GraphCast.input_vjp), through the fed-back predictions and forcings.  One target
    time delegates to the inner predictor; several need gradient_checkpointing=True."""
    inputs, targets_template = xs.from_xarray(inputs), xs.from_xarray(targets_template)
    forcings, cotangents = xs.from_xarray(forcings), xs.from_xarray(cotangents)
    if targets_template.sizes["time"] == 1:
      return self._predictor.input_vjp(inputs, targets_template, forcings, cotangents, **kwargs)
    model, norm_of = self._checkpointed_parts(inputs, targets_template, forcings, "input gradients")
    predictions, stash, first, plan = self._vjp_forward(model, norm_of, inputs, targets_template,
                                                        forcings)
    cot = [model._cotangent_planes(cotangents.isel(time=slice(t, t + 1)), first["targets"],
                                   stash.batch) for t in range(len(stash.steps))]
    input_grads, forcing_grads = model._input_grads(stash, plan, first["norm"], inputs, forcings,
                                                    cotangents=cot)
    return predictions, input_grads, forcing_grads

  def batched_input_vjp(self, inputs, targets_template, forcings, cotangents, *,
                        directions_per_pass=None, **kwargs):
    """input_vjp of K cotangents at once (GraphCast.batched_input_vjp), over every target time: each
    variable of `cotangents` has a leading "direction" dim followed by the shape of its
    targets_template namesake, and so do both gradient Datasets.  One target time delegates to the inner
    predictor; several need gradient_checkpointing=True.  The checkpointed rollout forward runs once
    per call and keeps every step's planes (graphcast.StepStash); each pass of directions_per_pass
    directions (None: all) then differentiates every step from that stash, its cotangents sharing each
    step's recompute and backward pass."""
    inputs, targets_template = xs.from_xarray(inputs), xs.from_xarray(targets_template)
    forcings, cotangents = xs.from_xarray(forcings), xs.from_xarray(cotangents)
    if targets_template.sizes["time"] == 1:
      return self._predictor.batched_input_vjp(inputs, targets_template, forcings, cotangents,
                                               directions_per_pass=directions_per_pass, **kwargs)
    model, norm_of = self._checkpointed_parts(inputs, targets_template, forcings, "input gradients")
    state = {}

    def one_pass(cot, first):
      if not state:                        # the forward, once, after every check has passed
        state["forward"] = self._vjp_forward(model, norm_of, inputs, targets_template, forcings)
      predictions, stash, first, plan = state["forward"]
      planes = [model._direction_cotangent_planes(cot.isel(time=slice(t, t + 1)), first["targets"],
                                                  stash.batch) for t in range(len(stash.steps))]
      return (predictions,) + model._input_grads(stash, plan, first["norm"], inputs, forcings,
                                                 cotangents=planes, directions=True)
    return graphcast.batched_vjp(one_pass, targets_template, cotangents, directions_per_pass)

  def _vjp_forward(self, model, norm_of, inputs, targets_template, forcings):
    """The forward of input_vjp over several target times: the rollout, keeping every step's input
    planes in pinned host memory.  Returns (predictions, graphcast.StepStash, first step's {inputs,
    targets, forcings, norm}, the all-channel feedback.FeedbackPlan)."""
    first = {}
    stash = None

    def step(rng, inputs, targets_template, forcings):
      nonlocal stash
      norm = norm_of(inputs, targets_template, forcings)
      predictions = model._call(inputs, targets_template, forcings, norm=norm)
      if stash is None:
        stash = graphcast.StepStash(model.engine.device)
        first.update(inputs=inputs, targets=targets_template, forcings=forcings, norm=norm)
      stash.save(model._planes_in)
      return predictions

    chunks = list(rollout.chunked_prediction_generator(
        step, rng=None, inputs=inputs, targets_template=targets_template, num_steps_per_chunk=1,
        forcings=forcings))
    plan = feedback.FeedbackPlan.all_channels(first["inputs"], first["targets"], first["forcings"])
    return xs.concat_time(chunks), stash, first, plan

  def input_jvp(self, inputs, targets_template, forcings, input_tangents, forcing_tangents=None,
                **kwargs):
    """(predictions, prediction_tangents): `predictions` as __call__ returns them, their derivative
    along the tangents of the inputs and of the forcings of every target time (GraphCast.input_jvp),
    through the fed-back predictions and forcings.  One target time delegates to the inner predictor.
    Several run forward with the rollout, step by step (no gradient_checkpointing needed, nothing kept
    per step): each step's tangent planes are fed on the device from the step before, by the rollout's
    channel map (feedback.FeedbackPlan.feed_index), its forcings slab from forcing_tangents."""
    inputs, targets_template = xs.from_xarray(inputs), xs.from_xarray(targets_template)
    forcings = xs.from_xarray(forcings)
    if targets_template.sizes["time"] == 1:
      return self._predictor.input_jvp(inputs, targets_template, forcings, input_tangents,
                                       forcing_tangents, **kwargs)
    return self._tangent_rollout(inputs, targets_template, forcings, input_tangents,
                                 forcing_tangents, directions=False)

  def batched_input_jvp(self, inputs, targets_template, forcings, input_tangents,
                        forcing_tangents=None, *, directions_per_pass=None, **kwargs):
    """input_jvp along K tangent directions at once (GraphCast.batched_input_jvp), over every target
    time: the tangent Datasets carry a leading "direction" dim, and so do prediction_tangents.  One
    target time delegates to the inner predictor.  Several run the rollout once per pass of
    directions_per_pass directions (None: all), feeding every direction's tangent planes on the device
    with one gather per step (feedback.FeedbackPlan.feed_index(K))."""
    inputs, targets_template = xs.from_xarray(inputs), xs.from_xarray(targets_template)
    forcings = xs.from_xarray(forcings)
    if targets_template.sizes["time"] == 1:
      return self._predictor.batched_input_jvp(inputs, targets_template, forcings, input_tangents,
                                               forcing_tangents,
                                               directions_per_pass=directions_per_pass, **kwargs)
    one_pass = lambda it, ft: self._tangent_rollout(inputs, targets_template, forcings, it, ft,
                                                    directions=True)
    return graphcast.batched_jvp(one_pass, inputs, forcings, input_tangents, forcing_tangents,
                                 directions_per_pass)

  def param_jvp(self, inputs, targets_template, forcings, param_tangents, **kwargs):
    """(predictions, prediction_tangents): `predictions` as __call__ returns them, their derivative
    along the parameter tangents (GraphCast.param_jvp) over every target time.  One target time
    delegates to the inner predictor.  Several run forward with the rollout, step by step, as input_jvp
    does (no gradient_checkpointing needed, nothing kept per step): step t > 0 gets the fed-back
    prediction tangent as its input tangent, plus its own weight-tangent terms."""
    inputs, targets_template = xs.from_xarray(inputs), xs.from_xarray(targets_template)
    forcings = xs.from_xarray(forcings)
    if targets_template.sizes["time"] == 1:
      return self._predictor.param_jvp(inputs, targets_template, forcings, param_tangents, **kwargs)
    return self._tangent_rollout(inputs, targets_template, forcings, None, None, directions=False,
                                 param_tangents=param_tangents)

  def loss_and_param_gnvp(self, inputs, targets, forcings, param_tangents, rng=None, *,
                          _noise_fold: int = 0, **kwargs):
    """(loss, diagnostics, gnvp): `loss` and `diagnostics` exactly as `loss` returns them, `gnvp` the
    generalised Gauss-Newton matrix of loss.mean() with respect to the params times v =
    param_tangents (a dict as param_jvp takes it), a dict shaped like the params (float32 numpy, exact
    zeros for the mesh2grid mesh-node MLP).  One target time delegates to the inner predictor
    (GraphCast.loss_and_param_gnvp).

    Several target times need gradient_checkpointing=True, and GraphCast directly or under a fused
    InputsAndResiduals.  gnvp is then sum_t J_t^T Lambda_t J_t v: r_t the normalised residual of step t,
    J_t = dr_t / d params through the whole rollout (fed-back predictions included) and Lambda_t =
    diag(coef * lat_weight), coef = 2 kappa / (batch * steps), the Hessian of the loss in r_t.  It is
    positive semi-definite, and where every step's targets equal the rollout's own predictions it is
    the full Hessian of the multi-step loss times v.  The forward is the rollout of param_jvp with the
    fused loss, which keeps every step's input and target planes and prediction tangents J_t v in pinned
    host memory; the backward then walks the steps last first as loss_and_grads does, each seeded with
    Lambda_t r-dot_t plus the feedback of the following step (gcb_output_loss_gn_seed_feedback).  With
    noise, everything is taken at noisy_inputs(inputs, targets, forcings, rng)."""
    inputs, targets = xs.from_xarray(inputs), xs.from_xarray(targets)
    forcings = xs.from_xarray(forcings)
    if targets.sizes["time"] == 1:
      return self._predictor.loss_and_param_gnvp(inputs, targets, forcings, param_tangents, **kwargs)
    if not self._gradient_checkpointing:
      raise NotImplementedError(
          "Gauss-Newton products cover one target time without gradient checkpointing: over several "
          "they recompute every step from its saved inputs; construct autoregressive.Predictor with "
          "gradient_checkpointing=True")
    model, norm_of = self._checkpointed_parts(inputs, targets, forcings, "Gauss-Newton products")
    one = lambda ds: ds.isel(time=slice(0, 1))
    run = model._param_tangent_run(inputs, targets, forcings, param_tangents, targets.sizes["time"],
                                   feedback.FeedbackPlan(inputs, one(targets), one(forcings)))
    loss, diagnostics, stash, first, lat_weight, coef = self._checkpointed_loss(
        model, norm_of, self._noised(inputs, targets, forcings, rng, _noise_fold), targets, forcings,
        tangent_run=run, keep_predictions=True)
    del run
    plan = feedback.FeedbackPlan(first["inputs"], first["targets"], first["forcings"])
    gnvp = model._bptt_grads(stash, plan, first["norm"], lat_weight, coef,
                             pred_tangents=first["tangents"])
    return loss, diagnostics, gnvp

  def loss_and_param_hvp(self, inputs, targets, forcings, param_tangents, **kwargs):
    """(loss, diagnostics, grads, hvp) of one target time (GraphCast.loss_and_param_hvp), delegated to
    the inner predictor; parameter Hessian-vector products over several target times are not provided,
    with or without gradient_checkpointing."""
    targets = xs.from_xarray(targets)
    if targets.sizes["time"] != 1:
      raise NotImplementedError("parameter Hessian-vector products cover one target time (several "
                                "are not provided)")
    return self._predictor.loss_and_param_hvp(inputs, targets, forcings, param_tangents, **kwargs)

  def _tangent_rollout(self, inputs, targets_template, forcings, input_tangents, forcing_tangents,
                       directions: bool, param_tangents=None):
    """input_jvp (batched_input_jvp with `directions`, param_jvp with `param_tangents`) over several
    target times."""
    what = "input_jvp" if param_tangents is None else "param_jvp"
    parts = self._device_parts()
    if parts is None:
      raise NotImplementedError(f"{what} over several target times needs a GraphCast predictor, "
                                "directly or inside InputsAndResiduals (the fused normalisation)")
    self._validate(inputs, targets_template, forcings)
    model, norm_of = parts
    num_steps = targets_template.sizes["time"]
    one = lambda ds: ds.isel(time=slice(0, 1))
    plan = feedback.FeedbackPlan(inputs, one(targets_template), one(forcings))
    if param_tangents is None:
      run = graphcast._TangentRun(inputs, forcings, input_tangents, forcing_tangents, num_steps, plan,
                                  directions=directions)
    else:
      run = model._param_tangent_run(inputs, targets_template, forcings, param_tangents, num_steps,
                                     plan)
    tangents = []

    def step(rng, inputs, targets_template, forcings):
      norm = norm_of(inputs, targets_template, forcings)
      predictions, step_tangents = model._input_jvp(inputs, targets_template, forcings, run, norm)
      tangents.append(step_tangents)
      return predictions

    chunks = list(rollout.chunked_prediction_generator(
        step, rng=None, inputs=inputs, targets_template=targets_template, num_steps_per_chunk=1,
        forcings=forcings))
    # the tangents of each step with the coordinates the rollout gives its predictions
    timed = []
    for chunk, step_tangents in zip(chunks, tangents):
      ds = xs.Dataset(coords=chunk.coords)
      if directions:
        ds.coords[feedback.DIRECTION] = step_tangents.coords[feedback.DIRECTION]
      for name in step_tangents.keys():
        ds[name] = step_tangents.data_vars[name]
      timed.append(ds)
    return xs.concat_time(chunks), xs.concat_time(timed)


def rng_seed(rng) -> int:
  """The 64-bit seed of an `rng`: an int in [0, 2**64), or a uint32 array of shape (2,) laid out as
  jax.random.PRNGKey(seed) lays out its key, [seed >> 32, seed & 0xffffffff]."""
  if isinstance(rng, (bool, np.bool_)):
    raise ValueError("rng must be an int seed or a uint32 [2] key, not a bool")
  if isinstance(rng, (int, np.integer)):
    if not 0 <= int(rng) < 2**64:
      raise ValueError(f"an int rng must lie in [0, 2**64), not {rng}")
    return int(rng)
  key = np.asarray(rng)
  if key.shape != (2,) or key.dtype != np.uint32:
    raise ValueError(f"rng must be an int seed or a uint32 array of shape (2,), not {key.dtype} "
                     f"{key.shape}")
  return (int(key[0]) << 32) | int(key[1])


def noise_plan(inputs: xs.Dataset, targets: xs.Dataset, forcings: xs.Dataset) -> List[Tuple[str, int]]:
  """(name, stream) of every input the noise applies to, in the order of `inputs`: the time-dependent
  inputs, which are targets or forcings (reference :238-242; the others are the constant inputs).
  stream = crc32 of the name, so that a variable's noise does not depend on which others are present;
  two variables with the same stream raise ValueError."""
  plan, seen = [], {}
  for name in inputs.keys():
    if name not in targets and name not in forcings:
      continue
    stream = zlib.crc32(name.encode())
    if stream in seen:
      raise ValueError(f"input variables {seen[stream]} and {name} have the same noise stream "
                       f"{stream:#010x} (crc32 of the name): rename one of them")
    seen[stream] = name
    plan.append((name, stream))
  return plan


def _layout(ds: xs.Dataset) -> xs.Dataset:
  """`ds` with each variable's data replaced by a zero-stride array of its shape: the names, dims,
  shapes and coords that the backward pass's channel plans read, without the values."""
  out = ds.copy()
  for name, v in ds.data_vars.items():
    out[name] = v.copy(np.broadcast_to(np.float32(0), v.shape))
  return out


def _mean_over_time(step_losses, step_diagnostics):
  """Mean over the steps of `(batch,)` losses and diagnostics (NaNs propagate)."""
  mean = lambda arrays: xs.DataArray(
      np.mean(np.stack([np.asarray(a.values, np.float64) for a in arrays]), axis=0
              ).astype(np.float32), step_losses[0].dims)
  diagnostics = xs.Dataset()
  for name in step_diagnostics[0].keys():
    diagnostics[name] = mean([d.data_vars[name] for d in step_diagnostics])
  return mean(step_losses), diagnostics
