"""GraphCast one-step predictor -- host-side mirror of the reference API.

Same public surface as `weathernext/weathernext1_graph/graphcast.py`:
  ModelConfig (:115-142), TaskConfig (utils/task.py:21-28), CheckPoint (:145-151),
  TASK / TASK_13 / TASK_13_PRECIP_OUT (:86-112),
  GraphCast(model_config, task_config).__call__(inputs, targets_template,
  forcings, is_training=False) -> Dataset (:184, :298-329),
  loss / loss_and_predictions(inputs, targets, forcings) (:331-366).

What differs is only *how* the step is computed: the three GNN calls
(`_run_grid2mesh_gnn` :550, `_run_mesh_gnn` :606, `_run_mesh2grid_gnn` :641) and
the channel (un)packing (`_inputs_to_grid_node_features` :680,
`_grid_node_outputs_to_prediction` :701) run as hand-written sm_90a kernels
behind the C ABI in include/graphcast_b200.h, and so does the loss's reduction
(`gcb_output_loss`, fused into the output unpack).  There is no CPU path: without a
CUDA device or the built library this module raises.

Parameters: the reference threads a Haiku parameter dict through
`hk.transform(...).apply(params, ...)`.  Here the same dict (module path ->
{"w","b"} / {"scale","offset"}; see SURVEY.md appendix B) is given to the
constructor (`params=`) or to `set_params`, e.g. `CheckPoint.params` loaded by
graphcast_b200.checkpoint.load.
"""

from __future__ import annotations

import abc
import dataclasses
import functools
from typing import Any, Dict, List, Mapping, Optional, Tuple

import numpy as np
import torch

from graphcast_b200 import _native
from graphcast_b200 import engine as engine_lib
from graphcast_b200 import feedback
from graphcast_b200 import graph as graph_lib
from graphcast_b200 import losses
from graphcast_b200 import model_utils
from graphcast_b200 import variables
from graphcast_b200 import xarray_shim as xs


@dataclasses.dataclass(frozen=True, eq=True)
class TaskConfig:
  """Inputs / targets / forcings of a task (reference utils/task.py:21-28)."""
  input_variables: Tuple[str, ...]
  target_variables: Tuple[str, ...]
  forcing_variables: Tuple[str, ...]
  pressure_levels: Tuple[int, ...]
  input_duration: str


@dataclasses.dataclass(frozen=True, eq=True)
class ModelConfig:
  """Architecture hyper-parameters (reference graphcast.py:115-142)."""
  resolution: float
  mesh_size: int
  latent_size: int
  gnn_msg_steps: int
  hidden_layers: int
  radius_query_fraction_edge_length: float
  mesh2grid_edge_normalization_factor: Optional[float] = None


@dataclasses.dataclass(frozen=True, eq=True)
class CheckPoint:
  params: Dict[str, Any]
  model_config: ModelConfig
  task_config: TaskConfig
  description: str
  license: str


_V = variables
TASK = TaskConfig(
    input_variables=(_V.TARGET_SURFACE_VARS + _V.TARGET_ATMOSPHERIC_VARS + _V.FORCING_VARS
                     + _V.STATIC_VARS),
    target_variables=_V.TARGET_SURFACE_VARS + _V.TARGET_ATMOSPHERIC_VARS,
    forcing_variables=_V.FORCING_VARS,
    pressure_levels=_V.PRESSURE_LEVELS_ERA5_37,
    input_duration="12h")
TASK_13 = dataclasses.replace(TASK, pressure_levels=_V.PRESSURE_LEVELS_WEATHERBENCH_13)
TASK_13_PRECIP_OUT = dataclasses.replace(
    TASK_13,
    input_variables=(_V.TARGET_SURFACE_NO_PRECIP_VARS + _V.TARGET_ATMOSPHERIC_VARS
                     + _V.FORCING_VARS + _V.STATIC_VARS))


class Predictor(abc.ABC):
  """xarray-style predictor interface (reference utils/predictor_base.py:27-84)."""

  @abc.abstractmethod
  def __call__(self, inputs, targets_template, forcings, **optional_kwargs):
    """Returns predictions shaped like `targets_template`."""

  def loss(self, inputs, targets, forcings, **optional_kwargs):
    """Returns (loss, diagnostics): `(batch,)` DataArray and Dataset of per-variable losses."""
    raise NotImplementedError(f"{type(self).__name__} does not implement a loss")

  def loss_and_predictions(self, inputs, targets, forcings, **optional_kwargs):
    """Returns ((loss, diagnostics), predictions)."""
    raise NotImplementedError(f"{type(self).__name__} does not implement a loss")

  def loss_and_grads(self, inputs, targets, forcings, **optional_kwargs):
    """Returns (loss, diagnostics, grads): `loss` / `diagnostics` as `loss` returns them, `grads`
    the gradient of loss.mean() (the mean over the batch) with respect to the parameters."""
    raise NotImplementedError(f"{type(self).__name__} does not implement parameter gradients")

  def loss_and_input_grads(self, inputs, targets, forcings, **optional_kwargs):
    """Returns (loss, diagnostics, input_grads, forcing_grads): `loss` / `diagnostics` as `loss`
    returns them, the gradients of loss.mean() with respect to every variable of `inputs` and
    `forcings`, as float32 Datasets shaped like them."""
    raise NotImplementedError(f"{type(self).__name__} does not implement input gradients")

  def input_vjp(self, inputs, targets_template, forcings, cotangents, **optional_kwargs):
    """Returns (predictions, input_grads, forcing_grads): the predictions of __call__ and the
    gradients of sum(cotangents * predictions) with respect to every variable of `inputs` and
    `forcings`; `cotangents` is shaped like `targets_template`."""
    raise NotImplementedError(f"{type(self).__name__} does not implement input gradients")

  def loss_and_input_hvp(self, inputs, targets, forcings, input_tangents, forcing_tangents=None,
                         **optional_kwargs):
    """Returns (loss, diagnostics, input_grads, forcing_grads, input_hvp, forcing_hvp): those of
    loss_and_input_grads, and the Hessian of loss.mean() with respect to the inputs and forcings times
    the tangents (Datasets as input_jvp takes them), shaped like `inputs` and `forcings`."""
    raise NotImplementedError(f"{type(self).__name__} does not implement Hessian-vector products")

  def batched_loss_and_input_hvp(self, inputs, targets, forcings, input_tangents, forcing_tangents=None,
                                 *, directions_per_pass=None, **optional_kwargs):
    """Returns (loss, diagnostics, input_grads, forcing_grads, input_hvp, forcing_hvp):
    loss_and_input_hvp along K tangent directions at once, the tangent Datasets' variables carrying a
    leading "direction" dim of size K; input_hvp and forcing_hvp have the same leading dim, the loss and
    gradients none.  directions_per_pass: directions that share one forward (None: all)."""
    raise NotImplementedError(f"{type(self).__name__} does not implement Hessian-vector products")

  def input_jvp(self, inputs, targets_template, forcings, input_tangents, forcing_tangents=None,
                **optional_kwargs):
    """Returns (predictions, prediction_tangents): the predictions of __call__ and their derivative
    along the tangents of the inputs and forcings (Datasets with some of their variables, each shaped
    like its namesake; a variable left out is held fixed), shaped like the predictions."""
    raise NotImplementedError(f"{type(self).__name__} does not implement input gradients")

  def batched_input_jvp(self, inputs, targets_template, forcings, input_tangents,
                        forcing_tangents=None, *, directions_per_pass=None, **optional_kwargs):
    """Returns (predictions, prediction_tangents): input_jvp along K tangent directions at once, the
    tangent Datasets' variables carrying a leading "direction" dim of size K; prediction_tangents has
    the same leading dim.  directions_per_pass: directions that share one forward (None: all)."""
    raise NotImplementedError(f"{type(self).__name__} does not implement input gradients")

  def batched_input_vjp(self, inputs, targets_template, forcings, cotangents, *,
                        directions_per_pass=None, **optional_kwargs):
    """Returns (predictions, input_grads, forcing_grads): input_vjp of K cotangents at once, each
    variable of `cotangents` carrying a leading "direction" dim of size K; both gradient Datasets have
    the same leading dim.  directions_per_pass: directions that share one forward (None: all)."""
    raise NotImplementedError(f"{type(self).__name__} does not implement input gradients")

  def param_jvp(self, inputs, targets_template, forcings, param_tangents, **optional_kwargs):
    """Returns (predictions, prediction_tangents): the predictions of __call__ and their derivative
    along `param_tangents`, a dict shaped like the params ({module: {field: array}}, entries left out
    being zero), shaped like the predictions: jax.jvp of the forecast with respect to the params."""
    raise NotImplementedError(f"{type(self).__name__} does not implement parameter tangents")

  def loss_and_param_gnvp(self, inputs, targets, forcings, param_tangents, **optional_kwargs):
    """Returns (loss, diagnostics, gnvp): `loss` / `diagnostics` as `loss` returns them, `gnvp` the
    generalised Gauss-Newton matrix of loss.mean() with respect to the params times `param_tangents`,
    a dict shaped like the params."""
    raise NotImplementedError(f"{type(self).__name__} does not implement parameter tangents")

  def loss_and_param_hvp(self, inputs, targets, forcings, param_tangents, **optional_kwargs):
    """Returns (loss, diagnostics, grads, hvp): `loss` / `diagnostics` as `loss` returns them, `grads`
    as loss_and_grads returns it, `hvp` the Hessian of loss.mean() with respect to the params times
    `param_tangents`, a dict shaped like the params."""
    raise NotImplementedError(f"{type(self).__name__} does not implement parameter tangents")

  def loss_and_joint_hvp(self, inputs, targets, forcings, param_tangents=None, input_tangents=None,
                         forcing_tangents=None, **optional_kwargs):
    """Returns (loss, diagnostics, grads, input_grads, forcing_grads, param_hvp, input_hvp,
    forcing_hvp): those of loss_and_grads and loss_and_input_grads, and the Hessian of loss.mean()
    jointly in the params, inputs and forcings times the tangents (param_tangents as
    loss_and_param_hvp takes them, input and forcing tangents as loss_and_input_hvp does, None: zero),
    its parameter side shaped like the params and its input side like `inputs` and `forcings`."""
    raise NotImplementedError(f"{type(self).__name__} does not implement joint Hessian-vector "
                              "products")


# Per-variable weights of GraphCast's loss (reference graphcast.py:341-356); others weigh 1.
LOSS_PER_VARIABLE_WEIGHTS = {
    "2m_temperature": 1.0,
    "10m_u_component_of_wind": 0.1,
    "10m_v_component_of_wind": 0.1,
    "mean_sea_level_pressure": 0.1,
    "total_precipitation_6hr": 0.1,
}


def num_outputs(task_config: TaskConfig) -> int:
  """Output channels: surface vars + levels * atmospheric vars (graphcast.py:236-241)."""
  atmos = set(task_config.target_variables) & set(_V.ALL_ATMOSPHERIC_VARS)
  surface = set(task_config.target_variables) - set(_V.ALL_ATMOSPHERIC_VARS)
  return len(surface) + len(task_config.pressure_levels) * len(atmos)


@dataclasses.dataclass
class FusedNormalization:
  """Per-channel constants that let the pack / unpack kernels apply
  normalization.InputsAndResiduals (utils/normalization.py:113-160) on the fly."""
  in_mean: torch.Tensor          # [c_in]
  in_scale: torch.Tensor         # [c_in]
  out_scale: torch.Tensor        # [n_out]
  out_offset: torch.Tensor       # [n_out]
  add_plane_index: torch.Tensor  # [n_out] int32: input plane to add (-1 = none)


class GraphCast(Predictor):
  """GraphCast predictor running on one H100."""

  def __init__(self, model_config: ModelConfig, task_config: TaskConfig, *,
               params: Optional[Mapping[str, Mapping[str, np.ndarray]]] = None,
               precision: str = "bf16x3", device: Optional[Any] = None,
               pregather: bool = True, fuse: bool = True, chain_lag: int = 0,
               image_residual: bool = True, deep_chains: bool = True, static_cache: bool = True):
    if model_config.latent_size != engine_lib.LATENT:
      raise ValueError(f"latent_size {model_config.latent_size} is not supported by the "
                       f"sm_90a kernels (only {engine_lib.LATENT})")
    if model_config.hidden_layers != 1:
      raise ValueError("only hidden_layers=1 is supported by the sm_90a kernels")
    self._model_config = model_config
    self._task_config = task_config
    self._precision = precision
    self._pregather = pregather
    self._fuse, self._chain_lag, self._image_residual = fuse, chain_lag, image_residual
    self._deep_chains = deep_chains
    # Engine.static_cache: the weight-only edge terms of the step are computed once per weight
    # version and precision (10.3 GiB at 0.25 degree), not every step.
    self._static_cache = static_cache
    self._device = device
    self._engine: Optional[engine_lib.Engine] = None
    self._params = params
    # Where the gradients of _loss_and_grads / _bptt_grads go: None = host numpy dicts (the public
    # loss_and_grads), else a callable(engine) that takes them on the device (optim.AdamW).
    self._grad_sink = None
    self._num_outputs = num_outputs(task_config)
    self._initialized = False
    self._static_graph: Optional[graph_lib.StaticGraph] = None
    self._planes_in: Optional[torch.Tensor] = None
    self._planes_out: Optional[torch.Tensor] = None
    # Host->device staging: two input-plane buffers filled on a dedicated copy stream, so
    # the H2D transfer of call k+1 overlaps the kernels of call k when the caller does not
    # synchronise in between (serving loop / ensemble members).
    self._h2d_stream: Optional[torch.cuda.Stream] = None
    self._planes_bufs: List[Optional[torch.Tensor]] = [None, None]
    self._buf_free: List[Optional[torch.cuda.Event]] = [None, None]
    self._call_index = 0
    # The loss: target planes staged like the inputs (same slots, same events), the latitude
    # weights of the last target grid, the per-channel sums of the last call.
    self._target_bufs: List[Optional[torch.Tensor]] = [None, None]
    self._planes_tgt: Optional[torch.Tensor] = None
    self._lat_weight_cache = None
    self._channel_sums: Optional[torch.Tensor] = None

  # -- parameters ------------------------------------------------------------------
  @property
  def _params(self):
    """The host parameters: while an engine exists, the engine's (Engine.params, which follows
    device reloads); otherwise those of the constructor or the last set_params."""
    return self._engine.params if self._engine is not None else self._host_params

  @_params.setter
  def _params(self, params) -> None:
    self._host_params = params

  def set_params(self, params: Mapping[str, Mapping[str, np.ndarray]]) -> None:
    """New weights.  An engine that exists already is reloaded in place (Engine.load_params) when
    the shapes match: no graph upload, no new workspace.  Otherwise it is dropped and the next call
    builds one."""
    if self._engine is not None:
      try:
        self._engine.load_params(params)
      except ValueError:
        self._engine = None
    self._params = params

  def set_precision(self, precision: str) -> None:
    """Arithmetic mode of the fused layers: "bf16x3" (parity), "bf16", "fp32_simt"."""
    from graphcast_b200 import _native
    if precision not in _native.PRECISIONS:
      raise ValueError(f"unknown precision {precision!r}; expected one of "
                       f"{sorted(_native.PRECISIONS)}")
    self._precision = precision
    if self._engine is not None:
      self._engine.set_precision(precision)

  @property
  def engine(self) -> engine_lib.Engine:
    if self._engine is None:
      raise RuntimeError("GraphCast has not been called yet")
    return self._engine

  def compute_device(self) -> torch.device:
    """The device the model runs on: its engine's, or the one the next call builds its engine on."""
    if self._engine is not None:
      return self._engine.device
    return torch.device(self._device if self._device is not None
                        else f"cuda:{torch.cuda.current_device()}")

  # -- lazy initialisation (reference _maybe_init :368-378) -------------------------
  def _maybe_init(self, sample_inputs: xs.Dataset, c_in: int) -> None:
    if not self._initialized:
      cfg = self._model_config
      self._static_graph = graph_lib.cached_static_graph(
          grid_lat=np.asarray(sample_inputs.lat.values),
          grid_lon=np.asarray(sample_inputs.lon.values),
          mesh_size=cfg.mesh_size,
          radius_query_fraction_edge_length=cfg.radius_query_fraction_edge_length,
          mesh2grid_edge_normalization_factor=cfg.mesh2grid_edge_normalization_factor)
      self._initialized = True
    if self._engine is None:
      if self._params is None:
        raise ValueError("GraphCast has no parameters: pass params= or call set_params()")
      self._engine = engine_lib.Engine(
          self._static_graph, self._params, c_in=c_in, n_out=self._num_outputs,
          msg_steps=self._model_config.gnn_msg_steps, precision=self._precision,
          device=self._device, pregather=self._pregather, fuse=self._fuse,
          chain_lag=self._chain_lag, image_residual=self._image_residual,
          deep_chains=self._deep_chains, static_cache=self._static_cache)
    elif self._engine.c_in != c_in:
      raise ValueError(f"inputs+forcings stack to {c_in} channels but the model was "
                       f"built for {self._engine.c_in}")

  # -- the step ----------------------------------------------------------------------
  def __call__(self, inputs, targets_template, forcings, is_training: bool = False,
               **unused_kwargs):
    return self._call(inputs, targets_template, forcings, norm=None)

  # -- the loss (reference loss_and_predictions / loss :331-366) ------------------------
  def loss_and_predictions(self, inputs, targets, forcings, **unused_kwargs):
    """((loss, diagnostics), predictions): the step, then `losses.weighted_mse_per_level` of the
    predictions against `targets` with GraphCast's per-variable weights.  The error is reduced on the
    device in the kernel that unpacks the outputs (gcb_output_loss: fp32 differences, fp64 sums)."""
    return self._loss(inputs, targets, forcings, norm=None, predictions=True)

  def loss(self, inputs, targets, forcings, **unused_kwargs):
    """(loss, diagnostics) of `loss_and_predictions`; the predictions are not materialised."""
    return self._loss(inputs, targets, forcings, norm=None, predictions=False)[0]

  def loss_and_grads(self, inputs, targets, forcings, **unused_kwargs):
    """(loss, diagnostics, grads) for one target time.

    `loss` and `diagnostics` are exactly what `loss()` returns for the same call.  `grads` is the
    gradient of the MEAN OVER THE BATCH of `loss` -- the scalar the reference demo's `loss_fn` hands
    to `jax.value_and_grad` (`loss.mean()`) -- with respect to every parameter: a dict shaped like
    `params` ({module path: {"w", "b"} | {"scale", "offset"}}, float32 numpy arrays), with exact
    zeros for the parameters the step never reads (the mesh2grid mesh-node MLP).  The forward runs
    stage by stage on the device, the backward pass through the sm_90a kernels of the C ABI (see
    graphcast_b200/backward.py) in the model's precision ("bf16x3" or "bf16")."""
    return self._loss_and_grads(inputs, targets, forcings, norm=None)

  def _loss_and_grads(self, inputs, targets, forcings, norm: Optional[FusedNormalization]):
    def begin(eng, tangents):
      eng.grads_begin()
      return eng.loss_and_grads_element
    loss, diagnostics = self._param_call(
        inputs, targets, forcings, norm, "parameter gradients cover one target time (no backprop "
        "through time)", None, begin)
    return loss, diagnostics, self._export_grads()

  def _param_call(self, inputs, targets, forcings, norm: Optional[FusedNormalization], refusal: str,
                  param_tangents, begin):
    """The calls of one target time that accumulate in the engine's gradient accumulators
    (loss_and_grads, loss_and_param_gnvp, loss_and_param_hvp), up to what they export.  Several target
    times raise NotImplementedError(refusal), and param_tangents (None: the call takes none) are
    checked, before anything runs.  Then `_call` runs begin(engine, checked tangents) once, which
    prepares the engine and returns its per-element call f(targets_planes, lat_weight, coef,
    channel_sums=..., **affine), and f for every batch element.  Returns (loss, diagnostics)."""
    inputs, targets = xs.from_xarray(inputs), xs.from_xarray(targets)
    if targets.sizes.get("time", 1) != 1:
      raise NotImplementedError(refusal)
    tangents = None if param_tangents is None else self._checked_param_tangents(param_tangents)
    slabs, coef = loss_coefficients(targets, inputs.sizes["lat"] * inputs.sizes["lon"],
                                    dict(inputs.sizes).get("batch", 1))
    run = lat_weight = coef_dev = None

    def start():
      nonlocal run, lat_weight, coef_dev
      eng = self._engine
      run = begin(eng, tangents)
      lat_weight, coef_dev = self._lat_weight(targets, eng.device), _device_coef(coef, eng.device)

    def element(b, planes_tgt, planes_out, channel_sums, affine):
      run(planes_tgt, lat_weight, coef_dev, channel_sums=channel_sums, **affine)

    self._call(inputs, targets, forcings, norm=norm, targets=targets, predictions=False, begin=start,
               element=element)
    run = coef_dev = None                  # with the weight tangents the element call holds
    return self._losses(slabs)

  def loss_and_input_grads(self, inputs, targets, forcings, **unused_kwargs):
    """(loss, diagnostics, input_grads, forcing_grads) for one target time.

    `loss` and `diagnostics` are exactly what `loss()` returns for the same call.  `input_grads` and
    `forcing_grads` are the gradient of loss.mean() (the scalar of loss_and_grads) with respect to
    every data variable of `inputs` and of `forcings`: float32 Datasets with their variables, dims and
    coords, in the variables' physical units.  A variable the packing broadcast over batch, lat or lon
    gets the sum over those axes.  The backward pass is Backward.element(param_grads=False) in the
    model's precision, seeded and carried over every input channel (feedback.FeedbackPlan
    .all_channels); the parameter gradients are neither computed nor touched."""
    return self._loss_and_input_grads(inputs, targets, forcings, norm=None)

  def loss_and_input_hvp(self, inputs, targets, forcings, input_tangents, forcing_tangents=None,
                         **unused_kwargs):
    """(loss, diagnostics, input_grads, forcing_grads, input_hvp, forcing_hvp) for one target time:
    what jax.jvp(jax.grad(loss), (x,), (v,)) gives, with the loss and gradient of loss_and_input_grads.

    `loss`, `diagnostics`, `input_grads` and `forcing_grads` are bit for bit what loss_and_input_grads
    returns.  `input_hvp` and `forcing_hvp` (float32, shaped like `inputs` and `forcings`, physical
    units) are H v, H the Hessian of loss.mean() with respect to every variable of the inputs and
    forcings and v = (input_tangents, forcing_tangents); the tangents are Datasets as input_jvp takes
    them, a variable left out (every forcing for forcing_tangents=None) being zero.  Variables the
    packing broadcast are summed as in loss_and_input_grads.  Every refusal of loss_and_input_grads and
    of input_jvp's tangents applies, before anything runs.

    The forward runs stage by stage with its tangent (Backward.tangent), keeping the tangent state the
    backward walk reads; the gradient and its tangent then share one backward walk
    (Backward.element(hvp=...)), forward-over-reverse: one forward, one tangent and one two-direction
    backward pass in place of the two gradients of a central difference."""
    return self._loss_and_input_grads(inputs, targets, forcings, norm=None,
                                      tangents=(input_tangents, forcing_tangents))

  def batched_loss_and_input_hvp(self, inputs, targets, forcings, input_tangents, forcing_tangents=None,
                                 *, directions_per_pass=None, **unused_kwargs):
    """(loss, diagnostics, input_grads, forcing_grads, input_hvp, forcing_hvp) of loss_and_input_hvp
    along K tangent directions at once, for one target time: what jax.vmap over the tangents of
    jax.jvp(jax.grad(loss), (x,), (v,)) gives.

    Every variable of input_tangents / forcing_tangents has a leading "direction" dim of size K >= 1,
    followed by its namesake's dims and shape; a variable left out (every forcing for
    forcing_tangents=None) is zero in every direction.  A missing direction dim, K differing between
    variables or Datasets, an unknown variable or a wrong shape and a bad directions_per_pass raise
    ValueError before anything runs, and every refusal of loss_and_input_hvp applies.  `loss`,
    `diagnostics`, `input_grads` and `forcing_grads` are bit for bit what loss_and_input_grads returns
    (no direction dim); input_hvp and forcing_hvp (float32) are shaped like `inputs` and `forcings` with
    a leading "direction" dim, its coordinate input_tangents' "direction" coordinate when it has one,
    else 0..K-1.  Direction k is bit for bit loss_and_input_hvp along tangent k alone, for any K and
    directions_per_pass.

    The directions share one stage-wise forward with their K tangents and one backward walk of 1 + K
    directions, the gradient and its K tangents (Backward.element(dirs=1 + K, hvp=...)): every GEMM
    streams its weights once for all of them, and every MLP's h and z recomputes, the embedder
    recomputes and the edge projections are formed once; the two coupled nonlinearities form their
    primal terms once per element.  directions_per_pass = g (None: K) runs ceil(K / g) such passes,
    each what a g-direction call runs, for memory: the kept tangent tables and the stacked gradient
    state grow with the directions of a pass.  The loss, diagnostics and gradients are the first
    pass's (every pass forms the same bits).  Measured on an 80 GB H100 at 1 degree / 13 levels
    (DESIGN.md section 8): a pass peaks at 15.4 GiB for one direction and 56.0 GiB for 8, about 5.8 GiB
    per further direction (3.5 GiB of it the kept tangent tables), so about 11 directions fit per pass
    (16 do not); 8 directions take 1.87x (T = 1) and 2.02x (T = 4) less time than 8 loss_and_input_hvp
    calls.  0.25 degree / 37 levels is not measured: one direction is not expected to fit there."""
    one_pass = lambda it, ft: self._loss_and_input_grads(inputs, targets, forcings, norm=None,
                                                         tangents=(it, ft), directions=True)
    return batched_hvp(one_pass, inputs, forcings, input_tangents, forcing_tangents,
                       directions_per_pass)

  def input_vjp(self, inputs, targets_template, forcings, cotangents, **unused_kwargs):
    """(predictions, input_grads, forcing_grads) for one target time: `predictions` is what __call__
    returns, bit for bit; the gradients (as in loss_and_input_grads) are those of
    J = sum over variables, batch, time, level, lat and lon of cotangents * predictions, with
    `cotangents` a Dataset shaped like `targets_template`."""
    return self._input_vjp(inputs, targets_template, forcings, cotangents, norm=None)

  def batched_input_vjp(self, inputs, targets_template, forcings, cotangents, *,
                        directions_per_pass=None, **unused_kwargs):
    """(predictions, input_grads, forcing_grads) of input_vjp for K cotangents at once, for one target
    time: what jax.vmap of the vjp function of jax.vjp over the cotangents gives.

    Every variable of `cotangents` has a leading "direction" dim of size K >= 1, followed by the shape
    of the `targets_template` variable of the same name; the variables are the template's.  A missing
    direction dim, K differing between variables, a wrong variable set or shape and a bad
    directions_per_pass raise ValueError before anything runs, and every refusal of input_vjp applies.
    `predictions` is what __call__ returns, bit for bit; input_grads and forcing_grads (float32) are
    shaped like `inputs` and `forcings` with a leading "direction" dim, its coordinate the cotangents'
    "direction" coordinate when they have one, else 0..K-1.  Direction k is bit for bit input_vjp with
    cotangent k alone, for any K and directions_per_pass.

    The directions share one stage-wise forward and one backward walk (Backward.element(dirs=K)): the
    gradient state is stacked direction-major, so every dX product streams its weights once for all of
    them and every MLP's h and z, the embedder recomputes and the edge projections are formed once; the
    seed, segment sums and input reductions run per direction.  directions_per_pass = g (None: K) runs
    ceil(K / g) such passes, for memory: the stacked state, and the bipartite chunks' temporaries
    (the chunks are those of one direction, whose boundaries the sender sums depend on), grow with the
    directions of a pass.  Measured on an 80 GB H100 (DESIGN.md section 8): at 0.25 degree / 37 levels
    input_vjp already peaks at 73.8 GiB, so run one direction per pass there (directions_per_pass=1),
    which peaks as input_vjp does (but measured slower than K input_vjp calls there, 0.69x at T = 1); at
    1 degree / 13 levels a pass peaks at 9.9 GiB for one direction and 33.9 GiB for 16, about 1.6 GiB per
    further direction, so about 40 fit, and 8 directions take 1.71x less time than 8 input_vjp calls."""
    if xs.from_xarray(targets_template).sizes.get("time", 1) != 1:
      raise NotImplementedError("input gradients of GraphCast cover one target time (several: "
                                "autoregressive.Predictor with gradient_checkpointing=True)")
    one_pass = lambda cot, first: self._input_vjp(inputs, targets_template, forcings, cot, norm=None,
                                                  directions=True, predictions=first)
    return batched_vjp(one_pass, targets_template, cotangents, directions_per_pass)

  def input_jvp(self, inputs, targets_template, forcings, input_tangents, forcing_tangents=None,
                **unused_kwargs):
    """(predictions, prediction_tangents) for one target time: `predictions` is what __call__ returns,
    bit for bit; `prediction_tangents` (float32, shaped like it) is d(predictions)/d eps at eps = 0 for
    the inputs + eps * input_tangents and forcings + eps * forcing_tangents, what jax.jvp of the
    predictor gives.  The tangent Datasets hold variables of `inputs` / `forcings` with their dims and
    shapes, in physical units; a variable left out (every forcing for forcing_tangents=None) is held
    fixed.  An unknown variable or a wrong shape raises ValueError before anything runs.  The tangent
    runs forward with the step, stage by stage (Backward.tangent), in the model's precision."""
    run = self._one_step_tangents(inputs, targets_template, forcings, input_tangents,
                                  forcing_tangents)
    return self._input_jvp(inputs, targets_template, forcings, run, norm=None)

  def batched_input_jvp(self, inputs, targets_template, forcings, input_tangents,
                        forcing_tangents=None, *, directions_per_pass=None, **unused_kwargs):
    """(predictions, prediction_tangents) of input_jvp along K tangent directions at once, for one
    target time: what jax.vmap of jax.jvp over the directions gives.

    Every variable of input_tangents / forcing_tangents has a leading "direction" dim of size K >= 1,
    followed by its namesake's dims and shape; a variable left out (every forcing for
    forcing_tangents=None) is held fixed in every direction.  A missing direction dim, K differing
    between variables or Datasets, an unknown variable or a wrong shape raise ValueError before anything
    runs, and every refusal of input_jvp applies.  `predictions` is what __call__ returns, bit for bit;
    `prediction_tangents` (float32) has a leading "direction" dim followed by the predictions' dims, its
    coordinate input_tangents' "direction" coordinate when it has one, else 0..K-1.  Direction k is
    bit for bit input_jvp along direction k alone, for any K and directions_per_pass.

    The directions share one stage-wise forward: their tangent state is stacked direction-major
    (Backward.tangent), so every tangent GEMM streams its weights once for all of them and every MLP's
    h and z are recomputed once.  directions_per_pass = g (None: K) runs ceil(K / g) such passes, for
    memory.  Measured on an 80 GB H100 (DESIGN.md section 8): at 0.25 degree / 37 levels a pass peaks
    at 57.4 GiB for one direction and 68.7-69.6 GiB for two, 11.3-12.2 GiB per direction, so at most
    2 directions fit per pass; at 1 degree / 13 levels 16 directions peak at 17.6 GiB (T = 4), about
    0.8 GiB per direction, so about 90 fit."""
    def one_pass(it, ft):
      run = self._one_step_tangents(inputs, targets_template, forcings, it, ft, directions=True)
      return self._input_jvp(inputs, targets_template, forcings, run, norm=None)
    return batched_jvp(one_pass, inputs, forcings, input_tangents, forcing_tangents,
                       directions_per_pass)

  def param_jvp(self, inputs, targets_template, forcings, param_tangents, **unused_kwargs):
    """(predictions, prediction_tangents) for one target time: `predictions` is what __call__ returns,
    bit for bit; `prediction_tangents` (float32, shaped like it, physical units) is d(predictions)/d eps
    at eps = 0 for the params + eps * param_tangents, what jax.jvp of the predictor with respect to the
    params gives (several target times: autoregressive.Predictor).

    `param_tangents` is a dict shaped like the params, {module path: {field: array}} with each array
    the shape of its parameter (cast to float32); a module or field left out is zero.  A non-mapping,
    an unknown module or field and a wrong shape raise ValueError, and the fp32_simt precision
    NotImplementedError, before anything runs.  The tangents are packed once per call into tangent
    weight images at the model's precision (Engine.weight_tangents); the engine's weights are not
    touched.  The tangent runs forward with the step, stage by stage (Backward.tangent(wts=...)):
    every layer adds X W-dot + b-dot to the tangent of its input's term, every LayerNorm
    scale-dot * zhat + offset-dot, and the mesh-node encoder, the edge embedders and the processor's
    e_0 get the tangents their parameters give them.  A module with no tangent costs no extra GEMM."""
    run = self._param_tangent_run(inputs, targets_template, forcings, param_tangents, num_steps=1)
    return self._input_jvp(inputs, targets_template, forcings, run, norm=None)

  def loss_and_param_gnvp(self, inputs, targets, forcings, param_tangents, **unused_kwargs):
    """(loss, diagnostics, gnvp) for one target time.

    `loss` and `diagnostics` are bit for bit what `loss()` returns.  `gnvp` is G v = J^T H J v, the
    generalised Gauss-Newton matrix of loss.mean() (the scalar of loss_and_grads) with respect to the
    params times v = param_tangents (a dict as param_jvp takes it): J the Jacobian of the decoder output
    y with respect to the params and H = diag(coef * lat_weight) the Hessian of the loss, a quadratic
    in y.  It is a dict shaped like the params, float32 numpy arrays as loss_and_grads returns `grads`,
    with exact zeros for the mesh2grid mesh-node MLP, which the step never reads; a batch averages over
    its elements as loss_and_grads does.  Where the predictions equal the targets the residual term of
    the Hessian vanishes, and G v is the full parameter Hessian times v.  Every refusal of param_jvp
    and loss_and_grads applies, before anything runs.

    Per batch element: the step with its tangent along v (param_jvp's forward), the seed
    coef * lat_weight * y-dot (gcb_output_loss_gn_seed), then the parameter backward pass of
    loss_and_grads from that seed, which recomputes the step with its snapshots."""
    return self._loss_and_param_gnvp(inputs, targets, forcings, param_tangents, norm=None)

  def loss_and_param_hvp(self, inputs, targets, forcings, param_tangents, **unused_kwargs):
    """(loss, diagnostics, grads, hvp) for one target time: what jax.jvp(jax.grad(loss), (params,),
    (v,)) gives, with the loss and gradient of loss_and_grads.

    `loss` and `diagnostics` are bit for bit what `loss()` returns, `grads` what loss_and_grads
    returns.  `hvp` is H v, H the Hessian of loss.mean() (the scalar of loss_and_grads; a batch
    averages over its elements) with respect to the params and v = param_tangents (a dict as param_jvp
    takes it, modules and fields left out being zero): a dict shaped like the params, float32 numpy
    arrays, with exact zeros for the mesh2grid mesh-node MLP, which the step never reads.  Unlike
    loss_and_param_gnvp's G v it keeps the residual term, the loss residual times the network's second
    derivatives.  Every refusal of param_jvp and loss_and_grads applies, before anything runs;
    several target times raise NotImplementedError.

    Per batch element (Engine.param_hvp_element): one forward with the tangent along v that keeps its
    tangent tables, then one backward walk of two directions, the gradient and its tangent, which
    accumulates both the parameter gradients and their tangents."""
    return self._loss_and_param_hvp(inputs, targets, forcings, param_tangents, norm=None)

  def _loss_and_param_hvp(self, inputs, targets, forcings, param_tangents,
                          norm: Optional[FusedNormalization]):
    def begin(eng, tangents):
      eng.param_hvp_begin()
      self._release_idle_staging()
      return functools.partial(eng.param_hvp_element,
                               weight_tangents=eng.weight_tangents(tangents, transposed=True))
    loss, diagnostics = self._param_call(
        inputs, targets, forcings, norm, "parameter Hessian-vector products cover one target time "
        "(several are not provided)", param_tangents, begin)
    return (loss, diagnostics, _host_grads(self._engine.grads()),
            _host_grads(self._engine.param_hvp()))

  def loss_and_joint_hvp(self, inputs, targets, forcings, param_tangents=None, input_tangents=None,
                         forcing_tangents=None, **unused_kwargs):
    """(loss, diagnostics, grads, input_grads, forcing_grads, param_hvp, input_hvp, forcing_hvp) for
    one target time: what jax.jvp(jax.grad(loss, argnums=(params, inputs)), ...) gives along
    (param_tangents, input and forcing tangents), with the Hessian's mixed blocks.

    `loss` and `diagnostics` are bit for bit what `loss()` returns, `grads` what loss_and_grads returns
    and `input_grads` / `forcing_grads` what loss_and_input_grads returns.  With H the Hessian of
    loss.mean() in (params, inputs and forcings) and v = (v_theta, v_x) the tangents, `param_hvp` is
    H_theta,theta v_theta + H_theta,x v_x, a dict shaped like the params (float32 numpy, exact zeros for
    the mesh2grid mesh-node MLP), and `input_hvp` / `forcing_hvp` are H_x,theta v_theta + H_x,x v_x,
    float32 Datasets shaped like `inputs` and `forcings` in physical units (variables the packing
    broadcast summed as in loss_and_input_grads).  param_tangents is checked as loss_and_param_hvp
    checks it, the input and forcing tangents as loss_and_input_hvp checks them; what a tangent leaves
    out (all of it for None) is zero.  Every refusal of loss_and_param_hvp applies, before anything
    runs.

    Per batch element (Engine.joint_hvp_element): one forward with its tangent along both v_theta and
    v_x that keeps its tangent tables, then one backward walk of two directions, the gradient and its
    tangent, which accumulates the parameter side and forms the input side."""
    tangents = self._joint_hvp_tangents(inputs, targets, forcings, param_tangents, input_tangents,
                                        forcing_tangents)
    return self._loss_and_joint_hvp(inputs, targets, forcings, tangents, norm=None)

  def _joint_hvp_tangents(self, inputs, targets, forcings, param_tangents, input_tangents,
                          forcing_tangents):
    """The checks of loss_and_joint_hvp, before anything runs: one target time, the parameter tangents
    (_checked_param_tangents; None: none) and the input and forcing tangents (hvp_tangent_planes).
    Returns (checked parameter tangents, [batch, c_in, Ng] host tangent planes)."""
    if xs.from_xarray(targets).sizes.get("time", 1) != 1:
      raise NotImplementedError("joint Hessian-vector products cover one target time (several are "
                                "not provided)")
    return (self._checked_param_tangents({} if param_tangents is None else param_tangents),
            hvp_tangent_planes(xs.from_xarray(inputs), xs.from_xarray(forcings), input_tangents,
                               forcing_tangents))

  def _loss_and_joint_hvp(self, inputs, targets, forcings, tangents,
                          norm: Optional[FusedNormalization]):
    """loss_and_joint_hvp of the checked tangents of _joint_hvp_tangents."""
    inputs, targets = xs.from_xarray(inputs), xs.from_xarray(targets)
    forcings = xs.from_xarray(forcings)
    param_tangents, planes = tangents
    slabs, coef = loss_coefficients(targets, inputs.sizes["lat"] * inputs.sizes["lon"],
                                    dict(inputs.sizes).get("batch", 1))
    run = self._one_step_input_grads(inputs, targets, forcings, norm, targets=targets, coef=coef,
                                     tangent_planes=planes, param_tangents=param_tangents)
    input_grads, forcing_grads, input_hvp, forcing_hvp = run.finish()
    del run                                # with the weight tangents it holds
    loss, diagnostics = self._losses(slabs)
    eng = self._engine
    return (loss, diagnostics, _host_grads(eng.grads()), input_grads, forcing_grads,
            _host_grads(eng.param_hvp()), input_hvp, forcing_hvp)

  def _param_tangent_run(self, inputs, targets_template, forcings, param_tangents, num_steps: int,
                         plan=None) -> "_TangentRun":
    """The checked parameter tangents of a param_jvp of `num_steps` target times, as a _TangentRun of
    zero input tangents; raises before anything runs."""
    inputs, forcings = xs.from_xarray(inputs), xs.from_xarray(forcings)
    if num_steps == 1 and xs.from_xarray(targets_template).sizes.get("time", 1) != 1:
      raise NotImplementedError("param_jvp of GraphCast covers one target time (several: "
                                "autoregressive.Predictor)")
    tangents = self._checked_param_tangents(param_tangents)
    run = _TangentRun(inputs, forcings, None, None, num_steps=num_steps, plan=plan)
    run.param_tangents = tangents
    return run

  def _checked_param_tangents(self, param_tangents) -> Dict[str, Dict[str, np.ndarray]]:
    """param_tangents checked against the params (check_param_tangents) and the precision."""
    if self._precision not in ("bf16x3", "bf16"):
      raise NotImplementedError(f"parameter tangents support the tensor-core precisions 'bf16x3' and "
                                f"'bf16', not {self._precision!r}")
    if self._params is None:
      raise ValueError("GraphCast has no parameters: pass params= or call set_params()")
    return check_param_tangents(param_tangents, self._params)

  def _loss_and_param_gnvp(self, inputs, targets, forcings, param_tangents,
                           norm: Optional[FusedNormalization]):
    def begin(eng, tangents):
      eng.grads_begin()
      self._release_idle_staging()
      return functools.partial(eng.param_gnvp_element, weight_tangents=eng.weight_tangents(tangents))
    loss, diagnostics = self._param_call(
        inputs, targets, forcings, norm, "Gauss-Newton products cover one target time (several are "
        "not provided)", param_tangents, begin)
    return loss, diagnostics, _host_grads(self._engine.grads())

  @staticmethod
  def _one_step_tangents(inputs, targets_template, forcings, input_tangents,
                         forcing_tangents, directions: bool = False) -> "_TangentRun":
    """The checked and packed tangents of an input_jvp (with `directions`: batched_input_jvp) of one
    target time."""
    if xs.from_xarray(targets_template).sizes.get("time", 1) != 1:
      raise NotImplementedError("input_jvp of GraphCast covers one target time (several: "
                                "autoregressive.Predictor)")
    return _TangentRun(xs.from_xarray(inputs), xs.from_xarray(forcings), input_tangents,
                       forcing_tangents, num_steps=1, directions=directions)

  def _input_jvp(self, inputs, targets_template, forcings, run: "_TangentRun",
                 norm: Optional[FusedNormalization]):
    """input_jvp of one step, the tangent planes carried by `run` (from the step before, in a
    rollout).  `_call` stages the planes once and, for every batch element, runs the stage-wise
    forward and its tangent (Engine.input_jvp_element) in place of its step."""
    inputs, forcings = xs.from_xarray(inputs), xs.from_xarray(forcings)
    targets_template = xs.from_xarray(targets_template)
    out = None

    def begin():
      nonlocal out
      eng = self._engine
      eng.input_grads_begin("input gradients" if run.param_tangents is None else "parameter tangents")
      self._release_idle_staging()
      out = torch.empty([run.dirs, run.batch, eng.n_out, eng.num_grid], dtype=torch.float32,
                        device=eng.device)

    def element(b, planes_tgt, planes_out, channel_sums, affine):
      run.element(self._engine, b, out[:, b], planes_out, norm, affine)

    predictions = self._call(inputs, targets_template, forcings, norm=norm, begin=begin,
                             element=element)
    run.step += 1
    if not run.directions:
      return predictions, self._planes_to_dataset(out[0], targets_template, run.n_lat, run.n_lon)
    return predictions, self._planes_to_dataset(out, targets_template, run.n_lat, run.n_lon,
                                                directions=run.labels)

  def _loss_and_input_grads(self, inputs, targets, forcings, norm: Optional[FusedNormalization],
                            tangents=None, directions: bool = False):
    """loss_and_input_grads of one target time; with tangents = (input_tangents, forcing_tangents),
    loss_and_input_hvp; with `directions` too, batched_loss_and_input_hvp of one pass, the tangents
    carrying a leading "direction" dim (hvp_direction_tangent_planes)."""
    inputs, targets = xs.from_xarray(inputs), xs.from_xarray(targets)
    forcings = xs.from_xarray(forcings)
    if targets.sizes.get("time", 1) != 1:
      raise NotImplementedError("input gradients of GraphCast cover one target time (several: "
                                "autoregressive.Predictor with gradient_checkpointing=True)")
    tangent = None
    if tangents is not None:
      pack = hvp_direction_tangent_planes if directions else hvp_tangent_planes
      tangent = pack(inputs, forcings, *tangents)
    slabs, coef = loss_coefficients(targets, inputs.sizes["lat"] * inputs.sizes["lon"],
                                    dict(inputs.sizes).get("batch", 1))
    run = self._one_step_input_grads(inputs, targets, forcings, norm, targets=targets, coef=coef,
                                     tangent_planes=tangent)
    return self._losses(slabs) + run.finish()

  def _input_vjp(self, inputs, targets_template, forcings, cotangents,
                 norm: Optional[FusedNormalization], directions: bool = False,
                 predictions: bool = True):
    """input_vjp of one target time; with `directions`, batched_input_vjp of one pass, the cotangents
    (checked) carrying a leading "direction" dim.  predictions=False: None in place of the predictions,
    which are then not unpacked."""
    inputs, forcings = xs.from_xarray(inputs), xs.from_xarray(forcings)
    targets_template = xs.from_xarray(targets_template)
    if targets_template.sizes.get("time", 1) != 1:
      raise NotImplementedError("input gradients of GraphCast cover one target time (several: "
                                "autoregressive.Predictor with gradient_checkpointing=True)")
    holder = {"predictions": None}
    run = self._one_step_input_grads(inputs, targets_template, forcings, norm, cotangents=cotangents,
                                     predictions=holder if predictions else None,
                                     directions=directions)
    return (holder["predictions"],) + run.finish()

  def _one_step_input_grads(self, inputs, template, forcings, norm, *, targets=None, coef=None,
                            cotangents=None, predictions=None, directions: bool = False,
                            tangent_planes: Optional[torch.Tensor] = None,
                            param_tangents=None) -> "_InputGradRun":
    """One target time: `_call` stages the planes once and, for every batch element, runs the
    stage-wise forward, the seed and the backward pass of Engine.input_grads_element in place of its
    step (no second forward, no host round trip).  With `targets` the loss sums land in
    self._channel_sums as in `loss`; with `cotangents`, predictions["predictions"] receives the
    predictions, unpacked from that forward as __call__ unpacks its step's; with `directions`, the
    cotangents have a leading "direction" dim and every direction shares that forward and backward
    pass; with `tangent_planes` ([batch, c_in, Ng] host planes of the input tangents, or [K, batch,
    c_in, Ng] for K directions, with `targets`) every element runs Engine.input_hvp_element, and with
    param_tangents as well (checked parameter tangents, one direction) Engine.joint_hvp_element, the
    parameter side accumulating in the engine (param_hvp_begin).  Returns the run, whose finish() gives
    (input_grads, forcing_grads), with tangent_planes followed by (input_hvp, forcing_hvp), these with
    a leading "direction" dim for K directions."""
    batch = dict(inputs.sizes).get("batch", 1)
    run = cot = lat_weight = coef_dev = None

    def begin():
      nonlocal run, cot, lat_weight, coef_dev
      eng = self._engine
      plan = feedback.FeedbackPlan.all_channels(inputs, template, forcings)
      dirs = None
      if directions:
        cot = self._direction_cotangent_planes(cotangents, template, batch)
        dirs = cot.shape[0]
      if param_tangents is not None:         # zeroes both accumulator sets before the run is built
        eng.param_hvp_begin()
      run = _InputGradRun(self, plan, norm, inputs, forcings, 1, batch, release_staging=False,
                          dirs=dirs, hvp=_hvp_directions(tangent_planes, 0))
      if param_tangents is not None:
        run.weight_tangents = eng.weight_tangents(param_tangents, transposed=True, input_grad=True)
      if cotangents is not None and not directions:
        cot = self._cotangent_planes(cotangents, template, batch)
      if targets is not None:
        lat_weight, coef_dev = self._lat_weight(targets, eng.device), _device_coef(coef, eng.device)

    def element(b, planes_tgt, planes_out, channel_sums, affine):
      eng = self._engine
      operands = dict(affine)
      if tangent_planes is not None and tangent_planes.dim() == 4:    # [K, batch, c_in, Ng]
        operands["tangent_planes"] = torch.empty(
            [tangent_planes.shape[0], eng.c_in, eng.num_grid], dtype=torch.float32, device=eng.device)
        operands["tangent_planes"].copy_(tangent_planes[:, b])
      elif tangent_planes is not None:
        operands["tangent_planes"] = tangent_planes[b].to(eng.device)
      if targets is not None:
        operands["targets_planes"] = planes_tgt
        kw = dict(lat_weight=lat_weight, coef=coef_dev, channel_sums=channel_sums)
      else:
        host = cot[:, b] if directions else cot[b]
        seed = torch.empty(list(host.shape), dtype=torch.float32, device=eng.device)
        seed.copy_(host)
        operands["cotangent"] = seed
        kw = {}
      run.element(b, 0, operands, planes_out=planes_out, **kw)

    out = self._call(inputs, template, forcings, norm=norm, targets=targets,
                     predictions=predictions is not None, begin=begin, element=element)
    if predictions is not None:
      predictions["predictions"] = out
    return run

  def _cotangent_planes(self, cotangents, template: xs.Dataset, batch: int,
                        out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """[batch, n_out, Ng] float32 host planes of a cotangent Dataset shaped like the one-step
    `template`, in the predictions' channel order (written into `out` when given)."""
    cotangents = xs.from_xarray(cotangents)
    slabs = self._check_template(template, self._engine.n_out)
    if set(cotangents.keys()) != set(template.keys()):
      raise ValueError(f"cotangents have the variables {sorted(cotangents.keys())}, the predictions "
                       f"{sorted(template.keys())}")
    n_lat, n_lon = template.sizes["lat"], template.sizes["lon"]
    sizes = {"batch": batch, "lat": n_lat, "lon": n_lon}
    if out is None:
      out = torch.empty([batch, self._engine.n_out, n_lat * n_lon], dtype=torch.float32)
    for s in slabs:
      v = cotangents.data_vars[s.name]
      if tuple(v.shape) != tuple(template.data_vars[s.name].shape):
        raise ValueError(f"cotangent {s.name} has shape {tuple(v.shape)}, the prediction "
                         f"{tuple(template.data_vars[s.name].shape)}")
      src = model_utils.variable_to_planes(v.transpose(*template.data_vars[s.name].dims), sizes)
      out[:, s.start:s.start + s.count] = torch.as_tensor(
          np.asarray(src, np.float32)).reshape(batch, s.count, n_lat * n_lon)
    return out

  def _direction_cotangent_planes(self, cotangents, template: xs.Dataset, batch: int) -> torch.Tensor:
    """[K, batch, n_out, Ng] float32 host planes of cotangents with a leading "direction" dim, direction
    k packed as _cotangent_planes packs cotangent k alone."""
    cotangents = xs.from_xarray(cotangents)
    dirs = next(iter(cotangents.data_vars.values())).shape[0]
    out = torch.empty([dirs, batch, self._engine.n_out, self._engine.num_grid], dtype=torch.float32)
    for k in range(dirs):
      self._cotangent_planes(cotangents.isel({feedback.DIRECTION: k}), template, batch, out=out[k])
    return out

  def _input_grads(self, stash: "StepStash", plan, norm: Optional[FusedNormalization],
                   inputs: xs.Dataset, forcings: xs.Dataset, *, lat_weight=None, coef=None,
                   cotangents=None, directions: bool = False, tangents: Optional["StepStash"] = None):
    """Gradients with respect to the inputs and forcings of the steps `stash` holds (several target
    times): for every batch element, last step first, the step's planes are uploaded again, packed
    and differentiated by Engine.input_grads_element with the all-channel feedback `plan` of the
    following step.  The seed is the loss (lat_weight, coef; the stash holds the target planes) or,
    with `cotangents` (per step [batch, n_out, Ng] host planes), J = sum cotangents * predictions;
    with `directions`, per step [K, batch, n_out, Ng] planes of K cotangents that share every step's
    backward pass.  The stash is only read, so several calls can differentiate the same forward.
    Returns (input_grads, forcing_grads) Datasets shaped like `inputs` and `forcings` (with a leading
    "direction" dim for `directions`).  With `tangents` (a StepStash of each step's input tangent planes
    [batch, c_in, Ng], or [batch, K, c_in, Ng] for K directions; loss seed only) every step runs
    Engine.input_hvp_element, and (input_hvp, forcing_hvp) follow the gradients, with a leading
    "direction" dim for K directions."""
    run = _InputGradRun(self, plan, norm, inputs, forcings, len(stash.steps), stash.batch,
                        release_staging=True,
                        dirs=cotangents[0].shape[0] if directions else None,
                        hvp=None if tangents is None else _hvp_directions(tangents.steps[0][0][0], 1))
    eng = self._engine
    dev = eng.device
    coef_dev = None if coef is None else _device_coef(coef, dev)
    compute = torch.cuda.current_stream(dev)
    for b in range(run.batch):
      for t in range(run.num_steps - 1, -1, -1):
        saved, done = stash.steps[t]
        compute.wait_event(done)
        # The step's planes and seed live in `operands` only: the engine drops them after the seed,
        # so the backward pass reuses their 2.9 GB (0.25 degree).
        operands = {"planes": torch.empty([eng.c_in, eng.num_grid], dtype=torch.float32, device=dev)}
        operands["planes"].copy_(saved[0][b], non_blocking=True)
        operands.update(self._pack(eng, operands.pop("planes"), norm))
        if tangents is not None:
          (host_tangent,), tangent_done = tangents.steps[t]
          compute.wait_event(tangent_done)
          operands["tangent_planes"] = torch.empty(list(host_tangent[b].shape), dtype=torch.float32,
                                                   device=dev)
          operands["tangent_planes"].copy_(host_tangent[b], non_blocking=True)
        lead = [cotangents[t].shape[0]] if directions else []
        seed = torch.empty(lead + [eng.n_out, eng.num_grid], dtype=torch.float32, device=dev)
        if cotangents is None:
          seed.copy_(saved[1][b], non_blocking=True)
          operands["targets_planes"] = seed
          kw = dict(lat_weight=lat_weight, coef=coef_dev)
        else:
          seed.copy_(cotangents[t][:, b] if directions else cotangents[t][b])
          operands["cotangent"] = seed
          kw = {}
        del seed
        run.element(b, t, operands, **kw)
    return run.finish()

  def _export_grads(self):
    """The engine's accumulated gradients as host numpy dicts, or, with a _grad_sink, whatever the
    sink returns after taking them on the device."""
    if self._grad_sink is not None:
      return self._grad_sink(self._engine)
    return _host_grads(self._engine.grads())

  def _stash_step(self, stash: "StepStash") -> None:
    """Keeps the input and target planes of the last `_call` (with targets) in pinned host memory."""
    stash.save(self._planes_in, self._planes_tgt)

  def _release_staging(self) -> None:
    """Before a backward pass that reads its steps from a StepStash: the rollout's staging buffers are
    not needed any more, their memory goes to the backward pass."""
    self._planes_bufs, self._target_bufs, self._buf_free = [None, None], [None, None], [None, None]
    self._planes_in = self._planes_tgt = None
    # Return the rollout's cached blocks to the driver, so that the backward pass allocates from an
    # unfragmented pool: at 0.25 degree it peaks within a few GiB of an 80 GB card's capacity, and a
    # second call would otherwise find its 1 GiB tables only in the gaps the first one left.
    torch.cuda.empty_cache()

  def _release_idle_staging(self) -> None:
    """Inside a `_call`: drops the staging slot the call does not use (the one the next call would
    stage into), for a backward pass that runs inside the call.  Its blocks stay in the allocator's
    cache, where the backward pass's rows of the same size reuse them: emptying the cache here would
    cost 0.5 s at 0.25 degree."""
    idle = self._call_index % 2
    self._planes_bufs[idle] = self._target_bufs[idle] = self._buf_free[idle] = None

  def _bptt_grads(self, stash: "StepStash", plan, norm: Optional[FusedNormalization],
                  lat_weight: torch.Tensor, coef: np.ndarray,
                  pred_tangents: Optional["StepStash"] = None):
    """Parameter gradients of the multi-step loss whose steps `stash` holds (backprop through time,
    see autoregressive.Predictor.loss_and_grads).  For every batch element, last step first: the
    step's planes are uploaded again, packed and differentiated by Engine.loss_and_grads_element with
    the feedback of the following step; the gradients accumulate in this fixed order.

    With pred_tangents (a StepStash of each step's prediction tangents [batch, n_out, Ng] along the
    parameter tangents; autoregressive.Predictor.loss_and_param_gnvp) the result is the Gauss-Newton
    product instead: each step's tangent is uploaded in place of its target planes and seeds
    Engine.param_gnvp_bptt_element, the rest of the walk unchanged."""
    eng = self._engine
    dev = eng.device
    eng.grads_begin()
    fb = eng.feedback(plan, None if norm is None else norm.add_plane_index,
                      None if norm is None else norm.in_scale)
    self._release_staging()
    planes = torch.empty([eng.c_in, eng.num_grid], dtype=torch.float32, device=dev)
    tgt = torch.empty([eng.n_out, eng.num_grid], dtype=torch.float32, device=dev)
    scratch = torch.empty([eng.n_out], dtype=torch.float64, device=dev)
    coef_dev = _device_coef(coef, dev)
    compute = torch.cuda.current_stream(dev)
    for b in range(stash.batch):
      fb.a = None
      for t in range(len(stash.steps) - 1, -1, -1):
        (host_in, host_tgt), done = stash.steps[t]
        compute.wait_event(done)
        planes.copy_(host_in[b], non_blocking=True)
        if pred_tangents is None:
          tgt.copy_(host_tgt[b], non_blocking=True)
        else:
          (host_tangent,), tangent_done = pred_tangents.steps[t]
          compute.wait_event(tangent_done)
          tgt.copy_(host_tangent[b], non_blocking=True)
        affine = self._pack(eng, planes, norm)
        if pred_tangents is None:
          eng.loss_and_grads_element(tgt, lat_weight, coef_dev, channel_sums=scratch, feedback=fb,
                                     input_grad=t > 0, **affine)
        else:
          eng.param_gnvp_bptt_element(tgt, lat_weight, coef_dev, feedback=fb, input_grad=t > 0,
                                      scale=affine.get("scale"))
    return self._export_grads()

  def _loss(self, inputs, targets, forcings, norm: Optional[FusedNormalization], predictions: bool):
    finish, preds, sums = self._device_loss(inputs, targets, forcings, norm, predictions)
    return finish(sums.cpu().numpy()), preds

  def _device_loss(self, inputs, targets, forcings, norm: Optional[FusedNormalization],
                   predictions: bool):
    """Queues one step with the fused loss of every batch element and returns
    (finish, predictions or None, channel_sums): `channel_sums` [batch, n_out] fp64 on the device
    receives the latitude-weighted squared-error sums of gcb_output_loss, and
    finish(host copy of those sums) -> (loss, diagnostics).  Nothing is synchronised here, so a
    multi-step loss reads all its sums back once."""
    targets = xs.from_xarray(targets)
    preds = self._call(inputs, targets, forcings, norm=norm, targets=targets,
                       predictions=predictions)
    slabs = model_utils.channel_layout(targets)
    return (lambda sums: self._losses(slabs, sums)), preds, self._channel_sums

  def _losses(self, slabs, sums: Optional[np.ndarray] = None):
    """(loss, diagnostics), as `loss` returns them, of the host channel sums [batch, n_out] of targets
    laid out as `slabs`; by default those of the last call, read back from self._channel_sums."""
    if sums is None:
      sums = self._channel_sums.cpu().numpy()
    return losses.losses_from_channel_sums(sums, slabs, self._engine.num_grid,
                                           LOSS_PER_VARIABLE_WEIGHTS)

  def _device_loss_tangent(self, inputs, targets, forcings, norm: Optional[FusedNormalization],
                           run: "_TangentRun", keep_predictions: bool = False):
    """_device_loss with the tangent planes of `run` carried through the step (the forward of
    loss_and_input_hvp over several target times): every batch element runs the stage-wise forward with
    its tangent (_TangentRun.element, which also feeds the next step's tangent planes), then
    output_loss on that forward, which is the step _device_loss runs.  Returns (finish, predictions,
    channel_sums, this step's input tangent planes on the device: [batch, c_in, Ng] for a run of one
    direction, [batch, K, c_in, Ng] for a run of K (`run.directions`)).  keep_predictions (a run of one
    direction; loss_and_param_gnvp): this step's prediction tangents [batch, n_out, Ng] in their place."""
    targets = xs.from_xarray(targets)
    planes = lat_weight = None

    def begin():
      nonlocal planes, lat_weight
      eng = self._engine
      eng.input_grads_begin()
      lead = [run.dirs] if run.directions else []
      rows = eng.n_out if keep_predictions else eng.c_in
      planes = torch.empty([run.batch] + lead + [rows, eng.num_grid], dtype=torch.float32,
                           device=eng.device)
      lat_weight = self._lat_weight(targets, eng.device)

    def element(b, planes_tgt, planes_out, channel_sums, affine):
      eng = self._engine
      tangent_out = torch.empty([run.dirs, eng.n_out, eng.num_grid], dtype=torch.float32,
                                device=eng.device)
      keep = None if keep_predictions else (
          lambda p: planes[b].copy_(p if run.directions else p[0]))
      run.element(eng, b, tangent_out, None, norm, affine, keep=keep)
      if keep_predictions:
        planes[b].copy_(tangent_out[0])
      eng.output_loss(planes_tgt, lat_weight, channel_sums=channel_sums, planes_out=planes_out,
                      **affine)

    preds = self._call(inputs, targets, forcings, norm=norm, targets=targets, predictions=True,
                       begin=begin, element=element)
    run.step += 1
    slabs = model_utils.channel_layout(targets)
    return (lambda sums: self._losses(slabs, sums)), preds, self._channel_sums, planes

  def _lat_weight(self, targets: xs.Dataset, device) -> torch.Tensor:
    """Normalised latitude weights of the targets' grid (float32, on the device), cached."""
    name = sorted(targets.data_vars.keys())[0]
    w = losses.normalized_latitude_weights(targets[name])
    w = np.ascontiguousarray(w, np.float32)
    key = (w.tobytes(), str(device))
    if self._lat_weight_cache is None or self._lat_weight_cache[0] != key:
      self._lat_weight_cache = (key, torch.as_tensor(w).to(device))
    return self._lat_weight_cache[1]

  def _channel_plan(self, inputs: xs.Dataset, forcings: xs.Dataset):
    in_slabs = model_utils.channel_layout(inputs)
    n_in = sum(s.count for s in in_slabs)
    f_slabs = model_utils.channel_layout(forcings, start=n_in)
    return in_slabs, f_slabs, n_in + sum(s.count for s in f_slabs)

  def _staging(self, bufs: List[Optional[torch.Tensor]], buf: int, shape) -> Tuple[torch.Tensor, bool]:
    fresh = bufs[buf] is None or bufs[buf].shape != shape
    if fresh:
      bufs[buf] = torch.empty(list(shape), dtype=torch.float32, device=self._engine.device)
    return bufs[buf], fresh

  def _call(self, inputs, targets_template, forcings, norm: Optional[FusedNormalization],
            targets: Optional[xs.Dataset] = None, predictions: bool = True, begin=None,
            element=None):
    """The step for every batch element.  With `targets` (shaped like the template, usually the
    same Dataset) the outputs go through gcb_output_loss instead of the plain unpack: the loss sums
    land in a new [batch, n_out] fp64 device tensor, self._channel_sums, and the predictions are
    returned only when `predictions` is set (else None).  With `element`, element(b, target planes or
    None, prediction planes or None, channel sums or None, affine keywords of _pack) replaces the
    step of every batch element after its inputs are packed (the derivative calls of one target
    time); begin() runs once before the first element, after the planes are staged and the engine
    exists."""
    inputs = xs.from_xarray(inputs)
    forcings = xs.from_xarray(forcings)
    targets_template = xs.from_xarray(targets_template)
    in_slabs, f_slabs, c_in = self._channel_plan(inputs, forcings)
    self._maybe_init(inputs, c_in)
    eng = self._engine
    sizes = dict(inputs.sizes)
    batch = sizes.get("batch", 1)
    sizes.setdefault("batch", batch)
    n_lat, n_lon = sizes["lat"], sizes["lon"]
    if n_lat * n_lon != eng.num_grid:
      raise ValueError("inputs lat/lon grid differs from the grid the model was built on")
    if targets is not None:
      t_slabs = self._check_template(targets, eng.n_out)
      lat_weight = self._lat_weight(targets, eng.device)
      if lat_weight.shape[0] != n_lat:
        raise ValueError(f"targets have {lat_weight.shape[0]} latitudes, the inputs {n_lat}")
      channel_sums = torch.empty([batch, eng.n_out], dtype=torch.float64, device=eng.device)
      self._channel_sums = channel_sums

    # xarray -> channel-major planes [B, C, lat*lon] on the device
    # (reference _inputs_to_grid_node_features :680-699; dataset_to_stacked order); the targets of a
    # loss are staged the same way, in the order of the predictions' channels.
    buf = self._call_index % 2
    self._call_index += 1
    planes_in, fresh = self._staging(self._planes_bufs, buf, (batch, c_in, eng.num_grid))
    self._planes_in = planes_in
    jobs = [(planes_in, inputs, in_slabs), (planes_in, forcings, f_slabs)]
    staged = [(planes_in, fresh)]
    if targets is not None:
      planes_tgt, fresh_tgt = self._staging(self._target_bufs, buf, (batch, eng.n_out, eng.num_grid))
      self._planes_tgt = planes_tgt
      jobs.append((planes_tgt, targets, t_slabs))
      staged.append((planes_tgt, fresh_tgt))
    if all(f for _, f in staged):
      self._buf_free[buf] = None
    sources = []
    for dst_planes, ds, slabs in jobs:
      for s in slabs:
        src = model_utils.variable_to_planes(ds.data_vars[s.name], sizes)
        if not isinstance(src, torch.Tensor):
          src = torch.from_numpy(np.ascontiguousarray(src, dtype=np.float32))
        sources.append((dst_planes, s, src))
    compute = torch.cuda.current_stream(eng.device)
    all_host = all(src.device.type == "cpu" for _, _, src in sources)
    if all_host:
      if self._h2d_stream is None:
        self._h2d_stream = torch.cuda.Stream(device=eng.device)
      copy_stream = self._h2d_stream
      for planes, f in staged:
        if f:
          # The caching allocator may hand back a block whose previous user still has kernels
          # queued on the compute stream: order the first copy after them, and tell the allocator
          # that the copy stream uses this block too.
          copy_stream.wait_stream(compute)
          planes.record_stream(copy_stream)
      if self._buf_free[buf] is not None:
        copy_stream.wait_event(self._buf_free[buf])      # kernels of call k-2 are done with it
    else:
      copy_stream = compute                              # device-resident inputs: stay in order
    with torch.cuda.stream(copy_stream):
      for dst_planes, s, src in sources:
        dst = dst_planes[:, s.start:s.start + s.count].view(batch, s.count, n_lat, n_lon)
        dst.copy_(src, non_blocking=True)
      if all_host:
        ready = torch.cuda.Event()
        ready.record(copy_stream)
    if all_host:
      compute.wait_event(ready)

    # Predictions are produced into fresh planes each call (they are handed out).
    planes_out = None
    if predictions:
      planes_out = torch.empty([batch, eng.n_out, eng.num_grid], dtype=torch.float32,
                               device=eng.device)
    if begin is not None:
      begin()
    for b in range(batch):
      affine = self._pack(eng, planes_in[b], norm)
      tgt = None if targets is None else planes_tgt[b]
      out = None if planes_out is None else planes_out[b]
      sums = None if targets is None else channel_sums[b]
      if element is not None:
        element(b, tgt, out, sums, affine)
        continue
      eng.step()
      if targets is not None:
        eng.output_loss(tgt, lat_weight, channel_sums=sums, planes_out=out, **affine)
      else:
        eng.unpack_outputs(out, **affine)
    free = torch.cuda.Event()
    free.record(compute)
    self._buf_free[buf] = free

    if planes_out is None:
      return None
    # planes -> Dataset shaped like the template
    # (reference _grid_node_outputs_to_prediction :701-723, stacked_to_dataset).
    return self._planes_to_dataset(planes_out, targets_template, n_lat, n_lon)

  @staticmethod
  def _pack(eng: engine_lib.Engine, planes: torch.Tensor, norm: Optional[FusedNormalization]) -> dict:
    """Packs one batch element's input planes [c_in, Ng] into eng.grid_in_img, normalised by `norm`,
    and returns the affine keywords that unpack its step's outputs (unpack_outputs, output_loss): none
    without `norm`."""
    if norm is None:
      eng.pack_inputs(planes)
      return {}
    eng.pack_inputs(planes, mean=norm.in_mean, scale=norm.in_scale)
    return dict(scale=norm.out_scale, offset=norm.out_offset, add_planes=planes,
                add_plane_index=norm.add_plane_index)

  @staticmethod
  def _check_template(template: xs.Dataset, n_channels: int):
    """Channel slabs of `template`, with stacked_to_dataset's two errors (model_utils.py:713-776)."""
    preserved = ("batch", "lat", "lon")
    for name in sorted(template.data_vars.keys()):
      tv = template.data_vars[name]
      if not all(d in tv.dims for d in preserved):
        raise ValueError(
            f"stacked_to_dataset requires all Variables to have {preserved} "
            f"dimensions, but found only {tv.dims}.")
    slabs = model_utils.channel_layout(template)
    expected = sum(s.count for s in slabs)
    if expected != n_channels:
      raise ValueError(f"Expected {expected} channels but found {n_channels}, when "
                       f"trying to convert the model output to a dataset of shape {template}.")
    return slabs

  def _planes_to_dataset(self, planes_out: torch.Tensor, template: xs.Dataset,
                         n_lat: int, n_lon: int, directions=None) -> xs.Dataset:
    """planes_out [batch, n_out, Ng] -> a Dataset shaped like `template`.  With `directions` (labels),
    planes_out [K, batch, n_out, Ng] -> variables with a leading "direction" dim, labelled so."""
    lead, lead_dims = planes_out.shape[:-2], ("batch",)
    if directions is not None:
      lead_dims = (feedback.DIRECTION, "batch")
    slabs = self._check_template(template, planes_out.shape[-2])
    out = xs.Dataset(coords=template.coords)
    if directions is not None:
      out.coords[feedback.DIRECTION] = ((feedback.DIRECTION,), np.asarray(directions))
    for s in slabs:
      piece = planes_out[..., s.start:s.start + s.count, :]
      piece = piece.reshape(tuple(lead) + s.stack_sizes + (n_lat, n_lon))
      da = xs.DataArray(piece, lead_dims + s.stack_dims + ("lat", "lon"))
      out[s.name] = da.transpose(*lead_dims[:-1], *s.var_dims)
    return out


def check_param_tangents(param_tangents, params) -> Dict[str, Dict[str, np.ndarray]]:
  """param_tangents (param_jvp, loss_and_param_gnvp) as float32 host arrays, after its checks against
  `params`: a mapping of mappings whose modules and fields are those of the params and whose arrays
  have their parameter's shape.  Raises ValueError otherwise."""
  if not isinstance(param_tangents, Mapping):
    raise ValueError(f"param_tangents must be a mapping {{module: {{field: array}}}} shaped like the "
                     f"params, not {type(param_tangents).__name__}")
  out = {}
  for name, fields in param_tangents.items():
    if name not in params:
      raise ValueError(f"param_tangents has an unknown module {name!r}")
    if not isinstance(fields, Mapping):
      raise ValueError(f"param_tangents[{name!r}] must be a mapping {{field: array}}, not "
                       f"{type(fields).__name__}")
    for f, a in fields.items():
      if f not in params[name]:
        raise ValueError(f"param_tangents has an unknown field {name}:{f}")
      try:
        arr = np.asarray(a, dtype=np.float32)
      except (TypeError, ValueError) as e:
        raise ValueError(f"param_tangents {name}:{f} is not a float array: {e}") from None
      want = tuple(np.shape(params[name][f]))
      if arr.shape != want:
        raise ValueError(f"param_tangents {name}:{f} has shape {arr.shape}, the parameter {want}")
      out.setdefault(name, {})[f] = arr
  return out


def loss_coefficients(targets: xs.Dataset, num_grid: int, batch: int, steps: int = 1):
  """(channel slabs of `targets`, [n_out] float64 coefficients 2 kappa / (batch * steps)): the loss
  derivative with respect to the channel sums of gcb_output_loss (losses.channel_kappa) of the mean
  loss over `batch` elements and `steps` target times."""
  slabs = model_utils.channel_layout(targets)
  return slabs, 2.0 * losses.channel_kappa(slabs, num_grid, LOSS_PER_VARIABLE_WEIGHTS) / (batch * steps)


def _device_coef(coef: np.ndarray, device) -> torch.Tensor:
  """Loss coefficients (loss_coefficients) as a float64 tensor on `device`."""
  return torch.as_tensor(np.asarray(coef, np.float64)).to(device)


def _host_grads(grads) -> Dict[str, Dict[str, np.ndarray]]:
  """Device gradients {module: {field: tensor}} as host numpy arrays."""
  return {name: {f: t.cpu().numpy() for f, t in fields.items()} for name, fields in grads.items()}


def hvp_tangent_planes(inputs: xs.Dataset, forcings: xs.Dataset, input_tangents,
                       forcing_tangents) -> torch.Tensor:
  """[batch, c_in, Ng] float32 host planes of the tangent of a Hessian-vector product, inputs then
  forcings, packed as GraphCast stages the planes (feedback.tangent_planes), after input_jvp's checks."""
  input_tangents = None if input_tangents is None else xs.from_xarray(input_tangents)
  forcing_tangents = None if forcing_tangents is None else xs.from_xarray(forcing_tangents)
  feedback.check_tangents(input_tangents, inputs, "input_tangents")
  feedback.check_tangents(forcing_tangents, forcings, "forcing_tangents")
  sizes = {"batch": dict(inputs.sizes).get("batch", 1), "lat": inputs.sizes["lat"],
           "lon": inputs.sizes["lon"]}
  return torch.from_numpy(np.concatenate(
      [feedback.tangent_planes(input_tangents, inputs, sizes),
       feedback.tangent_planes(forcing_tangents, forcings, sizes)], axis=1))


def hvp_direction_tangent_planes(inputs: xs.Dataset, forcings: xs.Dataset, input_tangents,
                                 forcing_tangents) -> torch.Tensor:
  """[K, batch, c_in, Ng] float32 host planes of the K tangents of a batched_loss_and_input_hvp, after
  batched_input_jvp's checks (feedback.check_direction_tangents): direction k is what
  hvp_tangent_planes packs for tangent k alone."""
  it = None if input_tangents is None else xs.from_xarray(input_tangents)
  ft = None if forcing_tangents is None else xs.from_xarray(forcing_tangents)
  dirs, _ = feedback.check_direction_tangents(it, inputs, ft, forcings)
  sizes = {"batch": dict(inputs.sizes).get("batch", 1), "lat": inputs.sizes["lat"],
           "lon": inputs.sizes["lon"]}
  return torch.from_numpy(np.concatenate(
      [feedback.tangent_planes(it, inputs, sizes, dirs),
       feedback.tangent_planes(ft, forcings, sizes, dirs)], axis=2))


def _hvp_directions(planes: Optional[torch.Tensor], axis: int) -> Optional[Tuple[int, bool]]:
  """(K, directions) of the tangent planes of a Hessian-vector product: the planes of one tangent have
  no direction axis (K = 1, no "direction" dim in the results), those of K tangents one at `axis`
  ([K, batch, c_in, Ng] host planes: 0; [batch, K, c_in, Ng] stashed planes: 1)."""
  if planes is None:
    return None
  return (1, False) if planes.dim() == 3 else (int(planes.shape[axis]), True)


def batched_hvp(one_pass, inputs, forcings, input_tangents, forcing_tangents, directions_per_pass):
  """batched_loss_and_input_hvp of a predictor stack: checks the tangents
  (feedback.check_direction_tangents) and directions_per_pass before anything runs, then runs
  one_pass(input_tangents, forcing_tangents) -> (loss, diagnostics, input_grads, forcing_grads,
  input_hvp, forcing_hvp) on consecutive slices of the directions (direction_passes) and joins the
  Hessian-vector products along "direction".  The loss, diagnostics and gradients are the first
  pass's."""
  inputs, forcings = xs.from_xarray(inputs), xs.from_xarray(forcings)
  it = None if input_tangents is None else xs.from_xarray(input_tangents)
  ft = None if forcing_tangents is None else xs.from_xarray(forcing_tangents)
  dirs, labels = feedback.check_direction_tangents(it, inputs, ft, forcings)
  at = lambda ds, sl: None if ds is None else ds.isel({feedback.DIRECTION: sl})

  def pass_of(sl):
    out = one_pass(at(it, sl), at(ft, sl))
    return (out[:4],) + tuple(out[4:])
  first, input_hvp, forcing_hvp = direction_passes(pass_of, dirs, labels, directions_per_pass)
  return first + (input_hvp, forcing_hvp)


def batched_jvp(one_pass, inputs, forcings, input_tangents, forcing_tangents, directions_per_pass):
  """batched_input_jvp of a predictor stack: checks the tangents (feedback.check_direction_tangents)
  and directions_per_pass before anything runs, then runs one_pass(input_tangents, forcing_tangents)
  -> (predictions, prediction_tangents) on ceil(K / directions_per_pass) consecutive slices of the
  directions and joins the tangents along "direction".  The predictions are those of the first pass."""
  inputs, forcings = xs.from_xarray(inputs), xs.from_xarray(forcings)
  it = None if input_tangents is None else xs.from_xarray(input_tangents)
  ft = None if forcing_tangents is None else xs.from_xarray(forcing_tangents)
  dirs, labels = feedback.check_direction_tangents(it, inputs, ft, forcings)
  at = lambda ds, sl: None if ds is None else ds.isel({feedback.DIRECTION: sl})
  return direction_passes(lambda sl: one_pass(at(it, sl), at(ft, sl)), dirs, labels,
                          directions_per_pass)


def batched_vjp(one_pass, targets_template, cotangents, directions_per_pass):
  """batched_input_vjp of a predictor stack: checks the cotangents against the template
  (feedback.check_direction_cotangents) and directions_per_pass before anything runs, then runs
  one_pass(cotangents, first) -> (predictions, input_grads, forcing_grads) on consecutive slices of the
  directions (direction_passes).  Only the first pass (first=True) need form the predictions: the later
  ones' are dropped, so they need not hold a second copy on the device."""
  cot = xs.from_xarray(cotangents)
  dirs, labels = feedback.check_direction_cotangents(cot, xs.from_xarray(targets_template))
  return direction_passes(lambda sl: one_pass(cot.isel({feedback.DIRECTION: sl}), sl.start == 0),
                          dirs, labels, directions_per_pass)


def direction_passes(one_pass, dirs: int, labels, directions_per_pass):
  """The passes of a batched call of `dirs` directions: one_pass(sl) -> (predictions, *results) runs
  on ceil(K / directions_per_pass) consecutive slices sl of the directions (feedback.direction_slices,
  which checks directions_per_pass first), each result a Dataset with a leading "direction" dim.
  Returns (predictions of the first pass, *each result joined along "direction" over the passes and
  labelled `labels`)."""
  predictions, parts = None, None
  for sl in feedback.direction_slices(dirs, directions_per_pass):
    p, *results = one_pass(sl)
    predictions = p if predictions is None else predictions
    parts = [[r] for r in results] if parts is None else [a + [r] for a, r in zip(parts, results)]
  return (predictions,) + tuple(join_directions(a, labels) for a in parts)


def join_directions(parts, labels) -> xs.Dataset:
  """Datasets with the same variables, each with a leading "direction" dim (consecutive slices of the
  directions, in order), joined along it and labelled `labels`.  The data stay torch tensors or numpy
  arrays, as the parts hold them."""
  out = xs.Dataset(coords=parts[0].coords)
  out.coords[feedback.DIRECTION] = ((feedback.DIRECTION,), np.asarray(labels))
  for name, v in parts[0].data_vars.items():
    data = [p.data_vars[name].data for p in parts]
    if len(data) == 1:
      data = data[0]
    elif isinstance(data[0], torch.Tensor):
      data = torch.cat(data, dim=0)
    else:
      data = np.concatenate(data, axis=0)
    out[name] = xs.DataArray(data, v.dims)
  return out


def innermost_graphcast(predictor) -> Optional[GraphCast]:
  """The GraphCast at the bottom of a predictor stack (autoregressive.Predictor, InputsAndResiduals,
  Bfloat16Cast wrappers hold it as `_predictor`), or None."""
  p = predictor
  while p is not None and not isinstance(p, GraphCast):
    p = getattr(p, "_predictor", None)
  return p


def init_params(model_config: ModelConfig, task_config: TaskConfig, c_in: int,
                seed: int = 1) -> Dict[str, Dict[str, np.ndarray]]:
  """Haiku-default random initialisation of all GraphCast parameters
  (what `hk.transform(...).init` yields in the reference demo, notebook cell 10):
  w ~ TruncatedNormal(1/sqrt(fan_in)), b = 0, LayerNorm scale = 1 / offset = 0."""
  rng = np.random.default_rng(seed)
  D = model_config.latent_size
  n_out = num_outputs(task_config)
  params: Dict[str, Dict[str, np.ndarray]] = {}

  def trunc_normal(shape, std):
    x = rng.standard_normal(shape)
    bad = np.abs(x) > 2.0
    while bad.any():
      x[bad] = rng.standard_normal(int(bad.sum()))
      bad = np.abs(x) > 2.0
    return (x * std).astype(np.float32)

  def add(gnn, prefix, set_name, d_in, d_out, layer_norm=True):
    stem = engine_lib.mlp_stem(gnn, prefix, set_name)
    fan_in = d_in
    for i, size in enumerate([D] * model_config.hidden_layers + [d_out]):
      params[f"{stem}_mlp/~/linear_{i}"] = {
          "w": trunc_normal((fan_in, size), 1.0 / np.sqrt(fan_in)),
          "b": np.zeros([size], np.float32)}
      fan_in = size
    if layer_norm:
      params[f"{stem}_layer_norm"] = {"scale": np.ones([d_out], np.float32),
                                      "offset": np.zeros([d_out], np.float32)}

  g = "grid2mesh_gnn"
  add(g, "encoder_nodes_", "grid_nodes", c_in + 3, D)
  add(g, "encoder_nodes_", "mesh_nodes", c_in + 3, D)
  add(g, "encoder_edges_", "grid2mesh", 4, D)
  add(g, "processor_edges_0_", "grid2mesh", 3 * D, D)
  add(g, "processor_nodes_0_", "grid_nodes", D, D)
  add(g, "processor_nodes_0_", "mesh_nodes", 2 * D, D)
  g = "mesh_gnn"
  add(g, "encoder_edges_", "mesh", 4, D)
  for k in range(model_config.gnn_msg_steps):
    add(g, f"processor_edges_{k}_", "mesh", 3 * D, D)
    add(g, f"processor_nodes_{k}_", "mesh_nodes", 2 * D, D)
  g = "mesh2grid_gnn"
  add(g, "encoder_edges_", "mesh2grid", 4, D)
  add(g, "processor_edges_0_", "mesh2grid", 3 * D, D)
  add(g, "processor_nodes_0_", "grid_nodes", 2 * D, D)
  add(g, "processor_nodes_0_", "mesh_nodes", D, D)
  add(g, "decoder_nodes_", "grid_nodes", D, n_out, layer_norm=False)
  return params


class _InputGradRun:
  """The backward pass of one input-gradient call (GraphCast._input_grads / _one_step_input_grads):
  the all-channel feedback of `plan`, and the per-variable results.  release_staging: the steps come
  from a StepStash and every staging buffer goes; else the backward pass runs inside `_call`, which
  keeps the slot it staged into.  After step t of batch element b
  (element(b, t, ...)) the rows of its forcings slab, and after step 0 those of the inputs, are
  reduced on the device (gcb_broadcast_grad_sum: the transpose of the broadcast over lat / lon,
  batch-free variables summed over the batch in order) before the previous step consumes `a`.
  Batched inputs are reduced into a buffer allocated after the element's backward pass and copied
  without a synchronisation into pinned host memory (torch's caching host allocator: allocated on the
  first call, reused after), so that the 0.25 degree inputs' 1.9 GB never coexist with a backward pass
  and cross PCIe at full speed; finish() synchronises once.  The returned arrays are views of it.

  dirs = K (batched_input_vjp): K cotangents share every step, fb.a is [K, n_rows, Ng], and every
  result buffer has a leading axis of K directions, each reduced as one direction's would be.

  hvp = (K, directions) (loss_and_input_hvp: (1, False); batched_loss_and_input_hvp: (K, True)): every
  step runs Engine.input_hvp_element, the 1 + K directions are the gradient and its derivatives along
  the K tangents, and finish() gives (input_grads, forcing_grads) from direction 0 and (input_hvp,
  forcing_hvp) from directions 1..K, these with a leading "direction" dim when `directions`.  With
  weight_tangents set as well (loss_and_joint_hvp, K = 1, one target time): Engine.joint_hvp_element
  in its place, the tangent also along those packed parameter tangents."""

  def __init__(self, model: GraphCast, plan, norm: Optional[FusedNormalization], inputs: xs.Dataset,
               forcings: xs.Dataset, num_steps: int, batch: int, release_staging: bool,
               dirs: Optional[int] = None, hvp: Optional[Tuple[int, bool]] = None):
    eng = self.eng = model.engine
    self.hvp, self.zero_targets = hvp, None
    self.weight_tangents = None
    dirs = 1 + hvp[0] if hvp else dirs
    self.dirs = dirs
    lead = [] if dirs is None else [dirs]
    eng.input_grads_begin()
    self.fb = eng.feedback(plan, None if norm is None else norm.add_plane_index,
                           None if norm is None else norm.in_scale)
    if release_staging:
      model._release_staging()
    else:
      model._release_idle_staging()
    self.inputs, self.forcings = inputs, forcings
    self.num_steps, self.batch = num_steps, batch
    self.n_lat, self.n_lon = inputs.sizes["lat"], inputs.sizes["lon"]
    self.var_rows = feedback.variable_rows(inputs, forcings)
    dev = eng.device
    self.dev_bufs, self.host, self.rows = {}, {}, {}
    for v in self.var_rows:
      if v.forcing or not v.batched:
        shape = ([batch] if v.batched else []) + ([num_steps] if v.timed else []) + [v.count, self._width(v)]
        self.dev_bufs[v.key] = torch.zeros(lead + shape, dtype=torch.float32, device=dev)
      else:
        self.host[v.key] = torch.empty(lead + [batch, v.count, self._width(v)], dtype=torch.float32,
                                       pin_memory=True)
      self.rows[v.key] = torch.arange(v.start, v.start + v.count, dtype=torch.int32, device=dev)

  def _width(self, v) -> int:
    return (self.eng.num_grid, self.n_lon, 1)[v.mode]

  def element(self, b: int, t: int, operands: dict, **kw) -> None:
    """Step t of batch element b (t = num_steps - 1 first): Engine.input_grads_element, then the
    reductions of the rows that are complete."""
    if t == self.num_steps - 1:
      self.fb.a = None
    if self.hvp:
      if self.zero_targets is None:
        self.zero_targets = torch.zeros([self.eng.n_out, self.eng.num_grid], dtype=torch.float32,
                                        device=self.eng.device)
      if self.weight_tangents is not None:   # a loss: no predictions to unpack
        kw.pop("planes_out", None)
        self.eng.joint_hvp_element(self.fb, operands, weight_tangents=self.weight_tangents,
                                   zero_targets=self.zero_targets, **kw)
      else:
        self.eng.input_hvp_element(self.fb, operands, zero_targets=self.zero_targets, **kw)
    else:
      self.eng.input_grads_element(self.fb, operands, **kw)
    for v in self.var_rows:
      if v.forcing or t == 0:
        self._reduce(v, b, t)
    if t == 0:
      self.fb.a = None

  def _reduce(self, v, b: int, t: int) -> None:
    if self.dirs is None:
      self._reduce_one(v, b, t, self.fb.a, self.host.get(v.key), self.dev_bufs.get(v.key))
      return
    for k in range(self.dirs):
      host, dev = self.host.get(v.key), self.dev_bufs.get(v.key)
      self._reduce_one(v, b, t, self.fb.a[k], None if host is None else host[k],
                       None if dev is None else dev[k])

  def _reduce_one(self, v, b: int, t: int, a: torch.Tensor, host: Optional[torch.Tensor],
                  dev: Optional[torch.Tensor]) -> None:
    """The rows of one direction's gradient a [n_rows, Ng] into its result buffer (host or dev)."""
    eng = self.eng
    if host is not None:                   # a batched input
      out = torch.empty([v.count, self._width(v)], dtype=torch.float32, device=eng.device)
      eng.broadcast_grad_sum(a, self.n_lat, self.rows[v.key], v.mode, out, False)
      host[b].copy_(out, non_blocking=True)   # stream-ordered before out's reuse
      return
    out = dev[b] if v.batched else dev
    out = out[t] if v.timed else out
    accumulate = (not v.batched and b > 0) or (v.forcing and not v.timed and t < self.num_steps - 1)
    eng.broadcast_grad_sum(a, self.n_lat, self.rows[v.key], v.mode, out, accumulate)

  def finish(self):
    """(input_grads, forcing_grads) Datasets shaped like the inputs and forcings."""
    grads = {key: buf.cpu().numpy() for key, buf in self.dev_bufs.items()}   # synchronises
    torch.cuda.current_stream(self.eng.device).synchronize()
    grads.update({key: t.numpy() for key, t in self.host.items()})
    if self.hvp:
      nt, directions = self.hvp
      at = lambda k: {key: g[k] for key, g in grads.items()}
      return feedback.grads_to_datasets(self.var_rows, at(0), self.inputs, self.forcings, self.n_lat,
                                        self.n_lon) + feedback.grads_to_datasets(
          self.var_rows, at(slice(1, None)) if directions else at(1), self.inputs, self.forcings,
          self.n_lat, self.n_lon, directions=nt if directions else None)
    return feedback.grads_to_datasets(self.var_rows, grads, self.inputs, self.forcings, self.n_lat,
                                      self.n_lon, directions=self.dirs)


class _TangentRun:
  """The tangent planes of one input_jvp or batched_input_jvp call (GraphCast._input_jvp,
  autoregressive.Predictor.input_jvp).  The tangent Datasets are checked and packed into host planes
  on construction, before anything runs on the device.  Per batch element a device buffer [dirs,
  c_in + n_out, Ng] holds the tangent of the current step's input planes of every direction in its
  first c_in rows (dirs = 1 for input_jvp, K with `directions`).  After a step that has a successor,
  the prediction tangents are copied into the last n_out rows and the next step's first n_in rows of
  every direction are gathered from the buffer by one gcb_gather_rows with FeedbackPlan.feed_index
  (dirs) (every such row is a copy of one row of the two sources); the forcings slab comes from the
  forcing tangents of that target time.  The tangent planes stay on the device from step to step, and
  nothing is kept per step."""

  def __init__(self, inputs: xs.Dataset, forcings: xs.Dataset, input_tangents, forcing_tangents,
               num_steps: int, plan=None, directions: bool = False):
    input_tangents = None if input_tangents is None else xs.from_xarray(input_tangents)
    forcing_tangents = None if forcing_tangents is None else xs.from_xarray(forcing_tangents)
    self.directions = directions
    if directions:
      self.dirs, self.labels = feedback.check_direction_tangents(input_tangents, inputs,
                                                                 forcing_tangents, forcings)
    else:
      feedback.check_tangents(input_tangents, inputs, "input_tangents")
      feedback.check_tangents(forcing_tangents, forcings, "forcing_tangents")
      self.dirs, self.labels = 1, None
    self.batch = dict(inputs.sizes).get("batch", 1)
    self.n_lat, self.n_lon = inputs.sizes["lat"], inputs.sizes["lon"]
    self.sizes = {"batch": self.batch, "lat": self.n_lat, "lon": self.n_lon}
    if num_steps > 1 and (self.n_lat * self.n_lon) % 4:
      raise NotImplementedError("input_jvp over several target times needs a multiple of 4 grid "
                                "nodes (the tangent feed gathers 16-byte rows)")
    self.input_planes = self._planes(input_tangents, inputs)
    self.forcings, self.forcing_tangents = forcings, forcing_tangents
    self.num_steps, self.step = num_steps, 0
    self.feed = None if plan is None else torch.from_numpy(plan.feed_index(self.dirs))
    self.carry = [None] * self.batch
    self._slab = (-1, None)
    # param_jvp: the checked host parameter tangents, packed on the device by the first element
    self.param_tangents, self.weight_tangents = None, None

  def _planes(self, tangents, like) -> torch.Tensor:
    """[dirs, batch, channels, Ng] host planes of a tangent Dataset (feedback.tangent_planes)."""
    if self.directions:
      return torch.from_numpy(feedback.tangent_planes(tangents, like, self.sizes, self.dirs))
    return torch.from_numpy(feedback.tangent_planes(tangents, like, self.sizes)).unsqueeze(0)

  def _forcing_planes(self, t: int) -> torch.Tensor:
    """[dirs, batch, c_in - n_in, Ng] host tangent planes of the forcings of target time t."""
    if self._slab[0] != t:
      at = lambda ds: ds.isel(time=slice(t, t + 1)) if "time" in ds.sizes else ds
      tangents = None if self.forcing_tangents is None else at(self.forcing_tangents)
      self._slab = (t, self._planes(tangents, at(self.forcings)))
    return self._slab[1]

  def element(self, eng, b: int, tangent_out: torch.Tensor, planes_out: Optional[torch.Tensor],
              norm: Optional[FusedNormalization], affine: dict, keep=None) -> None:
    """This step of batch element b (tangent_out [dirs, n_out, Ng]): Engine.input_jvp_element, then the
    feed of the next step.  keep(planes): called with this step's input tangent planes [dirs, c_in, Ng]
    (a device view, valid until the next step's feed) before the step runs."""
    c_in, n_in, ng = eng.c_in, self.input_planes.shape[2], eng.num_grid
    buf, self.carry[b] = self.carry[b], None
    if buf is None:
      buf = torch.empty([self.dirs, c_in + eng.n_out, ng], dtype=torch.float32, device=eng.device)
      buf[:, :n_in].copy_(self.input_planes[:, b])
    buf[:, n_in:c_in].copy_(self._forcing_planes(self.step)[:, b])
    if keep is not None:
      keep(buf[:, :c_in])
    if self.param_tangents is not None and self.weight_tangents is None:
      self.weight_tangents = eng.weight_tangents(self.param_tangents)
    eng.input_jvp_element(buf[:, :c_in], tangent_out,
                          in_scale=None if norm is None else norm.in_scale, planes_out=planes_out,
                          weight_tangents=self.weight_tangents, **affine)
    if self.step + 1 < self.num_steps:
      if self.feed.device != eng.device:
        self.feed = self.feed.to(eng.device)
      buf[:, c_in:].copy_(tangent_out)
      nxt = torch.empty_like(buf)
      with eng._on_device():
        _native.check(eng._lib.gcb_gather_rows(buf.data_ptr(), ng, self.feed.data_ptr(),
                                               self.feed.shape[0], nxt.data_ptr(), ng, ng,
                                               eng._stream()), "gcb_gather_rows")
      self.carry[b] = nxt


class StepStash:
  """Pinned host copies of the input and target planes of every step of a multi-step loss, for the
  recompute of backprop through time.  Each step's planes are first copied on the device (the staging
  buffers are reused two calls later), then to the host on a side stream, so the copy overlaps the
  next step's kernels.  steps[t] = ((inputs [batch, c_in, Ng], targets [batch, n_out, Ng]), event)."""

  def __init__(self, device):
    self.device = torch.device(device)
    self.stream = torch.cuda.Stream(device=self.device)
    self.steps = []
    self.batch = 0

  def save(self, *planes: torch.Tensor) -> None:
    compute = torch.cuda.current_stream(self.device)
    copies = [p.clone() for p in planes]
    ready = torch.cuda.Event()
    ready.record(compute)
    hosts = [torch.empty(p.shape, dtype=p.dtype, pin_memory=True) for p in planes]
    with torch.cuda.stream(self.stream):
      self.stream.wait_event(ready)
      for h, c in zip(hosts, copies):
        h.copy_(c, non_blocking=True)
        c.record_stream(self.stream)
      done = torch.cuda.Event()
      done.record(self.stream)
    self.steps.append((tuple(hosts), done))
    self.batch = int(planes[0].shape[0])
