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
from typing import Any, Dict, List, Mapping, Optional, Tuple

import numpy as np
import torch

from graphcast_b200 import engine as engine_lib
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
               image_residual: bool = True, deep_chains: bool = True):
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
    self._device = device
    self._params = params
    self._num_outputs = num_outputs(task_config)
    self._initialized = False
    self._static_graph: Optional[graph_lib.StaticGraph] = None
    self._engine: Optional[engine_lib.Engine] = None
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
  def set_params(self, params: Mapping[str, Mapping[str, np.ndarray]]) -> None:
    self._params = params
    self._engine = None

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
          deep_chains=self._deep_chains)
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
    inputs, targets = xs.from_xarray(inputs), xs.from_xarray(targets)
    if targets.sizes.get("time", 1) != 1:
      raise NotImplementedError("parameter gradients cover one target time (no backprop through time)")
    sizes = dict(inputs.sizes)
    batch = sizes.get("batch", 1)
    num_grid = sizes["lat"] * sizes["lon"]
    slabs = model_utils.channel_layout(targets)
    coef = 2.0 * losses.channel_kappa(slabs, num_grid, LOSS_PER_VARIABLE_WEIGHTS) / batch
    self._call(inputs, targets, forcings, norm=norm, targets=targets, predictions=False,
               grad_coef=coef)
    loss, diagnostics = losses.losses_from_channel_sums(
        self._channel_sums.cpu().numpy(), slabs, self._engine.num_grid, LOSS_PER_VARIABLE_WEIGHTS)
    grads = {name: {f: t.cpu().numpy() for f, t in fields.items()}
             for name, fields in self._engine.grads().items()}
    return loss, diagnostics, grads

  def _stash_step(self, stash: "StepStash") -> None:
    """Keeps the input and target planes of the last `_call` (with targets) in pinned host memory."""
    stash.save(self._planes_in, self._planes_tgt)

  def _bptt_grads(self, stash: "StepStash", plan, norm: Optional[FusedNormalization],
                  lat_weight: torch.Tensor, coef: np.ndarray):
    """Parameter gradients of the multi-step loss whose steps `stash` holds (backprop through time,
    see autoregressive.Predictor.loss_and_grads).  For every batch element, last step first: the
    step's planes are uploaded again, packed and differentiated by Engine.loss_and_grads_element with
    the feedback of the following step; the gradients accumulate in this fixed order."""
    eng = self._engine
    dev = eng.device
    eng.grads_begin()
    fb = eng.feedback(plan, None if norm is None else norm.add_plane_index,
                      None if norm is None else norm.in_scale)
    # The rollout's staging buffers are not needed any more: their memory goes to the backward pass.
    self._planes_bufs, self._target_bufs, self._buf_free = [None, None], [None, None], [None, None]
    self._planes_in = self._planes_tgt = None
    # Return the rollout's cached blocks to the driver, so that the backward pass allocates from an
    # unfragmented pool: at 0.25 degree it peaks within a few GiB of an 80 GB card's capacity, and a
    # second call would otherwise find its 1 GiB tables only in the gaps the first one left.
    torch.cuda.empty_cache()
    planes = torch.empty([eng.c_in, eng.num_grid], dtype=torch.float32, device=dev)
    tgt = torch.empty([eng.n_out, eng.num_grid], dtype=torch.float32, device=dev)
    scratch = torch.empty([eng.n_out], dtype=torch.float64, device=dev)
    coef_dev = torch.as_tensor(np.asarray(coef, np.float64)).to(dev)
    compute = torch.cuda.current_stream(dev)
    for b in range(stash.batch):
      fb.a = None
      for t in range(len(stash.steps) - 1, -1, -1):
        (host_in, host_tgt), done = stash.steps[t]
        compute.wait_event(done)
        planes.copy_(host_in[b], non_blocking=True)
        tgt.copy_(host_tgt[b], non_blocking=True)
        affine = {}
        if norm is None:
          eng.pack_inputs(planes)
        else:
          eng.pack_inputs(planes, mean=norm.in_mean, scale=norm.in_scale)
          affine = dict(scale=norm.out_scale, offset=norm.out_offset, add_planes=planes,
                        add_plane_index=norm.add_plane_index)
        eng.loss_and_grads_element(tgt, lat_weight, coef_dev, channel_sums=scratch, feedback=fb,
                                   input_grad=t > 0, **affine)
    return {name: {f: t.cpu().numpy() for f, t in fields.items()}
            for name, fields in eng.grads().items()}

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
    num_grid = self._engine.num_grid
    finish = lambda sums: losses.losses_from_channel_sums(sums, slabs, num_grid,
                                                          LOSS_PER_VARIABLE_WEIGHTS)
    return finish, preds, self._channel_sums

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
            targets: Optional[xs.Dataset] = None, predictions: bool = True,
            grad_coef: Optional[np.ndarray] = None):
    """The step for every batch element.  With `targets` (shaped like the template, usually the
    same Dataset) the outputs go through gcb_output_loss instead of the plain unpack: the loss sums
    land in a new [batch, n_out] fp64 device tensor, self._channel_sums, and the predictions are
    returned only when `predictions` is set (else None).  With `grad_coef` ([n_out] coefficients
    2 kappa / batch of the loss derivative) every element also runs the backward pass, which
    accumulates the parameter gradients in the engine (Engine.loss_and_grads_element)."""
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
    if grad_coef is not None:
      coef_dev = torch.as_tensor(np.asarray(grad_coef, np.float64)).to(eng.device)
      eng.grads_begin()
    planes_out = None
    if predictions:
      planes_out = torch.empty([batch, eng.n_out, eng.num_grid], dtype=torch.float32,
                               device=eng.device)
    for b in range(batch):
      if targets is not None:
        affine = {} if norm is None else dict(
            scale=norm.out_scale, offset=norm.out_offset, add_planes=planes_in[b],
            add_plane_index=norm.add_plane_index)
        if norm is None:
          eng.pack_inputs(planes_in[b])
        else:
          eng.pack_inputs(planes_in[b], mean=norm.in_mean, scale=norm.in_scale)
        if grad_coef is not None:
          eng.loss_and_grads_element(planes_tgt[b], lat_weight, coef_dev,
                                     channel_sums=channel_sums[b], **affine)
          continue
        eng.step()
        eng.output_loss(planes_tgt[b], lat_weight, channel_sums=channel_sums[b],
                        planes_out=None if planes_out is None else planes_out[b], **affine)
      elif norm is None:
        eng.pack_inputs(planes_in[b])
        eng.step()
        eng.unpack_outputs(planes_out[b])
      else:
        eng.pack_inputs(planes_in[b], mean=norm.in_mean, scale=norm.in_scale)
        eng.step()
        eng.unpack_outputs(planes_out[b], scale=norm.out_scale, offset=norm.out_offset,
                           add_planes=planes_in[b], add_plane_index=norm.add_plane_index)
    free = torch.cuda.Event()
    free.record(compute)
    self._buf_free[buf] = free

    if planes_out is None:
      return None
    # planes -> Dataset shaped like the template
    # (reference _grid_node_outputs_to_prediction :701-723, stacked_to_dataset).
    return self._planes_to_dataset(planes_out, targets_template, n_lat, n_lon)

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
                         n_lat: int, n_lon: int) -> xs.Dataset:
    slabs = self._check_template(template, planes_out.shape[1])
    batch = planes_out.shape[0]
    out = xs.Dataset(coords=template.coords)
    for s in slabs:
      piece = planes_out[:, s.start:s.start + s.count]
      piece = piece.reshape((batch,) + s.stack_sizes + (n_lat, n_lon))
      da = xs.DataArray(piece, ("batch",) + s.stack_dims + ("lat", "lon"))
      out[s.name] = da.transpose(*s.var_dims)
    return out


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
