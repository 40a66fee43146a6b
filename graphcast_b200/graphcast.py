"""GraphCast one-step predictor -- host-side mirror of the reference API.

Same public surface as `weathernext/weathernext1_graph/graphcast.py`:
  ModelConfig (:115-142), TaskConfig (utils/task.py:21-28), CheckPoint (:145-151),
  TASK / TASK_13 / TASK_13_PRECIP_OUT (:86-112),
  GraphCast(model_config, task_config).__call__(inputs, targets_template,
  forcings, is_training=False) -> Dataset (:184, :298-329).

What differs is only *how* the step is computed: the three GNN calls
(`_run_grid2mesh_gnn` :550, `_run_mesh_gnn` :606, `_run_mesh2grid_gnn` :641) and
the channel (un)packing (`_inputs_to_grid_node_features` :680,
`_grid_node_outputs_to_prediction` :701) run as hand-written sm_90a kernels
behind the C ABI in include/graphcast_b200.h.  There is no CPU path: without a
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
    raise NotImplementedError("training losses are outside the inference hot path")

  def loss_and_predictions(self, inputs, targets, forcings, **optional_kwargs):
    raise NotImplementedError("training losses are outside the inference hot path")


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

  def _channel_plan(self, inputs: xs.Dataset, forcings: xs.Dataset):
    in_slabs = model_utils.channel_layout(inputs)
    n_in = sum(s.count for s in in_slabs)
    f_slabs = model_utils.channel_layout(forcings, start=n_in)
    return in_slabs, f_slabs, n_in + sum(s.count for s in f_slabs)

  def _call(self, inputs, targets_template, forcings, norm: Optional[FusedNormalization]):
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

    # xarray -> channel-major planes [B, C, lat*lon] on the device
    # (reference _inputs_to_grid_node_features :680-699; dataset_to_stacked order).
    buf = self._call_index % 2
    self._call_index += 1
    fresh = self._planes_bufs[buf] is None or self._planes_bufs[buf].shape != (batch, c_in, eng.num_grid)
    if fresh:
      self._planes_bufs[buf] = torch.empty([batch, c_in, eng.num_grid], dtype=torch.float32,
                                           device=eng.device)
      self._buf_free[buf] = None
    planes_in = self._planes_bufs[buf]
    self._planes_in = planes_in
    sources = []
    for ds, slabs in ((inputs, in_slabs), (forcings, f_slabs)):
      for s in slabs:
        src = model_utils.variable_to_planes(ds.data_vars[s.name], sizes)
        if not isinstance(src, torch.Tensor):
          src = torch.from_numpy(np.ascontiguousarray(src, dtype=np.float32))
        sources.append((s, src))
    compute = torch.cuda.current_stream(eng.device)
    all_host = all(src.device.type == "cpu" for _, src in sources)
    if all_host:
      if self._h2d_stream is None:
        self._h2d_stream = torch.cuda.Stream(device=eng.device)
      copy_stream = self._h2d_stream
      if fresh:
        # The caching allocator may hand back a block whose previous user still has kernels
        # queued on the compute stream: order the first copy after them, and tell the allocator
        # that the copy stream uses this block too.
        copy_stream.wait_stream(compute)
        planes_in.record_stream(copy_stream)
      if self._buf_free[buf] is not None:
        copy_stream.wait_event(self._buf_free[buf])      # kernels of call k-2 are done with it
    else:
      copy_stream = compute                              # device-resident inputs: stay in order
    with torch.cuda.stream(copy_stream):
      for s, src in sources:
        dst = planes_in[:, s.start:s.start + s.count].view(batch, s.count, n_lat, n_lon)
        dst.copy_(src, non_blocking=True)
      if all_host:
        ready = torch.cuda.Event()
        ready.record(copy_stream)
    if all_host:
      compute.wait_event(ready)

    # Predictions are produced into fresh planes each call (they are handed out).
    planes_out = torch.empty([batch, eng.n_out, eng.num_grid], dtype=torch.float32,
                             device=eng.device)
    for b in range(batch):
      if norm is None:
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

    # planes -> Dataset shaped like the template
    # (reference _grid_node_outputs_to_prediction :701-723, stacked_to_dataset).
    return self._planes_to_dataset(planes_out, targets_template, n_lat, n_lon)

  def _planes_to_dataset(self, planes_out: torch.Tensor, template: xs.Dataset,
                         n_lat: int, n_lon: int) -> xs.Dataset:
    preserved = ("batch", "lat", "lon")
    for name in sorted(template.data_vars.keys()):
      tv = template.data_vars[name]
      if not all(d in tv.dims for d in preserved):
        raise ValueError(
            f"stacked_to_dataset requires all Variables to have {preserved} "
            f"dimensions, but found only {tv.dims}.")
    slabs = model_utils.channel_layout(template)
    expected = sum(s.count for s in slabs)
    if expected != planes_out.shape[1]:
      raise ValueError(f"Expected {expected} channels but found {planes_out.shape[1]}, when "
                       f"trying to convert the model output to a dataset of shape {template}.")
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
