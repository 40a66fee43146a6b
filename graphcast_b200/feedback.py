"""Feedback plan of the autoregressive rollout: how one step's input planes and predictions make the
next step's input planes, in the stacked channel layout of GraphCast._call (inputs, then forcings,
each in `model_utils.channel_layout` order).  Pure numpy.

The rollout's feeding logic (rollout._get_next_inputs, reference autoregressive.py:114-125 and
rollout.py:581-604) on that layout is a fixed map of channels:

  * frame k of a time-dependent input is frame k + 1 of the same input in the previous step;
  * its last frame is the prediction of the same variable and level for a target variable, and the
    step's forcing (the forcings slab of the previous step's planes) for a forcing variable;
  * static inputs are copied; the forcings slab is the next target time's given forcings.

Backprop through time (autoregressive.Predictor.loss_and_grads) runs that map backwards.  The ROWS of
the plan are the input channels that depend on the parameters: every frame of every time-dependent
input variable that is also a target, frame-major (row k * n_fed + i is frame k of fed-back channel i).

Input gradients (loss_and_input_grads / input_vjp) run it backwards over every channel:
FeedbackPlan.all_channels has the rows 0..c_in-1 (row r = channel r), and `VariableRows` maps the rows
back to the variables of the inputs and forcings Datasets.
"""

from __future__ import annotations

from typing import Optional

import numpy as np

from graphcast_b200 import model_utils
from graphcast_b200 import xarray_shim as xs


class FeedbackPlan:
  """Channel maps between consecutive steps of a rollout (see the module docstring).

  n_in, c_in       channels of the inputs / of inputs + forcings (the planes of one step)
  n_frames         input frames of every time-dependent input
  n_fed            fed-back channels per frame
  next_from_input  [c_in] channel of this step's planes that becomes channel j of the next step's, -1
  next_from_pred   [c_in] prediction channel that becomes channel j of the next step's planes, -1
                   (both -1: the forcings slab, given per step)
  rows             [n_rows] input channel of row r
  dpred_row        [n_out] row holding the last input frame of prediction channel c, -1 if c is not fed
                   back (e.g. precipitation when it is not an input)
  carry_row        [n_rows] row of the NEXT step into which row r is shifted (row r - n_fed), -1 for
                   frame 0
  """

  def __init__(self, inputs: xs.Dataset, targets: xs.Dataset, forcings: xs.Dataset):
    in_slabs = model_utils.channel_layout(inputs)
    n_in = sum(s.count for s in in_slabs)
    f_slabs = model_utils.channel_layout(forcings, start=n_in)
    t_slabs = model_utils.channel_layout(targets)
    c_in = n_in + sum(s.count for s in f_slabs)
    n_out = sum(s.count for s in t_slabs)
    t_by_name = {s.name: s for s in t_slabs}
    f_by_name = {s.name: s for s in f_slabs}
    next_from_input = np.full([c_in], -1, np.int64)
    next_from_pred = np.full([c_in], -1, np.int64)
    fed_in, fed_out = [], []          # per fed-back channel: (input slab, index in frame), target channel
    n_frames = None
    for s in in_slabs:
      if "time" not in s.stack_dims:
        next_from_input[s.start:s.start + s.count] = np.arange(s.start, s.start + s.count)
        continue
      if s.stack_dims[0] != "time":
        raise ValueError(f"{s.name}: time must be the leading stacked dim of the inputs")
      n_time = s.stack_sizes[0]
      if n_frames is None:
        n_frames = n_time
      elif n_frames != n_time:
        raise ValueError(f"{s.name}: {n_time} input frames, other inputs have {n_frames}")
      per_frame = s.count // n_time
      for k in range(n_time - 1):
        dst = s.start + k * per_frame
        next_from_input[dst:dst + per_frame] = np.arange(dst + per_frame, dst + 2 * per_frame)
      last = s.start + (n_time - 1) * per_frame
      if s.name in t_by_name:
        t = t_by_name[s.name]
        if t.count != per_frame:
          raise ValueError(f"{s.name}: target has {t.count} channels per frame, input {per_frame}")
        next_from_pred[last:last + per_frame] = np.arange(t.start, t.start + per_frame)
        fed_in += [(s, i) for i in range(per_frame)]
        fed_out += list(range(t.start, t.start + per_frame))
      elif s.name in f_by_name:
        f = f_by_name[s.name]
        if f.count != per_frame:
          raise ValueError(f"{s.name}: forcing has {f.count} channels per step, input {per_frame}")
        next_from_input[last:last + per_frame] = np.arange(f.start, f.start + per_frame)
      else:
        raise ValueError("Found an input with a time index that is not predicted or forced.")
    n_frames = n_frames or 1
    n_fed = len(fed_in)
    rows = np.empty([n_frames * n_fed], np.int64)
    for i, (s, j) in enumerate(fed_in):
      per_frame = s.count // n_frames
      for k in range(n_frames):
        rows[k * n_fed + i] = s.start + k * per_frame + j
    dpred_row = np.full([n_out], -1, np.int64)
    dpred_row[np.asarray(fed_out, np.int64)] = (n_frames - 1) * n_fed + np.arange(n_fed)
    carry_row = np.arange(n_frames * n_fed) - n_fed
    carry_row[:n_fed] = -1
    self.n_in, self.c_in, self.n_out = n_in, c_in, n_out
    self.n_frames, self.n_fed = n_frames, n_fed
    self.next_from_input, self.next_from_pred = next_from_input, next_from_pred
    self.rows, self.dpred_row, self.carry_row = rows, dpred_row, carry_row
    self.all_rows = False

  @classmethod
  def all_channels(cls, inputs: xs.Dataset, targets: xs.Dataset,
                   forcings: xs.Dataset) -> "FeedbackPlan":
    """The plan whose rows are all c_in channels (row r = channel r), for gradients with respect to
    the inputs and forcings.  dpred_row, carry_row and resid_channel keep their meaning and follow
    next_from_input / next_from_pred: frame k + 1 -> frame k, static -> static, forcings slab -> the
    last input frame of the same forcing variable, frame 0 -> -1.  Every channel feeds at most one
    channel of the next step, so a single carry row per row suffices."""
    plan = cls(inputs, targets, forcings)
    c_in = plan.c_in
    carry_row = np.full([c_in], -1, np.int64)
    src = np.nonzero(plan.next_from_input >= 0)[0]
    if np.unique(plan.next_from_input[src]).size != src.size:
      raise ValueError("an input channel feeds several channels of the next step")
    carry_row[plan.next_from_input[src]] = src
    dpred_row = np.full([plan.n_out], -1, np.int64)
    pred = np.nonzero(plan.next_from_pred >= 0)[0]
    dpred_row[plan.next_from_pred[pred]] = pred
    plan.rows, plan.dpred_row, plan.carry_row = np.arange(c_in, dtype=np.int64), dpred_row, carry_row
    plan.all_rows = True
    return plan

  @property
  def n_rows(self) -> int:
    return int(self.rows.shape[0])

  def last_frame_channel(self) -> np.ndarray:
    """[n_out] input channel of the last frame of prediction channel c, -1 if c is not fed back."""
    return np.where(self.dpred_row >= 0, self.rows[np.maximum(self.dpred_row, 0)], -1)

  def resid_channel(self, add_plane_index: Optional[np.ndarray]) -> np.ndarray:
    """[n_rows] prediction channel whose residual add (normalization.InputsAndResiduals) reads row r,
    -1 for none; `add_plane_index` as FusedNormalization holds it (None: no residual add).  Every
    residual channel of a fed-back target must be its last input frame."""
    out = np.full([self.n_rows], -1, np.int64)
    if add_plane_index is None:
      return out
    add = np.asarray(add_plane_index, np.int64)
    if self.all_rows:                     # every channel is a row: any residual channel has its row
      c = np.nonzero(add >= 0)[0]
      out[add[c]] = c
      return out
    last = self.last_frame_channel()
    fed = self.dpred_row >= 0
    if not np.array_equal(add[fed], last[fed]):
      raise ValueError("the residual add does not read the last input frame of a fed-back target")
    c = np.nonzero(fed & (add >= 0))[0]
    out[self.dpred_row[c]] = c
    return out

  def feed_index(self, directions: int = 1) -> np.ndarray:
    """[n_in] int32: the row of [this step's planes (c_in rows) | its predictions (n_out rows)] that
    becomes input channel j of the next step (next_from_input, else c_in + next_from_pred).  The
    forcings slab, channels n_in.., is the next target time's, given.  The gather index of the tangent
    feed between the steps of input_jvp.

    directions > 1: the K-fold index of the feed of that many directions at once (batched_input_jvp),
    whose buffer stacks them as [directions, c_in + n_out] rows.  Direction k's first n_in rows read
    feed_index() + k (c_in + n_out); the rows between them (the forcings slab and the predictions of
    every direction but the last) are copied through unchanged, as the next step overwrites them:
    [(directions - 1) (c_in + n_out) + n_in] in all, so that one gather feeds every direction."""
    src, pred = self.next_from_input[:self.n_in], self.next_from_pred[:self.n_in]
    if not np.all((src >= 0) | (pred >= 0)):
      raise ValueError("an input channel is neither carried nor predicted")
    one = np.where(src >= 0, src, self.c_in + pred).astype(np.int32)
    if directions == 1:
      return one
    width = self.c_in + self.n_out
    out = np.arange((directions - 1) * width + self.n_in, dtype=np.int32)
    for k in range(directions):
      out[k * width:k * width + self.n_in] = one + k * width
    return out

  def next_planes(self, planes: np.ndarray, predictions: np.ndarray,
                  next_forcings: np.ndarray) -> np.ndarray:
    """The next step's planes [c_in, ...] from this step's planes [c_in, ...], its predictions
    [n_out, ...] and the next step's forcings slab [c_in - n_in, ...]."""
    out = np.empty_like(planes)
    src = self.next_from_input >= 0
    out[src] = planes[self.next_from_input[src]]
    pred = self.next_from_pred >= 0
    out[pred] = predictions[self.next_from_pred[pred]]
    out[self.n_in:] = next_forcings
    return out


class VariableRows:
  """Where one variable of the inputs or forcings Dataset sits in the rows of an all-channel plan and
  how its gradient is formed from them: rows [start, start + count) of a step (the forcings of target
  time t in step t), summed over the axes the packing broadcast the variable to.

  mode     0: the variable has lat and lon, 1: it lacks lat (summed over lat), 2: it lacks both
           (summed over lat and lon); these are gcb_broadcast_grad_sum's modes
  batched  the variable has a batch dim; a batch-free one is summed over the batch elements
  forcing  a variable of the forcings Dataset: its rows are those of every step's forcings slab
  timed    a forcing with a time dim: one slab per target time (else the steps' slabs are summed)"""

  def __init__(self, slab: model_utils.ChannelSlab, var: xs.DataArray, forcing: bool):
    self.name, self.start, self.count = slab.name, slab.start, slab.count
    self.stack_dims, self.stack_sizes = slab.stack_dims, slab.stack_sizes
    self.var_dims = tuple(var.dims)
    self.batched = "batch" in var.dims
    has_lat, has_lon = "lat" in var.dims, "lon" in var.dims
    if has_lat and not has_lon:
      raise NotImplementedError(f"{slab.name}: input gradients of a variable with lat but no lon")
    self.mode = 0 if has_lat else (1 if has_lon else 2)
    self.forcing = forcing
    self.timed = forcing and "time" in var.dims
    self.key = ("forcings" if forcing else "inputs", slab.name)   # forcings share inputs' names

  def plane_shape(self, n_lat: int, n_lon: int) -> tuple:
    """Shape of the reduced plane of one row: (n_lat, n_lon), (n_lon,) or ()."""
    return ((n_lat, n_lon), (n_lon,), ())[self.mode]

  def reduce(self, a: np.ndarray, n_lat: int, n_lon: int) -> np.ndarray:
    """The numpy statement of gcb_broadcast_grad_sum for this variable: a [c_in, n_lat * n_lon] (the
    gradient of one step's planes) -> [count, *plane_shape], in float64."""
    x = np.asarray(a[self.start:self.start + self.count], np.float64).reshape(self.count, n_lat, n_lon)
    return x if self.mode == 0 else (x.sum(axis=1) if self.mode == 1 else x.sum(axis=(1, 2)))

  def to_variable(self, g: np.ndarray, n_lat: int, n_lon: int, directions: bool = False) -> xs.DataArray:
    """g: [batch]? ([time] for a timed forcing) [count, *plane_shape] -> the gradient as a DataArray with
    the variable's dims, in its order.  A timed forcing's per-step slab has a time dim of size 1, whose
    place the time axis of g takes.  directions: g has a leading axis of directions, and the result a
    leading "direction" dim (one copy, as for one direction)."""
    lead = ([DIRECTION] if directions else []) + (["batch"] if self.batched else [])
    if self.timed:
      lead.append("time")
    stack = [d for d in self.stack_dims if not (self.timed and d == "time")]
    sizes = [s for d, s in zip(self.stack_dims, self.stack_sizes) if not (self.timed and d == "time")]
    spatial = [("lat", "lon"), ("lon",), ()][self.mode]
    arr = np.asarray(g).reshape(list(g.shape[:len(lead)]) + sizes + list(self.plane_shape(n_lat, n_lon)))
    dims = lead + stack + list(spatial)
    var_dims = ((DIRECTION,) if directions else ()) + self.var_dims
    return xs.DataArray(np.ascontiguousarray(np.transpose(arr, [dims.index(d) for d in var_dims])),
                        var_dims)


def variable_rows(inputs: xs.Dataset, forcings: xs.Dataset) -> list:
  """VariableRows of every variable of `inputs` and of `forcings` (one target time's slab layout), in
  channel order."""
  in_slabs = model_utils.channel_layout(inputs)
  n_in = sum(s.count for s in in_slabs)
  step = forcings.isel(time=slice(0, 1)) if "time" in forcings.sizes else forcings
  f_slabs = model_utils.channel_layout(step, start=n_in)
  return ([VariableRows(s, inputs.data_vars[s.name], False) for s in in_slabs] +
          [VariableRows(s, forcings.data_vars[s.name], True) for s in f_slabs])


DIRECTION = "direction"


def check_tangents(tangents: Optional[xs.Dataset], like: xs.Dataset, what: str,
                   directions: bool = False) -> Optional[int]:
  """ValueError unless every variable of `tangents` (None: none) has a namesake in `like` with the
  same dims, in any order, and the same sizes.  With `directions`, every variable instead has a leading
  "direction" dim followed by those dims, of one size K >= 1 for all of them; returns K (None for no
  variables)."""
  if tangents is None:
    return None
  dirs = None
  for name in sorted(tangents.keys()):
    if name not in like.data_vars:
      raise ValueError(f"{what}: unknown variable {name!r}, expected one of {sorted(like.keys())}")
    v, ref = tangents.data_vars[name], like.data_vars[name]
    if directions:
      if not v.dims or v.dims[0] != DIRECTION:
        raise ValueError(f"{what}: {name} has dims {tuple(v.dims)}; a tangent of several directions "
                         f"needs the leading dim {DIRECTION!r}")
      k = v.shape[0]
      if k < 1:
        raise ValueError(f"{what}: {name} has no directions")
      if dirs is not None and k != dirs:
        raise ValueError(f"{what}: {name} has {k} directions, other variables {dirs}")
      dirs = k
      v = v.isel({DIRECTION: 0})
    if set(v.dims) != set(ref.dims) or tuple(v.transpose(*ref.dims).shape) != tuple(ref.shape):
      raise ValueError(f"{what}: {name} has dims {tuple(v.dims)} and shape {tuple(v.shape)}, the "
                       f"variable {tuple(ref.dims)} and {tuple(ref.shape)}")
  return dirs


def check_direction_tangents(input_tangents: Optional[xs.Dataset], inputs: xs.Dataset,
                             forcing_tangents: Optional[xs.Dataset], forcings: xs.Dataset):
  """(K, direction labels) of the tangents of a batched_input_jvp, after check_tangents(directions=True)
  of both Datasets: ValueError unless they agree on K and have at least one variable.  The labels are
  input_tangents' "direction" coordinate when it has one, else 0..K-1."""
  k_in = check_tangents(input_tangents, inputs, "input_tangents", directions=True)
  k_f = check_tangents(forcing_tangents, forcings, "forcing_tangents", directions=True)
  if k_in is not None and k_f is not None and k_in != k_f:
    raise ValueError(f"input_tangents have {k_in} directions, forcing_tangents {k_f}")
  dirs = k_in if k_in is not None else k_f
  if dirs is None:
    raise ValueError("the tangents have no variables, so no direction dim: give at least one")
  labels = np.arange(dirs)
  coord = None if input_tangents is None else input_tangents.coords.get(DIRECTION)
  if coord is not None and coord[0] == (DIRECTION,) and np.asarray(coord[1]).shape == (dirs,):
    labels = np.asarray(coord[1])
  return dirs, labels


def check_direction_cotangents(cotangents: xs.Dataset, template: xs.Dataset):
  """(K, direction labels) of the cotangents of a batched_input_vjp: ValueError unless they have the
  variables of `template` and each has a leading "direction" dim of one size K >= 1 for all of them,
  followed by its namesake's shape.  The variable-set and shape errors are input_vjp's.  The labels
  are the cotangents' "direction" coordinate when they have one, else 0..K-1."""
  if set(cotangents.keys()) != set(template.keys()):
    raise ValueError(f"cotangents have the variables {sorted(cotangents.keys())}, the predictions "
                     f"{sorted(template.keys())}")
  dirs = None
  for name in sorted(cotangents.keys()):
    v = cotangents.data_vars[name]
    if not v.dims or v.dims[0] != DIRECTION:
      raise ValueError(f"cotangents: {name} has dims {tuple(v.dims)}; the cotangents of several "
                       f"directions need the leading dim {DIRECTION!r}")
    if v.shape[0] < 1:
      raise ValueError(f"cotangents: {name} has no directions")
    if dirs is not None and v.shape[0] != dirs:
      raise ValueError(f"cotangents: {name} has {v.shape[0]} directions, other variables {dirs}")
    dirs = v.shape[0]
    shape, want = tuple(v.shape[1:]), tuple(template.data_vars[name].shape)
    if shape != want:
      raise ValueError(f"cotangent {name} has shape {shape}, the prediction {want}")
  if dirs is None:
    raise ValueError("the cotangents have no variables, so no direction dim")
  labels = np.arange(dirs)
  coord = cotangents.coords.get(DIRECTION)
  if coord is not None and coord[0] == (DIRECTION,) and np.asarray(coord[1]).shape == (dirs,):
    labels = np.asarray(coord[1])
  return dirs, labels


def direction_slices(dirs: int, directions_per_pass) -> list:
  """The consecutive slices of `dirs` directions that share one pass, directions_per_pass (None: all)
  each; ValueError unless it is None or an int >= 1."""
  per = dirs if directions_per_pass is None else directions_per_pass
  if isinstance(per, bool) or not isinstance(per, (int, np.integer)) or per < 1:
    raise ValueError(f"directions_per_pass must be None or an int >= 1, not {directions_per_pass!r}")
  per = int(per)
  return [slice(k0, min(k0 + per, dirs)) for k0 in range(0, dirs, per)]


def tangent_planes(tangents: Optional[xs.Dataset], like: xs.Dataset,
                   sizes: dict, directions: Optional[int] = None) -> np.ndarray:
  """[batch, channels, lat * lon] float32 planes of a tangent Dataset (check_tangents), packed exactly
  as GraphCast stages `like`: channel_layout(like) order, model_utils.variable_to_planes broadcasting
  a variable over the batch, lat and lon it lacks.  Variables `tangents` leaves out (all of them for
  None) get zero planes.  With `directions` = K (a Dataset of check_tangents(directions=True)):
  [K, batch, channels, lat * lon], direction k packed as the Dataset's slice k alone would be."""
  batch, n_lat, n_lon = sizes["batch"], sizes["lat"], sizes["lon"]
  slabs = model_utils.channel_layout(like)
  lead = () if directions is None else (directions,)
  out = np.zeros(lead + (batch, sum(s.count for s in slabs), n_lat * n_lon), np.float32)
  if directions is None:
    _fill_planes(tangents, like, sizes, slabs, out)
  else:                                           # each direction packed in place, no stacking copy
    for k in range(directions):
      _fill_planes(None if tangents is None else tangents.isel({DIRECTION: k}), like, sizes, slabs,
                   out[k])
  return out


def _fill_planes(tangents, like, sizes, slabs, out: np.ndarray) -> None:
  batch, n_lat, n_lon = sizes["batch"], sizes["lat"], sizes["lon"]
  for s in slabs:
    if tangents is None or s.name not in tangents.data_vars:
      continue
    v = tangents.data_vars[s.name].transpose(*like.data_vars[s.name].dims)
    p = model_utils.variable_to_planes(v, sizes)
    p = p.detach().cpu().numpy() if xs._is_torch(p) else np.asarray(p)
    out[:, s.start:s.start + s.count] = np.broadcast_to(
        p, (batch, s.count, n_lat, n_lon)).reshape(batch, s.count, n_lat * n_lon)


def grads_to_datasets(rows: list, grads: dict, inputs: xs.Dataset, forcings: xs.Dataset,
                      n_lat: int, n_lon: int, directions: Optional[int] = None):
  """(input_grads, forcing_grads): Datasets with the variables, dims and coords of `inputs` and
  `forcings`, from grads[VariableRows.key] as VariableRows.to_variable takes them.  With `directions`
  = K, grads[key] has a leading axis of K directions, and so has every variable ("direction" dim,
  labelled 0..K-1)."""
  out_in, out_f = xs.Dataset(coords=inputs.coords), xs.Dataset(coords=forcings.coords)
  if directions is not None:
    for out in (out_in, out_f):
      out.coords[DIRECTION] = ((DIRECTION,), np.arange(directions))
  for v in rows:
    (out_f if v.forcing else out_in)[v.name] = v.to_variable(grads[v.key], n_lat, n_lon,
                                                             directions=directions is not None)
  return out_in, out_f
