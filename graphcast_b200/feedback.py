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
    last = self.last_frame_channel()
    fed = self.dpred_row >= 0
    if not np.array_equal(add[fed], last[fed]):
      raise ValueError("the residual add does not read the last input frame of a fed-back target")
    c = np.nonzero(fed & (add >= 0))[0]
    out[self.dpred_row[c]] = c
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
