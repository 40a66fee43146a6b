"""The feedback plan of backprop through time (graphcast_b200.feedback) against the rollout's feeding
logic (rollout._get_next_inputs, pinned to the reference in tests/test_reference_rollout_golden.py) and
against the residual channels of the fused InputsAndResiduals constants.  CPU only."""
import numpy as np
import pytest
import torch

from graphcast_b200 import feedback, graphcast, model_utils, normalization, rollout, synthetic
from graphcast_b200 import xarray_shim as xs

TASKS = {"TASK": graphcast.TASK, "TASK_13": graphcast.TASK_13,
         "TASK_13_PRECIP_OUT": graphcast.TASK_13_PRECIP_OUT}


def _planes(*datasets, batch, n_lat, n_lon):
  """[batch, channels, lat * lon] planes of datasets stacked one after the other, as GraphCast._call
  stages them."""
  sizes = {"batch": batch, "lat": n_lat, "lon": n_lon}
  out = []
  for ds in datasets:
    for s in model_utils.channel_layout(ds):
      p = np.asarray(model_utils.variable_to_planes(ds.data_vars[s.name], sizes), np.float32)
      out.append(p.reshape(batch, s.count, n_lat * n_lon))
  return np.concatenate(out, axis=1)


def _step(task, seed=3):
  inputs, template, forcings = synthetic.make_example(task, 30.0, batch=2, num_target_steps=2,
                                                      seed=seed)
  rng = np.random.default_rng(seed)
  t0 = template.isel(time=slice(0, 1))
  predictions = xs.Dataset(coords=t0.coords)
  for name, v in t0.data_vars.items():
    predictions[name] = xs.DataArray(rng.standard_normal(v.shape).astype(np.float32), v.dims)
  f0, f1 = forcings.isel(time=slice(0, 1)), forcings.isel(time=slice(1, 2))
  return inputs, t0, predictions, f0, f1


@pytest.mark.parametrize("name", sorted(TASKS))
def test_plan_reproduces_the_rollout_feeding(name):
  task = TASKS[name]
  inputs, t0, predictions, f0, f1 = _step(task)
  # the rollout: the step's forcings join the predictions, then the frames shift
  # (rollout.chunked_prediction_generator resets the forcings' time to the target's)
  f0_like = f0.assign_coords(time=np.asarray(t0.coords["time"][1]))
  next_inputs = rollout._get_next_inputs(inputs, predictions.assign(f0_like))
  n_lat, n_lon = inputs.sizes["lat"], inputs.sizes["lon"]
  kw = dict(batch=2, n_lat=n_lat, n_lon=n_lon)
  p0 = _planes(inputs, f0, **kw)
  pred = _planes(predictions, **kw)
  forcing_next = _planes(f1, **kw)
  want = _planes(next_inputs, f1, **kw)
  plan = feedback.FeedbackPlan(inputs, t0, f0)
  assert plan.c_in == p0.shape[1] == synthetic.num_input_channels(task) and plan.n_frames == 2
  for b in range(2):
    got = plan.next_planes(p0[b], pred[b], forcing_next[b])
    np.testing.assert_array_equal(got, want[b])
  # precipitation is fed back exactly when it is an input
  slabs = {s.name: s for s in model_utils.channel_layout(t0)}
  precip = slabs["total_precipitation_6hr"]
  fed = plan.dpred_row[precip.start:precip.start + precip.count] >= 0
  assert fed.all() == ("total_precipitation_6hr" in task.input_variables) and (fed.all() or not fed.any())


@pytest.mark.parametrize("name", sorted(TASKS))
def test_backward_maps_are_the_adjoint_of_the_feeding(name):
  """<next(P, pred), A> = <P, shift^T A> + <pred, feed^T A> for A on the rows: the rows are closed under
  the map, carry_row and dpred_row are its transpose."""
  inputs, t0, predictions, f0, _ = _step(TASKS[name])
  plan = feedback.FeedbackPlan(inputs, t0, f0)
  rng = np.random.default_rng(0)
  p = rng.standard_normal((plan.c_in, 5))
  pred = rng.standard_normal((plan.n_out, 5))
  a_next = rng.standard_normal((plan.n_rows, 5))
  full = np.zeros((plan.c_in, 5))
  full[plan.rows] = a_next
  lhs = (plan.next_planes(p, pred, np.zeros((plan.c_in - plan.n_in, 5))) * full).sum()
  a_p = np.zeros((plan.c_in, 5))
  carried = plan.carry_row >= 0
  a_p[plan.rows[carried]] = a_next[plan.carry_row[carried]]
  a_pred = np.where((plan.dpred_row >= 0)[:, None], a_next[np.maximum(plan.dpred_row, 0)], 0.0)
  rhs = (p * a_p).sum() + (pred * a_pred).sum()
  assert abs(lhs - rhs) <= 1e-9 * abs(lhs)
  # every row is a frame of a time-dependent input that is also a target
  layout = {s.name: s for s in model_utils.channel_layout(inputs)}
  targets = set(t0.keys())
  for ch in plan.rows:
    s = next(s for s in layout.values() if s.start <= ch < s.start + s.count)
    assert s.name in targets and s.stack_dims[0] == "time"


def _stats(task):
  rng = np.random.default_rng(0)
  levels = np.asarray(task.pressure_levels)
  ds = xs.Dataset(coords={"level": levels})
  for name in set(task.input_variables) | set(task.target_variables) | set(task.forcing_variables):
    if name in graphcast.variables.ALL_ATMOSPHERIC_VARS:
      ds[name] = xs.DataArray(rng.uniform(0.5, 2.0, len(levels)).astype(np.float32), ("level",))
    else:
      ds[name] = xs.DataArray(np.float32(rng.uniform(0.5, 2.0)), ())
  return ds


@pytest.mark.parametrize("name", sorted(TASKS))
def test_plan_agrees_with_the_residual_channels(name):
  task = TASKS[name]
  inputs, t0, _, f0, _ = _step(task)
  stats = _stats(task)
  iar = normalization.InputsAndResiduals(graphcast.GraphCast(
      graphcast.ModelConfig(30.0, 1, 512, 1, 1, 0.6), task), stats, stats, stats)
  add = iar._fused_constants(inputs, t0, f0, torch.device("cpu")).add_plane_index.numpy()
  plan = feedback.FeedbackPlan(inputs, t0, f0)
  fed = plan.dpred_row >= 0
  assert np.array_equal(fed, add >= 0)
  assert np.array_equal(plan.last_frame_channel()[fed], add[fed])
  resid = plan.resid_channel(add)
  assert np.array_equal(np.sort(resid[resid >= 0]), np.nonzero(add >= 0)[0])
  assert np.array_equal(plan.rows[plan.dpred_row[resid[resid >= 0]]], add[resid[resid >= 0]])
  assert (plan.resid_channel(None) == -1).all()
  bad = add.copy()
  bad[np.nonzero(fed)[0][0]] += 1
  with pytest.raises(ValueError, match="last input frame"):
    plan.resid_channel(bad)


def test_plan_rejects_time_not_leading():
  inputs, t0, _, f0, _ = _step(graphcast.TASK_13)
  v = inputs.data_vars["temperature"]
  inputs["temperature"] = v.transpose("batch", "level", "time", "lat", "lon")
  with pytest.raises(ValueError, match="leading stacked dim"):
    feedback.FeedbackPlan(inputs, t0, f0)
