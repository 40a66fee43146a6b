"""The host side of the input gradients (loss_and_input_grads / input_vjp): the all-channel feedback
plan as the exact transpose of the rollout's feeding, the row -> variable map and its broadcast sums
as the transpose of the packing, and the refusals that need no device.  CPU only."""
import numpy as np
import pytest

from graphcast_b200 import (autoregressive, casting, feedback, graphcast, model_utils,
                            normalization, synthetic)
from graphcast_b200 import xarray_shim as xs

TASKS = {"TASK": graphcast.TASK, "TASK_13": graphcast.TASK_13,
         "TASK_13_PRECIP_OUT": graphcast.TASK_13_PRECIP_OUT}


def _example(task, steps=2, seed=3):
  return synthetic.make_example(task, 30.0, batch=2, num_target_steps=steps, seed=seed)


def _one(ds):
  return ds.isel(time=slice(0, 1))


@pytest.mark.parametrize("name", sorted(TASKS))
def test_all_channel_plan_is_the_adjoint_of_the_feeding(name):
  """<next_planes(P, Y, F), A> = <P, A^T_P> + <Y, A^T_Y> + <F, A^T_F> with the transposes formed from
  carry_row, dpred_row and the forcings rows alone, for random fp64 P, Y, F and A."""
  inputs, template, forcings = _example(TASKS[name])
  plan = feedback.FeedbackPlan.all_channels(inputs, _one(template), _one(forcings))
  assert np.array_equal(plan.rows, np.arange(plan.c_in)) and plan.n_rows == plan.c_in
  rng = np.random.default_rng(1)
  n = 7
  p = rng.standard_normal((plan.c_in, n))
  y = rng.standard_normal((plan.n_out, n))
  f = rng.standard_normal((plan.c_in - plan.n_in, n))
  a = rng.standard_normal((plan.c_in, n))
  lhs = (plan.next_planes(p, y, f) * a).sum()
  a_p = np.where((plan.carry_row >= 0)[:, None], a[np.maximum(plan.carry_row, 0)], 0.0)
  a_y = np.where((plan.dpred_row >= 0)[:, None], a[np.maximum(plan.dpred_row, 0)], 0.0)
  a_f = a[plan.n_in:]
  rhs = (p * a_p).sum() + (y * a_y).sum() + (f * a_f).sum()
  assert abs(lhs - rhs) <= 1e-12 * max(1.0, abs(lhs))
  # every forcings row carries into the last input frame of the same variable, when it is an input
  layout = {s.name: s for s in model_utils.channel_layout(inputs)}
  for s in model_utils.channel_layout(_one(forcings), start=plan.n_in):
    carried = plan.carry_row[s.start:s.start + s.count]
    if s.name in layout:
      src = layout[s.name]
      assert np.array_equal(carried, src.start + src.count - s.count + np.arange(s.count))
    else:
      assert (carried == -1).all()


@pytest.mark.parametrize("name", sorted(TASKS))
def test_all_channel_plan_leaves_the_bptt_plan_alone(name):
  inputs, template, forcings = _example(TASKS[name])
  a = feedback.FeedbackPlan(inputs, _one(template), _one(forcings))
  feedback.FeedbackPlan.all_channels(inputs, _one(template), _one(forcings))
  b = feedback.FeedbackPlan(inputs, _one(template), _one(forcings))
  for field in ("rows", "dpred_row", "carry_row", "next_from_input", "next_from_pred"):
    assert np.array_equal(getattr(a, field), getattr(b, field))
  assert not a.all_rows


def test_all_channel_residual_rows():
  task = graphcast.TASK_13
  inputs, template, forcings = _example(task)
  plan = feedback.FeedbackPlan.all_channels(inputs, _one(template), _one(forcings))
  bptt = feedback.FeedbackPlan(inputs, _one(template), _one(forcings))
  add = np.where(bptt.dpred_row >= 0, bptt.last_frame_channel(), -1)
  resid = plan.resid_channel(add)
  c = np.nonzero(add >= 0)[0]
  assert np.array_equal(resid[add[c]], c)
  assert (np.delete(resid, add[c]) == -1).all()
  # the residual reads the channel the prediction feeds: the same row as dpred_row
  assert np.array_equal(plan.dpred_row[c], add[c])


def _random_like(ds, rng):
  out = xs.Dataset(coords=ds.coords)
  for name, v in ds.data_vars.items():
    out[name] = xs.DataArray(rng.standard_normal(v.shape), v.dims)
  return out


@pytest.mark.parametrize("name", sorted(TASKS))
def test_variable_rows_are_the_transpose_of_the_packing(name):
  """For random variables X and random planes A of every step: <pack(X), A> = <X, grads(A)>, where
  pack is GraphCast's staging (model_utils.variable_to_planes, broadcasting over batch, lat and lon)
  and grads the row -> variable map with its broadcast sums (the numpy statement of
  gcb_broadcast_grad_sum), batch-free variables summed over the batch, forcings per target time."""
  inputs, template, forcings = _example(TASKS[name], steps=3)
  rng = np.random.default_rng(2)
  x_in, x_f = _random_like(inputs, rng), _random_like(forcings, rng)
  batch, n_lat, n_lon = inputs.sizes["batch"], inputs.sizes["lat"], inputs.sizes["lon"]
  sizes = {"batch": batch, "lat": n_lat, "lon": n_lon}
  rows = feedback.variable_rows(inputs, forcings)
  c_in = sum(v.count for v in rows)
  steps = forcings.sizes["time"]
  a = rng.standard_normal((steps, batch, c_in, n_lat * n_lon))
  # step t's planes: the inputs (only step 0 is read for them) and the forcings of target time t
  lhs = 0.0
  for v in rows:
    for t in range(steps if v.forcing else 1):
      src = x_f.isel(time=slice(t, t + 1)) if v.forcing else x_in
      planes = np.asarray(model_utils.variable_to_planes(src.data_vars[v.name], sizes), np.float64)
      lhs += (planes.reshape(batch, v.count, -1) * a[t, :, v.start:v.start + v.count]).sum()
  grads = {}
  for v in rows:
    per = [[v.reduce(a[t, b], n_lat, n_lon) for t in range(steps if v.forcing else 1)]
           for b in range(batch)]
    g = np.asarray(per)                                   # [batch, steps, count, *plane]
    g = g if v.timed else g.sum(axis=1)
    grads[v.key] = g if v.batched else g.sum(axis=0)
  g_in, g_f = feedback.grads_to_datasets(rows, grads, inputs, forcings, n_lat, n_lon)
  rhs = 0.0
  for x, g in ((x_in, g_in), (x_f, g_f)):
    assert set(g.keys()) == set(x.keys())
    for k in x.keys():
      assert g.data_vars[k].dims == x.data_vars[k].dims
      assert tuple(g.data_vars[k].shape) == tuple(x.data_vars[k].shape)
      rhs += (np.asarray(x.data_vars[k].values) * np.asarray(g.data_vars[k].values)).sum()
  assert abs(lhs - rhs) <= 1e-10 * abs(lhs)
  # the broadcast variables of the synthetic data take the three modes
  mode = {v.name: (v.mode, v.batched) for v in rows}
  assert mode["land_sea_mask"] == (0, False)
  assert mode["year_progress_sin"] == (2, True)
  assert mode["day_progress_cos"] == (1, True)


def test_variable_rows_reject_lat_without_lon():
  inputs, _, forcings = _example(graphcast.TASK_13)
  v = inputs.data_vars["land_sea_mask"]
  inputs["land_sea_mask"] = xs.DataArray(np.asarray(v.values)[:, 0], ("lat",))
  with pytest.raises(NotImplementedError, match="lat but no lon"):
    feedback.variable_rows(inputs, forcings)


def test_refusals_without_a_device():
  task = graphcast.TASK_13
  inputs, template, forcings = _example(task)
  cfg = graphcast.ModelConfig(30.0, 1, 512, 1, 1, 0.6)
  model = graphcast.GraphCast(cfg, task)

  class Other(graphcast.Predictor):
    def __call__(self, inputs, targets_template, forcings, **kwargs):
      raise AssertionError

  with pytest.raises(NotImplementedError, match="input gradients"):
    Other().loss_and_input_grads(inputs, template, forcings)
  with pytest.raises(NotImplementedError, match="input gradients"):
    Other().input_vjp(inputs, template, forcings, template)
  # several target times without checkpointing, or around a predictor that is not GraphCast
  ar = autoregressive.Predictor(model)
  with pytest.raises(NotImplementedError, match="gradient_checkpointing=True"):
    ar.loss_and_input_grads(inputs, template, forcings)
  with pytest.raises(NotImplementedError, match="gradient_checkpointing=True"):
    ar.input_vjp(inputs, template, forcings, template)
  with pytest.raises(NotImplementedError, match="GraphCast predictor"):
    autoregressive.Predictor(Other(), gradient_checkpointing=True).loss_and_input_grads(
        inputs, template, forcings)
  # GraphCast itself covers one target time
  with pytest.raises(NotImplementedError, match="one target time"):
    model.loss_and_input_grads(inputs, template, forcings)
  with pytest.raises(NotImplementedError, match="one target time"):
    model.input_vjp(inputs, template, forcings, template)
  # the generic (non-fused) normalisation
  stats = xs.Dataset()
  generic = normalization.InputsAndResiduals(casting.Bfloat16Cast(Other()), stats, stats, stats)
  with pytest.raises(NotImplementedError, match="fused normalisation"):
    generic.loss_and_input_grads(inputs, _one(template), _one(forcings))
  with pytest.raises(NotImplementedError, match="fused normalisation"):
    generic.input_vjp(inputs, _one(template), _one(forcings), _one(template))
