"""The host side of the tangent-linear forecast (input_jvp): tangent Datasets packed exactly as the
primal inputs are, the tangent feed between steps as the rollout's feeding of the next inputs, and
the refusals that need no device.  CPU only."""
import numpy as np
import pytest

from graphcast_b200 import (autoregressive, casting, feedback, graphcast, model_utils,
                            normalization, rollout, synthetic)
from graphcast_b200 import xarray_shim as xs

TASKS = {"TASK": graphcast.TASK, "TASK_13": graphcast.TASK_13,
         "TASK_13_PRECIP_OUT": graphcast.TASK_13_PRECIP_OUT}


def _example(task, steps=2, seed=3):
  return synthetic.make_example(task, 30.0, batch=2, num_target_steps=steps, seed=seed)


def _one(ds, t=0):
  return ds.isel(time=slice(t, t + 1))


def _random_like(ds, rng, names=None):
  out = xs.Dataset(coords=ds.coords)
  for name, v in ds.data_vars.items():
    if names is None or name in names:
      out[name] = xs.DataArray(rng.standard_normal(v.shape).astype(np.float32), v.dims)
  return out


def _sizes(ds):
  return {"batch": ds.sizes["batch"], "lat": ds.sizes["lat"], "lon": ds.sizes["lon"]}


def _packed(ds, sizes):
  """The primal packing of GraphCast._call: [batch, channels, lat * lon]."""
  stacked = model_utils.dataset_to_stacked(ds, sizes)          # [batch, lat, lon, channels]
  return np.transpose(stacked, (0, 3, 1, 2)).reshape(sizes["batch"], stacked.shape[-1], -1)


@pytest.mark.parametrize("name", sorted(TASKS))
def test_tangent_planes_follow_the_primal_packing(name):
  inputs, _, forcings = _example(TASKS[name])
  rng = np.random.default_rng(4)
  sizes = _sizes(inputs)
  for like in (inputs, _one(forcings)):
    full = _random_like(like, rng)
    got = feedback.tangent_planes(full, like, sizes)
    assert got.dtype == np.float32
    assert np.array_equal(got, _packed(full, sizes))
    # a subset: the variables left out are zero rows, the others unchanged
    keep = sorted(like.keys())[::2]
    sub = xs.Dataset(coords=like.coords)
    for k in keep:
      sub[k] = full.data_vars[k]
    part = feedback.tangent_planes(sub, like, sizes)
    for s in model_utils.channel_layout(like):
      rows = slice(s.start, s.start + s.count)
      want = got[:, rows] if s.name in keep else np.zeros_like(got[:, rows])
      assert np.array_equal(part[:, rows], want), s.name
    assert not feedback.tangent_planes(None, like, sizes).any()
  # the broadcast variables: no batch (land_sea_mask), no lat (day_progress_cos), neither lat nor lon
  # (year_progress_sin), and a tangent given in another dim order
  full = _random_like(inputs, rng)
  dims = {n: full.data_vars[n].dims for n in ("land_sea_mask", "day_progress_cos", "year_progress_sin")}
  assert "batch" not in dims["land_sea_mask"] and "lat" not in dims["day_progress_cos"]
  assert "lon" not in dims["year_progress_sin"]
  turned = xs.Dataset(coords=full.coords)
  for k, v in full.data_vars.items():
    turned[k] = v.transpose(*reversed(v.dims))
  assert np.array_equal(feedback.tangent_planes(turned, inputs, sizes), _packed(full, sizes))


@pytest.mark.parametrize("name", sorted(TASKS))
def test_feed_index_is_the_rollout_feeding(name):
  """The next step's tangent planes gathered from [planes | predictions] by feed_index equal the
  packing of rollout._get_next_inputs applied to the tangent Datasets, for random tangents of the
  inputs, the predictions and the forcings of the step."""
  inputs, template, forcings = _example(TASKS[name])
  plan = feedback.FeedbackPlan(inputs, _one(template), _one(forcings))
  rng = np.random.default_rng(5)
  sizes = _sizes(inputs)
  d_in, d_pred, d_f = _random_like(inputs, rng), _random_like(_one(template), rng), \
      _random_like(_one(forcings), rng)
  planes = np.concatenate([feedback.tangent_planes(d_in, inputs, sizes),
                           feedback.tangent_planes(d_f, _one(forcings), sizes),
                           feedback.tangent_planes(d_pred, _one(template), sizes)], axis=1)
  idx = plan.feed_index()
  assert idx.dtype == np.int32 and idx.shape == (plan.n_in,)
  assert idx.min() >= 0 and idx.max() < plan.c_in + plan.n_out
  got = planes[:, idx]
  want = rollout._get_next_inputs(d_in, d_pred.assign(d_f))
  assert np.array_equal(got, feedback.tangent_planes(want, inputs, sizes))
  # the same map as next_planes, which also sets the forcings slab
  nxt = rng.standard_normal((plan.c_in - plan.n_in, 3))
  p, y = rng.standard_normal((plan.c_in, 3)), rng.standard_normal((plan.n_out, 3))
  assert np.array_equal(plan.next_planes(p, y, nxt)[:plan.n_in], np.concatenate([p, y])[idx])


def test_refusals_without_a_device():
  task = graphcast.TASK_13
  inputs, template, forcings = _example(task)
  cfg = graphcast.ModelConfig(30.0, 1, 512, 1, 1, 0.6)
  model = graphcast.GraphCast(cfg, task)
  rng = np.random.default_rng(6)
  d_in = _random_like(inputs, rng, names=["2m_temperature"])
  one = (inputs, _one(template), _one(forcings))

  class Other(graphcast.Predictor):
    def __call__(self, inputs, targets_template, forcings, **kwargs):
      raise AssertionError

  with pytest.raises(NotImplementedError, match="input gradients"):
    Other().input_jvp(*one, d_in)
  # an unknown variable, a wrong shape, wrong dims: ValueError before the engine exists
  bad = xs.Dataset(coords=inputs.coords)
  bad["not_a_variable"] = d_in.data_vars["2m_temperature"]
  with pytest.raises(ValueError, match="unknown variable 'not_a_variable'"):
    model.input_jvp(*one, bad)
  v = d_in.data_vars["2m_temperature"]
  short = xs.Dataset(coords=inputs.coords)
  short["2m_temperature"] = xs.DataArray(np.asarray(v.values)[:1], v.dims)
  with pytest.raises(ValueError, match="2m_temperature has dims"):
    model.input_jvp(*one, short)
  with pytest.raises(ValueError, match="forcing_tangents"):
    model.input_jvp(*one, d_in, short)
  lost = xs.Dataset(coords=inputs.coords)
  lost["2m_temperature"] = xs.DataArray(np.asarray(v.values)[:, 0], tuple(d for d in v.dims if d != "time"))
  with pytest.raises(ValueError, match="2m_temperature has dims"):
    model.input_jvp(*one, lost)
  assert model._engine is None
  # GraphCast covers one target time; several target times check the tangents before the rollout
  with pytest.raises(NotImplementedError, match="one target time"):
    model.input_jvp(inputs, template, forcings, d_in)
  with pytest.raises(ValueError, match="unknown variable"):
    autoregressive.Predictor(model).input_jvp(inputs, template, forcings, bad)
  with pytest.raises(ValueError, match="forcing_tangents"):
    autoregressive.Predictor(model).input_jvp(inputs, template, forcings, d_in,
                                              _random_like(_one(forcings), rng))
  assert model._engine is None
  # several target times around a predictor that is not GraphCast
  with pytest.raises(NotImplementedError, match="GraphCast predictor"):
    autoregressive.Predictor(Other()).input_jvp(inputs, template, forcings, d_in)
  # the generic (non-fused) normalisation, directly and over several target times
  stats = xs.Dataset()
  generic = normalization.InputsAndResiduals(casting.Bfloat16Cast(Other()), stats, stats, stats)
  with pytest.raises(NotImplementedError, match="fused normalisation"):
    generic.input_jvp(*one, d_in)
  with pytest.raises(NotImplementedError, match="fused normalisation"):
    autoregressive.Predictor(generic).input_jvp(inputs, template, forcings, d_in)
