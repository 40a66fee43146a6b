"""The host side of the tangent-linear forecast of several directions (batched_input_jvp): the stacked
tangent planes against separate packings of each direction, the K-fold tangent feed between steps, and
every refusal that needs no device.  CPU only."""
import numpy as np
import pytest

from graphcast_b200 import autoregressive, casting, feedback, graphcast, normalization
from graphcast_b200 import xarray_shim as xs

TASKS = {"TASK": graphcast.TASK, "TASK_13": graphcast.TASK_13,
         "TASK_13_PRECIP_OUT": graphcast.TASK_13_PRECIP_OUT}


def _example(task, steps=2, seed=3):
  from graphcast_b200 import synthetic
  return synthetic.make_example(task, 30.0, batch=2, num_target_steps=steps, seed=seed)


def _one(ds, t=0):
  return ds.isel(time=slice(t, t + 1))


def _directions(ds, rng, k, names=None, labels=None):
  """Random tangents of `ds`'s variables (or of `names`) along k directions: a leading direction dim."""
  out = xs.Dataset(coords=ds.coords)
  if labels is not None:
    out.coords["direction"] = (("direction",), np.asarray(labels))
  for name, v in ds.data_vars.items():
    if names is None or name in names:
      out[name] = xs.DataArray(rng.standard_normal((k,) + tuple(v.shape)).astype(np.float32),
                               ("direction",) + tuple(v.dims))
  return out


def _sizes(ds):
  return {"batch": ds.sizes["batch"], "lat": ds.sizes["lat"], "lon": ds.sizes["lon"]}


@pytest.mark.parametrize("name", sorted(TASKS))
def test_stacked_tangent_planes_are_separate_packings(name):
  inputs, _, forcings = _example(TASKS[name])
  rng = np.random.default_rng(4)
  sizes = _sizes(inputs)
  for like in (inputs, _one(forcings)):
    for names in (None, sorted(like.keys())[::3]):
      d = _directions(like, rng, 3, names)
      assert feedback.check_tangents(d, like, "t", directions=True) == 3
      got = feedback.tangent_planes(d, like, sizes, 3)
      assert got.dtype == np.float32 and got.shape[0] == 3
      for k in range(3):
        assert np.array_equal(got[k], feedback.tangent_planes(d.isel(direction=k), like, sizes))
    assert not feedback.tangent_planes(None, like, sizes, 2).any()
    assert feedback.tangent_planes(None, like, sizes, 2).shape[0] == 2


@pytest.mark.parametrize("name", sorted(TASKS))
def test_kfold_feed_index_is_k_copies_with_offsets(name):
  """Direction k's fed rows read feed_index() + k (c_in + n_out); the rows between are copied through;
  gathering the stacked buffer equals K separate gathers."""
  inputs, template, forcings = _example(TASKS[name])
  plan = feedback.FeedbackPlan(inputs, _one(template), _one(forcings))
  one = plan.feed_index()
  width = plan.c_in + plan.n_out
  for dirs in (1, 2, 5):
    idx = plan.feed_index(dirs)
    assert idx.dtype == np.int32 and idx.shape == ((dirs - 1) * width + plan.n_in,)
    assert idx.min() >= 0 and idx.max() < dirs * width
    for k in range(dirs):
      assert np.array_equal(idx[k * width:k * width + plan.n_in], one + k * width)
      if k < dirs - 1:
        gap = np.arange(k * width + plan.n_in, (k + 1) * width)
        assert np.array_equal(idx[gap], gap)
    rng = np.random.default_rng(dirs)
    buf = rng.standard_normal((dirs, width, 3))
    nxt = buf.reshape(dirs * width, 3)[idx]
    for k in range(dirs):
      assert np.array_equal(nxt[k * width:k * width + plan.n_in], buf[k][one])


def test_direction_labels():
  inputs, _, forcings = _example(graphcast.TASK_13)
  rng = np.random.default_rng(5)
  f1 = _one(forcings)
  d = _directions(inputs, rng, 3, ["2m_temperature"], labels=[10, 20, 30])
  k, labels = feedback.check_direction_tangents(d, inputs, None, f1)
  assert k == 3 and list(labels) == [10, 20, 30]
  k, labels = feedback.check_direction_tangents(None, inputs, _directions(f1, rng, 2), f1)
  assert k == 2 and list(labels) == [0, 1]


def test_refusals_without_a_device():
  task = graphcast.TASK_13
  inputs, template, forcings = _example(task)
  cfg = graphcast.ModelConfig(30.0, 1, 512, 1, 1, 0.6)
  model = graphcast.GraphCast(cfg, task)
  rng = np.random.default_rng(6)
  one = (inputs, _one(template), _one(forcings))
  d_in = _directions(inputs, rng, 2, ["2m_temperature"])
  d_f = _directions(_one(forcings), rng, 2)

  class Other(graphcast.Predictor):
    def __call__(self, inputs, targets_template, forcings, **kwargs):
      raise AssertionError

  with pytest.raises(NotImplementedError, match="input gradients"):
    Other().batched_input_jvp(*one, d_in)
  stats = xs.Dataset()
  generic = normalization.InputsAndResiduals(casting.Bfloat16Cast(Other()), stats, stats, stats)
  stacks = [model, casting.Bfloat16Cast(model), autoregressive.Predictor(model)]
  v = d_in.data_vars["2m_temperature"]

  def ds(**variables):
    out = xs.Dataset(coords=inputs.coords)
    for k, a in variables.items():
      out[k] = a
    return out

  # a missing direction dim (an input_jvp tangent), directions of different sizes, an unknown
  # variable, a wrong shape, no variables at all, a bad directions_per_pass
  plain = xs.DataArray(np.asarray(v.values)[0], v.dims[1:])
  cases = [
      ((ds(**{"2m_temperature": plain}),), {}, "leading dim 'direction'"),
      ((ds(**{"2m_temperature": v, "temperature": xs.DataArray(
          rng.standard_normal((3,) + inputs.data_vars["temperature"].shape).astype(np.float32),
          ("direction",) + inputs.data_vars["temperature"].dims)}),), {}, "3 directions"),
      ((d_in, _directions(_one(forcings), rng, 3)), {}, "input_tangents have 2 directions, "
                                                         "forcing_tangents 3"),
      ((ds(not_a_variable=v),), {}, "unknown variable 'not_a_variable'"),
      ((ds(**{"2m_temperature": xs.DataArray(np.asarray(v.values)[:, :1], v.dims)}),), {},
       "2m_temperature has dims"),
      ((d_in, ds(**{"2m_temperature": v})), {}, "forcing_tangents"),
      ((xs.Dataset(coords=inputs.coords),), {}, "no variables"),
      ((ds(**{"2m_temperature": xs.DataArray(np.zeros((0,) + v.shape[1:], np.float32), v.dims)}),),
       {}, "no directions"),
      ((d_in, d_f), {"directions_per_pass": 0}, "directions_per_pass"),
      ((d_in, d_f), {"directions_per_pass": 1.5}, "directions_per_pass"),
  ]
  for stack in stacks:
    for args, kw, match in cases:
      with pytest.raises(ValueError, match=match):
        stack.batched_input_jvp(*one, *args, **kw)
  assert model._engine is None
  # the refusals of input_jvp, with its messages
  with pytest.raises(NotImplementedError, match="one target time"):
    model.batched_input_jvp(inputs, template, forcings, d_in)
  with pytest.raises(ValueError, match="unknown variable"):
    autoregressive.Predictor(model).batched_input_jvp(inputs, template, forcings, ds(bad=v))
  with pytest.raises(NotImplementedError, match="GraphCast predictor"):
    autoregressive.Predictor(Other()).batched_input_jvp(inputs, template, forcings, d_in)
  with pytest.raises(NotImplementedError, match="fused normalisation"):
    generic.batched_input_jvp(*one, d_in)
  with pytest.raises(NotImplementedError, match="fused normalisation"):
    autoregressive.Predictor(generic).batched_input_jvp(inputs, template, forcings, d_in)
  assert model._engine is None
