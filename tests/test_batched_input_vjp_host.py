"""The host side of input_vjp for several cotangents (batched_input_vjp): every refusal before anything
runs on the device, and the passes' helper, which joins the gradient Datasets of consecutive slices of
the directions along "direction" with either kind of label.  CPU only."""
import numpy as np
import pytest

from graphcast_b200 import autoregressive, casting, feedback, graphcast, normalization
from graphcast_b200 import xarray_shim as xs


def _example(task, steps=2, seed=3):
  from graphcast_b200 import synthetic
  return synthetic.make_example(task, 30.0, batch=2, num_target_steps=steps, seed=seed)


def _one(ds, t=0):
  return ds.isel(time=slice(t, t + 1))


def _directions(ds, rng, k, labels=None):
  """Random values of every variable of `ds` along k directions: a leading direction dim."""
  out = xs.Dataset(coords=ds.coords)
  if labels is not None:
    out.coords["direction"] = (("direction",), np.asarray(labels))
  for name, v in ds.data_vars.items():
    out[name] = xs.DataArray(rng.standard_normal((k,) + tuple(v.shape)).astype(np.float32),
                             ("direction",) + tuple(v.dims))
  return out


def test_cotangent_checks_and_labels():
  _, template, _ = _example(graphcast.TASK_13)
  rng = np.random.default_rng(4)
  one = _one(template)
  assert feedback.check_direction_cotangents(_directions(one, rng, 3), one)[0] == 3
  k, labels = feedback.check_direction_cotangents(_directions(one, rng, 2, labels=[7, 9]), one)
  assert k == 2 and list(labels) == [7, 9]
  k, labels = feedback.check_direction_cotangents(_directions(template, rng, 1), template)
  assert k == 1 and list(labels) == [0]
  assert feedback.direction_slices(5, None) == [slice(0, 5)]
  assert feedback.direction_slices(5, 2) == [slice(0, 2), slice(2, 4), slice(4, 5)]
  assert feedback.direction_slices(3, np.int64(7)) == [slice(0, 3)]


@pytest.mark.parametrize("labels", [None, [30, 10, 20, 40, 50]])
@pytest.mark.parametrize("per", [None, 1, 2, 5])
def test_passes_join_gradients_along_direction(labels, per):
  """direction_passes over slices of 5 directions, each pass returning per-direction gradient Datasets
  as _InputGradRun.finish does (feedback.grads_to_datasets with directions), gives the Datasets of
  all directions at once, with the labels given or 0..K-1."""
  inputs, template, forcings = _example(graphcast.TASK_13)
  f1 = _one(forcings)
  rows = feedback.variable_rows(inputs, f1)
  n_lat, n_lon = inputs.sizes["lat"], inputs.sizes["lon"]
  rng = np.random.default_rng(5)
  width = lambda v: (n_lat * n_lon, n_lon, 1)[v.mode]
  shape = lambda v: ([2] if v.batched else []) + ([1] if v.timed else []) + [v.count, width(v)]
  grads = {v.key: rng.standard_normal([5] + shape(v)).astype(np.float32) for v in rows}
  want_in, want_f = feedback.grads_to_datasets(rows, grads, inputs, f1, n_lat, n_lon, directions=5)
  for out, ds in ((want_in, inputs), (want_f, f1)):
    assert set(out.keys()) == set(ds.keys())
    for name, v in out.data_vars.items():
      assert v.dims == ("direction",) + ds.data_vars[name].dims
      assert tuple(v.shape) == (5,) + tuple(ds.data_vars[name].shape)
  for k in range(5):                      # direction k is what one direction's grads give
    one_in, one_f = feedback.grads_to_datasets(rows, {key: g[k] for key, g in grads.items()}, inputs,
                                               f1, n_lat, n_lon)
    for got, one in ((want_in, one_in), (want_f, one_f)):
      for name in one.keys():
        assert np.array_equal(np.asarray(got.data_vars[name].values)[k],
                              np.asarray(one.data_vars[name].values)), (k, name)
  seen = []

  def one_pass(sl):
    seen.append(sl)
    part = {key: g[sl] for key, g in grads.items()}
    pi, pf = feedback.grads_to_datasets(rows, part, inputs, f1, n_lat, n_lon,
                                        directions=sl.stop - sl.start)
    return ("predictions" if sl.start == 0 else None), pi, pf

  want_labels = np.arange(5) if labels is None else np.asarray(labels)
  p, gi, gf = graphcast.direction_passes(one_pass, 5, want_labels, per)
  assert p == "predictions" and len(seen) == -(-5 // (per or 5))
  for got, want in ((gi, want_in), (gf, want_f)):
    assert list(np.asarray(got.coords["direction"][1])) == list(want_labels)
    assert set(got.keys()) == set(want.keys())
    for name, v in want.data_vars.items():
      assert got.data_vars[name].dims == v.dims
      assert np.array_equal(np.asarray(got.data_vars[name].values), np.asarray(v.values)), name


def test_refusals_without_a_device():
  task = graphcast.TASK_13
  inputs, template, forcings = _example(task)
  cfg = graphcast.ModelConfig(30.0, 1, 512, 1, 1, 0.6)
  model = graphcast.GraphCast(cfg, task)
  rng = np.random.default_rng(6)
  one = (inputs, _one(template), forcings.isel(time=slice(0, 1)))
  cot = _directions(_one(template), rng, 2)

  class Other(graphcast.Predictor):
    def __call__(self, inputs, targets_template, forcings, **kwargs):
      raise AssertionError

  with pytest.raises(NotImplementedError, match="input gradients"):
    Other().batched_input_vjp(*one, cot)
  stats = xs.Dataset()
  generic = normalization.InputsAndResiduals(casting.Bfloat16Cast(Other()), stats, stats, stats)
  fused = normalization.InputsAndResiduals(model, stats, stats, stats)
  stacks = [model, casting.Bfloat16Cast(model), fused, autoregressive.Predictor(model),
            autoregressive.Predictor(fused, gradient_checkpointing=True)]
  name = "2m_temperature"
  v = cot.data_vars[name]

  def ds(**variables):
    out = xs.Dataset(coords=cot.coords)
    for k, a in cot.data_vars.items():
      out[k] = a
    for k, a in variables.items():
      out[k] = a
    return out

  def without(drop):
    out = xs.Dataset(coords=cot.coords)
    for k, a in cot.data_vars.items():
      if k != drop:
        out[k] = a
    return out

  three = xs.DataArray(rng.standard_normal((3,) + tuple(v.shape[1:])).astype(np.float32), v.dims)
  cases = [
      # a missing direction dim (an input_vjp cotangent)
      ((ds(**{name: xs.DataArray(np.asarray(v.values)[0], v.dims[1:])}),), {},
       "leading dim 'direction'"),
      ((ds(**{name: three}),), {}, "3 directions, other variables 2|2 directions, other variables 3"),
      ((without(name),), {}, "cotangents have the variables"),             # input_vjp's message
      ((ds(not_a_variable=v),), {}, "cotangents have the variables"),
      ((ds(**{name: xs.DataArray(np.asarray(v.values)[:, :1], v.dims)}),), {},
       f"cotangent {name} has shape"),                                      # input_vjp's message
      ((ds(**{name: xs.DataArray(np.zeros((0,) + tuple(v.shape[1:]), np.float32), v.dims)}),), {},
       "no directions"),
      ((cot,), {"directions_per_pass": 0}, "directions_per_pass"),
      ((cot,), {"directions_per_pass": 1.5}, "directions_per_pass"),
      ((cot,), {"directions_per_pass": True}, "directions_per_pass"),
  ]
  for stack in stacks:
    for args, kw, match in cases:
      with pytest.raises(ValueError, match=match):
        stack.batched_input_vjp(*one, *args, **kw)
  assert model._engine is None
  # several target times: the cotangents follow the whole template
  ar = autoregressive.Predictor(fused, gradient_checkpointing=True)
  with pytest.raises(ValueError, match="cotangent .* has shape"):
    ar.batched_input_vjp(inputs, template, forcings, cot)
  with pytest.raises(ValueError, match="directions_per_pass"):
    ar.batched_input_vjp(inputs, template, forcings, _directions(template, rng, 2),
                         directions_per_pass=-1)
  assert model._engine is None
  # the refusals of input_vjp, with its messages
  full = _directions(template, rng, 2)
  with pytest.raises(NotImplementedError, match="one target time"):
    model.batched_input_vjp(inputs, template, forcings, full)
  with pytest.raises(NotImplementedError, match="gradient_checkpointing=True"):
    autoregressive.Predictor(model).batched_input_vjp(inputs, template, forcings, full)
  with pytest.raises(NotImplementedError, match="GraphCast predictor"):
    autoregressive.Predictor(Other(), gradient_checkpointing=True).batched_input_vjp(
        inputs, template, forcings, full)
  with pytest.raises(NotImplementedError, match="fused normalisation"):
    generic.batched_input_vjp(*one, cot)
  with pytest.raises(NotImplementedError, match="fused normalisation"):
    autoregressive.Predictor(generic, gradient_checkpointing=True).batched_input_vjp(
        inputs, template, forcings, full)
  assert model._engine is None
