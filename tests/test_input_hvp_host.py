"""The refusals of loss_and_input_hvp that need no device: those of loss_and_input_grads and the
tangent checks of input_jvp, with their messages, on every stack, before an engine exists; and the
packing of the tangent planes.  CPU only."""
import numpy as np
import pytest

from graphcast_b200 import autoregressive, casting, feedback, graphcast, normalization, synthetic
from graphcast_b200 import xarray_shim as xs


def _example(task, steps=2, seed=3):
  return synthetic.make_example(task, 30.0, batch=2, num_target_steps=steps, seed=seed)


def _one(ds):
  return ds.isel(time=slice(0, 1))


def _random_like(ds, rng, names=None):
  out = xs.Dataset(coords=ds.coords)
  for name, v in ds.data_vars.items():
    if names is None or name in names:
      out[name] = xs.DataArray(rng.standard_normal(v.shape).astype(np.float32), v.dims)
  return out


class _Other(graphcast.Predictor):
  def __call__(self, inputs, targets_template, forcings, **kwargs):
    raise AssertionError


def test_tangent_planes_are_inputs_then_forcings():
  inputs, template, forcings = _example(graphcast.TASK_13)
  rng = np.random.default_rng(2)
  d_in, d_f = _random_like(inputs, rng), _random_like(_one(forcings), rng)
  planes = graphcast.hvp_tangent_planes(inputs, _one(forcings), d_in, d_f).numpy()
  sizes = {"batch": 2, "lat": inputs.sizes["lat"], "lon": inputs.sizes["lon"]}
  want = np.concatenate([feedback.tangent_planes(d_in, inputs, sizes),
                         feedback.tangent_planes(d_f, _one(forcings), sizes)], axis=1)
  assert np.array_equal(planes, want)
  no_f = graphcast.hvp_tangent_planes(inputs, _one(forcings), d_in, None).numpy()
  n_in = feedback.tangent_planes(d_in, inputs, sizes).shape[1]
  assert np.array_equal(no_f[:, :n_in], want[:, :n_in]) and not np.any(no_f[:, n_in:])


def test_refusals_without_a_device():
  task = graphcast.TASK_13
  inputs, template, forcings = _example(task)
  cfg = graphcast.ModelConfig(30.0, 1, 512, 1, 1, 0.6)
  model = graphcast.GraphCast(cfg, task)
  rng = np.random.default_rng(6)
  d_in = _random_like(inputs, rng, names=["2m_temperature"])
  one = (inputs, _one(template), _one(forcings))

  with pytest.raises(NotImplementedError, match="Hessian-vector products"):
    _Other().loss_and_input_hvp(*one, d_in)
  bad = xs.Dataset(coords=inputs.coords)
  bad["not_a_variable"] = d_in.data_vars["2m_temperature"]
  v = d_in.data_vars["2m_temperature"]
  short = xs.Dataset(coords=inputs.coords)
  short["2m_temperature"] = xs.DataArray(np.asarray(v.values)[:1], v.dims)
  lost = xs.Dataset(coords=inputs.coords)
  lost["2m_temperature"] = xs.DataArray(np.asarray(v.values)[:, 0],
                                        tuple(d for d in v.dims if d != "time"))
  stacks = [model, casting.Bfloat16Cast(model), autoregressive.Predictor(model),
            autoregressive.Predictor(model, gradient_checkpointing=True)]
  for pred in stacks:
    with pytest.raises(ValueError, match="unknown variable 'not_a_variable'"):
      pred.loss_and_input_hvp(*one, bad)
    with pytest.raises(ValueError, match="2m_temperature has dims"):
      pred.loss_and_input_hvp(*one, short)
    with pytest.raises(ValueError, match="forcing_tangents"):
      pred.loss_and_input_hvp(*one, d_in, short)
    with pytest.raises(ValueError, match="2m_temperature has dims"):
      pred.loss_and_input_hvp(*one, lost)
  # GraphCast and Bfloat16Cast cover one target time, as loss_and_input_grads does
  for pred in stacks[:2]:
    with pytest.raises(NotImplementedError, match="one target time"):
      pred.loss_and_input_hvp(inputs, template, forcings, d_in)
    with pytest.raises(NotImplementedError, match="one target time"):
      pred.loss_and_input_grads(inputs, template, forcings)
  # several target times: the refusals of loss_and_input_grads, then the tangent checks
  with pytest.raises(NotImplementedError, match="gradient_checkpointing=True"):
    stacks[2].loss_and_input_hvp(inputs, template, forcings, d_in)
  with pytest.raises(NotImplementedError, match="gradient_checkpointing=True"):
    stacks[2].loss_and_input_grads(inputs, template, forcings)
  with pytest.raises(NotImplementedError, match="GraphCast predictor"):
    autoregressive.Predictor(_Other(), gradient_checkpointing=True).loss_and_input_hvp(
        inputs, template, forcings, d_in)
  with pytest.raises(ValueError, match="unknown variable 'not_a_variable'"):
    stacks[3].loss_and_input_hvp(inputs, template, forcings, bad)
  with pytest.raises(ValueError, match="forcing_tangents"):
    stacks[3].loss_and_input_hvp(inputs, template, forcings, d_in, _random_like(_one(forcings), rng))
  assert model._engine is None
  # the generic (non-fused) normalisation refuses as loss_and_input_grads does
  stats = xs.Dataset()
  generic = normalization.InputsAndResiduals(casting.Bfloat16Cast(_Other()), stats, stats, stats)
  with pytest.raises(NotImplementedError) as want:
    generic.loss_and_input_grads(*one)
  with pytest.raises(NotImplementedError) as got:
    generic.loss_and_input_hvp(*one, d_in)
  assert str(got.value) == str(want.value)
