"""The host side of loss_and_joint_hvp: every refusal on the four predictor stacks before an engine
exists (those of loss_and_param_hvp, the parameter-tangent checks and the input and forcing tangent
checks), and the node-partitioned refusal of the gradient workspace.  CPU only."""
import types

import numpy as np
import pytest

from graphcast_b200 import autoregressive, casting, engine, graphcast, normalization, synthetic
from graphcast_b200 import xarray_shim as xs


def _example(task, steps=2, seed=3):
  return synthetic.make_example(task, 30.0, batch=2, num_target_steps=steps, seed=seed)


def _one(ds):
  return ds.isel(time=slice(0, 1))


def _model(task, precision="bf16x3"):
  cfg = graphcast.ModelConfig(30.0, 1, 512, 1, 1, 0.6)
  params = graphcast.init_params(cfg, task, synthetic.num_input_channels(task), seed=1)
  return graphcast.GraphCast(cfg, task, params=params, precision=precision), params


def _random_like(ds, rng, names=None):
  out = xs.Dataset(coords=ds.coords)
  for name, v in ds.data_vars.items():
    if names is None or name in names:
      out[name] = xs.DataArray(rng.standard_normal(v.shape).astype(np.float32), v.dims)
  return out


class _Other(graphcast.Predictor):
  def __call__(self, inputs, targets_template, forcings, **kwargs):
    raise AssertionError


def test_refusals_without_a_device():
  task = graphcast.TASK_13
  inputs, template, forcings = _example(task)
  model, params = _model(task)
  name = sorted(params)[0]
  v = {name: {f: np.zeros(np.shape(a), np.float32) for f, a in params[name].items()}}
  rng = np.random.default_rng(6)
  d_in = _random_like(inputs, rng, names=["2m_temperature"])
  one = (inputs, _one(template), _one(forcings))

  with pytest.raises(NotImplementedError, match="does not implement joint Hessian-vector products"):
    _Other().loss_and_joint_hvp(*one, v, d_in)
  with pytest.raises(NotImplementedError, match="does not implement joint Hessian-vector products"):
    casting.Bfloat16Cast(_Other()).loss_and_joint_hvp(*one, v, d_in)
  stats = xs.Dataset()
  generic = normalization.InputsAndResiduals(casting.Bfloat16Cast(_Other()), stats, stats, stats)
  fused = normalization.InputsAndResiduals(model, stats, stats, stats)

  bad = xs.Dataset(coords=inputs.coords)
  bad["not_a_variable"] = d_in.data_vars["2m_temperature"]
  t2m = d_in.data_vars["2m_temperature"]
  short = xs.Dataset(coords=inputs.coords)
  short["2m_temperature"] = xs.DataArray(np.asarray(t2m.values)[:1], t2m.dims)
  stacks = (model, casting.Bfloat16Cast(model), fused, autoregressive.Predictor(model),
            autoregressive.Predictor(fused))
  for pred in stacks:
    fn = pred.loss_and_joint_hvp
    # the parameter tangents, as loss_and_param_hvp checks them
    with pytest.raises(ValueError, match="unknown module"):
      fn(*one, {"no/such/module": {}})
    with pytest.raises(ValueError, match=f"unknown field {name}:nope"):
      fn(*one, {name: {"nope": np.zeros(3)}})
    with pytest.raises(ValueError, match="has shape"):
      fn(*one, {name: {f: np.zeros([1, 1, 1], np.float32) for f in params[name]}})
    with pytest.raises(ValueError, match="must be a mapping"):
      fn(*one, [v])
    # the input and forcing tangents, as loss_and_input_hvp checks them
    with pytest.raises(ValueError, match="unknown variable 'not_a_variable'"):
      fn(*one, v, bad)
    with pytest.raises(ValueError, match="2m_temperature has dims"):
      fn(*one, None, short)
    with pytest.raises(ValueError, match="forcing_tangents"):
      fn(*one, v, d_in, short)
    with pytest.raises(ValueError, match="forcing_tangents"):
      fn(*one, forcing_tangents=short)
  # the generic (non-fused) normalisation: loss_and_param_hvp's message, directly and over time
  for pred in (generic, autoregressive.Predictor(generic)):
    with pytest.raises(NotImplementedError) as want:
      pred.loss_and_param_hvp(*one, v)
    with pytest.raises(NotImplementedError, match="fused normalisation") as got:
      pred.loss_and_joint_hvp(*one, v, d_in)
    assert str(got.value) == str(want.value)
  # several target times, with or without gradient checkpointing, tangents or none
  for pred in stacks + (autoregressive.Predictor(model, gradient_checkpointing=True),
                        autoregressive.Predictor(fused, gradient_checkpointing=True)):
    for args in ((v, d_in), ()):
      with pytest.raises(NotImplementedError,
                         match="joint Hessian-vector products cover one target time"):
        pred.loss_and_joint_hvp(inputs, template, forcings, *args)
  assert model._engine is None
  # the fp32_simt precision, with tangents or none
  simt, _ = _model(task, precision="fp32_simt")
  for pred in (simt, autoregressive.Predictor(simt)):
    for args in ((v, d_in), ()):
      with pytest.raises(NotImplementedError, match="tensor-core precisions"):
        pred.loss_and_joint_hvp(*one, *args)
  assert simt._engine is None
  # a model without parameters
  bare = graphcast.GraphCast(graphcast.ModelConfig(30.0, 1, 512, 1, 1, 0.6), task)
  for args in ((v, d_in), ()):
    with pytest.raises(ValueError, match="no parameters"):
      bare.loss_and_joint_hvp(*one, *args)
  assert bare._engine is None


def test_node_partitioned_engine_is_refused():
  """loss_and_joint_hvp builds the gradient workspace through Engine.param_hvp_begin and
  Engine._grad_workspace, which refuses the node-partitioned engine (num_grid_owned set) before
  building anything; joint_hvp_element then refuses to run without it."""
  stub = types.SimpleNamespace(num_grid_owned=7, precision="bf16x3", _backward=None,
                               release_static_cache=lambda: None)
  stub._grad_workspace = lambda *a: engine.Engine._grad_workspace(stub, *a)
  stub.grads_begin = lambda: engine.Engine.grads_begin(stub)
  with pytest.raises(NotImplementedError, match="not available in the node-partitioned engine"):
    engine.Engine.param_hvp_begin(stub)
  assert stub._backward is None
  with pytest.raises(RuntimeError, match="param_hvp_begin"):
    engine.Engine.joint_hvp_element(stub, None, {}, lat_weight=None, coef=None, weight_tangents={},
                                    channel_sums=None)
