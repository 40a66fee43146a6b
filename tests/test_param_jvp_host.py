"""The host side of param_jvp and loss_and_param_gnvp: the checks of the parameter tangents, every
refusal on the four predictor stacks before an engine exists, and the GPU-free refusals of the two new
C entry points.  CPU only."""
import numpy as np
import pytest

from graphcast_b200 import _native, autoregressive, casting, graphcast, normalization, synthetic
from graphcast_b200 import xarray_shim as xs


def _example(task, steps=2, seed=3):
  return synthetic.make_example(task, 30.0, batch=2, num_target_steps=steps, seed=seed)


def _one(ds, t=0):
  return ds.isel(time=slice(t, t + 1))


def _model(task, precision="bf16x3"):
  cfg = graphcast.ModelConfig(30.0, 1, 512, 1, 1, 0.6)
  params = graphcast.init_params(cfg, task, synthetic.num_input_channels(task), seed=1)
  return graphcast.GraphCast(cfg, task, params=params, precision=precision), params


def test_param_tangents_are_checked_against_the_params():
  _, params = _model(graphcast.TASK_13)
  name = sorted(params)[0]
  field = sorted(params[name])[0]
  shape = np.shape(params[name][field])
  good = {name: {field: np.ones(shape, np.float64)}}
  got = graphcast.check_param_tangents(good, params)
  assert got[name][field].dtype == np.float32 and got[name][field].shape == shape
  assert graphcast.check_param_tangents({}, params) == {}
  for bad, why in (
      ([1, 2], "must be a mapping"),
      ({"no/such/module": {"w": np.zeros(3)}}, "unknown module 'no/such/module'"),
      ({name: np.zeros(shape)}, f"param_tangents[{name!r}] must be a mapping"),
      ({name: {"nope": np.zeros(shape)}}, f"unknown field {name}:nope"),
      ({name: {field: np.zeros(shape + (1,))}}, f"{name}:{field} has shape"),
      ({name: {field: "text"}}, "is not a float array"),
  ):
    with pytest.raises(ValueError, match=None) as e:
      graphcast.check_param_tangents(bad, params)
    assert why in str(e.value), (why, str(e.value))


def test_refusals_without_a_device():
  task = graphcast.TASK_13
  inputs, template, forcings = _example(task)
  model, params = _model(task)
  name = sorted(params)[0]
  v = {name: {f: np.zeros(np.shape(a), np.float32) for f, a in params[name].items()}}
  one = (inputs, _one(template), _one(forcings))

  class Other(graphcast.Predictor):
    def __call__(self, inputs, targets_template, forcings, **kwargs):
      raise AssertionError

  for call in ("param_jvp", "loss_and_param_gnvp"):
    with pytest.raises(NotImplementedError, match="does not implement parameter tangents"):
      getattr(Other(), call)(*one, v)
  stats = xs.Dataset()
  generic = normalization.InputsAndResiduals(casting.Bfloat16Cast(Other()), stats, stats, stats)
  fused = normalization.InputsAndResiduals(model, stats, stats, stats)
  stacks = [model, casting.Bfloat16Cast(Other()), fused, autoregressive.Predictor(model),
            autoregressive.Predictor(fused)]
  for call in ("param_jvp", "loss_and_param_gnvp"):
    for pred in (model, fused, autoregressive.Predictor(model), autoregressive.Predictor(fused)):
      fn = getattr(pred, call)
      with pytest.raises(ValueError, match="unknown module"):
        fn(*one, {"no/such/module": {}})
      with pytest.raises(ValueError, match="has shape"):
        fn(*one, {name: {f: np.zeros([1, 1, 1], np.float32) for f in params[name]}})
      with pytest.raises(ValueError, match="must be a mapping"):
        fn(*one, [v])
    # the generic (non-fused) normalisation: loss_and_grads' message, directly and over time
    with pytest.raises(NotImplementedError, match="fused normalisation"):
      getattr(generic, call)(*one, v)
  assert stacks and model._engine is None
  # several target times: GraphCast covers one, the Gauss-Newton product one everywhere
  with pytest.raises(NotImplementedError, match="one target time"):
    model.param_jvp(inputs, template, forcings, v)
  for pred in (model, fused, autoregressive.Predictor(model)):
    with pytest.raises(NotImplementedError, match="Gauss-Newton products cover one target time"):
      pred.loss_and_param_gnvp(inputs, template, forcings, v)
  with pytest.raises(ValueError, match="unknown module"):
    autoregressive.Predictor(model).param_jvp(inputs, template, forcings, {"x": {}})
  with pytest.raises(NotImplementedError, match="param_jvp over several target times needs a GraphCast"):
    autoregressive.Predictor(Other()).param_jvp(inputs, template, forcings, v)
  with pytest.raises(NotImplementedError, match="fused normalisation"):
    autoregressive.Predictor(generic).param_jvp(inputs, template, forcings, v)
  assert model._engine is None
  # the fp32_simt precision
  simt, _ = _model(task, precision="fp32_simt")
  for call in ("param_jvp", "loss_and_param_gnvp"):
    with pytest.raises(NotImplementedError, match="tensor-core precisions"):
      getattr(simt, call)(*one, v)
  with pytest.raises(NotImplementedError, match="tensor-core precisions"):
    autoregressive.Predictor(simt).param_jvp(inputs, template, forcings, v)
  assert simt._engine is None
  # a model without parameters
  bare = graphcast.GraphCast(graphcast.ModelConfig(30.0, 1, 512, 1, 1, 0.6), task)
  with pytest.raises(ValueError, match="no parameters"):
    bare.param_jvp(*one, v)


def test_native_refusals_without_a_device():
  """The two new entry points refuse bad arguments with status -1 and a message; dummy pointers and
  zero rows, so no accepted call here launches anything (the seed kernel launches whenever its checks
  pass, so only its refusals are called)."""
  lib = _native.lib()
  P = 256

  def ln(z=P, ld_z=512, dz=P, ld_dz=512, scale=P, rows=0, n=512, res=None, ld_res=512, ds=None, do=None,
         out=P, ld_out=512):
    return lib.gcb_layernorm_jvp_params(z, ld_z, dz, ld_dz, scale, rows, n, res, ld_res, ds, do, out,
                                        ld_out, None)

  def seed(dy=P, ld_dy=256, n_out=83, n_lat=2, n_lon=4, lat=P, coef=P, g=P, ld_g=256):
    return lib.gcb_output_loss_gn_seed(dy, ld_dy, n_out, n_lat, n_lon, lat, coef, g, ld_g, None)

  def refused(fn, why, **kw):
    assert fn(**kw) == -1, (why, kw)
    assert why in lib.gcb_last_error(), (lib.gcb_last_error(), kw)

  for k in ("z", "dz", "scale", "out"):
    refused(ln, b"null pointer", **{k: None})
  refused(ln, b"needs n = 512", n=256)
  refused(ln, b"rows < 0 or leading dimension < n", rows=-1)
  for k in ("ld_z", "ld_dz", "ld_out"):
    refused(ln, b"rows < 0 or leading dimension < n", **{k: 508})
  refused(ln, b"rows < 0 or leading dimension < n", res=P, ld_res=508)
  for kw in ({}, dict(res=P, ds=P, do=P, ld_z=516), dict(ds=P), dict(do=P)):
    assert ln(**kw) == 0, (lib.gcb_last_error(), kw)
  for k in ("dy", "lat", "coef", "g"):
    refused(seed, b"null pointer", **{k: None})
  refused(seed, b"ld_dy / ld_g too small", n_out=0)
  refused(seed, b"ld_dy / ld_g too small", ld_dy=82)
  refused(seed, b"ld_dy / ld_g too small", ld_g=82)
  refused(seed, b"empty grid", n_lat=0)
  refused(seed, b"empty grid", n_lon=0)
