"""The host side of loss_and_param_gnvp over several target times: every refusal on every predictor
stack before an engine exists, and the GPU-free refusals of the new C entry point
gcb_output_loss_gn_seed_feedback.  CPU only."""
import numpy as np
import pytest

from graphcast_b200 import _native, autoregressive, casting, graphcast, normalization, synthetic
from graphcast_b200 import xarray_shim as xs


def _example(task, steps=2, seed=3, resolution=30.0):
  return synthetic.make_example(task, resolution, batch=2, num_target_steps=steps, seed=seed)


def _model(task, precision="bf16x3"):
  cfg = graphcast.ModelConfig(30.0, 1, 512, 1, 1, 0.6)
  params = graphcast.init_params(cfg, task, synthetic.num_input_channels(task), seed=1)
  return graphcast.GraphCast(cfg, task, params=params, precision=precision), params


class _Other(graphcast.Predictor):
  def __call__(self, inputs, targets_template, forcings, **kwargs):
    raise AssertionError


def test_refusals_without_a_device():
  task = graphcast.TASK_13
  inputs, targets, forcings = _example(task)
  model, params = _model(task)
  name = sorted(params)[0]
  v = {name: {f: np.zeros(np.shape(a), np.float32) for f, a in params[name].items()}}
  stats = xs.Dataset()
  fused = normalization.InputsAndResiduals(model, stats, stats, stats)
  demo = normalization.InputsAndResiduals(casting.Bfloat16Cast(model), stats, stats, stats)
  generic = normalization.InputsAndResiduals(casting.Bfloat16Cast(_Other()), stats, stats, stats)
  ck = lambda p, **kw: autoregressive.Predictor(p, gradient_checkpointing=True, **kw)
  # without gradient checkpointing: the one-target-time message, pointing at the option
  for inner in (model, fused, demo, _Other(), generic):
    with pytest.raises(NotImplementedError,
                       match="Gauss-Newton products cover one target time") as e:
      autoregressive.Predictor(inner).loss_and_param_gnvp(inputs, targets, forcings, v)
    assert "gradient_checkpointing=True" in str(e.value)
  # stacks backprop through time does not accept
  for inner in (_Other(), casting.Bfloat16Cast(_Other())):
    with pytest.raises(NotImplementedError, match="backprop through time needs a GraphCast"):
      ck(inner).loss_and_param_gnvp(inputs, targets, forcings, v)
  with pytest.raises(NotImplementedError, match="fused normalisation"):
    ck(generic).loss_and_param_gnvp(inputs, targets, forcings, v)
  # bad tangents, on the plain, fused and demo stacks
  for inner in (model, fused, demo):
    fn = ck(inner).loss_and_param_gnvp
    with pytest.raises(ValueError, match="unknown module"):
      fn(inputs, targets, forcings, {"no/such/module": {}})
    with pytest.raises(ValueError, match=f"unknown field {name}:nope"):
      fn(inputs, targets, forcings, {name: {"nope": np.zeros(3)}})
    with pytest.raises(ValueError, match="has shape"):
      fn(inputs, targets, forcings, {name: {f: np.zeros([1, 1, 1], np.float32) for f in params[name]}})
    with pytest.raises(ValueError, match="must be a mapping"):
      fn(inputs, targets, forcings, [v])
  # noise without an rng
  for inner in (model, fused):
    with pytest.raises(ValueError, match="input noise needs an rng"):
      ck(inner, noise_level=0.05).loss_and_param_gnvp(inputs, targets, forcings, v)
  # GraphCast and the fused normalisation called directly keep their one-target-time refusal
  for pred in (model, fused):
    with pytest.raises(NotImplementedError, match="Gauss-Newton products cover one target time"):
      pred.loss_and_param_gnvp(inputs, targets, forcings, v)
  assert model._engine is None
  # the fp32_simt precision, directly and under the fused normalisation
  simt, _ = _model(task, precision="fp32_simt")
  for inner in (simt, normalization.InputsAndResiduals(simt, stats, stats, stats)):
    with pytest.raises(NotImplementedError, match="tensor-core precisions"):
      ck(inner).loss_and_param_gnvp(inputs, targets, forcings, v)
  assert simt._engine is None
  # a grid that is not a multiple of 4 nodes: the tangent feed gathers 16-byte rows
  odd_in, odd_tgt, odd_f = (ds.isel(lon=slice(0, 11)) for ds in (inputs, targets, forcings))
  assert (odd_in.sizes["lat"] * odd_in.sizes["lon"]) % 4
  for inner in (model, fused):
    with pytest.raises(NotImplementedError, match="multiple of 4 grid nodes"):
      ck(inner).loss_and_param_gnvp(odd_in, odd_tgt, odd_f, v)
  assert model._engine is None


def test_native_refusals_without_a_device():
  """gcb_output_loss_gn_seed_feedback refuses bad arguments with status -1 and a message; dummy
  pointers, and only refusals are called (an accepted call launches)."""
  lib = _native.lib()
  P = 256

  def call(pdot=P, n_out=83, n_lat=2, n_lon=4, scale=None, lat=P, coef=P, a_next=None, dpred=None,
           n_rows=0, resid=None, carry=None, a_out=None, g=P, ld_g=256):
    return lib.gcb_output_loss_gn_seed_feedback(pdot, n_out, n_lat, n_lon, scale, lat, coef, a_next,
                                                dpred, n_rows, resid, carry, a_out, g, ld_g, None)

  def refused(why, **kw):
    assert call(**kw) == -1, (why, kw)
    assert why in lib.gcb_last_error(), (lib.gcb_last_error(), kw)

  for k in ("pdot", "lat", "coef", "g"):
    refused(b"null pointer", **{k: None})
  refused(b"ld_g too small", n_out=0)
  refused(b"ld_g too small", n_out=-3)
  refused(b"ld_g too small", ld_g=82)
  refused(b"empty grid", n_lat=0)
  refused(b"empty grid", n_lon=0)
  refused(b"a_next needs dpred_row", a_next=P)
  refused(b"rows need a_out and resid_channel", n_rows=-1)
  refused(b"rows need a_out and resid_channel", n_rows=3, resid=P)
  refused(b"rows need a_out and resid_channel", n_rows=3, a_out=P)
  refused(b"too many channels / rows", n_rows=65535 * 32, resid=P, a_out=P)
