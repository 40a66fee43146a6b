"""The host side of loss_and_param_hvp: every refusal on the four predictor stacks before an engine
exists, the node-partitioned refusal of the gradient workspace, and the GPU-free refusals of the new C
entry point gcb_layernorm_backward_jvp_params.  CPU only."""
import types

import numpy as np
import pytest

from graphcast_b200 import _native, autoregressive, casting, engine, graphcast, normalization, synthetic
from graphcast_b200 import xarray_shim as xs


def _example(task, steps=2, seed=3):
  return synthetic.make_example(task, 30.0, batch=2, num_target_steps=steps, seed=seed)


def _one(ds, t=0):
  return ds.isel(time=slice(t, t + 1))


def _model(task, precision="bf16x3"):
  cfg = graphcast.ModelConfig(30.0, 1, 512, 1, 1, 0.6)
  params = graphcast.init_params(cfg, task, synthetic.num_input_channels(task), seed=1)
  return graphcast.GraphCast(cfg, task, params=params, precision=precision), params


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

  with pytest.raises(NotImplementedError, match="does not implement parameter tangents"):
    Other().loss_and_param_hvp(*one, v)
  stats = xs.Dataset()
  generic = normalization.InputsAndResiduals(casting.Bfloat16Cast(Other()), stats, stats, stats)
  fused = normalization.InputsAndResiduals(model, stats, stats, stats)
  with pytest.raises(NotImplementedError, match="does not implement parameter tangents"):
    casting.Bfloat16Cast(Other()).loss_and_param_hvp(*one, v)
  for pred in (model, casting.Bfloat16Cast(model), fused, autoregressive.Predictor(model),
               autoregressive.Predictor(fused)):
    fn = pred.loss_and_param_hvp
    with pytest.raises(ValueError, match="unknown module"):
      fn(*one, {"no/such/module": {}})
    with pytest.raises(ValueError, match=f"unknown field {name}:nope"):
      fn(*one, {name: {"nope": np.zeros(3)}})
    with pytest.raises(ValueError, match="has shape"):
      fn(*one, {name: {f: np.zeros([1, 1, 1], np.float32) for f in params[name]}})
    with pytest.raises(ValueError, match="must be a mapping"):
      fn(*one, [v])
  # the generic (non-fused) normalisation: loss_and_grads' message, directly and over time
  for pred in (generic, autoregressive.Predictor(generic)):
    with pytest.raises(NotImplementedError, match="fused normalisation"):
      pred.loss_and_param_hvp(*one, v)
  # several target times, with or without gradient checkpointing
  for pred in (model, casting.Bfloat16Cast(model), fused, autoregressive.Predictor(model),
               autoregressive.Predictor(model, gradient_checkpointing=True),
               autoregressive.Predictor(fused, gradient_checkpointing=True)):
    with pytest.raises(NotImplementedError,
                       match="parameter Hessian-vector products cover one target time"):
      pred.loss_and_param_hvp(inputs, template, forcings, v)
  assert model._engine is None
  # the fp32_simt precision
  simt, _ = _model(task, precision="fp32_simt")
  for pred in (simt, autoregressive.Predictor(simt)):
    with pytest.raises(NotImplementedError, match="tensor-core precisions"):
      pred.loss_and_param_hvp(*one, v)
  assert simt._engine is None
  # a model without parameters
  bare = graphcast.GraphCast(graphcast.ModelConfig(30.0, 1, 512, 1, 1, 0.6), task)
  with pytest.raises(ValueError, match="no parameters"):
    bare.loss_and_param_hvp(*one, v)


def test_node_partitioned_engine_is_refused():
  """param_hvp_begin builds the gradient workspace through Engine._grad_workspace, which refuses the
  node-partitioned engine (num_grid_owned set) before building anything."""
  stub = types.SimpleNamespace(num_grid_owned=7, precision="bf16x3", _backward=None,
                               release_static_cache=lambda: None)
  with pytest.raises(NotImplementedError, match="not available in the node-partitioned engine"):
    engine.Engine._grad_workspace(stub, None, "parameter gradients")
  stub._grad_workspace = lambda *a: engine.Engine._grad_workspace(stub, *a)
  stub.grads_begin = lambda: engine.Engine.grads_begin(stub)
  with pytest.raises(NotImplementedError, match="not available in the node-partitioned engine"):
    engine.Engine.param_hvp_begin(stub)


def test_native_refusals_without_a_device():
  """gcb_layernorm_backward_jvp_params refuses bad arguments with status -1 and a message; dummy
  pointers, and only refusals are called (an accepted call launches, even with zero rows, since the
  column sums are written)."""
  lib = _native.lib()
  P = 256
  ws_bytes = lib.gcb_rowwise_workspace_bytes(512)

  def call(dy=P, ld_dy=512, stride=0, z=P, ld_z=512, zd=P, ld_zd=512, scale=P, sd=None, rows=0, n=512,
           dz=P, ld_dz=512, ws=P, ws_bytes=ws_bytes, sums=(P,) * 6, acc=1):
    return lib.gcb_layernorm_backward_jvp_params(dy, ld_dy, stride, z, ld_z, zd, ld_zd, scale, sd, rows,
                                                 n, dz, ld_dz, ws, ws_bytes, *sums, acc, None)

  def refused(why, **kw):
    assert call(**kw) == -1, (why, kw)
    assert why in lib.gcb_last_error(), (lib.gcb_last_error(), kw)

  for k in ("dy", "z", "zd", "scale", "dz", "ws"):
    refused(b"null pointer", **{k: None})
  for i in range(6):
    sums = [P] * 6
    sums[i] = None
    refused(b"null column-sum output", sums=tuple(sums))
  refused(b"needs n = 512", n=256)
  refused(b"rows < 0", rows=-1)
  for k in ("ld_dy", "ld_z", "ld_zd", "ld_dz"):
    refused(b"leading dimension < n", **{k: 508})
  refused(b"dir_stride < rows", rows=10, stride=9)
  refused(b"workspace too small", ws_bytes=ws_bytes - 4)
  # the refusal comes before anything is launched, with scale_dot given as well
  refused(b"dir_stride < rows", rows=10, stride=9, sd=P)
