"""The host side of Hessian-vector products along several tangent directions
(batched_loss_and_input_hvp): the stacked tangent planes against separate packings of each direction,
and every refusal that needs no device, with its message, on every stack, before an engine exists.
CPU only."""
import numpy as np
import pytest

from graphcast_b200 import autoregressive, casting, feedback, graphcast, normalization, synthetic
from graphcast_b200 import xarray_shim as xs


def _example(task, steps=2, seed=3):
  return synthetic.make_example(task, 30.0, batch=2, num_target_steps=steps, seed=seed)


def _one(ds):
  return ds.isel(time=slice(0, 1))


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


class _Other(graphcast.Predictor):
  def __call__(self, inputs, targets_template, forcings, **kwargs):
    raise AssertionError


@pytest.mark.parametrize("task", [graphcast.TASK_13, graphcast.TASK])
def test_stacked_tangent_planes_are_single_packings(task):
  inputs, _, forcings = _example(task)
  f = _one(forcings)
  rng = np.random.default_rng(5)
  for k in (1, 2, 5):
    for d_in, d_f in ((_directions(inputs, rng, k), _directions(f, rng, k)),
                      (_directions(inputs, rng, k, names=sorted(inputs.keys())[::2]), None),
                      (None, _directions(f, rng, k, names=sorted(f.keys())[:1]))):
      got = graphcast.hvp_direction_tangent_planes(inputs, f, d_in, d_f).numpy()
      assert got.dtype == np.float32 and got.shape[0] == k
      for j in range(k):
        want = graphcast.hvp_tangent_planes(
            inputs, f, None if d_in is None else d_in.isel(direction=j),
            None if d_f is None else d_f.isel(direction=j)).numpy()
        assert np.array_equal(got[j], want)


def test_refusals_without_a_device():
  task = graphcast.TASK_13
  inputs, template, forcings = _example(task)
  cfg = graphcast.ModelConfig(30.0, 1, 512, 1, 1, 0.6)
  model = graphcast.GraphCast(cfg, task)
  rng = np.random.default_rng(6)
  d_in = _directions(inputs, rng, 2, names=["2m_temperature"])
  d_f = _directions(_one(forcings), rng, 2)
  one = (inputs, _one(template), _one(forcings))

  with pytest.raises(NotImplementedError, match="does not implement Hessian-vector products"):
    _Other().batched_loss_and_input_hvp(*one, d_in)
  v = d_in.data_vars["2m_temperature"]
  no_dir = xs.Dataset(coords=inputs.coords)
  no_dir["2m_temperature"] = xs.DataArray(np.asarray(v.values)[0], v.dims[1:])
  mixed = xs.Dataset(coords=inputs.coords)
  mixed["2m_temperature"] = v
  w = _directions(inputs, rng, 3, names=["geopotential"]).data_vars["geopotential"]
  mixed["geopotential"] = w
  bad = xs.Dataset(coords=inputs.coords)
  bad["not_a_variable"] = v
  short = xs.Dataset(coords=inputs.coords)
  short["2m_temperature"] = xs.DataArray(np.asarray(v.values)[:, :1], v.dims)
  stacks = [model, casting.Bfloat16Cast(model), autoregressive.Predictor(model),
            autoregressive.Predictor(model, gradient_checkpointing=True)]
  for pred in stacks:
    call = lambda *a, **kw: pred.batched_loss_and_input_hvp(*one, *a, **kw)
    with pytest.raises(ValueError, match="needs the leading dim 'direction'"):
      call(no_dir)
    with pytest.raises(ValueError, match="has 3 directions, other variables 2"):
      call(mixed)
    with pytest.raises(ValueError, match="input_tangents have 2 directions, forcing_tangents 3"):
      call(d_in, _directions(_one(forcings), rng, 3))
    with pytest.raises(ValueError, match="the tangents have no variables"):
      call(None, None)
    with pytest.raises(ValueError, match="unknown variable 'not_a_variable'"):
      call(bad)
    with pytest.raises(ValueError, match="2m_temperature has dims"):
      call(short)
    for per in (0, -1, 1.5, True, "2"):
      with pytest.raises(ValueError, match="directions_per_pass must be None or an int >= 1"):
        call(d_in, d_f, directions_per_pass=per)
  # GraphCast and Bfloat16Cast cover one target time, as loss_and_input_hvp does
  for pred in stacks[:2]:
    with pytest.raises(NotImplementedError, match="one target time"):
      pred.batched_loss_and_input_hvp(inputs, template, forcings, d_in)
  # several target times: the refusals of loss_and_input_hvp, then the tangent checks
  with pytest.raises(NotImplementedError, match="gradient_checkpointing=True"):
    stacks[2].batched_loss_and_input_hvp(inputs, template, forcings, d_in)
  with pytest.raises(NotImplementedError, match="GraphCast predictor"):
    autoregressive.Predictor(_Other(), gradient_checkpointing=True).batched_loss_and_input_hvp(
        inputs, template, forcings, d_in)
  with pytest.raises(ValueError, match="needs the leading dim 'direction'"):
    stacks[3].batched_loss_and_input_hvp(inputs, template, forcings, no_dir)
  with pytest.raises(ValueError, match="input_tangents have 2 directions, forcing_tangents 3"):
    stacks[3].batched_loss_and_input_hvp(inputs, template, forcings, d_in,
                                         _directions(forcings, rng, 3))
  with pytest.raises(ValueError, match="directions_per_pass must be None or an int >= 1"):
    stacks[3].batched_loss_and_input_hvp(inputs, template, forcings, d_in,
                                         _directions(forcings, rng, 2), directions_per_pass=0)
  with pytest.raises(ValueError, match="forcing_tangents"):
    stacks[3].batched_loss_and_input_hvp(inputs, template, forcings, d_in, d_f)
  assert model._engine is None
  # the fused normalisation checks the tangents the same way; the generic one refuses as
  # loss_and_input_grads does
  stats = xs.Dataset()
  generic = normalization.InputsAndResiduals(casting.Bfloat16Cast(_Other()), stats, stats, stats)
  with pytest.raises(NotImplementedError) as want:
    generic.loss_and_input_grads(*one)
  with pytest.raises(NotImplementedError) as got:
    generic.batched_loss_and_input_hvp(*one, d_in)
  assert str(got.value) == str(want.value)
  with pytest.raises(ValueError, match="needs the leading dim 'direction'"):
    generic.batched_loss_and_input_hvp(*one, no_dir)
  with pytest.raises(ValueError, match="directions_per_pass must be None or an int >= 1"):
    generic.batched_loss_and_input_hvp(*one, d_in, directions_per_pass=0)
  fused = normalization.InputsAndResiduals(model, stats, stats, stats)
  with pytest.raises(ValueError, match="has 3 directions, other variables 2"):
    fused.batched_loss_and_input_hvp(*one, mixed)
  with pytest.raises(ValueError, match="directions_per_pass must be None or an int >= 1"):
    fused.batched_loss_and_input_hvp(*one, d_in, directions_per_pass=2.0)
  assert model._engine is None


def test_direction_labels_and_pass_slices():
  """The labels come from input_tangents' direction coordinate, else 0..K-1; the passes are
  consecutive slices of directions_per_pass directions."""
  inputs, _, forcings = _example(graphcast.TASK_13)
  rng = np.random.default_rng(8)
  d = _directions(inputs, rng, 3, names=["2m_temperature"], labels=[7, 3, 5])
  assert feedback.check_direction_tangents(d, inputs, None, _one(forcings))[1].tolist() == [7, 3, 5]
  d = _directions(inputs, rng, 3, names=["2m_temperature"])
  assert feedback.check_direction_tangents(d, inputs, None, _one(forcings))[1].tolist() == [0, 1, 2]
  assert feedback.direction_slices(5, 2) == [slice(0, 2), slice(2, 4), slice(4, 5)]
  assert feedback.direction_slices(5, None) == [slice(0, 5)]
  assert feedback.direction_slices(2, 7) == [slice(0, 2)]
