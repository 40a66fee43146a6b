"""The tangent-linear forecast of several directions on the device (batched_input_jvp): the two direction
kernels against their one-direction counterparts (bit for bit) and fp64 torch, every direction of a
batched call against input_jvp along it alone (bit for bit) on every stack, precision and number of
target times, the independence of directions_per_pass, no interference with the other calls, and at
0.25 degree the bit equality and the memory of two directions."""
import gc

import numpy as np
import pytest
import torch

from graphcast_b200 import _native, graphcast
from graphcast_b200 import xarray_shim as xs
from test_gpu_grads import _frob
from test_gpu_input_grads import _full_problem, _random_cotangents, _stack

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _st():
  return torch.cuda.current_stream().cuda_stream


# ---- kernels -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [1, 7, 1003])
@pytest.mark.parametrize("dirs", [1, 3, 8])
def test_direction_kernels_equal_the_one_direction_kernels(rows, dirs):
  lib = _native.lib()
  gen = torch.Generator(device=DEV).manual_seed(rows * 10 + dirs)
  n = 512
  stride = (rows + 127) // 128 * 128 + 128 * (dirs % 2)   # any stride >= rows
  total = (dirs - 1) * stride + rows
  h = torch.randn(rows, n, generator=gen, device=DEV) * 3
  z = torch.randn(rows, n, generator=gen, device=DEV) * 2 + 0.5
  scale = torch.rand(n, generator=gen, device=DEV) + 0.5
  d = torch.randn(total, n, generator=gen, device=DEV)
  res = torch.randn(total, n, generator=gen, device=DEV)
  ws = torch.empty(lib.gcb_rowwise_workspace_bytes(n), dtype=torch.uint8, device=DEV)
  sink = torch.empty(n, device=DEV)

  da = torch.full((total, n), float("nan"), device=DEV)
  _native.check(lib.gcb_swish_jvp(h.data_ptr(), n, rows, n, d.data_ptr(), n, stride, dirs, da.data_ptr(),
                                  n, _st()), "gcb_swish_jvp")
  inplace = d.clone()
  _native.check(lib.gcb_swish_jvp(h.data_ptr(), n, rows, n, inplace.data_ptr(), n, stride, dirs,
                                  inplace.data_ptr(), n, _st()), "gcb_swish_jvp in place")
  outs = {}
  for residual in (None, res):
    out = torch.full((total, n), float("nan"), device=DEV)
    _native.check(lib.gcb_layernorm_jvp_dirs(
        z.data_ptr(), n, d.data_ptr(), n, scale.data_ptr(), rows, n, stride, dirs,
        None if residual is None else residual.data_ptr(), n, out.data_ptr(), n, _st()),
        "gcb_layernorm_jvp_dirs")
    outs[residual is None] = out
  hd, zd, sd = h.double(), z.double(), scale.double()
  sg = torch.sigmoid(hd)
  ln = lambda x: (x - x.mean(-1, keepdim=True)) * torch.rsqrt(x.var(-1, unbiased=False, keepdim=True)
                                                              + 1e-5) * sd
  for k in range(dirs):
    r = slice(k * stride, k * stride + rows)
    one = torch.empty(rows, n, device=DEV)
    _native.check(lib.gcb_swish_backward(d[r].data_ptr(), n, h.data_ptr(), n, rows, n, one.data_ptr(), n,
                                         ws.data_ptr(), ws.numel(), sink.data_ptr(), 0, _st()), "swish")
    assert torch.equal(da[r], one), k
    assert torch.equal(inplace[r], one), k
    assert _frob(da[r], sg * (1 + hd * (1 - sg)) * d[r].double()) <= 1e-6
    _, want = torch.func.jvp(ln, (zd,), (d[r].double(),))
    for no_res, residual in ((True, None), (False, res[r])):
      one = torch.empty(rows, n, device=DEV)
      _native.check(lib.gcb_layernorm_jvp(
          z.data_ptr(), n, d[r].data_ptr(), n, scale.data_ptr(), rows, n,
          None if residual is None else residual.data_ptr(), n, one.data_ptr(), n, _st()), "ln")
      assert torch.equal(outs[no_res][r], one), (k, no_res)
      ref = want if residual is None else want + residual.double()
      assert _frob(outs[no_res][r], ref) <= 1e-6
  print(f"rows {rows}, {dirs} directions: bit-equal to gcb_swish_backward and gcb_layernorm_jvp")


# ---- batched_input_jvp against input_jvp -----------------------------------------------------------------
def _values(ds):
  return {k: np.asarray(v.values) for k, v in ds.data_vars.items()}


def _directions(ds, rng, dirs, names=None, zero=(), only=None):
  """Tangents of `ds`'s variables (or of `names`) along `dirs` directions: random, except the
  directions in `zero` (all zero) and, for direction k in `only`, every variable but only[k] zero."""
  out = xs.Dataset(coords=ds.coords)
  for name, v in ds.data_vars.items():
    if names is not None and name not in names:
      continue
    a = rng.standard_normal((dirs,) + tuple(v.shape)).astype(np.float32)
    for k in zero:
      a[k] = 0
    for k, keep in (only or {}).items():
      if name != keep:
        a[k] = 0
    out[name] = xs.DataArray(a, ("direction",) + tuple(v.dims))
  return out


def _at(ds, k):
  return None if ds is None else ds.isel(direction=k)


def _check_directions(pred, inputs, targets, forcings, d_in, d_f, dirs, zero=(), **kw):
  call = _values(pred(inputs, targets, forcings))
  predictions, tangents = pred.batched_input_jvp(inputs, targets, forcings, d_in, d_f, **kw)
  assert all(np.array_equal(a, call[k]) for k, a in _values(predictions).items())
  assert np.array_equal(np.asarray(tangents.coords["direction"][1]), np.arange(dirs))
  for name, v in tangents.data_vars.items():
    p = predictions.data_vars[name]
    assert v.dims == ("direction",) + p.dims and tuple(v.shape) == (dirs,) + tuple(p.shape)
    assert np.asarray(v.values).dtype == np.float32
  got = _values(tangents)
  for k in range(dirs):
    _, one = pred.input_jvp(inputs, targets, forcings, _at(d_in, k), _at(d_f, k))
    for name, a in _values(one).items():
      assert np.array_equal(got[name][k], a), (k, name)
      if k in zero:
        assert not np.any(got[name][k]), (k, name)
  return got


@pytest.mark.parametrize("task_name,stack,steps,dirs,which", [
    ("TASK_13", "plain", 1, 2, "all"),
    ("TASK_13", "normalized", 1, 5, "some"),
    ("TASK_13", "demo", 1, 2, "all"),                   # bf16
    ("TASK_13_PRECIP_OUT", "plain", 3, 2, "some"),
    ("TASK_13", "normalized", 3, 5, "all"),
    ("TASK_13", "demo", 3, 5, "some"),
    ("TASK", "normalized", 1, 2, "some"),               # 37 levels
    ("TASK", "plain", 3, 5, "all"),
    ("TASK", "normalized", 3, 1, "all"),
    ("TASK_13", "normalized", 1, 1, "some"),
])
def test_each_direction_is_input_jvp_along_it(task_name, stack, steps, dirs, which):
  _, pred, inputs, targets, forcings, _ = _stack(task_name, stack, steps)
  rng = np.random.default_rng(21)
  zero = (dirs - 1,) if dirs > 1 else ()
  if which == "all":
    d_in = _directions(inputs, rng, dirs, zero=zero)
    d_f = _directions(forcings, rng, dirs, zero=zero)
  else:                   # a subset of the inputs, directions that touch one variable, forcings fixed
    only = {0: "temperature", 1: "2m_temperature"} if dirs > 2 else {0: "temperature"}
    d_in = _directions(inputs, rng, dirs, names=["temperature", "2m_temperature", "specific_humidity"],
                       zero=zero, only=only)
    d_f = None
  _check_directions(pred, inputs, targets, forcings, d_in, d_f, dirs, zero)
  print(f"{task_name} {stack} T={steps}, {dirs} directions ({which}): bit-equal to input_jvp")


def test_directions_per_pass_does_not_change_the_result():
  _, pred, inputs, targets, forcings, _ = _stack("TASK_13", "normalized", 3)
  rng = np.random.default_rng(22)
  d_in, d_f = _directions(inputs, rng, 5), _directions(forcings, rng, 5)
  d_in.coords["direction"] = (("direction",), np.array([3, 1, 4, 1, 5]))
  results = {}
  for per in (None, 1, 2, 5, 7):
    predictions, tangents = pred.batched_input_jvp(inputs, targets, forcings, d_in, d_f,
                                                   directions_per_pass=per)
    assert list(np.asarray(tangents.coords["direction"][1])) == [3, 1, 4, 1, 5]
    results[per] = (_values(predictions), _values(tangents))
  for per, (p, t) in results.items():
    for name in t:
      assert np.array_equal(t[name], results[None][1][name]), (per, name)
      assert np.array_equal(p[name], results[None][0][name]), (per, name)


def test_no_interference_with_the_other_calls():
  model, pred, inputs, targets, forcings, _ = _stack("TASK_13", "normalized", 1)
  rng = np.random.default_rng(23)
  v_in, v_f = _directions(inputs, rng, 1), _directions(forcings, rng, 1)
  d_in, d_f = _directions(inputs, rng, 4), _directions(forcings, rng, 4)
  w = _random_cotangents(targets)
  before = (pred.loss_and_grads(inputs, targets, forcings)[2],
            pred.input_vjp(inputs, targets, forcings, w),
            pred.input_jvp(inputs, targets, forcings, _at(v_in, 0), _at(v_f, 0)))
  pred.batched_input_jvp(inputs, targets, forcings, d_in, d_f, directions_per_pass=3)
  after = (pred.input_jvp(inputs, targets, forcings, _at(v_in, 0), _at(v_f, 0)),
           pred.input_vjp(inputs, targets, forcings, w),
           pred.loss_and_grads(inputs, targets, forcings)[2])
  g0, g1 = before[0], after[2]
  for k in g0:
    for f in g0[k]:
      assert np.array_equal(g0[k][f], g1[k][f]), (k, f)
  for a, b in zip(before[1] + before[2], after[1] + after[0]):
    for k in a.keys():
      assert np.array_equal(np.asarray(a.data_vars[k].values), np.asarray(b.data_vars[k].values)), k
  # the refusals of input_jvp
  model.set_precision("fp32_simt")
  with pytest.raises(NotImplementedError, match="tensor-core precisions"):
    pred.batched_input_jvp(inputs, targets, forcings, d_in)
  model.set_precision("bf16x3")


# ---- full size -------------------------------------------------------------------------------------------
def _peak(fn):
  gc.collect()
  torch.cuda.empty_cache()
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  out = fn()
  torch.cuda.synchronize()
  return torch.cuda.max_memory_allocated(), out


def test_full_size_two_directions():
  """0.25 degree / 37 levels, one target time: two directions at once equal two input_jvp calls bit
  for bit, and peak below 80 GiB."""
  if torch.cuda.get_device_properties(0).total_memory < 75e9:
    pytest.skip("needs an 80 GB GPU")
  model, ar, inputs, targets, forcings = _full_problem(graphcast.TASK, 0.25, 6, 1)
  ar(inputs, targets, forcings)                           # builds the engine
  rng = np.random.default_rng(24)
  d_in = _directions(inputs, rng, 2)
  d_f = _directions(forcings, rng, 2, names=["toa_incident_solar_radiation"])
  peak_one, (_, one) = _peak(lambda: ar.input_jvp(inputs, targets, forcings, _at(d_in, 0), _at(d_f, 0)))
  one = _values(one)
  peak_two, (_, two) = _peak(lambda: ar.batched_input_jvp(inputs, targets, forcings, d_in, d_f))
  two = _values(two)
  print(f"0.25 deg, T = 1: peak input_jvp {peak_one / 2**30:.2f} GiB, batched_input_jvp (K = 2) "
        f"{peak_two / 2**30:.2f} GiB on {torch.cuda.get_device_name(0)}")
  assert peak_two < 80 * 2**30
  for name, a in one.items():
    assert np.array_equal(two[name][0], a), name
  del one
  _, other = ar.input_jvp(inputs, targets, forcings, _at(d_in, 1), _at(d_f, 1))
  for name, a in _values(other).items():
    assert np.array_equal(two[name][1], a), name
