"""input_vjp of several cotangents on the device (batched_input_vjp): the LayerNorm backward of several
directions against gcb_layernorm_backward (bit for bit) and fp64 torch, every direction of a batched
call against input_vjp with its cotangent alone (bit for bit) on every stack, precision and number of
target times, with several bipartite chunks, the independence of directions_per_pass, no interference
with the other calls, the adjoint identity with batched_input_jvp, and at 0.25 degree the bit equality
and the memory of two directions run one per pass."""
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


# ---- kernel ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [1, 7, 1003])
@pytest.mark.parametrize("dirs", [1, 3, 8])
def test_layernorm_backward_dirs_equals_the_one_direction_kernel(rows, dirs):
  lib = _native.lib()
  gen = torch.Generator(device=DEV).manual_seed(rows * 10 + dirs)
  n = 512
  stride = (rows + 127) // 128 * 128 + 128 * (dirs % 2)   # any stride >= rows, here > rows
  total = (dirs - 1) * stride + rows
  z = torch.randn(rows, n, generator=gen, device=DEV) * 2 + 0.5
  scale = torch.rand(n, generator=gen, device=DEV) + 0.5
  dy = torch.randn(total, n, generator=gen, device=DEV)
  ws = torch.empty(lib.gcb_rowwise_workspace_bytes(n), dtype=torch.uint8, device=DEV)
  sums = [torch.empty(n, device=DEV) for _ in range(3)]
  dz = torch.full((total, n), float("nan"), device=DEV)
  _native.check(lib.gcb_layernorm_backward_dirs(
      dy.data_ptr(), n, z.data_ptr(), n, scale.data_ptr(), rows, n, stride, dirs, dz.data_ptr(), n,
      _st()), "gcb_layernorm_backward_dirs")
  zd, sd = z.double(), scale.double()
  ln = lambda x: (x - x.mean(-1, keepdim=True)) * torch.rsqrt(x.var(-1, unbiased=False, keepdim=True)
                                                              + 1e-5) * sd
  valid = torch.zeros(total, dtype=torch.bool, device=DEV)
  for k in range(dirs):
    r = slice(k * stride, k * stride + rows)
    valid[r] = True
    one = torch.empty(rows, n, device=DEV)
    _native.check(lib.gcb_layernorm_backward(
        dy[r].data_ptr(), n, z.data_ptr(), n, scale.data_ptr(), rows, n, one.data_ptr(), n,
        ws.data_ptr(), ws.numel(), sums[0].data_ptr(), sums[1].data_ptr(), sums[2].data_ptr(), 0,
        _st()), "gcb_layernorm_backward")
    assert torch.equal(dz[r], one), k
    _, vjp = torch.func.vjp(ln, zd)
    assert _frob(dz[r], vjp(dy[r].double())[0]) <= 1e-6
  assert torch.isnan(dz[~valid]).all()                    # the pad rows are never written
  print(f"rows {rows}, {dirs} directions: bit-equal to gcb_layernorm_backward")


# ---- batched_input_vjp against input_vjp -----------------------------------------------------------------
def _values(ds):
  return {k: np.asarray(v.values) for k, v in ds.data_vars.items()}


def _cotangents(targets, dirs, seed=9, zero=(), labels=None):
  """Random cotangents shaped like `targets` along `dirs` directions; the directions in `zero` are 0."""
  rng = np.random.default_rng(seed)
  out = xs.Dataset(coords=targets.coords)
  if labels is not None:
    out.coords["direction"] = (("direction",), np.asarray(labels))
  for name, v in targets.data_vars.items():
    a = rng.standard_normal((dirs,) + tuple(v.shape)).astype(np.float32)
    for k in zero:
      a[k] = 0
    out[name] = xs.DataArray(a, ("direction",) + tuple(v.dims))
  return out


def _check_directions(pred, inputs, targets, forcings, cot, dirs, zero=(), **kw):
  call = _values(pred(inputs, targets, forcings))
  predictions, ig, fg = pred.batched_input_vjp(inputs, targets, forcings, cot, **kw)
  assert all(np.array_equal(a, call[k]) for k, a in _values(predictions).items())
  for got, like in ((ig, inputs), (fg, forcings)):
    assert np.array_equal(np.asarray(got.coords["direction"][1]), np.arange(dirs))
    assert set(got.keys()) == set(like.keys())
    for name, v in got.data_vars.items():
      ref = like.data_vars[name]
      assert v.dims == ("direction",) + ref.dims and tuple(v.shape) == (dirs,) + tuple(ref.shape)
      assert np.asarray(v.values).dtype == np.float32
  got = (_values(ig), _values(fg))
  for k in range(dirs):
    _, one_i, one_f = pred.input_vjp(inputs, targets, forcings, cot.isel(direction=k))
    for g, one in zip(got, (one_i, one_f)):
      for name, a in _values(one).items():
        assert np.array_equal(g[name][k], a), (k, name)
        if k in zero:
          assert not np.any(g[name][k]), (k, name)
  return got


@pytest.mark.parametrize("task_name,stack,steps,dirs", [
    ("TASK_13", "plain", 1, 2),
    ("TASK_13", "normalized", 1, 5),
    ("TASK_13", "demo", 1, 2),                          # bf16
    ("TASK_13_PRECIP_OUT", "plain", 3, 2),
    ("TASK_13", "normalized", 3, 5),
    ("TASK_13", "demo", 3, 2),
    ("TASK", "normalized", 1, 2),                       # 37 levels
    ("TASK", "plain", 3, 5),
    ("TASK", "normalized", 3, 1),
    ("TASK_13", "normalized", 1, 1),
])
def test_each_direction_is_input_vjp_with_its_cotangent(task_name, stack, steps, dirs):
  _, pred, inputs, targets, forcings, _ = _stack(task_name, stack, steps)
  zero = (dirs - 1,) if dirs > 1 else ()
  _check_directions(pred, inputs, targets, forcings, _cotangents(targets, dirs, zero=zero), dirs, zero)
  print(f"{task_name} {stack} T={steps}, {dirs} directions: bit-equal to input_vjp")


@pytest.mark.parametrize("steps", [1, 3])
def test_several_bipartite_chunks(steps):
  """With chunks of 2000 (and 500) edges, every direction equals input_vjp at the same chunk_rows: the
  batched pass keeps the chunks of one direction, whose boundaries the sender sums depend on."""
  model, pred, inputs, targets, forcings, _ = _stack("TASK_13", "normalized", steps)
  pred(inputs, targets, forcings)                         # builds the engine
  for chunk_rows in (2000, 500):
    model.engine.grads_begin(chunk_rows=chunk_rows)
    assert len(model.engine._backward.chunks["m2g"]) > 1
    _check_directions(pred, inputs, targets, forcings, _cotangents(targets, 3, seed=chunk_rows), 3)


def test_directions_per_pass_does_not_change_the_result():
  _, pred, inputs, targets, forcings, _ = _stack("TASK_13", "normalized", 3)
  cot = _cotangents(targets, 5, seed=22, labels=[3, 1, 4, 1, 5])
  results = {}
  for per in (None, 1, 2, 5, 7):
    predictions, ig, fg = pred.batched_input_vjp(inputs, targets, forcings, cot, directions_per_pass=per)
    for g in (ig, fg):
      assert list(np.asarray(g.coords["direction"][1])) == [3, 1, 4, 1, 5]
    results[per] = (_values(predictions), _values(ig), _values(fg))
  for per, parts in results.items():
    for part, ref in zip(parts, results[None]):
      for name in ref:
        assert np.array_equal(part[name], ref[name]), (per, name)
  _, pred1, inputs1, targets1, forcings1, _ = _stack("TASK_13", "plain", 1)
  cot1 = _cotangents(targets1, 4, seed=23)
  ref = pred1.batched_input_vjp(inputs1, targets1, forcings1, cot1)
  for per in (1, 2, 3):
    got = pred1.batched_input_vjp(inputs1, targets1, forcings1, cot1, directions_per_pass=per)
    for a, b in zip(got, ref):
      for name, v in _values(b).items():
        assert np.array_equal(_values(a)[name], v), (per, name)


def _tangents(ds, rng, dirs):
  out = xs.Dataset(coords=ds.coords)
  for name, v in ds.data_vars.items():
    out[name] = xs.DataArray(rng.standard_normal((dirs,) + tuple(v.shape)).astype(np.float32),
                             ("direction",) + tuple(v.dims))
  return out


def _calls(pred, inputs, targets, forcings, d_in, d_f, cot, w):
  """batched_input_jvp, batched_input_vjp with the same K, input_vjp and loss_and_grads, in this order
  on one engine."""
  return [pred.batched_input_jvp(inputs, targets, forcings, d_in, d_f)[1],
          pred.batched_input_vjp(inputs, targets, forcings, cot)[1:],
          pred.input_vjp(inputs, targets, forcings, w)[1:],
          pred.loss_and_grads(inputs, targets, forcings)[2]]


@pytest.mark.parametrize("steps", [1, 2])
def test_no_interference_with_the_other_calls(steps):
  """On one engine with several bipartite chunks, batched_input_jvp of K directions (whose chunks are
  not the backward pass's) and then batched_input_vjp of K cotangents, input_vjp and loss_and_grads
  give what a fresh engine gives each of them, bit for bit."""
  dirs = 3
  runs = []
  for order in ("after", "fresh"):
    model, pred, inputs, targets, forcings, _ = _stack("TASK_13", "normalized", steps)
    pred(inputs, targets, forcings)
    model.engine.grads_begin(chunk_rows=500)
    rng = np.random.default_rng(31)
    d_in, d_f = _tangents(inputs, rng, dirs), _tangents(forcings, rng, dirs)
    cot, w = _cotangents(targets, dirs, seed=32), _random_cotangents(targets, seed=33)
    if order == "after":
      runs.append(_calls(pred, inputs, targets, forcings, d_in, d_f, cot, w))
    else:                                 # each call on an engine that has run nothing else
      out = [pred.batched_input_jvp(inputs, targets, forcings, d_in, d_f)[1]]
      for call in (lambda p: p.batched_input_vjp(inputs, targets, forcings, cot)[1:],
                   lambda p: p.input_vjp(inputs, targets, forcings, w)[1:],
                   lambda p: p.loss_and_grads(inputs, targets, forcings)[2]):
        m, p, *_ = _stack("TASK_13", "normalized", steps)
        p(inputs, targets, forcings)
        m.engine.grads_begin(chunk_rows=500)
        out.append(call(p))
      runs.append(out)
  after, fresh = runs
  assert np.all([np.array_equal(a, b) for a, b in zip(_values(after[0]).values(),
                                                       _values(fresh[0]).values())])
  for a, b in zip(after[1] + after[2], fresh[1] + fresh[2]):
    for name, v in _values(b).items():
      assert np.array_equal(_values(a)[name], v), name
  for k, fields in fresh[3].items():
    for f, v in fields.items():
      assert np.array_equal(after[3][k][f], v), (k, f)


def _dot(a, b):
  """<a, b> over every variable of the Datasets a and b (same variables; b transposed to a's dims)."""
  return sum(float((np.asarray(a.data_vars[k].values, np.float64) *
                    np.asarray(b.data_vars[k].transpose(*a.data_vars[k].dims).values, np.float64)).sum())
             for k in a.keys())


@pytest.mark.parametrize("steps", [1, 3])
def test_adjoint_identity_between_the_batched_calls(steps):
  """<c_k, J d_j> = <J^T c_k, d_j> for K = 3 cotangents and J = 4 tangents, with both sides formed by
  the batched calls."""
  _, pred, inputs, targets, forcings, _ = _stack("TASK_13", "normalized", steps)
  rng = np.random.default_rng(41)
  d_in, d_f = _tangents(inputs, rng, 4), _tangents(forcings, rng, 4)
  cot = _cotangents(targets, 3, seed=42)
  _, tangents = pred.batched_input_jvp(inputs, targets, forcings, d_in, d_f)
  _, ig, fg = pred.batched_input_vjp(inputs, targets, forcings, cot)
  lhs, rhs = np.empty((3, 4)), np.empty((3, 4))
  for k in range(3):
    for j in range(4):
      lhs[k, j] = _dot(cot.isel(direction=k), tangents.isel(direction=j))
      rhs[k, j] = (_dot(d_in.isel(direction=j), ig.isel(direction=k)) +
                   _dot(d_f.isel(direction=j), fg.isel(direction=k)))
  # relative to the matrix: an entry near zero (cancellation in a random inner product) is no gauge
  rel = np.linalg.norm(lhs - rhs) / max(np.linalg.norm(lhs), np.linalg.norm(rhs))
  worst = (np.abs(lhs - rhs) / np.maximum(np.abs(lhs), np.abs(rhs))).max()
  print(f"T={steps}: <c_k, J d_j> against <J^T c_k, d_j>, relative gap of the matrix {rel:.3g} "
        f"(worst entry {worst:.3g})")
  assert rel <= 1e-4


# ---- full size -------------------------------------------------------------------------------------------
def _peak(fn):
  gc.collect()
  torch.cuda.empty_cache()
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  out = fn()
  torch.cuda.synchronize()
  return torch.cuda.max_memory_allocated(), out


def test_full_size_two_directions_one_per_pass():
  """0.25 degree / 37 levels, one target time: two cotangents, one per pass, equal two input_vjp calls
  bit for bit, and peak no higher than input_vjp."""
  if torch.cuda.get_device_properties(0).total_memory < 75e9:
    pytest.skip("needs an 80 GB GPU")
  model, ar, inputs, targets, forcings = _full_problem(graphcast.TASK, 0.25, 6, 1)
  ar(inputs, targets, forcings)                           # builds the engine
  cot = _cotangents(targets, 2, seed=51)
  # nothing of one call (its predictions are device tensors) is alive while the other is measured
  peak_one, out = _peak(lambda: ar.input_vjp(inputs, targets, forcings, cot.isel(direction=0)))
  one = (_values(out[1]), _values(out[2]))
  del out
  peak_two, out = _peak(lambda: ar.batched_input_vjp(inputs, targets, forcings, cot,
                                                      directions_per_pass=1))
  two = (_values(out[1]), _values(out[2]))
  del out
  print(f"0.25 deg, T = 1: peak input_vjp {peak_one / 2**30:.2f} GiB, batched_input_vjp (K = 2, one "
        f"per pass) {peak_two / 2**30:.2f} GiB on {torch.cuda.get_device_name(0)}")
  # Within the caching allocator's granularity: a cached block up to 1 MiB larger than a request is
  # handed out whole, and the second pass meets the cache the first one left.
  assert peak_two <= peak_one + 2**21
  for g, o in zip(two, one):
    for name, a in o.items():
      assert np.array_equal(g[name][0], a), name
  del one
  _, ig, fg = ar.input_vjp(inputs, targets, forcings, cot.isel(direction=1))
  for g, o in zip(two, (_values(ig), _values(fg))):
    for name, a in o.items():
      assert np.array_equal(g[name][1], a), name
