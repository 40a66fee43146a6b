"""Hessian-vector products along several tangent directions on the device (batched_loss_and_input_hvp):
the two coupled backward kernels for K = 1, 2 and 5 tangents against the one-direction and one-tangent
kernels; every direction of the whole call bit for bit loss_and_input_hvp along it alone (T = 1 and 3,
plain, fused-normalised and bf16 stacks, 13 and 37 levels, with and without forcing tangents, several
directions_per_pass), with the loss, diagnostics and gradients bit for bit loss_and_input_grads in every
pass; noise at T = 2; labels, exact scaling, zero directions and symmetry; and K = 2 at 1 degree /
13 levels with 16 message-passing steps."""
import numpy as np
import pytest
import torch

from graphcast_b200 import _native, autoregressive, graphcast
from graphcast_b200 import xarray_shim as xs
from test_gpu_input_grads import _full_problem, _stack

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
N = 512


def _st():
  return torch.cuda.current_stream().cuda_stream


# ---- kernels ---------------------------------------------------------------------------------------
def _stacked(gen, dirs, rows, stride, scale=1.0):
  """A stacked table of `dirs` directions of `rows` rows, `stride` rows apart, NaN in the pad rows."""
  t = torch.full([(dirs - 1) * stride + rows, N], float("nan"), device=DEV)
  for k in range(dirs):
    t[k * stride:k * stride + rows] = torch.randn(rows, N, generator=gen, device=DEV) * scale
  return t


def _pads_untouched(out, dirs, rows, stride):
  for k in range(dirs - 1):
    assert torch.isnan(out[k * stride + rows:(k + 1) * stride]).all()


@pytest.mark.parametrize("rows", [1, 77, 1003])
@pytest.mark.parametrize("tangents", [1, 2, 5])
def test_swish_backward_jvp_dirs_kernel(tangents, rows):
  lib = _native.lib()
  gen = torch.Generator(device=DEV).manual_seed(7 + tangents)
  stride = (rows + 127) // 128 * 128 + 128             # larger than rows, pad rows in between
  h = torch.randn(rows, N, generator=gen, device=DEV) * 3
  hd = _stacked(gen, tangents, rows, stride)
  da = _stacked(gen, 1 + tangents, rows, stride)

  def run(src, dst=None):
    out = torch.full_like(src, float("nan")) if dst is None else dst
    _native.check(lib.gcb_swish_backward_jvp_dirs(
        h.data_ptr(), N, hd.data_ptr(), N, rows, N, src.data_ptr(), N, stride, out.data_ptr(), N,
        tangents, _st()), "gcb_swish_backward_jvp_dirs")
    return out

  out = run(da)
  want0 = torch.empty(rows, N, device=DEV)
  _native.check(lib.gcb_swish_jvp(h.data_ptr(), N, rows, N, da.data_ptr(), N, rows, 1,
                                  want0.data_ptr(), N, _st()), "gcb_swish_jvp")
  assert torch.equal(out[:rows], want0)
  for j in range(1, tangents + 1):                      # the one-tangent call on (0, j, j - 1)
    pair = torch.cat([da[:rows], da[j * stride:j * stride + rows]])
    one = torch.empty_like(pair)
    _native.check(lib.gcb_swish_backward_jvp(
        h.data_ptr(), N, hd[(j - 1) * stride:].data_ptr(), N, rows, N, pair.data_ptr(), N, rows,
        one.data_ptr(), N, _st()), "gcb_swish_backward_jvp")
    assert torch.equal(out[j * stride:j * stride + rows], one[rows:]), j
    assert torch.equal(one[:rows], want0)
  assert torch.isfinite(out[:rows]).all()
  _pads_untouched(out, 1 + tangents, rows, stride)
  inplace = da.clone()
  run(inplace, inplace)                                   # dh may alias da
  for k in range(1 + tangents):
    assert torch.equal(inplace[k * stride:k * stride + rows], out[k * stride:k * stride + rows]), k


@pytest.mark.parametrize("rows", [1, 77, 1003])
@pytest.mark.parametrize("tangents", [1, 2, 5])
def test_layernorm_backward_jvp_dirs_kernel(tangents, rows):
  lib = _native.lib()
  gen = torch.Generator(device=DEV).manual_seed(11 + tangents)
  stride = (rows + 127) // 128 * 128 + 128
  z = torch.randn(rows, N, generator=gen, device=DEV) * 2 + 0.5
  zd = _stacked(gen, tangents, rows, stride)
  dy = _stacked(gen, 1 + tangents, rows, stride)
  scale = torch.rand(N, generator=gen, device=DEV) + 0.5
  out = torch.full_like(dy, float("nan"))
  _native.check(lib.gcb_layernorm_backward_jvp_dirs(
      dy.data_ptr(), N, z.data_ptr(), N, zd.data_ptr(), N, scale.data_ptr(), rows, N, stride,
      out.data_ptr(), N, tangents, _st()), "gcb_layernorm_backward_jvp_dirs")
  want0 = torch.empty(rows, N, device=DEV)
  _native.check(lib.gcb_layernorm_backward_dirs(
      dy.data_ptr(), N, z.data_ptr(), N, scale.data_ptr(), rows, N, rows, 1, want0.data_ptr(), N,
      _st()), "gcb_layernorm_backward_dirs")
  assert torch.equal(out[:rows], want0)
  for j in range(1, tangents + 1):
    pair = torch.cat([dy[:rows], dy[j * stride:j * stride + rows]])
    one = torch.empty_like(pair)
    _native.check(lib.gcb_layernorm_backward_jvp(
        pair.data_ptr(), N, z.data_ptr(), N, zd[(j - 1) * stride:].data_ptr(), N, scale.data_ptr(),
        rows, N, rows, one.data_ptr(), N, _st()), "gcb_layernorm_backward_jvp")
    assert torch.equal(out[j * stride:j * stride + rows], one[rows:]), j
  assert torch.isfinite(out[:rows]).all()
  _pads_untouched(out, 1 + tangents, rows, stride)


def test_kernel_argument_checks():
  lib = _native.lib()
  t = torch.zeros(8, N, device=DEV)
  p = t.data_ptr()
  assert lib.gcb_swish_backward_jvp_dirs(p, N, p, N, 4, N, p, N, 4, p, N, 0, _st()) != 0
  assert lib.gcb_layernorm_backward_jvp_dirs(p, N, p, N, p, N, p, 4, N, 4, p, N, 0, _st()) != 0
  assert lib.gcb_layernorm_backward_jvp_dirs(p, N, p, N, p, N, p, 4, N, 3, p, N, 1, _st()) != 0


# ---- the model ---------------------------------------------------------------------------------------
def _directions(ds, seed, k, names=None, labels=None):
  rng = np.random.default_rng(seed)
  out = xs.Dataset(coords=ds.coords)
  if labels is not None:
    out.coords["direction"] = (("direction",), np.asarray(labels))
  for name, v in ds.data_vars.items():
    if names is None or name in names:
      out[name] = xs.DataArray(rng.standard_normal((k,) + tuple(v.shape)).astype(np.float32),
                               ("direction",) + tuple(v.dims))
  return out


def _vals(ds):
  return {k: np.asarray(v.values) for k, v in ds.data_vars.items()}


def _same(a, b):
  va, vb = _vals(a), _vals(b)
  assert set(va) == set(vb)
  for k in va:
    assert np.array_equal(va[k], vb[k]), k


def _at(ds, j):
  return None if ds is None else ds.isel(direction=j)


def _check_direction(got, j, want, like):
  """Direction j of a batched HVP Dataset `got` is bit for bit the Dataset `want`, shaped like `like`."""
  for name, v in like.data_vars.items():
    g = got.data_vars[name]
    assert g.dims == ("direction",) + tuple(v.dims), (name, g.dims)
    gj = np.asarray(g.values)[j]
    assert gj.dtype == np.float32
    assert np.array_equal(gj, np.asarray(want.data_vars[name].values)), (name, j)


def _check_grads(out, grads):
  loss, diag, ig, fg = out[:4]
  assert np.array_equal(np.asarray(loss.values), np.asarray(grads[0].values))
  _same(diag, grads[1])
  _same(ig, grads[2])
  _same(fg, grads[3])


@pytest.mark.parametrize("task_name,stack", [
    ("TASK_13", "plain"), ("TASK_13", "normalized"), ("TASK_13", "demo"), ("TASK", "normalized"),
    ("TASK", "demo"),
])
@pytest.mark.parametrize("with_forcings", [False, True])
@pytest.mark.parametrize("steps", [1, 3])
def test_every_direction_is_loss_and_input_hvp(task_name, stack, with_forcings, steps):
  """Direction k of the batched call is bit for bit loss_and_input_hvp along tangent k alone, for
  K = 1, 2 and 5 and directions_per_pass None, 1 and 2; the loss, diagnostics and gradients are bit for
  bit loss_and_input_grads."""
  _, pred, inputs, targets, forcings, _ = _stack(task_name, stack, steps)
  it = _directions(inputs, 3, 5)
  ft = _directions(forcings, 4, 5) if with_forcings else None
  grads = pred.loss_and_input_grads(inputs, targets, forcings)
  singles = [pred.loss_and_input_hvp(inputs, targets, forcings, _at(it, j), _at(ft, j))
             for j in range(5)]
  for s in singles:
    _check_grads(s, grads)
  for k, per in ((1, None), (2, 1), (2, None), (5, 2), (5, None)):
    sl = slice(0, k)
    out = pred.batched_loss_and_input_hvp(inputs, targets, forcings, it.isel(direction=sl),
                                          None if ft is None else ft.isel(direction=sl),
                                          directions_per_pass=per)
    assert len(out) == 6
    _check_grads(out, grads)
    for j in range(k):
      _check_direction(out[4], j, singles[j][4], inputs)
      _check_direction(out[5], j, singles[j][5], forcings)
    assert np.asarray(out[4].coords["direction"][1]).tolist() == list(range(k))


def test_every_pass_forms_the_same_loss_and_gradients():
  """A call of directions_per_pass = 2 over 5 directions runs three passes; each is what the call on
  its own directions runs, so each forms the loss and gradients of loss_and_input_grads."""
  _, pred, inputs, targets, forcings, _ = _stack("TASK_13", "normalized", 3)
  it, ft = _directions(inputs, 5, 5), _directions(forcings, 6, 5)
  grads = pred.loss_and_input_grads(inputs, targets, forcings)
  whole = pred.batched_loss_and_input_hvp(inputs, targets, forcings, it, ft, directions_per_pass=2)
  _check_grads(whole, grads)
  for sl in (slice(0, 2), slice(2, 4), slice(4, 5)):
    part = pred.batched_loss_and_input_hvp(inputs, targets, forcings, it.isel(direction=sl),
                                           ft.isel(direction=sl))
    _check_grads(part, grads)
    for j in range(sl.stop - sl.start):
      for got, want, like in ((whole[4], part[4], inputs), (whole[5], part[5], forcings)):
        for name in like.keys():
          assert np.array_equal(np.asarray(got.data_vars[name].values)[sl.start + j],
                                np.asarray(want.data_vars[name].values)[j]), (name, sl, j)


def test_noise_matches_single_calls():
  _, pred, inputs, targets, forcings, _ = _stack("TASK_13", "normalized", 2)
  noisy = autoregressive.Predictor(pred._predictor, noise_level=0.1, gradient_checkpointing=True)
  it, ft = _directions(inputs, 15, 2), _directions(forcings, 16, 2)
  out = noisy.batched_loss_and_input_hvp(inputs, targets, forcings, it, ft, rng=7,
                                         directions_per_pass=1)
  _check_grads(out, noisy.loss_and_input_grads(inputs, targets, forcings, rng=7))
  for j in range(2):
    one = noisy.loss_and_input_hvp(inputs, targets, forcings, _at(it, j), _at(ft, j), rng=7)
    _check_direction(out[4], j, one[4], inputs)
    _check_direction(out[5], j, one[5], forcings)


def test_labels_scaling_zeros_and_symmetry():
  _, pred, inputs, targets, forcings, _ = _stack("TASK_13", "normalized", 1)
  v = _directions(inputs, 8, 1)
  vf = _directions(forcings, 9, 1)
  w = _directions(inputs, 21, 1)
  wf = _directions(forcings, 22, 1)

  def stack(parts, labels):
    out = xs.Dataset(coords=parts[0].coords)
    out.coords["direction"] = (("direction",), np.asarray(labels))
    for name, x in parts[0].data_vars.items():
      out[name] = xs.DataArray(np.concatenate([np.asarray(p.data_vars[name].values) for p in parts]),
                               x.dims)
    return out

  def scaled(ds, c):
    out = xs.Dataset(coords=ds.coords)
    for k, x in ds.data_vars.items():
      out[k] = xs.DataArray(np.asarray(x.values) * np.float32(c), x.dims)
    return out

  labels = [10, 20, 30, 40]
  it = stack([v, scaled(v, 0.0), scaled(v, 4.0), w], labels)
  ft = stack([vf, scaled(vf, 0.0), scaled(vf, 4.0), wf], labels)
  out = pred.batched_loss_and_input_hvp(inputs, targets, forcings, it, ft)
  for ds in out[4:]:
    assert np.asarray(ds.coords["direction"][1]).tolist() == labels
    for name, x in _vals(ds).items():
      assert not np.any(x[1]), name                          # a zero direction gives exact zeros
      assert np.array_equal(x[0] * np.float32(4.0), x[2]), name   # 4 v gives exactly 4 H v

  def dot(a_in, a_f, ja, b_in, b_f, jb):
    s = 0.0
    for a, b in ((a_in, b_in), (a_f, b_f)):
      for k, x in a.data_vars.items():
        s += float(np.sum(np.asarray(x.values, np.float64)[ja] *
                          np.asarray(b.data_vars[k].values, np.float64)[jb]))
    return s

  lhs, rhs = dot(it, ft, 3, out[4], out[5], 0), dot(it, ft, 0, out[4], out[5], 3)
  print(f"<w, Hv> = {lhs:.9g}, <v, Hw> = {rhs:.9g}")
  assert abs(lhs - rhs) <= 1e-4 * max(abs(lhs), abs(rhs))
  # and the call did not change what the others compute
  again = pred.batched_loss_and_input_hvp(inputs, targets, forcings, it, ft, directions_per_pass=3)
  for a, b in zip(out[2:], again[2:]):
    _same(a, b)


def test_two_directions_at_one_degree():
  """K = 2 at 1 degree / 13 levels with 16 message-passing steps (every tangent edge snapshot of the
  processor is read, the bipartite edge sets run in several chunks) against two loss_and_input_hvp
  calls, bit for bit."""
  model, ar, inputs, targets, forcings = _full_problem(graphcast.TASK_13, 1.0, 5, 1)
  pred = ar._predictor
  it, ft = _directions(inputs, 17, 2), _directions(forcings, 18, 2)
  out = pred.batched_loss_and_input_hvp(inputs, targets, forcings, it, ft)
  for j in range(2):
    one = pred.loss_and_input_hvp(inputs, targets, forcings, _at(it, j), _at(ft, j))
    if j == 0:
      _check_grads(out, one)
    _check_direction(out[4], j, one[4], inputs)
    _check_direction(out[5], j, one[5], forcings)
