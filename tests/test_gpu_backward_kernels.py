"""The backward, tangent and HVP kernels (csrc/backward_kernels.cuh) against float64 references of the
same operations, through the C ABI, on seeded device data.  The references are formed on the device
from the values each kernel actually read (hi + lo for an operand image, the fp32 tables otherwise).

Every output buffer carries NaN sentinels (padding columns, a row past the end, pad rows between
stacked directions, rows above and below a weight-gradient row range) that must come back untouched.
Each axis (source, stride, width, row count, accumulate mode, direction count, arithmetic edge) is
varied against a base case; the production shapes run in full.

Every tolerance is an elementwise (or per-row) bound from an fp32 rounding model, derived in the
docstring of the test that uses it; each case prints its largest error / bound ratio.  Bit equality
is asserted only where the header promises it: run to run, accumulate onto +0 against accumulate = 0,
with and without the heavy list of gcb_segment_sum_sorted, and the direction kernels against the
one-direction kernels.  The refusals of these entry points are in test_native_abi.py."""
import numpy as np
import pytest
import torch

from graphcast_b200 import _native
from test_gpu_layer import _image_values

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
U = 2.0 ** -24                        # fp32 unit roundoff
NAN = float("nan")


def _st():
  return torch.cuda.current_stream().cuda_stream


def _gen(seed):
  return torch.Generator(device=DEV).manual_seed(seed)


def _padded(rows, n, ld, values=None):
  """[rows + 1, ld] fp32, NaN everywhere but [:rows, :n] (= values when given): NaN padding columns
  and a NaN row past the end."""
  t = torch.full((rows + 1, ld), NAN, device=DEV)
  if values is not None:
    t[:rows, :n] = values
  return t


def _stacked(dirs, rows, stride, ld, n, values=None):
  """dirs tables of [rows, n] stacked direction-major at row stride `stride` in a [dirs * stride + 1,
  ld] buffer; NaN in the padding columns, the pad rows between directions and the row past the end.
  values: [dirs, rows, n] or None (all NaN)."""
  t = torch.full((dirs * stride + 1, ld), NAN, device=DEV)
  if values is not None:
    for k in range(dirs):
      t[k * stride:k * stride + rows, :n] = values[k]
  return t


def _dir(t, k, rows, stride, n):
  return t[k * stride:k * stride + rows, :n]


def _dir_ptr(t, k, stride):
  """Device address of direction k (valid at rows = 0 too, where the direction is empty)."""
  return t[k * stride:].data_ptr()


def _sentinels_intact(t, dirs, rows, stride, n):
  """Every element of a _stacked / _padded buffer outside the data is still NaN."""
  mask = torch.ones_like(t, dtype=torch.bool)
  for k in range(dirs):
    mask[k * stride:k * stride + rows, :n] = False
  return bool(torch.isnan(t[mask]).all())


def _check(name, err, bound):
  """err <= bound elementwise; prints the largest ratio."""
  ratio = (err / bound).max().item() if err.numel() else 0.0
  print(f"{name}: max error / bound {ratio:.3g}")
  assert not torch.isnan(err).any(), f"{name}: NaN in the output"
  assert ratio <= 1.0, f"{name}: error exceeds the rounding bound by {ratio:.3g}x"


def _ids(v):
  return "-".join(map(str, v)) if isinstance(v, tuple) else str(v)


def _swish64(x):
  return x * torch.sigmoid(x)


# ---- weight gradient ------------------------------------------------------------------------------
WG_BASE = dict(prec="bf16x3", source="fp32", k=512, k_valid=512, ld_x=516, n=256, ld_g=260, rows=2049)


def _wg_run(lib, x, ld_x, k_valid, img, swish, g, ld_g, rows, k, n, prec, dw, acc):
  nb = lib.gcb_weight_grad_workspace_bytes(k, n)
  ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
  _native.check(lib.gcb_weight_grad(
      None if img is not None else x.data_ptr(), 0 if img is not None else ld_x,
      0 if img is not None else k_valid, None if img is None else img.data_ptr(), 1 if swish else 0,
      g.data_ptr(), ld_g, rows, k, n, _native.PRECISIONS[prec], ws.data_ptr(), nb, dw.data_ptr(), acc,
      _st()), "gcb_weight_grad")


def _weight_grad_case(prec, source, k, k_valid, ld_x, n, ld_g, rows, seed=0):
  """dw = X^T G against fp64, with the sentinels and the three accumulate modes (see the test)."""
  lib = _native.lib()
  gen = _gen(seed + 7 * rows + k + n)
  swish = source.startswith("swish")
  xv = torch.zeros(rows, k, device=DEV)
  xv[:, :k_valid] = torch.randn(rows, k_valid, generator=gen, device=DEV) * (2.0 if swish else 1.0)
  x = _padded(rows, k_valid, ld_x, xv[:, :k_valid])       # NaN beyond k_valid: never read
  img = None
  if source.endswith("image"):
    dense = xv.contiguous()
    img = torch.zeros(lib.gcb_a_image_bytes(max(rows, 1), k), dtype=torch.uint8, device=DEV)
    if rows:
      _native.check(lib.gcb_rows_to_image(dense.data_ptr(), k, 1, rows, k, img.data_ptr(), _st()), "img")
    xr = _image_values(img, rows, k).double()               # the values the kernel reads
  else:
    xr = xv.double()
  if swish:
    xr = _swish64(xr)
  g = _padded(rows, n, ld_g, torch.randn(rows, n, generator=gen, device=DEV))
  gd = g[:rows, :n].double()
  ref = xr.t() @ gd
  mag = xr.abs().t() @ gd.abs()                            # sum_r |x_r| |g_r|
  # the rounding model (docstring of test_weight_grad_matrix)
  if prec == "bf16x3":
    c = 3 * 2.0 ** -16 + 2 * 768 * U
  else:
    c = 2 * 2.0 ** -8 + 2 * 256 * U
  c += 2 * U + (4 * U if swish else 0.0)

  def fresh(fill):
    big = torch.full((k + 2, n), NAN, device=DEV)           # NaN rows above and below dw
    if fill is not None:
      big[1:k + 1] = fill
    return big

  args = (x, ld_x, k_valid, img, swish, g, ld_g, rows, k, n, prec)
  out = {}
  for name, fill, acc in (("acc0", None, 0), ("again", None, 0), ("onto0", 0.0, 1)):
    big = fresh(fill)
    _wg_run(lib, *args, big[1:k + 1], acc)
    out[name] = big
  base = torch.randn(k, n, generator=gen, device=DEV)
  big = fresh(base)
  _wg_run(lib, *args, big[1:k + 1], 1)
  out["base"] = big
  torch.cuda.synchronize()
  for name, big in out.items():
    assert torch.isnan(big[0]).all() and torch.isnan(big[k + 1]).all(), f"{name}: sentinel rows written"
  dw = out["acc0"][1:k + 1]
  assert torch.equal(dw, out["again"][1:k + 1]), "two runs differ"
  assert torch.equal(dw, out["onto0"][1:k + 1]), "accumulate onto +0 differs from accumulate = 0"
  tag = f"wgrad {prec} {source} k={k}/{k_valid} ld_x={ld_x} n={n} ld_g={ld_g} rows={rows}"
  _check(tag, (dw.double() - ref).abs(), c * mag + U * dw.double().abs() + 1e-38)
  got = out["base"][1:k + 1].double()
  want = ref + base.double()
  _check(tag + " onto a base", (got - want).abs(), c * mag + U * got.abs() + 1e-38)


@pytest.mark.parametrize("axis,value", (
    [("source", s) for s in ("fp32", "image", "swish", "swish_image")]
    + [("prec,source", ("bf16", s)) for s in ("fp32", "image", "swish", "swish_image")]
    + [("k,k_valid,ld_x,source", (k, kv, ld, s))
       for k, kv, ld in ((16, 4, 4), (48, 44, 52), (192, 188, 196), (480, 476, 480), (512, 512, 516),
                         (528, 512, 528))
       for s in ("fp32", "image")]
    + [("k,k_valid,ld_x,source,prec", (192, 188, 196, "swish_image", "bf16"))]
    + [("n,ld_g", (n, ld)) for n in (64, 128, 256, 512) for ld in (n, n + 4)]
    + [("rows", r) for r in (0, 1, 31, 33, 2047, 2049, 16384, 16385, 300_001)]
    + [("rows,source", (r, "image")) for r in (1, 33, 16385)]), ids=_ids)
def test_weight_grad_matrix(axis, value):
  """gcb_weight_grad against fp64 X^T G, one axis varied against WG_BASE.  Bound, elementwise with
  S = sum_r |x_r| |g_r| (u = 2^-24):
    split:  bf16x3 drops lo*lo and the residues of the split, |x g - (hh + hl + lh)| <= 3 * 2^-16 |x g|
            (2^-8 per bf16 rounding, conservatively); bf16 keeps hi*hi only, <= 2 * 2^-8 |x g|.
    fp32 accumulation between fp64 flushes: at most 256 rows x (3 | 1) exact products per flush,
            each addition off by at most 2u (the tensor core may truncate): 2 * 768 u S | 2 * 256 u S.
    the slice partial rounded to fp32 and the final fp64 sum rounded once: u S + u |dw| (with
            accumulate the base is exact in fp64 and shares only this last rounding).
    swish sources: x / (1 + expf(-x)) in fp32 is off by <= 4u relative (expf 2 ulp, add, divide).
  dw is written into a row range of a NaN tensor (accumulate = 0), onto +0 (must be accumulate = 0
  bit for bit) and onto a random base; a second run must be bit-identical."""
  case = dict(WG_BASE)
  names = axis.split(",")
  vals = value if len(names) > 1 else (value,)
  case.update(zip(names, vals))
  if case["source"].endswith("image") and "ld_x" not in names:
    case["ld_x"] = max(case["k_valid"], 4)
  _weight_grad_case(**case)


# ---- row-wise backward with column sums ------------------------------------------------------------
def _ln_model(z):
  """fp64 LayerNorm statistics of the fp32 rows z and the error model of their fp32 recomputation
  in the kernels (ln_row_stats and its pinned restatement: the row sum in chains of 21 roundings, 16
  per lane then five butterfly steps; the variance two-pass from z - mean):
    |d mean| <= 21 u max|z|,  |d var| <= 3 * 21 u M^2 + d_mean^2   (M = max|z - mean|),
    rstd relative error  e_r <= |d var| / (2 (var + eps)) + 6u   (rsqrtf 2 ulp, two roundings),
    |d zhat| <= rstd |d mean| + Zm (e_r + 2u)                      (Zm = max|zhat|)."""
  mean = z.mean(1, keepdim=True)
  var = ((z - mean) ** 2).mean(1, keepdim=True)
  rstd = torch.rsqrt(var + 1e-5)
  zhat = (z - mean) * rstd
  d_mean = 21 * U * z.abs().amax(1, keepdim=True)
  big_m = (z - mean).abs().amax(1, keepdim=True)
  d_var = 3 * 21 * U * big_m ** 2 + d_mean ** 2
  e_r = d_var / (2 * (var + 1e-5)) + 6 * U
  zm = zhat.abs().amax(1, keepdim=True)
  d_zhat = rstd * d_mean + zm * (e_r + 2 * U)
  return dict(rstd=rstd, zhat=zhat, e_r=e_r, zm=zm, d_zhat=d_zhat)


def _ln_bracket(x, m):
  """B = rstd (x - mean(x) - zhat mean(zhat x)) in fp64, and the per-row bound of its fp32 error:
  with Xm = max|x|, |mean(x)| <= Xm, |mean(zhat x)| <= Xm Zm, the sums in chains of <= 23 roundings,
  and three roundings in the bracket,
    |dB| <= rstd Xm (30u + 26u Zm^2 + 2 Zm |d zhat| + (2 + Zm^2) e_r)."""
  zhat = m["zhat"]
  b = m["rstd"] * (x - x.mean(1, keepdim=True) - zhat * (zhat * x).mean(1, keepdim=True))
  xm = x.abs().amax(1, keepdim=True)
  zm = m["zm"]
  db = m["rstd"] * xm * (30 * U + 26 * U * zm ** 2 + 2 * zm * m["d_zhat"] + (2 + zm ** 2) * m["e_r"])
  return b, db


def _z_rows(kind, rows, n, gen):
  """Pre-LayerNorm / pre-activation rows: 'normal' 2 N(0,1) + 0.5, 'offset' 1e3 + N(0, 2), 'const'
  0.75 in every column, 'spread' linspace(-100, 100) across the columns plus 0.1 N(0, 1)."""
  if kind == "normal":
    return torch.randn(rows, n, generator=gen, device=DEV) * 2 + 0.5
  if kind == "offset":
    return 1e3 + torch.randn(rows, n, generator=gen, device=DEV) * 2 ** 0.5
  if kind == "const":
    return torch.full((rows, n), 0.75, device=DEV)
  return torch.linspace(-100, 100, n, device=DEV) + 0.1 * torch.randn(rows, n, generator=gen, device=DEV)


def _swish_d1(h):
  s = torch.sigmoid(h)
  return s * (1 + h * (1 - s))


def _swish_d2(h):
  s = torch.sigmoid(h)
  return s * (1 - s) * (2 + h * (1 - 2 * s))


SWISH_FLOOR = 1e-36   # below exp(-88.7) expf overflows and sg = 0: s, s', s'' then lose <= 3e-37


def _swish_err(h):
  """|error| of the kernels' fp32 s'(h) and s''(h): sg = 1 / (1 + expf(-h)) is off by <= 6u
  relative, 1 - sg by <= 7u absolute, and the few products / fmas each round once, so both are
  within 16u (1 + |h|) (|s'| <= 1.1, |s''| <= 0.5), plus the underflow floor."""
  return 16 * U * (1 + h.abs()) + SWISH_FLOOR


def _col_sum_bound(terms, rows):
  """Column sums: each of kRowSlices = 256 blocks sums its rows in fp64 (exact to 2^-53), rounds
  once to fp32, and the blocks are summed in fp64 and rounded again:  u sum_b |S_b| + u |S|."""
  per = -(-rows // 256) if rows else 1
  padded = torch.zeros(256 * per, terms.shape[1], dtype=torch.float64, device=DEV)
  padded[:rows] = terms
  blocks = padded.view(256, per, -1).sum(1)
  return U * blocks.abs().sum(0) + U * terms.sum(0).abs() + 1e-38


ROW_BASE = dict(mode="ln", n=512, ld=516, rows=257, acc=0, z="normal")


def _rowwise_case(mode, n, ld, rows, acc, z, seed=1):
  lib = _native.lib()
  gen = _gen(seed + rows + n + ld)
  dyv = torch.randn(rows, n, generator=gen, device=DEV)
  zv = _z_rows(z, rows, n, gen)
  scale = torch.rand(n, generator=gen, device=DEV) + 0.5
  dy, zt = _padded(rows, n, ld, dyv), _padded(rows, n, ld, zv)
  with_dz = mode != "copy_nodz"
  dz = _padded(rows, n, ld) if with_dz else None
  nsums = 3 if mode == "ln" else 1
  bases = [torch.randn(n, generator=gen, device=DEV) if acc else None for _ in range(nsums)]
  sums = [torch.full((n + 8,), NAN, device=DEV) for _ in range(nsums)]   # 4 NaN either side
  for s, b in zip(sums, bases):
    if b is not None:
      s[4:4 + n] = b
  nb = lib.gcb_rowwise_workspace_bytes(n)
  ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
  sp = [s[4:].data_ptr() for s in sums]
  if mode == "ln":
    rc = lib.gcb_layernorm_backward(dy.data_ptr(), ld, zt.data_ptr(), ld, scale.data_ptr(), rows, n,
                                    dz.data_ptr(), ld, ws.data_ptr(), nb, sp[0], sp[1], sp[2], acc, _st())
  elif mode == "swish":
    rc = lib.gcb_swish_backward(dy.data_ptr(), ld, zt.data_ptr(), ld, rows, n, dz.data_ptr(), ld,
                                ws.data_ptr(), nb, sp[0], acc, _st())
  else:
    rc = lib.gcb_layernorm_backward(dy.data_ptr(), ld, None, 0, None, rows, n,
                                    dz.data_ptr() if with_dz else None, ld, ws.data_ptr(), nb, sp[0],
                                    None, None, acc, _st())
  _native.check(rc, f"rowwise {mode}")
  torch.cuda.synchronize()
  tag = f"rowwise {mode} n={n} ld={ld} rows={rows} acc={acc} z={z}"
  d = dyv.double()
  h = zv.double()
  if mode == "ln":
    m = _ln_model(h)
    g = d * scale.double()
    want_dz, bnd = _ln_bracket(g, m)
    bnd = bnd + U * want_dz.abs()
    col = [("dbias", None), ("dscale", d * m["zhat"]), ("doffset", d)]
  elif mode == "swish":
    want_dz = d * _swish_d1(h)
    bnd = d.abs() * _swish_err(h) + U * want_dz.abs()
    col = [("dbias", None)]
  else:
    want_dz, bnd = d, torch.zeros_like(d)
    col = [("dbias", None)]
  if with_dz:
    assert _sentinels_intact(dz, 1, rows, rows, n), f"{tag}: dz sentinels written"
    got_dz = dz[:rows, :n].double()
    if mode.startswith("copy"):
      assert torch.equal(dz[:rows, :n], dyv), tag
    else:
      _check(tag + " dz", (got_dz - want_dz).abs(), bnd + 1e-38)
  for q, (name, terms) in enumerate(col):
    s = sums[q]
    assert torch.isnan(s[:4]).all() and torch.isnan(s[4 + n:]).all(), f"{tag}: {name} sentinels written"
    if name == "dbias":
      # the kernel sums its own fp32 dz: the reference sums fp64 dz, plus dz's error bound per row
      terms, prop = want_dz, bnd.sum(0)
    elif name == "dscale":
      prop = (d.abs() * m["d_zhat"]).sum(0)                  # the kernel's zhat
    else:
      prop = 0.0
    want = terms.sum(0) + (bases[q].double() if acc else 0.0)
    b = _col_sum_bound(terms, rows) + prop + U * want.abs()
    _check(f"{tag} {name}", (s[4:4 + n].double() - want).abs(), b)
    if name == "dscale" and z == "const" and not acc:
      assert torch.equal(s[4:4 + n], torch.zeros(n, device=DEV)), "zhat of a constant row must be 0"


@pytest.mark.parametrize("axis,value", (
    [("mode,n", (m, n)) for m, n in (("ln", 512), ("swish", 512), ("swish", 256), ("copy", 512),
                                     ("copy", 256), ("copy_nodz", 256), ("copy_nodz", 512))]
    + [("ld", 512)]
    + [("mode,n,ld", (m, 256, 256)) for m in ("swish", "copy")]
    + [("rows", r) for r in (0, 1, 255, 256, 70_001, 1_048_577)]
    + [("mode,rows", (m, r)) for m in ("swish", "copy") for r in (0, 1, 255, 256, 1_048_577)]
    + [("acc", 1)] + [("mode,n,acc", (m, 256, 1)) for m in ("swish", "copy", "copy_nodz")]
    + [("acc,rows", (1, r)) for r in (0, 70_001)]
    + [("z", z) for z in ("offset", "const")]
    + [("mode,z", ("swish", "spread")), ("mode,n,z", ("swish", 256, "spread"))]), ids=_ids)
def test_rowwise_backward_matrix(axis, value):
  """gcb_layernorm_backward (LayerNorm and copy modes, dz = NULL too) and gcb_swish_backward against
  fp64, one axis varied against ROW_BASE: dz and every column sum, with NaN sentinels in dz and
  around the sums, accumulate 0 and 1 (onto a random base).  Bounds:
    LayerNorm dz: _ln_model / _ln_bracket with x = dy * scale, plus u |dz| for the last rounding.
    swish dz: |dy| * 16u (1 + |h|) (+ floor) + u |dz|  (_swish_err).
    column sums: _col_sum_bound, plus the propagated error of the summed fp32 terms: dz's bound
    summed over the rows for dbias, sum_r |dy| |d zhat| for dscale, none for doffset (dy is exact);
    and u |sum| for the base's rounding.
  Constant rows must give zhat = 0 exactly, so dscale is exactly 0."""
  case = dict(ROW_BASE)
  names = axis.split(",")
  vals = value if len(names) > 1 else (value,)
  case.update(zip(names, vals))
  if "ld" not in names:
    case["ld"] = case["n"] + 4
  _rowwise_case(**case)


# ---- tangent and HVP row kernels --------------------------------------------------------------------
def _swish_rows_out(lib, h, rows, n, ld):
  a = _padded(rows, n, ld)
  _native.check(lib.gcb_swish_rows(h.data_ptr(), ld, rows, n, a.data_ptr(), ld, _st()), "swish_rows")
  return a


@pytest.mark.parametrize("rows,n,z", [(0, 512, "normal"), (1, 512, "normal"), (1003, 512, "normal"),
                                      (1003, 256, "spread"), (9, 512, "spread"), (1003, 12, "normal")])
def test_swish_rows(rows, n, z):
  """gcb_swish_rows: a = h / (1 + expf(-h)) against fp64 swish.  expf is within 2 ulp, the add and
  the division round once each: <= 6u |a|, bounded by 8u |a|; below h = -88.7 expf overflows and a is
  -0 where fp64 gives at most 3e-37 (SWISH_FLOOR).  ld = n + 4 with NaN sentinels."""
  lib = _native.lib()
  hv = _z_rows(z, rows, n, _gen(rows + n))
  h = _padded(rows, n, n + 4, hv)
  a = _swish_rows_out(lib, h, rows, n, n + 4)
  torch.cuda.synchronize()
  assert _sentinels_intact(a, 1, rows, rows, n)
  want = _swish64(hv.double())
  got = a[:rows, :n].double()
  assert torch.isfinite(got).all()
  _check(f"swish_rows rows={rows} n={n} {z}", (got - want).abs(), 8 * U * want.abs() + SWISH_FLOOR)


TAN_CASES = ([(r, 2, r + 5, "normal") for r in (0, 1, 7, 8, 9, 1003)]
             + [(1003, k, s, "normal") for k in (1, 3) for s in (1003, 1008)]
             + [(1003, 2, 1003, z) for z in ("offset", "const", "spread")]
             + [(9, 3, 9, "const")])


@pytest.mark.parametrize("rows,dirs,stride,z", TAN_CASES)
def test_layernorm_jvp_kernels(rows, dirs, stride, z):
  """gcb_layernorm_jvp and gcb_layernorm_jvp_dirs against fp64
    out[k] = residual[k] + scale rstd (dz[k] - mean(dz[k]) - zhat mean(zhat dz[k])),
  with and without the residual, ld = 516 for every operand, `dirs` directions at `stride`.
  Bound per element: |scale| |dB| (_ln_bracket with x = dz) + 2u (|out| + |residual|) for the
  product with scale and the residual add.  Direction k of the dirs kernel must be the one-direction
  kernel on direction k bit for bit."""
  lib = _native.lib()
  n, ld = 512, 516
  gen = _gen(rows + 31 * dirs + stride)
  zv = _z_rows(z, rows, n, gen)
  zt = _padded(rows, n, ld, zv)
  dzv = torch.randn(dirs, rows, n, generator=gen, device=DEV)
  resv = torch.randn(dirs, rows, n, generator=gen, device=DEV)
  dz = _stacked(dirs, rows, stride, ld, n, dzv)
  res = _stacked(dirs, rows, stride, ld, n, resv)
  scale = torch.rand(n, generator=gen, device=DEV) + 0.5
  m = _ln_model(zv.double())
  for with_res in (False, True):
    out = _stacked(dirs, rows, stride, ld, n)
    _native.check(lib.gcb_layernorm_jvp_dirs(
        zt.data_ptr(), ld, dz.data_ptr(), ld, scale.data_ptr(), rows, n, stride, dirs,
        res.data_ptr() if with_res else None, ld, out.data_ptr(), ld, _st()), "ln_jvp_dirs")
    torch.cuda.synchronize()
    assert _sentinels_intact(out, dirs, rows, stride, n)
    for k in range(dirs):
      one = _padded(rows, n, ld)
      _native.check(lib.gcb_layernorm_jvp(
          zt.data_ptr(), ld, _dir_ptr(dz, k, stride), ld, scale.data_ptr(), rows, n,
          _dir_ptr(res, k, stride) if with_res else None, ld, one.data_ptr(), ld, _st()),
          "ln_jvp")
      torch.cuda.synchronize()
      assert _sentinels_intact(one, 1, rows, rows, n)
      got = _dir(out, k, rows, stride, n)
      assert torch.equal(got, one[:rows, :n]), f"direction {k} differs from the one-direction kernel"
      b, db = _ln_bracket(dzv[k].double(), m)
      r = resv[k].double() if with_res else 0.0
      want = r + scale.double() * b
      bound = scale.double() * db + 2 * U * (want.abs() + (resv[k].double().abs() if with_res else 0.0))
      _check(f"ln_jvp rows={rows} dir {k}/{dirs} stride={stride} {z} res={with_res}",
             (got.double() - want).abs(), bound + 1e-38)


@pytest.mark.parametrize("rows,dirs,stride,z", TAN_CASES)
def test_layernorm_backward_dirs_kernel(rows, dirs, stride, z):
  """gcb_layernorm_backward_dirs against fp64 dz[k] = _ln_bracket(dy[k] * scale) (bound: _ln_bracket
  plus u |dz|), ld = 516, and direction k bit for bit the dz of gcb_layernorm_backward for dy[k]
  alone, as the header promises."""
  lib = _native.lib()
  n, ld = 512, 516
  gen = _gen(rows + 17 * dirs + stride)
  zv = _z_rows(z, rows, n, gen)
  zt = _padded(rows, n, ld, zv)
  dyv = torch.randn(dirs, rows, n, generator=gen, device=DEV)
  dy = _stacked(dirs, rows, stride, ld, n, dyv)
  scale = torch.rand(n, generator=gen, device=DEV) + 0.5
  out = _stacked(dirs, rows, stride, ld, n)
  _native.check(lib.gcb_layernorm_backward_dirs(dy.data_ptr(), ld, zt.data_ptr(), ld, scale.data_ptr(),
                                                rows, n, stride, dirs, out.data_ptr(), ld, _st()), "dirs")
  nb = lib.gcb_rowwise_workspace_bytes(n)
  ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
  sums = torch.empty(3, n, device=DEV)
  torch.cuda.synchronize()
  assert _sentinels_intact(out, dirs, rows, stride, n)
  m = _ln_model(zv.double())
  for k in range(dirs):
    one = _padded(rows, n, ld)
    _native.check(lib.gcb_layernorm_backward(
        _dir_ptr(dy, k, stride), ld, zt.data_ptr(), ld, scale.data_ptr(), rows, n,
        one.data_ptr(), ld, ws.data_ptr(), nb, sums[0].data_ptr(), sums[1].data_ptr(), sums[2].data_ptr(),
        0, _st()), "ln_backward")
    torch.cuda.synchronize()
    got = _dir(out, k, rows, stride, n)
    assert torch.equal(got, one[:rows, :n]), f"direction {k} differs from gcb_layernorm_backward"
    want, db = _ln_bracket(dyv[k].double() * scale.double(), m)
    _check(f"ln_backward_dirs rows={rows} dir {k}/{dirs} stride={stride} {z}",
           (got.double() - want).abs(), db + U * want.abs() + 1e-38)


def _ln_hvp64(dy, dyd, z, zd, scale, m):
  """fp64 direction-j tangent of dz along zdot (formulas in backward_kernels.cuh) and the per-element
  bound of its fp32 error, first order in the input errors of every term (see the test)."""
  r, zhat, zm, dzh, e_r = m["rstd"], m["zhat"], m["zm"], m["d_zhat"], m["e_r"]
  mean = lambda x: x.mean(1, keepdim=True)
  amax = lambda x: x.abs().amax(1, keepdim=True)
  g, gd = dy * scale, dyd * scale
  mm = mean(g * zhat)
  a = g - mean(g) - zhat * mm
  rdot = -r * r * mean(zhat * zd)
  zhd = r * (zd - mean(zd) - zhat * mean(zhat * zd))
  mdot = mean(gd * zhat + g * zhd)
  b = gd - mean(gd) - zhd * mm - zhat * mdot
  want = rdot * a + r * b
  gm, gdm, tm = amax(g), amax(gd), amax(zd)
  c = 30 * U + 26 * U * zm ** 2 + 2 * zm * dzh       # the bracket's rounding factor (_ln_bracket)
  hm = r * tm * (2 + zm ** 2)                        # max |zhat-dot|
  d_h = r * tm * (c + (2 + zm ** 2) * e_r)
  rdm = r * r * zm * tm                              # max |rdot|
  d_rd = r * r * (tm * dzh + 23 * U * zm * tm) + rdm * (2 * e_r + 2 * U)
  d_mm = gm * dzh + 23 * U * gm * zm
  mdm = gdm * zm + gm * hm
  d_md = gdm * dzh + gm * d_h + 24 * U * mdm
  am = gm * (2 + zm ** 2)
  d_a = gm * c
  bm = 2 * gdm + hm * gm * zm + zm * mdm
  d_b = 25 * U * gdm + d_h * gm * zm + hm * d_mm + dzh * mdm + zm * d_md + 4 * U * bm
  bound = r * d_b + r * bm * e_r + rdm * d_a + am * d_rd + 2 * U * (r * bm + rdm * am)
  return want, bound


@pytest.mark.parametrize("rows,dirs,stride,z", TAN_CASES)
def test_layernorm_backward_jvp_kernels(rows, dirs, stride, z):
  """gcb_layernorm_backward_jvp_dirs with K = dirs tangents (1 + K directions) against fp64, ld = 516.
  Direction 0 must be gcb_layernorm_backward_dirs bit for bit; direction j the K = 1 call
  (gcb_layernorm_backward_jvp) on (0, j, tangent j - 1) bit for bit.  Bound of direction j, first
  order: every term of  dzdot = rdot a + rstd b  carries the error of its inputs (d zhat, e_r from
  _ln_model, the bracket factor of _ln_bracket for zhat-dot and a) and <= 25 roundings of its sums,
  each bounded through the row maxima |g|, |gdot|, |zdot|, |zhat| (_ln_hvp64)."""
  lib = _native.lib()
  n, ld = 512, 516
  gen = _gen(rows + 13 * dirs + stride)
  zv = _z_rows(z, rows, n, gen)
  zt = _padded(rows, n, ld, zv)
  dyv = torch.randn(1 + dirs, rows, n, generator=gen, device=DEV)
  zdv = torch.randn(dirs, rows, n, generator=gen, device=DEV)
  dy = _stacked(1 + dirs, rows, stride, ld, n, dyv)
  zd = _stacked(dirs, rows, stride, ld, n, zdv)
  scale = torch.rand(n, generator=gen, device=DEV) + 0.5
  out = _stacked(1 + dirs, rows, stride, ld, n)
  _native.check(lib.gcb_layernorm_backward_jvp_dirs(
      dy.data_ptr(), ld, zt.data_ptr(), ld, zd.data_ptr(), ld, scale.data_ptr(), rows, n, stride,
      out.data_ptr(), ld, dirs, _st()), "ln_hvp")
  back = _padded(rows, n, ld)
  _native.check(lib.gcb_layernorm_backward_dirs(dy.data_ptr(), ld, zt.data_ptr(), ld, scale.data_ptr(),
                                                rows, n, stride, 1, back.data_ptr(), ld, _st()), "dirs")
  torch.cuda.synchronize()
  assert _sentinels_intact(out, 1 + dirs, rows, stride, n)
  assert torch.equal(_dir(out, 0, rows, stride, n), back[:rows, :n]), "direction 0 != the backward"
  m = _ln_model(zv.double())
  for j in range(1, 1 + dirs):
    s1 = rows + 3                                    # a K = 1 call at its own stride
    dy1 = _stacked(2, rows, s1, ld, n, torch.stack([dyv[0], dyv[j]]))
    zd1 = _padded(rows, n, ld, zdv[j - 1])
    one = _stacked(2, rows, s1, ld, n)
    _native.check(lib.gcb_layernorm_backward_jvp(
        dy1.data_ptr(), ld, zt.data_ptr(), ld, zd1.data_ptr(), ld, scale.data_ptr(), rows, n, s1,
        one.data_ptr(), ld, _st()), "ln_hvp K=1")
    torch.cuda.synchronize()
    got = _dir(out, j, rows, stride, n)
    assert torch.equal(got, _dir(one, 1, rows, s1, n)), f"direction {j} differs from the K = 1 call"
    want, bound = _ln_hvp64(dyv[0].double(), dyv[j].double(), zv.double(), zdv[j - 1].double(),
                            scale.double(), m)
    _check(f"ln_hvp rows={rows} dir {j}/{dirs} stride={stride} {z}", (got.double() - want).abs(),
           bound + U * want.abs() + 1e-38)


SWISH_TAN = ([(r, 2, r + 5, 512, "normal") for r in (0, 1, 7, 8, 9, 1003)]
             + [(1003, k, s, 512, "normal") for k in (1, 3) for s in (1003, 1008)]
             + [(1003, 2, 1008, 256, "spread"), (1003, 3, 1003, 512, "spread"), (9, 2, 14, 12, "spread")])


@pytest.mark.parametrize("rows,dirs,stride,n,z", SWISH_TAN)
def test_swish_jvp_kernel(rows, dirs, stride, n, z):
  """gcb_swish_jvp: da[k] = s'(h) dh[k] against fp64, ld = n + 4, with da apart from dh and aliasing
  it (the header allows da = dh).  Bound: |dh| 16u (1 + |h|) (+ floor, _swish_err) + u |da|.
  Direction k must be the one-direction call bit for bit, aliased or not."""
  lib = _native.lib()
  ld = n + 4
  gen = _gen(rows + 7 * dirs + stride + n)
  hv = _z_rows(z, rows, n, gen)
  h = _padded(rows, n, ld, hv)
  dhv = torch.randn(dirs, rows, n, generator=gen, device=DEV)
  dh = _stacked(dirs, rows, stride, ld, n, dhv)
  out = _stacked(dirs, rows, stride, ld, n)
  _native.check(lib.gcb_swish_jvp(h.data_ptr(), ld, rows, n, dh.data_ptr(), ld, stride, dirs,
                                  out.data_ptr(), ld, _st()), "swish_jvp")
  inplace = dh.clone()
  _native.check(lib.gcb_swish_jvp(h.data_ptr(), ld, rows, n, inplace.data_ptr(), ld, stride, dirs,
                                  inplace.data_ptr(), ld, _st()), "swish_jvp in place")
  torch.cuda.synchronize()
  assert _sentinels_intact(out, dirs, rows, stride, n) and _sentinels_intact(inplace, dirs, rows, stride, n)
  assert torch.equal(torch.nan_to_num(out), torch.nan_to_num(inplace)), "da aliasing dh changes the result"
  f = _swish_d1(hv.double())
  err = _swish_err(hv.double())
  for k in range(dirs):
    one = _padded(rows, n, ld)
    _native.check(lib.gcb_swish_jvp(h.data_ptr(), ld, rows, n, _dir_ptr(dh, k, stride),
                                    ld, 0, 1, one.data_ptr(), ld, _st()), "swish_jvp one")
    torch.cuda.synchronize()
    got = _dir(out, k, rows, stride, n)
    assert torch.equal(got, one[:rows, :n]), f"direction {k} differs from the one-direction call"
    want = dhv[k].double() * f
    _check(f"swish_jvp rows={rows} n={n} dir {k}/{dirs} stride={stride} {z}", (got.double() - want).abs(),
           dhv[k].double().abs() * err + U * want.abs())


@pytest.mark.parametrize("rows,dirs,stride,n,z", SWISH_TAN)
def test_swish_backward_jvp_kernels(rows, dirs, stride, n, z):
  """gcb_swish_backward_jvp_dirs with K = dirs tangents against fp64, ld = n + 4, apart and with dh
  aliasing da.  Direction 0 = s'(h) da must be gcb_swish_jvp bit for bit; direction j =
  s'(h) dadot_j + s''(h) hdot_j da must be the K = 1 call on (0, j, j - 1) bit for bit.  Bound of
  direction j: |dadot| E + |hdot da| (E + 2u |s''|) + u |dhdot|, E = _swish_err(h) (the fma adds
  one rounding, the product (s'' hdot) da two)."""
  lib = _native.lib()
  ld = n + 4
  gen = _gen(rows + 11 * dirs + stride + n)
  hv = _z_rows(z, rows, n, gen)
  h = _padded(rows, n, ld, hv)
  dav = torch.randn(1 + dirs, rows, n, generator=gen, device=DEV)
  hdv = torch.randn(dirs, rows, n, generator=gen, device=DEV)
  da = _stacked(1 + dirs, rows, stride, ld, n, dav)
  hd = _stacked(dirs, rows, stride, ld, n, hdv)
  out = _stacked(1 + dirs, rows, stride, ld, n)
  _native.check(lib.gcb_swish_backward_jvp_dirs(h.data_ptr(), ld, hd.data_ptr(), ld, rows, n, da.data_ptr(),
                                                ld, stride, out.data_ptr(), ld, dirs, _st()), "swish_hvp")
  inplace = da.clone()
  _native.check(lib.gcb_swish_backward_jvp_dirs(h.data_ptr(), ld, hd.data_ptr(), ld, rows, n,
                                                inplace.data_ptr(), ld, stride, inplace.data_ptr(), ld,
                                                dirs, _st()), "swish_hvp in place")
  jvp = _padded(rows, n, ld)
  _native.check(lib.gcb_swish_jvp(h.data_ptr(), ld, rows, n, da.data_ptr(), ld, 0, 1, jvp.data_ptr(), ld,
                                  _st()), "swish_jvp")
  torch.cuda.synchronize()
  assert _sentinels_intact(out, 1 + dirs, rows, stride, n)
  assert _sentinels_intact(inplace, 1 + dirs, rows, stride, n)
  assert torch.equal(torch.nan_to_num(out), torch.nan_to_num(inplace)), "dh aliasing da changes the result"
  assert torch.equal(_dir(out, 0, rows, stride, n), jvp[:rows, :n]), "direction 0 != gcb_swish_jvp"
  hd64, d0 = hv.double(), dav[0].double()
  f1, f2, err = _swish_d1(hd64), _swish_d2(hd64), _swish_err(hd64)
  for j in range(1, 1 + dirs):
    s1 = rows + 1
    da1 = _stacked(2, rows, s1, ld, n, torch.stack([dav[0], dav[j]]))
    hd1 = _stacked(1, rows, s1, ld, n, hdv[j - 1:j])
    one = _stacked(2, rows, s1, ld, n)
    _native.check(lib.gcb_swish_backward_jvp(h.data_ptr(), ld, hd1.data_ptr(), ld, rows, n, da1.data_ptr(),
                                             ld, s1, one.data_ptr(), ld, _st()), "swish_hvp K=1")
    torch.cuda.synchronize()
    got = _dir(out, j, rows, stride, n)
    assert torch.equal(got, _dir(one, 1, rows, s1, n)), f"direction {j} differs from the K = 1 call"
    dj, tj = dav[j].double(), hdv[j - 1].double()
    want = dj * f1 + f2 * tj * d0
    bound = dj.abs() * err + (tj * d0).abs() * (err + 2 * U * f2.abs()) + U * want.abs()
    _check(f"swish_hvp rows={rows} n={n} dir {j}/{dirs} stride={stride} {z}", (got.double() - want).abs(),
           bound)


# ---- index operations --------------------------------------------------------------------------------
def _big_nodes():
  """More nodes than the light grid's cap of 16 blocks x 8 warps per SM: the warps stride."""
  return max(40_962, 16 * 8 * _native.lib().gcb_sm_count(0) + 1001)


def _segment_graph(num_nodes, seed, heavy_nodes=()):
  """Random degrees 0..5 with the first and last nodes empty and `heavy_nodes` given 300..700
  entries; returns the degrees and the CSR pointer."""
  rng = np.random.default_rng(seed)
  deg = rng.integers(0, 6, num_nodes)
  if num_nodes:
    deg[0] = deg[-1] = 0
  for v in heavy_nodes:
    deg[v] = rng.integers(300, 700)
  ptr = np.zeros(num_nodes + 1, np.int32)
  np.cumsum(deg, out=ptr[1:])
  return deg, ptr


def _seg_bound(msg_abs_sum, deg):
  """fp32 sums of `deg` terms in a fixed order: deg - 1 roundings along one chain, and the heavy
  receiver blocks' eight partial sums add at most 7 more, so |error| <= (deg + 7) u sum |m|."""
  return (torch.as_tensor(deg + 7, device=DEV, dtype=torch.float64)[:, None] * U * msg_abs_sum + 1e-38)


@pytest.mark.parametrize("num_nodes", [0, 1, 1000, "big"])
@pytest.mark.parametrize("ld", [512, 516])
def test_segment_sum_sorted(num_nodes, ld):
  """gcb_segment_sum_sorted (the backward of a sender gather) against fp64, with ld_msg = ld_out = ld,
  empty first and last nodes, NaN sentinels, and a heavy list that holds node 0 (empty), the last
  node (empty), an empty inner node and many heavy nodes.  The result must equal the run without the
  list bit for bit (the header promises it), and a second run.  Bound: _seg_bound."""
  lib = _native.lib()
  if num_nodes == "big":
    num_nodes = _big_nodes()
  hv_nodes = []
  if num_nodes >= 1000:
    hv_nodes = list(range(3, num_nodes - 1, max(1, num_nodes // 40)))
  deg, ptr = _segment_graph(num_nodes, num_nodes + ld, hv_nodes)
  n_edges = int(ptr[-1])
  rng = np.random.default_rng(num_nodes)
  snd = np.repeat(np.arange(num_nodes), deg)
  perm = rng.permutation(n_edges)                         # edge e = perm[j] belongs to node snd[j]
  order = np.empty(n_edges, np.int32)
  order[:] = perm
  edge_node = np.empty(n_edges, np.int64)
  edge_node[perm] = snd
  msgv = torch.randn(max(n_edges, 1), 512, generator=_gen(num_nodes + 3), device=DEV)
  msg = _padded(max(n_edges, 1), 512, ld, msgv)
  t = lambda a: torch.as_tensor(a).to(DEV)
  order_d, ptr_d = t(order if n_edges else np.zeros(1, np.int32)), t(ptr)
  heavy = sorted(set(hv_nodes) | ({0, num_nodes - 1, int(np.nonzero(deg[1:-1] == 0)[0][0]) + 1}
                                  if num_nodes >= 1000 else set()))
  heavy_d = t(np.asarray(heavy or [0], np.int32))

  def run(with_heavy):
    out = _padded(num_nodes, 512, ld)
    _native.check(lib.gcb_segment_sum_sorted(msg.data_ptr(), ld, order_d.data_ptr(), ptr_d.data_ptr(),
                                             num_nodes, heavy_d.data_ptr() if with_heavy else None,
                                             len(heavy) if with_heavy else 0, out.data_ptr(), ld, 512,
                                             _st()), "segment_sum_sorted")
    return out

  a, b, c = run(True), run(False), run(True)
  torch.cuda.synchronize()
  for o in (a, b):
    assert _sentinels_intact(o, 1, num_nodes, num_nodes, 512)
  assert torch.equal(a[:num_nodes, :512], b[:num_nodes, :512]), "the heavy list changes the result"
  assert torch.equal(a[:num_nodes, :512], c[:num_nodes, :512]), "two runs differ"
  ids = t(edge_node)
  want = torch.zeros(num_nodes, 512, dtype=torch.float64, device=DEV)
  mags = torch.zeros_like(want)
  if n_edges:
    want.index_add_(0, ids, msgv.double())
    mags.index_add_(0, ids, msgv.double().abs())
  got = a[:num_nodes, :512].double()
  if num_nodes:
    assert (got[0] == 0).all() and (got[-1] == 0).all()
  _check(f"segment_sum_sorted nodes={num_nodes} ld={ld} heavy={len(heavy)}", (got - want).abs(),
         _seg_bound(mags, deg))


@pytest.mark.parametrize("num_nodes", [0, 1, 1000, "big"])
@pytest.mark.parametrize("ld", [512, 516])
def test_segment_sum_receivers(num_nodes, ld):
  """gcb_segment_sum and gcb_segment_sum_heavy (receiver-sorted messages) against fp64, ld_msg =
  ld_out = ld, empty first and last nodes, NaN sentinels.  The heavy list is every node of more than
  256 entries, as the header asks; its blocks sum in another order than the warps, so only the rows
  outside the list must equal the run without it bit for bit.  Both must be deterministic.  Bound:
  _seg_bound."""
  lib = _native.lib()
  if num_nodes == "big":
    num_nodes = _big_nodes()
  hv_nodes = list(range(3, num_nodes - 1, max(1, num_nodes // 40))) if num_nodes >= 1000 else []
  deg, ptr = _segment_graph(num_nodes, num_nodes + ld + 1, hv_nodes)
  n_edges = int(ptr[-1])
  msgv = torch.randn(max(n_edges, 1), 512, generator=_gen(num_nodes + 5), device=DEV)
  msg = _padded(max(n_edges, 1), 512, ld, msgv)
  ptr_d = torch.as_tensor(ptr).to(DEV)
  heavy = np.nonzero(deg > 256)[0].astype(np.int32)
  heavy_d = torch.as_tensor(heavy if heavy.size else np.zeros(1, np.int32)).to(DEV)

  def run(with_heavy):
    out = _padded(num_nodes, 512, ld)
    if with_heavy:
      rc = lib.gcb_segment_sum_heavy(msg.data_ptr(), ld, ptr_d.data_ptr(), num_nodes, heavy_d.data_ptr(),
                                     heavy.size, out.data_ptr(), ld, 512, _st())
    else:
      rc = lib.gcb_segment_sum(msg.data_ptr(), ld, ptr_d.data_ptr(), num_nodes, out.data_ptr(), ld, 512,
                               _st())
    _native.check(rc, "segment_sum")
    return out

  outs = [run(False), run(True), run(False), run(True)]
  torch.cuda.synchronize()
  for o in outs:
    assert _sentinels_intact(o, 1, num_nodes, num_nodes, 512)
  assert torch.equal(torch.nan_to_num(outs[0]), torch.nan_to_num(outs[2])), "two runs differ"
  assert torch.equal(torch.nan_to_num(outs[1]), torch.nan_to_num(outs[3])), "two runs differ"
  light = torch.as_tensor(deg <= 256, device=DEV)
  assert torch.equal(outs[0][:num_nodes, :512][light], outs[1][:num_nodes, :512][light])
  ids = torch.as_tensor(np.repeat(np.arange(num_nodes), deg), device=DEV)
  want = torch.zeros(num_nodes, 512, dtype=torch.float64, device=DEV)
  mags = torch.zeros_like(want)
  if n_edges:
    want.index_add_(0, ids, msgv.double())
    mags.index_add_(0, ids, msgv.double().abs())
  for name, o in (("plain", outs[0]), ("heavy", outs[1])):
    got = o[:num_nodes, :512].double()
    if num_nodes:
      assert (got[0] == 0).all() and (got[-1] == 0).all()
    _check(f"segment_sum {name} nodes={num_nodes} ld={ld} heavy={heavy.size}", (got - want).abs(),
           _seg_bound(mags, deg))


@pytest.mark.parametrize("width", [4, 252, 512])
@pytest.mark.parametrize("with_addend", [False, True])
@pytest.mark.parametrize("n", [0, 1, 40_962])
def test_gather_add(width, with_addend, n):
  """gcb_gather_add: dst = addend + src[idx] with ld = width + 4 for src, addend and dst, NaN
  sentinels around every operand.  One fp32 addition per element, so the result is exact against
  the same fp32 addition (and bit for bit src[idx] without the addend)."""
  lib = _native.lib()
  ld = width + 4
  gen = _gen(width + n)
  n_src = 3001
  srcv = torch.randn(n_src, width, generator=gen, device=DEV)
  src = _padded(n_src, width, ld, srcv)
  idx = torch.randint(0, n_src, (max(n, 1),), generator=gen, device=DEV, dtype=torch.int32)
  addv = torch.randn(max(n, 1), width, generator=gen, device=DEV)
  add = _padded(max(n, 1), width, ld, addv)
  dst = _padded(n, width, ld)
  _native.check(lib.gcb_gather_add(src.data_ptr(), ld, idx.data_ptr(), n,
                                   add.data_ptr() if with_addend else None, ld, dst.data_ptr(), ld, width,
                                   _st()), "gather_add")
  torch.cuda.synchronize()
  assert _sentinels_intact(dst, 1, n, n, width)
  want = srcv[idx[:n].long()]
  if with_addend:
    want = addv[:n] + want
  assert torch.equal(dst[:n, :width], want)
