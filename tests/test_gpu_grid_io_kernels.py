"""The kernels on the grid boundary of the step against float64 references of the same operations, through
the C ABI, on seeded device data: the input packing (gcb_pack_grid_features, gcb_pack_grid_image), the
output unpacking (gcb_unpack_grid_outputs), the fused loss reduction (gcb_output_loss), the five seeds of
the backward passes (gcb_output_loss_grad, gcb_output_loss_gn_seed, gcb_output_loss_grad_feedback,
gcb_output_loss_gn_seed_feedback, gcb_output_cotangent_grad_feedback) and the input-side transposes
(gcb_input_grad, gcb_broadcast_grad_sum).

The conventions are those of test_gpu_backward_kernels.py.  References are formed on the device from the
values each kernel read.  Every output buffer carries NaN sentinels (a row before, a row after, padding
columns up to ld); images carry a 0xA5 byte tail on a 0xFF prefill.  Inputs hold NaN where a kernel must
not read (y's columns >= n_out, a row behind every plane stack).  Every kernel runs twice (same bits) and
once more into a 0xFF-prefilled buffer: it must give the same bits on every element it owns and keep the
prefill everywhere else.  Each matrix varies one axis against a base case.

u = 2^-24, u53 = 2^-53.  Each bound is derived in the docstring of the test that uses it, and each case
prints its largest error / bound ratio.  Bit equality is asserted where the header promises it, or where
the kernel evaluates the reference's fp32 IEEE operations in the same order (the build uses no fast-math,
so its divisions are correctly rounded, as torch's are).  The refusals of these entry points are in
test_native_abi.py and test_gpu_loss.py."""
import numpy as np
import pytest
import torch

from graphcast_b200 import _native
from test_gpu_backward_kernels import _check, _ids, _padded, _sentinels_intact
from test_gpu_layer import _image_values
from test_gpu_loss import _lat_weight

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
U = 2.0 ** -24                        # fp32 unit roundoff
U53 = 2.0 ** -53                      # fp64 unit roundoff
NAN = float("nan")
TAIL = 64                             # 0xA5 bytes behind every image
K_LOSS_GROUPS = 512                   # kLossGroups of aux_kernels.cuh

# n_lat x n_lon; "np": latitude rows at +-(90 - d/2), otherwise rows at the poles.  128 x 128 is exactly
# 512 loss tiles of 32 nodes (one per group), 5 x 3277 is 513 (one group gets a second, one-node tile);
# 721 x 1440 is 0.25 degree (32 445 tiles: 63 or 64 per group).
BIG = "721x1440"
GRIDS = ("1x1", "1x31", "1x33", "2x64", "3x43np", "19x37np", "128x128np", "5x3277", "181x360", BIG)
NODES = (1, 31, 33, 128, 129, 16_384, 16_385, 65_160, 1_038_240)
# (n_out, ld_y = ld_g); the base case is (83, 256).  Scalar loads: odd strides are legal.
SHAPES = ((1, 1), (31, 31), (32, 32), (33, 37), (227, 256), (227, 227), (256, 256))
AFFINE = tuple((s, o, a) for s in (0, 1) for o in (0, 1) for a in (0, 1) if (s, o, a) != (1, 1, 1))
ROWS = (0, 1, 31, 32, 33, 454)


def _st():
  return torch.cuda.current_stream().cuda_stream


def _gen(seed):
  return torch.Generator(device=DEV).manual_seed(seed)


def _ptr(t):
  return None if t is None else t.data_ptr()


def _bits(t):
  return t.contiguous().view(torch.int64 if t.element_size() == 8 else torch.int32)


def _case(base, axis, value):
  case = dict(base)
  names = axis.split(",")
  case.update(zip(names, value if len(names) > 1 else (value,)))
  return case


def _tag(name, case):
  return name + " " + " ".join(f"{k}={v}" for k, v in case.items())


def _need_memory(n_nodes):
  if n_nodes > 500_000 and torch.cuda.get_device_properties(0).total_memory < 75e9:
    pytest.skip("needs an 80 GB GPU")


# ---- buffers -------------------------------------------------------------------------------------------
def _framed(rows, n, ld, values=None, ff=False):
  """[rows + 2, ld] fp32 with the data at [1:rows + 1, :n] (= values when given) and NaN everywhere else:
  a row before, a row after and the padding columns.  ff: every element 0xFFFFFFFF instead."""
  if ff:
    return torch.full((rows + 2, ld), -1, dtype=torch.int32, device=DEV).view(torch.float32)
  t = _padded(rows + 1, n, ld)
  if values is not None:
    t[1:rows + 1, :n] = values
  return t


def _body(t, rows, n):
  return t[1:rows + 1, :n]


def _at(t):
  """Device address of the data of a _framed buffer."""
  return t[1:].data_ptr()


def _intact(t, rows, n):
  return bool(torch.isnan(t[0]).all()) and _sentinels_intact(t[1:], 1, rows, rows, n)


def _runs(tag, run, shapes):
  """run(*outputs) launches the kernel.  It runs into NaN-framed outputs twice and into 0xFF-prefilled
  ones once; shapes holds (rows, n, ld) of each fp32 output.  The sentinels must be intact, the two runs
  must give the same bits, and the 0xFF run must give them on every element the kernel owns and keep its
  prefill elsewhere.  Returns the first run's outputs."""
  outs = [[_framed(*s, ff=ff) for s in shapes] for ff in (False, False, True)]
  for o in outs:
    run(*o)
  torch.cuda.synchronize()
  for (rows, n, _), a, b, f in zip(shapes, *outs):
    assert _intact(a, rows, n) and _intact(b, rows, n), f"{tag}: a sentinel was written"
    assert torch.equal(_bits(a), _bits(b)), f"{tag}: two runs differ"
    assert torch.equal(_bits(_body(a, rows, n)), _bits(_body(f, rows, n))), \
        f"{tag}: the output depends on what the buffer held"
    rest = _bits(f).clone()
    rest[1:rows + 1, :n] = -1
    assert bool((rest == -1).all()), f"{tag}: an element outside the output was written"
  return outs[0]


def _same_bits(tag, got, want):
  assert torch.equal(_bits(got), _bits(want)), f"{tag}: not bit for bit the reference"
  print(f"{tag}: max error / bound 0 (bit for bit)")


def _cmp(tag, got, want, bound):
  """_check where the reference is finite; got must be NaN exactly where the reference is."""
  nan = torch.isnan(want)
  assert torch.equal(torch.isnan(got), nan), f"{tag}: NaN pattern differs from the reference"
  _check(tag, torch.where(nan, 0.0, (got.double() - want).abs()), torch.where(nan, 1.0, bound))


def _pairwise_sum(x):
  """Sum over the last dimension of fp64 x by repeated halving, and the number of halvings L: each level
  rounds every partial once, so the error is at most L u53 sum |x|."""
  levels = 0
  while x.shape[-1] > 1:
    h = (x.shape[-1] + 1) // 2
    if x.shape[-1] % 2:
      x = torch.cat([x, x.new_zeros(x.shape[:-1] + (1,))], -1)
    x = x[..., :h] + x[..., h:]
    levels += 1
  return x[..., 0], levels


# ---- the output side: y, targets, affine ----------------------------------------------------------------
def _grid(name):
  """(n_lat, n_lon) of a GRIDS name, and its fp32 latitude weights on the device (mean 1)."""
  poles = not name.endswith("np")
  n_lat, n_lon = (int(v) for v in name.replace("np", "").split("x"))
  _need_memory(n_lat * n_lon)
  if n_lat == 1:
    w = np.ones(1, np.float32)
  elif poles:
    w = _lat_weight(np.linspace(-90.0, 90.0, n_lat))
  else:
    d = 180.0 / n_lat
    w = _lat_weight(np.linspace(-90.0 + d / 2, 90.0 - d / 2, n_lat))
  return n_lat, n_lon, torch.as_tensor(w).to(DEV)


class _Out:
  """Seeded data of the output side and the fp32 quantities the kernels form from it, computed with the
  same IEEE operations in the same order.

  y [n, ld] (NaN in the columns >= n_out and in the rows around it, y[0, 0] = -0), targets [n_out, n]
  with NaN behind them, n_out + 5 add planes, the add index with -1 entries, a repeated plane and the
  last plane, offset 0 on the residual channels (as InputsAndResiduals sets them).  scale / offset / add
  0 pass NULL.  Edges: 'cancel' targets and add planes 1e3 + N(0, 1), so t - add cancels; 'small_scale'
  / 'big_scale' scales near 1e-3 / 1e3; 'offset_on_add' offsets on the residual channels too, which the
  header allows and which fixes the order of the offset and the add; 'nan_target' one NaN target."""

  def __init__(self, grid, n_out, ld, scale=1, offset=1, add=1, edge="none", seed=0):
    self.n_lat, self.n_lon, self.w = _grid(grid)
    n = self.n = self.n_lat * self.n_lon
    self.n_out, self.ld = n_out, ld
    gen = self.gen = _gen(seed + 7 * n + 131 * n_out + ld)
    rnd = lambda *s: torch.randn(*s, generator=gen, device=DEV)
    self.yv = rnd(n, n_out)
    self.yv[0, 0] = -0.0
    self.y = _framed(n, n_out, ld, self.yv)
    n_planes = n_out + 5
    cancel = edge == "cancel"
    tv = 1e3 + rnd(n_out, n) if cancel else rnd(n_out, n) * 3 + 1
    if edge == "nan_target":
      tv[n_out // 2, n // 2] = NAN
    planes = rnd(n_planes, n) + (1e3 if cancel else 0.0)
    self.targets = _padded(n_out, n, n, tv)
    self.planes = _padded(n_planes, n, n, planes)
    sc = (torch.rand(n_out, generator=gen, device=DEV) + 0.5) * {"small_scale": 1e-3,
                                                                 "big_scale": 1e3}.get(edge, 1.0)
    idx = torch.randint(0, n_planes, (n_out,), generator=gen, device=DEV, dtype=torch.int32)
    idx[::3] = -1                                    # targets that are not inputs
    idx[-1] = n_planes - 1                           # the last plane ...
    if n_out >= 3:
      idx[1] = n_planes - 1                          # ... twice
    of = rnd(n_out)
    if edge != "offset_on_add":
      of[idx >= 0] = 0
    self.coef = torch.rand(n_out, generator=gen, device=DEV, dtype=torch.float64) + 0.1
    self.scale, self.offset = (sc if scale else None), (of if offset else None)
    self.idx = idx if add else None
    self.wn = self.w.double().repeat_interleave(self.n_lon)          # [n] the weight of each node
    self.s64 = sc.double() if scale else torch.ones(n_out, dtype=torch.float64, device=DEV)
    has = (idx >= 0)[:, None]
    av = torch.where(has, planes[idx.clamp(min=0).long()], 0.0) if add else torch.zeros_like(tv)
    t_norm = ((tv - av) - (of if offset else torch.zeros_like(of))[:, None]) / \
        (sc if scale else torch.ones_like(sc))[:, None]
    self.d = self.yv.t() - t_norm                    # [n_out, n]: y - t_norm, rounded as the kernels do
    pred = self.yv.t()
    if scale:
      pred = pred * sc[:, None]
    if offset:
      pred = pred + of[:, None]
    if add:
      pred = torch.where(has, pred + av, pred)
    self.pred = pred                                 # [n_out, n]: the unpacked predictions

  def affine(self):
    return (_ptr(self.scale), _ptr(self.offset), _ptr(self.planes if self.idx is not None else None),
            _ptr(self.idx))

  def gl64(self, d):
    """coef[c] * w[node] * d in fp64, in the kernels' order ((coef w) d), [n_out, n]."""
    return (self.coef[:, None] * self.wn[None]) * d.double()


class _Rows:
  """The feedback rows: a_next [n_rows + 4, n] (or NULL), dpred_row / resid_channel / carry_row with -1
  entries and repeats (row 0 has resid = carry = -1), carry_row NULL when carry == 'null'."""

  def __init__(self, o, n_rows, a_next, carry):
    gen, n_out = o.gen, o.n_out
    n_next = n_rows + 4
    self.n_rows, self.n = n_rows, o.n
    self.a_next = _padded(n_next, o.n, o.n, torch.randn(n_next, o.n, generator=gen, device=DEV)) \
        if a_next else None
    ri = lambda hi, size: torch.randint(0, hi, (size,), generator=gen, device=DEV, dtype=torch.int32)
    self.dpred = ri(n_next, n_out)
    self.dpred[::4] = -1
    self.dpred[-1] = n_next - 1
    if n_out >= 3:
      self.dpred[1] = n_next - 1
    self.resid = ri(n_out, max(n_rows, 1))
    self.resid[::3] = -1
    if n_rows >= 3:
      self.resid[1] = self.resid[2] = n_out - 1
    self.carry = None
    if carry != "null":
      self.carry = ri(n_next, max(n_rows, 1))
      self.carry[::5] = -1

  def dp64(self, n_out):
    """a_next[dpred_row[c]] in fp64 (0 where there is none), [n_out, n]."""
    dp = torch.zeros(n_out, self.n, dtype=torch.float64, device=DEV)
    if self.a_next is not None:
      ok = self.dpred >= 0
      dp[ok] = self.a_next[self.dpred[ok].long()].double()
    return dp

  def carry64(self):
    """a_next[carry_row[r]] in fp64 where the carry applies, 0 elsewhere, and where it applies."""
    k = torch.zeros(self.n_rows, self.n, dtype=torch.float64, device=DEV)
    on = torch.zeros(self.n_rows, dtype=torch.bool, device=DEV)
    if self.a_next is not None and self.carry is not None:
      on = self.carry[:self.n_rows] >= 0
      k[on] = self.a_next[self.carry[:self.n_rows][on].long()].double()
    return k, on

  def args(self):
    return (_ptr(self.a_next), self.dpred.data_ptr(), self.n_rows, self.resid.data_ptr(), _ptr(self.carry))


def _check_rows(tag, a, r, x, mx):
  """a_out against fp64: row r = x[resid[r]] (0 when resid[r] < 0) + the carry k.  x is the kernel's
  fp64 value before its fp32 rounding, mx the sum of the magnitudes of its terms.  The kernel rounds x
  to fp32 and adds k in fp32; with e the fp64 error of x (kernel and reference) and a64 = x + k:
    |a - a64| <= e + u |x| + u |a64| + O(u^2) <= (2 + 2^-20) u (|a64| + |k|) + 2e,
  using |x| <= |a64| + |k|.  Rows with resid < 0 and no carry must be exactly +0."""
  if r.n_rows == 0:
    return
  res = r.resid[:r.n_rows].long()
  on = (res >= 0)[:, None]
  k, carried = r.carry64()
  want = torch.where(on, x[res.clamp(min=0)], 0.0) + k
  mag = torch.where(on, mx[res.clamp(min=0)], 0.0) + k.abs()
  got = _body(a, r.n_rows, r.n)
  _cmp(tag + " a_out", got, want, (2 + 2.0 ** -20) * U * (want.abs() + k.abs()) + 2.0 ** -47 * mag + 1e-300)
  zero = (res < 0) & ~carried
  assert bool((_bits(got[zero]) == 0).all()), f"{tag}: a row without residual or carry is not +0"


OUT_BASE = dict(grid="19x37", n_out=83, ld=256, scale=1, offset=1, add=1, edge="none")
OUT_AXES = ([("grid", g) for g in GRIDS] + [("n_out,ld", s) for s in SHAPES]
            + [("scale,offset,add", a) for a in AFFINE])
EDGES = ("cancel", "small_scale", "big_scale", "offset_on_add", "nan_target")


# ---- unpack and loss -------------------------------------------------------------------------------------
def _unpack(lib, o, out):
  _native.check(lib.gcb_unpack_grid_outputs(_at(o.y), o.ld, o.n_out, o.n, *o.affine(), out, _st()),
                "gcb_unpack_grid_outputs")


@pytest.mark.parametrize("axis,value", OUT_AXES + [("edge", e) for e in EDGES[:-1]], ids=_ids)
def test_unpack_grid_outputs_matrix(axis, value):
  """gcb_unpack_grid_outputs is bit for bit ((y * scale) + offset) + add in that order, each term only
  when given (the add only where add_plane_index >= 0): its sm_90a SASS has one FMUL and FADDs and no
  FFMA, so nothing is contracted.  planes_out is NaN-framed [n_out, n]."""
  case = _case(OUT_BASE, axis, value)
  tag = _tag("unpack", case)
  o = _Out(**case)
  lib = _native.lib()
  (p,) = _runs(tag, lambda p: _unpack(lib, o, _at(p)), [(o.n_out, o.n, o.n)])
  _same_bits(tag, _body(p, o.n_out, o.n), o.pred)


@pytest.mark.parametrize("axis,value", OUT_AXES + [("edge", e) for e in EDGES], ids=_ids)
def test_output_loss_matrix(axis, value):
  """gcb_output_loss: the channel sums against S = sum over nodes of w d^2 in fp64, with d = y - t_norm
  formed by torch in the kernel's order (((t - add) - offset) / scale, then y - t_norm).  d^2 is exact in
  fp64 and each term carries at most one rounding (the kernel's DFMA into its accumulator).  A thread adds
  m = ceil(n_tiles / 512) terms, then 5 butterfly steps, then the 512 group partials are added in
  sequence; the reference halves L = ceil(log2 n) times:  |S_gpu - S| <= (m + 520 + L) u53 S.  An fp32
  accumulator lands orders of magnitude outside this bound, and so does a dropped group on grids of 512
  tiles or more.  The workspace is NaN-prefilled, so every group must write its partials.

  planes_out must be gcb_unpack_grid_outputs bit for bit, and the sums must not depend on planes_out or
  on what the sums buffer held; a NaN target makes exactly its channel's sum NaN."""
  case = _case(OUT_BASE, axis, value)
  tag = _tag("loss", case)
  o = _Out(**case)
  lib = _native.lib()
  nbytes = lib.gcb_output_loss_workspace_bytes(o.n_out)

  def run(with_po, ff):
    sums = torch.full((o.n_out + 2,), -1 if ff else NAN, dtype=torch.int64 if ff else torch.float64,
                      device=DEV).view(torch.float64)
    ws = torch.full((nbytes // 8,), NAN, dtype=torch.float64, device=DEV)
    po = _framed(o.n_out, o.n, o.n, ff=ff) if with_po else None
    _native.check(lib.gcb_output_loss(
        _at(o.y), o.ld, o.n_out, o.n_lat, o.n_lon, *o.affine(), o.targets.data_ptr(), o.w.data_ptr(),
        _at(po) if with_po else None, ws.data_ptr(), nbytes, sums[1:].data_ptr(), _st()), "gcb_output_loss")
    return sums, po

  (s1, p1), (s2, p2), (s3, _), (s4, p4) = run(True, False), run(True, False), run(False, False), run(True, True)
  unpacked = _framed(o.n_out, o.n, o.n)
  _unpack(lib, o, _at(unpacked))
  torch.cuda.synchronize()
  for s in (s1, s2, s3):
    assert bool(torch.isnan(s[0]) and torch.isnan(s[-1])), f"{tag}: a sentinel of the sums was written"
  assert int(_bits(s4)[0]) == -1 and int(_bits(s4)[-1]) == -1, f"{tag}: a sentinel of the sums was written"
  for s in (s2, s3, s4):
    assert torch.equal(_bits(s[1:-1]), _bits(s1[1:-1])), f"{tag}: the sums differ between runs"
  assert _intact(p1, o.n_out, o.n) and torch.equal(_bits(p1), _bits(p2)), tag
  assert torch.equal(_bits(_body(p4, o.n_out, o.n)), _bits(_body(p1, o.n_out, o.n))), tag
  assert torch.equal(_bits(p1), _bits(unpacked)), f"{tag}: planes_out is not gcb_unpack_grid_outputs"
  _same_bits(tag + " planes_out", _body(p1, o.n_out, o.n), o.pred)
  d64 = o.d.double()
  sums, levels = _pairwise_sum(o.wn[None] * d64 * d64)
  tiles = -(-o.n // 32)
  m = -(-tiles // K_LOSS_GROUPS)
  _cmp(tag, s1[1:-1], sums, (m + 520 + levels) * U53 * sums.abs() + 1e-300)


# ---- seeds ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("axis,value", OUT_AXES + [("edge", e) for e in EDGES], ids=_ids)
def test_output_loss_grad_matrix(axis, value):
  """gcb_output_loss_grad against g64 = coef w d in fp64 from the kernel's fp32 d.  The kernel rounds
  twice in fp64 and once to fp32, the reference twice in fp64: |g - g64| <= u |g64| + 2^-49 |coef w d|.
  g is NaN-framed at ld_g = ld_y; its columns >= n_out are not written.  A NaN target makes exactly its
  own element NaN."""
  case = _case(OUT_BASE, axis, value)
  tag = _tag("loss_grad", case)
  o = _Out(**case)
  lib = _native.lib()
  run = lambda g: _native.check(lib.gcb_output_loss_grad(
      _at(o.y), o.ld, o.n_out, o.n_lat, o.n_lon, *o.affine(), o.targets.data_ptr(), o.w.data_ptr(),
      o.coef.data_ptr(), _at(g), o.ld, _st()), "gcb_output_loss_grad")
  (g,) = _runs(tag, run, [(o.n, o.n_out, o.ld)])
  g64 = o.gl64(o.d)
  _cmp(tag, _body(g, o.n, o.n_out).t(), g64, U * g64.abs() + 2.0 ** -49 * g64.abs() + 1e-300)


GN_AXES = [("grid", g) for g in GRIDS] + [("n_out,ld", s) for s in SHAPES]


@pytest.mark.parametrize("axis,value", GN_AXES, ids=_ids)
def test_output_loss_gn_seed_matrix(axis, value):
  """gcb_output_loss_gn_seed is bit for bit gcb_output_loss_grad with y = dy, all-zero targets and NULL
  scale, offset and add planes, NaN padding columns included (dy[0, 0] = -0).  Against fp64 g64 =
  coef w dy: |g - g64| <= u |g64| + 2^-49 |g64| (two fp64 roundings on either side, one fp32)."""
  case = _case(OUT_BASE, axis, value)
  tag = _tag("gn_seed", case)
  o = _Out(**case)
  lib = _native.lib()
  run = lambda g: _native.check(lib.gcb_output_loss_gn_seed(
      _at(o.y), o.ld, o.n_out, o.n_lat, o.n_lon, o.w.data_ptr(), o.coef.data_ptr(), _at(g), o.ld, _st()),
      "gcb_output_loss_gn_seed")
  (g,) = _runs(tag, run, [(o.n, o.n_out, o.ld)])
  zeros = torch.zeros(o.n_out, o.n, device=DEV)
  want = _framed(o.n, o.n_out, o.ld)
  _native.check(lib.gcb_output_loss_grad(
      _at(o.y), o.ld, o.n_out, o.n_lat, o.n_lon, None, None, None, None, zeros.data_ptr(), o.w.data_ptr(),
      o.coef.data_ptr(), _at(want), o.ld, _st()), "gcb_output_loss_grad")
  torch.cuda.synchronize()
  assert torch.equal(_bits(g), _bits(want)), f"{tag}: not gcb_output_loss_grad with zero targets"
  g64 = o.gl64(o.yv.t())
  _cmp(tag, _body(g, o.n, o.n_out).t(), g64, U * g64.abs() + 2.0 ** -49 * g64.abs() + 1e-300)


FB_BASE = dict(OUT_BASE, rows=70, a_next=1, carry="given")
FB_AXES = ([("rows", r) for r in ROWS] + [("a_next", 0), ("carry", "null"), ("a_next,rows", (0, 0))])


@pytest.mark.parametrize("axis,value", OUT_AXES + FB_AXES + [("edge", e) for e in EDGES], ids=_ids)
def test_output_loss_grad_feedback_matrix(axis, value):
  """gcb_output_loss_grad_feedback against fp64, with gl = coef w d from the kernel's fp32 d and dp =
  a_next[dpred_row[c]]:
    g64 = gl + scale dp: scale dp is exact in fp64; the kernel rounds three times in fp64 (possibly fused)
      and once to fp32, the reference three times: |g - g64| <= u |g64| + 2^-49 (|gl| + |scale dp|).
    a_out rows: x = gl / scale + dp (four fp64 roundings in the kernel, as many in the reference, so
      e <= 2^-48 (|gl / scale| + |dp|)), rounded to fp32, plus the carry in fp32: _check_rows.
  With a_next = NULL, g must be gcb_output_loss_grad bit for bit (the same rows passed)."""
  case = _case(FB_BASE, axis, value)
  tag = _tag("grad_feedback", case)
  rows, a_next, carry = case.pop("rows"), case.pop("a_next"), case.pop("carry")
  o = _Out(**case)
  r = _Rows(o, rows, a_next, carry)
  lib = _native.lib()

  def launch(rw, g, a):
    _native.check(lib.gcb_output_loss_grad_feedback(
        _at(o.y), o.ld, o.n_out, o.n_lat, o.n_lon, *o.affine(), o.targets.data_ptr(), o.w.data_ptr(),
        o.coef.data_ptr(), *rw, _at(a), _at(g), o.ld, _st()), "gcb_output_loss_grad_feedback")

  g, a = _runs(tag, lambda g, a: launch(r.args(), g, a), [(o.n, o.n_out, o.ld), (rows, o.n, o.n)])
  gl = o.gl64(o.d)
  dp = r.dp64(o.n_out)
  sdp = o.s64[:, None] * dp
  g64 = gl + sdp
  _cmp(tag + " g", _body(g, o.n, o.n_out).t(), g64,
       U * g64.abs() + 2.0 ** -49 * (gl.abs() + sdp.abs()) + 1e-300)
  x = gl / o.s64[:, None]
  _check_rows(tag, a, r, x + dp, x.abs() + dp.abs())
  # without the following step, g is gcb_output_loss_grad
  g_null, a_null, g_plain = _framed(o.n, o.n_out, o.ld), _framed(rows, o.n, o.n), _framed(o.n, o.n_out, o.ld)
  launch((None,) + r.args()[1:], g_null, a_null)
  _native.check(lib.gcb_output_loss_grad(
      _at(o.y), o.ld, o.n_out, o.n_lat, o.n_lon, *o.affine(), o.targets.data_ptr(), o.w.data_ptr(),
      o.coef.data_ptr(), _at(g_plain), o.ld, _st()), "gcb_output_loss_grad")
  torch.cuda.synchronize()
  assert torch.equal(_bits(g_null), _bits(g_plain)), f"{tag}: a_next = NULL is not gcb_output_loss_grad"


GNFB_BASE = dict(grid="19x37", n_out=83, ld=256, scale=1, edge="none", rows=70, a_next=1, carry="given")
GNFB_AXES = (GN_AXES + [("scale", 0)] + FB_AXES + [("edge", e) for e in ("small_scale", "big_scale")])


@pytest.mark.parametrize("axis,value", GNFB_AXES, ids=_ids)
def test_output_loss_gn_seed_feedback_matrix(axis, value):
  """gcb_output_loss_gn_seed_feedback against fp64, d = pdot / scale formed by torch (one fp32 division,
  the kernel's), gl = coef w d, dp = a_next[dpred_row[c]]: g and a_out with the bounds of
  test_output_loss_grad_feedback_matrix.  pdot [n_out, n] is channel-major with a NaN row behind it.
  Bit for bit, as the header promises: with scale NULL, g and a_out are gcb_output_loss_grad_feedback
  with y = pdot^T, zero targets and no offset or add planes (the same rows); with no a_next and n_rows =
  0 too, g is gcb_output_loss_gn_seed on dy = pdot^T."""
  case = _case(GNFB_BASE, axis, value)
  tag = _tag("gn_seed_feedback", case)
  rows, a_next, carry, scale = case.pop("rows"), case.pop("a_next"), case.pop("carry"), case.pop("scale")
  o = _Out(**case, scale=scale, offset=0, add=0)
  r = _Rows(o, rows, a_next, carry)
  pdot = _padded(o.n_out, o.n, o.n, o.yv.t())            # y = pdot^T at ld
  lib = _native.lib()

  def launch(sc, rw, g, a):
    _native.check(lib.gcb_output_loss_gn_seed_feedback(
        pdot.data_ptr(), o.n_out, o.n_lat, o.n_lon, _ptr(sc), o.w.data_ptr(), o.coef.data_ptr(), *rw,
        _at(a), _at(g), o.ld, _st()), "gcb_output_loss_gn_seed_feedback")

  g, a = _runs(tag, lambda g, a: launch(o.scale, r.args(), g, a), [(o.n, o.n_out, o.ld), (rows, o.n, o.n)])
  d = o.yv.t() / o.scale[:, None] if scale else o.yv.t()
  gl = o.gl64(d)
  dp = r.dp64(o.n_out)
  sdp = o.s64[:, None] * dp
  g64 = gl + sdp
  _cmp(tag + " g", _body(g, o.n, o.n_out).t(), g64,
       U * g64.abs() + 2.0 ** -49 * (gl.abs() + sdp.abs()) + 1e-300)
  x = gl / o.s64[:, None]
  _check_rows(tag, a, r, x + dp, x.abs() + dp.abs())
  # the identities of the header
  zeros = torch.zeros(o.n_out, o.n, device=DEV)
  bufs = [_framed(o.n, o.n_out, o.ld), _framed(rows, o.n, o.n), _framed(o.n, o.n_out, o.ld),
          _framed(rows, o.n, o.n)]
  launch(None, r.args(), bufs[0], bufs[1])
  _native.check(lib.gcb_output_loss_grad_feedback(
      _at(o.y), o.ld, o.n_out, o.n_lat, o.n_lon, None, None, None, None, zeros.data_ptr(), o.w.data_ptr(),
      o.coef.data_ptr(), *r.args(), _at(bufs[3]), _at(bufs[2]), o.ld, _st()), "gcb_output_loss_grad_feedback")
  g0, gn = _framed(o.n, o.n_out, o.ld), _framed(o.n, o.n_out, o.ld)
  launch(None, (None, r.dpred.data_ptr(), 0, r.resid.data_ptr(), _ptr(r.carry)), g0, _framed(0, o.n, o.n))
  _native.check(lib.gcb_output_loss_gn_seed(_at(o.y), o.ld, o.n_out, o.n_lat, o.n_lon, o.w.data_ptr(),
                                            o.coef.data_ptr(), _at(gn), o.ld, _st()), "gcb_output_loss_gn_seed")
  torch.cuda.synchronize()
  assert torch.equal(_bits(bufs[0]), _bits(bufs[2])), f"{tag}: g is not the feedback seed's with scale NULL"
  assert torch.equal(_bits(bufs[1]), _bits(bufs[3])), f"{tag}: a_out is not the feedback seed's"
  assert torch.equal(_bits(g0), _bits(gn)), f"{tag}: without feedback g is not gcb_output_loss_gn_seed"


@pytest.mark.parametrize("axis,value", GNFB_AXES, ids=_ids)
def test_output_cotangent_grad_feedback_matrix(axis, value):
  """gcb_output_cotangent_grad_feedback against fp64: d = cot + dp (dp = a_next[dpred_row[c]]; one fp64
  rounding at most), g64 = scale d (one more, then fp32): |g - g64| <= u |g64| + 2^-49 |scale| (|cot| +
  |dp|).  a_out rows: x = d rounded to fp32, plus the carry in fp32: _check_rows.  cot [n_out, n] has a
  NaN row behind it."""
  case = _case(GNFB_BASE, axis, value)
  tag = _tag("cotangent_seed", case)
  rows, a_next, carry, scale = case.pop("rows"), case.pop("a_next"), case.pop("carry"), case.pop("scale")
  o = _Out(**case, scale=scale, offset=0, add=0)
  r = _Rows(o, rows, a_next, carry)
  cotv = torch.randn(o.n_out, o.n, generator=o.gen, device=DEV)
  cot = _padded(o.n_out, o.n, o.n, cotv)
  lib = _native.lib()
  run = lambda g, a: _native.check(lib.gcb_output_cotangent_grad_feedback(
      o.n_out, o.n, _ptr(o.scale), cot.data_ptr(), *r.args(), _at(a), _at(g), o.ld, _st()),
      "gcb_output_cotangent_grad_feedback")
  g, a = _runs(tag, run, [(o.n, o.n_out, o.ld), (rows, o.n, o.n)])
  dp = r.dp64(o.n_out)
  d = cotv.double() + dp
  g64 = o.s64[:, None] * d
  _cmp(tag + " g", _body(g, o.n, o.n_out).t(), g64,
       U * g64.abs() + 2.0 ** -49 * o.s64[:, None] * (cotv.double().abs() + dp.abs()) + 1e-300)
  _check_rows(tag, a, r, d, cotv.double().abs() + dp.abs())


# ---- the input side ------------------------------------------------------------------------------------
class _Pack:
  """Input planes [n_ch, n] (a NaN plane behind them), node_static [n, n_static] (a NaN row behind it),
  mean / scale (0 passes NULL), and the packed features [n, k] as two separate torch ops compute them:
  (planes - mean) / scale, the static columns copied, +0 up to k.  Edges: 'cancel' planes and mean near
  1e3; 'small_scale' / 'big_scale' scales near 1e-3 / 1e3."""

  def __init__(self, nodes, ch, mean, scale, edge, seed=0):
    _need_memory(nodes)
    self.n = n = nodes
    self.n_ch, self.n_static, self.k = ch
    gen = _gen(seed + n + 7 * self.k)
    rnd = lambda *s: torch.randn(*s, generator=gen, device=DEV)
    base = 1e3 if edge == "cancel" else 0.0
    pv = rnd(self.n_ch, n) + base
    self.planes = _padded(self.n_ch, n, n, pv)
    sv = rnd(n, self.n_static)
    self.static = _padded(n, self.n_static, self.n_static, sv) if self.n_static else None
    self.mean = rnd(self.n_ch) + base if mean else None
    self.scale = ((torch.rand(self.n_ch, generator=gen, device=DEV) + 0.5)
                  * {"small_scale": 1e-3, "big_scale": 1e3}.get(edge, 1.0)) if scale else None
    x = pv
    if mean:
      x = x - self.mean[:, None]
    if scale:
      x = x / self.scale[:, None]
    self.want = torch.zeros(n, self.k, device=DEV)
    self.want[:, :self.n_ch] = x.t()
    self.want[:, self.n_ch:self.n_ch + self.n_static] = sv

  def args(self):
    return (self.planes.data_ptr(), self.n_ch, self.n, _ptr(self.mean), _ptr(self.scale), _ptr(self.static),
            self.n_static)


PACK_BASE = dict(nodes=19 * 37, ch=(471, 3, 480), mean=1, scale=1, edge="none")
PACK_AXES = ([("nodes", n) for n in NODES] + [("ch", c) for c in ((183, 3, 192), (1, 0, 16), (13, 3, 16),
                                                                   (740, 3, 752))]
             + [("mean,scale", m) for m in ((0, 0), (0, 1), (1, 0))]
             + [("edge", e) for e in ("cancel", "small_scale", "big_scale")])


@pytest.mark.parametrize("axis,value", PACK_AXES, ids=_ids)
def test_pack_grid_features_matrix(axis, value):
  """gcb_pack_grid_features at ld = k (k = 752 is the largest k under the image's 96 KB shared-memory
  cap) is bit for bit (planes - mean) / scale as two torch ops (no fast-math: the SASS division is the
  IEEE sequence), the static columns copied, and +0 in every column up to ld; NaN-framed output."""
  case = _case(PACK_BASE, axis, value)
  tag = _tag("pack_features", case)
  p = _Pack(**case)
  lib = _native.lib()
  run = lambda f: _native.check(lib.gcb_pack_grid_features(*p.args(), _at(f), p.k, _st()),
                                "gcb_pack_grid_features")
  (f,) = _runs(tag, run, [(p.n, p.k, p.k)])
  _same_bits(tag, _body(f, p.n, p.k), p.want)


@pytest.mark.parametrize("axis,value", PACK_AXES, ids=_ids)
def test_pack_grid_image_matrix(axis, value):
  """gcb_pack_grid_image is byte for byte gcb_rows_to_image of gcb_pack_grid_features packed at ld = k,
  pad rows of the last 128-row tile included: on a 0xFF-prefilled buffer they must be zero bytes.  A
  second run gives the same bytes, a zero-prefilled buffer the same bytes everywhere but in the 64-byte
  skews of the layout, which no kernel writes; the 0xA5 tail stays.  Decoded, hi + lo is within
  2^-17 |v| of the feature v (two bf16 roundings of 2^-9 each)."""
  case = _case(PACK_BASE, axis, value)
  tag = _tag("pack_image", case)
  p = _Pack(**case)
  lib = _native.lib()
  n, k = p.n, p.k
  feats = torch.full((n, k), NAN, device=DEV)
  _native.check(lib.gcb_pack_grid_features(*p.args(), feats.data_ptr(), k, _st()), "gcb_pack_grid_features")
  nbytes = lib.gcb_a_image_bytes(n, k)

  def image(fill):
    t = torch.full((nbytes + TAIL,), fill, dtype=torch.uint8, device=DEV)
    t[nbytes:] = 0xA5
    return t

  imgs = [image(0xFF), image(0xFF), image(0)]
  for img in imgs:
    _native.check(lib.gcb_pack_grid_image(*p.args(), k, img.data_ptr(), _st()), "gcb_pack_grid_image")
  ref = image(0xFF)
  _native.check(lib.gcb_rows_to_image(feats.data_ptr(), k, 1, n, k, ref.data_ptr(), _st()), "gcb_rows_to_image")
  torch.cuda.synchronize()
  assert torch.equal(_bits(feats), _bits(p.want)), f"{tag}: the features are not the reference"
  img = imgs[0]
  assert torch.equal(img, imgs[1]), f"{tag}: two runs differ"
  assert torch.equal(img, ref), f"{tag}: not gcb_rows_to_image of gcb_pack_grid_features"
  for t in imgs:
    assert bool((t[nbytes:] == 0xA5).all()), f"{tag}: the tail was written"
  blocks = lambda t: t[:nbytes].view(-1, k // 16, 2, 2, 2112)     # tile, K-step, hi|lo, chunk
  assert torch.equal(blocks(img)[..., :2048], blocks(imgs[2])[..., :2048]), \
      f"{tag}: the image depends on what the buffer held"
  assert bool((blocks(img)[..., 2048:] == 0xFF).all()) and bool((blocks(imgs[2])[..., 2048:] == 0).all()), \
      f"{tag}: a skew byte was written"
  rows = blocks(img)[..., :2048].reshape(-1, k // 16, 2, 2, 128, 16).permute(0, 4, 1, 2, 3, 5)
  rows = rows.reshape(-1, (k // 16) * 2 * 2 * 16)
  assert bool((rows[n:] == 0).all()), f"{tag}: a pad row of the last tile is not zero"
  v = feats.double()
  _check(tag, (_image_values(img[:nbytes], n, k).double() - v).abs(), 2.0 ** -17 * v.abs() + 1e-38)


IN_BASE = dict(nodes=19 * 37, ld=480, rows=471, scale=1, acc=0, edge="none")
IN_AXES = ([("nodes", n) for n in NODES] + [("ld", v) for v in (192, 77)] + [("rows", v) for v in (1, 31, 33)]
           + [("scale", 0), ("acc", 1), ("acc,scale", (1, 0)), ("acc,nodes", (1, 16_385))]
           + [("edge", e) for e in ("small_scale", "big_scale")])


@pytest.mark.parametrize("axis,value", IN_AXES, ids=_ids)
def test_input_grad_matrix(axis, value):
  """gcb_input_grad is bit for bit a + dx[:, ch] / scale[ch] in fp32 (torch's division and addition are
  the kernel's __fdiv_rn and __fadd_rn), with repeated channels and the last column of dx, dx NaN-framed.
  accumulate = 0 overwrites a NaN prefill (and a 0xFF one, with the same bits); accumulate = 1 adds onto
  a random base."""
  case = _case(IN_BASE, axis, value)
  tag = _tag("input_grad", case)
  n, ld, rows = case["nodes"], case["ld"], case["rows"]
  _need_memory(n)
  gen = _gen(n + ld + rows)
  dxv = torch.randn(n, ld, generator=gen, device=DEV)
  dx = _framed(n, ld, ld, dxv)
  ch = torch.randint(0, ld, (rows,), generator=gen, device=DEV, dtype=torch.int32)
  ch[0] = ld - 1
  if rows >= 3:
    ch[2] = ch[1]
  scale = (torch.rand(ld, generator=gen, device=DEV) + 0.3) * {"small_scale": 1e-3,
                                                               "big_scale": 1e3}.get(case["edge"], 1.0)
  sc = scale if case["scale"] else None
  term = dxv[:, ch.long()].t()
  if sc is not None:
    term = term / scale[ch.long()][:, None]
  lib = _native.lib()
  launch = lambda a, acc: _native.check(lib.gcb_input_grad(
      _at(dx), ld, n, rows, ch.data_ptr(), _ptr(sc), _at(a), acc, _st()), "gcb_input_grad")
  if not case["acc"]:
    (a,) = _runs(tag, lambda a: launch(a, 0), [(rows, n, n)])
    _same_bits(tag, _body(a, rows, n), term)
    return
  base = torch.randn(rows, n, generator=gen, device=DEV)
  a1, a2 = _framed(rows, n, n, base), _framed(rows, n, n, base)
  launch(a1, 1)
  launch(a2, 1)
  torch.cuda.synchronize()
  assert _intact(a1, rows, n) and torch.equal(_bits(a1), _bits(a2)), tag
  _same_bits(tag, _body(a1, rows, n), base + term)


BC_BASE = dict(grid="181x360", mode=2, rows="repeated", acc=0, edge="none")
BC_AXES = ([("mode", m) for m in (0, 1)]
           + [("grid,mode", (g, m)) for g in ("1x33", "37x1", BIG) for m in (0, 1, 2)]
           + [("rows,mode", ("none", m)) for m in (0, 1, 2)] + [("acc,mode", (1, m)) for m in (0, 1, 2)]
           + [("edge,mode", ("offset", m)) for m in (1, 2)])


@pytest.mark.parametrize("axis,value", BC_AXES, ids=_ids)
def test_broadcast_grad_sum_matrix(axis, value):
  """gcb_broadcast_grad_sum in its three modes against fp64 sums of the planes a[rows[i]] (rows 7, 0, 3,
  3 and the last of 9 planes; a NaN plane behind them).  The kernel's fp64 sum is a chain of `chain`
  roundings: 0 for mode 0 (a copy), n_lat for mode 1, ceil(n / 256) + 8 for mode 2 (a thread's strided
  terms, then an 8-level tree); the reference halves L times (_pairwise_sum); the result is rounded once
  to fp32:  |out - sum64| <= u |sum64| + (chain + 1 + L) u53 sum |a|.  With accumulate the base enters
  the same fp64 sum (one more rounding) before the same fp32 rounding.  n_rows = 0 leaves out untouched.
  Edge 'offset': planes 1e3 + N(0, 1)."""
  case = _case(BC_BASE, axis, value)
  tag = _tag("broadcast", case)
  mode, acc = case["mode"], case["acc"]
  n_lat, n_lon = (int(v) for v in case["grid"].split("x"))
  n = n_lat * n_lon
  _need_memory(n)
  gen = _gen(n + 17 * mode + acc)
  n_planes = 9
  av = torch.randn(n_planes, n, generator=gen, device=DEV) + (1e3 if case["edge"] == "offset" else 0.0)
  a = _padded(n_planes, n, n, av)
  rows = [7, 0, 3, 3, n_planes - 1] if case["rows"] == "repeated" else []
  rows_d = torch.as_tensor(rows or [0], dtype=torch.int32, device=DEV)
  n_rows = len(rows)
  width = (n, n_lon, 1)[mode]
  lib = _native.lib()
  launch = lambda out, accumulate: _native.check(lib.gcb_broadcast_grad_sum(
      a.data_ptr(), n_lat, n_lon, n_rows, rows_d.data_ptr(), mode, _at(out), accumulate, _st()),
      "gcb_broadcast_grad_sum")
  base = torch.randn(max(n_rows, 1), width, generator=gen, device=DEV)
  if n_rows == 0:
    out = _framed(1, width, width, base)
    before = out.clone()
    launch(out, acc)
    torch.cuda.synchronize()
    _same_bits(tag, out, before)
    return
  if acc:
    o1, o2 = _framed(n_rows, width, width, base), _framed(n_rows, width, width, base)
    launch(o1, 1)
    launch(o2, 1)
    torch.cuda.synchronize()
    assert _intact(o1, n_rows, width) and torch.equal(_bits(o1), _bits(o2)), tag
    out = o1
  else:
    (out,) = _runs(tag, lambda o: launch(o, 0), [(n_rows, width, width)])
  x = av.double()[torch.as_tensor(rows, device=DEV)]
  if mode == 0:
    want, mag, chain, levels = x, x.abs(), 0, 0
  elif mode == 1:
    xt = x.view(n_rows, n_lat, n_lon).transpose(1, 2)
    (want, levels), (mag, _) = _pairwise_sum(xt), _pairwise_sum(xt.abs())
    chain = n_lat
  else:
    (want, levels), (mag, _) = _pairwise_sum(x), _pairwise_sum(x.abs())
    want, mag = want[:, None], mag[:, None]
    chain = -(-n // 256) + 8
  if acc:
    want, mag, chain = want + base.double(), mag + base.double().abs(), chain + 1
  _cmp(tag, _body(out, n_rows, width), want,
       U * want.abs() + (chain + 1 + levels) * U53 * mag * (1 + 2.0 ** -20) + 1e-300)
