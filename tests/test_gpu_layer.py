"""Parity of the fused layer kernel (through the C ABI) against a float64 reference of the same op:
gathers, fan-in sums, operand-image segments, zero padding, bias, swish, LayerNorm, residual, all
three outputs, ragged row counts, both output widths.  The tensor-core arms run at every cluster
size (gcb_set_cluster_size: the N-split schedule at 2 with n = 512, the unsplit one otherwise), and
their results must be bit-identical across sizes.  LayerNorm statistics and swish are checked at the
edges of their fp32 arithmetic.  The refusals of gcb_layer_forward that need no GPU are in
test_native_abi.py."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

import _cases
from graphcast_b200 import _native, engine

pytestmark = pytest.mark.gpu

TOL = {"bf16x3": 3e-5, "bf16": 2e-2, "fp32_simt": 5e-6}
U32 = 2.0 ** -24                       # fp32 unit roundoff


@pytest.fixture(autouse=True)
def _default_cluster_size():
  """The cluster size is process-wide: put the default (2) back after every test, pass or fail."""
  yield
  assert _native.lib().gcb_set_cluster_size(2) == 0


def _pack(lib, w, k_pad, n_pad, dev):
  img = np.empty(lib.gcb_packed_weight_bytes(k_pad, n_pad), np.uint8)
  wp = np.zeros((k_pad, n_pad), np.float32)
  wp[:w.shape[0], :w.shape[1]] = w
  assert lib.gcb_pack_weight_host(wp.ctypes.data, k_pad, n_pad, k_pad, n_pad, img.ctypes.data) == 0
  return torch.as_tensor(img).to(dev), torch.as_tensor(wp).to(dev)


def _rel(got, want):
  return float((got - want).abs().max() / want.abs().max())


def _wrap_rows(extra=77):
  """Two waves of 128-row tiles over every SM plus a ragged tile: every CTA loops, and at cluster
  size 4 (and 2 with n = 256) some CTAs of the last clusters get dummy tiles."""
  return 2 * _native.lib().gcb_sm_count(0) * 128 + extra


def _image_values(img, rows, k):
  """fp32 values hi + lo of the operand image of a [rows, k] matrix (layout: gcb_layer_desc)."""
  h = img.view(torch.bfloat16).float().view(-1, k // 16, 2, 2, 1056)[..., :1024]  # tile, K-step, hi|lo, chunk
  v = (h[:, :, 0] + h[:, :, 1]).reshape(-1, k // 16, 2, 128, 8)
  return v.permute(0, 3, 1, 2, 4).reshape(-1, k)[:rows]


def _layer_norm64(x, scale, offset):
  return torch.nn.functional.layer_norm(x, (x.shape[1],), scale.double(), offset.double(), 1e-5)


class _Layer:
  """One fused layer on seeded device data, and its float64 reference, formed once on the device
  and shared by every precision and cluster size the layer runs at.

  segs: ("img", k), an operand-image segment of a random [rows, k] matrix, or
        (table_rows, k_valid, k_pad, use_idx, fan), an fp32 table segment (table_rows None: rows),
        gathered through a random index when use_idx."""

  def __init__(self, rows, segs, n, n_valid, *, act=False, ln=False, residual=False, out=True,
               out_y=False, out_img=False, seed=0, bias=None, w_scale=1.0):
    lib = self.lib = _native.lib()
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(seed)
    randn = lambda *shape: torch.randn(*shape, generator=g, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    self.rows, self.n_valid, self.ln = rows, n_valid, ln
    d = self.desc = _native.LayerDesc()
    d.rows, d.n, d.n_valid, d.nseg = rows, n, n_valid, len(segs)
    self._keep, cols, widths = [], [], []
    for i, sg in enumerate(segs):
      s = d.seg[i]
      if sg[0] == "img":
        k = sg[1]
        x = randn(max(rows, 1), k)
        img = torch.zeros(lib.gcb_a_image_bytes(rows, k), dtype=torch.uint8, device=dev)
        _native.check(lib.gcb_rows_to_image(x.data_ptr(), k, 1, rows, k, img.data_ptr(), st), "to_image")
        s.img, s.k = img.data_ptr(), k
        self._keep.append(img)
        cols.append(_image_values(img, rows, k).double())      # what the layer reads
        widths.append((k, k))
        continue
      trows, kv, kp, use_idx, fan = sg
      trows = rows if trows is None else trows
      ld = kv + 4                                  # row stride wider than the data
      table = randn(trows * fan, ld)
      s.table, s.ld, s.k, s.k_valid, s.fan = table.data_ptr(), ld, kp, kv, fan
      if use_idx:
        idx = torch.randint(0, trows, (rows,), generator=g, device=dev, dtype=torch.int32)
        s.idx = idx.data_ptr()
        self._keep.append(idx)
        src = idx.long()
      else:
        assert trows >= rows
        src = torch.arange(rows, device=dev)
      self._keep.append(table)
      cols.append(table.view(trows, fan, ld)[src][:, :, :kv].double().sum(1))
      widths.append((kv, kp))
    # weight rows laid out with per-segment padding
    k_real, k_pad = sum(kv for kv, _ in widths), sum(kp for _, kp in widths)
    w = randn(k_real, n_valid) * (w_scale / np.sqrt(k_real))
    wp = torch.zeros(k_pad, n_valid, device=dev)
    s0 = dst = 0
    for kv, kp in widths:
      wp[dst:dst + kv] = w[s0:s0 + kv]
      s0 += kv
      dst += kp
    self.w_img, self.w_f32 = _pack(lib, wp.cpu().numpy(), k_pad, n, dev)
    self.bias = 0.1 * randn(n) if bias is None else torch.as_tensor(bias, dtype=torch.float32).to(dev)
    self.scale, self.offset = 1 + 0.1 * randn(n), 0.1 * randn(n)
    d.w_packed, d.w_f32, d.bias = self.w_img.data_ptr(), self.w_f32.data_ptr(), self.bias.data_ptr()
    d.act = _native.ACT_SWISH if act else _native.ACT_NONE
    ld_out = n_valid + (4 - n_valid % 4) % 4 + 4
    self.res = randn(rows, ld_out) if residual else None
    if residual:
      d.residual, d.ld_res = self.res.data_ptr(), ld_out
    # one row more than the layer has: it must stay untouched, like the columns past n_valid
    self.out = torch.empty(rows + 1, ld_out, device=dev) if out else None
    if out:
      d.out, d.ld_out = self.out.data_ptr(), ld_out
    self.outy = torch.empty(rows + 1, ld_out + 8, device=dev) if out_y else None
    if out_y:
      d.out_y, d.ld_out_y = self.outy.data_ptr(), ld_out + 8
    self.img = torch.empty(lib.gcb_a_image_bytes(rows, 512), dtype=torch.uint8, device=dev) if out_img else None
    if out_img:
      d.out_img = self.img.data_ptr()
    # float64 reference
    z = torch.cat(cols, 1)
    self.pre = z @ w.double() + self.bias[:n_valid].double()
    y = self.pre * torch.sigmoid(self.pre) if act else self.pre
    if ln:
      y = _layer_norm64(y, self.scale[:n_valid], self.offset[:n_valid])
    self.want_y = y
    self.want = y + self.res[:, :n_valid].double() if residual else y

  def run(self, prec, cluster=2, *, ln=None):
    """Launches the layer (ln=False: without its LayerNorm) and returns gcb_layer_forward's status."""
    d = self.desc
    _native.check(self.lib.gcb_set_cluster_size(cluster), "gcb_set_cluster_size")
    use_ln = self.ln if ln is None else ln
    d.ln_scale = self.scale.data_ptr() if use_ln else None
    d.ln_offset = self.offset.data_ptr() if use_ln else None
    d.precision = _native.PRECISIONS[prec]
    for t in (self.out, self.outy):
      if t is not None:
        t.fill_(float("nan"))
    if self.img is not None:
      self.img.fill_(0xFF)                       # bf16 NaN
    rc = self.lib.gcb_layer_forward(C.byref(d), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc

  def outputs(self):
    """Every output buffer as raw bytes, padding included."""
    return [t.view(torch.uint8).clone() for t in (self.out, self.outy, self.img) if t is not None]

  def errors(self):
    """Relative error of each output against the reference; asserts nothing was written outside
    [rows, n_valid]."""
    r, nv = self.rows, self.n_valid
    errs = {}
    for name, t, want in (("out", self.out, self.want), ("out_y", self.outy, self.want_y)):
      if t is None:
        continue
      assert torch.isnan(t[:, nv:]).all() and torch.isnan(t[r:]).all(), f"{name} written outside"
      errs[name] = _rel(t[:r, :nv].double(), want)
    if self.img is not None:
      got = _image_values(self.img, r, 512)
      if self.out is not None:     # hi + lo of the fp32 result: 2^-17 relative
        torch.testing.assert_close(got, self.out[:r, :512], rtol=2e-5, atol=2e-5)
      errs["out_img"] = _rel(got.double(), self.want)
    return errs

  def check(self, prec, what):
    for name, err in self.errors().items():
      tol = TOL[prec] + (2 ** -16 if name == "out_img" else 0.0)   # the image's hi + lo rounding
      assert err < tol, f"{what}: {name} relative error {err:.3e} (tolerance {tol:.1e})"


def _run_case(prec, rows, segs, n, n_valid, act, ln, residual, out_y, seed=0, cluster=2):
  """segs: list of (table_rows, k_valid, k_pad, use_idx, fan) or ("img", k).  Largest relative
  error of the layer's outputs against float64."""
  layer = _Layer(rows, segs, n, n_valid, act=act, ln=ln, residual=residual, out_y=out_y, seed=seed)
  _native.check(layer.run(prec, cluster), "layer")
  return max(layer.errors().values())


@pytest.mark.parametrize("prec", ["fp32_simt", "bf16x3", "bf16"])
def test_edge_block_three_gathered_segments(prec):
  err = _run_case(prec, rows=1000, segs=[(1000, 512, 512, False, 1), (300, 512, 512, True, 1),
                                         (77, 512, 512, True, 1)],
                  n=512, n_valid=512, act=True, ln=False, residual=False, out_y=False)
  assert err < TOL[prec], err


@pytest.mark.parametrize("prec", ["fp32_simt", "bf16x3", "bf16"])
def test_layernorm_residual_and_message_output(prec):
  err = _run_case(prec, rows=333, segs=[(333, 512, 512, False, 1)], n=512, n_valid=512,
                  act=False, ln=True, residual=True, out_y=True)
  assert err < TOL[prec], err


@pytest.mark.parametrize("prec", ["fp32_simt", "bf16x3"])
def test_padded_inputs_and_narrow_output(prec):
  # K=474 real columns padded to 480 (first encoder layer), K=4 padded to 16 (edge embed)
  err = _run_case(prec, rows=257, segs=[(257, 476, 480, False, 1)], n=512, n_valid=512,
                  act=True, ln=False, residual=False, out_y=False)
  assert err < TOL[prec], err
  err = _run_case(prec, rows=129, segs=[(129, 4, 16, False, 1)], n=512, n_valid=512,
                  act=True, ln=False, residual=False, out_y=False)
  assert err < TOL[prec], err
  # decoder output layer: 227 of 256 columns, no LayerNorm
  err = _run_case(prec, rows=500, segs=[(500, 512, 512, False, 1)], n=256, n_valid=227,
                  act=False, ln=False, residual=False, out_y=False)
  assert err < TOL[prec], err


@pytest.mark.parametrize("prec", ["fp32_simt", "bf16x3"])
def test_fan_in_three_segment(prec):
  err = _run_case(prec, rows=700, segs=[(700, 512, 512, False, 1), (700, 512, 512, False, 3)],
                  n=512, n_valid=512, act=True, ln=False, residual=False, out_y=False)
  assert err < TOL[prec], err


@pytest.mark.parametrize("rows", [1, 127, 128, 129, 148 * 128 + 5])
def test_ragged_row_counts(rows):
  err = _run_case("bf16x3", rows=rows, segs=[(max(rows, 1), 512, 512, False, 1)], n=512,
                  n_valid=512, act=False, ln=True, residual=True, out_y=False)
  assert err < TOL["bf16x3"], err


@pytest.mark.parametrize("prec", ["fp32_simt", "bf16x3", "bf16"])
@pytest.mark.parametrize("rows", [700, 128 * 148 + 77])
def test_gathered_pre_activation_addends(prec, rows):
  """Split first edge-MLP layer: swish(e @ W_e + b + P_s[snd] + P_r[rcv])."""
  lib = _native.lib()
  dev = torch.device("cuda:0")
  g = torch.Generator().manual_seed(3)
  e = torch.randn(rows, 512, generator=g)
  ps, pr = torch.randn(301, 512, generator=g), torch.randn(97, 516, generator=g)
  snd = torch.randint(0, 301, (rows,), generator=g, dtype=torch.int32)
  rcv = torch.randint(0, 97, (rows,), generator=g, dtype=torch.int32)
  w = torch.randn(512, 512, generator=g) / np.sqrt(512)
  bias = 0.1 * torch.randn(512, generator=g)
  img, wf = _pack(lib, w.numpy(), 512, 512, dev)
  ed, psd, prd, sd, rd, bd = (t.to(dev) for t in (e, ps, pr, snd, rcv, bias))
  out = torch.empty(rows, 512, device=dev)
  d = _native.LayerDesc()
  d.rows, d.n, d.n_valid, d.nseg = rows, 512, 512, 1
  d.seg[0].table, d.seg[0].ld, d.seg[0].k, d.seg[0].k_valid, d.seg[0].fan = ed.data_ptr(), 512, 512, 512, 1
  d.w_packed, d.w_f32, d.bias, d.act = img.data_ptr(), wf.data_ptr(), bd.data_ptr(), 1
  d.out, d.ld_out = out.data_ptr(), 512
  d.precision = _native.PRECISIONS[prec]
  d.n_pre_add = 2
  d.pre_add[0].table, d.pre_add[0].idx, d.pre_add[0].ld = psd.data_ptr(), sd.data_ptr(), 512
  d.pre_add[1].table, d.pre_add[1].idx, d.pre_add[1].ld = prd.data_ptr(), rd.data_ptr(), 516
  _native.check(lib.gcb_layer_forward(C.byref(d), torch.cuda.current_stream().cuda_stream), "layer")
  torch.cuda.synchronize()
  y = e.double() @ w.double() + bias.double() + ps.double()[snd.long()] + pr.double()[rcv.long(), :512]
  want = y * torch.sigmoid(y)
  err = float((out.cpu().double() - want).abs().max() / want.abs().max())
  assert err < TOL[prec], err
  # LayerNorm + pre_add is rejected
  d.ln_scale, d.ln_offset = bd.data_ptr(), bd.data_ptr()
  assert lib.gcb_layer_forward(C.byref(d), None) == -1


@pytest.mark.parametrize("prec", ["fp32_simt", "bf16x3", "bf16"])
@pytest.mark.parametrize("rows", [1, 333, 128 * 148 * 2 + 5])
def test_operand_image_chain(prec, rows):
  """Two-layer MLP with the hidden activations handed over as an operand image:
  layer 0 writes out_img, layer 1 reads a_img (TMA-fed A operand, no gather warps)."""
  lib = _native.lib()
  dev = torch.device("cuda:0")
  g = torch.Generator().manual_seed(5)
  x = torch.randn(rows, 512, generator=g)
  w0 = torch.randn(512, 512, generator=g) / np.sqrt(512)
  w1 = torch.randn(512, 512, generator=g) / np.sqrt(512)
  b0, b1 = 0.1 * torch.randn(512, generator=g), 0.1 * torch.randn(512, generator=g)
  sc, of = 1 + 0.1 * torch.randn(512, generator=g), 0.1 * torch.randn(512, generator=g)
  img0, wf0 = _pack(lib, w0.numpy(), 512, 512, dev)
  img1, wf1 = _pack(lib, w1.numpy(), 512, 512, dev)
  xd, b0d, b1d, scd, ofd = (t.to(dev) for t in (x, b0, b1, sc, of))
  nbytes = lib.gcb_a_image_bytes(rows, 512)
  assert nbytes == ((rows + 127) // 128) * 32 * 8448
  himg = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
  out = torch.empty(rows, 512, device=dev)
  st = torch.cuda.current_stream().cuda_stream
  d = _native.LayerDesc()
  d.rows, d.n, d.n_valid, d.nseg = rows, 512, 512, 1
  d.seg[0].table, d.seg[0].ld, d.seg[0].k, d.seg[0].k_valid, d.seg[0].fan = xd.data_ptr(), 512, 512, 512, 1
  d.w_packed, d.w_f32, d.bias, d.act = img0.data_ptr(), wf0.data_ptr(), b0d.data_ptr(), 1
  d.out_img = himg.data_ptr()
  d.precision = _native.PRECISIONS[prec]
  _native.check(lib.gcb_layer_forward(C.byref(d), st), "layer0")
  d1 = _native.LayerDesc()
  d1.rows, d1.n, d1.n_valid, d1.nseg = rows, 512, 512, 1
  d1.seg[0].img, d1.seg[0].k = himg.data_ptr(), 512
  d1.w_packed, d1.w_f32, d1.bias = img1.data_ptr(), wf1.data_ptr(), b1d.data_ptr()
  d1.ln_scale, d1.ln_offset = scd.data_ptr(), ofd.data_ptr()
  d1.out, d1.ld_out = out.data_ptr(), 512
  d1.precision = _native.PRECISIONS[prec]
  _native.check(lib.gcb_layer_forward(C.byref(d1), st), "layer1")
  torch.cuda.synchronize()
  h = x.double() @ w0.double() + b0.double()
  h = h * torch.sigmoid(h)
  y = torch.nn.functional.layer_norm(h @ w1.double() + b1.double(), (512,), sc.double(), of.double(), 1e-5)
  err = float((out.cpu().double() - y).abs().max() / y.abs().max())
  assert err < 2 * TOL[prec], err


@pytest.mark.parametrize("prec", ["fp32_simt", "bf16x3"])
def test_mixed_image_and_gathered_segments_with_residual_image(prec):
  """[image segment | gathered fp32 segment], LayerNorm + residual, result delivered as
  fp32 AND as an operand image (which must include the residual)."""
  lib = _native.lib()
  dev = torch.device("cuda:0")
  rows = 1000
  g = torch.Generator().manual_seed(9)
  a0 = torch.randn(rows, 512, generator=g)
  tab = torch.randn(222, 512, generator=g)
  idx = torch.randint(0, 222, (rows,), generator=g, dtype=torch.int32)
  w = torch.randn(1024, 512, generator=g) / np.sqrt(1024)
  bias, sc, of = 0.1 * torch.randn(512, generator=g), 1 + 0.1 * torch.randn(512, generator=g), 0.1 * torch.randn(512, generator=g)
  res = torch.randn(rows, 512, generator=g)
  img, wf = _pack(lib, w.numpy(), 1024, 512, dev)
  a0d, tabd, idxd, bd, scd, ofd, resd = (t.to(dev) for t in (a0, tab, idx, bias, sc, of, res))
  st = torch.cuda.current_stream().cuda_stream
  a0img = torch.zeros(lib.gcb_a_image_bytes(rows, 512), dtype=torch.uint8, device=dev)
  _native.check(lib.gcb_rows_to_image(a0d.data_ptr(), 512, 1, rows, 512, a0img.data_ptr(), st), "to_image")
  out = torch.empty(rows, 512, device=dev)
  oimg = torch.zeros(lib.gcb_a_image_bytes(rows, 512), dtype=torch.uint8, device=dev)
  d = _native.LayerDesc()
  d.rows, d.n, d.n_valid, d.nseg = rows, 512, 512, 2
  d.seg[0].img, d.seg[0].k = a0img.data_ptr(), 512
  d.seg[1].table, d.seg[1].idx, d.seg[1].ld, d.seg[1].k, d.seg[1].k_valid, d.seg[1].fan = \
      tabd.data_ptr(), idxd.data_ptr(), 512, 512, 512, 1
  d.w_packed, d.w_f32, d.bias = img.data_ptr(), wf.data_ptr(), bd.data_ptr()
  d.ln_scale, d.ln_offset = scd.data_ptr(), ofd.data_ptr()
  d.residual, d.ld_res, d.out, d.ld_out, d.out_img = resd.data_ptr(), 512, out.data_ptr(), 512, oimg.data_ptr()
  d.precision = _native.PRECISIONS[prec]
  _native.check(lib.gcb_layer_forward(C.byref(d), st), "layer")
  torch.cuda.synchronize()
  z = torch.cat([a0.double(), tab.double()[idx.long()]], 1)
  y = torch.nn.functional.layer_norm(z @ w.double() + bias.double(), (512,), sc.double(), of.double(), 1e-5)
  want = y + res.double()
  assert float((out.cpu().double() - want).abs().max() / want.abs().max()) < 2 * TOL[prec]
  # decode the output image and compare with the fp32 output (bf16 hi+lo ~ 2^-17 relative)
  blocks = oimg.cpu().numpy().view(np.uint16).reshape(-1, 32, 2, 2112)   # tile, kstep, hi|lo, halfwords
  def part(p):
    x = blocks[:, :, p, :].astype(np.uint32) << 16
    x = x.view(np.float32).reshape(-1, 32, 2, 1056)[..., :1024].reshape(-1, 32, 2, 128, 8)
    return x.transpose(0, 3, 1, 2, 4).reshape(-1, 512)                   # [tile*128, 512]
  dec = (part(0) + part(1))[:rows]
  np.testing.assert_allclose(dec, out.cpu().numpy(), rtol=2e-5, atol=2e-5)


def test_rows_to_image_fan_in():
  lib = _native.lib()
  dev = torch.device("cuda:0")
  rows, fan, k = 301, 3, 512
  src = torch.randn(rows * fan, 516, device=dev)
  img = torch.zeros(lib.gcb_a_image_bytes(rows, k), dtype=torch.uint8, device=dev)
  _native.check(lib.gcb_rows_to_image(src.data_ptr(), 516, fan, rows, k, img.data_ptr(),
                                      torch.cuda.current_stream().cuda_stream), "to_image")
  torch.cuda.synchronize()
  blocks = img.cpu().numpy().view(np.uint16).reshape(-1, 32, 2, 2112)
  def part(p):
    x = blocks[:, :, p, :].astype(np.uint32) << 16
    x = x.view(np.float32).reshape(-1, 32, 2, 1056)[..., :1024].reshape(-1, 32, 2, 128, 8)
    return x.transpose(0, 3, 1, 2, 4).reshape(-1, 512)
  dec = part(0) + part(1)
  want = src[:, :k].view(rows, fan, k).sum(1).cpu().numpy()
  np.testing.assert_allclose(dec[:rows], want, rtol=2e-5, atol=2e-5)
  assert np.all(dec[rows:] == 0)


def test_zero_rows_is_a_noop():
  lib = _native.lib()
  d = _native.LayerDesc()
  t = torch.zeros(16, 16, device="cuda:0")
  d.rows, d.n, d.n_valid, d.nseg = 0, 512, 512, 1
  d.seg[0].table, d.seg[0].ld, d.seg[0].k, d.seg[0].k_valid, d.seg[0].fan = t.data_ptr(), 16, 16, 16, 1
  d.w_packed, d.bias, d.out, d.ld_out = t.data_ptr(), t.data_ptr(), t.data_ptr(), 512
  assert lib.gcb_layer_forward(C.byref(d), None) == 0


def test_tensor_path_matches_simt_arm_selftest():
  lib = _native.lib()
  for prec, tol in (("bf16x3", 3e-5), ("bf16", 2e-2)):
    err = C.c_float(-1)
    assert lib.gcb_selftest_layer(3000, 1024, 512, _native.PRECISIONS[prec], C.byref(err)) == 0
    assert 0 <= err.value < tol


# ---- every schedule against float64, and against each other ------------------------------------
# rows: 1, 127, 129, 4 * 128 + 1 and WRAP (_wrap_rows); (n, n_valid): (512, 512), (512, 474),
# (512, 200), (256, 256), (256, 227); T: a table of `rows` rows read without an index.
WRAP, T = "wrap", None
CASES = {
    "rows1_image_gather_swish": dict(
        rows=1, segs=[("img", 512), (50, 512, 512, True, 1)], n=512, n_valid=512, act=True,
        residual=True, out_y=True, out_img=True),
    "rows127_padded_k_layernorm": dict(
        rows=127, segs=[(T, 476, 480, False, 1)], n=512, n_valid=512, ln=True, residual=True,
        out_y=True, out_img=True),
    "rows513_image_fan3_layernorm": dict(
        rows=513, segs=[("img", 512), (T, 508, 512, False, 3)], n=512, n_valid=512, ln=True,
        residual=True, out_y=True, out_img=True),
    "wrap_image_gather_layernorm": dict(
        rows=WRAP, segs=[("img", 512), (1000, 512, 512, True, 1)], n=512, n_valid=512, ln=True,
        residual=True, out_y=True, out_img=True),
    "wrap_three_segments_swish": dict(
        rows=WRAP, segs=[("img", 512), (T, 512, 512, False, 1), (5000, 256, 256, True, 3)], n=512,
        n_valid=512, act=True, out_y=True, out_img=True),
    "rows129_k2048_three_segments": dict(      # kMaxKSteps = 128 K-steps
        rows=129, segs=[(T, 1024, 1024, False, 1), ("img", 512), (300, 512, 512, True, 1)], n=512,
        n_valid=512, residual=True, out_y=True),
    "rows129_fan3_gather_swish_474": dict(
        rows=129, segs=[(T, 512, 512, False, 3), (40, 256, 256, True, 1)], n=512, n_valid=474,
        act=True, residual=True, out_y=True),
    "rows127_three_segments_swish_474": dict(
        rows=127, segs=[(60, 512, 512, True, 1), ("img", 512), (T, 512, 512, False, 1)], n=512,
        n_valid=474, act=True, residual=True, out_y=True),
    "rows513_three_segments_200": dict(
        rows=513, segs=[("img", 256), (300, 512, 512, True, 1), (90, 128, 128, True, 3)], n=512,
        n_valid=200, residual=True, out_y=True),
    "wrap_gather_200": dict(
        rows=WRAP, segs=[(3000, 512, 512, True, 1)], n=512, n_valid=200, out_y=True),
    "rows1_narrow_k_swish_256": dict(
        rows=1, segs=[(T, 4, 16, False, 1)], n=256, n_valid=256, act=True, out_y=True),
    "rows129_image_layernorm_256": dict(
        rows=129, segs=[("img", 512)], n=256, n_valid=256, ln=True, residual=True, out_y=True),
    "rows513_gather_fan3_layernorm_227": dict(
        rows=513, segs=[(200, 512, 512, True, 1), (T, 64, 64, False, 3)], n=256, n_valid=227,
        ln=True, residual=True, out_y=True),
    "wrap_image_227": dict(
        rows=WRAP, segs=[("img", 512)], n=256, n_valid=227, residual=True, out_y=True),
    "wrap_table_image_layernorm_227": dict(
        rows=WRAP, segs=[(T, 512, 512, False, 1), ("img", 256)], n=256, n_valid=227, ln=True,
        residual=True, out_y=True),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_every_schedule_matches_fp64_and_the_default_bit_for_bit(name):
  """fp32_simt once (it has no clusters); bf16x3 and bf16 at cluster sizes 2, 1 and 4.  Each output
  column goes through the same K-ordered MMAs and the same epilogue in the N-split and the unsplit
  schedule, so sizes 1 and 4 must reproduce size 2 bit for bit.  LayerNorm over 512 columns needs
  the N-split pair and is refused at 1 and 4."""
  spec = dict(CASES[name])
  if spec["rows"] == WRAP:
    spec["rows"] = _wrap_rows()
  layer = _Layer(**spec, seed=zlib.crc32(name.encode()))
  lib = layer.lib
  _native.check(layer.run("fp32_simt"), "fp32_simt")
  layer.check("fp32_simt", "fp32_simt")
  ln512 = spec.get("ln", False) and spec["n"] == 512
  for prec in ("bf16x3", "bf16"):
    _native.check(layer.run(prec, 2), f"{prec} cluster 2")
    layer.check(prec, f"{prec} cluster 2")
    want = layer.outputs()
    for cs in (1, 4):
      rc = layer.run(prec, cs)
      if ln512:
        assert rc == -1 and b"needs the cluster size 2" in lib.gcb_last_error(), (prec, cs)
        continue
      _native.check(rc, f"{prec} cluster {cs}")
      layer.check(prec, f"{prec} cluster {cs}")
      for got, ref in zip(layer.outputs(), want):
        assert torch.equal(got, ref), f"{prec}: cluster size {cs} differs from 2"


def test_model_step_is_bit_identical_at_every_cluster_size():
  """The fused step at cluster sizes 1 and 4 (what bench.py --cluster sets): only its layer-by-layer
  launches change schedule -- the decoder's n = 256 output layer and the node projections; the chains
  always run pairs -- and the result must equal the default's bit for bit, through graph replay."""
  lib = _native.lib()
  g, params, x = _cases.small_case(c_in=31, n_out=23, msg_steps=2)
  xt = torch.as_tensor(x)
  _native.check(lib.gcb_set_graph_replay(1), "gcb_set_graph_replay")
  eng = engine.Engine(g, params, c_in=31, n_out=23, msg_steps=2, precision="bf16x3")
  want = eng.forward_features(xt).clone()
  for cs in (1, 4, 2):
    _native.check(lib.gcb_set_cluster_size(cs), "gcb_set_cluster_size")
    for call in ("direct", "capture", "replay"):
      assert torch.equal(eng.forward_features(xt), want), (cs, call)


def test_layer_by_layer_model_step_needs_cluster_size_2():
  """fuse=False runs every MLP's LayerNorm layer (n = 512) through gcb_layer_forward, so cluster
  sizes 1 and 4 refuse the step; the step graph recorded at size 2 is not replayed for them (the
  replay cache keys on the cluster size), and size 2 replays it again afterwards."""
  lib = _native.lib()
  g, params, x = _cases.small_case(c_in=31, n_out=23, msg_steps=2)
  xt = torch.as_tensor(x)
  _native.check(lib.gcb_set_graph_replay(1), "gcb_set_graph_replay")
  eng = engine.Engine(g, params, c_in=31, n_out=23, msg_steps=2, precision="bf16x3", fuse=False)
  want = [eng.forward_features(xt).clone() for _ in range(3)][0]     # direct, capture, replay
  for cs in (1, 4):
    _native.check(lib.gcb_set_cluster_size(cs), "gcb_set_cluster_size")
    with pytest.raises(ValueError, match="needs the cluster size 2"):
      eng.forward_features(xt)
  _native.check(lib.gcb_set_cluster_size(2), "gcb_set_cluster_size")
  assert torch.equal(eng.forward_features(xt), want)


# ---- LayerNorm statistics -------------------------------------------------------------------------
def _ln_runs(n):
  """(precision, cluster size) pairs of a LayerNorm layer of width n."""
  return [("fp32_simt", 2)] + [("bf16x3", cs) for cs in ((2,) if n == 512 else (1, 2, 4))]


@pytest.mark.parametrize("n,n_valid", [(512, 512), (256, 256), (256, 227)])
def test_layernorm_statistics_at_a_large_common_offset(n, n_valid):
  """Pre-LayerNorm values 1e3 + N(0, 2) per row.  The reference is the float64 LayerNorm of the
  layer's own fp32 pre-LayerNorm values (the same launch without LayerNorm: bit for bit the same
  MMAs and bias add), so the statistics are all that is compared."""
  rows = 1000
  bias = 1e3 + torch.randn(n, generator=torch.Generator().manual_seed(23))
  layer = _Layer(rows, [(T, 512, 512, False, 1)], n, n_valid, ln=True, out=False, out_y=True,
                 bias=bias, seed=23)
  sc, of = layer.scale[:n_valid].double(), layer.offset[:n_valid].double()
  for prec, cs in _ln_runs(n):
    _native.check(layer.run(prec, cs, ln=False), f"{prec} cluster {cs} without LayerNorm")
    x = layer.outy[:rows, :n_valid].double()                   # fp32 values, |x| < 1024
    _native.check(layer.run(prec, cs), f"{prec} cluster {cs}")
    got = layer.outy[:rows, :n_valid].double()
    want = _layer_norm64(x, sc, of)
    # Bound from fp32 rounding (u = 2^-24) per row, M = max |x - mean| (~5 here).  The tensor-core
    # epilogue sums d = x - x[0] (|d| <= D, the row's largest deviation from its column 0, ~10 here)
    # and d^2 in chains of 66 roundings (64 columns per thread, two shuffles) and divides by the
    # column count:  |d mean| <= 66 u D,  |d var| <= 3 * 66 u D^2  (s2 / m, and the square of
    # s1 / m; the N-split pair's combination of its halves adds a few u var).  The fp32 SIMT arm
    # sums x itself for the mean, in chains of 21 (16 per lane, five shuffles), and then (x - mean)^2:
    # |d mean| <= 21 u max|x| (~1.3e-3 at the offset),  |d var| <= 3 * 21 u M^2.  Through
    #   y = (x - mean) rstd scale + offset
    # that is  |dy| <= max|scale| rstd (|d mean| + M |d var| / (2 var)) + 16 u max|y|,  the last
    # term for the epilogue's own roundings and rsqrtf.  The offset enters the variance error only
    # through D.  A one-pass E[x^2] - E[x]^2 sums x^2 ~ 1e6: the same variance bound with max|x| ~ 1e3
    # in place of D is (1e3 / 10)^2 = 1e4 times larger; its actual error is checked below.
    big_d = (x - x[:, :1]).abs().amax(1)
    var = x.var(1, unbiased=False)
    big_m = (x - x.mean(1, keepdim=True)).abs().amax(1)
    if prec == "fp32_simt":
      d_mean, d_var = 21 * U32 * x.abs().amax(1), 3 * 21 * U32 * big_m ** 2
    else:
      d_mean, d_var = 66 * U32 * big_d, 3 * 66 * U32 * big_d ** 2
    bound = (sc.abs().max() * torch.rsqrt(var + 1e-5) * (d_mean + big_m * d_var / (2 * var))
             + 16 * U32 * want.abs().amax(1))
    err = (got - want).abs().amax(1)
    worst = int(torch.argmax(err / bound))
    assert (err <= bound).all(), f"{prec} cluster {cs}: row {worst} error {err[worst]:.2e} > {bound[worst]:.2e}"
    # what a one-pass variance in fp32 gives on the same values
    xf = x.float()
    m1 = xf.mean(1, keepdim=True)
    v1 = ((xf * xf).mean(1, keepdim=True) - m1 * m1).clamp_min(0)
    one_pass = ((xf - m1) * torch.rsqrt(v1 + 1e-5) * sc.float() + of.float()).double()
    assert (one_pass - want).abs().max() > 10 * bound.max()


@pytest.mark.parametrize("n,n_valid", [(512, 512), (256, 256), (256, 227)])
def test_layernorm_of_constant_rows_is_the_offset_exactly(n, n_valid):
  """Zero weights and a bias of 0.75 in every column: every row is constant, its deviations from the
  mean are exactly 0 on both arms and all schedules, and the outputs are ln_offset and
  residual + ln_offset exactly (with rstd = rsqrt(1e-5))."""
  rows = 300
  layer = _Layer(rows, [(T, 512, 512, False, 1)], n, n_valid, ln=True, residual=True, out_y=True,
                 bias=torch.full((n,), 0.75), w_scale=0.0, seed=29)
  want_y = layer.offset[:n_valid].expand(rows, n_valid)
  want = layer.res[:, :n_valid] + want_y
  for prec, cs in _ln_runs(n) + [("bf16", cs) for _, cs in _ln_runs(n)[1:]]:
    _native.check(layer.run(prec, cs), f"{prec} cluster {cs}")
    assert torch.equal(layer.outy[:rows, :n_valid], want_y), (prec, cs)
    assert torch.equal(layer.out[:rows, :n_valid], want), (prec, cs)


# ---- swish -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [512, 256])
def test_swish_at_extreme_pre_activations(n):
  """Biases from -100 to 100 across the columns: exp(-x) overflows fp32 below x ~ -88.7 and passes
  2^126 (where __fdividef returns 0) just above it, and underflows at the top.  The outputs must be
  finite and within |dy| <= 1.1 e_pre + 2e-5 |y| of float64 swish: e_pre = TOL * max|z W| is the
  product error the parity tolerances allow (1.1 bounds swish'), and 2e-5 the relative error of
  __expf / __fdividef including the rounding of x log2(e) at |x| <= 101."""
  rows = 700
  layer = _Layer(rows, [(T, 512, 512, False, 1)], n, n, act=True, out=False, out_y=True,
                 bias=torch.linspace(-100.0, 100.0, n), seed=31)
  zw = (layer.pre - layer.bias.double()).abs().max()
  want = layer.want_y
  for prec, cs in [("fp32_simt", 2)] + [(p, cs) for p in ("bf16x3", "bf16") for cs in (1, 2, 4)]:
    _native.check(layer.run(prec, cs), f"{prec} cluster {cs}")
    got = layer.outy[:rows, :n].double()
    assert torch.isfinite(got).all(), (prec, cs)
    excess = (got - want).abs() - (1.1 * TOL[prec] * zw + 2e-5 * want.abs())
    assert excess.max() <= 0, f"{prec} cluster {cs}: {excess.max():.2e} over the bound"
