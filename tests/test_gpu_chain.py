"""Fused layer chains (gcb_chain_forward): the results must be BIT-IDENTICAL to running the same
layers one by one through gcb_layer_forward (same tiles, same products, same order of operations;
only the hand-over of intermediate results changes: L2-resident scratch instead of HBM images),
and within the usual tolerance of a torch fp64 reference.  Row counts give every cluster several
tiles so that the scratch slots are reused and the pipeline fills and drains."""
import ctypes as C

import numpy as np
import pytest
import torch

import _cases
from graphcast_b200 import _native, engine
from oracle import gnn as oracle_gnn

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _stream():
  return torch.cuda.current_stream().cuda_stream


class Layer:
  """One linear layer's parameters on the device + its fp64 reference pieces."""

  def __init__(self, lib, k_real, k_pad, g, ln, bias=True):
    self.k_real, self.k_pad = k_real, k_pad
    self.w = torch.randn(k_real, 512, generator=g) / np.sqrt(k_real)
    wp = np.zeros((k_pad, 512), np.float32)
    wp[:k_real] = self.w.numpy()
    img = np.empty(lib.gcb_packed_weight_bytes(k_pad, 512), np.uint8)
    assert lib.gcb_pack_weight_host(wp.ctypes.data, k_pad, 512, k_pad, 512, img.ctypes.data) == 0
    self.w_img = torch.as_tensor(img).to(DEV)
    self.has_bias = bias
    self.bias = torch.randn(512, generator=g) * 0.1 if bias else torch.zeros(512)
    self.bias_dev = self.bias.to(DEV)
    self.ln = ln
    self.scale = 1 + 0.1 * torch.randn(512, generator=g)
    self.offset = 0.1 * torch.randn(512, generator=g)
    self.scale_dev, self.offset_dev = self.scale.to(DEV), self.offset.to(DEV)


def _image(lib, x_dev, rows, k):
  img = torch.zeros(lib.gcb_a_image_bytes(rows, k), dtype=torch.uint8, device=DEV)
  _native.check(lib.gcb_rows_to_image(x_dev.data_ptr(), x_dev.shape[1], 1, rows, k, img.data_ptr(),
                                      _stream()), "rows_to_image")
  return img


def _scratch(lib, n_keep, lag, dist):
  n = lib.gcb_chain_scratch_bytes(0, n_keep, lag, dist)
  assert n > 0
  return torch.zeros(n, dtype=torch.uint8, device=DEV)


def _layer_forward(lib, prec, rows, segs, layer, act, residual=None, out=None, out_y=None,
                   out_img=None, pre=()):
  d = _native.LayerDesc()
  d.rows, d.n, d.n_valid, d.nseg = rows, 512, 512, len(segs)
  for i, s in enumerate(segs):
    d.seg[i] = s
  d.w_packed, d.bias = layer.w_img.data_ptr(), layer.bias_dev.data_ptr()
  if layer.ln:
    d.ln_scale, d.ln_offset = layer.scale_dev.data_ptr(), layer.offset_dev.data_ptr()
  d.act = 1 if act else 0
  if residual is not None:
    d.residual, d.ld_res = residual.data_ptr(), 512
  if out is not None:
    d.out, d.ld_out = out.data_ptr(), 512
  if out_y is not None:
    d.out_y, d.ld_out_y = out_y.data_ptr(), 512
  if out_img is not None:
    d.out_img = out_img.data_ptr()
  d.n_pre_add = len(pre)
  for i, (t, idx) in enumerate(pre):
    d.pre_add[i].table, d.pre_add[i].ld = t.data_ptr(), 512
    d.pre_add[i].idx = idx.data_ptr() if idx is not None else None
  d.precision = _native.PRECISIONS[prec]
  _native.check(lib.gcb_layer_forward(C.byref(d), _stream()), "layer")


_ALIVE = []     # descriptors hold raw pointers: every tensor they name must outlive the launch


def _seg_img(img, k):
  _ALIVE.append(img)
  s = _native.Segment()
  s.img, s.k, s.k_valid, s.fan = img.data_ptr(), k, k, 1
  return s


def _seg_table(t, k_valid, k_pad):
  _ALIVE.append(t)
  s = _native.Segment()
  s.table, s.ld, s.k, s.k_valid, s.fan = t.data_ptr(), t.shape[1], k_pad, k_valid, 1
  return s


def _fill_chain_layer(cl, segs, seg_from, layer, act, keep, residual=None, out=None, out_y=None,
                      out_img=None, pre=()):
  cl.nseg = len(segs)
  for i, s in enumerate(segs):
    if s is not None:
      cl.seg[i] = s
    else:
      cl.seg[i].k = 512
    cl.seg_from[i] = seg_from[i]
  for i in range(len(segs), 3):
    cl.seg_from[i] = -1
  cl.w_packed = layer.w_img.data_ptr()
  cl.bias = layer.bias_dev.data_ptr() if layer.has_bias else None
  if layer.ln:
    cl.ln_scale, cl.ln_offset = layer.scale_dev.data_ptr(), layer.offset_dev.data_ptr()
  cl.act, cl.keep = (1 if act else 0), (1 if keep else 0)
  if residual is not None:
    cl.residual, cl.ld_res = residual.data_ptr(), 512
  if out is not None:
    cl.out, cl.ld_out = out.data_ptr(), 512
  if out_y is not None:
    cl.out_y, cl.ld_out_y = out_y.data_ptr(), 512
  if out_img is not None:
    cl.out_img = out_img.data_ptr()
  cl.n_pre_add = len(pre)
  for i, (t, idx) in enumerate(pre):
    cl.pre_add[i].table, cl.pre_add[i].ld = t.data_ptr(), 512
    cl.pre_add[i].idx = idx.data_ptr() if idx is not None else None


def _swish(x):
  return x * torch.sigmoid(x)


@pytest.fixture(autouse=True)
def _release_tensors():
  yield
  torch.cuda.synchronize()
  _ALIVE.clear()


@pytest.mark.parametrize("prec,tol", [("bf16x3", 3e-5), ("bf16", 3e-2)])
@pytest.mark.parametrize("lag", [1, 2])
@pytest.mark.parametrize("kind", ["edge", "node", "embed"])
def test_two_layer_mlp_chain_is_bit_identical_to_two_layer_launches(prec, tol, lag, kind):
  lib = _native.lib()
  g = torch.Generator().manual_seed(5)
  rows = 128 * 330 + 77            # > 4 tiles per cluster on 66 clusters, ragged last tile
  n_nodes = 5000
  f = lambda *shape: torch.randn(*shape, generator=g)
  nan = lambda: torch.full((rows, 512), float("nan"), device=DEV)
  pre, segs, ref_cols = [], [], []
  if kind == "edge":          # e image + two gathered node projections (pre-activation addends)
    x = f(rows, 512); xd = x.to(DEV)
    segs = [_seg_img(_image(lib, xd, rows, 512), 512)]
    k_real = k_pad = 512
    ref_cols = [x.double()]
    pa, pb = f(n_nodes, 512), f(n_nodes, 512)
    ia = torch.randint(0, n_nodes, (rows,), generator=g, dtype=torch.int32)
    ib = torch.randint(0, n_nodes, (rows,), generator=g, dtype=torch.int32)
    keepalive = [pa.to(DEV), pb.to(DEV), ia.to(DEV), ib.to(DEV)]
    pre = [(keepalive[0], keepalive[2]), (keepalive[1], keepalive[3])]
    pre_ref = pa.double()[ia.long()] + pb.double()[ib.long()]
  elif kind == "node":        # two image segments [v | agg]
    x, a = f(rows, 512), f(rows, 512)
    xd, ad = x.to(DEV), a.to(DEV)
    segs = [_seg_img(_image(lib, xd, rows, 512), 512), _seg_img(_image(lib, ad, rows, 512), 512)]
    k_real = k_pad = 1024
    ref_cols = [x.double(), a.double()]
    pre_ref = 0
  else:                       # edge-feature embedder: fp32 table, 4 real columns padded to 16
    x = f(rows, 4); xd = x.to(DEV)
    segs = [_seg_table(xd, 4, 16)]
    k_real, k_pad = 4, 16
    ref_cols = [x.double()]
    pre_ref = 0
  l0 = Layer(lib, k_real, k_pad, g, ln=False)
  l1 = Layer(lib, 512, 512, g, ln=True)
  res = f(rows, 512); resd = res.to(DEV)

  # layer-by-layer (hidden image through HBM)
  hidden = torch.zeros(lib.gcb_a_image_bytes(rows, 512), dtype=torch.uint8, device=DEV)
  o1, y1 = nan(), nan()
  img1 = torch.zeros_like(hidden)
  _layer_forward(lib, prec, rows, segs, l0, act=True, out_img=hidden, pre=pre)
  _layer_forward(lib, prec, rows, [_seg_img(hidden, 512)], l1, act=False, residual=resd, out=o1,
                 out_y=y1, out_img=img1)
  # one chain launch
  o2, y2 = nan(), nan()
  img2 = torch.zeros_like(hidden)
  scratch = _scratch(lib, 1, lag, 1)
  ch = _native.ChainDesc()
  ch.rows, ch.nlayers, ch.precision, ch.lag = rows, 2, _native.PRECISIONS[prec], lag
  ch.scratch, ch.scratch_bytes = scratch.data_ptr(), scratch.numel()
  _fill_chain_layer(ch.layer[0], segs, [-1] * len(segs), l0, act=True, keep=True, pre=pre)
  _fill_chain_layer(ch.layer[1], [None], [0], l1, act=False, keep=False, residual=resd, out=o2,
                    out_y=y2, out_img=img2)
  _native.check(lib.gcb_chain_forward(C.byref(ch), _stream()), "chain")
  torch.cuda.synchronize()
  assert torch.equal(o1, o2)
  assert torch.equal(y1, y2)
  n_img = (rows // 128) * 32 * 8448          # full tiles (rows of the ragged tail tile are don't-care)
  assert torch.equal(img1[:n_img], img2[:n_img])
  # fp64 reference
  z = torch.cat(ref_cols, 1) @ l0.w.double() + l0.bias.double() + pre_ref
  h = _swish(z)
  y = h @ l1.w.double() + l1.bias.double()
  y = torch.nn.functional.layer_norm(y, (512,), l1.scale.double(), l1.offset.double(), 1e-5)
  err = float((y2.cpu().double() - y).abs().max() / y.abs().max())
  err_o = float((o2.cpu().double() - (y + res.double())).abs().max() / (y + res.double()).abs().max())
  assert max(err, err_o) < tol, (err, err_o)


@pytest.mark.parametrize("lag", [1, 2])
def test_four_layer_chain_with_skip_consumers(lag):
  """node MLP (2 layers) followed by two projections of its result -- the shape of the processor's
  node block -- with a layer that is consumed at distance 1 and 2 (three scratch slots at lag 1)."""
  lib = _native.lib()
  prec = "bf16x3"
  g = torch.Generator().manual_seed(11)
  rows = 128 * 300 + 5
  f = lambda *shape: torch.randn(*shape, generator=g)
  nan = lambda: torch.full((rows, 512), float("nan"), device=DEV)
  v, a = f(rows, 512), f(rows, 512)
  vd, ad = v.to(DEV), a.to(DEV)
  v_img, a_img = _image(lib, vd, rows, 512), _image(lib, ad, rows, 512)
  l0 = Layer(lib, 1024, 1024, g, ln=False)
  l1 = Layer(lib, 512, 512, g, ln=True)
  ps = Layer(lib, 512, 512, g, ln=False, bias=False)
  pr = Layer(lib, 512, 512, g, ln=False, bias=False)
  # layer by layer
  hidden = torch.zeros(lib.gcb_a_image_bytes(rows, 512), dtype=torch.uint8, device=DEV)
  vnew1, vimg1 = nan(), torch.zeros_like(hidden)
  s1, r1 = nan(), nan()
  _layer_forward(lib, prec, rows, [_seg_img(v_img, 512), _seg_img(a_img, 512)], l0, act=True, out_img=hidden)
  _layer_forward(lib, prec, rows, [_seg_img(hidden, 512)], l1, act=False, residual=vd, out=vnew1, out_img=vimg1)
  _layer_forward(lib, prec, rows, [_seg_img(vimg1, 512)], ps, act=False, out=s1)
  _layer_forward(lib, prec, rows, [_seg_img(vimg1, 512)], pr, act=False, out=r1)
  # chain: layer 1's result is consumed by layers 2 (distance 1) and 3 (distance 2)
  vnew2, vimg2, s2, r2 = nan(), torch.zeros_like(hidden), nan(), nan()
  scratch = _scratch(lib, 2, lag, 2)
  ch = _native.ChainDesc()
  ch.rows, ch.nlayers, ch.precision, ch.lag = rows, 4, _native.PRECISIONS[prec], lag
  ch.scratch, ch.scratch_bytes = scratch.data_ptr(), scratch.numel()
  _fill_chain_layer(ch.layer[0], [_seg_img(v_img, 512), _seg_img(a_img, 512)], [-1, -1], l0, act=True, keep=True)
  _fill_chain_layer(ch.layer[1], [None], [0], l1, act=False, keep=True, residual=vd, out=vnew2, out_img=vimg2)
  _fill_chain_layer(ch.layer[2], [None], [1], ps, act=False, keep=False, out=s2)
  _fill_chain_layer(ch.layer[3], [None], [1], pr, act=False, keep=False, out=r2)
  _native.check(lib.gcb_chain_forward(C.byref(ch), _stream()), "chain")
  torch.cuda.synchronize()
  assert torch.equal(vnew1, vnew2)
  assert torch.equal(s1, s2)
  assert torch.equal(r1, r2)
  n_img = (rows // 128) * 32 * 8448
  assert torch.equal(vimg1[:n_img], vimg2[:n_img])


def test_chain_argument_validation():
  lib = _native.lib()
  ch = _native.ChainDesc()
  ch.rows, ch.nlayers, ch.precision = 128, 5, 0
  assert lib.gcb_chain_forward(C.byref(ch), None) == -1
  ch.nlayers, ch.precision = 1, _native.PRECISIONS["fp32_simt"]
  assert lib.gcb_chain_forward(C.byref(ch), None) == -1
  assert b"tensor-core" in lib.gcb_last_error()
  assert lib.gcb_chain_scratch_bytes(0, 1, 1, 1) == (lib.gcb_sm_count(0) // 2) * 2 * 32 * 8448


@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
def test_fused_step_is_bit_identical_to_the_layer_by_layer_step(prec):
  g, params, x = _cases.small_case(c_in=31, n_out=23, msg_steps=3, batch=1)
  xt = torch.as_tensor(x)
  a = engine.Engine(g, params, c_in=31, n_out=23, msg_steps=3, precision=prec, fuse=False)
  ya = a.forward_features(xt).clone()
  b = engine.Engine(g, params, c_in=31, n_out=23, msg_steps=3, precision=prec, fuse=True,
                    image_residual=False)
  yb = b.forward_features(xt).clone()
  assert torch.equal(ya, yb)
  assert torch.equal(a.mesh_lat, b.mesh_lat) and torch.equal(a.grid_lat, b.grid_lat)
  # every MLP but the decoder's (n = 256 output) is one launch instead of two
  n_mlp = 6 + 1 + 2 * 3 + 4
  assert a.launches_per_step - b.launches_per_step == n_mlp - 1
  ref = oracle_gnn.Oracle(params, torch.float32).forward(g.as_dict(), x).numpy()
  if prec == "bf16x3":
    assert float(np.abs(yb.cpu().numpy() - ref).max() / np.abs(ref).max()) <= 1e-4


def _decode_image(img, rows):
  """Operand image -> fp32 [rows, 512] (hi + lo), on the host."""
  raw = img.cpu().numpy().view(np.uint16).reshape(-1, 32, 2, 2112)      # [tile, kstep, hi|lo, 2112 u16]
  pieces = np.stack([raw[..., :1024], raw[..., 1056:2080]], axis=3)      # chunks c = 0, 1 (64 B skew)
  pieces = pieces.reshape(-1, 32, 2, 2, 128, 8)                           # [tile, ks, part, c, row, 8]
  f = (pieces.astype(np.uint32) << 16).view(np.float32)
  x = f[:, :, 0] + f[:, :, 1]                                             # hi + lo: [tile, ks, c, row, 8]
  x = x.transpose(0, 3, 1, 2, 4).reshape(-1, 512)
  return x[:rows]


def test_image_residual_update_matches_the_fp32_master_update():
  """x += LN(MLP([x | a])) with x held ONLY as an operand image (residual read back from the
  image, result written in place) against the same update with an fp32 master."""
  lib = _native.lib()
  prec = "bf16x3"
  g = torch.Generator().manual_seed(3)
  rows = 128 * 200 + 9
  f = lambda *shape: torch.randn(*shape, generator=g)
  x, a = f(rows, 512), f(rows, 512)
  xd, ad = x.to(DEV), a.to(DEV)
  x_img, a_img = _image(lib, xd, rows, 512), _image(lib, ad, rows, 512)
  x_from_img = torch.as_tensor(_decode_image(x_img, rows))
  assert float((x_from_img - x).abs().max() / x.abs().max()) < 2 ** -16      # the image IS x to 2^-17
  l0 = Layer(lib, 1024, 1024, g, ln=False)
  l1 = Layer(lib, 512, 512, g, ln=True)
  scratch = _scratch(lib, 1, 1, 1)

  def run(image_residual):
    out_img = x_img.clone()
    xm = x_from_img.to(DEV)              # master holding exactly what the image holds
    y = torch.full((rows, 512), float("nan"), device=DEV)
    ch = _native.ChainDesc()
    ch.rows, ch.nlayers, ch.precision, ch.lag = rows, 2, _native.PRECISIONS[prec], 1
    ch.scratch, ch.scratch_bytes = scratch.data_ptr(), scratch.numel()
    _fill_chain_layer(ch.layer[0], [_seg_img(out_img, 512), _seg_img(a_img, 512)], [-1, -1], l0, act=True, keep=True)
    _fill_chain_layer(ch.layer[1], [None], [0], l1, act=False, keep=False,
                      residual=None if image_residual else xm, out_y=y, out_img=out_img)
    if image_residual:
      ch.layer[1].residual_img = out_img.data_ptr()
    _native.check(lib.gcb_chain_forward(C.byref(ch), _stream()), "chain")
    torch.cuda.synchronize()
    return y, _decode_image(out_img, rows)

  y_m, x_m = run(False)
  y_i, x_i = run(True)
  assert torch.equal(y_m, y_i)                       # the MLP output itself is untouched
  np.testing.assert_array_equal(x_m, x_i)            # same residual values -> same updated image
  want = x_from_img.double() + y_m.cpu().double()
  assert float((torch.as_tensor(x_i).double() - want).abs().max() / want.abs().max()) < 2 ** -16


@pytest.mark.parametrize("msg_steps", [3])
def test_image_residual_step_stays_within_the_parity_gate(msg_steps):
  g, params, x = _cases.small_case(c_in=31, n_out=23, msg_steps=msg_steps, batch=1)
  ref = oracle_gnn.Oracle(params, torch.float64).forward(g.as_dict(), x).numpy()
  xt = torch.as_tensor(x)
  a = engine.Engine(g, params, c_in=31, n_out=23, msg_steps=msg_steps, precision="bf16x3",
                    image_residual=False)
  b = engine.Engine(g, params, c_in=31, n_out=23, msg_steps=msg_steps, precision="bf16x3",
                    image_residual=True, deep_chains=False)
  ya, yb = a.forward_features(xt).cpu().numpy(), b.forward_features(xt).cpu().numpy()
  ea = float(np.abs(ya - ref).max() / np.abs(ref).max())
  eb = float(np.abs(yb - ref).max() / np.abs(ref).max())
  print(f"vs fp64 oracle: fp32 masters {ea:.3e}, image-only latents {eb:.3e}")
  assert eb <= 1e-4


@pytest.mark.parametrize("lag", [1, 2])
def test_descending_order_chain_is_bit_identical(lag):
  """Same 4-layer node block with the last layer first inside each pipeline step (one scratch
  slot less per ring)."""
  lib = _native.lib()
  prec = "bf16x3"
  g = torch.Generator().manual_seed(13)
  rows = 128 * 300 + 5
  f = lambda *shape: torch.randn(*shape, generator=g)
  nan = lambda: torch.full((rows, 512), float("nan"), device=DEV)
  v, a = f(rows, 512), f(rows, 512)
  vd, ad = v.to(DEV), a.to(DEV)
  v_img, a_img = _image(lib, vd, rows, 512), _image(lib, ad, rows, 512)
  l0 = Layer(lib, 1024, 1024, g, ln=False)
  l1 = Layer(lib, 512, 512, g, ln=True)
  ps = Layer(lib, 512, 512, g, ln=False, bias=False)
  pr = Layer(lib, 512, 512, g, ln=False, bias=False)
  outs = []
  for order in (0, 1):
    vnew, vimg, s_, r_ = nan(), torch.zeros_like(v_img), nan(), nan()
    scratch = _scratch(lib, 2, lag, 2)
    ch = _native.ChainDesc()
    ch.rows, ch.nlayers, ch.precision, ch.lag, ch.order = rows, 4, _native.PRECISIONS[prec], lag, order
    ch.scratch, ch.scratch_bytes = scratch.data_ptr(), scratch.numel()
    _fill_chain_layer(ch.layer[0], [_seg_img(v_img, 512), _seg_img(a_img, 512)], [-1, -1], l0, act=True, keep=True)
    _fill_chain_layer(ch.layer[1], [None], [0], l1, act=False, keep=True, residual=vd, out=vnew, out_img=vimg)
    _fill_chain_layer(ch.layer[2], [None], [1], ps, act=False, keep=False, out=s_)
    _fill_chain_layer(ch.layer[3], [None], [1], pr, act=False, keep=False, out=r_)
    _native.check(lib.gcb_chain_forward(C.byref(ch), _stream()), "chain")
    torch.cuda.synchronize()
    outs.append((vnew, vimg, s_, r_))
  n_img = (rows // 128) * 32 * 8448
  for x, y in zip(outs[0], outs[1]):
    assert torch.equal(x[:n_img] if x.dtype == torch.uint8 else x, y[:n_img] if y.dtype == torch.uint8 else y)


def test_embedder_plus_edge_mlp_chain_with_on_chip_residual():
  """[edge embedder MLP -> edge MLP] as one 4-layer chain, the embedded latent e0 kept on chip and
  used both as the edge MLP's input and as its residual (e1 = e0 + m): against the same four layers
  run one by one with e0 written to HBM."""
  lib = _native.lib()
  prec = "bf16x3"
  g = torch.Generator().manual_seed(17)
  rows, n_nodes = 128 * 290 + 31, 7000
  f = lambda *shape: torch.randn(*shape, generator=g)
  nan = lambda: torch.full((rows, 512), float("nan"), device=DEV)
  feat = f(rows, 4).to(DEV)
  e0l0, e0l1 = Layer(lib, 4, 16, g, ln=False), Layer(lib, 512, 512, g, ln=True)
  m0, m1 = Layer(lib, 512, 512, g, ln=False), Layer(lib, 512, 512, g, ln=True)
  pa, pb = f(n_nodes, 512).to(DEV), f(n_nodes, 512).to(DEV)
  ia = torch.randint(0, n_nodes, (rows,), generator=g, dtype=torch.int32).to(DEV)
  ib = torch.randint(0, n_nodes, (rows,), generator=g, dtype=torch.int32).to(DEV)
  pre = [(pa, ia), (pb, ib)]
  nbytes = lib.gcb_a_image_bytes(rows, 512)
  zimg = lambda: torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
  # layer by layer: e0 as fp32 master (the residual) + image
  hidden, e0_img, e0, msg1, e1_img = zimg(), zimg(), nan(), nan(), zimg()
  _layer_forward(lib, prec, rows, [_seg_table(feat, 4, 16)], e0l0, act=True, out_img=hidden)
  _layer_forward(lib, prec, rows, [_seg_img(hidden, 512)], e0l1, act=False, out=e0, out_img=e0_img)
  _layer_forward(lib, prec, rows, [_seg_img(e0_img, 512)], m0, act=True, out_img=hidden, pre=pre)
  e1 = nan()
  _layer_forward(lib, prec, rows, [_seg_img(hidden, 512)], m1, act=False, residual=e0, out=e1, out_y=msg1,
                 out_img=e1_img)
  # one chain
  msg2, e2_img = nan(), zimg()
  scratch = _scratch(lib, 3, 1, 2)
  ch = _native.ChainDesc()
  ch.rows, ch.nlayers, ch.precision, ch.lag, ch.order = rows, 4, _native.PRECISIONS[prec], 1, 1
  ch.scratch, ch.scratch_bytes = scratch.data_ptr(), scratch.numel()
  _fill_chain_layer(ch.layer[0], [_seg_table(feat, 4, 16)], [-1], e0l0, act=True, keep=True)
  _fill_chain_layer(ch.layer[1], [None], [0], e0l1, act=False, keep=True)
  _fill_chain_layer(ch.layer[2], [None], [1], m0, act=True, keep=True, pre=pre)
  _fill_chain_layer(ch.layer[3], [None], [2], m1, act=False, keep=False, out_y=msg2, out_img=e2_img)
  ch.layer[3].residual_keep = 2
  _native.check(lib.gcb_chain_forward(C.byref(ch), _stream()), "chain")
  torch.cuda.synchronize()
  assert torch.equal(msg1, msg2)                    # the MLP outputs are bit-identical
  # e1 = e0 + m: the chain adds the image form of e0 (hi + lo, 2^-17), the reference its fp32 master
  x1, x2 = _decode_image(e1_img, rows), _decode_image(e2_img, rows)
  assert float(np.abs(x1 - x2).max() / np.abs(x1).max()) < 2 ** -15


@pytest.mark.parametrize("deep", [False, True])
def test_image_residual_step_stagewise_and_deep_chains(deep):
  g, params, x = _cases.small_case(c_in=31, n_out=23, msg_steps=3, batch=1)
  ref = oracle_gnn.Oracle(params, torch.float64).forward(g.as_dict(), x).numpy()
  eng = engine.Engine(g, params, c_in=31, n_out=23, msg_steps=3, precision="bf16x3",
                      image_residual=True, deep_chains=deep)
  y = eng.forward_features(torch.as_tensor(x)).cpu().numpy()
  err = float(np.abs(y - ref).max() / np.abs(ref).max())
  print(f"image-only latents, deep_chains={deep}: {err:.3e} vs fp64 oracle, {eng.launches_per_step} launches")
  assert err <= 1e-4
  # stage by stage == whole step
  planes = torch.as_tensor(x[:, 0, :]).t().contiguous().to(eng.device)
  eng.pack_inputs(planes)
  n = eng.run_stage("encode") + eng.run_stage("process_embed")
  for k in range(3):
    n += eng.run_stage("process_step", k)
  n += eng.run_stage("decode")
  torch.cuda.synchronize()
  assert n == eng.launches_per_step
  np.testing.assert_array_equal(eng.grid_out[:, :23].cpu().numpy(), y[:, 0])
