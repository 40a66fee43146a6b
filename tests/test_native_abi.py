"""The C-ABI library loads and exports every symbol include/graphcast_b200.h
declares; host-only entry points and argument validation (no GPU compute)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from graphcast_b200 import _native

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                      "include", "graphcast_b200.h")


def _declared_functions():
  text = open(HEADER).read()
  text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
  return sorted(set(re.findall(r"\b(gcb_[a-z0-9_]+)\s*\(", text)))


def test_every_declared_symbol_is_exported_and_bound():
  lib = _native.lib()
  names = _declared_functions()
  assert len(names) >= 12
  for name in names:
    assert hasattr(lib, name), f"{name} declared in the header but not exported"
    assert name in _native.EXPORTS, f"{name} has no ctypes signature in _native.EXPORTS"
  assert lib.gcb_abi_version() == _native.GCB_ABI_VERSION == 2


def test_missing_library_fails_loudly(monkeypatch):
  monkeypatch.setattr(_native, "_lib", None)
  monkeypatch.setattr(_native, "_LIB_PATH", "/nonexistent/libgraphcast_b200.so")
  with pytest.raises(_native.NativeLibraryError, match="no CPU / PyTorch fallback"):
    _native.lib()


def _bf16_to_f32(u16):
  return (u16.astype(np.uint32) << 16).view(np.float32)


def test_pack_weight_host_layout_and_split_accuracy():
  lib = _native.lib()
  k_real, n_real, k, n = 20, 227, 32, 256
  w = np.random.default_rng(0).standard_normal((k_real, n_real)).astype(np.float32)
  assert lib.gcb_packed_weight_bytes(k, n) == k * n * 4
  img = np.zeros(k * n * 4, np.uint8)
  assert lib.gcb_pack_weight_host(w.ctypes.data, k_real, n_real, k, n, img.ctypes.data) == 0
  im = img.view(np.uint16).reshape(k // 16, n // 256, 2, 2, 256, 8)   # kstep, block, hi|lo, chunk, row, j
  hi, lo = _bf16_to_f32(im[:, :, 0]), _bf16_to_f32(im[:, :, 1])        # [ks, h, c, r, j]
  rec = (hi + lo).transpose(0, 2, 4, 1, 3).reshape(k, n)               # [ks, c, j, h, r] -> [k, n]
  np.testing.assert_allclose(rec[:k_real, :n_real], w, rtol=2 ** -16, atol=1e-30)
  assert np.all(rec[k_real:] == 0) and np.all(rec[:, n_real:] == 0)
  # hi is the round-to-nearest-even bf16 of w
  want_hi = (((w.view(np.uint32) + 0x7fff + ((w.view(np.uint32) >> 16) & 1)) >> 16) << 16).view(np.float32)
  np.testing.assert_array_equal(hi.transpose(0, 2, 4, 1, 3).reshape(k, n)[:k_real, :n_real], want_hi)
  # 512-wide layer: two 256-column blocks per K-step
  w2 = np.random.default_rng(1).standard_normal((32, 512)).astype(np.float32)
  img2 = np.zeros(32 * 512 * 4, np.uint8)
  assert lib.gcb_pack_weight_host(w2.ctypes.data, 32, 512, 32, 512, img2.ctypes.data) == 0
  im2 = img2.view(np.uint16).reshape(2, 2, 2, 2, 256, 8)
  rec2 = (_bf16_to_f32(im2[:, :, 0]) + _bf16_to_f32(im2[:, :, 1])).transpose(0, 2, 4, 1, 3).reshape(32, 512)
  np.testing.assert_allclose(rec2, w2, rtol=2 ** -16, atol=1e-30)
  assert lib.gcb_pack_weight_host(w.ctypes.data, k_real, n_real, 24, n, img.ctypes.data) == -1
  assert b"multiple of 16" in lib.gcb_last_error()


def test_layer_validation_rejects_bad_descriptors():
  lib = _native.lib()
  d = _native.LayerDesc()
  d.rows, d.n, d.n_valid, d.nseg = 10, 300, 300, 1
  assert lib.gcb_layer_forward(C.byref(d), None) == -1
  assert b"n must be 256 or 512" in lib.gcb_last_error()
  d.n, d.n_valid = 512, 512
  d.seg[0].table, d.seg[0].ld, d.seg[0].k, d.seg[0].k_valid, d.seg[0].fan = 256, 8, 20, 8, 1
  assert lib.gcb_layer_forward(C.byref(d), None) == -1
  assert b"multiple of 16" in lib.gcb_last_error()
  with pytest.raises(ValueError):
    _native.check(-1, "x")


def test_layer_refusals_name_the_unsupported_case():
  """Layers the kernels cannot compute are refused by the argument checks: status -1, and
  gcb_last_error says why.  The pointers are dummies and rows = 0, so a descriptor that passed the
  checks would return 0 without a launch."""
  lib = _native.lib()

  def layer(n=512, n_valid=512, ks=(512,), act=_native.ACT_NONE, ln=False, ld_res=None,
            prec=_native.PREC_BF16X3):
    d = _native.LayerDesc()
    d.rows, d.n, d.n_valid, d.nseg = 0, n, n_valid, len(ks)
    for i, k in enumerate(ks):
      d.seg[i].table, d.seg[i].ld, d.seg[i].k, d.seg[i].k_valid, d.seg[i].fan = 256, k, k, k, 1
    d.w_packed, d.w_f32, d.bias, d.out, d.ld_out = 256, 256, 256, 256, 512
    d.act = act
    if ln:
      d.ln_scale = d.ln_offset = 256
    if ld_res is not None:
      d.residual, d.ld_res = 256, ld_res
    d.precision = prec
    return d

  def refused(d, why):
    assert lib.gcb_layer_forward(C.byref(d), None) == -1
    assert why in lib.gcb_last_error(), lib.gcb_last_error()

  def accepted(d):
    assert lib.gcb_layer_forward(C.byref(d), None) == 0, lib.gcb_last_error()

  refused(layer(ks=(1024, 512, 528)), b"K too large")           # 129 K-steps: 2048 is the limit
  accepted(layer(ks=(1024, 512, 512)))
  for prec in (_native.PREC_BF16X3, _native.PREC_BF16, _native.PREC_FP32_SIMT):
    # the tensor-core epilogue takes the LayerNorm statistics before the activation
    refused(layer(act=_native.ACT_SWISH, ln=True, prec=prec), b"swish OR LayerNorm")
    refused(layer(act=_native.ACT_SWISH, ln=True, n=256, n_valid=256, prec=prec), b"swish OR LayerNorm")
    # ... and over 512 columns combines two 256-column halves of equal width
    for n_valid in (508, 474, 256, 200):
      refused(layer(n_valid=n_valid, ln=True, prec=prec), b"needs n_valid = 512")
    refused(layer(n_valid=474, ld_res=472, prec=prec), b"ld_res must be >= n_valid")
    d = layer(ld_res=512, prec=prec)    # the tensor-core epilogue adds it to out_img only beside out
    d.out, d.out_img = None, 256
    refused(d, b"a residual needs out or out_y")
    d.out_y, d.ld_out_y = 256, 512
    accepted(d)
  for bad in (0, 3, 8, -1):
    assert lib.gcb_set_cluster_size(bad) == -1
    assert b"cluster size must be 1, 2 or 4" in lib.gcb_last_error()
  try:
    for cs in (1, 4):     # one 256-column accumulator per warpgroup: LayerNorm over 512 needs the pair
      assert lib.gcb_set_cluster_size(cs) == 0
      refused(layer(ln=True), b"needs the cluster size 2")
      accepted(layer(ln=True, n=256, n_valid=227))
      accepted(layer(ln=True, prec=_native.PREC_FP32_SIMT))     # no clusters on the SIMT arm
  finally:
    assert lib.gcb_set_cluster_size(2) == 0


def test_chain_refusals_name_the_unsupported_case():
  """Chains the kernel cannot run are refused by gcb_chain_forward's argument checks, as layers are
  above: rows = 0 and dummy pointers, so an accepted descriptor returns 0 without a launch.  The
  scratch is far larger than any chain needs (the need depends on the SM count, which a machine
  without a GPU takes to be 132)."""
  lib = _native.lib()
  LN = dict(ln_scale=256, ln_offset=256)

  def chain(*layers, lag=1, order=0):
    """layers: gcb_chain_layer fields per layer, and `reads`: its seg_from entries (-1: an external
    fp32 table of 512 columns).  Every layer is plain with a bias and an fp32 `out` unless told
    otherwise."""
    d = _native.ChainDesc()
    d.rows, d.nlayers, d.precision, d.lag, d.order = 0, len(layers), _native.PREC_BF16X3, lag, order
    d.scratch, d.scratch_bytes = 256, 1 << 40
    for cl, spec in zip(d.layer, layers):
      spec = dict(spec)
      reads = spec.pop("reads", (-1,))
      cl.nseg = len(reads)
      for s in range(3):
        cl.seg_from[s] = reads[s] if s < len(reads) else -1
      for s, j in enumerate(reads):
        cl.seg[s].k = 512
        if j < 0:
          cl.seg[s].table, cl.seg[s].ld, cl.seg[s].k_valid, cl.seg[s].fan = 256, 512, 512, 1
      cl.w_packed, cl.bias, cl.out, cl.ld_out = 256, 256, 256, 512
      for name, value in spec.items():
        setattr(cl, name, value)
    return d

  def line(n, **kw):
    """n layers, layer l reading layer l - 1 and the last also layer 0: distance n - 1."""
    layers = [dict(keep=1)] + [dict(reads=(l - 1,), keep=1) for l in range(1, n - 1)]
    return chain(*layers, dict(reads=(n - 2, 0) if n > 2 else (n - 2,)), **kw)

  def refused(d, why):
    assert lib.gcb_chain_forward(C.byref(d), None) == -1
    assert why in lib.gcb_last_error(), lib.gcb_last_error()

  def accepted(d):
    assert lib.gcb_chain_forward(C.byref(d), None) == 0, lib.gcb_last_error()

  swish_kept = dict(act=_native.ACT_SWISH, out=None, keep=1)
  # A kept layer's scratch slot is released for reuse only by its seg_from readers.
  no_reader = b"a kept layer must be read through seg_from by a later layer"
  refused(chain(dict(keep=1)), no_reader)
  refused(chain(dict(keep=1, out=None)), no_reader)
  refused(chain(swish_kept, dict(LN, out=None, out_y=256, ld_out_y=512, residual_keep=1)), no_reader)
  accepted(chain(swish_kept, dict(LN, reads=(0,), out=None, out_y=256, ld_out_y=512, residual_keep=1)))
  refused(chain(swish_kept, dict(reads=(0,), keep=1)), no_reader)
  accepted(chain(swish_kept, dict(reads=(0,))))
  # slots per ring: lag x distance (+ 1 in ascending order), at most 5
  too_far = b"lag x distance too large"
  refused(line(4, lag=2, order=0), too_far)
  refused(line(4, lag=2, order=1), too_far)
  accepted(line(3, lag=2, order=1))
  refused(line(6, lag=1, order=0), too_far)
  accepted(line(6, lag=1, order=1))
  accepted(line(6, lag=0, order=1))
  accepted(line(5, lag=1, order=0))
  refused(line(6, lag=3, order=1), b"lag must be 0 (default), 1 or 2")
  refused(chain(*[dict()] * 7), b"nlayers must be 1..GCB_MAX_CHAIN")
  # at most 8 bias / LayerNorm parameter vectors
  refused(chain(dict(LN, keep=1), dict(LN, reads=(0,), keep=1), dict(LN, reads=(1,))),
          b"too many bias / LayerNorm vectors")
  accepted(chain(dict(LN, keep=1), dict(LN, reads=(0,), keep=1), dict(LN, reads=(1,), bias=None)))
  # the descending order needs 3 layers
  refused(line(2, order=1), b"order must be 0, or 1 for chains of at least 3 layers")
  accepted(line(2, order=0))
  accepted(line(3, order=1))
  # residuals on LayerNorm layers only; swish layers deliver operand images only
  refused(chain(dict(residual=256, ld_res=512)), b"residual needs a LayerNorm layer")
  refused(chain(dict(residual_img=256, out=None, out_y=256, ld_out_y=512)), b"residual needs a LayerNorm layer")
  accepted(chain(dict(LN, residual=256, ld_res=512)))
  refused(chain(dict(act=_native.ACT_SWISH)), b"a swish chain layer delivers operand images only")
  refused(chain(dict(act=_native.ACT_SWISH, out=None, out_y=256, ld_out_y=512)),
          b"a swish chain layer delivers operand images only")
  accepted(chain(dict(act=_native.ACT_SWISH, out=None, out_img=256)))
  refused(chain(dict(LN, act=_native.ACT_SWISH, out=None, out_img=256)), b"swish OR LayerNorm")
  # residual_keep names an earlier kept layer
  bad_keep = b"residual_keep must name an earlier kept layer"
  rk = dict(LN, out=None, out_y=256, ld_out_y=512)
  refused(chain(dict(act=_native.ACT_SWISH, out=None, out_img=256), dict(rk, residual_keep=1)), bad_keep)
  refused(chain(dict(rk, residual_keep=2), dict(keep=1), dict(reads=(1,))), bad_keep)
  refused(chain(swish_kept, dict(rk, reads=(0,), residual_keep=2)), bad_keep)
  refused(chain(swish_kept, dict(rk, reads=(0,), residual_keep=1, out=256)), bad_keep)


def _refuser(lib, fn):
  """(refused, accepted) checkers of one entry point called with keyword overrides of its defaults."""
  def refused(why, **kw):
    assert fn(**kw) == -1, (why, kw)
    assert why in lib.gcb_last_error(), (lib.gcb_last_error(), kw)

  def accepted(**kw):
    assert fn(**kw) == 0, (lib.gcb_last_error(), kw)
  return refused, accepted


def test_backward_kernel_refusals_name_the_unsupported_case():
  """Refusals of the backward, tangent and HVP row kernels and the index operations: status -1, and
  gcb_last_error says why.  The pointers are dummies and rows / nodes = 0: the direction kernels, the
  index operations and gcb_swish_rows return without a launch once their checks pass, so the
  accepted cases do no device work.  gcb_weight_grad and the column-sum kernels launch even at
  rows = 0, so only their refusals are called here."""
  lib = _native.lib()
  P = 256                                   # a dummy, 16-byte aligned device address

  def wgrad(x=P, ld_x=64, k_valid=64, x_img=None, swish=0, g=P, ld_g=64, rows=0, k=64, n=64,
            prec=_native.PREC_BF16X3, ws=P, ws_bytes=None, dw=P, acc=0):
    ws_bytes = lib.gcb_weight_grad_workspace_bytes(k, n) if ws_bytes is None else ws_bytes
    return lib.gcb_weight_grad(x, ld_x, k_valid, x_img, swish, g, ld_g, rows, k, n, prec, ws, ws_bytes,
                               dw, acc, None)

  refused, _ = _refuser(lib, wgrad)
  shape = b"k must be a multiple of 16, n of 64"
  refused(shape, k=24, k_valid=24, ld_x=24)
  refused(shape, n=96, ld_g=96)
  refused(shape, n=0, ld_g=64)
  refused(b"rows < 0", rows=-1)
  refused(b"G must have 16-byte rows and ld_g >= n", ld_g=60)
  refused(b"G must have 16-byte rows and ld_g >= n", ld_g=66)
  table = b"x must have 16-byte rows, k_valid a multiple of 4 in (0, k]"
  refused(table, k_valid=6, ld_x=8)
  refused(table, k_valid=80, ld_x=80)
  refused(table, k_valid=0)
  refused(table, ld_x=60)
  refused(table, ld_x=66)
  refused(table, x=None)
  refused(b"weight gradients support the tensor-core precisions only", prec=_native.PREC_FP32_SIMT)
  refused(b"workspace too small", ws_bytes=lib.gcb_weight_grad_workspace_bytes(64, 64) - 1)
  refused(b"workspace too small", k=64, n=128, ld_g=128, ws_bytes=lib.gcb_weight_grad_workspace_bytes(64, 64))
  refused(b"x_img unaligned", x=None, x_img=P + 8)

  nb = lambda n: lib.gcb_rowwise_workspace_bytes(n)

  def ln_bwd(dy=P, ld_dy=512, z=P, ld_z=512, scale=P, rows=0, n=512, dz=P, ld_dz=512, ws=P,
             ws_bytes=None, sums=(P, P, P)):
    return lib.gcb_layernorm_backward(dy, ld_dy, z, ld_z, scale, rows, n, dz, ld_dz, ws,
                                      nb(n) if ws_bytes is None else ws_bytes, *sums, 0, None)

  refused, _ = _refuser(lib, ln_bwd)
  refused(b"the LayerNorm backward needs n = 512", n=256, ld_dy=256, ld_z=256, ld_dz=256)
  refused(b"n must be 256 or 512", n=384, ld_dy=384, ld_z=384, ld_dz=384)
  refused(b"n must be 256 or 512", scale=None, z=None, n=128, ld_dy=128, ld_dz=128)
  refused(b"rows < 0", rows=-1)
  for ld in ("ld_dy", "ld_z", "ld_dz"):
    refused(b"leading dimension < n", **{ld: 508})
  refused(b"leading dimension < n", scale=None, z=None, n=256, ld_dy=256, ld_dz=252)
  refused(b"workspace too small", ws_bytes=nb(512) - 1)
  refused(b"the LayerNorm backward needs z and dz", dz=None)
  refused(b"the LayerNorm backward needs z and dz", z=None)
  refused(b"null column-sum output", sums=(P, None, P))
  refused(b"null column-sum output", scale=None, z=None, sums=(None, None, None))
  refused(b"null pointer", ws=None)

  def swish_bwd(da=P, ld_da=256, h=P, ld_h=256, rows=0, n=256, dh=P, ld_dh=256, ws=P, ws_bytes=None,
                dbias=P):
    return lib.gcb_swish_backward(da, ld_da, h, ld_h, rows, n, dh, ld_dh, ws,
                                  nb(n) if ws_bytes is None else ws_bytes, dbias, 0, None)

  refused, _ = _refuser(lib, swish_bwd)
  refused(b"n must be 256 or 512", n=128, ld_da=128, ld_h=128, ld_dh=128)
  for ld in ("ld_da", "ld_h", "ld_dh"):
    refused(b"leading dimension < n", **{ld: 252})
  refused(b"null pointer", h=None)
  refused(b"null pointer", dh=None)
  refused(b"workspace too small", n=512, ld_da=512, ld_h=512, ld_dh=512, ws_bytes=nb(256))
  refused(b"null column-sum output", dbias=None)

  # ---- direction kernels: rows = 0 returns without a launch --------------------------------------
  def swish_jvp(h=P, ld_h=256, rows=0, n=256, dh=P, ld_dh=256, stride=0, dirs=1, da=P, ld_da=256):
    return lib.gcb_swish_jvp(h, ld_h, rows, n, dh, ld_dh, stride, dirs, da, ld_da, None)

  refused, accepted = _refuser(lib, swish_jvp)
  dirs_msg = b"rows < 0, dirs < 1 or dir_stride < rows"
  refused(dirs_msg, dirs=0)
  refused(dirs_msg, dirs=2, stride=-1)
  refused(dirs_msg, rows=-1)
  accepted(dirs=1, stride=-1)                     # ignored for one direction
  accepted(dirs=3, stride=0)
  ld_msg = b"n / leading dimensions must be multiples of 4 with 16-byte rows"
  refused(ld_msg, n=254)
  for ld in ("ld_h", "ld_dh", "ld_da"):
    refused(ld_msg, **{ld: 252})
    refused(ld_msg, **{ld: 258})
  refused(ld_msg, dh=P + 4)
  refused(b"null pointer", da=None)

  def ln_jvp(z=P, ld_z=512, dz=P, ld_dz=512, scale=P, rows=0, n=512, res=None, ld_res=0, out=P,
             ld_out=512):
    return lib.gcb_layernorm_jvp(z, ld_z, dz, ld_dz, scale, rows, n, res, ld_res, out, ld_out, None)

  refused, accepted = _refuser(lib, ln_jvp)
  refused(b"the LayerNorm tangent needs n = 512", n=256, ld_z=256, ld_dz=256, ld_out=256)
  for kw in (dict(ld_z=508), dict(ld_dz=508), dict(ld_out=508), dict(res=P, ld_res=508), dict(rows=-1)):
    refused(b"rows < 0 or leading dimension < n", **kw)
  refused(b"null pointer", scale=None)
  accepted(res=P, ld_res=516)

  def ln_jvp_dirs(z=P, ld_z=512, dz=P, ld_dz=512, scale=P, rows=0, n=512, stride=0, dirs=2, res=None,
                  ld_res=0, out=P, ld_out=512):
    return lib.gcb_layernorm_jvp_dirs(z, ld_z, dz, ld_dz, scale, rows, n, stride, dirs, res, ld_res,
                                      out, ld_out, None)

  refused, accepted = _refuser(lib, ln_jvp_dirs)
  refused(b"the LayerNorm tangent needs n = 512", n=256, ld_z=256, ld_dz=256, ld_out=256)
  refused(b"dirs < 1 or dir_stride < rows", dirs=0)
  refused(b"dirs < 1 or dir_stride < rows", stride=-1)
  refused(b"rows < 0 or leading dimension < n", ld_out=508)
  refused(b"rows < 0 or leading dimension < n", res=P, ld_res=500)
  accepted(dirs=1, stride=-1)
  accepted(dirs=3, stride=5, res=P, ld_res=512)

  def ln_bwd_dirs(dy=P, ld_dy=512, z=P, ld_z=512, scale=P, rows=0, n=512, stride=0, dirs=2, dz=P,
                  ld_dz=512):
    return lib.gcb_layernorm_backward_dirs(dy, ld_dy, z, ld_z, scale, rows, n, stride, dirs, dz, ld_dz,
                                           None)

  refused, accepted = _refuser(lib, ln_bwd_dirs)
  refused(b"the LayerNorm backward of several directions needs n = 512", n=256, ld_dy=256, ld_z=256,
          ld_dz=256)
  refused(b"dirs < 1 or dir_stride < rows", dirs=0)
  refused(b"dirs < 1 or dir_stride < rows", stride=-1)
  for ld in ("ld_dy", "ld_z", "ld_dz"):
    refused(b"rows < 0 or leading dimension < n", **{ld: 508})
  refused(b"null pointer", scale=None)
  accepted(dirs=1, stride=-1)
  accepted(dirs=3, stride=7)

  def swish_hvp(h=P, ld_h=256, hdot=P, ld_hdot=256, rows=0, n=256, da=P, ld_da=256, stride=0, dh=P,
                ld_dh=256, tangents=1):
    return lib.gcb_swish_backward_jvp_dirs(h, ld_h, hdot, ld_hdot, rows, n, da, ld_da, stride, dh, ld_dh,
                                           tangents, None)

  refused, accepted = _refuser(lib, swish_hvp)
  refused(b"tangents < 1", tangents=0)
  refused(b"rows < 0 or dir_stride < rows", stride=-1)
  refused(b"rows < 0 or dir_stride < rows", rows=-1)
  for ld in ("ld_h", "ld_hdot", "ld_da", "ld_dh"):
    refused(ld_msg, **{ld: 252})
  refused(ld_msg, n=6)
  refused(b"null pointer", hdot=None)
  accepted(tangents=3, stride=9)

  def ln_hvp(dy=P, ld_dy=512, z=P, ld_z=512, zdot=P, ld_zdot=512, scale=P, rows=0, n=512, stride=0,
             dz=P, ld_dz=512, tangents=1):
    return lib.gcb_layernorm_backward_jvp_dirs(dy, ld_dy, z, ld_z, zdot, ld_zdot, scale, rows, n, stride,
                                               dz, ld_dz, tangents, None)

  refused, accepted = _refuser(lib, ln_hvp)
  refused(b"the LayerNorm backward tangent needs n = 512", n=256, ld_dy=256, ld_z=256, ld_zdot=256,
          ld_dz=256)
  refused(b"tangents < 1", tangents=0)
  refused(b"dir_stride < rows", stride=-1)
  for ld in ("ld_dy", "ld_z", "ld_zdot", "ld_dz"):
    refused(b"rows < 0 or leading dimension < n", **{ld: 508})
  refused(b"null pointer", zdot=None)
  accepted(tangents=3, stride=0)

  def swish_rows(h=P, ld_h=256, rows=0, n=256, a=P, ld_a=256):
    return lib.gcb_swish_rows(h, ld_h, rows, n, a, ld_a, None)

  refused, accepted = _refuser(lib, swish_rows)
  refused(ld_msg, ld_a=252)
  refused(ld_msg, ld_h=258)
  refused(ld_msg, n=0)
  accepted(ld_h=260, ld_a=260)

  def gather(src=P, ld_src=512, idx=P, n=0, add=None, ld_add=0, dst=P, ld_dst=512, width=512):
    return lib.gcb_gather_add(src, ld_src, idx, n, add, ld_add, dst, ld_dst, width, None)

  refused, accepted = _refuser(lib, gather)
  gather_msg = b"width / leading dimensions must be multiples of 4 with 16-byte rows"
  refused(gather_msg, width=6)
  refused(gather_msg, ld_src=508)
  refused(gather_msg, ld_dst=508)
  refused(gather_msg, width=4, ld_dst=2)
  refused(b"addend unaligned", add=P, ld_add=508)
  accepted(width=4, ld_src=4, ld_dst=4)
  accepted(width=252, ld_src=256, ld_dst=256, add=P, ld_add=252)

  # ---- index operations: num_nodes = 0 returns without a launch ----------------------------------
  def sorted_sum(msg=P, ld_msg=512, order=P, ptr=P, nodes=0, heavy=None, nheavy=0, out=P, ld_out=512,
                 width=512):
    return lib.gcb_segment_sum_sorted(msg, ld_msg, order, ptr, nodes, heavy, nheavy, out, ld_out, width,
                                      None)

  def receiver_sum(msg=P, ld_msg=512, ptr=P, nodes=0, heavy=None, nheavy=0, out=P, ld_out=512,
                   width=512):
    return lib.gcb_segment_sum_heavy(msg, ld_msg, ptr, nodes, heavy, nheavy, out, ld_out, width, None)

  for fn in (sorted_sum, receiver_sum):
    refused, accepted = _refuser(lib, fn)
    # rows narrower than the 512 summed columns would overlap, and their writes race
    refused(b"ld_msg and ld_out must be >= width", ld_out=508)
    refused(b"ld_msg and ld_out must be >= width", ld_out=256)
    refused(b"ld_msg and ld_out must be >= width", ld_msg=508)
    refused(b"num_nodes < 0", nodes=-1)
    refused(b"num_nodes < 0", nodes=-8)
    refused(b"heavy list is null", nheavy=2)
    refused(b"unaligned", ld_out=514)
    refused(b"supports width 512", width=256, ld_msg=256, ld_out=256)
    accepted(ld_msg=516, ld_out=516)
    accepted(heavy=P, nheavy=3)


def test_debug_flags_accepts_only_zero():
  """The build has no kernel experiment switches: 0 is accepted, anything else is an error."""
  lib = _native.lib()
  assert lib.gcb_debug_flags(0) == 0
  with pytest.raises(ValueError, match="no experiment switches"):
    _native.check(lib.gcb_debug_flags(2), "gcb_debug_flags")


def test_struct_layouts_match_the_header():
  """ctypes mirrors vs the C structs: sizes computed by a C compiler from the header itself."""
  import subprocess
  import tempfile
  src = ('#include <stdio.h>\n#include "graphcast_b200.h"\n'
         'int main(void){printf("%zu %zu %zu %zu %zu\\n", sizeof(gcb_segment), sizeof(gcb_layer_desc),'
         ' sizeof(gcb_chain_layer), sizeof(gcb_chain_desc), sizeof(gcb_model)); return 0;}\n')
  with tempfile.TemporaryDirectory() as d:
    c = os.path.join(d, "s.c")
    open(c, "w").write(src)
    exe = os.path.join(d, "s")
    subprocess.run(["gcc", "-I", os.path.dirname(HEADER), c, "-o", exe], check=True)
    sizes = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
  assert sizes == [C.sizeof(_native.Segment), C.sizeof(_native.LayerDesc), C.sizeof(_native.ChainLayer),
                   C.sizeof(_native.ChainDesc), C.sizeof(_native.Model)]
