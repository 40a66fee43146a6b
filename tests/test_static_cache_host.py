"""The table-accumulator chain layer (gcb_chain_layer.acc_table) and the raw accumulator output
(acc_out) that fills such tables: every refusal of gcb_chain_forward, with its message, and the
refusals of gcb_forward_static.  No GPU needed: the descriptors are checked before anything runs."""
import ctypes as C

import pytest

from graphcast_b200 import _native

LN = dict(ln_scale=256, ln_offset=256)


@pytest.fixture(scope="module")
def lib():
  try:
    return _native.lib()
  except _native.NativeLibraryError as e:
    pytest.skip(str(e))


def _chain(*layers, order=0):
  """rows = 0 (validation only); each layer reads an external fp32 table unless it says otherwise."""
  d = _native.ChainDesc()
  d.rows, d.nlayers, d.precision, d.lag, d.order = 0, len(layers), _native.PREC_BF16X3, 1, order
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


# a table layer: no segments, no weights
TABLE = dict(reads=(), w_packed=None, acc_table=256, ld_acc=512)


def _refused(lib, d, why):
  assert lib.gcb_chain_forward(C.byref(d), None) == -1
  assert why in lib.gcb_last_error(), lib.gcb_last_error()


def _accepted(lib, d):
  assert lib.gcb_chain_forward(C.byref(d), None) == 0, lib.gcb_last_error()


def test_acc_table_layer_refusals(lib):
  no_seg = b"an acc_table layer has no segments and no weights (nseg = 0, w_packed = NULL)"
  _accepted(lib, _chain(TABLE))
  _accepted(lib, _chain(dict(TABLE, act=_native.ACT_SWISH, out=None, keep=1), dict(LN, reads=(0,))))
  _accepted(lib, _chain(dict(TABLE, bias=None, n_pre_add=1,
                             pre_add=(_native.PreAdd * 2)(_native.PreAdd(256, None, 512, 0)))))
  _refused(lib, _chain(dict(TABLE, reads=(-1,))), no_seg)                    # a segment
  _refused(lib, _chain(dict(TABLE, w_packed=256)), no_seg)                   # weights
  _refused(lib, _chain(dict(TABLE, **LN)), b"an acc_table layer cannot have LayerNorm")
  _refused(lib, _chain(dict(TABLE, ld_acc=510)), b"acc_table unaligned")
  _refused(lib, _chain(dict(TABLE, ld_acc=256)), b"acc_table unaligned")
  _refused(lib, _chain(dict(TABLE, acc_table=260)), b"acc_table unaligned")
  # nseg = 0 without a table keeps its message
  _refused(lib, _chain(dict(reads=())), b"nseg must be 1..3")


def test_acc_out_refusals(lib):
  raw = dict(bias=None, acc_out=1)
  _accepted(lib, _chain(raw))
  _accepted(lib, _chain(dict(keep=1, bias=None), dict(raw, reads=(0,))))
  why = (b"acc_out needs out and excludes bias, LayerNorm, swish, pre_add, keep, out_y, out_img "
         b"and acc_table")
  _refused(lib, _chain(dict(raw, bias=256)), why)
  _refused(lib, _chain(dict(raw, acc_out=2)), why)
  _refused(lib, _chain(dict(raw, out=None, out_img=256)), why)
  _refused(lib, _chain(dict(raw, out_y=256, ld_out_y=512)), why)
  _refused(lib, _chain(dict(raw, out_img=256)), why)
  _refused(lib, _chain(dict(raw, **LN)), why)
  _refused(lib, _chain(dict(raw, act=_native.ACT_SWISH)), why)
  _refused(lib, _chain(dict(raw, n_pre_add=1,
                            pre_add=(_native.PreAdd * 2)(_native.PreAdd(256, None, 512, 0)))), why)
  _refused(lib, _chain(dict(raw, keep=1), dict(reads=(0,))), why)
  _refused(lib, _chain(dict(TABLE, **raw)), why)


def test_forward_static_refusals(lib):
  assert lib.gcb_forward_static(None, None, None) == -1
  assert b"null model" in lib.gcb_last_error()
  m = _native.Model()                     # no workspace: refused before any launch
  m.msg_steps = 1
  assert lib.gcb_forward_static(C.byref(m), None, None) == -1
  assert b"workspace pointer is null" in lib.gcb_last_error()
