"""The table-accumulator chain layer (gcb_chain_layer.acc_table) reads its table through the chain
kernel's operand ring: the TMA warp copies the rows of a tile into the stages, 16 rows per stage in
bf16x3 (8 stages) and 8 in bf16 (16 pseudo-K-steps on 12 stages, so the ring wraps inside the unit).
Every case runs a chain whose first layer takes its accumulator from a table filled by an acc_out
chain, and checks every output bit for bit against the same chain with that layer's MMAs: at row
counts that leave the last tile's stages empty or partly filled, at table strides and offsets, next to
a layer that gathers an fp32-table segment (the producer warps then arrive on every stage), at lag 2,
in a three-layer chain in descending order, and with many tiles per cluster."""
import ctypes as C

import pytest
import torch

import test_gpu_chain as tc
from graphcast_b200 import _native
from test_gpu_chain import DEV, Layer, _fill_chain_layer, _image, _image_words, _seg_img, _seg_table, _stream

pytestmark = pytest.mark.gpu

PRECS = ["bf16x3", "bf16"]
N_NODES = 300


@pytest.fixture(autouse=True)
def _release_tensors():
  yield
  torch.cuda.synchronize()
  tc._ALIVE.clear()


def _many_tiles():
  sm = torch.cuda.get_device_properties(0).multi_processor_count
  return 128 * (sm // 2) * 3 + 77


def _run(lib, d):
  _native.check(lib.gcb_chain_forward(C.byref(d), _stream()), "chain")


def _check(prec, rows, chain="two", lag=1, ld=512, offset=0):
  """chain: "two" = [swish(X W0 + b0 + addends), kept] -> LN; "gathered" = the same, the LN layer also
  reading an fp32 table gathered through row indices; "three" = [swish(X W0 + b0 + addends), kept] ->
  [swish, kept] -> LN, in descending order.  The first layer runs once with MMAs and once from the
  table X W0 ([rows, ld] at `offset` bytes into a larger buffer)."""
  lib = _native.lib()
  g = torch.Generator().manual_seed(rows * 7 + ld + offset)
  x = torch.randn(rows, 512, generator=g).to(DEV)
  x[1::5] = 0.0                                             # rows whose products are all zero
  x_img = _image(lib, x, rows, 512)
  l0 = Layer(lib, 512, 512, g, ln=False)
  pa, pb = torch.randn(N_NODES, 512, generator=g).to(DEV), torch.randn(N_NODES, 512, generator=g).to(DEV)
  pa[:, :64] = -0.0
  pb[:, :64] = -0.0
  ia = torch.randint(0, N_NODES, (rows,), generator=g, dtype=torch.int32).to(DEV)
  ib = torch.randint(0, N_NODES, (rows,), generator=g, dtype=torch.int32).to(DEV)
  pre = [(pa, ia), (pb, ib)]
  if chain == "gathered":
    l1 = Layer(lib, 1024, 1024, g, ln=True)
    gt = torch.randn(N_NODES, 512, generator=g).to(DEV)
    gi = torch.randint(0, N_NODES, (rows,), generator=g, dtype=torch.int32).to(DEV)
    gseg = _seg_table(gt, 512, 512)
    gseg.idx = gi.data_ptr()
    tc._ALIVE.append(gi)
  else:
    l1 = Layer(lib, 512, 512, g, ln=chain == "two")
  l2 = Layer(lib, 512, 512, g, ln=True) if chain == "three" else None
  nlayers = 3 if chain == "three" else 2
  scratch = tc._scratch(lib, nlayers - 1, lag, 1)
  nan = lambda: torch.full((rows, 512), float("nan"), device=DEV)

  def desc(n, order=0):
    d = _native.ChainDesc()
    d.rows, d.nlayers, d.precision, d.lag, d.order = rows, n, _native.PRECISIONS[prec], lag, order
    d.scratch, d.scratch_bytes = scratch.data_ptr(), scratch.numel()
    return d

  # the table: X @ W0, the raw accumulator, written with row stride ld at `offset` bytes into a buffer
  assert offset % 16 == 0
  buf = torch.full((rows * ld + offset // 4 + 16,), float("nan"), device=DEV)
  table = buf[offset // 4:offset // 4 + rows * ld].view(rows, ld)
  d = desc(1)
  _fill_chain_layer(d.layer[0], [_seg_img(x_img, 512)], [-1], l0, act=False, keep=False, out=table)
  d.layer[0].bias, d.layer[0].acc_out, d.layer[0].ld_out = None, 1, ld
  _run(lib, d)

  results = []
  for use_table in (False, True):
    img0, out, out_y = torch.zeros_like(x_img), nan(), nan()
    d = desc(nlayers, order=1 if chain == "three" else 0)
    _fill_chain_layer(d.layer[0], [_seg_img(x_img, 512)], [-1], l0, act=True, keep=True, out_img=img0, pre=pre)
    if use_table:
      cl = d.layer[0]
      cl.nseg, cl.w_packed, cl.seg_from[0] = 0, None, -1
      cl.acc_table, cl.ld_acc = table.data_ptr(), ld
    if chain == "two":
      _fill_chain_layer(d.layer[1], [None], [0], l1, act=False, keep=False, out=out, out_y=out_y)
    elif chain == "gathered":
      _fill_chain_layer(d.layer[1], [None, gseg], [0, -1], l1, act=False, keep=False, out=out, out_y=out_y)
    else:
      _fill_chain_layer(d.layer[1], [None], [0], l1, act=True, keep=True)
      _fill_chain_layer(d.layer[2], [None], [1], l2, act=False, keep=False, out=out, out_y=out_y)
    _run(lib, d)
    results.append((_image_words(img0, rows), out, out_y))
  torch.cuda.synchronize()

  assert torch.isfinite(table[:, :512]).all()             # columns 512.. of a wider stride stay unwritten
  bits = lambda t: t.view(torch.int32)
  (mma_img, mma_out, mma_y), (tab_img, tab_out, tab_y) = results
  for a, b in zip(mma_img, tab_img):
    assert torch.equal(a, b)
  assert torch.isfinite(tab_out).all() and torch.isfinite(tab_y).all()
  assert torch.equal(bits(mma_out), bits(tab_out))
  assert torch.equal(bits(mma_y), bits(tab_y))


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("extra", [1, 8, 16, 17, 120])
def test_last_tile_boundaries(prec, extra):
  _check(prec, 256 + extra)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("ld,offset", [(516, 0), (1024, 0), (512, 16), (516, 48)])
def test_table_stride_and_offset(prec, ld, offset):
  _check(prec, 1000, ld=ld, offset=offset)


@pytest.mark.parametrize("prec", PRECS)
def test_next_to_a_gathered_table_segment(prec):
  _check(prec, 1000, chain="gathered")


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("chain,lag", [("two", 2), ("three", 1), ("three", 2)])
def test_schedules(prec, chain, lag):
  _check(prec, 1000, chain=chain, lag=lag)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("chain", ["two", "gathered", "three"])
def test_many_tiles_per_cluster(prec, chain):
  _check(prec, _many_tiles(), chain=chain)
