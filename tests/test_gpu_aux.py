"""Segment sum and halo row packing kernels against PyTorch references (the channel pack / unpack
kernels are checked in test_gpu_grid_io_kernels.py)."""
import numpy as np
import pytest
import torch

from graphcast_b200 import _native

pytestmark = pytest.mark.gpu


def test_segment_sum_skewed_degrees_and_empty_rows():
  lib = _native.lib()
  dev = torch.device("cuda:0")
  rng = np.random.default_rng(0)
  deg = rng.integers(0, 12, 3000)
  deg[5] = 0; deg[17] = 3753; deg[2999] = 1             # empty, pole-like, last
  row_ptr = np.zeros(3001, np.int32); np.cumsum(deg, out=row_ptr[1:])
  e = int(row_ptr[-1])
  msg = torch.randn(e, 512, device=dev)
  out = torch.full((3000, 512), float("nan"), device=dev)
  rp = torch.as_tensor(row_ptr).to(dev)
  _native.check(lib.gcb_segment_sum(msg.data_ptr(), 512, rp.data_ptr(), 3000, out.data_ptr(), 512,
                                    512, torch.cuda.current_stream().cuda_stream), "segsum")
  ids = torch.repeat_interleave(torch.arange(3000, device=dev), torch.as_tensor(deg, device=dev))
  want = torch.zeros(3000, 512, device=dev, dtype=torch.float64).index_add_(0, ids, msg.double())
  # fp32 running sums of up to 3753 N(0,1) terms: absolute error grows with the degree
  torch.testing.assert_close(out.double(), want, rtol=1e-5, atol=2e-3)
  assert (out[5] == 0).all()
  # deterministic: bit-identical on a second run
  out2 = torch.empty_like(out)
  lib.gcb_segment_sum(msg.data_ptr(), 512, rp.data_ptr(), 3000, out2.data_ptr(), 512, 512,
                      torch.cuda.current_stream().cuda_stream)
  assert torch.equal(out, out2)
  # heavy-receiver path: nodes with > 256 in-edges get one block each; same result, deterministic
  heavy = torch.as_tensor(np.nonzero(deg > 256)[0].astype(np.int32)).to(dev)
  out3 = torch.full((3000, 512), float("nan"), device=dev)
  _native.check(lib.gcb_segment_sum_heavy(msg.data_ptr(), 512, rp.data_ptr(), 3000, heavy.data_ptr(),
                                          heavy.numel(), out3.data_ptr(), 512, 512,
                                          torch.cuda.current_stream().cuda_stream), "segsum_heavy")
  torch.testing.assert_close(out3.double(), want, rtol=1e-5, atol=2e-3)
  assert torch.equal(out3[5], out[5]) and torch.equal(out3[100], out[100])
  out4 = torch.empty_like(out3)
  lib.gcb_segment_sum_heavy(msg.data_ptr(), 512, rp.data_ptr(), 3000, heavy.data_ptr(), heavy.numel(),
                            out4.data_ptr(), 512, 512, torch.cuda.current_stream().cuda_stream)
  assert torch.equal(out3, out4)


def test_halo_row_packing_fp32_rows_and_image_rows():
  """Send / receive side of the halo exchange (graphcast_b200/partitioned.py): gcb_gather_rows on an
  fp32 table, and gcb_image_rows_pack / _unpack on an operand image -- the unpacked image rows must be
  the packed rows' bytes (the receiver holds the owner's image rows bit for bit)."""
  lib = _native.lib()
  st = torch.cuda.current_stream().cuda_stream
  g = torch.Generator().manual_seed(5)
  rows, n = 1000, 333                                   # ragged: not multiples of the 128-row tile
  x = torch.randn(rows, 512, generator=g).to("cuda:0")
  idx = torch.randperm(rows, generator=g)[:n].to(torch.int32).to("cuda:0")
  dense = torch.empty(n, 512, device="cuda:0")
  _native.check(lib.gcb_gather_rows(x.data_ptr(), 512, idx.data_ptr(), n, dense.data_ptr(), 512, 512,
                                    st), "gather_rows")
  assert torch.equal(dense, x[idx.long()])

  def image_of(t, r):
    img = torch.zeros(lib.gcb_a_image_bytes(r, 512), dtype=torch.uint8, device="cuda:0")
    _native.check(lib.gcb_rows_to_image(t.data_ptr(), 512, 1, r, 512, img.data_ptr(), st), "image")
    return img

  img = image_of(x, rows)
  buf = torch.zeros(n, 2048, dtype=torch.uint8, device="cuda:0")
  _native.check(lib.gcb_image_rows_pack(img.data_ptr(), idx.data_ptr(), n, buf.data_ptr(), st), "pack")
  # receiver: rows 256.. of a second image (a halo block behind 256 owned rows)
  first = 256
  other = torch.randn(first + n, 512, generator=g).to("cuda:0")
  img2 = image_of(other, first + n)
  untouched = img2.clone()
  _native.check(lib.gcb_image_rows_unpack(buf.data_ptr(), n, img2.data_ptr(), first, st), "unpack")
  expect = image_of(torch.cat([other[:first], x[idx.long()]]), first + n)
  torch.cuda.synchronize()
  assert torch.equal(img2, expect)
  tile0 = 32 * 8448 * (first // 128)
  assert torch.equal(img2[:tile0], untouched[:tile0])   # owned tiles untouched
  # n = 0 is a no-op, bad arguments are refused
  assert lib.gcb_image_rows_pack(img.data_ptr(), idx.data_ptr(), 0, buf.data_ptr(), st) == 0
  assert lib.gcb_image_rows_unpack(buf.data_ptr(), -1, img2.data_ptr(), 0, st) != 0
