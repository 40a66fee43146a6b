"""Timeline of CTA 0 for one fused-layer launch (debug aid).

  python tools/trace_layer.py            # six layer shapes, 1184 tiles
  python tools/trace_layer.py big        # two image-fed shapes at 3.0M rows (HBM resident)
  python tools/trace_layer.py cluster    # cluster 1 vs 2

Columns: cycles (clock64) of consumer warp 4 for the first units of CTA 0 (wait for the first
operands, MMA phase and its cycles per K-step against the tensor-pipe ideal, LayerNorm statistics,
epilogue stores), plus the cycles the TMA warp spent waiting on `empty` barriers (tma_blocked)."""
import ctypes as C, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from graphcast_b200 import _native
lib = _native.lib()
dev = torch.device("cuda:0")

def run(rows, k, n, ln, act, csize, out_y=False, residual=False, idx=False, pre=0, img_in=False, img_out=False):
  lib.gcb_set_cluster_size(csize)
  a = torch.randn(rows, k, device=dev)
  w = (torch.randn(k, n) / np.sqrt(k)).numpy().astype(np.float32)
  img = np.empty(lib.gcb_packed_weight_bytes(k, n), np.uint8)
  lib.gcb_pack_weight_host(w.ctypes.data, k, n, k, n, img.ctypes.data)
  img_d = torch.as_tensor(img).to(dev)
  bias = torch.zeros(n, device=dev); sc = torch.ones(n, device=dev); of = torch.zeros(n, device=dev)
  out = torch.empty(rows, n, device=dev); oy = torch.empty(rows, 512, device=dev); res = torch.randn(rows, n, device=dev)
  d = _native.LayerDesc()
  d.rows, d.n, d.n_valid, d.nseg = rows, n, n, 1
  d.seg[0].table, d.seg[0].ld, d.seg[0].k, d.seg[0].k_valid, d.seg[0].fan = a.data_ptr(), k, k, k, 1
  if idx:
    ix = torch.randint(0, rows, (rows,), dtype=torch.int32, device=dev); d.seg[0].idx = ix.data_ptr()
  d.w_packed, d.bias = img_d.data_ptr(), bias.data_ptr()
  if ln: d.ln_scale, d.ln_offset = sc.data_ptr(), of.data_ptr()
  d.act = 1 if act else 0
  d.out, d.ld_out = out.data_ptr(), n
  if out_y: d.out_y, d.ld_out_y = oy.data_ptr(), 512
  if residual: d.residual, d.ld_res = res.data_ptr(), n
  d.precision = 0
  if img_in:
    ai = torch.zeros(lib.gcb_a_image_bytes(rows, k), dtype=torch.uint8, device=dev)
    d.seg[0].img, d.seg[0].k, d.nseg = ai.data_ptr(), k, 1
  if img_out:
    oi = torch.zeros(lib.gcb_a_image_bytes(rows, n), dtype=torch.uint8, device=dev)
    d.out_img, d.out, = oi.data_ptr(), None
  if pre:
    ptab = [torch.randn(40962, 512, device=dev) for _ in range(pre)]
    pidx = [torch.sort(torch.randint(0, 40962, (rows,), dtype=torch.int32, device=dev))[0] if i else
            torch.randint(0, 40962, (rows,), dtype=torch.int32, device=dev) for i in range(pre)]
    d.n_pre_add = pre
    for i in range(pre):
      d.pre_add[i].table, d.pre_add[i].idx, d.pre_add[i].ld = ptab[i].data_ptr(), pidx[i].data_ptr(), 512
  tr = torch.zeros(64 * 16, dtype=torch.int64, device=dev)
  for _ in range(2):
    lib.gcb_layer_forward(C.byref(d), None)
  torch.cuda.synchronize()
  lib.gcb_debug_trace(tr.data_ptr())
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record(); lib.gcb_layer_forward(C.byref(d), None); e1.record()
  torch.cuda.synchronize()
  lib.gcb_debug_trace(None)
  t = tr.cpu().numpy().reshape(64, 16)
  ntile = min(64, (rows + 127) // 128 // 132)
  print(f"rows={rows} k={k} n={n} ln={ln} act={act} cluster={csize} out_y={out_y} res={residual} idx={idx} pre={pre} img_in={img_in} img_out={img_out}: {e0.elapsed_time(e1):.3f} ms; tiles/CTA~{ntile}")
  base = t[1, 0]
  ideal = 128 * (6 if d.precision == 0 else 2)   # tensor cycles per K-step: bf16x3 | bf16, 2 warpgroups
  for i in range(1, min(ntile, 6)):
    r = t[i]
    mma = r[3] - r[1]
    ln = r[4] - r[3] if r[4] > 0 else 0
    print(f"  unit {i}: start@{r[0]-base:8d} ops_ready+{r[1]-r[0]:6d} mma+{mma:7d} "
          f"({mma / max(r[9], 1):5.0f}/K-step, ideal {ideal}) | ln_stats+{ln:6d} stored+{r[5]-max(r[4], r[3]):6d} | "
          f"next unit+{t[i+1,0]-r[0]:7d} | tma_blocked={r[7]}")

import sys
big = len(sys.argv) > 1 and sys.argv[1] in ("big", "cluster")
if len(sys.argv) > 1 and sys.argv[1] == "cluster":
  for cs in (1, 2):
    print("== cluster", cs)
    run(132 * 128 * 160, 512, 512, False, True, cs, img_in=True, img_out=True)
    run(132 * 128 * 160, 512, 512, True, False, cs, img_in=True)
  sys.exit(0)
rows = 132 * 128 * (160 if big else 8)
for cs in (2,):
  run(rows, 512, 512, False, True, cs, img_in=True, img_out=True)
  run(rows, 512, 512, True, False, cs, img_in=True)
  if not big:
    run(rows, 512, 512, False, True, cs, img_out=True)
    run(rows, 512, 512, False, True, cs, pre=2, img_in=True, img_out=True)
    run(rows, 512, 512, True, False, cs, out_y=True, residual=True, img_in=True)
    run(rows, 1536, 512, False, True, cs, idx=True, img_out=True)
