"""Fused chain vs layer-by-layer launches on MLP-shaped problems (debug / attribution aid).

  python tools/trace_chain.py [rows] [lag]

For an edge-MLP-shaped problem (image A operand + two gathered addends -> swish -> LN + residual,
fp32 + image outputs) and a node-MLP-shaped one it prints: NaN diagnostics, bitwise equality of
the two paths, CUDA-event times, and the in-kernel timeline of cluster 0 / CTA 0 of the chain
launch (cycles; per executed unit: barrier waits, MMA phase per K-step against the 768-cycle
tensor-pipe ideal, LayerNorm statistics, epilogue stores, scratch hand-over).  The "edge-table" case
is the edge problem with the first layer's accumulator read from a table (gcb_chain_layer.acc_table,
filled by an acc_out chain) instead of computed: its layer-0 units have no MMAs; their operand wait
is the wait for the first stage of table rows, and their "mma" column the walk over the rest."""
import ctypes as C, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np, torch
from graphcast_b200 import _native
import test_gpu_chain as tc

lib = _native.lib()
rows = int(sys.argv[1]) if len(sys.argv) > 1 else 327660
lag = int(sys.argv[2]) if len(sys.argv) > 2 else 1
DEV = "cuda:0"


def timed(fn, reps=5):
  fn(); torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(reps):
    fn()
  e1.record(); torch.cuda.synchronize()
  return e0.elapsed_time(e1) / reps


IMG_RES = len(sys.argv) > 3 and sys.argv[3] == "img"


def case(kind, table=False):
  g = torch.Generator().manual_seed(5)
  f = lambda *shape: torch.randn(*shape, generator=g)
  n_nodes = 40962
  pre = []
  if kind == "edge":
    x = f(rows, 512); xd = x.to(DEV)
    segs = [tc._seg_img(tc._image(lib, xd, rows, 512), 512)]
    k = 512
    pa, pb = f(n_nodes, 512).to(DEV), f(n_nodes, 512).to(DEV)
    ia = torch.randint(0, n_nodes, (rows,), generator=g, dtype=torch.int32).to(DEV)
    ib = torch.sort(torch.randint(0, n_nodes, (rows,), generator=g, dtype=torch.int32))[0].to(DEV)
    pre = [(pa, ia), (pb, ib)]
  else:
    x, a = f(rows, 512).to(DEV), f(rows, 512).to(DEV)
    segs = [tc._seg_img(tc._image(lib, x, rows, 512), 512), tc._seg_img(tc._image(lib, a, rows, 512), 512)]
    k = 1024
  l0 = tc.Layer(lib, k, k, g, ln=False)
  l1 = tc.Layer(lib, 512, 512, g, ln=True)
  res = f(rows, 512).to(DEV)
  nan = lambda: torch.full((rows, 512), float("nan"), device=DEV)
  hidden = torch.zeros(lib.gcb_a_image_bytes(rows, 512), dtype=torch.uint8, device=DEV)
  o1, y1, o2, y2 = nan(), nan(), nan(), nan()
  img1, img2 = torch.zeros_like(hidden), torch.zeros_like(hidden)

  def unfused():
    tc._layer_forward(lib, "bf16x3", rows, segs, l0, act=True, out_img=hidden, pre=pre)
    tc._layer_forward(lib, "bf16x3", rows, [tc._seg_img(hidden, 512)], l1, act=False, residual=res,
                      out=o1, out_y=y1, out_img=img1)

  scratch = tc._scratch(lib, 1, lag, 1)
  ch = _native.ChainDesc()
  ch.rows, ch.nlayers, ch.precision, ch.lag = rows, 2, 0, lag
  ch.scratch, ch.scratch_bytes = scratch.data_ptr(), scratch.numel()
  tc._fill_chain_layer(ch.layer[0], segs, [-1] * len(segs), l0, act=True, keep=True, pre=pre)
  if IMG_RES:     # latent as image only: residual read back from the image, updated in place
    img2.copy_(tc._image(lib, res, rows, 512))
    tc._fill_chain_layer(ch.layer[1], [None], [0], l1, act=False, keep=False, out_y=y2, out_img=img2)
    ch.layer[1].residual_img = img2.data_ptr()
  else:
    tc._fill_chain_layer(ch.layer[1], [None], [0], l1, act=False, keep=False, residual=res, out=o2,
                         out_y=y2, out_img=img2)

  if table:
    acc = nan()
    tab = _native.ChainDesc()
    tab.rows, tab.nlayers, tab.precision, tab.lag = rows, 1, 0, lag
    tab.scratch, tab.scratch_bytes = scratch.data_ptr(), scratch.numel()
    tc._fill_chain_layer(tab.layer[0], segs, [-1] * len(segs), l0, act=False, keep=False, out=acc)
    tab.layer[0].bias, tab.layer[0].acc_out = None, 1
    _native.check(lib.gcb_chain_forward(C.byref(tab), None), "acc_out chain")
    cl = ch.layer[0]
    cl.nseg, cl.w_packed, cl.seg_from[0] = 0, None, -1
    cl.acc_table, cl.ld_acc = acc.data_ptr(), 512
    kind += "-table"

  def fused():
    _native.check(lib.gcb_chain_forward(C.byref(ch), None), "chain")

  t_u, t_f = timed(unfused), timed(fused)
  for name, t in (("o1", o1), ("y1", y1), ("o2", o2), ("y2", y2)):
    bad = ~torch.isfinite(t)
    if bad.any():
      r = bad.any(1).nonzero().flatten()
      print(f"  {name}: {int(bad.sum())} non-finite values in {r.numel()} rows, first rows {r[:8].tolist()}, last {r[-3:].tolist()}")
  print(f"{kind}: rows={rows} lag={lag}: unfused {t_u:.3f} ms, fused {t_f:.3f} ms; "
        f"bitwise out {torch.equal(o1, o2)} out_y {torch.equal(y1, y2)} "
        f"img {torch.equal(img1[:(rows // 128) * 32 * 8448], img2[:(rows // 128) * 32 * 8448])}")
  tr = torch.zeros(64 * 16, dtype=torch.int64, device=DEV)
  lib.gcb_debug_trace(tr.data_ptr())
  fused(); torch.cuda.synchronize()
  lib.gcb_debug_trace(None)
  print_timeline(tr.cpu().numpy().reshape(64, 16))


IDEAL_KSTEP = 768   # tensor cycles per K-step and CTA: 6 x m64n256k16 (bf16x3, 2 warpgroups) at 128


def print_timeline(t):
  """Events: see the trace comment in graphcast_b200/csrc/mlp_tc.cuh.  Cycles after the previous
  event of the same unit; per K-step = MMA phase (first full barrier -> MMAs retired) / K-steps.  A
  table unit (0 K-steps) reads its stages of table rows before the h_free wait: its "ops_ready" is the
  wait for the first stage after the unit start, and its "mma" the walk over the stages plus the
  h_free wait."""
  base = t[2, 0]
  print("   u L | start  h_free  ops_ready  mma (per K-step / ideal) | ln_stats  columns  handed"
        " | next unit | tma: blocked h_full_wait")
  tot = np.zeros(8)
  per_layer = {}
  for u in range(2, 14):
    r = t[u]
    if r[9] > 0:
      hfree, ops, mma = r[2] - r[0], r[1] - r[2], r[3] - r[1]
    elif r[1] > 0:
      hfree, ops, mma = 0, r[1] - r[0], r[3] - r[1]
    else:                                # table read by the consumers' own global loads: no stages
      hfree, ops, mma = r[2] - r[0], 0, 0
    ln = r[4] - r[3] if r[4] > 0 else 0
    stored = r[5] - max(r[4], r[3])      # column loop
    handed = r[6] - r[5]                 # last store issued -> h_full arrives done
    nxt = t[u + 1, 0] - r[0]
    tot += [hfree, ops, mma if r[9] > 0 else 0, ln + stored + handed, nxt, r[9], stored, handed]
    per_layer.setdefault(int(r[11]), []).append((nxt, stored, ops, mma, r[9]))
    per_k = f"{mma / r[9]:6.0f}" if r[9] > 0 else " table"
    print(f"  {u:2d} {r[11]} | {r[0]-base:8d} +{hfree:6d} +{ops:6d} +{mma:7d} ({per_k} / {IDEAL_KSTEP}) | "
          f"+{ln:6d} +{stored:7d} +{handed:6d} | +{nxt:7d} | {r[7]:7d} {r[8]:7d}")
  print(f"  units 2-13: h_free wait {tot[0]:.0f}, operand wait {tot[1]:.0f}, MMA {tot[2]:.0f} "
        f"({tot[2] / max(tot[5], 1):.0f} cycles per K-step vs {IDEAL_KSTEP}), epilogue + hand-over {tot[3]:.0f}, "
        f"unit to unit {tot[4]:.0f} cycles")
  print(f"  epilogue of units 2-13: column loop {tot[6]:.0f}, last store -> h_full arrive {tot[7]:.0f} cycles")
  for l, v in sorted(per_layer.items()):
    ks = sum(x[4] for x in v)
    phase = (f"MMA {sum(x[3] for x in v) / ks:.0f} cycles per K-step" if ks > 0 else
             f"table walk {np.mean([x[3] for x in v]):.0f} cycles")
    print(f"  layer {l}: {len(v)} units, mean unit to unit {np.mean([x[0] for x in v]):.0f} cycles, "
          f"mean column loop {np.mean([x[1] for x in v]):.0f} cycles, mean operand wait "
          f"{np.mean([x[2] for x in v]):.0f} cycles, {phase}")


case("edge")
case("edge", table=True)
case("node")
