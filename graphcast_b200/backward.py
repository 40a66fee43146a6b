"""Parameter gradients of one step's forecast loss on the device (Engine.loss_and_grads).

The forward runs stage by stage (gcb_forward_stage, bit-identical to gcb_forward) and keeps what the
backward pass reads: the operand images of the latents after every stage and the aggregates.  The
backward pass then walks decoder, processor steps (last first) and encoder, following the forward of
SURVEY.md appendix A:

  * every MLP y = LN(swish(X W0 + b0) W1 + b1) is recomputed layer by layer with gcb_layer_forward
    (h, swish(h), z: bit-identical to the fused chains by the header's guarantee) and differentiated
    with gcb_layernorm_backward / gcb_swish_backward (column sums -> bias, scale, offset),
    gcb_weight_grad (dW = X^T G) and gcb_layer_forward with the transposed packed weight (dX);
  * the first edge layer stays in its pre-gathered form [e | v_s | v_r] W = e W_e + (v W_s)[snd] +
    (v W_r)[rcv]: with dH its pre-activation gradient, S / R = dH summed by sender / receiver are
    node tables (gcb_segment_sum_sorted / gcb_segment_sum_heavy), dW_s = v^T S, dW_r = v^T R,
    dW_e = e^T dH, dv += S W_s^T + R W_r^T, de = dH W_e^T -- no [E, 1536] tensor is formed;
  * residuals v' = v + N([v | agg]) and e' = e + m: the aggregate is of m (not e + m), the edge MLP
    sees the pre-update nodes; the grid2mesh edge residual and the mesh2grid mesh-node MLP are dead,
    their parameters get exact zeros;
  * inputs (grid features, mesh zeros + structural, edge features) are constants: their MLPs get dW,
    never dX.

All arithmetic is in libgraphcast_b200.so; this module only sequences the launches and owns the
buffers.  Allocation is lazy: nothing here exists until the first loss_and_grads call.
"""

from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional

import numpy as np
import torch

from graphcast_b200 import _native
from graphcast_b200 import graph as graph_lib

D = 512


def _stem(gnn: str, prefix: str, set_name: str) -> str:
  return f"{gnn}/~_networks_builder/{prefix}{set_name}"


class _MlpInfo:
  """One MLP of the model: forward weights (from the engine's gcb_model), transposed packed weights
  for the dX products, and its gradient buffers."""

  def __init__(self, stem: str, w: "_native.Mlp", k_segs: List[int], ln: bool, n1: int, n1_valid: int,
               split: Optional["_native.MlpSplit"] = None):
    self.stem, self.w, self.k_segs, self.ln = stem, w, k_segs, ln
    self.n1, self.n1_valid, self.split = n1, n1_valid, split
    self.g: Dict[str, torch.Tensor] = {}
    self.t: Dict[str, torch.Tensor] = {}     # transposed packed weights


class Backward:
  """Gradient workspace and launch sequence of one Engine (created on the first loss_and_grads)."""

  def __init__(self, eng, params, chunk_rows: int = 1 << 19):
    if not eng.pregather:
      raise NotImplementedError("parameter gradients need the pre-gathered edge layers (pregather=True)")
    self.eng = eng
    self.lib = eng._lib
    self.m = eng._model
    dev = eng.device
    self.dev = dev
    m = self.m
    cin = eng.c_in_pad
    specs = [
        ("enc_grid", _stem("grid2mesh_gnn", "encoder_nodes_", "grid_nodes"), [cin], None),
        ("enc_mesh", _stem("grid2mesh_gnn", "encoder_nodes_", "mesh_nodes"), [cin], None),
        ("enc_e_g2m", _stem("grid2mesh_gnn", "encoder_edges_", "grid2mesh"), [16], None),
        ("proc_e_g2m", _stem("grid2mesh_gnn", "processor_edges_0_", "grid2mesh"), [D] * 3,
         m.proc_e_g2m_split),
        ("proc_n_mesh_g2m", _stem("grid2mesh_gnn", "processor_nodes_0_", "mesh_nodes"), [D] * 2, None),
        ("proc_n_grid_g2m", _stem("grid2mesh_gnn", "processor_nodes_0_", "grid_nodes"), [D], None),
        ("enc_e_mesh", _stem("mesh_gnn", "encoder_edges_", "mesh"), [16], None),
        ("enc_e_m2g", _stem("mesh2grid_gnn", "encoder_edges_", "mesh2grid"), [16], None),
        ("proc_e_m2g", _stem("mesh2grid_gnn", "processor_edges_0_", "mesh2grid"), [D] * 3,
         m.proc_e_m2g_split),
        ("proc_n_grid_m2g", _stem("mesh2grid_gnn", "processor_nodes_0_", "grid_nodes"), [D] * 2, None),
        ("dec_grid", _stem("mesh2grid_gnn", "decoder_nodes_", "grid_nodes"), [D], None),
    ]
    self.mlps: Dict[str, _MlpInfo] = {}
    for key, stem, ks, split in specs:
      w = getattr(m, key)
      self.mlps[key] = _MlpInfo(stem, w, ks, key != "dec_grid", w.n1, w.n1_valid, split)
    self.proc_e = [_MlpInfo(_stem("mesh_gnn", f"processor_edges_{k}_", "mesh"), m.proc_e_mesh[k],
                            [D] * 3, True, D, D, m.proc_e_mesh_split[k]) for k in range(eng.msg_steps)]
    self.proc_n = [_MlpInfo(_stem("mesh_gnn", f"processor_nodes_{k}_", "mesh_nodes"), m.proc_n_mesh[k],
                            [D] * 2, True, D, D) for k in range(eng.msg_steps)]
    self.params = params
    self._all = list(self.mlps.values()) + self.proc_e + self.proc_n
    for info in self._all:
      self._pack_transposed(info)
      self._alloc_grads(info)
    # sender CSR of the three edge sets (execution order), receiver rows of mesh2grid (fan-in 3)
    self.csr = {"mesh": self._csr(eng.exec_senders["mesh"], m.num_mesh)}
    self.m2g_row_ptr = self._i32(np.arange(0, 3 * m.num_grid + 1, 3))
    # The bipartite edge sets (3.1 M mesh2grid and 1.6 M grid2mesh edges at 0.25 degree) are
    # differentiated in chunks of at most `chunk_rows` edges whose boundaries fall on receiver
    # boundaries (for mesh2grid: grid nodes, 3 edges each), so that every receiver sum is complete
    # inside its chunk; the sender sums of the chunks are added in chunk order.
    self.chunk_rows = int(chunk_rows)
    self.chunks = {
        "m2g": self._chunks(np.arange(0, 3 * m.num_grid + 1, 3, dtype=np.int64),
                            eng.exec_senders["m2g"], m.num_mesh),
        "g2m": self._chunks(eng.exec_row_ptr["g2m"].astype(np.int64), eng.exec_senders["g2m"],
                            m.num_grid),
    }
    self.iota = self._i32(np.arange(max(m.num_grid, m.num_mesh)))
    self.zero_bias = torch.zeros([D], dtype=torch.float32, device=dev)
    self.prec = _native.PRECISIONS[eng.precision]
    self.ws_rows = torch.empty([max(self.lib.gcb_rowwise_workspace_bytes(D), 16)], dtype=torch.uint8, device=dev)
    nb = self.lib.gcb_weight_grad_workspace_bytes(D, D)     # the largest single call: k = n = 512
    self.ws_wg = torch.empty([nb], dtype=torch.uint8, device=dev)

  # -- setup ---------------------------------------------------------------------------------
  def _i32(self, a):
    return torch.as_tensor(np.ascontiguousarray(a, np.int32)).to(self.dev)

  def _csr(self, senders: np.ndarray, n_nodes: int):
    order, ptr, heavy = graph_lib.sender_csr(senders, n_nodes)
    return (self._i32(order), self._i32(ptr),
            self._i32(heavy if heavy.size else np.zeros([1], np.int32)), int(heavy.size))

  def _chunks(self, row_ptr: np.ndarray, senders: np.ndarray, n_senders: int):
    """Receiver-aligned chunks of a bipartite edge set: (r0, r1, g0, g1, local receiver row_ptr,
    local heavy receivers, count, sender CSR of the chunk's edges)."""
    out = []
    n_rcv = row_ptr.shape[0] - 1
    g0 = 0
    while g0 < n_rcv:
      # the last receiver whose edges still fit (at least one receiver per chunk)
      g1 = int(np.searchsorted(row_ptr, row_ptr[g0] + self.chunk_rows, side="right")) - 1
      g1 = min(max(g1, g0 + 1), n_rcv)
      r0, r1 = int(row_ptr[g0]), int(row_ptr[g1])
      rp = row_ptr[g0:g1 + 1] - row_ptr[g0]
      heavy = np.nonzero(np.diff(rp) > 256)[0].astype(np.int32)
      out.append((r0, r1, g0, g1, self._i32(rp),
                  self._i32(heavy if heavy.size else np.zeros([1], np.int32)), int(heavy.size),
                  self._csr(senders[r0:r1], n_senders)))
      g0 = g1
    return out

  def _pack(self, w: np.ndarray, k_pad: int, n_pad: int) -> torch.Tensor:
    w = np.ascontiguousarray(w, np.float32)
    nbytes = self.lib.gcb_packed_weight_bytes(k_pad, n_pad)
    img = np.empty([nbytes], np.uint8)
    _native.check(self.lib.gcb_pack_weight_host(w.ctypes.data, w.shape[0], w.shape[1], k_pad, n_pad,
                                                img.ctypes.data), "gcb_pack_weight_host")
    return torch.as_tensor(img).to(self.dev)

  def _pack_transposed(self, info: _MlpInfo) -> None:
    p = self.params
    w1 = np.asarray(p[f"{info.stem}_mlp/~/linear_1"]["w"], np.float32)       # [512, n1_valid]
    info.t["w1"] = self._pack(w1.T, info.n1, D)                               # [n1, 512]
    w0 = np.asarray(p[f"{info.stem}_mlp/~/linear_0"]["w"], np.float32)
    if len(info.k_segs) >= 2 and w0.shape[0] == len(info.k_segs) * D:
      for s in range(len(info.k_segs)):
        info.t[f"w0_{s}"] = self._pack(w0[s * D:(s + 1) * D].T, D, D)        # block s, transposed
    elif w0.shape[0] == D:
      info.t["w0_0"] = self._pack(w0.T, D, D)

  def input_transposed(self):
    """(packed [512, n] transpose of the grid embedder's first layer, n): the dX product of the grid
    inputs (backprop through time), n = 256 | 512 >= c_in_pad.  Packed on first use, so the one-step
    gradient never holds it."""
    info = self.mlps["enc_grid"]
    if "w0_in" not in info.t:
      cin = self.eng.c_in_pad
      if cin > 2 * 256:
        raise NotImplementedError(f"input gradients support at most 512 padded input channels, "
                                  f"not {cin}")
      n = 256 if cin <= 256 else 512
      w0 = np.asarray(self.params[f"{info.stem}_mlp/~/linear_0"]["w"], np.float32)   # [c_in + 3, 512]
      info.t["w0_in"] = self._pack(w0.T, D, n)
      self.n_in_t = n
    return info.t["w0_in"], self.n_in_t

  def _alloc_grads(self, info: _MlpInfo) -> None:
    z = lambda *s: torch.zeros(list(s), dtype=torch.float32, device=self.dev)
    info.g = {"w0": z(sum(info.k_segs), D), "b0": z(D), "w1": z(D, info.n1), "b1": z(info.n1)}
    if info.ln:
      info.g["scale"], info.g["offset"] = z(D), z(D)

  def zero_grads(self) -> None:
    for info in self._all:
      for t in info.g.values():
        t.zero_()

  # -- launch helpers ------------------------------------------------------------------------------
  def _st(self) -> int:
    return torch.cuda.current_stream(self.dev).cuda_stream

  @staticmethod
  def img(t: torch.Tensor, k: int = D):
    return ("img", t, k)

  @staticmethod
  def tab(t: torch.Tensor, k: int = D, k_valid: Optional[int] = None, ld: Optional[int] = None):
    return ("tab", t, k, k_valid or k, ld or t.shape[1])

  def layer(self, rows: int, segs, w_packed, bias, act: int = _native.ACT_NONE, *,
            out_y: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
            residual: Optional[torch.Tensor] = None, ln=None, pre=None, n: int = D,
            n_valid: Optional[int] = None) -> None:
    d = _native.LayerDesc()
    d.rows, d.n, d.n_valid, d.nseg = rows, n, n_valid or n, len(segs)
    for i, s in enumerate(segs):
      g = d.seg[i]
      if s[0] == "img":
        g.img, g.k = s[1].data_ptr(), s[2]
      else:
        g.table, g.k, g.k_valid, g.ld, g.fan = s[1].data_ptr(), s[2], s[3], s[4], 1
    d.w_packed = w_packed if isinstance(w_packed, int) else w_packed.data_ptr()
    d.bias = bias if isinstance(bias, int) else bias.data_ptr()
    if ln is not None:
      d.ln_scale, d.ln_offset = ln
    d.act = act
    if residual is not None:
      d.residual, d.ld_res = residual.data_ptr(), residual.shape[1]
    if out is not None:
      d.out, d.ld_out = out.data_ptr(), out.shape[1]
    if out_y is not None:
      d.out_y, d.ld_out_y = out_y.data_ptr(), out_y.shape[1]
    d.precision = self.prec
    if pre is not None:
      d.n_pre_add = len(pre)
      for i, (table, idx) in enumerate(pre):
        d.pre_add[i].table, d.pre_add[i].idx, d.pre_add[i].ld = table.data_ptr(), idx.data_ptr(), D
    _native.check(self.lib.gcb_layer_forward(C.byref(d), self._st()), "gcb_layer_forward")

  def empty(self, rows: int, cols: int = D) -> torch.Tensor:
    return torch.empty([max(rows, 1), cols], dtype=torch.float32, device=self.dev)

  def wgrad(self, x, g: torch.Tensor, rows: int, dw: torch.Tensor, *, n: int = D, swish: bool = False):
    """dw += X^T g (X an image or fp32 table segment, dw a contiguous [k, n] view)."""
    if x[0] == "img":
      xp, ld, kv, img, k = None, 0, 0, x[1].data_ptr(), x[2]
    else:
      xp, k, kv, ld, img = x[1].data_ptr(), x[2], x[3], x[4], None
    assert dw.is_contiguous() and tuple(dw.shape) == (k, n)
    _native.check(self.lib.gcb_weight_grad(
        xp, ld, kv, img, 1 if swish else 0, g.data_ptr(), g.shape[1], rows, k, n, self.prec,
        self.ws_wg.data_ptr(), self.ws_wg.numel(), dw.data_ptr(), 1, self._st()), "gcb_weight_grad")

  # -- MLP forward recompute and backward ------------------------------------------------------------
  def fwd_mlp(self, info: _MlpInfo, rows: int, segs) -> torch.Tensor:
    """y = LN(swish(X W0 + b0) W1 + b1) in fp32 (an embedder output the forward kept on chip)."""
    w = info.w
    a = self.empty(rows)
    self.layer(rows, segs, w.w0_packed, w.b0, _native.ACT_SWISH, out_y=a)
    y = self.empty(rows)
    self.layer(rows, [self.tab(a)], w.w1_packed, w.b1, out_y=y, ln=(w.ln_scale, w.ln_offset))
    return y

  def mlp_backward(self, info: _MlpInfo, rows: int, segs, dy: torch.Tensor, *, pre=None,
                   w0=None, dw_segs=None) -> torch.Tensor:
    """Backward of one MLP at the recomputed forward; accumulates its parameter gradients and returns
    dh [rows, 512], the gradient of the first layer's pre-activation (incl. pre-gathered addends).
    dw_segs: the layer-0 inputs whose weight blocks get X^T dh (default: all of `segs`)."""
    w = info.w
    h = self.empty(rows)
    self.layer(rows, segs, w0 or w.w0_packed, w.b0, _native.ACT_NONE, out_y=h, pre=pre)
    g = info.g
    ws = self.ws_rows
    if info.ln:
      a = self.empty(rows)
      _native.check(self.lib.gcb_swish_rows(h.data_ptr(), D, rows, D, a.data_ptr(), D, self._st()),
                    "gcb_swish_rows")
      z = self.empty(rows)
      self.layer(rows, [self.tab(a)], w.w1_packed, w.b1, out_y=z)
      del a
      dz = self.empty(rows)
      _native.check(self.lib.gcb_layernorm_backward(
          dy.data_ptr(), dy.shape[1], z.data_ptr(), D, w.ln_scale, rows, D, dz.data_ptr(), D,
          ws.data_ptr(), ws.numel(), g["b1"].data_ptr(), g["scale"].data_ptr(),
          g["offset"].data_ptr(), 1, self._st()), "gcb_layernorm_backward")
      del z
    else:
      dz = dy
      _native.check(self.lib.gcb_layernorm_backward(
          dy.data_ptr(), dy.shape[1], None, 0, None, rows, info.n1, None, 0, ws.data_ptr(),
          ws.numel(), g["b1"].data_ptr(), None, None, 1, self._st()), "gcb_layernorm_backward")
    self.wgrad(self.tab(h), dz, rows, g["w1"], n=info.n1, swish=True)     # dW1 = swish(h)^T dz
    da = self.empty(rows)
    self.layer(rows, [self.tab(dz, info.n1)], info.t["w1"], self.zero_bias, out_y=da)
    dh = self.empty(rows)
    _native.check(self.lib.gcb_swish_backward(
        da.data_ptr(), D, h.data_ptr(), D, rows, D, dh.data_ptr(), D, ws.data_ptr(), ws.numel(),
        g["b0"].data_ptr(), 1, self._st()), "gcb_swish_backward")
    del da, h
    off = 0
    for s in (dw_segs if dw_segs is not None else segs):
      k = s[2]
      self.wgrad(s, dh, rows, g["w0"][off:off + k])
      off += k
    return dh

  def seg_sum_sender(self, name: str, dh: torch.Tensor, num_nodes: int) -> torch.Tensor:
    order, ptr, heavy, n_heavy = self.csr[name]
    out = self.empty(num_nodes)
    _native.check(self.lib.gcb_segment_sum_sorted(
        dh.data_ptr(), D, order.data_ptr(), ptr.data_ptr(), num_nodes, heavy.data_ptr(), n_heavy,
        out.data_ptr(), D, D, self._st()), "gcb_segment_sum_sorted")
    return out

  def seg_sum_receiver(self, dh: torch.Tensor, row_ptr, num_nodes: int, heavy=None, n_heavy=0):
    out = self.empty(num_nodes)
    _native.check(self.lib.gcb_segment_sum_heavy(
        dh.data_ptr(), D, row_ptr.data_ptr(), num_nodes, heavy.data_ptr() if n_heavy else None,
        n_heavy, out.data_ptr(), D, D, self._st()), "gcb_segment_sum_heavy")
    return out

  def gather_add(self, src: torch.Tensor, idx: torch.Tensor, n: int,
                 addend: Optional[torch.Tensor] = None) -> torch.Tensor:
    out = self.empty(n)
    _native.check(self.lib.gcb_gather_add(
        src.data_ptr(), D, idx.data_ptr(), n, None if addend is None else addend.data_ptr(), D,
        out.data_ptr(), D, D, self._st()), "gcb_gather_add")
    return out

  def projection(self, rows: int, v, w_packed) -> torch.Tensor:
    out = self.empty(rows)
    self.layer(rows, [v], w_packed, self.zero_bias, out_y=out)
    return out

  def edge_backward(self, info: _MlpInfo, rows: int, e_seg, dm: torch.Tensor, snd_name: str,
                    v_s, n_s: int, snd: torch.Tensor, v_r, n_r: int, rcv: torch.Tensor,
                    rcv_sum) -> tuple:
    """Backward of a pre-gathered edge MLP m = MLP([e | v_s[snd] | v_r[rcv]]): accumulates its
    parameter gradients, returns (dH, S, R)."""
    sp = info.split
    ps = self.projection(n_s, v_s, sp.ws_packed)
    pr = self.projection(n_r, v_r, sp.wr_packed)
    dh = self.mlp_backward(info, rows, [e_seg], dm, pre=[(ps, snd), (pr, rcv)], w0=sp.we_packed)
    del ps, pr
    s = self.seg_sum_sender(snd_name, dh, n_s)
    r = rcv_sum(dh)
    w0 = info.g["w0"]
    self.wgrad(v_s, s, n_s, w0[D:2 * D])
    self.wgrad(v_r, r, n_r, w0[2 * D:3 * D])
    return dh, s, r

  def bipartite_backward(self, name: str, info: _MlpInfo, enc: _MlpInfo, feat_t: torch.Tensor,
                         dagg: torch.Tensor, snd: torch.Tensor, rcv: torch.Tensor, v_s, n_s: int,
                         v_r, n_r: int) -> tuple:
    """Backward of a grid2mesh / mesh2grid edge MLP m = MLP([e | v_s[snd] | v_r[rcv]]) with
    e = MLP(edge features) and dm = dagg[rcv] (its edge residual is dead), chunk by chunk (see
    self.chunks): accumulates the parameter gradients of both MLPs and returns the node tables
    (S [n_s, 512], R [n_r, 512]) of dH summed by sender / receiver."""
    sp = info.split
    ps = self.projection(n_s, v_s, sp.ws_packed)
    pr = self.projection(n_r, v_r, sp.wr_packed)
    s_tab, r_tab = None, self.empty(n_r)
    for r0, r1, g0, g1, rp, heavy, n_heavy, csr in self.chunks[name]:
      n = r1 - r0
      f = self.tab(feat_t[r0:r1], 16, 4, 4)                 # 16-byte rows: the view stays aligned
      snd_c, rcv_c = snd[r0:r1].clone(), rcv[r0:r1].clone()  # index arrays from an aligned base
      e = self.fwd_mlp(enc, n, [f])
      dm = self.gather_add(dagg, rcv_c, n)
      dh = self.mlp_backward(info, n, [self.tab(e)], dm, pre=[(ps, snd_c), (pr, rcv_c)],
                             w0=sp.we_packed)
      del dm, e, snd_c, rcv_c
      order, ptr, sh, n_sh = csr
      s_c = self.empty(n_s)
      _native.check(self.lib.gcb_segment_sum_sorted(
          dh.data_ptr(), D, order.data_ptr(), ptr.data_ptr(), n_s, sh.data_ptr(), n_sh,
          s_c.data_ptr(), D, D, self._st()), "gcb_segment_sum_sorted")
      s_tab = s_c if s_tab is None else self.gather_add(s_c, self.iota, n_s, s_tab)
      del s_c
      _native.check(self.lib.gcb_segment_sum_heavy(
          dh.data_ptr(), D, rp.data_ptr(), g1 - g0, heavy.data_ptr() if n_heavy else None, n_heavy,
          r_tab[g0:g1].data_ptr(), D, D, self._st()), "gcb_segment_sum_heavy")
      de = self.empty(n)
      self.layer(n, [self.tab(dh)], info.t["w0_0"], self.zero_bias, out_y=de)
      del dh
      self.mlp_backward(enc, n, [f], de)
      del de
    del ps, pr
    w0 = info.g["w0"]
    self.wgrad(v_s, s_tab, n_s, w0[D:2 * D])
    self.wgrad(v_r, r_tab, n_r, w0[2 * D:3 * D])
    return s_tab, r_tab

  # -- one batch element ---------------------------------------------------------------------------
  def element(self, grid_in_img: torch.Tensor, g_out: torch.Tensor, snaps: dict,
              dgrid_in: bool = False) -> Optional[torch.Tensor]:
    """Accumulates the parameter gradients of one batch element whose loss derivative with respect
    to the decoder output is g_out [Ng, 256] (gcb_output_loss_grad) and whose forward left `snaps`
    (whose entries are dropped as they are consumed).  dgrid_in: also return the derivative with
    respect to the packed grid inputs, dh_enc_grid W0^T [Ng, n] (see input_transposed; columns >=
    c_in + 3 are zero)."""
    eng, m = self.eng, self.m
    ng, nm = m.num_grid, m.num_mesh
    K = eng.msg_steps
    mp = self.mlps
    img, tab = self.img, self.tab
    feat = lambda t: tab(t, 16, 4, 4)

    # ---- decoder: out = MLP(vg2);  vg2 = vg1 + MLP([vg1 | agg3]);  m3 = MLP([e3 | v[snd] | vg1[rcv]])
    dh = self.mlp_backward(mp["dec_grid"], ng, [img(snaps["vg2"])], g_out)
    dvg2 = self.empty(ng)
    self.layer(ng, [tab(dh)], mp["dec_grid"].t["w0_0"], self.zero_bias, out_y=dvg2)
    info = mp["proc_n_grid_m2g"]
    dh = self.mlp_backward(info, ng, [img(snaps["vg1"]), img(snaps["agg3"])], dvg2)
    dvg1 = self.empty(ng)
    self.layer(ng, [tab(dh)], info.t["w0_0"], self.zero_bias, residual=dvg2, out=dvg1)
    dagg3 = self.empty(ng)
    self.layer(ng, [tab(dh)], info.t["w0_1"], self.zero_bias, out_y=dagg3)
    del dh, dvg2
    info = mp["proc_e_m2g"]
    S, R = self.bipartite_backward("m2g", info, mp["enc_e_m2g"], eng.m2g_feat, dagg3, eng.m2g_snd,
                                   eng.m2g_rcv, img(snaps["v"][K]), nm, img(snaps["vg1"]), ng)
    del dagg3
    # snapshots are released as soon as the backward pass is past their stage
    snaps["vg2"] = snaps["agg3"] = snaps["vg1"] = None
    dvg1_new = self.empty(ng)
    self.layer(ng, [tab(R)], info.t["w0_2"], self.zero_bias, residual=dvg1, out=dvg1_new)
    dvg1 = dvg1_new
    dv = self.empty(nm)
    self.layer(nm, [tab(S)], info.t["w0_1"], self.zero_bias, out_y=dv)
    del S, R

    # ---- processor, last step first:  m = MLP([e | v[snd] | v[rcv]]);  v' = v + MLP([v | agg]);
    #      e' = e + m
    de_next = None
    for k in range(K - 1, -1, -1):
      v_k = img(snaps["v"][k])
      agg_k = img(snaps["agg"][k])
      nfo, efo = self.proc_n[k], self.proc_e[k]
      dh_n = self.mlp_backward(nfo, nm, [v_k, agg_k], dv)
      dagg = self.empty(nm)
      self.layer(nm, [tab(dh_n)], nfo.t["w0_1"], self.zero_bias, out_y=dagg)
      dm = self.gather_add(dagg, eng.mesh_rcv, m.e_mesh, de_next)
      del dagg
      if k == 0:
        e0 = self.fwd_mlp(mp["enc_e_mesh"], m.e_mesh, [feat(eng.mesh_feat)])
        e_k = tab(e0)
      else:
        e_k = img(snaps["e"][k])
      dH, S, R = self.edge_backward(
          efo, m.e_mesh, e_k, dm, "mesh", v_k, nm, eng.mesh_snd, v_k, nm, eng.mesh_rcv,
          lambda d: self.seg_sum_receiver(d, eng.mesh_row_ptr, nm))
      del dm
      de = self.empty(m.e_mesh)              # de_k = de_{k+1} + dH W_e^T  (e' = e + m)
      if de_next is None:
        self.layer(m.e_mesh, [tab(dH)], efo.t["w0_0"], self.zero_bias, out_y=de)
      else:
        self.layer(m.e_mesh, [tab(dH)], efo.t["w0_0"], self.zero_bias, residual=de_next, out=de)
      del dH
      de_next = de
      # dv_k = dv_{k+1} + dh_n W0a^T + S W_s^T + R W_r^T
      dv_new = self.empty(nm)
      self.layer(nm, [tab(dh_n)], nfo.t["w0_0"], self.zero_bias, residual=dv, out=dv_new)
      dv2 = self.empty(nm)
      self.layer(nm, [tab(S)], efo.t["w0_1"], self.zero_bias, residual=dv_new, out=dv2)
      self.layer(nm, [tab(R)], efo.t["w0_2"], self.zero_bias, residual=dv2, out=dv_new)
      dv = dv_new
      del dh_n, S, R, dv2
      snaps["v"][k + 1] = snaps["agg"][k] = snaps["e"][k] = None
    # mesh edge embedder: e0 = MLP(edge features)
    self.mlp_backward(mp["enc_e_mesh"], m.e_mesh, [feat(eng.mesh_feat)], de_next)
    del de_next, e0

    # ---- encoder: vg1 = vg0 + MLP([vg0]);  vm1 = vm0 + MLP([vm0 | agg1]);
    #      m1 = MLP([e1 | vg0[snd] | vm0[rcv]]);  vg0 = MLP(grid_in);  vm0 = MLP(mesh_in)
    grid_in = img(grid_in_img, eng.c_in_pad)
    mesh_in = img(eng.mesh_in_img, eng.c_in_pad)
    vg0 = self.fwd_mlp(mp["enc_grid"], ng, [grid_in])
    vm0 = self.fwd_mlp(mp["enc_mesh"], nm, [mesh_in])
    info = mp["proc_n_grid_g2m"]
    dh = self.mlp_backward(info, ng, [tab(vg0)], dvg1)
    dvg0 = self.empty(ng)
    self.layer(ng, [tab(dh)], info.t["w0_0"], self.zero_bias, residual=dvg1, out=dvg0)
    del dh, dvg1
    info = mp["proc_n_mesh_g2m"]
    dh = self.mlp_backward(info, nm, [tab(vm0), img(snaps["agg1"])], dv)
    dvm0 = self.empty(nm)
    self.layer(nm, [tab(dh)], info.t["w0_0"], self.zero_bias, residual=dv, out=dvm0)
    dagg1 = self.empty(nm)
    self.layer(nm, [tab(dh)], info.t["w0_1"], self.zero_bias, out_y=dagg1)
    del dh, dv
    info = mp["proc_e_g2m"]
    S, R = self.bipartite_backward("g2m", info, mp["enc_e_g2m"], eng.g2m_feat, dagg1, eng.g2m_snd,
                                   eng.g2m_rcv, tab(vg0), ng, tab(vm0), nm)
    del dagg1
    t = self.empty(ng)
    self.layer(ng, [tab(S)], info.t["w0_1"], self.zero_bias, residual=dvg0, out=t)
    dvg0 = t
    t = self.empty(nm)
    self.layer(nm, [tab(R)], info.t["w0_2"], self.zero_bias, residual=dvm0, out=t)
    dvm0 = t
    del S, R, vg0, vm0
    dh = self.mlp_backward(mp["enc_grid"], ng, [grid_in], dvg0)
    dx = None
    if dgrid_in:
      w0t, n = self.input_transposed()
      dx = self.empty(ng, n)
      self.layer(ng, [tab(dh)], w0t, self.zero_bias, out_y=dx, n=n)
    del dh, dvg0
    self.mlp_backward(mp["enc_mesh"], nm, [mesh_in], dvm0)
    return dx

  # -- result ----------------------------------------------------------------------------------------
  def grads(self) -> Dict[str, Dict[str, torch.Tensor]]:
    """Device fp32 gradients keyed and shaped like the params; parameters the step never reads (the
    mesh2grid mesh-node MLP) get zeros."""
    out: Dict[str, Dict[str, torch.Tensor]] = {}
    for info in self._all:
      p = self.params
      l0, l1 = f"{info.stem}_mlp/~/linear_0", f"{info.stem}_mlp/~/linear_1"
      k_real = np.asarray(p[l0]["w"]).shape[0]
      g = info.g
      if len(info.k_segs) == 1:
        w0 = g["w0"][:k_real]
      else:
        w0 = g["w0"]
      n = info.n1_valid
      out[l0] = {"w": w0.clone(), "b": g["b0"].clone()}
      out[l1] = {"w": g["w1"][:, :n].clone(), "b": g["b1"][:n].clone()}
      if info.ln:
        out[f"{info.stem}_layer_norm"] = {"scale": g["scale"].clone(), "offset": g["offset"].clone()}
    for name, fields in self.params.items():
      if name not in out:
        out[name] = {f: torch.zeros(np.asarray(a).shape, dtype=torch.float32, device=self.dev)
                     for f, a in fields.items()}
    return out
