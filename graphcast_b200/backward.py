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

The tangent-linear model (input_jvp, batched_input_jvp) walks the same graph in forward order with the
same helpers (Backward.tangent): each stage of the stage-wise forward is followed by its tangent, every
MLP's tangent formed at its recomputed h and z (mlp_jvp; gcb_swish_jvp and gcb_layernorm_jvp_dirs for
the two nonlinearities).  Several tangent directions share that walk: their state is stacked
direction-major, so every tangent GEMM runs once over all of them and h and z are recomputed once.
Tangents along the parameters (param_jvp) walk the same graph with packed tangent weight images
(weight_tangents): every layer with one adds its weight-tangent GEMM X W-dot + b-dot at the primal
rows, and every LayerNorm scale-dot * zhat + offset-dot (gcb_layernorm_jvp_params).
Several cotangents (batched_input_vjp) share the backward walk the same way: element(dirs=K) stacks the
gradient state like the tangent's, runs every dX product once over all directions, and differentiates
the two nonlinearities with gcb_layernorm_backward_dirs and gcb_swish_jvp.
A parameter Hessian-vector product (loss_and_param_hvp) joins the two: the tangent along weight tangents keeps
its snapshots, and the two-direction walk element(hvp=..., param_grads=True) accumulates the gradient and its
tangent, with every layer's weight-tangent terms (mlp_backward, dx, wgrad_dot).  A joint one in the
parameters and the inputs (loss_and_joint_hvp) runs that walk along an input tangent as well, and also
forms the input gradient and its tangent, with the grid embedder's two coupling terms.

All arithmetic is in libgraphcast_b200.so; this module only sequences the launches and owns the
buffers.  Allocation is lazy: nothing here exists until the first loss_and_grads call.
"""

from __future__ import annotations

import ctypes as C
import weakref
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


class _WeightTangent:
  """The tangent of one MLP's parameters (param_jvp), packed as the engine packs its weights
  (Backward.weight_tangents): the tangent weight images at the engine's precision with the primal's
  padding, for a pre-gathered edge layer its split blocks (`split`: we / ws / wr) in place of w0, and the
  padded tangent biases and LayerNorm vectors.  A layer with no tangent has w0 / split / w1 None (a
  tangent bias alone comes with a zero weight image); a LayerNorm field with no tangent is None.
  w0_f32 / w1_f32: the padded fp32 tangent weights the images were packed from; `t`: their transposed
  images (Backward.pack_transposed_tangents, keyed as _MlpInfo.t), for the dX products of a parameter
  Hessian-vector product."""

  def __init__(self):
    self.w0 = self.split = self.b0 = self.w1 = self.b1 = self.scale = self.offset = None
    self.w0_f32 = self.w1_f32 = None
    self.t: Dict[str, torch.Tensor] = {}


class Backward:
  """Gradient workspace and launch sequence of one Engine (created on the first loss_and_grads)."""

  def __init__(self, eng, chunk_rows: int = 1 << 19):
    if not eng.pregather:
      raise NotImplementedError("parameter gradients need the pre-gathered edge layers (pregather=True)")
    # The engine owns this workspace: a weak reference, so that dropping the engine frees both at
    # once instead of leaving a cycle for the garbage collector.
    self.eng = weakref.proxy(eng)
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
    self.shapes = eng.param_shapes
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
    self._chunk_src = {
        "m2g": (np.arange(0, 3 * m.num_grid + 1, 3, dtype=np.int64), eng.exec_senders["m2g"],
                m.num_mesh),
        "g2m": (eng.exec_row_ptr["g2m"].astype(np.int64), eng.exec_senders["g2m"], m.num_grid),
    }
    self.chunks = {name: self._chunks(*src, self.chunk_rows) for name, src in self._chunk_src.items()}
    self.iota = self._i32(np.arange(max(m.num_grid, m.num_mesh)))
    self._edge_iota = None
    # the tangent of several directions (tangent(dirs=...)): their K-fold gather indices and chunks
    self.dirs = 1
    # kfold's indices: {fold count: {key: index}}, the two fold counts used last (a Hessian-vector
    # product's walk reads K-fold and (1 + K)-fold indices in one pass)
    self._kfold = {}
    self._tangent_chunks = {}
    self.zero_bias = torch.zeros([D], dtype=torch.float32, device=dev)
    self.prec = _native.PRECISIONS[eng.precision]
    self.ws_rows = torch.empty([max(self.lib.gcb_rowwise_workspace_bytes(D), 16)], dtype=torch.uint8, device=dev)
    nb = self.lib.gcb_weight_grad_workspace_bytes(D, D)     # the largest single call: k = n = 512
    self.ws_wg = torch.empty([nb], dtype=torch.uint8, device=dev)
    # element(param_grads=False): the column sums of the row-wise kernels land here, never in info.g
    self.param_grads = True
    # element(hvp=...): the tangent snapshots of the forward (tangent(snaps=...)) of self.tdirs = K
    # directions; the walk then carries the gradient (direction 0) and its K tangents (directions 1..K)
    self.hvp, self.tdirs = None, 0
    self.sink = {f: torch.zeros([D], dtype=torch.float32, device=dev)
                 for f in ("b0", "b1", "scale", "offset")}
    # tangent(wts=...): the packed parameter tangents of param_jvp, {MLP stem: _WeightTangent}
    self.wts: Dict[str, _WeightTangent] = {}
    # element(hvp=..., param_grads=True, wts=...): a parameter Hessian-vector product, whose gradient
    # tangents accumulate into info.gt (allocated by the first one, zero_hvp)
    self.phvp = False

  # -- setup ---------------------------------------------------------------------------------
  def _i32(self, a):
    return torch.as_tensor(np.ascontiguousarray(a, np.int32)).to(self.dev)

  def _csr(self, senders: np.ndarray, n_nodes: int):
    order, ptr, heavy = graph_lib.sender_csr(senders, n_nodes)
    return (self._i32(order), self._i32(ptr),
            self._i32(heavy if heavy.size else np.zeros([1], np.int32)), int(heavy.size))

  def _chunks(self, row_ptr: np.ndarray, senders: np.ndarray, n_senders: int, chunk_rows: int,
              csr: bool = True):
    """Receiver-aligned chunks of at most chunk_rows edges (at least one receiver) of a bipartite edge
    set: (r0, r1, g0, g1, local receiver row_ptr, local heavy receivers, count, sender CSR of the
    chunk's edges, or None without `csr`)."""
    out = []
    n_rcv = row_ptr.shape[0] - 1
    g0 = 0
    while g0 < n_rcv:
      # the last receiver whose edges still fit (at least one receiver per chunk)
      g1 = int(np.searchsorted(row_ptr, row_ptr[g0] + chunk_rows, side="right")) - 1
      g1 = min(max(g1, g0 + 1), n_rcv)
      r0, r1 = int(row_ptr[g0]), int(row_ptr[g1])
      rp = row_ptr[g0:g1 + 1] - row_ptr[g0]
      heavy = np.nonzero(np.diff(rp) > 256)[0].astype(np.int32)
      out.append((r0, r1, g0, g1, self._i32(rp),
                  self._i32(heavy if heavy.size else np.zeros([1], np.int32)), int(heavy.size),
                  self._csr(senders[r0:r1], n_senders) if csr else None))
      g0 = g1
    return out

  def _pack_t(self, info, key: str, w: int, ld: int, k: int, n: int, n_cols: int) -> None:
    """info.t[key] (an _MlpInfo or _WeightTangent) = the packed image of the transpose of the device fp32 matrix at address w (rows of
    `ld` floats), of padded shape [k, n] (n_cols real columns), written in place when it exists."""
    if key not in info.t:
      info.t[key] = torch.empty([self.lib.gcb_packed_weight_bytes(k, n)], dtype=torch.uint8,
                                device=self.dev)
    self.eng.pack_weight(w, ld, True, k, n_cols, k, n, info.t[key])

  def _pack_transposed(self, info: _MlpInfo) -> None:
    """Packs the transposed weights of one MLP on the device, from the engine's zero-padded fp32 weight
    buffers (so they follow every reload, from host or device): w1^T [n1, 512], and w0^T per 512-row
    block of the first layer."""
    w = info.w
    self._pack_t(info, "w1", w.w1_f32, info.n1, info.n1, D, D)
    k0 = self.shapes[f"{info.stem}_mlp/~/linear_0"]["w"][0]
    if len(info.k_segs) >= 2 and k0 == len(info.k_segs) * D:
      for s in range(len(info.k_segs)):
        self._pack_t(info, f"w0_{s}", w.w0_f32 + 4 * s * D * D, D, D, D, D)   # block s, transposed
    elif k0 == D:
      self._pack_t(info, "w0_0", w.w0_f32, D, D, D, D)
    if "w0_in" in info.t:                                  # the grid embedder's input transpose
      self._pack_t(info, "w0_in", w.w0_f32, D, D, self.n_in_t, self.eng.c_in_pad)

  def weight_tangents(self, tangents) -> Dict[str, _WeightTangent]:
    """Packs parameter tangents, device fp32 tensors keyed and shaped like the params (modules and
    fields may be left out: zero), into tangent weight images on the current stream, with the padding
    and split blocks of the engine's own (Engine._make_mlp, _make_split).  MLPs with no tangent at all
    are absent, so their tangent GEMMs are skipped; the mesh2grid mesh-node MLP, which the step never
    reads, is never packed.  The engine's weights are not touched."""
    zeros = lambda *s: torch.zeros(list(s), dtype=torch.float32, device=self.dev)
    image = lambda k, n: torch.zeros([self.lib.gcb_packed_weight_bytes(k, n)], dtype=torch.uint8,
                                     device=self.dev)
    out = {}
    for info in self._all:
      l0, l1 = f"{info.stem}_mlp/~/linear_0", f"{info.stem}_mlp/~/linear_1"
      t0, t1 = tangents.get(l0, {}), tangents.get(l1, {})
      tn = tangents.get(f"{info.stem}_layer_norm", {}) if info.ln else {}
      if not (t0 or t1 or tn):
        continue
      wt = _WeightTangent()
      if t0:
        w = t0["w"] if "w" in t0 else zeros(*self.shapes[l0]["w"])
        if info.split is not None:           # row blocks [edge | sender | receiver], each packed alone
          wt.split, wt.w0_f32 = {}, w
          for i, name in enumerate(("we", "ws", "wr")):
            wt.split[name] = image(D, D)
            self.eng.pack_weight(w.data_ptr() + 4 * i * D * D, D, False, D, D, D, D, wt.split[name])
        else:
          seg_real = [w.shape[0]] if len(info.k_segs) == 1 else info.k_segs
          wt.w0, wt.w0_f32 = image(sum(info.k_segs), D), zeros(sum(info.k_segs), D)
          self.eng._pack_linear_device(w, seg_real, info.k_segs, wt.w0, wt.w0_f32)
        wt.b0 = t0["b"] if "b" in t0 else zeros(D)
      if t1:
        w = t1["w"] if "w" in t1 else zeros(*self.shapes[l1]["w"])
        wt.w1, wt.w1_f32 = image(D, info.n1), zeros(D, info.n1)
        self.eng._pack_linear_device(w, [D], [D], wt.w1, wt.w1_f32)
        wt.b1 = zeros(info.n1)
        if "b" in t1:
          wt.b1[:info.n1_valid].copy_(t1["b"])
      for f in ("scale", "offset"):
        if f in tn:
          v = zeros(info.n1)
          v[:info.n1_valid].copy_(tn[f])
          setattr(wt, f, v)
      out[info.stem] = wt
    return out

  def pack_transposed_tangents(self, wts: Dict[str, _WeightTangent], input_grad: bool = False) -> None:
    """The transposed images of packed parameter tangents (weight_tangents), packed on the device as
    _pack_transposed packs the primal ones: W1-dot^T and W0-dot^T per 512-row block (for a pre-gathered
    edge layer: we, ws, wr), so that a parameter Hessian-vector product's dX products can add their
    dY W-dot^T terms.  Layers without a tangent get none.  input_grad (a joint Hessian-vector product,
    whose walk also forms the input gradient): the grid embedder's W0-dot^T in input_transposed's
    [512, n] layout too (w0_in), when that layer has a tangent."""
    for info in self._all:
      wt = wts.get(info.stem)
      if wt is None:
        continue
      if wt.w1_f32 is not None:
        self._pack_t(wt, "w1", wt.w1_f32.data_ptr(), info.n1, info.n1, D, D)
      if wt.w0_f32 is not None:
        k0 = self.shapes[f"{info.stem}_mlp/~/linear_0"]["w"][0]
        if len(info.k_segs) >= 2 and k0 == len(info.k_segs) * D:
          for s in range(len(info.k_segs)):
            self._pack_t(wt, f"w0_{s}", wt.w0_f32.data_ptr() + 4 * s * D * D, D, D, D, D)
        elif k0 == D:
          self._pack_t(wt, "w0_0", wt.w0_f32.data_ptr(), D, D, D, D)
        if input_grad and info is self.mlps["enc_grid"]:
          _, n = self.input_transposed()
          self._pack_t(wt, "w0_in", wt.w0_f32.data_ptr(), D, D, n, self.eng.c_in_pad)

  def repack(self, stems=None) -> None:
    """The engine's weights were rewritten (Engine.load_params / load_params_device): repacks the
    transposed weights of the MLPs whose module path stem is in `stems` (None: all), in place."""
    for info in self._all:
      if stems is None or info.stem in stems:
        self._pack_transposed(info)

  def input_transposed(self):
    """(packed [512, n] transpose of the grid embedder's first layer, n): the dX product of the grid
    inputs (backprop through time), n = 256 | 512 >= c_in_pad.  Packed on first use, from the
    engine's current weights, so the one-step gradient never holds it."""
    info = self.mlps["enc_grid"]
    if "w0_in" not in info.t:
      cin = self.eng.c_in_pad
      if cin > 2 * 256:
        raise NotImplementedError(f"input gradients support at most 512 padded input channels, "
                                  f"not {cin}")
      self.n_in_t = 256 if cin <= 256 else 512
      self._pack_t(info, "w0_in", info.w.w0_f32, D, D, self.n_in_t, cin)   # [512, c_in_pad]
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

  def zero_hvp(self) -> None:
    """Zeroes (allocating on first use) the accumulators of a parameter Hessian-vector product, the
    tangents of the gradient accumulators info.g, shaped like them."""
    for info in self._all:
      if not hasattr(info, "gt"):
        info.gt = {f: torch.zeros_like(t) for f, t in info.g.items()}
      for t in info.gt.values():
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
      for i, (table, idx) in enumerate(pre):             # idx None: row r adds row r of the table
        d.pre_add[i].table, d.pre_add[i].idx = table.data_ptr(), None if idx is None else idx.data_ptr()
        d.pre_add[i].ld = table.shape[1]
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
                   w0=None, dw_segs=None, tan=None, xdot=None) -> torch.Tensor:
    """Backward of one MLP at the recomputed forward; accumulates its parameter gradients and returns
    dh [rows, 512], the gradient of the first layer's pre-activation (incl. pre-gathered addends).
    dw_segs: the layer-0 inputs whose weight blocks get X^T dh (default: all of `segs`).

    With self.dirs > 1 (no parameter gradients), dy and dh are stacked tables of that many directions
    of `rows` rows (dir_rows): h and z are recomputed once, the dX products run once over every
    direction, and the two nonlinearities are gcb_layernorm_backward_dirs and gcb_swish_jvp, whose
    results are those of the one-direction kernels without the column sums.

    In a Hessian-vector product (self.hvp set, 1 + K directions: the gradient and its tangents along K
    primal tangents, K = self.tdirs), `tan` = (dsegs, dpre, dw0) is the tangent of the layer-0 input as
    mlp_jvp takes it (stacked tables of K directions, K-fold gather indices): h-dot = dsegs W0 + the
    gathered addends, z-dot = W1 (swish'(h) h-dot), each one GEMM over the K directions, and the two
    nonlinearities are gcb_layernorm_backward_jvp_dirs and gcb_swish_backward_jvp_dirs, which form the
    primal terms once for all K.

    A parameter Hessian-vector product (self.phvp: two directions, parameter gradients, the weight
    tangents self.wts) runs that walk with K = 1 and every launch of direction 0 on the operands of the
    one-direction walk, and also forms the tangents of the parameter gradients in info.gt: h-dot and
    z-dot get the MLP's weight-tangent terms X W0-dot + b0-dot and a W1-dot + b1-dot; the LayerNorm is
    gcb_layernorm_backward_jvp_params (its scale-dot, the sums of both directions); da-dot gets
    dz W1-dot^T; dW-dot = X-dot^T g + X^T g-dot for each weight, with `xdot` the tangents of the layer-0
    inputs aligned with dw_segs (default segs; None entries or xdot None: zero) and a-dot for layer 1;
    the bias sums of both directions run in gcb_layernorm_backward's column-sum mode."""
    w = info.w
    w0 = w0 or w.w0_packed
    nd, stride, rk = self.dirs, self.dir_stride(rows), self.dir_rows(rows)
    ph = self.phvp
    wt = self.wts.get(info.stem) if ph else None
    h = self.empty(rows)
    self.layer(rows, segs, w0, w.b0, _native.ACT_NONE, out_y=h, pre=pre)
    hd = None if self.hvp is None else self._hdot(rows, w0, tan, segs, wt)
    g = info.g if self.param_grads else self.sink
    ad = None
    ws = self.ws_rows
    if info.ln:
      a = self.empty(rows)
      _native.check(self.lib.gcb_swish_rows(h.data_ptr(), D, rows, D, a.data_ptr(), D, self._st()),
                    "gcb_swish_rows")
      z = self.empty(rows)
      self.layer(rows, [self.tab(a)], w.w1_packed, w.b1, out_y=z)
      if wt is None or wt.w1 is None:
        del a
      dz = self.empty(rk)
      if hd is not None:                     # z-dot = W1 (swish'(h) h-dot), K directions
        nt = self.tdirs
        rt = self.dir_rows(rows, nt)
        ad = self.empty(rt)
        _native.check(self.lib.gcb_swish_jvp(h.data_ptr(), D, rows, D, hd.data_ptr(), D, stride, nt,
                                             ad.data_ptr(), D, self._st()), "gcb_swish_jvp")
        zd = self.empty(rt)
        self.layer(rt, [self.tab(ad)], w.w1_packed, self.zero_bias, out_y=zd)
        if not ph:
          ad = None
        if wt is not None and wt.w1 is not None:   # + a W1-dot + b1-dot
          zdt = self.empty(rows)
          self.layer(rows, [self.tab(a)], wt.w1, wt.b1, out_y=zdt, pre=[(zd, None)])
          zd = zdt
          del a
        if ph:
          gt = info.gt
          _native.check(self.lib.gcb_layernorm_backward_jvp_params(
              dy.data_ptr(), dy.shape[1], stride, z.data_ptr(), D, zd.data_ptr(), D, w.ln_scale,
              self._ptr(None if wt is None else wt.scale), rows, D, dz.data_ptr(), D, ws.data_ptr(),
              ws.numel(), g["b1"].data_ptr(), g["scale"].data_ptr(), g["offset"].data_ptr(),
              gt["b1"].data_ptr(), gt["scale"].data_ptr(), gt["offset"].data_ptr(), 1, self._st()),
              "gcb_layernorm_backward_jvp_params")
        else:
          _native.check(self.lib.gcb_layernorm_backward_jvp_dirs(
              dy.data_ptr(), dy.shape[1], z.data_ptr(), D, zd.data_ptr(), D, w.ln_scale, rows, D,
              stride, dz.data_ptr(), D, nt, self._st()), "gcb_layernorm_backward_jvp_dirs")
        del zd
      elif nd == 1:
        _native.check(self.lib.gcb_layernorm_backward(
            dy.data_ptr(), dy.shape[1], z.data_ptr(), D, w.ln_scale, rows, D, dz.data_ptr(), D,
            ws.data_ptr(), ws.numel(), g["b1"].data_ptr(), g["scale"].data_ptr(),
            g["offset"].data_ptr(), 1, self._st()), "gcb_layernorm_backward")
      else:
        _native.check(self.lib.gcb_layernorm_backward_dirs(
            dy.data_ptr(), dy.shape[1], z.data_ptr(), D, w.ln_scale, rows, D, stride, nd,
            dz.data_ptr(), D, self._st()), "gcb_layernorm_backward_dirs")
      del z
    else:
      dz = dy
      if nd == 1:                            # its column sums only (several directions: none)
        self.col_sums(dy, rows, info.n1, g["b1"])
      elif ph:                               # both directions' (a parameter HVP)
        self.col_sums(dy, rows, info.n1, g["b1"])
        self.col_sums(dy[stride:], rows, info.n1, info.gt["b1"])
      if ph:                                 # a-dot = swish'(h) h-dot, for dW1-dot
        ad = self.empty(rows)
        _native.check(self.lib.gcb_swish_jvp(h.data_ptr(), D, rows, D, hd.data_ptr(), D, stride, 1,
                                             ad.data_ptr(), D, self._st()), "gcb_swish_jvp")
    if self.param_grads:
      self.wgrad(self.tab(h), dz, rows, g["w1"], n=info.n1, swish=True)     # dW1 = swish(h)^T dz
    if ph:                                   # dW1-dot = a-dot^T dz + swish(h)^T dz-dot
      self.wgrad(self.tab(ad), dz, rows, info.gt["w1"], n=info.n1)
      self.wgrad(self.tab(h), dz[stride:], rows, info.gt["w1"], n=info.n1, swish=True)
      del ad
    da = self.empty(rk)
    self.layer(rk, [self.tab(dz, info.n1)], info.t["w1"], self.zero_bias, out_y=da)
    if wt is not None and "w1" in wt.t:      # da-dot += dz W1-dot^T
      self.add_dot_product(rows, dz, wt.t["w1"], da, k=info.n1)
    if hd is not None:                       # [swish'(h) da; its K tangents] in place
      dh = da
      _native.check(self.lib.gcb_swish_backward_jvp_dirs(
          h.data_ptr(), D, hd.data_ptr(), D, rows, D, da.data_ptr(), D, stride, dh.data_ptr(), D,
          self.tdirs, self._st()), "gcb_swish_backward_jvp_dirs")
      del hd
      if ph:                                 # the bias sums of dh and dh-dot
        self.col_sums(dh, rows, D, g["b0"])
        self.col_sums(dh[stride:], rows, D, info.gt["b0"])
    elif nd == 1:
      dh = self.empty(rows)
      _native.check(self.lib.gcb_swish_backward(
          da.data_ptr(), D, h.data_ptr(), D, rows, D, dh.data_ptr(), D, ws.data_ptr(), ws.numel(),
          g["b0"].data_ptr(), 1, self._st()), "gcb_swish_backward")
    else:                                    # swish'(h) da in place
      dh = da
      _native.check(self.lib.gcb_swish_jvp(h.data_ptr(), D, rows, D, da.data_ptr(), D, stride, nd,
                                           dh.data_ptr(), D, self._st()), "gcb_swish_jvp")
    del da, h
    if self.param_grads:
      off = 0
      wsegs = dw_segs if dw_segs is not None else segs
      if xdot is None and tan is not None and tan[2] is None and len(tan[0]) == len(wsegs):
        xdot = tan[0]                        # the input tangents, one per segment
      for i, s in enumerate(wsegs):
        k = s[2]
        self.wgrad(s, dh, rows, g["w0"][off:off + k])
        if ph:                               # dW0-dot = X-dot^T dh + X^T dh-dot
          self.wgrad_dot(s, None if xdot is None else xdot[i], dh, rows, info.gt["w0"][off:off + k])
        off += k
    return dh

  def _hdot(self, rows: int, w0, tan, segs=None, wt: Optional[_WeightTangent] = None) -> torch.Tensor:
    """h-dot of an MLP's first layer, a stacked table of self.tdirs directions of `rows` rows, from
    tan = (dsegs, dpre, dw0) (see mlp_backward): dsegs W0 (dw0: the weight of those segments, default
    w0) plus the gathered addends dpre, or the addends alone; zeros when the layer input has no
    tangent.  With a layer-0 weight tangent wt (a parameter HVP, one direction), + segs W0-dot + b0-dot
    (for a pre-gathered edge layer, segs is the edge segment and W0-dot its block we)."""
    dsegs, dpre, dw0 = tan if tan is not None else ([], (), None)
    rt = self.dir_rows(rows, self.tdirs)
    if dsegs:
      hd = self.empty(rt)
      self.layer(rt, dsegs, dw0 or w0, self.zero_bias, out_y=hd, pre=list(dpre) or None)
    else:
      hd = None
      for table, idx in dpre:
        hd = self.gather_add(table, idx, rt, hd)
    t0 = None if wt is None else (wt.split["we"] if wt.split is not None else wt.w0)
    if t0 is not None:
      hdt = self.empty(rows)
      self.layer(rows, segs, t0, wt.b0, out_y=hdt, pre=None if hd is None else [(hd, None)])
      return hdt
    return hd if hd is not None else torch.zeros([max(rt, 1), D], dtype=torch.float32, device=self.dev)

  def col_sums(self, t: torch.Tensor, rows: int, n: int, out: torch.Tensor) -> None:
    """out += the column sums of t's first `rows` rows (gcb_layernorm_backward's column-sum mode: the
    row split and fp64 fold of every row-wise backward kernel's sums)."""
    ws = self.ws_rows
    _native.check(self.lib.gcb_layernorm_backward(
        t.data_ptr(), t.shape[1], None, 0, None, rows, n, None, 0, ws.data_ptr(), ws.numel(),
        out.data_ptr(), None, None, 1, self._st()), "gcb_layernorm_backward")

  def add_dot_product(self, rows: int, src: torch.Tensor, img, out: torch.Tensor, k: int = D,
                      n: int = D) -> None:
    """A parameter HVP's dX product: direction 1 of the stacked out (= src W^T over both directions,
    n columns) += direction 0 of src times the transposed tangent image img (dY W-dot^T), through one
    GEMM with that direction as an identity addend."""
    s = self.dir_stride(rows)
    t = self.empty(rows, n)
    self.layer(rows, [self.tab(src, k)], img, self.zero_bias, out_y=t, pre=[(out[s:s + rows], None)],
               n=n)
    out[s:s + rows].copy_(t)

  def dx(self, info: _MlpInfo, key: str, rows: int, src: torch.Tensor,
         residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    """A dX product of the walk, [residual +] src W^T over every direction with the transposed block
    info.t[key]; in a parameter HVP, direction 1 also gets src_0 W-dot^T when that block has a
    tangent."""
    rows_k = self.dir_rows(rows)
    out = self.empty(rows_k)
    if residual is None:
      self.layer(rows_k, [self.tab(src)], info.t[key], self.zero_bias, out_y=out)
    else:
      self.layer(rows_k, [self.tab(src)], info.t[key], self.zero_bias, residual=residual, out=out)
    wt = self.wts.get(info.stem) if self.phvp else None
    if wt is not None and key in wt.t:
      self.add_dot_product(rows, src, wt.t[key], out)
    return out

  def wgrad_dot(self, x, xdot, g: torch.Tensor, rows: int, dw: torch.Tensor, *, n: int = D) -> None:
    """dw += X-dot^T g_0 + X^T g_1 (g a stacked table of two directions; xdot None: zero)."""
    if xdot is not None:
      self.wgrad(xdot, g, rows, dw, n=n)
    self.wgrad(x, g[self.dir_stride(rows):], rows, dw, n=n)

  def sender_sums(self, dh: torch.Tensor, rows: int, csr, num_nodes: int) -> torch.Tensor:
    """gcb_segment_sum_sorted (sender CSR `csr`) of every direction of the stacked edge table dh (`rows`
    rows per direction) into a new stacked node table of num_nodes rows per direction, one launch per
    direction."""
    order, ptr, heavy, n_heavy = csr
    out = self.empty(self.dir_rows(num_nodes))
    s_in, s_out = self.dir_stride(rows), self.dir_stride(num_nodes)
    for k in range(self.dirs):
      _native.check(self.lib.gcb_segment_sum_sorted(
          dh[k * s_in:].data_ptr(), D, order.data_ptr(), ptr.data_ptr(), num_nodes, heavy.data_ptr(),
          n_heavy, out[k * s_out:].data_ptr(), D, D, self._st()), "gcb_segment_sum_sorted")
    return out

  def seg_sum_receiver(self, dh: torch.Tensor, rows: int, row_ptr, num_nodes: int, heavy=None,
                       n_heavy=0):
    out = self.empty(self.dir_rows(num_nodes))
    self.receiver_sums(dh, rows, row_ptr, num_nodes, out, self.dir_stride(num_nodes), heavy, n_heavy)
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
                    rcv_sum, tan=None) -> tuple:
    """Backward of a pre-gathered edge MLP m = MLP([e | v_s[snd] | v_r[rcv]]): accumulates its
    parameter gradients, returns (dH, S, R).  tan (Hessian-vector products): (edge tangent segments,
    sender node tangent table, receiver node tangent table), stacked tables of self.tdirs directions;
    their projections are gathered with K-fold indices keyed (snd_name, "snd" | "rcv"), those of
    tangent()."""
    sp = info.split
    ps = self.projection(n_s, v_s, sp.ws_packed)
    pr = self.projection(n_r, v_r, sp.wr_packed)
    t = None
    if tan is not None:                      # in a parameter HVP the projections get v W-dot too
      de_segs, dv_s, dv_r = tan
      nt = self.tdirs
      dps = self.proj_tangent(n_s, v_s, dv_s, sp.ws_packed, self._split_tangent(info, "ws"), nt)
      dpr = self.proj_tangent(n_r, v_r, dv_r, sp.wr_packed, self._split_tangent(info, "wr"), nt)
      t = (de_segs, [(dps, self.kfold(snd, n_s, (snd_name, "snd"), nt)),
                     (dpr, self.kfold(rcv, n_r, (snd_name, "rcv"), nt))], None)
    dh = self.mlp_backward(info, rows, [e_seg], dm, pre=[(ps, snd), (pr, rcv)], w0=sp.we_packed,
                           tan=t, xdot=None if t is None or not t[0] else t[0])
    del ps, pr, t
    s = self.sender_sums(dh, rows, self.csr[snd_name], n_s)
    r = rcv_sum(dh)
    if self.param_grads:
      w0 = info.g["w0"]
      self.wgrad(v_s, s, n_s, w0[D:2 * D])
      self.wgrad(v_r, r, n_r, w0[2 * D:3 * D])
      if self.phvp:                          # the node blocks: v-dot^T S + v^T S-dot
        gt = info.gt["w0"]
        self.wgrad_dot(v_s, self.tab(tan[1]), s, n_s, gt[D:2 * D])
        self.wgrad_dot(v_r, self.tab(tan[2]), r, n_r, gt[2 * D:3 * D])
    return dh, s, r

  def bipartite_backward(self, name: str, info: _MlpInfo, enc: _MlpInfo, feat_t: torch.Tensor,
                         dagg: torch.Tensor, snd: torch.Tensor, rcv: torch.Tensor, v_s, n_s: int,
                         v_r, n_r: int, tan=None) -> tuple:
    """Backward of a grid2mesh / mesh2grid edge MLP m = MLP([e | v_s[snd] | v_r[rcv]]) with
    e = MLP(edge features) and dm = dagg[rcv] (its edge residual is dead), chunk by chunk (see
    self.chunks): accumulates the parameter gradients of both MLPs and returns the node tables
    (S [n_s, 512], R [n_r, 512]) of dH summed by sender / receiver.

    Several directions (self.dirs > 1, stacked dagg) use these same chunks, not tangent_chunks: S is
    added chunk by chunk, so its bits depend on where the chunks fall, and direction k is to be what
    one direction alone gives.  The stacked temporaries of a chunk therefore grow with the direction
    count.

    tan (Hessian-vector products): the node tangent tables (sender, receiver or None), stacked tables
    of self.tdirs directions; the edge embedder's output has no tangent.  Their projections are
    gathered in a chunk with K-fold indices of that chunk (keys (name, "hvp", i, ...))."""
    sp = info.split
    ps = self.projection(n_s, v_s, sp.ws_packed)
    pr = self.projection(n_r, v_r, sp.wr_packed)
    dps = dpr = None
    nt = self.tdirs
    if tan is not None:                      # in a parameter HVP the projections get v W-dot too
      dps = self.proj_tangent(n_s, v_s, tan[0], sp.ws_packed, self._split_tangent(info, "ws"), nt)
      dpr = self.proj_tangent(n_r, v_r, tan[1], sp.wr_packed, self._split_tangent(info, "wr"), nt)
    enc_t = self.phvp and enc.stem in self.wts
    s_tab, r_tab = None, self.empty(self.dir_rows(n_r))
    for i, (r0, r1, g0, g1, rp, heavy, n_heavy, csr) in enumerate(self.chunks[name]):
      n = r1 - r0
      f = self.tab(feat_t[r0:r1], 16, 4, 4)                 # 16-byte rows: the view stays aligned
      snd_c, rcv_c = snd[r0:r1].clone(), rcv[r0:r1].clone()  # index arrays from an aligned base
      e = self.fwd_mlp(enc, n, [f])
      # the embedded edges' tangent (their embedder's parameters), recomputed as e is
      de = self.weight_jvp(enc, n, [f]) if enc_t else None
      dm = self.gather_add(dagg, self.kfold(rcv_c, n_r, (name, "backward", i, "rcv")),
                           self.dir_rows(n))
      t = None
      if dps is not None:
        t = ([] if de is None else [self.tab(de)],
             [(dps, self.kfold(snd_c, n_s, (name, "hvp", i, "snd"), nt))] + (
                 [] if dpr is None else [(dpr, self.kfold(rcv_c, n_r, (name, "hvp", i, "rcv"), nt))]),
             None)
      dh = self.mlp_backward(info, n, [self.tab(e)], dm, pre=[(ps, snd_c), (pr, rcv_c)],
                             w0=sp.we_packed, tan=t, xdot=None if de is None else [self.tab(de)])
      del dm, e, de, snd_c, rcv_c, t
      s_c = self.sender_sums(dh, n, csr, n_s)
      s_tab = s_c if s_tab is None else self.gather_add(
          s_c, self.kfold(self.iota[:n_s], n_s, ("iota", n_s)), self.dir_rows(n_s), s_tab)
      del s_c
      self.receiver_sums(dh, n, rp, g1 - g0, r_tab[g0:], self.dir_stride(n_r), heavy, n_heavy)
      if self.param_grads:                  # the edge embedder's backward: parameters only
        de = self.dx(info, "w0_0", n, dh)
        del dh
        self.mlp_backward(enc, n, [f], de)
        del de
      else:
        del dh
    del ps, pr, dps, dpr
    if self.param_grads:
      w0 = info.g["w0"]
      self.wgrad(v_s, s_tab, n_s, w0[D:2 * D])
      self.wgrad(v_r, r_tab, n_r, w0[2 * D:3 * D])
      if self.phvp:                          # the node blocks: v-dot^T S + v^T S-dot
        gt = info.gt["w0"]
        self.wgrad_dot(v_s, self.tab(tan[0]), s_tab, n_s, gt[D:2 * D])
        self.wgrad_dot(v_r, None if tan[1] is None else self.tab(tan[1]), r_tab, n_r, gt[2 * D:3 * D])
    return s_tab, r_tab

  # -- one batch element ---------------------------------------------------------------------------
  def element(self, grid_in_img: torch.Tensor, g_out: torch.Tensor, snaps: dict,
              dgrid_in: bool = False, param_grads: bool = True,
              dirs: int = 1, hvp: Optional[dict] = None,
              wts: Optional[Dict[str, _WeightTangent]] = None) -> Optional[torch.Tensor]:
    """Accumulates the parameter gradients of one batch element whose loss derivative with respect
    to the decoder output is g_out [Ng, 256] (gcb_output_loss_grad) and whose forward left `snaps`
    (whose entries are dropped as they are consumed).  dgrid_in: also return the derivative with
    respect to the packed grid inputs, dh_enc_grid W0^T [Ng, n] (see input_transposed; columns >=
    c_in + 3 are zero).

    param_grads=False (with dgrid_in: the input gradient alone) leaves the accumulators untouched and
    skips what only the parameters need: every gcb_weight_grad, the backward passes of the three edge
    embedders and of the mesh-node encoder, and the de product of the first processor step.  The
    row-wise kernels' column sums go to scratch.  The recomputes and the dX products that remain are
    the same launches on the same operands, so dx is bit-identical to that of param_grads=True.

    dirs = K > 1 (param_grads=False only) differentiates K cotangents at once: g_out is the stacked
    table of K directions of Ng rows (dir_rows), and so is dx.  The gradient state is stacked like the
    tangent's, so every dX product is one GEMM over all directions and every MLP's h and z, the
    embedder recomputes and the sender / receiver projections are formed once; the segment sums run
    per direction.  Direction k is bit for bit what g_out's direction k alone gives.

    hvp (Hessian-vector products, dirs = 1 + K with K >= 1, param_grads=False): the tangent snapshots
    of tangent(dirs=K, snaps=...), stacked tables of K directions, entries dropped as they are consumed.
    Direction 0 of g_out is the loss seed, direction j its tangent along primal tangent j - 1; the walk
    is the same, every MLP also forms h-dot and z-dot of the K tangents from the snapshots (one GEMM
    each over the K directions) and differentiates its two nonlinearities with
    gcb_layernorm_backward_jvp_dirs and gcb_swish_backward_jvp_dirs, so direction j of dx is the
    tangent of direction 0 along tangent j - 1.  Direction 0 is bit for bit what g_out's direction 0
    alone gives, and direction j what the K = 1 walk gives for tangent j - 1 and seed direction j.

    hvp with param_grads (a parameter Hessian-vector product, loss_and_param_hvp): dirs = 2, the
    snapshots of tangent(wts=wts, snaps=..., tsnaps=...) along the packed parameter tangents `wts`
    (with pack_transposed_tangents), g_out's direction 1 the seed's tangent.  The walk above with K = 1
    then also accumulates the parameter gradients (direction 0, bit for bit those of the one-direction
    walk) and their tangents into info.gt (see mlp_backward), runs the parts that only the parameters
    need on both directions (the edge embedders, the mesh-node encoder, the first step's de product), and
    adds every weight tangent's terms: h-dot and z-dot get X W-dot + b-dot, every dX product of a layer
    with a tangent dY_0 W-dot^T, and the node projections of the edge layers v W-dot.  The input
    tangent is taken to be zero, and the grid embedder's dW0-dot has no X-dot^T dh term.

    That walk with dgrid_in (a joint Hessian-vector product in the parameters and the inputs,
    loss_and_joint_hvp): the tangent ran along the parameter tangents and a non-zero input tangent, so
    the grid embedder's dW0-dot also gets X-dot^T dh (X-dot the packed input tangent of the snapshots),
    and direction 1 of dx also gets dh_0 W0-dot^T (pack_transposed_tangents(input_grad=True)).  Direction
    0 of dx is bit for bit what param_grads=False gives."""
    phvp = hvp is not None and param_grads
    if phvp:
      if dirs != 2:
        raise ValueError("a parameter Hessian-vector product runs two directions")
    else:
      if dirs > 1 and param_grads:
        raise ValueError("several directions are supported without parameter gradients only")
      if hvp is not None and dirs < 2:
        raise ValueError("a Hessian-vector product runs 1 + K directions (K >= 1) without parameter "
                         "gradients")
    self.param_grads, self.dirs, self.hvp = bool(param_grads), int(dirs), hvp
    self.tdirs = 0 if hvp is None else int(dirs) - 1
    self.phvp, self.wts = phvp, (wts or {}) if phvp else {}
    try:
      return self._element(grid_in_img, g_out, snaps, dgrid_in)
    finally:
      self.param_grads, self.dirs, self.hvp, self.tdirs = True, 1, None, 0
      self.phvp, self.wts = False, {}

  def _element(self, grid_in_img, g_out, snaps, dgrid_in):
    eng, m = self.eng, self.m
    ng, nm = m.num_grid, m.num_mesh
    K = eng.msg_steps
    mp = self.mlps
    img, tab = self.img, self.tab
    feat = lambda t: tab(t, 16, 4, 4)
    rk = self.dir_rows                       # rows of a stacked table (n rows for one direction)
    T = self.hvp                             # tangent snapshots (Hessian-vector products) or None
    tan = (lambda *segs, dw0=None: None) if T is None else (
        lambda *segs, dw0=None: ([tab(t) for t in segs], (), dw0))

    # ---- decoder: out = MLP(vg2);  vg2 = vg1 + MLP([vg1 | agg3]);  m3 = MLP([e3 | v[snd] | vg1[rcv]])
    dh = self.mlp_backward(mp["dec_grid"], ng, [img(snaps["vg2"])], g_out,
                           tan=tan(*(() if T is None else (T.pop("vg2"),))))
    dvg2 = self.dx(mp["dec_grid"], "w0_0", ng, dh)
    info = mp["proc_n_grid_m2g"]
    dh = self.mlp_backward(info, ng, [img(snaps["vg1"]), img(snaps["agg3"])], dvg2,
                           tan=tan(*(() if T is None else (T["vg1"], T.pop("agg3")))))
    dvg1 = self.dx(info, "w0_0", ng, dh, residual=dvg2)
    dagg3 = self.dx(info, "w0_1", ng, dh)
    del dh, dvg2
    info = mp["proc_e_m2g"]
    S, R = self.bipartite_backward("m2g", info, mp["enc_e_m2g"], eng.m2g_feat, dagg3, eng.m2g_snd,
                                   eng.m2g_rcv, img(snaps["v"][K]), nm, img(snaps["vg1"]), ng,
                                   tan=None if T is None else (T["v"][K], T.pop("vg1")))
    del dagg3
    # snapshots are released as soon as the backward pass is past their stage
    snaps["vg2"] = snaps["agg3"] = snaps["vg1"] = None
    dvg1 = self.dx(info, "w0_2", ng, R, residual=dvg1)
    dv = self.dx(info, "w0_1", nm, S)
    del S, R

    # ---- processor, last step first:  m = MLP([e | v[snd] | v[rcv]]);  v' = v + MLP([v | agg]);
    #      e' = e + m
    de_next = None
    rcv_k = self.kfold(eng.mesh_rcv, nm, ("mesh", "rcv"))
    for k in range(K - 1, -1, -1):
      v_k = img(snaps["v"][k])
      agg_k = img(snaps["agg"][k])
      nfo, efo = self.proc_n[k], self.proc_e[k]
      dh_n = self.mlp_backward(nfo, nm, [v_k, agg_k], dv,
                               tan=tan(*(() if T is None else (T["v"][k], T["agg"][k]))))
      dagg = self.dx(nfo, "w0_1", nm, dh_n)
      dm = self.gather_add(dagg, rcv_k, rk(m.e_mesh), de_next)
      del dagg
      if k == 0:
        e0 = self.fwd_mlp(mp["enc_e_mesh"], m.e_mesh, [feat(eng.mesh_feat)])
        e_k = tab(e0)
      else:
        e_k = img(snaps["e"][k])
      dH, S, R = self.edge_backward(
          efo, m.e_mesh, e_k, dm, "mesh", v_k, nm, eng.mesh_snd, v_k, nm, eng.mesh_rcv,
          lambda d: self.seg_sum_receiver(d, m.e_mesh, eng.mesh_row_ptr, nm),
          tan=None if T is None else ([] if T["e"][k] is None else [tab(T["e"][k])], T["v"][k],
                                      T["v"][k]))
      del dm
      if k == 0 and not self.param_grads:    # de_0 feeds the mesh edge embedder's parameters only
        de = None
      else:                                  # de_k = de_{k+1} + dH W_e^T  (e' = e + m)
        de = self.dx(efo, "w0_0", m.e_mesh, dH, residual=de_next)
      del dH
      de_next = de
      # dv_k = dv_{k+1} + dh_n W0a^T + S W_s^T + R W_r^T
      dv_new = self.dx(nfo, "w0_0", nm, dh_n, residual=dv)
      dv2 = self.dx(efo, "w0_1", nm, S, residual=dv_new)
      dv = self.dx(efo, "w0_2", nm, R, residual=dv2)
      del dh_n, S, R, dv2, dv_new
      snaps["v"][k + 1] = snaps["agg"][k] = snaps["e"][k] = None
      if T is not None:
        T["v"][k + 1] = T["agg"][k] = T["e"][k] = None
    # mesh edge embedder: e0 = MLP(edge features)
    if self.param_grads:
      self.mlp_backward(mp["enc_e_mesh"], m.e_mesh, [feat(eng.mesh_feat)], de_next)
    del de_next, e0

    # ---- encoder: vg1 = vg0 + MLP([vg0]);  vm1 = vm0 + MLP([vm0 | agg1]);
    #      m1 = MLP([e1 | vg0[snd] | vm0[rcv]]);  vg0 = MLP(grid_in);  vm0 = MLP(mesh_in)
    grid_in = img(grid_in_img, eng.c_in_pad)
    mesh_in = img(eng.mesh_in_img, eng.c_in_pad)
    vg0 = self.fwd_mlp(mp["enc_grid"], ng, [grid_in])
    vm0 = self.fwd_mlp(mp["enc_mesh"], nm, [mesh_in])
    info = mp["proc_n_grid_g2m"]
    dh = self.mlp_backward(info, ng, [tab(vg0)], dvg1,
                           tan=tan(*(() if T is None else (T["vg0"],))))
    dvg0 = self.dx(info, "w0_0", ng, dh, residual=dvg1)
    del dh, dvg1
    info = mp["proc_n_mesh_g2m"]
    dvm0_t = None if T is None else T.pop("vm0", None)   # v_m0's tangent (its encoder's parameters)
    if dvm0_t is None:                       # vm0 has no tangent: block 1 of W0 alone
      dh = self.mlp_backward(info, nm, [tab(vm0), img(snaps["agg1"])], dv,
                             tan=None if T is None else tan(T["agg1"], dw0=self.w0_block(info, 1)),
                             xdot=None if T is None else [None, tab(T["agg1"])])
    else:
      dh = self.mlp_backward(info, nm, [tab(vm0), img(snaps["agg1"])], dv,
                             tan=tan(dvm0_t, T["agg1"]))
    if T is not None:
      del T["agg1"]
    dvm0 = self.dx(info, "w0_0", nm, dh, residual=dv)
    dagg1 = self.dx(info, "w0_1", nm, dh)
    del dh, dv
    info = mp["proc_e_g2m"]
    S, R = self.bipartite_backward("g2m", info, mp["enc_e_g2m"], eng.g2m_feat, dagg1, eng.g2m_snd,
                                   eng.g2m_rcv, tab(vg0), ng, tab(vm0), nm,
                                   tan=None if T is None else (T.pop("vg0"), dvm0_t))
    del dagg1, dvm0_t
    dvg0 = self.dx(info, "w0_1", ng, S, residual=dvg0)
    dvm0 = self.dx(info, "w0_2", nm, R, residual=dvm0)
    del S, R, vg0, vm0
    # A parameter HVP has a zero input tangent; a joint one (phvp with dgrid_in) has one, whose
    # X-dot^T dh the grid embedder's weight-gradient tangent takes.
    joint = self.phvp and dgrid_in
    gin_t = None if T is None else img(T.pop("grid_in"), eng.c_in_pad)
    dh = self.mlp_backward(mp["enc_grid"], ng, [grid_in], dvg0,
                           tan=None if T is None else ([gin_t], (), None),
                           xdot=[gin_t if joint else None])
    del gin_t
    dx = None
    if dgrid_in:
      w0t, n = self.input_transposed()
      dx = self.empty(rk(ng), n)
      self.layer(rk(ng), [tab(dh)], w0t, self.zero_bias, out_y=dx, n=n)
      wt = self.wts.get(mp["enc_grid"].stem)
      if joint and wt is not None and "w0_in" in wt.t:    # direction 1 += dh_0 W0-dot^T
        self.add_dot_product(ng, dh, wt.t["w0_in"], dx, n=n)
    del dh, dvg0
    if self.param_grads:
      self.mlp_backward(mp["enc_mesh"], nm, [mesh_in], dvm0)
    return dx

  # -- tangent-linear model (Engine.input_jvp_element) ------------------------------------------------
  # The tangent (or, in element(dirs=K), gradient) state of `dirs` directions is stacked direction-major: a table of n rows per direction
  # holds direction k in rows [k * dir_stride(n), k * dir_stride(n) + n), the stride rounded up to the
  # 128-row tiles of the operand images.  The last direction is not padded, so that one direction is
  # exactly the table of n rows.  The pad rows between directions are never read into a valid row: the
  # GEMMs and row-wise kernels treat every row on its own, and the segment sums and unpacks run per
  # direction.
  @staticmethod
  def dir_stride(rows: int) -> int:
    return (rows + 127) // 128 * 128

  def dir_rows(self, rows: int, dirs: Optional[int] = None) -> int:
    """Rows of a stacked tangent table of `dirs` (default self.dirs) directions of `rows` rows each."""
    return ((self.dirs if dirs is None else dirs) - 1) * self.dir_stride(rows) + rows

  def kfold(self, idx: torch.Tensor, n_src: int, key, folds: Optional[int] = None) -> torch.Tensor:
    """The gather index `idx` (into a table of n_src rows per direction) for `folds` (default
    self.dirs) directions: idx + k * dir_stride(n_src) in the rows of direction k of a stacked table of
    len(idx) rows per direction, 0 in the pad rows.  Built on first use per (folds, key) and kept while
    the fold count is one of the two used last (a Hessian-vector product's walk reads K-fold and
    (1 + K)-fold indices in one pass, and its tangent forward K-fold ones).  The key names the index
    and, for a bipartite chunk, the chunk set it belongs to ("tangent" | "backward" | "hvp"): with
    several directions the sets differ, so chunk i of one is not chunk i of the other."""
    folds = self.dirs if folds is None else int(folds)
    if folds == 1:
      return idx
    cache = self._kfold.pop(folds, None)
    cache = {} if cache is None else cache
    self._kfold[folds] = cache               # most recently used last
    while len(self._kfold) > 2:
      del self._kfold[next(iter(self._kfold))]
    out = cache.get(key)
    if out is None:
      n, s_src, s = idx.shape[0], self.dir_stride(n_src), self.dir_stride(idx.shape[0])
      out = torch.zeros([self.dir_rows(n, folds)], dtype=torch.int32, device=self.dev)
      for k in range(folds):
        out[k * s:k * s + n] = idx + k * s_src
      cache[key] = out
    return out

  def tangent_chunks(self, name: str):
    """The receiver-aligned chunks of a bipartite edge set for the tangent of self.dirs directions: those
    of the backward pass for one direction, else chunks of chunk_rows // dirs edges (built on first
    use, without the sender CSR), so that the stacked temporaries stay the size of one direction's.
    Every receiver's sum is complete inside its chunk, so the results do not depend on the chunking."""
    if self.dirs == 1:
      return self.chunks[name]
    key = (name, self.dirs)
    if key not in self._tangent_chunks:
      row_ptr, senders, n_senders = self._chunk_src[name]
      self._tangent_chunks[key] = self._chunks(row_ptr, senders, n_senders,
                                               max(self.chunk_rows // self.dirs, 1), csr=False)
    return self._tangent_chunks[key]

  def w0_block(self, info: _MlpInfo, s: int) -> int:
    """Address of the packed image of the 512-row block s of an MLP's first layer (the image is K-step
    major, so a row block is a contiguous slice)."""
    return info.w.w0_packed + s * self.lib.gcb_packed_weight_bytes(D, D)

  def mlp_jvp(self, info: _MlpInfo, rows: int, segs, dsegs, *, pre=None, dpre=(), w0=None,
              dw0=None, residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Tangent of one MLP y = LN(swish(X W0 + b0) W1 + b1) at the recomputed forward (h, z as
    mlp_backward forms them, once for all directions), along the layer-0 input tangents `dsegs` with the
    weight dw0 (default: that of the primal, w0) and the pre-gathered addends `dpre` (K-fold indices);
    with no dsegs the addends alone are the pre-activation tangent.  Tangents are stacked tables of
    self.dirs directions of `rows` rows.  Returns residual + dy (LayerNorm MLPs) or dy [., n1] (the
    decoder).

    With a parameter tangent of this MLP in self.wts (param_jvp, one direction), each layer also gets
    its weight-tangent term, one GEMM at the primal rows with the previous tangent as an identity
    pre-gathered addend: h-dot = X-dot W0 + X W0-dot + b0-dot (for a pre-gathered edge layer X is the
    edge segment and W0-dot its block we; the node blocks' terms come in dpre), z-dot = a-dot W1 +
    a W1-dot + b1-dot, and the LayerNorm adds scale-dot * zhat + offset-dot (gcb_layernorm_jvp_params).
    A layer without a tangent runs exactly what it runs without self.wts."""
    w = info.w
    w0 = w0 or w.w0_packed
    wt = self.wts.get(info.stem)
    t0 = None if wt is None else (wt.split["we"] if wt.split is not None else wt.w0)
    nd, stride, rk = self.dirs, self.dir_stride(rows), self.dir_rows(rows)
    dh = None
    if dsegs:
      dh = self.empty(rk)
      self.layer(rk, dsegs, dw0 or w0, self.zero_bias, out_y=dh, pre=list(dpre) or None)
      dpre = ()
    if t0 is not None:                       # + X W0-dot + b0-dot (and the addends not yet added)
      pre_t = list(dpre) + ([] if dh is None else [(dh, None)])
      dht = self.empty(rows)
      self.layer(rows, segs, t0, wt.b0, out_y=dht, pre=pre_t or None)
      dh = dht
    else:
      for table, idx in dpre:
        dh = self.gather_add(table, idx, rk, dh)
      if dh is None:                         # neither the input nor the first layer has a tangent
        dh = torch.zeros([max(rk, 1), D], dtype=torch.float32, device=self.dev)
    h = self.empty(rows)
    self.layer(rows, segs, w0, w.b0, _native.ACT_NONE, out_y=h, pre=pre)
    da = dh                                  # swish'(h) dh in place: the Jacobian of swish is diagonal
    _native.check(self.lib.gcb_swish_jvp(h.data_ptr(), D, rows, D, dh.data_ptr(), D, stride, nd,
                                         da.data_ptr(), D, self._st()), "gcb_swish_jvp")
    del dh
    t1 = None if wt is None else wt.w1
    if not info.ln:
      dy = self.empty(rk, info.n1)
      self.layer(rk, [self.tab(da)], w.w1_packed, self.zero_bias, out_y=dy, n=info.n1,
                 n_valid=info.n1_valid)
      if t1 is not None:                     # + a W1-dot + b1-dot (padded columns: zero weights)
        a = self.empty(rows)
        _native.check(self.lib.gcb_swish_rows(h.data_ptr(), D, rows, D, a.data_ptr(), D, self._st()),
                      "gcb_swish_rows")
        dyt = self.empty(rows, info.n1)
        self.layer(rows, [self.tab(a)], t1, wt.b1, out_y=dyt, pre=[(dy, None)], n=info.n1)
        dy = dyt
      return dy
    a = self.empty(rows)
    _native.check(self.lib.gcb_swish_rows(h.data_ptr(), D, rows, D, a.data_ptr(), D, self._st()),
                  "gcb_swish_rows")
    del h
    z = self.empty(rows)
    self.layer(rows, [self.tab(a)], w.w1_packed, w.b1, out_y=z)
    if t1 is None:
      del a
    dz = self.empty(rk)
    self.layer(rk, [self.tab(da)], w.w1_packed, self.zero_bias, out_y=dz)
    del da
    if t1 is not None:                       # + a W1-dot + b1-dot
      dzt = self.empty(rows)
      self.layer(rows, [self.tab(a)], t1, wt.b1, out_y=dzt, pre=[(dz, None)])
      dz = dzt
      del a
    out = self.empty(rk)
    if wt is not None and (wt.scale is not None or wt.offset is not None):
      _native.check(self.lib.gcb_layernorm_jvp_params(
          z.data_ptr(), D, dz.data_ptr(), D, w.ln_scale, rows, D, self._ptr(residual), D,
          self._ptr(wt.scale), self._ptr(wt.offset), out.data_ptr(), D, self._st()),
          "gcb_layernorm_jvp_params")
      return out
    _native.check(self.lib.gcb_layernorm_jvp_dirs(
        z.data_ptr(), D, dz.data_ptr(), D, w.ln_scale, rows, D, stride, nd, self._ptr(residual), D,
        out.data_ptr(), D, self._st()), "gcb_layernorm_jvp_dirs")
    return out

  def proj_tangent(self, rows: int, v, dv: Optional[torch.Tensor], w_packed, tw_packed,
                   dirs: Optional[int] = None):
    """Tangent of a node projection v W (a pre-gathered edge layer's sender or receiver block), a
    stacked table of `dirs` (default self.dirs) directions of `rows` rows: dv W + v W-dot, each term
    only when its tangent exists (dv, the image tw_packed of W-dot, one direction); None when neither
    does."""
    out = None
    if dv is not None:
      out = self.projection(self.dir_rows(rows, dirs), self.tab(dv), w_packed)
    if tw_packed is not None:
      t = self.empty(rows)
      self.layer(rows, [v], tw_packed, self.zero_bias, out_y=t,
                 pre=None if out is None else [(out, None)])
      out = t
    return out

  def _split_tangent(self, info: _MlpInfo, name: str):
    """The image of the tangent of split block `name` (ws | wr) of an edge MLP, or None."""
    wt = self.wts.get(info.stem)
    return None if wt is None or wt.split is None else wt.split[name]

  @staticmethod
  def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()

  def receiver_sums(self, dm: torch.Tensor, rows: int, row_ptr: torch.Tensor, n_nodes: int,
                    out: torch.Tensor, out_stride: int, heavy=None, n_heavy: int = 0) -> None:
    """gcb_segment_sum_heavy of every direction of the stacked edge tangent dm (`rows` rows per
    direction) into n_nodes rows of every direction of the stacked node table `out` (a view starting at
    direction 0's first row, out_stride rows per direction), one launch per direction."""
    s_in, s_out = self.dir_stride(rows), out_stride
    for k in range(self.dirs):
      _native.check(self.lib.gcb_segment_sum_heavy(
          dm[k * s_in:].data_ptr(), D, row_ptr.data_ptr(), n_nodes,
          heavy.data_ptr() if n_heavy else None, n_heavy, out[k * s_out:].data_ptr(), D, D,
          self._st()), "gcb_segment_sum_heavy")

  def bipartite_jvp(self, name: str, info: _MlpInfo, enc: _MlpInfo, feat_t: torch.Tensor,
                    snd: torch.Tensor, rcv: torch.Tensor, v_s, n_s: int, v_r, n_r: int,
                    dv_s: torch.Tensor, dv_r: Optional[torch.Tensor]) -> torch.Tensor:
    """Tangent of the receiver sums of a grid2mesh / mesh2grid edge MLP m = MLP([e | v_s[snd] |
    v_r[rcv]]) with e = MLP(edge features), chunk by chunk (tangent_chunks): dagg (n_r rows per
    direction), from the stacked sender and (when dv_r is given) receiver node tangents.  e has a tangent
    only through the edge embedder's parameters (self.wts), and so do the node blocks' W_s, W_r."""
    sp = info.split
    ps = self.projection(n_s, v_s, sp.ws_packed)
    pr = self.projection(n_r, v_r, sp.wr_packed)
    dps = self.proj_tangent(n_s, v_s, dv_s, sp.ws_packed, self._split_tangent(info, "ws"))
    dpr = self.proj_tangent(n_r, v_r, dv_r, sp.wr_packed, self._split_tangent(info, "wr"))
    enc_t = enc.stem in self.wts
    dagg = self.empty(self.dir_rows(n_r))
    for i, (r0, r1, g0, g1, rp, heavy, n_heavy, _) in enumerate(self.tangent_chunks(name)):
      n = r1 - r0
      f = self.tab(feat_t[r0:r1], 16, 4, 4)                 # 16-byte rows: the view stays aligned
      snd_c, rcv_c = snd[r0:r1].clone(), rcv[r0:r1].clone()  # index arrays from an aligned base
      e = self.fwd_mlp(enc, n, [f])
      de = self.mlp_jvp(enc, n, [f], []) if enc_t else None
      dpre = [(dps, self.kfold(snd_c, n_s, (name, "tangent", i, "snd")))]
      if dpr is not None:
        dpre.append((dpr, self.kfold(rcv_c, n_r, (name, "tangent", i, "rcv"))))
      dm = self.mlp_jvp(info, n, [self.tab(e)], [] if de is None else [self.tab(de)],
                        pre=[(ps, snd_c), (pr, rcv_c)], dpre=dpre, w0=sp.we_packed)
      del e, de
      self.receiver_sums(dm, n, rp, g1 - g0, dagg[g0:], self.dir_stride(n_r), heavy, n_heavy)
      del dm
    return dagg

  def tangent(self, grid_in_img: torch.Tensor, dgrid_in_img: torch.Tensor, dirs: int = 1,
              snaps: Optional[dict] = None, tsnaps: Optional[dict] = None,
              wts: Optional[Dict[str, _WeightTangent]] = None) -> torch.Tensor:
    """One step stage by stage (Engine.run_stage, from the packed inputs grid_in_img) and, interleaved
    with it, its tangent along `dirs` directions at once: dgrid_in_img is the stacked operand image of
    the packed input tangents ([Ng, c_in_pad] per direction, dir_stride(Ng) rows apart, structural
    columns zero).  Returns dy, the stacked tangents of the decoder output ([Ng, 256] per direction,
    n_out valid columns).  Each stage's tangent runs right after the stage, from the engine's buffers
    and copies of that stage's inputs alone; the tangent state is stacked fp32 tables, and every MLP's
    h and z are recomputed once for all directions.  Exactly zero tangents are not formed: the
    mesh-node encoder, the three edge embedders, e_0 of the processor, and the v_m0 and edge terms of
    the grid2mesh edge MLP.

    With `snaps` and `tsnaps` (dicts; Hessian-vector products, any number of directions) they receive
    what element(dirs=1 + dirs, hvp=tsnaps) reads: snaps the primal copies of
    Engine._forward_snapshots, tsnaps the tangent tables v-dot_k (k = 0..K), e-dot_k (k = 1..K-1),
    agg-dot_k, and the v-dot / agg-dot of the grid and mesh nodes around the encoder and decoder (vg0,
    agg1, vg1, agg3, vg2), and the packed input tangent image (grid_in).  The tangent tables are the
    stacked tables of `dirs` directions the forward forms anyway: keeping them costs no copy, and their
    memory grows with the directions.  Without them nothing more is kept or launched.

    With `wts` (weight_tangents; param_jvp and loss_and_param_hvp, one direction) the tangent is also
    along those parameter tangents: every MLP with one adds its weight-tangent terms (mlp_jvp,
    proj_tangent), and the tangents that are zero along the inputs alone are formed when their
    parameters have one: the mesh-node encoder's (so the grid2mesh receiver block and the mesh-node
    residual get theirs), the edge embedders' and with it e_0 of the processor.  With snapshots as well
    (a parameter Hessian-vector product), tsnaps also keeps v-dot_m0 ("vm0") and e-dot_0 (e[0]) when they
    exist; the embedded edges' tangents of the two bipartite graphs are not kept (the backward pass
    recomputes them per chunk)."""
    if wts and dirs != 1:
      raise ValueError("parameter tangents run one direction")
    self.dirs, self.wts = int(dirs), wts or {}
    try:
      return self._tangent(grid_in_img, dgrid_in_img, snaps, tsnaps)
    finally:
      self.dirs, self.wts = 1, {}

  def _tangent(self, grid_in_img, dgrid_in_img, snaps=None, ts=None):
    eng, m = self.eng, self.m
    ng, nm = m.num_grid, m.num_mesh
    K = eng.msg_steps
    mp = self.mlps
    img, tab = self.img, self.tab
    cin = eng.c_in_pad

    # ---- encoder: vg0 = MLP(grid_in);  m1 = MLP([e1 | vg0[snd] | vm0[rcv]]);  agg1 = sum m1;
    #      vm1 = vm0 + MLP([vm0 | agg1]);  vg1 = vg0 + MLP([vg0]).  agg1 is read from the engine.
    eng.run_stage("encode", grid_in=grid_in_img)
    keep = ts is not None
    if keep:
      snaps.update(v=[], agg=[], e=[None], vg1=eng.grid_lat_img.clone(), agg1=eng.mesh_agg_img.clone())
      snaps["v"].append(eng.mesh_lat_img.clone())
      ts.update(v=[], agg=[], e=[None], grid_in=dgrid_in_img)
    grid_in = img(grid_in_img, cin)
    info = mp["enc_grid"]
    dvg0 = self.mlp_jvp(info, ng, [grid_in], [img(dgrid_in_img, cin)])
    vg0 = self.fwd_mlp(info, ng, [grid_in])
    mesh_in = [img(eng.mesh_in_img, cin)]
    vm0 = self.fwd_mlp(mp["enc_mesh"], nm, mesh_in)
    # vm0 (from the static mesh inputs) has a tangent only through the mesh-node encoder's parameters
    dvm0 = self.mlp_jvp(mp["enc_mesh"], nm, mesh_in, []) if mp["enc_mesh"].stem in self.wts else None
    dagg = self.bipartite_jvp("g2m", mp["proc_e_g2m"], mp["enc_e_g2m"], eng.g2m_feat, eng.g2m_snd,
                              eng.g2m_rcv, tab(vg0), ng, tab(vm0), nm, dvg0, dvm0)
    info = mp["proc_n_mesh_g2m"]
    if dvm0 is None:                             # vm0 has no tangent: block 1 of W0 alone
      dv = self.mlp_jvp(info, nm, [tab(vm0), img(eng.mesh_agg_img)], [tab(dagg)],
                        dw0=self.w0_block(info, 1))
    else:
      dv = self.mlp_jvp(info, nm, [tab(vm0), img(eng.mesh_agg_img)], [tab(dvm0), tab(dagg)],
                        residual=dvm0)
      if keep:
        ts["vm0"] = dvm0
      del dvm0
    if keep:
      ts.update(vg0=dvg0, agg1=dagg)
      ts["v"].append(dv)
    del dagg, vm0
    dvg = self.mlp_jvp(mp["proc_n_grid_g2m"], ng, [tab(vg0)], [tab(dvg0)], residual=dvg0)
    if keep:
      ts["vg1"] = dvg
    del dvg0, vg0

    # ---- processor:  m = MLP([e | v[snd] | v[rcv]]);  v' = v + MLP([v | agg]);  e' = e + m.
    #      v_k and e_k are copied before step k, agg_k read after it.
    eng.run_stage("process_embed")
    de = None
    snd_k, rcv_k = (self.kfold(eng.mesh_snd, nm, ("mesh", "snd")),
                    self.kfold(eng.mesh_rcv, nm, ("mesh", "rcv")))
    for k in range(K):
      v_k = eng.mesh_lat_img.clone()
      if k == 0:
        feat = [tab(eng.mesh_feat, 16, 4, 4)]
        e_k = tab(self.fwd_mlp(mp["enc_e_mesh"], m.e_mesh, feat))
        if mp["enc_e_mesh"].stem in self.wts:    # e_0 has a tangent through the embedder's parameters
          de = self.mlp_jvp(mp["enc_e_mesh"], m.e_mesh, feat, [])
          if keep:
            ts["e"][0] = de
      else:
        e_k = img(eng.mesh_edge_img.clone())
      eng.run_stage("process_step", k)
      if keep:
        snaps["v"].append(eng.mesh_lat_img.clone())
        snaps["agg"].append(eng.mesh_agg_img.clone())
        if k < K - 1:
          snaps["e"].append(eng.mesh_edge_img.clone())
        if k > 0:
          ts["e"].append(de)
      nfo, efo = self.proc_n[k], self.proc_e[k]
      sp = efo.split
      ps, pr = self.projection(nm, img(v_k), sp.ws_packed), self.projection(nm, img(v_k), sp.wr_packed)
      dps = self.proj_tangent(nm, img(v_k), dv, sp.ws_packed, self._split_tangent(efo, "ws"))
      dpr = self.proj_tangent(nm, img(v_k), dv, sp.wr_packed, self._split_tangent(efo, "wr"))
      dpre = [(dps, snd_k), (dpr, rcv_k)]
      dm = self.mlp_jvp(efo, m.e_mesh, [e_k], [] if de is None else [tab(de)],
                        pre=[(ps, eng.mesh_snd), (pr, eng.mesh_rcv)], dpre=dpre, w0=sp.we_packed)
      del ps, pr, dps, dpr, e_k
      dagg = self.empty(self.dir_rows(nm))
      self.receiver_sums(dm, m.e_mesh, eng.mesh_row_ptr, nm, dagg, self.dir_stride(nm))
      if k < K - 1:                              # the last step's edge update is never read
        de = dm if de is None else self.gather_add(dm, self.edge_iota(), self.dir_rows(m.e_mesh), de)
      del dm
      if keep:
        ts["agg"].append(dagg)
      dv = self.mlp_jvp(nfo, nm, [img(v_k), img(eng.mesh_agg_img)], [tab(dv), tab(dagg)],
                        residual=dv)
      if keep:
        ts["v"].append(dv)
      del dagg, v_k
    del de

    # ---- decoder: m3 = MLP([e3 | v[snd] | vg1[rcv]]);  agg3 = fan-in-3 sum;
    #      vg2 = vg1 + MLP([vg1 | agg3]);  out = MLP(vg2).  agg3 and vg2 are read from the engine.
    v_k, vg1 = eng.mesh_lat_img.clone(), eng.grid_lat_img.clone()
    eng.run_stage("decode", grid_in=grid_in_img)
    if keep:
      snaps.update(vg2=eng.grid_lat_img.clone(), agg3=eng.grid_agg_img.clone())
    dagg = self.bipartite_jvp("m2g", mp["proc_e_m2g"], mp["enc_e_m2g"], eng.m2g_feat, eng.m2g_snd,
                              eng.m2g_rcv, img(v_k), nm, img(vg1), ng, dv, dvg)
    del v_k, dv
    dvg = self.mlp_jvp(mp["proc_n_grid_m2g"], ng, [img(vg1), img(eng.grid_agg_img)],
                       [tab(dvg), tab(dagg)], residual=dvg)
    if keep:
      ts.update(agg3=dagg, vg2=dvg)
    del vg1, dagg
    return self.mlp_jvp(mp["dec_grid"], ng, [img(eng.grid_lat_img)], [tab(dvg)])

  def weight_jvp(self, info: _MlpInfo, rows: int, segs) -> torch.Tensor:
    """The tangent of an MLP of constant inputs along its parameter tangent (self.wts), one direction
    (mlp_jvp with no input tangent), inside a walk of any direction count."""
    dirs, self.dirs = self.dirs, 1
    try:
      return self.mlp_jvp(info, rows, segs, [])
    finally:
      self.dirs = dirs

  def edge_iota(self) -> torch.Tensor:
    """0..dir_rows(E_mesh)-1 (the identity gather of the edge-tangent update e' = e + m over every
    direction), made on first use."""
    n = self.dir_rows(self.m.e_mesh)
    if self._edge_iota is None or self._edge_iota.shape[0] != n:
      self._edge_iota = self._i32(np.arange(n))
    return self._edge_iota

  # -- result ----------------------------------------------------------------------------------------
  def _accumulators(self, tangent: bool = False) -> Dict[str, Dict[str, torch.Tensor]]:
    """The valid slices of the gradient accumulators (views; `tangent`: those of a parameter
    Hessian-vector product, info.gt), keyed and shaped like the params; the parameters the step never
    reads (the mesh2grid mesh-node MLP) are absent."""
    out: Dict[str, Dict[str, torch.Tensor]] = {}
    for info in self._all:
      l0, l1 = f"{info.stem}_mlp/~/linear_0", f"{info.stem}_mlp/~/linear_1"
      k_real = self.shapes[l0]["w"][0]
      g = info.gt if tangent else info.g
      if len(info.k_segs) == 1:
        w0 = g["w0"][:k_real]
      else:
        w0 = g["w0"]
      n = info.n1_valid
      out[l0] = {"w": w0, "b": g["b0"]}
      out[l1] = {"w": g["w1"][:, :n], "b": g["b1"][:n]}
      if info.ln:
        out[f"{info.stem}_layer_norm"] = {"scale": g["scale"], "offset": g["offset"]}
    return out

  def grads(self, tangent: bool = False) -> Dict[str, Dict[str, torch.Tensor]]:
    """Device fp32 gradients keyed and shaped like the params (`tangent`: the Hessian-vector products
    accumulated by parameter HVPs, zero_hvp); parameters the step never reads (the mesh2grid mesh-node
    MLP) get zeros."""
    out = {name: {f: t.clone() for f, t in fields.items()}
           for name, fields in self._accumulators(tangent).items()}
    for name, fields in self.shapes.items():
      if name not in out:
        out[name] = {f: torch.zeros(shape, dtype=torch.float32, device=self.dev)
                     for f, shape in fields.items()}
    return out

  def grads_into(self, out) -> None:
    """The gradients of `grads` copied into the device tensors out[name][field]."""
    acc = self._accumulators()
    for name, fields in self.shapes.items():
      for f in fields:
        if name in acc:
          out[name][f].copy_(acc[name][f])
        else:
          out[name][f].zero_()
