"""Device engine: uploads the static graph and weights, owns the HBM workspace and
drives the C ABI (`gcb_forward`) for one GraphCast instance on one GPU.

PyTorch is used for device memory and streams only; all arithmetic of the step
runs in libgraphcast_b200.so.  HBM layout (fp32 unless noted):

  grid_in    image [Ng, c_in_pad]  packed, normalised inputs + 3 structural + zero pad
  grid_lat   [Ng, 512]          latent grid nodes (updated in place vg0->vg1->vg2)
  mesh_lat   [Nm, 512]          latent mesh nodes (updated in place, 1 + 16 times)
  mesh_agg   [Nm, 512]          segment sums
  mesh_edge  [E_mesh, 512]      latent multi-mesh edges (receiver-sorted order)
  mesh_msg   [E_mesh, 512]      messages of the current step
  edge_a/b   [max(E_g2m,E_m2g), 512]  bipartite edge latents / messages
  hidden     image [max rows, 512]  hidden activations between the two layers of an MLP
  *_img      operand images (bf16 hi|lo in the tensor-core A layout) of every tensor that
             is consumed as an identity-row A operand: grid_in, grid_lat, mesh_lat,
             mesh_agg, mesh_edge, the embedded bipartite edges, the summed m2g messages
  grid_out   [Ng, 256]          decoder output (n_out valid columns)
  weights    per linear layer: bf16 hi|lo tile image (wgmma B operand) + fp32 copy
"""

from __future__ import annotations

import ctypes as C
from typing import Mapping, Optional

import numpy as np
import torch

from graphcast_b200 import _native
from graphcast_b200 import graph as graph_lib

LATENT = 512


def _ceil(x: int, m: int) -> int:
  return (x + m - 1) // m * m


def mlp_stem(gnn: str, prefix: str, set_name: str) -> str:
  """Haiku module path stem of one MLP (reference deep_typed_graph_net.py:205-208,
  251-262, 295-307, 315-319; gnn names graphcast.py:217,233,261)."""
  return f"{gnn}/~_networks_builder/{prefix}{set_name}"


class Engine:
  """One GraphCast model resident on one CUDA device."""

  def __init__(self, static_graph: graph_lib.StaticGraph,
               params: Mapping[str, Mapping[str, np.ndarray]], *,
               c_in: int, n_out: int, msg_steps: int, precision: str = "bf16x3",
               device: Optional[torch.device] = None, pregather: bool = True,
               fuse: bool = True, chain_lag: int = 0, image_residual: bool = True,
               deep_chains: bool = True, num_grid_owned: int = 0, num_mesh_owned: int = 0,
               reorder_mesh: bool = False):
    if precision not in _native.PRECISIONS:
      raise ValueError(f"unknown precision {precision!r}; expected one of "
                       f"{sorted(_native.PRECISIONS)}")
    self._lib = _native.lib()            # raises if the CUDA library is missing
    self._step_stream = None             # created on first use (see step)
    self._loss_workspace = None          # fp64 partial sums of output_loss, created on first use
    if not torch.cuda.is_available():
      raise RuntimeError("graphcast_b200 requires a CUDA device (no CPU fallback)")
    self.device = torch.device(device if device is not None else
                               f"cuda:{torch.cuda.current_device()}")
    if not 1 <= msg_steps <= _native.GCB_MAX_MSG_STEPS:
      raise ValueError("gnn_msg_steps out of range")
    if n_out > 256:
      raise ValueError("at most 256 output channels are supported")
    self.c_in = c_in                      # data channels (without structural)
    self.n_out = n_out
    self.msg_steps = msg_steps
    self.precision = precision
    # pregather: evaluate the first edge-MLP layer as  e@W_e + (v@W_s)[snd] + (v@W_r)[rcv]
    # (node-level projections gathered in the epilogue) -- 30 % fewer tensor-core MACs.
    self.pregather = bool(pregather)
    # fuse: both linears of every MLP run as one chain launch, the hidden activation stays in
    # an L2-resident scratch (gcb_chain_forward); False = one launch per linear (round-1 path).
    self.fuse = bool(fuse)
    self.chain_lag = int(chain_lag)
    # image_residual: latent streams live in HBM only as operand images (no fp32 masters).
    self.image_residual = bool(image_residual)
    # deep_chains (with image_residual): [edge embedder -> edge MLP] and [node MLP -> next
    # projections] as single launches; see gcb_model.deep_chains.
    self.deep_chains = bool(deep_chains)
    self.c_in_pad = _ceil(c_in + 3, 16)
    self.c_in_valid = _ceil(c_in + 3, 4)
    g = static_graph
    # Optional internal numbering of the mesh nodes along a space-filling curve (graph.spatial_order),
    # so that gathers through the mesh indices are local.  Measured at 0.25 degree: the processor's
    # edge block 1.33 -> 1.29 ms, but the segment sum 0.15 -> 0.19 ms (the high-degree coarse-level
    # nodes no longer sit together), no net gain: off by default.  mesh_order[new] = reference id;
    # `mesh_rows_in_reference_order` undoes it for tests.  Not used for partition-local graphs
    # (their owned / halo blocks are fixed by the exchange plan).
    self.mesh_order = None
    if reorder_mesh and not (num_grid_owned or num_mesh_owned):
      f = g.mesh_node_feats.astype(np.float64)
      cos_lat = np.sqrt(np.maximum(0.0, 1.0 - f[:, 0] ** 2))
      order = graph_lib.spatial_order(np.stack([cos_lat * f[:, 1], cos_lat * f[:, 2], f[:, 0]], 1))
      new_of_old = np.empty_like(order)
      new_of_old[order] = np.arange(order.size)
      import dataclasses as _dc
      g = _dc.replace(
          g, mesh_node_feats=np.ascontiguousarray(g.mesh_node_feats[order]),
          g2m_receivers=new_of_old[g.g2m_receivers].astype(np.int32),
          mesh_senders=new_of_old[g.mesh_senders].astype(np.int32),
          mesh_receivers=new_of_old[g.mesh_receivers].astype(np.int32),
          m2g_senders=new_of_old[g.m2g_senders].astype(np.int32))
      self.mesh_order = order
    self.num_grid, self.num_mesh = g.num_grid_nodes, g.num_mesh_nodes
    # Node-partitioned execution (partitioned.py): the local tables are [owned | halo]; node
    # updates, aggregation and the decoder cover the owned rows only.  0 = every row is owned.
    self.num_grid_owned, self.num_mesh_owned = int(num_grid_owned), int(num_mesh_owned)
    self._keep = []                       # device tensors referenced by raw pointer
    self._model = _native.Model()
    self._upload_graph(g)
    self._upload_weights(params)
    self._alloc_workspace()
    self.launches_per_step = 0

  # -- helpers -------------------------------------------------------------------
  def _dev(self, array: np.ndarray, dtype) -> torch.Tensor:
    t = torch.as_tensor(np.ascontiguousarray(array)).to(dtype).to(self.device)
    self._keep.append(t)
    return t

  @staticmethod
  def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()

  # -- static graph --------------------------------------------------------------
  def _upload_graph(self, g: graph_lib.StaticGraph) -> None:
    m = self._model
    m.num_grid, m.num_mesh = g.num_grid_nodes, g.num_mesh_nodes
    m.num_grid_owned, m.num_mesh_owned = self.num_grid_owned, self.num_mesh_owned
    # grid2mesh and multi-mesh edges in receiver-sorted execution order.
    p1, s1, r1, rp1 = graph_lib.receiver_sorted(g.g2m_senders, g.g2m_receivers, g.num_mesh_nodes)
    p2, s2, r2, rp2 = graph_lib.receiver_sorted(g.mesh_senders, g.mesh_receivers, g.num_mesh_nodes)
    expected = np.repeat(np.arange(self.num_grid_owned or g.num_grid_nodes, dtype=np.int64), 3)
    if g.m2g_receivers.shape[0] != expected.shape[0] or not np.array_equal(
        g.m2g_receivers.astype(np.int64), expected):
      raise ValueError("mesh2grid edges must be grouped by grid node with fan-in 3")
    m.e_g2m, m.e_mesh, m.e_m2g = len(s1), len(s2), len(g.m2g_senders)
    self.g2m_snd, self.g2m_rcv = self._dev(s1, torch.int32), self._dev(r1, torch.int32)
    self.g2m_row_ptr = self._dev(rp1, torch.int32)
    self.g2m_feat = self._dev(g.g2m_edge_feats[p1], torch.float32)
    heavy = np.nonzero(np.diff(rp1) > 256)[0].astype(np.int32)     # pole-side receivers
    self.g2m_heavy = self._dev(heavy if heavy.size else np.zeros([1], np.int32), torch.int32)
    m.g2m_heavy, m.n_g2m_heavy = self._ptr(self.g2m_heavy), int(heavy.size)
    self.mesh_snd, self.mesh_rcv = self._dev(s2, torch.int32), self._dev(r2, torch.int32)
    self.mesh_row_ptr = self._dev(rp2, torch.int32)
    self.mesh_feat = self._dev(g.mesh_edge_feats[p2], torch.float32)
    self.m2g_snd = self._dev(g.m2g_senders, torch.int32)
    self.m2g_rcv = self._dev(g.m2g_receivers, torch.int32)
    self.m2g_feat = self._dev(g.m2g_edge_feats, torch.float32)
    # Mesh-node encoder input: zeros for the data channels + 3 structural
    # features (reference graphcast.py:573-583).
    mesh_in = np.zeros([g.num_mesh_nodes, self.c_in_pad], np.float32)
    mesh_in[:, self.c_in:self.c_in + 3] = g.mesh_node_feats
    self.mesh_in = self._dev(mesh_in, torch.float32)
    self.grid_static = self._dev(g.grid_node_feats, torch.float32)   # [Ng,3]
    m.g2m_snd, m.g2m_rcv = self._ptr(self.g2m_snd), self._ptr(self.g2m_rcv)
    m.g2m_row_ptr, m.g2m_feat = self._ptr(self.g2m_row_ptr), self._ptr(self.g2m_feat)
    m.mesh_snd, m.mesh_rcv = self._ptr(self.mesh_snd), self._ptr(self.mesh_rcv)
    m.mesh_row_ptr, m.mesh_feat = self._ptr(self.mesh_row_ptr), self._ptr(self.mesh_feat)
    m.m2g_snd, m.m2g_rcv = self._ptr(self.m2g_snd), self._ptr(self.m2g_rcv)
    m.m2g_feat = self._ptr(self.m2g_feat)
    m.mesh_in = self._ptr(self.mesh_in)
    m.c_in_pad, m.c_in_valid = self.c_in_pad, self.c_in_valid
    m.msg_steps = self.msg_steps
    m.precision = _native.PRECISIONS[self.precision]
    m.pregather = 1 if self.pregather else 0

  # -- weights ---------------------------------------------------------------------
  def _pack_linear(self, w: np.ndarray, seg_real, seg_pad, n_pad: int):
    """w [sum(seg_real), n_real] -> (packed image tensor, fp32 padded tensor).

    Rows are re-laid so that segment s occupies seg_pad[s] rows (zero padded)."""
    w = np.asarray(w, np.float32)
    k_real, n_real = w.shape
    if k_real != sum(seg_real):
      raise ValueError(f"weight has {k_real} input rows, expected {sum(seg_real)}")
    k_pad = sum(seg_pad)
    wp = np.zeros([k_pad, n_pad], np.float32)
    src = dst = 0
    for real, pad in zip(seg_real, seg_pad):
      wp[dst:dst + real, :n_real] = w[src:src + real]
      src += real
      dst += pad
    nbytes = self._lib.gcb_packed_weight_bytes(k_pad, n_pad)
    img = np.empty([nbytes], np.uint8)
    _native.check(self._lib.gcb_pack_weight_host(
        wp.ctypes.data, k_pad, n_pad, k_pad, n_pad, img.ctypes.data), "gcb_pack_weight_host")
    return self._dev(img, torch.uint8), self._dev(wp, torch.float32), k_pad

  def _make_mlp(self, params, stem: str, seg_real, seg_pad, n1_real: int,
                layer_norm: bool) -> _native.Mlp:
    def get(name, field):
      try:
        return np.asarray(params[name][field], np.float32)
      except KeyError as e:
        raise KeyError(f"missing parameter {name}:{field}") from e
    if f"{stem}_mlp/~/linear_2" in params:
      raise ValueError("only hidden_layers=1 MLPs are supported")
    w0, b0 = get(f"{stem}_mlp/~/linear_0", "w"), get(f"{stem}_mlp/~/linear_0", "b")
    w1, b1 = get(f"{stem}_mlp/~/linear_1", "w"), get(f"{stem}_mlp/~/linear_1", "b")
    if w0.shape[1] != LATENT or w1.shape[0] != LATENT:
      raise ValueError(f"{stem}: only latent/hidden size {LATENT} is supported")
    if w1.shape[1] != n1_real:
      raise ValueError(f"{stem}: output width {w1.shape[1]} != expected {n1_real}")
    n1_pad = 512 if n1_real > 256 else 256
    if n1_real == LATENT:
      n1_pad = 512
    mlp = _native.Mlp()
    img0, f0, k0 = self._pack_linear(w0, seg_real, seg_pad, LATENT)
    img1, f1, _ = self._pack_linear(w1, [LATENT], [LATENT], n1_pad)
    pad = lambda v, n: np.concatenate([v, np.zeros([n - v.shape[0]], np.float32)])
    mlp.w0_packed, mlp.w0_f32 = self._ptr(img0), self._ptr(f0)
    mlp.b0 = self._ptr(self._dev(b0, torch.float32))
    mlp.w1_packed, mlp.w1_f32 = self._ptr(img1), self._ptr(f1)
    mlp.b1 = self._ptr(self._dev(pad(b1, n1_pad), torch.float32))
    if layer_norm:
      mlp.ln_scale = self._ptr(self._dev(pad(get(f"{stem}_layer_norm", "scale"), n1_pad),
                                         torch.float32))
      mlp.ln_offset = self._ptr(self._dev(pad(get(f"{stem}_layer_norm", "offset"), n1_pad),
                                          torch.float32))
    mlp.k0, mlp.n1, mlp.n1_valid = k0, n1_pad, n1_real
    return mlp

  def _make_split(self, params, stem: str) -> _native.MlpSplit:
    """Row blocks [edge | sender | receiver] of a [1536,512] first edge-MLP layer
    (concat order of the reference, typed_graph_net.py:637-638), each packed alone."""
    w0 = np.asarray(params[f"{stem}_mlp/~/linear_0"]["w"], np.float32)
    D = LATENT
    if w0.shape != (3 * D, D):
      raise ValueError(f"{stem}: expected a [{3 * D},{D}] first layer")
    sp = _native.MlpSplit()
    for name, block in (("we", w0[:D]), ("ws", w0[D:2 * D]), ("wr", w0[2 * D:])):
      img, f32, _ = self._pack_linear(block, [D], [D], D)
      setattr(sp, f"{name}_packed", self._ptr(img))
      setattr(sp, f"{name}_f32", self._ptr(f32))
    return sp

  def _upload_weights(self, params) -> None:
    m = self._model
    D = LATENT
    cin_real, cin_pad = self.c_in + 3, self.c_in_pad
    mk = self._make_mlp
    g = "grid2mesh_gnn"
    m.enc_grid = mk(params, mlp_stem(g, "encoder_nodes_", "grid_nodes"), [cin_real], [cin_pad], D, True)
    m.enc_mesh = mk(params, mlp_stem(g, "encoder_nodes_", "mesh_nodes"), [cin_real], [cin_pad], D, True)
    m.enc_e_g2m = mk(params, mlp_stem(g, "encoder_edges_", "grid2mesh"), [4], [16], D, True)
    m.proc_e_g2m = mk(params, mlp_stem(g, "processor_edges_0_", "grid2mesh"), [D] * 3, [D] * 3, D, True)
    m.proc_n_mesh_g2m = mk(params, mlp_stem(g, "processor_nodes_0_", "mesh_nodes"), [D] * 2, [D] * 2, D, True)
    m.proc_n_grid_g2m = mk(params, mlp_stem(g, "processor_nodes_0_", "grid_nodes"), [D], [D], D, True)
    g = "mesh_gnn"
    m.enc_e_mesh = mk(params, mlp_stem(g, "encoder_edges_", "mesh"), [4], [16], D, True)
    for k in range(self.msg_steps):
      m.proc_e_mesh[k] = mk(params, mlp_stem(g, f"processor_edges_{k}_", "mesh"), [D] * 3, [D] * 3, D, True)
      m.proc_n_mesh[k] = mk(params, mlp_stem(g, f"processor_nodes_{k}_", "mesh_nodes"), [D] * 2, [D] * 2, D, True)
    g = "mesh2grid_gnn"
    m.enc_e_m2g = mk(params, mlp_stem(g, "encoder_edges_", "mesh2grid"), [4], [16], D, True)
    m.proc_e_m2g = mk(params, mlp_stem(g, "processor_edges_0_", "mesh2grid"), [D] * 3, [D] * 3, D, True)
    m.proc_n_grid_m2g = mk(params, mlp_stem(g, "processor_nodes_0_", "grid_nodes"), [D] * 2, [D] * 2, D, True)
    m.dec_grid = mk(params, mlp_stem(g, "decoder_nodes_", "grid_nodes"), [D], [D], self.n_out, False)
    if self.pregather:
      m.proc_e_g2m_split = self._make_split(params, mlp_stem("grid2mesh_gnn", "processor_edges_0_", "grid2mesh"))
      m.proc_e_m2g_split = self._make_split(params, mlp_stem("mesh2grid_gnn", "processor_edges_0_", "mesh2grid"))
      for k in range(self.msg_steps):
        m.proc_e_mesh_split[k] = self._make_split(params, mlp_stem("mesh_gnn", f"processor_edges_{k}_", "mesh"))
      m.zero_bias = self._ptr(self._dev(np.zeros([D], np.float32), torch.float32))

  # -- workspace ---------------------------------------------------------------------
  def _image(self, rows: int, k: int = LATENT) -> torch.Tensor:
    # zeros: rows of the last 128-row tile beyond `rows` are never written by some producers
    return torch.zeros([self._lib.gcb_a_image_bytes(max(rows, 1), k)], dtype=torch.uint8,
                       device=self.device)

  def _alloc_workspace(self) -> None:
    m = self._model
    f = lambda rows, cols: torch.empty([max(rows, 1), cols], dtype=torch.float32, device=self.device)
    max_rows = max(m.num_grid, m.num_mesh, m.e_g2m, m.e_mesh, m.e_m2g)
    big_edges = max(m.e_g2m, m.e_m2g)
    # operand images (bf16 hi/lo in tensor-core A layout) and fp32 masters
    self.hidden = self._image(max_rows)
    self.edge_a_img = self._image(big_edges)
    self.edge_b = f(big_edges, LATENT)
    self.grid_in_img = self._image(m.num_grid, self.c_in_pad)
    self.mesh_in_img = self._image(m.num_mesh, self.c_in_pad)
    self.grid_lat, self.grid_lat_img = f(m.num_grid, LATENT), self._image(m.num_grid)
    self.mesh_lat, self.mesh_lat_img = f(m.num_mesh, LATENT), self._image(m.num_mesh)
    self.mesh_agg, self.mesh_agg_img = f(m.num_mesh, LATENT), self._image(m.num_mesh)
    self.mesh_edge, self.mesh_edge_img = f(m.e_mesh, LATENT), self._image(m.e_mesh)
    self.mesh_msg = f(m.e_mesh, LATENT)
    self.grid_agg_img = self._image(m.num_grid)
    self.grid_out = f(m.num_grid, 256)
    # static mesh-node encoder input as an image, built once
    with self._on_device():
      _native.check(self._lib.gcb_rows_to_image(self.mesh_in.data_ptr(), self.c_in_pad, 1, m.num_mesh,
                                                self.c_in_pad, self.mesh_in_img.data_ptr(),
                                                self._stream()), "gcb_rows_to_image")
    for name in ("hidden", "edge_a_img", "edge_b", "mesh_in_img", "grid_lat",
                 "grid_lat_img", "mesh_lat", "mesh_lat_img", "mesh_agg", "mesh_agg_img",
                 "mesh_edge", "mesh_edge_img", "mesh_msg", "grid_agg_img"):
      setattr(m, name, self._ptr(getattr(self, name)))
    m.fuse, m.chain_lag = (1 if self.fuse else 0), self.chain_lag
    m.image_residual = 1 if self.image_residual else 0
    m.deep_chains = 1 if self.deep_chains else 0
    nbytes = self._lib.gcb_chain_scratch_bytes(self.device.index or 0, 3, 2, 2)
    if nbytes <= 0:
      raise RuntimeError("gcb_chain_scratch_bytes failed")
    self.chain_scratch = torch.zeros([nbytes], dtype=torch.uint8, device=self.device)
    m.chain_scratch, m.chain_scratch_bytes = self._ptr(self.chain_scratch), nbytes
    if self.pregather:
      self.proj_grid = f(m.num_grid, LATENT)
      self.proj_mesh_a, self.proj_mesh_b = f(m.num_mesh, LATENT), f(m.num_mesh, LATENT)
      m.proj_grid = self._ptr(self.proj_grid)
      m.proj_mesh_a, m.proj_mesh_b = self._ptr(self.proj_mesh_a), self._ptr(self.proj_mesh_b)
      self.proj_grid_b = f(m.num_grid, LATENT)
      m.proj_grid_b = self._ptr(self.proj_grid_b)

  def mesh_rows_in_reference_order(self, table: torch.Tensor) -> torch.Tensor:
    """A [num_mesh, ...] device table (e.g. `mesh_lat`) re-indexed by the reference's mesh node ids."""
    if self.mesh_order is None:
      return table
    inv = torch.empty(self.num_mesh, dtype=torch.long, device=table.device)
    inv[torch.as_tensor(self.mesh_order, device=table.device)] = torch.arange(self.num_mesh, device=table.device)
    return table[inv]

  def workspace_bytes(self) -> int:
    ts = [self.hidden, self.edge_a_img, self.edge_b, self.grid_in_img,
          self.mesh_in_img, self.grid_lat, self.grid_lat_img, self.mesh_lat, self.mesh_lat_img,
          self.mesh_agg, self.mesh_agg_img, self.mesh_edge, self.mesh_edge_img, self.mesh_msg,
          self.grid_agg_img, self.grid_out]
    if self.pregather:
      ts += [self.proj_grid, self.proj_mesh_a, self.proj_mesh_b]
    return sum(t.numel() * t.element_size() for t in ts)

  # -- execution ---------------------------------------------------------------------
  def _stream(self) -> int:
    """Raw handle of the current stream of THIS engine's device (not of the current device)."""
    return torch.cuda.current_stream(self.device).cuda_stream

  def _on_device(self):
    """The C ABI launches on the calling thread's current CUDA device; make that ours."""
    return torch.cuda.device(self.device)

  def set_precision(self, precision: str) -> None:
    self._model.precision = _native.PRECISIONS[precision]
    self.precision = precision

  def pack_inputs(self, planes: torch.Tensor, mean: Optional[torch.Tensor] = None,
                  scale: Optional[torch.Tensor] = None,
                  out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """planes [c_in, Ng] (device, fp32, contiguous) -> operand image of the packed,
    normalised grid features [Ng, c_in_pad] (with the 3 structural features)."""
    if planes.shape != (self.c_in, self.num_grid) or planes.dtype != torch.float32 \
        or not planes.is_contiguous() or planes.device != self.device:
      raise ValueError(f"planes must be a contiguous fp32 [{self.c_in}, {self.num_grid}] "
                       f"tensor on {self.device}")
    out = self.grid_in_img if out is None else out
    with self._on_device():
      _native.check(self._lib.gcb_pack_grid_image(
          planes.data_ptr(), self.c_in, self.num_grid, self._ptr(mean), self._ptr(scale),
          self.grid_static.data_ptr(), 3, self.c_in_pad, out.data_ptr(), self._stream()),
          "gcb_pack_grid_image")
    return out

  def step(self, grid_in: Optional[torch.Tensor] = None,
           grid_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """grid_in (operand image of [Ng, c_in_pad]) -> grid_out [Ng, 256] (n_out valid columns)."""
    grid_in = self.grid_in_img if grid_in is None else grid_in
    grid_out = self.grid_out if grid_out is None else grid_out
    n = C.c_int32(0)
    cur = torch.cuda.current_stream(self.device)
    # The step replays a CUDA graph (gcb_set_graph_replay), which the legacy default stream
    # cannot capture: run it on the engine's own stream, fenced against the current one.
    side = cur.cuda_stream == 0
    if side:
      if self._step_stream is None:
        self._step_stream = torch.cuda.Stream(self.device)
      self._step_stream.wait_stream(cur)
    st = self._step_stream if side else cur
    with self._on_device():
      _native.check(self._lib.gcb_forward(C.byref(self._model), grid_in.data_ptr(),
                                          grid_out.data_ptr(), st.cuda_stream, C.byref(n)),
                    "gcb_forward")
    if side:
      cur.wait_stream(self._step_stream)
    self.launches_per_step = int(n.value)
    return grid_out

  def run_stage(self, stage: str, step: int = 0, grid_in: Optional[torch.Tensor] = None,
                grid_out: Optional[torch.Tensor] = None) -> int:
    """One stage of the step on the current stream (gcb_forward_stage): "encode",
    "process_embed", "process_step" (with `step`), "decode".  encode, process_embed,
    process_step 0..msg_steps-1, decode == step().  Returns the number of kernel launches."""
    stages = {"encode": _native.STAGE_ENCODE, "process_embed": _native.STAGE_PROCESS_EMBED,
              "process_step": _native.STAGE_PROCESS_STEP, "decode": _native.STAGE_DECODE}
    if stage not in stages:
      raise ValueError(f"unknown stage {stage!r}")
    grid_in = self.grid_in_img if grid_in is None else grid_in
    grid_out = self.grid_out if grid_out is None else grid_out
    n = C.c_int32(0)
    with self._on_device():
      _native.check(self._lib.gcb_forward_stage(
          C.byref(self._model), stages[stage], step, grid_in.data_ptr(), grid_out.data_ptr(),
          self._stream(), C.byref(n)), "gcb_forward_stage")
    return int(n.value)

  def unpack_outputs(self, planes_out: torch.Tensor, grid_out: Optional[torch.Tensor] = None,
                     scale: Optional[torch.Tensor] = None, offset: Optional[torch.Tensor] = None,
                     add_planes: Optional[torch.Tensor] = None,
                     add_plane_index: Optional[torch.Tensor] = None) -> torch.Tensor:
    """grid_out [Ng,256] -> planes_out [n_out, Ng] (optionally un-normalised +
    residual-added, see gcb_unpack_grid_outputs)."""
    grid_out = self.grid_out if grid_out is None else grid_out
    if planes_out.shape != (self.n_out, self.num_grid) or not planes_out.is_contiguous():
      raise ValueError("planes_out must be a contiguous [n_out, Ng] tensor")
    with self._on_device():
      _native.check(self._lib.gcb_unpack_grid_outputs(
          grid_out.data_ptr(), 256, self.n_out, self.num_grid, self._ptr(scale), self._ptr(offset),
          self._ptr(add_planes), self._ptr(add_plane_index), planes_out.data_ptr(), self._stream()),
          "gcb_unpack_grid_outputs")
    return planes_out

  def output_loss(self, targets_planes: torch.Tensor, lat_weight: torch.Tensor, *,
                  channel_sums: torch.Tensor, scale: Optional[torch.Tensor] = None,
                  offset: Optional[torch.Tensor] = None, add_planes: Optional[torch.Tensor] = None,
                  add_plane_index: Optional[torch.Tensor] = None,
                  planes_out: Optional[torch.Tensor] = None,
                  grid_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Latitude-weighted squared error of grid_out against the normalised targets, per output
    channel, into `channel_sums` ([n_out] fp64 device slice; see gcb_output_loss).  Optionally
    writes the predictions to `planes_out` as unpack_outputs would.  Launches on the current stream
    and does not synchronise, so a multi-step loss stays on the device until it is read."""
    if self.num_grid_owned:
      raise NotImplementedError(
          "the loss is not available in the node-partitioned engine: each rank holds only its own "
          "grid rows; evaluate it with a single-GPU GraphCast")
    grid_out = self.grid_out if grid_out is None else grid_out
    n_lat = lat_weight.shape[0]
    if n_lat == 0 or self.num_grid % n_lat:
      raise ValueError(f"{n_lat} latitude weights do not tile {self.num_grid} grid nodes")
    for name, t, dt, shape in (("targets_planes", targets_planes, torch.float32, (self.n_out, self.num_grid)),
                               ("lat_weight", lat_weight, torch.float32, (n_lat,)),
                               ("channel_sums", channel_sums, torch.float64, (self.n_out,)),
                               ("planes_out", planes_out, torch.float32, (self.n_out, self.num_grid))):
      if t is not None and (tuple(t.shape) != shape or t.dtype != dt or not t.is_contiguous()
                            or t.device != self.device):
        raise ValueError(f"{name} must be a contiguous {dt} {list(shape)} tensor on {self.device}")
    nbytes = self._lib.gcb_output_loss_workspace_bytes(self.n_out)
    ws = self._loss_workspace
    if ws is None or ws.numel() < nbytes:
      ws = self._loss_workspace = torch.empty([nbytes], dtype=torch.uint8, device=self.device)
    with self._on_device():
      _native.check(self._lib.gcb_output_loss(
          grid_out.data_ptr(), 256, self.n_out, n_lat, self.num_grid // n_lat, self._ptr(scale),
          self._ptr(offset), self._ptr(add_planes), self._ptr(add_plane_index),
          targets_planes.data_ptr(), lat_weight.data_ptr(), self._ptr(planes_out), ws.data_ptr(),
          nbytes, channel_sums.data_ptr(), self._stream()), "gcb_output_loss")
    return channel_sums

  def forward_features(self, grid_features: torch.Tensor) -> torch.Tensor:
    """Convenience for parity tests: grid_features [Ng, B, c_in] (the reference's
    `_inputs_to_grid_node_features` layout) -> [Ng, B, n_out]."""
    ng, batch, c = grid_features.shape
    outs = []
    for b in range(batch):
      planes = grid_features[:, b, :].t().contiguous().to(self.device, torch.float32)
      self.pack_inputs(planes)
      self.step()
      outs.append(self.grid_out[:, :self.n_out].clone())
    return torch.stack(outs, dim=1)
