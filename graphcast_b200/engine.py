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
from typing import List, Mapping, Optional

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
               reorder_mesh: bool = False, static_cache: bool = True):
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
    # static_cache (deep-chain path only): the weight-only edge terms -- the embedded edges' product
    # with the first edge-MLP layer's edge block, per graph, and the embedded mesh edges e0 -- are
    # computed once per weight version and precision (gcb_forward_static) instead of every step.
    # Built by step() when absent or stale and no gradient workspace exists; released by every
    # gradient, tangent and HVP path before it builds its workspace.
    self.static_cache = bool(static_cache)
    self._static = None                   # {name: tensor} of the cache, or None
    self._static_key = None               # (weights_version, precision) the cache was built for
    self._static_events = None            # CUDA events around the last build
    self.static_cache_builds = 0
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
    self._weights = {}                    # weight buffer groups, rewritten by load_params
    self._model = _native.Model()
    self._upload_graph(g)
    self._upload_weights(params)
    self._alloc_workspace()
    self.launches_per_step = 0
    self.param_shapes = {name: {f: tuple(np.shape(a)) for f, a in fields.items()}
                         for name, fields in params.items()}
    # The host dict of the weights (see `params`).  After load_params_device it is stale until read,
    # and so are the host copies by which load_params skips unchanged groups.
    self._host_params = params
    self._params_stale = False
    self._copies_stale = False
    self.weights_version = 0              # counts the reloads (load_params, load_params_device)
    self._backward = None                 # gradient workspace, created by the first loss_and_grads

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
    # senders in execution order (host): the sender CSRs of the backward pass are built from them
    self.exec_senders = {"g2m": s1, "mesh": s2, "m2g": np.asarray(g.m2g_senders, np.int32)}
    self.exec_row_ptr = {"g2m": rp1}      # receiver CSR of grid2mesh: the backward's edge chunks
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
    """w [sum(seg_real), n_real] -> (packed image, fp32 padded weight), host arrays.

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
    return img, wp

  def pack_weight(self, w: int, ld: int, transpose: bool, k_rows: int, n_cols: int, k: int, n: int,
                  img: torch.Tensor, f32: Optional[torch.Tensor] = None) -> None:
    """gcb_pack_weight on the current stream: the device fp32 matrix at address w (rows of `ld`
    floats, read transposed with `transpose`) -> the packed image `img` of padded shape [k, n] and,
    optionally, the zero-padded fp32 copy `f32` [k, n]."""
    _native.check(self._lib.gcb_pack_weight(w, ld, 1 if transpose else 0, k_rows, n_cols, k, n,
                                            img.data_ptr(), self._ptr(f32), self._stream()),
                  "gcb_pack_weight")

  def _pack_linear_device(self, w: torch.Tensor, seg_real, seg_pad, img: torch.Tensor,
                          f32: torch.Tensor) -> None:
    """The device twin of _pack_linear, into the existing buffers: one launch per padded segment
    (one in all for the unpadded multi-segment layers)."""
    k_real, n_real = w.shape
    n_pad = f32.shape[1]
    if list(seg_real) == list(seg_pad):
      seg_real = seg_pad = [k_real]
    src = dst = 0
    for real, pad in zip(seg_real, seg_pad):
      self.pack_weight(w.data_ptr() + 4 * src * n_real, n_real, False, real, n_real, pad, n_pad,
                       img[4 * dst * n_pad:], f32[dst:])
      src += real
      dst += pad

  def _upload_group(self, key, build, device_build, read, params, sources) -> dict:
    """Uploads the host arrays build(self, params) of one group of weight buffers and remembers how
    to rebuild them in place: from host arrays (load_params) and, with device_build(self, params,
    bufs), from device tensors (load_params_device).  read(self, bufs) -> {(module, field): device
    tensor} recovers the parameters the buffers hold (the `params` refresh).  sources: the (module,
    field) parameters they are made of.  The callables take the engine as an argument rather than
    closing over it: the engine keeps them, and a cycle would keep a dropped engine's device memory
    alive until the garbage collector ran."""
    bufs = {name: self._dev(a, torch.uint8 if a.dtype == np.uint8 else torch.float32)
            for name, a in build(self, params).items()}
    copies = [np.array(params[n][f], np.float32) for n, f in sources]
    self._weights[key] = (build, device_build, read, bufs, sources, copies)
    return bufs

  def _make_mlp(self, params, stem: str, seg_real, seg_pad, n1_real: int,
                layer_norm: bool) -> _native.Mlp:
    def get(params, name, field):
      try:
        return np.asarray(params[name][field], np.float32)
      except KeyError as e:
        raise KeyError(f"missing parameter {name}:{field}") from e
    if f"{stem}_mlp/~/linear_2" in params:
      raise ValueError("only hidden_layers=1 MLPs are supported")
    l0, l1, ln = f"{stem}_mlp/~/linear_0", f"{stem}_mlp/~/linear_1", f"{stem}_layer_norm"
    n1_pad = 512 if n1_real > 256 else 256
    if n1_real == LATENT:
      n1_pad = 512
    pad = lambda v, n: np.concatenate([v, np.zeros([n - v.shape[0]], np.float32)])

    def build(eng, params):
      w0, w1 = get(params, l0, "w"), get(params, l1, "w")
      if w0.shape[1] != LATENT or w1.shape[0] != LATENT:
        raise ValueError(f"{stem}: only latent/hidden size {LATENT} is supported")
      if w1.shape[1] != n1_real:
        raise ValueError(f"{stem}: output width {w1.shape[1]} != expected {n1_real}")
      out = {}
      out["w0_packed"], out["w0_f32"] = eng._pack_linear(w0, seg_real, seg_pad, LATENT)
      out["w1_packed"], out["w1_f32"] = eng._pack_linear(w1, [LATENT], [LATENT], n1_pad)
      out["b0"], out["b1"] = get(params, l0, "b"), pad(get(params, l1, "b"), n1_pad)
      if layer_norm:
        out["ln_scale"] = pad(get(params, ln, "scale"), n1_pad)
        out["ln_offset"] = pad(get(params, ln, "offset"), n1_pad)
      return out

    def device_build(eng, params, bufs):      # the padding of every buffer stays zero
      eng._pack_linear_device(params[l0]["w"], seg_real, seg_pad, bufs["w0_packed"], bufs["w0_f32"])
      eng._pack_linear_device(params[l1]["w"], [LATENT], [LATENT], bufs["w1_packed"], bufs["w1_f32"])
      bufs["b0"].copy_(params[l0]["b"])
      bufs["b1"][:n1_real].copy_(params[l1]["b"])
      if layer_norm:
        bufs["ln_scale"][:n1_real].copy_(params[ln]["scale"])
        bufs["ln_offset"][:n1_real].copy_(params[ln]["offset"])

    def read(eng, bufs):
      w0, rows, dst = bufs["w0_f32"], [], 0
      for real, padded in zip(seg_real, seg_pad):
        rows.append(w0[dst:dst + real])
        dst += padded
      out = {(l0, "w"): torch.cat(rows), (l0, "b"): bufs["b0"],
             (l1, "w"): bufs["w1_f32"][:, :n1_real], (l1, "b"): bufs["b1"][:n1_real]}
      if layer_norm:
        out[(ln, "scale")], out[(ln, "offset")] = bufs["ln_scale"][:n1_real], bufs["ln_offset"][:n1_real]
      return out
    sources = [(l0, "w"), (l0, "b"), (l1, "w"), (l1, "b")]
    if layer_norm:
      sources += [(ln, "scale"), (ln, "offset")]
    bufs = self._upload_group(stem, build, device_build, read, params, sources)
    mlp = _native.Mlp()
    for name, t in bufs.items():
      setattr(mlp, name, self._ptr(t))
    mlp.k0, mlp.n1, mlp.n1_valid = sum(seg_pad), n1_pad, n1_real
    return mlp

  def _make_split(self, params, stem: str) -> _native.MlpSplit:
    """Row blocks [edge | sender | receiver] of a [1536,512] first edge-MLP layer
    (concat order of the reference, typed_graph_net.py:637-638), each packed alone."""
    l0 = f"{stem}_mlp/~/linear_0"
    D = LATENT

    def build(eng, params):
      w0 = np.asarray(params[l0]["w"], np.float32)
      if w0.shape != (3 * D, D):
        raise ValueError(f"{stem}: expected a [{3 * D},{D}] first layer")
      out = {}
      for name, block in (("we", w0[:D]), ("ws", w0[D:2 * D]), ("wr", w0[2 * D:])):
        out[f"{name}_packed"], out[f"{name}_f32"] = eng._pack_linear(block, [D], [D], D)
      return out

    def device_build(eng, params, bufs):      # row block i: a pointer offset into w0
      w0 = params[l0]["w"]
      for i, name in enumerate(("we", "ws", "wr")):
        eng.pack_weight(w0.data_ptr() + 4 * i * D * D, D, False, D, D, D, D, bufs[f"{name}_packed"],
                        bufs[f"{name}_f32"])
    bufs = self._upload_group((stem, "split"), build, device_build, lambda eng, bufs: {}, params,
                              [(l0, "w")])
    sp = _native.MlpSplit()
    for name, t in bufs.items():
      setattr(sp, name, self._ptr(t))
    return sp

  def load_params(self, params: Mapping[str, Mapping[str, np.ndarray]]) -> None:
    """Rewrites every weight buffer from `params`, which must have the shapes of the current ones:
    packed and fp32 weights, padded biases and LayerNorm vectors, the pre-gathered split blocks, and
    the transposed weights of the gradient workspace if it exists.  The device pointers stay the
    same, so the recorded step graph stays valid and device memory does not grow.  Groups whose
    arrays equal what was loaded last are not repacked.  Raises ValueError on a missing parameter or
    a shape mismatch, before anything is written."""
    self._check_params(params, lambda b: np.shape(b))
    changed = set()
    for key, (build, _, _, bufs, sources, copies) in self._weights.items():
      new = [np.asarray(params[n][f], np.float32) for n, f in sources]
      if not self._copies_stale and all(np.array_equal(a, c) for a, c in zip(new, copies)):
        continue
      with self._on_device():
        for name, a in build(self, params).items():
          bufs[name].copy_(torch.from_numpy(a))
      for c, a in zip(copies, new):
        c[...] = a
      changed.add(key if isinstance(key, str) else key[0])
    self._host_params, self._params_stale, self._copies_stale = params, False, False
    self.weights_version += 1
    self._static_detach()                 # stale until the next step() rebuilds it
    if self._backward is not None:
      with self._on_device():
        self._backward.repack(changed)

  def load_params_device(self, params: Mapping[str, Mapping[str, torch.Tensor]]) -> None:
    """load_params from device tensors: `params` shaped like the params, contiguous fp32 tensors on
    this engine's device (views into one flat buffer are fine).  Rewrites the same buffers on the
    device, on the current stream and without a host synchronisation: the packed images and fp32
    copies through gcb_pack_weight, the padded biases and LayerNorm vectors, the split blocks and the
    backward pass's transposed weights.  Pointers stay the same and nothing is allocated.  Raises
    ValueError on a missing parameter or a shape, dtype or device mismatch, before anything is
    written.  Afterwards `params` and the host copies of load_params are stale: the next read of
    `params` refreshes it from the device, and the next load_params repacks every group."""
    def shape(t):
      if not (isinstance(t, torch.Tensor) and t.dtype == torch.float32 and t.device == self.device
              and t.is_contiguous()):
        raise ValueError(f"load_params_device takes contiguous float32 tensors on {self.device}")
      return tuple(t.shape)
    self._check_params(params, shape)
    with self._on_device():
      for build, device_build, _, bufs, _, _ in self._weights.values():
        device_build(self, params, bufs)
      if self._backward is not None:
        self._backward.repack()
    self._params_stale = self._copies_stale = True
    self.weights_version += 1
    self._static_detach()

  def _check_params(self, params, shape) -> None:
    for name, fields in self.param_shapes.items():
      for f, want in fields.items():
        try:
          b = params[name][f]
        except KeyError:
          raise ValueError(f"missing parameter {name}:{f}") from None
        if shape(b) != want:
          raise ValueError(f"{name}:{f} has shape {shape(b)}, the engine holds {want}")

  @property
  def params(self) -> Mapping[str, Mapping[str, np.ndarray]]:
    """The host dict of the weights the engine holds: the dict of the last load_params (or of the
    constructor), or, after load_params_device, a refresh from the engine's fp32 weight buffers, made
    on first read with one device-to-host copy.  Parameters the step never reads (the mesh2grid
    mesh-node MLP) keep their last host values."""
    if self._params_stale:
      held = {}
      for _, _, read, bufs, _, _ in self._weights.values():
        held.update(read(self, bufs))
      keys = sorted(held)
      with self._on_device():
        flat = torch.cat([held[k].reshape(-1) for k in keys]).cpu().numpy()
      new = {name: dict(fields) for name, fields in self._host_params.items()}
      off = 0
      for name, f in keys:
        shape = self.param_shapes[name][f]
        size = int(np.prod(shape))
        new[name][f] = flat[off:off + size].reshape(shape)
        off += size
      self._host_params, self._params_stale = new, False
    return self._host_params

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
    if self._static is not None:
      ts += list(self._static.values())
    return sum(t.numel() * t.element_size() for t in ts)

  # -- static-edge cache (gcb_forward_static) ------------------------------------------------
  def _static_eligible(self) -> bool:
    """The deep-chain path runs (the C side's condition for gcb_model.deep_chains)."""
    return (self.static_cache and self.image_residual and self.fuse and self.pregather and
            self.deep_chains and self.precision in ("bf16x3", "bf16") and
            not (self.num_grid_owned or self.num_mesh_owned))

  def _static_detach(self) -> None:
    """The step stops reading the cache (its tables are kept for a rebuild in place)."""
    m = self._model
    m.static_acc_g2m = m.static_acc_m2g = m.static_acc_mesh = m.static_e0_img = None
    self._static_key = None

  def release_static_cache(self) -> None:
    """Frees the static-edge cache; the next step() builds it again."""
    self._static_detach()
    self._static = None

  def _ensure_static_cache(self, stream: torch.cuda.Stream) -> None:
    """Builds the static-edge cache on `stream` when the step can use it and it is absent or stale."""
    if not self._static_eligible():
      if self._static is not None:
        self.release_static_cache()
      return
    if self._backward is not None:
      # A gradient workspace exists: the steps are most likely the forward of the next gradient,
      # tangent or HVP call, which frees the cache again before its backward pass, so a build would
      # cost 10 GiB (0.25 degree) next to the workspace for a few steps.  Inference gets the cache
      # back after release_gradient_workspace().
      return
    key = (self.weights_version, self.precision)
    if self._static is not None and self._static_key == key:
      return
    m = self._model
    self._static_detach()
    if self._static is None:
      f = lambda rows: torch.empty([max(rows, 1), LATENT], dtype=torch.float32, device=self.device)
      self._static = {"acc_g2m": f(m.e_g2m), "acc_m2g": f(m.e_m2g), "acc_mesh": f(m.e_mesh),
                      "e0_img": self._image(m.e_mesh)}
      cur = torch.cuda.current_stream(self.device)
      if stream != cur:
        # The tables were allocated, and the image zero-filled, on the current stream; the build
        # and the steps that read them run on `stream`.
        stream.wait_stream(cur)
        for t in self._static.values():
          t.record_stream(stream)
    t = self._static
    m.static_acc_g2m, m.static_acc_m2g = self._ptr(t["acc_g2m"]), self._ptr(t["acc_m2g"])
    m.static_acc_mesh, m.static_e0_img = self._ptr(t["acc_mesh"]), self._ptr(t["e0_img"])
    ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
    ev[0].record(stream)
    try:
      _native.check(self._lib.gcb_forward_static(C.byref(m), stream.cuda_stream, None),
                    "gcb_forward_static")
    except Exception:
      self.release_static_cache()
      raise
    ev[1].record(stream)
    self._static_events = ev
    self._static_key = key
    self.static_cache_builds += 1

  def static_cache_build_ms(self) -> Optional[float]:
    """Device time of the last static-edge cache build in ms (synchronises with it), or None."""
    if self._static_events is None:
      return None
    self._static_events[1].synchronize()
    return self._static_events[0].elapsed_time(self._static_events[1])

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
    self._static_detach()                 # the cache holds products of the old precision

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
      self._ensure_static_cache(st)
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

  # -- parameter gradients (graphcast_b200/backward.py) ------------------------------------------------
  def grads_begin(self, chunk_rows: Optional[int] = None) -> None:
    """Zeroes the gradient accumulators of `loss_and_grads_element`; the gradient workspace (transposed
    weights, sender CSRs, accumulators) is created by the first call, so inference never holds it.
    chunk_rows: edges per chunk of the grid2mesh / mesh2grid edge-MLP backward passes (default 2^19;
    the peak memory of the backward pass scales with it)."""
    self._grad_workspace(chunk_rows, "parameter gradients")
    self._backward.zero_grads()

  def release_gradient_workspace(self) -> None:
    """Frees the gradient workspace of the gradient, tangent and HVP paths, with the parameter
    gradients it accumulated (the next such call builds it again).  While it exists, step() runs
    without the static-edge cache."""
    self._backward = None

  def _grad_workspace(self, chunk_rows: Optional[int], what: str) -> None:
    """The checks of every gradient and the gradient workspace, created on first use.  The static-edge
    cache is released first: the derivative paths run the step without it, and at 0.25 degree their
    peaks leave no room for it."""
    self.release_static_cache()
    if self.num_grid_owned:
      raise NotImplementedError(
          f"{what} are not available in the node-partitioned engine: each rank holds "
          "only its own grid rows; compute them with a single-GPU GraphCast")
    if self.precision not in ("bf16x3", "bf16"):
      raise NotImplementedError(f"{what} support the tensor-core precisions 'bf16x3' "
                                f"and 'bf16', not {self.precision!r}")
    if self._backward is None or (chunk_rows and chunk_rows != self._backward.chunk_rows):
      from graphcast_b200 import backward
      self._backward = None
      with self._on_device():
        self._backward = (backward.Backward(self, chunk_rows) if chunk_rows
                          else backward.Backward(self))
    self._backward.prec = _native.PRECISIONS[self.precision]

  def loss_and_grads_element(self, targets_planes: torch.Tensor, lat_weight: torch.Tensor,
                             coef: torch.Tensor, *, channel_sums: torch.Tensor,
                             grid_in: Optional[torch.Tensor] = None,
                             feedback: Optional["Feedback"] = None, input_grad: bool = False,
                             **affine) -> None:
    """One batch element: the step stage by stage from `grid_in` (default: the packed grid_in_img)
    with snapshots of what the backward pass reads, the loss sums of `output_loss` into channel_sums,
    the loss derivative seed (gcb_output_loss_grad with coef = 2 kappa / batch) and the backward pass,
    which ADDS this element's parameter gradients to the accumulators (see grads_begin / grads).

    feedback: one step of backprop through time.  The seed also carries feedback.a, dL/d(inputs) of
    the following step (None for the last step), into the predictions (gcb_output_loss_grad_feedback);
    with input_grad, feedback.a is then replaced by dL/d(inputs) of this step, the residual and
    frame-shift terms from the seed plus the derivative through the grid embedder (gcb_input_grad),
    else it is dropped."""
    if self._backward is None:
      raise RuntimeError("call grads_begin() first")
    if feedback is not None:
      self._bptt_element(targets_planes, lat_weight, coef, channel_sums, grid_in, feedback,
                         input_grad, affine)
      return
    grid_in = self.grid_in_img if grid_in is None else grid_in
    snaps = self._forward_snapshots(grid_in)
    self.output_loss(targets_planes, lat_weight, channel_sums=channel_sums, **affine)
    g_out = torch.zeros([self.num_grid, 256], dtype=torch.float32, device=self.device)
    with self._on_device():
      self._loss_seed(self.grid_out, targets_planes, lat_weight, coef, g_out, affine)
      self._backward.element(grid_in, g_out, snaps)

  def _loss_seed(self, y: torch.Tensor, targets_planes: torch.Tensor, lat_weight: torch.Tensor,
                 coef: torch.Tensor, g: torch.Tensor, affine: dict, fb: Optional["Feedback"] = None,
                 a_next: Optional[torch.Tensor] = None, a_out: Optional[torch.Tensor] = None,
                 n_rows: int = 0) -> None:
    """The loss derivative seed of the decoder output y [Ng, ld] into the rows of g (row stride 256),
    with `affine` the output normalisation (scale, offset, add_planes, add_plane_index; absent: none):
    gcb_output_loss_grad, or with fb, gcb_output_loss_grad_feedback, which also carries a_next (the
    following step's gradient on fb's rows, or None) into the seed and writes the residual and
    frame-shift terms of n_rows rows to a_out."""
    n_lat = lat_weight.shape[0]
    head = (y.data_ptr(), y.shape[1], self.n_out, n_lat, self.num_grid // n_lat,
            self._ptr(affine.get("scale")), self._ptr(affine.get("offset")),
            self._ptr(affine.get("add_planes")), self._ptr(affine.get("add_plane_index")),
            targets_planes.data_ptr(), lat_weight.data_ptr(), coef.data_ptr())
    if fb is None:
      _native.check(self._lib.gcb_output_loss_grad(*head, g.data_ptr(), 256, self._stream()),
                    "gcb_output_loss_grad")
      return
    _native.check(self._lib.gcb_output_loss_grad_feedback(
        *head, self._ptr(a_next), fb.dpred_row.data_ptr(), n_rows, fb.resid_channel.data_ptr(),
        fb.carry_row.data_ptr(), self._ptr(a_out), g.data_ptr(), 256, self._stream()),
        "gcb_output_loss_grad_feedback")

  def _gn_seed(self, dy: torch.Tensor, lat_weight: torch.Tensor, coef: torch.Tensor,
               g: torch.Tensor) -> None:
    """The Gauss-Newton seed coef * lat_weight * dy of the decoder tangent dy [Ng, ld] into the rows
    of g (row stride 256): gcb_output_loss_gn_seed."""
    n_lat = lat_weight.shape[0]
    _native.check(self._lib.gcb_output_loss_gn_seed(
        dy.data_ptr(), dy.shape[1], self.n_out, n_lat, self.num_grid // n_lat, lat_weight.data_ptr(),
        coef.data_ptr(), g.data_ptr(), 256, self._stream()), "gcb_output_loss_gn_seed")

  def _pack_tangents(self, planes: List[torch.Tensor], in_scale: Optional[torch.Tensor],
                     stride: int) -> torch.Tensor:
    """The stacked operand image of K tangent planes [c_in, Ng] (direction k from row k * stride),
    each packed as pack_inputs packs the planes, without the mean (in_scale: the input normalisation's
    scale) and with zero structural features."""
    dgrid_in = self._image((len(planes) - 1) * stride + self.num_grid, self.c_in_pad)
    img_stride = self._lib.gcb_a_image_bytes(stride, self.c_in_pad)
    no_static = torch.zeros([self.num_grid, 3], dtype=torch.float32, device=self.device)
    for k, p in enumerate(planes):
      _native.check(self._lib.gcb_pack_grid_image(
          p.data_ptr(), self.c_in, self.num_grid, None, self._ptr(in_scale), no_static.data_ptr(), 3,
          self.c_in_pad, dgrid_in.data_ptr() + k * img_stride, self._stream()), "gcb_pack_grid_image")
    return dgrid_in

  def _input_grad_tail(self, dx: torch.Tensor, fb: "Feedback", a_outs, stride: int) -> None:
    """gcb_input_grad of every direction k of the backward pass's input-image gradient dx (from row
    k * stride) into a_outs[k] [fb.n_rows, Ng]: the derivative through the grid embedder, added to the
    seed's terms there."""
    for k, a in enumerate(a_outs):
      _native.check(self._lib.gcb_input_grad(
          dx[k * stride:].data_ptr(), dx.shape[1], self.num_grid, fb.n_rows, fb.rows.data_ptr(),
          self._ptr(fb.in_scale), a.data_ptr(), 1, self._stream()), "gcb_input_grad")

  def _forward_snapshots(self, grid_in: torch.Tensor) -> dict:
    """The step stage by stage, with copies of what the backward pass reads."""
    snaps = {"v": [], "agg": [], "e": [None]}
    self.run_stage("encode", grid_in=grid_in)
    snaps["vg1"], snaps["agg1"] = self.grid_lat_img.clone(), self.mesh_agg_img.clone()
    snaps["v"].append(self.mesh_lat_img.clone())
    self.run_stage("process_embed")
    for k in range(self.msg_steps):
      self.run_stage("process_step", k)
      snaps["v"].append(self.mesh_lat_img.clone())
      snaps["agg"].append(self.mesh_agg_img.clone())
      if k < self.msg_steps - 1:
        snaps["e"].append(self.mesh_edge_img.clone())
    self.run_stage("decode", grid_in=grid_in)
    snaps["vg2"], snaps["agg3"] = self.grid_lat_img.clone(), self.grid_agg_img.clone()
    return snaps

  def _bptt_element(self, targets_planes, lat_weight, coef, channel_sums, grid_in, fb: "Feedback",
                    input_grad: bool, affine) -> None:
    def seed(g_out, a_out, n_rows):
      self.output_loss(targets_planes, lat_weight, channel_sums=channel_sums, **affine)
      self._loss_seed(self.grid_out, targets_planes, lat_weight, coef, g_out, affine, fb=fb,
                      a_next=fb.a, a_out=a_out, n_rows=n_rows)
    self._bptt_walk(grid_in, fb, input_grad, seed)

  def param_gnvp_bptt_element(self, pred_tangent: torch.Tensor, lat_weight: torch.Tensor,
                              coef: torch.Tensor, *, feedback: "Feedback", input_grad: bool,
                              grid_in: Optional[torch.Tensor] = None,
                              scale: Optional[torch.Tensor] = None) -> None:
    """One step of one batch element of a Gauss-Newton product over several target times (call
    grads_begin() first): loss_and_grads_element(feedback=...) with the Gauss-Newton seed in place of
    the loss seed, and no loss.  pred_tangent [n_out, Ng] is this step's tangent of the physical
    predictions along the parameter tangents, through the whole rollout before it (the stash of the
    forward); scale the output normalisation's scale (None: 1).  The step runs again stage by stage
    from `grid_in` with its snapshots, gcb_output_loss_gn_seed_feedback seeds coef * lat_weight *
    pred_tangent / scale plus the feedback of the following step, and the backward pass ADDS this
    step's J^T Lambda J v terms to the gradient accumulators; with input_grad, feedback.a becomes this
    step's input-plane cotangent (gcb_input_grad).  No tangent runs here: J v is pred_tangent."""
    if self._backward is None:
      raise RuntimeError("call grads_begin() first")
    if (tuple(pred_tangent.shape) != (self.n_out, self.num_grid) or pred_tangent.dtype != torch.float32
        or not pred_tangent.is_contiguous() or pred_tangent.device != self.device):
      raise ValueError(f"pred_tangent must be a contiguous float32 [{self.n_out}, {self.num_grid}] "
                       f"tensor on {self.device}")
    n_lat = lat_weight.shape[0]
    fb = feedback

    def seed(g_out, a_out, n_rows):
      _native.check(self._lib.gcb_output_loss_gn_seed_feedback(
          pred_tangent.data_ptr(), self.n_out, n_lat, self.num_grid // n_lat, self._ptr(scale),
          lat_weight.data_ptr(), coef.data_ptr(), self._ptr(fb.a), fb.dpred_row.data_ptr(), n_rows,
          fb.resid_channel.data_ptr(), fb.carry_row.data_ptr(), self._ptr(a_out), g_out.data_ptr(),
          256, self._stream()), "gcb_output_loss_gn_seed_feedback")
    self._bptt_walk(grid_in, fb, input_grad, seed)

  def _bptt_walk(self, grid_in, fb: "Feedback", input_grad: bool, seed) -> None:
    """The step of a backprop-through-time element: the recompute with snapshots, seed(g_out, a_out,
    n_rows) (which reads fb.a), the backward pass with parameter gradients and, with input_grad, the
    input gradient into fb.a."""
    grid_in = self.grid_in_img if grid_in is None else grid_in
    snaps = self._forward_snapshots(grid_in)
    g_out = torch.zeros([self.num_grid, 256], dtype=torch.float32, device=self.device)
    n_rows = fb.n_rows if input_grad else 0
    a_out = torch.empty([n_rows, self.num_grid], dtype=torch.float32, device=self.device) \
        if n_rows else None
    with self._on_device():
      seed(g_out, a_out, n_rows)
      fb.a = a_out                         # the following step's rows are consumed: release them
      dx = self._backward.element(grid_in, g_out, snaps, dgrid_in=bool(n_rows))
      if n_rows:
        self._input_grad_tail(dx, fb, [a_out], 0)

  # -- input gradients (loss_and_input_grads, input_vjp) ---------------------------------------------
  def input_grads_begin(self, what: str = "input gradients") -> None:
    """The gradient workspace of `input_grads_element`, with the checks of grads_begin (`what` names
    the call in their messages); the parameter accumulators are neither zeroed nor touched."""
    self._grad_workspace(None, what)

  def input_grads_element(self, fb: "Feedback", operands: dict, *,
                          lat_weight: Optional[torch.Tensor] = None, coef: Optional[torch.Tensor] = None,
                          channel_sums: Optional[torch.Tensor] = None,
                          planes_out: Optional[torch.Tensor] = None,
                          grid_in: Optional[torch.Tensor] = None) -> None:
    """One step of one batch element of an input gradient: the step stage by stage from `grid_in`
    (default: the packed grid_in_img), the seed, and the backward pass without parameter gradients
    (Backward.element(param_grads=False)).  Afterwards fb.a [fb.n_rows, Ng] is the derivative with
    respect to this step's input planes (physical units) on fb's rows, fb.a of the following step
    having been consumed by the seed.

    With channel_sums the forward's loss sums go there (output_loss); with planes_out its predictions
    (unpack_outputs), as the step and unpack of __call__ would give them.  Both are optional: a
    recomputed step of a rollout needs neither.

    The seed is either the loss of loss_and_grads_element (operands["targets_planes"], lat_weight,
    coef = 2 kappa / (batch * steps): gcb_output_loss_grad_feedback) or, with
    operands["cotangent"] [n_out, Ng], J = sum cotangent * prediction
    (gcb_output_cotangent_grad_feedback).  `operands` also holds the affine keywords of output_loss
    (scale, offset, add_planes, add_plane_index).  The seed is their last reader: the dict is cleared
    after it, so that planes the caller no longer references are free during the backward pass.

    Several cotangents at once (batched_input_vjp): operands["cotangent"] [K, n_out, Ng], contiguous.
    fb.a is then [K, fb.n_rows, Ng], direction k's rows; the seed and gcb_input_grad run per direction,
    the backward pass once for all of them (Backward.element(dirs=K)), and direction k is bit for bit
    what its cotangent alone gives."""
    if self._backward is None:
      raise RuntimeError("call input_grads_begin() first")
    affine = {k: operands[k] for k in ("scale", "offset", "add_planes", "add_plane_index")
              if k in operands}
    targets_planes, cotangent = operands.get("targets_planes"), operands.get("cotangent")
    operands.clear()
    single = cotangent is None or cotangent.dim() == 2
    dirs = 1 if single else cotangent.shape[0]
    if not single and (tuple(cotangent.shape) != (dirs, self.n_out, self.num_grid) or dirs < 1
                       or not cotangent.is_contiguous()):
      raise ValueError(f"cotangent must be a contiguous [K, {self.n_out}, {self.num_grid}] tensor")
    grid_in = self.grid_in_img if grid_in is None else grid_in
    snaps = self._forward_snapshots(grid_in)
    stride = self._backward.dir_stride(self.num_grid)
    g_out = torch.zeros([(dirs - 1) * stride + self.num_grid, 256], dtype=torch.float32,
                        device=self.device)
    a_out = torch.empty(([] if single else [dirs]) + [fb.n_rows, self.num_grid], dtype=torch.float32,
                        device=self.device)
    a_outs = [a_out] if single else list(a_out.unbind(0))
    with self._on_device():
      if planes_out is not None:
        self.unpack_outputs(planes_out, **affine)
      if channel_sums is not None:
        self.output_loss(targets_planes, lat_weight, channel_sums=channel_sums, **affine)
      if cotangent is None:
        self._loss_seed(self.grid_out, targets_planes, lat_weight, coef, g_out, affine, fb=fb,
                        a_next=fb.a, a_out=a_out, n_rows=fb.n_rows)
      else:
        if single and (tuple(cotangent.shape) != (self.n_out, self.num_grid)
                       or not cotangent.is_contiguous()):
          raise ValueError(f"cotangent must be a contiguous [{self.n_out}, {self.num_grid}] tensor")
        cots = [cotangent] if single else list(cotangent.unbind(0))
        a_next = [fb.a] if single else [None] * dirs if fb.a is None else list(fb.a.unbind(0))
        for k in range(dirs):
          _native.check(self._lib.gcb_output_cotangent_grad_feedback(
              self.n_out, self.num_grid, self._ptr(affine.get("scale")), cots[k].data_ptr(),
              self._ptr(a_next[k]), fb.dpred_row.data_ptr(), fb.n_rows, fb.resid_channel.data_ptr(),
              fb.carry_row.data_ptr(), a_outs[k].data_ptr(), g_out[k * stride:].data_ptr(), 256,
              self._stream()), "gcb_output_cotangent_grad_feedback")
        del cots, a_next
      # the following step's rows, the planes, targets and cotangent are consumed: release them
      fb.a = a_out
      affine = targets_planes = cotangent = None
      dx = self._backward.element(grid_in, g_out, snaps, dgrid_in=True, param_grads=False, dirs=dirs)
      self._input_grad_tail(dx, fb, a_outs, stride)

  # -- Hessian-vector products (loss_and_input_hvp) ---------------------------------------------------
  def input_hvp_element(self, fb: "Feedback", operands: dict, *, lat_weight: torch.Tensor,
                        coef: torch.Tensor, channel_sums: Optional[torch.Tensor] = None,
                        planes_out: Optional[torch.Tensor] = None,
                        grid_in: Optional[torch.Tensor] = None,
                        zero_targets: Optional[torch.Tensor] = None) -> None:
    """One step of one batch element of a Hessian-vector product of the loss (call input_grads_begin()
    first).  operands: "targets_planes", "tangent_planes" [c_in, Ng] (the tangent v of this step's
    input planes, physical units) or [K, c_in, Ng] (K tangents v_1..v_K, each direction's planes
    contiguous; batched_loss_and_input_hvp) and the affine keywords of output_loss.  fb.a is None or
    [1 + K, fb.n_rows, Ng] of the following step: direction 0 its gradient, direction j that gradient's
    derivative along v_j; afterwards it is this step's.  channel_sums and planes_out as in
    input_grads_element; zero_targets: a zero [n_out, Ng] float32 plane for the seed's tangents, shared
    by the elements of a call (None: one is allocated here).

    The step runs stage by stage with its K tangents (Backward.tangent(dirs=K)), each packed into its
    slice of one stacked image as input_jvp_element packs them, keeping the primal and tangent
    snapshots.  Direction 0 of the seed is input_grads_element's loss seed.  The seed is affine in
    (y, the add planes, fb.a), so direction j is the same kernel on their tangents along v_j with zero
    targets: y-dot_j, add_planes = v_j (so that t_norm = -v_j[add] / scale), no offset and fb.a's
    direction j.  All 1 + K directions then share one backward walk (Backward.element(dirs=1 + K,
    hvp=...)), and gcb_input_grad runs per direction.  Direction 0 is bit for bit what
    input_grads_element gives, and direction j what the [c_in, Ng] call gives along v_j alone."""
    if self._backward is None:
      raise RuntimeError("call input_grads_begin() first")
    affine = {k: operands[k] for k in ("scale", "offset", "add_planes", "add_plane_index")
              if k in operands}
    targets_planes, tangent = operands["targets_planes"], operands["tangent_planes"]
    operands.clear()
    single = tangent.dim() == 2
    nt = 1 if single else tangent.shape[0]
    lead = () if single else (nt,)
    if (tuple(tangent.shape) != lead + (self.c_in, self.num_grid) or tangent.dtype != torch.float32
        or tangent.stride()[-2:] != (self.num_grid, 1) or nt < 1):
      raise ValueError(f"tangent_planes must be a float32 {list(lead + (self.c_in, self.num_grid))} "
                       f"tensor with contiguous [{self.c_in}, {self.num_grid}] planes per direction")
    planes = [tangent] if single else list(tangent.unbind(0))
    grid_in = self.grid_in_img if grid_in is None else grid_in
    stride = self._backward.dir_stride(self.num_grid)
    add_index = affine.get("add_plane_index")
    with self._on_device():
      dgrid_in = self._pack_tangents(planes, fb.in_scale, stride)
      snaps, tsnaps = {}, {}
      dy = self._backward.tangent(grid_in, dgrid_in, nt, snaps=snaps, tsnaps=tsnaps)
      del dgrid_in
      if planes_out is not None:
        self.unpack_outputs(planes_out, **affine)
      if channel_sums is not None:
        self.output_loss(targets_planes, lat_weight, channel_sums=channel_sums, **affine)
      g_out = torch.zeros([nt * stride + self.num_grid, 256], dtype=torch.float32, device=self.device)
      a_out = torch.empty([1 + nt, fb.n_rows, self.num_grid], dtype=torch.float32, device=self.device)
      a_next = [None] * (1 + nt) if fb.a is None else list(fb.a.unbind(0))
      if zero_targets is None:
        zero_targets = torch.zeros([self.n_out, self.num_grid], dtype=torch.float32,
                                   device=self.device)
      seeds = [(self.grid_out, affine, targets_planes)]
      seeds += [(dy[k * stride:], dict(scale=affine.get("scale"), add_plane_index=add_index,
                                       add_planes=None if add_index is None else p), zero_targets)
                for k, p in enumerate(planes)]
      for k, (y, seed_affine, targets) in enumerate(seeds):
        self._loss_seed(y, targets, lat_weight, coef, g_out[k * stride:], seed_affine, fb=fb,
                        a_next=a_next[k], a_out=a_out[k], n_rows=fb.n_rows)
      # the following step's rows, the planes, targets and tangents are consumed: release them
      fb.a = a_out
      del seeds, y, seed_affine, targets, a_next, zero_targets, dy, planes
      affine = targets_planes = tangent = None
      dx = self._backward.element(grid_in, g_out, snaps, dgrid_in=True, param_grads=False,
                                  dirs=1 + nt, hvp=tsnaps)
      del g_out, snaps, tsnaps
      self._input_grad_tail(dx, fb, a_out.unbind(0), stride)

  # -- tangent-linear model (input_jvp, batched_input_jvp) --------------------------------------------
  def input_jvp_element(self, tangent_planes: torch.Tensor, tangent_out: torch.Tensor, *,
                        in_scale: Optional[torch.Tensor] = None,
                        planes_out: Optional[torch.Tensor] = None,
                        grid_in: Optional[torch.Tensor] = None, weight_tangents=None,
                        **affine) -> None:
    """One step of one batch element of the tangent-linear forecast (call input_grads_begin() first):
    the step stage by stage from `grid_in` (default: the packed grid_in_img) interleaved with its
    tangent (Backward.tangent) along tangent_planes [c_in, Ng], the tangent of this step's input planes
    in physical units, or along several directions at once, tangent_planes [K, c_in, Ng] (each
    direction's planes contiguous).  They are packed as pack_inputs packs the planes, without the mean
    (in_scale: the input normalisation's scale) and with zero structural features, each direction into
    its slice of one stacked image.  tangent_out [n_out, Ng] ([K, n_out, Ng]) receives the tangent of
    the physical predictions: the decoder tangent times affine["scale"] plus, through the residual add,
    tangent_planes[affine["add_plane_index"]] (gcb_unpack_grid_outputs without the offset), unpacked
    per direction.  With planes_out, the predictions as unpack_outputs gives them from the same
    forward.  `affine`: the keywords of unpack_outputs (scale, offset, add_planes, add_plane_index).

    weight_tangents (param_jvp, one direction): packed parameter tangents (weight_tangents()), along
    which the step's tangent also runs (Backward.tangent(wts=...)); tangent_planes is then the input
    tangent fed back from the step before (zeros for the first step)."""
    if self._backward is None:
      raise RuntimeError("call input_grads_begin() first")
    single = tangent_planes.dim() == 2
    dirs = 1 if single else tangent_planes.shape[0]
    if weight_tangents is not None and dirs != 1:
      raise ValueError("parameter tangents run one direction")
    for name, t, rows in (("tangent_planes", tangent_planes, self.c_in),
                          ("tangent_out", tangent_out, self.n_out)):
      lead = () if single else (dirs,)
      if (tuple(t.shape) != lead + (rows, self.num_grid) or t.dtype != torch.float32
          or t.stride()[-2:] != (self.num_grid, 1) or t.device != self.device or dirs < 1):
        raise ValueError(f"{name} must be a float32 {list(lead + (rows, self.num_grid))} tensor on "
                         f"{self.device} with contiguous [{rows}, {self.num_grid}] planes per direction")
    planes = [tangent_planes] if single else list(tangent_planes.unbind(0))
    outs = [tangent_out] if single else list(tangent_out.unbind(0))
    grid_in = self.grid_in_img if grid_in is None else grid_in
    stride = self._backward.dir_stride(self.num_grid)
    add_index = affine.get("add_plane_index")
    with self._on_device():
      dgrid_in = self._pack_tangents(planes, in_scale, stride)
      dy = self._backward.tangent(grid_in, dgrid_in, dirs, wts=weight_tangents)
      del dgrid_in
      if planes_out is not None:
        self.unpack_outputs(planes_out, **affine)
      for k, (p, out) in enumerate(zip(planes, outs)):
        _native.check(self._lib.gcb_unpack_grid_outputs(
            dy[k * stride:].data_ptr(), dy.shape[1], self.n_out, self.num_grid,
            self._ptr(affine.get("scale")), None, None if add_index is None else p.data_ptr(),
            self._ptr(add_index), out.data_ptr(), self._stream()), "gcb_unpack_grid_outputs")

  # -- parameter tangents (param_jvp, loss_and_param_gnvp) ---------------------------------------------
  def weight_tangents(self, param_tangents: Mapping[str, Mapping[str, np.ndarray]],
                      transposed: bool = False, input_grad: bool = False):
    """Packs parameter tangents (host float32 arrays keyed and shaped like the params, modules and
    fields optional) into tangent weight images on the device (Backward.weight_tangents), for
    input_jvp_element, param_gnvp_element and (with `transposed`: also their transposed images,
    Backward.pack_transposed_tangents) param_hvp_element; with `input_grad` as well, the grid
    embedder's transposed image of the input gradient, for joint_hvp_element.  Call
    input_grads_begin() or grads_begin() first.  The engine's weights and weights_version are not
    touched."""
    if self._backward is None:
      raise RuntimeError("call input_grads_begin() or grads_begin() first")
    with self._on_device():
      dev = {name: {f: torch.as_tensor(np.ascontiguousarray(a, np.float32)).to(self.device)
                    for f, a in fields.items()} for name, fields in param_tangents.items()}
      wts = self._backward.weight_tangents(dev)
      if transposed:
        self._backward.pack_transposed_tangents(wts, input_grad=input_grad)
      return wts

  def param_gnvp_element(self, targets_planes: torch.Tensor, lat_weight: torch.Tensor,
                         coef: torch.Tensor, weight_tangents, *, channel_sums: torch.Tensor,
                         **affine) -> None:
    """One batch element of a Gauss-Newton product (call grads_begin() first): the step from the
    packed grid_in_img with its tangent along the packed parameter tangents (Backward.tangent(wts=...),
    zero input tangent), whose decoder tangent y-dot = J v seeds g = coef * lat_weight * y-dot
    (gcb_output_loss_gn_seed: the loss Hessian with respect to y is that diagonal).  The step then runs
    again stage by stage with the snapshots of loss_and_grads_element, whose loss sums go to
    channel_sums, and the backward pass from g ADDS this element's J^T H J v to the gradient
    accumulators.  Recomputing the step rather than keeping snapshots through the tangent keeps the
    peak that of the larger of the two passes."""
    if self._backward is None:
      raise RuntimeError("call grads_begin() first")
    grid_in = self.grid_in_img
    with self._on_device():
      dgrid_in = self._image(self.num_grid, self.c_in_pad)
      dy = self._backward.tangent(grid_in, dgrid_in, wts=weight_tangents)
      del dgrid_in
      g_out = torch.zeros([self.num_grid, 256], dtype=torch.float32, device=self.device)
      self._gn_seed(dy, lat_weight, coef, g_out)
      del dy
    # The tangent pass leaves its blocks cached in shapes the backward pass cannot reuse: at 0.25
    # degree the backward pass peaks within a few GiB of an 80 GB card and would not find its 1 GiB
    # tables in them.
    torch.cuda.empty_cache()
    snaps = self._forward_snapshots(grid_in)
    self.output_loss(targets_planes, lat_weight, channel_sums=channel_sums, **affine)
    with self._on_device():
      self._backward.element(grid_in, g_out, snaps)

  # -- parameter Hessian-vector products (loss_and_param_hvp) -----------------------------------------
  def param_hvp_begin(self) -> None:
    """grads_begin() for loss_and_param_hvp: zeroes the gradient accumulators and those of the
    Hessian-vector product (param_hvp)."""
    self.grads_begin()
    self._backward.zero_hvp()

  def param_hvp_element(self, targets_planes: torch.Tensor, lat_weight: torch.Tensor,
                        coef: torch.Tensor, weight_tangents, *, channel_sums: torch.Tensor,
                        **affine) -> None:
    """One batch element of a Hessian-vector product of the loss with respect to the parameters (call
    param_hvp_begin() first; weight_tangents from weight_tangents(..., transposed=True)).

    The step runs from the packed grid_in_img with its tangent along the parameter tangents v and a
    zero input tangent (Backward.tangent(wts=..., snaps=..., tsnaps=...)), keeping the primal and
    tangent snapshots; the loss sums of that forward go to channel_sums (output_loss).  The seed has
    two directions: direction 0 is loss_and_grads_element's (gcb_output_loss_grad), direction 1 its
    tangent.  Targets and the normalisation do not move with the parameters, so that tangent is
    coef * lat_weight * y-dot (gcb_output_loss_gn_seed).  One coupled backward walk
    (Backward.element(dirs=2, hvp=..., param_grads=True)) then ADDS this element's gradient to the
    gradient accumulators, bit for bit as loss_and_grads_element does, and its H v to those of
    param_hvp()."""
    if self._backward is None:
      raise RuntimeError("call param_hvp_begin() first")
    bw = self._backward
    grid_in = self.grid_in_img
    stride = bw.dir_stride(self.num_grid)
    with self._on_device():
      dgrid_in = self._image(self.num_grid, self.c_in_pad)
      snaps, tsnaps = {}, {}
      dy = bw.tangent(grid_in, dgrid_in, snaps=snaps, tsnaps=tsnaps, wts=weight_tangents)
      del dgrid_in
      self.output_loss(targets_planes, lat_weight, channel_sums=channel_sums, **affine)
      g_out = torch.zeros([stride + self.num_grid, 256], dtype=torch.float32, device=self.device)
      self._loss_seed(self.grid_out, targets_planes, lat_weight, coef, g_out, affine)
      self._gn_seed(dy, lat_weight, coef, g_out[stride:])
      del dy
      bw.element(grid_in, g_out, snaps, dirs=2, hvp=tsnaps, wts=weight_tangents)

  def param_hvp(self):
    """The accumulated Hessian-vector products of param_hvp_element (or the parameter side of
    joint_hvp_element's): device fp32 tensors keyed and shaped like the params, zeros for the
    parameters the step never reads."""
    return self._backward.grads(tangent=True)

  # -- joint Hessian-vector products (loss_and_joint_hvp) ----------------------------------------------
  def joint_hvp_element(self, fb: "Feedback", operands: dict, *, lat_weight: torch.Tensor,
                        coef: torch.Tensor, weight_tangents, channel_sums: torch.Tensor,
                        zero_targets: Optional[torch.Tensor] = None) -> None:
    """One batch element of a Hessian-vector product of the loss jointly in the parameters and the
    inputs (call param_hvp_begin() first, then build fb; weight_tangents from weight_tangents(...,
    transposed=True, input_grad=True)).  operands: "targets_planes", "tangent_planes" [c_in, Ng] (the
    input tangent v_x, physical units) and the affine keywords of output_loss.  Afterwards fb.a is
    [2, fb.n_rows, Ng]: direction 0 the gradient with respect to the input planes, direction 1 its
    derivative along (v_theta, v_x); the parameter gradients and their derivatives are ADDED to the
    accumulators of grads() and param_hvp().  zero_targets as in input_hvp_element.

    The step runs from the packed grid_in_img with its tangent along the parameter tangents and v_x,
    packed as input_hvp_element packs it (Backward.tangent(wts=..., snaps=..., tsnaps=...)); the loss
    sums of that forward go to channel_sums.  Direction 0 of the seed is input_grads_element's loss
    seed with no following step.  The seed is affine in (y, the add planes, fb.a) and the parameters
    reach it only through y, so direction 1 is the same kernel on y-dot, add_planes = v_x, zero targets
    and no offset, as input_hvp_element seeds its tangent.  One coupled walk
    (Backward.element(dirs=2, hvp=..., param_grads=True, dgrid_in=True)) then forms both sides, and
    gcb_input_grad runs per direction.  The loss sums, the parameter gradients and direction 0 are bit
    for bit those of loss_and_grads_element and input_grads_element."""
    if self._backward is None:
      raise RuntimeError("call param_hvp_begin() first")
    bw = self._backward
    affine = {k: operands[k] for k in ("scale", "offset", "add_planes", "add_plane_index")
              if k in operands}
    targets_planes, tangent = operands["targets_planes"], operands["tangent_planes"]
    operands.clear()
    if (tuple(tangent.shape) != (self.c_in, self.num_grid) or tangent.dtype != torch.float32
        or not tangent.is_contiguous()):
      raise ValueError(f"tangent_planes must be a contiguous float32 [{self.c_in}, {self.num_grid}] "
                       "tensor")
    grid_in = self.grid_in_img
    stride = bw.dir_stride(self.num_grid)
    add_index = affine.get("add_plane_index")
    with self._on_device():
      dgrid_in = self._pack_tangents([tangent], fb.in_scale, stride)
      snaps, tsnaps = {}, {}
      dy = bw.tangent(grid_in, dgrid_in, snaps=snaps, tsnaps=tsnaps, wts=weight_tangents)
      del dgrid_in
      self.output_loss(targets_planes, lat_weight, channel_sums=channel_sums, **affine)
      g_out = torch.zeros([stride + self.num_grid, 256], dtype=torch.float32, device=self.device)
      a_out = torch.empty([2, fb.n_rows, self.num_grid], dtype=torch.float32, device=self.device)
      if zero_targets is None:
        zero_targets = torch.zeros([self.n_out, self.num_grid], dtype=torch.float32,
                                   device=self.device)
      self._loss_seed(self.grid_out, targets_planes, lat_weight, coef, g_out, affine, fb=fb,
                      a_out=a_out[0], n_rows=fb.n_rows)
      self._loss_seed(dy, zero_targets, lat_weight, coef, g_out[stride:],
                      dict(scale=affine.get("scale"), add_plane_index=add_index,
                           add_planes=None if add_index is None else tangent),
                      fb=fb, a_out=a_out[1], n_rows=fb.n_rows)
      # the planes, targets and tangents are consumed: release them
      fb.a = a_out
      del dy, zero_targets
      affine = targets_planes = tangent = None
      dx = bw.element(grid_in, g_out, snaps, dgrid_in=True, dirs=2, hvp=tsnaps, wts=weight_tangents)
      del g_out, snaps, tsnaps
      self._input_grad_tail(dx, fb, a_out.unbind(0), stride)

  def broadcast_grad_sum(self, a: torch.Tensor, n_lat: int, rows: torch.Tensor, mode: int,
                         out: torch.Tensor, accumulate: bool) -> None:
    """gcb_broadcast_grad_sum on the current stream: the planes a[rows] ([*, Ng] fp32) reduced into
    `out` ([len(rows), Ng | n_lon | 1]) over the axes of `mode` (_native.BCAST_*)."""
    n_lon = self.num_grid // n_lat
    width = (self.num_grid, n_lon, 1)[mode]
    if out.numel() != rows.numel() * width or not out.is_contiguous() or out.dtype != torch.float32:
      raise ValueError(f"out must be a contiguous float32 tensor of {rows.numel() * width} elements")
    with self._on_device():
      _native.check(self._lib.gcb_broadcast_grad_sum(
          a.data_ptr(), n_lat, n_lon, rows.numel(), rows.data_ptr(), mode, out.data_ptr(),
          1 if accumulate else 0, self._stream()), "gcb_broadcast_grad_sum")

  def grads(self):
    """The accumulated gradients: device fp32 tensors keyed and shaped like the params."""
    return self._backward.grads()

  def grads_into(self, out: Mapping[str, Mapping[str, torch.Tensor]]) -> None:
    """The accumulated gradients copied into `out`, device tensors keyed and shaped like the params
    (e.g. views into an optimiser's flat buffer): the valid slices of the accumulators, no copy in
    between; zeros for the parameters the step never reads."""
    with self._on_device():
      self._backward.grads_into(out)

  def feedback(self, plan, add_plane_index=None, in_scale: Optional[torch.Tensor] = None) -> "Feedback":
    """Backprop-through-time state of one batch element for a feedback.FeedbackPlan (host) of this
    engine's channels; add_plane_index / in_scale as in FusedNormalization (None: no normalisation).
    Packs the transposed grid-embedder weight of the input gradient."""
    if plan.c_in != self.c_in or plan.n_out != self.n_out:
      raise ValueError(f"feedback plan of {plan.c_in} -> {plan.n_out} channels, engine "
                       f"{self.c_in} -> {self.n_out}")
    if self._backward is None:
      raise RuntimeError("call grads_begin() or input_grads_begin() first")
    with self._on_device():
      self._backward.input_transposed()
    if add_plane_index is not None and isinstance(add_plane_index, torch.Tensor):
      add_plane_index = add_plane_index.cpu().numpy()
    i32 = lambda a: torch.as_tensor(np.ascontiguousarray(a, np.int32)).to(self.device)
    return Feedback(i32(plan.rows), i32(plan.dpred_row), i32(plan.resid_channel(add_plane_index)),
                    i32(plan.carry_row), in_scale)

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


class Feedback:
  """Backprop through time of one batch element (Engine.loss_and_grads_element(feedback=...)): the
  device copies of a feedback.FeedbackPlan's row maps and `a`, dL/d(input planes) [n_rows, Ng] of the
  step after the one being differentiated (None before the last step)."""

  def __init__(self, rows: torch.Tensor, dpred_row: torch.Tensor, resid_channel: torch.Tensor,
               carry_row: torch.Tensor, in_scale: Optional[torch.Tensor]):
    self.rows, self.dpred_row = rows, dpred_row
    self.resid_channel, self.carry_row = resid_channel, carry_row
    self.in_scale = in_scale
    self.n_rows = int(rows.shape[0])
    self.a: Optional[torch.Tensor] = None
