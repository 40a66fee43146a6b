"""Oracle: GraphCast encode-process-decode forward on the CPU (torch-CPU tensors).

TEST INFRASTRUCTURE -- see oracle/__init__.py.  Pinned against the reference's own wiring,
executed on numpy stand-ins for jax / jraph / haiku (tests/test_reference_gnn_golden.py,
tests/test_reference_gnn_latent512.py: 5.5e-7); the third-party primitives listed below are
restatements of their published definitions (the packages cannot be installed here).

Restates, for explicit index arrays and a Haiku-named parameter dict:
  * hk.nets.MLP + hk.LayerNorm + jraph.concatenated_args as wired by
    `build_mlp_with_maybe_layer_norm`  (utils/legacy/deep_typed_graph_net.py:205-247)
  * GraphMapFeatures embedders / decoder (utils/typed_graph_net.py:657-696,
    deep_typed_graph_net.py:250-271, 314-322)
  * InteractionNetwork step: gather senders/receivers, edge fn on
    concat[edge, sender, receiver] (typed_graph_net.py:369-484, 637-638),
    segment_sum over receivers and node fn on concat[node, agg]
    (typed_graph_net.py:487-546, 646-647), node and edge residuals
    (deep_typed_graph_net.py:372-393)
  * the three GNN calls and their glue (weathernext1_graph/graphcast.py:550-678).

Third-party arithmetic restated from its published definition (packages are not
in the reference; versions unpinned in its setup.py:37,43):
  hk.Linear      y = x @ w + b, w:[in,out]
  hk.nets.MLP    activation between layers, none after the last
  hk.LayerNorm   axis=-1, eps=1e-5: (x-mean)*rsqrt(var_biased+eps)*scale+offset
  jax.nn.swish   x*sigmoid(x)
  jraph.segment_sum  sum of rows per segment id
"""

from __future__ import annotations

from typing import Dict, Mapping, Optional

import numpy as np
import torch

Params = Dict[str, Dict[str, np.ndarray]]


def mlp_name(gnn: str, prefix: str, set_name: str) -> str:
  """Haiku module path stem (deep_typed_graph_net.py:205-208,251-262,295-307,
  315-319; gnn names graphcast.py:217,233,261)."""
  return f"{gnn}/~_networks_builder/{prefix}{set_name}"


def swish(x: torch.Tensor) -> torch.Tensor:
  return x * torch.sigmoid(x)


def layer_norm(x, scale, offset, eps: float = 1e-5):
  mean = x.mean(dim=-1, keepdim=True)
  var = ((x - mean) ** 2).mean(dim=-1, keepdim=True)       # biased
  return (x - mean) * torch.rsqrt(var + eps) * scale + offset


class Oracle:
  """Holds params as torch-CPU tensors of one dtype and runs the forward."""

  def __init__(self, params: Params, dtype=torch.float32):
    self.dtype = dtype
    self.p = {k: {n: torch.as_tensor(np.asarray(a)).to(dtype) for n, a in v.items()}
              for k, v in params.items()}

  def matmul(self, x, w):
    """x @ w.  Hook so tests can emulate reduced-precision tensor-core products."""
    return x @ w

  # Further hooks (identity arithmetic here) so that a subclass can place roundings where a
  # reduced-precision execution of the reference has them (ReferenceBf16Oracle below).
  def bias_add(self, x, b):
    return x + b

  def activation(self, x):
    return swish(x)

  def normalize(self, x, scale, offset):
    return layer_norm(x, scale, offset)

  def add(self, a, b):
    """Residual connections (deep_typed_graph_net.py:372-393, graphcast.py:596-604,668-672)."""
    return a + b

  def aggregate(self, gnn: str, data, segment_ids, num_segments):
    """jraph.segment_sum of the edge messages of GNN `gnn` (typed_graph_net.py:532-538)."""
    return self.segment_sum(data, segment_ids, num_segments)

  # hk.nets.MLP (+ optional hk.LayerNorm) on the concatenation of `args`.
  def mlp(self, stem: str, args, use_layer_norm: bool = True):
    x = torch.cat(list(args), dim=-1)
    i = 0
    while f"{stem}_mlp/~/linear_{i}" in self.p:
      lin = self.p[f"{stem}_mlp/~/linear_{i}"]
      if i > 0:
        x = self.activation(x)
      x = self.bias_add(self.matmul(x, lin["w"]), lin["b"])
      i += 1
    if use_layer_norm:
      ln = self.p[f"{stem}_layer_norm"]
      x = self.normalize(x, ln["scale"], ln["offset"])
    return x

  @staticmethod
  def segment_sum(data, segment_ids, num_segments):
    out = torch.zeros((num_segments,) + tuple(data.shape[1:]), dtype=data.dtype)
    out.index_add_(0, segment_ids, data)
    return out

  # The three GNN calls of GraphCast.__call__ as separate stages (graphcast.py:309-323), so that
  # the 0.25 degree parity tests can check the CUDA path stage by stage (SURVEY section 8d).
  def _t(self, a):
    return torch.as_tensor(np.asarray(a)).to(self.dtype)

  @staticmethod
  def _idx(a):
    return torch.as_tensor(np.asarray(a)).to(torch.int64)

  def encoder(self, graph: Mapping[str, np.ndarray], grid_features, inter: Optional[dict] = None):
    """grid2mesh_gnn (graphcast.py:550-604): [Ng,B,C_in] -> (vm1 [Nm,B,D], vg1 [Ng,B,D])."""
    X = self._t(grid_features)
    n_grid, batch, _ = X.shape
    bcast = lambda f: self._t(f)[:, None, :].expand(-1, batch, -1)   # _add_batch_second_axis :726-730
    sg, sm = bcast(graph["grid_node_feats"]), bcast(graph["mesh_node_feats"])
    n_mesh = sm.shape[0]
    grid_in = torch.cat([X, sg], dim=-1)
    mesh_in = torch.cat([torch.zeros((n_mesh,) + tuple(X.shape[1:]), dtype=self.dtype), sm],
                        dim=-1)                                 # :573-583
    g = "grid2mesh_gnn"
    vg0 = self.mlp(mlp_name(g, "encoder_nodes_", "grid_nodes"), [grid_in])
    vm0 = self.mlp(mlp_name(g, "encoder_nodes_", "mesh_nodes"), [mesh_in])
    e1 = self.mlp(mlp_name(g, "encoder_edges_", "grid2mesh"), [bcast(graph["g2m_edge_feats"])])
    s1, r1 = self._idx(graph["g2m_senders"]), self._idx(graph["g2m_receivers"])
    m1 = self.mlp(mlp_name(g, "processor_edges_0_", "grid2mesh"), [e1, vg0[s1], vm0[r1]])
    agg1 = self.aggregate(g, m1, r1, n_mesh)       # f32_aggregation is a no-op in f32
    vm1 = self.add(vm0, self.mlp(mlp_name(g, "processor_nodes_0_", "mesh_nodes"), [vm0, agg1]))
    vg1 = self.add(vg0, self.mlp(mlp_name(g, "processor_nodes_0_", "grid_nodes"), [vg0]))
    if inter is not None:
      inter.update(vg0=vg0, vm0=vm0, e1=e1, m1=m1, agg1=agg1, vm1=vm1, vg1=vg1)
    return vm1, vg1

  def processor_embed(self, graph: Mapping[str, np.ndarray], batch: int = 1):
    """Embedded multi-mesh edge latents (the mesh GNN's `_embed`, deep_typed_graph_net.py:250-271)."""
    bcast = lambda f: self._t(f)[:, None, :].expand(-1, batch, -1)
    return self.mlp(mlp_name("mesh_gnn", "encoder_edges_", "mesh"), [bcast(graph["mesh_edge_feats"])])

  def processor_step(self, graph: Mapping[str, np.ndarray], v, e, k: int):
    """One InteractionNetwork step with node and edge residuals (deep_typed_graph_net.py:372-393):
    returns (v_new, e_new)."""
    g = "mesh_gnn"
    s2, r2 = self._idx(graph["mesh_senders"]), self._idx(graph["mesh_receivers"])
    m = self.mlp(mlp_name(g, f"processor_edges_{k}_", "mesh"), [e, v[s2], v[r2]])
    agg = self.aggregate(g, m, r2, v.shape[0])
    v_new = self.add(v, self.mlp(mlp_name(g, f"processor_nodes_{k}_", "mesh_nodes"), [v, agg]))
    return v_new, self.add(e, m)

  def num_message_steps(self) -> int:
    k = 0
    while mlp_name("mesh_gnn", f"processor_edges_{k}_", "mesh") + "_mlp/~/linear_0" in self.p:
      k += 1
    return k

  def processor(self, graph: Mapping[str, np.ndarray], vm1, inter: Optional[dict] = None):
    """mesh_gnn (graphcast.py:606-639): all message-passing steps on the multi-mesh."""
    v = self._t(vm1)
    e = self.processor_embed(graph, v.shape[1])
    for k in range(self.num_message_steps()):
      v, e = self.processor_step(graph, v, e, k)
    if inter is not None:
      inter.update(v_mesh=v, e_mesh=e)
    return v

  def decoder(self, graph: Mapping[str, np.ndarray], v_mesh, vg1, inter: Optional[dict] = None):
    """mesh2grid_gnn + output MLP (graphcast.py:641-678) -> [Ng,B,n_out]."""
    v, vg1 = self._t(v_mesh), self._t(vg1)
    n_grid, batch = vg1.shape[0], vg1.shape[1]
    bcast = lambda f: self._t(f)[:, None, :].expand(-1, batch, -1)
    g = "mesh2grid_gnn"
    e3 = self.mlp(mlp_name(g, "encoder_edges_", "mesh2grid"), [bcast(graph["m2g_edge_feats"])])
    s3, r3 = self._idx(graph["m2g_senders"]), self._idx(graph["m2g_receivers"])
    m3 = self.mlp(mlp_name(g, "processor_edges_0_", "mesh2grid"), [e3, v[s3], vg1[r3]])
    agg3 = self.aggregate(g, m3, r3, n_grid)
    vg2 = self.add(vg1, self.mlp(mlp_name(g, "processor_nodes_0_", "grid_nodes"), [vg1, agg3]))
    out = self.mlp(mlp_name(g, "decoder_nodes_", "grid_nodes"), [vg2], use_layer_norm=False)
    if inter is not None:
      inter.update(vg2=vg2)
    return out

  def forward(self, graph: Mapping[str, np.ndarray], grid_features: np.ndarray,
              return_intermediates: bool = False):
    """One step.  grid_features [Ng, B, C_in] (already normalised + packed).

    graph keys: grid_node_feats [Ng,3], mesh_node_feats [Nm,3],
      g2m_senders/g2m_receivers [E1], g2m_edge_feats [E1,4],
      mesh_senders/mesh_receivers [E2], mesh_edge_feats [E2,4],
      m2g_senders/m2g_receivers [E3], m2g_edge_feats [E3,4].
    Returns [Ng, B, n_out].
    """
    inter = {} if return_intermediates else None
    vm1, vg1 = self.encoder(graph, grid_features, inter)
    v = self.processor(graph, vm1, inter)
    out = self.decoder(graph, v, vg1, inter)
    if return_intermediates:
      return out, inter
    return out


class Bf16OperandOracle(Oracle):
  """The product's "bf16" mode, emulated: every contraction takes its two operands rounded to
  bfloat16 (round-to-nearest-even) and accumulates in this oracle's dtype; everything else
  (bias, swish, LayerNorm, residuals, aggregation) stays in that dtype.  This is what
  `precision="bf16"` / `casting.Bfloat16Cast` computes on the device (one tensor-core product per MAC,
  fp32 accumulation, latents as 2 x bf16) -- NOT the reference's all-bf16 execution, where XLA also
  rounds every activation, the LayerNorm and (outside grid2mesh) the aggregation to bf16
  (utils/casting.py:31-65, graphcast.py:215,232,260); see graphcast_b200/casting.py."""

  def matmul(self, x, w):
    r = lambda t: t.to(torch.float32).to(torch.bfloat16).to(self.dtype)
    return r(x) @ r(w)


class ReferenceBf16Oracle(Oracle):
  """The reference's OWN bf16 execution, emulated op by op (what `casting.Bfloat16Cast` makes of the
  model): inputs and parameters are bfloat16 (utils/casting.py:53-58 with `_all_inputs_to_bfloat16`
  :135-145 and `bfloat16_variable_view` :156-205), so every jnp op returns a bfloat16 array -- the linear layers
  (fp32 accumulation inside the dot, result rounded), bias adds, `jax.nn.swish` (sigmoid, then the
  product), `hk.LayerNorm` (mean, variance, rsqrt, scale, shift: each a bf16 result), the residual adds
  and the segment sums; only grid2mesh aggregates in fp32 (`f32_aggregation`, graphcast.py:215,232,260
  with utils/legacy/deep_typed_graph_net.py:273-288) before rounding the sum.  Every rounding is round-to-nearest-even of
  a value computed in fp32 from bf16 operands, i.e. the semantics of the individual XLA ops; a fused
  XLA executable may keep some intermediates wider, and a bf16 scatter-add may round after every
  addend, so this is one admissible execution, not a bit-level model of any backend.

  Used to place the product's "bf16" mode (Bf16OperandOracle: bf16 operands, everything else fp32)
  against what the reference computes under `Bfloat16Cast` (tests/test_oracle.py)."""

  F32_AGGREGATION = ("grid2mesh_gnn",)

  def __init__(self, params: Params):
    super().__init__(params, torch.float32)
    self.p = {k: {n: self._r(a) for n, a in v.items()} for k, v in self.p.items()}

  @staticmethod
  def _r(t):
    return t.to(torch.bfloat16).to(torch.float32)

  def _t(self, a):
    return self._r(super()._t(a))

  def matmul(self, x, w):
    return self._r(x @ w)

  def bias_add(self, x, b):
    return self._r(x + b)

  def activation(self, x):
    return self._r(x * self._r(torch.sigmoid(x)))

  def normalize(self, x, scale, offset, eps: float = 1e-5):
    r = self._r
    mean = r(x.mean(dim=-1, keepdim=True))
    var = r(((x - x.mean(dim=-1, keepdim=True)) ** 2).mean(dim=-1, keepdim=True))   # jnp.var: fp32 inside
    inv = r(scale * r(torch.rsqrt(r(var + eps))))
    return r(r(inv * r(x - mean)) + offset)

  def add(self, a, b):
    return self._r(a + b)

  def aggregate(self, gnn, data, segment_ids, num_segments):
    # fp32 accumulation either way here (optimistic for the GNNs without f32_aggregation)
    return self._r(self.segment_sum(data, segment_ids, num_segments))


def truncated_normal(rng: np.random.Generator, shape, stddev: float) -> np.ndarray:
  """hk.initializers.TruncatedNormal: N(0,1) truncated to [-2,2], times stddev."""
  x = rng.standard_normal(shape)
  bad = np.abs(x) > 2.0
  while bad.any():
    x[bad] = rng.standard_normal(int(bad.sum()))
    bad = np.abs(x) > 2.0
  return (x * stddev).astype(np.float32)


def init_params(*, c_in: int, n_out: int, latent: int = 512, msg_steps: int = 16,
                hidden_layers: int = 1, seed: int = 1, randomize_affine: bool = False
                ) -> Params:
  """Haiku-default initialisation of every GraphCast parameter (SURVEY App. B):
  w ~ TruncNormal(1/sqrt(fan_in)), b = 0, LN scale = 1, offset = 0.
  `randomize_affine` perturbs b / scale / offset so tests exercise those terms.
  Shapes follow deep_typed_graph_net.py:205-322 with the concat orders of
  typed_graph_net.py:637-647."""
  rng = np.random.default_rng(seed)
  params: Params = {}

  def add_mlp(gnn, prefix, set_name, d_in, d_out, layer_norm=True):
    stem = mlp_name(gnn, prefix, set_name)
    sizes = [latent] * hidden_layers + [d_out]
    fan_in = d_in
    for i, size in enumerate(sizes):
      w = truncated_normal(rng, (fan_in, size), 1.0 / np.sqrt(fan_in))
      b = np.zeros([size], np.float32)
      if randomize_affine:
        b = (0.1 * rng.standard_normal(size)).astype(np.float32)
      params[f"{stem}_mlp/~/linear_{i}"] = {"w": w, "b": b}
      fan_in = size
    if layer_norm:
      scale = np.ones([d_out], np.float32)
      offset = np.zeros([d_out], np.float32)
      if randomize_affine:
        scale = (1.0 + 0.1 * rng.standard_normal(d_out)).astype(np.float32)
        offset = (0.1 * rng.standard_normal(d_out)).astype(np.float32)
      params[f"{stem}_layer_norm"] = {"scale": scale, "offset": offset}

  D = latent
  g = "grid2mesh_gnn"
  add_mlp(g, "encoder_nodes_", "grid_nodes", c_in + 3, D)
  add_mlp(g, "encoder_nodes_", "mesh_nodes", c_in + 3, D)
  add_mlp(g, "encoder_edges_", "grid2mesh", 4, D)
  add_mlp(g, "processor_edges_0_", "grid2mesh", 3 * D, D)
  add_mlp(g, "processor_nodes_0_", "grid_nodes", D, D)
  add_mlp(g, "processor_nodes_0_", "mesh_nodes", 2 * D, D)
  g = "mesh_gnn"
  add_mlp(g, "encoder_edges_", "mesh", 4, D)
  for k in range(msg_steps):
    add_mlp(g, f"processor_edges_{k}_", "mesh", 3 * D, D)
    add_mlp(g, f"processor_nodes_{k}_", "mesh_nodes", 2 * D, D)
  g = "mesh2grid_gnn"
  add_mlp(g, "encoder_edges_", "mesh2grid", 4, D)
  add_mlp(g, "processor_edges_0_", "mesh2grid", 3 * D, D)
  add_mlp(g, "processor_nodes_0_", "grid_nodes", 2 * D, D)
  add_mlp(g, "processor_nodes_0_", "mesh_nodes", D, D)       # traced but dead
  add_mlp(g, "decoder_nodes_", "grid_nodes", D, n_out, layer_norm=False)
  return params
