"""One forecast step spread over the GPUs of a box by MESH NODE (BASELINE config 4).

The reference has no spatially sharded GraphCast; its newer models shard gathers / segment sums
with an `all_gather` in front of every gather and a `psum_scatter` behind every segment sum
(utils/gather_scatter_ops.py:278,423), dropping both when all indices are shard-local (:102-144).
Here the rule "an edge lives on the rank that owns its RECEIVER" makes every aggregation
(`_node_update`, utils/typed_graph_net.py:532-538) rank-local, so the only collective left is, once
per message-passing step, the exchange of the latents of the HALO mesh nodes (remote senders of
owned edges): one grouped NCCL all-to-all-v of <= 1 MB per rank (SURVEY.md section 8e).

Ownership
  mesh node   recursive coordinate bisection of the vertices (partition.py)
  grid node   the owner of the first vertex of its containing mesh triangle (its mesh2grid senders)
  edge        the owner of its receiver (all three graphs)
Local tables of rank r
  mesh  [owned | padding to a multiple of 128 | halo]   halo = remote senders of owned multi-mesh
        and mesh2grid edges, grouped by owner: a peer's rows arrive contiguously -- as rows of the
        operand image (default: image-only latents, gcb_image_rows_pack / _unpack) or, with fp32
        masters, straight into the fp32 table; the 128-row alignment gives the halo its own tiles
        of the operand image
  grid  [owned | halo]    halo = remote senders of owned grid2mesh edges; their encoder latents are
        recomputed locally from the raw inputs (a per-node MLP) instead of being exchanged
A rank's local arrays form an ordinary `StaticGraph` (local numbering) for `engine.Engine`, which
restricts node updates / aggregation / the decoder to the owned rows (gcb_model.num_*_owned).

`build_local_graph` is pure numpy (CPU-tested against the oracle in tests/test_partitioned_host.py);
`PartitionedEngine` drives the stage-wise C ABI and `torch.distributed` (NCCL).
"""

from __future__ import annotations

import dataclasses
from typing import Dict, List, Optional

import numpy as np

from graphcast_b200 import graph as graph_lib
from graphcast_b200 import partition

TILE = 128


@dataclasses.dataclass
class LocalGraph:
  rank: int
  num_parts: int
  graph: graph_lib.StaticGraph          # local numbering
  grid_owned: np.ndarray                # [ng_own] global grid ids (ascending)
  grid_halo: np.ndarray                 # [ng_halo] global grid ids
  mesh_owned: np.ndarray                # [nm_own] global mesh ids (ascending)
  mesh_halo: np.ndarray                 # [nm_halo] global mesh ids, grouped by owner
  mesh_owned_pad: int                   # first local row of the halo part (multiple of 128)
  send_rows: np.ndarray                 # [n_send] local owned rows to send, grouped by peer
  send_counts: List[int]                # per rank
  recv_counts: List[int]                # per rank (sum = nm_halo)

  @property
  def local_grid_ids(self) -> np.ndarray:
    return np.concatenate([self.grid_owned, self.grid_halo])


def mesh_xyz(g: graph_lib.StaticGraph) -> np.ndarray:
  """Unit vectors of the mesh nodes from their structural features [sin lat, cos lon, sin lon]."""
  f = g.mesh_node_feats.astype(np.float64)
  cos_lat = np.sqrt(np.maximum(0.0, 1.0 - f[:, 0] ** 2))
  return np.stack([cos_lat * f[:, 1], cos_lat * f[:, 2], f[:, 0]], axis=1)


def ownership(g: graph_lib.StaticGraph, num_parts: int):
  """(mesh node -> rank, grid node -> rank)."""
  mesh_part = partition.recursive_coordinate_bisection(mesh_xyz(g), num_parts)
  if not np.array_equal(g.m2g_receivers, np.repeat(np.arange(g.num_grid_nodes), 3)):
    raise ValueError("mesh2grid edges must be grouped by grid node with fan-in 3")
  grid_part = mesh_part[g.m2g_senders[0::3]]
  return mesh_part, grid_part


def _mesh_halo(g, mesh_part, grid_part, r):
  """Remote mesh senders rank r needs: of its multi-mesh edges and of its mesh2grid edges."""
  em = mesh_part[g.mesh_receivers] == r
  ed = grid_part[g.m2g_receivers] == r
  snd = np.concatenate([g.mesh_senders[em], g.m2g_senders[ed]])
  remote = np.unique(snd[mesh_part[snd] != r])
  order = np.lexsort((remote, mesh_part[remote]))          # grouped by owner, ascending id inside
  return remote[order]


def build_local_graph(g: graph_lib.StaticGraph, num_parts: int, rank: int) -> LocalGraph:
  mesh_part, grid_part = ownership(g, num_parts)
  mesh_owned = np.flatnonzero(mesh_part == rank)
  grid_owned = np.flatnonzero(grid_part == rank)
  mesh_halo = _mesh_halo(g, mesh_part, grid_part, rank)
  owned_pad = (mesh_owned.size + TILE - 1) // TILE * TILE
  # edges owned by this rank (receiver rule), in their global relative order
  e1 = np.flatnonzero(mesh_part[g.g2m_receivers] == rank)
  e2 = np.flatnonzero(mesh_part[g.mesh_receivers] == rank)
  e3 = np.flatnonzero(grid_part[g.m2g_receivers] == rank)
  g2m_snd = g.g2m_senders[e1]
  grid_halo = np.unique(g2m_snd[grid_part[g2m_snd] != rank])
  # global -> local
  mesh_local = np.full(g.num_mesh_nodes, -1, np.int64)
  mesh_local[mesh_owned] = np.arange(mesh_owned.size)
  mesh_local[mesh_halo] = owned_pad + np.arange(mesh_halo.size)
  grid_local = np.full(g.num_grid_nodes, -1, np.int64)
  grid_local[grid_owned] = np.arange(grid_owned.size)
  grid_local[grid_halo] = grid_owned.size + np.arange(grid_halo.size)
  n_mesh_local = owned_pad + mesh_halo.size
  mesh_feats = np.zeros([n_mesh_local, 3], np.float32)
  mesh_feats[:mesh_owned.size] = g.mesh_node_feats[mesh_owned]
  mesh_feats[owned_pad:] = g.mesh_node_feats[mesh_halo]
  grid_ids = np.concatenate([grid_owned, grid_halo])
  i32 = lambda a: np.ascontiguousarray(a, np.int32)
  local = graph_lib.StaticGraph(
      num_grid_nodes=int(grid_ids.size), num_mesh_nodes=int(n_mesh_local),
      grid_lat=g.grid_lat, grid_lon=g.grid_lon,
      grid_node_feats=np.ascontiguousarray(g.grid_node_feats[grid_ids]), mesh_node_feats=mesh_feats,
      g2m_senders=i32(grid_local[g2m_snd]), g2m_receivers=i32(mesh_local[g.g2m_receivers[e1]]),
      g2m_edge_feats=np.ascontiguousarray(g.g2m_edge_feats[e1]),
      mesh_senders=i32(mesh_local[g.mesh_senders[e2]]), mesh_receivers=i32(mesh_local[g.mesh_receivers[e2]]),
      mesh_edge_feats=np.ascontiguousarray(g.mesh_edge_feats[e2]),
      m2g_senders=i32(mesh_local[g.m2g_senders[e3]]), m2g_receivers=i32(grid_local[g.m2g_receivers[e3]]),
      m2g_edge_feats=np.ascontiguousarray(g.m2g_edge_feats[e3]))
  for a in (local.g2m_senders, local.g2m_receivers, local.mesh_senders, local.mesh_receivers,
            local.m2g_senders, local.m2g_receivers):
    assert a.size == 0 or a.min() >= 0
  # halo exchange: what I receive (my halo, grouped by owner) and what every peer needs from me
  recv_counts = [int(np.count_nonzero(mesh_part[mesh_halo] == p)) for p in range(num_parts)]
  send_rows, send_counts = [], []
  for p in range(num_parts):
    if p == rank:
      send_counts.append(0)
      continue
    theirs = _mesh_halo(g, mesh_part, grid_part, p)
    mine = theirs[mesh_part[theirs] == rank]               # in THEIR halo order
    send_rows.append(mesh_local[mine])
    send_counts.append(int(mine.size))
  send_rows = np.concatenate(send_rows) if send_rows else np.zeros([0], np.int64)
  return LocalGraph(rank=rank, num_parts=num_parts, graph=local, grid_owned=grid_owned,
                    grid_halo=grid_halo, mesh_owned=mesh_owned, mesh_halo=mesh_halo,
                    mesh_owned_pad=int(owned_pad), send_rows=i32(send_rows),
                    send_counts=send_counts, recv_counts=recv_counts)


def plan_statistics(g: graph_lib.StaticGraph, num_parts: int) -> Dict[str, List[int]]:
  lgs = [build_local_graph(g, num_parts, r) for r in range(num_parts)]
  return {
      "grid_owned": [int(l.grid_owned.size) for l in lgs], "grid_halo": [int(l.grid_halo.size) for l in lgs],
      "mesh_owned": [int(l.mesh_owned.size) for l in lgs], "mesh_halo": [int(l.mesh_halo.size) for l in lgs],
      "g2m_edges": [int(l.graph.g2m_senders.size) for l in lgs],
      "mesh_edges": [int(l.graph.mesh_senders.size) for l in lgs],
      "m2g_edges": [int(l.graph.m2g_senders.size) for l in lgs],
      "halo_bytes_per_step": [int(l.mesh_halo.size) * 512 * 4 for l in lgs],
      "peers": [int(sum(1 for c in l.recv_counts if c)) for l in lgs],
  }


class PartitionedEngine:
  """One rank's share of one forecast: a local `Engine` + the per-step halo exchange."""

  def __init__(self, g: graph_lib.StaticGraph, params, *, c_in: int, n_out: int, msg_steps: int,
               rank: int, world: int, device, precision: str = "bf16x3", group=None,
               image_residual: bool = True):
    import torch
    from graphcast_b200 import _native, engine
    self.local = build_local_graph(g, world, rank)
    self.rank, self.world, self.group = rank, world, group
    lg = self.local
    # The halo rows travel as 2048-byte rows: fp32 rows gathered from the fp32 master, or -- image-only
    # latents (default) -- the rows of the operand image themselves (bf16 hi + lo pieces), which the
    # receiver stores into its own image unchanged.
    self.image_residual = bool(image_residual)
    self.engine = engine.Engine(lg.graph, params, c_in=c_in, n_out=n_out, msg_steps=msg_steps,
                                precision=precision, device=device, image_residual=self.image_residual,
                                deep_chains=False, num_grid_owned=int(lg.grid_owned.size),
                                num_mesh_owned=int(lg.mesh_owned.size))
    eng = self.engine
    self._lib = _native.lib()
    self._native = _native
    self._torch = torch
    self.send_rows = torch.as_tensor(lg.send_rows, dtype=torch.int32, device=eng.device)
    self.n_send, self.n_halo = int(lg.send_rows.size), int(lg.mesh_halo.size)
    self.send_buf = torch.empty([max(self.n_send, 1), 512], dtype=torch.float32, device=eng.device)
    if self.image_residual:
      self.halo_view = torch.empty([max(self.n_halo, 1), 512], dtype=torch.float32,
                                   device=eng.device)[:self.n_halo]
    else:
      self.halo_view = eng.mesh_lat[lg.mesh_owned_pad:lg.mesh_owned_pad + self.n_halo]
    self.skip_exchange = False      # measurement aid (bench.py): time a step without exchanges
    self._events = []

  def output_loss(self, *args, **kwargs):
    """Not provided: a rank holds only its own grid rows, and the loss is a mean over all of them."""
    raise NotImplementedError("the loss is not available in the node-partitioned engine; "
                              "evaluate it with a single-GPU GraphCast")

  def exchange_halo(self, timed: bool = False) -> None:
    """Owned boundary rows of mesh_lat -> the halo rows of the peers that need them; then the
    halo part of the operand image is rebuilt."""
    if self.world == 1 or self.skip_exchange:
      return
    import torch.distributed as dist
    torch, eng, lg = self._torch, self.engine, self.local
    ev = None
    if timed:
      ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
      ev[0].record()
    with eng._on_device():
      if self.image_residual:
        self._native.check(self._lib.gcb_image_rows_pack(
            eng.mesh_lat_img.data_ptr(), self.send_rows.data_ptr(), self.n_send,
            self.send_buf.data_ptr(), eng._stream()), "gcb_image_rows_pack")
      else:
        self._native.check(self._lib.gcb_gather_rows(
            eng.mesh_lat.data_ptr(), 512, self.send_rows.data_ptr(), self.n_send,
            self.send_buf.data_ptr(), 512, 512, eng._stream()), "gcb_gather_rows")
    dist.all_to_all_single(self.halo_view, self.send_buf[:self.n_send],
                           output_split_sizes=lg.recv_counts, input_split_sizes=lg.send_counts,
                           group=self.group)
    if self.n_halo:
      with eng._on_device():
        if self.image_residual:
          self._native.check(self._lib.gcb_image_rows_unpack(
              self.halo_view.data_ptr(), self.n_halo, eng.mesh_lat_img.data_ptr(),
              lg.mesh_owned_pad, eng._stream()), "gcb_image_rows_unpack")
        else:
          img_off = (lg.mesh_owned_pad // TILE) * 32 * 8448
          self._native.check(self._lib.gcb_rows_to_image(
              self.halo_view.data_ptr(), 512, 1, self.n_halo, 512,
              eng.mesh_lat_img.data_ptr() + img_off, eng._stream()), "gcb_rows_to_image")
    if ev is not None:
      ev[1].record()
      self._events.append(ev)

  def step(self, planes_local, timed_halo: bool = False):
    """planes_local [c_in, n_grid_local] (owned + halo grid rows, `local.local_grid_ids` order) ->
    grid_out [n_grid_owned, 256] of the owned grid rows."""
    eng = self.engine
    eng.pack_inputs(planes_local)
    eng.run_stage("encode")
    self.exchange_halo(timed_halo)
    eng.run_stage("process_embed")
    for k in range(eng.msg_steps):
      eng.run_stage("process_step", k)
      self.exchange_halo(timed_halo)
    eng.run_stage("decode")
    return eng.grid_out[:self.local.grid_owned.size]

  def step_from_host(self, host_planes, host_out):
    """End-to-end step with HOST buffers, pipelined over successive calls.

    host_planes: pinned fp32 [c_in, n_grid_local] (this rank's owned + halo grid columns);
    host_out: pinned fp32 [n_out, n_grid_owned].  The upload runs on a copy stream into one of two
    staging buffers, the download on a second side stream out of one of two result buffers, so call
    i + 1's upload and call i's download overlap the kernels of the neighbouring steps (the host
    returns as soon as everything is queued).  Returns the event after which `host_out` is complete."""
    torch, eng = self._torch, self.engine
    n_owned = int(self.local.grid_owned.size)
    if tuple(host_planes.shape) != (eng.c_in, eng.num_grid) or tuple(host_out.shape) != (eng.n_out, n_owned) \
        or not (host_planes.is_pinned() and host_out.is_pinned()):
      raise ValueError(f"expected pinned fp32 host buffers [{eng.c_in}, {eng.num_grid}] and "
                       f"[{eng.n_out}, {n_owned}]")
    io = getattr(self, "_io", None)
    if io is None:
      f = lambda *shape: torch.empty(shape, dtype=torch.float32, device=eng.device)
      io = self._io = {
          "h2d": torch.cuda.Stream(eng.device), "d2h": torch.cuda.Stream(eng.device), "n": 0,
          "dev_in": [f(eng.c_in, eng.num_grid) for _ in range(2)],
          "dev_out": [f(eng.n_out, n_owned) for _ in range(2)],
          "in_free": [None, None], "out_free": [None, None]}
    b = io["n"] % 2
    io["n"] += 1
    compute = torch.cuda.current_stream(eng.device)
    with torch.cuda.stream(io["h2d"]):
      if io["in_free"][b] is not None:
        io["h2d"].wait_event(io["in_free"][b])        # the step two calls ago has packed this buffer
      io["dev_in"][b].copy_(host_planes, non_blocking=True)
      uploaded = torch.cuda.Event()
      uploaded.record(io["h2d"])
    compute.wait_event(uploaded)
    self.step(io["dev_in"][b])
    io["in_free"][b] = torch.cuda.Event()
    io["in_free"][b].record(compute)                  # conservative: after the whole step
    if io["out_free"][b] is not None:
      compute.wait_event(io["out_free"][b])           # its previous download has finished
    with eng._on_device():
      self._native.check(self._lib.gcb_unpack_grid_outputs(
          eng.grid_out.data_ptr(), 256, eng.n_out, n_owned, None, None, None, None,
          io["dev_out"][b].data_ptr(), eng._stream()), "gcb_unpack_grid_outputs")
    unpacked = torch.cuda.Event()
    unpacked.record(compute)
    with torch.cuda.stream(io["d2h"]):
      io["d2h"].wait_event(unpacked)
      host_out.copy_(io["dev_out"][b], non_blocking=True)
      done = torch.cuda.Event()
      done.record(io["d2h"])
    io["out_free"][b] = done
    return done

  def halo_ms_per_exchange(self) -> Optional[float]:
    if not self._events:
      return None
    self._torch.cuda.synchronize()
    ms = [a.elapsed_time(b) for a, b in self._events]
    self._events = []
    return float(np.mean(ms))
