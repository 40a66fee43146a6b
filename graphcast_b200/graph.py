"""Static graph assembly for GraphCast (host side, once per model instance).

Builds the three typed graphs of reference graphcast.py `_maybe_init`:368-378
(`_init_mesh_properties`:380, `_init_grid_properties`:396,
`_init_grid2mesh_graph`:408, `_init_mesh_graph`:460,
`_init_mesh2grid_graph`:499) as plain numpy arrays in the *reference's* node
numbering and edge order, then derives the device execution order
(receiver-sorted edge permutations, CSR row pointers) that the CUDA kernels
consume.  Edge latents never leave the model, so permuting edges internally is
invisible at the API boundary; node numbering is never changed.
"""

from __future__ import annotations

import dataclasses
from typing import Dict, Optional

import numpy as np

from graphcast_b200 import grid_mesh_connectivity
from graphcast_b200 import icosahedral_mesh
from graphcast_b200 import model_utils


@dataclasses.dataclass
class StaticGraph:
  """All index / feature arrays of one GraphCast instance (reference order)."""
  num_grid_nodes: int
  num_mesh_nodes: int
  grid_lat: np.ndarray              # [n_lat] float32
  grid_lon: np.ndarray              # [n_lon] float32
  grid_node_feats: np.ndarray       # [Ng,3] float32
  mesh_node_feats: np.ndarray       # [Nm,3] float32
  g2m_senders: np.ndarray           # [E1] grid index
  g2m_receivers: np.ndarray         # [E1] mesh index
  g2m_edge_feats: np.ndarray        # [E1,4] float32
  mesh_senders: np.ndarray          # [E2]
  mesh_receivers: np.ndarray        # [E2]
  mesh_edge_feats: np.ndarray       # [E2,4] float32
  m2g_senders: np.ndarray           # [E3] mesh index
  m2g_receivers: np.ndarray         # [E3] grid index (fan-in 3, sorted)
  m2g_edge_feats: np.ndarray        # [E3,4] float32

  def as_dict(self) -> Dict[str, np.ndarray]:
    return {f.name: getattr(self, f.name) for f in dataclasses.fields(self)
            if isinstance(getattr(self, f.name), np.ndarray)}


def build_static_graph(*, grid_lat: np.ndarray, grid_lon: np.ndarray,
                       mesh_size: int, radius_query_fraction_edge_length: float,
                       mesh2grid_edge_normalization_factor: Optional[float] = None,
                       connectivity: Optional[Dict[str, np.ndarray]] = None
                       ) -> StaticGraph:
  """`connectivity` (optional) supplies the results of the two spatial queries
  (`g2m_grid`, `g2m_mesh`, `m2g_grid`, `m2g_mesh` index arrays) so that they are
  not recomputed; everything else is always derived here."""
  meshes = icosahedral_mesh.get_hierarchy_of_triangular_meshes_for_sphere(
      splits=mesh_size)
  finest = meshes[-1]

  # Mesh node lat/lon, float32 (graphcast.py:380-394).
  phi, theta = model_utils.cartesian_to_spherical(
      finest.vertices[:, 0], finest.vertices[:, 1], finest.vertices[:, 2])
  mesh_lat, mesh_lon = model_utils.spherical_to_lat_lon(phi=phi, theta=theta)
  mesh_lat = mesh_lat.astype(np.float32)
  mesh_lon = mesh_lon.astype(np.float32)

  # Grid node lat/lon, node id = lat_i * n_lon + lon_i (graphcast.py:396-406).
  grid_lat = np.asarray(grid_lat).astype(np.float32)
  grid_lon = np.asarray(grid_lon).astype(np.float32)
  lon2d, lat2d = np.meshgrid(grid_lon, grid_lat)
  grid_nodes_lon = lon2d.reshape([-1]).astype(np.float32)
  grid_nodes_lat = lat2d.reshape([-1]).astype(np.float32)
  num_grid = grid_nodes_lat.shape[0]
  num_mesh = finest.vertices.shape[0]

  # grid2mesh (graphcast.py:264-267, 408-458).
  radius = (icosahedral_mesh.max_edge_length(finest)
            * radius_query_fraction_edge_length)
  if connectivity is not None:
    g_idx, m_idx = connectivity["g2m_grid"], connectivity["g2m_mesh"]
  else:
    g_idx, m_idx = grid_mesh_connectivity.radius_query_indices(
        grid_latitude=grid_lat, grid_longitude=grid_lon, mesh=finest, radius=radius)
  grid_feats, mesh_feats, g2m_edge = model_utils.get_bipartite_graph_spatial_features(
      senders_node_lat=grid_nodes_lat, senders_node_lon=grid_nodes_lon,
      receivers_node_lat=mesh_lat, receivers_node_lon=mesh_lon,
      senders=g_idx, receivers=m_idx, edge_normalization_factor=None)

  # multi-mesh (graphcast.py:460-497).
  merged = icosahedral_mesh.merge_meshes(meshes)
  ms, mr = icosahedral_mesh.faces_to_edges(merged.faces)
  mesh_feats2, mesh_edge = model_utils.get_graph_spatial_features(
      node_lat=mesh_lat, node_lon=mesh_lon, senders=ms, receivers=mr)
  del mesh_feats2  # identical to mesh_feats; the processor does not embed nodes

  # mesh2grid (graphcast.py:499-548).
  if connectivity is not None:
    g_idx3, m_idx3 = connectivity["m2g_grid"], connectivity["m2g_mesh"]
  else:
    g_idx3, m_idx3 = grid_mesh_connectivity.in_mesh_triangle_indices(
        grid_latitude=grid_lat, grid_longitude=grid_lon, mesh=finest)
  _, _, m2g_edge = model_utils.get_bipartite_graph_spatial_features(
      senders_node_lat=mesh_lat, senders_node_lon=mesh_lon,
      receivers_node_lat=grid_nodes_lat, receivers_node_lon=grid_nodes_lon,
      senders=m_idx3, receivers=g_idx3,
      edge_normalization_factor=mesh2grid_edge_normalization_factor)

  f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
  i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)
  return StaticGraph(
      num_grid_nodes=num_grid, num_mesh_nodes=num_mesh,
      grid_lat=grid_lat, grid_lon=grid_lon,
      grid_node_feats=f32(grid_feats), mesh_node_feats=f32(mesh_feats),
      g2m_senders=i32(g_idx), g2m_receivers=i32(m_idx), g2m_edge_feats=f32(g2m_edge),
      mesh_senders=i32(ms), mesh_receivers=i32(mr), mesh_edge_feats=f32(mesh_edge),
      m2g_senders=i32(m_idx3), m2g_receivers=i32(g_idx3), m2g_edge_feats=f32(m2g_edge))


def receiver_sorted(senders: np.ndarray, receivers: np.ndarray, num_receivers: int):
  """Stable sort of edges by receiver.  Returns (perm, senders_p, receivers_p,
  row_ptr) with row_ptr [num_receivers+1] the CSR offsets of each receiver's
  in-edges in the permuted order."""
  perm = np.argsort(receivers, kind="stable")
  counts = np.bincount(receivers, minlength=num_receivers)
  row_ptr = np.zeros([num_receivers + 1], dtype=np.int32)
  np.cumsum(counts, out=row_ptr[1:])
  return (perm.astype(np.int64), np.ascontiguousarray(senders[perm], np.int32),
          np.ascontiguousarray(receivers[perm], np.int32), row_ptr)


def sender_csr(senders: np.ndarray, num_senders: int, heavy_threshold: int = 256):
  """CSR of an edge set by SENDER, for the backward of the sender gather (gcb_segment_sum_sorted).
  `senders` are in the edges' execution order.  Returns (order, ptr, heavy): order [E] int32 edge ids
  grouped by sender (stable, so each sender's edges stay in execution order), ptr [num_senders+1]
  int32 offsets into order, heavy int32 ids of the senders with more than `heavy_threshold` edges."""
  senders = np.asarray(senders).astype(np.int64)
  order = np.argsort(senders, kind="stable").astype(np.int32)
  counts = np.bincount(senders, minlength=num_senders)
  ptr = np.zeros([num_senders + 1], dtype=np.int32)
  np.cumsum(counts, out=ptr[1:])
  heavy = np.nonzero(counts > heavy_threshold)[0].astype(np.int32)
  return order, ptr, heavy


def cached_static_graph(*, grid_lat: np.ndarray, grid_lon: np.ndarray,
                        mesh_size: int, radius_query_fraction_edge_length: float,
                        mesh2grid_edge_normalization_factor: Optional[float] = None,
                        cache_dir: Optional[str] = None) -> StaticGraph:
  """`build_static_graph` with an on-disk .npz cache keyed by the arguments.

  Only the results of the two spatial queries (grid2mesh radius query and
  mesh2grid containing-triangle lookup: 4 index arrays, a few MB compressed) are
  cached - they dominate the build time; features are recomputed on load.  The
  cache is purely a start-up optimisation: a missing / unreadable file falls
  back to the full build."""
  import hashlib
  import os
  if cache_dir is None:
    cache_dir = os.environ.get(
        "GRAPHCAST_B200_CACHE",
        os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                     ".graph_cache"))
  h = hashlib.sha1()
  h.update(np.ascontiguousarray(grid_lat, dtype=np.float32).tobytes())
  h.update(np.ascontiguousarray(grid_lon, dtype=np.float32).tobytes())
  h.update(repr((mesh_size, float(radius_query_fraction_edge_length),
                 mesh2grid_edge_normalization_factor, "v3")).encode())
  path = os.path.join(cache_dir, f"connectivity_{h.hexdigest()[:16]}.npz")
  build = lambda conn: build_static_graph(
      grid_lat=grid_lat, grid_lon=grid_lon, mesh_size=mesh_size,
      radius_query_fraction_edge_length=radius_query_fraction_edge_length,
      mesh2grid_edge_normalization_factor=mesh2grid_edge_normalization_factor,
      connectivity=conn)
  if os.path.exists(path):
    try:
      with np.load(path) as z:
        conn = {k: z[k] for k in ("g2m_grid", "g2m_mesh", "m2g_grid", "m2g_mesh")}
      return build(conn)
    except Exception:  # corrupt cache -> rebuild
      pass
  g = build(None)
  try:
    os.makedirs(cache_dir, exist_ok=True)
    tmp = path + f".tmp{os.getpid()}.npz"
    np.savez_compressed(tmp, g2m_grid=g.g2m_senders, g2m_mesh=g.g2m_receivers,
                        m2g_grid=g.m2g_receivers, m2g_mesh=g.m2g_senders)
    os.replace(tmp, path)
  except OSError:
    pass
  return g


def spatial_order(xyz: np.ndarray, bits: int = 10) -> np.ndarray:
  """Permutation that sorts points of the unit sphere along a 3-D Morton (Z-order) curve:
  `order[new] = old`.  Used for the INTERNAL numbering of the mesh nodes on the device: the
  reference numbers them by refinement level (children appended after their parents), so the senders
  of consecutive receivers are scattered over an 84 MB projection table; along a space-filling curve
  they are neighbours in memory and the gathers of the edge blocks hit the L2.  Mesh nodes never
  leave the model, so the renumbering is invisible at the API (grid node numbering is untouched)."""
  q = np.clip(((np.asarray(xyz, np.float64) + 1.0) * 0.5 * ((1 << bits) - 1)).round().astype(np.uint64),
              0, (1 << bits) - 1)
  code = np.zeros(q.shape[0], np.uint64)
  for b in range(bits):
    for axis in range(3):
      code |= ((q[:, axis] >> np.uint64(b)) & np.uint64(1)) << np.uint64(3 * b + axis)
  return np.argsort(code, kind="stable")
