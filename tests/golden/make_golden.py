"""Generates tests/golden/*.npz by IMPORTING THE REFERENCE (a checkout of
google-deepmind/graphcast, `weathernext`):
  GRAPHCAST_REFERENCE=<path of the checkout> python tests/golden/make_golden.py

The reference's JAX model stack is not installable here, but
`weathernext.utils.icosahedral_mesh` is pure numpy/scipy and imports fine; its
outputs pin the static-graph half of the oracle / product:
  * mesh hierarchy (vertices, faces) for splits 0..3, full arrays;
  * splits 4..6: faces hashed (sha256 of int32 bytes) + vertex checksums;
  * multi-mesh `faces_to_edges` senders/receivers for splits 3 (full) and 6 (hash).
"""
import hashlib
import os
import sys

import numpy as np

sys.path.insert(0, os.environ["GRAPHCAST_REFERENCE"])
from weathernext.utils import icosahedral_mesh as ref  # noqa: E402

here = os.path.dirname(os.path.abspath(__file__))
out = {}
for splits in range(0, 7):
  meshes = ref.get_hierarchy_of_triangular_meshes_for_sphere(splits)
  m = meshes[-1]
  faces = np.ascontiguousarray(m.faces, np.int32)
  verts = np.ascontiguousarray(m.vertices, np.float32)
  if splits <= 3:
    out[f"vertices_{splits}"] = verts
    out[f"faces_{splits}"] = faces
  out[f"faces_sha_{splits}"] = np.frombuffer(hashlib.sha256(faces.tobytes()).digest(), np.uint8)
  out[f"vertices_sha_{splits}"] = np.frombuffer(hashlib.sha256(verts.tobytes()).digest(), np.uint8)
  out[f"vertex_sum_{splits}"] = verts.astype(np.float64).sum(0)
  out[f"vertex_abs_sum_{splits}"] = np.abs(verts.astype(np.float64)).sum(0)
  merged = ref.merge_meshes(meshes)
  s, r = ref.faces_to_edges(merged.faces)
  s, r = np.ascontiguousarray(s, np.int32), np.ascontiguousarray(r, np.int32)
  if splits == 3:
    out["multimesh_senders_3"], out["multimesh_receivers_3"] = s, r
  out[f"multimesh_edges_sha_{splits}"] = np.frombuffer(
      hashlib.sha256(s.tobytes() + r.tobytes()).digest(), np.uint8)
np.savez_compressed(os.path.join(here, "icosahedral_mesh_reference.npz"), **out)
print("wrote", os.path.join(here, "icosahedral_mesh_reference.npz"))


# ---- checkpoint format (weathernext/utils/checkpoint.py is pure numpy and imports fine) ----
# A GraphCast-CheckPoint-shaped tree (graphcast.py:115-151: params, model_config, task_config,
# description, license) written by the REFERENCE's `checkpoint.dump`; the test loads it with
# this repo's `checkpoint.load` into this repo's dataclasses and re-dumps it.
import dataclasses  # noqa: E402
from typing import Any, Optional  # noqa: E402

from weathernext.utils import checkpoint as ref_ckpt  # noqa: E402


@dataclasses.dataclass(frozen=True)
class TaskConfig:
  input_variables: tuple[str, ...]      # annotations as in weathernext/utils/task.py:21-28
  target_variables: tuple[str, ...]
  forcing_variables: tuple[str, ...]
  pressure_levels: tuple[int, ...]
  input_duration: str


@dataclasses.dataclass(frozen=True)
class ModelConfig:
  resolution: float
  mesh_size: int
  latent_size: int
  gnn_msg_steps: int
  hidden_layers: int
  radius_query_fraction_edge_length: float
  mesh2grid_edge_normalization_factor: Optional[float] = None


@dataclasses.dataclass(frozen=True)
class CheckPoint:
  params: dict[str, Any]
  model_config: ModelConfig
  task_config: TaskConfig
  description: str
  license: str


rng = np.random.default_rng(5)
ck = CheckPoint(
    params={
        "grid2mesh_gnn/~_networks_builder/encoder_nodes_grid_nodes_mlp/~/linear_0":
            {"w": rng.standard_normal((7, 4)).astype(np.float32), "b": np.zeros(4, np.float32)},
        "grid2mesh_gnn/~_networks_builder/encoder_nodes_grid_nodes_layer_norm":
            {"scale": np.ones(4, np.float32), "offset": rng.standard_normal(4).astype(np.float32)},
    },
    model_config=ModelConfig(1.0, 5, 512, 16, 1, 0.6, None),
    task_config=TaskConfig(("2m_temperature", "geopotential"), ("2m_temperature",),
                           ("toa_incident_solar_radiation",), (50, 500, 1000), "12h"),
    description="golden checkpoint written by the reference's checkpoint.dump",
    license="n/a")
path = os.path.join(here, "reference_checkpoint.npz")
with open(path, "wb") as f:
  ref_ckpt.dump(f, ck)
with open(path, "rb") as f:                       # the reference reads its own file back
  back = ref_ckpt.load(f, CheckPoint)
assert back.model_config == ck.model_config and back.task_config == ck.task_config
print("wrote", path)


# ---- static-graph geometry and features, computed by the reference's own numpy code ----------
# `weathernext/utils/model_utils.py` and `utils/legacy/grid_mesh_connectivity.py` import jax /
# xarray / trimesh at module scope but the functions below are pure numpy + scipy.  The missing
# packages are replaced by empty stub modules (attribute access yields dummy types, enough for
# the annotations evaluated at import time); no reference code is modified or re-implemented.
# Not reachable this way: `in_mesh_triangle_indices` (really calls trimesh) and everything that
# touches xarray data.
import types  # noqa: E402


class _Stub(types.ModuleType):

  def __getattr__(self, name):
    if name.startswith("__"):
      raise AttributeError(name)
    return type(name, (), {})


for _name in ("jax", "jax.numpy", "xarray", "xarray.ufuncs", "trimesh"):
  sys.modules.setdefault(_name, _Stub(_name))
sys.modules["jax"].numpy = sys.modules["jax.numpy"]
sys.modules["xarray"].ufuncs = sys.modules["xarray.ufuncs"]

from weathernext.utils import model_utils as ref_mu  # noqa: E402
from weathernext.utils.legacy import grid_mesh_connectivity as ref_gm  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(here)))
from graphcast_b200 import grid_mesh_connectivity as our_gm  # noqa: E402  (only for m2g INPUT indices)

geo = {}
lat = np.linspace(-90, 90, 19).astype(np.float32)     # float32 like GraphCast._init_grid_properties
lon = np.arange(0, 360, 10.0).astype(np.float32)      # (graphcast.py:396-406)
meshes = ref.get_hierarchy_of_triangular_meshes_for_sphere(2)
finest = meshes[-1]
geo["grid_lat"], geo["grid_lon"] = lat, lon
geo["grid_coordinates"] = ref_gm._grid_lat_lon_to_coordinates(lat, lon)
es, er = ref.faces_to_edges(finest.faces)
max_edge = np.linalg.norm(finest.vertices[es] - finest.vertices[er], axis=-1).max()
geo["radius"] = np.float64(0.6 * max_edge)
g_idx, m_idx = ref_gm.radius_query_indices(grid_latitude=lat, grid_longitude=lon, mesh=finest,
                                           radius=0.6 * max_edge)
geo["g2m_grid_indices"], geo["g2m_mesh_indices"] = g_idx, m_idx
phi, theta = ref_mu.cartesian_to_spherical(finest.vertices[:, 0], finest.vertices[:, 1],
                                           finest.vertices[:, 2])
mesh_lat, mesh_lon = ref_mu.spherical_to_lat_lon(phi=phi, theta=theta)
geo["mesh_lat"], geo["mesh_lon"] = mesh_lat, mesh_lon
lon2d, lat2d = np.meshgrid(lon, lat)
glat, glon = lat2d.reshape(-1).astype(np.float32), lon2d.reshape(-1).astype(np.float32)
kw = dict(add_node_positions=False, add_node_latitude=True, add_node_longitude=True,
          add_relative_positions=True, relative_longitude_local_coordinates=True,
          relative_latitude_local_coordinates=True)      # graphcast.py:408-548 call sites
sn, rn, ef = ref_mu.get_bipartite_graph_spatial_features(
    senders_node_lat=glat, senders_node_lon=glon,
    receivers_node_lat=mesh_lat.astype(np.float32), receivers_node_lon=mesh_lon.astype(np.float32),
    senders=g_idx, receivers=m_idx, edge_normalization_factor=None, **kw)
geo["g2m_grid_node_feats"], geo["g2m_mesh_node_feats"], geo["g2m_edge_feats"] = sn, rn, ef
merged = ref.merge_meshes(meshes)
ms, mr = ref.faces_to_edges(merged.faces)
nf, mef = ref_mu.get_graph_spatial_features(
    node_lat=mesh_lat.astype(np.float32), node_lon=mesh_lon.astype(np.float32),
    senders=ms, receivers=mr, **kw)
geo["mesh_node_feats"], geo["mesh_edge_feats"] = nf, mef
geo["mesh_senders"], geo["mesh_receivers"] = ms, mr
# mesh2grid: the containing-triangle lookup itself needs trimesh; the edge FEATURES for a given
# index list do not.  The indices are an input of this golden (stored), the features the output.
g3, m3 = our_gm.in_mesh_triangle_indices(grid_latitude=lat, grid_longitude=lon, mesh=finest)
geo["m2g_grid_indices"], geo["m2g_mesh_indices"] = g3, m3
for tag, norm in (("", None), ("_norm2", 2.0)):
  _, _, ef3 = ref_mu.get_bipartite_graph_spatial_features(
      senders_node_lat=mesh_lat.astype(np.float32), senders_node_lon=mesh_lon.astype(np.float32),
      receivers_node_lat=glat, receivers_node_lon=glon, senders=m3, receivers=g3,
      edge_normalization_factor=norm, **kw)
  geo["m2g_edge_feats" + tag] = ef3
np.savez_compressed(os.path.join(here, "reference_geometry.npz"), **geo)

# Grid->mesh connectivity at the BASELINE resolutions, by the reference's own
# `radius_query_indices` on the reference's own mesh (utils/legacy/grid_mesh_connectivity.py:40-86,
# grid exactly as GraphCast._init_grid_properties builds it, graphcast.py:396-406): edge count and
# sha256 of the int64 index arrays.  The radius query is tie-sensitive (1-ulp vertex differences
# flip edges at 0.25 degree), so index parity is pinned at the sizes the benchmark runs.
conn = {}
for tag, res, splits in (("1deg_mesh5", 1.0, 5), ("0p25deg_mesh6", 0.25, 6)):
  clat = np.linspace(-90, 90, int(round(180 / res)) + 1).astype(np.float32)
  clon = (np.arange(int(round(360 / res))) * res).astype(np.float32)
  cmesh = ref.get_hierarchy_of_triangular_meshes_for_sphere(splits)[-1]
  ces, cer = ref.faces_to_edges(cmesh.faces)
  cmax = np.linalg.norm(cmesh.vertices[ces] - cmesh.vertices[cer], axis=-1).max()
  gi, mi = ref_gm.radius_query_indices(grid_latitude=clat, grid_longitude=clon, mesh=cmesh,
                                       radius=0.6 * cmax)
  gi, mi = np.ascontiguousarray(gi, np.int64), np.ascontiguousarray(mi, np.int64)
  conn[f"num_edges_{tag}"] = np.int64(gi.shape[0])
  conn[f"grid_sha_{tag}"] = np.frombuffer(hashlib.sha256(gi.tobytes()).digest(), np.uint8)
  conn[f"mesh_sha_{tag}"] = np.frombuffer(hashlib.sha256(mi.tobytes()).digest(), np.uint8)
  conn[f"radius_{tag}"] = np.float64(0.6 * cmax)
np.savez_compressed(os.path.join(here, "reference_connectivity.npz"), **conn)
print("wrote reference_connectivity.npz", {k: (int(v) if v.ndim == 0 and v.dtype.kind == "i" else v.shape)
                                          for k, v in conn.items()})
print("wrote", os.path.join(here, "reference_geometry.npz"),
      {k: (v.shape, str(v.dtype)) for k, v in geo.items() if hasattr(v, "shape")})


# ---- channel packing: the reference's dataset_to_stacked / stacked_to_dataset ----------------
# These functions (model_utils.py:645-776) decide the channel ORDER of the model's inputs and
# outputs: variables sorted by name, non-(batch, lat, lon) dims stacked in the variable's own dim
# order.  They only use a small part of the xarray API, which is provided below by a numpy-backed
# stand-in following xarray's documented semantics (Variable.stack: stacked dims moved to the
# end and flattened in C order, first listed dim slowest; set_dims: broadcast to the requested
# dims, in the requested order; unstack: the inverse reshape).  The reference code itself runs
# unmodified on top of it.
class _Sizes(dict):
  pass


class FakeVariable:

  def __init__(self, dims, data):
    self.dims = tuple(dims)
    self.data = np.asarray(data)
    assert self.data.ndim == len(self.dims)

  @property
  def sizes(self):
    return _Sizes(zip(self.dims, self.data.shape))

  def transpose(self, *dims):
    if Ellipsis in dims:                              # transpose("lat", "lon", ...)
      named = [d for d in dims if d is not Ellipsis]
      rest = [d for d in self.dims if d not in named]
      i = dims.index(Ellipsis)
      dims = tuple(dims[:i]) + tuple(rest) + tuple(dims[i + 1:])
    return FakeVariable(dims, np.transpose(self.data, [self.dims.index(d) for d in dims]))

  @property
  def variable(self):
    return self

  def stack(self, **kw):
    (new_dim, stacked), = kw.items()
    keep = [d for d in self.dims if d not in stacked]
    v = self.transpose(*keep, *stacked)
    shape = v.data.shape[:len(keep)] + (-1,)
    return FakeVariable(tuple(keep) + (new_dim,), v.data.reshape(shape))

  def unstack(self, mapping):
    (old_dim, sizes), = mapping.items()
    assert self.dims[-1] == old_dim
    new_dims = self.dims[:-1] + tuple(sizes.keys())
    return FakeVariable(new_dims, self.data.reshape(self.data.shape[:-1] + tuple(sizes.values())))

  def set_dims(self, dims):
    names = list(dims.keys())
    missing = [d for d in names if d not in self.dims]
    data = self.data.reshape((1,) * len(missing) + self.data.shape)
    v = FakeVariable(tuple(missing) + self.dims, data).transpose(*names)
    return FakeVariable(names, np.broadcast_to(v.data, [dims[d] for d in names]))

  def isel(self, indexers):
    idx = tuple(indexers.get(d, slice(None)) for d in self.dims)
    return FakeVariable(self.dims, self.data[idx])

  @staticmethod
  def concat(variables, dim):
    axis = variables[0].dims.index(dim)
    return FakeVariable(variables[0].dims, np.concatenate([v.data for v in variables], axis=axis))


class FakeDataArray(FakeVariable):

  def __init__(self, data, coords=None, dims=None, name=None):
    if isinstance(data, FakeVariable):
      dims, data = data.dims, data.data
    super().__init__(dims, data)
    self.coords = dict(coords or {})
    self.name = name


class FakeDataset(dict):

  def __init__(self, data_vars, coords=None):
    super().__init__(data_vars)
    self.coords = dict(coords or {})

  @property
  def data_vars(self):
    return self

  @property
  def variables(self):
    return self

  @property
  def sizes(self):
    out = {}
    for v in self.values():
      out.update(v.sizes)
    return out


ref_mu.xr.Variable = FakeVariable
ref_mu.xr.DataArray = FakeDataArray
ref_mu.xr.Dataset = FakeDataset

B, T, L, LA, LO = 2, 2, 3, 4, 5
rng = np.random.default_rng(9)
mk = lambda *shape: rng.standard_normal(shape).astype(np.float32)
inputs_np = {
    "2m_temperature": (("batch", "time", "lat", "lon"), mk(B, T, LA, LO)),
    "geopotential": (("batch", "time", "level", "lat", "lon"), mk(B, T, L, LA, LO)),
    "land_sea_mask": (("lat", "lon"), mk(LA, LO)),                       # static: broadcast over batch
    "toa_incident_solar_radiation": (("batch", "time", "lat", "lon"), mk(B, T, LA, LO)),
    "10m_u_component_of_wind": (("batch", "time", "lat", "lon"), mk(B, T, LA, LO)),
}
ds = FakeDataset({k: FakeDataArray(v, dims=d, name=k) for k, (d, v) in inputs_np.items()})
stacked = ref_mu.dataset_to_stacked(ds)
assert stacked.dims == ("batch", "lat", "lon", "channels")
pack = {"stacked_inputs": stacked.data}
for k, (d, v) in inputs_np.items():
  pack["in:" + k] = v
  pack["in_dims:" + k] = np.array(d)
template_np = {
    "2m_temperature": (("batch", "time", "lat", "lon"), (B, 1, LA, LO)),
    "geopotential": (("batch", "time", "level", "lat", "lon"), (B, 1, L, LA, LO)),
    "total_precipitation_6hr": (("batch", "time", "lat", "lon"), (B, 1, LA, LO)),
}
tmpl = FakeDataset({k: FakeDataArray(np.zeros(shape, np.float32), dims=d, name=k)
                    for k, (d, shape) in template_np.items()})
n_out = sum(int(np.prod([s for dd, s in zip(d, shape) if dd not in ("batch", "lat", "lon")]))
            for d, shape in template_np.values())
flat = rng.standard_normal((B, LA, LO, n_out)).astype(np.float32)
out_ds = ref_mu.stacked_to_dataset(FakeVariable(("batch", "lat", "lon", "channels"), flat), tmpl)
pack["stacked_outputs"] = flat
for k, (d, shape) in template_np.items():
  assert out_ds[k].dims == d
  pack["out:" + k] = out_ds[k].data
  pack["out_dims:" + k] = np.array(d)
np.savez_compressed(os.path.join(here, "reference_packing.npz"), **pack)
print("wrote", os.path.join(here, "reference_packing.npz"), stacked.data.shape, n_out)


# ---- the GNN forward: the reference's GraphCast wiring executed on numpy stand-ins -----------
# weathernext1_graph/graphcast.py, utils/legacy/deep_typed_graph_net.py and utils/typed_graph_net.py
# are imported and RUN (graph construction, `_run_grid2mesh_gnn`, `_run_mesh_gnn`,
# `_run_mesh2grid_gnn`: concat orders, gathers, per-receiver aggregation, residuals, which node
# set is updated when, the three-GNN composition) with jax / jraph / haiku / chex replaced by
# the few numpy primitives of tests/golden/numpy_standins.py.  Only `in_mesh_triangle_indices`
# (needs trimesh) is taken from this repo; the xarray I/O of `__call__` is bypassed by calling
# the three `_run_*` methods on a raw [Ng, B, C] array.
import numpy_standins as ns  # noqa: E402

ns.install()
from weathernext.weathernext1_graph import graphcast as ref_gc  # noqa: E402
from weathernext.utils.legacy import grid_mesh_connectivity as ref_gm2  # noqa: E402

ref_gm2.in_mesh_triangle_indices = our_gm.in_mesh_triangle_indices
task = ref_gc.TaskConfig(
    input_variables=("2m_temperature", "geopotential", "toa_incident_solar_radiation"),
    target_variables=("2m_temperature", "geopotential"),
    forcing_variables=("toa_incident_solar_radiation",), pressure_levels=(500, 850),
    input_duration="12h")
cfg = ref_gc.ModelConfig(resolution=10.0, mesh_size=2, latent_size=32, gnn_msg_steps=3,
                         hidden_layers=1, radius_query_fraction_edge_length=0.6)
model = ref_gc.GraphCast(cfg, task)
glat = np.linspace(-90, 90, 19).astype(np.float32)
glon = np.arange(0, 360, 10.0).astype(np.float32)
model._maybe_init(types.SimpleNamespace(lat=glat, lon=glon))
# Inputs as (stand-in) xarray datasets, converted by the reference's own
# `_inputs_to_grid_node_features` (graphcast.py:680-699); the full `__call__` is run below.
ref_gc.xarray.concat = lambda arrays, dim: FakeDataArray(FakeVariable.concat(list(arrays), dim))
ref_gc.xarray_jax.unwrap = lambda v: v
ref_gc.xarray_jax.DataArray = lambda data, dims: FakeDataArray(data, dims=dims)
NB, NLAT, NLON = 2, 19, 36
rng = np.random.default_rng(0)
mk = lambda *shape: rng.standard_normal(shape).astype(np.float32)
api_inputs = {
    "2m_temperature": (("batch", "time", "lat", "lon"), mk(NB, 2, NLAT, NLON)),
    "geopotential": (("batch", "time", "level", "lat", "lon"), mk(NB, 2, 2, NLAT, NLON)),
    "toa_incident_solar_radiation": (("batch", "time", "lat", "lon"), mk(NB, 2, NLAT, NLON)),
}
api_forcings = {"toa_incident_solar_radiation": (("batch", "time", "lat", "lon"), mk(NB, 1, NLAT, NLON))}
api_template = {
    "2m_temperature": (("batch", "time", "lat", "lon"), np.zeros((NB, 1, NLAT, NLON), np.float32)),
    "geopotential": (("batch", "time", "level", "lat", "lon"), np.zeros((NB, 1, 2, NLAT, NLON), np.float32)),
}
to_ds = lambda spec: FakeDataset({k: FakeDataArray(v, dims=d, name=k) for k, (d, v) in spec.items()})
ds_inputs, ds_forcings, ds_template = to_ds(api_inputs), to_ds(api_forcings), to_ds(api_template)
ds_inputs.lat, ds_inputs.lon = glat, glon
x = model._inputs_to_grid_node_features(ds_inputs, ds_forcings)
assert x.shape == (NLAT * NLON, NB, 9)
latent_mesh, latent_grid = model._run_grid2mesh_gnn(x)
updated_mesh = model._run_mesh_gnn(latent_mesh)
output = model._run_mesh2grid_gnn(updated_mesh, latent_grid)
predictions = model(ds_inputs, ds_template, ds_forcings)          # the reference's __call__, end to end
gnn = {"grid_lat": glat, "grid_lon": glon, "grid_features": x,
       "latent_mesh_after_grid2mesh": latent_mesh, "latent_grid_after_grid2mesh": latent_grid,
       "latent_mesh_after_mesh_gnn": updated_mesh, "output": output,
       "mesh_size": np.int64(2), "gnn_msg_steps": np.int64(3)}


def _edges(graph, name):
  key = graph.edge_key_by_name(name)
  es = graph.edges[key]
  return es.indices.senders, es.indices.receivers, es.features


g2m, mesh_g, m2g = (model._grid2mesh_graph_structure, model._mesh_graph_structure,
                    model._mesh2grid_graph_structure)
gnn["grid_node_feats"] = g2m.nodes["grid_nodes"].features
gnn["mesh_node_feats"] = g2m.nodes["mesh_nodes"].features
for tag, graph, name in (("g2m", g2m, "grid2mesh"), ("mesh", mesh_g, "mesh"), ("m2g", m2g, "mesh2grid")):
  s_, r_, f_ = _edges(graph, name)
  gnn[f"{tag}_senders"], gnn[f"{tag}_receivers"], gnn[f"{tag}_edge_feats"] = s_, r_, f_
for tag, spec in (("api_in", api_inputs), ("api_forcing", api_forcings)):
  for k, (d, v) in spec.items():
    gnn[f"{tag}:{k}"], gnn[f"{tag}_dims:{k}"] = v, np.array(d)
for k, (d, v) in api_template.items():
  assert predictions[k].dims == d
  gnn[f"api_out:{k}"], gnn[f"api_out_dims:{k}"] = predictions[k].data, np.array(d)
for path, entry in ns.PARAMS.items():
  for leaf, value in entry.items():
    gnn[f"param:{path}:{leaf}"] = value
# sanity: the manifest + seed reproduce the parameters bit for bit
_regen = ns.regenerate(ns.MANIFEST, ns.SEED)
assert all(np.array_equal(_regen[k][l], v) for k, e in ns.PARAMS.items() for l, v in e.items())
np.savez_compressed(os.path.join(here, "reference_gnn_forward.npz"), **gnn)

# Same wiring at the CUDA kernels' width (latent 512) for the GPU test: the parameters (40 MB) are
# not stored, only the seed and the creation manifest they are regenerated from.
ns.reset(seed=512512)
cfg512 = ref_gc.ModelConfig(resolution=10.0, mesh_size=2, latent_size=512, gnn_msg_steps=2,
                            hidden_layers=1, radius_query_fraction_edge_length=0.6)
model512 = ref_gc.GraphCast(cfg512, task)
model512._maybe_init(types.SimpleNamespace(lat=glat, lon=glon))
x512 = np.random.default_rng(1).standard_normal((NLAT * NLON, NB, 9)).astype(np.float32)
lm512, lg512 = model512._run_grid2mesh_gnn(x512)
um512 = model512._run_mesh_gnn(lm512)
out512 = model512._run_mesh2grid_gnn(um512, lg512)
g512 = {k: v for k, v in gnn.items()
        if k.split("_")[0] in ("grid", "mesh", "g2m", "m2g") and not k.startswith("grid_features")}
g512.update(grid_features=x512, output=out512, seed=np.int64(ns.SEED), gnn_msg_steps=np.int64(2),
            manifest_path=np.array([m[0] for m in ns.MANIFEST]),
            manifest_kind=np.array([m[1] for m in ns.MANIFEST]),
            manifest_shape=np.array([[m[2], m[3]] for m in ns.MANIFEST], np.int64),
            mesh_rms_after_mesh_gnn=np.sqrt(np.mean(um512.astype(np.float64) ** 2)))
np.savez_compressed(os.path.join(here, "reference_gnn_forward_latent512.npz"), **g512)
print("wrote", os.path.join(here, "reference_gnn_forward_latent512.npz"), out512.shape, sorted(g512)[:30])
print("wrote", os.path.join(here, "reference_gnn_forward.npz"), output.shape, len(ns.PARAMS), "param entries")


# ---- normalisation wrapper: the reference's InputsAndResiduals.__call__ executed ---------------
# utils/normalization.py and utils/xarray_tree.py run unmodified on the stand-in datasets, which
# get the remaining xarray behaviour they need: arithmetic that broadcasts by dimension NAME
# (result dims = dims of the left operand, then the new dims of the right one), `astype`,
# `isel(time=-1)` (an integer index drops the dim), `rename`, `merge`.
def _binary(a, b, op):
  if not isinstance(b, FakeVariable):
    return FakeDataArray(op(a.data, b), dims=a.dims, name=getattr(a, "name", None))
  dims = tuple(a.dims) + tuple(d for d in b.dims if d not in a.dims)

  def expand(v):
    have = [d for d in dims if d in v.dims]
    data = np.transpose(v.data, [v.dims.index(d) for d in have])
    return data.reshape([v.sizes[d] if d in v.dims else 1 for d in dims])

  return FakeDataArray(op(expand(a), expand(b)), dims=dims, name=getattr(a, "name", None))


FakeVariable.__sub__ = lambda a, b: _binary(a, b, np.subtract)
FakeVariable.__add__ = lambda a, b: _binary(a, b, np.add)
FakeVariable.__mul__ = lambda a, b: _binary(a, b, np.multiply)
FakeVariable.__truediv__ = lambda a, b: _binary(a, b, np.divide)
FakeVariable.dtype = property(lambda self: self.data.dtype)
FakeVariable.astype = lambda self, dt: FakeDataArray(self.data.astype(dt), dims=self.dims,
                                                     name=getattr(self, "name", None))
FakeDataArray.rename = lambda self, name: FakeDataArray(self.data, dims=self.dims, name=name)
_isel_dict = FakeVariable.isel


def _isel(self, indexers=None, **kw):
  indexers = dict(indexers or {}, **kw)
  out = _isel_dict(self, {k: v for k, v in indexers.items() if isinstance(v, slice)})
  for k, v in indexers.items():
    if not isinstance(v, slice):                        # integer: index and drop the dim
      ax = out.dims.index(k)
      out = FakeVariable(out.dims[:ax] + out.dims[ax + 1:], np.take(out.data, v, axis=ax))
  return FakeDataArray(out.data, dims=out.dims, name=getattr(self, "name", None))


FakeVariable.isel = _isel
import importlib  # noqa: E402

xr_mod = sys.modules["xarray"]
xr_mod.Dataset, xr_mod.DataArray = FakeDataset, FakeDataArray
xr_mod.merge = lambda arrays, join=None, compat=None: FakeDataset({a.name: a for a in arrays})
ref_norm = importlib.import_module("weathernext.utils.normalization")

levels = 2
stats_spec = lambda fn: FakeDataset({
    "2m_temperature": FakeDataArray(np.float32(fn(0)), dims=(), name="2m_temperature"),
    "geopotential": FakeDataArray(np.array([fn(1), fn(2)], np.float32), dims=("level",), name="geopotential"),
    "toa_incident_solar_radiation": FakeDataArray(np.float32(fn(3)), dims=(), name="toa_incident_solar_radiation"),
    "total_precipitation_6hr": FakeDataArray(np.float32(fn(4)), dims=(), name="total_precipitation_6hr"),
})
mean_by_level = stats_spec(lambda i: 1.5 * i - 2.0)
stddev_by_level = stats_spec(lambda i: 0.5 + 0.75 * i)
diffs_stddev_by_level = stats_spec(lambda i: 0.1 + 0.05 * i)
captured = {}


def inner_predictor(norm_inputs, targets_template, forcings):
  """Stands for the model: records what it is given, returns a fixed function of it."""
  captured["norm_inputs"], captured["norm_forcings"] = norm_inputs, forcings
  out = {}
  for name in targets_template.keys():
    if name in norm_inputs.keys():
      v = norm_inputs[name]
      out[name] = FakeDataArray(0.5 * v.data[:, -1:] + 0.25, dims=v.dims, name=name)
    else:                                                   # target-only variable
      t = targets_template[name]
      out[name] = FakeDataArray(np.full(t.data.shape, 0.125, np.float32) * (1 + np.arange(t.data.shape[-1], dtype=np.float32)),
                                dims=t.dims, name=name)
  return FakeDataset(out)


norm_template = dict(api_template)
norm_template["total_precipitation_6hr"] = (("batch", "time", "lat", "lon"), np.zeros((NB, 1, NLAT, NLON), np.float32))
wrapped = ref_norm.InputsAndResiduals(inner_predictor, stddev_by_level=stddev_by_level,
                                      mean_by_level=mean_by_level,
                                      diffs_stddev_by_level=diffs_stddev_by_level)
norm_out = wrapped(ds_inputs, to_ds(norm_template), ds_forcings)
nz = {}
for tag, spec in (("in", api_inputs), ("forcing", api_forcings)):
  for k, (d, v) in spec.items():
    nz[f"{tag}:{k}"], nz[f"{tag}_dims:{k}"] = v, np.array(d)
for k, (d, v) in norm_template.items():
  nz[f"template_dims:{k}"], nz[f"template_shape:{k}"] = np.array(d), np.array(v.shape)
for sname, sds in (("mean", mean_by_level), ("std", stddev_by_level), ("diffs_std", diffs_stddev_by_level)):
  for k in sds.keys():
    nz[f"{sname}:{k}"], nz[f"{sname}_dims:{k}"] = sds[k].data, np.array(sds[k].dims, dtype=str)
for k in captured["norm_inputs"].keys():
  nz[f"norm_in:{k}"] = captured["norm_inputs"][k].data
for k in captured["norm_forcings"].keys():
  nz[f"norm_forcing:{k}"] = captured["norm_forcings"][k].data
for k in norm_out.keys():
  nz[f"out:{k}"], nz[f"out_dims:{k}"] = norm_out[k].data, np.array(norm_out[k].dims)
np.savez_compressed(os.path.join(here, "reference_normalization.npz"), **nz)
print("wrote", os.path.join(here, "reference_normalization.npz"), sorted(norm_out.keys()))


# ---- rollout: the reference's chunked_prediction_generator / _get_next_inputs executed ----------
# utils/rollout.py runs unmodified.  Its xarray use needs a dataset with coordinates: `RDataset`
# below adds `coords` (name -> DataArray), `copy`, `isel(time=slice)` (data and time coordinates),
# `assign_coords`, `assign`, `compute`, `__getitem__(list)`, `dims`, and `xarray.concat(...,
# dim="time", data_vars="different")` + `tail` as used by `_get_next_inputs` (variables without
# the concat dim are taken from the first dataset).  jax.jit / vmap / random.split are identity
# functions here (no randomness is used by the recording predictor).
class RDataset(FakeDataset):

  def __init__(self, data_vars, coords=None):
    super().__init__(data_vars, coords)

  def copy(self):
    return RDataset(dict(self), dict(self.coords))

  def compute(self):
    return self

  def __getitem__(self, key):
    if isinstance(key, list):
      return RDataset({k: dict.__getitem__(self, k) for k in key}, dict(self.coords))
    return dict.__getitem__(self, key)

  @property
  def dims(self):
    out = []
    for v in self.values():
      out.extend(d for d in v.dims if d not in out)
    return tuple(out)

  def isel(self, **kw):
    data = {k: (v.isel(kw) if all(d in v.dims for d in kw) else v) for k, v in self.items()}
    coords = {k: (c.isel(kw) if all(d in c.dims for d in kw) else c) for k, c in self.coords.items()}
    return RDataset(data, coords)

  def assign_coords(self, coords=None, **kw):
    new = dict(self.coords)
    for k, v in dict(coords or {}, **kw).items():
      new[k] = v if isinstance(v, FakeVariable) else FakeDataArray(np.asarray(v), dims=(k,), name=k)
    return RDataset(dict(self), new)

  def assign(self, other):
    data = dict(self)
    data.update(other)
    return RDataset(data, dict(self.coords))

  def tail(self, **kw):
    (dim, n), = kw.items()
    return self.isel(**{dim: slice(-n, None)})


def _concat(datasets, dim, data_vars=None, compat=None):
  first = datasets[0]
  out = {}
  for k, v in first.items():
    if dim in v.dims:
      parts = [ds[k].transpose(*v.dims) for ds in datasets]
      out[k] = FakeDataArray(FakeVariable.concat(parts, dim), name=k)
    else:
      out[k] = v                                            # data_vars="different": not concatenated
  coords = dict(first.coords)
  if dim in coords:
    coords[dim] = FakeDataArray(np.concatenate([ds.coords[dim].data for ds in datasets]), dims=(dim,), name=dim)
  return RDataset(out, coords)


jax_mod = sys.modules["jax"]
jax_mod.jit = lambda f, **kw: f
jax_mod.vmap = lambda f, **kw: f
jax_mod.pmap = lambda f, **kw: f
jax_mod.random = types.SimpleNamespace(split=lambda rng: (rng, rng))
xr_mod.Dataset = RDataset
xr_mod.concat = _concat
ref_rollout = importlib.import_module("weathernext.utils.rollout")

NSTEPS = 4
hour = np.timedelta64(6, "h")
roll_inputs_np = {
    "2m_temperature": (("batch", "time", "lat", "lon"), mk(NB, 2, 3, 4)),
    "geopotential": (("batch", "time", "level", "lat", "lon"), mk(NB, 2, 2, 3, 4)),
    "toa_incident_solar_radiation": (("batch", "time", "lat", "lon"), mk(NB, 2, 3, 4)),
    "land_sea_mask": (("lat", "lon"), mk(3, 4)),
}
roll_forcings_np = {"toa_incident_solar_radiation": (("batch", "time", "lat", "lon"), mk(NB, NSTEPS, 3, 4))}
roll_template_np = {
    "2m_temperature": (("batch", "time", "lat", "lon"), np.zeros((NB, NSTEPS, 3, 4), np.float32)),
    "geopotential": (("batch", "time", "level", "lat", "lon"), np.zeros((NB, NSTEPS, 2, 3, 4), np.float32)),
}
time_coord = lambda values: {"time": FakeDataArray(np.asarray(values), dims=("time",), name="time")}
to_rds = lambda spec, times: RDataset({k: FakeDataArray(v, dims=d, name=k) for k, (d, v) in spec.items()},
                                      time_coord(times))
in_times = np.array([-1, 0]) * hour
tgt_times = (np.arange(NSTEPS) + 1) * hour
calls = []


def recording_predictor(rng, inputs, targets_template, forcings):
  """Depends on both input frames and on the forcing of the target time, so that the order of
  the frames and the forcing slice fed at every step show up in the trajectory."""
  calls.append({"in_time": inputs.coords["time"].data.copy(),
                "target_time": targets_template.coords["time"].data.copy()})
  f = forcings["toa_incident_solar_radiation"].data                 # [B, 1, lat, lon]
  out = {}
  for name in targets_template.keys():
    x = inputs[name].data                                            # [B, 2, ...]
    fb = f.reshape(f.shape[:2] + (1,) * (x.ndim - 4) + f.shape[2:])
    out[name] = FakeDataArray(0.9 * x[:, 1:] + 0.1 * x[:, :1] + 0.05 * fb + 0.01 * inputs["land_sea_mask"].data,
                              dims=inputs[name].dims, name=name)
  return RDataset(out, dict(targets_template.coords))


chunks = list(ref_rollout.chunked_prediction_generator(
    recording_predictor, rng=0, inputs=to_rds(roll_inputs_np, in_times),
    targets_template=to_rds(roll_template_np, tgt_times), num_steps_per_chunk=1,
    forcings=to_rds(roll_forcings_np, tgt_times)))
assert len(chunks) == NSTEPS
ro = {"in_times": in_times.astype("timedelta64[h]").astype(np.int64),
      "target_times": tgt_times.astype("timedelta64[h]").astype(np.int64)}
for tag, spec in (("in", roll_inputs_np), ("forcing", roll_forcings_np), ("template", roll_template_np)):
  for k, (d, v) in spec.items():
    ro[f"{tag}:{k}"], ro[f"{tag}_dims:{k}"] = v, np.array(d)
for i, (chunk, call) in enumerate(zip(chunks, calls)):
  for k in chunk.keys():
    ro[f"chunk{i}:{k}"] = chunk[k].data
  ro[f"chunk{i}_time"] = chunk.coords["time"].data.astype("timedelta64[h]").astype(np.int64)
  ro[f"call{i}_in_time"] = call["in_time"].astype("timedelta64[h]").astype(np.int64)
  ro[f"call{i}_target_time"] = call["target_time"].astype("timedelta64[h]").astype(np.int64)
np.savez_compressed(os.path.join(here, "reference_rollout.npz"), **ro)
print("wrote", os.path.join(here, "reference_rollout.npz"), [c["in_time"].astype("timedelta64[h]").astype(int).tolist() for c in calls],
      [c.coords["time"].data.astype("timedelta64[h]").astype(int).tolist() for c in chunks])


# ---- ensemble driver: the reference's chunked_prediction_generator_multiple_runs executed -------
# Non-pmap branch (one member after the other).  Inputs carry a leading "sample" dim; the stand-in
# dataset gets `isel(sample=i, drop=True)`, `sizes` including coordinates and item assignment on
# `coords`.
_r_isel = RDataset.isel


def _r_isel_drop(self, drop=False, **kw):
  return _r_isel(self, **kw)


RDataset.isel = _r_isel_drop
absl_logging = sys.modules["absl.logging"]
absl_logging.info = lambda *a, **k: None
absl_logging.flush = lambda *a, **k: None
sys.modules["absl"].logging = absl_logging
ref_rollout.logging = absl_logging
NS = 3
ens_inputs_np = {k: ((("sample",) + d) if "time" in d else d,
                     (np.stack([v * (1.0 + 0.5 * s) for s in range(NS)]) if "time" in d else v))
                 for k, (d, v) in roll_inputs_np.items()}
ens_forcings_np = {k: (("sample",) + d, np.stack([v + 0.25 * s for s in range(NS)]))
                   for k, (d, v) in roll_forcings_np.items()}
ens_chunks = list(ref_rollout.chunked_prediction_generator_multiple_runs(
    recording_predictor, rngs=np.arange(NS), inputs=to_rds(ens_inputs_np, in_times),
    targets_template=to_rds(roll_template_np, tgt_times), forcings=to_rds(ens_forcings_np, tgt_times),
    num_samples=NS, num_steps_per_chunk=1))
assert len(ens_chunks) == NS * NSTEPS
en = {"in_times": ro["in_times"], "target_times": ro["target_times"], "num_samples": np.int64(NS)}
for tag, spec in (("in", ens_inputs_np), ("forcing", ens_forcings_np), ("template", roll_template_np)):
  for k, (d, v) in spec.items():
    en[f"{tag}:{k}"], en[f"{tag}_dims:{k}"] = v, np.array(d)
for i, chunk in enumerate(ens_chunks):
  for k in chunk.keys():
    en[f"chunk{i}:{k}"] = chunk[k].data
  en[f"chunk{i}_time"] = chunk.coords["time"].data.astype("timedelta64[h]").astype(np.int64)
  en[f"chunk{i}_sample"] = np.int64(chunk.coords["sample"] if not hasattr(chunk.coords["sample"], "data")
                                    else chunk.coords["sample"].data)
np.savez_compressed(os.path.join(here, "reference_rollout_ensemble.npz"), **en)
print("wrote", os.path.join(here, "reference_rollout_ensemble.npz"),
      [(int(en[f"chunk{i}_sample"]), en[f"chunk{i}_time"].tolist()) for i in range(len(ens_chunks))])


# ---- forcing generation: the reference's progress features and TISR executed ---------------------
# utils/data_utils.py (get_year_progress, get_day_progress, featurize_progress) and
# utils/solar_radiation.py (get_tsi, get_toa_incident_solar_radiation with the default ERA5 TSI
# series) run unmodified; pandas is the real package, jnp is numpy, jax.jit is the identity and
# jax.scipy.integrate.trapezoid is numpy's.
jax_mod.jit = lambda f, **kw: f
jax_mod.scipy = types.SimpleNamespace(integrate=types.SimpleNamespace(trapezoid=np.trapezoid))
xr_mod.Variable = FakeVariable
_fda_init = FakeDataArray.__init__


def _fda_init_coords(self, data, coords=None, dims=None, name=None):
  _fda_init(self, data, coords=None, dims=dims, name=name)
  self.coords = {k: (v if isinstance(v, FakeVariable) else FakeDataArray(np.asarray(v), dims=(k,), name=k))
                 for k, v in (coords or {}).items()}


FakeDataArray.__init__ = _fda_init_coords
ref_solar = importlib.import_module("weathernext.utils.solar_radiation")
ref_du = importlib.import_module("weathernext.utils.data_utils")
stamps = np.array(["2020-02-29T18:00", "1989-11-08T21:00", "2033-07-01T00:00", "2000-01-01T12:00",
                   "1979-12-31T06:00"], dtype="datetime64[ns]")
f_lat = np.linspace(-90.0, 90.0, 7)
f_lon = np.arange(0.0, 360.0, 45.0)
seconds = stamps.astype("datetime64[s]").astype(np.int64)
fg = {"timestamps_ns": stamps.astype(np.int64), "lat": f_lat, "lon": f_lon,
      "year_progress": ref_du.get_year_progress(seconds),
      "day_progress": ref_du.get_day_progress(seconds, f_lon),
      "tsi": np.asarray(ref_solar.get_tsi(list(stamps), ref_solar.era5_tsi_data())),
      "tisr_1h_360": np.asarray(ref_solar.get_toa_incident_solar_radiation(list(stamps), f_lat, f_lon)),
      "tisr_6h_24_reference_tsi": np.asarray(ref_solar.get_toa_incident_solar_radiation(
          list(stamps[:2]), f_lat, f_lon, tsi_data=ref_solar.reference_tsi_data(),
          integration_period="6h", num_integration_bins=24))}
feat = ref_du.featurize_progress("day_progress", ("time", "lon"), fg["day_progress"])
for k, v in feat.items():
  fg["feat:" + k], fg["feat_dims:" + k] = v.data, np.array(v.dims)
np.savez_compressed(os.path.join(here, "reference_forcings.npz"), **fg)
print("wrote", os.path.join(here, "reference_forcings.npz"), fg["tisr_1h_360"].shape, fg["tisr_1h_360"].dtype,
      float(fg["tisr_1h_360"].max()), fg["tsi"])


# ---- example batch -> (inputs, targets, forcings): the reference's data_utils executed -----------
# `extract_inputs_targets_forcings` / `extract_input_target_times` (data_utils.py:214-333) run
# unmodified with real pandas Timedeltas; the stand-in dataset gets label selection (`sel` on
# level / time, inclusive slices), `drop_vars` and integer indexing of a coordinate.
import pandas as pd  # noqa: E402


def _labels(values):
  return np.asarray([np.timedelta64(pd.Timedelta(v).value, "ns") if isinstance(v, (pd.Timedelta, str)) else v
                     for v in values])


def _r_sel(self, indexers=None, **kw):
  indexers = dict(indexers or {}, **kw)
  out = self
  for dim, sel in indexers.items():
    coord = out.coords[dim].data
    if isinstance(sel, slice):
      lo, hi = _labels([sel.start])[0], _labels([sel.stop])[0]
      idx = np.flatnonzero((coord >= lo) & (coord <= hi))
    else:
      idx = np.asarray([int(np.flatnonzero(coord == l)[0]) for l in _labels(list(sel))])
    data = {k: (FakeDataArray(np.take(v.data, idx, axis=v.dims.index(dim)), dims=v.dims, name=k)
                if dim in v.dims else v) for k, v in out.items()}
    coords = {k: (FakeDataArray(np.take(c.data, idx, axis=c.dims.index(dim)), dims=c.dims, name=k)
                  if dim in c.dims else c) for k, c in out.coords.items()}
    out = RDataset(data, coords)
  return out


RDataset.sel = _r_sel
RDataset.drop_vars = lambda self, name: RDataset(dict(self), {k: c for k, c in self.coords.items() if k != name})
FakeVariable.__getitem__ = lambda self, i: FakeDataArray(self.data[i], dims=self.dims[1:], name=getattr(self, "name", None))
_prev_binary = _binary


def _binary_td(a, b, op):
  if isinstance(b, pd.Timedelta):
    b = np.timedelta64(b.value, "ns")
  return _prev_binary(a, b, op)


FakeVariable.__sub__ = lambda a, b: _binary_td(a, b, np.subtract)
FakeVariable.__add__ = lambda a, b: _binary_td(a, b, np.add)
rngd = np.random.default_rng(21)
mkd = lambda *s: rngd.standard_normal(s).astype(np.float32)
DB, DT, DL, DLAT, DLON = 2, 5, 4, 3, 4
batch_np = {
    "2m_temperature": (("batch", "time", "lat", "lon"), mkd(DB, DT, DLAT, DLON)),
    "geopotential": (("batch", "time", "level", "lat", "lon"), mkd(DB, DT, DL, DLAT, DLON)),
    "toa_incident_solar_radiation": (("batch", "time", "lat", "lon"), mkd(DB, DT, DLAT, DLON)),
    "land_sea_mask": (("lat", "lon"), mkd(DLAT, DLON)),
}
d_time = (np.arange(DT) * np.timedelta64(6, "h")).astype("timedelta64[ns]")
d_level = np.array([50, 500, 850, 1000])
d_datetime = (np.datetime64("2021-03-04T00:00", "ns") + d_time)[None].repeat(DB, 0)
example = RDataset(
    {k: FakeDataArray(v, dims=d, name=k) for k, (d, v) in batch_np.items()},
    {"time": FakeDataArray(d_time, dims=("time",), name="time"),
     "level": FakeDataArray(d_level, dims=("level",), name="level"),
     "lat": FakeDataArray(np.linspace(-45, 45, DLAT), dims=("lat",), name="lat"),
     "lon": FakeDataArray(np.arange(DLON) * 90.0, dims=("lon",), name="lon"),
     "datetime": FakeDataArray(d_datetime, dims=("batch", "time"), name="datetime")})
du = {"time_ns": d_time.astype(np.int64), "level": d_level, "datetime_ns": d_datetime.astype(np.int64)}
for k, (d, v) in batch_np.items():
  du[f"in:{k}"], du[f"in_dims:{k}"] = v, np.array(d)
task_kw = dict(input_variables=("2m_temperature", "geopotential", "toa_incident_solar_radiation", "land_sea_mask"),
               target_variables=("2m_temperature", "geopotential"),
               forcing_variables=("toa_incident_solar_radiation",), pressure_levels=(500, 1000),
               input_duration="12h")
for tag, lead in (("slice", slice("6h", "18h")), ("list", ["12h"])):
  parts = ref_du.extract_inputs_targets_forcings(example, target_lead_times=lead, **task_kw)
  for part_name, part in zip(("inputs", "targets", "forcings"), parts):
    du[f"{tag}:{part_name}:time_ns"] = part.coords["time"].data.astype("timedelta64[ns]").astype(np.int64)
    du[f"{tag}:{part_name}:names"] = np.array(sorted(part.keys()))
    assert "datetime" not in part.coords
    for k in part.keys():
      du[f"{tag}:{part_name}:{k}"] = part[k].data
      du[f"{tag}:{part_name}_dims:{k}"] = np.array(part[k].dims)
np.savez_compressed(os.path.join(here, "reference_data_utils.npz"), **du)
print("wrote", os.path.join(here, "reference_data_utils.npz"),
      {t: (du[f"{t}:inputs:time_ns"] // 3600e9).tolist() for t in ("slice", "list")},
      {t: (du[f"{t}:targets:time_ns"] // 3600e9).tolist() for t in ("slice", "list")})


# ---- variable tables (weathernext/utils/variables.py is plain data and imports fine) -------------
from weathernext.utils import variables as ref_vars  # noqa: E402

vt = {name: np.array(getattr(ref_vars, name)) for name in dir(ref_vars)
      if name.isupper() and isinstance(getattr(ref_vars, name), tuple)}
vt["PRESSURE_LEVELS_keys"] = np.array(sorted(ref_vars.PRESSURE_LEVELS))
np.savez_compressed(os.path.join(here, "reference_variables.npz"), **vt)
print("wrote", os.path.join(here, "reference_variables.npz"), sorted(vt))


# ---- task definitions (weathernext1_graph/graphcast.py:86-112), via the stand-in import ----------
tk = {}
for tname in ("TASK", "TASK_13", "TASK_13_PRECIP_OUT"):
  t = getattr(ref_gc, tname)
  for field in ("input_variables", "target_variables", "forcing_variables", "pressure_levels"):
    tk[f"{tname}:{field}"] = np.array(getattr(t, field))
  tk[f"{tname}:input_duration"] = np.array(t.input_duration)
np.savez_compressed(os.path.join(here, "reference_tasks.npz"), **tk)
print("wrote", os.path.join(here, "reference_tasks.npz"), {k: len(v) for k, v in tk.items() if v.ndim})
