"""Generates tests/golden/reference_losses.npz by EXECUTING THE REFERENCE's loss code:
  GRAPHCAST_REFERENCE=<path of the checkout> python tests/golden/make_golden_losses.py

Run unmodified: `weathernext/utils/losses.py` (weighted_mse_per_level / weighted_mae_per_level,
sum_per_variable_losses, the latitude / level weights), `GraphCast.loss_and_predictions` / `loss`
(`weathernext1_graph/graphcast.py:331-366`, called unbound on a stand-in whose `__call__` returns fixed
predictions: pins the per-variable weights), `InputsAndResiduals.loss` / `loss_and_predictions`
(`utils/normalization.py:134-196`) around a recording predictor, and `autoregressive.Predictor.loss`
(`utils/autoregressive.py:224-312`, T = 3 and T = 1) around a predictor that depends on its inputs.

jax / haiku are the numpy stand-ins of tests/golden/numpy_standins.py.  xarray and xarray_jax are
replaced by the small numpy-backed `DataArray` / `Dataset` below, which follow xarray's documented
semantics for what this code calls: arithmetic that broadcasts by dimension NAME (result dims = dims of
the left operand, then the new dims of the right one) and keeps the operands' coordinates, `**`, `abs`,
`astype`, `notnull`, `where`, `mean` / `sum` over named dims (NaNs propagate: skipna=False), numpy
ufuncs on a coordinate returning an array with the same dims, item assignment, `isel` (an integer drops
the dim), `rename`, `transpose` with `...`; on datasets `isel`, `transpose`, `expand_dims`, `drop_vars`,
`assign_coords`, `tail`, `xarray.merge`, `xarray.concat` (along `time` for datasets, a new `variable`
dim for arrays), and xarray_jax's flattening of a dataset into its arrays (dims and coordinates in the
tree definition).  hk.scan is a Python loop that stacks the per-step outputs.
"""
import importlib
import os
import sys

import numpy as np

sys.path.insert(0, os.environ["GRAPHCAST_REFERENCE"])
here = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, here)
import numpy_standins as ns  # noqa: E402


# ---- xarray stand-in --------------------------------------------------------------------------
class DataArray:

  def __init__(self, data, coords=None, dims=(), name=None):
    self.data = np.asarray(data) if not isinstance(data, np.ndarray) else data
    self.dims = tuple(dims)
    assert self.data.ndim == len(self.dims), (self.data.shape, self.dims)
    self.name = name
    self.coords = {k: (v if isinstance(v, DataArray) else DataArray(np.asarray(v), dims=(k,), name=k))
                   for k, v in (coords or {}).items()}

  @property
  def sizes(self):
    return dict(zip(self.dims, self.data.shape))

  @property
  def dtype(self):
    return self.data.dtype

  def _new(self, data, dims=None, coords=None):
    return DataArray(data, coords=dict(self.coords) if coords is None else coords,
                     dims=self.dims if dims is None else dims, name=self.name)

  def _binary(self, other, op):
    if not isinstance(other, DataArray):
      return self._new(op(self.data, other))
    dims = self.dims + tuple(d for d in other.dims if d not in self.dims)

    def expand(v):
      have = [d for d in dims if d in v.dims]
      x = np.transpose(v.data, [v.dims.index(d) for d in have])
      return x.reshape([v.sizes[d] if d in v.dims else 1 for d in dims])

    coords = dict(other.coords)
    coords.update(self.coords)
    return self._new(op(expand(self), expand(other)), dims, coords)

  __add__ = lambda a, b: a._binary(b, np.add)
  __sub__ = lambda a, b: a._binary(b, np.subtract)
  __mul__ = lambda a, b: a._binary(b, np.multiply)
  __truediv__ = lambda a, b: a._binary(b, np.divide)
  __pow__ = lambda a, p: a._new(a.data ** p)
  __abs__ = lambda a: a._new(np.abs(a.data))

  def __array__(self, dtype=None, copy=None):
    return np.asarray(self.data, dtype=dtype)

  def __array_ufunc__(self, ufunc, method, *inputs, **kw):
    raw = [x.data if isinstance(x, DataArray) else x for x in inputs]
    result = getattr(ufunc, method)(*raw, **kw)
    if method == "__call__" and np.shape(result) == self.data.shape:
      return self._new(result)
    return result

  def __getitem__(self, index):                    # positional, first dim (coordinates)
    if isinstance(index, slice):
      return self._new(self.data[index])
    return DataArray(self.data[index], dims=self.dims[1:], name=self.name)

  def __setitem__(self, index, value):
    self.data = np.array(self.data)
    self.data[index] = value

  def astype(self, dtype):
    return self._new(self.data.astype(dtype))

  def notnull(self):
    return self._new(~np.isnan(self.data))

  def where(self, cond, other):
    return self._new(np.where(cond.data if isinstance(cond, DataArray) else cond, self.data, other))

  def _reduce(self, fn, dim=None, skipna=None):
    assert skipna is False
    dims = self.dims if dim is None else ((dim,) if isinstance(dim, str) else tuple(dim))
    kept = tuple(d for d in self.dims if d not in dims)
    out = fn(self.data, axis=tuple(self.dims.index(d) for d in dims))
    return DataArray(np.asarray(out), coords={k: c for k, c in self.coords.items() if k in kept},
                     dims=kept, name=self.name)

  def mean(self, dim=None, skipna=None):
    return self._reduce(np.mean, dim, skipna)

  def sum(self, dim=None, skipna=None):
    return self._reduce(np.sum, dim, skipna)

  def rename(self, name):
    out = self._new(self.data)
    out.name = name
    return out

  def transpose(self, *dims):
    if Ellipsis in dims:
      i = dims.index(Ellipsis)
      rest = [d for d in self.dims if d not in dims]
      dims = tuple(dims[:i]) + tuple(rest) + tuple(dims[i + 1:])
    return self._new(np.transpose(self.data, [self.dims.index(d) for d in dims]), tuple(dims))

  def isel(self, indexers=None, drop=False, **kw):
    indexers = dict(indexers or {}, **kw)
    data, dims = self.data, list(self.dims)
    for d, sel in indexers.items():
      if d not in dims:
        continue
      ax = dims.index(d)
      data = data[(slice(None),) * ax + (sel,)]
      if not isinstance(sel, slice):
        dims.pop(ax)
    coords = {k: c for k, c in self.coords.items() if k not in indexers}
    return DataArray(data, coords=coords, dims=dims, name=self.name)


class Dataset(dict):

  def __init__(self, data_vars=None, coords=None):
    super().__init__(data_vars or {})
    self.coords = dict(coords or {})

  def __getitem__(self, key):
    if isinstance(key, list):
      return Dataset({k: dict.__getitem__(self, k) for k in key}, self.coords)
    v = dict.__getitem__(self, key)
    coords = {k: c for k, c in self.coords.items() if all(d in v.dims for d in c.dims)}
    coords.update(v.coords)
    return DataArray(v.data, coords=coords, dims=v.dims, name=key)

  @property
  def data_vars(self):
    return self

  @property
  def sizes(self):
    out = {}
    for v in self.values():
      out.update(v.sizes)
    return out

  @property
  def dims(self):
    return self.sizes

  def _map(self, fn, coords=None):
    return Dataset({k: fn(self[k]) for k in self.keys()}, self.coords if coords is None else coords)

  def copy(self):
    return Dataset(dict(self), dict(self.coords))

  def isel(self, drop=False, **kw):
    coords = {k: (c.isel(**{d: s for d, s in kw.items() if d in c.dims}) if any(d in c.dims for d in kw) else c)
              for k, c in self.coords.items()}
    coords = {k: c for k, c in coords.items() if c.dims or not drop}
    return self._map(lambda v: v.isel(**kw), coords)

  def transpose(self, *dims):
    return self._map(lambda v: v.transpose(*dims))

  def expand_dims(self, axis=0, **kw):
    (dim, coord), = kw.items()
    n = len(coord.data)
    coords = dict(self.coords)
    coords[dim] = coord

    def one(v):
      return DataArray(np.repeat(np.expand_dims(v.data, axis), n, axis), coords=v.coords,
                       dims=v.dims[:axis] + (dim,) + v.dims[axis:], name=v.name)
    return self._map(one, coords)

  def drop_vars(self, names, errors="raise"):
    names = {names} if isinstance(names, str) else set(names)
    return Dataset({k: v for k, v in self.items() if k not in names},
                   {k: c for k, c in self.coords.items() if k not in names})

  def assign_coords(self, coords=None, **kw):
    new = dict(self.coords)
    for k, v in dict(coords or {}, **kw).items():
      new[k] = v if isinstance(v, DataArray) else DataArray(np.asarray(v), dims=(k,), name=k)
    return Dataset(dict(self), new)

  def tail(self, **kw):
    (dim, n), = kw.items()
    return self.isel(**{dim: slice(-n, None)})


def merge(objects, join=None, compat=None):
  data, coords = {}, {}
  for o in objects:
    if isinstance(o, Dataset):
      data.update(o)
      coords.update(o.coords)
    else:
      data[o.name] = o
      coords.update(o.coords)
  return Dataset(data, coords)


def concat(objs, dim, join=None, **kw):
  objs = list(objs)
  if not isinstance(objs[0], Dataset):                     # DataArrays along a new dim
    return DataArray(np.stack([o.data for o in objs]), dims=(dim,) + objs[0].dims)
  first = objs[0]
  out = {}
  for k, v in first.items():
    if dim in v.dims:
      parts = [ds[k].transpose(*v.dims).data for ds in objs]
      out[k] = DataArray(np.concatenate(parts, axis=v.dims.index(dim)), coords=v.coords, dims=v.dims, name=k)
    else:
      out[k] = v
  coords = dict(first.coords)
  if dim in coords:
    coords[dim] = DataArray(np.concatenate([ds.coords[dim].data for ds in objs]), dims=(dim,), name=dim)
  return Dataset(out, coords)


# ---- install the stand-ins, then import the reference modules -----------------------------------
ns.install()
xr_mod, xj_mod = sys.modules["xarray"], sys.modules["xarray_jax"]
xr_mod.Dataset, xr_mod.DataArray, xr_mod.merge, xr_mod.concat = Dataset, DataArray, merge, concat
xj_mod.unwrap_data = lambda v: v.data
xj_mod.DataArray = lambda data, dims: DataArray(np.asarray(data), dims=dims)
sys.modules["absl.logging"].info = lambda *a, **k: None
sys.modules["absl.logging"].warning = lambda *a, **k: None
sys.modules["absl"].logging = sys.modules["absl.logging"]


def _tree_flatten(tree):
  """xarray_jax: a dataset flattens into its arrays (sorted names); dims / coords are the treedef."""
  if isinstance(tree, Dataset):
    keys = sorted(tree.keys())
    return [tree[k].data for k in keys], ("dataset", keys, [tree[k].dims for k in keys],
                                          [dict(tree[k].coords) for k in keys], dict(tree.coords))
  return ns.tree_flatten(tree)


def _tree_unflatten(treedef, leaves):
  if isinstance(treedef, tuple) and treedef and treedef[0] == "dataset":
    _, keys, dims, vcoords, coords = treedef
    return Dataset({k: DataArray(np.asarray(x), coords=c, dims=d, name=k)
                    for k, x, d, c in zip(keys, leaves, dims, vcoords)}, dict(coords))
  return ns.tree_unflatten(treedef, leaves)


def _tree_map(f, tree, *rest):
  leaves, treedef = _tree_flatten(tree)
  others = [_tree_flatten(r)[0] for r in rest]
  return _tree_unflatten(treedef, [f(*x) for x in zip(leaves, *others)])


for _m in (sys.modules["jax.tree_util"], sys.modules["jax.tree"]):
  _m.tree_flatten = _m.flatten = _tree_flatten
  _m.tree_unflatten = _m.unflatten = _tree_unflatten
  _m.tree_leaves = _m.leaves = lambda t: _tree_flatten(t)[0]
  _m.tree_map = _m.map = _tree_map


def _scan(f, init, xs_):
  """hk.scan: carry through f, per-step outputs stacked on a new leading axis."""
  leaves, treedef = _tree_flatten(xs_)
  carry, outs = init, []
  for t in range(leaves[0].shape[0]):
    carry, out = f(carry, _tree_unflatten(treedef, [x[t] for x in leaves]))
    outs.append(out)
  stacked, out_def = _tree_flatten(outs[0])
  per_step = [_tree_flatten(o)[0] for o in outs]
  return carry, _tree_unflatten(out_def, [np.stack([s[i] for s in per_step]) for i in range(len(stacked))])


sys.modules["haiku"].scan = _scan
ref_losses = importlib.import_module("weathernext.utils.losses")
ref_norm = importlib.import_module("weathernext.utils.normalization")
ref_ar = importlib.import_module("weathernext.utils.autoregressive")
ref_gc = importlib.import_module("weathernext.weathernext1_graph.graphcast")

# ---- the cases ----------------------------------------------------------------------------------
rngl = np.random.default_rng(77)
mkl = lambda *s: rngl.standard_normal(s).astype(np.float32)
LB, LLON = 2, 8
HOUR = np.timedelta64(6, "h")
l_levels = np.array([50, 500, 850])
grids = {"poles": np.linspace(-90, 90, 7).astype(np.float32), "nopoles": np.arange(-75.0, 90.0, 30.0)}
S2 = ("batch", "time", "lat", "lon")
S3 = ("batch", "time", "level", "lat", "lon")
lo = {"levels": l_levels}


def _ds(spec, lat, times=None):
  coords = {"lat": lat, "lon": np.arange(LLON) * 45.0, "level": l_levels}
  if times is not None:
    coords["time"] = np.asarray(times) * HOUR
  data = {k: DataArray(v, coords={c: coords[c] for c in d if c in coords}, dims=d, name=k)
          for k, (d, v) in spec.items()}
  return Dataset(data, {k: DataArray(np.asarray(v), dims=(k,), name=k) for k, v in coords.items()})


def _store(prefix, spec):
  for k, (d, v) in spec.items():
    lo[f"{prefix}:{k}"], lo[f"{prefix}_dims:{k}"] = v, np.array(d)


def _store_loss(prefix, loss_and_diag):
  total, per_var = loss_and_diag
  lo[f"{prefix}:total"] = np.asarray(total.data)
  for k, v in per_var.items():
    lo[f"{prefix}:var:{k}"] = np.asarray(v.data if hasattr(v, "data") else v)


def _raises(fn):
  try:
    fn()
  except ValueError:
    return np.bool_(True)
  return np.bool_(False)


# losses.py on a grid with and one without pole rows, with and without `level`, batch 2, one NaN target
for gname, glat in grids.items():
  nl = len(glat)
  pred_spec = {"2m_temperature": (S2, mkl(LB, 1, nl, LLON)), "geopotential": (S3, mkl(LB, 1, 3, nl, LLON)),
               "total_precipitation_6hr": (S2, mkl(LB, 1, nl, LLON))}
  tgt_spec = {k: (d, mkl(*v.shape)) for k, (d, v) in pred_spec.items()}
  tgt_spec["total_precipitation_6hr"][1][1, 0, 2, 3] = np.nan            # batch element 1 only
  lo[f"{gname}:lat"] = glat
  _store(f"{gname}:pred", pred_spec)
  _store(f"{gname}:tgt", tgt_spec)
  p_ds, t_ds = _ds(pred_spec, glat), _ds(tgt_spec, glat)
  w = {"2m_temperature": 1.0, "total_precipitation_6hr": 0.1}
  _store_loss(f"{gname}:mse", ref_losses.weighted_mse_per_level(p_ds, t_ds, per_variable_weights=w))
  _store_loss(f"{gname}:mae", ref_losses.weighted_mae_per_level(p_ds, t_ds))
  _store_loss(f"{gname}:mse_nan", ref_losses.weighted_mse_per_level(
      p_ds, t_ds, per_variable_weights=w, vars_with_nan_targets=("total_precipitation_6hr",),
      loss_for_nan_targets=0.5))
  lo[f"{gname}:lat_weights"] = np.asarray(ref_losses.normalized_latitude_weights(t_ds["geopotential"]).data)
  lo[f"{gname}:level_weights"] = np.asarray(ref_losses.normalized_level_weights(t_ds["geopotential"]).data)
bad_lats = {"nonuniform": np.array([-90.0, -60.0, 0.0, 60.0, 90.0]),
            "no_pole_wrong_ends": np.array([-80.0, -40.0, 0.0, 40.0, 80.0]),
            "one_pole": np.array([-90.0, -45.0, 0.0, 45.0])}
for bname, blat in bad_lats.items():
  da = DataArray(np.zeros(len(blat), np.float32), coords={"lat": blat}, dims=("lat",), name="x")
  lo[f"bad_lat:{bname}"] = blat
  lo[f"bad_lat_raises:{bname}"] = _raises(lambda: ref_losses.normalized_latitude_weights(da))
lo["unknown_weight_raises"] = _raises(lambda: ref_losses.sum_per_variable_losses(
    Dataset({"a": DataArray(np.ones(2), dims=("batch",), name="a")}), {"b": 1.0}))

# GraphCast.loss_and_predictions / loss, unbound, on a stand-in whose __call__ returns fixed predictions
glat = grids["poles"]
nl = len(glat)
gc_vars = {"2m_temperature": S2, "10m_u_component_of_wind": S2, "10m_v_component_of_wind": S2,
           "mean_sea_level_pressure": S2, "total_precipitation_6hr": S2, "geopotential": S3}
shape_of = lambda d: tuple({"batch": LB, "time": 1, "level": 3, "lat": nl, "lon": LLON}[x] for x in d)
gc_pred = {k: (d, mkl(*shape_of(d))) for k, d in gc_vars.items()}
gc_tgt = {k: (d, mkl(*shape_of(d))) for k, d in gc_vars.items()}


class FixedGraphCast:

  def __call__(self, inputs, targets_template, forcings, is_training=False):
    assert is_training
    return _ds({k: v for k, v in gc_pred.items() if k in targets_template}, glat)

  loss_and_predictions = ref_gc.GraphCast.loss_and_predictions
  loss = ref_gc.GraphCast.loss


(gc_loss, gc_diag), _ = FixedGraphCast().loss_and_predictions(None, _ds(gc_tgt, glat), None)
_store("gc:pred", gc_pred)
_store("gc:tgt", gc_tgt)
_store_loss("gc", (gc_loss, gc_diag))
_store_loss("gc_loss", FixedGraphCast().loss(None, _ds(gc_tgt, glat), None))
lo["gc:missing_weighted_var_raises"] = _raises(lambda: FixedGraphCast().loss(
    None, _ds({k: v for k, v in gc_tgt.items() if k != "mean_sea_level_pressure"}, glat), None))

# InputsAndResiduals.loss / loss_and_predictions around a recording predictor (normalised space)
iar_in = {"2m_temperature": (S2, mkl(LB, 2, nl, LLON)), "geopotential": (S3, mkl(LB, 2, 3, nl, LLON)),
          "toa_incident_solar_radiation": (S2, mkl(LB, 2, nl, LLON))}
iar_forcing = {"toa_incident_solar_radiation": (S2, mkl(LB, 1, nl, LLON))}
iar_tgt = {"2m_temperature": (S2, mkl(LB, 1, nl, LLON)), "geopotential": (S3, mkl(LB, 1, 3, nl, LLON)),
           "total_precipitation_6hr": (S2, mkl(LB, 1, nl, LLON))}
iar_stats = lambda fn: Dataset({
    "2m_temperature": DataArray(np.float32(fn(0)), dims=(), name="2m_temperature"),
    "geopotential": DataArray(np.array([fn(1), fn(2), fn(5)], np.float32), dims=("level",), name="geopotential"),
    "toa_incident_solar_radiation": DataArray(np.float32(fn(3)), dims=(), name="toa_incident_solar_radiation"),
    "total_precipitation_6hr": DataArray(np.float32(fn(4)), dims=(), name="total_precipitation_6hr")})
iar_mean, iar_std = iar_stats(lambda i: 1.5 * i - 2.0), iar_stats(lambda i: 0.5 + 0.75 * i)
iar_dstd = iar_stats(lambda i: 0.1 + 0.05 * i)
iar_seen = []


class RecordingLossPredictor:
  """Prediction = a fixed function of the normalised inputs; loss = the reference MSE against the
  (normalised) targets it is given, which it records."""

  def loss_and_predictions(self, inputs, targets, forcings):
    iar_seen.append({k: np.asarray(targets[k].data) for k in targets.keys()})
    out = {}
    for name in sorted(targets.keys()):
      t = targets[name]
      if name in inputs:
        x = inputs[name]                                   # (batch, time, [level], lat, lon)
        out[name] = DataArray(0.5 * x.data[:, -1:] + 0.25, coords=t.coords, dims=x.dims, name=name)
      else:
        out[name] = DataArray(np.full(t.data.shape, 0.125, np.float32), coords=t.coords, dims=t.dims, name=name)
    pred = Dataset(out, dict(targets.coords))
    return ref_losses.weighted_mse_per_level(pred, targets), pred

  def loss(self, inputs, targets, forcings):
    return self.loss_and_predictions(inputs, targets, forcings)[0]


iar = ref_norm.InputsAndResiduals(RecordingLossPredictor(), stddev_by_level=iar_std, mean_by_level=iar_mean,
                                  diffs_stddev_by_level=iar_dstd)
_store_loss("iar_loss", iar.loss(_ds(iar_in, glat), _ds(iar_tgt, glat, [1]), _ds(iar_forcing, glat, [1])))
(iar_l, iar_d), iar_pred = iar.loss_and_predictions(_ds(iar_in, glat), _ds(iar_tgt, glat, [1]),
                                                    _ds(iar_forcing, glat, [1]))
_store_loss("iar", (iar_l, iar_d))
for k in iar_tgt:
  lo[f"iar:norm_target:{k}"] = iar_seen[-1][k]
  lo[f"iar:pred:{k}"] = np.asarray(iar_pred[k].transpose(*iar_tgt[k][0]).data)
_store("iar:in", iar_in)
_store("iar:forcing", iar_forcing)
_store("iar:tgt", iar_tgt)
for sname, sds in (("mean", iar_mean), ("std", iar_std), ("diffs_std", iar_dstd)):
  for k in sds.keys():
    lo[f"iar:{sname}:{k}"] = np.asarray(sds[k].data)

# autoregressive.Predictor.loss for T = 3 (scan over loss_and_predictions, feedback) and T = 1
AT = 3
ar_in = {"2m_temperature": (S2, mkl(LB, 2, nl, LLON)), "geopotential": (S3, mkl(LB, 2, 3, nl, LLON)),
         "land_sea_mask": (("lat", "lon"), mkl(nl, LLON))}
ar_forcing = {"toa_incident_solar_radiation": (S2, mkl(LB, AT, nl, LLON))}
ar_tgt = {"2m_temperature": (S2, mkl(LB, AT, nl, LLON)), "geopotential": (S3, mkl(LB, AT, 3, nl, LLON))}


class FeedbackLossPredictor:
  """Depends on both input frames, the step's forcing and a constant input, so that the fed-back
  predictions and the forcing slices show in the loss."""

  def loss_and_predictions(self, inputs, targets, forcings):
    # the scan hands over targets / forcings with `time` leading (expand_dims(axis=0)): index by name
    f = forcings["toa_incident_solar_radiation"].transpose("batch", "time", "lat", "lon").data
    out = {}
    for name in sorted(targets.keys()):
      x = inputs[name]                                     # (batch, time, [level], lat, lon)
      fb = f.reshape(f.shape[:2] + (1,) * (x.data.ndim - 4) + f.shape[2:])
      out[name] = DataArray(0.9 * x.data[:, 1:] + 0.1 * x.data[:, :1] + 0.05 * fb
                            + 0.01 * inputs["land_sea_mask"].data,
                            coords=targets[name].coords, dims=x.dims, name=name)
    pred = Dataset(out, dict(targets.coords))
    return ref_losses.weighted_mse_per_level(pred, targets, per_variable_weights={"2m_temperature": 0.5}), pred

  def loss(self, inputs, targets, forcings):
    return self.loss_and_predictions(inputs, targets, forcings)[0]


ar = ref_ar.Predictor(FeedbackLossPredictor())
ar_inputs = _ds(ar_in, glat, [-1, 0])
_store_loss("ar3", ar.loss(ar_inputs, _ds(ar_tgt, glat, [1, 2, 3]), _ds(ar_forcing, glat, [1, 2, 3])))
one = lambda spec: {k: (d, v[:, :1]) for k, (d, v) in spec.items()}
_store_loss("ar1", ar.loss(ar_inputs, _ds(one(ar_tgt), glat, [1]), _ds(one(ar_forcing), glat, [1])))
_store("ar:in", ar_in)
_store("ar:forcing", ar_forcing)
_store("ar:tgt", ar_tgt)
np.savez_compressed(os.path.join(here, "reference_losses.npz"), **lo)
print("wrote", os.path.join(here, "reference_losses.npz"),
      {k: np.asarray(v).round(5).tolist() for k, v in lo.items() if k.endswith(":total")})
