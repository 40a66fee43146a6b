"""Parameter gradients at the production shapes, tensor by tensor.

At 0.25 deg and 1 deg there is no affordable autograd reference, so every live parameter tensor t is
checked by a central difference of the device loss along its own gradient, u_t = g_t / |g_t|, with
the weights reloaded in place (Engine.load_params) for each evaluation.  A single check along the
whole gradient g / |g| cannot see a zeroed tensor at all, nor a sign-flipped tensor that holds a few
per cent of |g|^2; the sensitivity test below plants such errors and shows both verdicts.

Only bf16x3: the bf16 forward is not smooth in the weights, so finite differences mean nothing there.
"""
import gc
import time
import weakref

import numpy as np
import pytest
import torch

import _cases
from graphcast_b200 import (autoregressive, engine, graph as graph_lib, graphcast, losses, model_utils,
                            normalization, synthetic)
from graphcast_b200 import xarray_shim as xs
from oracle import gnn as oracle_gnn
from test_gpu_loss import _lat_weight, _model_and_data, _stats

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
DEAD = "mesh2grid_gnn/~_networks_builder/processor_nodes_0_mesh_nodes"   # never read by the step
GATE = 1e-2             # per tensor: a sign flip moves the check by 2, a dropped chunk of six by ~0.17
REL_CHANGE = 1e-4       # eps_t |g_t| = REL_CHANGE * loss


# ---- Engine.load_params --------------------------------------------------------------------------
def _small_problem():
  g, p1, x = _cases.small_case(c_in=31, n_out=23, msg_steps=3)
  _, p2, _ = _cases.small_case(c_in=31, n_out=23, msg_steps=3, seed=1)
  rng = np.random.default_rng(3)
  planes = torch.as_tensor(x[:, 0, :].T.copy()).to(DEV)
  targets = torch.as_tensor(rng.standard_normal((23, g.num_grid_nodes)).astype(np.float32)).to(DEV)
  lat_w = torch.as_tensor(_lat_weight(np.linspace(-90, 90, len(g.grid_lat)))).to(DEV)
  coef = torch.as_tensor(rng.uniform(0.5, 2.0, 23) / (23 * g.num_grid_nodes)).to(DEV)
  return g, p1, p2, planes, targets, lat_w, coef


def _outputs(eng, planes, targets, lat_w, coef):
  """Everything the engine computes from its weights, as device tensors (of the decoder output, the
  n_out valid columns: the step never writes the padding)."""
  eng.pack_inputs(planes)
  steps = [eng.step()[:, :23].clone() for _ in range(3)]   # eager, captured, replayed
  sums = torch.empty(23, dtype=torch.float64, device=DEV)
  eng.output_loss(targets, lat_w, channel_sums=sums)
  eng.grads_begin()
  grad_sums = torch.empty(23, dtype=torch.float64, device=DEV)
  eng.loss_and_grads_element(targets, lat_w, coef, channel_sums=grad_sums)
  grads = [t.clone() for _, v in sorted(eng.grads().items()) for _, t in sorted(v.items())]
  w0_in = eng._backward.input_transposed()[0].clone()      # the input transpose of backprop in time
  eng.set_precision("fp32_simt")                           # reads the fp32 weight copies
  simt = eng.step()[:, :23].clone()
  eng.set_precision("bf16x3")
  return steps + [sums, grad_sums] + grads + [w0_in, simt]


def _equal(a, b):
  return len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


def test_load_params_matches_a_fresh_engine():
  g, p1, p2, planes, targets, lat_w, coef = _small_problem()
  args = (planes, targets, lat_w, coef)
  eng = engine.Engine(g, p1, c_in=31, n_out=23, msg_steps=3, precision="bf16x3")
  first = _outputs(eng, *args)
  assert torch.equal(first[0], first[1]) and torch.equal(first[0], first[2])
  eng.load_params(p2)                 # the step graph recorded with p1's buffers is replayed
  reloaded = _outputs(eng, *args)
  fresh = engine.Engine(g, p2, c_in=31, n_out=23, msg_steps=3, precision="bf16x3")
  want = _outputs(fresh, *args)
  del fresh
  assert not torch.equal(reloaded[0], first[0])
  assert _equal(reloaded, want)
  eng.load_params(p1)
  assert _equal(_outputs(eng, *args), first)
  # in place: ten reloads allocate nothing
  torch.cuda.synchronize()
  before = torch.cuda.memory_allocated()
  for i in range(10):
    eng.load_params(p2 if i % 2 == 0 else p1)
  torch.cuda.synchronize()
  assert torch.cuda.memory_allocated() == before
  # a shape mismatch or a missing tensor raises before anything is written
  name = "mesh_gnn/~_networks_builder/processor_edges_1_mesh_mlp/~/linear_0"
  bad = {k: dict(v) for k, v in p2.items()}
  bad[name]["w"] = np.asarray(bad[name]["w"])[:-1]
  with pytest.raises(ValueError, match="shape"):
    eng.load_params(bad)
  missing = {k: v for k, v in p2.items() if k != name}
  with pytest.raises(ValueError, match="missing"):
    eng.load_params(missing)
  eng.pack_inputs(planes)
  assert torch.equal(eng.step()[:, :23], first[0])


def test_dropped_engine_frees_its_memory_at_once():
  """Callers free an engine's workspace with `del`: neither the reload machinery nor the gradient
  workspace may put the engine in a reference cycle that only the garbage collector would break."""
  g, p1, p2, planes, targets, lat_w, coef = _small_problem()
  gc.collect()
  torch.cuda.synchronize()
  before = torch.cuda.memory_allocated()
  gc.disable()
  try:
    for with_grads in (False, True):
      eng = engine.Engine(g, p1, c_in=31, n_out=23, msg_steps=3, precision="bf16x3")
      eng.load_params(p2)
      if with_grads:
        _outputs(eng, planes, targets, lat_w, coef)
        eng.load_params(p1)
      ref = weakref.ref(eng)
      del eng
      assert ref() is None, with_grads
      torch.cuda.synchronize()
      assert torch.cuda.memory_allocated() == before, with_grads
  finally:
    gc.enable()


def test_graphcast_set_params_reloads_the_engine():
  task, model, inputs, targets, forcings = _model_and_data(batch=1)
  model.loss(inputs, targets, forcings)
  eng = model.engine
  c_in = synthetic.num_input_channels(task)
  p2 = oracle_gnn.init_params(c_in=c_in, n_out=83, msg_steps=2, seed=9, randomize_affine=True)
  model.set_params(p2)
  assert model.engine is eng
  fresh = graphcast.GraphCast(graphcast.ModelConfig(10.0, 2, 512, 2, 1, 0.6), task, params=p2)
  assert np.array_equal(model.loss(inputs, targets, forcings)[0].values,
                        fresh.loss(inputs, targets, forcings)[0].values)
  other = oracle_gnn.init_params(c_in=c_in, n_out=83, msg_steps=1, seed=9)
  model.set_params(other)                       # other shapes: the engine is rebuilt on the next call
  assert model._engine is None


# ---- the per-tensor check ------------------------------------------------------------------------
def _live(params):
  return [(n, f) for n in sorted(params) for f in sorted(params[n]) if not n.startswith(DEAD)]


def _with(params, group, arrays):
  """params with the (module, field) tensors of `group` replaced by `arrays`."""
  out = dict(params)
  for n in {n for n, _ in group}:
    out[n] = dict(params[n])
  for (n, f), a in zip(group, arrays):
    out[n][f] = a
  return out


def _directional(loss_at, params, grads, loss0, group):
  """Central differences of loss_at along u = g_group / |g_group| with steps eps and eps / 2, where
  eps |g_group| = REL_CHANGE * loss0.  Each is divided by the change <g, theta+ - theta-> / 2 that the
  gradient predicts for the fp32 weights actually evaluated, which removes their rounding.  Returns
  (ratio at eps, ratio at eps / 2, |Richardson extrapolation of the ratio - 1|)."""
  g = [np.asarray(grads[n][f], np.float64) for n, f in group]
  gn = np.sqrt(sum(float((a * a).sum()) for a in g))
  if gn == 0:                                   # a live tensor without a gradient: no direction
    return float("nan"), float("nan"), float("inf")
  eps = REL_CHANGE * abs(loss0) / gn
  theta = [np.asarray(params[n][f], np.float64) for n, f in group]
  ratios = []
  for e in (eps, eps / 2):
    plus = [(t + e * a / gn).astype(np.float32) for t, a in zip(theta, g)]
    minus = [(t - e * a / gn).astype(np.float32) for t, a in zip(theta, g)]
    diff = loss_at(_with(params, group, plus)) - loss_at(_with(params, group, minus))
    pred = sum(float((a * (p.astype(np.float64) - m.astype(np.float64))).sum())
               for a, p, m in zip(g, plus, minus))
    ratios.append(diff / pred)
  return ratios[0], ratios[1], abs((4 * ratios[1] - ratios[0]) / 3 - 1)


def _whole_vector(loss_at, params, grads, loss0):
  """The check the per-tensor one replaces: the central difference along g / |g| against |g|."""
  keys = [(n, f) for n in params for f in params[n]]
  gn = np.sqrt(sum(float((np.asarray(grads[n][f], np.float64) ** 2).sum()) for n, f in keys))
  eps = 1e-2 * loss0 / gn
  shifted = [loss_at({n: {f: (np.asarray(a, np.float64) + s * eps * np.asarray(grads[n][f], np.float64)
                              / gn).astype(np.float32) for f, a in v.items()} for n, v in params.items()})
             for s in (1.0, -1.0)]
  fd = (shifted[0] - shifted[1]) / (2 * eps)
  return fd, gn, abs(fd - gn) / gn


def _per_tensor(loss_at, params, grads, loss0, joint, tag):
  """The check over every live tensor; the MLPs whose stem is in `joint` are checked as one group.
  Prints one row per group and returns {label: Richardson error}."""
  for n in params:
    if n.startswith(DEAD):
      for f in params[n]:
        assert not np.any(grads[n][f]), (n, f)
  groups = {}
  for n, f in _live(params):
    stem = next((s for s in joint if n.startswith(s)), None)
    groups.setdefault(stem or f"{n}:{f}", []).append((n, f))
  assert sum(len(v) for v in groups.values()) == len(_live(params))
  total = sum(float((np.asarray(grads[n][f], np.float64) ** 2).sum()) for n, f in _live(params))
  out, spread = {}, []
  t0 = time.time()
  print(f"\n{tag}: {len(groups)} groups of {len(_live(params))} tensors; columns: share of |g|^2, "
        f"FD(eps) / predicted, FD(eps/2) / predicted, Richardson |error|")
  for label, group in groups.items():
    share = sum(float((np.asarray(grads[n][f], np.float64) ** 2).sum()) for n, f in group) / total
    r1, r2, err = _directional(loss_at, params, grads, loss0, group)
    out[label] = err
    spread.append(abs(r1 - r2))
    print(f"  {label:<90s} {share:9.3e} {r1:.8f} {r2:.8f} {err:9.3e}")
  worst = max(out.items(), key=lambda kv: kv[1])
  print(f"{tag}: worst {worst[1]:.3g} at {worst[0]}; |FD(eps) - FD(eps/2)| / predicted: median "
        f"{np.median(spread):.3g}, max {np.max(spread):.3g}; {4 * len(groups)} loss evaluations in "
        f"{time.time() - t0:.1f} s")
  return out


# ---- engine-level problems at 1 deg and 0.25 deg ---------------------------------------------------
def _engine_problem(task, resolution, mesh_size):
  lat, lon = synthetic.grid_coords(resolution)
  g = graph_lib.cached_static_graph(grid_lat=lat, grid_lon=lon, mesh_size=mesh_size,
                                    radius_query_fraction_edge_length=0.6)
  c_in, n_out = synthetic.num_input_channels(task), graphcast.num_outputs(task)
  params = graphcast.init_params(graphcast.ModelConfig(resolution, mesh_size, 512, 16, 1, 0.6), task,
                                 c_in, seed=1)
  gen = torch.Generator(device=DEV).manual_seed(0)
  planes = torch.randn(c_in, g.num_grid_nodes, device=DEV, generator=gen)
  targets = torch.randn(n_out, g.num_grid_nodes, device=DEV, generator=gen)
  lat_w = torch.as_tensor(_lat_weight(lat)).to(DEV)
  kappa = np.random.default_rng(1).uniform(0.5, 2.0, n_out) / (n_out * g.num_grid_nodes)
  eng = engine.Engine(g, params, c_in=c_in, n_out=n_out, msg_steps=16, precision="bf16x3")
  return eng, params, planes, targets, lat_w, torch.as_tensor(kappa).to(DEV)


class _EngineLoss:
  """The device loss sum_c kappa_c sum_node w (y - t)^2 of one step at the given weights."""

  def __init__(self, eng, planes, targets, lat_w, kappa):
    self.eng, self.planes, self.targets, self.lat_w, self.kappa = eng, planes, targets, lat_w, kappa
    self.sums = torch.empty(eng.n_out, dtype=torch.float64, device=DEV)

  def __call__(self, params):
    self.eng.load_params(params)
    self.eng.pack_inputs(self.planes)
    self.eng.step()
    self.eng.output_loss(self.targets, self.lat_w, channel_sums=self.sums)
    return float((self.sums * self.kappa).sum())

  def gradient(self):
    """(loss, host fp64 gradients) from the stage-wise forward and the backward pass."""
    eng = self.eng
    eng.grads_begin()
    eng.pack_inputs(self.planes)
    eng.loss_and_grads_element(self.targets, self.lat_w, 2 * self.kappa, channel_sums=self.sums)
    grads = {k: {f: t.double().cpu().numpy() for f, t in v.items()} for k, v in eng.grads().items()}
    return float((self.sums * self.kappa).sum()), grads


def _gpu():
  return (f"{torch.cuda.get_device_name(0)}, "
          f"{torch.cuda.get_device_properties(0).total_memory / 2**30:.0f} GiB")


# Groups checked together, each with the measured reason (empty: every tensor meets the gate alone).
_JOINT_FULL_SIZE = {}
_JOINT_BPTT = {}


def test_full_size_per_tensor_directional_derivatives_and_peak_memory():
  """0.25 deg / 37 levels, one step: every live tensor's gradient against central differences of the
  device loss; the peak device memory of the gradient is reported."""
  if torch.cuda.get_device_properties(0).total_memory < 75e9:
    pytest.skip("needs an 80 GB GPU")
  gc.collect()                                  # the gradient peaks within a few GiB of 80 GB
  torch.cuda.empty_cache()
  eng, params, *data = _engine_problem(graphcast.TASK, 0.25, 6)
  loss_at = _EngineLoss(eng, *data)
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  t0 = time.time()
  loss0, grads = loss_at.gradient()
  torch.cuda.synchronize()
  peak = torch.cuda.max_memory_allocated()
  print(f"\n0.25 deg gradient: {time.time() - t0:.2f} s, peak device memory {peak / 2**30:.1f} GiB "
        f"on {_gpu()}")
  eng._backward = None                          # the gradient workspace is not needed any more
  torch.cuda.empty_cache()
  base = loss_at(params)
  fd, gn, rel = _whole_vector(loss_at, params, grads, loss0)
  print(f"0.25 deg whole vector: loss {loss0:.9g}, |g| {gn:.6g}, central difference {fd:.6g} "
        f"(relative {rel:.3g})")
  errs = _per_tensor(loss_at, params, grads, loss0, _JOINT_FULL_SIZE, "0.25 deg, one step")
  assert loss_at(params) == base                # the reloads restore the weights bit for bit
  assert base == loss0                          # stage-wise forward == gcb_forward
  assert rel <= 1e-2
  bad = {k: v for k, v in errs.items() if not v <= GATE}
  assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])


def test_config1_bptt_per_tensor_directional_derivatives():
  """BASELINE config 1 (1 deg, mesh 5, 13 levels, 16 steps), backprop through four target times of
  autoregressive.Predictor(InputsAndResiduals(GraphCast)); each loss through set_params and loss."""
  task = graphcast.TASK_13
  inputs, template, forcings = synthetic.make_example(task, 1.0, batch=1, num_target_steps=4, seed=2)
  rng = np.random.default_rng(3)
  targets = xs.Dataset(coords=template.coords)
  for name, v in template.data_vars.items():
    targets[name] = xs.DataArray(rng.standard_normal(v.shape).astype(np.float32), v.dims)
  cfg = graphcast.ModelConfig(1.0, 5, 512, 16, 1, 0.6)
  params = graphcast.init_params(cfg, task, synthetic.num_input_channels(task), seed=1)
  model = graphcast.GraphCast(cfg, task, params=params)
  ar = autoregressive.Predictor(normalization.InputsAndResiduals(model, *_stats(task, seed=1)),
                                gradient_checkpointing=True)
  t0 = time.time()
  loss, _, grads = ar.loss_and_grads(inputs, targets, forcings)
  print(f"\n1 deg, T = 4 gradient: {time.time() - t0:.2f} s on {_gpu()}")
  eng = model.engine
  # `loss` returns float32, whose rounding (one ulp of this loss is 8.5e-4 of the difference at eps / 2)
  # would dominate the check: the same loss is taken in fp64 from the per-step device channel sums
  # that `loss` reduces, sum_c kappa_c sums_c averaged over the steps.
  kappa = torch.as_tensor(losses.channel_kappa(model_utils.channel_layout(targets.isel(time=slice(0, 1))),
                                               eng.num_grid, graphcast.LOSS_PER_VARIABLE_WEIGHTS)).to(DEV)
  step_sums, device_loss = [], model._device_loss

  def recording_device_loss(*args, **kwargs):
    finish, predictions, sums = device_loss(*args, **kwargs)
    step_sums.append(sums)
    return finish, predictions, sums
  model._device_loss = recording_device_loss

  def loss_at(p):
    model.set_params(p)
    step_sums.clear()
    api = float(np.asarray(ar.loss(inputs, targets, forcings)[0].values, np.float64)[0])
    assert len(step_sums) == 4
    exact = float(sum((s[0] * kappa).sum() for s in step_sums)) / 4
    assert abs(exact - api) <= 1e-6 * abs(exact)          # the float32 API value, unrounded
    return exact

  base = loss_at(params)
  loss0 = base
  assert abs(base - float(loss.values[0])) <= 1e-6 * base   # the loss of the gradient
  fd, gn, rel = _whole_vector(loss_at, params, grads, loss0)
  print(f"1 deg, T = 4 whole vector: loss {loss0:.9g}, |g| {gn:.6g}, central difference {fd:.6g} "
        f"(relative {rel:.3g})")
  errs = _per_tensor(loss_at, params, grads, loss0, _JOINT_BPTT, "1 deg, T = 4")
  assert model.engine is eng                    # reloaded in place, never rebuilt
  assert loss_at(params) == base
  assert rel <= 1e-2
  bad = {k: v for k, v in errs.items() if not v <= GATE}
  assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])


def test_per_tensor_check_flags_planted_errors():
  """1 deg, one step: errors planted in a host copy of the true gradient.  The per-tensor check flags
  each; the whole-vector check passes the sign flip of a small tensor and a zeroed tensor."""
  eng, params, *data = _engine_problem(graphcast.TASK_13, 1.0, 5)
  loss_at = _EngineLoss(eng, *data)
  loss0, grads = loss_at.gradient()
  eng._backward = None
  live = _live(params)
  sq = {k: float((grads[k[0]][k[1]] ** 2).sum()) for k in live}
  total = sum(sq.values())
  flip = max((k for k in live if sq[k] <= 4e-3 * total), key=sq.get)
  g2m = ("grid2mesh_gnn/~_networks_builder/processor_edges_0_grid2mesh_mlp/~/linear_0", "w")
  m2g = ("mesh2grid_gnn/~_networks_builder/processor_edges_0_mesh2grid_mlp/~/linear_0", "w")
  mesh = ("mesh_gnn/~_networks_builder/processor_edges_0_mesh_mlp/~/linear_0", "w")
  zero = max((k for k in live if k not in (flip, g2m, m2g)), key=sq.get)

  def swap(a):
    b = a.copy()
    b[512:1024], b[1024:1536] = a[1024:1536], a[512:1024]
    return b
  # (what, tensor, error, the old check passes it, the new check flags it)
  mutations = [("sign flip", flip, lambda a: -a, True, True),
               ("zeroed", zero, np.zeros_like, True, True),
               ("x0.8 (a dropped chunk)", g2m, lambda a: 0.8 * a, None, True),
               ("sender/receiver blocks swapped", m2g, swap, None, True),
               # Measured blind spot of any check along g_t: in the mesh processor the sender and
               # receiver blocks' gradients nearly coincide, so the error e of the swap has
               # <e, g_t> / |g_t|^2 = -3.6e-5, below the check's noise (it reads 1.8e-4).  The
               # small-case autograd comparison, element by element, is what catches it.
               ("swapped, mesh processor", mesh, swap, None, False)]
  print(f"\n1 deg planted errors (|g|^2 share of the tensor; old: central difference along g'/|g'| "
        f"against |g'|; new: per-tensor Richardson error, gate {GATE}; first order: <e, g_t> / |g_t|^2 "
        f"of the planted error e)")
  for what, key, fn, old_passes, flagged in mutations:
    _, _, control = _directional(loss_at, params, grads, loss0, [key])
    assert control <= GATE, (key, control)      # the true gradient of the same tensor passes
    bad = {n: dict(v) for n, v in grads.items()}
    g_t = grads[key[0]][key[1]]
    bad[key[0]][key[1]] = fn(g_t)
    first = float(((bad[key[0]][key[1]] - g_t) * g_t).sum()) / sq[key]
    _, _, old = _whole_vector(loss_at, params, bad, loss0)
    _, _, new = _directional(loss_at, params, bad, loss0, [key])
    print(f"  {what:<32s} {key[0]}:{key[1]} share {sq[key] / total:.3e}: old {old:.3g} "
          f"({'pass' if old <= 1e-2 else 'fail'}), new {new:.3g} "
          f"({'pass' if new <= GATE else 'flagged'}); first order {first:.3g}; true gradient {control:.3g}")
    assert (new > GATE) == flagged, what
    if old_passes:
      assert old <= 1e-2, what
