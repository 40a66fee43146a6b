"""The static-edge cache of the deep-chain step (Engine(static_cache=True), gcb_forward_static): the
step with the cache is bit for bit the step without it, stage by stage as well as whole; the cache
follows every weight write and change of precision; every derivative path releases it and computes
what an engine that never built one computes; and the table-accumulator chain layer it relies on is
bit for bit the chain that forms the same accumulator with MMAs."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

import _cases
from graphcast_b200 import _native, engine, graphcast, optim, synthetic
from graphcast_b200 import xarray_shim as xs
from test_gpu_chain import DEV, Layer, _fill_chain_layer, _image, _scratch, _seg_img, _stream

pytestmark = pytest.mark.gpu


def _engine(params, msg_steps, prec="bf16x3", **kw):
  g, _, _ = _cases.small_case(c_in=31, n_out=23, msg_steps=msg_steps)
  return engine.Engine(g, params, c_in=31, n_out=23, msg_steps=msg_steps, precision=prec, **kw)


def _planes(eng, seed):
  gen = torch.Generator(device=DEV).manual_seed(seed)
  return torch.randn(31, eng.num_grid, generator=gen, device=DEV)


def _step(eng, planes):
  eng.pack_inputs(planes)
  eng.step()
  torch.cuda.synchronize()
  return eng.grid_out[:, :23].clone()


# ---- engine: cache on == cache off ------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
@pytest.mark.parametrize("msg_steps", [1, 2, 4])
def test_cache_on_equals_cache_off_over_repeated_steps(prec, msg_steps):
  _, params, _ = _cases.small_case(c_in=31, n_out=23, msg_steps=msg_steps, seed=msg_steps)
  on, off = _engine(params, msg_steps, prec), _engine(params, msg_steps, prec, static_cache=False)
  for seed in range(4):                   # eager, captured and replayed steps
    planes = _planes(on, seed)
    assert torch.equal(_step(on, planes), _step(off, planes)), seed
  assert on.static_cache_builds == 1 and off.static_cache_builds == 0
  assert on.launches_per_step == off.launches_per_step
  assert on.workspace_bytes() - off.workspace_bytes() == sum(
      t.numel() * t.element_size() for t in on._static.values())
  assert on.static_cache_build_ms() > 0
  # stage by stage == whole step, with the cache and with the same launch count
  planes = _planes(on, 9)
  y = _step(on, planes)
  on.pack_inputs(planes)
  n = on.run_stage("encode") + on.run_stage("process_embed")
  for k in range(msg_steps):
    n += on.run_stage("process_step", k)
  n += on.run_stage("decode")
  torch.cuda.synchronize()
  assert n == on.launches_per_step
  assert torch.equal(on.grid_out[:, :23], y)
  assert on.static_cache_builds == 1


def test_cache_follows_weights_and_precision():
  msg_steps = 2
  _, pa, _ = _cases.small_case(c_in=31, n_out=23, msg_steps=msg_steps, seed=1)
  _, pb, _ = _cases.small_case(c_in=31, n_out=23, msg_steps=msg_steps, seed=2)
  eng = _engine(pa, msg_steps)
  planes = _planes(eng, 0)
  y_a = _step(eng, planes)
  fresh = lambda p, prec="bf16x3": _step(_engine(p, msg_steps, prec), planes)
  eng.load_params(pb)
  assert torch.equal(_step(eng, planes), fresh(pb))
  assert torch.equal(_step(eng, planes), fresh(pb))        # replayed graph, rebuilt tables
  dev_a = {k: {f: torch.as_tensor(np.asarray(a, np.float32)).to(DEV).contiguous() for f, a in v.items()}
           for k, v in pa.items()}
  eng.load_params_device(dev_a)
  assert torch.equal(_step(eng, planes), y_a)
  eng.set_precision("bf16")
  assert torch.equal(_step(eng, planes), fresh(pa, "bf16"))
  eng.set_precision("fp32_simt")                            # no deep chains: the cache is freed
  _step(eng, planes)
  assert eng._static is None
  eng.set_precision("bf16x3")
  assert torch.equal(_step(eng, planes), y_a)
  assert eng.static_cache_builds == 5


# ---- GraphCast: 13 and 37 levels, AdamW, and the derivative paths ---------------------------------
def _problem(task, msg_steps=2, seed=2):
  inputs, template, forcings = synthetic.make_example(task, 10.0, batch=1, num_target_steps=1, seed=seed)
  rng = np.random.default_rng(seed)
  targets = xs.Dataset(coords=template.coords)
  for name, v in template.data_vars.items():
    targets[name] = xs.DataArray(rng.standard_normal(v.shape).astype(np.float32), v.dims)
  cfg = graphcast.ModelConfig(10.0, 2, 512, msg_steps, 1, 0.6)
  params = graphcast.init_params(cfg, task, synthetic.num_input_channels(task), seed=1)
  return cfg, params, inputs, template, targets, forcings


def _tangent(ds, seed):
  rng = np.random.default_rng(seed)
  out = xs.Dataset(coords=ds.coords)
  name, v = next(iter(ds.data_vars.items()))
  out[name] = xs.DataArray(rng.standard_normal(v.shape).astype(np.float32), v.dims)
  return out


def _arrays(x):
  """Every array of a result (Datasets, DataArrays, parameter dicts, tuples) in a fixed order."""
  if isinstance(x, (tuple, list)):
    return [a for e in x for a in _arrays(e)]
  if isinstance(x, dict):
    return [a for k in sorted(x) for a in _arrays(x[k])]
  if hasattr(x, "data_vars"):
    return [np.asarray(x.data_vars[k].values) for k in sorted(x.data_vars)]
  if hasattr(x, "values"):
    return [np.asarray(x.values)]
  return [np.asarray(x)]


def _same(a, b):
  xa, xb = _arrays(a), _arrays(b)
  assert len(xa) == len(xb)
  for u, v in zip(xa, xb):
    assert u.shape == v.shape and np.array_equal(u, v, equal_nan=True)


@pytest.mark.parametrize("task", ["TASK_13", "TASK"])
@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
def test_graphcast_predictions_cache_on_equals_off(task, prec):
  cfg, params, inputs, template, _, forcings = _problem(getattr(graphcast, task), msg_steps=3)
  on = graphcast.GraphCast(cfg, getattr(graphcast, task), params=params, precision=prec)
  off = graphcast.GraphCast(cfg, getattr(graphcast, task), params=params, precision=prec,
                            static_cache=False)
  for _ in range(3):
    _same(on(inputs, template, forcings), off(inputs, template, forcings))
  assert on.engine._static is not None and off.engine._static is None


def test_adamw_step_rebuilds_the_cache():
  task = graphcast.TASK_13
  cfg, params, inputs, template, targets, forcings = _problem(task)
  model = graphcast.GraphCast(cfg, task, params=params)
  model(inputs, template, forcings)
  opt = optim.AdamW(model, learning_rate=1e-3)
  opt.step(inputs, targets, forcings)
  assert model.engine._static is None                       # released by the gradient
  fresh = graphcast.GraphCast(cfg, task, params=model.engine.params)
  want = fresh(inputs, template, forcings)
  _same(model(inputs, template, forcings), want)
  assert model.engine._static is None                       # not rebuilt next to the workspace
  model.engine.release_gradient_workspace()
  _same(model(inputs, template, forcings), want)            # rebuilt from the new weights
  assert model.engine._static is not None


@pytest.mark.parametrize("what", ["loss_and_grads", "loss_and_input_grads", "input_jvp",
                                  "loss_and_input_hvp"])
def test_derivatives_after_a_call_release_the_cache_and_match(what):
  task = graphcast.TASK_13
  cfg, params, inputs, template, targets, forcings = _problem(task)
  tangent = _tangent(inputs, 5)
  args = {"loss_and_grads": (inputs, targets, forcings),
          "loss_and_input_grads": (inputs, targets, forcings),
          "input_jvp": (inputs, template, forcings, tangent),
          "loss_and_input_hvp": (inputs, targets, forcings, tangent)}[what]
  called = graphcast.GraphCast(cfg, task, params=params)
  called(inputs, template, forcings)
  assert called.engine._static is not None
  got = getattr(called, what)(*args)
  assert called.engine._static is None
  never = graphcast.GraphCast(cfg, task, params=params)
  want = getattr(never, what)(*args)
  assert never.engine.static_cache_builds == 0
  _same(got, want)
  # no cache next to the gradient workspace; without the workspace the next call builds it again,
  # and both predict what a fresh model predicts
  want = graphcast.GraphCast(cfg, task, params=params)(inputs, template, forcings)
  _same(called(inputs, template, forcings), want)
  assert called.engine._static is None
  called.engine.release_gradient_workspace()
  _same(called(inputs, template, forcings), want)
  assert called.engine._static is not None


# ---- the table-accumulator layer against the MMA chain --------------------------------------------
def _rows(which):
  sm = torch.cuda.get_device_properties(0).multi_processor_count
  return {"many_tiles": 128 * (sm // 2) * 3 + 77}.get(which, which)


@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
@pytest.mark.parametrize("rows", [1, 127, 129, "many_tiles"])
def test_table_layer_is_bit_identical_to_the_mma_layer(prec, rows):
  lib = _native.lib()
  rows = _rows(rows)
  g = torch.Generator().manual_seed(rows)
  n_nodes = 300
  x = torch.randn(rows, 512, generator=g).to(DEV)
  x[1::5] = 0.0                                             # rows whose products are all zero
  x_img = _image(lib, x, rows, 512)
  l0 = Layer(lib, 512, 512, g, ln=False)
  l1 = Layer(lib, 512, 512, g, ln=True)
  pa, pb = torch.randn(n_nodes, 512, generator=g).to(DEV), torch.randn(n_nodes, 512, generator=g).to(DEV)
  pb[:, :64] = -0.0
  pa[:, :64] = -0.0
  ia = torch.randint(0, n_nodes, (rows,), generator=g, dtype=torch.int32).to(DEV)
  ib = torch.randint(0, n_nodes, (rows,), generator=g, dtype=torch.int32).to(DEV)
  pre = [(pa, ia), (pb, ib)]
  scratch = _scratch(lib, 3, 1, 2)
  nan = lambda: torch.full((rows, 512), float("nan"), device=DEV)

  def desc(n):
    d = _native.ChainDesc()
    d.rows, d.nlayers, d.precision, d.lag, d.order = rows, n, _native.PRECISIONS[prec], 1, 0
    d.scratch, d.scratch_bytes = scratch.data_ptr(), scratch.numel()
    return d

  def run(d):
    _native.check(lib.gcb_chain_forward(C.byref(d), _stream()), "chain")

  def as_table(cl, table):
    cl.nseg, cl.w_packed = 0, None
    cl.seg_from[0] = -1
    cl.acc_table, cl.ld_acc = table.data_ptr(), 512

  # the table: X @ W0, the raw accumulator
  table = nan()
  d = desc(1)
  _fill_chain_layer(d.layer[0], [_seg_img(x_img, 512)], [-1], l0, act=False, keep=False, out=table)
  d.layer[0].bias, d.layer[0].acc_out = None, 1
  run(d)
  # [swish(X @ W0 + b0 + addends), kept] -> LN: MMAs vs table
  outs = []
  for use_table in (False, True):
    out = nan()
    d = desc(2)
    _fill_chain_layer(d.layer[0], [_seg_img(x_img, 512)], [-1], l0, act=True, keep=True, pre=pre)
    if use_table:
      as_table(d.layer[0], table)
    _fill_chain_layer(d.layer[1], [None], [0], l1, act=False, keep=False, out=out)
    run(d)
    outs.append(out)
  # a plain layer with an fp32 output: X @ W0 + b0
  for use_table in (False, True):
    out = nan()
    d = desc(1)
    _fill_chain_layer(d.layer[0], [_seg_img(x_img, 512)], [-1], l0, act=False, keep=False, out=out)
    if use_table:
      as_table(d.layer[0], table)
    run(d)
    outs.append(out)
  torch.cuda.synchronize()
  as_bits = lambda t: t.view(torch.int32)
  assert torch.equal(as_bits(outs[0]), as_bits(outs[1]))
  assert torch.equal(as_bits(outs[2]), as_bits(outs[3]))
  assert torch.isfinite(outs[1]).all() and torch.isfinite(table).all()
  assert (table[1::5] == 0).all()
  ref = x.double() @ l0.w.double().to(DEV)
  err = float((table.double() - ref).abs().max() / ref.abs().max())
  assert err <= (3e-5 if prec == "bf16x3" else 3e-2), err


# ---- 0.25 degree: the cache is released before the gradient workspace ----------------------------
def test_full_size_call_then_input_grads():
  if torch.cuda.get_device_properties(0).total_memory < 75e9:
    pytest.skip("needs an 80 GB GPU")
  from test_gpu_input_grads import _full_problem
  model, ar, inputs, targets, forcings = _full_problem(graphcast.TASK, 0.25, 6, 1)
  torch.cuda.reset_peak_memory_stats()
  model(inputs, targets, forcings)
  torch.cuda.synchronize()
  eng = model.engine
  call_peak = torch.cuda.max_memory_allocated()
  cache = sum(t.numel() * t.element_size() for t in eng._static.values())
  build_ms = eng.static_cache_build_ms()
  torch.cuda.reset_peak_memory_stats()
  loss, _, ig, fg = ar.loss_and_input_grads(inputs, targets, forcings)
  torch.cuda.synchronize()
  grad_peak = torch.cuda.max_memory_allocated()
  assert eng._static is None
  assert np.isfinite(float(loss.values[0]))
  assert all(np.isfinite(np.asarray(v.values)).all() for ds in (ig, fg) for v in ds.data_vars.values())
  print(f"\n0.25 deg: static-edge cache {cache / 2**30:.2f} GiB built in {build_ms:.1f} ms; peak of "
        f"__call__ {call_peak / 2**30:.2f} GiB, of loss_and_input_grads after it {grad_peak / 2**30:.2f} "
        f"GiB on {torch.cuda.get_device_name(0)}")
  del ig, fg
  gc.collect()
