"""The device training step (optim.AdamW): gcb_pack_weight against the host packer, gcb_sum_squares and
gcb_adamw_step against fp64, Engine.load_params_device against load_params, the stale-host-weights
paths, and opt.step end to end against loss_and_grads and the fp64 restatement of AdamW."""
import gc

import numpy as np
import pytest
import torch

import _cases
from graphcast_b200 import (_native, autoregressive, casting, engine, graphcast, normalization, optim,
                            synthetic)
from graphcast_b200 import xarray_shim as xs
from test_gpu_grad_tensors import _equal, _outputs
from test_gpu_loss import _lat_weight, _model_and_data, _stats
from test_optim_host import restate

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _st():
  return torch.cuda.current_stream().cuda_stream


# ---- 1. gcb_pack_weight --------------------------------------------------------------------------
def _host_pack(w, k, n):
  lib = _native.lib()
  w = np.ascontiguousarray(w, np.float32)
  img = np.empty([lib.gcb_packed_weight_bytes(k, n)], np.uint8)
  _native.check(lib.gcb_pack_weight_host(w.ctypes.data, w.shape[0], w.shape[1], k, n, img.ctypes.data),
                "gcb_pack_weight_host")
  return img


def _dev_pack(src, offset, ld, transpose, k_rows, n_cols, k, n):
  lib = _native.lib()
  img = torch.full([lib.gcb_packed_weight_bytes(k, n)], 0xAB, dtype=torch.uint8, device=DEV)
  f32 = torch.full([k, n], float("nan"), dtype=torch.float32, device=DEV)
  _native.check(lib.gcb_pack_weight(src.data_ptr() + 4 * offset, ld, transpose, k_rows, n_cols, k, n,
                                    img.data_ptr(), f32.data_ptr(), _st()), "gcb_pack_weight")
  return img.cpu().numpy(), f32.cpu().numpy()


# (name, source shape, element offset, ld, transpose, k_rows, n_cols, k, n): every use of the engine
PACK_CASES = [
    ("grid_embedder_474_to_480", (474, 512), 0, 512, 0, 474, 512, 480, 512),
    ("edge_embedder_4_to_16", (4, 512), 0, 512, 0, 4, 512, 16, 512),
    ("decoder_227_to_256", (512, 227), 0, 227, 0, 512, 227, 512, 256),
    ("split_block_sender", (1536, 512), 512 * 512, 512, 0, 512, 512, 512, 512),
    ("split_block_receiver", (1536, 512), 2 * 512 * 512, 512, 0, 512, 512, 512, 512),
    ("w1_t_decoder", (512, 227), 0, 227, 1, 227, 512, 256, 512),
    ("w1_t_latent", (512, 512), 0, 512, 1, 512, 512, 512, 512),
    ("w0_t_block_2", (1536, 512), 2 * 512 * 512, 512, 1, 512, 512, 512, 512),
    ("w0_in_n256", (200, 512), 0, 512, 1, 512, 200, 512, 256),
    ("w0_in_n512", (474, 512), 0, 512, 1, 512, 474, 512, 512),
    ("k_rows_0", (16, 512), 0, 512, 0, 0, 512, 16, 512),
]


@pytest.mark.parametrize("case", PACK_CASES, ids=[c[0] for c in PACK_CASES])
def test_pack_weight_is_byte_identical_to_the_host_packer(case):
  _, shape, off, ld, tr, k_rows, n_cols, k, n = case
  rng = np.random.default_rng(0)
  src = rng.standard_normal(shape).astype(np.float32) * np.float32(0.05)
  src.reshape(-1)[::97] = 0.0
  src.reshape(-1)[1::89] = -0.0
  src.reshape(-1)[2::83] *= np.float32(1e-39) / np.float32(0.05)  # subnormals
  flat = src.reshape(-1)
  if tr:
    logical = flat[off:off + n_cols * ld].reshape(n_cols, ld)[:, :k_rows].T
  else:
    logical = flat[off:off + k_rows * ld].reshape(k_rows, ld)[:, :n_cols]
  want = _host_pack(logical, k, n)
  img, f32 = _dev_pack(torch.as_tensor(src).to(DEV), off, ld, tr, k_rows, n_cols, k, n)
  assert np.array_equal(img, want)
  padded = np.zeros([k, n], np.float32)
  padded[:k_rows, :n_cols] = logical
  assert np.array_equal(f32.view(np.uint32), padded.view(np.uint32))


def test_pack_weight_rejects_bad_arguments():
  lib = _native.lib()
  t = torch.zeros([64 * 256], dtype=torch.float32, device=DEV)
  assert lib.gcb_pack_weight(t.data_ptr(), 256, 0, 20, 256, 24, 256, t.data_ptr(), None, _st()) == -1
  assert b"multiple of 16" in lib.gcb_last_error()
  assert lib.gcb_pack_weight(t.data_ptr(), 100, 0, 16, 256, 16, 256, t.data_ptr(), None, _st()) == -1
  assert lib.gcb_pack_weight(t.data_ptr(), 256, 0, 32, 256, 16, 256, t.data_ptr(), None, _st()) == -1


# ---- 2. gcb_sum_squares --------------------------------------------------------------------------
def _sum_squares(x):
  lib = _native.lib()
  ws = torch.empty([lib.gcb_sum_squares_workspace_bytes()], dtype=torch.uint8, device=DEV)
  out = torch.full([1], float("nan"), dtype=torch.float64, device=DEV)
  _native.check(lib.gcb_sum_squares(x.data_ptr(), x.numel(), ws.data_ptr(), ws.numel(), out.data_ptr(),
                                    _st()), "gcb_sum_squares")
  return out


@pytest.mark.parametrize("n", [0, 1, 2 ** 10 - 1, 2 ** 10 + 1, 2 ** 18 - 1, 2 ** 18 + 1, 2 ** 20 + 1,
                               36_348_131])
def test_sum_squares_against_fp64(n):
  g = torch.Generator(device=DEV).manual_seed(n)
  x = torch.randn(max(n, 1), generator=g, device=DEV)[:n] * 3 + 0.5
  got = _sum_squares(x)
  again = _sum_squares(x)
  assert torch.equal(got, again)                              # bit-identical reruns
  want = float(np.sum(x.cpu().numpy().astype(np.float64) ** 2))
  got = float(got.item())
  if n == 0:
    assert got == 0.0
  else:
    assert abs(got - want) <= 1e-12 * want


# ---- 3. gcb_adamw_step ---------------------------------------------------------------------------
def _gate(before, after, ref):
  """The per-element gate of the device update against the fp64 restatement from the same fp32 state:
  |dp_dev - dp_ref| <= 1e-5 |dp_ref| + ulp(p_new); m and v within 1e-6 relative."""
  (p0, _, _), (p1, m1, v1), (pr, mr, vr) = before, after, ref
  p0, p1, m1, v1 = (np.asarray(a, np.float64) for a in (p0, p1, m1, v1))
  dp_dev, dp_ref = p1 - p0, pr - p0
  ulp = np.spacing(np.abs(pr).astype(np.float32)).astype(np.float64)
  bad = np.abs(dp_dev - dp_ref) > 1e-5 * np.abs(dp_ref) + ulp
  assert not bad.any(), f"{int(bad.sum())} elements off, e.g. {dp_dev[bad][:3]} vs {dp_ref[bad][:3]}"
  assert np.all(np.abs(m1 - mr) <= 1e-6 * np.abs(mr))
  assert np.all(np.abs(v1 - vr) <= 1e-6 * np.abs(vr))


def _adamw(p, g, m, v, t, hp, n_decay, max_norm):
  lib = _native.lib()
  sumsq = _sum_squares(g)
  _native.check(lib.gcb_adamw_step(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel(),
                                   n_decay, t, hp["lr"], hp["b1"], hp["b2"], hp["eps"], hp["eps_root"],
                                   hp["wd"], sumsq.data_ptr(), max_norm or 0.0, _st()), "gcb_adamw_step")


@pytest.mark.parametrize("t", [1, 2, 1000])
@pytest.mark.parametrize("clip", [False, True])
@pytest.mark.parametrize("offset", [0, 1], ids=["aligned", "unaligned"])
def test_adamw_step_against_the_fp64_restatement(t, clip, offset):
  n = 1_000_003
  g = torch.Generator(device=DEV).manual_seed(t)
  buf = lambda: torch.empty([n + 4], dtype=torch.float32, device=DEV)[offset:offset + n]
  state = [torch.randn(n, generator=g, device=DEV) * 0.1,                  # p
           torch.randn(n, generator=g, device=DEV) * 1e-2,                 # g
           torch.randn(n, generator=g, device=DEV) * 1e-3,                 # m
           torch.rand(n, generator=g, device=DEV) * 1e-5]                  # v
  hp = dict(lr=1e-3, b1=0.9, b2=0.95, eps=1e-8, eps_root=1e-12, wd=0.1)
  n_decay = 612_345
  norm = float(torch.linalg.vector_norm(state[1].double()))
  max_norm = 0.25 * norm if clip else None
  before = [s.cpu().numpy() for s in (state[0], state[2], state[3])]
  results = []
  for _ in range(2):
    p, gg, m, v = (buf().copy_(s) for s in state)
    _adamw(p, gg, m, v, t, hp, n_decay, max_norm)
    results.append([s.cpu().numpy() for s in (p, m, v)])
  assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(*results))
  pr, mr, vr, _ = restate(before[0], state[1].cpu().numpy(), before[1], before[2], t, n_decay=n_decay,
                          max_norm=max_norm, **hp)
  _gate(before, results[0], (pr, mr, vr))


# ---- 4. Engine.load_params_device ----------------------------------------------------------------
def _problem(res):
  g, p1, x = _cases.small_case(c_in=31, n_out=23, msg_steps=3, res=res)
  _, p2, _ = _cases.small_case(c_in=31, n_out=23, msg_steps=3, seed=1, res=res)
  rng = np.random.default_rng(3)
  planes = torch.as_tensor(x[:, 0, :].T.copy()).to(DEV)
  targets = torch.as_tensor(rng.standard_normal((23, g.num_grid_nodes)).astype(np.float32)).to(DEV)
  lat_w = torch.as_tensor(_lat_weight(np.linspace(-90, 90, len(g.grid_lat)))).to(DEV)
  coef = torch.as_tensor(rng.uniform(0.5, 2.0, 23) / (23 * g.num_grid_nodes)).to(DEV)
  return g, p1, p2, (planes, targets, lat_w, coef)


def _to_device(params):
  return {k: {f: torch.as_tensor(np.asarray(a, np.float32)).to(DEV) for f, a in v.items()}
          for k, v in params.items()}


def _buffers(eng):
  """Every weight buffer of the engine and its gradient workspace, by name."""
  out = {}
  for key, (_, _, _, bufs, _, _) in eng._weights.items():
    for name, t in bufs.items():
      out[(str(key), name)] = t
  for info in eng._backward._all:
    for name, t in info.t.items():
      out[(info.stem, "t", name)] = t
  return out


@pytest.mark.parametrize("res", [4.0, 2.0])
def test_load_params_device_equals_load_params(res):
  g, p1, p2, args = _problem(res)
  make = lambda p: engine.Engine(g, p, c_in=31, n_out=23, msg_steps=3, precision="bf16x3")
  dev_eng, host_eng = make(p1), make(p1)
  _outputs(dev_eng, *args)                   # gradient workspace and the input transpose exist
  _outputs(host_eng, *args)
  ptrs = {k: t.data_ptr() for k, t in _buffers(dev_eng).items()}
  p2_dev = _to_device(p2)
  dev_eng.load_params_device(p2_dev)
  host_eng.load_params(p2)
  a, b = _buffers(dev_eng), _buffers(host_eng)
  assert set(a) == set(b) and any("w0_in" in k for k in a)
  for k in a:
    assert torch.equal(a[k], b[k]), k
  assert {k: t.data_ptr() for k, t in a.items()} == ptrs
  # replayed step graph, loss, gradients, input transpose, fp32 path: as a fresh engine
  fresh = make(p2)
  want = _outputs(fresh, *args)
  del fresh
  assert _equal(_outputs(dev_eng, *args), want)
  # the host view of the weights follows the device
  for name, fields in dev_eng.params.items():
    for f, arr in fields.items():
      if not name.startswith("mesh2grid_gnn/~_networks_builder/processor_nodes_0_mesh_nodes"):
        assert np.array_equal(arr, np.asarray(p2[name][f], np.float32)), (name, f)
  # in place: ten reloads allocate nothing
  p1_dev = _to_device(p1)
  torch.cuda.synchronize()
  before = torch.cuda.memory_allocated()
  for i in range(10):
    dev_eng.load_params_device(p1_dev if i % 2 == 0 else p2_dev)
  torch.cuda.synchronize()
  assert torch.cuda.memory_allocated() == before
  assert {k: t.data_ptr() for k, t in _buffers(dev_eng).items()} == ptrs
  # bad shapes, dtypes or devices raise before anything is written
  snapshot = {k: t.clone() for k, t in _buffers(dev_eng).items()}
  name = "mesh_gnn/~_networks_builder/processor_edges_1_mesh_mlp/~/linear_0"
  for bad_t, match in ((p1_dev[name]["w"][:-1], "shape"), (p1_dev[name]["w"].double(), "float32"),
                       (p1_dev[name]["w"].cpu(), "float32")):
    bad = {k: dict(v) for k, v in p1_dev.items()}
    bad[name]["w"] = bad_t
    with pytest.raises(ValueError, match=match):
      dev_eng.load_params_device(bad)
  with pytest.raises(ValueError, match="missing"):
    dev_eng.load_params_device({k: v for k, v in p1_dev.items() if k != name})
  assert all(torch.equal(t, snapshot[k]) for k, t in _buffers(dev_eng).items())


# ---- helpers of the end-to-end tests ---------------------------------------------------------------
def _one(ds):
  return ds.isel(time=slice(0, 1))


def _stack(kind, model, task):
  std, mean, dstd = _stats(task, seed=1)
  if kind == "graphcast":
    return model
  if kind == "ar_norm_bf16_T1":
    return autoregressive.Predictor(normalization.InputsAndResiduals(casting.Bfloat16Cast(model),
                                                                     std, mean, dstd))
  return autoregressive.Predictor(normalization.InputsAndResiduals(model, std, mean, dstd),
                                  gradient_checkpointing=True)


def _dev_state(opt):
  return [opt._bufs[k].cpu().numpy() for k in ("p", "m", "v")]


HP = dict(lr=1e-3, b1=0.9, b2=0.95, eps=1e-8, eps_root=0.0, wd=0.1)


def _make_opt(predictor, **kw):
  return optim.AdamW(predictor, learning_rate=HP["lr"], b1=HP["b1"], b2=HP["b2"], eps=HP["eps"],
                     eps_root=HP["eps_root"], weight_decay=HP["wd"], **kw)


# ---- 5. stale host weights -----------------------------------------------------------------------
def test_no_path_reads_stale_host_weights():
  task, model, inputs, targets, forcings = _model_and_data(batch=1, steps=2)
  p_before = {k: {f: np.array(a) for f, a in v.items()} for k, v in model._params.items()}
  opt = _make_opt(model)
  for _ in range(2):
    opt.step(inputs, _one(targets), _one(forcings))        # one target time: no input transpose yet
  p_after = opt.params()
  ar = autoregressive.Predictor(model, gradient_checkpointing=True)
  got = ar.loss_and_grads(inputs, targets, forcings)       # packs w0_in for the first time

  def fresh(params):
    m = graphcast.GraphCast(model._model_config, task, params=params)
    return autoregressive.Predictor(m, gradient_checkpointing=True).loss_and_grads(inputs, targets,
                                                                                   forcings)

  def same(a, b):
    assert np.array_equal(a[0].values, b[0].values)
    for k in b[2]:
      for f in b[2][k]:
        assert np.array_equal(a[2][k][f], b[2][k][f]), (k, f)
  live = [k for k in p_after
          if not k.startswith("mesh2grid_gnn/~_networks_builder/processor_nodes_0_mesh_nodes")]
  for k in live:                                           # the predictor's host params are refreshed
    for f in p_after[k]:
      assert np.array_equal(model._params[k][f], p_after[k][f]), (k, f)
  same(got, fresh(p_after))
  model.set_params(p_before)                               # equal to the host copies: still reloaded
  same(ar.loss_and_grads(inputs, targets, forcings), fresh(p_before))


# ---- 6. opt.step end to end ----------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["graphcast", "ar_norm_bf16_T1", "ar_norm_T2"])
def test_step_matches_loss_and_grads_and_the_restatement(kind):
  task, model, inputs, targets, forcings = _model_and_data(batch=2, steps=2)
  if kind != "ar_norm_T2":
    targets, forcings = _one(targets), _one(forcings)
  pred = _stack(kind, model, task)
  mask = lambda module, field: field == "w"
  opt = _make_opt(pred, mask=mask, max_grad_norm=0.5)
  layout = optim.FlatLayout.of(model._params, mask)
  for t in range(1, 4):
    ref_loss, ref_diag, ref_grads = pred.loss_and_grads(inputs, targets, forcings)
    if t == 1:                                             # the state is created by the first step
      before = [layout.flatten(model._params)] + [np.zeros(layout.size, np.float32)] * 2
    else:
      before = _dev_state(opt)
    loss, diag, grad_norm = opt.step(inputs, targets, forcings)
    assert np.array_equal(loss.values, ref_loss.values)
    for name in ref_diag.keys():
      assert np.array_equal(diag.data_vars[name].values, ref_diag.data_vars[name].values)
    g = opt._bufs["g"].cpu().numpy()
    assert np.array_equal(g, opt.layout.flatten(ref_grads))
    pr, mr, vr, norm = restate(*[before[0], g, before[1], before[2]], t, n_decay=opt.layout.n_decay,
                               max_norm=0.5, **HP)
    assert abs(grad_norm - norm) <= 1e-12 * norm
    _gate(before, _dev_state(opt), (pr, mr, vr))
  # training lowers the loss on a fixed batch
  first = float(np.mean(loss.values))
  for _ in range(17):
    loss, _, _ = opt.step(inputs, targets, forcings)
  assert float(np.mean(loss.values)) < first


# ---- 7. state() / load_state() -------------------------------------------------------------------
def test_state_round_trip_resumes_bit_identically():
  task, model_a, inputs, targets, forcings = _model_and_data(batch=1)
  params0 = model_a._params
  opt_a = _make_opt(model_a)
  for _ in range(4):
    opt_a.step(inputs, targets, forcings)
  model_b = graphcast.GraphCast(model_a._model_config, task, params=params0)
  opt_b = _make_opt(model_b)
  for _ in range(2):
    opt_b.step(inputs, targets, forcings)
  state, params = opt_b.state(), opt_b.params()
  assert state["count"] == 2
  del opt_b, model_b
  model_c = graphcast.GraphCast(model_a._model_config, task, params=params)
  opt_c = _make_opt(model_c)
  opt_c.load_state(state)
  for _ in range(2):
    opt_c.step(inputs, targets, forcings)
  assert opt_c.count == opt_a.count == 4
  for a, c in zip(_dev_state(opt_a), _dev_state(opt_c)):
    assert np.array_equal(a.view(np.uint32), c.view(np.uint32))


# ---- 8. 0.25 degree / 37 levels ------------------------------------------------------------------
def _full_size(steps):
  gc.collect()
  torch.cuda.empty_cache()
  task = graphcast.TASK
  inputs, template, forcings = synthetic.make_example(task, 0.25, batch=1, num_target_steps=steps,
                                                      seed=2)
  rng = np.random.default_rng(3)
  targets = xs.Dataset(coords=template.coords)
  for name, v in template.data_vars.items():
    targets[name] = xs.DataArray(rng.standard_normal(v.shape).astype(np.float32), v.dims)
  cfg = graphcast.ModelConfig(0.25, 6, 512, 16, 1, 0.6)
  params = graphcast.init_params(cfg, task, synthetic.num_input_channels(task), seed=1)
  model = graphcast.GraphCast(cfg, task, params=params)
  std, mean, dstd = _stats(task, seed=1)
  pred = autoregressive.Predictor(normalization.InputsAndResiduals(model, std, mean, dstd),
                                  gradient_checkpointing=True)
  return model, pred, inputs, targets, forcings


def test_full_size_step_matches_the_restatement_and_fits():
  """0.25 deg / 37 levels on an 80 GB GPU: one step (T = 1) checked tensor by tensor, then the peak
  device memory of a T = 2 (backprop through time) step."""
  if torch.cuda.get_device_properties(0).total_memory < 75e9:
    pytest.skip("needs an 80 GB GPU")
  model, pred, inputs, targets, forcings = _full_size(2)
  opt = _make_opt(pred)
  layout = optim.FlatLayout.of(model._params)
  before = [layout.flatten(model._params)] + [np.zeros(layout.size, np.float32)] * 2
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  _, _, grad_norm = opt.step(inputs, _one(targets), _one(forcings))
  torch.cuda.synchronize()
  peak1 = torch.cuda.max_memory_allocated()
  g = opt._bufs["g"].cpu().numpy()
  after = _dev_state(opt)
  pr, mr, vr, norm = restate(before[0], g, before[1], before[2], 1, n_decay=layout.n_decay,
                             max_norm=32.0, **HP)
  assert abs(grad_norm - norm) <= 1e-12 * norm
  for name, f, off, shape in layout.entries:            # every tensor through the gate
    sl = slice(off, off + int(np.prod(shape)))
    _gate([b[sl] for b in before], [a[sl] for a in after], (pr[sl], mr[sl], vr[sl]))
  del g, after, pr, mr, vr, before
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  opt.step(inputs, targets, forcings)
  torch.cuda.synchronize()
  peak2 = torch.cuda.max_memory_allocated()
  print(f"0.25 deg / 37 levels, {layout.size} parameters, |g| {grad_norm:.6g}: peak device memory of "
        f"an optimiser step {peak1 / 2**30:.1f} GiB (T = 1), {peak2 / 2**30:.1f} GiB (T = 2) on "
        f"{torch.cuda.get_device_name(0)}")
