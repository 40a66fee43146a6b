"""Parameter gradients on the device: the backward kernels against fp64 PyTorch, and the gradients of
the whole step (Engine / GraphCast.loss_and_grads) against torch autograd of the fp64 oracle."""
import numpy as np
import pytest
import torch

import _cases
from graphcast_b200 import _native, autoregressive, casting, engine, graph as graph_lib, normalization
from oracle import gnn as oracle_gnn
from test_gpu_loss import _HostLoss, _lat_weight, _model_and_data, _stats

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _st():
  return torch.cuda.current_stream().cuda_stream


def _frob(got, ref):
  got, ref = got.double(), ref.double()
  return float(torch.linalg.norm(got - ref) / torch.linalg.norm(ref))


def _wgrad(lib, x, g, rows, k, n, prec, *, img=None, k_valid=None, swish=False, dw=None, acc=0):
  nb = lib.gcb_weight_grad_workspace_bytes(k, n)
  ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
  dw = torch.full((k, n), float("nan"), device=DEV) if dw is None else dw
  _native.check(lib.gcb_weight_grad(
      None if img is not None else x.data_ptr(), 0 if img is not None else x.shape[1],
      0 if img is not None else (k_valid or k), None if img is None else img.data_ptr(),
      1 if swish else 0, g.data_ptr(), g.shape[1], rows, k, n, _native.PRECISIONS[prec],
      ws.data_ptr(), nb, dw.data_ptr(), acc, _st()), "gcb_weight_grad")
  return dw


@pytest.mark.parametrize("prec,tol", [("bf16x3", 1e-5), ("bf16", 1e-2)])
@pytest.mark.parametrize("k,n", [(16, 512), (48, 256), (512, 256), (512, 512)])
@pytest.mark.parametrize("source", ["fp32", "image"])
def test_weight_grad_kernel_against_fp64(prec, tol, k, n, source):
  lib = _native.lib()
  gen = torch.Generator(device=DEV).manual_seed(k + n)
  rows = 5003                                       # not a multiple of 128 nor of the slice size
  k_valid = 4 if k == 16 else k
  x = torch.zeros(rows, k, device=DEV)
  x[:, :k_valid] = torch.randn(rows, k_valid, generator=gen, device=DEV)
  g = torch.randn(rows, n, generator=gen, device=DEV)
  img = None
  if source == "image":
    img = torch.zeros(lib.gcb_a_image_bytes(rows, k), dtype=torch.uint8, device=DEV)
    _native.check(lib.gcb_rows_to_image(x.data_ptr(), k, 1, rows, k, img.data_ptr(), _st()), "img")
    xs = x
  else:
    xs = x[:, :k_valid].contiguous() if k == 16 else x
  ref = x.double().t() @ g.double()
  dw = _wgrad(lib, xs, g, rows, k, n, prec, img=img, k_valid=k_valid)
  err = _frob(dw, ref)
  assert err <= tol, err
  again = _wgrad(lib, xs, g, rows, k, n, prec, img=img, k_valid=k_valid)
  assert torch.equal(dw, again)                     # deterministic, bit for bit
  # accumulate mode adds to what is there
  base = torch.randn(k, n, generator=gen, device=DEV)
  acc = _wgrad(lib, xs, g, rows, k, n, prec, img=img, k_valid=k_valid, dw=base.clone(), acc=1)
  assert _frob(acc, ref + base.double()) <= tol


def test_weight_grad_swish_source_and_many_rows():
  lib = _native.lib()
  gen = torch.Generator(device=DEV).manual_seed(1)
  rows, k, n = 300_001, 512, 512
  h = torch.randn(rows, k, generator=gen, device=DEV)
  g = torch.randn(rows, n, generator=gen, device=DEV)
  hd = h.double()
  ref = (hd * torch.sigmoid(hd)).t() @ g.double()
  dw = _wgrad(lib, h, g, rows, k, n, "bf16x3", swish=True)
  assert _frob(dw, ref) <= 1e-5


def _rowwise(lib, mode, dy, z, scale, n):
  rows = dy.shape[0]
  nb = lib.gcb_rowwise_workspace_bytes(n)
  ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
  dz = torch.full_like(dy, float("nan"))
  sums = [torch.full((n,), float("nan"), device=DEV) for _ in range(3)]
  if mode == "ln":
    _native.check(lib.gcb_layernorm_backward(
        dy.data_ptr(), n, z.data_ptr(), n, scale.data_ptr(), rows, n, dz.data_ptr(), n, ws.data_ptr(),
        nb, sums[0].data_ptr(), sums[1].data_ptr(), sums[2].data_ptr(), 0, _st()), "ln")
  elif mode == "swish":
    _native.check(lib.gcb_swish_backward(dy.data_ptr(), n, z.data_ptr(), n, rows, n, dz.data_ptr(), n,
                                         ws.data_ptr(), nb, sums[0].data_ptr(), 0, _st()), "swish")
  else:
    _native.check(lib.gcb_layernorm_backward(dy.data_ptr(), n, None, 0, None, rows, n, dz.data_ptr(),
                                             n, ws.data_ptr(), nb, sums[0].data_ptr(), None, None, 0,
                                             _st()), "copy")
  return dz, sums


@pytest.mark.parametrize("mode,n", [("ln", 512), ("swish", 512), ("swish", 256), ("copy", 256)])
def test_rowwise_backward_against_autograd(mode, n):
  lib = _native.lib()
  gen = torch.Generator(device=DEV).manual_seed(2)
  rows = 70_001
  dy = torch.randn(rows, n, generator=gen, device=DEV)
  z = torch.randn(rows, n, generator=gen, device=DEV) * 2 + 0.5
  scale = torch.rand(n, generator=gen, device=DEV) + 0.5
  dz, sums = _rowwise(lib, mode, dy, z, scale, n)
  zd = z.double().requires_grad_(True)
  if mode == "ln":
    sd = scale.double().requires_grad_(True)
    od = torch.zeros(n, dtype=torch.float64, device=DEV, requires_grad=True)
    y = oracle_gnn.layer_norm(zd, sd, od)
    y.backward(dy.double())
    want = [zd.grad.sum(0), sd.grad, od.grad]
  elif mode == "swish":
    (zd * torch.sigmoid(zd)).backward(dy.double())
    want = [zd.grad.sum(0)]
  else:
    zd.grad = dy.double()
    want = [dy.double().sum(0)]
  assert _frob(dz, zd.grad) <= 1e-6
  for got, ref in zip(sums, want):
    assert _frob(got, ref) <= 1e-6
  dz2, sums2 = _rowwise(lib, mode, dy, z, scale, n)
  assert torch.equal(dz, dz2) and all(torch.equal(a, b) for a, b in zip(sums[:len(want)], sums2))


def test_sender_segment_sum_and_gather_add():
  lib = _native.lib()
  rng = np.random.default_rng(3)
  n_nodes, n_edges = 1000, 40_000
  snd = rng.integers(0, n_nodes, n_edges)
  snd[:3000] = 17                                   # one heavy sender (a pole-side mesh node)
  rng.shuffle(snd)
  order, ptr, heavy = graph_lib.sender_csr(snd, n_nodes)
  assert heavy.tolist() == [17]
  msg = torch.randn(n_edges, 512, device=DEV, dtype=torch.float32)
  t = lambda a: torch.as_tensor(a).to(DEV)
  out = torch.full((n_nodes, 512), float("nan"), device=DEV)
  order_d, ptr_d, hv = t(order), t(ptr), t(heavy)   # kept alive while the kernels read them
  args = (msg.data_ptr(), 512, order_d.data_ptr(), ptr_d.data_ptr(), n_nodes)
  _native.check(lib.gcb_segment_sum_sorted(*args, hv.data_ptr(), 1, out.data_ptr(), 512, 512, _st()), "s")
  ref = torch.zeros(n_nodes, 512, dtype=torch.float64, device=DEV)
  ref.index_add_(0, t(snd).long(), msg.double())
  err = _frob(out, ref)
  print(f"sender segment sum: relative error {err:.3g}")
  assert err <= 1e-6
  # without the heavy list the same rows are summed in the same order: bit-identical
  out2 = torch.full_like(out, float("nan"))
  _native.check(lib.gcb_segment_sum_sorted(*args, None, 0, out2.data_ptr(), 512, 512, _st()), "s")
  assert torch.equal(out, out2)
  # gather-add: dst = addend + src[idx]
  src = torch.randn(n_nodes, 512, device=DEV)
  idx = t(snd.astype(np.int32))
  add = torch.randn(n_edges, 512, device=DEV)
  dst = torch.empty(n_edges, 512, device=DEV)
  _native.check(lib.gcb_gather_add(src.data_ptr(), 512, idx.data_ptr(), n_edges, add.data_ptr(), 512,
                                   dst.data_ptr(), 512, 512, _st()), "gather_add")
  assert torch.equal(dst, add + src[idx.long()])


# ---- the whole step -------------------------------------------------------------------------------
class _GradOracle(oracle_gnn.Oracle):
  """The oracle with its stage outputs kept as tensors, so that autograd sees the whole step."""

  def _t(self, a):
    return a if isinstance(a, torch.Tensor) else super()._t(a)


def _oracle_grads(g, params, x, targets, lat_w, coef, dtype=torch.float64):
  """Gradient of  sum_b sum_c coef_c / 2 * sum_node w (y - t)^2  by torch autograd of the oracle."""
  orc = _GradOracle(params, dtype)
  for fields in orc.p.values():
    for t in fields.values():
      t.requires_grad_(True)
  y = orc.forward(g.as_dict(), x)                                    # [Ng, B, n_out]
  n_lon = g.num_grid_nodes // lat_w.shape[0]
  wn = torch.as_tensor(np.repeat(lat_w, n_lon)).to(dtype)[:, None, None]
  d = y - torch.as_tensor(targets).to(dtype)
  loss = (torch.as_tensor(coef).to(dtype) / 2 * wn * d * d).sum()
  loss.backward()
  return {k: {f: t.grad for f, t in v.items()} for k, v in orc.p.items()}


def _engine_grads(eng, x, targets, lat_w, coef, chunk_rows=None):
  n_out = eng.n_out
  eng.grads_begin(chunk_rows)
  w = torch.as_tensor(lat_w).to(DEV)
  c = torch.as_tensor(coef).to(DEV)
  sums = torch.empty(x.shape[1], n_out, dtype=torch.float64, device=DEV)
  for b in range(x.shape[1]):
    eng.pack_inputs(torch.as_tensor(x[:, b, :].T.copy()).to(DEV))
    eng.loss_and_grads_element(torch.as_tensor(targets[:, b, :].T.copy()).to(DEV), w, c,
                               channel_sums=sums[b])
  return {k: {f: t.cpu() for f, t in v.items()} for k, v in eng.grads().items()}, sums


def _compare(got, ref, params, tol):
  """Per-tensor relative error (against the global norm for tensors with a tiny reference)."""
  gnorm = np.sqrt(sum(float((t.double() ** 2).sum()) for v in ref.values() for t in v.values()
                      if t is not None))
  worst = {}
  for name, fields in params.items():
    for f, a in fields.items():
      g = got[name][f]
      assert tuple(g.shape) == np.asarray(a).shape, (name, f)
      r = ref[name][f]
      if r is None:                                  # never reached by the loss: exact zeros
        assert torch.count_nonzero(g) == 0, (name, f)
        continue
      rn = float(torch.linalg.norm(r.double()))
      den = rn if rn >= 1e-6 * gnorm else gnorm
      worst[(name, f)] = float(torch.linalg.norm(g.double() - r.double())) / den
  bad = {k: v for k, v in worst.items() if v > tol}
  assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])[:10]
  return worst


_REFERENCE = {}          # fp64 autograd gradients of a small case, shared by its engine variants


def _small_grad_case(res, mesh_size):
  """The small case on a res-degree grid: graph, params, inputs, targets, latitude weights, coef, and
  the fp64 autograd reference (computed once per grid)."""
  g, params, x = _cases.small_case(c_in=31, n_out=23, msg_steps=3, batch=2, res=res,
                                   mesh_size=mesh_size, randomize_affine=True)
  n_lat = len(g.grid_lat)
  assert g.num_grid_nodes == n_lat * len(g.grid_lon)
  lat_w = _lat_weight(np.linspace(-90, 90, n_lat))
  rng = np.random.default_rng(7)
  targets = rng.standard_normal((g.num_grid_nodes, 2, 23)).astype(np.float32)
  kappa = rng.uniform(0.5, 2.0, 23) / (23 * g.num_grid_nodes)
  coef = 2 * kappa / 2                                       # 2 kappa / batch
  if (res, mesh_size) not in _REFERENCE:
    _REFERENCE[(res, mesh_size)] = _oracle_grads(g, params, x, targets, lat_w, coef)
  return g, params, x, targets, lat_w, coef, _REFERENCE[(res, mesh_size)]


def _chunk_plan(eng):
  """Counts over the grid2mesh and mesh2grid edge chunks of the backward pass: chunks, chunks with
  heavy receivers (> 256 edges), single-receiver chunks larger than chunk_rows, chunks whose sender
  CSR has heavy senders."""
  chunks = eng._backward.chunks["g2m"] + eng._backward.chunks["m2g"]
  cr = eng._backward.chunk_rows
  return {"chunks": len(chunks),
          "heavy_receivers": sum(c[6] > 0 for c in chunks),
          "oversized": sum(c[3] - c[2] == 1 and c[1] - c[0] > cr for c in chunks),
          "heavy_senders": sum(c[7][3] > 0 for c in chunks)}


_MODES = [{"fuse": False}, {"image_residual": False}, {"deep_chains": False}, {"chain_lag": 1},
          {"chain_lag": 2}, {"reorder_mesh": True}]


@pytest.mark.parametrize("prec,tol,chunk_rows,res,mode", [
    pytest.param("bf16x3", 1e-4, None, 4.0, {}, id="bf16x3-0.0001-None"),
    pytest.param("bf16x3", 1e-4, 2000, 4.0, {}, id="bf16x3-0.0001-2000"),
    pytest.param("bf16", 5e-2, None, 4.0, {}, id="bf16-0.05-None"),
    # 2 deg / mesh 3: in-degree up to 467 and mesh2grid out-degree up to 757, so the chunks meet
    # heavy receivers, receivers with more edges than chunk_rows and heavy senders
    pytest.param("bf16x3", 1e-4, None, 2.0, {}, id="2deg-bf16x3-0.0001-None"),
    pytest.param("bf16x3", 1e-4, 300, 2.0, {}, id="2deg-bf16x3-0.0001-300"),
] + [pytest.param("bf16x3", 1e-4, None, 4.0, m, id="-".join(f"{k}={v}" for k, v in m.items()))
     for m in _MODES])
def test_model_grads_against_fp64_autograd(prec, tol, chunk_rows, res, mode):
  g, params, x, targets, lat_w, coef, ref = _small_grad_case(res, 3)
  eng = engine.Engine(g, params, c_in=31, n_out=23, msg_steps=3, precision=prec, **mode)
  got, sums = _engine_grads(eng, x, targets, lat_w, coef, chunk_rows)
  plan = _chunk_plan(eng)
  if chunk_rows:                                  # several receiver-aligned edge chunks
    assert len(eng._backward.chunks["m2g"]) > 3 and len(eng._backward.chunks["g2m"]) > 3
  if res == 2.0:
    assert plan["heavy_receivers"] > 0
    if chunk_rows:
      assert plan["oversized"] > 0
    else:                                         # a chunk holds all of a heavy sender's edges
      assert plan["heavy_senders"] > 0
  assert set(got) == set(params)
  worst = _compare(got, ref, params, tol)
  name, err = max(worst.items(), key=lambda kv: kv[1])
  print(f"{res} deg, {prec}, chunk_rows={chunk_rows}, {mode or 'default mode'}: max per-tensor "
        f"relative error {err:.3g} ({name[0]}:{name[1]}); chunk plan {plan}")
  dead = "mesh2grid_gnn/~_networks_builder/processor_nodes_0_mesh_nodes_mlp/~/linear_0"
  assert torch.count_nonzero(got[dead]["w"]) == 0
  again, sums2 = _engine_grads(eng, x, targets, lat_w, coef, chunk_rows)
  assert torch.equal(sums, sums2)
  for name in got:
    for f in got[name]:
      assert torch.equal(got[name][f], again[name][f]), (name, f)
  # the stage-wise forward of the gradient is gcb_forward: the same loss sums, bit for bit
  w = torch.as_tensor(lat_w).to(DEV)
  for b in range(x.shape[1]):
    eng.pack_inputs(torch.as_tensor(x[:, b, :].T.copy()).to(DEV))
    eng.step()
    step_sums = torch.empty(23, dtype=torch.float64, device=DEV)
    eng.output_loss(torch.as_tensor(targets[:, b, :].T.copy()).to(DEV), w, channel_sums=step_sums)
    assert torch.equal(step_sums, sums[b]), b


def test_gradients_need_the_pregathered_edge_layers():
  g, params, _ = _cases.small_case(c_in=31, n_out=23, msg_steps=3)
  eng = engine.Engine(g, params, c_in=31, n_out=23, msg_steps=3, pregather=False)
  with pytest.raises(NotImplementedError, match="pregather"):
    eng.grads_begin()


def test_graphcast_loss_and_grads_surface():
  task, model, inputs, targets, forcings = _model_and_data(batch=2)
  loss, diag, grads = model.loss_and_grads(inputs, targets, forcings)
  loss_ref, diag_ref = model.loss(inputs, targets, forcings)
  assert np.array_equal(loss.values, loss_ref.values)
  for name in diag_ref.keys():
    assert np.array_equal(diag.data_vars[name].values, diag_ref.data_vars[name].values)
  params = model._params
  assert set(grads) == set(params)
  for name, fields in params.items():
    assert set(grads[name]) == set(fields)
    for f, a in fields.items():
      assert grads[name][f].shape == np.asarray(a).shape and grads[name][f].dtype == np.float32
      assert np.isfinite(grads[name][f]).all()
  dead = "mesh2grid_gnn/~_networks_builder/processor_nodes_0_mesh_nodes_mlp/~/linear_1"
  assert not grads[dead]["w"].any()
  _, _, again = model.loss_and_grads(inputs, targets, forcings)
  for name in grads:
    for f in grads[name]:
      assert np.array_equal(grads[name][f], again[name][f])


def test_wrapper_stack_grads():
  task, model, inputs, targets, forcings = _model_and_data(batch=1, steps=1)
  std, mean, dstd = _stats(task, seed=1)
  cast = casting.Bfloat16Cast(model)
  fused = normalization.InputsAndResiduals(cast, std, mean, dstd)
  demo = autoregressive.Predictor(fused)
  loss, diag, grads = demo.loss_and_grads(inputs, targets, forcings)
  loss2, diag2, grads2 = fused.loss_and_grads(inputs, targets, forcings)
  assert np.array_equal(loss.values, loss2.values)
  for name in grads:
    for f in grads[name]:
      assert np.array_equal(grads[name][f], grads2[name][f])
  assert np.array_equal(loss.values, fused.loss(inputs, targets, forcings)[0].values)
  _, _, t_in, t_tg, t_fc = _model_and_data(batch=1, steps=2)
  with pytest.raises(NotImplementedError):
    demo.loss_and_grads(t_in, t_tg, t_fc)
  generic = normalization.InputsAndResiduals(_HostLoss(model), std, mean, dstd)
  with pytest.raises(NotImplementedError):
    generic.loss_and_grads(inputs, targets, forcings)
  model.set_precision("fp32_simt")
  with pytest.raises(NotImplementedError):
    model.loss_and_grads(inputs, targets, forcings)


def test_partitioned_engine_refuses_gradients():
  from graphcast_b200 import partitioned
  g, params, _ = _cases.small_case(c_in=31, n_out=23, msg_steps=3)
  pe = partitioned.PartitionedEngine(g, params, c_in=31, n_out=23, msg_steps=3, rank=0, world=2,
                                     device=DEV)
  with pytest.raises(NotImplementedError, match="node-partitioned"):
    pe.engine.grads_begin()


class _CheckpointedOracle(_GradOracle):
  """fp32 oracle whose processor steps are recomputed in the backward pass (host memory bounded)."""

  def processor(self, graph, vm1, inter=None):
    from torch.utils.checkpoint import checkpoint
    v = self._t(vm1)
    e = self.processor_embed(graph, v.shape[1])
    for k in range(self.num_message_steps()):
      v, e = checkpoint(lambda v_, e_, k_=k: self.processor_step(graph, v_, e_, k_), v, e,
                        use_reentrant=False)
    return v


def test_config1_grads_against_fp32_autograd():
  """BASELINE config 1 (1 deg, mesh 5, 13 levels, 16 steps): every parameter gradient against
  torch autograd of the fp32 oracle on the CPU."""
  import os
  from graphcast_b200 import graphcast, synthetic
  torch.set_num_threads(min(32, os.cpu_count() or 1))
  task = graphcast.TASK_13
  lat, lon = synthetic.grid_coords(1.0)
  g = graph_lib.cached_static_graph(grid_lat=lat, grid_lon=lon, mesh_size=5,
                                    radius_query_fraction_edge_length=0.6)
  c_in, n_out = synthetic.num_input_channels(task), graphcast.num_outputs(task)
  params = oracle_gnn.init_params(c_in=c_in, n_out=n_out, msg_steps=16, seed=1, randomize_affine=True)
  rng = np.random.default_rng(0)
  x = rng.standard_normal((g.num_grid_nodes, 1, c_in)).astype(np.float32)
  targets = rng.standard_normal((g.num_grid_nodes, 1, n_out)).astype(np.float32)
  lat_w = _lat_weight(lat)
  coef = 2 * rng.uniform(0.5, 2.0, n_out) / (n_out * g.num_grid_nodes)
  eng = engine.Engine(g, params, c_in=c_in, n_out=n_out, msg_steps=16, precision="bf16x3")
  got, _ = _engine_grads(eng, x, targets, lat_w, coef)
  del eng
  torch.cuda.empty_cache()
  orc = _CheckpointedOracle(params, torch.float32)
  for fields in orc.p.values():
    for t in fields.values():
      t.requires_grad_(True)
  y = orc.forward(g.as_dict(), x)
  wn = torch.as_tensor(np.repeat(lat_w, len(lon)))[:, None, None]
  d = y - torch.as_tensor(targets)
  (torch.as_tensor(coef, dtype=torch.float32) / 2 * wn * d * d).sum().backward()
  ref = {k: {f: t.grad for f, t in v.items()} for k, v in orc.p.items()}
  worst = _compare(got, ref, params, 1e-4)
  print(f"config 1: max per-tensor relative error {max(worst.values()):.3g}")

