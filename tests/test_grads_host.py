"""Host-side pieces of the parameter gradients: the loss coefficients kappa, the sender CSRs, and a
torch restatement of the loss written with kappa against graphcast_b200.losses (pinned to the
executed reference), which ties the autograd ground truth of tests/test_gpu_grads.py to the loss."""
import numpy as np
import torch

import _cases
from graphcast_b200 import engine, graph as graph_lib, graphcast, losses, model_utils, synthetic
from graphcast_b200 import xarray_shim as xs


def _targets_and_predictions(seed=0):
  task = graphcast.TASK_13_PRECIP_OUT
  _, template, _ = synthetic.make_example(task, 10.0, batch=2, num_target_steps=1, seed=seed)
  rng = np.random.default_rng(seed)
  targets, preds = xs.Dataset(coords=template.coords), xs.Dataset(coords=template.coords)
  for name, v in template.data_vars.items():
    targets[name] = xs.DataArray(rng.standard_normal(v.shape).astype(np.float32), v.dims)
    preds[name] = xs.DataArray(rng.standard_normal(v.shape).astype(np.float32), v.dims)
  return targets, preds


def _planes(ds, slabs):
  sizes = dict(ds.sizes)
  out = [np.asarray(model_utils.variable_to_planes(ds.data_vars[s.name], sizes)) for s in slabs]
  return np.concatenate([o.reshape(sizes["batch"], s.count, -1) for o, s in zip(out, slabs)], axis=1)


def test_kappa_is_the_linear_map_of_losses_from_channel_sums():
  targets, _ = _targets_and_predictions()
  slabs = model_utils.channel_layout(targets)
  n = sum(s.count for s in slabs)
  num_nodes = 18 * 36
  kappa = losses.channel_kappa(slabs, num_nodes, graphcast.LOSS_PER_VARIABLE_WEIGHTS)
  basis = np.eye(n) * 1e3
  total, _ = losses.losses_from_channel_sums(basis, slabs, num_nodes, graphcast.LOSS_PER_VARIABLE_WEIGHTS)
  np.testing.assert_allclose(np.asarray(total.values, np.float64) / 1e3, kappa, rtol=1e-6)


def test_torch_loss_with_kappa_equals_the_pinned_loss():
  targets, preds = _targets_and_predictions(seed=1)
  slabs = model_utils.channel_layout(targets)
  want, _ = losses.weighted_mse_per_level(preds, targets,
                                          per_variable_weights=graphcast.LOSS_PER_VARIABLE_WEIGHTS)
  lat = np.asarray(targets.lat.values)
  w = losses.normalized_latitude_weights(xs.DataArray(np.zeros(len(lat), np.float32), ("lat",),
                                                      coords={"lat": lat}))
  n_lon = targets.sizes["lon"]
  num_nodes = len(lat) * n_lon
  kappa = torch.as_tensor(losses.channel_kappa(slabs, num_nodes, graphcast.LOSS_PER_VARIABLE_WEIGHTS))
  y = torch.as_tensor(_planes(preds, slabs), dtype=torch.float64)
  t = torch.as_tensor(_planes(targets, slabs), dtype=torch.float64)
  wn = torch.as_tensor(np.repeat(w, n_lon), dtype=torch.float64)
  got = (kappa[None, :, None] * wn * (y - t) ** 2).sum(dim=(1, 2))
  np.testing.assert_allclose(got.numpy(), np.asarray(want.values, np.float64), rtol=1e-6)


def test_sender_csr_covers_every_edge_once():
  g = _cases.small_graph()
  eng_senders = {
      "g2m": (graph_lib.receiver_sorted(g.g2m_senders, g.g2m_receivers, g.num_mesh_nodes)[1], g.num_grid_nodes),
      "mesh": (graph_lib.receiver_sorted(g.mesh_senders, g.mesh_receivers, g.num_mesh_nodes)[1], g.num_mesh_nodes),
      "m2g": (np.asarray(g.m2g_senders, np.int32), g.num_mesh_nodes),
  }
  for name, (snd, n_nodes) in eng_senders.items():
    order, ptr, heavy = graph_lib.sender_csr(snd, n_nodes, heavy_threshold=8)
    assert order.dtype == np.int32 and ptr.dtype == np.int32
    assert ptr[0] == 0 and ptr[-1] == len(snd) and np.all(np.diff(ptr) >= 0), name
    assert np.array_equal(np.sort(order), np.arange(len(snd))), name      # every edge exactly once
    for i in range(n_nodes):
      edges = order[ptr[i]:ptr[i + 1]]
      assert np.all(snd[edges] == i) and np.all(np.diff(edges) > 0), name  # stable within a sender
    assert np.array_equal(heavy, np.nonzero(np.diff(ptr) > 8)[0]), name
