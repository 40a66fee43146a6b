"""GPU parity against the fp32 CPU oracle on BASELINE.json's configurations (SURVEY section 8d):

  config 1  GraphCast_small 1 deg (181x360, 13 levels, mesh 5, 16 message steps): the WHOLE step
            output against the oracle's full step.
  config 2  GraphCast 0.25 deg (721x1440, 37 levels, mesh 6): stage by stage --
              encoder   mesh rows with the largest in-degree (the pole rows: up to 3 753 incoming
                        grid points) plus a random sample, and every grid row that sends to them
                        (the encoder is 1-hop: a mesh row depends only on its incoming grid rows);
              processor IN FULL on the CPU from the GPU's own encoder output (its receptive field
                        is global: it cannot be sampled);
              decoder   sampled grid rows incl. both poles and the lon = 0 / 180 lines, from the
                        GPU's processor output (1-hop again: 3 mesh rows per grid row).
Gate: max-abs error / max-abs reference <= 1e-4 (bf16x3), for the fp32-master layout and for the
image-only latent layout.  A 29 TFLOP oracle step does not finish in a test; the processor alone
(12 TFLOP) takes about a minute on the GPU host."""
import os

import numpy as np
import pytest
import torch

from graphcast_b200 import engine, graph as graph_lib, graphcast, synthetic
from oracle import gnn as oracle_gnn

pytestmark = pytest.mark.gpu

TOL = 1e-4


def _rel(a, b):
  return float(np.abs(a - b).max() / np.abs(b).max())


def _threads():
  torch.set_num_threads(min(32, os.cpu_count() or 1))


def _setup(res, mesh, task):
  lat, lon = synthetic.grid_coords(res)
  g = graph_lib.cached_static_graph(grid_lat=lat, grid_lon=lon, mesh_size=mesh,
                                    radius_query_fraction_edge_length=0.6)
  c_in = synthetic.num_input_channels(task)
  n_out = graphcast.num_outputs(task)
  params = oracle_gnn.init_params(c_in=c_in, n_out=n_out, msg_steps=16, seed=1)
  return g, params, c_in, n_out


def test_config1_small_1deg_full_step_matches_the_oracle():
  _threads()
  g, params, c_in, n_out = _setup(1.0, 5, graphcast.TASK_13)
  assert (g.num_grid_nodes, g.num_mesh_nodes, len(g.g2m_senders), len(g.mesh_senders)) == \
      (65160, 10242, 101892, 81900)
  x = np.random.default_rng(0).standard_normal((g.num_grid_nodes, 1, c_in)).astype(np.float32)
  ref = oracle_gnn.Oracle(params, torch.float32).forward(g.as_dict(), x).numpy()
  for image_residual in (False, True):
    eng = engine.Engine(g, params, c_in=c_in, n_out=n_out, msg_steps=16, precision="bf16x3",
                        image_residual=image_residual)
    y = eng.forward_features(torch.as_tensor(x)).cpu().numpy()
    err = _rel(y, ref)
    print(f"config 1 (1 deg, mesh 5, 13 levels, 16 steps), image_residual={image_residual}: "
          f"bf16x3 vs fp32 oracle, whole step output: {err:.3e}")
    assert err <= TOL
    del eng
    torch.cuda.empty_cache()


def _subgraph_encoder(g, mesh_rows):
  """Encoder restricted to the given mesh rows and every grid row that sends to them."""
  keep = np.isin(g.g2m_receivers, mesh_rows)
  snd, rcv = g.g2m_senders[keep], g.g2m_receivers[keep]
  grid_rows = np.unique(snd)
  sub = {
      "grid_node_feats": g.grid_node_feats[grid_rows], "mesh_node_feats": g.mesh_node_feats[mesh_rows],
      "g2m_senders": np.searchsorted(grid_rows, snd), "g2m_receivers": np.searchsorted(mesh_rows, rcv),
      "g2m_edge_feats": g.g2m_edge_feats[keep],
  }
  return sub, grid_rows


def _subgraph_decoder(g, grid_rows):
  e = (grid_rows[:, None] * 3 + np.arange(3)[None, :]).reshape(-1)      # fan-in 3, receiver-sorted
  assert np.array_equal(g.m2g_receivers[e], np.repeat(grid_rows, 3))
  snd = g.m2g_senders[e]
  mesh_rows = np.unique(snd)
  sub = {
      "m2g_senders": np.searchsorted(mesh_rows, snd),
      "m2g_receivers": np.repeat(np.arange(grid_rows.shape[0]), 3),
      "m2g_edge_feats": g.m2g_edge_feats[e],
  }
  return sub, mesh_rows


def test_config2_quarter_degree_stagewise_matches_the_oracle():
  if torch.cuda.get_device_properties(0).total_memory < 75e9:
    pytest.skip("needs an 80 GB GPU")
  _threads()
  task = graphcast.TASK
  g, params, c_in, n_out = _setup(0.25, 6, task)
  assert (g.num_grid_nodes, g.num_mesh_nodes, len(g.g2m_senders)) == (1038240, 40962, 1618818)
  orc = oracle_gnn.Oracle(params, torch.float32)
  rng = np.random.default_rng(7)
  gen = torch.Generator(device="cuda:0").manual_seed(0)
  planes = torch.randn(c_in, g.num_grid_nodes, device="cuda:0", generator=gen)

  eng = engine.Engine(g, params, c_in=c_in, n_out=n_out, msg_steps=16, precision="bf16x3",
                      image_residual=False)
  eng.pack_inputs(planes)

  # ---- encoder -------------------------------------------------------------------------
  eng.run_stage("encode")
  torch.cuda.synchronize()
  vm1 = eng.mesh_rows_in_reference_order(eng.mesh_lat).cpu().numpy()   # [Nm, 512], reference node ids
  deg = np.bincount(g.g2m_receivers, minlength=g.num_mesh_nodes)
  assert deg.max() == 3753
  mesh_rows = np.unique(np.concatenate([np.argsort(deg)[-24:], rng.choice(g.num_mesh_nodes, 300, False)]))
  sub, grid_rows = _subgraph_encoder(g, mesh_rows)
  x_sub = planes[:, torch.as_tensor(grid_rows, device="cuda:0")].t().cpu().numpy()[:, None, :]
  vm1_ref, vg1_ref = orc.encoder(sub, x_sub)
  e_mesh = _rel(vm1[mesh_rows], vm1_ref[:, 0].numpy())
  vg1_gpu = eng.grid_lat[torch.as_tensor(grid_rows, device="cuda:0")].cpu().numpy()
  e_grid = _rel(vg1_gpu, vg1_ref[:, 0].numpy())
  print(f"config 2 encoder: {mesh_rows.size} mesh rows (max in-degree {deg[mesh_rows].max()}), "
        f"{grid_rows.size} grid rows: mesh latents {e_mesh:.3e}, grid latents {e_grid:.3e}")
  assert e_mesh <= TOL and e_grid <= TOL

  # ---- processor, in full --------------------------------------------------------------
  eng.run_stage("process_embed")
  for k in range(16):
    eng.run_stage("process_step", k)
  torch.cuda.synchronize()
  v_gpu = eng.mesh_rows_in_reference_order(eng.mesh_lat).cpu().numpy()
  v_ref = orc.processor(g.as_dict(), vm1[:, None, :])[:, 0].numpy()
  e_proc = _rel(v_gpu, v_ref)
  print(f"config 2 processor (16 steps, 327 660 edges, in full, from the GPU's encoder output): {e_proc:.3e}")
  assert e_proc <= TOL

  # ---- decoder -------------------------------------------------------------------------
  vg1_all = eng.grid_lat.clone()                        # decode updates grid_lat in place
  eng.run_stage("decode")
  torch.cuda.synchronize()
  n_lon = 1440
  rows = np.unique(np.concatenate([
      np.arange(0, 2 * n_lon), np.arange(g.num_grid_nodes - 2 * n_lon, g.num_grid_nodes),   # both poles
      np.arange(0, g.num_grid_nodes, n_lon)[::4], np.arange(n_lon // 2, g.num_grid_nodes, n_lon)[::4],
      rng.choice(g.num_grid_nodes, 3000, False)]))
  sub, mrows = _subgraph_decoder(g, rows)
  out_ref = orc.decoder(sub, v_gpu[mrows][:, None, :],
                        vg1_all[torch.as_tensor(rows, device="cuda:0")].cpu().numpy()[:, None, :])[:, 0].numpy()
  out_gpu = eng.grid_out[torch.as_tensor(rows, device="cuda:0"), :n_out].cpu().numpy()
  e_dec = _rel(out_gpu, out_ref)
  print(f"config 2 decoder: {rows.size} grid rows: outputs {e_dec:.3e}")
  assert e_dec <= TOL

  # ---- whole step: stages == gcb_forward, and the image-only latent layout -----------------
  full = eng.grid_out[:, :n_out].clone()
  eng.step()
  torch.cuda.synchronize()
  assert torch.equal(full, eng.grid_out[:, :n_out])
  del eng, vg1_all
  torch.cuda.empty_cache()
  eng2 = engine.Engine(g, params, c_in=c_in, n_out=n_out, msg_steps=16, precision="bf16x3",
                       image_residual=True)
  eng2.pack_inputs(planes)
  eng2.step()
  torch.cuda.synchronize()
  y2 = eng2.grid_out[:, :n_out]
  scale = float(full.abs().max())
  e_img = float((y2 - full).abs().max()) / scale
  e_img_rows = _rel(y2[torch.as_tensor(rows, device="cuda:0")].cpu().numpy(), out_ref)
  print(f"config 2 whole step, image-only latents vs fp32 masters: {e_img:.3e}; "
        f"decoder rows vs oracle (stage input from the master run): {e_img_rows:.3e}")
  assert e_img <= TOL
