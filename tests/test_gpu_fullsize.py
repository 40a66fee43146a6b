"""Full-size (GraphCast 0.25 deg, 721x1440, 37 levels, mesh 6, 16 steps) checks that do not
need the CPU oracle (a 29 TFLOP step does not finish in seconds on the host):
  * the tensor-core bf16x3 path against the exact-fp32 CUDA-core arm of the same library
    (itself <= 2e-6 vs the fp64 oracle on the small cases) over the WHOLE step output;
  * bitwise determinism of two runs;
  * the bf16 single-product mode stays within its documented error.
"""
import numpy as np
import pytest
import torch

from graphcast_b200 import engine, graph as graph_lib, graphcast, synthetic

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def full_engine():
  if torch.cuda.get_device_properties(0).total_memory < 75e9:
    pytest.skip("needs an 80 GB GPU")
  task = graphcast.TASK
  lat, lon = synthetic.grid_coords(0.25)
  g = graph_lib.cached_static_graph(grid_lat=lat, grid_lon=lon, mesh_size=6,
                                    radius_query_fraction_edge_length=0.6)
  cfg = graphcast.ModelConfig(0.25, 6, 512, 16, 1, 0.6)
  c_in = synthetic.num_input_channels(task)
  params = graphcast.init_params(cfg, task, c_in, seed=1)
  eng = engine.Engine(g, params, c_in=c_in, n_out=graphcast.num_outputs(task), msg_steps=16,
                      precision="bf16x3")
  planes = torch.randn(c_in, g.num_grid_nodes, device="cuda:0",
                       generator=torch.Generator(device="cuda:0").manual_seed(0))
  return eng, planes


def _run(eng, planes):
  eng.pack_inputs(planes)
  eng.step()
  torch.cuda.synchronize()
  return eng.grid_out[:, :eng.n_out].clone()


def test_full_size_parity_determinism_and_bf16_error(full_engine):
  eng, planes = full_engine
  assert (eng.num_grid, eng.num_mesh) == (1038240, 40962)
  y = _run(eng, planes)
  assert torch.isfinite(y).all()
  assert torch.equal(y, _run(eng, planes))                 # bitwise deterministic
  eng.set_precision("fp32_simt")
  ref = _run(eng, planes)
  eng.set_precision("bf16")
  y16 = _run(eng, planes)
  eng.set_precision("bf16x3")
  scale = float(ref.abs().max())
  err = float((y - ref).abs().max()) / scale
  err16 = float((y16 - ref).abs().max()) / scale
  print(f"full-size step: bf16x3 vs fp32 arm max-abs rel err {err:.3e}; bf16 {err16:.3e}")
  assert err <= 1e-4
  assert err16 <= 5e-2
