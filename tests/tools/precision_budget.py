#!/usr/bin/env python
"""Per-layer-group precision budget of the GraphCast step (CPU, test infrastructure: uses oracle/).

VERDICT r1 item 6 asked whether some layers can run with fewer than the three bf16 tensor-core
products per MAC (bf16x3: a_hi*w_hi + a_hi*w_lo + a_lo*w_hi) inside the 1e-4 parity budget.  This tool
answers it without a GPU: an fp64 oracle in which ONE group of MLPs computes its contractions with
emulated reduced products while everything else stays exact, on a real workload graph with all 16
message-passing steps; the error is max|y - y_ref| / max|y_ref| of the step output against the exact
fp64 oracle (the parity metric of tests/ and bench.py).

  modes:  x1  = one product, both operands rounded to bf16          (1/3 of the MMAs)
          x2w = two products, weights rounded to bf16 (a_hi+a_lo)*w_hi   (2/3 of the MMAs)
          x2a = two products, activations rounded to bf16 a_hi*(w_hi+w_lo)
          x3  = the product's parity mode (drops only a_lo*w_lo), for scale

  python tests/tools/precision_budget.py --workload sample_2deg_13lvl [--out precision_budget.md]
"""
import argparse
import os
import sys
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)

from graphcast_b200 import graph as graph_lib, graphcast, synthetic   # noqa: E402
from oracle import gnn                                                # noqa: E402

WORKLOADS = {"graphcast_small_1deg_13lvl": (1.0, 5, "TASK_13"), "sample_2deg_13lvl": (2.0, 4, "TASK_13"),
             "tiny_4deg_13lvl": (4.0, 3, "TASK_13")}

# group name -> substrings of the MLP stem (oracle/gnn.py mlp_name) that select it
GROUPS = {
    "edge-feature embedders (K=4 -> 512 -> 512; g2m, mesh, m2g)": ["encoder_edges_"],
    "grid node embedder (K=c_in+3)": ["grid2mesh_gnn/~_networks_builder/encoder_nodes_grid_nodes"],
    "mesh node embedder": ["grid2mesh_gnn/~_networks_builder/encoder_nodes_mesh_nodes"],
    "grid2mesh edge MLP (K=1536)": ["grid2mesh_gnn/~_networks_builder/processor_edges_0_"],
    "grid2mesh node MLPs (mesh K=1024, grid K=512)": ["grid2mesh_gnn/~_networks_builder/processor_nodes_0_"],
    "processor edge MLPs, 16 steps (K=1536)": ["mesh_gnn/~_networks_builder/processor_edges_"],
    "processor node MLPs, 16 steps (K=1024)": ["mesh_gnn/~_networks_builder/processor_nodes_"],
    "mesh2grid edge MLP (K=1536)": ["mesh2grid_gnn/~_networks_builder/processor_edges_0_"],
    "mesh2grid grid-node MLP (K=1024)": ["mesh2grid_gnn/~_networks_builder/processor_nodes_0_"],
    "output MLP (512 -> 512 -> n_out, no LayerNorm)": ["decoder_nodes_"],
    "ALL layers": [""],
}


def _bf16(t):
  return t.to(torch.float32).to(torch.bfloat16).to(t.dtype)


class SelectiveOracle(gnn.Oracle):
  """fp64 oracle; MLPs whose stem contains one of `select` use `mode` products."""

  def __init__(self, params, select, mode):
    super().__init__(params, torch.float64)
    self.select, self.mode, self._on = select, mode, False
    self.hits = 0

  def mlp(self, stem, args, use_layer_norm=True):
    self._on = any(s in stem for s in self.select)
    self.hits += self._on
    try:
      return super().mlp(stem, args, use_layer_norm)
    finally:
      self._on = False

  def matmul(self, x, w):
    if not self._on:
      return x @ w
    # the device splits fp32 values: start from the fp32 rounding of both operands
    x, w = x.to(torch.float32).to(self.dtype), w.to(torch.float32).to(self.dtype)
    xh, wh = _bf16(x), _bf16(w)
    if self.mode == "x1":
      return xh @ wh
    xl, wl = _bf16(x - xh), _bf16(w - wh)
    if self.mode == "x2w":
      return (xh + xl) @ wh
    if self.mode == "x2a":
      return xh @ (wh + wl)
    if self.mode == "x3":
      return xh @ wh + xh @ wl + xl @ wh
    raise ValueError(self.mode)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--workload", default="sample_2deg_13lvl", choices=sorted(WORKLOADS))
  ap.add_argument("--modes", default="x1,x2w,x2a,x3")
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  res, mesh, task_name = WORKLOADS[args.workload]
  task = getattr(graphcast, task_name)
  lat, lon = synthetic.grid_coords(res)
  g = graph_lib.cached_static_graph(grid_lat=lat, grid_lon=lon, mesh_size=mesh,
                                    radius_query_fraction_edge_length=0.6).as_dict()
  c_in, n_out = synthetic.num_input_channels(task), graphcast.num_outputs(task)
  params = gnn.init_params(c_in=c_in, n_out=n_out, msg_steps=16, seed=1)
  x = np.random.default_rng(0).standard_normal((g["grid_node_feats"].shape[0], 1, c_in)).astype(np.float32)
  t0 = time.time()
  ref = gnn.Oracle(params, torch.float64).forward(g, x)
  scale = ref.abs().max().item()
  print(f"# exact fp64 step: {time.time() - t0:.1f} s", file=sys.stderr)
  modes = args.modes.split(",")
  rows = []
  for name, select in GROUPS.items():
    errs = []
    for mode in modes:
      o = SelectiveOracle(params, select, mode)
      y = o.forward(g, x)
      errs.append((y - ref).abs().max().item() / scale)
      assert o.hits > 0, name
    rows.append((name, errs))
    print(name, " ".join(f"{m}={e:.2e}" for m, e in zip(modes, errs)), file=sys.stderr, flush=True)
  lines = [f"# Precision budget per layer group -- {args.workload}, 16 message-passing steps, Haiku-default weights",
           "",
           "Error = max|y - y_ref| / max|y_ref| of the step output vs the exact fp64 oracle when ONLY the named",
           "group computes its contractions with the reduced products (tests/tools/precision_budget.py; parity gate 1e-4).",
           "",
           "| layer group | " + " | ".join(modes) + " |", "|---|" + "---|" * len(modes)]
  for name, errs in rows:
    lines.append(f"| {name} | " + " | ".join(f"{e:.2e}" for e in errs) + " |")
  text = "\n".join(lines) + "\n"
  print(text)
  if args.out:
    with open(args.out, "w") as f:
      f.write(text)


if __name__ == "__main__":
  main()
