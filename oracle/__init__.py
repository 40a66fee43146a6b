"""CPU oracle for the GraphCast hot path -- TEST INFRASTRUCTURE ONLY.

This package restates, on the CPU (numpy / torch-CPU, float32 or float64), the
arithmetic of the reference's GraphCast single 6 h step and the host logic
around it.  Every function cites the reference file:line it follows
(paths relative to the root of the reference, google-deepmind/graphcast).

Who may import it: `tests/`, `__graft_entry__.smoke()` and `bench.py`'s
`cpu_baseline` / `--impl reference` legs -- as the checker or the reported CPU
baseline, never as the product.  Nothing under `graphcast_b200/` imports it;
the product path fails loudly when its CUDA library is missing.

Pinning status (SURVEY.md section 8c):
  * static graph (icosahedral mesh, faces->edges order, grid coordinates):
    PINNED against the reference's own known-answer tests
    (icosahedral_mesh_test.py:36-94, grid_mesh_connectivity_test.py:23-47) and
    against golden vectors generated here by importing the reference's
    `icosahedral_mesh` module (tests/golden/, script tests/golden/make_golden.py).
  * structural features (node features, receiver-local edge features of the three
    graphs; `oracle/graph_features.py`) and the grid2mesh radius query: PINNED
    against golden vectors computed by the reference's own numpy code
    (`model_utils.py`, `legacy/grid_mesh_connectivity.py`, imported with jax /
    xarray / trimesh stubbed out; tests/test_reference_geometry_golden.py).
  * channel packing order and checkpoint format (product-side host logic):
    PINNED against the reference's `dataset_to_stacked` / `stacked_to_dataset`
    and `checkpoint.dump` (tests/golden/reference_packing.npz,
    reference_checkpoint.npz).
  * GNN forward (`oracle/gnn.py`): PINNED against the reference's own wiring, executed:
    tests/golden/make_golden.py imports and runs weathernext1_graph/graphcast.py
    (`_maybe_init`, `_run_grid2mesh_gnn`, `_run_mesh_gnn`, `_run_mesh2grid_gnn`),
    legacy/deep_typed_graph_net.py and typed_graph_net.py on numpy stand-ins for jax / jraph /
    haiku / chex (tests/golden/numpy_standins.py); the oracle reproduces its outputs and
    intermediate latents to 5.5e-7 (tests/test_reference_gnn_golden.py).  Only the third-party
    primitives (Linear, LayerNorm, swish, segment_sum, concatenated_args) are restated there.
  * `GraphCast.__call__` I/O conversion, normalisation wrapper (`InputsAndResiduals`) and
    rollout (`chunked_prediction_generator`, `_get_next_inputs`): the product's host logic is
    PINNED the same way -- the reference functions are executed on numpy-backed stand-in
    datasets (tests/golden/reference_{gnn_forward,normalization,rollout}.npz).
  * Not exercised anywhere: the real jax / haiku / jraph / xarray packages (not installable in
    this image).  The stand-ins restate only the primitives the executed reference code calls;
    they are listed at the top of tests/golden/numpy_standins.py and make_golden.py.
"""
