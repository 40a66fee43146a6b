"""`casting.Bfloat16Cast` of the reference (weathernext/utils/casting.py:31-65) for this backend.

The reference wrapper casts inputs, parameters and activations to bfloat16 and the predictions
back to the targets' dtype, so that the whole model runs in bf16 on the accelerator.  Here the
numerics are a property of the CUDA kernels: wrapping a `GraphCast` selects its "bf16" mode
(one bf16 tensor-core product per MAC, fp32 accumulation, fp32 latents and LayerNorm) instead
of the default 3-product "bf16x3" parity mode.  This is a defined arithmetic of its own -- both
operands of every contraction rounded to bfloat16, everything else in fp32 (latents as two bf16) --
tested against an oracle that emulates exactly that (`oracle.gnn.Bf16OperandOracle`,
tests/test_gpu_model.py::test_bf16_mode_matches_its_emulation, <= 2e-4).  It is NOT the reference's
all-bf16 execution, where XLA additionally rounds every activation, the LayerNorm and -- outside
grid2mesh (graphcast.py:215,232,260) -- the aggregation to bf16: those rounding points depend on
XLA's fusion decisions and cannot be reproduced bit for bit, and two bf16 implementations of a
40-GEMM-deep chain differ by far more than any tolerance worth stating.  The op-by-op form of that
execution is emulated too (`oracle.gnn.ReferenceBf16Oracle`, the jnp semantics of every op with
bfloat16 inputs and parameters): against the exact step it is off by 8.7e-3 where this mode is off by
6.0e-3 on the same case (tests/test_oracle.py asserts ours <= theirs; 5e-3 to 7e-3 measured on the GPU
at 0.25 degree), so switching to this backend does not lose accuracy against what `Bfloat16Cast` gives
in the reference.  Inputs and predictions stay float32 Datasets, which is what the reference wrapper
returns.

The same holds for `loss` / `loss_and_predictions` (reference :67-117): the reference evaluates the
loss in bfloat16 and casts it back to the targets' dtype; here the outputs of the bf16 step are
compared with the targets in float32 and the weighted squared errors are summed in float64
(`gcb_output_loss`), so the loss is not rounded to bfloat16 anywhere.

To keep the demo's wrapper stack working unchanged,

    predictor = graphcast.GraphCast(model_config, task_config, params=...)
    predictor = casting.Bfloat16Cast(predictor)
    predictor = normalization.InputsAndResiduals(predictor, ...)

`Bfloat16Cast(graphcast_model)` returns the SAME `GraphCast` object (switched to "bf16"), so
that `InputsAndResiduals` still recognises it and fuses the normalisation into the pack /
unpack kernels.  Any other predictor is wrapped in a pass-through object (there is nothing to
cast on the host)."""

from __future__ import annotations

from graphcast_b200 import graphcast


class Bfloat16Cast(graphcast.Predictor):
  """See the module docstring.  `enabled=False` leaves the predictor untouched (reference :37-43)."""

  def __new__(cls, predictor, enabled: bool = True):
    if isinstance(predictor, graphcast.GraphCast):
      if enabled:
        predictor.set_precision("bf16")
      return predictor
    return super().__new__(cls)

  def __init__(self, predictor, enabled: bool = True):
    self._predictor = predictor
    self._enabled = enabled

  def __call__(self, inputs, targets_template, forcings, **kwargs):
    return self._predictor(inputs, targets_template, forcings, **kwargs)

  def loss(self, inputs, targets, forcings, **kwargs):
    return self._predictor.loss(inputs, targets, forcings, **kwargs)

  def loss_and_predictions(self, inputs, targets, forcings, **kwargs):
    return self._predictor.loss_and_predictions(inputs, targets, forcings, **kwargs)

  def loss_and_grads(self, inputs, targets, forcings, **kwargs):
    return self._predictor.loss_and_grads(inputs, targets, forcings, **kwargs)
