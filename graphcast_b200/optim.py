"""AdamW on the device: the optax chain clip_by_global_norm(max_grad_norm) -> adamw(learning_rate, b1,
b2, eps, eps_root, weight_decay, mask), fused into the training step of a GraphCast predictor stack.

    opt = optim.AdamW(predictor, learning_rate=1e-4)
    loss, diagnostics, grad_norm = opt.step(inputs, targets, forcings)

One `step` is `predictor.loss_and_grads` with the gradients left on the device: the valid slices of
the backward pass's accumulators are copied into a flat fp32 gradient buffer, gcb_sum_squares reduces
it to the squared global norm (fp64, on the device), gcb_adamw_step clips and applies AdamW to the
flat fp32 master weights and moments in one pass, and Engine.load_params_device repacks the engine's
weights from the master weights on the device.  Nothing goes through the host but the loss and the
norm that `step` returns.

The input noise of an autoregressive.Predictor(noise_level=...) is keyed per step: `step(..., rng=None)`
draws with (seed, fold = count), so each step gets fresh noise, a run is reproducible from the
constructor's `seed`, and a run resumed with load_state() replays its noise exactly; an explicit `rng`
(an int seed or a uint32 [2] key, as autoregressive.Predictor.loss_and_grads takes it) uses fold 0.

Differences from optax: the master weights are fp32 whatever the predictor's precision, the gradient
is the one the kernels compute (see GraphCast.loss_and_grads), and `step` returns no next state.
GraphCast was trained with b1 = 0.9, b2 = 0.95, weight decay 0.1 and clipping at global
norm 32 (the paper's supplement); those are the defaults here.
"""

from __future__ import annotations

import weakref
from typing import Callable, Dict, List, Mapping, Optional, Tuple, Union

import numpy as np
import torch

from graphcast_b200 import _native
from graphcast_b200 import autoregressive
from graphcast_b200 import graphcast


class FlatLayout:
  """Where every parameter lives in the optimiser's flat fp32 buffers: the weight-decayed tensors
  first, then the others, each class in sorted (module, field) order, so that the decay mask is the
  split index `n_decay`.  entries: (module, field, offset, shape)."""

  def __init__(self, shapes: Mapping[str, Mapping[str, Tuple[int, ...]]],
               mask: Optional[Callable[[str, str], bool]] = None):
    keys = sorted((name, f) for name, fields in shapes.items() for f in fields)
    decay = [k for k in keys if mask is None or bool(mask(*k))]
    keep = [k for k in keys if not (mask is None or bool(mask(*k)))]
    self.entries: List[Tuple[str, str, int, Tuple[int, ...]]] = []
    off = 0
    for name, f in decay + keep:
      shape = tuple(int(s) for s in shapes[name][f])
      self.entries.append((name, f, off, shape))
      off += int(np.prod(shape))
    self.n_decay = sum(int(np.prod(shapes[name][f])) for name, f in decay)
    self.size = off

  @classmethod
  def of(cls, params, mask=None) -> "FlatLayout":
    return cls({name: {f: np.shape(a) for f, a in fields.items()} for name, fields in params.items()},
               mask)

  def views(self, flat) -> Dict[str, Dict[str, object]]:
    """A params-shaped dict of views into `flat` (numpy array or torch tensor of `size` elements)."""
    out: Dict[str, Dict[str, object]] = {}
    for name, f, off, shape in self.entries:
      out.setdefault(name, {})[f] = flat[off:off + int(np.prod(shape))].reshape(shape)
    return out

  def flatten(self, params) -> np.ndarray:
    """A params dict -> a new flat fp32 host array."""
    flat = np.empty([self.size], np.float32)
    for name, f, off, shape in self.entries:
      a = np.asarray(params[name][f], np.float32)
      if a.shape != shape:
        raise ValueError(f"{name}:{f} has shape {a.shape}, expected {shape}")
      flat[off:off + a.size] = a.reshape(-1)
    return flat

  def unflatten(self, flat: np.ndarray) -> Dict[str, Dict[str, np.ndarray]]:
    """A flat host array -> a params dict of new arrays."""
    return {name: {f: np.array(v) for f, v in fields.items()}
            for name, fields in self.views(np.asarray(flat)).items()}


def _graphcast_of(predictor) -> graphcast.GraphCast:
  """The GraphCast at the bottom of a predictor stack (graphcast.innermost_graphcast)."""
  p = graphcast.innermost_graphcast(predictor)
  if p is None:
    raise NotImplementedError(
        f"optim.AdamW trains a GraphCast predictor, directly or inside autoregressive.Predictor, "
        f"InputsAndResiduals or Bfloat16Cast; {type(predictor).__name__} holds none")
  return p


class AdamW:
  """optax.chain(clip_by_global_norm(max_grad_norm), adamw(...)) on the device for a predictor stack
  whose `loss_and_grads` runs on the GPU (see the module docstring).

  learning_rate: a float, or callable(count) -> float evaluated on the host with count = the number
    of steps already taken (0 for the first), as optax evaluates a schedule.
  mask: None = weight decay on every parameter (optax's default), or callable(module, field) -> bool,
    True for the parameters to decay.
  max_grad_norm: None (or <= 0) disables clipping.

  State: four flat fp32 device buffers of the parameter count (master weights, gradient, mu, nu),
  allocated by the first step from the predictor's current parameters."""

  def __init__(self, predictor, learning_rate: Union[float, Callable[[int], float]] = 1e-4, *,
               b1: float = 0.9, b2: float = 0.95, eps: float = 1e-8, eps_root: float = 0.0,
               weight_decay: float = 0.1, mask: Optional[Callable[[str, str], bool]] = None,
               max_grad_norm: Optional[float] = 32.0, seed: int = 0):
    if not callable(learning_rate):
      learning_rate = float(learning_rate)
      if not np.isfinite(learning_rate) or learning_rate < 0:
        raise ValueError(f"learning_rate must be a finite float >= 0 or a callable, not {learning_rate}")
    for name, x in (("b1", b1), ("b2", b2)):
      if not 0.0 <= float(x) < 1.0:
        raise ValueError(f"{name} must lie in [0, 1), not {x}")
    for name, x in (("eps", eps), ("eps_root", eps_root), ("weight_decay", weight_decay)):
      if not (np.isfinite(float(x)) and float(x) >= 0.0):
        raise ValueError(f"{name} must be a finite float >= 0, not {x}")
    if mask is not None and not callable(mask):
      raise ValueError("mask must be None or a callable(module, field) -> bool")
    if max_grad_norm is not None and not np.isfinite(float(max_grad_norm)):
      raise ValueError(f"max_grad_norm must be None or a finite float, not {max_grad_norm}")
    self.seed = autoregressive.rng_seed(seed)
    self._predictor = predictor
    self._model = _graphcast_of(predictor)
    self._lr = learning_rate
    self.b1, self.b2, self.eps, self.eps_root = float(b1), float(b2), float(eps), float(eps_root)
    self.weight_decay = float(weight_decay)
    self.max_grad_norm = None if max_grad_norm is None or max_grad_norm <= 0 else float(max_grad_norm)
    self._mask = mask
    self.layout: Optional[FlatLayout] = None
    self._count = 0
    self._bufs: Optional[Dict[str, torch.Tensor]] = None   # p, g, m, v (flat fp32), sumsq, workspace
    self._synced = None                                     # (weakref to the engine, weights_version)

  # -- state -------------------------------------------------------------------------------------
  def _ensure_state(self) -> None:
    if self._bufs is not None:
      return
    model = self._model
    params = model._params
    if params is None:
      raise ValueError("GraphCast has no parameters: pass params= or call set_params()")
    device = model.compute_device()
    self.layout = FlatLayout.of(params, self._mask)
    lib = _native.lib()
    p = torch.from_numpy(self.layout.flatten(params)).to(device)
    z = lambda: torch.zeros([self.layout.size], dtype=torch.float32, device=device)
    self._bufs = {"p": p, "g": z(), "m": z(), "v": z(),
                  "sumsq": torch.zeros([1], dtype=torch.float64, device=device),
                  "ws": torch.empty([lib.gcb_sum_squares_workspace_bytes()], dtype=torch.uint8,
                                    device=device)}
    self._p_views = self.layout.views(p)
    self._g_views = self.layout.views(self._bufs["g"])
    self.device = device

  @property
  def count(self) -> int:
    """Steps taken (optax's ScaleByAdamState.count)."""
    return self._count

  def params(self) -> Dict[str, Dict[str, np.ndarray]]:
    """The master weights: a host dict with the keys and shapes of the params, float32."""
    self._ensure_state()
    return self.layout.unflatten(self._bufs["p"].cpu().numpy())

  def state(self) -> dict:
    """{"count": int, "mu": host dict, "nu": host dict}: the AdamW moments, shaped like the params."""
    self._ensure_state()
    return {"count": self._count, "mu": self.layout.unflatten(self._bufs["m"].cpu().numpy()),
            "nu": self.layout.unflatten(self._bufs["v"].cpu().numpy())}

  def load_state(self, state: Mapping) -> None:
    """Restores what `state` returned (the master weights stay those of the predictor)."""
    self._ensure_state()
    count = int(state["count"])
    if count < 0:
      raise ValueError(f"count must be >= 0, not {count}")
    mu, nu = self.layout.flatten(state["mu"]), self.layout.flatten(state["nu"])
    self._bufs["m"].copy_(torch.from_numpy(mu))
    self._bufs["v"].copy_(torch.from_numpy(nu))
    self._count = count

  # -- the step ------------------------------------------------------------------------------------
  def _sync_engine(self) -> None:
    """The engine computes the gradient at the master weights: reload them if its weights changed
    since this optimiser last wrote them (or it is not the same engine)."""
    eng = self._model._engine
    if eng is None:
      if self._synced is not None:          # the engine was dropped: the next one is built from these
        self._model._params = self.params()
      return
    if self._synced is not None and self._synced[0]() is eng and self._synced[1] == eng.weights_version:
      return
    if eng.device != self.device:
      raise ValueError(f"the predictor's engine is on {eng.device}, the optimiser on {self.device}")
    eng.load_params_device(self._p_views)
    self._synced = (weakref.ref(eng), eng.weights_version)

  def step(self, inputs, targets, forcings, rng=None):
    """One training step on a batch: returns (loss, diagnostics, grad_norm), `loss` and `diagnostics`
    exactly as predictor.loss_and_grads returns them at the current weights, grad_norm the global
    norm of the gradient before clipping.  Raises NotImplementedError where loss_and_grads does.

    rng: the key of the input noise of an autoregressive.Predictor with noise_level (used with several
    target times only).  None draws with the optimiser's seed and the step count as the fold, so every
    step gets fresh noise and a run resumed from state() replays it; an explicit rng uses fold 0."""
    kwargs = {}
    if isinstance(self._predictor, autoregressive.Predictor):
      kwargs = (dict(rng=self.seed, _noise_fold=self._count) if rng is None
                else dict(rng=rng, _noise_fold=0))
    self._ensure_state()
    model = self._model
    self._sync_engine()
    lr = float(self._lr(self._count)) if callable(self._lr) else self._lr
    taken = []

    def sink(eng):
      if eng.device != self.device:
        raise ValueError(f"the predictor's engine is on {eng.device}, the optimiser on {self.device}")
      eng.grads_into(self._g_views)
      taken.append(eng)
    model._grad_sink = sink
    try:
      loss, diagnostics, _ = self._predictor.loss_and_grads(inputs, targets, forcings, **kwargs)
    finally:
      model._grad_sink = None
    if not taken:
      raise RuntimeError("the predictor's loss_and_grads did not compute its gradient on the device")
    eng = taken[0]
    b = self._bufs
    lib = _native.lib()
    n = self.layout.size
    with torch.cuda.device(self.device):
      st = torch.cuda.current_stream(self.device).cuda_stream
      _native.check(lib.gcb_sum_squares(b["g"].data_ptr(), n, b["ws"].data_ptr(), b["ws"].numel(),
                                        b["sumsq"].data_ptr(), st), "gcb_sum_squares")
      _native.check(lib.gcb_adamw_step(
          b["p"].data_ptr(), b["g"].data_ptr(), b["m"].data_ptr(), b["v"].data_ptr(), n,
          self.layout.n_decay, self._count + 1, lr, self.b1, self.b2, self.eps, self.eps_root,
          self.weight_decay, b["sumsq"].data_ptr(), self.max_grad_norm or 0.0, st), "gcb_adamw_step")
      eng.load_params_device(self._p_views)
    self._synced = (weakref.ref(eng), eng.weights_version)
    self._count += 1
    grad_norm = float(np.sqrt(b["sumsq"].item()))
    return loss, diagnostics, grad_norm
