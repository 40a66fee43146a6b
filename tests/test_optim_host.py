"""optim.AdamW without a GPU: the fp64 restatement of clip_by_global_norm -> adamw that the device
tests hold the kernels to, checked against torch.optim.AdamW; the flat layout; argument checks."""
import numpy as np
import pytest
import torch

from graphcast_b200 import casting, graphcast, optim


def restate(p, g, m, v, t, *, lr, b1, b2, eps, eps_root, wd, n_decay, max_norm):
  """One step of optax's clip_by_global_norm(max_norm) -> adamw on flat fp64 arrays, from the formulas:
  g <- g * max_norm / |g| when |g| >= max_norm (None: no clipping); m = b1 m + (1 - b1) g;
  v = b2 v + (1 - b2) g^2; u = (m / (1 - b1^t)) / (sqrt(v / (1 - b2^t) + eps_root) + eps), plus
  wd p for the first n_decay elements; p - lr u.  Returns (p, m, v, |g| before clipping)."""
  p, g, m, v = (np.asarray(a, np.float64) for a in (p, g, m, v))
  norm = np.sqrt(np.sum(g * g))
  if max_norm is not None and not norm < max_norm:
    g = g * (max_norm / norm)
  m = b1 * m + (1 - b1) * g
  v = b2 * v + (1 - b2) * g * g
  u = (m / (1 - b1 ** t)) / (np.sqrt(v / (1 - b2 ** t) + eps_root) + eps)
  u[:n_decay] += wd * p[:n_decay]
  return p - lr * u, m, v, norm


def _rel(a, b):
  return float(np.max(np.abs(a - b)) / np.max(np.abs(b)))


@pytest.mark.parametrize("max_norm", [None, 1e3, 0.5], ids=["no_clip", "clip_inactive", "clip_active"])
@pytest.mark.parametrize("n_decay", [0, 700, 1000])
def test_restatement_matches_torch_adamw(max_norm, n_decay):
  rng = np.random.default_rng(0)
  n = 1000
  hp = dict(lr=3e-3, b1=0.9, b2=0.95, eps=1e-8, eps_root=0.0, wd=0.1)
  p0 = rng.standard_normal(n)
  grads = [rng.standard_normal(n) * 0.1 for _ in range(5)]
  # torch: the decayed block and the rest as two parameter groups, the clip applied by hand
  a = torch.tensor(p0[:n_decay], dtype=torch.float64, requires_grad=True)
  b = torch.tensor(p0[n_decay:], dtype=torch.float64, requires_grad=True)
  groups = [{"params": [a], "weight_decay": hp["wd"]}, {"params": [b], "weight_decay": 0.0}]
  opt = torch.optim.AdamW([gr for gr in groups if gr["params"][0].numel()],
                          lr=hp["lr"], betas=(hp["b1"], hp["b2"]), eps=hp["eps"])
  p, m, v = p0.copy(), np.zeros(n), np.zeros(n)
  clipped = 0
  for t, g in enumerate(grads, start=1):
    p, m, v, norm = restate(p, g, m, v, t, n_decay=n_decay, max_norm=max_norm, **hp)
    c = 1.0 if max_norm is None or norm < max_norm else max_norm / norm
    clipped += c < 1.0
    a.grad = torch.tensor(g[:n_decay] * c, dtype=torch.float64)
    b.grad = torch.tensor(g[n_decay:] * c, dtype=torch.float64)
    opt.step()
    want = torch.cat([a.detach(), b.detach()]).numpy()
    assert _rel(p, want) <= 1e-12, t
    sa, sb = opt.state[a], opt.state[b]
    if n_decay:
      assert _rel(m[:n_decay], sa["exp_avg"].numpy()) <= 1e-12
    if n_decay < n:
      assert _rel(v[n_decay:], sb["exp_avg_sq"].numpy()) <= 1e-12
  assert (clipped == 5) == (max_norm == 0.5)


def test_restatement_eps_root():
  rng = np.random.default_rng(1)
  p, g = rng.standard_normal(64), rng.standard_normal(64)
  hp = dict(lr=1e-2, b1=0.9, b2=0.95, eps=1e-8, wd=0.0, n_decay=0, max_norm=None)
  q0 = restate(p, g, 0 * p, 0 * p, 1, eps_root=0.0, **hp)[0]
  q1 = restate(p, g, 0 * p, 0 * p, 1, eps_root=1e-3, **hp)[0]
  # first step: u = g / (sqrt(g^2 + eps_root) + eps)  (p - q cancels ~ |p| / |lr u| = 100x: 1e-12)
  np.testing.assert_allclose(p - q1, 1e-2 * g / (np.sqrt(g * g + 1e-3) + 1e-8), rtol=1e-12)
  assert np.all(np.abs(p - q1) < np.abs(p - q0))


def _params():
  cfg = graphcast.ModelConfig(10.0, 2, 512, 2, 1, 0.6)
  task = graphcast.TASK_13
  return cfg, task, graphcast.init_params(cfg, task, 20, seed=3)


def test_flat_layout_covers_every_parameter_once_decayed_first():
  _, _, params = _params()
  mask = lambda module, field: field == "w"
  layout = optim.FlatLayout.of(params, mask)
  keys = [(n, f) for n, f, _, _ in layout.entries]
  assert sorted(keys) == sorted((n, f) for n, v in params.items() for f in v)
  assert len(set(keys)) == len(keys)
  off = 0
  for name, f, o, shape in layout.entries:
    assert o == off and shape == np.shape(params[name][f])
    size = int(np.prod(shape))
    assert (o + size <= layout.n_decay) == (f == "w")        # every decayed tensor before the split
    off += size
  assert layout.size == off == sum(np.size(a) for v in params.values() for a in v.values())
  assert 0 < layout.n_decay < layout.size
  flat = layout.flatten(params)
  back = layout.unflatten(flat)
  for name, fields in params.items():
    for f, a in fields.items():
      assert back[name][f].dtype == np.float32 and np.array_equal(back[name][f], a)
  views = layout.views(flat)
  first = layout.entries[0]
  views[first[0]][first[1]][...] = 7.0                       # views, not copies
  assert np.all(flat[:int(np.prod(first[3]))] == 7.0)
  t = torch.from_numpy(layout.flatten(params))
  tv = layout.views(t)
  assert all(torch.equal(tv[n][f], torch.from_numpy(np.asarray(a))) for n, v in params.items()
             for f, a in v.items())
  every = optim.FlatLayout.of(params)                         # mask None: decay everything
  assert every.n_decay == every.size


class _NotGraphCast(graphcast.Predictor):
  def __call__(self, inputs, targets_template, forcings, **kw):
    raise AssertionError


def test_bad_arguments_and_unsupported_stacks_raise():
  cfg, task, params = _params()
  model = graphcast.GraphCast(cfg, task, params=params)
  optim.AdamW(model)                                          # no device work before the first step
  optim.AdamW(model, learning_rate=lambda count: 1e-3 / (1 + count), max_grad_norm=None,
              mask=lambda module, field: field != "offset")
  for kw in (dict(learning_rate=-1.0), dict(learning_rate=float("nan")), dict(b1=1.0), dict(b2=-0.1),
             dict(eps=-1e-8), dict(eps_root=-1.0), dict(weight_decay=-0.1), dict(mask=3),
             dict(max_grad_norm=float("inf"))):
    with pytest.raises(ValueError):
      optim.AdamW(model, **kw)
  with pytest.raises(NotImplementedError, match="GraphCast"):
    optim.AdamW(_NotGraphCast())
  with pytest.raises(NotImplementedError, match="GraphCast"):
    optim.AdamW(casting.Bfloat16Cast(_NotGraphCast()))
