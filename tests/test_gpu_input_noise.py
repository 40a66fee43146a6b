"""Input noise on the device (gcb_add_gaussian_noise, autoregressive.Predictor(noise_level=...)): the
kernel against the numpy restatement (tests/noise_oracle.py), the statistics of its draws, the noisy
loss and gradients against the noiseless path on noisy_inputs, the reference's rules on what is noised,
reproducible training steps, and the 0.25 degree gradient's memory peak."""
import gc
import zlib

import numpy as np
import pytest
import torch
from scipy import stats as sstats

import noise_oracle
from graphcast_b200 import (_native, autoregressive, graphcast, model_utils, normalization, optim)
from graphcast_b200 import xarray_shim as xs
from test_gpu_bptt import _data
from test_gpu_input_grads import _full_problem
from test_gpu_loss import _stats

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
SIGMA = 0.3


def _st():
  return torch.cuda.current_stream().cuda_stream


def _launch(segments, seed, fold, sigma):
  """segments: [(src tensor or None, dst tensor, offset, stream)], one launch."""
  table = (_native.NoiseSegment * len(segments))()
  for entry, (src, dst, offset, stream) in zip(table, segments):
    entry.src = None if src is None else src.data_ptr()
    entry.dst, entry.n, entry.offset, entry.stream = dst.data_ptr(), dst.numel(), offset, stream
  _native.check(_native.lib().gcb_add_gaussian_noise(table, len(segments), seed, fold, sigma, _st()),
                "gcb_add_gaussian_noise")


def _ulps(a, b):
  """|a - b| in float32 ulps (ordered integer distance)."""
  order = lambda x: np.where(x.view(np.int32) < 0, np.int64(-2**31) - x.view(np.int32).astype(np.int64),
                             x.view(np.int32).astype(np.int64))
  return np.abs(order(np.asarray(a, np.float32)) - order(np.asarray(b, np.float32)))


def _close_to_restatement(got, want, what):
  d = _ulps(got, want)
  assert d.max() <= 1, (what, int(d.max()))
  assert (d == 0).mean() >= 0.999, (what, float((d == 0).mean()))


# ---- the kernel ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fold", [0, 7])
def test_kernel_against_the_restatement(fold):
  rng = np.random.default_rng(fold)
  seed = 0x0123456789ABCDEF
  sigma = np.float32(0.7)
  # (n, offset, stream, src misalignment in floats, dst misalignment, with src)
  cases = [(1, 0, 1, 0, 0, True), (7, 0, 2, 1, 3, True), (1000, 2, 3, 2, 2, True),
           (4099, 2**32 + 1, 4, 3, 1, True), (65537, 3 * 2**32 - 2, 5, 0, 0, True),
           (513, 5, 6, 0, 1, False), (200003, 0, 7, 0, 0, True), (31, 2**40 + 3, 8, 1, 1, False)]
  segments, expected, keep = [], [], []
  for n, offset, stream, mis_src, mis_dst, with_src in cases:
    x = rng.standard_normal(n).astype(np.float32)
    src = None
    if with_src:
      buf = torch.empty(n + 8, device=DEV)
      src = buf[mis_src:mis_src + n]
      src.copy_(torch.from_numpy(x))
      keep.append(buf)
    dbuf = torch.full([n + 8], float("nan"), device=DEV)
    dst = dbuf[mis_dst:mis_dst + n]
    segments.append((src, dst, offset, stream))
    want = (noise_oracle.add_noise(x, sigma, seed, fold, stream, offset) if with_src
            else noise_oracle.noise_only(sigma, seed, fold, stream, offset, n))
    expected.append((dbuf, mis_dst, want))
  _launch(segments, seed, fold, float(sigma))
  first = [d.clone() for d, _, _ in expected]
  for (dbuf, mis, want), case in zip(expected, cases):
    got = dbuf.cpu().numpy()
    _close_to_restatement(got[mis:mis + case[0]], want, case)
    assert np.all(np.isnan(got[:mis])) and np.all(np.isnan(got[mis + case[0]:])), case   # no overrun
  _launch(segments, seed, fold, float(sigma))                   # deterministic
  for (dbuf, _, _), f in zip(expected, first):
    assert np.array_equal(dbuf.cpu().numpy(), f.cpu().numpy(), equal_nan=True)


def test_kernel_in_place_zero_sigma_and_segment_independence():
  x = torch.randn(10001, device=DEV)
  y = x.clone()
  _launch([(y, y, 0, 9)], 5, 1, 0.5)                            # in place
  z = torch.empty_like(x)
  _launch([(x, z, 0, 9)], 5, 1, 0.5)
  assert torch.equal(y, z)
  # the same elements drawn as a slice of a longer stream, alone or with other segments
  part = torch.empty(4000, device=DEV)
  other = torch.empty(77, device=DEV)
  _launch([(None, other, 3, 1), (x[17:4017], part, 17, 9)], 5, 1, 0.5)
  assert torch.equal(part, z[17:4017])
  # sigma = 0 leaves every non-zero value unchanged
  w = torch.empty_like(x)
  _launch([(x, w, 0, 9)], 5, 1, 0.0)
  assert torch.equal(w, x)


def test_kernel_statistics():
  n = 1 << 24
  draws = {}
  for key, (stream, fold) in {"a": (1, 0), "b": (2, 0), "c": (1, 1)}.items():
    d = torch.empty(n, device=DEV)
    _launch([(None, d, 0, stream)], 12345, fold, 1.0)
    draws[key] = d.double()
  z = draws["a"]
  bound = 5 / np.sqrt(n)
  mean, var = float(z.mean()), float(z.var())
  assert abs(mean) < bound, mean
  assert abs(var - 1) < 5 * np.sqrt(2 / n), var
  corr = lambda u, v: float(((u - u.mean()) * (v - v.mean())).mean() / (u.std() * v.std()))
  for lag in (1, 2, 3, 4):
    assert abs(corr(z[:-lag], z[lag:])) < bound, lag
  assert abs(corr(z, draws["b"])) < bound
  assert abs(corr(z, draws["c"])) < bound
  p = sstats.kstest(z.cpu().numpy(), "norm").pvalue
  assert p > 1e-3, p
  print(f"2^24 draws: mean {mean:.2e}, variance - 1 {var - 1:.2e}, KS p {p:.3f}")


def test_kernel_argument_checks():
  lib = _native.lib()
  d = torch.empty(8, device=DEV)
  table = (_native.NoiseSegment * 1)()
  table[0].dst, table[0].n = d.data_ptr(), 8
  assert lib.gcb_add_gaussian_noise(table, 1, 0, 0, float("nan"), _st()) == -1
  assert lib.gcb_add_gaussian_noise(table, _native.GCB_NOISE_MAX_SEGMENTS + 1, 0, 0, 1.0, _st()) == -1
  table[0].src = d.data_ptr() + 4                                # overlapping, not equal
  assert lib.gcb_add_gaussian_noise(table, 1, 0, 0, 1.0, _st()) == -1
  assert b"overlap" in lib.gcb_last_error()
  table[0].src, table[0].offset = None, -1
  assert lib.gcb_add_gaussian_noise(table, 1, 0, 0, 1.0, _st()) == -1


# ---- the loss and its gradients ------------------------------------------------------------------------
def _stacks(stack, precision, steps, seed=5):
  task = graphcast.TASK_13
  model, inputs, targets, forcings = _data(task, steps=steps, seed=seed)
  model.set_precision(precision)
  inner = model
  if stack == "norm":
    inner = normalization.InputsAndResiduals(model, *_stats(task, seed=1))
  noisy = autoregressive.Predictor(inner, noise_level=SIGMA, gradient_checkpointing=True)
  clean = autoregressive.Predictor(inner, gradient_checkpointing=True)
  return model, noisy, clean, inputs, targets, forcings


def _same_ds(a, b, what):
  assert set(a.keys()) == set(b.keys()), what
  for name in a.keys():
    assert np.array_equal(a.data_vars[name].values, b.data_vars[name].values, equal_nan=True), (what, name)


def _same_grads(a, b):
  assert set(a) == set(b)
  for module in a:
    for field in a[module]:
      assert np.array_equal(a[module][field], b[module][field]), (module, field)


@pytest.mark.parametrize("stack", ["plain", "norm"])
@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("steps", [2, 3])
def test_noisy_loss_and_gradients_are_the_noiseless_ones_at_the_noised_inputs(stack, precision, steps):
  model, noisy, clean, inputs, targets, forcings = _stacks(stack, precision, steps)
  key = np.array([0, 42], np.uint32)
  noised = noisy.noisy_inputs(inputs, targets, forcings, key)
  loss, diag = noisy.loss(inputs, targets, forcings, rng=key)
  ref_loss, ref_diag = clean.loss(noised, targets, forcings)
  assert np.array_equal(loss.values, ref_loss.values)
  _same_ds(diag, ref_diag, "diagnostics")
  plain_loss, _ = clean.loss(inputs, targets, forcings)
  assert not np.array_equal(loss.values, plain_loss.values)      # the noise reaches the loss
  got = noisy.loss_and_grads(inputs, targets, forcings, rng=42)   # the int seed of the same key
  want = clean.loss_and_grads(noised, targets, forcings)
  assert np.array_equal(got[0].values, want[0].values) and np.array_equal(got[0].values, loss.values)
  _same_grads(got[2], want[2])
  got = noisy.loss_and_input_grads(inputs, targets, forcings, rng=key)
  want = clean.loss_and_input_grads(noised, targets, forcings)
  assert np.array_equal(got[0].values, want[0].values)
  _same_ds(got[2], want[2], "input gradients")
  _same_ds(got[3], want[3], "forcing gradients")
  # the input gradients have the caller's variables, dims and shapes
  for name, v in inputs.data_vars.items():
    assert got[2].data_vars[name].dims == v.dims and got[2].data_vars[name].shape == v.shape


def test_one_target_time_ignores_the_noise():
  model, noisy, clean, inputs, targets, forcings = _stacks("norm", "bf16x3", 1)
  a = noisy.loss(inputs, targets, forcings, rng=3)
  b = clean.loss(inputs, targets, forcings)
  assert np.array_equal(a[0].values, b[0].values)
  ga = noisy.loss_and_grads(inputs, targets, forcings, rng=3)
  gb = clean.loss_and_grads(inputs, targets, forcings)
  assert np.array_equal(ga[0].values, gb[0].values)
  _same_grads(ga[2], gb[2])
  assert noisy.noisy_inputs(inputs, targets, forcings, 3) is inputs


# ---- what is noised -------------------------------------------------------------------------------------
def test_noisy_inputs_follow_the_reference_rules():
  model, noisy, clean, inputs, targets, forcings = _stacks("norm", "bf16x3", 2)
  before = {k: np.array(v.values, copy=True) for k, v in inputs.data_vars.items()}
  seed, fold = 2**64 - 3, 5
  noised = noisy.noisy_inputs(inputs, targets, forcings, seed, _noise_fold=fold)
  plan = dict(autoregressive.noise_plan(inputs, targets, forcings))
  sizes = {"batch": inputs.sizes["batch"], "lat": inputs.sizes["lat"], "lon": inputs.sizes["lon"]}
  for name, v in inputs.data_vars.items():
    assert np.array_equal(v.values, before[name]), name           # the caller's arrays are untouched
    out = noised.data_vars[name]
    assert out.dims == v.dims and out.shape == v.shape
    if name not in plan:                                           # constant inputs: unchanged
      assert out.data is v.data, name
      continue
    assert isinstance(out.data, torch.Tensor) and out.data.device == DEV
    assert out.data.dtype == torch.float32
    want = noise_oracle.add_noise(before[name], SIGMA, seed, fold, zlib.crc32(name.encode()))
    _close_to_restatement(out.values, want, name)
    # the noise has the variable's own shape: broadcast by the packing, constant where it is
    diff = (np.asarray(model_utils.variable_to_planes(xs.DataArray(out.values, out.dims), sizes),
                       np.float64)
            - np.asarray(model_utils.variable_to_planes(v, sizes), np.float64))
    if "lat" not in v.dims:
      assert np.all(diff == diff[:, :, :1]), name
    if "lon" not in v.dims:
      assert np.all(diff == diff[:, :, :, :1]), name
  assert {"year_progress_sin", "day_progress_cos", "toa_incident_solar_radiation"} <= set(plan)
  # host- and device-resident inputs give the same noise
  on_dev = xs.Dataset(coords=inputs.coords)
  for name, v in inputs.data_vars.items():
    on_dev[name] = xs.DataArray(torch.as_tensor(np.asarray(v.values)).to(DEV), v.dims)
  from_dev = noisy.noisy_inputs(on_dev, targets, forcings, seed, _noise_fold=fold)
  _same_ds(from_dev, noised, "device-resident inputs")
  for name in plan:                                                # not noised in place
    assert torch.equal(on_dev.data_vars[name].data.cpu(), torch.from_numpy(before[name]))
  # sigma = 0 is no noise: bit-identical to the noiseless path
  zero = autoregressive.Predictor(noisy._predictor, noise_level=0.0, gradient_checkpointing=True)
  assert np.array_equal(zero.loss(inputs, targets, forcings, rng=1)[0].values,
                        clean.loss(inputs, targets, forcings)[0].values)


# ---- training --------------------------------------------------------------------------------------------
def _trainer(params=None):
  task = graphcast.TASK_13
  model, inputs, targets, forcings = _data(task, steps=2, seed=5)
  if params is not None:
    model = graphcast.GraphCast(model._model_config, task, params=params)
  pred = autoregressive.Predictor(normalization.InputsAndResiduals(model, *_stats(task, seed=1)),
                                  noise_level=SIGMA, gradient_checkpointing=True)
  return pred, optim.AdamW(pred, learning_rate=1e-3, seed=3), (inputs, targets, forcings)


def test_training_steps_are_reproducible_and_resume_exactly():
  pred_a, opt_a, batch = _trainer()
  for _ in range(3):
    opt_a.step(*batch)
  final_a = opt_a.params()
  pred_b, opt_b, _ = _trainer()
  for _ in range(3):
    opt_b.step(*batch)
  _same_grads(opt_b.params(), final_a)
  del pred_b, opt_b
  # resumed after step 2 from state() and the master weights
  pred_c, opt_c, _ = _trainer()
  for _ in range(2):
    opt_c.step(*batch)
  state, params = opt_c.state(), opt_c.params()
  del pred_c, opt_c
  pred_d, opt_d, _ = _trainer(params)
  opt_d.load_state(state)
  opt_d.step(*batch)
  _same_grads(opt_d.params(), final_a)
  # every step draws fresh noise: fold = the step count
  first = pred_d.noisy_inputs(*batch, 3, _noise_fold=0)
  second = pred_d.noisy_inputs(*batch, 3, _noise_fold=1)
  name = "2m_temperature"
  assert not np.array_equal(first.data_vars[name].values, second.data_vars[name].values)
  # an explicit rng uses fold 0: the step's loss is the loss at noisy_inputs(rng) (weights unchanged
  # between the two calls below, as the loss is taken before the update)
  clean = autoregressive.Predictor(pred_d._predictor, gradient_checkpointing=True)
  want = clean.loss(pred_d.noisy_inputs(*batch, 11), *batch[1:])[0].values
  loss, _, _ = opt_d.step(*batch, rng=11)
  assert np.array_equal(loss.values, want)


# ---- full size -------------------------------------------------------------------------------------------
def test_full_size_noisy_gradient_and_peak_memory():
  """0.25 deg / 37 levels, two target times: the noisy loss_and_grads is the noiseless one at
  noisy_inputs, bit for bit, and its peak is within 0.1 GiB of the noiseless call's."""
  if torch.cuda.get_device_properties(0).total_memory < 75e9:
    pytest.skip("needs an 80 GB GPU")
  model, ar, inputs, targets, forcings = _full_problem(graphcast.TASK, 0.25, 6, 2)
  noisy = autoregressive.Predictor(ar._predictor, noise_level=SIGMA, gradient_checkpointing=True)
  ar.loss(inputs, targets, forcings)
  peaks, out = {}, {}
  for what, call in (("clean", lambda: ar.loss_and_grads(inputs, targets, forcings)),
                     ("noisy", lambda: noisy.loss_and_grads(inputs, targets, forcings, rng=7))):
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    out[what] = call()
    torch.cuda.synchronize()
    peaks[what] = torch.cuda.max_memory_allocated()
  noised = noisy.noisy_inputs(inputs, targets, forcings, 7)
  want = ar.loss_and_grads(noised, targets, forcings)
  del noised
  assert np.array_equal(out["noisy"][0].values, want[0].values)
  _same_grads(out["noisy"][2], want[2])
  assert not np.array_equal(out["noisy"][0].values, out["clean"][0].values)
  print(f"0.25 deg, T = 2: peak device memory loss_and_grads {peaks['clean'] / 2**30:.2f} GiB, with "
        f"noise {peaks['noisy'] / 2**30:.2f} GiB on {torch.cuda.get_device_name(0)}")
  assert peaks["noisy"] <= peaks["clean"] + 0.1 * 2**30
