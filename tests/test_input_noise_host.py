"""The host side of the input noise (autoregressive.Predictor(noise_level=...)): the numpy restatement of
the generator against published Philox4x32-10 answers, the range of its uniforms and normals, the
choice of the noised variables and their streams, and the argument checks that need no device.  CPU
only."""
import zlib

import numpy as np
import pytest

import noise_oracle
from graphcast_b200 import autoregressive, graphcast, optim, synthetic
from graphcast_b200 import xarray_shim as xs

TASKS = {"TASK": graphcast.TASK, "TASK_13": graphcast.TASK_13,
         "TASK_13_PRECIP_OUT": graphcast.TASK_13_PRECIP_OUT}


@pytest.mark.parametrize("counter, key, words", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_known_answers(counter, key, words):
  got = noise_oracle.philox4x32_10(counter, key)
  assert tuple(int(w) for w in got) == words


def test_uniforms_open_and_normals_bounded():
  for w in (0, 1, 0x7FFFFFFF, 0xFFFFFFFE, 0xFFFFFFFF):
    u = noise_oracle.unit_open(np.uint32(w))
    assert 0.0 < u < 1.0
  z = noise_oracle.normals(seed=2**63 + 5, fold=3, stream=11, offset=2**33 - 7, n=1 << 18)
  assert z.dtype == np.float32 and np.all(np.isfinite(z))
  assert np.abs(z).max() <= np.sqrt(66 * np.log(2))          # r at the smallest u = 2^-33
  # the extremes of the words give the extremes of r, exactly as stated
  u_min = noise_oracle.unit_open(np.uint32(0))
  assert u_min == 2.0 ** -33
  assert np.sqrt(-2.0 * np.log(u_min)) == pytest.approx(np.sqrt(66 * np.log(2)), rel=1e-15)


def test_normals_depend_on_the_element_index_only():
  whole = noise_oracle.normals(7, 1, 5, 0, 40)
  for off in (1, 2, 3, 4, 13):
    assert np.array_equal(noise_oracle.normals(7, 1, 5, off, 40 - off - 1), whole[off:-1])
  assert not np.array_equal(noise_oracle.normals(7, 2, 5, 0, 40), whole)     # fold
  assert not np.array_equal(noise_oracle.normals(7, 1, 6, 0, 40), whole)     # stream
  assert not np.array_equal(noise_oracle.normals(8, 1, 5, 0, 40), whole)     # seed


def test_sincospi_restatement_near_its_zeros():
  x = np.array([0.0, 0.5, 1.0, 1.5, 2.0, 2.0 ** -31, 1.0 - 2.0 ** -31, 1.0 + 2.0 ** -31])
  s, c = noise_oracle.sincospi(x)
  assert np.array_equal(s[:5], [0.0, 1.0, 0.0, -1.0, 0.0]) and np.array_equal(c[:5], [1, 0, -1, 0, 1])
  np.testing.assert_allclose(s[5:], [np.pi * 2.0 ** -31, np.pi * 2.0 ** -31, -np.pi * 2.0 ** -31],
                             rtol=1e-15)


@pytest.mark.parametrize("name", sorted(TASKS))
def test_streams_are_distinct_for_every_input(name):
  task = TASKS[name]
  names = sorted(set(task.input_variables) | set(task.forcing_variables) | set(task.target_variables))
  streams = {zlib.crc32(n.encode()) for n in names}
  assert len(streams) == len(names)


@pytest.mark.parametrize("name", sorted(TASKS))
def test_noised_variables_are_the_time_dependent_inputs(name):
  task = TASKS[name]
  inputs, targets, forcings = synthetic.make_example(task, 30.0, batch=2, num_target_steps=2, seed=1)
  plan = autoregressive.noise_plan(inputs, targets, forcings)
  names = [n for n, _ in plan]
  want = [n for n in inputs.keys() if n in targets or n in forcings]
  assert names == want
  static = {n for n, v in inputs.data_vars.items() if "time" not in v.dims}
  assert {"geopotential_at_surface", "land_sea_mask"} <= static
  assert set(inputs.keys()) - set(names) == static
  for n in names:
    assert "time" in inputs.data_vars[n].dims
  assert not set(names) & set(targets.keys()) - set(inputs.keys())
  # the forcings that are inputs (solar radiation, progress features) are noised too
  assert set(task.forcing_variables) & set(inputs.keys()) <= set(names)
  assert [s for _, s in plan] == [zlib.crc32(n.encode()) for n in names]
  # own-shape noise: the year progress has one value per (batch, time), the day progress one per
  # (batch, time, lon), each broadcast over the rest of the grid by the packing, noise included
  for n, dims in (("year_progress_sin", ("batch", "time")), ("year_progress_cos", ("batch", "time")),
                  ("day_progress_sin", ("batch", "time", "lon")),
                  ("day_progress_cos", ("batch", "time", "lon"))):
    assert n in names
    v = inputs.data_vars[n]
    assert v.dims == dims
    x = np.asarray(v.values, np.float32)
    noised = noise_oracle.add_noise(x, 0.5, 9, 0, zlib.crc32(n.encode()))
    assert noised.shape == x.shape and np.all(noised != x)


def _collision_example():
  """Two time-dependent inputs whose names have the same crc32 (a known pair)."""
  assert zlib.crc32(b"plumless") == zlib.crc32(b"buckeroo")
  coords = {"lat": np.arange(3.0), "lon": np.arange(4.0), "time": np.arange(2)}
  data = lambda: xs.DataArray(np.zeros([1, 2, 3, 4], np.float32), ("batch", "time", "lat", "lon"))
  inputs = xs.Dataset({"plumless": data(), "buckeroo": data()}, coords)
  targets = xs.Dataset({"plumless": data(), "buckeroo": data()}, coords)
  return inputs, targets, xs.Dataset(coords={"time": np.arange(2)})


def _model():
  cfg = graphcast.ModelConfig(30.0, 1, 512, 16, 1, 0.6)
  return graphcast.GraphCast(cfg, graphcast.TASK_13)


def test_noise_level_validation():
  for bad in (float("nan"), float("inf"), -float("inf")):
    with pytest.raises(ValueError, match="finite"):
      autoregressive.Predictor(_model(), noise_level=bad)
  for off in (None, 0, 0.0):
    p = autoregressive.Predictor(_model(), noise_level=off)
    assert p._noise_level is None
  assert autoregressive.Predictor(_model(), noise_level=0.25)._noise_level == 0.25


def test_rng_validation():
  assert autoregressive.rng_seed(0) == 0
  assert autoregressive.rng_seed(2**64 - 1) == 2**64 - 1
  assert autoregressive.rng_seed(np.uint64(7)) == 7
  # jax.random.PRNGKey(seed) layout: [seed >> 32, seed & 0xffffffff]
  assert autoregressive.rng_seed(np.array([1, 2], np.uint32)) == (1 << 32) | 2
  assert autoregressive.rng_seed(np.array([0, 42], np.uint32)) == 42
  for bad in (-1, 2**64, True, np.array([1, 2], np.int64), np.zeros(3, np.uint32),
              np.zeros([1, 2], np.uint32), 1.5, "key"):
    with pytest.raises(ValueError):
      autoregressive.rng_seed(bad)


def test_missing_or_malformed_rng_raises_before_any_device_work():
  inputs, targets, forcings = synthetic.make_example(graphcast.TASK_13, 30.0, batch=1,
                                                     num_target_steps=2, seed=1)
  p = autoregressive.Predictor(_model(), noise_level=0.1, gradient_checkpointing=True)
  for call in (p.loss, p.loss_and_grads, p.loss_and_input_grads):
    with pytest.raises(ValueError, match="needs an rng"):
      call(inputs, targets, forcings)
    with pytest.raises(ValueError, match="rng"):
      call(inputs, targets, forcings, rng=np.array([1, 2, 3], np.uint32))
  with pytest.raises(ValueError, match="needs an rng"):
    p.noisy_inputs(inputs, targets, forcings, None)
  with pytest.raises(ValueError, match="fold"):
    p.noisy_inputs(inputs, targets, forcings, 1, _noise_fold=2**32)


def test_stream_collision_raises():
  inputs, targets, forcings = _collision_example()
  with pytest.raises(ValueError, match="same noise stream"):
    autoregressive.noise_plan(inputs, targets, forcings)
  p = autoregressive.Predictor(_model(), noise_level=0.1)
  with pytest.raises(ValueError, match="same noise stream"):
    p.noisy_inputs(inputs, targets, forcings, 3)
  # one of the pair alone is fine
  one = xs.Dataset({"plumless": inputs.data_vars["plumless"]}, inputs.coords)
  assert [n for n, _ in autoregressive.noise_plan(one, targets, forcings)] == ["plumless"]


def test_no_noise_without_noise_level_or_with_one_target_time():
  inputs, targets, forcings = synthetic.make_example(graphcast.TASK_13, 30.0, batch=1,
                                                     num_target_steps=2, seed=1)
  assert autoregressive.Predictor(_model()).noisy_inputs(inputs, targets, forcings, 1) is inputs
  one = targets.isel(time=slice(0, 1))
  p = autoregressive.Predictor(_model(), noise_level=0.1)
  assert p.noisy_inputs(inputs, one, forcings.isel(time=slice(0, 1)), None) is inputs


def test_noise_needs_a_graphcast_in_the_stack():
  inputs, targets, forcings = synthetic.make_example(graphcast.TASK_13, 30.0, batch=1,
                                                     num_target_steps=2, seed=1)

  class Other:
    pass
  p = autoregressive.Predictor(Other(), noise_level=0.1)
  with pytest.raises(NotImplementedError, match="GraphCast"):
    p.noisy_inputs(inputs, targets, forcings, 1)
  with pytest.raises(NotImplementedError, match="GraphCast"):
    p.loss(inputs, targets, forcings, rng=1)


def test_adamw_seed_validation():
  p = autoregressive.Predictor(_model(), noise_level=0.1, gradient_checkpointing=True)
  assert optim.AdamW(p).seed == 0
  assert optim.AdamW(p, seed=3).seed == 3
  for bad in (-1, 2**64):
    with pytest.raises(ValueError):
      optim.AdamW(p, seed=bad)
