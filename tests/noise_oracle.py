"""numpy restatement of the input-noise generator (gcb_add_gaussian_noise, csrc/noise_kernels.cuh), with
uint64 arithmetic and no loop over elements: Philox4x32-10, then u = (w + 0.5) 2^-32, then Box-Muller in
fp64 rounded once to fp32, then the fp32 add.  Test infrastructure: the GPU tests hold the kernel to it."""
import numpy as np

_MASK = np.uint64(0xFFFFFFFF)
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)


def philox4x32_10(counter, key):
  """counter: four uint32 arrays (broadcastable), key: two uint32 values -> the four uint32 words."""
  c0, c1, c2, c3 = (np.asarray(c, np.uint64) & _MASK for c in counter)
  k0, k1 = (np.asarray(k, np.uint64) & _MASK for k in key)
  for _ in range(10):
    p0, p1 = _M0 * c0, _M1 * c2                       # < 2^64: exact in uint64
    c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _MASK,
                      (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _MASK)
    k0, k1 = (k0 + _W0) & _MASK, (k1 + _W1) & _MASK
  return tuple(c.astype(np.uint32) for c in (c0, c1, c2, c3))


def unit_open(w):
  """(w + 0.5) 2^-32 in fp64: exact, strictly inside (0, 1)."""
  return (np.asarray(w, np.float64) + 0.5) * 2.0 ** -32


def sincospi(x):
  """(sin(pi x), cos(pi x)) in fp64 for x in [0, 2]: reduced exactly to r = x - n / 2, |r| <= 1/4,
  then rotated by n quarter turns, so that values near the zeros keep their relative accuracy."""
  x = np.asarray(x, np.float64)
  n = np.rint(2.0 * x)
  r = x - 0.5 * n                                     # exact: x is a multiple of 2^-32
  s, c = np.sin(np.pi * r), np.cos(np.pi * r)
  q = n.astype(np.int64) % 4
  sin = np.choose(q, [s, c, -s, -c])
  cos = np.choose(q, [c, -s, -c, s])
  return sin, cos


def normals(seed: int, fold: int, stream: int, offset: int, n: int) -> np.ndarray:
  """z of elements offset .. offset + n - 1 of `stream`: float32 [n]."""
  if n == 0:
    return np.zeros([0], np.float32)
  g0, g1 = offset // 4, (offset + n - 1) // 4
  j = np.arange(g1 - g0 + 1, dtype=np.uint64) + np.uint64(g0)
  w = philox4x32_10((j & _MASK, j >> np.uint64(32), np.uint64(stream), np.uint64(fold)),
                    (np.uint64(seed & 0xFFFFFFFF), np.uint64(seed >> 32)))
  u = [unit_open(x) for x in w]
  r0, r1 = np.sqrt(-2.0 * np.log(u[0])), np.sqrt(-2.0 * np.log(u[2]))
  s0, c0 = sincospi(2.0 * u[1])
  s1, c1 = sincospi(2.0 * u[3])
  z = np.stack([r0 * c0, r0 * s0, r1 * c1, r1 * s1], axis=1).astype(np.float32).reshape(-1)
  start = offset - 4 * g0
  return z[start:start + n]


def add_noise(x, sigma: float, seed: int, fold: int, stream: int, offset: int = 0) -> np.ndarray:
  """fl32(x + fl32(sigma z)) over the C-order elements of x, element k being stream element offset + k."""
  x = np.asarray(x, np.float32)
  z = normals(seed, fold, stream, offset, x.size).reshape(x.shape)
  return x + np.float32(sigma) * z


def noise_only(sigma: float, seed: int, fold: int, stream: int, offset: int, n: int) -> np.ndarray:
  """fl32(sigma z) of n elements (the kernel with src = NULL)."""
  return np.float32(sigma) * normals(seed, fold, stream, offset, n)
