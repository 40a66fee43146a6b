// Gaussian input noise of the multi-step training loss (autoregressive.Predictor(noise_level=...)):
// dst = src + sigma * z, z a standard normal drawn by a counter-based generator, so that the draw of
// an element depends only on (seed, fold, stream, element index) and not on the launch, the device or
// how the elements are split into launches.  The generator is restated in numpy in tests/noise_oracle.py.
//
// Element i of stream s: Philox4x32-10 with key (seed lo, seed hi) and counter (j lo, j hi, s, fold),
// j = i / 4, gives words w0..w3; u_k = (w_k + 0.5) 2^-32 in fp64 lies strictly inside (0, 1); Box-Muller
// in fp64 turns (u0, u1) into z0 = r cos 2 pi u1, z1 = r sin 2 pi u1 with r = sqrt(-2 ln u0), and (u2, u3)
// into z2, z3 the same way; each is rounded to fp32 once, and element i takes z_{i mod 4}.  Then
// dst = fl32(x + fl32(sigma z)) (src == NULL: dst = fl32(sigma z)).
#pragma once
#include <stdint.h>

namespace gcb {

// Segments of one launch (gcb_add_gaussian_noise), passed in the kernel parameters.
constexpr int kMaxNoiseSegments = 64;

struct NoiseSeg {
  const float* src;     // NULL: the noise alone
  float* dst;
  long long n;          // elements
  long long offset;     // element index of dst[0] in the stream
  long long group0;     // first counter j of the segment: offset / 4
  long long begin;      // first work item (one per counter j) of the segment in the launch
  unsigned stream;
  int vec4;             // src and dst 16-byte aligned at every counter group's first element
};

struct NoiseArgs {
  NoiseSeg seg[kMaxNoiseSegments];
  int nseg;
  unsigned key0, key1, fold;
  float sigma;
  long long items;      // work items of all segments
};

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, unsigned k0, unsigned k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const unsigned hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const unsigned hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c;
}

// (w + 0.5) 2^-32: exact in fp64, strictly inside (0, 1).
__device__ __forceinline__ double unit_open(unsigned w) {
  return (static_cast<double>(w) + 0.5) * 0x1p-32;
}

// The four normals of counter group j of `stream`.
__device__ __forceinline__ float4 normal4(const NoiseArgs& a, unsigned stream, long long j) {
  const unsigned long long uj = static_cast<unsigned long long>(j);
  const uint4 w = philox4x32_10(make_uint4(static_cast<unsigned>(uj), static_cast<unsigned>(uj >> 32),
                                           stream, a.fold), a.key0, a.key1);
  double s0, c0, s1, c1;
  const double r0 = sqrt(-2.0 * log(unit_open(w.x)));
  sincospi(2.0 * unit_open(w.y), &s0, &c0);
  const double r1 = sqrt(-2.0 * log(unit_open(w.z)));
  sincospi(2.0 * unit_open(w.w), &s1, &c1);
  return make_float4(static_cast<float>(r0 * c0), static_cast<float>(r0 * s0),
                     static_cast<float>(r1 * c1), static_cast<float>(r1 * s1));
}

__device__ __forceinline__ float noised(float x, float z, float sigma, bool has_src) {
  const float n = __fmul_rn(sigma, z);
  return has_src ? __fadd_rn(x, n) : n;
}

// One work item per (segment, counter group j): the thread draws the group's four normals and writes
// the elements of the group that lie in the segment, with one 16-byte load and store when the group is
// whole and the segment's pointers are aligned at group boundaries, else element by element.  Work
// items are numbered segment after segment; a grid-stride loop walks them in increasing order, so
// each thread finds its segment by advancing from the last one.
__global__ void __launch_bounds__(256)
gaussian_noise_kernel(const __grid_constant__ NoiseArgs a) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  int s = 0;
  for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < a.items;
       t += stride) {
    while (s + 1 < a.nseg && t >= a.seg[s + 1].begin) ++s;
    const NoiseSeg& g = a.seg[s];
    const long long j = g.group0 + (t - g.begin);
    const float4 z = normal4(a, g.stream, j);
    const long long first = 4 * j - g.offset;          // dst index of the group's first element
    const bool has_src = g.src != nullptr;
    if (g.vec4 && first >= 0 && first + 4 <= g.n) {
      float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
      if (has_src) x = *reinterpret_cast<const float4*>(g.src + first);
      float4 y;
      y.x = noised(x.x, z.x, a.sigma, has_src);
      y.y = noised(x.y, z.y, a.sigma, has_src);
      y.z = noised(x.z, z.z, a.sigma, has_src);
      y.w = noised(x.w, z.w, a.sigma, has_src);
      *reinterpret_cast<float4*>(g.dst + first) = y;
      continue;
    }
    const float zs[4] = {z.x, z.y, z.z, z.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const long long e = first + k;
      if (e < 0 || e >= g.n) continue;
      g.dst[e] = noised(has_src ? g.src[e] : 0.f, zs[k], a.sigma, has_src);
    }
  }
}

}  // namespace gcb
