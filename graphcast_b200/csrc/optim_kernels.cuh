// Device side of the training step: the weight packer (the device twin of gcb_pack_weight_host), the
// fp64 sum of squares of a flat buffer (the global gradient norm) and the fused AdamW update.
#pragma once
#include <stdint.h>

namespace gcb {

// Round-to-nearest-even bf16 of an fp32 value, bit for bit the host packer's f32_to_bf16_rne.
__device__ __forceinline__ uint16_t f32_to_bf16_rne_dev(float f) {
  uint32_t u = __float_as_uint(f);
  if ((u & 0x7fffffffu) > 0x7f800000u) return static_cast<uint16_t>((u >> 16) | 0x40);  // NaN
  const uint32_t lsb = (u >> 16) & 1u;
  u += 0x7fffu + lsb;
  return static_cast<uint16_t>(u >> 16);
}

// One block per (K-step ks, 256-column block h) of the image, 256 threads: thread r owns column
// h * 256 + r and writes its 2 x 8 hi and 2 x 8 lo values (16-byte stores) of the block
//   [hi | lo][K chunk c][256 rows][8 elements]
// (layout of gcb_pack_weight_host).  Element (kk, nn) of the logical W is w[kk * ld + nn], or
// w[nn * ld + kk] when `transpose`; outside [k_rows, n_cols] it is zero.  f32 (optional): the
// zero-padded fp32 [k, n] copy of W, row-major.
__global__ void __launch_bounds__(256)
pack_weight_kernel(const float* __restrict__ w, int ld, int transpose, int k_rows, int n_cols, int n,
                   uint16_t* __restrict__ img, float* __restrict__ f32) {
  const int ks = blockIdx.x, h = blockIdx.y, halves = gridDim.y;
  const int r = threadIdx.x;
  const int nn = h * 256 + r;
  uint16_t* hi = img + (static_cast<size_t>(ks) * halves + h) * 8192;
  uint16_t* lo = hi + 4096;
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    uint16_t hv[8], lv[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int kk = ks * 16 + c * 8 + j;
      float v = 0.f;
      if (kk < k_rows && nn < n_cols)
        v = transpose ? w[static_cast<size_t>(nn) * ld + kk] : w[static_cast<size_t>(kk) * ld + nn];
      hv[j] = f32_to_bf16_rne_dev(v);
      lv[j] = f32_to_bf16_rne_dev(__fsub_rn(v, __uint_as_float(static_cast<uint32_t>(hv[j]) << 16)));
      if (f32) f32[static_cast<size_t>(kk) * n + nn] = v;
    }
    const size_t off = (static_cast<size_t>(c) * 256 + r) * 8;
    uint4 ph, pl;
    ph.x = hv[0] | (static_cast<uint32_t>(hv[1]) << 16); ph.y = hv[2] | (static_cast<uint32_t>(hv[3]) << 16);
    ph.z = hv[4] | (static_cast<uint32_t>(hv[5]) << 16); ph.w = hv[6] | (static_cast<uint32_t>(hv[7]) << 16);
    pl.x = lv[0] | (static_cast<uint32_t>(lv[1]) << 16); pl.y = lv[2] | (static_cast<uint32_t>(lv[3]) << 16);
    pl.z = lv[4] | (static_cast<uint32_t>(lv[5]) << 16); pl.w = lv[6] | (static_cast<uint32_t>(lv[7]) << 16);
    *reinterpret_cast<uint4*>(hi + off) = ph;
    *reinterpret_cast<uint4*>(lo + off) = pl;
  }
}

// Fixed number of element groups of the sum of squares: every device splits the buffer the same way,
// so the fp64 result is bit-identical run to run and on any GPU.
constexpr int kSumGroups = 1024;

// partial[g] = sum of x[i]^2 (fp64; exact squares) over i = (t * kSumGroups + g) * 256 + thread,
// t = 0, 1, ...: each thread sums its elements in order, the block folds its lanes with a fixed
// butterfly and its eight warps in order.  No atomics.
__global__ void __launch_bounds__(256)
sum_squares_kernel(const float* __restrict__ x, long long n, double* __restrict__ partial) {
  __shared__ double warp_sum[8];
  double s = 0.0;
  const long long stride = static_cast<long long>(kSumGroups) * 256;
  for (long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x; i < n; i += stride) {
    const double v = static_cast<double>(x[i]);
    s = fma(v, v, s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double b = 0.0;
    for (int w = 0; w < 8; ++w) b += warp_sum[w];
    partial[blockIdx.x] = b;
  }
}

// out = sum over g = 0..kSumGroups-1 of partial[g]: thread t sums partial[4t .. 4t+3] in order, then
// the same fixed fold as above.  One block of 256 threads.
__global__ void __launch_bounds__(256)
sum_partials_kernel(const double* __restrict__ partial, double* __restrict__ out) {
  __shared__ double warp_sum[8];
  static_assert(kSumGroups == 4 * 256, "sum_partials_kernel folds four partials per thread");
  const int t = threadIdx.x;
  double s = ((partial[4 * t] + partial[4 * t + 1]) + partial[4 * t + 2]) + partial[4 * t + 3];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((t & 31) == 0) warp_sum[t >> 5] = s;
  __syncthreads();
  if (t == 0) {
    double b = 0.0;
    for (int w = 0; w < 8; ++w) b += warp_sum[w];
    *out = b;
  }
}

struct AdamWArgs {
  double lr, b1, b2, eps, eps_root, weight_decay, bc1, bc2, max_norm;
  long long n, n_decay;
};

// One element of clip_by_global_norm -> adamw (optax semantics), all in fp64 from the fp32 state.
__device__ __forceinline__ void adamw_element(const AdamWArgs& a, double clip, long long i, float& p,
                                              float g, float& m, float& v) {
  const double gd = static_cast<double>(g) * clip;
  const double mn = a.b1 * static_cast<double>(m) + (1.0 - a.b1) * gd;
  const double vn = a.b2 * static_cast<double>(v) + (1.0 - a.b2) * (gd * gd);
  const double pd = static_cast<double>(p);
  double u = (mn / a.bc1) / (sqrt(vn / a.bc2 + a.eps_root) + a.eps);
  if (i < a.n_decay) u += a.weight_decay * pd;
  p = static_cast<float>(pd - a.lr * u);
  m = static_cast<float>(mn);
  v = static_cast<float>(vn);
}

// The clip factor of optax.clip_by_global_norm from the device sum of squares: 1 while
// |g| < max_norm, else max_norm / |g| (a NaN norm propagates; max_norm <= 0 disables clipping).
__device__ __forceinline__ double clip_factor(const AdamWArgs& a, const double* sumsq) {
  if (!(a.max_norm > 0.0) || sumsq == nullptr) return 1.0;
  const double norm = sqrt(*sumsq);
  return norm < a.max_norm ? 1.0 : a.max_norm / norm;
}

// Grid-stride over float4 groups when every buffer is 16-byte aligned (vec4), else over elements.
__global__ void __launch_bounds__(256)
adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
             float* __restrict__ v, const double* __restrict__ sumsq, AdamWArgs a, int vec4) {
  const double clip = clip_factor(a, sumsq);
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long t0 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  long long tail = 0;
  if (vec4) {
    const long long n4 = a.n / 4;
    for (long long q = t0; q < n4; q += stride) {
      float4 pp = reinterpret_cast<const float4*>(p)[q];
      const float4 gg = reinterpret_cast<const float4*>(g)[q];
      float4 mm = reinterpret_cast<const float4*>(m)[q];
      float4 vv = reinterpret_cast<const float4*>(v)[q];
      adamw_element(a, clip, 4 * q + 0, pp.x, gg.x, mm.x, vv.x);
      adamw_element(a, clip, 4 * q + 1, pp.y, gg.y, mm.y, vv.y);
      adamw_element(a, clip, 4 * q + 2, pp.z, gg.z, mm.z, vv.z);
      adamw_element(a, clip, 4 * q + 3, pp.w, gg.w, mm.w, vv.w);
      reinterpret_cast<float4*>(p)[q] = pp;
      reinterpret_cast<float4*>(m)[q] = mm;
      reinterpret_cast<float4*>(v)[q] = vv;
    }
    tail = n4 * 4;
  }
  for (long long i = tail + t0; i < a.n; i += stride) {
    float pp = p[i], mm = m[i], vv = v[i];
    adamw_element(a, clip, i, pp, g[i], mm, vv);
    p[i] = pp;
    m[i] = mm;
    v[i] = vv;
  }
}

}  // namespace gcb
