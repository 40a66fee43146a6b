// FP32 CUDA-core arm of the fused layer (GCB_PREC_FP32_SIMT).  Same contract as
// the tensor-core kernel in mlp_tc.cuh (segments, gather, fan-in sum, bias,
// swish, LayerNorm, residual), exact fp32 FFMA arithmetic.  It exists to
// validate the tensor-core (wgmma) path on the device; it is not a performance path.
#pragma once
#include <cuda_bf16.h>

#include "../../include/graphcast_b200.h"

namespace gcb {

// Element (row, col) of an operand image (see gcb_layer_desc.a_img): byte offset of its
// bf16 "hi" part; the "lo" part is 4224 bytes further.
__device__ __forceinline__ size_t a_image_offset(long long row, int col, int k) {
  const long long tile = row >> 7;
  const int r = static_cast<int>(row & 127), ks = col >> 4, c = (col >> 3) & 1, j = col & 7;
  return (static_cast<size_t>(tile) * (k >> 4) + ks) * GCB_A_IMAGE_BLOCK + c * 2112 + r * 16 + j * 2;
}
__device__ __forceinline__ float bf16_bits_to_float(unsigned short h) {
  return __uint_as_float(static_cast<unsigned int>(h) << 16);
}

constexpr int kSimtRows = 32;
constexpr int kSimtThreads = 256;
constexpr int kSimtK = 16;

__device__ __forceinline__ float swish_exact(float x) { return x / (1.0f + expf(-x)); }

// dynamic smem: ytile [32][n] floats, then a_tile [32][17], w_tile [16][n]
__global__ void __launch_bounds__(kSimtThreads)
mlp_layer_simt_kernel(const __grid_constant__ gcb_layer_desc d) {
  extern __shared__ float sm[];
  const int n = d.n;
  float* ytile = sm;                         // [32][n]
  float* a_tile = ytile + kSimtRows * n;     // [32][17]
  float* w_tile = a_tile + kSimtRows * 17;   // [16][n]
  const int tid = threadIdx.x;
  const int ty = tid >> 6;                   // 0..3 -> rows ty*8 .. +7
  const int tx = tid & 63;                   // cols tx + 64*j
  const int ncol = n / 64;                   // 4 or 8
  const long long row0 = static_cast<long long>(blockIdx.x) * kSimtRows;

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  int kglobal = 0;
  for (int s = 0; s < d.nseg; ++s) {
    gcb_segment sg = d.seg[s];
    if (sg.img) { sg.k_valid = sg.k; sg.fan = 1; sg.idx = nullptr; }
    for (int k0 = 0; k0 < sg.k; k0 += kSimtK, kglobal += kSimtK) {
      // A tile: 32 rows x 16 -> 512 elements, 2 per thread.
      for (int e = tid; e < kSimtRows * kSimtK; e += kSimtThreads) {
        const int r = e / kSimtK, kk = e % kSimtK;
        const long long grow = row0 + r;
        float v = 0.f;
        if (grow < d.rows && (k0 + kk) < sg.k_valid) {
          if (sg.img) {
            const unsigned char* p = static_cast<const unsigned char*>(sg.img) +
                                     a_image_offset(grow, k0 + kk, sg.k);
            v = bf16_bits_to_float(*reinterpret_cast<const unsigned short*>(p)) +
                bf16_bits_to_float(*reinterpret_cast<const unsigned short*>(p + 4224));
          } else {
            const long long src = sg.idx ? static_cast<long long>(sg.idx[grow]) : grow;
            for (int j = 0; j < sg.fan; ++j)
              v += sg.table[(src * sg.fan + j) * sg.ld + k0 + kk];
          }
        }
        a_tile[r * 17 + kk] = v;
      }
      for (int e = tid; e < kSimtK * n; e += kSimtThreads) {
        const int kk = e / n, c = e % n;
        w_tile[kk * n + c] = d.w_f32[static_cast<long long>(kglobal + kk) * n + c];
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < kSimtK; ++kk) {
        float a[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) a[i] = a_tile[(ty * 8 + i) * 17 + kk];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (j < ncol) {
            const float w = w_tile[kk * n + tx + 64 * j];
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[i][j] = fmaf(a[i], w, acc[i][j]);
          }
        }
      }
      __syncthreads();
    }
  }
  // bias + activation into the row tile
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (j < ncol) {
        const int c = tx + 64 * j;
        float x = acc[i][j] + d.bias[c];
        const long long grow = row0 + ty * 8 + i;
        if (grow < d.rows) {
          for (int pa = 0; pa < d.n_pre_add; ++pa) {
            const long long src = d.pre_add[pa].idx ? static_cast<long long>(d.pre_add[pa].idx[grow]) : grow;
            x += d.pre_add[pa].table[src * d.pre_add[pa].ld + c];
          }
        }
        if (d.act == GCB_ACT_SWISH) x = swish_exact(x);
        ytile[(ty * 8 + i) * n + c] = x;
      }
  __syncthreads();
  // per-row LayerNorm / residual / store: warp w handles rows w*4 .. w*4+3
  const int warp = tid >> 5, lane = tid & 31;
  const int nv = d.n_valid;
  for (int rr = 0; rr < 4; ++rr) {
    const int r = warp * 4 + rr;
    const long long grow = row0 + r;
    if (grow >= d.rows) continue;
    float mean = 0.f, rstd = 1.f;
    if (d.ln_scale) {
      float s1 = 0.f;
      for (int c = lane; c < nv; c += 32) s1 += ytile[r * n + c];
      for (int o = 16; o > 0; o >>= 1) s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      mean = s1 / nv;
      float s2 = 0.f;
      for (int c = lane; c < nv; c += 32) {
        const float t = ytile[r * n + c] - mean;
        s2 += t * t;
      }
      for (int o = 16; o > 0; o >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, o);
      rstd = rsqrtf(s2 / nv + 1e-5f);
    }
    for (int c = lane; c < nv; c += 32) {
      float x = ytile[r * n + c];
      if (d.ln_scale) x = (x - mean) * rstd * d.ln_scale[c] + d.ln_offset[c];
      if (d.out_img) {
        unsigned char* p = static_cast<unsigned char*>(d.out_img) + a_image_offset(grow, c, n);
        const float xo = x + (d.residual ? d.residual[grow * d.ld_res + c] : 0.f);
        const __nv_bfloat16 hi = __float2bfloat16_rn(xo);
        const __nv_bfloat16 lo = __float2bfloat16_rn(xo - __bfloat162float(hi));
        *reinterpret_cast<__nv_bfloat16*>(p) = hi;
        *reinterpret_cast<__nv_bfloat16*>(p + 4224) = lo;
      }
      if (d.out_y) d.out_y[grow * d.ld_out_y + c] = x;
      if (d.out) d.out[grow * d.ld_out + c] = x + (d.residual ? d.residual[grow * d.ld_res + c] : 0.f);
    }
  }
}

}  // namespace gcb
