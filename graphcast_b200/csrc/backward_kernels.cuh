// Kernels of the parameter-gradient (backward) pass: the weight-gradient GEMM, the row-wise
// LayerNorm / swish / column-sum backward with fixed-order column partials, the sender-ordered
// segment sum, the receiver gather-add and the seed of the loss derivative.  Every reduction here
// runs over a FIXED split of the rows (not derived from the SM count) and is summed slice by slice
// in a fixed order, so two runs are bit-identical on any device; no atomics.
#pragma once
#include <cuda_bf16.h>

#include "../../include/graphcast_b200.h"
#include "mlp_simt.cuh"

namespace gcb {

// ---- weight-gradient GEMM:  dW[K, N] = sum_r X[r, 0:K]^T G[r, 0:N] ------------------------------
// Tensor cores through mma.sync.m16n8k16 (bf16 operands, fp32 accumulation); the reduction dimension
// is the row index, so both operands are read TRANSPOSED from shared memory while the fragments are
// built (X is staged row-major [rows][K-tile], the A fragment wants [K-tile][rows]).  BF16X3 splits
// each fp32 operand into hi + lo and issues hi*hi + hi*lo + lo*hi, as the forward does.
constexpr int kWgSlices = 64;     // fixed row split -> partial tiles per slice
constexpr int kWgBM = 64;         // K (output rows) per CTA
constexpr int kWgBN = 64;         // N (output cols) per CTA
constexpr int kWgRows = 32;       // rows staged per iteration
constexpr int kWgLd = kWgBM + 4;  // smem row stride: conflict-free transposed fragment reads
constexpr int kWgFlush = 8;       // iterations (256 rows) between fp32 -> fp64 accumulator flushes

__device__ __forceinline__ uint32_t pack_bf16x2(float lo_col, float hi_col) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo_col, hi_col);
  return *reinterpret_cast<uint32_t*>(&v);
}

__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat16 ha = __float2bfloat16_rn(a), hb = __float2bfloat16_rn(b);
  __nv_bfloat162 h; h.x = ha; h.y = hb;
  hi = *reinterpret_cast<uint32_t*>(&h);
  lo = pack_bf16x2(a - __bfloat162float(ha), b - __bfloat162float(hb));
}

__device__ __forceinline__ void mma_bf16(float* c, const uint32_t* a, const uint32_t* b) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};\n"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

__device__ __forceinline__ float swish_fwd(float x) { return x / (1.0f + expf(-x)); }

// grid (N / 64, ceil(K / 64), kWgSlices), 128 threads (2 x 2 warps of 32 x 32).
// X: fp32 table (ld_x, columns >= k_valid read as 0) or operand image x_img of [rows, k_img].
template <bool kSplit>
__global__ void __launch_bounds__(128)
weight_grad_kernel(const float* __restrict__ x, int ld_x, int k_valid,
                   const unsigned char* __restrict__ x_img, int k_img, int x_swish,
                   const float* __restrict__ g, int ld_g, long long rows, int k, int n,
                   float* __restrict__ partial) {
  __shared__ __align__(16) float xs[kWgRows][kWgLd];
  __shared__ __align__(16) float gs[kWgRows][kWgLd];
  const int n0 = blockIdx.x * kWgBN, m0 = blockIdx.y * kWgBM, slice = blockIdx.z;
  const long long per = ((rows + kWgSlices - 1) / kWgSlices + kWgRows - 1) / kWgRows * kWgRows;
  const long long r_beg = min(rows, per * slice), r_end = min(rows, r_beg + per);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;
  const int gq = lane >> 2, tq = lane & 3;
  float acc[2][4][4];
  double dacc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) { acc[i][j][q] = 0.f; dacc[i][j][q] = 0.0; }
  int iter = 0;
  for (long long r0 = r_beg; r0 < r_end; r0 += kWgRows) {
    // stage X[r0:r0+32, m0:m0+64] and G[r0:r0+32, n0:n0+64] (zeros outside)
    if (x_img) {
      for (int p = tid; p < kWgRows * (kWgBM / 8); p += 128) {
        const int rr = p / (kWgBM / 8), c8 = (p % (kWgBM / 8)) * 8;
        const long long r = r0 + rr;
        const int col = m0 + c8;
        float v[8];
        if (r < r_end && col < k_img) {
          const unsigned char* base = x_img + a_image_offset(r, col, k_img);
          const uint4 hv = *reinterpret_cast<const uint4*>(base);
          const uint4 lv = *reinterpret_cast<const uint4*>(base + 4224);
          const unsigned short* h = reinterpret_cast<const unsigned short*>(&hv);
          const unsigned short* l = reinterpret_cast<const unsigned short*>(&lv);
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] = bf16_bits_to_float(h[j]) + bf16_bits_to_float(l[j]);
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] = 0.f;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) xs[rr][c8 + j] = x_swish ? swish_fwd(v[j]) : v[j];
      }
    } else {
      for (int p = tid; p < kWgRows * (kWgBM / 4); p += 128) {
        const int rr = p / (kWgBM / 4), c4 = (p % (kWgBM / 4)) * 4;
        const long long r = r0 + rr;
        const int col = m0 + c4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (r < r_end && col < k_valid) v = __ldg(reinterpret_cast<const float4*>(x + r * ld_x + col));
        if (x_swish) { v.x = swish_fwd(v.x); v.y = swish_fwd(v.y); v.z = swish_fwd(v.z); v.w = swish_fwd(v.w); }
        *reinterpret_cast<float4*>(&xs[rr][c4]) = v;
      }
    }
    for (int p = tid; p < kWgRows * (kWgBN / 4); p += 128) {
      const int rr = p / (kWgBN / 4), c4 = (p % (kWgBN / 4)) * 4;
      const long long r = r0 + rr;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r < r_end) v = __ldg(reinterpret_cast<const float4*>(g + r * ld_g + n0 + c4));
      *reinterpret_cast<float4*>(&gs[rr][c4]) = v;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kWgRows; kk += 16) {
      uint32_t ah[2][4], al[2][4], bh[4][2], bl[4][2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int m = wm + i * 16 + gq;
        // A[m][kk'] = X[kk'][m]: (row g, cols 2t, 2t+1), (row g+8, ...), (row g, cols +8), (g+8, +8)
        const float* c0 = &xs[kk + 2 * tq][0];
        const float* c1 = &xs[kk + 2 * tq + 1][0];
        const float* c8 = &xs[kk + 2 * tq + 8][0];
        const float* c9 = &xs[kk + 2 * tq + 9][0];
        if (kSplit) {
          split2(c0[m], c1[m], ah[i][0], al[i][0]);
          split2(c0[m + 8], c1[m + 8], ah[i][1], al[i][1]);
          split2(c8[m], c9[m], ah[i][2], al[i][2]);
          split2(c8[m + 8], c9[m + 8], ah[i][3], al[i][3]);
        } else {
          ah[i][0] = pack_bf16x2(c0[m], c1[m]);
          ah[i][1] = pack_bf16x2(c0[m + 8], c1[m + 8]);
          ah[i][2] = pack_bf16x2(c8[m], c9[m]);
          ah[i][3] = pack_bf16x2(c8[m + 8], c9[m + 8]);
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int nn = wn + j * 8 + gq;
        const float b00 = gs[kk + 2 * tq][nn], b01 = gs[kk + 2 * tq + 1][nn];
        const float b10 = gs[kk + 2 * tq + 8][nn], b11 = gs[kk + 2 * tq + 9][nn];
        if (kSplit) {
          split2(b00, b01, bh[j][0], bl[j][0]);
          split2(b10, b11, bh[j][1], bl[j][1]);
        } else {
          bh[j][0] = pack_bf16x2(b00, b01);
          bh[j][1] = pack_bf16x2(b10, b11);
        }
      }
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (kSplit) {
            mma_bf16(acc[i][j], al[i], bh[j]);
            mma_bf16(acc[i][j], ah[i], bl[j]);
          }
          mma_bf16(acc[i][j], ah[i], bh[j]);
        }
    }
    __syncthreads();
    if (++iter == kWgFlush) {
      iter = 0;
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int q = 0; q < 4; ++q) { dacc[i][j][q] += acc[i][j][q]; acc[i][j][q] = 0.f; }
    }
  }
  float* out = partial + static_cast<long long>(slice) * k * n;
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int m = m0 + wm + i * 16 + gq + (q >> 1) * 8;
        const int nn = n0 + wn + j * 8 + 2 * tq + (q & 1);
        if (m < k) out[static_cast<long long>(m) * n + nn] = static_cast<float>(dacc[i][j][q] + acc[i][j][q]);
      }
}

// out[i] = (accumulate ? out[i] : 0) + sum over s = 0..slices-1 (in this order) of partial[s*stride + i],
// in fp64, rounded once to fp32.
__global__ void __launch_bounds__(256)
slices_reduce_kernel(const float* __restrict__ partial, int slices, long long stride, long long count,
                     float* __restrict__ out, int accumulate) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= count) return;
  double s = accumulate ? static_cast<double>(out[i]) : 0.0;
  for (int q = 0; q < slices; ++q) s += static_cast<double>(partial[q * stride + i]);
  out[i] = static_cast<float>(s);
}

// ---- row-wise backward kernels -------------------------------------------------------------------
// One warp per row, lane owns columns lane + 32 j.  Block b (of kRowSlices) owns a contiguous row
// range; its 8 warps stride through it, each keeping fp64 column sums in registers; the warps are
// folded in order through shared memory into partial[b][q][col] (fp32).
constexpr int kRowSlices = 256;
enum RowMode { kRowLayerNorm = 0, kRowCopy = 1, kRowSwish = 2 };

// The LayerNorm statistics (eps 1e-5) of one n = 32 * kCols row held by a warp, lane owning v[j] =
// column lane + 32 j: its mean and 1 / sqrt(var + eps), with fixed butterfly sums.
template <int kCols>
__device__ __forceinline__ void ln_row_stats(const float* v, float& mean, float& rstd) {
  constexpr int n = kCols * 32;
  mean = 0.f;
#pragma unroll
  for (int j = 0; j < kCols; ++j) mean += v[j];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mean += __shfl_xor_sync(0xffffffffu, mean, o);
  mean *= (1.0f / n);
  float var = 0.f;
#pragma unroll
  for (int j = 0; j < kCols; ++j) { const float t = v[j] - mean; var += t * t; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
  rstd = rsqrtf(var * (1.0f / n) + 1e-5f);
}

template <int kMode, int kCols>   // kCols = n / 32 (8 or 16)
__global__ void __launch_bounds__(256)
rowwise_backward_kernel(const float* __restrict__ dy, int ld_dy, const float* __restrict__ z, int ld_z,
                        const float* __restrict__ scale, long long rows, float* __restrict__ dz,
                        int ld_dz, float* __restrict__ partial) {
  constexpr int kSums = kMode == kRowLayerNorm ? 3 : 1;
  constexpr int n = kCols * 32;
  __shared__ double red[8][n];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long per = (rows + kRowSlices - 1) / kRowSlices;
  const long long r_beg = min(rows, per * blockIdx.x), r_end = min(rows, r_beg + per);
  double s0[kCols], s1[kCols], s2[kCols];
  float sc[kCols];
#pragma unroll
  for (int j = 0; j < kCols; ++j) {
    s0[j] = s1[j] = s2[j] = 0.0;
    sc[j] = (kMode == kRowLayerNorm) ? scale[lane + 32 * j] : 1.f;
  }
  for (long long r = r_beg + warp; r < r_end; r += 8) {
    float d[kCols], v[kCols];
#pragma unroll
    for (int j = 0; j < kCols; ++j) d[j] = dy[r * ld_dy + lane + 32 * j];
    if (kMode == kRowLayerNorm) {
#pragma unroll
      for (int j = 0; j < kCols; ++j) v[j] = z[r * ld_z + lane + 32 * j];
      float mean, rstd;
      ln_row_stats<kCols>(v, mean, rstd);
      float mg = 0.f, mgz = 0.f;
#pragma unroll
      for (int j = 0; j < kCols; ++j) {
        v[j] = (v[j] - mean) * rstd;                   // z-hat
        const float gg = d[j] * sc[j];
        mg += gg;
        mgz += gg * v[j];
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        mg += __shfl_xor_sync(0xffffffffu, mg, o);
        mgz += __shfl_xor_sync(0xffffffffu, mgz, o);
      }
      mg *= (1.0f / n);
      mgz *= (1.0f / n);
#pragma unroll
      for (int j = 0; j < kCols; ++j) {
        const float out = rstd * (d[j] * sc[j] - mg - v[j] * mgz);
        dz[r * ld_dz + lane + 32 * j] = out;
        s0[j] += out;                                  // bias of the linear before the LayerNorm
        s1[j] += static_cast<double>(d[j]) * v[j];     // LayerNorm scale
        s2[j] += d[j];                                 // LayerNorm offset
      }
    } else if (kMode == kRowSwish) {
#pragma unroll
      for (int j = 0; j < kCols; ++j) {
        const float h = z[r * ld_z + lane + 32 * j];
        const float sg = 1.0f / (1.0f + expf(-h));
        const float out = d[j] * (sg * (1.0f + h * (1.0f - sg)));
        dz[r * ld_dz + lane + 32 * j] = out;
        s0[j] += out;
      }
    } else {
#pragma unroll
      for (int j = 0; j < kCols; ++j) {
        if (dz) dz[r * ld_dz + lane + 32 * j] = d[j];
        s0[j] += d[j];
      }
    }
  }
#pragma unroll
  for (int q = 0; q < kSums; ++q) {
#pragma unroll
    for (int j = 0; j < kCols; ++j) red[warp][lane + 32 * j] = q == 0 ? s0[j] : (q == 1 ? s1[j] : s2[j]);
    __syncthreads();
    for (int c = threadIdx.x; c < n; c += 256) {
      double t = 0.0;
      for (int w = 0; w < 8; ++w) t += red[w][c];
      partial[(static_cast<long long>(blockIdx.x) * kSums + q) * n + c] = static_cast<float>(t);
    }
    __syncthreads();
  }
}

// ---- tangent-linear model ------------------------------------------------------------------------
// The LayerNorm tangent of one row (n = 512, lane owns columns lane + 32 j) from zhat v, rstd and the
// row sums md_sum = sum dz and mdz_sum = sum zhat * dz:
//   out = [residual +] scale * (rstd * (dz - md_sum / n - zhat * (mdz_sum / n)))
// with every rounding pinned by an intrinsic, so that each kernel applying it gives the same bits.  The
// roundings are those layernorm_jvp_kernel was first compiled to, which input_jvp's results have been
// since: md_sum / n folded into one fma with dz, mdz_sum / n rounded once, and the residual of column
// 0 (j = 0) added to the rounded product, that of every other column fused with it into one fma.
__device__ __forceinline__ void ln_jvp_apply(const float (&d)[16], const float (&v)[16], float rstd,
                                             float md_sum, float mdz_sum, const float (&sc)[16],
                                             const float* __restrict__ res_row, float* __restrict__ out_row,
                                             int lane) {
  const float mdz = __fmul_rn(mdz_sum, 1.0f / 512);
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int c = lane + 32 * j;
    const float t = __fmul_rn(rstd, __fmaf_rn(v[j], -mdz, __fmaf_rn(md_sum, -1.0f / 512, d[j])));
    float o;
    if (!res_row) o = __fmul_rn(t, sc[j]);
    else if (j == 0) o = __fadd_rn(__fmul_rn(t, sc[j]), res_row[c]);
    else o = __fmaf_rn(t, sc[j], res_row[c]);
    out_row[c] = o;
  }
}

// Tangent of hk.LayerNorm at the pre-LayerNorm z along dz, one warp per row of n = 512 (lane owns
// columns lane + 32 j), 8 rows per block:
//   out = (residual ? residual : 0) + scale * (rstd * (dz - mean(dz) - zhat * mean(zhat * dz)))
// zhat = (z - mu) * rstd, mu and rstd from ln_row_stats as rowwise_backward_kernel forms them.  The
// Jacobian is symmetric, so with unit scale this is that kernel's dz for dy = dz.  Row-wise: no column
// sums, no atomics.  The output arithmetic is ln_jvp_apply.
__global__ void __launch_bounds__(256)
layernorm_jvp_kernel(const float* __restrict__ z, int ld_z, const float* __restrict__ dz, int ld_dz,
                     const float* __restrict__ scale, long long rows, const float* __restrict__ residual,
                     int ld_res, float* __restrict__ out, int ld_out) {
  constexpr int kCols = 16;
  const int lane = threadIdx.x & 31;
  const long long r = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (r >= rows) return;
  float v[kCols], d[kCols], sc[kCols];
#pragma unroll
  for (int j = 0; j < kCols; ++j) {
    v[j] = z[r * ld_z + lane + 32 * j];
    d[j] = dz[r * ld_dz + lane + 32 * j];
    sc[j] = scale[lane + 32 * j];
  }
  float mean, rstd;
  ln_row_stats<kCols>(v, mean, rstd);
  float md = 0.f, mdz = 0.f;
#pragma unroll
  for (int j = 0; j < kCols; ++j) {
    v[j] = (v[j] - mean) * rstd;                       // z-hat
    md += d[j];
    mdz += d[j] * v[j];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    md += __shfl_xor_sync(0xffffffffu, md, o);
    mdz += __shfl_xor_sync(0xffffffffu, mdz, o);
  }
  ln_jvp_apply(d, v, rstd, md, mdz, sc, residual ? residual + r * ld_res : nullptr, out + r * ld_out,
               lane);
}

// ---- tangents with respect to the parameters (param_jvp) --------------------------------------------
// layernorm_jvp_kernel plus the tangent of the LayerNorm's own parameters:
//   out = (residual ? residual : 0) + scale * (rstd * (dz - mean(dz) - zhat * mean(zhat * dz)))
//         + dscale * zhat + doffset
// The statements up to ln_jvp_apply are those of layernorm_jvp_kernel, so with dscale = doffset = NULL
// the result is its bits.  The two parameter terms are then added to the stored row in order, each
// rounded once: fma(dscale, zhat, out), then + doffset.  One warp per row of n = 512, 8 rows per block.
__global__ void __launch_bounds__(256)
layernorm_jvp_params_kernel(const float* __restrict__ z, int ld_z, const float* __restrict__ dz,
                            int ld_dz, const float* __restrict__ scale, long long rows,
                            const float* __restrict__ residual, int ld_res,
                            const float* __restrict__ dscale, const float* __restrict__ doffset,
                            float* __restrict__ out, int ld_out) {
  constexpr int kCols = 16;
  const int lane = threadIdx.x & 31;
  const long long r = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (r >= rows) return;
  float v[kCols], d[kCols], sc[kCols];
#pragma unroll
  for (int j = 0; j < kCols; ++j) {
    v[j] = z[r * ld_z + lane + 32 * j];
    d[j] = dz[r * ld_dz + lane + 32 * j];
    sc[j] = scale[lane + 32 * j];
  }
  float mean, rstd;
  ln_row_stats<kCols>(v, mean, rstd);
  float md = 0.f, mdz = 0.f;
#pragma unroll
  for (int j = 0; j < kCols; ++j) {
    v[j] = (v[j] - mean) * rstd;                       // z-hat
    md += d[j];
    mdz += d[j] * v[j];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    md += __shfl_xor_sync(0xffffffffu, md, o);
    mdz += __shfl_xor_sync(0xffffffffu, mdz, o);
  }
  float* out_row = out + r * ld_out;
  ln_jvp_apply(d, v, rstd, md, mdz, sc, residual ? residual + r * ld_res : nullptr, out_row, lane);
  if (!dscale && !doffset) return;
#pragma unroll
  for (int j = 0; j < kCols; ++j) {
    const int c = lane + 32 * j;
    float o = out_row[c];
    if (dscale) o = __fmaf_rn(dscale[c], v[j], o);
    if (doffset) o = __fadd_rn(o, doffset[c]);
    out_row[c] = o;
  }
}

// The seed of a Gauss-Newton product: the loss Hessian with respect to the decoder output is diagonal,
// coef[c] * lat_weight, so  g[node, c] = coef[c] * lat_weight[node / n_lon] * dy[node, c]  (fp64, rounded
// once): output_loss_grad_kernel with zero targets and no scale / offset / add planes, whose t_norm is
// then +0 and y - t_norm is y.  One thread per (node, channel), channels fastest.
__global__ void __launch_bounds__(256)
output_loss_gn_seed_kernel(const float* __restrict__ dy, int ld_dy, int n_out, int n_lon,
                           long long n_nodes, const float* __restrict__ lat_weight,
                           const double* __restrict__ coef, float* __restrict__ g, int ld_g) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n_nodes * n_out) return;
  const long long node = i / n_out;
  const int c = static_cast<int>(i - node * n_out);
  const double d = static_cast<double>(__fsub_rn(dy[node * ld_dy + c], 0.f));
  g[node * ld_g + c] = static_cast<float>(coef[c] * static_cast<double>(lat_weight[node / n_lon]) * d);
}

// ---- several tangent directions (batched_input_jvp) -----------------------------------------------
// The tangent tables of `dirs` directions are stacked direction-major: row r of direction k is row
// k * stride + r.  Each kernel reads the primal row once and applies it to the dirs tangent rows with,
// per element, exactly the arithmetic of its one-direction counterpart, so every direction is bit for
// bit what that kernel gives it alone.

// da[k] = swish'(h) * dh[k], swish'(h) = sg * (1 + h * (1 - sg)), sg = 1 / (1 + exp(-h)): the dz of
// rowwise_backward_kernel<kRowSwish> without its column sums.  One thread per 4 columns of a row; da
// may alias dh (each thread reads its dh before it writes the same da).
__global__ void __launch_bounds__(256)
swish_jvp_kernel(const float* __restrict__ h, int ld_h, long long rows, int n4,
                 const float* dh, int ld_dh, long long stride, int dirs, float* da, int ld_da) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= rows * n4) return;
  const long long r = i / n4;
  const int c = static_cast<int>(i - r * n4) * 4;
  const float4 hv = *reinterpret_cast<const float4*>(h + r * ld_h + c);
  const float hq[4] = {hv.x, hv.y, hv.z, hv.w};
  float f[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float sg = 1.0f / (1.0f + expf(-hq[q]));
    f[q] = sg * (1.0f + hq[q] * (1.0f - sg));
  }
  for (int k = 0; k < dirs; ++k) {
    const long long rk = k * stride + r;
    const float4 d = *reinterpret_cast<const float4*>(dh + rk * ld_dh + c);
    *reinterpret_cast<float4*>(da + rk * ld_da + c) =
        make_float4(d.x * f[0], d.y * f[1], d.z * f[2], d.w * f[3]);
  }
}

// layernorm_jvp_kernel for dirs directions: the statistics and zhat of z's row once, then per direction
//   out[k] = (residual ? residual[k] : 0) + scale * (rstd * (dz[k] - mean(dz[k]) - zhat * mean(zhat * dz[k])))
// One warp per row of n = 512, 8 rows per block.
__global__ void __launch_bounds__(256)
layernorm_jvp_dirs_kernel(const float* __restrict__ z, int ld_z, const float* __restrict__ dz,
                          int ld_dz, const float* __restrict__ scale, long long rows, long long stride,
                          int dirs, const float* __restrict__ residual, int ld_res,
                          float* __restrict__ out, int ld_out) {
  constexpr int kCols = 16;
  const int lane = threadIdx.x & 31;
  const long long r = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (r >= rows) return;
  float v[kCols], sc[kCols];
#pragma unroll
  for (int j = 0; j < kCols; ++j) {
    v[j] = z[r * ld_z + lane + 32 * j];
    sc[j] = scale[lane + 32 * j];
  }
  float mean, rstd;
  ln_row_stats<kCols>(v, mean, rstd);
#pragma unroll
  for (int j = 0; j < kCols; ++j) v[j] = (v[j] - mean) * rstd;     // z-hat
  for (int k = 0; k < dirs; ++k) {
    const long long rk = k * stride + r;
    float d[kCols];
#pragma unroll
    for (int j = 0; j < kCols; ++j) d[j] = dz[rk * ld_dz + lane + 32 * j];
    float md = 0.f, mdz = 0.f;
#pragma unroll
    for (int j = 0; j < kCols; ++j) {
      md += d[j];
      mdz += d[j] * v[j];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      md += __shfl_xor_sync(0xffffffffu, md, o);
      mdz += __shfl_xor_sync(0xffffffffu, mdz, o);
    }
    ln_jvp_apply(d, v, rstd, md, mdz, sc, residual ? residual + rk * ld_res : nullptr,
                 out + rk * ld_out, lane);
  }
}

// ---- several cotangents (batched_input_vjp) -------------------------------------------------------
// The dz of rowwise_backward_kernel<kRowLayerNorm, 16> for dirs stacked dy tables (row r of direction k
// is row k * stride + r), without its column sums:
//   dz[k] = rstd * (dy[k]*scale - mean(dy[k]*scale) - zhat * mean(dy[k]*scale*zhat))
// One warp per row of n = 512 (lane owns columns lane + 32 j), 8 rows per block; z's row is read once.
// Every rounding is pinned by an intrinsic to what rowwise_backward_kernel<kRowLayerNorm, 16> compiles
// to (its SASS): the row sum s of z in column order then butterfly order, z - mean as fma(s, -1/n, z)
// (the mean itself never rounded), the variance as a chain of fmas from 0, rstd = rsqrt(fma(var, 1/n,
// 1e-5)), zhat = (z - mean) * rstd; g = dy * scale rounded, sum g added in column order, sum g * zhat
// as a chain of fmas from 0; dz = rstd * fma(zhat, -mgz, fma(sum g, -1/n, g)) with mgz = (sum g * zhat)
// / n rounded once.
__global__ void __launch_bounds__(256)
layernorm_backward_dirs_kernel(const float* __restrict__ dy, int ld_dy, const float* __restrict__ z,
                               int ld_z, const float* __restrict__ scale, long long rows,
                               long long stride, int dirs, float* __restrict__ dz, int ld_dz) {
  constexpr int kCols = 16;
  constexpr float kInvN = 1.0f / (kCols * 32);
  const int lane = threadIdx.x & 31;
  const long long r = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (r >= rows) return;
  float v[kCols], sc[kCols];
#pragma unroll
  for (int j = 0; j < kCols; ++j) {
    v[j] = z[r * ld_z + lane + 32 * j];
    sc[j] = scale[lane + 32 * j];
  }
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < kCols; ++j) s = __fadd_rn(s, v[j]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
  float var = 0.f;
#pragma unroll
  for (int j = 0; j < kCols; ++j) {
    v[j] = __fmaf_rn(s, -kInvN, v[j]);                 // z - mean
    var = __fmaf_rn(v[j], v[j], var);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) var = __fadd_rn(var, __shfl_xor_sync(0xffffffffu, var, o));
  const float rstd = rsqrtf(__fmaf_rn(var, kInvN, 1e-5f));
#pragma unroll
  for (int j = 0; j < kCols; ++j) v[j] = __fmul_rn(v[j], rstd);     // z-hat
  for (int k = 0; k < dirs; ++k) {
    const long long rk = k * stride + r;
    float g[kCols];
    float mg = 0.f, mgz = 0.f;
#pragma unroll
    for (int j = 0; j < kCols; ++j) {
      g[j] = __fmul_rn(dy[rk * ld_dy + lane + 32 * j], sc[j]);
      mg = __fadd_rn(mg, g[j]);
      mgz = __fmaf_rn(v[j], g[j], mgz);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mg = __fadd_rn(mg, __shfl_xor_sync(0xffffffffu, mg, o));
      mgz = __fadd_rn(mgz, __shfl_xor_sync(0xffffffffu, mgz, o));
    }
    const float mgz_n = __fmul_rn(mgz, kInvN);
#pragma unroll
    for (int j = 0; j < kCols; ++j)
      dz[rk * ld_dz + lane + 32 * j] = __fmul_rn(rstd, __fmaf_rn(v[j], -mgz_n, __fmaf_rn(mg, -kInvN, g[j])));
  }
}

// ---- Hessian-vector products (loss_and_input_hvp, batched_loss_and_input_hvp) ---------------------
// The backward pass of the gradient (direction 0) coupled with its tangents along K primal tangents
// (directions 1..K), stacked as above with 1 + K directions, at the primal h / z and their tangents
// hdot / zdot (stacked tables of K directions at the same stride).  Direction 0 is bit for bit what
// swish_jvp_kernel / layernorm_backward_dirs_kernel give it alone; direction j is its derivative along
// tangent j - 1, in fp32, with the same roundings whatever K is (pinned below to the sequence the
// one-tangent kernel compiled to), so direction j is bit for bit the K = 1 launch on (0, j, j - 1).
// The primal terms (s', s'', the row statistics, z-hat, g) are formed once per element / row.

// dh = s'(h) da, dhdot_j = s'(h) dadot_j + s''(h) hdot_j da, with s'(h) = sg (1 + h (1 - sg)) rounded
// as swish_jvp_kernel compiles it and s''(h) = sg (1 - sg) (2 + h (1 - 2 sg)).  One thread per 4 columns
// of a row; dh may alias da (each thread reads direction j of da before it writes direction j of dh,
// and no other thread touches those columns).
__global__ void __launch_bounds__(256)
swish_backward_jvp_kernel(const float* __restrict__ h, int ld_h, const float* __restrict__ hdot,
                          int ld_hdot, long long rows, int n4, const float* da, int ld_da,
                          long long stride, int tangents, float* dh, int ld_dh) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= rows * n4) return;
  const long long r = i / n4;
  const int c = static_cast<int>(i - r * n4) * 4;
  const float4 hv = *reinterpret_cast<const float4*>(h + r * ld_h + c);
  const float4 a0 = *reinterpret_cast<const float4*>(da + r * ld_da + c);
  const float hq[4] = {hv.x, hv.y, hv.z, hv.w}, d0[4] = {a0.x, a0.y, a0.z, a0.w};
  float f[4], f2[4], o0[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float sg = 1.0f / (1.0f + expf(-hq[q]));
    const float om = __fsub_rn(1.0f, sg);
    f[q] = __fmul_rn(sg, __fmaf_rn(hq[q], om, 1.0f));
    f2[q] = __fmul_rn(__fmul_rn(sg, om),
                      __fmaf_rn(hq[q], __fsub_rn(1.0f, __fadd_rn(sg, sg)), 2.0f));
    o0[q] = __fmul_rn(d0[q], f[q]);
  }
  *reinterpret_cast<float4*>(dh + r * ld_dh + c) = make_float4(o0[0], o0[1], o0[2], o0[3]);
  for (int t = 0; t < tangents; ++t) {
    const long long rt = static_cast<long long>(t) * stride + r;
    const float4 tv = *reinterpret_cast<const float4*>(hdot + rt * ld_hdot + c);
    const float4 a1 = *reinterpret_cast<const float4*>(da + (stride + rt) * ld_da + c);
    const float tq[4] = {tv.x, tv.y, tv.z, tv.w}, d1[4] = {a1.x, a1.y, a1.z, a1.w};
    float o1[4];
#pragma unroll
    for (int q = 0; q < 4; ++q)            // s'(h) dadot + (s''(h) hdot) da
      o1[q] = __fmaf_rn(d1[q], f[q], __fmul_rn(__fmul_rn(f2[q], tq[q]), d0[q]));
    *reinterpret_cast<float4*>(dh + (stride + rt) * ld_dh + c) = make_float4(o1[0], o1[1], o1[2], o1[3]);
  }
}

// The LayerNorm backward of layernorm_backward_dirs_kernel for [dy; dydot_1..K] (direction 0: its dz,
// with its pinned roundings) and the tangents of that dz along zdot_1..K (directions 1..K).  With r =
// rstd, zhat = (z - mu) r, g = dy*scale, m = mean(g*zhat), per tangent:
//   rdot    = -r^2 mean(zhat*zdot)
//   zhatdot = r (zdot - mean(zdot) - zhat mean(zhat*zdot))
//   gdot    = dydot*scale,  mdot = mean(gdot*zhat + g*zhatdot)
//   dzdot   = rdot (g - mean(g) - zhat m) + r (gdot - mean(gdot) - zhatdot m - zhat mdot)
// One warp per row of n = 512 (lane owns columns lane + 32 j), 8 rows per block; z's row is read once,
// the statistics, zhat, g and (g - mean(g) - zhat m) are formed once for every tangent.
__global__ void __launch_bounds__(256)
layernorm_backward_jvp_kernel(const float* __restrict__ dy, int ld_dy, const float* __restrict__ z,
                              int ld_z, const float* __restrict__ zdot, int ld_zdot,
                              const float* __restrict__ scale, long long rows, long long stride,
                              int tangents, float* __restrict__ dz, int ld_dz) {
  constexpr int kCols = 16;
  constexpr float kInvN = 1.0f / (kCols * 32);
  const int lane = threadIdx.x & 31;
  const long long r = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (r >= rows) return;
  float v[kCols], sc[kCols];
#pragma unroll
  for (int j = 0; j < kCols; ++j) {
    v[j] = z[r * ld_z + lane + 32 * j];
    sc[j] = scale[lane + 32 * j];
  }
  // the primal statistics and direction 0: layernorm_backward_dirs_kernel's arithmetic
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < kCols; ++j) s = __fadd_rn(s, v[j]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
  float var = 0.f;
#pragma unroll
  for (int j = 0; j < kCols; ++j) {
    v[j] = __fmaf_rn(s, -kInvN, v[j]);                 // z - mean
    var = __fmaf_rn(v[j], v[j], var);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) var = __fadd_rn(var, __shfl_xor_sync(0xffffffffu, var, o));
  const float rstd = rsqrtf(__fmaf_rn(var, kInvN, 1e-5f));
#pragma unroll
  for (int j = 0; j < kCols; ++j) v[j] = __fmul_rn(v[j], rstd);     // z-hat
  float g[kCols], a[kCols];
  float mg = 0.f, mgz = 0.f;
#pragma unroll
  for (int j = 0; j < kCols; ++j) {
    g[j] = __fmul_rn(dy[r * ld_dy + lane + 32 * j], sc[j]);
    mg = __fadd_rn(mg, g[j]);
    mgz = __fmaf_rn(v[j], g[j], mgz);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mg = __fadd_rn(mg, __shfl_xor_sync(0xffffffffu, mg, o));
    mgz = __fadd_rn(mgz, __shfl_xor_sync(0xffffffffu, mgz, o));
  }
  const float mgz_n = __fmul_rn(mgz, kInvN);
#pragma unroll
  for (int j = 0; j < kCols; ++j) {
    a[j] = __fmaf_rn(v[j], -mgz_n, __fmaf_rn(mg, -kInvN, g[j]));     // g - mean(g) - zhat m
    dz[r * ld_dz + lane + 32 * j] = __fmul_rn(rstd, a[j]);
  }
  const float rr = __fmul_rn(rstd, rstd);
  // directions 1..K: the tangents.  mean(x) = sum(x) / 512 is folded into an fma with -1/512 where the
  // mean is subtracted (exact: a power of two).
  for (int t = 0; t < tangents; ++t) {
    const long long rt = static_cast<long long>(t) * stride + r;
    float zd[kCols];
    float mzd = 0.f, mvz = 0.f;
#pragma unroll
    for (int j = 0; j < kCols; ++j) {
      zd[j] = zdot[rt * ld_zdot + lane + 32 * j];
      mzd = __fadd_rn(mzd, zd[j]);
      mvz = __fmaf_rn(v[j], zd[j], mvz);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mzd = __fadd_rn(mzd, __shfl_xor_sync(0xffffffffu, mzd, o));
      mvz = __fadd_rn(mvz, __shfl_xor_sync(0xffffffffu, mvz, o));
    }
    mvz = __fmul_rn(mvz, kInvN);
    const float nrdot = __fmul_rn(mvz, rr);                          // -rdot
    float gd[kCols];
    float mgd = 0.f, mdot = 0.f;
#pragma unroll
    for (int j = 0; j < kCols; ++j) {
      zd[j] = __fmul_rn(rstd, __fmaf_rn(v[j], -mvz, __fmaf_rn(mzd, -kInvN, zd[j])));   // zhat-dot
      gd[j] = __fmul_rn(dy[(stride + rt) * ld_dy + lane + 32 * j], sc[j]);
      mgd = __fadd_rn(mgd, gd[j]);
      mdot = __fadd_rn(mdot, __fmaf_rn(v[j], gd[j], __fmul_rn(g[j], zd[j])));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mgd = __fadd_rn(mgd, __shfl_xor_sync(0xffffffffu, mgd, o));
      mdot = __fadd_rn(mdot, __shfl_xor_sync(0xffffffffu, mdot, o));
    }
    mdot = __fmul_rn(mdot, kInvN);
#pragma unroll
    for (int j = 0; j < kCols; ++j) {
      const float b = __fmaf_rn(v[j], -mdot, __fmaf_rn(-mgz_n, zd[j], __fmaf_rn(mgd, -kInvN, gd[j])));
      dz[(stride + rt) * ld_dz + lane + 32 * j] = __fmaf_rn(rstd, b, -__fmul_rn(nrdot, a[j]));
    }
  }
}

// ---- Hessian-vector products with respect to the parameters (loss_and_param_hvp) ------------------
// Direction 1 of layernorm_backward_jvp_kernel (one tangent, dy and dydot = rows [0, rows) and
// [stride, stride + rows)) with the tangent of the scale as well, g-dot = dydot*scale + dy*scale_dot
// (scale_dot NULL: dydot*scale, so that dzdot is that kernel's bits), and the tangents of the three
// column sums of rowwise_backward_kernel<kRowLayerNorm, 16>:
//   sum dzdot (bias), sum dydot*zhat + dy*zhatdot (scale), sum dydot (offset)
// over rowwise_backward_kernel's row split: block b of kRowSlices owns a contiguous row range, its 8
// warps stride through it keeping fp64 column sums, and the warps are folded in order into
// partial[b][q][col].  Direction 0 (dz and its sums) is rowwise_backward_kernel's launch itself.
__global__ void __launch_bounds__(256)
layernorm_backward_jvp_params_kernel(const float* __restrict__ dy, int ld_dy, long long stride,
                                     const float* __restrict__ z, int ld_z,
                                     const float* __restrict__ zdot, int ld_zdot,
                                     const float* __restrict__ scale,
                                     const float* __restrict__ scale_dot, long long rows,
                                     float* __restrict__ dz, int ld_dz, float* __restrict__ partial) {
  constexpr int kCols = 16;
  constexpr int n = kCols * 32;
  constexpr float kInvN = 1.0f / n;
  __shared__ double red[8][n];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long per = (rows + kRowSlices - 1) / kRowSlices;
  const long long r_beg = min(rows, per * blockIdx.x), r_end = min(rows, r_beg + per);
  double s0[kCols], s1[kCols], s2[kCols];
#pragma unroll
  for (int j = 0; j < kCols; ++j) s0[j] = s1[j] = s2[j] = 0.0;
  for (long long r = r_beg + warp; r < r_end; r += 8) {
    // the primal statistics, z-hat, g and a = g - mean(g) - zhat m: layernorm_backward_jvp_kernel's
    float v[kCols];
#pragma unroll
    for (int j = 0; j < kCols; ++j) v[j] = z[r * ld_z + lane + 32 * j];
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < kCols; ++j) s = __fadd_rn(s, v[j]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
    float var = 0.f;
#pragma unroll
    for (int j = 0; j < kCols; ++j) {
      v[j] = __fmaf_rn(s, -kInvN, v[j]);               // z - mean
      var = __fmaf_rn(v[j], v[j], var);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) var = __fadd_rn(var, __shfl_xor_sync(0xffffffffu, var, o));
    const float rstd = rsqrtf(__fmaf_rn(var, kInvN, 1e-5f));
#pragma unroll
    for (int j = 0; j < kCols; ++j) v[j] = __fmul_rn(v[j], rstd);   // z-hat
    float g[kCols], a[kCols];
    float mg = 0.f, mgz = 0.f;
#pragma unroll
    for (int j = 0; j < kCols; ++j) {
      g[j] = __fmul_rn(dy[r * ld_dy + lane + 32 * j], scale[lane + 32 * j]);
      mg = __fadd_rn(mg, g[j]);
      mgz = __fmaf_rn(v[j], g[j], mgz);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mg = __fadd_rn(mg, __shfl_xor_sync(0xffffffffu, mg, o));
      mgz = __fadd_rn(mgz, __shfl_xor_sync(0xffffffffu, mgz, o));
    }
    const float mgz_n = __fmul_rn(mgz, kInvN);
#pragma unroll
    for (int j = 0; j < kCols; ++j) a[j] = __fmaf_rn(v[j], -mgz_n, __fmaf_rn(mg, -kInvN, g[j]));
    const float rr = __fmul_rn(rstd, rstd);
    // the tangent: layernorm_backward_jvp_kernel's direction 1, g-dot with the scale's tangent term
    const long long rt = stride + r;
    float zd[kCols];
    float mzd = 0.f, mvz = 0.f;
#pragma unroll
    for (int j = 0; j < kCols; ++j) {
      zd[j] = zdot[r * ld_zdot + lane + 32 * j];
      mzd = __fadd_rn(mzd, zd[j]);
      mvz = __fmaf_rn(v[j], zd[j], mvz);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mzd = __fadd_rn(mzd, __shfl_xor_sync(0xffffffffu, mzd, o));
      mvz = __fadd_rn(mvz, __shfl_xor_sync(0xffffffffu, mvz, o));
    }
    mvz = __fmul_rn(mvz, kInvN);
    const float nrdot = __fmul_rn(mvz, rr);                          // -rdot
    float mgd = 0.f, mdot = 0.f;
#pragma unroll
    for (int j = 0; j < kCols; ++j) {
      const int c = lane + 32 * j;
      zd[j] = __fmul_rn(rstd, __fmaf_rn(v[j], -mvz, __fmaf_rn(mzd, -kInvN, zd[j])));   // zhat-dot
      float gd = __fmul_rn(dy[rt * ld_dy + c], scale[c]);
      if (scale_dot) gd = __fmaf_rn(dy[r * ld_dy + c], scale_dot[c], gd);
      mgd = __fadd_rn(mgd, gd);
      mdot = __fadd_rn(mdot, __fmaf_rn(v[j], gd, __fmul_rn(g[j], zd[j])));
      g[j] = gd;                                                     // g is not read again
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mgd = __fadd_rn(mgd, __shfl_xor_sync(0xffffffffu, mgd, o));
      mdot = __fadd_rn(mdot, __shfl_xor_sync(0xffffffffu, mdot, o));
    }
    mdot = __fmul_rn(mdot, kInvN);
#pragma unroll
    for (int j = 0; j < kCols; ++j) {
      const int c = lane + 32 * j;
      const float b = __fmaf_rn(v[j], -mdot, __fmaf_rn(-mgz_n, zd[j], __fmaf_rn(mgd, -kInvN, g[j])));
      const float out = __fmaf_rn(rstd, b, -__fmul_rn(nrdot, a[j]));
      dz[rt * ld_dz + c] = out;
      const float d0 = dy[r * ld_dy + c], d1 = dy[rt * ld_dy + c];
      s0[j] += out;                                                  // bias of the linear before it
      s1[j] += static_cast<double>(d1) * v[j] + static_cast<double>(d0) * zd[j];   // LayerNorm scale
      s2[j] += d1;                                                   // LayerNorm offset
    }
  }
#pragma unroll
  for (int q = 0; q < 3; ++q) {
#pragma unroll
    for (int j = 0; j < kCols; ++j) red[warp][lane + 32 * j] = q == 0 ? s0[j] : (q == 1 ? s1[j] : s2[j]);
    __syncthreads();
    for (int c = threadIdx.x; c < n; c += 256) {
      double t = 0.0;
      for (int w = 0; w < 8; ++w) t += red[w][c];
      partial[(static_cast<long long>(blockIdx.x) * 3 + q) * n + c] = static_cast<float>(t);
    }
    __syncthreads();
  }
}

// ---- index operations ----------------------------------------------------------------------------
// out[i, 0:512] = sum_{j in [ptr[i], ptr[i+1])} msg[order[j], 0:512], summed in j order.  Rows listed
// in `heavy` (ascending node ids): one 128-thread block each (thread owns one float4 column); every
// other row: one warp (lane owns 4 float4 columns), which looks its node up in the list (binary
// search) and leaves listed rows to their block.  Both walk j in the same order, so the result does
// not depend on which rows are listed.
__device__ __forceinline__ bool in_sorted_list(const int* __restrict__ list, int n, int v) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    const int x = list[mid];
    if (x == v) return true;
    if (x < v) lo = mid + 1; else hi = mid;
  }
  return false;
}

__global__ void __launch_bounds__(256)
segment_sum_sorted_kernel(const float* __restrict__ msg, int ld_msg, const int* __restrict__ order,
                          const int* __restrict__ ptr, int num_nodes, const int* __restrict__ heavy,
                          int num_heavy, int light_blocks, float* __restrict__ out, int ld_out) {
  if (static_cast<int>(blockIdx.x) >= light_blocks) {
    const int node = heavy[blockIdx.x - light_blocks];
    if (threadIdx.x >= 128) return;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = ptr[node]; j < ptr[node + 1]; ++j) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(msg + static_cast<long long>(order[j]) * ld_msg) + threadIdx.x);
      acc.x += t.x; acc.y += t.y; acc.z += t.z; acc.w += t.w;
    }
    reinterpret_cast<float4*>(out + static_cast<long long>(node) * ld_out)[threadIdx.x] = acc;
    return;
  }
  const int lane = threadIdx.x & 31;
  for (int node = blockIdx.x * 8 + (threadIdx.x >> 5); node < num_nodes; node += light_blocks * 8) {
    const int b = ptr[node], e = ptr[node + 1];
    if (in_sorted_list(heavy, num_heavy, node)) continue;   // a listed row: its own block
    float4 acc[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[q] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = b; j < e; ++j) {
      const float4* row = reinterpret_cast<const float4*>(msg + static_cast<long long>(order[j]) * ld_msg);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 t = __ldg(row + lane + 32 * q);
        acc[q].x += t.x; acc[q].y += t.y; acc[q].z += t.z; acc[q].w += t.w;
      }
    }
    float4* o = reinterpret_cast<float4*>(out + static_cast<long long>(node) * ld_out);
#pragma unroll
    for (int q = 0; q < 4; ++q) o[lane + 32 * q] = acc[q];
  }
}

// a[r, 0:n] = swish(h[r, 0:n]): the hidden activation of an MLP from its recomputed pre-activation.
__global__ void __launch_bounds__(256)
swish_rows_kernel(const float* __restrict__ h, int ld_h, long long rows, int n4, float* __restrict__ a,
                  int ld_a) {
  const long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= rows * n4) return;
  const long long r = t / n4;
  const int c = static_cast<int>(t % n4);
  float4 v = __ldg(reinterpret_cast<const float4*>(h + r * ld_h) + c);
  v.x = swish_fwd(v.x); v.y = swish_fwd(v.y); v.z = swish_fwd(v.z); v.w = swish_fwd(v.w);
  reinterpret_cast<float4*>(a + r * ld_a)[c] = v;
}

// dst[i, 0:w] = (addend ? addend[i, 0:w] : 0) + src[idx[i], 0:w]   (w a multiple of 4)
__global__ void __launch_bounds__(256)
gather_add_kernel(const float* __restrict__ src, int ld_src, const int* __restrict__ idx, long long n,
                  const float* __restrict__ addend, int ld_add, float* __restrict__ dst, int ld_dst, int w4) {
  const long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= n * w4) return;
  const long long i = t / w4;
  const int c = static_cast<int>(t % w4);
  float4 v = __ldg(reinterpret_cast<const float4*>(src + static_cast<long long>(idx[i]) * ld_src) + c);
  if (addend) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(addend + i * ld_add) + c);
    v.x = a.x + v.x; v.y = a.y + v.y; v.z = a.z + v.z; v.w = a.w + v.w;
  }
  reinterpret_cast<float4*>(dst + i * ld_dst)[c] = v;
}

// ---- seed of the loss derivative -----------------------------------------------------------------
// g[node, c] = coef[c] * lat_weight[node / n_lon] * (y[node, c] - t_norm[c, node]), t_norm exactly as
// output_loss_kernel forms it; the product in fp64, rounded once.  32 x 32 tiles: the target planes
// are read node-major (coalesced) into shared memory, y and g channel-major.
__global__ void __launch_bounds__(256)
output_loss_grad_kernel(const float* __restrict__ y, int ld_y, int n_out, int n_lon, long long n_nodes,
                        const float* __restrict__ scale, const float* __restrict__ offset,
                        const float* __restrict__ add_planes, const int* __restrict__ add_plane_index,
                        const float* __restrict__ targets, const float* __restrict__ lat_weight,
                        const double* __restrict__ coef, float* __restrict__ g, int ld_g) {
  __shared__ float tile[32][33];
  const long long node0 = static_cast<long long>(blockIdx.x) * 32;
  const int c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int r = ty; r < 32; r += 8) {
    const int c = c0 + r;
    const long long node = node0 + tx;
    float t_norm = 0.f;
    if (c < n_out && node < n_nodes) {
      const float sc = scale ? scale[c] : 1.f, of = offset ? offset[c] : 0.f;
      const int ap = add_plane_index ? add_plane_index[c] : -1;
      const float av = ap >= 0 ? add_planes[static_cast<long long>(ap) * n_nodes + node] : 0.f;
      t_norm = __fdiv_rn(__fsub_rn(__fsub_rn(targets[static_cast<long long>(c) * n_nodes + node], av), of), sc);
    }
    tile[r][tx] = t_norm;
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const long long node = node0 + r;
    const int c = c0 + tx;
    if (c < n_out && node < n_nodes) {
      const double d = static_cast<double>(__fsub_rn(y[node * ld_y + c], tile[tx][r]));
      g[node * ld_g + c] = static_cast<float>(coef[c] * static_cast<double>(lat_weight[node / n_lon]) * d);
    }
  }
}

// ---- backprop through time -----------------------------------------------------------------------
// Differentiates the feeding of one step's predictions into the next step's inputs
// (autoregressive.py:114-125, the loss unroll :262-310) through the residual add and the target
// normalisation of InputsAndResiduals (normalization.py:113-146).  A = dL / d(input planes) of a step,
// restricted to a list of rows (input channels); a_next is that of the following step.
//
// Blocks with blockIdx.y < c_tiles: the seed, node-major, as output_loss_grad_kernel plus the derivative
// that reaches the prediction through the next step's inputs:
//   g[node, c] = coef[c] * w * (y - t_norm) + scale[c] * a_next[dpred_row[c], node]   (fp64, rounded once)
// the second term only when a_next != NULL and dpred_row[c] >= 0, so that without it g is bit-identical
// to output_loss_grad_kernel.  The other blocks: rows r of a_out, channel-major,
//   a_out[r, node] = (c = resid_channel[r]) >= 0 ? (float)(g_loss[node, c] / scale[c] + a_next[dpred_row[c], node]) : 0
//                    (+ a_next[carry_row[r], node] when carry_row[r] >= 0)
// g_loss the first term of g: the residual add and the target normalisation both read the same last
// input frame; the carry is the frame shift.  Both tile kinds use the 32 x 32 shared-memory transpose.
__device__ __forceinline__ float loss_t_norm(int c, long long node, long long n_nodes,
                                             const float* __restrict__ scale, const float* __restrict__ offset,
                                             const float* __restrict__ add_planes,
                                             const int* __restrict__ add_plane_index,
                                             const float* __restrict__ targets) {
  const float sc = scale ? scale[c] : 1.f, of = offset ? offset[c] : 0.f;
  const int ap = add_plane_index ? add_plane_index[c] : -1;
  const float av = ap >= 0 ? add_planes[static_cast<long long>(ap) * n_nodes + node] : 0.f;
  return __fdiv_rn(__fsub_rn(__fsub_rn(targets[static_cast<long long>(c) * n_nodes + node], av), of), sc);
}

__global__ void __launch_bounds__(256)
output_loss_grad_feedback_kernel(const float* __restrict__ y, int ld_y, int n_out, int n_lon,
                                 long long n_nodes, const float* __restrict__ scale,
                                 const float* __restrict__ offset, const float* __restrict__ add_planes,
                                 const int* __restrict__ add_plane_index, const float* __restrict__ targets,
                                 const float* __restrict__ lat_weight, const double* __restrict__ coef,
                                 const float* __restrict__ a_next, const int* __restrict__ dpred_row,
                                 int n_rows, const int* __restrict__ resid_channel,
                                 const int* __restrict__ carry_row, float* __restrict__ a_out,
                                 float* __restrict__ g, int ld_g, int c_tiles) {
  __shared__ float tile[32][33];
  __shared__ float tile_dp[32][33];
  const long long node0 = static_cast<long long>(blockIdx.x) * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  if (static_cast<int>(blockIdx.y) < c_tiles) {
    const int c0 = blockIdx.y * 32;
    for (int r = ty; r < 32; r += 8) {
      const int c = c0 + r;
      const long long node = node0 + tx;
      float t_norm = 0.f, dp = 0.f;
      if (c < n_out && node < n_nodes) {
        t_norm = loss_t_norm(c, node, n_nodes, scale, offset, add_planes, add_plane_index, targets);
        const int q = a_next ? dpred_row[c] : -1;
        if (q >= 0) dp = a_next[static_cast<long long>(q) * n_nodes + node];
      }
      tile[r][tx] = t_norm;
      tile_dp[r][tx] = dp;
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {
      const long long node = node0 + r;
      const int c = c0 + tx;
      if (c < n_out && node < n_nodes) {
        const double d = static_cast<double>(__fsub_rn(y[node * ld_y + c], tile[tx][r]));
        double v = coef[c] * static_cast<double>(lat_weight[node / n_lon]) * d;
        if (a_next && dpred_row[c] >= 0)
          v += static_cast<double>(scale ? scale[c] : 1.f) * static_cast<double>(tile_dp[tx][r]);
        g[node * ld_g + c] = static_cast<float>(v);
      }
    }
    return;
  }
  const int r0 = (static_cast<int>(blockIdx.y) - c_tiles) * 32;
  // y[node, resid_channel[r]] of the tile's rows, node-major reads
  for (int q = ty; q < 32; q += 8) {
    const long long node = node0 + q;
    const int r = r0 + tx;
    float v = 0.f;
    if (r < n_rows && node < n_nodes) {
      const int c = resid_channel[r];
      if (c >= 0) v = y[node * ld_y + c];
    }
    tile[q][tx] = v;
  }
  __syncthreads();
  for (int q = ty; q < 32; q += 8) {
    const int r = r0 + q;
    const long long node = node0 + tx;
    if (r >= n_rows || node >= n_nodes) continue;
    float v = 0.f;
    const int c = resid_channel[r];
    if (c >= 0) {
      const float t_norm = loss_t_norm(c, node, n_nodes, scale, offset, add_planes, add_plane_index, targets);
      const double d = static_cast<double>(__fsub_rn(tile[tx][q], t_norm));
      const double gl = coef[c] * static_cast<double>(lat_weight[node / n_lon]) * d;
      const int p = a_next ? dpred_row[c] : -1;
      const double dp = p >= 0 ? static_cast<double>(a_next[static_cast<long long>(p) * n_nodes + node]) : 0.0;
      v = static_cast<float>(gl / static_cast<double>(scale ? scale[c] : 1.f) + dp);
    }
    const int k = (a_next && carry_row) ? carry_row[r] : -1;
    if (k >= 0) v = __fadd_rn(v, a_next[static_cast<long long>(k) * n_nodes + node]);
    a_out[static_cast<long long>(r) * n_nodes + node] = v;
  }
}

// The seed of a Gauss-Newton product over several target times.  The loss is a quadratic in the
// normalised residual r = y - t_norm = (pred - target) / scale, so its Gauss-Newton cotangent is
// coef[c] * w * d with d = pdot / scale (fp32, true division; scale NULL = 1) the tangent of r, pdot
// [n_out, n_nodes] the channel-major tangent of the physical predictions.  With d in place of y - t_norm
// this is output_loss_grad_feedback_kernel's arithmetic:
//   g[node, c]     = coef[c] * w * d + scale[c] * a_next[dpred_row[c], node]   (fp64, rounded once)
//   a_out[r, node] = c >= 0 ? (float)(coef[c] * w * d / scale[c] + a_next[dpred_row[c], node]) : 0
//                    (+ a_next[carry_row[r], node] when carry_row[r] >= 0)
// d is rounded as that kernel rounds y - t_norm with t_norm = +0, so with scale NULL both outputs are its
// bits for y = pdot^T and all-zero targets.  The c-tile blocks transpose d and the feedback row through
// the 32 x 32 shared-memory tiles; the row blocks read pdot channel-major as they write a_out.
__device__ __forceinline__ float gn_residual_tangent(int c, long long node, long long n_nodes,
                                                     const float* __restrict__ scale,
                                                     const float* __restrict__ pdot) {
  const float p = pdot[static_cast<long long>(c) * n_nodes + node];
  return __fsub_rn(scale ? __fdiv_rn(p, scale[c]) : p, 0.f);
}

__global__ void __launch_bounds__(256)
output_loss_gn_seed_feedback_kernel(const float* __restrict__ pdot, int n_out, int n_lon,
                                    long long n_nodes, const float* __restrict__ scale,
                                    const float* __restrict__ lat_weight, const double* __restrict__ coef,
                                    const float* __restrict__ a_next, const int* __restrict__ dpred_row,
                                    int n_rows, const int* __restrict__ resid_channel,
                                    const int* __restrict__ carry_row, float* __restrict__ a_out,
                                    float* __restrict__ g, int ld_g, int c_tiles) {
  const long long node0 = static_cast<long long>(blockIdx.x) * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  if (static_cast<int>(blockIdx.y) < c_tiles) {
    __shared__ float tile[32][33];
    __shared__ float tile_dp[32][33];
    const int c0 = blockIdx.y * 32;
    for (int r = ty; r < 32; r += 8) {
      const int c = c0 + r;
      const long long node = node0 + tx;
      float d = 0.f, dp = 0.f;
      if (c < n_out && node < n_nodes) {
        d = gn_residual_tangent(c, node, n_nodes, scale, pdot);
        const int q = a_next ? dpred_row[c] : -1;
        if (q >= 0) dp = a_next[static_cast<long long>(q) * n_nodes + node];
      }
      tile[r][tx] = d;
      tile_dp[r][tx] = dp;
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {
      const long long node = node0 + r;
      const int c = c0 + tx;
      if (c < n_out && node < n_nodes) {
        const double d = static_cast<double>(tile[tx][r]);
        double v = coef[c] * static_cast<double>(lat_weight[node / n_lon]) * d;
        if (a_next && dpred_row[c] >= 0)
          v += static_cast<double>(scale ? scale[c] : 1.f) * static_cast<double>(tile_dp[tx][r]);
        g[node * ld_g + c] = static_cast<float>(v);
      }
    }
    return;
  }
  const int r0 = (static_cast<int>(blockIdx.y) - c_tiles) * 32;
  for (int q = ty; q < 32; q += 8) {
    const int r = r0 + q;
    const long long node = node0 + tx;
    if (r >= n_rows || node >= n_nodes) continue;
    float v = 0.f;
    const int c = resid_channel[r];
    if (c >= 0) {
      const double d = static_cast<double>(gn_residual_tangent(c, node, n_nodes, scale, pdot));
      const double gl = coef[c] * static_cast<double>(lat_weight[node / n_lon]) * d;
      const int p = a_next ? dpred_row[c] : -1;
      const double dp = p >= 0 ? static_cast<double>(a_next[static_cast<long long>(p) * n_nodes + node]) : 0.0;
      v = static_cast<float>(gl / static_cast<double>(scale ? scale[c] : 1.f) + dp);
    }
    const int k = (a_next && carry_row) ? carry_row[r] : -1;
    if (k >= 0) v = __fadd_rn(v, a_next[static_cast<long long>(k) * n_nodes + node]);
    a_out[static_cast<long long>(r) * n_nodes + node] = v;
  }
}

// Transpose of pack_grid_image_kernel's normalisation for a list of rows (normalization.py:113-146,
// the input side of InputsAndResiduals): a[r, node] (+)= dx[node, channel[r]] / scale[channel[r]]
// (true division; scale == NULL divides by 1).  dx is read node-major through a 32 x 32 shared tile,
// a written channel-major.  One addition per element: deterministic.
__global__ void __launch_bounds__(256)
input_grad_kernel(const float* __restrict__ dx, int ld_dx, long long n_nodes, int n_rows,
                  const int* __restrict__ channel, const float* __restrict__ scale,
                  float* __restrict__ a, int accumulate) {
  __shared__ float tile[32][33];
  const long long node0 = static_cast<long long>(blockIdx.x) * 32;
  const int r0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int q = ty; q < 32; q += 8) {
    const long long node = node0 + q;
    const int r = r0 + tx;
    tile[q][tx] = (r < n_rows && node < n_nodes) ? __ldg(dx + node * ld_dx + channel[r]) : 0.f;
  }
  __syncthreads();
  for (int q = ty; q < 32; q += 8) {
    const int r = r0 + q;
    const long long node = node0 + tx;
    if (r < n_rows && node < n_nodes) {
      float v = tile[tx][q];
      if (scale) v = __fdiv_rn(v, scale[channel[r]]);
      float* p = a + static_cast<long long>(r) * n_nodes + node;
      *p = accumulate ? __fadd_rn(*p, v) : v;
    }
  }
}

// ---- input gradients of a vector-Jacobian product ---------------------------------------------------
// The seed of J = sum cot * pred over the physical predictions pred = y * scale + (offset | add), with
// the feedback of output_loss_grad_feedback_kernel: d[c, node] = cot[c, node] + a_next[dpred_row[c], node]
// (the second term when a_next != NULL and dpred_row[c] >= 0; fp64, rounded once) is dJ/dpred.
// Blocks with blockIdx.y < c_tiles: g[node, c] = (float)(scale[c] * d), node-major through the 32 x 32
// shared-memory transpose.  The other blocks: rows r of a_out, channel-major,
//   a_out[r, node] = (c = resid_channel[r]) >= 0 ? (float)d[c, node] : 0  (+ a_next[carry_row[r], node])
__device__ __forceinline__ double cotangent_d(int c, long long node, long long n_nodes,
                                              const float* __restrict__ cot,
                                              const float* __restrict__ a_next,
                                              const int* __restrict__ dpred_row) {
  double d = static_cast<double>(cot[static_cast<long long>(c) * n_nodes + node]);
  const int q = a_next ? dpred_row[c] : -1;
  if (q >= 0) d += static_cast<double>(a_next[static_cast<long long>(q) * n_nodes + node]);
  return d;
}

__global__ void __launch_bounds__(256)
output_cotangent_grad_feedback_kernel(int n_out, long long n_nodes, const float* __restrict__ scale,
                                      const float* __restrict__ cot, const float* __restrict__ a_next,
                                      const int* __restrict__ dpred_row, int n_rows,
                                      const int* __restrict__ resid_channel,
                                      const int* __restrict__ carry_row, float* __restrict__ a_out,
                                      float* __restrict__ g, int ld_g, int c_tiles) {
  const long long node0 = static_cast<long long>(blockIdx.x) * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  if (static_cast<int>(blockIdx.y) < c_tiles) {
    __shared__ float tile[32][33];
    const int c0 = blockIdx.y * 32;
    for (int r = ty; r < 32; r += 8) {
      const int c = c0 + r;
      const long long node = node0 + tx;
      float v = 0.f;
      if (c < n_out && node < n_nodes) {
        const double sc = scale ? static_cast<double>(scale[c]) : 1.0;
        v = static_cast<float>(sc * cotangent_d(c, node, n_nodes, cot, a_next, dpred_row));
      }
      tile[r][tx] = v;
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {
      const long long node = node0 + r;
      const int c = c0 + tx;
      if (c < n_out && node < n_nodes) g[node * ld_g + c] = tile[tx][r];
    }
    return;
  }
  const int r0 = (static_cast<int>(blockIdx.y) - c_tiles) * 32;
  for (int q = ty; q < 32; q += 8) {
    const int r = r0 + q;
    const long long node = node0 + tx;
    if (r >= n_rows || node >= n_nodes) continue;
    const int c = resid_channel[r];
    float v = c >= 0 ? static_cast<float>(cotangent_d(c, node, n_nodes, cot, a_next, dpred_row)) : 0.f;
    const int k = (a_next && carry_row) ? carry_row[r] : -1;
    if (k >= 0) v = __fadd_rn(v, a_next[static_cast<long long>(k) * n_nodes + node]);
    a_out[static_cast<long long>(r) * n_nodes + node] = v;
  }
}

// Transpose of the host broadcast of a variable that lacks lat and / or lon (model_utils
// .variable_to_planes): for row i of the list, the plane a[rows[i]] [n_lat, n_lon] summed over lat
// (kMode 1: out [n_rows, n_lon]), over lat and lon (kMode 2: out [n_rows]) or not at all (kMode 0: out
// [n_rows, n_lat * n_lon]).  fp64 sums in a fixed order, one rounding per output element, optionally
// added to out (accumulate: out = (float)(out + sum)).
constexpr int kBcastNone = 0, kBcastLat = 1, kBcastLatLon = 2;

template <int kMode>
__global__ void __launch_bounds__(256)
broadcast_grad_sum_kernel(const float* __restrict__ a, int n_lat, int n_lon,
                          const int* __restrict__ rows, float* __restrict__ out, int accumulate) {
  const long long n_nodes = static_cast<long long>(n_lat) * n_lon;
  const int i = blockIdx.y;
  const float* src = a + static_cast<long long>(rows[i]) * n_nodes;
  if constexpr (kMode == kBcastLatLon) {
    __shared__ double part[256];
    double s = 0.0;
    for (long long j = threadIdx.x; j < n_nodes; j += 256) s += static_cast<double>(__ldg(src + j));
    part[threadIdx.x] = s;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
      if (static_cast<int>(threadIdx.x) < w) part[threadIdx.x] += part[threadIdx.x + w];
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      float* p = out + i;
      *p = static_cast<float>(accumulate ? static_cast<double>(*p) + part[0] : part[0]);
    }
  } else {
    const long long width = kMode == kBcastLat ? n_lon : n_nodes;
    const long long j = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
    if (j >= width) return;
    double s;
    if constexpr (kMode == kBcastLat) {
      s = 0.0;
      for (int la = 0; la < n_lat; ++la) s += static_cast<double>(__ldg(src + static_cast<long long>(la) * n_lon + j));
    } else {
      s = static_cast<double>(__ldg(src + j));
    }
    float* p = out + static_cast<long long>(i) * width + j;
    *p = static_cast<float>(accumulate ? static_cast<double>(*p) + s : s);
  }
}

}  // namespace gcb
