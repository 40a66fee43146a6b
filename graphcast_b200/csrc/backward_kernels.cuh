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
      float mean = 0.f;
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
      const float rstd = rsqrtf(var * (1.0f / n) + 1e-5f);
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

}  // namespace gcb
