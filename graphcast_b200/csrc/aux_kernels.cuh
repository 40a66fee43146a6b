// HBM-bound helper kernels of the GraphCast step: receiver-sorted segment sum and
// the channel pack / unpack transposes (with the normalisation affine fused in).
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

#include "ptx.cuh"

namespace gcb {

// out[node, :] = sum over in-edges (CSR row_ptr, edges receiver-sorted) of msg[e, :].
// One warp per receiver node; lane l owns float4 columns l, l+32, ... so every
// edge row is read with fully coalesced 512-byte warp loads and each output row
// is written once -- no atomics, deterministic order.
//
// Receivers with more than kHeavyDegree in-edges (the mesh nodes next to the poles collect
// thousands of grid points) would serialise one warp for milliseconds; they are listed in
// `heavy` and handled by the last `num_heavy` blocks, one block per node: eight warps sum
// contiguous slices of the node's edges and combine them in a fixed order (still
// deterministic).
constexpr int kHeavyDegree = 256;

// Four consecutive columns (col % 4 == 0) of row `row` into an operand image of a [rows, k]
// matrix: 8 bytes of bf16 "hi" and 8 bytes of "lo" (layout: GCB_A_IMAGE_BLOCK, graphcast_b200.h).
__device__ __forceinline__ void store_image_f4(unsigned char* img, long long row, int col, int k,
                                               const float4& v) {
  uint2 hi, lo;
  ptx::split_bf16x4(v, hi, lo);
  unsigned char* dst = img + (static_cast<size_t>(row >> 7) * (k >> 4) + (col >> 4)) * 8448 +
                       ((col >> 3) & 1) * 2112 + (row & 127) * 16 + (col & 7) * 2;
  *reinterpret_cast<uint2*>(dst) = hi;
  *reinterpret_cast<uint2*>(dst + 4224) = lo;
}

// `img` (optional): also emit the sums as an operand image of the [num_nodes, 128*kVecPerLane]
// result, so that the consuming layer needs no separate conversion pass.
template <int kVecPerLane>
__global__ void __launch_bounds__(256)
segment_sum_kernel(const float* __restrict__ msg, int ld_msg, const int* __restrict__ row_ptr,
                   int num_nodes, float* __restrict__ out, int ld_out,
                   const int* __restrict__ heavy, int num_heavy, unsigned char* __restrict__ img) {
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const int light_blocks = gridDim.x - num_heavy;
  if (static_cast<int>(blockIdx.x) >= light_blocks) {
    // ---- one block per heavy receiver ----
    __shared__ float4 part[8][32 * kVecPerLane];
    const int node = heavy[blockIdx.x - light_blocks];
    const int beg = row_ptr[node], end = row_ptr[node + 1];
    const int w = threadIdx.x >> 5;
    const int per = (end - beg + 7) / 8;
    const int lo = beg + w * per, hi = min(end, lo + per);
    float4 acc[kVecPerLane];
#pragma unroll
    for (int j = 0; j < kVecPerLane; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int e = lo; e < hi; ++e) {
      const float4* pa = reinterpret_cast<const float4*>(msg + static_cast<long long>(e) * ld_msg);
#pragma unroll
      for (int j = 0; j < kVecPerLane; ++j) {
        const float4 a = __ldg(pa + lane + 32 * j);
        acc[j].x += a.x; acc[j].y += a.y; acc[j].z += a.z; acc[j].w += a.w;
      }
    }
#pragma unroll
    for (int j = 0; j < kVecPerLane; ++j) part[w][lane + 32 * j] = acc[j];
    __syncthreads();
    for (int i = threadIdx.x; i < 32 * kVecPerLane; i += blockDim.x) {
      float4 s = part[0][i];
      for (int k = 1; k < 8; ++k) { s.x += part[k][i].x; s.y += part[k][i].y; s.z += part[k][i].z; s.w += part[k][i].w; }
      reinterpret_cast<float4*>(out + static_cast<long long>(node) * ld_out)[i] = s;
      if (img) store_image_f4(img, node, 4 * i, 128 * kVecPerLane, s);
    }
    return;
  }
  const long long gwarp = static_cast<long long>(blockIdx.x) * warps_per_block + (threadIdx.x >> 5);
  const long long nwarps = static_cast<long long>(light_blocks) * warps_per_block;
  for (long long node = gwarp; node < num_nodes; node += nwarps) {
    const int beg = row_ptr[node], end = row_ptr[node + 1];
    if (num_heavy > 0 && end - beg > kHeavyDegree) continue;   // done by a heavy block
    float4 acc[kVecPerLane];
#pragma unroll
    for (int j = 0; j < kVecPerLane; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    int e = beg;
    for (; e + 1 < end; e += 2) {
      float4 a[kVecPerLane], b[kVecPerLane];
      const float4* pa = reinterpret_cast<const float4*>(msg + static_cast<long long>(e) * ld_msg);
      const float4* pb = reinterpret_cast<const float4*>(msg + static_cast<long long>(e + 1) * ld_msg);
#pragma unroll
      for (int j = 0; j < kVecPerLane; ++j) { a[j] = __ldg(pa + lane + 32 * j); b[j] = __ldg(pb + lane + 32 * j); }
#pragma unroll
      for (int j = 0; j < kVecPerLane; ++j) {
        acc[j].x += a[j].x; acc[j].y += a[j].y; acc[j].z += a[j].z; acc[j].w += a[j].w;
        acc[j].x += b[j].x; acc[j].y += b[j].y; acc[j].z += b[j].z; acc[j].w += b[j].w;
      }
    }
    if (e < end) {
      const float4* pa = reinterpret_cast<const float4*>(msg + static_cast<long long>(e) * ld_msg);
#pragma unroll
      for (int j = 0; j < kVecPerLane; ++j) {
        const float4 a = __ldg(pa + lane + 32 * j);
        acc[j].x += a.x; acc[j].y += a.y; acc[j].z += a.z; acc[j].w += a.w;
      }
    }
    float4* po = reinterpret_cast<float4*>(out + node * ld_out);
#pragma unroll
    for (int j = 0; j < kVecPerLane; ++j) po[lane + 32 * j] = acc[j];
    if (img) {
#pragma unroll
      for (int j = 0; j < kVecPerLane; ++j)
        store_image_f4(img, node, 4 * (lane + 32 * j), 128 * kVecPerLane, acc[j]);
    }
  }
}

// dst[i, 0:width] = src[idx[i], 0:width]  (width a multiple of 4 floats).  The send side of the
// halo exchange of the node-partitioned processor: boundary rows of the latent table, gathered
// into one contiguous buffer per step.  One warp per row, float4 lanes: coalesced both ways.
__global__ void __launch_bounds__(256)
gather_rows_kernel(const float* __restrict__ src, int ld_src, const int* __restrict__ idx,
                   long long n, float* __restrict__ dst, int ld_dst, int width) {
  const int lane = threadIdx.x & 31;
  const long long warp = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nwarps = static_cast<long long>(gridDim.x) * (blockDim.x >> 5);
  for (long long i = warp; i < n; i += nwarps) {
    const float4* s = reinterpret_cast<const float4*>(src + static_cast<long long>(idx[i]) * ld_src);
    float4* d = reinterpret_cast<float4*>(dst + i * ld_dst);
    for (int c = lane; c < (width >> 2); c += 32) d[c] = __ldg(s + c);
  }
}

// Rows of an operand image of a [*, 512] matrix <-> a dense buffer of 2048-byte packed rows (the
// send / receive side of a halo exchange when the latent stream exists only as an image).  A packed
// row holds, per (K-step, 8-column chunk) piece, the 16 bytes of bf16 "hi" then the 16 bytes of "lo"
// exactly as the image stores them, so the receiver's image rows are the owner's bit for bit.
// kToImage = false: buf[i] = image row idx[i];  true: image row first_row + i = buf[i].
template <bool kToImage>
__global__ void __launch_bounds__(256)
image_rows_kernel(unsigned char* __restrict__ img, const int* __restrict__ idx, long long first_row,
                  long long n, unsigned char* __restrict__ buf) {
  const int lane = threadIdx.x & 31;
  const long long warp = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nwarps = static_cast<long long>(gridDim.x) * (blockDim.x >> 5);
  for (long long i = warp; i < n; i += nwarps) {
    const long long row = kToImage ? first_row + i : static_cast<long long>(idx[i]);
    unsigned char* tile = img + static_cast<size_t>(row >> 7) * 32 * 8448 + (row & 127) * 16;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int piece = lane + 32 * h;              // (K-step, chunk) = (piece >> 1, piece & 1)
      unsigned char* p = tile + static_cast<size_t>(piece >> 1) * 8448 + (piece & 1) * 2112;
      uint4* b = reinterpret_cast<uint4*>(buf + i * 2048 + piece * 32);
      if (kToImage) {
        *reinterpret_cast<uint4*>(p) = b[0];
        *reinterpret_cast<uint4*>(p + 4224) = b[1];
      } else {
        b[0] = *reinterpret_cast<const uint4*>(p);
        b[1] = *reinterpret_cast<const uint4*>(p + 4224);
      }
    }
  }
}

// planes [n_ch, n_nodes] (+ node_static [n_nodes, n_static]) -> feats [n_nodes, ld],
// feats[i, c] = (planes[c, i] - mean[c]) / scale[c]; 32x32 smem-tiled transpose so
// both the plane reads (along nodes) and the feature writes (along channels) are
// coalesced.
__global__ void __launch_bounds__(256)
pack_grid_features_kernel(const float* __restrict__ planes, int n_ch, long long n_nodes,
                          const float* __restrict__ mean, const float* __restrict__ scale,
                          const float* __restrict__ node_static, int n_static,
                          float* __restrict__ feats, int ld) {
  __shared__ float tile[32][33];
  const long long node0 = static_cast<long long>(blockIdx.x) * 32;
  const int c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
  for (int r = ty; r < 32; r += 8) {
    const int c = c0 + r;
    const long long node = node0 + tx;
    float v = 0.f;
    if (node < n_nodes) {
      if (c < n_ch) {
        v = planes[static_cast<long long>(c) * n_nodes + node];
        if (mean) v -= mean[c];
        if (scale) v /= scale[c];
      } else if (c < n_ch + n_static) {
        v = node_static[node * n_static + (c - n_ch)];
      }
    }
    tile[r][tx] = v;
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const long long node = node0 + r;
    const int c = c0 + tx;
    if (node < n_nodes && c < ld) feats[node * ld + c] = tile[tx][r];
  }
}

// planes [n_ch, n_nodes] (+ node_static) -> operand image of the packed, normalised feature
// rows [n_nodes, k] (k = padded channel count, multiple of 16): the fp32 feature matrix is
// never materialised.  A block handles 32 nodes: phase 1 reads every channel plane with
// 128-byte coalesced loads into a shared tile, phase 2 lets lane = node emit the 16-byte
// image pieces (512-byte warp stores), as in rows_to_image_kernel.
__global__ void __launch_bounds__(256)
pack_grid_image_kernel(const float* __restrict__ planes, int n_ch, long long n_nodes,
                       const float* __restrict__ mean, const float* __restrict__ scale,
                       const float* __restrict__ node_static, int n_static, int k,
                       unsigned char* __restrict__ img) {
  extern __shared__ float tile[];                 // [32][k + 4]
  const int kp = k + 4;
  const long long node0 = static_cast<long long>(blockIdx.x) * 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long node = node0 + lane;
  // Phase 1 is pure latency (one 128-byte line per warp and channel): keep kU independent
  // plane loads in flight per warp instead of one.
  constexpr int kU = 6;
  for (int c0 = warp; c0 < k; c0 += 8 * kU) {
    float v[kU], mu[kU], sd[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const int c = c0 + 8 * u;
      v[u] = 0.f; mu[u] = 0.f; sd[u] = 1.f;
      if (c < n_ch) {
        if (node < n_nodes) v[u] = planes[static_cast<long long>(c) * n_nodes + node];
        if (mean) mu[u] = mean[c];
        if (scale) sd[u] = scale[c];
      } else if (c < n_ch + n_static && node < n_nodes) {
        v[u] = node_static[node * n_static + (c - n_ch)];
      }
    }
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const int c = c0 + 8 * u;
      if (c < k) {
        float x = v[u];
        if (c < n_ch && node < n_nodes) {
          if (mean) x -= mu[u];
          if (scale) x /= sd[u];
        }
        tile[lane * kp + c] = x;
      }
    }
  }
  __syncthreads();
  const long long t = node >> 7;
  const int r = static_cast<int>(node & 127);
  const int ksteps = k >> 4;
  for (int piece = warp; piece < ksteps * 2; piece += 8) {
    const int ks = piece >> 1, c = piece & 1;
    const float* x = tile + lane * kp + ks * 16 + c * 8;
    const float4 a = *reinterpret_cast<const float4*>(x), b = *reinterpret_cast<const float4*>(x + 4);
    __nv_bfloat162 h0 = __floats2bfloat162_rn(a.x, a.y), h1 = __floats2bfloat162_rn(a.z, a.w);
    __nv_bfloat162 h2 = __floats2bfloat162_rn(b.x, b.y), h3 = __floats2bfloat162_rn(b.z, b.w);
    const float2 f0 = __bfloat1622float2(h0), f1 = __bfloat1622float2(h1);
    const float2 f2 = __bfloat1622float2(h2), f3 = __bfloat1622float2(h3);
    __nv_bfloat162 l0 = __floats2bfloat162_rn(a.x - f0.x, a.y - f0.y), l1 = __floats2bfloat162_rn(a.z - f1.x, a.w - f1.y);
    __nv_bfloat162 l2 = __floats2bfloat162_rn(b.x - f2.x, b.y - f2.y), l3 = __floats2bfloat162_rn(b.z - f3.x, b.w - f3.y);
    if (node < ((n_nodes + 127) >> 7 << 7)) {
      unsigned char* dst = img + (static_cast<size_t>(t) * ksteps + ks) * 8448 + c * 2112 + r * 16;
      uint4 hv, lv;
      hv.x = *reinterpret_cast<unsigned int*>(&h0); hv.y = *reinterpret_cast<unsigned int*>(&h1);
      hv.z = *reinterpret_cast<unsigned int*>(&h2); hv.w = *reinterpret_cast<unsigned int*>(&h3);
      lv.x = *reinterpret_cast<unsigned int*>(&l0); lv.y = *reinterpret_cast<unsigned int*>(&l1);
      lv.z = *reinterpret_cast<unsigned int*>(&l2); lv.w = *reinterpret_cast<unsigned int*>(&l3);
      *reinterpret_cast<uint4*>(dst) = hv;
      *reinterpret_cast<uint4*>(dst + 4224) = lv;
    }
  }
}

// TOA incident solar radiation (the reference's solar_radiation.get_toa_incident_solar_radiation,
// :443-521): out[t, h, w] = sum_b f[t,b] * max(cos_lat[h] * cd[t,b] * cos(H0[t,b] + lon[w]) +
// sin_lat[h] * sd[t,b], 0), the trapezoidal time integral of the instantaneous flux.  The per-bin
// orbital quantities are scalars computed on the host in float64 (`table`: [T, B, 5] =
// cos / sin of the declination, cos / sin of the hour angle at longitude 0, and
// weight * TSI / d^2 * dx); cos(H0 + lon) is expanded with the angle-sum identity, so the bin loop
// has no transcendental.  One thread per grid point, the bin table of the block's timestamp in
// shared memory; reads 3 small vectors, writes the field once (HBM-bound at 0.25 degree).
__global__ void __launch_bounds__(256)
tisr_kernel(const float* __restrict__ table, int bins, const float* __restrict__ sin_lat,
            const float* __restrict__ cos_lat, const float* __restrict__ cos_lon,
            const float* __restrict__ sin_lon, int n_lat, int n_lon, float* __restrict__ out) {
  extern __shared__ float s_tab[];                  // [bins][5]
  const int t = blockIdx.z, h = blockIdx.y;
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  const float* tab = table + static_cast<size_t>(t) * bins * 5;
  for (int i = threadIdx.x; i < bins * 5; i += blockDim.x) s_tab[i] = tab[i];
  __syncthreads();
  if (w >= n_lon) return;
  const float sl = sin_lat[h], cl = cos_lat[h], cw = cos_lon[w], sw = sin_lon[w];
  float acc = 0.f;
  for (int b = 0; b < bins; ++b) {
    const float* p = s_tab + 5 * b;
    const float cos_h = p[2] * cw - p[3] * sw;      // cos(H0 + lon)
    const float sin_alt = fmaf(cl * p[0], cos_h, sl * p[1]);
    acc = fmaf(p[4], fmaxf(sin_alt, 0.f), acc);
  }
  out[(static_cast<size_t>(t) * n_lat + h) * n_lon + w] = acc;
}

// y [n_nodes, ld_y] -> planes_out [n_out, n_nodes] with per-channel affine and an
// optional additive plane (the last input frame for residual targets).
__global__ void __launch_bounds__(256)
unpack_grid_outputs_kernel(const float* __restrict__ y, int ld_y, int n_out, long long n_nodes,
                           const float* __restrict__ scale, const float* __restrict__ offset,
                           const float* __restrict__ add_planes,
                           const int* __restrict__ add_plane_index,
                           float* __restrict__ planes_out) {
  __shared__ float tile[32][33];
  const long long node0 = static_cast<long long>(blockIdx.x) * 32;
  const int c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int r = ty; r < 32; r += 8) {
    const long long node = node0 + r;
    const int c = c0 + tx;
    tile[r][tx] = (node < n_nodes && c < n_out) ? y[node * ld_y + c] : 0.f;
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const int c = c0 + r;
    const long long node = node0 + tx;
    if (c < n_out && node < n_nodes) {
      float v = tile[tx][r];
      if (scale) v *= scale[c];
      if (offset) v += offset[c];
      if (add_plane_index) {
        const int ap = add_plane_index[c];
        if (ap >= 0) v += add_planes[static_cast<long long>(ap) * n_nodes + node];
      }
      planes_out[static_cast<long long>(c) * n_nodes + node] = v;
    }
  }
}

// Fixed number of node groups of the loss reduction: every device splits the node tiles the same
// way, so the fp64 partial sums -- and the result -- are bit-identical on any GPU.
constexpr int kLossGroups = 512;

// Latitude-weighted squared error of the raw outputs against normalised targets (the loss of
// normalization.InputsAndResiduals / GraphCast.loss_and_predictions), per channel:
//   t_norm = ((target - add) - offset) / scale           (fp32, true division)
//   partial[g, c] = sum over the node tiles of group g of lat_weight[node / n_lon] * (y - t_norm)^2
// in fp64.  Same 32x32 transpose as unpack_grid_outputs_kernel (y is node-major, the target and
// prediction planes channel-major); `planes_out` (optional) receives exactly what that kernel
// writes, from the same expression.  Block (g, channel tile) walks the node tiles g, g + G, ... in
// order; each warp owns four channels and folds its 32 lanes with a fixed butterfly.  No atomics.
__global__ void __launch_bounds__(256)
output_loss_kernel(const float* __restrict__ y, int ld_y, int n_out, int n_lon, long long n_nodes,
                   const float* __restrict__ scale, const float* __restrict__ offset,
                   const float* __restrict__ add_planes, const int* __restrict__ add_plane_index,
                   const float* __restrict__ targets, const float* __restrict__ lat_weight,
                   float* __restrict__ planes_out, double* __restrict__ partial) {
  __shared__ float tile[32][33];
  const int c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const long long n_tiles = (n_nodes + 31) / 32;
  // The thread's four channels c0 + ty + 8j: their constants once, outside the node loop.
  float sc[4], of[4];
  int ap[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int c = min(c0 + ty + 8 * j, n_out - 1);
    sc[j] = scale ? scale[c] : 1.f;
    of[j] = offset ? offset[c] : 0.f;
    ap[j] = add_plane_index ? add_plane_index[c] : -1;
  }
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  for (long long t = blockIdx.x; t < n_tiles; t += kLossGroups) {
    const long long node0 = t * 32;
    for (int r = ty; r < 32; r += 8) {
      const long long node = node0 + r;
      const int c = c0 + tx;
      tile[r][tx] = (node < n_nodes && c < n_out) ? y[node * ld_y + c] : 0.f;
    }
    const long long node = node0 + tx;
    // the plane reads of the tile, issued together
    float tv[4], av[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = c0 + ty + 8 * j;
      const bool ok = c < n_out && node < n_nodes;
      tv[j] = ok ? targets[static_cast<long long>(c) * n_nodes + node] : 0.f;
      av[j] = ok && ap[j] >= 0 ? add_planes[static_cast<long long>(ap[j]) * n_nodes + node] : 0.f;
    }
    const double w = node < n_nodes ? static_cast<double>(lat_weight[node / n_lon]) : 0.0;
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = c0 + ty + 8 * j;
      if (c < n_out && node < n_nodes) {
        const float raw = tile[tx][ty + 8 * j];
        // the prediction: the expression of unpack_grid_outputs_kernel, same operations in order
        float v = raw;
        if (scale) v *= sc[j];
        if (offset) v += of[j];
        if (ap[j] >= 0) v += av[j];
        if (planes_out) planes_out[static_cast<long long>(c) * n_nodes + node] = v;
        const float t_norm = __fdiv_rn(__fsub_rn(__fsub_rn(tv[j], av[j]), of[j]), sc[j]);
        const double d = static_cast<double>(__fsub_rn(raw, t_norm));
        acc[j] += w * (d * d);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    double s = acc[j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const int c = c0 + ty + 8 * j;
    if (tx == 0 && c < n_out) partial[static_cast<long long>(blockIdx.x) * n_out + c] = s;
  }
}

// channel_sums[c] = sum over g = 0..kLossGroups-1 (in this order) of partial[g, c].
__global__ void __launch_bounds__(128)
loss_partials_kernel(const double* __restrict__ partial, int n_out, double* __restrict__ channel_sums) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_out) return;
  double s = 0.0;
  for (int g = 0; g < kLossGroups; ++g) s += partial[static_cast<long long>(g) * n_out + c];
  channel_sums[c] = s;
}

// img[r, 0:k] = sum_{j<fan} src[r*fan + j, 0:k] written as an operand image (bf16 hi/lo
// in the tensor-core A layout, see gcb_layer_desc).  A block handles 32 output rows:
// phase 1 sums the fan input rows with coalesced float4 reads into a padded shared tile,
// phase 2 lets lane = row emit the 16-byte image pieces, so a warp stores 512 contiguous
// bytes.  HBM-bound: fan*k*4 bytes read + ~k*4 written per row.
__global__ void __launch_bounds__(256)
rows_to_image_kernel(const float* __restrict__ src, int ld, int fan, long long rows, int k,
                     unsigned char* __restrict__ img) {
  extern __shared__ float tile[];                 // [32][k + 4]
  const int kp = k + 4;
  const long long row0 = static_cast<long long>(blockIdx.x) * 32;
  const int nvec = k >> 2;                        // float4 per row
  for (int e = threadIdx.x; e < 32 * nvec; e += blockDim.x) {
    const int r = e / nvec, c4 = e % nvec;
    const long long grow = row0 + r;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (grow < rows) {
      const float* p = src + grow * fan * ld + c4 * 4;
      for (int j = 0; j < fan; ++j) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(p + static_cast<long long>(j) * ld));
        acc.x += t.x; acc.y += t.y; acc.z += t.z; acc.w += t.w;
      }
    }
    *reinterpret_cast<float4*>(tile + r * kp + c4 * 4) = acc;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long grow = row0 + lane;
  const long long t = grow >> 7;
  const int r = static_cast<int>(grow & 127);
  const int ksteps = k >> 4;
  // 16-byte pieces: (K-step, chunk) pairs distributed over the 8 warps
  for (int piece = warp; piece < ksteps * 2; piece += 8) {
    const int ks = piece >> 1, c = piece & 1;
    const float* x = tile + lane * kp + ks * 16 + c * 8;
    const float4 a = *reinterpret_cast<const float4*>(x), b = *reinterpret_cast<const float4*>(x + 4);
    __nv_bfloat162 h0 = __floats2bfloat162_rn(a.x, a.y), h1 = __floats2bfloat162_rn(a.z, a.w);
    __nv_bfloat162 h2 = __floats2bfloat162_rn(b.x, b.y), h3 = __floats2bfloat162_rn(b.z, b.w);
    const float2 f0 = __bfloat1622float2(h0), f1 = __bfloat1622float2(h1);
    const float2 f2 = __bfloat1622float2(h2), f3 = __bfloat1622float2(h3);
    __nv_bfloat162 l0 = __floats2bfloat162_rn(a.x - f0.x, a.y - f0.y), l1 = __floats2bfloat162_rn(a.z - f1.x, a.w - f1.y);
    __nv_bfloat162 l2 = __floats2bfloat162_rn(b.x - f2.x, b.y - f2.y), l3 = __floats2bfloat162_rn(b.z - f3.x, b.w - f3.y);
    if (grow < ((rows + 127) >> 7 << 7)) {        // rows of the last tile beyond `rows` get zeros
      unsigned char* dst = img + (static_cast<size_t>(t) * ksteps + ks) * 8448 + c * 2112 + r * 16;
      uint4 hv, lv;
      hv.x = *reinterpret_cast<unsigned int*>(&h0); hv.y = *reinterpret_cast<unsigned int*>(&h1);
      hv.z = *reinterpret_cast<unsigned int*>(&h2); hv.w = *reinterpret_cast<unsigned int*>(&h3);
      lv.x = *reinterpret_cast<unsigned int*>(&l0); lv.y = *reinterpret_cast<unsigned int*>(&l1);
      lv.z = *reinterpret_cast<unsigned int*>(&l2); lv.w = *reinterpret_cast<unsigned int*>(&l3);
      *reinterpret_cast<uint4*>(dst) = hv;
      *reinterpret_cast<uint4*>(dst + 4224) = lv;
    }
  }
}

}  // namespace gcb
