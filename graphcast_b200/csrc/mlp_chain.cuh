// Fused layer CHAINS on Hopper tensor cores (sm_90a, wgmma): up to GCB_MAX_CHAIN fused layers
// (see mlp_tc.cuh for one layer) over the same rows in ONE persistent kernel.
//
//   layer l:  y_l[r] = residual_l[r] + LN|swish( concat_s A_{l,s}(r) @ W_l + b_l + gathered addends )
//   where a segment A_{l,s} is an external operand image, an external fp32 table (gathered /
//   fan-in summed by the producer warps), or the RESULT OF AN EARLIER LAYER of the chain.
//
// A cluster pair owns a 128-row tile (N-split: CTA r computes output columns [256r, 256r+256)
// of every layer, the A block of each K-step is fetched once and multicast to both CTAs, as in
// mlp_tc.cuh) and takes it through the layers.  A layer whose result later layers consume
// ("keep") writes it, as an operand image, into a per-cluster SCRATCH ring in global memory:
// (lag * max_distance + 1) slots of 264 KB per kept layer and cluster, 40 MB for a whole
// two-layer MLP launch.  The ring is rewritten in place tile after tile by the same cluster and
// read back within microseconds, and its lines are written with the L2 evict_last policy so
// that they stay in the L2 rather than go to HBM; the consumer streams it with the same TMA bulk copies as any other operand image.  This
// keeps the [rows, 512] hidden activation of every MLP (84 GB of HBM traffic per 0.25 degree
// step when the two linears were separate launches) on chip.
//
// Schedule.  Work is a sequence of UNITS (tile, layer); per cluster, step s runs the units
// (tile_{s - l*lag}, layer l) for l = 0..L-1 (or L-1..0: gcb_chain_desc.order), i.e. a tile advances one layer per `lag` steps, so
// that between a layer's MMAs and the dependent layer's MMAs the tensor pipe has `lag` other
// units to execute while the epilogue converts the accumulator and hands it over.  Each of the
// two consumer warpgroups holds the 64 x 256 fp32 accumulator of its half of the tile in
// registers and runs the MMAs and the epilogue of every unit in turn (mlp_tc.cuh).
//
// Hand-over protocol of a kept layer's scratch slot (both CTAs write half of the columns and
// both read all of them):
//   h_full[q][slot]  count 16: the 8 consumer warps of BOTH CTAs arrive (release.cluster) after
//                    their st.global + fence.proxy.async; the TMA warp of each CTA waits
//                    (acquire.cluster) before the first bulk copy out of the slot.
//   h_free[q][slot]  count 16 x consumers: every consumer warp of a consuming unit arrives (CTA
//                    scope) in both CTAs once its last MMA has retired, i.e. when all bulk copies out of
//                    the slot have landed and been consumed in that CTA; the consumers wait for
//                    it before overwriting the slot.
#pragma once
#include <type_traits>

#include "mlp_tc.cuh"

namespace gcb {

constexpr int kChainSlotsMax = 5;
constexpr int kScratchTileBytes = (kMaxN / kKStep) * GCB_A_IMAGE_BLOCK;   // 32 x 8448 = 270336
constexpr int kChainTailBytes = 3072;

// kBig: room for 8 instead of 4 [512]-float parameter vectors (biases, LayerNorm scale / offset):
// chains of two MLPs; costs 8 KB of shared memory (one operand stage in some variants).
template <bool kSplit, bool kPre, bool kBig>
struct ChainConfig {
  static constexpr int kParamVecs = kBig ? 8 : 4;
  static constexpr int kAStageBytes = kSplit ? 2 * kAPartBytes : kAPartBytes;
  static constexpr int kBStageBytes = kSplit ? 2 * kBPartBytes : kBPartBytes;
  static constexpr int kStageBytes = kAStageBytes + kBStageBytes;
  static constexpr int kParamBytes = kParamVecs * kMaxN * 4;
  static constexpr int kFixedBytes = kParamBytes + kLnxBytes + kChainTailBytes;
  static constexpr int kFit = (kSmemLimit - kFixedBytes) / kStageBytes;
#ifdef GCB_FORCE_STAGES          // experiment: sensitivity of a launch to the ring depth
  static constexpr int kStages = GCB_FORCE_STAGES < kFit ? GCB_FORCE_STAGES : kFit;
#else
  static constexpr int kStages = kFit < 12 ? kFit : 12;
#endif
  static constexpr int kSmemBytes = kStages * kStageBytes + kFixedBytes;
  static_assert(kStages >= 4, "operand ring too shallow");
};

struct ChainSeg {
  const float* table;
  const int32_t* idx;
  const uint8_t* img;
  int ld, k_valid, fan, ksteps;
  int src_q;          // >= 0: scratch ring q (result of an earlier layer); else external
  int pad_;
};

// kKindLN*: LayerNorm without residual / with an fp32 residual / with an operand-image residual
enum { kKindPlain = 0, kKindSwish = 1, kKindLN = 2, kKindLNRes = 3, kKindLNImg = 4 };

struct ChainLayer {
  const uint8_t* w;
  const float* residual;
  float* out;
  float* out_y;
  uint8_t* out_img;
  const uint8_t* res_img;
  int ld_res, ld_out, ld_outy;
  int nseg, ksteps, n_pre, kind;
  int bias_off, scale_off, offset_off;   // float offsets into the parameter area, -1 = none
  int keep_q;                            // scratch ring this layer writes, -1 = none
  int has_table;                         // some segment is an fp32 table (producer warps)
  int res_q;                             // residual = the kept result in scratch ring res_q, -1 = none
};

// ---- epilogue ----------------------------------------------------------------------------
// A consumer thread owns rows lr0 + 8h (h = 0, 1) of the tile and, in each 32-column chunk of its
// 256 unit columns, the column pairs 8jj + 2q (jj = 0..3): 16 results per chunk, kept in
// acc[16 * chunk .. + 16) at acc[4jj + 2h], acc[4jj + 2h + 1].  Every pointer below addresses
// column col_base + 2q of the first chunk of the unit; a chunk's accesses are the pointer plus a
// compile-time offset, and the column loop advances the pointers once per iteration.
struct ChainEpi {
  const float* pre[2][2];     // [table][h]: gathered pre-activation addend rows
  const float* res[2];        // [h]: fp32 residual rows
  float* out[2];              // [h]: result + residual, fp32
  float* outy[2];             // [h]: result without residual, fp32
  uint8_t* img0;              // operand images at the piece of (column col_base + 2q, row lr0)
  uint8_t* img1;              // (scratch slot of a kept layer)
  const uint8_t* res_img;
  uint32_t s_bias, s_scale, s_offset;   // shared-memory parameter vectors
  bool row_ok[2];             // [h]: row < rows (rows past the end exist in the images only)
  bool pre_b;                 // second addend table present
  bool has_bias, st_out, st_outy, st_img0, st_img1;
  float mean[2], rstd[2];
};

// Chunks per column-loop iteration.  The loop cannot be unrolled (8 chunks of straight-line code
// per unit overflow the instruction cache, DESIGN.md §3.1b), and a rolled loop can only index the
// accumulator with constants by shifting it down after every iteration: two chunks per
// iteration shift 96 registers 4 times per unit instead of 112 registers 8 times.
constexpr int kEpiChunks = 2;
constexpr int kEpiIters = kUnitN / 32 / kEpiChunks;
static_assert(kEpiChunks % 2 == 0 && kEpiIters * kEpiChunks * 32 == kUnitN,
              "the residual double buffer alternates halves chunk by chunk");

// p + bytes as integer arithmetic: also defined for p == nullptr (an absent output or input,
// whose accesses are predicated off).
template <typename T>
__device__ __forceinline__ T* byte_offset(T* p, long long bytes) {
  return reinterpret_cast<T*>(reinterpret_cast<uintptr_t>(p) + bytes);
}

// Byte offset, in an operand image, of (chunk c, column pair jj, row h) from the thread's piece
// in chunk 0 (image_offset with gc = col_base + 32c + 8jj + 2q, r = lr0 + 8h).
__device__ __forceinline__ constexpr int epi_img_off(int c, int jj, int h) {
  return (2 * c + (jj >> 1)) * GCB_A_IMAGE_BLOCK + (jj & 1) * kALbo + h * 8 * 16;
}

// Gathered addends of chunk c: buf[2jj + h] = table a, buf[8 + 2jj + h] = table b.  Table a
// reads as 0 and table b as -0 where they are missing (rows past the end; no second table): the
// sum a + b is then exactly a, or +0, as when the missing addends were skipped.
__device__ __forceinline__ void epi_load_pre(const ChainEpi& e, uint2 (&buf)[16], int c, bool ok) {
#pragma unroll
  for (int jj = 0; jj < 4; ++jj)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int o = 32 * c + 8 * jj;
      buf[2 * jj + h] = ptx::ld_global_nc_v2_pred(e.pre[0][h] + o, ok && e.row_ok[h], 0u);
      buf[8 + 2 * jj + h] = ptx::ld_global_nc_v2_pred(e.pre[1][h] + o, ok && e.row_ok[h] && e.pre_b, 0x80000000u);
    }
}
// fp32 residual of chunk c into buf[half + 2jj + h] (rows past the end: 0).
__device__ __forceinline__ void epi_load_res(const ChainEpi& e, uint2 (&buf)[16], int half, int c, bool ok) {
#pragma unroll
  for (int jj = 0; jj < 4; ++jj)
#pragma unroll
    for (int h = 0; h < 2; ++h)
      buf[half + 2 * jj + h] = ptx::ld_global_v2_pred(e.res[h] + 32 * c + 8 * jj, ok && e.row_ok[h]);
}
// Operand-image residual of chunk c: buf[half + 2jj + h] = (hi, lo) words.
__device__ __forceinline__ void epi_load_res_img(const ChainEpi& e, uint2 (&buf)[16], int half, int c, bool ok) {
#pragma unroll
  for (int jj = 0; jj < 4; ++jj)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint8_t* p = e.res_img + epi_img_off(c, jj, h);
      buf[half + 2 * jj + h] = make_uint2(ptx::ld_global_b32_pred(p, ok), ptx::ld_global_b32_pred(p + kAPartBytes, ok));
    }
}

// The column loop of one unit for one layer kind (kAdd: Plain / Swish with gathered addends).
// buf holds chunk 0's inputs on entry (loaded before the MMAs).  Each chunk adds the addends, then
// loads the next chunk's inputs, then computes and stores its 16 results; nothing in the loop
// branches, so the 16 independent element chains of a chunk interleave.  The arithmetic per
// element is that of mlp_layer_tc_kernel, in the same order, so the two kernels agree bit for
// bit (including the + 0 of an absent residual, which turns -0 into +0).
template <int kKind, bool kAdd>
__device__ __forceinline__ void chain_epilogue(float (&acc)[128], uint2 (&buf)[16], ChainEpi e,
                                               uint64_t keep_policy) {
  constexpr bool kLN = kKind >= kKindLN;
  constexpr bool kFp32Out = kKind != kKindSwish;     // swish layers deliver operand images only
  constexpr bool kOut = kFp32Out && kKind != kKindLNImg;
#pragma unroll 1
  for (int it = 0; it < kEpiIters; ++it) {
    const bool more = it + 1 < kEpiIters;
#pragma unroll
    for (int cc = 0; cc < kEpiChunks; ++cc) {
      float* v = &acc[16 * cc];
      const bool next = cc + 1 < kEpiChunks || more;
      const int cur = 8 * (cc & 1);                  // residual: this chunk in buf[cur..], next in the other half
      if constexpr (kAdd) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float gx = __uint_as_float(buf[i].x) + __uint_as_float(buf[8 + i].x);
          const float gy = __uint_as_float(buf[i].y) + __uint_as_float(buf[8 + i].y);
          v[4 * (i >> 1) + 2 * (i & 1)] += gx;
          v[4 * (i >> 1) + 2 * (i & 1) + 1] += gy;
        }
        epi_load_pre(e, buf, cc + 1, next);
      } else if constexpr (kKind == kKindLNRes) {
        epi_load_res(e, buf, 8 - cur, cc + 1, next);
      } else if constexpr (kKind == kKindLNImg) {
        epi_load_res_img(e, buf, 8 - cur, cc + 1, next);
      }
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int co = 4 * (32 * cc + 8 * jj);       // byte offset of the column pair in a row
        const float2 b = ptx::ld_shared_v2_pred(e.s_bias + co, e.has_bias);
        float2 sc = make_float2(1.f, 1.f), of = make_float2(0.f, 0.f);
        if constexpr (kLN) {
          sc = ptx::ld_shared_v2_pred(e.s_scale + co, true);
          of = ptx::ld_shared_v2_pred(e.s_offset + co, true);
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float* a = &v[4 * jj + 2 * h];
          const uint2 rin = buf[cur + 2 * jj + h];
          float2 y = make_float2(a[0] + b.x, a[1] + b.y);
          if constexpr (kKind == kKindSwish) { y.x = swish_f(y.x); y.y = swish_f(y.y); }
          if constexpr (kLN) {
            y.x = (y.x - e.mean[h]) * e.rstd[h] * sc.x + of.x;
            y.y = (y.y - e.mean[h]) * e.rstd[h] * sc.y + of.y;
          }
          float2 rs = make_float2(0.f, 0.f);
          if constexpr (kKind == kKindLNRes) rs = make_float2(__uint_as_float(rin.x), __uint_as_float(rin.y));
          float2 x = make_float2(y.x + rs.x, y.y + rs.y);
          if constexpr (kFp32Out) ptx::st_global_v2_pred(e.outy[h] + co / 4, y, e.st_outy && e.row_ok[h]);
          if constexpr (kOut) ptx::st_global_v2_pred(e.out[h] + co / 4, x, e.st_out && e.row_ok[h]);
          if constexpr (kKind == kKindLNImg) {
            // (hi, lo) bf16 words; a packed word holds the even column in its low half
            x.x += __uint_as_float(rin.x << 16) + __uint_as_float(rin.y << 16);
            x.y += __uint_as_float(rin.x & 0xffff0000u) + __uint_as_float(rin.y & 0xffff0000u);
          }
          uint32_t hi, lo;
          ptx::split_bf16x2(x.x, x.y, hi, lo);
          const int io = epi_img_off(cc, jj, h);
          ptx::st_global_b32_pred(e.img0 + io, hi, e.st_img0);
          ptx::st_global_b32_pred(e.img0 + io + kAPartBytes, lo, e.st_img0);
          ptx::st_global_b32_hint_pred(e.img1 + io, hi, keep_policy, e.st_img1);
          ptx::st_global_b32_hint_pred(e.img1 + io + kAPartBytes, lo, keep_policy, e.st_img1);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 128 - 16 * kEpiChunks; ++i) acc[i] = acc[i + 16 * kEpiChunks];
    constexpr int kCols = 32 * kEpiChunks;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      e.pre[0][h] += kCols; e.pre[1][h] += kCols; e.res[h] += kCols;
      e.out[h] += kCols; e.outy[h] += kCols;
    }
    e.img0 += 2 * kEpiChunks * GCB_A_IMAGE_BLOCK;
    e.img1 += 2 * kEpiChunks * GCB_A_IMAGE_BLOCK;
    e.res_img += 2 * kEpiChunks * GCB_A_IMAGE_BLOCK;
    e.s_bias += 4 * kCols; e.s_scale += 4 * kCols; e.s_offset += 4 * kCols;
  }
}

template <bool kSplit, bool kPre, bool kBig>
__global__ void __launch_bounds__(kThreads, 1)
mlp_chain_tc_kernel(const __grid_constant__ gcb_chain_desc d, const int nq, const int nslots) {
  using Cfg = ChainConfig<kSplit, kPre, kBig>;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* stage_base = smem;
  float* s_param = reinterpret_cast<float*>(smem + Cfg::kStages * Cfg::kStageBytes);
  float2* s_lnx = reinterpret_cast<float2*>(s_param + Cfg::kParamBytes / 4);   // [2][128]
  uint8_t* tail = reinterpret_cast<uint8_t*>(s_lnx) + kLnxBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(tail);          // [12]
  uint64_t* empty_bar = full_bar + 12;                             // [12]
  uint64_t* lnx_bar = empty_bar + 12;                              // [2 warpgroups][2]
  uint64_t* h_full_bar = lnx_bar + 4;                              // [GCB_MAX_CHAIN][kChainSlotsMax]
  uint64_t* h_free_bar = h_full_bar + GCB_MAX_CHAIN * kChainSlotsMax;
  ChainLayer* s_layer = reinterpret_cast<ChainLayer*>(h_free_bar + GCB_MAX_CHAIN * kChainSlotsMax);  // [4]
  ChainSeg* s_seg = reinterpret_cast<ChainSeg*>(s_layer + GCB_MAX_CHAIN);            // [4][3]
  PreAddInfo* s_pre = reinterpret_cast<PreAddInfo*>(s_seg + GCB_MAX_CHAIN * 3);      // [4][2]
  static_assert((2 * 12 + 4 + 2 * GCB_MAX_CHAIN * kChainSlotsMax) * 8 +
                    GCB_MAX_CHAIN * (sizeof(ChainLayer) + 3 * sizeof(ChainSeg) + 2 * sizeof(PreAddInfo))
                    <= kChainTailBytes, "tail region too small");

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int L = d.nlayers;
  const int lag = d.lag > 0 ? d.lag : 1;
  // Unit order inside a step: ascending (layer 0 first) or descending.  Descending, a kept
  // result is consumed (by the next layer, one step later) BEFORE the producing layer's next
  // unit writes again, so lag*distance slots per scratch ring suffice instead of lag*distance+1
  // - what keeps the rings of a 4-layer chain inside the L2.  It shortens the distance between
  // dependent units from L+1 to L-1 units, so it is used for chains of 3 and more layers.
  const bool desc = d.order != 0;
  const long long rows_total = d.rows;
  const int num_tiles = (d.rows + kTileM - 1) / kTileM;
  const uint32_t crank = ptx::cluster_ctarank();
  const uint32_t cid = ptx::cluster_id_x();
  const uint32_t ncl = ptx::num_clusters_x();
  const uint32_t peer = crank ^ 1u;
  constexpr uint16_t cmask = 3;
  // Tiles of this cluster: cid, cid + ncl, ...
  const int T = (num_tiles > static_cast<int>(cid))
                    ? (num_tiles - static_cast<int>(cid) + static_cast<int>(ncl) - 1) / static_cast<int>(ncl)
                    : 0;
  const int nsteps = T > 0 ? T + (L - 1) * lag : 0;
  uint8_t* const scratch = static_cast<uint8_t*>(d.scratch) +
                           static_cast<size_t>(cid) * nq * nslots * kScratchTileBytes;
  auto scratch_slot = [&](int q, int ti) -> uint8_t* {
    return scratch + (static_cast<size_t>(q) * nslots + (ti % nslots)) * kScratchTileBytes;
  };
  bool any_table = false;
  for (int l = 0; l < L; ++l)
    for (int s = 0; s < d.layer[l].nseg; ++s)
      any_table = any_table || (d.layer[l].seg_from[s] < 0 && d.layer[l].seg[s].img == nullptr);

  // ---- one-time setup ---------------------------------------------------------
  {
    // Parameter vectors in layer order: [bias] [ln scale, ln offset] per layer (every thread
    // derives the same offsets, so no synchronisation is needed before the copy).
    int off = 0;
    for (int l = 0; l < L; ++l) {
      const gcb_chain_layer& gl = d.layer[l];
      if (gl.bias != nullptr) {
        for (int i = threadIdx.x; i < kMaxN; i += kThreads) s_param[off + i] = gl.bias[i];
        off += kMaxN;
      }
      if (gl.ln_scale != nullptr) {
        for (int i = threadIdx.x; i < kMaxN; i += kThreads) {
          s_param[off + i] = gl.ln_scale[i];
          s_param[off + kMaxN + i] = gl.ln_offset[i];
        }
        off += 2 * kMaxN;
      }
    }
  }
  if (threadIdx.x == 0) {
    int off = 0, q = 0;
    int q_of_layer[GCB_MAX_CHAIN];
    int consumers[GCB_MAX_CHAIN];
    for (int l = 0; l < L; ++l) { q_of_layer[l] = -1; consumers[l] = 0; }
    for (int l = 0; l < L; ++l) {
      const gcb_chain_layer& gl = d.layer[l];
      ChainLayer& cl = s_layer[l];
      cl.w = static_cast<const uint8_t*>(gl.w_packed);
      cl.residual = gl.residual; cl.out = gl.out; cl.out_y = gl.out_y;
      cl.out_img = static_cast<uint8_t*>(gl.out_img);
      cl.res_img = static_cast<const uint8_t*>(gl.residual_img);
      cl.ld_res = gl.ld_res; cl.ld_out = gl.ld_out; cl.ld_outy = gl.ld_out_y;
      cl.nseg = gl.nseg; cl.n_pre = gl.n_pre_add;
      cl.res_q = gl.residual_keep > 0 ? q_of_layer[gl.residual_keep - 1] : -1;
      cl.kind = gl.ln_scale != nullptr
                    ? (gl.residual != nullptr
                           ? kKindLNRes
                           : ((gl.residual_img != nullptr || gl.residual_keep > 0) ? kKindLNImg : kKindLN))
                    : (gl.act == GCB_ACT_SWISH ? kKindSwish : kKindPlain);
      cl.bias_off = -1; cl.scale_off = -1; cl.offset_off = -1;
      if (gl.bias != nullptr) { cl.bias_off = off; off += kMaxN; }
      if (gl.ln_scale != nullptr) { cl.scale_off = off; cl.offset_off = off + kMaxN; off += 2 * kMaxN; }
      cl.keep_q = -1;
      if (gl.keep) { cl.keep_q = q; q_of_layer[l] = q; ++q; }
      int ks = 0, has_table = 0;
      for (int s = 0; s < gl.nseg; ++s) {
        ChainSeg& cs = s_seg[l * 3 + s];
        const int from = gl.seg_from[s];
        cs.table = gl.seg[s].table; cs.idx = gl.seg[s].idx;
        cs.img = static_cast<const uint8_t*>(gl.seg[s].img);
        cs.ld = gl.seg[s].ld; cs.k_valid = gl.seg[s].k_valid; cs.fan = gl.seg[s].fan;
        cs.ksteps = (from >= 0 ? kMaxN : gl.seg[s].k) / kKStep;
        cs.src_q = from >= 0 ? q_of_layer[from] : -1;
        if (from >= 0) { cs.img = nullptr; ++consumers[from]; }
        else if (cs.img == nullptr) has_table = 1;
        ks += cs.ksteps;
      }
      cl.ksteps = ks; cl.has_table = has_table;
      for (int s = 0; s < gl.n_pre_add; ++s) {
        s_pre[l * 2 + s].table = gl.pre_add[s].table;
        s_pre[l * 2 + s].idx = gl.pre_add[s].idx;
        s_pre[l * 2 + s].ld = gl.pre_add[s].ld;
      }
    }
    for (int s = 0; s < Cfg::kStages; ++s) {
      ptx::mbar_init(&full_bar[s], any_table ? 1 + kProducerWarps : 1);   // TMA lane (+ the producer warps)
      ptx::mbar_init(&empty_bar[s], 2 * kConsumerWarps);                   // every consumer warp of both CTAs
    }
    for (int b = 0; b < 2; ++b) {
      ptx::mbar_init(&lnx_bar[b], 1);
      ptx::mbar_init(&lnx_bar[2 + b], 1);
    }
    for (int l = 0; l < L; ++l) {
      if (q_of_layer[l] < 0) continue;
      for (int sl = 0; sl < nslots; ++sl) {
        ptx::mbar_init(&h_full_bar[q_of_layer[l] * kChainSlotsMax + sl], 2 * kConsumerWarps);
        ptx::mbar_init(&h_free_bar[q_of_layer[l] * kChainSlotsMax + sl],
                       2 * kConsumerWarps * (consumers[l] > 0 ? consumers[l] : 1));
      }
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();
  ptx::cluster_sync_all();

  // ---- roles ------------------------------------------------------------------
  if (warp < 4) {
    ptx::setmaxnreg_dec<kChainProducerRegs>();       // whole warpgroup 0, before its warps split up
    if (warp == 0) {
      // ===== TMA warp (converged; every lane polls, one elected lane issues) =====
      const uint32_t b_bytes = Cfg::kBStageBytes;
      const size_t b_block = 2 * kBPartBytes;
      const size_t b_stride = 2 * b_block;                          // n = 512: two blocks per K-step
      const uint32_t a_bytes = Cfg::kAStageBytes;
      const uint32_t a_half = a_bytes / 2;
      uint32_t stage = 0, phase = 0, tu = 0;
      const uint64_t keep_policy = ptx::l2_policy_evict_last();
      for (int st = 0; st < nsteps; ++st) {
        for (int li = 0; li < L; ++li) {
          const int l = desc ? L - 1 - li : li;
          const int ti = st - l * lag;
          if (ti < 0 || ti >= T) continue;
          const uint32_t tile = cid + static_cast<uint32_t>(ti) * ncl;
          const int nseg = s_layer[l].nseg;
          const uint8_t* b_ptr = s_layer[l].w + static_cast<size_t>(crank) * b_block;
          const bool tr = tracing(tu);
          long long blocked = 0, hwait = 0;
          for (int s = 0; s < nseg; ++s) {
            const ChainSeg sg = s_seg[l * 3 + s];
            const uint8_t* a_ptr = nullptr;
            bool a_copy = false;
            const bool a_scratch = sg.src_q >= 0;
            if (sg.src_q >= 0) {
              const long long w0 = tr ? clock64() : 0;
              // Poll at CTA scope (a cluster-scope acquire per retry is far more expensive), then
              // take the cluster-scope acquire once on the completed phase.
              ptx::mbar_wait(&h_full_bar[sg.src_q * kChainSlotsMax + (ti % nslots)],
                             static_cast<uint32_t>(ti / nslots) & 1u);
              ptx::mbar_wait_cluster(&h_full_bar[sg.src_q * kChainSlotsMax + (ti % nslots)],
                                     static_cast<uint32_t>(ti / nslots) & 1u);
              if (tr) hwait += clock64() - w0;
              a_ptr = scratch_slot(sg.src_q, ti) + crank * a_half;
              a_copy = true;
            } else if (sg.img != nullptr) {
              a_ptr = sg.img + static_cast<size_t>(tile) * sg.ksteps * GCB_A_IMAGE_BLOCK + crank * a_half;
              a_copy = true;
            }
            const uint32_t tx = b_bytes + (a_copy ? a_bytes : 0u);
            for (int k = 0; k < sg.ksteps; ++k) {
              const long long w0 = tr ? clock64() : 0;
              ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
              if (tr) blocked += clock64() - w0;
              uint8_t* a_dst = stage_base + stage * Cfg::kStageBytes;
              if (ptx::elect_one()) {
                ptx::mbar_arrive_expect_tx(&full_bar[stage], tx);
                if (a_scratch)
                  ptx::bulk_g2s_multicast_hint(a_dst + crank * a_half, a_ptr, a_half, &full_bar[stage], cmask, keep_policy);
                else if (a_copy)
                  ptx::bulk_g2s_multicast(a_dst + crank * a_half, a_ptr, a_half, &full_bar[stage], cmask);
                ptx::bulk_g2s(a_dst + Cfg::kAStageBytes, b_ptr, b_bytes, &full_bar[stage]);
              }
              __syncwarp();
              a_ptr += GCB_A_IMAGE_BLOCK;
              b_ptr += b_stride;
              if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
            }
          }
          if (lane == 0) { trace_val(tu, 7, blocked); trace_val(tu, 8, hwait); trace_val(tu, 11, l); }
          ++tu;
        }
      }
    } else if (warp >= 4 - kProducerWarps) {
      // ===== producers (warps 2-3): fp32-table segments, unit by unit =====
      // A table segment is gathered through its index (optional fan-in sum), split to bf16 hi / lo
      // and stored in the K-major core-matrix layout.  The producers arrive on EVERY K-step's full
      // barrier when some layer has a table segment (for image / scratch K-steps without writing
      // anything), so the barrier count is uniform.
      const int t64 = threadIdx.x - 32 * (4 - kProducerWarps);
      const int sub = t64 & 3;                        // which float4 of the 16-wide K-step
      const int rg = t64 >> 2;                        // 0..15; rows rg + 16*i
      const uint32_t sts_off = (sub >> 1) * kALbo + (sub & 1) * 8;
      uint32_t stage = 0, phase = 0;
      for (int st = 0; st < nsteps; ++st) {
        for (int li = 0; li < L; ++li) {
          const int l = desc ? L - 1 - li : li;
          const int ti = st - l * lag;
          if (ti < 0 || ti >= T) continue;
          const uint32_t tile = cid + static_cast<uint32_t>(ti) * ncl;
          const int nseg = s_layer[l].nseg;
          for (int s = 0; any_table && s < nseg; ++s) {
            const ChainSeg sg = s_seg[l * 3 + s];
            const bool is_tab = sg.src_q < 0 && sg.img == nullptr;
            int src[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              src[i] = -1;
              if (is_tab) {
                const long long grow = static_cast<long long>(tile) * kTileM + rg + 16 * i;
                if (grow < rows_total) src[i] = sg.idx ? __ldg(sg.idx + grow) : static_cast<int>(grow);
              }
            }
            for (int k = 0; k < sg.ksteps; ++k) {
              float4 cur[8];
              if (is_tab) {
                const int koff = k * kKStep + sub * 4;
                const bool kvalid = koff < sg.k_valid;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
                  if (kvalid && src[i] >= 0) {
                    const float* p = sg.table + static_cast<long long>(src[i]) * sg.fan * sg.ld + koff;
                    a = __ldg(reinterpret_cast<const float4*>(p));
                    for (int j = 1; j < sg.fan; ++j) {
                      const float4 t = __ldg(reinterpret_cast<const float4*>(p + static_cast<long long>(j) * sg.ld));
                      a.x += t.x; a.y += t.y; a.z += t.z; a.w += t.w;
                    }
                  }
                  cur[i] = a;
                }
              }
              ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
              if (is_tab) {
                uint8_t* a_hi = stage_base + stage * Cfg::kStageBytes;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                  uint2 hi, lo;
                  ptx::split_bf16x4(cur[i], hi, lo);
                  const uint32_t off = sts_off + (rg + 16 * i) * 16;
                  *reinterpret_cast<uint2*>(a_hi + off) = hi;
                  if (kSplit) *reinterpret_cast<uint2*>(a_hi + kAPartBytes + off) = lo;
                }
                ptx::fence_proxy_async_smem();
              }
              __syncwarp();
              if (lane == 0) ptx::mbar_arrive(&full_bar[stage]);
              if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
            }
          }
        }
      }
    }
  } else {
    ptx::setmaxnreg_inc<consumer_regs(kChainProducerRegs)>();
    // ===== consumers: MMA + epilogue =====
    const int eg = (warp - 4) >> 2;                // warpgroup: tile rows [64 eg, 64 eg + 64)
    const int q = lane & 3;
    const int lr0 = eg * 64 + (warp & 3) * 16 + (lane >> 2);   // tile rows lr0, lr0 + 8
    const bool lead = lane == 0 && (warp & 3) == 0;
    const int col_base = static_cast<int>(crank) * kUnitN;   // my 256 columns of every layer
    uint32_t stage = 0, phase = 0, ln_count = 0, u = 0;
    const uint64_t keep_policy = ptx::l2_policy_evict_last();
    float acc[128];

    for (int st = 0; st < nsteps; ++st) {
      for (int li = 0; li < L; ++li) {
        const int l = desc ? L - 1 - li : li;
        const int ti = st - l * lag;
        if (ti < 0 || ti >= T) continue;
        const uint32_t tile = cid + static_cast<uint32_t>(ti) * ncl;
        const ChainLayer& cl = s_layer[l];
        const int kind = cl.kind;
        const float* const s_bias = cl.bias_off >= 0 ? s_param + cl.bias_off : nullptr;
        if (eg == 0 && ti + 1 < T && (cl.residual != nullptr || cl.res_img != nullptr)) {
          // Pull the residual of this layer's NEXT tile into L2 now (a whole step ahead).
          const uint32_t ntile = tile + ncl;
          const int pr = (warp & 3) * 32 + lane;      // 128 threads: one row each
          if (cl.residual != nullptr) {
            const long long nrow = static_cast<long long>(ntile) * kTileM + pr;
            if (nrow < rows_total) ptx::bulk_prefetch_l2(cl.residual + nrow * cl.ld_res + col_base, kUnitN * 4);
          } else if (pr < kUnitN / kKStep) {
            ptx::bulk_prefetch_l2(cl.res_img + (static_cast<size_t>(ntile) * (kMaxN / kKStep) +
                                                (col_base >> 4) + pr) * GCB_A_IMAGE_BLOCK,
                                  GCB_A_IMAGE_BLOCK);
          }
        }
        const bool is_ln = kind >= kKindLN;
        const bool want_pre = kPre && !is_ln && cl.n_pre > 0;
        const int keep_q = cl.keep_q;
        // Epilogue state of this unit (ChainEpi).  Pointers of absent outputs are formed from
        // nullptr; their stores are predicated off.
        ChainEpi e;
        {
          const long long grow0 = static_cast<long long>(tile) * kTileM + lr0;
          const int c0 = col_base + 2 * q;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const long long grow = grow0 + 8 * h;
            e.row_ok[h] = grow < rows_total;
            e.out[h] = byte_offset(cl.out, 4 * (grow * cl.ld_out + c0));
            e.outy[h] = byte_offset(cl.out_y, 4 * (grow * cl.ld_outy + c0));
            e.res[h] = byte_offset(cl.residual, 4 * (grow * cl.ld_res + c0));
            if (want_pre) {
              const PreAddInfo pa = s_pre[l * 2];
              const PreAddInfo pb = s_pre[l * 2 + 1];
              int ra = 0, rb = 0;
              if (e.row_ok[h]) {
                ra = pa.idx ? __ldg(pa.idx + grow) : static_cast<int>(grow);
                if (cl.n_pre > 1) rb = pb.idx ? __ldg(pb.idx + grow) : static_cast<int>(grow);
              }
              e.pre[0][h] = byte_offset(pa.table, 4 * (static_cast<long long>(ra) * pa.ld + c0));
              e.pre[1][h] = byte_offset(pb.table, 4 * (static_cast<long long>(rb) * pb.ld + c0));
            }
          }
          const long long piece = static_cast<long long>(image_offset(c0, lr0));
          const long long tile_img = static_cast<long long>(tile) * (kMaxN / kKStep) * GCB_A_IMAGE_BLOCK;
          e.img0 = byte_offset(cl.out_img, tile_img + piece);
          // keep: this tile's slot of the scratch ring (written once h_free has been passed below)
          e.img1 = byte_offset(keep_q >= 0 ? scratch_slot(keep_q, ti) : nullptr, piece);
          // Residual = the kept result of an earlier layer: the slot this CTA's consumers wrote for
          // this tile (same threads, same rows and columns: program order makes it visible, and the
          // slot cannot be rewritten before these warps reach tile ti + nslots themselves).
          e.res_img = cl.res_q >= 0 ? scratch_slot(cl.res_q, ti) + piece : byte_offset(cl.res_img, tile_img + piece);
          e.pre_b = cl.n_pre > 1;
          e.has_bias = s_bias != nullptr;
          e.st_out = cl.out != nullptr;
          e.st_outy = cl.out_y != nullptr;
          e.st_img0 = cl.out_img != nullptr;
          // Through a vote: a predicate the compiler knows to be warp-uniform lets it predicate the
          // cache-hinted stores (it branches around them otherwise).
          e.st_img1 = __all_sync(0xffffffffu, keep_q >= 0);
          e.s_bias = ptx::smem_addr(s_param + (cl.bias_off >= 0 ? cl.bias_off : 0) + c0);
          e.s_scale = ptx::smem_addr(s_param + (cl.scale_off >= 0 ? cl.scale_off : 0) + c0);
          e.s_offset = ptx::smem_addr(s_param + (cl.offset_off >= 0 ? cl.offset_off : 0) + c0);
        }
        // Inputs of the epilogue that live in global memory - the gathered pre-activation addends
        // (two tables, gathered through their row indices) or the residual (fp32 rows or an operand
        // image) - are loaded into registers one 32-column chunk ahead of their use, chunk 0 before
        // the MMAs, so that their latency hides behind the MMAs and the previous chunk.  Loading
        // ahead is safe for the in-place updates (out_img == res_img, out == residual): every word
        // is read and then written by the same thread, and a chunk's loads touch other columns than
        // the stores they move ahead of.
        uint2 buf[16];
        if (want_pre) epi_load_pre(e, buf, 0, true);
        else if (kind == kKindLNRes) epi_load_res(e, buf, 0, 0, true);
        else if (kind == kKindLNImg) epi_load_res_img(e, buf, 0, 0, true);
        if (lead && eg == 0) trace(u, 0);
        if (keep_q >= 0) {
          // previous readers of this slot (tile ti - nslots) are done in both CTAs
          ptx::mbar_wait(&h_free_bar[keep_q * kChainSlotsMax + (ti % nslots)],
                         (static_cast<uint32_t>(ti / nslots) & 1u) ^ 1u);
        }
        if (lead && eg == 0) { trace(u, 2); trace_val(u, 9, cl.ksteps); }
        mma_unit<kSplit, Cfg::kStages, Cfg::kStageBytes, Cfg::kAStageBytes>(
            acc, stage_base, full_bar, empty_bar, stage, phase, cl.ksteps, eg * 64 * 16, cmask, u);
        if (lane == 0) {
          // Every scratch slot this unit read is reusable (in both CTAs) once these MMAs retired.
          // The slot's readers are bulk copies that have completed (their bytes were counted on
          // full barriers this warp passed); the next writers wait on h_free first.  So, as for
          // the stage release in mma_unit, a CTA-scope arrive suffices.
          for (int s = 0; s < cl.nseg; ++s) {
            const int sq = s_seg[l * 3 + s].src_q;
            if (sq >= 0) {
              const uint32_t a = ptx::smem_addr(&h_free_bar[sq * kChainSlotsMax + (ti % nslots)]);
              ptx::mbar_arrive_remote_cta(ptx::mapa(a, 0));
              ptx::mbar_arrive_remote_cta(ptx::mapa(a, 1));
            }
          }
        }
        if (lead && eg == 0) trace(u, 3);
        e.mean[0] = e.mean[1] = 0.f;
        e.rstd[0] = e.rstd[1] = 1.f;
        if (is_ln) {
          // Each CTA computes (mean, M2) of its 256 columns of a row, hands them to the partner
          // through distributed shared memory, and both combine them (Chan's parallel update).
          float shift[2], s1[2], s2[2];
          row_shifted_sums(acc, s_bias != nullptr ? s_bias + col_base : nullptr, kUnitN, shift, s1, s2);
          const uint32_t lb = ln_count & 1, par = (ln_count >> 1) & 1;
          uint64_t* bar = &lnx_bar[eg * 2 + lb];
          float mh[2], m2h[2];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            mh[h] = shift[h] + s1[h] * (1.0f / kUnitN);
            m2h[h] = fmaxf(s2[h] - s1[h] * s1[h] * (1.0f / kUnitN), 0.f);
            if (q == 0)
              ptx::st_async_f32x2(ptx::mapa(ptx::smem_addr(&s_lnx[lb * kTileM + lr0 + 8 * h]), peer),
                                  mh[h], m2h[h], ptx::mapa(ptx::smem_addr(bar), peer));
          }
          if (lead) ptx::mbar_arrive_expect_tx(bar, 64 * 8);
          ptx::mbar_wait(bar, par);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float2 other = s_lnx[lb * kTileM + lr0 + 8 * h];
            const float delta = other.x - mh[h];
            e.mean[h] = 0.5f * (mh[h] + other.x);
            const float var = (m2h[h] + other.y + delta * delta * (0.5f * kUnitN)) * (1.0f / (2 * kUnitN));
            e.rstd[h] = rsqrtf(var + 1e-5f);
          }
          ++ln_count;
          if (lead && eg == 0) trace(u, 4);
        }
        // One column loop per layer kind, chosen once per unit.
        if (kPre && want_pre) {
          if (kind == kKindSwish) chain_epilogue<kKindSwish, kPre>(acc, buf, e, keep_policy);
          else chain_epilogue<kKindPlain, kPre>(acc, buf, e, keep_policy);
        } else if (kind == kKindSwish) {
          chain_epilogue<kKindSwish, false>(acc, buf, e, keep_policy);
        } else if (kind == kKindPlain) {
          chain_epilogue<kKindPlain, false>(acc, buf, e, keep_policy);
        } else if (kind == kKindLN) {
          chain_epilogue<kKindLN, false>(acc, buf, e, keep_policy);
        } else if (kind == kKindLNRes) {
          chain_epilogue<kKindLNRes, false>(acc, buf, e, keep_policy);
        } else {
          chain_epilogue<kKindLNImg, false>(acc, buf, e, keep_policy);
        }
        if (lead && eg == 0) trace(u, 5);
        if (keep_q >= 0) {
          // Hand the slot to the TMA warps of both CTAs: my generic-proxy global stores must be
          // visible to their async-proxy bulk copies.
          ptx::fence_proxy_async_global();
          __syncwarp();
          if (lane == 0) {
            uint64_t* hb = &h_full_bar[keep_q * kChainSlotsMax + (ti % nslots)];
            ptx::mbar_arrive_release_cluster(hb);
            ptx::mbar_arrive_remote(ptx::mapa(ptx::smem_addr(hb), peer));
          }
        }
        if (lead && eg == 0) trace(u, 6);
        ++u;
      }
    }
  }

  // ---- teardown ---------------------------------------------------------------
  __syncthreads();
  ptx::cluster_sync_all();
}

}  // namespace gcb
