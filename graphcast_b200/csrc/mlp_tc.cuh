// Fused linear layer on Hopper tensor cores (sm_90a, wgmma).
//
//   out[r] = residual[r] + LN( act( concat_s A_s(r) @ W + bias + gathered addends ) )
//
// One persistent 384-thread CTA per SM.  Work is cut into UNITS of 128 rows x 256 output
// columns.  Two schedules:
//   N-split (n = 512, cluster of 2): both CTAs of the cluster work on the SAME 128-row
//     tile, CTA r owning output columns [256r, 256r+256).  The A block of every K-step is
//     fetched once and multicast to both CTAs, each CTA streams only its half of the
//     weights, and LayerNorm row statistics are combined across the pair through
//     distributed shared memory.  Consecutive units of a CTA are consecutive tiles.
//   unsplit (n = 256, or cluster of 1 / 4): every CTA walks its own tiles (n/256 units per
//     tile); the CTAs of a cluster share the weight stream by multicast.  LayerNorm over
//     512 columns needs the N-split schedule (the launcher enforces it).
// Warp roles:
//   warp 0        TMA lane: per K-step streams (a) 1/cluster of the pre-packed bf16 weight
//                 tile with cp.async.bulk, multicast to every CTA of the cluster, and (b)
//                 the A block of segments that are stored as operand images.
//   warps 4-11    two consumer warpgroups, rows [0, 64) and [64, 128) of the tile: wgmma
//                 (M=64, N=256, K=16), three products per K-step in BF16X3 mode (hi*hi,
//                 hi*lo, lo*hi), fp32 accumulation in registers (128 per thread), then the
//                 epilogue straight from the accumulator fragment: bias, gathered
//                 pre-activation addends, swish | LayerNorm (+ residual), fp32 and / or
//                 operand-image outputs.
//   warps 2-3     producers.  A segments given as fp32 tables (optionally gathered through
//                 an index, optionally a fan-in sum) are converted to bf16 hi/lo and stored
//                 in the K-major core-matrix layout; gathered pre-activation addends (node
//                 projections of the split edge MLP) are staged into shared memory in
//                 32-column chunks, unit by unit after that unit's A operand.
//
// Shared-memory operand layout (no swizzle, K-major): a [R x 16] bf16 operand of one
// K-step is two "K chunks" of 8 elements; chunk c, row r lives at byte c*LBO + r*16.
// Eight consecutive rows form one 128-byte core matrix, so SBO = 128; LBO = 256*16 for the
// weights and 128*16 + 64 for the activations (see kALbo and ptx.cuh make_smem_desc).
#pragma once
#include "../../include/graphcast_b200.h"
#include "ptx.cuh"

namespace gcb {

constexpr int kTileM = 128;
constexpr int kUnitN = 256;                       // output columns per unit / accumulator
constexpr int kKStep = 16;
constexpr int kThreads = 384;
// A operand: the two 8-element K chunks of a K-step are 2048 + 64 bytes apart.  The
// 64-byte skew puts chunk 1 on the other 16 banks so that the producers' 8-byte
// stores (rows 0-3 of both chunks per half-warp) are conflict-free.
constexpr int kALbo = kTileM * 16 + 64;           // 2112
constexpr int kAPartBytes = 2 * kALbo;            // 4224: one of {hi, lo}
constexpr int kBLbo = kUnitN * 16;                // 4096
constexpr int kBPartBytes = 2 * kBLbo;            // 8192: one of {hi, lo} of a 256-row weight block
constexpr int kEpiRowFloats = 36;                 // 32 + 4 pad: conflict-free 16 B accesses
// Pre-activation addend chunks (gathered node projections), double buffered:
// [2][128 rows][36 floats], filled by the producer groups, read by the epilogue.
constexpr int kGBufFloats = kTileM * kEpiRowFloats;
constexpr int kGBytes = 2 * kGBufFloats * 4;
constexpr int kMaxN = 512;
constexpr int kMaxKSteps = 128;                   // K <= 2048
constexpr int kConsumerWarps = 8;                 // warps 4-11: two warpgroups of 64 tile rows each
constexpr int kProducerWarps = 2;                 // warps 2-3
static_assert(2 * kAPartBytes == GCB_A_IMAGE_BLOCK, "A image block must match the stage layout");

// Shared-memory budget: everything the variant does not need goes to pipeline stages.
// LayerNorm variants never stage gathered addends (only the 2 KB statistics exchange
// aliases that region); the others carry no LayerNorm scale / offset.
constexpr int kSmemLimit = 227 * 1024;            // opt-in dynamic shared memory per CTA
constexpr int kTailBytes = 1024;                  // barriers, segment tables
constexpr int kLnxBytes = 2 * kTileM * 8;         // [2][128] (mean, M2) pairs

template <bool kSplit, bool kLN>
struct TcConfig {
  static constexpr int kAStageBytes = kSplit ? 2 * kAPartBytes : kAPartBytes;
  static constexpr int kBStageBytes = kSplit ? 2 * kBPartBytes : kBPartBytes;
  static constexpr int kStageBytes = kAStageBytes + kBStageBytes;
  static constexpr int kParamBytes = (kLN ? 3 : 1) * kMaxN * 4;   // bias (, ln scale, ln offset)
  static constexpr int kGRegionBytes = kLN ? kLnxBytes : kGBytes;
  static constexpr int kFixedBytes = kParamBytes + kGRegionBytes + kTailBytes;
  static constexpr int kFit = (kSmemLimit - kFixedBytes) / kStageBytes;
  static constexpr int kStages = kFit < 12 ? kFit : 12;           // tail holds 2*12+8 barriers
  static constexpr int kSmemBytes = kStages * kStageBytes + kFixedBytes;
  static_assert(kStages >= 4, "operand ring too shallow");
};

// Register split between warpgroup 0 (TMA, idle and producer warps) and the two consumer
// warpgroups.  __launch_bounds__(kThreads, 1) gives every warp kLaunchRegs (65536 / 384, rounded
// down to a multiple of 8); warpgroup 0 hands registers back so that the consumers, which hold a
// 128-register accumulator through the epilogue, can run it without spilling:
// 128 * producer registers + 256 * consumer registers <= 384 * kLaunchRegs.  The splits were
// picked from ptxas spill counts and H100 step times: the layer kernel's producers keep 24
// source rows and two K-steps of A in flight and need 120 (consumers 192); the chain kernel
// runs faster at 56 / 224 than at 88 / 208 (its producers only convert fp32-table segments).
constexpr int kLaunchRegs = 168;
constexpr int kLayerProducerRegs = 120;
constexpr int kChainProducerRegs = 56;
__host__ __device__ constexpr int consumer_regs(int producer_regs) { return (3 * kLaunchRegs - producer_regs) / 2 / 8 * 8; }
static_assert(kLayerProducerRegs % 8 == 0 && kLayerProducerRegs >= 24 && consumer_regs(kLayerProducerRegs) <= 256 &&
              kChainProducerRegs % 8 == 0 && kChainProducerRegs >= 24 && consumer_regs(kChainProducerRegs) <= 256,
              "setmaxnreg takes a multiple of 8 in [24, 256]");

__device__ __forceinline__ float swish_f(float x) {
  // x * sigmoid(x) = x / (1 + 2^(-x*log2 e)): one ex2.approx and one rcp.approx,
  // branch-free (~2 ulp), so 32 independent elements pipeline through the SFU.
  return __fdividef(x, 1.0f + __expf(-x));
}

// Optional timeline trace (debug): when non-null, CTA 0 records clock64() at a few
// points of each of its first kTraceTiles units; see gcb_debug_trace in api.cu.  Events of a
// unit (clock64 stamps of consumer warp 4 unless a count):
//   0 unit start  1 first full barrier passed  2 h_free passed (chain)  3 MMAs retired
//   4 LayerNorm statistics combined  5 epilogue stored  6 hand-over done (chain)
//   7 cycles the TMA warp waited on empty barriers  8 cycles it waited on h_full (chain)
//   9 K-steps  11 layer (chain)
constexpr int kTraceTiles = 64;
constexpr int kTraceEvents = 16;
__device__ long long* g_trace = nullptr;
// Debug-only experiment switches (gcb_debug_flags); 0 in production.
__device__ int g_dbg_flags = 0;

__device__ __forceinline__ void trace(uint32_t unit, int ev) {
  if (g_trace != nullptr && blockIdx.x == 0 && unit < kTraceTiles)
    g_trace[unit * kTraceEvents + ev] = clock64();
}
__device__ __forceinline__ bool tracing(uint32_t unit) {
  return g_trace != nullptr && blockIdx.x == 0 && unit < kTraceTiles;
}
__device__ __forceinline__ void trace_val(uint32_t unit, int ev, long long v) {
  if (tracing(unit)) g_trace[unit * kTraceEvents + ev] = v;
}

struct KStepInfo {
  uint8_t seg;
  uint8_t is_img;  // 1: this K-step's A block comes from the segment's operand image (TMA)
  uint16_t koff;   // element offset of this K-step inside its segment
};

// Per-segment fields copied to shared memory once: reading them from the kernel
// parameter (constant bank) inside the hot loops costs an exposed ~100-cycle LDC each.
struct SegInfo {
  const float* table;
  const int32_t* idx;
  const uint8_t* img;
  int ld, k_valid, fan, ksteps;
};
struct PreAddInfo {
  const float* table;
  const int32_t* idx;
  long long ld;
};

// ---- consumer warpgroup helpers (shared with mlp_chain.cuh) ------------------------
// Fragment coordinates: consumer thread t of warp w of warpgroup g holds tile rows
// frag_row(h) = 64g + 16w + t/4 + 8h and columns 8j + 2(t%4) + e of the unit (ptx.cuh).

// The MMAs of one unit for this warpgroup's 64 rows (A rows start a_row_off bytes into the
// stage).  After each K-step the previous one is retired and its stage released: one arrival
// per warp, on the local barrier (rel_mask == 0) or on the barrier of every CTA in rel_mask.
// `unit` only indexes the timeline trace (event 1: first full barrier passed).
template <bool kSplit, int kStages, int kStageBytes, int kAStageBytes>
__device__ __forceinline__ void mma_unit(float (&acc)[128], uint8_t* stage_base, uint64_t* full_bar,
                                         uint64_t* empty_bar, uint32_t& stage, uint32_t& phase,
                                         int ksteps, uint32_t a_row_off, uint32_t rel_mask, uint32_t unit) {
  const bool lead = (threadIdx.x & 31) == 0;
  // The stage's readers are this warpgroup's wgmma operand fetches (async proxy), retired by
  // the wgmma.wait_group before the call; its next writers are TMA bulk copies and producer
  // st.shared, both issued by a thread that has observed the empty barrier.  This warp made no
  // generic-proxy writes the writers must see, so the arrive needs no release beyond CTA scope.
  // A release.cluster arrive would put MEMBAR.ALL.GPU in front of every arrive, i.e. stall the
  // warpgroup's next wgmma per K-step, right after an epilogue until all its stores are acked.
  auto release = [&](uint32_t s) {
    if (!lead) return;
    if (rel_mask == 0) {
      ptx::mbar_arrive(&empty_bar[s]);
    } else {
      const uint32_t a = ptx::smem_addr(&empty_bar[s]);
      for (uint32_t r = 0; r < 4; ++r)
        if ((rel_mask >> r) & 1u) ptx::mbar_arrive_remote_cta(ptx::mapa(a, r));
    }
  };
  uint32_t prev = 0;
  for (int ks = 0; ks < ksteps; ++ks) {
    ptx::mbar_wait(&full_bar[stage], phase);
    if (ks == 0 && threadIdx.x == 4 * 32) trace(unit, 1);      // operands of the unit arrived
    const uint32_t sa = ptx::smem_addr(stage_base + stage * kStageBytes);
    const uint64_t a_hi = ptx::make_smem_desc(sa + a_row_off, kALbo, 128);
    const uint64_t b_hi = ptx::make_smem_desc(sa + kAStageBytes, kBLbo, 128);
    ptx::fence_regs(acc);
    ptx::wgmma_fence();
    ptx::wgmma_bf16_m64n256(acc, a_hi, b_hi, ks > 0 ? 1u : 0u);
    if (kSplit) {
      // descriptors differ only in the 16-byte-unit start address field
      ptx::wgmma_bf16_m64n256(acc, a_hi, b_hi + (kBPartBytes >> 4), 1u);
      ptx::wgmma_bf16_m64n256(acc, a_hi + (kAPartBytes >> 4), b_hi, 1u);
    }
    ptx::wgmma_commit();
    ptx::fence_regs(acc);
    if (ks > 0) {
      ptx::wgmma_wait<1>();
      release(prev);
    }
    prev = stage;
    if (++stage == kStages) { stage = 0; phase ^= 1; }
  }
  ptx::wgmma_wait<0>();
  ptx::fence_regs(acc);
  release(prev);
}

// Shifted sums of this thread's two rows over the unit columns c < ncols, bias included:
// s1 = sum(x - shift), s2 = sum((x - shift)^2) with shift = the row's value in column 0,
// reduced over the four threads that share a row.
__device__ __forceinline__ void row_shifted_sums(const float (&acc)[128], const float* bias, int ncols,
                                                 float (&shift)[2], float (&s1)[2], float (&s2)[2]) {
  const int q = threadIdx.x & 3;
  const float b0 = bias != nullptr ? bias[0] : 0.f;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    shift[h] = __shfl_sync(0xffffffffu, acc[2 * h] + b0, (threadIdx.x & 31) & ~3);
    s1[h] = 0.f;
    s2[h] = 0.f;
  }
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int c = 8 * j + 2 * q;
    const float2 b = bias != nullptr ? *reinterpret_cast<const float2*>(bias + c) : make_float2(0.f, 0.f);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (c < ncols) {
        const float x = acc[4 * j + 2 * h] + b.x - shift[h];
        s1[h] += x; s2[h] = fmaf(x, x, s2[h]);
      }
      if (c + 1 < ncols) {
        const float x = acc[4 * j + 2 * h + 1] + b.y - shift[h];
        s1[h] += x; s2[h] = fmaf(x, x, s2[h]);
      }
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
      s1[h] += __shfl_xor_sync(0xffffffffu, s1[h], o);
      s2[h] += __shfl_xor_sync(0xffffffffu, s2[h], o);
    }
  }
}

// Adds the staged pre-activation addends of one 32-column chunk (rows of this thread).
__device__ __forceinline__ void add_staged_chunk(float (&acc)[128], int j0, const float* gbuf, int lr0) {
  const int q = threadIdx.x & 3;
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float2 g = *reinterpret_cast<const float2*>(gbuf + (lr0 + 8 * h) * kEpiRowFloats + 8 * jj + 2 * q);
      acc[4 * (j0 + jj) + 2 * h] += g.x;
      acc[4 * (j0 + jj) + 2 * h + 1] += g.y;
    }
  }
}

// Byte offset of the 4-byte (two-column) piece of global column gc (even) of tile row r in
// the operand image of one 128-row tile; "lo" lives kAPartBytes further.
__device__ __forceinline__ size_t image_offset(int gc, int r) {
  return static_cast<size_t>(gc >> 4) * GCB_A_IMAGE_BLOCK + ((gc >> 3) & 1) * kALbo + r * 16 + (gc & 7) * 2;
}

// Gathered pre-activation addends (node projections of the split edge MLP) of the 256 columns
// [gcol_lo, gcol_lo + 256) of one tile, staged 32 columns at a time into the double buffer s_g
// ([2][128][36]; chunk count gc selects buffer and phase) by the kProducerWarps producer warps.
// Thread t: rows t/8 + 8p (p < 16), 16-byte column group t%8 of each chunk, so that 8 lanes read
// one 128-byte line segment of a gathered row.  Returns the updated chunk count.
__device__ __forceinline__ uint32_t stage_addends(float* s_g, uint64_t* g_full_bar, uint64_t* g_empty_bar,
                                                  const PreAddInfo* s_pre, int n_pre, long long trow0,
                                                  long long rows_total, int gcol_lo, uint32_t gc, int t64) {
  const int cgp = t64 & 7, rp = t64 >> 3;
  const PreAddInfo a = s_pre[0];
  const PreAddInfo b = s_pre[n_pre > 1 ? 1 : 0];
  int r0[16], r1[16];                            // source rows (-1: past the end)
#pragma unroll
  for (int p = 0; p < 16; ++p) {
    const long long grow = trow0 + rp + 8 * p;
    r0[p] = -1; r1[p] = -1;
    if (grow < rows_total) {
      r0[p] = a.idx ? __ldg(a.idx + grow) : static_cast<int>(grow);
      if (n_pre > 1) r1[p] = b.idx ? __ldg(b.idx + grow) : static_cast<int>(grow);
    }
  }
  for (int c0 = gcol_lo; c0 < gcol_lo + kUnitN; c0 += 32, ++gc) {
    const uint32_t gb = gc & 1;
    ptx::mbar_wait(&g_empty_bar[gb], ((gc >> 1) & 1) ^ 1);
    float* gdst = s_g + gb * kGBufFloats + rp * kEpiRowFloats + cgp * 4;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      float4 v[8];
#pragma unroll
      for (int p = 0; p < 8; ++p) {
        const int i = 8 * half + p;
        v[p] = r0[i] >= 0 ? __ldg(reinterpret_cast<const float4*>(a.table + static_cast<long long>(r0[i]) * a.ld + c0 + cgp * 4))
                          : make_float4(0.f, 0.f, 0.f, 0.f);
        if (r1[i] >= 0) {
          const float4 t = __ldg(reinterpret_cast<const float4*>(b.table + static_cast<long long>(r1[i]) * b.ld + c0 + cgp * 4));
          v[p].x += t.x; v[p].y += t.y; v[p].z += t.z; v[p].w += t.w;
        }
      }
#pragma unroll
      for (int p = 0; p < 8; ++p)
        *reinterpret_cast<float4*>(gdst + 8 * (8 * half + p) * kEpiRowFloats) = v[p];
    }
    __syncwarp();
    if ((t64 & 31) == 0) ptx::mbar_arrive(&g_full_bar[gb]);
  }
  return gc;
}

// kSplit: bf16x3 (hi/lo) vs single bf16 product.  kSwish / kLN: epilogue variant,
// compile-time so the per-element loops are straight-line code.
template <bool kSplit, bool kSwish, bool kLN>
__global__ void __launch_bounds__(kThreads, 1)
mlp_layer_tc_kernel(const __grid_constant__ gcb_layer_desc d) {
  using Cfg = TcConfig<kSplit, kLN>;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* stage_base = smem;
  float* s_bias = reinterpret_cast<float*>(smem + Cfg::kStages * Cfg::kStageBytes);
  float* s_scale = s_bias + kMaxN;                                  // LayerNorm variants only
  float* s_offset = s_scale + kMaxN;                                // LayerNorm variants only
  float* s_g = s_bias + Cfg::kParamBytes / 4;                       // [2][128][36] (not kLN)
  uint8_t* tail = reinterpret_cast<uint8_t*>(s_g) + Cfg::kGRegionBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(tail);          // [kStages]
  uint64_t* empty_bar = full_bar + Cfg::kStages;                   // [kStages]
  uint64_t* g_full_bar = empty_bar + Cfg::kStages;                 // [2]
  uint64_t* g_empty_bar = g_full_bar + 2;                          // [2]
  uint64_t* lnx_bar = g_empty_bar + 2;                             // [2 warpgroups][2] LayerNorm pair exchange
  SegInfo* s_seg = reinterpret_cast<SegInfo*>(lnx_bar + 4);               // [3]
  PreAddInfo* s_pre = reinterpret_cast<PreAddInfo*>(s_seg + 3);           // [2]
  KStepInfo* ks_info = reinterpret_cast<KStepInfo*>(s_pre + 2);           // [kMaxKSteps]
  // [2][128] LayerNorm statistics received from the partner CTA (N-split).  Aliases the
  // addend buffers, which LayerNorm layers never use (pre_add excludes LayerNorm).
  float2* s_lnx = reinterpret_cast<float2*>(s_g);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int n = d.n;
  const int n_halves = n / kUnitN;             // units per 128-row tile (1 or 2)
  const int num_tiles = (d.rows + kTileM - 1) / kTileM;
  // Segments backed by an operand image are streamed by TMA; if every segment is,
  // the producer warps have no A work at all (a_is_img).
  int ksteps = 0;
  bool a_is_img = true;
  for (int s = 0; s < d.nseg; ++s) {
    ksteps += d.seg[s].k / kKStep;
    a_is_img = a_is_img && (d.seg[s].img != nullptr);
  }
  const int dbg = g_dbg_flags;
  uint8_t* const out_img = (dbg & 2) ? nullptr : static_cast<uint8_t*>(d.out_img);
  // Descriptor fields used inside hot loops, hoisted into registers once.
  const long long rows_total = d.rows;
  const int nseg = d.nseg;
  const int n_pre = d.n_pre_add;               // gathered pre-activation addends (0..2)
  float* const out_ptr = (dbg & 2) ? nullptr : d.out;
  float* const outy_ptr = (dbg & 2) ? nullptr : d.out_y;
  const float* const res_ptr = d.residual;
  const long long ld_out = d.ld_out, ld_outy = d.ld_out_y, ld_res = d.ld_res;
  // Cluster schedule: the CTAs of a cluster walk the K-steps of `csize` consecutive
  // tiles in lockstep and share every weight tile through TMA multicast.
  const uint32_t crank = ptx::cluster_ctarank();
  const uint32_t csize = ptx::cluster_nctarank();
  const bool nsplit = (csize == 2) && (n_halves == 2);
  const uint32_t tiles_per_iter = nsplit ? 1u : csize;       // tiles a cluster covers per iteration
  const uint32_t tile_first = ptx::cluster_id_x() * tiles_per_iter;
  const uint32_t tile_stride = ptx::num_clusters_x() * tiles_per_iter;
  const uint32_t tile_off = nsplit ? 0u : crank;             // my tile = base + tile_off
  const int units_per_tile = nsplit ? 1 : n_halves;          // units this CTA runs per tile
  const uint16_t cmask = static_cast<uint16_t>((1u << csize) - 1u);
  // (experiment, debug flag 4) N-split pair without A multicast: each CTA streams the whole
  // block itself and recycles its stages on its own MMAs only.
  const bool decouple = nsplit && (dbg & 4);
  const bool gather_mode = !kLN && n_pre > 0;

  // ---- one-time setup ---------------------------------------------------------
  for (int i = threadIdx.x; i < n; i += kThreads) {
    s_bias[i] = d.bias[i];
    if (kLN) {
      s_scale[i] = d.ln_scale[i];
      s_offset[i] = d.ln_offset[i];
    }
  }
  if (threadIdx.x == 0) {
    int ks = 0;
    for (int s = 0; s < d.nseg; ++s) {
      s_seg[s].table = d.seg[s].table;
      s_seg[s].idx = d.seg[s].idx;
      s_seg[s].img = static_cast<const uint8_t*>(d.seg[s].img);
      s_seg[s].ld = d.seg[s].ld;
      s_seg[s].k_valid = d.seg[s].k_valid;
      s_seg[s].fan = d.seg[s].fan;
      s_seg[s].ksteps = d.seg[s].k / kKStep;
    }
    for (int s = 0; s < n_pre; ++s) {
      s_pre[s].table = d.pre_add[s].table;
      s_pre[s].idx = d.pre_add[s].idx;
      s_pre[s].ld = d.pre_add[s].ld;
    }
    for (int s = 0; s < d.nseg; ++s)
      for (int k = 0; k < d.seg[s].k; k += kKStep) {
        ks_info[ks].seg = static_cast<uint8_t>(s);
        ks_info[ks].is_img = d.seg[s].img != nullptr ? 1 : 0;
        ks_info[ks].koff = static_cast<uint16_t>(k);
        ++ks;
      }
    for (int s = 0; s < Cfg::kStages; ++s) {
      // 1 TMA lane (+ the producer warps unless A comes from images only)
      ptx::mbar_init(&full_bar[s], a_is_img ? 1 : 1 + kProducerWarps);
      // every consumer warp of every CTA that shares the stage
      ptx::mbar_init(&empty_bar[s], (decouple ? 1 : csize) * kConsumerWarps);
    }
    for (int b = 0; b < 2; ++b) {
      ptx::mbar_init(&g_full_bar[b], kProducerWarps);     // every producer warp
      ptx::mbar_init(&g_empty_bar[b], kConsumerWarps);    // every consumer warp
      ptx::mbar_init(&lnx_bar[b], 1);          // my expect_tx; the partner's 64 st.async complete it
      ptx::mbar_init(&lnx_bar[2 + b], 1);
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();
  ptx::cluster_sync_all();          // barrier inits visible cluster-wide before remote arrives

  // ---- roles ------------------------------------------------------------------
  if (warp < 4) {
    ptx::setmaxnreg_dec<kLayerProducerRegs>();       // whole warpgroup 0, before its warps split up
    if (warp == 0) {
      // ===== TMA warp =====
      // Converged warp, every lane polls, ONE elected lane issues.  The loop body is kept
      // minimal - running pointers, ring counters, one SegInfo read per segment.
      const uint32_t b_bytes = Cfg::kBStageBytes;                 // hi (| lo) of a 256-row block
      const size_t b_block = 2 * kBPartBytes;                     // image always holds hi|lo
      const size_t b_stride = static_cast<size_t>(n_halves) * b_block;   // next K-step, same half
      const uint32_t slice = b_bytes / csize;
      const uint32_t a_bytes = Cfg::kAStageBytes;                 // hi (| lo) block of one K-step
      const uint32_t a_half = a_bytes / 2;
      const bool b_own = (csize == 1) || nsplit;                  // my own weight block, no multicast
      const uint8_t* wimg = static_cast<const uint8_t*>(d.w_packed);
      uint32_t stage = 0, phase = 0, tu = 0;
      for (uint32_t base = tile_first; base < static_cast<uint32_t>(num_tiles); base += tile_stride) {
        const uint32_t tile = base + tile_off;
        const bool tile_ok = tile < static_cast<uint32_t>(num_tiles);   // else: dummy tile
        for (int uh = 0; uh < units_per_tile; ++uh, ++tu) {
          const int h = nsplit ? static_cast<int>(crank) : uh;          // my 256-column block
          const uint8_t* b_ptr = wimg + static_cast<size_t>(h) * b_block + (b_own ? 0u : crank * slice);
          const bool tr = tracing(tu);
          long long blocked = 0;
          for (int s = 0; s < nseg; ++s) {
            const SegInfo sg = s_seg[s];
            const bool a_copy = tile_ok && sg.img != nullptr;
            // Same tile in both CTAs of an N-split pair: each fetches half of every block and
            // multicasts it to both.
            const uint8_t* a_ptr = sg.img + static_cast<size_t>(tile) * sg.ksteps * GCB_A_IMAGE_BLOCK +
                                   (nsplit && !decouple ? crank * a_half : 0u);
            const uint32_t tx = b_bytes + (a_copy ? a_bytes : 0u);
            // (experiment, debug flag 16) L2 prefetch of the same block of my next tile
            const bool pf_next = (dbg & 16) && uh == units_per_tile - 1 &&
                                 tile + tile_stride < static_cast<uint32_t>(num_tiles);
            const size_t pf_off = static_cast<size_t>(tile_stride) * sg.ksteps * GCB_A_IMAGE_BLOCK;
            for (int k = 0; k < sg.ksteps; ++k) {
              const long long w0 = tr ? clock64() : 0;
              ptx::mbar_wait(&empty_bar[stage], phase ^ 1);   // free in every CTA of the cluster
              if (tr) blocked += clock64() - w0;
              uint8_t* a_dst = stage_base + stage * Cfg::kStageBytes;
              if (ptx::elect_one()) {
                ptx::mbar_arrive_expect_tx(&full_bar[stage], tx);
                if (pf_next && a_copy) ptx::bulk_prefetch_l2(a_ptr + pf_off, nsplit ? a_half : a_bytes);
                if (a_copy) {
                  if (nsplit && !decouple) ptx::bulk_g2s_multicast(a_dst + crank * a_half, a_ptr, a_half, &full_bar[stage], cmask);
                  else ptx::bulk_g2s(a_dst, a_ptr, a_bytes, &full_bar[stage]);
                }
                if (b_own) {
                  ptx::bulk_g2s(a_dst + Cfg::kAStageBytes, b_ptr, b_bytes, &full_bar[stage]);
                } else {
                  // Same block in every CTA: each fetches 1/csize and multicasts it to all.
                  ptx::bulk_g2s_multicast(a_dst + Cfg::kAStageBytes + crank * slice, b_ptr, slice,
                                          &full_bar[stage], cmask);
                }
              }
              __syncwarp();
              a_ptr += GCB_A_IMAGE_BLOCK;
              b_ptr += b_stride;
              if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
            }
          }
          if (lane == 0) trace_val(tu, 7, blocked);
        }
      }
    } else if (warp >= 4 - kProducerWarps) {
      // ===== producers (warps 2-3) =====
      const int t64 = threadIdx.x - 32 * (4 - kProducerWarps);
      const int sub = t64 & 3;                      // which float4 of the 16-wide K-step
      const int rg = t64 >> 2;                      // 0..15; rows rg + 16*i
      const uint32_t sts_off = (sub >> 1) * kALbo + (sub & 1) * 8;
      uint32_t it = 0, gc = 0;
      for (uint32_t base = tile_first; base < static_cast<uint32_t>(num_tiles); base += tile_stride) {
        const uint32_t tile = base + tile_off;       // may be past the end: all-zero dummy tile
        for (int uh = 0; uh < units_per_tile; ++uh) {
          if (!a_is_img) {
            // ----- activation (A operand) producer -----
            // Source row of each of my 8 tile rows, per segment (-1 = out of range).
            int src[3][8];
#pragma unroll
            for (int s = 0; s < 3; ++s) {
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                src[s][i] = -1;
                if (s < nseg) {
                  const long long grow = static_cast<long long>(tile) * kTileM + rg + 16 * i;
                  const int32_t* ip = s_seg[s].idx;
                  if (grow < rows_total) src[s][i] = ip ? __ldg(ip + grow) : static_cast<int>(grow);
                }
              }
            }
            float4 cur[8];
            bool have_cur = false, cur_img = false;
            uint32_t cur_it = 0;
            // Software pipeline over the K-steps: the loads of the next K-step are in flight
            // while the current one is converted and stored.
            for (int ks = 0; ks <= ksteps; ++ks) {
              const uint32_t this_it = it + ks;
              const bool mine = ks < ksteps;
              float4 nxt[8];
              const bool img_step = mine && ks_info[ks].is_img;   // TMA brings the data: arrive only
              if (mine && !img_step) {
                const int s = ks_info[ks].seg;
                const int koff = ks_info[ks].koff + sub * 4;
                const SegInfo sg = s_seg[s];
                const bool kvalid = koff < sg.k_valid;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
                  const int sr = (s == 0) ? src[0][i] : (s == 1 ? src[1][i] : src[2][i]);
                  if (kvalid && sr >= 0) {
                    const float* p = sg.table + static_cast<long long>(sr) * sg.fan * sg.ld + koff;
                    a = __ldg(reinterpret_cast<const float4*>(p));
                    for (int j = 1; j < sg.fan; ++j) {
                      const float4 t = __ldg(reinterpret_cast<const float4*>(p + static_cast<long long>(j) * sg.ld));
                      a.x += t.x; a.y += t.y; a.z += t.z; a.w += t.w;
                    }
                  }
                  nxt[i] = a;
                }
              }
              if (have_cur) {
                const uint32_t stage = cur_it % Cfg::kStages;
                const uint32_t phase = (cur_it / Cfg::kStages) & 1;
                ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
                uint8_t* a_hi = stage_base + stage * Cfg::kStageBytes;
                if (!cur_img) {
#pragma unroll
                  for (int i = 0; i < 8; ++i) {
                    uint2 hi, lo;
                    ptx::split_bf16x4(cur[i], hi, lo);
                    const uint32_t off = sts_off + (rg + 16 * i) * 16;
                    *reinterpret_cast<uint2*>(a_hi + off) = hi;
                    if (kSplit) *reinterpret_cast<uint2*>(a_hi + kAPartBytes + off) = lo;
                  }
                }
                ptx::fence_proxy_async_smem();
                __syncwarp();
                if (lane == 0) ptx::mbar_arrive(&full_bar[stage]);
                have_cur = false;
              }
              if (mine) {
#pragma unroll
                for (int i = 0; i < 8; ++i) cur[i] = nxt[i];
                cur_it = this_it;
                cur_img = img_step;
                have_cur = true;
              }
            }
            it += ksteps;
          }
          if (gather_mode) {
            const int gcol_lo = (nsplit ? static_cast<int>(crank) : uh) * kUnitN;
            gc = stage_addends(s_g, g_full_bar, g_empty_bar, s_pre, n_pre,
                               static_cast<long long>(tile) * kTileM, rows_total, gcol_lo, gc, t64);
          }
        }
      }
    }
  } else {
    ptx::setmaxnreg_inc<consumer_regs(kLayerProducerRegs)>();
    // ===== consumers: MMA + epilogue =====
    const int eg = (warp - 4) >> 2;                // warpgroup: tile rows [64 eg, 64 eg + 64)
    const int q = lane & 3;
    const int lr0 = eg * 64 + (warp & 3) * 16 + (lane >> 2);   // tile rows lr0, lr0 + 8
    const int n_valid = d.n_valid;
    const bool lead = lane == 0 && (warp & 3) == 0;
    const uint32_t rel_mask = (csize == 1 || decouple) ? 0u : cmask;
    // The image holds residual + y when an fp32 output is written, y otherwise.
    const bool img_res = res_ptr != nullptr && (out_ptr != nullptr || outy_ptr != nullptr);
    uint32_t stage = 0, phase = 0, g_count = 0, ln_count = 0, u = 0;
    float acc[128];
    for (uint32_t base = tile_first; base < static_cast<uint32_t>(num_tiles); base += tile_stride) {
      const uint32_t tile = base + tile_off;
      const bool tile_ok = tile < static_cast<uint32_t>(num_tiles);
      const long long grow0 = static_cast<long long>(tile) * kTileM + lr0;
      for (int uh = 0; uh < units_per_tile; ++uh, ++u) {
        const int h_blk = nsplit ? static_cast<int>(crank) : uh;
        const int col_base = h_blk * kUnitN;
        const int ncols = min(kUnitN, n_valid - col_base);
        if (lead && eg == 0) trace(u, 0);
        mma_unit<kSplit, Cfg::kStages, Cfg::kStageBytes, Cfg::kAStageBytes>(
            acc, stage_base, full_bar, empty_bar, stage, phase, ksteps, eg * 64 * 16, rel_mask, u);
        if (lead && eg == 0) { trace(u, 3); trace_val(u, 9, ksteps); }
        float mean[2] = {0.f, 0.f}, rstd[2] = {1.f, 1.f};
        if (kLN) {
          float shift[2], s1[2], s2[2];
          row_shifted_sums(acc, s_bias + col_base, ncols, shift, s1, s2);
          if (nsplit) {
            // LayerNorm over a row whose two halves live in the two CTAs of the cluster: each
            // CTA computes (mean, M2) of its 256 columns, hands them to the partner through
            // distributed shared memory, and both combine them (Chan's parallel update).
            const uint32_t lb = ln_count & 1, par = (ln_count >> 1) & 1;
            uint64_t* bar = &lnx_bar[eg * 2 + lb];
            const uint32_t peer = crank ^ 1u;
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
              mean[h] = 0.5f * (mh[h] + other.x);
              const float var = (m2h[h] + other.y + delta * delta * (0.5f * kUnitN)) * (1.0f / (2 * kUnitN));
              rstd[h] = rsqrtf(var + 1e-5f);
            }
            ++ln_count;
          } else {
            const float inv_n = 1.0f / static_cast<float>(ncols);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const float m1 = s1[h] * inv_n;
              mean[h] = shift[h] + m1;
              rstd[h] = rsqrtf(fmaxf(s2[h] * inv_n - m1 * m1, 0.f) + 1e-5f);
            }
          }
          if (lead && eg == 0) trace(u, 4);
        }
        // Epilogue, 32 columns (j0 .. j0 + 3) at a time; unrolled so that the accumulator is
        // only ever indexed with constants (it must stay in registers).
#pragma unroll
        for (int c0 = 0; c0 < kUnitN; c0 += 32) {
          if (c0 >= ncols) continue;
          const int j0 = c0 >> 3;
          if (gather_mode) {
            // Add the gathered node projections staged by the producer warps.
            const uint32_t gb = g_count & 1;
            ptx::mbar_wait(&g_full_bar[gb], (g_count >> 1) & 1);
            add_staged_chunk(acc, j0, s_g + gb * kGBufFloats, lr0);
            __syncwarp();
            if (lane == 0) ptx::mbar_arrive(&g_empty_bar[gb]);
            ++g_count;
          }
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const int c = c0 + 8 * jj + 2 * q;                 // unit column of this pair
            const int gc = col_base + c;
            const float2 b = *reinterpret_cast<const float2*>(s_bias + gc);
            float2 sc = make_float2(1.f, 1.f), of = make_float2(0.f, 0.f);
            if (kLN) {
              sc = *reinterpret_cast<const float2*>(s_scale + gc);
              of = *reinterpret_cast<const float2*>(s_offset + gc);
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float* v = &acc[4 * (j0 + jj) + 2 * h];
              v[0] += b.x; v[1] += b.y;
              if (kSwish) { v[0] = swish_f(v[0]); v[1] = swish_f(v[1]); }
              if (kLN) {
                v[0] = (v[0] - mean[h]) * rstd[h] * sc.x + of.x;
                v[1] = (v[1] - mean[h]) * rstd[h] * sc.y + of.y;
              }
              const long long grow = grow0 + 8 * h;
              const bool row_ok = grow < rows_total;
              float2 y = make_float2(v[0], v[1]);
              float2 r = make_float2(0.f, 0.f);
              if (res_ptr != nullptr && row_ok) {
                if (c + 1 < ncols) r = *reinterpret_cast<const float2*>(res_ptr + grow * ld_res + gc);
                else if (c < ncols) r.x = res_ptr[grow * ld_res + gc];
              }
              if (row_ok && c < ncols) {
                if (c + 1 < ncols) {
                  if (outy_ptr != nullptr) *reinterpret_cast<float2*>(outy_ptr + grow * ld_outy + gc) = y;
                  if (out_ptr != nullptr)
                    *reinterpret_cast<float2*>(out_ptr + grow * ld_out + gc) = make_float2(y.x + r.x, y.y + r.y);
                } else {
                  if (outy_ptr != nullptr) outy_ptr[grow * ld_outy + gc] = y.x;
                  if (out_ptr != nullptr) out_ptr[grow * ld_out + gc] = y.x + r.x;
                }
              }
              if (out_img != nullptr && tile_ok) {
                // Operand image of this tile for a later layer (n = n_valid = 512): the four
                // threads of a row complete one 16-byte piece, eight rows a 128-byte line.
                if (img_res) { y.x += r.x; y.y += r.y; }
                uint32_t hi, lo;
                ptx::split_bf16x2(y.x, y.y, hi, lo);
                uint8_t* dst = out_img + static_cast<size_t>(tile) * (n >> 4) * GCB_A_IMAGE_BLOCK +
                               image_offset(gc, lr0 + 8 * h);
                *reinterpret_cast<uint32_t*>(dst) = hi;
                *reinterpret_cast<uint32_t*>(dst + kAPartBytes) = lo;
              }
            }
          }
        }
        if (lead && eg == 0) trace(u, 5);
      }
    }
  }

  // ---- teardown ---------------------------------------------------------------
  // No CTA may exit while a peer can still multicast into its shared memory or arrive
  // on its barriers.
  __syncthreads();
  ptx::cluster_sync_all();
}

}  // namespace gcb
