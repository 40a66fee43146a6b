// Thin inline-PTX wrappers for the sm_90a features the MLP kernels use:
// mbarrier, 1-D bulk async copy (TMA engine), thread-block clusters and wgmma.
// Descriptor bit layouts follow the PTX ISA wgmma "matrix descriptor" table.
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

namespace gcb {
namespace ptx {

__device__ __forceinline__ uint32_t smem_addr(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier ---------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count)
               : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_addr(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)),
               "r"(bytes)
               : "memory");
}
// Blocking wait on the phase with the given parity.  With GCB_BOUNDED_WAIT a
// wait that exceeds ~1-2 s of SM clocks traps: a protocol bug then surfaces as
// a launch failure instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_addr(bar);
  uint32_t done = 0;
#ifdef GCB_BOUNDED_WAIT
  const long long t0 = clock64();
#endif
  for (;;) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, 0x2710;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
    if (done) return;
#ifdef GCB_BOUNDED_WAIT
    if (clock64() - t0 > 3000000000ll) asm volatile("trap;");
#endif
  }
}

// Busy-polling wait (mbarrier.test_wait, no suspend): lowest wake-up latency; for the
// single issuing lanes of the TMA / MMA warps, which have nothing else to do.
__device__ __forceinline__ void mbar_spin(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_addr(bar);
  uint32_t done = 0;
#ifdef GCB_BOUNDED_WAIT
  const long long t0 = clock64();
#endif
  for (;;) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
    if (done) return;
#ifdef GCB_BOUNDED_WAIT
    if (clock64() - t0 > 3000000000ll) asm volatile("trap;");
#endif
  }
}

// ---- proxies / fences ---------------------------------------------------------
// Make generic-proxy shared-memory writes (st.shared) visible to the async
// proxy (wgmma operand reads, bulk copies).
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// Same for global memory: generic-proxy st.global made visible to later bulk copies
// (cp.async.bulk reads through the async proxy) that are ordered after this thread.
__device__ __forceinline__ void fence_proxy_async_global() {
  asm volatile("fence.proxy.async.global;" ::: "memory");
}

// ---- bulk async copy global -> shared (TMA engine, no tensor map) ------------
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes,
                                         uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(smem_addr(smem_dst)),
      "l"(gmem_src), "r"(bytes), "r"(smem_addr(bar))
      : "memory");
}

// ---- L2 cache policies -----------------------------------------------------------------
// evict_last: lines of the chain kernel's scratch ring.  They are rewritten in place every few
// units; with the default policy the GBs streaming through the L2 in between evict them and every
// scratch write ends up in DRAM (ncu: 10.7 GB written by a launch whose only HBM output is 3.3 GB).
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void st_global_b32_hint(void* ptr, uint32_t v, uint64_t policy) {
  asm volatile("st.global.L2::cache_hint.b32 [%0], %1, %2;" ::"l"(ptr), "r"(v), "l"(policy) : "memory");
}

// ---- predicated accesses (the chain kernel's epilogue) ----------------------------------
// Predicated instructions instead of branches: a load whose predicate is false leaves `fill` in
// its destination, a store whose predicate is false does nothing, and the code around them stays
// one straight-line block that the compiler can schedule freely.
__device__ __forceinline__ uint2 ld_global_nc_v2_pred(const void* ptr, bool pred, uint32_t fill) {
  uint2 v;
  asm volatile(
      "{\n .reg .pred p;\n setp.ne.b32 p, %3, 0;\n mov.b32 %0, %4;\n mov.b32 %1, %4;\n"
      " @p ld.global.nc.v2.b32 {%0, %1}, [%2];\n}"
      : "=r"(v.x), "=r"(v.y) : "l"(ptr), "r"(static_cast<uint32_t>(pred)), "r"(fill));
  return v;
}
// Coherent (not .nc): the fp32 residual may be the output this kernel updates in place.
__device__ __forceinline__ uint2 ld_global_v2_pred(const void* ptr, bool pred) {
  uint2 v;
  asm volatile(
      "{\n .reg .pred p;\n setp.ne.b32 p, %3, 0;\n mov.b32 %0, 0;\n mov.b32 %1, 0;\n"
      " @p ld.global.v2.b32 {%0, %1}, [%2];\n}"
      : "=r"(v.x), "=r"(v.y) : "l"(ptr), "r"(static_cast<uint32_t>(pred)));
  return v;
}
__device__ __forceinline__ uint32_t ld_global_b32_pred(const void* ptr, bool pred) {
  uint32_t v;
  asm volatile(
      "{\n .reg .pred p;\n setp.ne.b32 p, %2, 0;\n mov.b32 %0, 0;\n @p ld.global.b32 %0, [%1];\n}"
      : "=r"(v) : "l"(ptr), "r"(static_cast<uint32_t>(pred)));
  return v;
}
__device__ __forceinline__ float2 ld_shared_v2_pred(uint32_t saddr, bool pred) {
  float2 v;
  asm volatile(
      "{\n .reg .pred p;\n setp.ne.b32 p, %3, 0;\n mov.b32 %0, 0f00000000;\n mov.b32 %1, 0f00000000;\n"
      " @p ld.shared.v2.f32 {%0, %1}, [%2];\n}"
      : "=f"(v.x), "=f"(v.y) : "r"(saddr), "r"(static_cast<uint32_t>(pred)));
  return v;
}
// 8 bytes from shared memory into integer registers, unpredicated (ld_shared_v2_pred is predicated).
__device__ __forceinline__ uint2 ld_shared_v2_u32(uint32_t saddr) {
  uint2 v;
  asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(saddr));
  return v;
}
__device__ __forceinline__ void st_global_v2_pred(void* ptr, float2 v, bool pred) {
  asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %3, 0;\n @p st.global.v2.f32 [%0], {%1, %2};\n}"
               ::"l"(ptr), "f"(v.x), "f"(v.y), "r"(static_cast<uint32_t>(pred)) : "memory");
}
__device__ __forceinline__ void st_global_b32_pred(void* ptr, uint32_t v, bool pred) {
  asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %2, 0;\n @p st.global.b32 [%0], %1;\n}"
               ::"l"(ptr), "r"(v), "r"(static_cast<uint32_t>(pred)) : "memory");
}
__device__ __forceinline__ void st_global_b32_hint_pred(void* ptr, uint32_t v, uint64_t policy, bool pred) {
  asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %3, 0;\n @p st.global.L2::cache_hint.b32 [%0], %1, %2;\n}"
               ::"l"(ptr), "r"(v), "l"(policy), "r"(static_cast<uint32_t>(pred)) : "memory");
}
// bulk copy global -> shared, multicast, with an L2 cache policy for the source lines
__device__ __forceinline__ void bulk_g2s_multicast_hint(void* smem_dst, const void* gmem_src,
                                                        uint32_t bytes, uint64_t* bar,
                                                        uint16_t cta_mask, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster.L2::cache_hint "
      "[%0], [%1], %2, [%3], %4, %5;"
      ::"r"(smem_addr(smem_dst)),
      "l"(gmem_src), "r"(bytes), "r"(smem_addr(bar)), "h"(cta_mask), "l"(policy)
      : "memory");
}

// Hint: bring [gmem_src, +bytes) into L2 (no shared-memory destination, no completion).
__device__ __forceinline__ void bulk_prefetch_l2(const void* gmem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gmem_src), "r"(bytes) : "memory");
}

// Same, multicast to every CTA of the cluster selected by cta_mask: the bytes land at
// the same CTA-relative offset in each destination CTA and complete_tx is signalled on
// the mbarrier at the same CTA-relative offset there.
__device__ __forceinline__ void bulk_g2s_multicast(void* smem_dst, const void* gmem_src,
                                                   uint32_t bytes, uint64_t* bar,
                                                   uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster "
      "[%0], [%1], %2, [%3], %4;"
      ::"r"(smem_addr(smem_dst)),
      "l"(gmem_src), "r"(bytes), "r"(smem_addr(bar)), "h"(cta_mask)
      : "memory");
}

// ---- thread-block cluster -----------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t cluster_nctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t cluster_id_x() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t num_clusters_x() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%nclusterid.x;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// Distributed shared memory: address of the same CTA-relative location in CTA `rank`.
__device__ __forceinline__ uint32_t mapa(uint32_t saddr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(saddr), "r"(rank));
  return r;
}
__device__ __forceinline__ void st_cluster_f32x2(uint32_t raddr, float a, float b) {
  asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(raddr), "f"(a), "f"(b) : "memory");
}
// Asynchronous 8-byte store into another CTA's shared memory that signals that CTA's
// mbarrier (complete_tx, 8 bytes) when the data is visible there.  No release fence in the
// sender: the alternative, st.shared::cluster followed by `mbarrier.arrive.release.cluster`
// (mbar_arrive_remote), compiles to MEMBAR.ALL.GPU, which first waits until every global
// store the thread has outstanding is acknowledged.
__device__ __forceinline__ void st_async_f32x2(uint32_t raddr, float a, float b, uint32_t rbar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v2.f32 [%0], {%1, %2}, [%3];"
               ::"r"(raddr), "f"(a), "f"(b), "r"(rbar) : "memory");
}
// Arrive with release at cluster scope on an mbarrier of THIS CTA (pairs with a
// mbar_wait_cluster by a thread that then acts on behalf of the whole cluster).
__device__ __forceinline__ void mbar_arrive_release_cluster(uint64_t* bar) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cta.b64 _, [%0];" ::"r"(smem_addr(bar)) : "memory");
}
// Arrive (release at cluster scope) on an mbarrier of another CTA of the cluster.  Compiles
// to MEMBAR.ALL.CTA + MEMBAR.ALL.GPU before the arrive: for hand-overs of generic-proxy
// writes only.
__device__ __forceinline__ void mbar_arrive_remote(uint32_t raddr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(raddr) : "memory");
}
// Arrive (default semantics: release at CTA scope) on an mbarrier of another CTA of the
// cluster: a bare SYNCS.ARRIVE, no memory fence.  Enough to free a buffer whose readers were
// async-proxy operations that have already completed (retired wgmma, landed bulk copies) and
// whose next writer is a bulk copy or a thread that first observes the barrier.
__device__ __forceinline__ void mbar_arrive_remote_cta(uint32_t raddr) {
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(raddr) : "memory");
}
// Wait with acquire at cluster scope (pairs with mbar_arrive_remote).
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_addr(bar);
  uint32_t done = 0;
#ifdef GCB_BOUNDED_WAIT
  const long long t0 = clock64();
#endif
  for (;;) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2, 0x2710;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
    if (done) return;
#ifdef GCB_BOUNDED_WAIT
    if (clock64() - t0 > 3000000000ll) asm volatile("trap;");
#endif
  }
}

// ---- wgmma ---------------------------------------------------------------------
// Shared-memory matrix descriptor, K-major operand, no swizzle ("interleave"):
// the operand is a grid of core matrices, each 8 rows x 16 bytes stored as 128
// contiguous bytes;  SBO = byte distance between core matrices adjacent along
// M/N (next 8 rows),  LBO = byte distance between core matrices adjacent along
// K (next 16 bytes of K).  Fields are in units of 16 bytes.
//   [0,14)  start address >> 4      [16,30) LBO >> 4      [32,46) SBO >> 4
//   [49,52) base offset = 0         [62,64) layout type = 0 (no swizzle)
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes,
                                                   uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  return d;
}

// The accumulator of a 64 x 256 fp32 tile, owned by one warpgroup: thread t of warp w holds
// d[4j + 2h + e] = D[16w + t/4 + 8h][8j + 2(t%4) + e]  (j < 32, h, e < 2).
// D (+)= A[smem] * B[smem]^T for one K-step of 16, issued by the whole warpgroup.
__device__ __forceinline__ void wgmma_bf16_m64n256(float (&d)[128], uint64_t a_desc, uint64_t b_desc,
                                                   uint32_t scale_d) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
        "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
        "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
        "}, %128, %129, p, 1, 1, 0, 0;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]),
          "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]),
          "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]),
          "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
          "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]),
          "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]),
          "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]),
          "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]),
          "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]),
          "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]),
          "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]),
          "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]),
          "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]),
          "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]),
          "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]),
          "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(a_desc), "l"(b_desc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_fence() {
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
template <int kPending>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory");
}
// Keeps the compiler from moving accesses of the accumulator across wgmma issue / wait.
__device__ __forceinline__ void fence_regs(float (&d)[128]) {
#pragma unroll
  for (int i = 0; i < 128; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ---- register reallocation between warpgroups ---------------------------------------
// Every warp of a warpgroup must execute the same one; kRegs is a multiple of 8 in [24, 256].
template <int kRegs>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs));
}
template <int kRegs>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs));
}

// ---- misc ---------------------------------------------------------------------
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(pred));
  return pred != 0;
}

// Split four floats into packed bf16 "hi" and "lo" parts: x ~= hi + lo with
// |x - hi - lo| <= 2^-17 |x|.
__device__ __forceinline__ void split_bf16x4(const float4& x, uint2& hi, uint2& lo) {
  __nv_bfloat162 h01 = __floats2bfloat162_rn(x.x, x.y);
  __nv_bfloat162 h23 = __floats2bfloat162_rn(x.z, x.w);
  float2 f01 = __bfloat1622float2(h01);
  float2 f23 = __bfloat1622float2(h23);
  __nv_bfloat162 l01 = __floats2bfloat162_rn(x.x - f01.x, x.y - f01.y);
  __nv_bfloat162 l23 = __floats2bfloat162_rn(x.z - f23.x, x.w - f23.y);
  hi.x = *reinterpret_cast<uint32_t*>(&h01);
  hi.y = *reinterpret_cast<uint32_t*>(&h23);
  lo.x = *reinterpret_cast<uint32_t*>(&l01);
  lo.y = *reinterpret_cast<uint32_t*>(&l23);
}

// Same for two floats (two adjacent columns): one packed 32-bit word each for hi and lo,
// the first float in the low half.
__device__ __forceinline__ void split_bf16x2(float a, float b, uint32_t& hi, uint32_t& lo) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  const float2 f = __bfloat1622float2(h);
  __nv_bfloat162 l = __floats2bfloat162_rn(a - f.x, b - f.y);
  hi = *reinterpret_cast<uint32_t*>(&h);
  lo = *reinterpret_cast<uint32_t*>(&l);
}

}  // namespace ptx
}  // namespace gcb
