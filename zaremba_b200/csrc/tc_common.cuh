// sm_90a primitives used by the tensor-core kernels: mbarrier, TMA (cp.async.bulk[.tensor]),
// warpgroup MMA (wgmma.mma_async, fence / commit / wait) and its shared-memory descriptors.
// Inline PTX only (no CUTLASS); formats follow the PTX ISA "asynchronous warpgroup level
// matrix" section.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <stdlib.h>
#include "common.cuh"

namespace zrb {
// host: whether rec_launch (lstm_rec_fwd.cu, where the launch modes of the persistent recurrence kernels are described)
// launches a cluster grid programmatically.  A plain launch is only as safe as its occupancy check, so the default is
// programmatic only while ONE tensor-core context is alive on the device -- a process that holds several (an ensemble,
// two trainers) gets the cooperative launch.  ZRB_REC_PDL=0 forces cooperative, =1 forces programmatic.
static inline int rec_pdl_env() {
    static const int mode = [] { const char* e = getenv("ZRB_REC_PDL"); return e ? (atoi(e) != 0 ? 1 : 0) : -1; }();
    return mode;
}
static inline bool rec_pdl_enabled() { return rec_pdl_env() != 0; }   // (GEMMs: trigger early; harmless before a cooperative launch)
static inline bool rec_launch_programmatic(int dev) {
    const int m = rec_pdl_env();
    return m < 0 ? g_live_tc_ctx[dev & 63].load(std::memory_order_relaxed) <= 1 : m == 1;
}
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier ---------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// arrive on the mbarrier at `bar`'s offset in the shared memory of cluster rank `rank` (this CTA's own included), with
// the default CTA-scope release: it hands back a stage whose reads (wgmma) have completed, and orders no memory writes.
// (.release.cluster would put a MEMBAR.GPU in front of every arrive: ~1 us per stage, measured.)
__device__ __forceinline__ void mbar_arrive_rank(uint64_t* bar, uint32_t rank) {
    uint32_t a;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(a) : "r"(smem_u32(bar)), "r"(rank));
    asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(a) : "memory");
}
__device__ __forceinline__ uint32_t cta_rank_in_cluster() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
// every thread of every CTA in the cluster (warp-converged)
__device__ __forceinline__ void cluster_barrier() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}

// ---- proxies / fences ---------------------------------------------------------------------
// generic-proxy writes to shared memory -> visible to the async proxy (TMA, wgmma operands)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// generic-proxy writes to global memory -> visible to async-proxy reads (bulk copies)
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }
// the same for the global state space only: a single FENCE.VIEW.ASYNC.G (the all-spaces form adds a MEMBAR.GPU)
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

// ---- TMA ----------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)m) : "memory");
}
// 2-D tiled load: box at (c0 = innermost coordinate, c1) -> smem, completes on `bar`
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        :: "r"(smem_u32(dst)), "l"((uint64_t)m), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
// the same box written to the same shared-memory offset of every CTA in `cta_mask` (cluster ranks), each of which has
// its mbarrier at `bar`'s offset signalled with the box's bytes
__device__ __forceinline__ void tma_load_2d_multicast(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                                      uint16_t cta_mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
        " [%0], [%1, {%3, %4}], [%2], %5;"
        :: "r"(smem_u32(dst)), "l"((uint64_t)m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask)
        : "memory");
}
// 1-D bulk copy global -> shared (bytes multiple of 16, 16-byte aligned both sides)
__device__ __forceinline__ void bulk_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        :: "r"(smem_u32(dst)), "l"((uint64_t)src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}

// ---- wgmma ----------------------------------------------------------------------------------------
// A warpgroup (4 consecutive warps, the first a multiple of 4) issues every wgmma together: .sync.aligned, so the
// whole warpgroup must reach each of these with the same control flow.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int kPending>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across wgmma_wait
template <int R>
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// wgmma.mma_async m64nNk16, f32 accumulators in registers (N/2 per thread), A and B from shared-memory
// descriptors; TA / TB = 1 reads that operand MN-major.  scale_d = 0 overwrites the accumulators.
template <int N, int TA, int TB> struct Wgmma;
template <int TA, int TB> struct Wgmma<8, TA, TB> {
    static __device__ __forceinline__ void mma(float (&d)[4], uint64_t da, uint64_t db, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %6, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n8k16.f32.f16.f16 "
            "{%0, %1, %2, %3}, "
            "%4, %5, p, 1, 1, %7, %8;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
            : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
    }
};
template <int TA, int TB> struct Wgmma<16, TA, TB> {
    static __device__ __forceinline__ void mma(float (&d)[8], uint64_t da, uint64_t db, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %10, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7}, "
            "%8, %9, p, 1, 1, %11, %12;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
    }
};
template <int TA, int TB> struct Wgmma<24, TA, TB> {
    static __device__ __forceinline__ void mma(float (&d)[12], uint64_t da, uint64_t db, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %14, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n24k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11}, "
            "%12, %13, p, 1, 1, %15, %16;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11])
            : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
    }
};
template <int TA, int TB> struct Wgmma<32, TA, TB> {
    static __device__ __forceinline__ void mma(float (&d)[16], uint64_t da, uint64_t db, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
            "%16, %17, p, 1, 1, %19, %20;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
    }
};
template <int TA, int TB> struct Wgmma<64, TA, TB> {
    static __device__ __forceinline__ void mma(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %34, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
            "%32, %33, p, 1, 1, %35, %36;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
    }
};
template <int TA, int TB> struct Wgmma<128, TA, TB> {
    static __device__ __forceinline__ void mma(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %66, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
            "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
            "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
            "%64, %65, p, 1, 1, %67, %68;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
              "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
              "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
              "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
    }
};
template <int TA, int TB> struct Wgmma<256, TA, TB> {
    static __device__ __forceinline__ void mma(float (&d)[128], uint64_t da, uint64_t db, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %130, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
            "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
            "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
            "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
            "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
            "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
            "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
            "%128, %129, p, 1, 1, %131, %132;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
              "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
              "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
              "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
              "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
              "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
              "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
              "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
              "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
              "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
              "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
              "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
            : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
    }
};

// Accumulator fragment of m64nN: register 4 * c8 + 2 * h + e of thread t holds row 16 * (t / 32) + (t % 32) / 4 + 8 * h,
// column 8 * c8 + 2 * (t % 4) + e.
__device__ __forceinline__ int wgmma_row(int t, int h) { return 16 * (t >> 5) + ((t & 31) >> 2) + 8 * h; }
__device__ __forceinline__ int wgmma_col(int t, int c8) { return 8 * c8 + 2 * (t & 3); }

// ---- descriptors ------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptor (64 bit):
//   [0,14) start address >> 4   [16,30) leading byte offset >> 4   [32,46) stride byte offset >> 4
//   [49,52) base offset (0: every swizzled tile here starts 1024-byte aligned)   [62,64) swizzle: 0 none, 1 = 128B
// K-major: LBO = distance between the two 8-element K core matrices of a K=16 step (no swizzle; unused with 128B),
//          SBO = distance between 8-row groups.
// MN-major, 128B swizzle: LBO = distance between 64-element MN blocks, SBO = distance between 8-row K groups.
constexpr uint64_t kSwizzleNone = 0, kSwizzle128B = 1;
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes,
                                                   uint64_t swizzle) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) |
           ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32) | (swizzle << 62);
}

}  // namespace tc
}  // namespace zrb
