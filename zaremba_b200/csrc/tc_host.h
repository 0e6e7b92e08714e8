// Host-side helpers shared by the tensor-core kernels.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>

#include "common.cuh"

namespace zrb {
int tc_num_sms();
int tc_make_tmap_f16(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t box_inner,
                     uint32_t box_outer, int swizzle128);
// One fp16 operand of gemm_f16_tc, row pitch ld elements.  mn_major: stored with the M (A) or N (B) index contiguous,
// i.e. A as [K,M] and B as [K,N]; else K-major, A [M,K] and B [N,K].
struct GemmOperand {
    const __half* ptr = nullptr;
    int64_t ld = 0;
    bool mn_major = false;
};
// One launch of the wgmma GEMM: C[M,N] fp32 = alpha * op(A) * op(B)^T (+bias) (+C).  Every optional field is off by
// default.
struct Gemm {
    GemmOperand A, B;
    float* C = nullptr;
    int64_t ldc = 0;
    int M = 0, N = 0, K = 0;
    float alpha = 1.f;
    const float* bias = nullptr;    // [N] or null, added to every row
    const float* bias2 = nullptr;   // [N] or null: a second bias vector added with the first (needs bias)
    bool accumulate = false;        // add into C instead of storing
    // (plain-store launches only) gemm_f16_tc_sumsq_slots(*this).first floats whose sum is sum(C^2), by a fixed
    // summation tree
    float* sumsq = nullptr;
    // launch as a programmatic dependent of the kernel enqueued just before it on the stream (which must be one of the
    // persistent recurrence kernels: they release their dependents once all their CTAs are resident).  The GEMM must
    // not read anything that kernel writes; it runs on the SMs the recurrence leaves idle and waits for it before
    // completing.
    bool pdl = false;
    // Set dual.C for a second problem dual.C[M, dual.N] = alpha * op(A) * op(dual.B)^T computed by the same launch: the
    // same A, M and K, dual.B in B's layout with pitch dual.ldb, dual.C with pitch dual.ldc (the two weight gradients of
    // a layer share dG as their A operand; with per-layer widths dW_ih is [4H, In] and dW_hh [4H, H]).  Both problems
    // are tiled with the tile width of the wider one, and the work items of the second follow those of the first.  No
    // bias, no accumulate.
    struct Dual {
        const __half* B = nullptr;
        float* C = nullptr;
        int N = 0;
        int64_t ldb = 0, ldc = 0;
        float* sumsq = nullptr;     // gemm_f16_tc_sumsq_slots(the Gemm).dual floats, as sumsq
    } dual;
    // EXPERIMENT (zrb_gemm_f16_tiled): K-major operands also given as pre-tiled, pre-swizzled images with that many
    // 128-row tiles per K block
    const __half* a_tiled = nullptr;
    int a_nt128 = 0;
    const __half* b_tiled = nullptr;
    int b_nt128 = 0;
};
int gemm_f16_tc(const Gemm& g, cudaStream_t s);
// The sum-of-squares slot counts g's launch writes once g.sumsq (and g.dual.sumsq) are set: first for C, dual for the
// dual problem's C (0 without one)
struct GemmSlots {
    int first, dual;
};
GemmSlots gemm_f16_tc_sumsq_slots(const Gemm& g);
}  // namespace zrb
