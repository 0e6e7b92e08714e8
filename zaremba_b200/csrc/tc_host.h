// Host-side helpers shared by the tensor-core kernels.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>

#include "common.cuh"

namespace zrb {
int tc_num_sms();
int tc_make_tmap_f16(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t box_inner,
                     uint32_t box_outer, int swizzle128);
// The second problem of a dual launch: its N, its B operand's pitch and its output's pitch.  N = 0: the first
// problem's N, ldb and ldc.
struct DualB {
    int N = 0;
    int64_t ldb = 0, ldc = 0;
};
// C[M,N] fp32 = alpha * op(A) * op(B)^T (+bias) (+C); *_mn = operand stored with the M/N index contiguous
int gemm_f16_tc(const __half* A, int64_t lda, int a_mn, const __half* B, int64_t ldb, int b_mn, float* C, int64_t ldc,
                int M, int N, int K, float alpha, const float* bias, int accumulate, cudaStream_t s,
                float* sumsq_out = nullptr, const float* bias2 = nullptr, bool pdl = false, const __half* B2 = nullptr,
                float* C2 = nullptr, float* sumsq_out2 = nullptr, const __half* A_tiled = nullptr, int a_nt128 = 0,
                const __half* B_tiled = nullptr, int b_nt128 = 0, DualB d2 = DualB{});
// B2 / C2 (/ sumsq_out2): a second problem C2[M,N2] = alpha * op(A) * op(B2)^T with the same A, M and K, and N2 and
// pitches from d2, computed by the same launch (the two weight gradients of a layer share dG as their A operand; with
// per-layer widths dW_ih is [4H, In] and dW_hh [4H, H]).  Both problems are tiled with the tile width of the wider one,
// and the work items of the second follow those of the first.  No bias, no accumulate.
// pdl: launch as a programmatic dependent of the kernel enqueued just before it on `s` (which must be one of the
// persistent recurrence kernels: they release their dependents once all their CTAs are resident).  The GEMM must not
// read anything that kernel writes; it runs on the SMs the recurrence leaves idle and waits for it before completing.
// sumsq_out (plain-store calls only): gemm_f16_tc_sumsq_slots(M, N, K) floats whose sum is sum(C^2), fixed summation tree
int gemm_f16_tc_sumsq_slots(int M, int N, int K);
// ... and the two slot counts of a dual launch with N and N2 = d2.N (equal to gemm_f16_tc_sumsq_slots when N2 = N)
void gemm_f16_tc_dual_sumsq_slots(int M, int N1, int N2, int K, int* n1, int* n2);
}  // namespace zrb
