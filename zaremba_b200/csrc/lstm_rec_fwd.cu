// Persistent LSTM recurrence, forward, one launch per layer (sm_90a; launch modes: rec_launch below).
//
//   for t in 0..T-1:   gates_t = XG_t + h_{t-1} * W_hh^T ;  (i,f,g,o) ;  c_t, h_t     (model.py:34-45)
//
// Work split: CTA k owns U hidden units j in [k*U, k*U+U) (their cell math, c_t in registers for the whole
// window).  The slice of W_hh a CTA multiplies with (fp16, ~144 KB) is loaded ONCE into shared memory in the
// canonical no-swizzle K-major wgmma layout and stays there for all T steps (weight-stationary):
//   SPLIT = false  the 4U gate rows of its own units x the whole contraction, M = 64 tiles   (H < 256)
//   SPLIT = true   CTA PAIRS (clusters of 2): the 8U gate rows of the pair's units x ONE HALF of the contraction,
//                  M = 128 tiles; see the K-split note below.  The description below is the SPLIT = false flow;
//                  with SPLIT the drain pushes rows to their owner instead of staging them.
//
// Per step:
//   loader thread   polls the grid-barrier counter (relaxed loads, one fence.acquire.gpu after the last
//                   arrival, fence.proxy.async.global), then brings the 72 KB h_{t-1} operand image (written
//                   by all CTAs, already in wgmma layout; step 0: the image fwd_prep built from the incoming
//                   state) into shared memory as four cp.async.bulk pieces, each with its own mbarrier, so
//                   the MMAs start when the first quarter of K has landed
//   MMA warpgroup   H/16 wgmma m64nNk16 (N = pad8(B)) chained into register accumulators, then each
//                   accumulator row is staged in shared memory (rec_common.cuh: rec_mma_step)
//   8 epilogue warps add the x-part pre-activations prefetched during the MMAs to the staged rows,
//                   apply the cell rule (lstm_cell.cuh) and dropout (variational mode: the operand image holds h * rm, rm
//                   the cell's recurrent multiplier drawn once before the step loop and kept in a register).
//                   The next step's operand image is stored FIRST and published (one red.release.gpu on the grid-barrier counter, which is never reset:
//                   the launch gets its starting value); everything backward needs (activated gates, c_t,
//                   row-major fp16 h, dropout(h) for the next layer) is stored after the arrival, off the
//                   critical path.
//
// Roofline: latency/L2/shared-memory bound, not tensor bound -- per step each CTA streams its 144 KB
// weight slice from shared memory through the tensor core and all CTAs re-read the 72 KB h image
// from L2; algorithmic flops per layer call = 8*T*B*H^2.
#include <stdlib.h>

#include "lstm_rec_fwd.cuh"

namespace zrb {

// ---- weight / state image builders ---------------------------------------------------------------
// w_img[cta][kcl][g][r][e] = half(W_hh[q*H + j, k]) with cta = cluster * KS + rank, row i = g*8 + r = 4*uc + q,
// uc = unit within the cluster (UC = KS * U units), j = cluster*UC + uc, k = (rank*KcS + kcl)*8 + e
// m active (weight drop): W[r, k] * the multiplier of element r*H + k; a thread then writes 4 consecutive e (one quad of
// k), so that each quad of mask elements costs one Philox call
__global__ void pack_whh_fwd_kernel(const float* __restrict__ W, __half* __restrict__ img, int H, int UC, int G, int KcS,
                                    int KS, int nCTA, MaskSrc m) {
    const size_t per_cta = (size_t)KcS * G * 64;
    const size_t total = per_cta * nCTA;
    if (m.active) {
        for (size_t idx = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4; idx < total;
             idx += (size_t)gridDim.x * blockDim.x * 4) {
            int cta = (int)(idx / per_cta);
            size_t r0 = idx % per_cta;
            int e0 = (int)(r0 & 7), r = (int)((r0 >> 3) & 7);
            int g = (int)((r0 >> 6) % G), kcl = (int)((r0 >> 6) / G);
            int i = g * 8 + r, uc = i >> 2, q = i & 3;
            int cluster = cta / KS, rank = cta % KS;
            int j = cluster * UC + uc, k0 = (rank * KcS + kcl) * 8 + e0;
            const bool row_ok = uc < UC && j < H;
            const size_t row = (size_t)q * H + j;
            float mul[4] = {0.f, 0.f, 0.f, 0.f};
            if (row_ok && k0 < H) mask_mul4_at(m, row * H + k0, mul);
#pragma unroll
            for (int t = 0; t < 4; ++t)
                img[idx + t] = __float2half_rn(row_ok && k0 + t < H ? W[row * H + k0 + t] * mul[t] : 0.f);
        }
        return;
    }
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (size_t)gridDim.x * blockDim.x) {
        int cta = (int)(idx / per_cta);
        size_t r0 = idx % per_cta;
        int e = (int)(r0 & 7), r = (int)((r0 >> 3) & 7);
        int g = (int)((r0 >> 6) % G), kcl = (int)((r0 >> 6) / G);
        int i = g * 8 + r, uc = i >> 2, q = i & 3;
        int cluster = cta / KS, rank = cta % KS;
        int j = cluster * UC + uc, k = (rank * KcS + kcl) * 8 + e;
        float v = 0.f;
        if (uc < UC && j < H && k < H) v = W[((size_t)q * H + j) * H + k];
        img[idx] = __float2half_rn(v);
    }
}

// ---- host ------------------------------------------------------------------------------------------
size_t rec_smem_bytes(int Kc, int G, int GB) {
    return (size_t)Kc * G * 128 + (size_t)Kc * GB * 128 + 2 * 64 * (GB * 8 + 1) * 4 + 128 /*align*/ + 128 /*bars*/;
}

// 8-row batch groups of the K-split plans' operand images: the real ones (wgmma's m64nNk16 takes any N that is a multiple
// of 8), but two at B <= 8.  The receive area (2 x 64 x (8 GBi + 1) floats, rows of pitch 8 GBi + 4) holds the 8U rows a
// CTA receives for U <= 13 at N = 16, for U <= 12 only at N = 8; at H = 1500, U = 12 would need 16 backward clusters of 8,
// more than the GPCs hold, and the backward would fall back to clusters of 4
int rec_split_groups(int GB) { return GB < 2 ? 2 : GB; }

int rec_max_clusters(const void* kernel, int cluster, int smem, int nCTA) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(nCTA);
    cfg.blockDim = dim3(kRecThreads);
    cfg.dynamicSmemBytes = (size_t)smem;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = cluster; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    int n = 0;
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess ||
        cudaOccupancyMaxActiveClusters(&n, kernel, &cfg) != cudaSuccess) {
        (void)cudaGetLastError();
        return 0;
    }
    return n;
}

int rec_plan_finish(RecPlan* plan, const void* kernel, int cluster) {
    plan->kernel = kernel;
    plan->cluster = cluster;
    plan->max_clusters = rec_max_clusters(kernel, cluster, plan->smem, plan->nCTA);
    int dev = 0, per_sm = 0, reserved = 0;
    ZRB_CUDA(cudaGetDevice(&dev));
    ZRB_CUDA(cudaDeviceGetAttribute(&per_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev));
    ZRB_CUDA(cudaDeviceGetAttribute(&reserved, cudaDevAttrReservedSharedMemoryPerBlock, dev));
    plan->beside_smem = per_sm - 2 * reserved - plan->smem + 1;
    plan->ok = 1;
    return ZRB_OK;
}

static bool rec_no_coop() {
    // Profilers (Nsight Compute) refuse cooperative + cluster launches; under one (detected through the injection
    // environment it sets up) or with ZRB_NO_COOP=1 cluster kernels take the checked plain launch
    static const bool v = getenv("ZRB_NO_COOP") != nullptr || getenv("CUDA_INJECTION64_PATH") != nullptr ||
                          getenv("NV_COMPUTE_PROFILER_PERFWORKS_DIR") != nullptr || getenv("NVTX_INJECTION64_PATH") != nullptr;
    return v;
}

// How both persistent recurrence kernels are launched.  Their grid barrier needs all nCTA CTAs co-resident:
//   cooperative   -- the driver guarantees it or refuses the launch (cudaErrorCooperativeLaunchTooLarge: an error, no
//                    fallback).  Always for the unclustered forward, which has no plain mode; for cluster grids unless one
//                    of the next two applies.
//   programmatic  -- a plain cluster launch, checked against the plan's occupancy answer, with the programmatic-
//                    serialization attribute: the GEMM enqueued before it triggers at its start, so the recurrence CTAs
//                    take SMs as the GEMM's CTAs retire and fetch their resident weight slices while its tail is still
//                    running (pdl_wait in the kernels).  9 us per train step at the Large config; the cooperative
//                    attribute suppresses the early start (measured: no gain with both attributes).  Decided at every
//                    launch by rec_launch_programmatic (tc_common.cuh: while ONE tensor-core context is alive on the
//                    device, since a second context can appear at any time), never for a traced launch.
//   checked plain -- the same launch without the programmatic attribute: under a profiler (rec_no_coop), or when a
//                    cooperative cluster launch fails for another reason than the grid's size.
// A plain launch is only as safe as the occupancy check: two persistent grids launched at the same time from two
// streams could each get part of the device and spin on their barriers until the bounded waits give up and fail the
// zrb context (rec_common.cuh: RecWatch).
int rec_launch(const RecPlan& p, void** args, bool trace, cudaStream_t s, const char* name) {
    if (p.cluster == 1) {
        ZRB_CUDA(cudaLaunchCooperativeKernel(p.kernel, dim3(p.nCTA), dim3(kRecThreads), args, (size_t)p.smem, s));
        count_launch();
        return ZRB_OK;
    }
    int dev = 0;
    cudaGetDevice(&dev);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(p.nCTA);
    cfg.blockDim = dim3(kRecThreads);
    cfg.dynamicSmemBytes = (size_t)p.smem;
    cfg.stream = s;
    cudaLaunchAttribute attrs[2];
    attrs[0].id = cudaLaunchAttributeClusterDimension;
    attrs[0].val.clusterDim.x = p.cluster; attrs[0].val.clusterDim.y = 1; attrs[0].val.clusterDim.z = 1;
    cfg.attrs = attrs;
    const bool programmatic = rec_launch_programmatic(dev) && !trace;
    const bool plain = programmatic || rec_no_coop();
    cudaError_t e = cudaSuccess;
    if (!plain) {
        attrs[1].id = cudaLaunchAttributeCooperative;
        attrs[1].val.cooperative = 1;
        cfg.numAttrs = 2;
        e = cudaLaunchKernelExC(&cfg, p.kernel, args);
        if (e == cudaErrorCooperativeLaunchTooLarge) {
            (void)cudaGetLastError();
            set_error("%s: the %d-CTA grid cannot be co-resident on this device", name, p.nCTA);
            return ZRB_E_CUDA;
        }
        if (e != cudaSuccess) (void)cudaGetLastError();   // e.g. not supported under a tool: try the checked plain launch
    }
    if (plain || e != cudaSuccess) {
        if (p.max_clusters * p.cluster < p.nCTA) {
            set_error("%s: %d clusters of %d needed, the device can hold %d at once", name, p.nCTA / p.cluster, p.cluster,
                      p.max_clusters);
            return ZRB_E_CUDA;
        }
        cfg.numAttrs = 1;
        if (programmatic) {
            attrs[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
            attrs[1].val.programmaticStreamSerializationAllowed = 1;
            cfg.numAttrs = 2;
        }
        e = cudaLaunchKernelExC(&cfg, p.kernel, args);
    }
    if (e != cudaSuccess) {
        set_error("%s launch failed: %s", name, cudaGetErrorString(e));
        return ZRB_E_CUDA;
    }
    count_launch();
    return ZRB_OK;
}

int rec_fwd_plan(int H, int B, RecPlan* plan) {
    // [KS == 2]; naming <false> first keeps the order of the two kernels in the cubin
    const void* const kernel[2] = {(const void*)lstm_rec_fwd_kernel<false, false>,
                                   (const void*)lstm_rec_fwd_kernel<true, false>};
    int nsm = tc_num_sms();
    plan->GB = (B + 7) / 8;
    plan->ok = 0;
    plan->KS = 1;
    if (plan->GB * 8 > 32) return ZRB_OK;  // accumulators / staging sized for N <= 32
    // K-split pairs (see the kernel header); the operand image's batch groups: rec_split_groups
    if (H >= 256) {
        const int Kp = (H + 31) / 32 * 32, Kc = Kp / 8, KcS = Kc / 2, GBi = rec_split_groups(plan->GB);
        // first choice (rec_split_first_choice): one (unit, batch) cell per epilogue thread, and SMs left for the work
        // beside the recurrence; else the largest U that fits, up to kRecMaxCell cells per thread
        for (int pass = 0; pass < 2; ++pass)
            for (int U = 16; U >= 1; --U) {
                const int npair = (H + 2 * U - 1) / (2 * U);
                if (2 * npair > nsm) break;
                if (U * B > kRecMaxCell * kRecEpiThreads || (pass == 0 && !rec_split_first_choice(U, B, 2 * npair, nsm)))
                    continue;
                const int G = U;                              // 8U gate rows of the pair / 8
                const size_t smem = rec_smem_bytes(KcS, G, GBi);
                // two M = 64 tiles read 16 row groups per K chunk: the last chunk reaches (16-G)*128 B past the slice, into the h buffer
                if (smem <= 227 * 1024 && 2 * 4 * U * (GBi * 8 + 4) <= 2 * 64 * (GBi * 8 + 1)) {
                    plan->KS = 2; plan->U = U; plan->G = G; plan->nCTA = 2 * npair; plan->smem = (int)smem;
                    plan->Kc = Kc; plan->KcS = KcS; plan->GBi = GBi;
                    return rec_plan_finish(plan, kernel[1], 2);
                }
            }
    }
    int Kp = (H + 15) / 16 * 16;
    plan->Kc = Kp / 8;
    plan->KcS = plan->Kc;
    plan->GBi = plan->GB;
    for (int U = 16; U >= 1; --U) {
        int n = (H + U - 1) / U;
        if (n > nsm) break;
        int G = (4 * U + 7) / 8;
        size_t smem = rec_smem_bytes(plan->Kc, G, plan->GB);
        // the M=64 wgmma reads 8 row groups per K chunk: the last chunk reaches (8-G)*128 B past the
        // slice, which lands in the h image buffer that follows it
        if (smem <= 227 * 1024 && U * B <= kRecMaxCell * kRecEpiThreads) {
            plan->U = U; plan->G = G; plan->nCTA = n; plan->smem = (int)smem;
            return rec_plan_finish(plan, kernel[0], 1);
        }
    }
    return ZRB_OK;
}

int pack_whh_fwd(const float* W, __half* img, int H, const RecPlan& p, cudaStream_t s, MaskSrc m) {
    pack_whh_fwd_kernel<<<tc_num_sms() * 4, 256, 0, s>>>(W, img, H, p.KS * p.U, p.G, p.KcS, p.KS, p.nCTA, m);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

int lstm_rec_fwd(const RecPlan& p, const RecWatchdog& wd, RecFwdArgs a, cudaStream_t s) {
    a.U = p.U; a.G = p.G; a.GB = p.GB; a.Kc = p.Kc; a.nCTA = p.nCTA; a.KcS = p.KcS; a.GBi = p.GBi;
    ZRB_REQUIRE(wd.flag && wd.host, "lstm_rec_fwd needs the context's watchdog words");
    a.w = rec_watch_args(wd);
    a.base += rec_fault_base("fwd");   // (tests only)
    if (a.trace) ZRB_CUDA(cudaMemsetAsync(a.trace + 4, 0x80, 2 * sizeof(long long), s));
    void* args[] = {&a};
    if (!a.zo.on) return rec_launch(p, args, a.trace != nullptr, s, "lstm_rec_fwd");
    ZRB_REQUIRE(a.h0 && a.ctil, "zoneout needs h0 and the c~ buffer");
    RecPlan q = p;   // the same plan through the zoneout instantiation (same shared memory, one CTA per SM)
    q.kernel = rec_fwd_zoneout_kernel(p.KS == 2);
    if (!q.kernel) return ZRB_E_CUDA;
    return rec_launch(q, args, a.trace != nullptr, s, "lstm_rec_fwd (zoneout)");
}

}  // namespace zrb
