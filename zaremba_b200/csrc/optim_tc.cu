// SGD update fused with the rebuild of the fp16 operand images (tensor-core engine).
// The update pass already holds every new weight in registers; writing its fp16 images from there
// removes the separate pack pass (which re-read 348 MB of fp32 weights per step at the Large config).
#include "tc_kernels.h"

namespace zrb {

struct PackSpec {
    __half* row_img;     // [rows, ld] row-major image or null
    int64_t ld;
    __half* fwd_img;     // recurrent forward slices  [cta][kc][g][8][8] or null
    int fU, fG, fKc, fKS;   // units per cluster (KS * U), row groups, K chunks per CTA, K-split factor
    __half* bwd_img;     // recurrent backward slices [cluster][4][kc][g][8][8] or null
    int bUC, bG, bKc, bS;   // units per cluster, row groups, K chunks per CTA, K-split factor per gate
    int write_g;         // store coef * g back into the gradient buffer (clip_grad_norm_'s in-place scaling)
    int pdl;             // launched as a programmatic dependent of the forward recurrence kernel enqueued before it
                         // (deferred update, zrb_set_lazy_update): release the next dependent at once, and block 0 waits
                         // for the primary before it exits so that the grid cannot complete before the primary has
};

__device__ __forceinline__ void pdl_prologue(const PackSpec& sp) {
    if (sp.pdl && threadIdx.x == 0) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__device__ __forceinline__ void pdl_epilogue(const PackSpec& sp) {
    if (sp.pdl && blockIdx.x == 0 && threadIdx.x == 0) asm volatile("griddepcontrol.wait;" ::: "memory");
}

template <int VEC> struct VecT;
template <> struct VecT<4> { using type = float4; };
template <> struct VecT<2> { using type = float2; };
template <> struct VecT<1> { using type = float; };

template <int VEC>
__device__ __forceinline__ void load_vec(const float* p, float (&v)[VEC]) {
    typename VecT<VEC>::type t = __ldcs(reinterpret_cast<const typename VecT<VEC>::type*>(p));
    const float* f = reinterpret_cast<const float*>(&t);
#pragma unroll
    for (int i = 0; i < VEC; ++i) v[i] = f[i];
}
// VEC consecutive fp16 values (VEC-element aligned destination) with the widest stores
template <int VEC>
__device__ __forceinline__ void store_halves(__half* dst, const __half (&h)[VEC]) {
    if constexpr (VEC == 1) {
        dst[0] = h[0];
    } else {
#pragma unroll
        for (int x = 0; x < VEC; x += 2) reinterpret_cast<__half2*>(dst)[x >> 1] = __halves2half2(h[x], h[x + 1]);
    }
}

template <int VEC>
__device__ __forceinline__ void store_vec(float* p, const float (&v)[VEC]) {
    typename VecT<VEC>::type t;
    float* f = reinterpret_cast<float*>(&t);
#pragma unroll
    for (int i = 0; i < VEC; ++i) f[i] = v[i];
    __stcs(reinterpret_cast<typename VecT<VEC>::type*>(p), t);
}

// matrix [rows, cols] (cols % VEC == 0): g *= coef; p -= lr*g; row-major fp16 image of the new p.
template <int VEC>
__global__ void update_pack_kernel(float* __restrict__ p, float* __restrict__ g, int rows, int cols, float lr,
                                   const float* __restrict__ scalars, PackSpec sp) {
    pdl_prologue(sp);
    const float coef = scalars[1];
    const int cv = cols / VEC;
    const int64_t total = (int64_t)rows * cv;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int r = (int)(i / cv), c = (int)(i % cv) * VEC;
        const int64_t off = (int64_t)r * cols + c;
        float gv[VEC], pv[VEC];
        load_vec<VEC>(g + off, gv);
        load_vec<VEC>(p + off, pv);
#pragma unroll
        for (int x = 0; x < VEC; ++x) { gv[x] *= coef; pv[x] = sgd_elem(pv[x], gv[x], lr); }
        if (sp.write_g) store_vec<VEC>(g + off, gv);
        store_vec<VEC>(p + off, pv);
        if (sp.row_img) {
            __half hh[VEC];
#pragma unroll
            for (int x = 0; x < VEC; ++x) hh[x] = __float2half_rn(pv[x]);
            store_halves<VEC>(sp.row_img + (int64_t)r * sp.ld + c, hh);
        }
    }
    pdl_epilogue(sp);
}

// W_hh [4H, H] with both recurrent images: a thread owns an 8-row x VEC-column tile (rows j..j+7 of one gate
// block), so the backward image -- whose 16-byte vectors hold 8 consecutive K indices (= rows) of one unit
// (= column) -- is written with full 16-byte stores instead of 2-byte scatters.
template <int VEC>
__global__ void update_pack_whh_kernel(float* __restrict__ p, float* __restrict__ g, int H, float lr,
                                       const float* __restrict__ scalars, PackSpec sp) {
    pdl_prologue(sp);
    const float coef = scalars[1];
    const int cv = H / VEC, jb_n = (H + 7) >> 3;
    const int64_t total = (int64_t)4 * jb_n * cv;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % cv) * VEC;
        const int jb = (int)((i / cv) % jb_n), q = (int)(i / ((int64_t)cv * jb_n));
        const int j0 = jb << 3;
        __half hv[8][VEC];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const int j = j0 + e;
            if (j < H) {
                const int64_t off = ((int64_t)q * H + j) * H + c;
                float gv[VEC], pv[VEC];
                load_vec<VEC>(g + off, gv);
                load_vec<VEC>(p + off, pv);
#pragma unroll
                for (int x = 0; x < VEC; ++x) { gv[x] *= coef; pv[x] = sgd_elem(pv[x], gv[x], lr); hv[e][x] = __float2half_rn(pv[x]); }
                if (sp.write_g) store_vec<VEC>(g + off, gv);
                store_vec<VEC>(p + off, pv);
                if (sp.row_img) store_halves<VEC>(sp.row_img + ((int64_t)q * H + j) * sp.ld + c, hv[e]);
                if (sp.fwd_img) {   // slice of the CTA owning unit j, row 4u+q; K indices c..c+VEC-1 share a K chunk
                    const int cluster = j / sp.fU, u = j % sp.fU, row = 4 * u + q;
                    const int kc = c >> 3, cta = cluster * sp.fKS + kc / sp.fKc, kcl = kc % sp.fKc;
                    store_halves<VEC>(sp.fwd_img + (((int64_t)cta * sp.fKc + kcl) * sp.fG + (row >> 3)) * 64 +
                                          (row & 7) * 8 + (c & 7), hv[e]);
                }
            } else {
#pragma unroll
                for (int x = 0; x < VEC; ++x) hv[e][x] = __float2half_rn(0.f);
            }
        }
        if (sp.bwd_img) {   // units c..c+VEC-1, rank q, K chunk jb: one 16-byte vector per unit
#pragma unroll
            for (int x = 0; x < VEC; ++x) {
                const int cl = (c + x) / sp.bUC, u = (c + x) % sp.bUC;
                uint4 v;
                v.x = (uint32_t)__half_as_ushort(hv[0][x]) | ((uint32_t)__half_as_ushort(hv[1][x]) << 16);
                v.y = (uint32_t)__half_as_ushort(hv[2][x]) | ((uint32_t)__half_as_ushort(hv[3][x]) << 16);
                v.z = (uint32_t)__half_as_ushort(hv[4][x]) | ((uint32_t)__half_as_ushort(hv[5][x]) << 16);
                v.w = (uint32_t)__half_as_ushort(hv[6][x]) | ((uint32_t)__half_as_ushort(hv[7][x]) << 16);
                const int rank = q * sp.bS + jb / sp.bKc, kcl = jb % sp.bKc;
                *reinterpret_cast<uint4*>(sp.bwd_img + ((((int64_t)cl * 4 * sp.bS + rank) * sp.bKc + kcl) * sp.bG) * 64 +
                                          (u >> 3) * 64 + (u & 7) * 8) = v;
            }
        }
    }
    pdl_epilogue(sp);
}

template <int VEC>
static int update_pack_launch(float* p, float* g, int rows, int cols, float lr, const float* scalars, const PackSpec& sp,
                              bool whh, cudaStream_t s) {
    int64_t total = whh ? (int64_t)4 * ((cols + 7) / 8) * (cols / VEC) : (int64_t)rows * (cols / VEC);
    const int threads = whh ? 128 : 256;
    int blocks = (int)((total + threads - 1) / threads);
    if (blocks > 132 * 16) blocks = 132 * 16;
    if (sp.pdl) {
        // beside the persistent forward recurrence: a dynamic shared-memory request larger than what that kernel leaves
        // free on its SMs keeps these blocks on the ~23 idle SMs, off the latency-critical ones
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(blocks); cfg.blockDim = dim3(threads); cfg.dynamicSmemBytes = 12 * 1024; cfg.stream = s;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        if (whh) ZRB_CUDA(cudaLaunchKernelEx(&cfg, update_pack_whh_kernel<VEC>, p, g, cols, lr, scalars, sp));
        else ZRB_CUDA(cudaLaunchKernelEx(&cfg, update_pack_kernel<VEC>, p, g, rows, cols, lr, scalars, sp));
        count_launch();
        return ZRB_OK;
    }
    if (whh) update_pack_whh_kernel<VEC><<<blocks, threads, 0, s>>>(p, g, cols, lr, scalars, sp);
    else update_pack_kernel<VEC><<<blocks, threads, 0, s>>>(p, g, rows, cols, lr, scalars, sp);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

int update_pack(float* p, float* g, int rows, int cols, float lr, const float* scalars, __half* row_img, int64_t ld,
                __half* fwd_img, const RecPlan* fp, __half* bwd_img, const RecPlan* bp, bool write_g, cudaStream_t s,
                bool pdl) {
    PackSpec sp;
    sp.write_g = write_g ? 1 : 0;
    sp.pdl = pdl ? 1 : 0;
    sp.row_img = row_img; sp.ld = ld;
    sp.fwd_img = fwd_img; sp.fKS = fp ? fp->KS : 1; sp.fU = fp ? fp->KS * fp->U : 1; sp.fG = fp ? fp->G : 1;
    sp.fKc = fp ? fp->KcS : 1;
    sp.bwd_img = bwd_img; sp.bS = bp ? bp->KS : 1; sp.bUC = bp ? 4 * bp->KS * bp->U : 4; sp.bG = bp ? bp->G : 1;
    sp.bKc = bp ? bp->KcS : 1;
    const bool whh = (fwd_img || bwd_img) && rows == 4 * cols;
    const bool al16 = ((((uintptr_t)p) | ((uintptr_t)g)) & 15) == 0, al8 = ((((uintptr_t)p) | ((uintptr_t)g)) & 7) == 0;
    if (cols % 4 == 0 && al16) return update_pack_launch<4>(p, g, rows, cols, lr, scalars, sp, whh, s);
    if (cols % 2 == 0 && al8) return update_pack_launch<2>(p, g, rows, cols, lr, scalars, sp, whh, s);
    return update_pack_launch<1>(p, g, rows, cols, lr, scalars, sp, whh, s);
}

}  // namespace zrb
