// clip_grad_norm_ + SGD over a list of tensors -- main.py:114-117.
// Pure HBM streaming.  Pass 1 reads every gradient once (sum of squares); pass 2 reads g and p and
// writes g and p (and, for the tensor-core engine, the fp16 operand images of the new weights, so the
// weights are not re-read by a separate pack pass).  Algorithmic bytes per parameter element:
// 4 (norm) + 16 (update) [+ 2..6 for fp16 images of the matrices].
// Tensors that are adjacent in memory (the Trainer's flat buffers) are coalesced into one run and
// streamed with 128-bit accesses.
#include "kernels.h"

namespace zrb {

constexpr int kNormBlocks = 148 * 8;
constexpr int kThreads = 256;

__device__ __forceinline__ float block_sum(float acc, float* sh) {
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
    __syncthreads();
    float v = 0.f;
    if (threadIdx.x < 32) {
        v = threadIdx.x < kThreads / 32 ? sh[threadIdx.x] : 0.f;
        v = warp_sum(v);
    }
    return v;
}

// sum of squares of this block's grid-stride share (blocks bx of nbx) of one run of `n` floats
__device__ __forceinline__ float block_sumsq(const float* __restrict__ g, int64_t n, int bx, int nbx, float* sh) {
    float acc = 0.f;
    const int64_t tid = (int64_t)bx * blockDim.x + threadIdx.x, stride = (int64_t)nbx * blockDim.x;
    if ((((uintptr_t)g) & 15) == 0) {
        const float4* g4 = reinterpret_cast<const float4*>(g);
        const int64_t n4 = n >> 2;
        int64_t i = tid;
        for (; i + 3 * stride < n4; i += 4 * stride) {   // 4 independent 16-byte loads in flight
            float4 a = __ldcs(g4 + i), b = __ldcs(g4 + i + stride), c = __ldcs(g4 + i + 2 * stride),
                   d = __ldcs(g4 + i + 3 * stride);
            acc += a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w;
            acc += b.x * b.x + b.y * b.y + b.z * b.z + b.w * b.w;
            acc += c.x * c.x + c.y * c.y + c.z * c.z + c.w * c.w;
            acc += d.x * d.x + d.y * d.y + d.z * d.z + d.w * d.w;
        }
        for (; i < n4; i += stride) {
            float4 a = __ldcs(g4 + i);
            acc += a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w;
        }
        for (int64_t j = (n4 << 2) + tid; j < n; j += stride) acc += g[j] * g[j];
    } else {
        for (int64_t j = tid; j < n; j += stride) acc += g[j] * g[j];
    }
    return block_sum(acc, sh);
}

// runs of contiguous floats (the tensor list after merging neighbours); block (x, y) takes share x of run y and owns
// partial slot y * gridDim.x + x, so one launch covers the whole list and no slot is written twice
struct Runs {
    float* p[kMaxTensors];
    float* g[kMaxTensors];
    int64_t n[kMaxTensors];
};
__global__ void sumsq_kernel(Runs r, float* __restrict__ partials) {
    __shared__ float sh[kThreads / 32];
    float v = block_sumsq(r.g[blockIdx.y], r.n[blockIdx.y], blockIdx.x, gridDim.x, sh);
    if (threadIdx.x == 0) partials[blockIdx.y * gridDim.x + blockIdx.x] = v;
}

// scalars[0] = norm, scalars[1] = clip coefficient  (double accumulation of the partials)
__global__ void norm_finalize_kernel(const float* __restrict__ partials, int n, float max_norm,
                                     float* __restrict__ scalars, float* __restrict__ norm_out) {
    __shared__ double sh[32];
    double acc = 0.0;
    // up to ~15k partials: batches of 8 independent loads per thread (a rolled loop pays one L2 round trip per load)
    int i = threadIdx.x;
    for (; i + 7 * (int)blockDim.x < n; i += 8 * (int)blockDim.x) {
        float v[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = partials[i + k * (int)blockDim.x];
#pragma unroll
        for (int k = 0; k < 8; ++k) acc += (double)v[k];
    }
    for (; i < n; i += blockDim.x) acc += (double)partials[i];
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += sh[i];
        float norm = (float)sqrt(t);
        float coef = max_norm / (norm + 1e-6f);   // torch.nn.utils.clip_grad_norm_
        if (coef > 1.f) coef = 1.f;
        scalars[0] = norm;
        scalars[1] = coef;
        if (norm_out) *norm_out = norm;
    }
}

// g *= coef (clip_grad_norm_ scales .grad in place); p -= lr * g (main.py:117)
template <bool WRITE_G>
__global__ void clip_sgd_update_kernel(Runs r, float lr, const float* __restrict__ scalars) {
    float* __restrict__ p = r.p[blockIdx.y];
    float* __restrict__ g = r.g[blockIdx.y];
    const int64_t n = r.n[blockIdx.y];
    const float coef = scalars[1];
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
    if (((((uintptr_t)g) | ((uintptr_t)p)) & 15) == 0) {
        float4* g4 = reinterpret_cast<float4*>(g);
        float4* p4 = reinterpret_cast<float4*>(p);
        const int64_t n4 = n >> 2;
        for (int64_t i = tid; i < n4; i += stride) {
            float4 gv = __ldcs(g4 + i), pv = __ldcs(p4 + i);
            gv.x *= coef; gv.y *= coef; gv.z *= coef; gv.w *= coef;
            pv.x -= lr * gv.x; pv.y -= lr * gv.y; pv.z -= lr * gv.z; pv.w -= lr * gv.w;
            if (WRITE_G) __stcs(g4 + i, gv);
            __stcs(p4 + i, pv);
        }
        for (int64_t j = (n4 << 2) + tid; j < n; j += stride) {
            float gv = g[j] * coef;
            if (WRITE_G) g[j] = gv;
            p[j] -= lr * gv;
        }
    } else {
        for (int64_t j = tid; j < n; j += stride) {
            float gv = g[j] * coef;
            if (WRITE_G) g[j] = gv;
            p[j] -= lr * gv;
        }
    }
}

// merge tensors that are adjacent in memory (both p and g) into runs; returns the run count and the block
// count per run (sized for the longest run, all runs' partial slots fit in kNormBlocks)
static int coalesce(const TensorList& tl, Runs* r, int* blocks_per_run) {
    int runs = 0;
    int64_t longest = 0;
    for (int t = 0; t < tl.count; ++t) {
        if (tl.n[t] == 0) continue;
        if (runs && r->p[runs - 1] + r->n[runs - 1] == tl.p[t] && r->g[runs - 1] + r->n[runs - 1] == tl.g[t]) {
            r->n[runs - 1] += tl.n[t];
        } else {
            r->p[runs] = tl.p[t]; r->g[runs] = tl.g[t]; r->n[runs] = tl.n[t];
            ++runs;
        }
    }
    for (int i = runs; i < kMaxTensors; ++i) { r->p[i] = nullptr; r->g[i] = nullptr; r->n[i] = 0; }
    for (int i = 0; i < runs; ++i) longest = r->n[i] > longest ? r->n[i] : longest;
    int64_t b = (longest / 4 + kThreads - 1) / kThreads;
    if (b < 1) b = 1;
    const int cap = kNormBlocks / (runs > 0 ? runs : 1);
    *blocks_per_run = (int)(b > cap ? cap : b);
    return runs;
}

int norm_partials_base() { return kNormBlocks; }

int grad_norm(const TensorList& tl, float max_norm, float* partials, float* scalars, float* norm_out,
              cudaStream_t s, bool extra_used, int n_gemm) {
    Runs r;
    int bpr = 1;
    const int runs = coalesce(tl, &r, &bpr);
    ZRB_CUDA(cudaMemsetAsync(partials, 0, (kNormBlocks + (extra_used ? 0 : kNormExtra)) * sizeof(float), s));
    if (runs) {
        sumsq_kernel<<<dim3(bpr, runs), kThreads, 0, s>>>(r, partials);
        ZRB_KERNEL_CHECK();
    }
    // one block, 1024 threads: up to ~15k partials, a handful of independent loads per thread
    norm_finalize_kernel<<<1, 1024, 0, s>>>(partials, kNormBlocks + kNormExtra + n_gemm, max_norm, scalars, norm_out);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

// update only (norm / coefficient already in `scalars`)
int sgd_apply(const TensorList& tl, float lr, const float* scalars, bool write_g, cudaStream_t s) {
    Runs r;
    int bpr = 1;
    const int runs = coalesce(tl, &r, &bpr);
    if (!runs) return ZRB_OK;
    int64_t longest = 0;   // grid.x sized for the longest run (no slot limit here); shorter runs leave blocks idle
    for (int i = 0; i < runs; ++i) longest = r.n[i] > longest ? r.n[i] : longest;
    int64_t b = (longest / 4 + kThreads - 1) / kThreads;
    const int bx = (int)(b < 1 ? 1 : (b > kNormBlocks ? kNormBlocks : b)) * 2;
    if (write_g) clip_sgd_update_kernel<true><<<dim3(bx, runs), kThreads, 0, s>>>(r, lr, scalars);
    else clip_sgd_update_kernel<false><<<dim3(bx, runs), kThreads, 0, s>>>(r, lr, scalars);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

int clip_sgd(const TensorList& tl, float lr, float max_norm, float* partials, float* scalars, float* norm_out,
             bool write_g, cudaStream_t s) {
    ZRB_TRY(grad_norm(tl, max_norm, partials, scalars, norm_out, s));
    return sgd_apply(tl, lr, scalars, write_g, s);
}

// ---- dynamic evaluation (DESIGN.md section 14) ---------------------------------------------------------------------
// Tensors without an fp16 image (biases, fc.b, the untied embedding; every tensor on the validation engine).  Block
// (x, y) streams share x of tensor y; no coalescing, so theta_g and r need not be laid out like p.
struct DynRuns {
    float* p[kMaxTensors];
    const float* g[kMaxTensors];
    const float* tg[kMaxTensors];
    const float* r[kMaxTensors];
    int64_t n[kMaxTensors];
};

// the non-empty entries of the list; returns their count and sets *bx to the blocks per tensor (cap: no more in all)
static int dyn_runs(const TensorList& tl, float* const* tg, float* const* r, DynRuns* d, int* bx, int cap) {
    int k = 0;
    int64_t longest = 0;
    for (int t = 0; t < tl.count; ++t) {
        if (tl.n[t] == 0) continue;
        d->p[k] = tl.p[t]; d->g[k] = tl.g[t]; d->n[k] = tl.n[t];
        d->tg[k] = tg ? tg[t] : nullptr;
        d->r[k] = r ? r[t] : nullptr;
        longest = tl.n[t] > longest ? tl.n[t] : longest;
        ++k;
    }
    int64_t b = (longest / 4 + kThreads - 1) / kThreads;
    if (b < 1) b = 1;
    const int c = cap / (k > 0 ? k : 1);
    *bx = (int)(b > c ? c : b);
    return k;
}

template <bool RMS>
__global__ void dyneval_list_kernel(DynRuns d, DynArgs a) {
    float* __restrict__ p = d.p[blockIdx.y];
    const float* __restrict__ g = d.g[blockIdx.y];
    const float* __restrict__ tg = d.tg[blockIdx.y];
    const float* __restrict__ r = d.r[blockIdx.y];
    const int64_t n = d.n[blockIdx.y];
    const float rbar = RMS ? *a.rbar : 0.f;
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
    int64_t j0 = 0;
    if (((((uintptr_t)p) | ((uintptr_t)g) | ((uintptr_t)tg) | (RMS ? (uintptr_t)r : 0)) & 15) == 0) {
        const int64_t n4 = n >> 2;
        for (int64_t i = tid; i < n4; i += stride) {
            float4 pv = __ldcs(reinterpret_cast<const float4*>(p) + i), gv = __ldcs(reinterpret_cast<const float4*>(g) + i);
            float4 tv = __ldcs(reinterpret_cast<const float4*>(tg) + i), rv = make_float4(0.f, 0.f, 0.f, 0.f);
            if (RMS) rv = __ldcs(reinterpret_cast<const float4*>(r) + i);
            pv.x = dyneval_elem<RMS>(pv.x, gv.x, tv.x, rv.x, a.lr, a.lam, a.eps, rbar);
            pv.y = dyneval_elem<RMS>(pv.y, gv.y, tv.y, rv.y, a.lr, a.lam, a.eps, rbar);
            pv.z = dyneval_elem<RMS>(pv.z, gv.z, tv.z, rv.z, a.lr, a.lam, a.eps, rbar);
            pv.w = dyneval_elem<RMS>(pv.w, gv.w, tv.w, rv.w, a.lr, a.lam, a.eps, rbar);
            __stcs(reinterpret_cast<float4*>(p) + i, pv);
        }
        j0 = n4 << 2;
    }
    for (int64_t j = j0 + tid; j < n; j += stride)
        p[j] = dyneval_elem<RMS>(p[j], g[j], tg[j], RMS ? r[j] : 0.f, a.lr, a.lam, a.eps, rbar);
}

int dyneval_apply(const TensorList& tl, float* const* tg, float* const* r, const DynArgs& a, cudaStream_t s) {
    DynRuns d;
    int bx = 1;
    const int k = dyn_runs(tl, tg, a.rbar ? r : nullptr, &d, &bx, kNormBlocks * 2);
    if (!k) return ZRB_OK;
    if (a.rbar) dyneval_list_kernel<true><<<dim3(bx, k), kThreads, 0, s>>>(d, a);
    else dyneval_list_kernel<false><<<dim3(bx, k), kThreads, 0, s>>>(d, a);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

// ms += g * g, one fma per element, one streaming pass
__global__ void sq_accumulate_kernel(DynRuns d) {
    float* __restrict__ ms = d.p[blockIdx.y];
    const float* __restrict__ g = d.g[blockIdx.y];
    const int64_t n = d.n[blockIdx.y];
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
    int64_t j0 = 0;
    if (((((uintptr_t)ms) | ((uintptr_t)g)) & 15) == 0) {
        const int64_t n4 = n >> 2;
        for (int64_t i = tid; i < n4; i += stride) {
            float4 m = __ldcs(reinterpret_cast<const float4*>(ms) + i), v = __ldcs(reinterpret_cast<const float4*>(g) + i);
            m.x = __fmaf_rn(v.x, v.x, m.x); m.y = __fmaf_rn(v.y, v.y, m.y);
            m.z = __fmaf_rn(v.z, v.z, m.z); m.w = __fmaf_rn(v.w, v.w, m.w);
            __stcs(reinterpret_cast<float4*>(ms) + i, m);
        }
        j0 = n4 << 2;
    }
    for (int64_t j = j0 + tid; j < n; j += stride) ms[j] = __fmaf_rn(g[j], g[j], ms[j]);
}

int sq_accumulate(const TensorList& tl, cudaStream_t s) {
    DynRuns d;
    int bx = 1;
    const int k = dyn_runs(tl, nullptr, nullptr, &d, &bx, kNormBlocks * 2);
    if (!k) return ZRB_OK;
    sq_accumulate_kernel<<<dim3(bx, k), kThreads, 0, s>>>(d);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

// block-wide fp64 sum in a fixed order (xor tree in each warp, then the warps' sums in index order)
__device__ __forceinline__ double block_sum_f64(double v, double* sh) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x == 0)
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += sh[w];
    return t;
}

// r = sqrt(ms / K) in place; partials[y * gridDim.x + x] = fp64 sum of the r this block wrote
__global__ void stats_sqrt_kernel(DynRuns d, float kf, double* __restrict__ partials) {
    __shared__ double sh[kThreads / 32];
    float* __restrict__ ms = d.p[blockIdx.y];
    const int64_t n = d.n[blockIdx.y];
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
    double acc = 0.0;
    for (int64_t j = tid; j < n; j += stride) {
        const float r = __fsqrt_rn(__fdiv_rn(ms[j], kf));
        ms[j] = r;
        acc += (double)r;
    }
    const double t = block_sum_f64(acc, sh);
    if (threadIdx.x == 0) partials[blockIdx.y * gridDim.x + blockIdx.x] = t;
}

// rbar = fp32(sum of the partials in a fixed order / P): one block
__global__ void stats_mean_kernel(const double* __restrict__ partials, int n, double P, float* __restrict__ rbar) {
    __shared__ double sh[kThreads / 32];
    double acc = 0.0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) acc += partials[i];
    const double t = block_sum_f64(acc, sh);
    if (threadIdx.x == 0) *rbar = (float)(t / P);
}

int stats_finish(const TensorList& tl, int64_t windows, double* partials, float* rbar, cudaStream_t s) {
    DynRuns d;
    int bx = 1;
    const int k = dyn_runs(tl, nullptr, nullptr, &d, &bx, kStatsPartials);
    int64_t P = 0;
    for (int i = 0; i < k; ++i) P += d.n[i];
    if (!k) return ZRB_OK;
    stats_sqrt_kernel<<<dim3(bx, k), kThreads, 0, s>>>(d, (float)windows, partials);
    ZRB_KERNEL_CHECK();
    stats_mean_kernel<<<1, kThreads, 0, s>>>(partials, bx * k, (double)P, rbar);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

}  // namespace zrb
