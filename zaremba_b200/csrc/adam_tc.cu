// Adam in the train step's update (Kingma & Ba 2015; DESIGN.md section 21): the clipped gradient drives two moment
// streams, m and v, through the same pass as g and p.
// The matrices go through the tile kernels of update_tile.cuh (the moments are loaded with g and p and stored with p;
// the fp16 images are rebuilt from registers as by the SGD update); every tensor without an image -- the biases, the
// dense embedding, and every tensor on the validation engine or the unaligned fallback -- through the list kernel below.
#include "update_tile.cuh"

namespace zrb {

// One element of update t, in this fixed fp32 order (intrinsics, so that no kernel contracts it), with g' = coef * g:
//   m = b1 * m + omb1 * g';  v = b2 * v + omb2 * (g' * g');  denom = sqrt(v) / bc2s + eps;  p = p - step_size * (m / denom)
// (AdamScalars: step_size = fp32(lr / (1 - b1^t)), bc2s = fp32(sqrt(1 - b2^t)), omb1 = fp32(1 - b1), omb2 = fp32(1 - b2)).
// The ONE expression every kernel that applies Adam calls; g becomes g'.
__device__ __forceinline__ void adam_elem(float& p, float& g, float& m, float& v, float coef, const AdamScalars& k) {
    g = __fmul_rn(g, coef);
    m = __fadd_rn(__fmul_rn(k.beta1, m), __fmul_rn(k.omb1, g));
    v = __fadd_rn(__fmul_rn(k.beta2, v), __fmul_rn(k.omb2, __fmul_rn(g, g)));
    const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), k.bc2s), k.eps);
    p = __fsub_rn(p, __fmul_rn(k.step_size, __fdiv_rn(m, denom)));
}

// the tiles of m and v ride with the tiles of g and p.  The update needs all four, so it happens in finish(), the hook
// that sees the tile; apply() leaves p and g as loaded.
struct AdamRule : NoTileRule {
    float* m;
    float* v;
    AdamScalars k;
    const float* scalars;
    float coef;
    static constexpr bool kMayWriteG = true;
    // W_hh kernel: at most 168 registers.  The tiles of m and v add 64 live values at 4 columns to the 64 of g and p,
    // so the SGD bound (102) cannot hold them; ptxas (CUDA 12.9) gives the 4-column instantiation 164 with no spill.
    // 3 blocks x 128 threads x 512 B = 192 KB of loads in flight per SM.
    static constexpr int kWhhMinBlocks = 3;
    template <int VEC> struct Tile { float m[kTileRows][VEC], v[kTileRows][VEC]; };
    __device__ __forceinline__ void init() { coef = scalars[1]; }
    template <int VEC>
    __device__ __forceinline__ void apply(int64_t, float (&)[VEC], float (&)[VEC]) const {}
    template <int VEC> __device__ __forceinline__ void load(int64_t off, int e, Tile<VEC>& t) const {
        load_vec<VEC>(m + off, t.m[e]);
        load_vec<VEC>(v + off, t.v[e]);
    }
    template <int VEC>
    __device__ __forceinline__ void finish(int e, float (&pv)[VEC], float (&gv)[VEC], Tile<VEC>& t) const {
#pragma unroll
        for (int x = 0; x < VEC; ++x) adam_elem(pv[x], gv[x], t.m[e][x], t.v[e][x], coef, k);
    }
    template <int VEC> __device__ __forceinline__ void store(int64_t off, int e, const Tile<VEC>& t) const {
        store_vec<VEC>(m + off, t.m[e]);
        store_vec<VEC>(v + off, t.v[e]);
    }
};

int update_pack_adam(float* p, float* g, float* m, float* v, const AdamScalars& k, int rows, int cols,
                     const float* scalars, const WeightImages& img, bool write_g, cudaStream_t s, int pdl_smem) {
    AdamRule rule;
    rule.m = m; rule.v = v; rule.k = k; rule.scalars = scalars; rule.coef = 0.f;
    return update_pack_rule(p, g, rows, cols, rule, (uintptr_t)m | (uintptr_t)v, img, write_g, s, pdl_smem);
}

// ---- tensors without an fp16 image (and every tensor on the validation engine / the unaligned fallback) ------------
// Block (x, y) streams share x of tensor y, as the averaging list kernels do.
constexpr int kAdamListThreads = 256;
constexpr int kAdamListBlocks = 148 * 16;

struct AdamRuns {
    float* p[kMaxTensors];
    float* g[kMaxTensors];
    float* m[kMaxTensors];
    float* v[kMaxTensors];
    int64_t n[kMaxTensors];
};

template <bool WRITE_G>
__global__ void __launch_bounds__(kAdamListThreads) adam_list_kernel(AdamRuns d, AdamScalars k,
                                                                     const float* __restrict__ scalars) {
    float* __restrict__ p = d.p[blockIdx.y];
    float* __restrict__ g = d.g[blockIdx.y];
    float* __restrict__ m = d.m[blockIdx.y];
    float* __restrict__ v = d.v[blockIdx.y];
    const int64_t n = d.n[blockIdx.y];
    const float coef = scalars[1];
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
    int64_t j0 = 0;
    if (((((uintptr_t)p) | ((uintptr_t)g) | ((uintptr_t)m) | ((uintptr_t)v)) & 15) == 0) {
        const int64_t n4 = n >> 2;
        for (int64_t i = tid; i < n4; i += stride) {
            float pv[4], gv[4], mv[4], vv[4];
            load_vec<4>(g + 4 * i, gv);
            load_vec<4>(p + 4 * i, pv);
            load_vec<4>(m + 4 * i, mv);
            load_vec<4>(v + 4 * i, vv);
#pragma unroll
            for (int x = 0; x < 4; ++x) adam_elem(pv[x], gv[x], mv[x], vv[x], coef, k);
            if (WRITE_G) store_vec<4>(g + 4 * i, gv);
            store_vec<4>(p + 4 * i, pv);
            store_vec<4>(m + 4 * i, mv);
            store_vec<4>(v + 4 * i, vv);
        }
        j0 = n4 << 2;
    }
    for (int64_t j = j0 + tid; j < n; j += stride) {
        float pv = p[j], gv = g[j], mv = m[j], vv = v[j];
        adam_elem(pv, gv, mv, vv, coef, k);
        if (WRITE_G) g[j] = gv;
        p[j] = pv;
        m[j] = mv;
        v[j] = vv;
    }
}

int adam_apply(const TensorList& tl, const AdamStep& a, const float* scalars, bool write_g, cudaStream_t s) {
    AdamRuns d;
    int k = 0;
    int64_t longest = 0;
    for (int t = 0; t < tl.count; ++t) {
        if (tl.n[t] == 0) continue;
        d.p[k] = tl.p[t]; d.g[k] = tl.g[t]; d.m[k] = a.m[t]; d.v[k] = a.v[t]; d.n[k] = tl.n[t];
        longest = tl.n[t] > longest ? tl.n[t] : longest;
        ++k;
    }
    if (!k) return ZRB_OK;
    int64_t b = (longest / 4 + kAdamListThreads - 1) / kAdamListThreads;
    if (b < 1) b = 1;
    const int cap = kAdamListBlocks / k;
    const dim3 grid((unsigned)(b > cap ? cap : b), (unsigned)k);
    if (write_g) adam_list_kernel<true><<<grid, kAdamListThreads, 0, s>>>(d, a.k, scalars);
    else adam_list_kernel<false><<<grid, kAdamListThreads, 0, s>>>(d, a.k, scalars);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

}  // namespace zrb
