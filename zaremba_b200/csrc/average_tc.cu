// Iterate averaging (NT-ASGD, DESIGN.md section 16): the train step's SGD update with a running average of the
// weights streamed through the same pass, and the exchange of the weights with their average.
// The matrices go through the tile kernels of update_tile.cuh (one more stream: the average is loaded with g and p and
// stored with p; the fp16 images are rebuilt from registers as by the plain update); every tensor without an image
// through the list kernels below.
#include "update_tile.cuh"

namespace zrb {

// one element of the average after the update gave p: a copy at n = 1, else a + (p - a) * mu with mu = fp32(1 / n),
// in this fixed fp32 order (intrinsics, so that no kernel contracts it)
__device__ __forceinline__ float avg_elem(float a, float p, float mu, int first) {
    return first ? p : __fadd_rn(a, __fmul_rn(__fsub_rn(p, a), mu));
}

// SgdRule, then the average of the new p: a tile of the average rides with the tile of g and p
struct AvgRule : SgdRule {
    float* a;
    float mu;
    int first;
    // W_hh kernel: at most 168 registers.  The tile of the average adds 32 live values at 4 columns; bounded at 128,
    // ptxas spills in the 4-column instantiation.  3 blocks x 128 threads x 384 B = 144 KB of loads in flight per SM.
    static constexpr int kWhhMinBlocks = 3;
    template <int VEC> struct Tile { float v[kTileRows][VEC]; };
    template <int VEC> __device__ __forceinline__ void load(int64_t off, int e, Tile<VEC>& t) const {
        load_vec<VEC>(a + off, t.v[e]);
    }
    template <int VEC>
    __device__ __forceinline__ void finish(int e, float (&pv)[VEC], float (&)[VEC], Tile<VEC>& t) const {
#pragma unroll
        for (int x = 0; x < VEC; ++x) t.v[e][x] = avg_elem(t.v[e][x], pv[x], mu, first);
    }
    template <int VEC> __device__ __forceinline__ void store(int64_t off, int e, const Tile<VEC>& t) const {
        store_vec<VEC>(a + off, t.v[e]);
    }
};

// the kernels' g is the average: exchange it with p (both stored), images from the new p
struct SwapRule : NoTileRule {
    static constexpr bool kMayWriteG = true;
    // W_hh kernel: at most 128 registers (bounded at 102, ptxas spills in the 4-column instantiation: both old values
    // stay live until the stores)
    static constexpr int kWhhMinBlocks = 4;
    __device__ __forceinline__ void init() {}
    template <int VEC>
    __device__ __forceinline__ void apply(int64_t, float (&pv)[VEC], float (&gv)[VEC]) const {
#pragma unroll
        for (int x = 0; x < VEC; ++x) { const float t = pv[x]; pv[x] = gv[x]; gv[x] = t; }
    }
};

int update_pack_avg(float* p, float* g, float* a, float mu, bool first, int rows, int cols, float lr,
                    const float* scalars, const WeightImages& img, bool write_g, cudaStream_t s, int pdl_smem) {
    AvgRule rule;
    rule.lr = lr; rule.scalars = scalars; rule.coef = 0.f;
    rule.a = a; rule.mu = mu; rule.first = first ? 1 : 0;
    return update_pack_rule(p, g, rows, cols, rule, (uintptr_t)a, img, write_g, s, pdl_smem);
}

int swap_pack(float* p, float* a, int rows, int cols, const WeightImages& img, cudaStream_t s) {
    return update_pack_rule(p, a, rows, cols, SwapRule{}, 0, img, true, s, false);
}

// ---- tensors without an fp16 image (and every tensor on the validation engine / the unaligned fallback) ------------
// Block (x, y) streams share x of tensor y; no coalescing, so the averages need not be laid out like p.
constexpr int kListThreads = 256;
constexpr int kListBlocks = 148 * 16;

struct AvgRuns {
    float* p[kMaxTensors];
    float* g[kMaxTensors];
    float* a[kMaxTensors];
    int64_t n[kMaxTensors];
};

static int avg_runs(const TensorList& tl, float* const* a, AvgRuns* d, int* bx) {
    int k = 0;
    int64_t longest = 0;
    for (int t = 0; t < tl.count; ++t) {
        if (tl.n[t] == 0) continue;
        d->p[k] = tl.p[t]; d->g[k] = tl.g[t]; d->a[k] = a[t]; d->n[k] = tl.n[t];
        longest = tl.n[t] > longest ? tl.n[t] : longest;
        ++k;
    }
    int64_t b = (longest / 4 + kListThreads - 1) / kListThreads;
    if (b < 1) b = 1;
    const int cap = kListBlocks / (k > 0 ? k : 1);
    *bx = (int)(b > cap ? cap : b);
    return k;
}

// SGD: g *= coef; p = sgd_elem(p, g, lr) (clip_sgd's element rule), g stored back if WRITE_G; then the average of p.
// !SGD: the average of p only (p and g untouched: the embedding under the rows-only update).
template <bool SGD, bool WRITE_G>
__global__ void __launch_bounds__(kListThreads) sgd_avg_list_kernel(AvgRuns d, float lr, const float* __restrict__ scalars,
                                                                    float mu, int first) {
    float* __restrict__ p = d.p[blockIdx.y];
    float* __restrict__ g = d.g[blockIdx.y];
    float* __restrict__ a = d.a[blockIdx.y];
    const int64_t n = d.n[blockIdx.y];
    const float coef = SGD ? scalars[1] : 0.f;
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
    int64_t j0 = 0;
    if (((((uintptr_t)p) | ((uintptr_t)a) | (SGD ? (uintptr_t)g : 0)) & 15) == 0) {
        const int64_t n4 = n >> 2;
        for (int64_t i = tid; i < n4; i += stride) {
            float pv[4], av[4];
            load_vec<4>(p + 4 * i, pv);
            load_vec<4>(a + 4 * i, av);
            if constexpr (SGD) {
                float gv[4];
                load_vec<4>(g + 4 * i, gv);
#pragma unroll
                for (int x = 0; x < 4; ++x) { gv[x] *= coef; pv[x] = sgd_elem(pv[x], gv[x], lr); }
                if (WRITE_G) store_vec<4>(g + 4 * i, gv);
                store_vec<4>(p + 4 * i, pv);
            }
#pragma unroll
            for (int x = 0; x < 4; ++x) av[x] = avg_elem(av[x], pv[x], mu, first);
            store_vec<4>(a + 4 * i, av);
        }
        j0 = n4 << 2;
    }
    for (int64_t j = j0 + tid; j < n; j += stride) {
        float pv = p[j];
        if constexpr (SGD) {
            const float gv = g[j] * coef;
            if (WRITE_G) g[j] = gv;
            pv = sgd_elem(pv, gv, lr);
            p[j] = pv;
        }
        a[j] = avg_elem(a[j], pv, mu, first);
    }
}

__global__ void __launch_bounds__(kListThreads) swap_list_kernel(AvgRuns d) {
    float* __restrict__ p = d.p[blockIdx.y];
    float* __restrict__ a = d.a[blockIdx.y];
    const int64_t n = d.n[blockIdx.y];
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
    int64_t j0 = 0;
    if (((((uintptr_t)p) | ((uintptr_t)a)) & 15) == 0) {
        const int64_t n4 = n >> 2;
        for (int64_t i = tid; i < n4; i += stride) {
            float pv[4], av[4];
            load_vec<4>(p + 4 * i, pv);
            load_vec<4>(a + 4 * i, av);
            store_vec<4>(p + 4 * i, av);
            store_vec<4>(a + 4 * i, pv);
        }
        j0 = n4 << 2;
    }
    for (int64_t j = j0 + tid; j < n; j += stride) {
        const float t = p[j];
        p[j] = a[j];
        a[j] = t;
    }
}

int sgd_avg_apply(const TensorList& tl, float* const* a, float lr, const float* scalars, bool write_g, float mu,
                  bool first, cudaStream_t s) {
    AvgRuns d;
    int bx = 1;
    const int k = avg_runs(tl, a, &d, &bx);
    if (!k) return ZRB_OK;
    if (write_g) sgd_avg_list_kernel<true, true><<<dim3(bx, k), kListThreads, 0, s>>>(d, lr, scalars, mu, first ? 1 : 0);
    else sgd_avg_list_kernel<true, false><<<dim3(bx, k), kListThreads, 0, s>>>(d, lr, scalars, mu, first ? 1 : 0);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

int avg_apply(const TensorList& tl, float* const* a, float mu, bool first, cudaStream_t s) {
    AvgRuns d;
    int bx = 1;
    const int k = avg_runs(tl, a, &d, &bx);
    if (!k) return ZRB_OK;
    sgd_avg_list_kernel<false, false><<<dim3(bx, k), kListThreads, 0, s>>>(d, 0.f, nullptr, mu, first ? 1 : 0);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

int swap_apply(const TensorList& tl, float* const* a, cudaStream_t s) {
    AvgRuns d;
    int bx = 1;
    const int k = avg_runs(tl, a, &d, &bx);
    if (!k) return ZRB_OK;
    swap_list_kernel<<<dim3(bx, k), kListThreads, 0, s>>>(d);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

}  // namespace zrb
