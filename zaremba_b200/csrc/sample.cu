// Sampler of the decode loop (zrb_sample, zrb_generate): one token per row of a [B,V] fp32 score matrix, one CTA per
// row, no host synchronisation.  Gumbel-max over a kept set (DESIGN.md section 9):
//   greedy   temperature == 0: argmax_j z_j, lowest index on ties, no uniforms drawn
//   top-k    keep z_j >= the k-th largest z (ties at the boundary kept)
//   top-p    over the top-k set, p = softmax(z / tau): keep z_j >= v*, v* the largest score whose set {z >= v*} holds
//            at least top_p of the mass (ties kept)
//   draw     argmax over kept j of z_j / tau + g_j, g_j = -log(-log u_j), u_j from sample_words (common.cuh)
//   logprob  log softmax(z)[token] at temperature 1 over the whole vocabulary
// Both thresholds are radix selects on the order-preserving integer key of z, most significant 8-bit digit first.  The
// histograms hold integers -- counts for top-k, masses in fixed point (multiples of 2^-36 of the largest entry's mass)
// for top-p -- so their shared-memory atomics give the same sums in any order, and every other reduction is a fixed
// shuffle tree: a run is bit-reproducible.
#include <climits>

#include "engine.h"

namespace zrb {

constexpr int kSampleThreads = 512;
constexpr int kSampleSmemV = 4 * 512 * 8;            // rows up to softmax_nll_reg_kernel's register-path size stay on chip
constexpr float kMassOne = 68719476736.f;            // 2^36: fixed-point mass of the row's largest entry

// order-preserving key: key(a) < key(b) iff a < b for finite floats (-0 and +0 share the key of +0)
__device__ __forceinline__ uint32_t order_key(float z) {
    const uint32_t u = __float_as_uint(z == 0.f ? 0.f : z);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

struct ArgMax {
    float v;
    int i;
};
__device__ __forceinline__ ArgMax better(ArgMax a, ArgMax b) {
    if (b.i == INT_MAX) return a;
    if (a.i == INT_MAX) return b;
    return (b.v > a.v || (b.v == a.v && b.i < a.i)) ? b : a;
}
__device__ __forceinline__ ArgMax warp_argmax(ArgMax a) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        ArgMax t;
        t.v = __shfl_xor_sync(0xffffffffu, a.v, o);
        t.i = __shfl_xor_sync(0xffffffffu, a.i, o);
        a = better(a, t);
    }
    return a;
}
// every thread gets the block's (max, lowest index of the max)
__device__ ArgMax block_argmax(ArgMax a, float* shv, int* shi) {
    a = warp_argmax(a);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) { shv[w] = a.v; shi[w] = a.i; }
    __syncthreads();
    a.v = l < kSampleThreads / 32 ? shv[l] : -INFINITY;
    a.i = l < kSampleThreads / 32 ? shi[l] : INT_MAX;
    return warp_argmax(a);
}
__device__ float block_sum(float v, float* sh) {
    v = warp_sum(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) sh[w] = v;
    __syncthreads();
    v = l < kSampleThreads / 32 ? sh[l] : 0.f;
    return warp_sum(v);
}

__device__ __forceinline__ unsigned long long mass_fx(float z, float m, float t) {
    return __float2ull_rn(expf((z - m) / t) * kMassOne);
}

// The largest key K such that the weight of {j : lo_key <= key_j, K <= key_j} reaches `target` (>= 1, <= the weight
// of the whole set).  kMass: weight = mass_fx, else 1.
template <bool kMass>
__device__ uint32_t select_from_top(const float* row, int V, uint32_t lo_key, float m, float t, unsigned long long target,
                                    unsigned long long* hist, uint32_t* s_sel, unsigned long long* s_above) {
    uint32_t prefix = 0, pmask = 0;
    unsigned long long above = 0;   // weight of the keys above the current prefix's bucket
    for (int pass = 0; pass < 4; ++pass) {
        const int shift = 24 - 8 * pass;
        if (threadIdx.x < 256) hist[threadIdx.x] = 0;
        __syncthreads();
        // Most entries share their leading digits, so the lanes of a warp that hit the same bin first add their weights
        // (__match_any_sync groups them; integer sums, any order) and one of them issues the atomic.  The trip count is
        // warp-uniform: the whole warp takes part in every match.
        const int lane = threadIdx.x & 31;
        for (int j0 = threadIdx.x - lane; j0 < V; j0 += kSampleThreads) {
            const int j = j0 + lane;
            uint32_t bin = 256u;   // none
            unsigned long long w = 0;
            if (j < V) {
                const float z = row[j];
                const uint32_t k = order_key(z);
                if (k >= lo_key && (k & pmask) == prefix) {
                    bin = (k >> shift) & 255u;
                    w = kMass ? mass_fx(z, m, t) : 1ull;
                }
            }
            const unsigned peers = __match_any_sync(0xffffffffu, bin);
            unsigned long long sum = __popc(peers);
            if (kMass)   // w <= 2^36: 32 lanes' high (12-bit) and low (24-bit) parts each sum inside 32 bits
                sum = ((unsigned long long)__reduce_add_sync(peers, (unsigned)(w >> 24)) << 24) +
                      __reduce_add_sync(peers, (unsigned)(w & 0xFFFFFFu));
            if (bin < 256u && lane == __ffs(peers) - 1) atomicAdd(&hist[bin], sum);
        }
        __syncthreads();
        if (threadIdx.x < 32) {   // lane l owns digits 255-8l .. 248-8l (descending); the crossing digit is selected
            const int lane = threadIdx.x;
            unsigned long long s = 0;
#pragma unroll
            for (int i = 0; i < 8; ++i) s += hist[255 - 8 * lane - i];
            unsigned long long incl = s;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned long long v = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += v;
            }
            unsigned long long c = above + (incl - s);
            if (c < target && above + incl >= target) {
                for (int i = 0; i < 8; ++i) {
                    const int bin = 255 - 8 * lane - i;
                    if (c + hist[bin] >= target) { *s_sel = (uint32_t)bin; *s_above = c; break; }
                    c += hist[bin];
                }
            }
        }
        __syncthreads();
        prefix |= *s_sel << shift;
        pmask |= 255u << shift;
        above = *s_above;
    }
    return prefix;
}

__global__ void __launch_bounds__(kSampleThreads) sample_kernel(const float* __restrict__ scores, int64_t ld, int V,
                                                                zrb_sampling cfg, SampleSrc key, bool on_chip,
                                                                int64_t* __restrict__ tokens,
                                                                float* __restrict__ logprobs) {
    extern __shared__ float s_row[];
    __shared__ unsigned long long hist[256];
    __shared__ float shv[32];
    __shared__ int shi[32];
    __shared__ uint32_t s_sel;
    __shared__ unsigned long long s_above, s_total;
    const int b = blockIdx.x;
    const float* row = scores + (int64_t)b * ld;
    if (on_chip) {
        for (int j = threadIdx.x; j < V; j += kSampleThreads) s_row[j] = row[j];
        __syncthreads();
        row = s_row;
    }
    ArgMax a = {-INFINITY, INT_MAX};
    for (int j = threadIdx.x; j < V; j += kSampleThreads) a = better(a, ArgMax{row[j], j});
    a = block_argmax(a, shv, shi);
    const float m = a.v;
    float sum = 0.f;
    if (logprobs) {
        for (int j = threadIdx.x; j < V; j += kSampleThreads) sum += expf(row[j] - m);
        sum = block_sum(sum, shv);
    }
    int tok = a.i;
    const float t = cfg.temperature;
    if (t > 0.f) {
        uint32_t lo_key = 0;
        if (cfg.top_k > 0 && cfg.top_k < V)
            lo_key = select_from_top<false>(row, V, 0, m, t, (unsigned long long)cfg.top_k, hist, &s_sel, &s_above);
        if (cfg.top_p < 1.f) {
            if (threadIdx.x == 0) s_total = 0;
            __syncthreads();
            unsigned long long mine = 0;
            for (int j = threadIdx.x; j < V; j += kSampleThreads) {
                const float z = row[j];
                if (order_key(z) >= lo_key) mine += mass_fx(z, m, t);
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
            if ((threadIdx.x & 31) == 0) atomicAdd(&s_total, mine);
            __syncthreads();
            double want = ceil((double)cfg.top_p * (double)s_total);
            const unsigned long long target = want < 1.0 ? 1ull : (unsigned long long)want;
            lo_key = select_from_top<true>(row, V, lo_key, m, t, target, hist, &s_sel, &s_above);
        }
        ArgMax d = {-INFINITY, INT_MAX};
        const int groups = (V + 3) >> 2;
        for (int g = threadIdx.x; g < groups; g += kSampleThreads) {
            const Philox4 r = sample_words(key, (uint32_t)g, (uint32_t)b);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int j = 4 * g + i;
                if (j < V) {
                    const float z = row[j];
                    if (order_key(z) >= lo_key) d = better(d, ArgMax{z / t + -logf(-logf(sample_uniform(r.v[i]))), j});
                }
            }
        }
        tok = block_argmax(d, shv, shi).i;
    }
    if (threadIdx.x == 0) {
        tokens[b] = tok;
        if (logprobs) logprobs[b] = row[tok] - m - logf(sum);
    }
}

int sample_check(const zrb_sampling* cfg, int B, int V) {
    ZRB_REQUIRE(cfg, "null sampling config");
    ZRB_REQUIRE(cfg->temperature >= 0.f, "temperature %f must be >= 0", cfg->temperature);
    ZRB_REQUIRE(cfg->top_p > 0.f, "top_p %f must be > 0", cfg->top_p);
    ZRB_REQUIRE(cfg->top_k >= 0, "top_k %d must be >= 0", cfg->top_k);
    ZRB_REQUIRE(B >= 1 && V >= 1, "B=%d and V=%d must be >= 1", B, V);
    ZRB_REQUIRE(V <= (1 << 27), "V=%d above 2^27: the fixed-point top-p masses could overflow", V);
    return ZRB_OK;
}

int sample_rows(const float* scores, int64_t ld, int B, int V, const zrb_sampling* cfg, uint64_t pos, int64_t* tokens,
                float* logprobs, cudaStream_t s) {
    ZRB_TRY(sample_check(cfg, B, V));
    ZRB_REQUIRE(scores && tokens, "null argument");
    ZRB_REQUIRE(ld >= V, "ld=%lld < V=%d", (long long)ld, V);
    static bool attr[64] = {};   // per device: function attributes belong to the device's context
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (!attr[dev]) {
        ZRB_CUDA(cudaFuncSetAttribute(sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      kSampleSmemV * (int)sizeof(float)));
        attr[dev] = true;
    }
    const bool on_chip = V <= kSampleSmemV;
    sample_kernel<<<B, kSampleThreads, on_chip ? (size_t)V * sizeof(float) : 0, s>>>(
        scores, ld, V, *cfg, make_sample_src(cfg->seed, pos), on_chip, tokens, logprobs);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

}  // namespace zrb
