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
#include "engine.h"
#include "select.cuh"

namespace zrb {

constexpr int kSampleThreads = kSelectThreads;
constexpr int kSampleSmemV = 4 * 512 * 8;            // rows up to softmax_nll_reg_kernel's register-path size stay on chip

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
