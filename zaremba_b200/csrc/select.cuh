// Block-level selection helpers shared by the sampler (sample.cu) and the beam search (beam.cu): fixed-order
// reductions and the radix select on the order-preserving key of a float.  Every block using them has kSelectThreads
// threads.
#pragma once
#include <climits>

#include "common.cuh"

namespace zrb {

constexpr int kSelectThreads = 512;
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
__device__ inline ArgMax block_argmax(ArgMax a, float* shv, int* shi) {
    a = warp_argmax(a);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) { shv[w] = a.v; shi[w] = a.i; }
    __syncthreads();
    a.v = l < kSelectThreads / 32 ? shv[l] : -INFINITY;
    a.i = l < kSelectThreads / 32 ? shi[l] : INT_MAX;
    return warp_argmax(a);
}
__device__ inline float block_sum(float v, float* sh) {
    v = warp_sum(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) sh[w] = v;
    __syncthreads();
    v = l < kSelectThreads / 32 ? sh[l] : 0.f;
    return warp_sum(v);
}

__device__ __forceinline__ unsigned long long mass_fx(float z, float m, float t) {
    return __float2ull_rn(expf((z - m) / t) * kMassOne);
}

// The largest key K such that the weight of {j : lo_key <= key_j, K <= key_j} reaches `target` (>= 1, <= the weight
// of the whole set).  kMass: weight = mass_fx, else 1.  `row[j]` is the value of entry j: a pointer, or a functor that
// computes it.  On return *s_above holds the weight of {j : lo_key <= key_j, K < key_j}.
template <bool kMass, typename Row>
__device__ uint32_t select_from_top(const Row& row, int V, uint32_t lo_key, float m, float t, unsigned long long target,
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
        for (int j0 = threadIdx.x - lane; j0 < V; j0 += kSelectThreads) {
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

}  // namespace zrb
