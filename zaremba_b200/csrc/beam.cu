// Beam search of the decode loop (zrb_beam_step, zrb_beam_search; DESIGN.md section 10), no host synchronisation.
// One selection step over B prompts with K_in live rows each (row b*K_in + i is slot i of prompt b):
//   row r     m = max z, L = logf(sum expf(z_j - m)) (the sampler's reductions), logp_j = (z_j - m) - L,
//             cand_j = S_r + logp_j; a finished row (last token == eos) has the one candidate j = eos, logp 0, cand S_r
//   order     cand descending, then flat index i*V + j ascending
//   select    the K best of a prompt become its slots 0..K-1 in that order (parent i, token j, S = cand, logp)
// beam_row_kernel (one CTA per row) keeps each row's own K best under that order: a radix select on the
// order-preserving key of cand gives the K-th largest key, then every key above it and the ties at it in index order
// up to K.  The K best of a prompt are among the K best of its rows, so the two stages are exact.  beam_merge_kernel
// ranks a prompt's <= K_in*K survivors, writes the step's outputs and gathers the chosen parents' (h, c).
#include <algorithm>

#include "engine.h"
#include "select.cuh"

namespace zrb {

constexpr int kBeamSmemV = 4 * 512 * 8;   // rows up to this size are read from shared memory, longer ones from global
constexpr int kMergeThreads = 512;
constexpr uint32_t kNoCand = 0xFFFFFFFFu;   // flat index of an empty candidate slot (finished rows fill one of K)

// entry j of row r's candidates, computed where it is read
struct CandRow {
    const float* z;
    float m, L, S;
    __device__ __forceinline__ float logp(int j) const { return (z[j] - m) - L; }
    __device__ __forceinline__ float operator[](int j) const { return S + logp(j); }
};

__global__ void __launch_bounds__(kSelectThreads) beam_row_kernel(const float* __restrict__ scores, int64_t ld, int V,
                                                                  int K_in, int K, const float* __restrict__ cum_in,
                                                                  const int64_t* __restrict__ tok_in, int eos,
                                                                  bool on_chip, BeamCand* __restrict__ cands) {
    extern __shared__ float s_row[];
    __shared__ unsigned long long hist[256];
    __shared__ float shv[32];
    __shared__ int shi[32];
    __shared__ uint32_t s_sel;
    __shared__ unsigned long long s_above;
    __shared__ int s_na[kSelectThreads / 32], s_nt[kSelectThreads / 32];
    const int r = blockIdx.x, i = r % K_in;
    BeamCand* out = cands + (size_t)r * K;
    const float S = cum_in ? cum_in[r] : 0.f;
    if (tok_in && eos >= 0 && tok_in[r] == eos) {
        for (int e = threadIdx.x; e < K; e += kSelectThreads)
            out[e] = e == 0 ? BeamCand{S, 0.f, (uint32_t)i * (uint32_t)V + (uint32_t)eos} : BeamCand{-INFINITY, 0.f, kNoCand};
        return;
    }
    const float* row = scores + (int64_t)r * ld;
    if (on_chip) {
        for (int j = threadIdx.x; j < V; j += kSelectThreads) s_row[j] = row[j];
        __syncthreads();
        row = s_row;
    }
    // m and L exactly as sample_kernel computes them, so logp is bit-identical to zrb_sample's logprob
    ArgMax a = {-INFINITY, INT_MAX};
    for (int j = threadIdx.x; j < V; j += kSelectThreads) a = better(a, ArgMax{row[j], j});
    a = block_argmax(a, shv, shi);
    const float m = a.v;
    float sum = 0.f;
    for (int j = threadIdx.x; j < V; j += kSelectThreads) sum += expf(row[j] - m);
    sum = block_sum(sum, shv);
    const CandRow cr{row, m, logf(sum), S};
    const uint32_t thr = select_from_top<false>(cr, V, 0u, 0.f, 1.f, (unsigned long long)K, hist, &s_sel, &s_above);
    const int n_above = (int)s_above, n_ties = K - n_above;   // keys above the K-th largest, and ties of it to take
    // compaction in index order, 512 entries per round: above-threshold entries to slots [0, n_above), the first
    // n_ties ties to [n_above, K).  The counts are block-uniform, so the loop stops together once both are in.
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int base_a = 0, base_t = 0;
    for (int j0 = 0; j0 < V && (base_a < n_above || base_t < n_ties); j0 += kSelectThreads) {
        const int j = j0 + threadIdx.x;
        const uint32_t key = j < V ? order_key(cr[j]) : 0u;
        const bool above = j < V && key > thr, tie = j < V && key == thr;
        const unsigned ba = __ballot_sync(0xffffffffu, above), bt = __ballot_sync(0xffffffffu, tie);
        if (lane == 0) { s_na[w] = __popc(ba); s_nt[w] = __popc(bt); }
        __syncthreads();
        int pa = base_a, pt = base_t;
#pragma unroll
        for (int q = 0; q < kSelectThreads / 32; ++q) {
            if (q < w) { pa += s_na[q]; pt += s_nt[q]; }
            base_a += s_na[q];
            base_t += s_nt[q];
        }
        const unsigned lt = (1u << lane) - 1u;
        pa += __popc(ba & lt);
        pt += __popc(bt & lt);
        if (above || (tie && pt < n_ties)) {
            const float lp = cr.logp(j);
            out[above ? pa : n_above + pt] = BeamCand{S + lp, lp, (uint32_t)i * (uint32_t)V + (uint32_t)j};
        }
        __syncthreads();
    }
}

// grid (B, gy): every CTA of prompt b ranks its candidates; CTA (b, 0) writes the step's outputs, and the gy CTAs
// share the gather of the 2*L*K state rows (L = 0: no gather)
__global__ void __launch_bounds__(kMergeThreads) beam_merge_kernel(const BeamCand* __restrict__ cands, int K_in, int K,
                                                                   int V, int64_t* __restrict__ tokens,
                                                                   int32_t* __restrict__ parents, float* cum_out,
                                                                   float* __restrict__ logprobs, zrb_states src,
                                                                   zrb_states dst, int L, LayerWidths w) {
    __shared__ unsigned long long s_key[ZRB_MAX_BEAMS * ZRB_MAX_BEAMS];
    __shared__ int s_pick[ZRB_MAX_BEAMS];
    __shared__ const float* s_src[2 * ZRB_MAX_LAYERS];   // (h, c) of layer l at 2l, 2l+1: constant indices into the
    __shared__ float* s_dst[2 * ZRB_MAX_LAYERS];         // kernel parameters, so they stay out of local memory
    __shared__ int s_h[ZRB_MAX_LAYERS];                  // (the width of layer l, likewise)
    if (threadIdx.x == 0) {
#pragma unroll
        for (int l = 0; l < ZRB_MAX_LAYERS; ++l) {
            s_src[2 * l] = src.h[l]; s_src[2 * l + 1] = src.c[l];
            s_dst[2 * l] = dst.h[l]; s_dst[2 * l + 1] = dst.c[l];
            s_h[l] = w.h[l];
        }
    }
    const int b = blockIdx.x, n = K_in * K;
    const BeamCand* cb = cands + (size_t)b * n;
    // (order key of cand, bitwise NOT of the flat index) as one 64-bit key: larger is better, unique per candidate;
    // 0 for an empty slot (the order key of a finite float is at least 2^23)
    for (int e = threadIdx.x; e < n; e += kMergeThreads) {
        const BeamCand x = cb[e];
        s_key[e] = x.flat == kNoCand ? 0ull : ((unsigned long long)order_key(x.cand) << 32) | (uint32_t)~x.flat;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < n; e += kMergeThreads) {
        const unsigned long long k = s_key[e];
        if (k == 0ull) continue;
        int rank = 0;
        for (int f = 0; f < n; ++f) rank += s_key[f] > k;
        if (rank < K) s_pick[rank] = e;
    }
    __syncthreads();
    if (blockIdx.y == 0 && threadIdx.x < K) {
        const BeamCand x = cb[s_pick[threadIdx.x]];
        const int r = b * K + threadIdx.x;
        tokens[r] = (int64_t)(x.flat % (uint32_t)V);
        parents[r] = (int32_t)(x.flat / (uint32_t)V);
        cum_out[r] = x.cand;
        logprobs[r] = x.logp;
    }
    // row q = ((l, h or c), k'): dst row b*K + k' <- src row b*K_in + parent(k')
    for (int q = blockIdx.y; q < 2 * L * K; q += gridDim.y) {
        const int lhc = q / K, k = q % K, H = s_h[lhc >> 1];
        const int par = (int)(cb[s_pick[k]].flat / (uint32_t)V);
        const float* s = s_src[lhc] + ((size_t)b * K_in + par) * H;
        float* d = s_dst[lhc] + ((size_t)b * K + k) * H;
        for (int u = threadIdx.x; u < H; u += kMergeThreads) d[u] = s[u];
    }
}

// thread r = b*K + k follows final slot k of prompt b back through the parents
__global__ void beam_backtrack_kernel(const int64_t* __restrict__ step_tok, const int32_t* __restrict__ step_par,
                                      const float* __restrict__ step_lp, const float* __restrict__ cum, int n_new,
                                      int BK, int K, int64_t* __restrict__ tokens, float* __restrict__ logprobs,
                                      float* __restrict__ scores) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= BK) return;
    const int base = r - r % K;
    int slot = r % K;
    for (int t = n_new - 1; t >= 0; --t) {
        const size_t at = (size_t)t * BK + base + slot;
        tokens[(size_t)t * BK + r] = step_tok[at];
        if (logprobs) logprobs[(size_t)t * BK + r] = step_lp[at];
        slot = step_par[at];
    }
    if (scores) scores[r] = cum[r];
}

int beam_check(int B, int K, int V, int eos) {
    ZRB_REQUIRE(B >= 1 && V >= 1, "B=%d and V=%d must be >= 1", B, V);
    ZRB_REQUIRE(V <= (1 << 26), "V=%d above 2^26: flat candidate indices i*V + j must fit 32 bits", V);
    ZRB_REQUIRE(K >= 1 && K <= ZRB_MAX_BEAMS && K <= V, "beam width K=%d outside [1, min(%d, V=%d)]", K, ZRB_MAX_BEAMS,
                V);
    ZRB_REQUIRE(eos >= -1 && eos < V, "eos=%d outside [-1, V=%d)", eos, V);
    return ZRB_OK;
}

int beam_step(const float* scores, int64_t ld, int B, int K_in, int K, int V, const float* cum_in, const int64_t* tok_in,
              int eos, BeamCand* cands, int64_t* tokens, int32_t* parents, float* cum_out, float* logprobs,
              const zrb_states* src, const zrb_states* dst, int L, const LayerWidths& w, cudaStream_t s) {
    ZRB_TRY(beam_check(B, K, V, eos));
    // a step-0 row is never finished, so every step has at least K candidates per prompt
    ZRB_REQUIRE(K_in == K || (K_in == 1 && !tok_in), "K_in=%d must be K=%d, or 1 without tok_in (step 0)", K_in, K);
    ZRB_REQUIRE(scores && cands && tokens && parents && cum_out && logprobs, "null argument");
    ZRB_REQUIRE(ld >= V, "ld=%lld < V=%d", (long long)ld, V);
    static bool attr[64] = {};   // per device: function attributes belong to the device's context
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (!attr[dev]) {
        ZRB_CUDA(cudaFuncSetAttribute(beam_row_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      kBeamSmemV * (int)sizeof(float)));
        attr[dev] = true;
    }
    const bool on_chip = V <= kBeamSmemV;
    beam_row_kernel<<<B * K_in, kSelectThreads, on_chip ? (size_t)V * sizeof(float) : 0, s>>>(
        scores, ld, V, K_in, K, cum_in, tok_in, eos, on_chip, cands);
    ZRB_KERNEL_CHECK();
    // the gather is split over ~128 CTAs in all: at B = 1 one CTA alone would move K*L*2*H floats
    const int gy = L ? std::max(1, std::min(2 * L * K, 128 / B)) : 1;
    const zrb_states none = {};
    beam_merge_kernel<<<dim3(B, gy), kMergeThreads, 0, s>>>(cands, K_in, K, V, tokens, parents, cum_out, logprobs,
                                                            src ? *src : none, dst ? *dst : none, L, w);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

int beam_backtrack(const int64_t* step_tok, const int32_t* step_par, const float* step_lp, const float* cum, int n_new,
                   int BK, int K, int64_t* tokens, float* logprobs, float* scores, cudaStream_t s) {
    beam_backtrack_kernel<<<cdiv(BK, 128), 128, 0, s>>>(step_tok, step_par, step_lp, cum, n_new, BK, K, tokens, logprobs,
                                                        scores);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

}  // namespace zrb
