// Mixture of Softmaxes head (Yang et al. 2018; DESIGN.md section 19): the pointwise latent kernels and the mixture
// kernels that read the N*K logits rows the projection GEMM wrote.  Rows are token-major: logits row n*K + k is expert k
// of token n.  The prior scores a_n sit in columns [Ua, Ua + K) of the head GEMM's output row n, the latent in [0, K*E).
#include <math.h>

#include "tc_kernels.h"

namespace zrb {

namespace {

constexpr int kMosThreads = 256;

// lane k < K: log softmax_k(v); -inf on the other lanes
__device__ __forceinline__ float warp_log_softmax(float v, int K, int lane) {
    v = lane < K ? v : -INFINITY;
    const float m = warp_max(v);
    const float s = warp_sum(lane < K ? expf(v - m) : 0.f);
    return v - m - logf(s);
}
// logsumexp over the lanes (every lane gets it); t = -inf on lanes that take no part
__device__ __forceinline__ float warp_logsumexp(float t) {
    const float m = warp_max(t);
    return m + logf(warp_sum(t == -INFINITY ? 0.f : expf(t - m)));
}

// warp 0 of a block: log pi and the LSEs of token n into shared memory (lanes < K)
__device__ __forceinline__ void token_prior(const float* __restrict__ ua, int64_t ldu, int Ua, const float* __restrict__ lse,
                                            int64_t n, int K, float* lpi, float* lk) {
    const int lane = threadIdx.x;
    const float a = lane < K ? ua[n * ldu + Ua + lane] : 0.f;
    const float lp = warp_log_softmax(a, K, lane);
    if (lane < K) {
        lpi[lane] = lp;
        lk[lane] = lse[n * K + lane];
    }
}

// u + b -> c = tanh(u) (kept in ua for the backward), and the fp16 latent image row r*K + k, column e: c * mask
__global__ void mos_latent_fwd_kernel(float* __restrict__ ua, int64_t ldu, const float* __restrict__ b,
                                      __half* __restrict__ lat_h, int64_t ld_l, int rows, int K, int E, int64_t row0,
                                      MaskSrc m) {
    const int KE = K * E;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)rows * KE) return;
    const int64_t r = i / KE;
    const int j = (int)(i - r * KE), k = j / E, e = j - k * E;
    const float c = tanhf(ua[r * ldu + j] + b[j]);
    ua[r * ldu + j] = c;
    const float mul = mask_mul1(m, (uint64_t)(row0 + r) * KE + j, ~0ull);
    lat_h[(r * K + k) * ld_l + e] = __float2half_rn(c * mul);
}

// du = dc^ * mask * (1 - c^2), written kGradScale-scaled into columns [0, K*E) of the gradient image
__global__ void mos_latent_bwd_kernel(const float* __restrict__ dlat, const float* __restrict__ ua, int64_t ldu,
                                      __half* __restrict__ dua_h, int64_t ld_d, int N, int K, int E, MaskSrc m) {
    const int KE = K * E;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)N * KE) return;
    const int64_t n = i / KE;
    const int j = (int)(i - n * KE), k = j / E, e = j - k * E;
    const float c = ua[n * ldu + j];
    const float mul = mask_mul1(m, (uint64_t)n * KE + j, ~0ull);
    const float du = dlat[(n * K + k) * E + e] * mul * (1.f - c * c);
    dua_h[n * ld_d + j] = __float2half_rn(kGradScale * du);
}

// LSE of every logits row (one CTA per row, online max / sum; VEC: V % 4 == 0, 16-byte loads, one rescale per quad)
template <bool VEC>
__global__ void __launch_bounds__(kMosThreads) mos_lse_kernel(const float* __restrict__ Z, int V, float* __restrict__ lse) {
    const float* z = Z + (int64_t)blockIdx.x * V;
    float m = -INFINITY, s = 0.f;
    if (VEC) {
        for (int v = 4 * threadIdx.x; v < V; v += 4 * blockDim.x) {
            const float4 x = *reinterpret_cast<const float4*>(z + v);
            const float mx = fmaxf(fmaxf(x.x, x.y), fmaxf(x.z, x.w));
            if (mx > m) {
                s = m == -INFINITY ? 0.f : s * expf(m - mx);
                m = mx;
            }
            s += expf(x.x - m) + expf(x.y - m) + expf(x.z - m) + expf(x.w - m);
        }
    } else {
        for (int v = threadIdx.x; v < V; v += blockDim.x) {
            const float x = z[v];
            if (x > m) {
                s = s * expf(m - x) + 1.f;
                m = x;
            } else {
                s += expf(x - m);
            }
        }
    }
    __shared__ float sm[kMosThreads / 32], ss[kMosThreads / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
        const float mm = fmaxf(m, m2);
        s = (m == -INFINITY ? 0.f : s * expf(m - mm)) + (m2 == -INFINITY ? 0.f : s2 * expf(m2 - mm));
        m = mm;
    }
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { sm[w] = m; ss[w] = s; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float M = sm[0];
        for (int i = 1; i < kMosThreads / 32; ++i) M = fmaxf(M, sm[i]);
        float S = 0.f;
        for (int i = 0; i < kMosThreads / 32; ++i) S += sm[i] == -INFINITY ? 0.f : ss[i] * expf(sm[i] - M);
        lse[blockIdx.x] = M + logf(S);
    }
}

// the train step's mixture NLL and its gradient, one CTA per logits row (n, k): warp 0 forms log pi, log p[y] and
// r_k = pi_k q_k[y] / p[y] from the token's K statistics; the CTA writes the scaled fp16 row g r_k (q_k - onehot(y)).
// The CTA of k = 0 writes the row loss and da = g (pi - r).
template <bool VEC>
__global__ void __launch_bounds__(kMosThreads) mos_nll_grad_kernel(
    const float* __restrict__ Z, const float* __restrict__ lse, const float* __restrict__ ua, int64_t ldu, int Ua,
    const int64_t* __restrict__ y, int K, int V, float g, float* __restrict__ row_loss, __half* __restrict__ ds_h,
    int64_t ld_s, __half* __restrict__ dua_h, int64_t ld_d) {
    const int64_t row = blockIdx.x, n = row / K;
    const int k = (int)(row - n * K);
    const int64_t yn = y[n];
    __shared__ float sh_r, sh_l;
    if (threadIdx.x < 32) {
        const int lane = threadIdx.x;
        const float a = lane < K ? ua[n * ldu + Ua + lane] : 0.f;
        const float lp = warp_log_softmax(a, K, lane);
        const float lk = lane < K ? lse[n * K + lane] : 0.f;
        const float t = lane < K ? lp + Z[(n * K + lane) * V + yn] - lk : -INFINITY;
        const float logp = warp_logsumexp(t);
        const float r = lane < K ? expf(t - logp) : 0.f;
        if (lane == k) { sh_r = r; sh_l = lk; }
        if (k == 0) {
            if (lane < K) dua_h[n * ld_d + Ua + lane] = __float2half_rn(kGradScale * (g * (expf(lp) - r)));
            if (lane == 0) row_loss[n] = -logp;
        }
    }
    __syncthreads();
    const float rs = kGradScale * (g * sh_r), l = sh_l;
    const float* z = Z + row * V;
    __half* d = ds_h + row * ld_s;
    if (VEC) {   // V % 4 == 0: 16-byte loads, 8-byte stores
        for (int v = 4 * threadIdx.x; v < V; v += 4 * blockDim.x) {
            const float4 x = *reinterpret_cast<const float4*>(z + v);
            const float q0 = expf(x.x - l) - (v == yn), q1 = expf(x.y - l) - (v + 1 == yn);
            const float q2 = expf(x.z - l) - (v + 2 == yn), q3 = expf(x.w - l) - (v + 3 == yn);
            __half2 h[2] = {__floats2half2_rn(rs * q0, rs * q1), __floats2half2_rn(rs * q2, rs * q3)};
            *reinterpret_cast<uint2*>(d + v) = *reinterpret_cast<uint2*>(h);
        }
    } else {
        for (int v = threadIdx.x; v < V; v += blockDim.x) d[v] = __float2half_rn(rs * (expf(z[v] - l) - (v == yn)));
    }
}

// eval mode: row loss -log p[y] and (or null) p[y], one warp per token
__global__ void mos_nll_eval_kernel(const float* __restrict__ Z, const float* __restrict__ lse, const float* __restrict__ ua,
                                    int64_t ldu, int Ua, const int64_t* __restrict__ y, int K, int V,
                                    float* __restrict__ row_loss, float* __restrict__ tgt_prob) {
    const int64_t n = blockIdx.x;
    const int lane = threadIdx.x;
    const int64_t yn = y[n];
    const float a = lane < K ? ua[n * ldu + Ua + lane] : 0.f;
    const float lp = warp_log_softmax(a, K, lane);
    const float t = lane < K ? lp + Z[(n * K + lane) * V + yn] - lse[n * K + lane] : -INFINITY;
    const float logp = warp_logsumexp(t);
    if (lane == 0) {
        row_loss[n] = -logp;
        if (tgt_prob) tgt_prob[n] = expf(logp);
    }
}

// log p of token r at entry v: logsumexp_k(log pi_k + z_k[v] - LSE_k), two passes over the K rows
__device__ __forceinline__ float mix_logp(const float* __restrict__ Z, int64_t r, int K, int V, int v, const float* lpi,
                                          const float* lk) {
    float mx = -INFINITY;
    for (int k = 0; k < K; ++k) mx = fmaxf(mx, lpi[k] + Z[(r * K + k) * V + v] - lk[k]);
    float s = 0.f;
    for (int k = 0; k < K; ++k) s += expf(lpi[k] + Z[(r * K + k) * V + v] - lk[k] - mx);
    return mx + logf(s);
}

// out [rows, ldo] = log p, one CTA per token
__global__ void __launch_bounds__(kMosThreads) mos_logp_kernel(const float* __restrict__ Z, const float* __restrict__ lse,
                                                               const float* __restrict__ ua, int64_t ldu, int Ua, int K,
                                                               int V, float* __restrict__ out, int64_t ldo) {
    __shared__ float lpi[32], lk[32];
    const int64_t r = blockIdx.x;
    if (threadIdx.x < 32) token_prior(ua, ldu, Ua, lse, r, K, lpi, lk);
    __syncthreads();
    for (int v = threadIdx.x; v < V; v += blockDim.x) out[r * ldo + v] = mix_logp(Z, r, K, V, v, lpi, lk);
}

// the drop-in backward, pass 1 (one CTA per token): log p into P, s_k = sum_v G_v rho_kv into s, and
// da_k = s_k - pi_k sum_v G_v (scaled fp16) into the gradient image
__global__ void __launch_bounds__(kMosThreads) mos_vjp_token_kernel(
    const float* __restrict__ Z, const float* __restrict__ lse, const float* __restrict__ ua, int64_t ldu, int Ua, int K,
    int V, const float* __restrict__ G, float* __restrict__ P, float* __restrict__ s_out, __half* __restrict__ dua_h,
    int64_t ld_d) {
    __shared__ float lpi[32], lk[32], red[kMosThreads / 32][ZRB_MAX_EXPERTS + 1];
    const int64_t n = blockIdx.x;
    if (threadIdx.x < 32) token_prior(ua, ldu, Ua, lse, n, K, lpi, lk);
    __syncthreads();
    float acc[ZRB_MAX_EXPERTS + 1];
#pragma unroll
    for (int k = 0; k <= ZRB_MAX_EXPERTS; ++k) acc[k] = 0.f;
    for (int v = threadIdx.x; v < V; v += blockDim.x) {
        const float lp = mix_logp(Z, n, K, V, v, lpi, lk);
        const float gv = G[n * V + v];
        P[n * V + v] = lp;
        acc[ZRB_MAX_EXPERTS] += gv;
#pragma unroll
        for (int k = 0; k < ZRB_MAX_EXPERTS; ++k)
            if (k < K) acc[k] += gv * expf(lpi[k] + Z[(n * K + k) * V + v] - lk[k] - lp);
    }
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int k = 0; k <= ZRB_MAX_EXPERTS; ++k) {
        const float t = warp_sum(acc[k]);
        if (lane == 0) red[w][k] = t;
    }
    __syncthreads();
    if (threadIdx.x < K) {
        const int k = threadIdx.x;
        float sk = 0.f, sg = 0.f;
        for (int i = 0; i < kMosThreads / 32; ++i) { sk += red[i][k]; sg += red[i][ZRB_MAX_EXPERTS]; }
        s_out[n * K + k] = sk;
        dua_h[n * ld_d + Ua + k] = __float2half_rn(kGradScale * (sk - expf(lpi[k]) * sg));
    }
}

// pass 2 (one CTA per logits row n*K + k): dz_v = rho_kv G_v - q_kv s_k, scaled fp16
__global__ void __launch_bounds__(kMosThreads) mos_vjp_dz_kernel(
    const float* __restrict__ Z, const float* __restrict__ lse, const float* __restrict__ ua, int64_t ldu, int Ua, int K,
    int V, const float* __restrict__ G, const float* __restrict__ P, const float* __restrict__ s_in,
    __half* __restrict__ ds_h, int64_t ld_s) {
    __shared__ float lpi[32], lk[32];
    const int64_t row = blockIdx.x, n = row / K;
    const int k = (int)(row - n * K);
    if (threadIdx.x < 32) token_prior(ua, ldu, Ua, lse, n, K, lpi, lk);
    __syncthreads();
    const float l = lk[k], lp = lpi[k], sk = s_in[row];
    const float* z = Z + row * V;
    for (int v = threadIdx.x; v < V; v += blockDim.x) {
        const float q = expf(z[v] - l), rho = expf(lp + z[v] - l - P[n * V + v]);
        ds_h[row * ld_s + v] = __float2half_rn(kGradScale * (rho * G[n * V + v] - q * sk));
    }
}

}  // namespace

int mos_latent_fwd(float* ua, int64_t ldu, const float* b, __half* lat_h, int64_t ld_l, int rows, int K, int E,
                   int64_t row0, MaskSrc m, cudaStream_t s) {
    const int64_t n = (int64_t)rows * K * E;
    mos_latent_fwd_kernel<<<cdiv(n, kMosThreads), kMosThreads, 0, s>>>(ua, ldu, b, lat_h, ld_l, rows, K, E, row0, m);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

int mos_latent_bwd(const float* dlat, const float* ua, int64_t ldu, __half* dua_h, int64_t ld_d, int N, int K, int E,
                   MaskSrc m, cudaStream_t s) {
    const int64_t n = (int64_t)N * K * E;
    mos_latent_bwd_kernel<<<cdiv(n, kMosThreads), kMosThreads, 0, s>>>(dlat, ua, ldu, dua_h, ld_d, N, K, E, m);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

int mos_lse(const float* Z, int rows, int V, float* lse, cudaStream_t s) {
    if (V % 4 == 0) mos_lse_kernel<true><<<rows, kMosThreads, 0, s>>>(Z, V, lse);
    else mos_lse_kernel<false><<<rows, kMosThreads, 0, s>>>(Z, V, lse);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

int mos_nll_grad(const float* Z, const float* lse, const float* ua, int64_t ldu, int Ua, const int64_t* y, int N, int K,
                 int V, int B, float* row_loss, float* loss, __half* ds_h, int64_t ld_s, __half* dua_h, int64_t ld_d,
                 cudaStream_t s) {
    const float g = (float)B / (float)N;
    if (V % 4 == 0)
        mos_nll_grad_kernel<true><<<N * K, kMosThreads, 0, s>>>(Z, lse, ua, ldu, Ua, y, K, V, g, row_loss, ds_h, ld_s,
                                                                dua_h, ld_d);
    else
        mos_nll_grad_kernel<false><<<N * K, kMosThreads, 0, s>>>(Z, lse, ua, ldu, Ua, y, K, V, g, row_loss, ds_h, ld_s,
                                                                 dua_h, ld_d);
    ZRB_KERNEL_CHECK();
    return loss_reduce(row_loss, N, g, loss, s);
}

int mos_nll_eval(const float* Z, const float* lse, const float* ua, int64_t ldu, int Ua, const int64_t* y, int N, int K,
                 int V, int B, float* row_loss, float* loss, float* tgt_prob, cudaStream_t s) {
    mos_nll_eval_kernel<<<N, 32, 0, s>>>(Z, lse, ua, ldu, Ua, y, K, V, row_loss, tgt_prob);
    ZRB_KERNEL_CHECK();
    if (!loss) return ZRB_OK;
    return loss_reduce(row_loss, N, (float)B / (float)N, loss, s);
}

int mos_logp(const float* Z, const float* lse, const float* ua, int64_t ldu, int Ua, int rows, int K, int V, float* out,
             int64_t ldo, cudaStream_t s) {
    mos_logp_kernel<<<rows, kMosThreads, 0, s>>>(Z, lse, ua, ldu, Ua, K, V, out, ldo);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

int mos_vjp(const float* Z, const float* lse, const float* ua, int64_t ldu, int Ua, int N, int K, int V, const float* G,
            float* P, float* s_buf, __half* ds_h, int64_t ld_s, __half* dua_h, int64_t ld_d, cudaStream_t s) {
    mos_vjp_token_kernel<<<N, kMosThreads, 0, s>>>(Z, lse, ua, ldu, Ua, K, V, G, P, s_buf, dua_h, ld_d);
    ZRB_KERNEL_CHECK();
    mos_vjp_dz_kernel<<<N * K, kMosThreads, 0, s>>>(Z, lse, ua, ldu, Ua, K, V, G, P, s_buf, ds_h, ld_s);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

}  // namespace zrb
