// Shared host/device helpers for libzaremba_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>

#include "../../include/zaremba_b200.h"

namespace zrb {

void set_error(const char* fmt, ...);
extern std::atomic<int64_t> g_launches;
extern std::atomic<int> g_live_tc_ctx[64];   // live tensor-core-engine contexts per device (index = device & 63)
inline void count_launch(int n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

#define ZRB_CUDA(call)                                                                   \
    do {                                                                                 \
        cudaError_t e_ = (call);                                                         \
        if (e_ != cudaSuccess) {                                                         \
            zrb::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #call,                  \
                           cudaGetErrorString(e_));                                      \
            return ZRB_E_CUDA;                                                           \
        }                                                                                \
    } while (0)

#define ZRB_KERNEL_CHECK()                                                               \
    do {                                                                                 \
        zrb::count_launch();                                                             \
        ZRB_CUDA(cudaGetLastError());                                                    \
    } while (0)

#define ZRB_REQUIRE(cond, ...)                                                           \
    do {                                                                                 \
        if (!(cond)) {                                                                   \
            zrb::set_error(__VA_ARGS__);                                                 \
            return ZRB_E_INVALID;                                                        \
        }                                                                                \
    } while (0)

#define ZRB_TRY(expr)                                                                    \
    do {                                                                                 \
        int rc_ = (expr);                                                                \
        if (rc_ != ZRB_OK) return rc_;                                                   \
    } while (0)

static inline int cdiv(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// ---------------------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al. 2011).  Counter-based: dropout keep-masks are a pure
// function of (seed, step, site, element), so backward regenerates them instead of
// storing or re-reading a mask tensor.
// ---------------------------------------------------------------------------------------
struct Philox4 {
    uint32_t v[4];
};

__host__ __device__ inline Philox4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                                 uint32_t k0, uint32_t k1) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        uint64_t p0 = (uint64_t)M0 * c0;
        uint64_t p1 = (uint64_t)M1 * c2;
        uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
        uint32_t n1 = (uint32_t)p1;
        uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
        uint32_t n3 = (uint32_t)p0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += W0; k1 += W1;
    }
    Philox4 o;
    o.v[0] = c0; o.v[1] = c1; o.v[2] = c2; o.v[3] = c3;
    return o;
}

// How the keep-mask of one dropout site is obtained.
struct MaskSrc {
    const uint8_t* explicit_mask;  // if non-null: [n] bytes, 1 = keep (replayed reference masks)
    uint32_t k0, k1;               // Philox key   = seed
    uint32_t c2, c3;               // Philox ctr hi = (site, step)
    uint32_t thresh;               // keep iff (r >> 8) >= thresh, thresh = round(p * 2^24)
    float scale;                   // 1 / (1 - p)
    int active;                    // 0: identity (eval mode or p == 0)
    uint32_t period;               // 0, or B*H: variational mode, element e takes the flag of e % period (the mask of
                                   // time step 0 held fixed over the window; DESIGN.md section 11)
};

__host__ inline MaskSrc make_mask_src(const uint8_t* explicit_mask, uint64_t seed, uint64_t step, int site,
                                      float p, int train) {
    MaskSrc m;
    m.explicit_mask = explicit_mask;
    m.period = 0;
    m.k0 = (uint32_t)seed;
    m.k1 = (uint32_t)(seed >> 32) ^ (uint32_t)(step >> 32);
    m.c2 = (uint32_t)site;
    m.c3 = (uint32_t)step;
    double t = (double)p * 16777216.0;
    m.thresh = (uint32_t)(t + 0.5);
    m.scale = (float)(1.0 / (1.0 - (double)p));
    m.active = (train && p > 0.f) ? 1 : 0;
    return m;
}

// Uniforms of the sampler (zrb_sample): a pure function of (seed, pos, row b, vocabulary entry j).
//   key     = (seed lo32, seed hi32 XOR pos hi32)
//   counter = (j / 4, b, 0xFFFFFFFF, pos lo32); entry j reads word r[j % 4]
//   u       = ((r >> 9) + 0.5) * 2^-23: exact in float32, strictly inside (0, 1)
// Counter word 2 of a dropout mask is its site (<= 2 * ZRB_MAX_LAYERS with the recurrent sites of the variational
// mode), never 0xFFFFFFFF: the two streams cannot meet.
struct SampleSrc {
    uint32_t k0, k1, c3;
};

__host__ __device__ inline SampleSrc make_sample_src(uint64_t seed, uint64_t pos) {
    SampleSrc s;
    s.k0 = (uint32_t)seed;
    s.k1 = (uint32_t)(seed >> 32) ^ (uint32_t)(pos >> 32);
    s.c3 = (uint32_t)pos;
    return s;
}

// the four words of entries [4*g, 4*g+3] of row b
__host__ __device__ inline Philox4 sample_words(const SampleSrc& s, uint32_t g, uint32_t b) {
    return philox4x32_10(g, b, 0xFFFFFFFFu, s.c3, s.k0, s.k1);
}

__host__ __device__ inline float sample_uniform(uint32_t r) {
    return ((float)(r >> 9) + 0.5f) * 1.1920928955078125e-7f;   // 2^-23
}

// keep flags of the 4 consecutive elements [4*g, 4*g+3] packed in bits 0..3
__device__ inline uint32_t mask_keep4(const MaskSrc& m, uint64_t g, uint64_t n_total) {
    if (m.explicit_mask) {
        uint32_t bits = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            uint64_t e = 4 * g + i;
            if (e < n_total && m.explicit_mask[e]) bits |= 1u << i;
        }
        return bits;
    }
    Philox4 r = philox4x32_10((uint32_t)g, (uint32_t)(g >> 32), m.c2, m.c3, m.k0, m.k1);
    uint32_t bits = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i)
        if ((r.v[i] >> 8) >= m.thresh) bits |= 1u << i;
    return bits;
}

// the element of the site's Philox stream that element e of the activation reads (variational mode: e % period)
__device__ inline uint64_t mask_elem(const MaskSrc& m, uint64_t e) { return m.period ? e % m.period : e; }

// multiplier (0 or scale) of stream element e, without the period reduction: the persistent recurrence kernels pass
// b*H + j themselves and keep the 64-bit remainder out of their code
__device__ inline float mask_mul1_at(const MaskSrc& m, uint64_t e, uint64_t n_total) {
    if (!m.active) return 1.f;
    uint32_t bits = mask_keep4(m, e >> 2, n_total);
    return ((bits >> (e & 3)) & 1u) ? m.scale : 0.f;
}

// multiplier (0 or scale) for a single element e
__device__ inline float mask_mul1(const MaskSrc& m, uint64_t e, uint64_t n_total) {
    if (!m.active) return 1.f;
    return mask_mul1_at(m, mask_elem(m, e), n_total);
}

__device__ inline float sigmoidf_(float z) { return 1.f / (1.f + expf(-z)); }

// one SGD element (main.py:117) with the clipped gradient g = coef * grad: the ONE expression update_pack stores and the
// tied embedding's gather through a deferred update reads, so that the two agree bit for bit
__device__ __forceinline__ float sgd_elem(float p, float g, float lr) { return p - lr * g; }

// one element of the dynamic-evaluation update (DESIGN.md section 14), in this fixed fp32 order (intrinsics, so that no
// kernel contracts it differently):  d = tg - p;  u = g / (r + eps) (RMS rule) or g (SGD rule, RMS = false);
// a = min(1, (lam * r) / rbar) or min(1, lam);  p + fma(a, d, -(lr * u)).  tg = the trained weight theta_g, r = its RMS
// statistic, rbar = the mean of r over all parameters.  The ONE expression every kernel that applies the rule calls.
template <bool RMS>
__device__ __forceinline__ float dyneval_elem(float p, float g, float tg, float r, float lr, float lam, float eps,
                                              float rbar) {
    const float d = __fsub_rn(tg, p);
    const float u = RMS ? __fdiv_rn(g, __fadd_rn(r, eps)) : g;
    const float a = fminf(1.f, RMS ? __fdiv_rn(__fmul_rn(lam, r), rbar) : lam);
    return __fadd_rn(p, __fmaf_rn(a, d, -__fmul_rn(lr, u)));
}

// scalars of the dynamic-evaluation update; rbar is read on the device (zrb_grad_stats_finish writes it)
struct DynArgs {
    float lr, lam, eps;
    const float* rbar;   // null: the SGD rule
};

__device__ inline float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ inline float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

}  // namespace zrb
