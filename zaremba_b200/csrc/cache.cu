// Neural-cache evaluation (Grave, Joulin & Usunier, "Improving Neural Language Models with a Continuous Cache", ICLR
// 2017; DESIGN.md section 12 states it bit for bit).
//
// Per stream b the cache handle owns a ring of (key, next token) pairs: keys fp16 [B][cap][Hp], the last layer's output
// rounded to nearest with zero pad columns; tokens int32 [B][cap].  Stream position p lives in slot p % cap, and
// cap >= W + max_seq is a multiple of 64, so the W + T - 1 positions a window reads never collide and an aligned key tile
// never straddles the wrap.  Per window:
//
//   cache_append_kernel   the window's keys and targets into the ring, its queries into a contiguous staging image
//                         (q [B][Tq][Hp]: a 64-row query tile is one TMA box whatever the ring's wrap)
//   cache_attend_kernel   grid (key chunk, stream, 64-query tile).  A producer warp streams the chunk's key tiles
//                         through an mbarrier ring with TMA (128B swizzle); the consumer warpgroup holds the query tile in
//                         shared memory and runs wgmma m64nKNk16 (KN = 64 or 16 keys per tile) with fp32 accumulators.
//                         The epilogue in registers scales by theta, masks by position, and keeps the online softmax:
//                         running max, sum over all keys, sum over the keys whose token is the row's target.  One
//                         (m, S, S_match) partial per (row, chunk): the logits never reach HBM.
//   cache_combine_kernel  one CTA: merges the partials in chunk order (no atomics: a call is bit-reproducible), mixes
//                         with the eval step's row loss in log-add-exp form, writes p_cache, the row losses and the
//                         window loss with loss_reduce_kernel's summation tree (lambda = 0 gives its bits).
//
// Bound: HBM reads of the keys, B * (W + T) * Hp * 2 bytes per window (Large, W = 2000, B = 20: 125 MB).
#include <math.h>
#include <string.h>

#include <vector>

#include "engine.h"
#include "tc_common.cuh"
#include "tc_host.h"

namespace zrb {
constexpr int kCacheQT = 64;                  // query rows per tile (the wgmma M)
constexpr int kCacheKB = 64;                  // contraction block: one 128-byte swizzled row per key / query
constexpr int kCacheMaxHp = 1536;             // the query tile (64 x Hp fp16) stays resident in shared memory
constexpr int kCacheThreads = 160;            // warps 0-3: the consumer warpgroup; warp 4: the TMA producer
template <int KN> struct CacheCfg {
    static constexpr int kStages = KN == 64 ? 4 : 8;
    static constexpr int kStageBytes = KN * kCacheKB * 2;
};
static int cache_smem_bytes(int KN, int Hp) {
    const int stages = KN == 64 ? CacheCfg<64>::kStages : CacheCfg<16>::kStages;
    return kCacheQT * Hp * 2 + stages * KN * kCacheKB * 2 + 1024 /*align slack*/ + 256 /*barriers*/;
}
}  // namespace zrb

struct zrb_cache {
    int H = 0, Hp = 0, B = 0, W = 0, max_seq = 0, cap = 0, Tq = 0, nch_max = 0;
    int64_t pos = 0;                  // tokens fed since the last reset (host: no synchronisation)
    int device = 0;
    int slots64 = 0, slots16 = 0;     // CTAs of each attend variant resident on the device at once
    __half* keys = nullptr;           // [B][cap][Hp]
    int32_t* toks = nullptr;          // [B][cap]
    __half* q = nullptr;              // [B][Tq][Hp] the window's queries
    float4* part = nullptr;           // [nch_max][max_seq * B] (m, S, S_match, -)
    CUtensorMap kmap64, kmap16, qmap;
    std::vector<void*> allocs;
};

namespace zrb {

using namespace tc;

__global__ void cache_append_kernel(const __half* __restrict__ xh, const float* __restrict__ xf, int64_t ld,
                                    const int64_t* __restrict__ y, __half* __restrict__ keys, int32_t* __restrict__ toks,
                                    __half* __restrict__ q, int B, int H, int Hp, int cap, int Tq, int64_t P0) {
    const int n = blockIdx.x, t = n / B, b = n - t * B;
    const int slot = (int)((P0 + t) % cap);
    __half* krow = keys + ((int64_t)b * cap + slot) * Hp;
    __half* qrow = q + ((int64_t)b * Tq + t) * Hp;
    for (int j0 = 8 * threadIdx.x; j0 < Hp; j0 += 8 * blockDim.x) {
        union { uint4 u; __half h[8]; } v;
        if (xh && j0 + 8 <= H) {
            v.u = *reinterpret_cast<const uint4*>(xh + (int64_t)n * ld + j0);
        } else {
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const int j = j0 + e;
                v.h[e] = j < H ? (xh ? xh[(int64_t)n * ld + j] : __float2half_rn(xf[(int64_t)n * ld + j]))
                               : __float2half_rn(0.f);
            }
        }
        *reinterpret_cast<uint4*>(krow + j0) = v.u;
        *reinterpret_cast<uint4*>(qrow + j0) = v.u;
    }
    if (threadIdx.x == 0) toks[(int64_t)b * cap + slot] = (int32_t)y[n];
}

struct AttendArgs {
    const int32_t* toks;
    const int64_t* y;     // [T*B] the window's targets
    float4* part;         // [nch][T*B]
    int T, B, W, cap, Tq, nkb;
    int qrel0;            // position of the window's row 0, relative to key tile 0
    int base_slot;        // ring slot of key tile 0
    int nk, tpc;          // key tiles of the window, tiles per chunk
    float theta;
};

// combine two online-softmax partials (m, S, S_match); m = -inf is the empty partial
__device__ __forceinline__ void cache_merge(float& m, float& S, float& Sm, float om, float oS, float oSm) {
    const float nm = fmaxf(m, om);
    if (nm == -INFINITY) return;
    const float a = expf(m - nm), c = expf(om - nm);   // expf(-inf) = 0
    S = S * a + oS * c;
    Sm = Sm * a + oSm * c;
    m = nm;
}

template <int KN>
__global__ void __launch_bounds__(kCacheThreads)
cache_attend_kernel(const __grid_constant__ CUtensorMap kmap, const __grid_constant__ CUtensorMap qmap, AttendArgs p) {
    using Cfg = CacheCfg<KN>;
    constexpr int kStages = Cfg::kStages, kStageBytes = Cfg::kStageBytes;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint8_t* sQ = smem;                                   // [nkb][64 rows][128 B]
    uint8_t* sK = smem + p.nkb * (kCacheQT * 128);        // [kStages][KN rows][128 B]
    uint64_t* bars = (uint64_t*)(sK + kStages * kStageBytes);
    uint64_t* qbar = bars;
    uint64_t* full = bars + 1;
    uint64_t* empty = bars + 1 + kStages;

    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
    const int lane = threadIdx.x & 31;
    const int chunk = blockIdx.x, b = blockIdx.y, qt = blockIdx.z;
    const int t_lo = qt * kCacheQT, t_hi = min(p.T, t_lo + kCacheQT);
    // key tiles this CTA reads: its chunk, clipped to what its query rows can see ([first - W, last) relative positions)
    const int need_lo_rel = p.qrel0 + t_lo - p.W, need_hi_rel = p.qrel0 + t_hi - 1;
    int i0 = chunk * p.tpc, i1 = min(p.nk, i0 + p.tpc);
    if (need_lo_rel > 0) i0 = max(i0, need_lo_rel / KN);
    i1 = need_hi_rel > 0 ? min(i1, (need_hi_rel - 1) / KN + 1) : i0;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&kmap);
        tma_prefetch_desc(&qmap);
        mbar_init(qbar, 1);
        for (int i = 0; i < kStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 4); }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == 4) {
        // ===================== TMA producer =====================
        if (lane == 0 && i0 < i1) {
            mbar_expect_tx(qbar, p.nkb * kCacheQT * 128);
            for (int kb = 0; kb < p.nkb; ++kb)
                tma_load_2d(sQ + kb * (kCacheQT * 128), &qmap, qbar, kb * kCacheKB, b * p.Tq + t_lo);
            int s = 0; uint32_t ph = 0;
            for (int i = i0; i < i1; ++i) {
                const int row = b * p.cap + (p.base_slot + i * KN) % p.cap;
                for (int kb = 0; kb < p.nkb; ++kb) {
                    mbar_wait(&empty[s], ph ^ 1);
                    mbar_expect_tx(&full[s], kStageBytes);
                    tma_load_2d(sK + s * kStageBytes, &kmap, &full[s], kb * kCacheKB, row);
                    if (++s == kStages) { s = 0; ph ^= 1; }
                }
            }
        }
        return;
    }

    // ===================== consumer warpgroup =====================
    const int t = threadIdx.x;
    int prel[2], tgt[2];
    bool live[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int tl = t_lo + wgmma_row(t, h);
        live[h] = tl < t_hi;
        prel[h] = p.qrel0 + tl;
        tgt[h] = live[h] ? (int)p.y[(int64_t)tl * p.B + b] : -1;
    }
    float m[2] = {-INFINITY, -INFINITY}, S[2] = {0.f, 0.f}, Sm[2] = {0.f, 0.f};
    if (i0 < i1) {
        mbar_wait(qbar, 0);
        const uint32_t q_addr = smem_u32(sQ);
        int s = 0; uint32_t ph = 0;
        float acc[KN / 2];
        for (int i = i0; i < i1; ++i) {
            const int slot0 = (p.base_slot + i * KN) % p.cap;
            int2 tok[KN / 8];
#pragma unroll
            for (int c8 = 0; c8 < KN / 8; ++c8)
                tok[c8] = __ldg(reinterpret_cast<const int2*>(p.toks + (int64_t)b * p.cap + slot0 + wgmma_col(t, c8)));
#pragma unroll
            for (int r = 0; r < KN / 2; ++r) acc[r] = 0.f;
            wgmma_fence();
            wgmma_fence_acc(acc);
            int prev = -1;
            for (int kb = 0; kb < p.nkb; ++kb) {
                mbar_wait(&full[s], ph);
                const uint32_t a_addr = q_addr + kb * (kCacheQT * 128);
                const uint32_t b_addr = smem_u32(sK + s * kStageBytes);
#pragma unroll
                for (int k = 0; k < kCacheKB / 16; ++k) {
                    // both K-major, 128B swizzle: rows 128 B apart, 8-row groups 1024 B apart, +32 B per K=16 step
                    const uint64_t da = make_smem_desc(a_addr + k * 32, 16, 1024, kSwizzle128B);
                    const uint64_t db = make_smem_desc(b_addr + k * 32, 16, 1024, kSwizzle128B);
                    Wgmma<KN, 0, 0>::mma(acc, da, db, 1u);
                }
                wgmma_commit();
                wgmma_wait<1>();                   // the previous stage's wgmmas are done: hand it back
                if (prev >= 0) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty[prev]);
                }
                prev = s;
                if (++s == kStages) { s = 0; ph ^= 1; }
            }
            wgmma_wait<0>();
            wgmma_fence_acc(acc);
            if (prev >= 0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[prev]);
            }
            // epilogue: scale, mask by position, online update of this thread's share of its two rows
            const int krel0 = i * KN;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float lm = -INFINITY;
#pragma unroll
                for (int c8 = 0; c8 < KN / 8; ++c8)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int kr = krel0 + wgmma_col(t, c8) + e;
                        const bool ok = kr >= prel[h] - p.W && kr < prel[h];
                        const float sv = ok ? p.theta * acc[4 * c8 + 2 * h + e] : -INFINITY;
                        acc[4 * c8 + 2 * h + e] = sv;
                        lm = fmaxf(lm, sv);
                    }
                if (lm == -INFINITY) continue;
                const float nm = fmaxf(m[h], lm);
                const float sc = expf(m[h] - nm);
                float ts = 0.f, tm = 0.f;
#pragma unroll
                for (int c8 = 0; c8 < KN / 8; ++c8)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const float w = expf(acc[4 * c8 + 2 * h + e] - nm);
                        ts += w;
                        if ((e ? tok[c8].y : tok[c8].x) == tgt[h]) tm += w;
                    }
                S[h] = S[h] * sc + ts;
                Sm[h] = Sm[h] * sc + tm;
                m[h] = nm;
            }
        }
    }
    // the four threads of a row combine their shares (fixed xor order), one writes the chunk's partial
    const int N = p.T * p.B;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
            const float om = __shfl_xor_sync(0xffffffffu, m[h], o);
            const float oS = __shfl_xor_sync(0xffffffffu, S[h], o);
            const float oSm = __shfl_xor_sync(0xffffffffu, Sm[h], o);
            cache_merge(m[h], S[h], Sm[h], om, oS, oSm);
        }
        if ((t & 3) == 0 && live[h])
            p.part[(int64_t)chunk * N + (int64_t)(t_lo + wgmma_row(t, h)) * p.B + b] = make_float4(m[h], S[h], Sm[h], 0.f);
    }
}

// One CTA of 256 threads.  A group of G lanes (a power of two <= 32, as many as keep all threads busy: G = 1 for a
// 700-row window, more for short ones with many chunks) merges a row's partials: lane l of the group takes chunks
// l, l + G, ... in order, then a fixed xor tree.  The window loss then sums the row losses with loss_reduce_kernel's
// tree (thread i: rows i, i + 256, ...), so with lambda = 0 (row loss = the eval step's row loss) it has its bits.
constexpr int kCombineThreads = 256;
__global__ void __launch_bounds__(kCombineThreads)
cache_combine_kernel(const float4* __restrict__ part, int nch, int N, int G, float lam, float log1m_lam, float log_lam,
                     float* row_loss, float* __restrict__ cache_prob, float* __restrict__ loss, float scale) {
    __shared__ float sh[32];
    const int group = threadIdx.x / G, gl = threadIdx.x % G, ngroups = kCombineThreads / G;
    for (int n0 = 0; n0 < N; n0 += ngroups) {      // the same trip count for every thread: the shuffles below converge
        const int n = n0 + group;
        float m = -INFINITY, S = 0.f, Sm = 0.f;
        if (n < N)
            for (int c = gl; c < nch; c += G) {
                const float4 v = part[(int64_t)c * N + n];
                cache_merge(m, S, Sm, v.x, v.y, v.z);
            }
        for (int o = G >> 1; o > 0; o >>= 1) {
            const float om = __shfl_xor_sync(0xffffffffu, m, o);
            const float oS = __shfl_xor_sync(0xffffffffu, S, o);
            const float oSm = __shfl_xor_sync(0xffffffffu, Sm, o);
            cache_merge(m, S, Sm, om, oS, oSm);
        }
        if (gl != 0 || n >= N) continue;
        const bool empty = m == -INFINITY;    // no earlier position in the window of this row (a stream's first token)
        const float pc = empty ? 0.f : Sm / S;
        if (cache_prob) cache_prob[n] = pc;
        if (row_loss && !empty && lam != 0.f) {   // -log((1-lam) exp(-r) + lam pc) = -logaddexp(log(1-lam) - r, log(lam) + log(pc))
            const float a = log1m_lam - row_loss[n], c = log_lam + logf(pc);
            const float hi = fmaxf(a, c), lo = fminf(a, c);
            row_loss[n] = -(hi + log1pf(expf(lo - hi)));
        }
    }
    if (!loss) return;
    __syncthreads();
    float acc = 0.f;
    for (int n = threadIdx.x; n < N; n += blockDim.x) acc += row_loss[n];
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x < 32) {
        float v = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.f;
        v = warp_sum(v);
        if (threadIdx.x == 0) *loss = v * scale;
    }
}

// The dynamic shared memory limit is an attribute of the kernel on the device, shared by every handle: it is raised
// once per device to what the widest handle (Hp = kCacheMaxHp) needs, so that a narrower handle created later cannot
// lower it under a wider one.  The occupancy (slots) is the handle's own.
static bool g_attend_attr_set[64][2] = {};
template <int KN>
static int attend_setup(zrb_cache* k, int* slots) {
    auto kern = cache_attend_kernel<KN>;
    bool& done = g_attend_attr_set[k->device & 63][KN == 64 ? 0 : 1];
    if (!done) {
        ZRB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, cache_smem_bytes(KN, kCacheMaxHp)));
        done = true;
    }
    const int smem = cache_smem_bytes(KN, k->Hp);
    int per_sm = 0;
    ZRB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kCacheThreads, smem));
    *slots = (per_sm > 0 ? per_sm : 1) * tc_num_sms();
    return ZRB_OK;
}

// append + attend + combine for one window of T rows per stream; xh (fp16, pitch ld) or xf (fp32, pitch ld) = the
// last layer's output, row n = t*B + b.  row_loss: the eval step's row losses, mixed in place (or null: p_cache only).
static int cache_window(zrb_cache* k, const __half* xh, const float* xf, int64_t ld, const int64_t* y, int T, float theta,
                        float lam, float* row_loss, float* cache_prob, float* loss, cudaStream_t s) {
    const int B = k->B, N = T * B;
    const int64_t P0 = k->pos;
    cache_append_kernel<<<N, 64, 0, s>>>(xh, xf, ld, y, k->keys, k->toks, k->q, B, k->H, k->Hp, k->cap, k->Tq, P0);
    ZRB_KERNEL_CHECK();
    // keys the window reads: positions [lo, hi) (row t sees [max(0, P0 + t - W), P0 + t))
    const int64_t lo = P0 > k->W ? P0 - k->W : 0, hi = P0 + T - 1;
    int nch = 0;
    if (hi > lo) {
        const int nqt = cdiv(T, kCacheQT);
        // 16-key tiles when 64-key tiles, one per CTA, would not fill the device once (small B and W)
        const int64_t base64 = lo / 64 * 64;
        const int nk64 = cdiv(hi - base64, 64);
        const int KN = (int64_t)B * nqt * nk64 < k->slots64 ? 16 : 64;
        const int64_t base = lo / KN * KN;
        AttendArgs a;
        a.toks = k->toks; a.y = y; a.part = k->part;
        a.T = T; a.B = B; a.W = k->W; a.cap = k->cap; a.Tq = k->Tq; a.nkb = k->Hp / kCacheKB;
        a.qrel0 = (int)(P0 - base);
        a.base_slot = (int)(base % k->cap);
        a.nk = cdiv(hi - base, KN);
        a.theta = theta;
        // the fewest key tiles per CTA that still fit the grid in one wave of resident CTAs
        const int slots = KN == 64 ? k->slots64 : k->slots16;
        a.tpc = a.nk;
        for (int tpc = 1; tpc <= a.nk; ++tpc)
            if ((int64_t)B * nqt * cdiv(a.nk, tpc) <= slots) { a.tpc = tpc; break; }
        nch = cdiv(a.nk, a.tpc);
        const dim3 grid(nch, B, nqt);
        if (KN == 64)
            cache_attend_kernel<64><<<grid, kCacheThreads, cache_smem_bytes(64, k->Hp), s>>>(k->kmap64, k->qmap, a);
        else
            cache_attend_kernel<16><<<grid, kCacheThreads, cache_smem_bytes(16, k->Hp), s>>>(k->kmap16, k->qmap, a);
        ZRB_KERNEL_CHECK();
    }
    const float scale = (float)((double)B / (double)N);   // softmax_nll's: summed over the batch, averaged over time
    int G = 1;
    while (G < 32 && (int64_t)N * G * 2 <= kCombineThreads && G < nch) G *= 2;
    cache_combine_kernel<<<1, kCombineThreads, 0, s>>>(k->part, nch, N, G, lam, log1pf(-lam), logf(lam), row_loss,
                                                       cache_prob, loss, scale);
    ZRB_KERNEL_CHECK();
    k->pos = P0 + T;
    return ZRB_OK;
}

static int check_theta(float theta) {
    ZRB_REQUIRE(theta >= 0.f && isfinite(theta), "theta %f must be finite and >= 0", theta);
    return ZRB_OK;
}

// the ring lives in the memory of the device the handle was created on: its kernels must run there
static int check_device(const zrb_cache* k) {
    int dev = -1;
    ZRB_CUDA(cudaGetDevice(&dev));
    ZRB_REQUIRE(dev == k->device, "the cache was created on device %d, the current device is %d", k->device, dev);
    return ZRB_OK;
}

}  // namespace zrb

using namespace zrb;

extern "C" {

int zrb_cache_create(int32_t hidden, int32_t batch, int32_t size, int32_t max_seq, zrb_cache** out) {
    ZRB_REQUIRE(out, "null argument");
    *out = nullptr;
    ZRB_REQUIRE(hidden >= 1 && (hidden + 63) / 64 * 64 <= kCacheMaxHp, "hidden %d outside [1, %d]", hidden, kCacheMaxHp);
    ZRB_REQUIRE(batch >= 1 && size >= 1 && max_seq >= 1, "batch %d, size %d and max_seq %d must be >= 1", batch, size,
                max_seq);
    ZRB_REQUIRE((int64_t)size + max_seq <= (1 << 28), "size %d + max_seq %d too large", size, max_seq);
    zrb_cache* k = new zrb_cache();
    k->H = hidden; k->Hp = (hidden + 63) / 64 * 64; k->B = batch; k->W = size; k->max_seq = max_seq;
    k->cap = (size + max_seq + 63) / 64 * 64;
    k->Tq = (max_seq + kCacheQT - 1) / kCacheQT * kCacheQT;
    k->nch_max = k->cap / 16 + 1;
    cudaGetDevice(&k->device);
    auto alloc = [&](void** ptr, size_t bytes) -> int {
        if (cudaMalloc(ptr, bytes) != cudaSuccess) {
            set_error("cudaMalloc(%zu) failed for the neural cache", bytes);
            return ZRB_E_NOMEM;
        }
        k->allocs.push_back(*ptr);
        return cudaMemset(*ptr, 0, bytes) == cudaSuccess ? ZRB_OK : ZRB_E_CUDA;
    };
    int rc = alloc((void**)&k->keys, (size_t)batch * k->cap * k->Hp * sizeof(__half));
    if (rc == ZRB_OK) rc = alloc((void**)&k->toks, (size_t)batch * k->cap * sizeof(int32_t));
    if (rc == ZRB_OK) rc = alloc((void**)&k->q, (size_t)batch * k->Tq * k->Hp * sizeof(__half));
    if (rc == ZRB_OK) rc = alloc((void**)&k->part, (size_t)k->nch_max * max_seq * batch * sizeof(float4));
    if (rc == ZRB_OK) rc = tc_make_tmap_f16(&k->kmap64, k->keys, k->Hp, (uint64_t)batch * k->cap, k->Hp, kCacheKB, 64, 1);
    if (rc == ZRB_OK) rc = tc_make_tmap_f16(&k->kmap16, k->keys, k->Hp, (uint64_t)batch * k->cap, k->Hp, kCacheKB, 16, 1);
    if (rc == ZRB_OK) rc = tc_make_tmap_f16(&k->qmap, k->q, k->Hp, (uint64_t)batch * k->Tq, k->Hp, kCacheKB, kCacheQT, 1);
    if (rc == ZRB_OK) rc = attend_setup<64>(k, &k->slots64);
    if (rc == ZRB_OK) rc = attend_setup<16>(k, &k->slots16);
    if (rc != ZRB_OK) {
        zrb_cache_destroy(k);
        return rc;
    }
    *out = k;
    return ZRB_OK;
}

int zrb_cache_reset(zrb_cache* cache) {
    ZRB_REQUIRE(cache, "null cache");
    cache->pos = 0;   // stale slots are masked by position
    return ZRB_OK;
}

void zrb_cache_destroy(zrb_cache* cache) {
    if (!cache) return;
    for (void* p : cache->allocs) cudaFree(p);
    delete cache;
}

int zrb_cache_step(zrb_cache* cache, const float* h, const int64_t* y, int32_t T, int32_t B, float theta,
                   float* cache_prob, void* stream) {
    ZRB_REQUIRE(cache && h && y && cache_prob, "null argument");
    ZRB_TRY(check_theta(theta));
    ZRB_TRY(check_device(cache));
    ZRB_REQUIRE(B == cache->B, "B=%d but the cache holds %d streams", B, cache->B);
    ZRB_REQUIRE(T >= 1 && T <= cache->max_seq, "T=%d outside [1,%d]", T, cache->max_seq);
    return cache_window(cache, nullptr, h, cache->H, y, T, theta, 0.f, nullptr, cache_prob, nullptr, (cudaStream_t)stream);
}

int zrb_eval_step_cache(zrb_ctx* c, const zrb_params* p, const int64_t* x, const int64_t* y, int32_t T, int32_t B,
                        const zrb_states* in, const zrb_states* out, zrb_cache* cache, float theta, float lambda,
                        float* loss, float* tgt_prob, float* cache_prob, void* stream) {
    ZRB_REQUIRE(c && p && x && y && in && out && cache, "null argument");
    ZRB_REQUIRE(!c->experts, "the neural cache does not support a Mixture-of-Softmaxes context (experts = %d)", c->experts);
    ZRB_TRY(check_theta(theta));
    ZRB_TRY(check_device(cache));
    ZRB_REQUIRE(lambda >= 0.f && lambda < 1.f, "lambda %f outside [0,1)", lambda);
    ZRB_REQUIRE(B == cache->B, "B=%d but the cache holds %d streams", B, cache->B);
    const int H = c->width[c->cfg.layers];   // the last layer's width
    ZRB_REQUIRE(H == cache->H, "the model's last layer has H=%d but the cache %d", H, cache->H);
    ZRB_REQUIRE(T >= 1 && T <= cache->max_seq, "T=%d outside [1,%d] of the cache", T, cache->max_seq);
    cudaStream_t s = (cudaStream_t)stream;
    // zrb_eval_step's forward and softmax (the same row losses and tgt_prob), its loss reduction left to the combine
    ZRB_TRY(zrb_forward(c, p, x, T, B, in, out, c->scores, 0, 0, 0, stream));
    c->have_fwd = false;
    ZRB_TRY(softmax_nll(c->scores, y, T * B, c->cfg.vocab, B, c->row_loss, nullptr, nullptr, tgt_prob, s));
    const __half* xh = nullptr;
    const float* xf = nullptr;
    int64_t ld = H;
    if (c->cfg.engine == ZRB_ENGINE_TC) {
        xh = tc_last_layer_image(c);     // fp16 image of the last layer's output, pitch Hp: the projection's operand
        ld = cache->Hp;
    } else {
        xf = c->act[c->cfg.layers];      // eval mode: no dropout, act[L] = h
    }
    return cache_window(cache, xh, xf, ld, y, T, theta, lambda, c->row_loss, cache_prob, loss, s);
}

}  // extern "C"
