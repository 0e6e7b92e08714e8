// Persistent, warp-specialised wgmma GEMM for sm_90a:
//     C[M,N] (fp32) = alpha * A * B^T (+ bias[N]) (+ C)
// A is [M,K] (K-major) or stored [K,M] (MN-major); B is [N,K] (K-major) or stored [K,N]
// (MN-major).  fp16 operands, fp32 accumulation in registers.
//
//   warpgroup 0   TMA producer (one thread): cp.async.bulk.tensor 2-D boxes, 128B swizzle, mbarrier ring
//                 (6 stages of 128x128 tiles or 4 of 128x256)
//   warpgroups 1-2  consumers: warpgroup c owns rows [64c, 64c+64) of the 128-row tile, issues wgmma m64nNk16
//                 (N = tile width) on each landed stage, releases the stage once the next stage's wgmmas are in
//                 flight, and stores its accumulators (alpha, bias, fp32 stores or split-K atomics) itself; the two
//                 warpgroups run kStages-1 K blocks apart, so one's epilogue overlaps the other's wgmmas
//
// A split-K plan that leaves SMs idle runs instead as 64-row items in 2-CTA clusters that multicast the B tile they
// share (gemm_f16_tc_pair_kernel, below), with the same arithmetic per output element.
//
// Every batched contraction of the path runs here: X*W_ih^T, the vocabulary projection, their
// dgrads (weights read MN-major from the same fp16 image, no transposed copies) and the
// wgrads (both operands MN-major: contraction over tokens).  Roofline: tensor pipe
// (2*M*N*K flop per call); operands stream once from HBM/L2 via TMA.
#include <stdlib.h>
#include <string.h>

#include "kernels.h"
#include "tc_common.cuh"
#include "tc_host.h"

namespace zrb {

using namespace tc;

constexpr int GBM = 128, GBK = 64;
constexpr int kASubBytes = GBM * GBK * 2;   // the 128-row A tile of a K block
constexpr int kEpiWarps = 8;                 // consumer warps: sum-of-squares slots per tile
constexpr int kGemmThreads = 3 * 128;
// Tile N is a template parameter: 128 (6 stages) or 256 (4 stages).  128x256 tiles pull 25% fewer operand bytes per
// flop than 128x128 ones, so 256 is used whenever it still fills the machine.
template <int GBN> struct GemmCfg {
    static constexpr int kStages = GBN == 256 ? 4 : 6;
    static constexpr int kABytes = kASubBytes;
    static constexpr int kBBytes = GBN * GBK * 2;
    static constexpr int kSmem = kStages * (kABytes + kBBytes) + 1024 /*align slack*/ + 256 /*barriers*/;
};

struct GemmArgs {
    int M, N, K;
    float alpha;
    const float* bias;
    const float* bias2;   // or null: a second bias vector added with the first (b_ih + b_hh, model.py:35)
    float* C;
    int64_t ldc;
    int accumulate;
    int tiles_m, tiles_n;
    int splits;      // split-K factor (1 or 2); with 2 the epilogue adds atomically into a zeroed C
    float* sumsq_out; // or null: slot [tile * 8 + w] = sum of squares of the outputs consumer warp w stored for `tile`
                      // (the wgrads feed clip_grad_norm_ from here instead of re-reading 200 MB of gradients)
    float* C2;        // dual launch (or null): a second problem with the same A, M and K but its own B (tma_b2), N2, C2
    float* sumsq_out2;  // pitch, output and sum-of-squares slots; work items [num_tiles, num_tiles + tiles_m * tiles_n2)
    int N2, tiles_n2;   // belong to it, tile w - num_tiles (splits == 1)
    int64_t ldc2;
    const __half* a_tiled;   // EXPERIMENT (zrb_gemm_f16_tiled): pre-tiled, pre-swizzled K-major images ([K block][128-row
    const __half* b_tiled;   // tile][128][64] halves, chunk c of row r stored at c ^ (r % 8)): operand tiles are fetched with
    int a_nt128, b_nt128;    // 1-D bulk copies instead of 2-D tensor loads
    int pdl_trigger;  // release a programmatic dependent enqueued behind this kernel (a recurrence kernel) at once
    int pdl_tail;     // launched as a programmatic dependent of the kernel before it in the stream (it started while that
                      // kernel was still running and consumes none of its outputs): wait for that kernel before exiting,
                      // so that "this grid completed" keeps implying "everything before it in the stream completed"
    int epi_direct;   // ZRB_GEMM_EPI=direct: both consumer warpgroups in lockstep, one 4-byte store per element
};

// Staggered consumers (the default): warpgroup 1 starts its first work item only once warpgroup 0 has issued the
// wgmmas of kStagger K blocks (or all of its first item, if shorter).  Both stay that far apart -- the producer can
// only refill a stage that both have released -- so each warpgroup's epilogue runs while the other one issues wgmmas
// instead of leaving the tensor cores idle.  kStagger < kStages: warpgroup 0 gets there on stages the producer loads
// before anything is released.
template <int GBN> constexpr int kStagger = GemmCfg<GBN>::kStages - 1;
constexpr int kStaggerBar = 1;   // named barrier of the two consumer warpgroups (256 threads)

template <bool A_MN, bool B_MN, int GBN>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_f16_tc_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                   const __grid_constant__ CUtensorMap tma_b2, GemmArgs p) {
    using Cfg = GemmCfg<GBN>;
    constexpr int kStages = Cfg::kStages;
    constexpr int kABytes = Cfg::kABytes;
    constexpr int kBBytes = Cfg::kBBytes;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint8_t* sA = smem;
    uint8_t* sB = smem + kStages * kABytes;
    uint64_t* bars = (uint64_t*)(smem + kStages * (kABytes + kBBytes));
    uint64_t* full = bars;                       // [kStages]
    uint64_t* empty = bars + kStages;            // [kStages]

    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);   // warp-uniform for the compiler
    const int lane = threadIdx.x & 31;
    const int num_tiles = p.tiles_m * p.tiles_n;
    const int num_kb = (p.K + GBK - 1) / GBK;
    const bool dual = p.C2 != nullptr;
    // work item w: tile = w % num_tiles and K range w / num_tiles (split-K), or tile w - num_tiles of the second problem
    // once w >= num_tiles (dual launch)
    const int num_work = dual ? num_tiles + p.tiles_m * p.tiles_n2 : num_tiles * p.splits;
    const int kb_per = (num_kb + p.splits - 1) / p.splits;

    if (threadIdx.x == 0) {
        if (p.pdl_trigger) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
        tma_prefetch_desc(&tma_a);
        tma_prefetch_desc(&tma_b);
        if (dual) tma_prefetch_desc(&tma_b2);
        for (int i = 0; i < kStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], kEpiWarps); }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp < 4) {
        // ===================== TMA producer =====================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
        if (warp == 0 && lane == 0) {
            int s = 0; uint32_t ph = 0;
            for (int w = blockIdx.x; w < num_work; w += gridDim.x) {
                const bool second = dual && w >= num_tiles;
                const int tile = second ? w - num_tiles : w % num_tiles, sp = dual ? 0 : w / num_tiles;
                const int kb0 = sp * kb_per, kb1 = min(num_kb, kb0 + kb_per);
                const CUtensorMap* tmb = second ? &tma_b2 : &tma_b;
                const int m0 = (tile % p.tiles_m) * GBM, n0 = (tile / p.tiles_m) * GBN;
                for (int kb = kb0; kb < kb1; ++kb) {
                    mbar_wait(&empty[s], ph ^ 1);
                    mbar_expect_tx(&full[s], kABytes + kBBytes);
                    uint8_t* a = sA + s * kABytes;
                    uint8_t* b = sB + s * kBBytes;
                    if (!A_MN && p.a_tiled) {
                        bulk_load_1d(a, p.a_tiled + ((size_t)kb * p.a_nt128 + (m0 >> 7)) * (128 * GBK), kASubBytes, &full[s]);
                    } else if (!A_MN) {
                        tma_load_2d(a, &tma_a, &full[s], kb * GBK, m0);
                    } else {
                        tma_load_2d(a, &tma_a, &full[s], m0, kb * GBK);
                        tma_load_2d(a + kASubBytes / 2, &tma_a, &full[s], m0 + 64, kb * GBK);
                    }
                    if (!B_MN && p.b_tiled) {
                        bulk_load_1d(b, p.b_tiled + ((size_t)kb * p.b_nt128 + (n0 >> 7)) * (128 * GBK), kBBytes, &full[s]);
                    } else if (!B_MN) {
                        tma_load_2d(b, tmb, &full[s], kb * GBK, n0);
                    } else {
#pragma unroll
                        for (int j = 0; j < GBN / 64; ++j)
                            tma_load_2d(b + j * (GBK * 128), tmb, &full[s], n0 + 64 * j, kb * GBK);
                    }
                    if (++s == kStages) { s = 0; ph ^= 1; }
                }
            }
        }
    } else {
        // ===================== consumers: two warpgroups =====================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
        const int cw = warp - 4;                        // consumer warp 0..7
        const int wg = cw >> 2;                         // rows [64 wg, 64 wg + 64) of the tile
        const int t = (int)threadIdx.x - 128 * (1 + wg);
        int s = 0; uint32_t ph = 0;
        float acc[GBN / 2];
        bool started_wg1 = p.epi_direct || wg == 1;   // (warpgroup 0) has warpgroup 1 been let go
        if (!p.epi_direct && wg == 1) asm volatile("bar.sync %0, 256;" :: "n"(kStaggerBar) : "memory");
        int kb_issued = 0;
        // float2 stores (and float2 atomics for split-K): a quad of lanes writes one whole 32-byte sector of a row
        const bool pair_store = !p.epi_direct && !p.accumulate && (p.ldc & 1) == 0 && (p.ldc2 & 1) == 0 &&
                                ((uintptr_t)p.C & 7) == 0 && ((uintptr_t)p.C2 & 7) == 0;
        for (int w = blockIdx.x; w < num_work; w += gridDim.x) {
            const bool second = dual && w >= num_tiles;
            const int tile = second ? w - num_tiles : w % num_tiles, split = dual ? 0 : w / num_tiles;
            const int kb0 = split * kb_per, kb1 = min(num_kb, kb0 + kb_per);
            float* const Cout = second ? p.C2 : p.C;
            float* const ssq = second ? p.sumsq_out2 : p.sumsq_out;
            const int Nw = second ? p.N2 : p.N;
            const int64_t ldcw = second ? p.ldc2 : p.ldc;
            const int m0 = (tile % p.tiles_m) * GBM + 64 * wg, n0 = (tile / p.tiles_m) * GBN;
#pragma unroll
            for (int i = 0; i < GBN / 2; ++i) acc[i] = 0.f;
            wgmma_fence();
            wgmma_fence_acc(acc);
            int prev = -1;
            for (int kb = kb0; kb < kb1; ++kb) {
                mbar_wait(&full[s], ph);
                // this warpgroup's 64 rows start 8192 B into the stage's A tile in both layouts (K-major: 64 rows of
                // 128 B; MN-major: the second 64-element M block); 1024-byte aligned, so the swizzle phase is unchanged
                const uint32_t a_addr = smem_u32(sA + s * kABytes) + wg * (kASubBytes / 2);
                const uint32_t b_addr = smem_u32(sB + s * kBBytes);
#pragma unroll
                for (int k = 0; k < GBK / 16; ++k) {
                    // K-major, 128B swizzle: rows 128 B apart, 8-row groups 1024 B apart, +32 B per K=16 step.
                    // MN-major, 128B swizzle: 64-element blocks GBK*128 B apart (LBO), 8 k-rows per 1024 B group (SBO),
                    // +16 k-rows = 2048 B per step.
                    const uint64_t da = A_MN ? make_smem_desc(a_addr + k * 2048, GBK * 128, 1024, kSwizzle128B)
                                             : make_smem_desc(a_addr + k * 32, 16, 1024, kSwizzle128B);
                    const uint64_t db = B_MN ? make_smem_desc(b_addr + k * 2048, GBK * 128, 1024, kSwizzle128B)
                                             : make_smem_desc(b_addr + k * 32, 16, 1024, kSwizzle128B);
                    Wgmma<GBN, A_MN ? 1 : 0, B_MN ? 1 : 0>::mma(acc, da, db, 1u);
                }
                wgmma_commit();
                if (!started_wg1 && ++kb_issued == kStagger<GBN>) {
                    asm volatile("bar.arrive %0, 256;" :: "n"(kStaggerBar) : "memory");
                    started_wg1 = true;
                }
                wgmma_wait<1>();                        // the previous stage's wgmmas are done: hand it back
                if (prev >= 0) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty[prev]);
                }
                prev = s;
                if (++s == kStages) { s = 0; ph ^= 1; }
            }
            if (!started_wg1) {                         // a first work item shorter than kStagger K blocks
                asm volatile("bar.arrive %0, 256;" :: "n"(kStaggerBar) : "memory");
                started_wg1 = true;
            }
            wgmma_wait<0>();
            wgmma_fence_acc(acc);
            if (prev >= 0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[prev]);
            }
            // epilogue straight from the accumulator fragments (tc_common.cuh: wgmma_row / wgmma_col)
            const bool add_bias = p.bias != nullptr && split == 0;
            float ss = 0.f;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = m0 + wgmma_row(t, h);
                if (row >= p.M) continue;
                float* const crow = Cout + (int64_t)row * ldcw;
#pragma unroll
                for (int c8 = 0; c8 < GBN / 8; ++c8) {
                    const int col0 = n0 + wgmma_col(t, c8);   // even
                    if (pair_store && col0 + 1 < Nw) {
                        // the same two elements, values and sum-of-squares order as the per-element loop below
                        const float bv0 = add_bias ? p.bias[col0] + (p.bias2 ? p.bias2[col0] : 0.f) : 0.f;
                        const float bv1 = add_bias ? p.bias[col0 + 1] + (p.bias2 ? p.bias2[col0 + 1] : 0.f) : 0.f;
                        const float o0 = p.alpha * acc[4 * c8 + 2 * h] + bv0;
                        const float o1 = p.alpha * acc[4 * c8 + 2 * h + 1] + bv1;
                        if (p.splits > 1) {
                            atomicAdd(reinterpret_cast<float2*>(crow + col0), make_float2(o0, o1));
                        } else {
                            *reinterpret_cast<float2*>(crow + col0) = make_float2(o0, o1);
                            ss += o0 * o0;
                            ss += o1 * o1;
                        }
                        continue;
                    }
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int col = n0 + wgmma_col(t, c8) + e;
                        if (col >= Nw) continue;
                        const float bv = add_bias ? p.bias[col] + (p.bias2 ? p.bias2[col] : 0.f) : 0.f;
                        const float o = p.alpha * acc[4 * c8 + 2 * h + e] + bv;
                        if (p.splits > 1) {
                            atomicAdd(crow + col, o);
                        } else if (p.accumulate) {
                            crow[col] += o;
                        } else {
                            crow[col] = o;
                            ss += o * o;
                        }
                    }
                }
            }
            if (ssq) {
                ss = warp_sum(ss);
                if (lane == 0) ssq[tile * 8 + cw] = ss;
            }
        }
        if (!started_wg1) asm volatile("bar.arrive %0, 256;" :: "n"(kStaggerBar) : "memory");   // (a CTA without work)
    }
    // ONE CTA keeps the grid from completing before the primary has: a CTA blocked here holds its SM, and if every
    // CTA waited, the SMs the recurrence leaves idle would each run a single tile and then sit until it ends
    if (p.pdl_tail && blockIdx.x == 0 && threadIdx.x == 0) asm volatile("griddepcontrol.wait;" ::: "memory");
}

// ---- split-K in CTA pairs ----------------------------------------------------------------------
// A split-K plan of 128-row tiles leaves SMs idle (the dgrads: 6 x 6 tiles x 2 K halves = 72 CTAs on 132 SMs; M = 700 is
// 11 blocks of 64 rows, so 64-row items fill the machine).  This kernel runs the same plan as 64 x 256 x (one K half)
// work items, two per 2-CTA cluster.  A pair shares its K half; usually it is the two 64-row halves of one 128-row tile
// (same N block), and then each CTA loads its own A rows and one column half of the B tile, multicast into both.  Each
// consumer warpgroup takes 128 columns of the 64 rows, one wgmma chain over the same K blocks as in the 128-row plan:
// every output element gets the same k16 sequence, the same alpha and the same two atomically added partials, so the
// bits are those of the 128-row plan.
//
// Pairs of one K half: first the vertical ones (64-row blocks 2i and 2i+1 of an N block), then, when the number of
// 64-row blocks is odd, the last block's items two by two along N; those do not share B, and each CTA loads its whole
// B tile itself.  An odd one left over is paired with a copy of itself that stores nothing.  Both CTAs of a pair run the
// same K blocks, so their stage rings stay in step: a stage is refilled once the consumers of BOTH CTAs have released it
// (the partner's multicast writes into this CTA's copy of the stage).
//
// The two consumer warpgroups read the same stages in lockstep (no staggered start): a CTA of this plan runs one work
// item, so there is no epilogue to hide under the other warpgroup's wgmmas, and the producer can run a whole ring ahead
// of both.  The stage count is what fits in 227 KB (the 64-row A tile frees 8 KB per stage).  Only split plans of
// 256-wide tiles take it (gemm_f16_tc).
constexpr int PBM = 64, PBN = 256;
struct PairCfg {
    static constexpr int kStages = 5;
    static constexpr int kABytes = PBM * GBK * 2;
    static constexpr int kBBytes = PBN * GBK * 2;
    static constexpr int kSmem = kStages * (kABytes + kBBytes) + 1024 /*align slack*/ + 256 /*barriers*/;
};

// pairs per K half for tiles_m 64-row blocks and tiles_n N blocks
__host__ __device__ inline int pairs_per_split(int tiles_m, int tiles_n) {
    return (tiles_m / 2) * tiles_n + ((tiles_m & 1) ? (tiles_n + 1) / 2 : 0);
}

struct PairItem {
    int split, m_blk, n_blk;
    bool shared;   // both CTAs have this N block: each loads one column half of B for both
    bool live;     // false: a copy of the partner's item, nothing stored
};
__device__ __forceinline__ PairItem pair_item(int tiles_m, int tiles_n, int pair, int rank) {
    const int vert = (tiles_m / 2) * tiles_n, per = pairs_per_split(tiles_m, tiles_n);
    const int q = pair % per;
    PairItem it;
    it.split = pair / per;
    if (q < vert) {
        it.n_blk = q / (tiles_m / 2);
        it.m_blk = 2 * (q % (tiles_m / 2)) + rank;
        it.shared = it.live = true;
    } else {
        const int n_first = 2 * (q - vert);   // rank 0's N block
        it.m_blk = tiles_m - 1;
        it.live = n_first + rank < tiles_n;
        it.n_blk = it.live ? n_first + rank : n_first;
        it.shared = n_first + 1 >= tiles_n;
    }
    return it;
}

// p.tiles_m counts 64-row blocks here; p.splits == 2, no sum-of-squares slots, no accumulate, no dual problem.
template <bool A_MN, bool B_MN>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_f16_tc_pair_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                        GemmArgs p) {
    using Cfg = PairCfg;
    constexpr int GBN = PBN;
    constexpr int kStages = Cfg::kStages;
    constexpr int kABytes = Cfg::kABytes;
    constexpr int kBBytes = Cfg::kBBytes;
    constexpr int kBHalf = kBBytes / 2;   // GBN/2 columns: K-major GBN/2 rows of 128 B, MN-major GBN/128 64-column boxes
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint8_t* sA = smem;
    uint8_t* sB = smem + kStages * kABytes;
    uint64_t* bars = (uint64_t*)(smem + kStages * (kABytes + kBBytes));
    uint64_t* full = bars;                       // [kStages]
    uint64_t* empty = bars + kStages;            // [kStages]: the consumer warps of both CTAs

    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
    const int lane = threadIdx.x & 31;
    const int rank = (int)cta_rank_in_cluster();
    const int num_kb = (p.K + GBK - 1) / GBK;
    const int kb_per = (num_kb + 1) / 2;
    const int num_pairs = 2 * pairs_per_split(p.tiles_m, p.tiles_n);
    const int cluster = blockIdx.x >> 1, num_clusters = gridDim.x >> 1;

    if (threadIdx.x == 0) {
        if (p.pdl_trigger) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
        tma_prefetch_desc(&tma_a);
        tma_prefetch_desc(&tma_b);
        for (int i = 0; i < kStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 2 * kEpiWarps); }
        fence_mbar_init();
    }
    cluster_barrier();   // the partner's barriers exist before anything multicasts or arrives on them

    if (warp < 4) {
        // ===================== TMA producer =====================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
        if (warp == 0 && lane == 0) {
            int s = 0; uint32_t ph = 0;
            for (int pr = cluster; pr < num_pairs; pr += num_clusters) {
                const PairItem it = pair_item(p.tiles_m, p.tiles_n, pr, rank);
                const int kb0 = it.split * kb_per, kb1 = min(num_kb, kb0 + kb_per);
                const int m0 = it.m_blk * PBM, n0 = it.n_blk * GBN;
                for (int kb = kb0; kb < kb1; ++kb) {
                    mbar_wait(&empty[s], ph ^ 1);
                    mbar_expect_tx(&full[s], kABytes + kBBytes);
                    uint8_t* a = sA + s * kABytes;
                    uint8_t* b = sB + s * kBBytes;
                    if (!A_MN) tma_load_2d(a, &tma_a, &full[s], kb * GBK, m0);
                    else       tma_load_2d(a, &tma_a, &full[s], m0, kb * GBK);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        if (it.shared && h != rank) continue;
#pragma unroll
                        for (int j = 0; j < (B_MN ? GBN / 128 : 1); ++j) {
                            uint8_t* dst = b + h * kBHalf + j * (GBK * 128);
                            const int c0 = B_MN ? n0 + h * (GBN / 2) + 64 * j : kb * GBK;
                            const int c1 = B_MN ? kb * GBK : n0 + h * (GBN / 2);
                            if (it.shared) tma_load_2d_multicast(dst, &tma_b, &full[s], c0, c1, 0x3);
                            else           tma_load_2d(dst, &tma_b, &full[s], c0, c1);
                        }
                    }
                    if (++s == kStages) { s = 0; ph ^= 1; }
                }
            }
        }
    } else {
        // ===================== consumers: warpgroup wg takes columns [wg GBN/2, (wg + 1) GBN/2) =====================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
        const int cw = warp - 4;
        const int wg = cw >> 2;
        const int t = (int)threadIdx.x - 128 * (1 + wg);
        int s = 0; uint32_t ph = 0;
        float acc[GBN / 4];
        const bool pair_store = (p.ldc & 1) == 0 && ((uintptr_t)p.C & 7) == 0;
        for (int pr = cluster; pr < num_pairs; pr += num_clusters) {
            const PairItem it = pair_item(p.tiles_m, p.tiles_n, pr, rank);
            const int kb0 = it.split * kb_per, kb1 = min(num_kb, kb0 + kb_per);
            const int m0 = it.m_blk * PBM, n0 = it.n_blk * GBN + wg * (GBN / 2);
#pragma unroll
            for (int i = 0; i < GBN / 4; ++i) acc[i] = 0.f;
            wgmma_fence();
            wgmma_fence_acc(acc);
            int prev = -1;
            for (int kb = kb0; kb < kb1; ++kb) {
                mbar_wait(&full[s], ph);
                const uint32_t a_addr = smem_u32(sA + s * kABytes);
                const uint32_t b_addr = smem_u32(sB + s * kBBytes) + wg * kBHalf;   // 1024-byte aligned
#pragma unroll
                for (int k = 0; k < GBK / 16; ++k) {
                    const uint64_t da = A_MN ? make_smem_desc(a_addr + k * 2048, GBK * 128, 1024, kSwizzle128B)
                                             : make_smem_desc(a_addr + k * 32, 16, 1024, kSwizzle128B);
                    const uint64_t db = B_MN ? make_smem_desc(b_addr + k * 2048, GBK * 128, 1024, kSwizzle128B)
                                             : make_smem_desc(b_addr + k * 32, 16, 1024, kSwizzle128B);
                    Wgmma<GBN / 2, A_MN ? 1 : 0, B_MN ? 1 : 0>::mma(acc, da, db, 1u);
                }
                wgmma_commit();
                wgmma_wait<1>();
                if (prev >= 0) {
                    __syncwarp();
                    if (lane < 2) mbar_arrive_rank(&empty[prev], lane);   // this CTA's and the partner's
                }
                prev = s;
                if (++s == kStages) { s = 0; ph ^= 1; }
            }
            wgmma_wait<0>();
            wgmma_fence_acc(acc);
            if (prev >= 0) {
                __syncwarp();
                if (lane < 2) mbar_arrive_rank(&empty[prev], lane);
            }
            if (!it.live) continue;
            // the epilogue of gemm_f16_tc_kernel's split-K path, element for element
            const bool add_bias = p.bias != nullptr && it.split == 0;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = m0 + wgmma_row(t, h);
                if (row >= p.M) continue;
                float* const crow = p.C + (int64_t)row * p.ldc;
#pragma unroll
                for (int c8 = 0; c8 < GBN / 16; ++c8) {
                    const int col0 = n0 + wgmma_col(t, c8);
                    if (pair_store && col0 + 1 < p.N) {
                        const float bv0 = add_bias ? p.bias[col0] + (p.bias2 ? p.bias2[col0] : 0.f) : 0.f;
                        const float bv1 = add_bias ? p.bias[col0 + 1] + (p.bias2 ? p.bias2[col0 + 1] : 0.f) : 0.f;
                        const float o0 = p.alpha * acc[4 * c8 + 2 * h] + bv0;
                        const float o1 = p.alpha * acc[4 * c8 + 2 * h + 1] + bv1;
                        atomicAdd(reinterpret_cast<float2*>(crow + col0), make_float2(o0, o1));
                        continue;
                    }
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int col = col0 + e;
                        if (col >= p.N) continue;
                        const float bv = add_bias ? p.bias[col] + (p.bias2 ? p.bias2[col] : 0.f) : 0.f;
                        atomicAdd(crow + col, p.alpha * acc[4 * c8 + 2 * h + e] + bv);
                    }
                }
            }
        }
    }
    __syncwarp();
    cluster_barrier();   // no CTA leaves while its partner may still multicast into it or arrive on its barriers
}

// ---- host side ----------------------------------------------------------------------------------
namespace {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

int g_num_sms = 0;
bool g_attr_set[64][8] = {};   // per device: function attributes belong to the device's context

}  // namespace

int tc_num_sms() {
    if (!g_num_sms) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
        if (g_num_sms <= 0) g_num_sms = 132;
    }
    return g_num_sms;
}

// fp16 2-D tensor map: `inner` contiguous elements per row, `outer` rows, row pitch ld elements
int tc_make_tmap_f16(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t box_inner,
                     uint32_t box_outer, int swizzle128) {
    EncodeTiledFn enc = get_encode();
    if (!enc) {
        set_error("cuTensorMapEncodeTiled not available from the driver");
        return ZRB_E_CUDA;
    }
    ZRB_REQUIRE((ld * 2) % 16 == 0 && (((uintptr_t)ptr) & 15) == 0, "TMA operand needs 16-byte aligned base and pitch");
    cuuint64_t dims[2] = {inner, outer};
    cuuint64_t strides[1] = {ld * 2};
    cuuint32_t box[2] = {box_inner, box_outer};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed (%d) inner=%llu outer=%llu ld=%llu", (int)r,
                  (unsigned long long)inner, (unsigned long long)outer, (unsigned long long)ld);
        return ZRB_E_CUDA;
    }
    return ZRB_OK;
}

template <bool A_MN, bool B_MN, int GBN>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tb2, const GemmArgs& a,
                       cudaStream_t s) {
    auto kern = gemm_f16_tc_kernel<A_MN, B_MN, GBN>;
    const int idx = (A_MN ? 2 : 0) + (B_MN ? 1 : 0) + (GBN == 256 ? 4 : 0);
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (!g_attr_set[dev][idx]) {
        ZRB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, GemmCfg<GBN>::kSmem));
        g_attr_set[dev][idx] = true;
    }
    const int work = a.C2 ? a.tiles_m * (a.tiles_n + a.tiles_n2) : a.tiles_m * a.tiles_n * a.splits;
    int grid = work;
    if (grid > tc_num_sms()) grid = tc_num_sms();
    if (a.pdl_tail) {
        // programmatic dependent launch: the grid may start as soon as every CTA of the preceding kernel has executed
        // griddepcontrol.launch_dependents (the persistent recurrence kernels do so once they are all resident), and
        // fills the SMs that kernel leaves idle; CTAs that find no free SM start when it ends.  ONE work item per CTA
        // here (not the persistent one-CTA-per-SM grid): the hardware block scheduler then hands tiles to whichever
        // SMs are free, so the idle SMs work through most of the tiles while the recurrence runs, instead of each
        // late CTA still owning a full static share of them.
        grid = work;
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(grid); cfg.blockDim = dim3(kGemmThreads);
        cfg.dynamicSmemBytes = GemmCfg<GBN>::kSmem; cfg.stream = s;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        ZRB_CUDA(cudaLaunchKernelEx(&cfg, kern, ta, tb, tb2, a));
        count_launch();
        return ZRB_OK;
    }
    kern<<<grid, kGemmThreads, GemmCfg<GBN>::kSmem, s>>>(ta, tb, tb2, a);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

// the gemm_f16_tc_pair_kernel instantiation for the operand layouts
static const void* pair_kernel(bool a_mn, bool b_mn) {
    if (!a_mn) return b_mn ? (const void*)gemm_f16_tc_pair_kernel<false, true> : (const void*)gemm_f16_tc_pair_kernel<false, false>;
    return b_mn ? (const void*)gemm_f16_tc_pair_kernel<true, true> : (const void*)gemm_f16_tc_pair_kernel<true, false>;
}

static void pair_launch_config(cudaLaunchConfig_t* cfg, cudaLaunchAttribute* cluster, int grid) {
    *cfg = {};
    cfg->gridDim = dim3(grid); cfg->blockDim = dim3(kGemmThreads); cfg->dynamicSmemBytes = PairCfg::kSmem;
    cluster->id = cudaLaunchAttributeClusterDimension;
    cluster->val.clusterDim.x = 2; cluster->val.clusterDim.y = 1; cluster->val.clusterDim.z = 1;
    cfg->attrs = cluster; cfg->numAttrs = 1;
}

// per device and layout: 1 + cudaOccupancyMaxActiveClusters of the pair kernel (0: not asked yet; a failed query
// counts as none).  Asking also raises the kernel's shared-memory limit, which its launches rely on.
static int g_pair_clusters[64][4] = {};

// The pair plan when all its clusters are resident at once (one round of 64-row items instead of one of 128-row tiles);
// false: the caller keeps the 128-row plan.
static bool pair_plan_fits(int pairs, bool a_mn, bool b_mn) {
    int dev = 0;
    cudaGetDevice(&dev);
    int& slot = g_pair_clusters[dev & 63][(a_mn ? 2 : 0) + (b_mn ? 1 : 0)];
    if (!slot) {
        const void* kern = pair_kernel(a_mn, b_mn);
        cudaLaunchConfig_t cfg;
        cudaLaunchAttribute cluster;
        pair_launch_config(&cfg, &cluster, tc_num_sms() & ~1);
        int n = 0;
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, PairCfg::kSmem) != cudaSuccess ||
            cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess) {
            (void)cudaGetLastError();
            n = 0;
        }
        slot = 1 + n;
    }
    return pairs <= slot - 1;
}

static int launch_gemm_pair(const CUtensorMap& ta, const CUtensorMap& tb, const GemmArgs& a, int pairs, bool a_mn,
                            bool b_mn, cudaStream_t s) {
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute cluster;
    pair_launch_config(&cfg, &cluster, 2 * pairs);
    cfg.stream = s;
    void* args[] = {(void*)&ta, (void*)&tb, (void*)&a};
    ZRB_CUDA(cudaLaunchKernelExC(&cfg, pair_kernel(a_mn, b_mn), args));
    count_launch();
    return ZRB_OK;
}

template <int GBN>
static int dispatch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tb2, const GemmArgs& a,
                         int a_mn, int b_mn, cudaStream_t s) {
    if (!a_mn && !b_mn) return launch_gemm<false, false, GBN>(ta, tb, tb2, a, s);
    if (!a_mn && b_mn) return launch_gemm<false, true, GBN>(ta, tb, tb2, a, s);
    if (a_mn && !b_mn) return launch_gemm<true, false, GBN>(ta, tb, tb2, a, s);
    return launch_gemm<true, true, GBN>(ta, tb, tb2, a, s);
}

// Tile shape for an [M,N] output with K-block count num_kb: 128x256 when those tiles give every SM (nearly) a
// full wave, else 128x128; few output tiles but a long contraction (the dgrads) split K.
// With `retile` (outputs without sum-of-squares slots, ZRB_GEMM_EPI unset), an unsplit 256-wide plan whose last round
// of the persistent grid is mostly empty switches to 128-wide tiles when those need fewer rounds counted in
// 256-wide-tile units (X*W_ih^T at Large: 144 tiles = 2 rounds on 132 SMs, vs 282 half tiles = 3 half rounds).  The
// tile width does not change what is summed per output element, nor in which K order.
struct TileChoice { int bn, tiles_m, tiles_n, splits; };
static TileChoice choose_tiles(int M, int N, int num_kb, bool can_split, bool retile = false) {
    const int nsm = tc_num_sms();
    TileChoice c;
    c.tiles_m = cdiv(M, GBM);
    const int t256 = c.tiles_m * cdiv(N, 256);
    if (can_split && t256 * 2 <= nsm && t256 * 2 >= (nsm * 4) / 10 && num_kb / 2 >= 8) {
        // the dgrads ([700 x 1500] outputs, 94..157 K blocks): 36 tiles of 128x256 with the contraction split in two
        // move 25% fewer operand bytes per CTA than 72 tiles of 128x128.  Never more than two splits: two partials
        // added into a zeroed C give the same sum in either order, so a train step is reproducible run to run.
        c.bn = 256; c.tiles_n = cdiv(N, 256); c.splits = 2;
        return c;
    }
    c.bn = (t256 >= (nsm * 9) / 10) ? 256 : 128;
    if (retile && c.bn == 256 && cdiv(t256, nsm) * 2 > cdiv(c.tiles_m * cdiv(N, 128), nsm) &&
             c.tiles_m * cdiv(N, 128) * 2 > nsm)   // (never turns a whole plan into a split one)
        c.bn = 128;
    c.tiles_n = cdiv(N, c.bn);
    // few output tiles but a long contraction: split K in two so that ~all SMs work; partials added into a
    // zeroed C with atomics
    c.splits = (can_split && c.tiles_m * c.tiles_n * 2 <= nsm && num_kb >= 8) ? 2 : 1;
    return c;
}

// The tile plan of g's launch.  sumsq: it writes sum-of-squares slots.  A dual launch takes the tile width of its
// wider problem; both problems are cut into tiles of that width.
static TileChoice gemm_tiles(const Gemm& g, bool sumsq, bool direct) {
    if (g.dual.C) return choose_tiles(g.M, g.N > g.dual.N ? g.N : g.dual.N, cdiv(g.K, GBK), false);
    const bool plain = !sumsq && !g.accumulate;
    return choose_tiles(g.M, g.N, cdiv(g.K, GBK), plain && g.ldc == g.N, plain && !direct);
}

GemmSlots gemm_f16_tc_sumsq_slots(const Gemm& g) {
    const TileChoice c = gemm_tiles(g, true, false);
    GemmSlots n;
    n.first = c.tiles_m * cdiv(g.N, c.bn) * kEpiWarps;
    n.dual = g.dual.C ? c.tiles_m * cdiv(g.dual.N, c.bn) * kEpiWarps : 0;
    return n;
}

int gemm_f16_tc(const Gemm& g, cudaStream_t s) {
    const int M = g.M, N = g.N, K = g.K;
    const Gemm::Dual& d2 = g.dual;
    if (M <= 0 || N <= 0) return ZRB_OK;
    ZRB_REQUIRE(!d2.B == !d2.C, "dual launch needs both B2 and C2");
    ZRB_REQUIRE(!d2.C || (d2.N > 0 && !g.bias && !g.accumulate), "dual launch: N2 > 0, no bias, no accumulate");
    ZRB_REQUIRE(!g.bias2 || g.bias, "bias2 needs bias");
    ZRB_REQUIRE(!g.sumsq || !g.accumulate, "sumsq_out needs a plain store epilogue");
    ZRB_REQUIRE(K > 0, "gemm_f16_tc needs K > 0");
    // ZRB_GEMM_EPI=direct: the lockstep consumers with per-element stores and the tile plan they were tuned with (A/B
    // comparisons, bit for bit and in time); read at every launch so that one process can run both
    const char* epi = getenv("ZRB_GEMM_EPI");
    const bool direct = epi && strcmp(epi, "direct") == 0;
    const TileChoice tc = gemm_tiles(g, g.sumsq != nullptr, direct);
    const int bn = tc.bn;
    const bool a_mn = g.A.mn_major, b_mn = g.B.mn_major;
    // a split plan of 256-wide tiles runs in CTA pairs of 64-row items (gemm_f16_tc_pair_kernel) when that makes more
    // work items and all the pairs are resident at once; never under ZRB_GEMM_EPI=direct, whose plan is the reference.
    // (128-wide tiles stay: as pairs each warpgroup issues m64n64 wgmmas, and Medium's dS*W_fc measured 6% slower.)
    const int tiles_m64 = cdiv(M, PBM);
    const int pairs = 2 * pairs_per_split(tiles_m64, tc.tiles_n);
    const bool paired = !direct && tc.splits == 2 && bn == 256 && !g.a_tiled && !g.b_tiled && tiles_m64 > tc.tiles_m &&
                        pair_plan_fits(pairs, a_mn, b_mn);
    const int box_m = paired ? PBM : GBM, box_n = paired ? bn / 2 : bn;   // (K-major boxes; MN-major ones are 64 wide)
    CUtensorMap ta, tb;
    if (!a_mn) ZRB_TRY(tc_make_tmap_f16(&ta, g.A.ptr, K, M, g.A.ld, GBK, box_m, 1));
    else       ZRB_TRY(tc_make_tmap_f16(&ta, g.A.ptr, M, K, g.A.ld, 64, GBK, 1));
    if (!b_mn) ZRB_TRY(tc_make_tmap_f16(&tb, g.B.ptr, K, N, g.B.ld, GBK, box_n, 1));
    else       ZRB_TRY(tc_make_tmap_f16(&tb, g.B.ptr, N, K, g.B.ld, 64, GBK, 1));
    CUtensorMap tb2 = tb;
    if (d2.B) {
        if (!b_mn) ZRB_TRY(tc_make_tmap_f16(&tb2, d2.B, K, d2.N, d2.ldb, GBK, bn, 1));
        else       ZRB_TRY(tc_make_tmap_f16(&tb2, d2.B, d2.N, K, d2.ldb, 64, GBK, 1));
    }
    GemmArgs a;
    a.M = M; a.N = N; a.K = K; a.alpha = g.alpha; a.bias = g.bias; a.C = g.C; a.ldc = g.ldc;
    a.accumulate = g.accumulate;
    a.tiles_m = tc.tiles_m; a.tiles_n = cdiv(N, bn);   // (a dual plan's tile width comes from the wider problem)
    a.splits = tc.splits;
    a.sumsq_out = g.sumsq;
    a.bias2 = g.bias2;
    a.C2 = d2.C; a.sumsq_out2 = d2.sumsq;
    a.N2 = d2.N; a.ldc2 = d2.ldc; a.tiles_n2 = cdiv(d2.N, bn);
    a.a_tiled = a_mn ? nullptr : g.a_tiled; a.a_nt128 = g.a_nt128; a.b_tiled = b_mn ? nullptr : g.b_tiled;
    a.b_nt128 = g.b_nt128;
    a.pdl_tail = (g.pdl && a.splits == 1) ? 1 : 0;    // (a split launch is preceded by a memset: nothing to chain to)
    a.pdl_trigger = (rec_pdl_enabled() && !a.pdl_tail) ? 1 : 0;
    a.epi_direct = direct ? 1 : 0;
    // split partials are added into a zeroed C: order-independent for two (a+b == b+a)
    if (a.splits > 1 && !g.accumulate) ZRB_CUDA(cudaMemsetAsync(g.C, 0, (size_t)M * N * sizeof(float), s));
    if (paired) {
        a.tiles_m = tiles_m64;
        return launch_gemm_pair(ta, tb, a, pairs, a_mn, b_mn, s);
    }
    return bn == 256 ? dispatch_gemm<256>(ta, tb, tb2, a, a_mn, b_mn, s) : dispatch_gemm<128>(ta, tb, tb2, a, a_mn, b_mn, s);
}

}  // namespace zrb

// EXPERIMENT: the same GEMM (K-major A and B) with both operands given as pre-tiled images as well; a_nt128 / b_nt128 =
// 128-row tiles per K block in the images (b_nt128 even)
extern "C" int zrb_gemm_f16_tiled(const void* A, int64_t lda, const void* B, int64_t ldb, const void* A_tiled, int32_t a_nt128,
                                  const void* B_tiled, int32_t b_nt128, float* C, int64_t ldc, int32_t M, int32_t N, int32_t K,
                                  float alpha, void* stream) {
    ZRB_REQUIRE(A && B && C, "null argument");
    zrb::Gemm g;
    g.A = {(const __half*)A, lda}; g.B = {(const __half*)B, ldb};
    g.C = C; g.ldc = ldc; g.M = M; g.N = N; g.K = K; g.alpha = alpha;
    g.a_tiled = (const __half*)A_tiled; g.a_nt128 = a_nt128; g.b_tiled = (const __half*)B_tiled; g.b_nt128 = b_nt128;
    return zrb::gemm_f16_tc(g, (cudaStream_t)stream);
}

extern "C" int zrb_gemm_f16(const void* A, int64_t lda, int32_t a_mn_major, const void* B, int64_t ldb,
                            int32_t b_mn_major, float* C, int64_t ldc, int32_t M, int32_t N, int32_t K, float alpha,
                            const float* bias, int32_t accumulate, void* stream) {
    ZRB_REQUIRE(A && B && C, "null argument");
    zrb::Gemm g;
    g.A = {(const __half*)A, lda, a_mn_major != 0}; g.B = {(const __half*)B, ldb, b_mn_major != 0};
    g.C = C; g.ldc = ldc; g.M = M; g.N = N; g.K = K; g.alpha = alpha; g.bias = bias; g.accumulate = accumulate != 0;
    return zrb::gemm_f16_tc(g, (cudaStream_t)stream);
}
