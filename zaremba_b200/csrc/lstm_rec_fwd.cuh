// The persistent forward recurrence kernel (see lstm_rec_fwd.cu for the flow), included by the sources that
// instantiate it: lstm_rec_fwd.cu (the mode off) and lstm_rec_zoneout.cu (zoneout, DESIGN.md section 20).
#pragma once
#include "lstm_cell.cuh"
#include "rec_common.cuh"

namespace zrb {

// K-split variant (RecPlan::KS == 2, used when the shape allows): a CTA that owns 4U = 48 gate rows and the whole
// contraction issues H/16 = 94 chained, three-quarters-full M=64 wgmmas per step.  A CLUSTER OF TWO CTAs instead owns 2U
// units = 8U gate rows (two M = 64 tiles, N = pad8(B)): CTA r keeps the K half r of all 8U rows resident (168 KB at U = 14), loads
// only its half of the h image, runs half the K chain, and the MMA warpgroup pushes each accumulator pair straight from
// registers into the shared memory of the CTA that owns the row's unit (st.async, bytes counted on the owner's mbarrier:
// no fence, no staging pass); the owner adds the two partial sums in its cell math.

__device__ __forceinline__ uint32_t fwd_cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ uint32_t fwd_mapa(uint32_t local_addr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_addr), "r"(rank));
    return r;
}
__device__ __forceinline__ void fwd_cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ZO: zoneout (DESIGN.md section 20).  The cell keeps h_{t-1} in hreg beside c_{t-1} in creg, draws its two flags while
// the MMAs run, and stores c~_t for the backward; every ZO statement is under `if constexpr`, so the instantiations with
// ZO = false compile to the code they had before the mode existed.
template <bool SPLIT, bool ZO>
__global__ void __launch_bounds__(kRecThreads, 1) lstm_rec_fwd_kernel(RecFwdArgs a) {
    extern __shared__ uint8_t smem_raw[];
    // aligned by offsetting smem_raw itself: the compiler then knows every pointer below is a shared-memory one (LDS /
    // STS, 32-bit addresses) -- a round trip through an integer would leave them generic
    uint8_t* smem = smem_raw + ((128u - (smem_u32(smem_raw) & 127u)) & 127u);
    const int a_bytes = a.KcS * a.G * 128;     // this CTA's weight slice
    const int b_bytes = a.KcS * a.GBi * 128;   // the part of the h image this CTA multiplies with
    const int Bp = a.GBi * 8;                  // N of the MMA
    const int ldd = Bp + 1;
    const int ldr = Bp + 4;                    // K-split: pitch of the receive buffer rows (16-byte aligned)
    uint8_t* sA = smem;
    uint8_t* sB = smem + a_bytes;
    float* sD = (float*)(sB + b_bytes);        // [64][Bp+1] accumulator staging (sized for two) / K-split: receive buffer
    float* sR = sD;                            //   sR[source rank][gate * U + unit][batch]
    uint64_t* bars = (uint64_t*)((uint8_t*)sD + 2 * 64 * ldd * 4);
    uint64_t* bar_a = bars;        // weight slice landed
    uint64_t* bar_b = bars + 1;    // [kRecPieces] h image pieces of this step landed
    uint64_t* bar_mma = bars + 1 + kRecPieces;  // accumulators ready
    uint64_t* bar_recv = bar_mma + 1;           // K-split: both CTAs' partial sums of my rows have landed

    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);   // warp-uniform for the compiler
    const int lane = threadIdx.x & 31;
    const int cta = blockIdx.x;
    const uint32_t rank = SPLIT ? fwd_cluster_ctarank() : 0u;   // K half this CTA multiplies; also which units it owns
    const int j0 = cta * a.U;                  // (K-split: cta = 2 * pair + rank, the pair owns units [pair*2U, pair*2U + 2U))
    const int nu = max(0, min(a.U, a.H - j0));
    const int ksteps = a.KcS / 2;
    const int piece_steps = (ksteps + kRecPieces - 1) / kRecPieces;
    const bool tr = a.trace != nullptr && cta == 0;
    long long* const trs = a.trace + 8;
    if (a.trace && threadIdx.x == 0) rec_launch_stamps(a.trace, tr, false);

    if (threadIdx.x == 0) {
        mbar_init(bar_a, 1);
        for (int i = 0; i < kRecPieces; ++i) mbar_init(&bar_b[i], 1);
        mbar_init(bar_mma, kRecMmaThreads);
        mbar_init(bar_recv, 1);
        fence_mbar_init();
    }
    __syncthreads();
    if (SPLIT) fwd_cluster_sync();   // the partner's mbarriers are initialised before any st.async targets them

    if (warp == kRecLoadWarp && lane == 0) {
        // ===================== loader =====================
        const uint8_t* src = (const uint8_t*)a.w_img + (size_t)cta * a_bytes;
        mbar_expect_tx(bar_a, a_bytes);
        for (int off = 0; off < a_bytes; off += 32768) bulk_load_1d(sA + off, src + off, min(32768, a_bytes - off), bar_a);
        pdl_wait();   // everything below reads what the preceding kernel wrote
        bool dead = false;
        const int lbo_b = a.GBi * 128;
        const size_t img_bytes = (size_t)a.Kc * a.GBi * 128;   // one whole h image; this CTA reads K chunks [rank*KcS, +KcS)
        for (int t = 0; t < a.T; ++t) {
            if (t > 0) grid_counter_wait(a.counter, a.base + (unsigned int)t * a.nCTA, a.w, dead, t);
            if (dead) break;   // (watchdog: a thread that gave up starts no further asynchronous operation)
            if (tr) trs[t * 8 + 0] = clock64();
            fence_proxy_async_global();
            const uint8_t* img = (t == 0 ? (const uint8_t*)a.h0_img : (const uint8_t*)a.h_img + (size_t)t * img_bytes) +
                                 (size_t)rank * b_bytes;
            for (int pc = 0; pc < kRecPieces; ++pc) {
                const int k0 = pc * piece_steps, k1 = min(ksteps, k0 + piece_steps);
                if (k0 >= k1) { mbar_arrive(&bar_b[pc]); continue; }
                const int off = k0 * 2 * lbo_b, bytes = (k1 - k0) * 2 * lbo_b;
                mbar_expect_tx(&bar_b[pc], bytes);
                bulk_load_1d(sB + off, img + off, bytes, &bar_b[pc]);
            }
        }
    } else if (warp >= kRecMmaWarp && warp < kRecMmaWarp + kRecMmaWarps) {
        // ===================== MMA warpgroup =====================
        const uint32_t a_addr = smem_u32(sA), b_addr = smem_u32(sB);
        const uint32_t lbo_a = a.G * 128, lbo_b = a.GBi * 128;
        const int rows_pair = 8 * a.U;                                   // K-split: gate rows of the pair (4 x 2U)
        const int mt = SPLIT && rows_pair > 64 ? 2 : 1;
        const uint32_t sR_addr = smem_u32(sR), bar_recv_addr = smem_u32(bar_recv);
        // where each of this thread's (at most four) accumulator rows goes, worked out once: its first float in the
        // staging buffer (no K split), or its receive row in the owner's shared memory and the owner's mbarrier (K split)
        const int tm = (int)threadIdx.x - kRecMmaWarp * 32;
        uint32_t row_dst[2][2], row_owner[2][2], row_bar[2][2];
        bool row_ok[2][2];
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = rec_acc_row(tm, m, h);
                if (!SPLIT) {
                    row_dst[m][h] = (uint32_t)(row * ldd * 4);
                    row_owner[m][h] = 0u; row_bar[m][h] = 0u; row_ok[m][h] = true;
                } else {
                    // row = 4 * (unit within the pair) + gate: straight into the shared memory of the owning CTA.
                    // Receive rows are gate-major (q * U + u): the cell threads of a warp (consecutive u) then read
                    // addresses ldr floats apart, 4 banks apart, instead of 4 * ldr (2 distinct banks: 16-way conflicts)
                    const int up = row >> 2, owner = up / a.U, lrow = (row & 3) * a.U + (up - owner * a.U);
                    row_ok[m][h] = row < rows_pair;
                    row_owner[m][h] = row_ok[m][h] ? (uint32_t)owner : 0u;   // (rows past the pair's are never sent)
                    row_dst[m][h] = sR_addr + (uint32_t)(((int)rank * 4 * a.U + lrow) * ldr * 4);
                    row_bar[m][h] = fwd_mapa(bar_recv_addr, row_owner[m][h]);
                }
            }
        bool dead = false;
        bounded_mbar_wait(bar_a, 0, a.w, dead, kWaitWeights, 0);
        dead = rec_mma_any(dead);
        auto emit = [&](int m, int h, int col, float v0, float v1) {
            if (!SPLIT) {
                float* dst = (float*)((uint8_t*)sD + row_dst[m][h]) + col;
                dst[0] = v0;
                dst[1] = v1;
            } else if (row_ok[m][h]) {
                st_async_v2(fwd_mapa(row_dst[m][h] + (uint32_t)col * 4u, row_owner[m][h]), v0, v1, row_bar[m][h]);
            }
        };
        for (int t = 0; t < a.T && !dead; ++t) {
            rec_mma_step(a.GBi, mt, a_addr, b_addr, lbo_a, lbo_b, ksteps, piece_steps, bar_b, t & 1, a.w, dead, t,
                         tr ? &trs[t * 8 + 1] : nullptr, emit);
            if (!dead) mbar_arrive(bar_mma);
            if (tr && tm == 0) trs[t * 8 + 2] = clock64();
        }
    } else if (warp < kRecEpiWarps) {
        pdl_wait();
        if (threadIdx.x == 0) pdl_launch_dependents();   // after the wait: dependents of this kernel keep stream order with its predecessor
        // ===================== epilogue: 256 threads =====================
        const int tid = threadIdx.x;
        const int B = a.B, H = a.H;
        bool dead = false;
        const int cells = a.U * B;                     // cell = b * U + u (u fastest: contiguous j)
        const uint64_t n_total = (uint64_t)a.T * B * H;
        int cb[kRecMaxCell];   // rec_cell
        float creg[kRecMaxCell];
        float hreg[kRecMaxCell];   // (ZO only; 0 and unused otherwise)
        // the cell's mask multipliers held fixed over the window, drawn once here (variational mode; else 1 and unused):
        // recurrent rm on the next step's operand, ym on the output when the output site's mask has a period
        float rm[kRecMaxCell], ym[kRecMaxCell];
        const uint64_t bh = (uint64_t)B * H;
#pragma unroll
        for (int k = 0; k < kRecMaxCell; ++k) {
            cb[k] = (tid + kRecEpiThreads * k) / a.U;
            const auto [b, u, ok] = rec_cell(tid, k, cb[k], a.U, cells, nu);
            creg[k] = ok ? a.c0[(size_t)b * H + j0 + u] : 0.f;
            hreg[k] = ZO && ok ? a.h0[(size_t)b * H + j0 + u] : 0.f;
            const uint64_t e = (uint64_t)b * H + j0 + u;
            rm[k] = ok ? mask_mul1_at(a.rm, e, bh) : 1.f;
            ym[k] = ok && a.m.period ? mask_mul1_at(a.m, e, bh) : 1.f;
        }
        const uint32_t recv_bytes = 2u * 4u * (uint32_t)a.U * (uint32_t)Bp * 4u;   // 2 sources x 4U rows x Bp columns
        for (int t = 0; t < a.T; ++t) {
            if (SPLIT && tid == 0 && !dead) mbar_expect_tx(bar_recv, recv_bytes);
            // prefetch the x-part pre-activations of this step while the MMAs run
            float pre[kRecMaxCell][4];
#pragma unroll
            for (int k = 0; k < kRecMaxCell; ++k) {
                const auto [b, u, ok] = rec_cell(tid, k, cb[k], a.U, cells, nu);
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    pre[k][q] = ok ? __ldg(a.gates + ((size_t)t * B + b) * 4 * H + (size_t)q * H + j0 + u) : 0.f;
            }
            // ZO, train mode: bit 2k = cell k keeps c_{t-1}, bit 2k + 1 = it keeps h_{t-1} (loaded while the MMAs run)
            uint32_t zbits = 0;
            if constexpr (ZO) {
                if (a.zo.flags) {
#pragma unroll
                    for (int k = 0; k < kRecMaxCell; ++k) {
                        const auto [b, u, ok] = rec_cell(tid, k, cb[k], a.U, cells, nu);
                        if (ok) zbits |= (uint32_t)__ldg(a.zo.flags + ((size_t)t * B + b) * H + j0 + u) << (2 * k);
                    }
                }
            }
            bounded_mbar_wait(bar_mma, t & 1, a.w, dead, kWaitAcc, t);   // staged rows / my pushes are out
            if (tr && tid == 0) trs[t * 8 + 3] = clock64();
            if (SPLIT) bounded_mbar_wait(bar_recv, t & 1, a.w, dead, kWaitRecv, t);   // both K halves of my 4U rows have landed
            if (tr && tid == 0) trs[t * 8 + 4] = clock64();
            float o_i[kRecMaxCell], o_f[kRecMaxCell], o_g[kRecMaxCell], o_o[kRecMaxCell], o_h[kRecMaxCell];
#pragma unroll
            for (int k = 0; k < kRecMaxCell; ++k) {
                const auto [b, u, ok] = rec_cell(tid, k, cb[k], a.U, cells, nu);
                o_i[k] = o_f[k] = o_g[k] = o_o[k] = o_h[k] = 0.f;
                if (!ok) continue;
                float zi, zf, zg, zo;
                if (!SPLIT) {
                    const float* d0 = sD + (4 * u) * ldd + b;
                    zi = pre[k][0] + d0[0];
                    zf = pre[k][1] + d0[ldd];
                    zg = pre[k][2] + d0[2 * ldd];
                    zo = pre[k][3] + d0[3 * ldd];
                } else {
                    const float* r0 = sR + u * ldr + b;                  // K half 0, gate 0
                    const float* r1 = r0 + 4 * a.U * ldr;                // K half 1
                    const int gs = a.U * ldr;                            // gate stride
                    zi = pre[k][0] + (r0[0] + r1[0]);
                    zf = pre[k][1] + (r0[gs] + r1[gs]);
                    zg = pre[k][2] + (r0[2 * gs] + r1[2 * gs]);
                    zo = pre[k][3] + (r0[3 * gs] + r1[3 * gs]);
                }
                const CellFwd cf = cell_fwd<FastAct, ZO>(zi, zf, zg, zo, creg[k], hreg[k], (zbits >> (2 * k)) & 1u,
                                                          (zbits >> (2 * k)) & 2u, a.zo);
                if constexpr (ZO) {
                    a.ctil[((size_t)t * B + b) * H + j0 + u] = cf.ctil;
                    hreg[k] = cf.h;
                }
                creg[k] = cf.c;
                o_i[k] = cf.i; o_f[k] = cf.f; o_g[k] = cf.g; o_o[k] = cf.o; o_h[k] = cf.h;
                // critical path: the next step's operand image [kc][g][r][e], kc = j/8, e = j%8, g = b/8, r = b%8
                const int j = j0 + u;
                __half* img = a.h_img + (size_t)(t + 1) * ((size_t)a.Kc * a.GBi * 64);
                img[((size_t)(j >> 3) * a.GBi + (b >> 3)) * 64 + (b & 7) * 8 + (j & 7)] = __float2half_rn(cf.h * rm[k]);
            }
            if (tr && tid == 0) trs[t * 8 + 5] = clock64();
            asm volatile("bar.sync 1, 256;" ::: "memory");
            if (tid == 0) {
                if (tr) trs[t * 8 + 6] = clock64();
                grid_counter_arrive(a.counter);
                if (tr) trs[t * 8 + 7] = clock64();
            }
            // off the critical path: what backward and the next layer read after this kernel
#pragma unroll
            for (int k = 0; k < kRecMaxCell; ++k) {
                const auto [b, u, ok] = rec_cell(tid, k, cb[k], a.U, cells, nu);
                if (!ok) continue;
                const int j = j0 + u;
                const size_t n = (size_t)t * B + b;
                float* grow = a.gates + n * 4 * H + j;
                grow[0] = o_i[k]; grow[H] = o_f[k]; grow[2 * (size_t)H] = o_g[k]; grow[3 * (size_t)H] = o_o[k];
                a.cst[n * H + j] = creg[k];
                a.hprev_h[((size_t)B + n) * a.Hp + j] = __float2half_rn(o_h[k] * rm[k]);
                float y = o_h[k] * (a.m.period ? ym[k] : mask_mul1_at(a.m, (uint64_t)n * H + j, n_total));
                a.y_h[n * a.Hp + j] = __float2half_rn(y);
                if (a.h_f32) a.h_f32[n * H + j] = o_h[k];
                if (t == a.T - 1) {
                    if (a.h_last) a.h_last[(size_t)b * H + j] = o_h[k];
                    if (a.c_last) a.c_last[(size_t)b * H + j] = creg[k];
                }
            }
        }
    }
    __syncthreads();
    if (SPLIT) fwd_cluster_sync();   // nobody leaves while the partner could still address its shared memory
    if (a.trace && threadIdx.x == 0) rec_launch_stamps(a.trace, tr, true);
}

}  // namespace zrb
