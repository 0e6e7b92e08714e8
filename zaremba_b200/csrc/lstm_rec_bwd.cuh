// The persistent backward recurrence kernel (see lstm_rec_bwd.cu for the flow), included by the sources that
// instantiate it: lstm_rec_bwd.cu (the mode off) and lstm_rec_zoneout.cu (zoneout, DESIGN.md section 20).
#pragma once
#include "lstm_cell.cuh"
#include "rec_common.cuh"

namespace zrb {

__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ uint32_t mapa_shared(uint32_t local_addr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_addr), "r"(rank));
    return r;
}
__device__ __forceinline__ void st_dsmem_f32(uint32_t cluster_addr, float v) {
    asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(cluster_addr), "f"(v) : "memory");
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// S = 1: clusters of 4 (CTA rank = gate), one M = 64 tile, the whole gate block as contraction.
// S = 2: clusters of 8.  The cluster owns twice the units (8U = 120 rows at Large, two M = 64 tiles, N = pad8(B)) and CTA rank
//        r = 2*gate + half multiplies only HALF of its gate's rows: 47 K steps per step instead of 94, half the operand
//        image to fetch.
// Both push their CS partial products (st.async) into the owners' shared memory, where they are summed in fixed order.
// ZO: zoneout (DESIGN.md section 20): the cell rule (lstm_cell.cuh) reads c~_t (the forward's store) and keeps the carries
// dc and hcarry in registers; hcarry joins dh with the upstream gradient in the prefetch, so that it holds no register
// across the waits.  Under `if constexpr` like the forward's.
template <int S, bool ZO>
__global__ void __launch_bounds__(kRecThreads, 1) lstm_rec_bwd_kernel(RecBwdArgs a) {
    constexpr int CS = 4 * S;   // cluster size
    extern __shared__ uint8_t smem_raw[];
    // aligned by offsetting smem_raw itself: the compiler then knows every pointer below is a shared-memory one (LDS /
    // STS, 32-bit addresses) -- a round trip through an integer would leave them generic
    uint8_t* smem = smem_raw + ((128u - (smem_u32(smem_raw) & 127u)) & 127u);
    const int a_bytes = a.KcS * a.G * 128;     // this CTA's weight slice
    const int b_bytes = a.KcS * a.GBi * 128;   // the part of its gate's dG image this CTA multiplies with
    const int Bp = a.GBi * 8;                  // N of the MMA
    uint8_t* sA = smem;
    uint8_t* sB = smem + a_bytes;
    // receive buffer sR[source rank][unit][batch (pitch ldr, 16-byte rows)], in the 2 x 64 x (Bp + 1) floats that
    // rec_smem_bytes sets aside (the plans check that it fits)
    const int ldr = Bp + 4;
    float* sR = (float*)(sB + b_bytes);
    uint64_t* bars = (uint64_t*)((uint8_t*)sR + 2 * 64 * (Bp + 1) * 4);
    uint64_t* bar_a = bars;
    uint64_t* bar_b = bars + 1;                    // [kRecPieces]
    uint64_t* bar_mma = bars + 1 + kRecPieces;
    uint64_t* bar_recv = bar_mma + 1;              // all CS CTAs' partials of this CTA's units have landed

    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);   // warp-uniform for the compiler
    const int lane = threadIdx.x & 31;
    const uint32_t rank = cluster_ctarank();
    const int cluster = blockIdx.x / CS;
    const int UC = CS * a.U;
    const int jc0 = cluster * UC;            // first unit of the cluster
    const int j0 = jc0 + (int)rank * a.U;    // first unit whose cell math this CTA owns
    const int nu = max(0, min(a.U, a.H - j0));
    const int gate = (int)rank / S, khalf = (int)rank % S;   // contraction slice: rows [khalf*KcS*8, +KcS*8) of gate block `gate`
    const int T = a.T, B = a.B, H = a.H;
    const int ksteps = a.KcS / 2;
    const int piece_steps = (ksteps + kRecPieces - 1) / kRecPieces;
    const bool tr = a.trace != nullptr && blockIdx.x == 0;
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
    cluster_sync_all();   // every CTA's mbarriers are initialised before any remote arrive

    if (warp == kRecLoadWarp && lane == 0) {
        // ===================== loader =====================
        const uint8_t* src = (const uint8_t*)a.w_img + ((size_t)cluster * CS + rank) * a_bytes;
        mbar_expect_tx(bar_a, a_bytes);
        for (int off = 0; off < a_bytes; off += 32768) bulk_load_1d(sA + off, src + off, min(32768, a_bytes - off), bar_a);
        pdl_wait();   // everything below reads what the preceding kernel wrote
        bool dead = false;
        const int lbo_b = a.GBi * 128;
        const size_t gate_bytes = (size_t)a.Kc * a.GBi * 128;   // one gate's whole dG image
        for (int s = 1; s < T; ++s) {
            const int t = T - 1 - s;                      // step being computed; needs dG_{t+1}
            grid_counter_wait(a.counter, a.base + (unsigned int)s * a.nCTA, a.w, dead, s);
            if (dead) break;   // (watchdog: a thread that gave up starts no further asynchronous operation)
            if (tr) trs[s * 8 + 0] = clock64();
            fence_proxy_async_global();
            const uint8_t* img = (const uint8_t*)a.g_img + ((size_t)((t + 1) & 1) * 4 + gate) * gate_bytes +
                                 (size_t)khalf * b_bytes;
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
        const int mt = S == 2 && UC > 64 ? 2 : 1;
        const uint32_t sR_addr = smem_u32(sR), bar_recv_addr = smem_u32(bar_recv);
        // accumulator row = cluster-local unit.  Where each of this thread's (at most four) rows goes, worked out once:
        // its receive row in the owner's shared memory and the owner's mbarrier
        const int tm = (int)threadIdx.x - kRecMmaWarp * 32;
        uint32_t row_dst[2][2], row_owner[2][2], row_bar[2][2];
        bool row_ok[2][2];
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = rec_acc_row(tm, m, h);
                const int owner = row / a.U, uo = row - owner * a.U;
                row_ok[m][h] = row < UC;
                row_owner[m][h] = row_ok[m][h] ? (uint32_t)owner : 0u;   // (rows past the cluster's are never sent)
                row_dst[m][h] = sR_addr + (uint32_t)(((int)rank * a.U + uo) * ldr * 4);
                row_bar[m][h] = mapa_shared(bar_recv_addr, row_owner[m][h]);
            }
        // variational mode: the recurrent mask of each (unit = row, batch = column) value this thread emits, drawn once.
        // Bit 16 m + 4 (col / 8) + 2 h + e (e: column col + e) set = dropped; none set with the mode off.  Every
        // partial product is multiplied by 0 or scale(p_rec) (a.rm.scale, 1 with the mode off: exact), so the cell
        // math adds scale * m * (dG_{t+1} W_hh) with no register of its own -- the epilogue is at the register limit.
        uint32_t rdrop = 0;
        if (a.rm.active) {
            for (int m = 0; m < 2; ++m)
                for (int h = 0; h < 2; ++h) {
                    const int row = rec_acc_row(tm, m, h), j = jc0 + row;
                    for (int c8 = 0; c8 < 4; ++c8)
                        for (int e = 0; e < 2; ++e) {
                            const int b = wgmma_col(tm, c8) + e;
                            if (row < UC && j < H && b < B && mask_mul1_at(a.rm, (uint64_t)b * H + j, (uint64_t)B * H) == 0.f)
                                rdrop |= 1u << (16 * m + 4 * c8 + 2 * h + e);
                        }
                }
        }
        const float rscale = a.rm.scale;
        bool dead = false;
        bounded_mbar_wait(bar_a, 0, a.w, dead, kWaitWeights, 0);
        dead = rec_mma_any(dead);
        auto emit = [&](int m, int h, int col, float v0, float v1) {
            const int bit = 16 * m + 4 * (col >> 3) + 2 * h;
            v0 *= ((rdrop >> bit) & 1u) ? 0.f : rscale;
            v1 *= ((rdrop >> (bit + 1)) & 1u) ? 0.f : rscale;
            if (row_ok[m][h]) {
                // straight from the registers into the shared memory of the CTA that owns this unit
                st_async_v2(mapa_shared(row_dst[m][h] + (uint32_t)col * 4u, row_owner[m][h]), v0, v1, row_bar[m][h]);
            }
        };
        for (int s = 1; s < T && !dead; ++s) {
            rec_mma_step(a.GBi, mt, a_addr, b_addr, lbo_a, lbo_b, ksteps, piece_steps, bar_b, (s - 1) & 1, a.w, dead, s,
                         tr ? &trs[s * 8 + 1] : nullptr, emit);
            if (!dead) mbar_arrive(bar_mma);
            if (tr && tm == 0) trs[s * 8 + 2] = clock64();
        }
    } else if (warp < kRecEpiWarps) {
        pdl_wait();
        if (threadIdx.x == 0) pdl_launch_dependents();   // after the wait: dependents of this kernel keep stream order with its predecessor
        // ===================== epilogue: 256 threads, cells (u, b) of this CTA's U units =====================
        const int tid = threadIdx.x;
        bool dead = false;
        const int cells = a.U * B;                     // cell = b * U + u (u fastest: contiguous j)
        int cb[kRecMaxCell];   // rec_cell
        float dcreg[kRecMaxCell], bsum[kRecMaxCell][4];
        float hcarry[kRecMaxCell];   // (ZO only) zh * dh_t, added to dh_{t-1}
#pragma unroll
        for (int k = 0; k < kRecMaxCell; ++k) {
            cb[k] = (tid + kRecEpiThreads * k) / a.U;
            dcreg[k] = 0.f;
            hcarry[k] = 0.f;
#pragma unroll
            for (int q = 0; q < 4; ++q) bsum[k][q] = 0.f;
        }
        const uint64_t n_total = (uint64_t)T * B * H;
        const uint32_t recv_bytes = (uint32_t)CS * (uint32_t)a.U * (uint32_t)Bp * 4u;   // CS sources x U units x Bp columns
        const float inv = 1.f / kGradScale;
        const size_t img_gate = (size_t)a.Kc * a.GBi * 64;

        for (int s = 0; s < T; ++s) {
            const int t = T - 1 - s;
            // prefetch this step's saved activations and upstream gradient
            float gi[kRecMaxCell], gf[kRecMaxCell], gg[kRecMaxCell], go[kRecMaxCell], ct[kRecMaxCell], cp[kRecMaxCell],
                dyv[kRecMaxCell];
#pragma unroll
            for (int k = 0; k < kRecMaxCell; ++k) {
                gi[k] = gf[k] = gg[k] = go[k] = ct[k] = cp[k] = dyv[k] = 0.f;
                const auto [b, u, ok] = rec_cell(tid, k, cb[k], a.U, cells, nu);
                if (ok) {
                    const int j = j0 + u;
                    const size_t n = (size_t)t * B + b;
                    const float* grow = a.gates + n * 4 * H + j;
                    gi[k] = __ldg(grow); gf[k] = __ldg(grow + H); gg[k] = __ldg(grow + 2 * (size_t)H);
                    go[k] = __ldg(grow + 3 * (size_t)H);
                    ct[k] = __ldg((ZO ? a.ctil : a.cst) + n * H + j);   // (ZO: c~_t)
                    cp[k] = t > 0 ? __ldg(a.cst + (n - B) * H + j) : __ldg(a.c0 + (size_t)b * H + j);
                    // (variational mode: element b*H + j of the site's stream, the mask fixed over the window)
                    dyv[k] = __ldg(a.dy + n * H + j) *
                             mask_mul1_at(a.m, (uint64_t)(a.m.period ? b : (int)n) * H + j, n_total);
                    if (a.r) dyv[k] += __ldg(a.r + n * H + j);
                    if constexpr (ZO) dyv[k] += hcarry[k];   // (hcarry is dead from here to the cell math)
                }
            }
            uint32_t zbits = 0;   // ZO, train mode: bit 2k = cell k kept c_{t-1}, bit 2k + 1 = it kept h_{t-1}
            if constexpr (ZO) {
                if (a.zo.flags) {
#pragma unroll
                    for (int k = 0; k < kRecMaxCell; ++k) {
                        const auto [b, u, ok] = rec_cell(tid, k, cb[k], a.U, cells, nu);
                        if (ok) zbits |= (uint32_t)__ldg(a.zo.flags + ((size_t)t * B + b) * H + j0 + u) << (2 * k);
                    }
                }
            }
            if (s > 0) {
                if (tid == 0 && !dead) mbar_expect_tx(bar_recv, recv_bytes);
                bounded_mbar_wait(bar_mma, (s - 1) & 1, a.w, dead, kWaitAcc, s);
                if (tr && tid == 0) trs[s * 8 + 3] = clock64();   // my pushes are out
                bounded_mbar_wait(bar_recv, (s - 1) & 1, a.w, dead, kWaitRecv, s);   // all CS x U x Bp partial sums of my units have landed
                if (tr && tid == 0) trs[s * 8 + 4] = clock64();
            }
            __half hv[kRecMaxCell][4];
#pragma unroll
            for (int k = 0; k < kRecMaxCell; ++k) {
                const auto [b, u, ok] = rec_cell(tid, k, cb[k], a.U, cells, nu);
                if (!ok) continue;
                float dh = dyv[k];
                if (s > 0) {
                    float pp[CS];
#pragma unroll
                    for (int rr = 0; rr < CS; ++rr) pp[rr] = sR[(rr * a.U + u) * ldr + b];
                    float r = (pp[0] + pp[1]) + (pp[2] + pp[3]);
                    if constexpr (S == 2) r += (pp[4] + pp[5]) + (pp[6] + pp[7]);
                    dh += r * inv;
                }
                const CellGrad d = cell_bwd<FastAct, ZO>(gi[k], gf[k], gg[k], go[k], ct[k], cp[k], dh, dcreg[k], hcarry[k],
                                                          (zbits >> (2 * k)) & 1u, (zbits >> (2 * k)) & 2u, a.zo);
                const float dg4[4] = {d.i, d.f, d.g, d.o};
                const int j = j0 + u;
                // critical path: the four gate images the next step multiplies with
                __half* img = a.g_img + (size_t)(t & 1) * 4 * img_gate + ((size_t)(j >> 3) * a.GBi + (b >> 3)) * 64 +
                              (b & 7) * 8 + (j & 7);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    hv[k][q] = f16_sat(dg4[q] * kGradScale);
                    img[(size_t)q * img_gate] = hv[k][q];
                    bsum[k][q] += dg4[q];
                }
            }
            if (tr && tid == 0) trs[s * 8 + 5] = clock64();
            asm volatile("bar.sync 1, 256;" ::: "memory");
            if (tid == 0) {
                if (tr) trs[s * 8 + 6] = clock64();
                grid_counter_arrive(a.counter);
                if (tr) trs[s * 8 + 7] = clock64();
            }
            // off the critical path: row-major image for the batched dgrad / wgrad GEMMs
#pragma unroll
            for (int k = 0; k < kRecMaxCell; ++k) {
                const auto [b, u, ok] = rec_cell(tid, k, cb[k], a.U, cells, nu);
                if (!ok) continue;
                __half* hrow = a.dG_h + ((size_t)t * B + b) * a.G4p + j0 + u;
#pragma unroll
                for (int q = 0; q < 4; ++q) hrow[(size_t)q * H] = hv[k][q];
            }
        }
        if (a.db1) {
            // bias gradients: per-cell sums over the window -> a global scratch [4][B][H] -> fixed-order sum over the
            // batch by one thread per (gate, unit) of this CTA.  bar.sync orders the CTA's own global writes for its readers.
            // (ZO: nu and cells computed afresh from an opaque copy of U: held across the step loop, the two values
            // would be the zoneout epilogue's only spills)
            int nu_db = nu, cells_db = cells;
            if constexpr (ZO) {
                int U2;
                asm volatile("mov.b32 %0, %1;" : "=r"(U2) : "r"(a.U));
                nu_db = max(0, min(U2, H - (jc0 + (int)rank * U2)));
                cells_db = U2 * B;
            }
#pragma unroll
            for (int k = 0; k < kRecMaxCell; ++k) {
                const auto [b, u, ok] = rec_cell(tid, k, cb[k], a.U, cells_db, nu_db);
                if (ok) {
#pragma unroll
                    for (int q = 0; q < 4; ++q) a.db_scratch[((size_t)q * B + b) * H + j0 + u] = bsum[k][q];
                }
            }
            __threadfence_block();
            asm volatile("bar.sync 1, 256;" ::: "memory");
            if (tid < 4 * a.U) {
                const int q = tid / a.U, u = tid % a.U;
                if (u < nu_db) {
                    float sacc = 0.f;
                    for (int b = 0; b < B; ++b) sacc += a.db_scratch[((size_t)q * B + b) * H + j0 + u];
                    a.db1[(size_t)q * H + j0 + u] = sacc;
                    if (a.db2) a.db2[(size_t)q * H + j0 + u] = sacc;
                }
            }
        }
    }
    __syncthreads();
    cluster_sync_all();   // no CTA leaves while a peer could still address its shared memory
    if (a.trace && threadIdx.x == 0) rec_launch_stamps(a.trace, tr, true);
}

}  // namespace zrb
