// Persistent LSTM recurrence, backward, one launch per layer (sm_90a, thread-block clusters).
//
//   for t in T-1..0:  dh_t = mask * dY_t + dG_{t+1} * W_hh ;  cell backward -> dG_t, dc      (SURVEY 8a)
//   (variational mode: the second term times the cell's recurrent multiplier m * scale(p_rec); the MMA warpgroup
//   applies it to the partial products it pushes, from flags drawn once before the step loop)
//
// The contraction dG_{t+1}[B,4H] * W_hh[4H,H] runs over the 4H gate rows.  A CTA that owned only a few
// hidden units would fill 16 of the 64 rows of a wgmma tile, so a CLUSTER owns UC units and
// splits the contraction between its CTAs; every CTA keeps its slice W_hh[rows of its share, units]^T
// (K-major, canonical no-swizzle wgmma layout, ~150 KB) resident in shared memory for all T steps.
//   S = 1  clusters of 4: CTA rank = gate, one M = 64 tile, K = H          (small H)
//   S = 2  clusters of 8: CTA rank = 2*gate + K half, two M = 64 tiles, K = H/2: half the K chain per step,
//          half the operand image to fetch
// The partial products D_r[UC x B] are exchanged as a reduce-scatter by PUSHING: the MMA warpgroup writes each
// accumulator pair straight from registers into the shared memory of the CTA that owns the row's unit
// (st.async, the bytes are counted on the owner's mbarrier: no fence, no staging pass), and the owner adds
// the partials in fixed order in its cell math.  (The alternative stages them locally, announces them with a
// cluster-scope release arrive and pulls them through DSMEM; selectable for S = 1 with ZRB_BWD_PULL=1.)
// dc lives in registers for the whole window; the bias
// gradients sum_{t,b} dG are accumulated in registers and reduced over the batch at the end of the kernel.
//
// Per step and CTA: a bulk copy of its part of its gate's dG image (47-72 KB, four pieces), H/(16*S)
// wgmma, the push exchange, U*B cell updates, one grid-barrier arrival.
// Roofline: latency / L2 bound like the forward kernel; flops per layer call 8*T*B*H^2.
#include <stdlib.h>

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
__device__ __forceinline__ float ld_dsmem_f32(uint32_t cluster_addr) {
    float v;
    asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(cluster_addr));
    return v;
}
__device__ __forceinline__ void st_dsmem_f32(uint32_t cluster_addr, float v) {
    asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(cluster_addr), "f"(v) : "memory");
}
__device__ __forceinline__ void mbar_arrive_remote_release(uint32_t cluster_addr) {
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait_acq_cluster(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// S = 1: clusters of 4 (CTA rank = gate), one M = 64 tile, the whole gate block as contraction (S = 1 also keeps the
//        staging + DSMEM-pull exchange selectable with a.push = 0).
// S = 2: clusters of 8.  The cluster owns twice the units (8U = 96 rows, two M = 64 tiles, N = 32) and CTA rank
//        r = 2*gate + half multiplies only HALF of its gate's rows: 47 K steps per step instead of 94, half the operand
//        image to fetch; the eight partial products are pushed (st.async) into the owners' shared memory and summed in
//        fixed order.
template <int S>
__global__ void __launch_bounds__(kRecThreads, 1) lstm_rec_bwd_kernel(RecBwdArgs a) {
    constexpr int CS = 4 * S;   // cluster size
    extern __shared__ uint8_t smem_raw[];
    // aligned by offsetting smem_raw itself: the compiler then knows every pointer below is a shared-memory one (LDS /
    // STS, 32-bit addresses) -- a round trip through an integer would leave them generic
    uint8_t* smem = smem_raw + ((128u - (smem_u32(smem_raw) & 127u)) & 127u);
    const int a_bytes = a.KcS * a.G * 128;     // this CTA's weight slice
    const int b_bytes = a.KcS * a.GBi * 128;   // the part of its gate's dG image this CTA multiplies with
    const int Bp = a.GBi * 8;                  // N of the MMA
    const int ldd = Bp + 1;
    uint8_t* sA = smem;
    uint8_t* sB = smem + a_bytes;
    float* sD = (float*)(sB + b_bytes);  // [64][Bp+1] this CTA's partial product, all issuers' accumulators summed (sized for two)
    uint64_t* bars = (uint64_t*)((uint8_t*)sD + 2 * 64 * ldd * 4);
    uint64_t* bar_a = bars;
    uint64_t* bar_b = bars + 1;                    // [kRecPieces]
    uint64_t* bar_mma = bars + 1 + kRecPieces;
    uint64_t* bar_part = bar_mma + 1;              // 4 arrivals per step: every CTA of the cluster staged its partial
    uint64_t* bar_recv = bar_part + 1;             // push mode: all four CTAs' partials of this CTA's units have landed
    // push mode reuses the staging buffer as the receive buffer sR[source rank][unit][batch (pitch ldr, 16-byte rows)]
    const int ldr = Bp + 4;
    float* sR = sD;

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
        mbar_init(bar_part, CS);
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
        const bool publish = a.res_flag != nullptr && blockIdx.x == 0;
        if (publish && T == 1) asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(a.res_flag), "r"(a.res_value) : "memory");
        for (int s = 1; s < T; ++s) {
            const int t = T - 1 - s;                      // step being computed; needs dG_{t+1}
            grid_counter_wait(a.counter, a.base + (unsigned int)s * a.nCTA, a.w, dead, s);
            if (publish && s == 1)   // every CTA arrived once: the whole grid is resident (or gave up: a stream gated on this must not hang)
                asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(a.res_flag), "r"(a.res_value) : "memory");
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
        const bool push = S == 2 || a.push != 0;
        const uint32_t sR_addr = smem_u32(sR), bar_recv_addr = smem_u32(bar_recv);
        // accumulator row = cluster-local unit.  Where each of this thread's (at most four) rows goes, worked out once:
        // its first float in the staging buffer, or its receive row in the owner's shared memory and the owner's mbarrier
        const int tm = (int)threadIdx.x - kRecMmaWarp * 32;
        uint32_t row_dst[2][2], row_owner[2][2], row_bar[2][2];
        bool row_ok[2][2];
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = rec_acc_row(tm, m, h);
                if (!push) {
                    row_dst[m][h] = (uint32_t)(row * ldd * 4);
                    row_owner[m][h] = 0u; row_bar[m][h] = 0u; row_ok[m][h] = true;
                } else {
                    const int owner = row / a.U, uo = row - owner * a.U;
                    row_ok[m][h] = row < UC;
                    row_owner[m][h] = row_ok[m][h] ? (uint32_t)owner : 0u;   // (rows past the cluster's are never sent)
                    row_dst[m][h] = sR_addr + (uint32_t)(((int)rank * a.U + uo) * ldr * 4);
                    row_bar[m][h] = mapa_shared(bar_recv_addr, row_owner[m][h]);
                }
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
            if (!push) {
                float* dst = (float*)((uint8_t*)sD + row_dst[m][h]) + col;
                dst[0] = v0;
                dst[1] = v1;
            } else if (row_ok[m][h]) {
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
#pragma unroll
        for (int k = 0; k < kRecMaxCell; ++k) {
            cb[k] = (tid + kRecEpiThreads * k) / a.U;
            dcreg[k] = 0.f;
#pragma unroll
            for (int q = 0; q < 4; ++q) bsum[k][q] = 0.f;
        }
        const uint64_t n_total = (uint64_t)T * B * H;
        const uint32_t sD_addr = smem_u32(sD);
        uint32_t part_addr[4];
#pragma unroll
        for (int rr = 0; rr < 4; ++rr) part_addr[rr] = mapa_shared(sD_addr, rr);   // (pull exchange: S == 1 only)
        const uint32_t bar_part_addr = smem_u32(bar_part);
        const uint32_t sR_addr = smem_u32(sR), bar_recv_addr = smem_u32(bar_recv);
        const uint32_t recv_bytes = (uint32_t)CS * (uint32_t)a.U * (uint32_t)Bp * 4u;   // CS sources x U units x Bp columns
        const float inv = 1.f / kGradScale;
        const size_t img_gate = (size_t)a.Kc * a.GBi * 64;
        const bool push = S == 2 || a.push != 0;

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
                    ct[k] = __ldg(a.cst + n * H + j);
                    cp[k] = t > 0 ? __ldg(a.cst + (n - B) * H + j) : __ldg(a.c0 + (size_t)b * H + j);
                    // (variational mode: element b*H + j of the site's stream, the mask fixed over the window)
                    dyv[k] = __ldg(a.dy + n * H + j) *
                             mask_mul1_at(a.m, (uint64_t)(a.m.period ? b : (int)n) * H + j, n_total);
                    if (a.r) dyv[k] += __ldg(a.r + n * H + j);
                }
            }
            if (s > 0) {
                if (push && tid == 0 && !dead) mbar_expect_tx(bar_recv, recv_bytes);
                bounded_mbar_wait(bar_mma, (s - 1) & 1, a.w, dead, kWaitAcc, s);
                if (tr && tid == 0) trs[s * 8 + 3] = clock64();   // staged partial / my pushes are out
                if (!push) {
                    asm volatile("bar.sync 1, 256;" ::: "memory");
                    if (tid < 4) mbar_arrive_remote_release(mapa_shared(bar_part_addr, tid));
                    {   // wait until all four CTAs of the cluster staged their partials
                        uint32_t n = 0; long long t0 = 0;
                        while (!dead && !mbar_try_wait_acq_cluster(bar_part, (s - 1) & 1)) {
                            if ((++n & 0xFFFu) == 0 && rec_spin_check(a.w, t0, kWaitPart, s)) dead = true;
                        }
                    }
                } else {
                    bounded_mbar_wait(bar_recv, (s - 1) & 1, a.w, dead, kWaitRecv, s);   // all CS x U x Bp partial sums of my units have landed
                }
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
                    if (!push) {
                        const uint32_t off = (uint32_t)(((int)rank * a.U + u) * ldd + b) * 4u;
#pragma unroll             // issue all four DSMEM loads before the first use (each is ~200+ clk)
                        for (int rr = 0; rr < 4; ++rr) pp[rr] = ld_dsmem_f32(part_addr[rr] + off);
                    } else {
#pragma unroll
                        for (int rr = 0; rr < CS; ++rr) pp[rr] = sR[(rr * a.U + u) * ldr + b];
                    }
                    float r = (pp[0] + pp[1]) + (pp[2] + pp[3]);
                    if constexpr (S == 2) r += (pp[4] + pp[5]) + (pp[6] + pp[7]);
                    dh += r * inv;
                }
                const float tc = fast_tanh(ct[k]);
                const float d_o = dh * tc;
                const float dcc = dcreg[k] + dh * go[k] * (1.f - tc * tc);
                const float d_i = dcc * gg[k], d_g = dcc * gi[k], d_f = dcc * cp[k];
                dcreg[k] = dcc * gf[k];
                float dg4[4];
                dg4[0] = d_i * gi[k] * (1.f - gi[k]);
                dg4[1] = d_f * gf[k] * (1.f - gf[k]);
                dg4[2] = d_g * (1.f - gg[k] * gg[k]);
                dg4[3] = d_o * go[k] * (1.f - go[k]);
                const int j = j0 + u;
                // critical path: the four gate images the next step multiplies with
                __half* img = a.g_img + (size_t)(t & 1) * 4 * img_gate + ((size_t)(j >> 3) * a.GBi + (b >> 3)) * 64 +
                              (b & 7) * 8 + (j & 7);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    float v = fminf(fmaxf(dg4[q] * kGradScale, -65504.f), 65504.f);
                    hv[k][q] = __float2half_rn(v);
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
            // bias gradients: per-cell sums over the window -> a global scratch [4][B][H] (no shared-memory region of
            // a guaranteed size is free: peers may still read the staging buffer) -> fixed-order sum over the batch by
            // one thread per (gate, unit) of this CTA.  bar.sync orders the CTA's own global writes for its readers.
#pragma unroll
            for (int k = 0; k < kRecMaxCell; ++k) {
                const auto [b, u, ok] = rec_cell(tid, k, cb[k], a.U, cells, nu);
                if (ok) {
#pragma unroll
                    for (int q = 0; q < 4; ++q) a.db_scratch[((size_t)q * B + b) * H + j0 + u] = bsum[k][q];
                }
            }
            __threadfence_block();
            asm volatile("bar.sync 1, 256;" ::: "memory");
            if (tid < 4 * a.U) {
                const int q = tid / a.U, u = tid % a.U;
                if (u < nu) {
                    float sacc = 0.f;
                    for (int b = 0; b < B; ++b) sacc += a.db_scratch[((size_t)q * B + b) * H + j0 + u];
                    a.db1[(size_t)q * H + j0 + u] = sacc;
                    if (a.db2) a.db2[(size_t)q * H + j0 + u] = sacc;
                }
            }
        }
    }
    __syncthreads();
    cluster_sync_all();   // no CTA leaves while a peer may still read its staged partial
    if (a.trace && threadIdx.x == 0) rec_launch_stamps(a.trace, tr, true);
}

// w_img[cluster][rank][kcl][g][rr][e] = half(W_hh[gate*H + (khalf*KcS + kcl)*8 + e, cluster*UC + g*8 + rr]) with
// rank = gate*S + khalf: one warp per (cluster, rank, kcl) reads 8 rows x UC contiguous floats and writes one contiguous
// 16*UC-byte block.
// m active (weight drop): W[r, j] * the multiplier of element r*H + j, four consecutive u per lane (one Philox call per
// quad of mask elements; rows8 is a multiple of 8, so a quad of u never changes e)
__global__ void pack_whh_bwd_kernel(const float* __restrict__ W, __half* __restrict__ img, int H, int UC, int G, int KcS,
                                    int S, int nCluster, MaskSrc m) {
    __shared__ __half tile[8][8 * 128];
    const int warp_in_block = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int CS = 4 * S;
    const long long total = (long long)nCluster * CS * KcS;
    for (long long w = (long long)blockIdx.x * 8 + warp_in_block; w < total; w += (long long)gridDim.x * 8) {
        const int kcl = (int)(w % KcS);
        const int r = (int)((w / KcS) % CS);
        const int cl = (int)(w / ((long long)KcS * CS));
        const int gate = r / S, khalf = r % S;
        __half* t = tile[warp_in_block];
        const int rows8 = G * 8;
        if (m.active) {
            for (int idx = lane * 4; idx < 8 * rows8; idx += 128) {
                const int e = idx / rows8, u0 = idx % rows8;
                const int k = (khalf * KcS + kcl) * 8 + e, j0 = cl * UC + u0;
                const size_t row = (size_t)gate * H + k;
                float mul[4] = {0.f, 0.f, 0.f, 0.f};
                if (k < H && u0 < UC && j0 < H) mask_mul4_at(m, row * H + j0, mul);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int u = u0 + q, j = j0 + q;
                    t[u * 8 + e] = __float2half_rn((k < H && u < UC && j < H) ? W[row * H + j] * mul[q] : 0.f);
                }
            }
        } else {
            for (int idx = lane; idx < 8 * rows8; idx += 32) {
                int e = idx / rows8, u = idx % rows8;            // u fastest: contiguous global reads
                int k = (khalf * KcS + kcl) * 8 + e, j = cl * UC + u;
                float v = (k < H && u < UC && j < H) ? W[((size_t)gate * H + k) * H + j] : 0.f;
                t[u * 8 + e] = __float2half_rn(v);
            }
        }
        __syncwarp();
        __half* dst = img + (((size_t)cl * CS + r) * KcS + kcl) * ((size_t)G * 64);
        for (int idx = lane; idx < rows8 * 8; idx += 32) dst[idx] = t[idx];
        __syncwarp();
    }
}

int rec_bwd_plan(int H, int B, RecPlan* plan) {
    int nsm = tc_num_sms();
    plan->GB = (B + 7) / 8;
    plan->ok = 0;
    plan->KS = 1;
    if (plan->GB * 8 > 32) return ZRB_OK;
    static const bool no_split = getenv("ZRB_REC_NOSPLIT") != nullptr;   // A/B switch
    // clusters of 8, half a gate block per CTA (see the kernel header); image batch groups padded to an even count
    if (!no_split && H >= 256) {
        const int Kp = (H + 31) / 32 * 32, Kc = Kp / 8, KcS = Kc / 2, GBi = (plan->GB + 1) / 2 * 2;
        // first choice: at most one (unit, batch) cell per epilogue thread (see rec_fwd_plan)
        for (int pass = 0; pass < 2; ++pass)
            for (int U = 16; U >= 1; --U) {
                const int UC = 8 * U;
                if (UC > 128) continue;
                const int ncl = (H + UC - 1) / UC;
                if (ncl * 8 > nsm) break;
                if (U * B > (pass == 0 ? 1 : kRecMaxCell) * kRecEpiThreads) continue;
                const int G = UC / 8;
                const size_t smem = rec_smem_bytes(KcS, G, GBi);
                if (smem <= 227 * 1024 && 8 * U * (GBi * 8 + 4) <= 2 * 64 * (GBi * 8 + 1)) {
                    // the GPCs cannot hold that many 8-CTA clusters
                    if (rec_max_clusters((const void*)lstm_rec_bwd_kernel<2>, 8, (int)smem, 8 * 64) < ncl) continue;
                    plan->KS = 2; plan->U = U; plan->G = G; plan->nCTA = ncl * 8; plan->smem = (int)smem;
                    plan->Kc = Kc; plan->KcS = KcS; plan->GBi = GBi;
                    return rec_plan_finish(plan, (const void*)lstm_rec_bwd_kernel<2>, 8);
                }
            }
    }
    int Kp = (H + 15) / 16 * 16;
    plan->Kc = Kp / 8;
    plan->KcS = plan->Kc;
    plan->GBi = plan->GB;
    int max_clusters = (nsm - 16) / 4;   // clusters of 4 strand up to 16 SMs (GPC remainders)
    for (int U = 16; U >= 1; --U) {
        int UC = 4 * U;
        if (UC % 8) continue;
        int ncl = (H + UC - 1) / UC;
        if (ncl > max_clusters) break;
        int G = UC / 8;
        size_t smem = rec_smem_bytes(plan->Kc, G, plan->GB);
        if (smem <= 227 * 1024 && U * B <= kRecMaxCell * kRecEpiThreads) {
            plan->U = U; plan->G = G; plan->nCTA = ncl * 4; plan->smem = (int)smem;
            return rec_plan_finish(plan, (const void*)lstm_rec_bwd_kernel<1>, 4);
        }
    }
    return ZRB_OK;
}

int pack_whh_bwd(const float* W, __half* img, int H, const RecPlan& p, cudaStream_t s, MaskSrc m) {
    const int CS = 4 * p.KS;
    pack_whh_bwd_kernel<<<tc_num_sms() * 4, 256, 0, s>>>(W, img, H, CS * p.U, p.G, p.KcS, p.KS, p.nCTA / CS, m);
    ZRB_KERNEL_CHECK();
    return ZRB_OK;
}

int lstm_rec_bwd(const RecPlan& p, const RecWatchdog& wd, RecBwdArgs a, cudaStream_t s) {
    ZRB_REQUIRE(!a.db1 || a.db_scratch, "bias gradients need the scratch buffer");
    static const bool pull = getenv("ZRB_BWD_PULL") != nullptr;   // A/B switch: the r01 staging + DSMEM-pull exchange (S = 1)
    a.push = pull ? 0 : 1;
    a.U = p.U; a.G = p.G; a.GB = p.GB; a.Kc = p.Kc; a.nCTA = p.nCTA; a.KcS = p.KcS; a.GBi = p.GBi;
    if (!a.rm.active) a.rm.scale = 1.f;   // (the epilogue multiplies by it unconditionally)
    ZRB_REQUIRE(wd.flag && wd.host, "lstm_rec_bwd needs the context's watchdog words");
    a.w = rec_watch_args(wd);
    a.base += rec_fault_base("bwd");   // (tests only)
    if (a.trace) ZRB_CUDA(cudaMemsetAsync(a.trace + 4, 0x80, 2 * sizeof(long long), s));
    void* args[] = {&a};
    return rec_launch(p, args, a.trace != nullptr, s, "lstm_rec_bwd");
}

}  // namespace zrb
