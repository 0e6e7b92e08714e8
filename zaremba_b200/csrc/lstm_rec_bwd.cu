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
// the partials in fixed order in its cell math.
// dc lives in registers for the whole window; the bias
// gradients sum_{t,b} dG are accumulated in registers and reduced over the batch at the end of the kernel.
//
// Per step and CTA: a bulk copy of its part of its gate's dG image (47-72 KB, four pieces), H/(16*S)
// wgmma, the push exchange, U*B cell updates, one grid-barrier arrival.
// Roofline: latency / L2 bound like the forward kernel; flops per layer call 8*T*B*H^2.
#include <stdlib.h>

#include "lstm_rec_bwd.cuh"

namespace zrb {

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
    // clusters of 8, half a gate block per CTA (see the kernel header); the dG images' batch groups: rec_split_groups
    if (H >= 256) {
        const int Kp = (H + 31) / 32 * 32, Kc = Kp / 8, KcS = Kc / 2, GBi = rec_split_groups(plan->GB);
        // first choice: as in rec_fwd_plan (rec_split_first_choice)
        for (int pass = 0; pass < 2; ++pass)
            for (int U = 16; U >= 1; --U) {
                const int UC = 8 * U;
                if (UC > 128) continue;
                const int ncl = (H + UC - 1) / UC;
                if (ncl * 8 > nsm) break;
                if (U * B > kRecMaxCell * kRecEpiThreads || (pass == 0 && !rec_split_first_choice(U, B, 8 * ncl, nsm)))
                    continue;
                const int G = UC / 8;
                const size_t smem = rec_smem_bytes(KcS, G, GBi);
                if (smem <= 227 * 1024 && 8 * U * (GBi * 8 + 4) <= 2 * 64 * (GBi * 8 + 1)) {
                    // the GPCs cannot hold that many 8-CTA clusters
                    if (rec_max_clusters((const void*)lstm_rec_bwd_kernel<2, false>, 8, (int)smem, 8 * 64) < ncl) continue;
                    plan->KS = 2; plan->U = U; plan->G = G; plan->nCTA = ncl * 8; plan->smem = (int)smem;
                    plan->Kc = Kc; plan->KcS = KcS; plan->GBi = GBi;
                    return rec_plan_finish(plan, (const void*)lstm_rec_bwd_kernel<2, false>, 8);
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
            return rec_plan_finish(plan, (const void*)lstm_rec_bwd_kernel<1, false>, 4);
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
    a.U = p.U; a.G = p.G; a.GB = p.GB; a.Kc = p.Kc; a.nCTA = p.nCTA; a.KcS = p.KcS; a.GBi = p.GBi;
    if (!a.rm.active) a.rm.scale = 1.f;   // (the epilogue multiplies by it unconditionally)
    ZRB_REQUIRE(wd.flag && wd.host, "lstm_rec_bwd needs the context's watchdog words");
    a.w = rec_watch_args(wd);
    a.base += rec_fault_base("bwd");   // (tests only)
    if (a.trace) ZRB_CUDA(cudaMemsetAsync(a.trace + 4, 0x80, 2 * sizeof(long long), s));
    void* args[] = {&a};
    if (!a.zo.on) return rec_launch(p, args, a.trace != nullptr, s, "lstm_rec_bwd");
    ZRB_REQUIRE(a.ctil, "zoneout needs the forward's c~ buffer");
    RecPlan q = p;   // the same plan through the zoneout instantiation (same shared memory and cluster shape)
    q.kernel = rec_bwd_zoneout_kernel(p.KS);
    if (!q.kernel) return ZRB_E_CUDA;
    return rec_launch(q, args, a.trace != nullptr, s, "lstm_rec_bwd (zoneout)");
}

}  // namespace zrb
