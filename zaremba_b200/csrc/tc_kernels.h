// Launchers used only by the tensor-core engine.
#pragma once
#include "kernels.h"
#include "tc_host.h"

namespace zrb {

constexpr float kGradScale = 1024.f;   // fp16 gradient images hold kGradScale * value (exact power of two)

// m (weight drop, DESIGN.md section 15; inactive by default): src element r*ld_src + c times its multiplier first
int convert_pad_f16(const float* src, int64_t ld_src, __half* dst, int64_t ld_dst, int rows, int cols, float scale,
                    cudaStream_t s, MaskSrc m = MaskSrc{});
int colsum_h_scratch_floats(int M);
int colsum_h(const __half* A, int64_t ld, float* out, float* out2, int N, int M, float inv_scale, float* scratch,
             cudaStream_t s);

// ---- Mixture-of-Softmaxes head (mos.cu; DESIGN.md section 19) ----------------------------------------------------
// ua [rows, ldu]: the head GEMM's output, latent u in columns [0, K*E), prior a in [Ua, Ua + K).  Logits Z [rows*K, V],
// row r*K + k = expert k of token r; lse [rows*K].  K <= ZRB_MAX_EXPERTS (one warp holds a token's K statistics).
// c = tanh(u + b) back into ua, and lat_h row r*K + k = half(c * the latent mask of element (row0 + r)*K*E + j)
int mos_latent_fwd(float* ua, int64_t ldu, const float* b, __half* lat_h, int64_t ld_l, int rows, int K, int E,
                   int64_t row0, MaskSrc m, cudaStream_t s);
// dua_h columns [0, K*E) = kGradScale * dlat * mask * (1 - c^2), c from ua; dlat [N*K, E] fp32
int mos_latent_bwd(const float* dlat, const float* ua, int64_t ldu, __half* dua_h, int64_t ld_d, int N, int K, int E,
                   MaskSrc m, cudaStream_t s);
int mos_lse(const float* Z, int rows, int V, float* lse, cudaStream_t s);
// the mixture NLL of the train step: row_loss, loss = B/N sum, the scaled fp16 dz rows into ds_h and da into the
// columns [Ua, Ua + K) of dua_h
int mos_nll_grad(const float* Z, const float* lse, const float* ua, int64_t ldu, int Ua, const int64_t* y, int N, int K,
                 int V, int B, float* row_loss, float* loss, __half* ds_h, int64_t ld_s, __half* dua_h, int64_t ld_d,
                 cudaStream_t s);
// eval mode: row_loss, loss (or null) and tgt_prob = p[y] (or null)
int mos_nll_eval(const float* Z, const float* lse, const float* ua, int64_t ldu, int Ua, const int64_t* y, int N, int K,
                 int V, int B, float* row_loss, float* loss, float* tgt_prob, cudaStream_t s);
// out [rows, ldo] = log p
int mos_logp(const float* Z, const float* lse, const float* ua, int64_t ldu, int Ua, int rows, int K, int V, float* out,
             int64_t ldo, cudaStream_t s);
// the drop-in backward from G = dL / d log p [N, V]: dz into ds_h and da into dua_h.  Scratch: P [N, V], s_buf [N*K]
int mos_vjp(const float* Z, const float* lse, const float* ua, int64_t ldu, int Ua, int N, int K, int V, const float* G,
            float* P, float* s_buf, __half* ds_h, int64_t ld_s, __half* dua_h, int64_t ld_d, cudaStream_t s);

// cell pointwise with fp16 side outputs (tc_cell.cu).  rm: recurrent mask of element b*H + j (variational mode), applied
// to h_raw_h (the next step's operand) forward and to dh_rec backward
struct ZoneoutSrc;
// zo (or null: the mode off; zoneout, DESIGN.md section 20): h_prev [B,H] is h_{t-1} and c_til [B,H] receives c~_t
int lstm_cell_fwd_tc(float* pre, const float* c_prev, float* c_out, float* h_raw, __half* h_raw_h, __half* y_h,
                     int64_t ld_h, int B, int H, int64_t elem_off, int64_t n_total, MaskSrc m, MaskSrc rm, cudaStream_t s,
                     const ZoneoutSrc* zo = nullptr, const float* h_prev = nullptr, float* c_til = nullptr);
// zo (or null): c_t is c~_t and hcarry [B,H] the carried zh * dh (read, then overwritten; zero at t = T-1)
int lstm_cell_bwd_tc(const float* dy_post, const float* dh_rec, float* dc, const float* gates, const float* c_t,
                     const float* c_prev, float* dG, __half* dG_h, int64_t ld_g, int B, int H, int64_t elem_off,
                     int64_t n_total, MaskSrc m, MaskSrc rm, cudaStream_t s, const float* r = nullptr,
                     const ZoneoutSrc* zo = nullptr, float* hcarry = nullptr);
// r [B,H] (or null): the AR/TAR gradient of this step (DESIGN.md section 17), added to dh after the output mask

// Zoneout of one layer (DESIGN.md section 20).  Train mode (flags non-null): unit (t, b, j) keeps c_{t-1} where bit 0 of
// flags[t*B*H + b*H + j] is set, and h_{t-1} where bit 1 is (zoneout_flags).  Eval mode (flags null): the expectation
// c_t = fma(ec, c_{t-1}, ec1 * c~_t) and h_t = fma(eh, h_{t-1}, eh1 * h~_t).
struct ZoneoutSrc {
    const uint8_t* flags;     // [T*B*H] or null
    float ec, ec1, eh, eh1;   // fp32(z_c), fp32(1 - z_c), fp32(z_h), fp32(1 - z_h)
    int on;                   // the mode is on (z_c > 0 or z_h > 0): the kernels take the zoneout instantiations
};
// flags[e] = (dropped flag of element e of c's stream) | (dropped flag of element e of h's stream) << 1, e < n: one
// Philox call per site and quad of elements, drawn before the layer's recurrence so that neither recurrence kernel holds
// the generator's registers
int zoneout_flags(MaskSrc c, MaskSrc h, int64_t n, uint8_t* flags, cudaStream_t s);

// ---- persistent recurrence (lstm_rec_fwd.cu / lstm_rec_bwd.cu) ---------------------------------------
struct RecPlan {
    int ok;      // shape fits the persistent kernel (else the per-timestep path is used)
    int U;       // hidden units per CTA
    int G;       // 8-row groups of the weight slice (ceil(4U/8))
    int GB;      // 8-row groups of the batch operand (ceil(B/8))
    int Kc;      // 8-element K chunks of the whole contraction
    int nCTA;
    int smem;
    int KS;      // K-split: CTAs that share one set of output rows, each holding 1/KS of the contraction (clusters)
    int KcS;     // K chunks per CTA (Kc / KS)
    int GBi;     // 8-row batch groups of the operand images (GB; the K-split plans: rec_split_groups(GB))
    const void* kernel;   // the instantiation launched: lstm_rec_fwd_kernel<KS == 2> / lstm_rec_bwd_kernel<KS>
    int cluster;          // CTAs per thread-block cluster: 1 (unsplit forward), 2, 4 or 8
    int max_clusters;     // cudaOccupancyMaxActiveClusters at this cluster size and smem (0: the query failed)
    int beside_smem;      // dynamic shared memory per block that keeps a kernel launched beside this grid off its SMs:
                          // one byte more than an SM has left after one of its CTAs (the SM's shared memory less smem
                          // and two blocks' reserved shares)
};
size_t rec_smem_bytes(int Kc, int G, int GB);
int rec_split_groups(int GB);   // GBi of the K-split plans (see the definition)
// cudaOccupancyMaxActiveClusters of `kernel` on a grid of nCTA in clusters of `cluster`, after raising its dynamic
// shared-memory limit; 0 if either call fails, with the error cleared
int rec_max_clusters(const void* kernel, int cluster, int smem, int nCTA);
// the plan fits: record the kernel it launches, its cluster size, occupancy answer and beside_smem, and set ok
int rec_plan_finish(RecPlan* plan, const void* kernel, int cluster);
// launch the plan's kernel with args = {&RecFwdArgs} or {&RecBwdArgs}; the launch modes are described at the definition
// (lstm_rec_fwd.cu).  trace: the launch records a trace (never programmatic); name: for error messages
int rec_launch(const RecPlan& p, void** args, bool trace, cudaStream_t s, const char* name);
// the zoneout instantiations of the two kernels (lstm_rec_zoneout.cu): the forward with or without the K split, the
// backward for S = 1 or 2, with their shared-memory limit raised on the current device (null when that fails, the error
// set); the plans' occupancy answers hold for them (same shared memory, one CTA per SM, no spill)
const void* rec_fwd_zoneout_kernel(bool split);
const void* rec_bwd_zoneout_kernel(int S);
// Where a persistent kernel that gave up on a wait (rec_common.cuh: watchdog) reports it: `flag` is the device word the
// spinning threads poll, `host` a mapped host word the host reads without synchronising.  Owned by the context.
struct RecWatchdog {
    unsigned int* flag = nullptr;
    unsigned int* host = nullptr;
};
// ... and the kernels' copy of it, one per launch (rec_common.cuh: rec_watch_args)
struct RecWatch {
    unsigned int* flag;       // device word polled by the spinning threads (0 = healthy)
    unsigned int* host;       // mapped host word the first thread to give up writes the code to
    long long spin_cycles;    // ~3 s at 2 GHz unless ZRB_SPIN_CYCLES says otherwise
};
int rec_fwd_plan(int H, int B, RecPlan* plan);
// m (weight drop, DESIGN.md section 15; inactive by default): the image of fp32(W[r, k] * multiplier of r*H + k)
int pack_whh_fwd(const float* W, __half* img, int H, const RecPlan& p, cudaStream_t s, MaskSrc m = MaskSrc{});
struct RecFwdArgs {
    const __half* w_img;      // [nCTA][KcS][G][8][8]  (K-split: CTA = (pair, K half))
    const __half* h0_img;     // [Kc][GB][8][8] image of the state entering the window: the B operand of step 0
    __half* h_img;            // [T+1][Kc][GB][8][8]; image t (t >= 1) is the B operand of step t, written by step t-1
    float* gates;             // [N,4H] in: x-part pre-activations (+biases); out: activated gates
    const float* c0;          // [B,H]
    float* cst;               // [N,H]
    float* h_last;            // [B,H] or null
    float* c_last;            // [B,H] or null
    __half* hprev_h;          // [N+B,Hp] row-major, rows B.. written here
    __half* y_h;              // [N,Hp] row-major dropout(h)
    float* h_f32;             // or null: [N,H] fp32 h_t (the unit-level entry point zrb_lstm_layer_fwd returns it)
    unsigned int* counter;    // grid barrier: never reset, `base` is its value when this launch starts
    unsigned int base;
    int T, B, H, Hp, U, G, GB, Kc, nCTA;
    int KcS, GBi;             // K chunks per CTA (Kc / KS); 8-row batch groups of the operand image (RecPlan::GBi)
    MaskSrc m;                // the output site's dropout (period B*H: variational mode, fixed over the window)
    MaskSrc rm;               // variational mode: recurrent mask of element b*H + j on h_{t-1} (operand images, hprev_h)
    RecWatch w;               // watchdog (rec_common.cuh)
    long long* trace;         // optional (profiling): [8] launch stamps (rec_launch_stamps) + [T][8] clock64 stamps of CTA 0
    // zoneout (zo.on: the launch takes the zoneout instantiation; appended, so the other fields keep their offsets)
    ZoneoutSrc zo;
    const float* h0;          // [B,H] h entering the window (h_{-1} of the select)
    float* ctil;              // [N,H] c~_t, the cell value before the select (the backward reads it)
};
// Launch the forward recurrence with a's per-call fields; the launcher sets the plan's fields (U, G, GB, Kc, nCTA, KcS,
// GBi) and the watchdog's.  rm is never applied to h_last, h_f32 or the input of m.
int lstm_rec_fwd(const RecPlan& p, const RecWatchdog& wd, RecFwdArgs a, cudaStream_t s);
// Everything the forward needs from the incoming state and tokens in ONE launch (it replaced 9: five device
// copies, two fp16 conversions, two image packs): h0s/c0s = copies of the incoming (h, c) (the caller may pass
// the same buffers for the outgoing state), hprev_h rows [0,B) = half(h0) with zeroed pad columns, h0_img = the
// UMMA-layout image [kc][g][r][e] = half(h0[b = g*8+r, k = kc*8+e]) (null: not built), x_saved = x.  Variational mode:
// the half(h0) rows and the image hold h0 * rm[l] (element b*H + k); h0s stays unmasked.
struct FwdPrep {
    const float* in_h[ZRB_MAX_LAYERS];
    const float* in_c[ZRB_MAX_LAYERS];
    float* h0s[ZRB_MAX_LAYERS];
    float* c0s[ZRB_MAX_LAYERS];
    __half* hprev_h[ZRB_MAX_LAYERS];
    __half* h0_img[ZRB_MAX_LAYERS];
    MaskSrc rm[ZRB_MAX_LAYERS];
    const int64_t* x;
    int64_t* x_saved;
    int H[ZRB_MAX_LAYERS], Hp[ZRB_MAX_LAYERS];   // layer l's width and the pitch of its hprev_h rows
    int GB[ZRB_MAX_LAYERS], Kc[ZRB_MAX_LAYERS];  // ... and the shape of its h0_img (layer l's forward plan)
    int L, B, N;
};
int fwd_prep(const FwdPrep& a, cudaStream_t s);
// The fp16 operand images of one weight matrix, as the fused update rewrites them from registers.  Default: no image.
struct WeightImages {
    __half* row = nullptr;           // [rows, ld] row-major image
    int64_t ld = 0;
    __half* fwd = nullptr;           // forward recurrent slices (pack_whh_fwd's layout) under fplan
    const RecPlan* fplan = nullptr;
    __half* bwd = nullptr;           // backward recurrent slices (pack_whh_bwd's layout) under bplan
    const RecPlan* bplan = nullptr;
};
// SGD update of one matrix fused with its fp16 image rebuild (optim_tc.cu)
int update_pack(float* p, float* g, int rows, int cols, float lr, const float* scalars, const WeightImages& img,
                bool write_g, cudaStream_t s,
                int pdl_smem = 0);   // > 0: programmatic dependent of the forward recurrence kernel enqueued before it,
                                     // each block requesting this much dynamic shared memory (rec_beside_smem)
// the same kernels with the dynamic-evaluation rule (dyneval_elem): theta_g tg and r at p's offsets (r unused under the
// SGD rule, a.rbar null); g is read, never written; the same images
int update_pack_dyn(float* p, float* g, const float* tg, const float* r, int rows, int cols, const DynArgs& a,
                    const WeightImages& img, cudaStream_t s);
// iterate averaging (average_tc.cu, DESIGN.md section 16): update_pack's update, then a = first ? p : a + (p - a) * mu
// over the new p in the same pass; the same images
int update_pack_avg(float* p, float* g, float* a, float mu, bool first, int rows, int cols, float lr,
                    const float* scalars, const WeightImages& img, bool write_g, cudaStream_t s, int pdl_smem = 0);
// Adam (adam_tc.cu, DESIGN.md section 21): adam_apply's element rule with the moments m and v at p's offsets, in place of
// update_pack's SGD; the same images
int update_pack_adam(float* p, float* g, float* m, float* v, const AdamScalars& k, int rows, int cols,
                     const float* scalars, const WeightImages& img, bool write_g, cudaStream_t s, int pdl_smem = 0);
// exchange p and a, and write the images of the new p (update_pack's image stores)
int swap_pack(float* p, float* a, int rows, int cols, const WeightImages& img, cudaStream_t s);
int rec_bwd_plan(int H, int B, RecPlan* plan);   // U = units per CTA, nCTA = 4 * clusters
int pack_whh_bwd(const float* W, __half* img, int H, const RecPlan& p, cudaStream_t s, MaskSrc m = MaskSrc{});
struct RecBwdArgs {
    const __half* w_img;      // [nCluster][4][Kc][G][8][8]
    __half* g_img;            // [2][4][Kc][GB][8][8] ring: slot (t & 1) holds kGradScale * dG_t per gate
    const float* dy;          // [N,H] grad wrt the layer's dropout'ed output
    const float* r;           // [N,H] or null: AR/TAR gradient added after the mask (DESIGN.md section 17)
    const float* gates;       // [N,4H] activated (i,f,g,o)
    const float* cst;         // [N,H]
    const float* c0;          // [B,H]
    __half* dG_h;             // [N,G4p] row-major, kGradScale * dG
    float* db1;               // [4H] or null: bias gradient sum_{t,b} dG (model.py:35-36: b_ih and b_hh get the same
    float* db2;               //      gradient), accumulated in registers over the window and reduced over the batch here
    float* db_scratch;        // [4][B][H] fp32 scratch of that reduction (needed when db1 is set)
    unsigned int* counter;    // grid barrier: never reset, `base` is its value when this launch starts
    unsigned int base;
    int T, B, H, G4p, U, G, GB, Kc, nCTA;
    int KcS, GBi;             // K chunks per CTA (Kc / S); 8-row batch groups of the dG images (RecPlan::GBi)
    MaskSrc m;                // the output site's dropout (period B*H: variational mode, fixed over the window)
    MaskSrc rm;               // variational mode: recurrent mask of element b*H + j; scales the recurrent gradient
    RecWatch w;               // watchdog (rec_common.cuh)
    long long* trace;         // optional (profiling): [8] launch stamps (rec_launch_stamps) + [T][8] clock64 stamps of CTA 0
    ZoneoutSrc zo;            // zoneout (zo.on: the zoneout instantiation; the forward's flags), appended like RecFwdArgs'
    const float* ctil;        // [N,H] c~_t of the forward (zo.on)
};
// Launch the backward recurrence with a's per-call fields; the launcher sets the plan's and the watchdog's fields.
int lstm_rec_bwd(const RecPlan& p, const RecWatchdog& wd, RecBwdArgs a, cudaStream_t s);

}  // namespace zrb
