// ZRB_ENGINE_TC: every dense contraction of the path on wgmma tensor cores (fp16 operands,
// fp32 accumulation), pointwise math and state in fp32.
//
// fp16 images (K = contraction index):
//   w_ih_h[l], w_hh_h[l] [4H, Hp]   read K-major by the forward GEMMs (X*W^T, h*W^T) and MN-major
//   fc_w_h               [V,  Hp]   by the dgrads (dG*W, dS*W): one image serves both
//   x_h[l]      [N, Hp]  dropout'ed input of layer l (x_h[L] feeds the projection); MN-major B of wgrads
//   hprev_h[l]  [N+B,Hp] rows 0..B-1 = h entering the window, rows B.. = h_t: row block t is h_{t-1}
//                        (variational mode: times the layer's recurrent mask, so the dW_hh GEMM needs no change)
//   dG_h        [N, G4p] kGradScale * dG;  dS_h [N, Vp] kGradScale * dscores
// Gradient images are scaled by an exact power of two and unscaled by the consuming GEMM's alpha.
#include "engine.h"
#include <stdlib.h>
#include <string.h>

#include "tc_kernels.h"

struct zrb_tc_state {
    int Hp = 0, G4p = 0, Vp = 0;
    int device = 0;
    __half* w_ih_h[ZRB_MAX_LAYERS] = {};
    __half* w_hh_h[ZRB_MAX_LAYERS] = {};
    __half* fc_w_h = nullptr;
    __half* x_h[ZRB_MAX_LAYERS + 1] = {};
    __half* hprev_h[ZRB_MAX_LAYERS] = {};
    __half* dG_h = nullptr;            // scaled dG of the layer being differentiated ...
    __half* dG_h_alt = nullptr;        // ... double-buffered by layer parity: the weight gradients of layer l run
                                       //     underneath the recurrence of layer l-1, which writes the other buffer
    __half* dS_h = nullptr;
    // weight-gradient GEMMs deferred to run as programmatic dependents of the NEXT backward recurrence kernel (on the
    // ~20 SMs it leaves idle): 0 none, 1 = fc.W, 2 = (w_ih, w_hh) of layer `pending_layer`
    int pending = 0, pending_layer = 0;
    bool defer_wgrad = false;
    // deferred weight updates (zrb_set_lazy_update): items 1..L-1 = (w_ih, w_hh) of that layer, item L = fc.W; bit i of
    // upd_pending set = item i still to be applied with the (lr, coef in c->scalars[1]) of the step that deferred it
    unsigned upd_pending = 0;
    float upd_lr = 0.f;
    zrb::TensorList upd_tl{};
    bool in_train_step = false;   // tc_forward is running as the first half of a fused train step
    float* colsum_scratch = nullptr;   // row-split partials of the bias-gradient column sums
    int64_t packed_version = 0;
    zrb_params packed_params{};
    std::vector<void*> allocs;
    // persistent recurrence
    zrb::RecPlan fplan{};
    __half* w_img_f[ZRB_MAX_LAYERS] = {};
    __half* h0_img[ZRB_MAX_LAYERS] = {};   // image of the state entering the window (step 0's B operand)
    __half* h_img = nullptr;
    unsigned int* counter = nullptr;       // [0]: forward grid barrier, [32]: backward; never reset between launches,
    unsigned int cnt_f = 0, cnt_b = 0;     // their values when the next launch starts
    zrb::RecPlan bplan{};
    __half* w_img_b[ZRB_MAX_LAYERS] = {};
    __half* g_img = nullptr;
    long long* trace = nullptr;   // [2][8 + T*8]: launch stamps + per-step clock stamps (zrb_prof_rec_trace)
    // fused step (zrb_set_embed_sparse): the wgrad GEMMs leave sums of squares of the matrix gradients in
    // c->partials, so clip_grad_norm_ does not re-read them; valid for the gradient buffers keyed by wg_key
    bool wg_ok = false;
    int wg_slots = 0;
    const float* wg_key = nullptr;
};

namespace zrb {

static bool prof_keeps_pdl();
static int pad64(int n) { return (n + 63) / 64 * 64; }

template <typename T>
static int tc_alloc(zrb_ctx* c, T** p, size_t count) {
    void* q = nullptr;
    size_t bytes = count * sizeof(T);
    cudaError_t e = cudaMalloc(&q, bytes);
    if (e != cudaSuccess) {
        set_error("cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
        return ZRB_E_NOMEM;
    }
    cudaMemset(q, 0, bytes);
    c->tc->allocs.push_back(q);
    c->bytes += (int64_t)bytes;
    *p = (T*)q;
    return ZRB_OK;
}

static inline RecWatchdog tc_watchdog(const zrb_ctx* c) {
    RecWatchdog wd;
    wd.flag = c->wd_flag; wd.host = c->wd_host;
    return wd;
}

int tc_ctx_init(zrb_ctx* c) {
    int major = 0, dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    if (major != 9) {
        set_error("the tensor-core engine needs an sm_90 device (found compute capability %d.x)", major);
        return ZRB_E_INVALID;
    }
    c->tc = new zrb_tc_state();
    zrb_tc_state* t = c->tc;
    t->device = dev & 63;
    g_live_tc_ctx[t->device].fetch_add(1);
    const int H = c->cfg.hidden, L = c->cfg.layers, V = c->cfg.vocab;
    const size_t N = (size_t)c->cfg.max_seq * c->cfg.max_batch, B = c->cfg.max_batch;
    t->Hp = pad64(H); t->G4p = pad64(4 * H); t->Vp = pad64(V);
    for (int l = 0; l < L; ++l) {
        ZRB_TRY(tc_alloc(c, &t->w_ih_h[l], (size_t)4 * H * t->Hp));
        ZRB_TRY(tc_alloc(c, &t->w_hh_h[l], (size_t)4 * H * t->Hp));
        ZRB_TRY(tc_alloc(c, &t->hprev_h[l], (N + B) * t->Hp));
    }
    for (int l = 0; l <= L; ++l) ZRB_TRY(tc_alloc(c, &t->x_h[l], N * t->Hp));
    ZRB_TRY(tc_alloc(c, &t->fc_w_h, (size_t)V * t->Hp));
    ZRB_TRY(tc_alloc(c, &t->dG_h, N * t->G4p));
    ZRB_TRY(tc_alloc(c, &t->dG_h_alt, N * t->G4p));
    ZRB_TRY(tc_alloc(c, &t->dS_h, N * t->Vp));
    ZRB_TRY(tc_alloc(c, &t->colsum_scratch, (size_t)colsum_h_scratch_floats(V > 4 * H ? V : 4 * H)));
    ZRB_TRY(rec_fwd_plan(H, c->cfg.max_batch, &t->fplan));
    const char* force = getenv("ZRB_REC");
    if (force && !strcmp(force, "steps")) t->fplan.ok = 0;   // A/B switch: per-timestep launches
    if (t->fplan.ok) {
        const RecPlan& fp = t->fplan;
        for (int l = 0; l < L; ++l) {
            ZRB_TRY(tc_alloc(c, &t->w_img_f[l], (size_t)fp.nCTA * fp.KcS * fp.G * 64 + 16 * 64 /* M=128 over-read */));
            ZRB_TRY(tc_alloc(c, &t->h0_img[l], (size_t)fp.Kc * fp.GBi * 64));
        }
        ZRB_TRY(tc_alloc(c, &t->h_img, (size_t)(c->cfg.max_seq + 1) * fp.Kc * fp.GBi * 64));
        ZRB_TRY(tc_alloc(c, &t->counter, 64));
    }
    if (getenv("ZRB_REC_TRACE")) ZRB_TRY(tc_alloc(c, &t->trace, (size_t)2 * (8 + c->cfg.max_seq * 8)));
    ZRB_TRY(rec_bwd_plan(H, c->cfg.max_batch, &t->bplan));
    if (!t->fplan.ok || (force && !strcmp(force, "fwdonly"))) t->bplan.ok = 0;
    if (t->bplan.ok) {
        const RecPlan& bp = t->bplan;
        for (int l = 0; l < L; ++l) ZRB_TRY(tc_alloc(c, &t->w_img_b[l], (size_t)bp.nCTA * bp.KcS * bp.G * 64 + 16 * 64));
        ZRB_TRY(tc_alloc(c, &t->g_img, (size_t)2 * 4 * bp.Kc * bp.GBi * 64));
    }
    return ZRB_OK;
}

void tc_ctx_free(zrb_ctx* c) {
    if (!c->tc) return;
    g_live_tc_ctx[c->tc->device].fetch_sub(1);
    for (void* p : c->tc->allocs) cudaFree(p);
    delete c->tc;
    c->tc = nullptr;
}

// rebuild the fp16 weight images when parameter values changed (main.py:116-117 / zrb_clip_sgd)
static int tc_pack_weights(zrb_ctx* c, const zrb_params* p, cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    if (t->packed_version == c->weights_version && !memcmp(&t->packed_params, p, sizeof(*p))) return ZRB_OK;
    ProfScope ps(c, ZRB_PROF_PACK, s);
    const int H = c->cfg.hidden, L = c->cfg.layers, V = c->cfg.vocab;
    for (int l = 0; l < L; ++l) {
        ZRB_TRY(convert_pad_f16(p->w_ih[l], H, t->w_ih_h[l], t->Hp, 4 * H, H, 1.f, s));
        ZRB_TRY(convert_pad_f16(p->w_hh[l], H, t->w_hh_h[l], t->Hp, 4 * H, H, 1.f, s));
        if (t->fplan.ok) ZRB_TRY(pack_whh_fwd(p->w_hh[l], t->w_img_f[l], H, t->fplan, s));
        if (t->bplan.ok) ZRB_TRY(pack_whh_bwd(p->w_hh[l], t->w_img_b[l], H, t->bplan, s));
    }
    ZRB_TRY(convert_pad_f16(p->fc_w, H, t->fc_w_h, t->Hp, V, H, 1.f, s));
    t->packed_version = c->weights_version;
    t->packed_params = *p;
    return ZRB_OK;
}

// apply deferred update item `item` (see zrb_tc_state::upd_pending); pdl: as a programmatic dependent of the forward
// recurrence kernel just enqueued on `s`
static int tc_issue_update(zrb_ctx* c, int item, bool pdl, cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    const int H = c->cfg.hidden, L = c->cfg.layers, V = c->cfg.vocab;
    if (!(t->upd_pending & (1u << item))) return ZRB_OK;
    t->upd_pending &= ~(1u << item);
    const TensorList& tl = t->upd_tl;
    const bool persistent = t->fplan.ok && t->bplan.ok;
    if (item < L) {
        const int l = item, b = 1 + 4 * l;
        ZRB_TRY(update_pack(tl.p[b], tl.g[b], 4 * H, H, t->upd_lr, c->scalars, t->w_ih_h[l], t->Hp, nullptr, nullptr,
                            nullptr, nullptr, c->keep_clipped, s, pdl));
        return update_pack(tl.p[b + 1], tl.g[b + 1], 4 * H, H, t->upd_lr, c->scalars, persistent ? nullptr : t->w_hh_h[l],
                           t->Hp, t->fplan.ok ? t->w_img_f[l] : nullptr, &t->fplan,
                           t->bplan.ok ? t->w_img_b[l] : nullptr, &t->bplan, c->keep_clipped, s, pdl);
    }
    const int f = 1 + 4 * L;
    return update_pack(tl.p[f], tl.g[f], V, H, t->upd_lr, c->scalars, t->fc_w_h, t->Hp, nullptr, nullptr, nullptr,
                       nullptr, c->keep_clipped, s, pdl);
}

int tc_flush_updates(zrb_ctx* c, cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    if (!t || !t->upd_pending) return ZRB_OK;
    ProfScope ps(c, ZRB_PROF_CLIP_SGD, s);
    for (int item = 1; item <= c->cfg.layers; ++item) ZRB_TRY(tc_issue_update(c, item, false, s));
    return ZRB_OK;
}

int tc_forward(zrb_ctx* c, const zrb_params* p, const int64_t* x, const zrb_states* in, const zrb_states* out,
               float* scores, cudaStream_t s, bool last_only) {
    zrb_tc_state* t = c->tc;
    const int H = c->cfg.hidden, L = c->cfg.layers, V = c->cfg.vocab, T = c->T, B = c->B, N = T * B;
    const int Hp = t->Hp;
    const size_t bh = (size_t)B * H * sizeof(float);
    // deferred updates ride beside the forward recurrences of a fused train step; any other forward applies them first
    const bool ride = t->upd_pending && t->in_train_step && t->fplan.ok && (!c->prof_on || prof_keeps_pdl());
    if (t->upd_pending && !ride) ZRB_TRY(tc_flush_updates(c, s));
    ZRB_TRY(tc_pack_weights(c, p, s));
    {   // state copies (in / out may be the same buffers), fp16 h0 rows and images, saved tokens: one launch
        FwdPrep fp = {};
        for (int l = 0; l < L; ++l) {
            fp.in_h[l] = in->h[l]; fp.in_c[l] = in->c[l]; fp.h0s[l] = c->h0s[l]; fp.c0s[l] = c->c0s[l];
            fp.hprev_h[l] = t->hprev_h[l]; fp.h0_img[l] = t->fplan.ok ? t->h0_img[l] : nullptr;
            fp.rm[l] = rec_mask(c, l);
        }
        fp.x = x; fp.x_saved = c->x_saved;
        fp.L = L; fp.B = B; fp.H = H; fp.Hp = Hp; fp.GB = t->fplan.GBi; fp.Kc = t->fplan.Kc; fp.N = N;
        ZRB_TRY(fwd_prep(fp, s));
    }
    {
        ProfScope ps(c, ZRB_PROF_EMBED_FWD, s);
        // tied: E's update (item L) is still deferred -> gather through it; the update itself rides beside the last
        // recurrence, before the projection reads fc_w_h
        const bool through = ride && c->tied && (t->upd_pending & (1u << L));
        ZRB_TRY(embed_dropout_fwd(p->embed_w, x, nullptr, t->x_h[0], Hp, N, H, V, site_mask(c, 0), s,
                                  through ? t->upd_tl.g[1 + 4 * L] : nullptr, t->upd_lr, c->scalars));
    }
    for (int l = 0; l < L; ++l) {
        float* G = c->gates[l];
        {
            ProfScope ps(c, ZRB_PROF_GEMM_IN, s);
            ZRB_TRY(gemm_f16_tc(t->x_h[l], Hp, 0, t->w_ih_h[l], Hp, 0, G, 4 * H, N, 4 * H, H, 1.f, p->b_ih[l], 0, s, nullptr,
                                p->b_hh[l]));
        }
        MaskSrc m = site_mask(c, l + 1), rm = rec_mask(c, l);
        ProfScope ps(c, ZRB_PROF_REC_FWD, s);
        if (t->fplan.ok) {
            const unsigned int arrivals = (unsigned int)T * (unsigned int)t->fplan.nCTA;
            if (t->cnt_f > 0xF0000000u - arrivals) {   // far from wrapping: once per ~900k launches
                ZRB_CUDA(cudaMemsetAsync(t->counter, 0, sizeof(unsigned int), s));
                t->cnt_f = 0;
            }
            ZRB_TRY(lstm_rec_fwd(t->fplan, tc_watchdog(c), t->w_img_f[l], t->h0_img[l], t->h_img, G, c->c0s[l], c->cst[l], out->h[l],
                                 out->c[l], t->hprev_h[l], t->x_h[l + 1], t->counter, t->cnt_f, T, B, H, Hp, m, rm, s,
                                 t->trace));
            t->cnt_f += arrivals;
            // deferred update of the NEXT layer's matrices (or of fc.W after the last layer): on the idle SMs, beside
            // this recurrence; their consumers (the next input GEMM / the projection) are enqueued behind them
            if (ride) ZRB_TRY(tc_issue_update(c, l + 1, true, s));
            continue;
        }
        for (int tt = 0; tt < T; ++tt) {
            const float* c_prev = tt ? c->cst[l] + (size_t)(tt - 1) * B * H : c->c0s[l];
            float* Gt = G + (size_t)tt * B * 4 * H;
            ZRB_TRY(gemm_f16_tc(t->hprev_h[l] + (size_t)tt * B * Hp, Hp, 0, t->w_hh_h[l], Hp, 0, Gt, 4 * H, B, 4 * H, H,
                                1.f, nullptr, 1, s));
            ZRB_TRY(lstm_cell_fwd_tc(Gt, c_prev, c->cst[l] + (size_t)tt * B * H, c->hraw[l] + (size_t)tt * B * H,
                                     t->hprev_h[l] + (size_t)(tt + 1) * B * Hp, t->x_h[l + 1] + (size_t)tt * B * Hp, Hp, B,
                                     H, (int64_t)tt * B * H, (int64_t)N * H, m, rm, s));
        }
        ZRB_CUDA(cudaMemcpyAsync(out->h[l], c->hraw[l] + (size_t)(T - 1) * B * H, bh, cudaMemcpyDeviceToDevice, s));
        ZRB_CUDA(cudaMemcpyAsync(out->c[l], c->cst[l] + (size_t)(T - 1) * B * H, bh, cudaMemcpyDeviceToDevice, s));
    }
    if (scores) {
        ProfScope ps(c, ZRB_PROF_PROJ_FWD, s);
        const int rows = last_only ? B : N;
        ZRB_TRY(gemm_f16_tc(t->x_h[L] + (size_t)(N - rows) * Hp, Hp, 0, t->fc_w_h, Hp, 0, scores, V, rows, V, H, 1.f,
                            p->fc_b, 0, s));
    }
    return ZRB_OK;
}

const __half* tc_last_layer_image(const zrb_ctx* c) { return c->tc->x_h[c->cfg.layers]; }

static bool prof_keeps_pdl() {
    static const bool on = getenv("ZRB_PROF_KEEP_PDL") != nullptr;
    return on;
}

// next block of sum-of-squares slots for an [M,N] weight gradient, or null when the step does not fuse the norm
static float* wgrad_sumsq(zrb_ctx* c, int M, int N, int K) {
    zrb_tc_state* t = c->tc;
    if (!t->wg_ok) return nullptr;
    const int n = gemm_f16_tc_sumsq_slots(M, N, K);
    if (t->wg_slots + n > kNormGemm) {
        t->wg_ok = false;   // does not fit: the update takes the norm over the whole buffers instead
        return nullptr;
    }
    float* out = c->partials + norm_partials_base() + kNormExtra + t->wg_slots;
    t->wg_slots += n;
    return out;
}

// backward from the scaled fp16 image dS_h already in place
// projection backward: afterwards fc.W / fc.b gradients are complete and c->bwd_dy holds d loss / d act[L]
static int tc_backward_head(zrb_ctx* c, const zrb_params* p, const zrb_params* g, cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    const int H = c->cfg.hidden, L = c->cfg.layers, V = c->cfg.vocab, N = c->T * c->B;
    const int Hp = t->Hp, Vp = t->Vp;
    const float inv = 1.f / kGradScale;
    float* dY = c->dy;
    c->bwd_dy = c->dy;
    c->bwd_dx = c->dx;
    c->bwd_next_layer = L - 1;
    {
        ProfScope ps(c, ZRB_PROF_PROJ_BWD, s);
        // dA[N,H] = dS[N,V] * W[V,H]       (W image read MN-major)
        ZRB_TRY(gemm_f16_tc(t->dS_h, Vp, 0, t->fc_w_h, Hp, 1, dY, H, N, H, V, inv, nullptr, 0, s));
        t->wg_ok = c->fused_norm;
        t->wg_slots = 0;
        t->wg_key = g->fc_w;
        ZRB_TRY(colsum_h(t->dS_h, Vp, g->fc_b, nullptr, N, V, inv, t->colsum_scratch, s));
        // dW[V,H] = dS^T[V,N] * A[N,H]     (both operands MN-major: contraction over tokens).  Nothing downstream in
        // backward reads it: with deferral on it runs underneath the first backward recurrence instead of before it.
        t->pending = 0;
        if (t->defer_wgrad && t->bplan.ok && (!c->prof_on || prof_keeps_pdl())) t->pending = 1;
        else ZRB_TRY(gemm_f16_tc(t->dS_h, Vp, 1, t->x_h[L], Hp, 1, g->fc_w, H, V, H, N, inv, nullptr, 0, s,
                                 wgrad_sumsq(c, V, H, N)));
    }
    return ZRB_OK;
}

// the two weight gradients of layer l from dG (scaled fp16, [N,G4p]): ONE launch, dG is the shared A operand
static int tc_layer_wgrads(zrb_ctx* c, const zrb_params* g, int l, const __half* dG_h, bool pdl, cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    const int H = c->cfg.hidden, N = c->T * c->B;
    float* ss1 = wgrad_sumsq(c, 4 * H, H, N);
    float* ss2 = wgrad_sumsq(c, 4 * H, H, N);
    return gemm_f16_tc(dG_h, t->G4p, 1, t->x_h[l], t->Hp, 1, g->w_ih[l], H, 4 * H, H, N, 1.f / kGradScale, nullptr, 0, s,
                       ss1, nullptr, pdl, t->hprev_h[l], g->w_hh[l], ss2);
}

// launch what tc_backward_head / the previous layer deferred, as a programmatic dependent of the recurrence kernel
// that was just enqueued on `s`
static int tc_issue_pending(zrb_ctx* c, const zrb_params* g, cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    const int H = c->cfg.hidden, L = c->cfg.layers, V = c->cfg.vocab, N = c->T * c->B;
    const int kind = t->pending;
    t->pending = 0;
    // (no event bracket here: an event record between the recurrence kernel and its programmatic dependent would sit
    // between the two launches; while profiling with ZRB_PROF_KEEP_PDL=1 the time lands in the enclosing REC_BWD class)
    if (kind == 1) {
        return gemm_f16_tc(t->dS_h, t->Vp, 1, t->x_h[L], t->Hp, 1, g->fc_w, H, V, H, N, 1.f / kGradScale, nullptr, 0, s,
                           wgrad_sumsq(c, V, H, N), nullptr, true);
    }
    if (kind == 2) {
        const int l = t->pending_layer;
        return tc_layer_wgrads(c, g, l, (l & 1) ? t->dG_h_alt : t->dG_h, true, s);
    }
    return ZRB_OK;
}

// backward of layer l (must be called for l = L-1, ..., 0 in that order): afterwards the layer's four
// gradients are complete; l == 0 also finishes the embedding gradient
static int tc_backward_layer(zrb_ctx* c, const zrb_params* p, const zrb_params* g, int l, cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    const int H = c->cfg.hidden, V = c->cfg.vocab, T = c->T, B = c->B, N = T * B;
    const int Hp = t->Hp, G4p = t->G4p;
    const size_t bh = (size_t)B * H;
    const float inv = 1.f / kGradScale;
    if (l != c->bwd_next_layer) {
        set_error("backward layers must be visited in order L-1..0 (expected %d, got %d)", c->bwd_next_layer, l);
        return ZRB_E_STATE;
    }
    float* dY = c->bwd_dy;
    float* dX = c->bwd_dx;
    __half* dG_h = (l & 1) ? t->dG_h_alt : t->dG_h;
    {
        MaskSrc m = site_mask(c, l + 1), rm = rec_mask(c, l);
        if (t->bplan.ok) {
            ProfScope ps(c, ZRB_PROF_REC_BWD, s);
            const unsigned int arrivals = (unsigned int)T * (unsigned int)t->bplan.nCTA;
            if (t->cnt_b > 0xF0000000u - arrivals) {
                ZRB_CUDA(cudaMemsetAsync(t->counter + 32, 0, sizeof(unsigned int), s));
                t->cnt_b = 0;
            }
            ZRB_TRY(lstm_rec_bwd(t->bplan, tc_watchdog(c), t->w_img_b[l], t->g_img, dY, c->gates[l], c->cst[l], c->c0s[l], dG_h,
                                 t->counter + 32, t->cnt_b, T, B, H, G4p, m, rm, s,
                                 t->trace ? t->trace + 8 + (size_t)c->cfg.max_seq * 8 : nullptr, g->b_ih[l], g->b_hh[l],
                                 c->resident_flag, ++c->resident_seq, c->dG /* [N,4H] fp32, idle on this path */));
            t->cnt_b += arrivals;
            ZRB_TRY(tc_issue_pending(c, g, s));   // runs on the SMs the cluster kernel leaves idle
        } else {
            ProfScope ps(c, ZRB_PROF_REC_BWD, s);
            ZRB_CUDA(cudaMemsetAsync(c->dc, 0, bh * sizeof(float), s));   // (the persistent kernel keeps dc in registers)
            for (int tt = T - 1; tt >= 0; --tt) {
                const float* c_prev = tt ? c->cst[l] + (size_t)(tt - 1) * bh : c->c0s[l];
                ZRB_TRY(lstm_cell_bwd_tc(dY + (size_t)tt * bh, tt == T - 1 ? nullptr : c->dh_rec, c->dc,
                                         c->gates[l] + (size_t)tt * B * 4 * H, c->cst[l] + (size_t)tt * bh, c_prev,
                                         c->dG + (size_t)tt * B * 4 * H, dG_h + (size_t)tt * B * G4p, G4p, B, H,
                                         (int64_t)tt * bh, (int64_t)N * H, m, rm, s));
                if (tt > 0)  // dh_{t-1}[B,H] = dG_t[B,4H] * W_hh[4H,H]
                    ZRB_TRY(gemm_f16_tc(dG_h + (size_t)tt * B * G4p, G4p, 0, t->w_hh_h[l], Hp, 1, c->dh_rec, H, B, H,
                                        4 * H, inv, nullptr, 0, s));
            }
        }
        {
            ProfScope ps(c, ZRB_PROF_GEMM_DX, s);
            ZRB_TRY(gemm_f16_tc(dG_h, G4p, 0, t->w_ih_h[l], Hp, 1, dX, H, N, H, 4 * H, inv, nullptr, 0, s));
        }
        // dW_ih, dW_hh: nothing downstream in backward reads them -> for l > 0 they run underneath the next layer's
        // recurrence (which writes the other dG buffer); the bias gradients come out of the recurrence kernel itself
        if (t->defer_wgrad && t->bplan.ok && l > 0 && (!c->prof_on || prof_keeps_pdl())) {
            t->pending = 2;
            t->pending_layer = l;
        } else {
            ProfScope ps(c, ZRB_PROF_GEMM_WGRAD, s);
            ZRB_TRY(tc_layer_wgrads(c, g, l, dG_h, false, s));
        }
        if (!t->bplan.ok) ZRB_TRY(colsum(c->dG, g->b_ih[l], g->b_hh[l], N, 4 * H, s));
        float* tmp = dY; dY = dX; dX = tmp;
    }
    c->bwd_dy = dY;
    c->bwd_dx = dX;
    c->bwd_next_layer = l - 1;
    if (l > 0) return ZRB_OK;
    ProfScope ps(c, ZRB_PROF_EMBED_BWD, s);
    if (c->embed_rows_out) return embed_rows(dY, c->embed_rows_out, N, H, site_mask(c, 0), s);
    if (c->tied) {
        // g->embed_w holds G_proj (the projection's wgrad GEMM overwrote every row): add the fixed-point row sums, with
        // dX (free now) as the rows buffer; the fused norm's extra slots get the correction from G_proj^2 to dE^2
        ZRB_TRY(embed_rows(dY, dX, N, H, site_mask(c, 0), s));
        return embed_scatter_rows(c->x_saved, dX, g->embed_w, N, H, V, c->emb_first, c->emb_acc, s, true,
                                  c->fused_norm ? c->partials + norm_partials_base() : nullptr, kNormExtra);
    }
    if (c->emb_sparse && c->emb_prev_grad == g->embed_w) {
        ZRB_TRY(embed_zero_rows(g->embed_w, c->emb_prev_ids, c->emb_prev_n, H, V, s));   // only last window's rows are non-zero
    } else {
        ZRB_CUDA(cudaMemsetAsync(g->embed_w, 0, (size_t)V * H * sizeof(float), s));
    }
    ZRB_TRY(embed_dropout_bwd(dY, c->x_saved, g->embed_w, N, H, V, site_mask(c, 0), s));
    if (c->emb_sparse) {
        ZRB_CUDA(cudaMemcpyAsync(c->emb_prev_ids, c->x_saved, (size_t)N * sizeof(int64_t), cudaMemcpyDeviceToDevice, s));
        c->emb_prev_n = N;
        c->emb_prev_grad = g->embed_w;
    }
    return ZRB_OK;
}

static int tc_backward_from_image(zrb_ctx* c, const zrb_params* p, const zrb_params* g, cudaStream_t s) {
    static const bool no_overlap = getenv("ZRB_NO_OVERLAP") != nullptr;    // A/B switch
    c->tc->defer_wgrad = !no_overlap;
    ZRB_TRY(tc_backward_head(c, p, g, s));
    for (int l = c->cfg.layers - 1; l >= 0; --l) ZRB_TRY(tc_backward_layer(c, p, g, l, s));
    return ZRB_OK;
}

int tc_backward(zrb_ctx* c, const zrb_params* p, const float* dscores, const zrb_params* g, cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    const int N = c->T * c->B, V = c->cfg.vocab;
    ZRB_TRY(convert_pad_f16(dscores, V, t->dS_h, t->Vp, N, V, kGradScale, s));
    return tc_backward_from_image(c, p, g, s);
}

int tc_train_step_grads(zrb_ctx* c, const zrb_params* p, const zrb_params* g, const int64_t* x, const int64_t* y,
                        int T, int B, const zrb_states* in, const zrb_states* out, uint64_t seed, uint64_t step,
                        float* loss, cudaStream_t s) {
    c->T = T; c->B = B; c->train = 1; c->seed = seed; c->step = step;
    c->have_fwd = false;
    c->tc->in_train_step = true;
    const int frc = tc_forward(c, p, x, in, out, c->scores, s);
    c->tc->in_train_step = false;
    ZRB_TRY(frc);
    c->have_fwd = true;
    {
        ProfScope ps(c, ZRB_PROF_SOFTMAX, s);
        ZRB_TRY(softmax_nll(c->scores, y, T * B, c->cfg.vocab, B, c->row_loss, loss, nullptr, nullptr, s, c->tc->dS_h,
                            c->tc->Vp, kGradScale));
    }
    return tc_backward_from_image(c, p, g, s);
}

// the gradient of the eval-mode loss (DESIGN.md section 14): the fused gradient path with c->train = 0, so that every
// site_mask / rec_mask is off while tc_forward still keeps the activations; pending lazy updates are applied first (the
// forward runs outside a train step).  No clip norm follows, so the wgrad epilogues write no sum-of-squares slots.
int tc_eval_grads(zrb_ctx* c, const zrb_params* p, const zrb_params* g, const int64_t* x, const int64_t* y, int T, int B,
                  const zrb_states* in, const zrb_states* out, float* loss, cudaStream_t s) {
    c->T = T; c->B = B; c->train = 0; c->seed = 0; c->step = 0;
    c->have_fwd = false;
    ZRB_TRY(tc_forward(c, p, x, in, out, c->scores, s));
    c->have_fwd = true;
    {
        ProfScope ps(c, ZRB_PROF_SOFTMAX, s);
        ZRB_TRY(softmax_nll(c->scores, y, T * B, c->cfg.vocab, B, c->row_loss, loss, nullptr, nullptr, s, c->tc->dS_h,
                            c->tc->Vp, kGradScale));
    }
    const bool fused = c->fused_norm;
    c->fused_norm = false;
    const int rc = tc_backward_from_image(c, p, g, s);
    c->fused_norm = fused;
    c->tc->wg_ok = false;
    return rc;
}

int tc_train_step_begin(zrb_ctx* c, const zrb_params* p, const zrb_params* g, const int64_t* x, const int64_t* y,
                        int T, int B, const zrb_states* in, const zrb_states* out, uint64_t seed, uint64_t step,
                        float* loss, cudaStream_t s) {
    c->T = T; c->B = B; c->train = 1; c->seed = seed; c->step = step;
    c->have_fwd = false;
    c->tc->in_train_step = true;
    const int frc = tc_forward(c, p, x, in, out, c->scores, s);
    c->tc->in_train_step = false;
    ZRB_TRY(frc);
    c->have_fwd = true;
    {
        ProfScope ps(c, ZRB_PROF_SOFTMAX, s);
        ZRB_TRY(softmax_nll(c->scores, y, T * B, c->cfg.vocab, B, c->row_loss, loss, nullptr, nullptr, s, c->tc->dS_h,
                            c->tc->Vp, kGradScale));
    }
    c->tc->defer_wgrad = false;   // phased backward: every bucket is complete when its call returns
    return tc_backward_head(c, p, g, s);
}

int tc_train_step_layer(zrb_ctx* c, const zrb_params* p, const zrb_params* g, int l, cudaStream_t s) {
    return tc_backward_layer(c, p, g, l, s);
}

bool tc_persistent_bwd(const zrb_ctx* c) { return c->tc && c->tc->bplan.ok; }

void tc_rec_plans(const zrb_ctx* c, int32_t* h_out) {
    const RecPlan* plans[2] = {&c->tc->fplan, &c->tc->bplan};
    for (int d = 0; d < 2; ++d) {
        const RecPlan& p = *plans[d];
        int32_t* o = h_out + 8 * d;
        o[0] = p.ok;
        o[1] = p.ok ? p.KS : 0; o[2] = p.ok ? p.U : 0; o[3] = p.ok ? p.G : 0; o[4] = p.ok ? p.nCTA : 0;
        o[5] = p.ok ? p.GBi : 0; o[6] = p.ok ? p.Kc : 0; o[7] = p.ok ? p.KcS : 0;
    }
}

// ---- unit-level entry points: ONE recurrent layer through the persistent kernels (zrb_lstm_layer_fwd / _bwd) --------
// They borrow layer slot 0 of the context (images, activations) and leave the model-level weight images stale, so the
// next model-level call repacks.
int tc_layer_fwd(zrb_ctx* c, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, const float* x,
                 int T, int B, const float* h0, const float* c0, float* y, float* hT, float* cT, cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    const int H = c->cfg.hidden, N = T * B, Hp = t->Hp;
    if (!t->fplan.ok || !t->bplan.ok) {
        set_error("zrb_lstm_layer_fwd needs the persistent recurrence kernels (shape H=%d B=%d does not fit them)", H, B);
        return ZRB_E_INVALID;
    }
    ZRB_TRY(tc_flush_updates(c, s));
    c->T = T; c->B = B; c->train = 0;
    t->packed_version = 0;                       // slot 0 is about to hold this call's weights
    ZRB_TRY(convert_pad_f16(w_ih, H, t->w_ih_h[0], Hp, 4 * H, H, 1.f, s));
    ZRB_TRY(pack_whh_fwd(w_hh, t->w_img_f[0], H, t->fplan, s));
    ZRB_TRY(pack_whh_bwd(w_hh, t->w_img_b[0], H, t->bplan, s));
    ZRB_TRY(convert_pad_f16(x, H, t->x_h[0], Hp, N, H, 1.f, s));
    FwdPrep fp = {};
    fp.in_h[0] = h0; fp.in_c[0] = c0; fp.h0s[0] = c->h0s[0]; fp.c0s[0] = c->c0s[0];
    fp.hprev_h[0] = t->hprev_h[0]; fp.h0_img[0] = t->h0_img[0];
    fp.x = nullptr; fp.x_saved = nullptr;
    fp.L = 1; fp.B = B; fp.H = H; fp.Hp = Hp; fp.GB = t->fplan.GBi; fp.Kc = t->fplan.Kc; fp.N = 0;
    ZRB_TRY(fwd_prep(fp, s));
    ZRB_TRY(gemm_f16_tc(t->x_h[0], Hp, 0, t->w_ih_h[0], Hp, 0, c->gates[0], 4 * H, N, 4 * H, H, 1.f, b_ih, 0, s, nullptr, b_hh));
    const unsigned int arrivals = (unsigned int)T * (unsigned int)t->fplan.nCTA;
    if (t->cnt_f > 0xF0000000u - arrivals) {
        ZRB_CUDA(cudaMemsetAsync(t->counter, 0, sizeof(unsigned int), s));
        t->cnt_f = 0;
    }
    MaskSrc m = make_mask_src(nullptr, 0, 0, 0, 0.f, 0);    // no dropout at this level: the caller applies it (model.py:105,108)
    ZRB_TRY(lstm_rec_fwd(t->fplan, tc_watchdog(c), t->w_img_f[0], t->h0_img[0], t->h_img, c->gates[0], c->c0s[0], c->cst[0], hT, cT,
                         t->hprev_h[0], t->x_h[1], t->counter, t->cnt_f, T, B, H, Hp, m, m, s, nullptr, y));
    t->cnt_f += arrivals;
    c->have_fwd = false;                         // a model-level backward must not follow this
    c->layer_fwd_ok = true;
    return ZRB_OK;
}

int tc_layer_bwd(zrb_ctx* c, const float* dy, float* dx, float* dw_ih, float* dw_hh, float* db_ih, float* db_hh,
                 cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    const int H = c->cfg.hidden, T = c->T, B = c->B, N = T * B, Hp = t->Hp, G4p = t->G4p;
    if (!c->layer_fwd_ok) {
        set_error("zrb_lstm_layer_bwd without a preceding zrb_lstm_layer_fwd");
        return ZRB_E_STATE;
    }
    const unsigned int arrivals = (unsigned int)T * (unsigned int)t->bplan.nCTA;
    if (t->cnt_b > 0xF0000000u - arrivals) {
        ZRB_CUDA(cudaMemsetAsync(t->counter + 32, 0, sizeof(unsigned int), s));
        t->cnt_b = 0;
    }
    MaskSrc m = make_mask_src(nullptr, 0, 0, 0, 0.f, 0);
    ZRB_TRY(lstm_rec_bwd(t->bplan, tc_watchdog(c), t->w_img_b[0], t->g_img, dy, c->gates[0], c->cst[0], c->c0s[0], t->dG_h, t->counter + 32,
                         t->cnt_b, T, B, H, G4p, m, m, s, nullptr, db_ih, db_hh, c->resident_flag, ++c->resident_seq, c->dG));
    t->cnt_b += arrivals;
    const float inv = 1.f / kGradScale;
    if (dx) ZRB_TRY(gemm_f16_tc(t->dG_h, G4p, 0, t->w_ih_h[0], Hp, 1, dx, H, N, H, 4 * H, inv, nullptr, 0, s));
    ZRB_TRY(gemm_f16_tc(t->dG_h, G4p, 1, t->x_h[0], Hp, 1, dw_ih, H, 4 * H, H, N, inv, nullptr, 0, s, nullptr, nullptr, false,
                        t->hprev_h[0], dw_hh, nullptr));
    c->layer_fwd_ok = false;
    return ZRB_OK;
}

int tc_rec_trace(zrb_ctx* c, long long* h_out, int max_entries) {
    if (!c->tc || !c->tc->trace) { set_error("set ZRB_REC_TRACE=1 before creating the context"); return ZRB_E_STATE; }
    int n = 2 * (8 + c->cfg.max_seq * 8);
    if (n > max_entries) n = max_entries;
    ZRB_CUDA(cudaDeviceSynchronize());
    ZRB_CUDA(cudaMemcpy(h_out, c->tc->trace, (size_t)n * sizeof(long long), cudaMemcpyDeviceToHost));
    return n;
}

// clip + SGD (main.py:114-117).  The update pass also writes the fp16 operand images of the new weights,
// so the next forward needs no pack pass.
int tc_update(zrb_ctx* c, const zrb_params* p, const TensorList& tl, float lr, float max_norm, float* norm_out,
              cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    const int H = c->cfg.hidden, L = c->cfg.layers, V = c->cfg.vocab;
    ZRB_TRY(tc_flush_updates(c, s));   // (a second update without a forward in between)
    bool fuse = true;   // update_pack picks 16 / 8 / 4-byte accesses from the matrix width and alignment
    for (int i = 0; i < tl.count && fuse; ++i)
        fuse = ((((uintptr_t)tl.p[i]) | ((uintptr_t)tl.g[i])) & 3) == 0;
    ProfScope ps(c, ZRB_PROF_CLIP_SGD, s);
    if (!fuse) {
        ZRB_TRY(clip_sgd(tl, lr, max_norm, c->partials, c->scalars, norm_out, c->keep_clipped, s));
        c->weights_version++;
        return ZRB_OK;
    }
    // tensor order of param_list(): embed, (w_ih, w_hh, b_ih, b_hh) x L, fc_w, fc_b (tied: embed has n = 0, E is fc_w)
    const bool rows_only = !c->tied && c->emb_sparse && c->emb_prev_grad == tl.g[0] && c->emb_prev_n > 0;
    const bool tied_gemm_norm = c->tied && t->wg_ok && t->wg_key == tl.g[1 + 4 * L];
    if (tied_gemm_norm) {
        // matrices from the wgrad epilogue slots (E's describe G_proj); the extra slots hold the merge's correction
        // to dE (tc_backward_layer): no read of the matrices' gradients
        TensorList dense = tl;
        for (int l = 0; l < L; ++l) dense.n[1 + 4 * l] = dense.n[2 + 4 * l] = 0;
        dense.n[1 + 4 * L] = 0;
        ZRB_TRY(grad_norm(dense, max_norm, c->partials, c->scalars, norm_out, s, true, t->wg_slots));
    } else if (rows_only) {
        // embedding: only the rows of the last window can be non-zero -> norm and update over those rows
        TensorList dense = tl;
        dense.n[0] = 0;
        const bool gemm_norm = t->wg_ok && t->wg_key == tl.g[1 + 4 * L];   // matrices: summed by the wgrad GEMMs
        if (gemm_norm) {
            for (int l = 0; l < L; ++l) dense.n[1 + 4 * l] = dense.n[2 + 4 * l] = 0;
            dense.n[1 + 4 * L] = 0;
        }
        ZRB_TRY(embed_first_table(c->emb_prev_ids, c->emb_first, c->emb_prev_n, V, s));
        ZRB_TRY(embed_rows_sumsq(tl.g[0], c->emb_prev_ids, c->emb_first, c->emb_prev_n, H, V,
                                 c->partials + norm_partials_base(), kNormExtra, s));   // one token per block
        ZRB_TRY(grad_norm(dense, max_norm, c->partials, c->scalars, norm_out, s, true, gemm_norm ? t->wg_slots : 0));
        ZRB_TRY(embed_rows_update(tl.p[0], tl.g[0], c->emb_prev_ids, c->emb_first, c->emb_prev_n, H, V, lr, c->scalars,
                                  c->keep_clipped, s));
    } else {
        ZRB_TRY(grad_norm(tl, max_norm, c->partials, c->scalars, norm_out, s));
    }
    TensorList rest;
    rest.count = 0;
    auto push = [&](int i) { rest.p[rest.count] = tl.p[i]; rest.g[rest.count] = tl.g[i]; rest.n[rest.count] = tl.n[i]; rest.count++; };
    if (!rows_only) push(0);
    const bool persistent = t->fplan.ok && t->bplan.ok;
    // lazy update: layer 0 (needed by the very next kernels) now; layers >= 1 and fc.W beside the forward recurrences of
    // the next step (tc_forward), or at the next call that is not a fused train step (tc_flush_updates)
    const bool lazy = c->lazy_update && persistent && (!c->prof_on || prof_keeps_pdl());
    if (lazy) {
        t->upd_tl = tl;
        t->upd_lr = lr;
    }
    for (int l = 0; l < L; ++l) {
        const int b = 1 + 4 * l;
        push(b + 2);
        push(b + 3);
        if (lazy && l >= 1) {
            t->upd_pending |= 1u << l;
            continue;
        }
        ZRB_TRY(update_pack(tl.p[b], tl.g[b], 4 * H, H, lr, c->scalars, t->w_ih_h[l], t->Hp, nullptr, nullptr, nullptr,
                            nullptr, c->keep_clipped, s));
        ZRB_TRY(update_pack(tl.p[b + 1], tl.g[b + 1], 4 * H, H, lr, c->scalars, persistent ? nullptr : t->w_hh_h[l],
                            t->Hp, t->fplan.ok ? t->w_img_f[l] : nullptr, &t->fplan,
                            t->bplan.ok ? t->w_img_b[l] : nullptr, &t->bplan, c->keep_clipped, s));
    }
    const int f = 1 + 4 * L;
    if (lazy) t->upd_pending |= 1u << L;
    else ZRB_TRY(update_pack(tl.p[f], tl.g[f], V, H, lr, c->scalars, t->fc_w_h, t->Hp, nullptr, nullptr, nullptr, nullptr,
                             c->keep_clipped, s));
    push(f + 1);
    ZRB_TRY(sgd_apply(rest, lr, c->scalars, c->keep_clipped, s));
    t->wg_ok = false;
    c->weights_version++;
    t->packed_version = c->weights_version;      // images are current
    t->packed_params = *p;
    return ZRB_OK;
}

// The dynamic-evaluation update (DESIGN.md section 14): tc_update's schedule with the dynamic rule, no norm and no lazy
// deferral.  The matrices go through update_pack's kernels, which rebuild their fp16 images from registers; the rest
// through the list kernel.  tg / r: theta_g and the RMS statistic in param_list() order (r null: the SGD rule).
int tc_dyneval_update(zrb_ctx* c, const zrb_params* p, const TensorList& tl, float* const* tg, float* const* r,
                      const DynArgs& a, cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    const int H = c->cfg.hidden, L = c->cfg.layers, V = c->cfg.vocab;
    ZRB_TRY(tc_flush_updates(c, s));
    ProfScope ps(c, ZRB_PROF_CLIP_SGD, s);
    bool fuse = true;
    for (int i = 0; i < tl.count && fuse; ++i)
        fuse = ((((uintptr_t)tl.p[i]) | ((uintptr_t)tl.g[i]) | ((uintptr_t)tg[i]) | (r ? (uintptr_t)r[i] : 0)) & 3) == 0;
    if (!fuse) {   // images rebuilt by the next forward's pack
        ZRB_TRY(dyneval_apply(tl, tg, r, a, s));
        c->weights_version++;
        return ZRB_OK;
    }
    TensorList rest = tl;   // entries with an image get length 0 here (skipped by the list kernel)
    const bool persistent = t->fplan.ok && t->bplan.ok;
    for (int l = 0; l < L; ++l) {
        const int b = 1 + 4 * l;
        ZRB_TRY(update_pack_dyn(tl.p[b], tl.g[b], tg[b], r ? r[b] : nullptr, 4 * H, H, a, t->w_ih_h[l], t->Hp, nullptr,
                                nullptr, nullptr, nullptr, s));
        ZRB_TRY(update_pack_dyn(tl.p[b + 1], tl.g[b + 1], tg[b + 1], r ? r[b + 1] : nullptr, 4 * H, H, a,
                                persistent ? nullptr : t->w_hh_h[l], t->Hp, t->fplan.ok ? t->w_img_f[l] : nullptr,
                                &t->fplan, t->bplan.ok ? t->w_img_b[l] : nullptr, &t->bplan, s));
        rest.n[b] = rest.n[b + 1] = 0;
    }
    const int f = 1 + 4 * L;
    ZRB_TRY(update_pack_dyn(tl.p[f], tl.g[f], tg[f], r ? r[f] : nullptr, V, H, a, t->fc_w_h, t->Hp, nullptr, nullptr,
                            nullptr, nullptr, s));
    rest.n[f] = 0;
    ZRB_TRY(dyneval_apply(rest, tg, r, a, s));
    t->wg_ok = false;
    c->weights_version++;
    t->packed_version = c->weights_version;      // images are current
    t->packed_params = *p;
    return ZRB_OK;
}

}  // namespace zrb
