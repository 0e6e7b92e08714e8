// ZRB_ENGINE_TC: every dense contraction of the path on wgmma tensor cores (fp16 operands,
// fp32 accumulation), pointwise math and state in fp32.
//
// fp16 images (K = contraction index; Xp[s] = pad64(width of site s): Xp[l] = pad64(In_l), Xp[l+1] = pad64(H_l)):
//   w_ih_h[l] [4H_l, Xp[l]], w_hh_h[l] [4H_l, Xp[l+1]]   read K-major by the forward GEMMs (X*W^T, h*W^T) and MN-major
//   fc_w_h    [V,    Xp[L]]                             by the dgrads (dG*W, dS*W): one image serves both
//   x_h[l]      [N, Xp[l]]     dropout'ed input of layer l (x_h[L] feeds the projection); MN-major B of wgrads
//   hprev_h[l]  [N+B, Xp[l+1]] rows 0..B-1 = h entering the window, rows B.. = h_t: row block t is h_{t-1}
//                              (variational mode: times the layer's recurrent mask, so the dW_hh GEMM needs no change)
//   dG_h        [N, G4p[l]] kGradScale * dG;  dS_h [N, Vp] kGradScale * dscores
// Gradient images are scaled by an exact power of two and unscaled by the consuming GEMM's alpha.
#include "engine.h"
#include <stdlib.h>
#include <string.h>

#include "tc_kernels.h"

// One grid-barrier word of the persistent recurrence kernels.  The word is never reset between launches: each launch
// gets the value it starts from as its base, and its T * nCTA arrivals advance the word.
struct GridBarrier {
    unsigned int* word = nullptr;
    unsigned int base = 0;   // the word's value when the next launch starts
    // claim T * nCTA arrivals: enqueue launch(word, base), after resetting the word when the arrivals could wrap it (once
    // per ~900k launches; the reset stays before the launch, so nothing lands between a recurrence kernel and its
    // programmatic dependents).  The base advances only once the launch is enqueued: after a failed launch the next
    // one must not wait for arrivals that never came.
    template <typename Launch>
    int claim(int T, int nCTA, cudaStream_t s, Launch&& launch) {
        const unsigned int arrivals = (unsigned int)T * (unsigned int)nCTA;
        if (base > 0xF0000000u - arrivals) {
            ZRB_CUDA(cudaMemsetAsync(word, 0, sizeof(unsigned int), s));
            base = 0;
        }
        ZRB_TRY(launch(word, base));
        base += arrivals;
        return ZRB_OK;
    }
};

struct zrb_tc_state {
    int Xp[ZRB_MAX_LAYERS + 1] = {}, G4p[ZRB_MAX_LAYERS] = {}, Vp = 0;
    int Fp = 0;                        // pitch of fc_w_h: pad64 of fc.W's width (H_{L-1}; E in a Mixture-of-Softmaxes head)
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
    // upd_pending set = item i still to be applied with `upd`, the update of the step that deferred it (its rule and
    // constants; the clip coefficient in c->scalars[1])
    unsigned upd_pending = 0;
    zrb::UpdateStep upd{};
    bool in_train_step = false;   // tc_forward is running as the first half of a fused train step
    float* colsum_scratch = nullptr;   // row-split partials of the bias-gradient column sums
    int64_t packed_version = 0;
    zrb_mos_params packed_params{};    // (the head tensors only with experts)
    // Mixture-of-Softmaxes head (DESIGN.md section 19), with K = c->experts, E = width[0], H = H_{L-1}, Ua = pad64(K*E),
    // HW = Ua + pad64(K): head_w_h [HW, Xp[L]] = latent.W in rows [0, K*E) and prior.W in rows [Ua, Ua + K), zero rows
    // between; ua [N, HW] fp32 the head GEMM's output (u, then c = tanh(u); a); lat_h [N*K, pad64(E)] the dropped latent
    // rows; logits [N*K, V] and lse [N*K]; dua_h [N, HW] the scaled fp16 [du | da]; dlat [N*K, E] fp32 dc^; headg
    // [Ua + K, H] the head's weight gradients before they are copied out; vjp_s [N*K] the drop-in backward's s.
    int Ua = 0, HW = 0;
    __half* head_w_h = nullptr;
    float* ua = nullptr;
    __half* lat_h = nullptr;
    float* logits = nullptr;
    float* lse = nullptr;
    __half* dua_h = nullptr;
    float* dlat = nullptr;
    float* headg = nullptr;
    float* vjp_s = nullptr;
    bool head_loss_only = false;       // tc_forward of a fused step or eval step: the head stops at the LSEs (no log p)
    std::vector<void*> allocs;
    // persistent recurrence: one plan per layer and direction, each for the layer's width.  Either direction is on for
    // every layer or for none (tc_ctx_init), so fplan[0].ok / bplan[0].ok say which path a step takes.
    zrb::RecPlan fplan[ZRB_MAX_LAYERS] = {};
    __half* w_img_f[ZRB_MAX_LAYERS] = {};
    __half* h0_img[ZRB_MAX_LAYERS] = {};   // image of the state entering the window (step 0's B operand)
    __half* h_img = nullptr;
    GridBarrier fwd_bar, bwd_bar;          // words 0 and 32 of one allocation; shared by the model- and layer-level calls
    zrb::RecPlan bplan[ZRB_MAX_LAYERS] = {};
    __half* w_img_b[ZRB_MAX_LAYERS] = {};
    __half* g_img = nullptr;
    long long* trace = nullptr;   // [2][8 + T*8]: launch stamps + per-step clock stamps (zrb_prof_rec_trace)
    // fused step (zrb_set_embed_sparse): the wgrad GEMMs leave sums of squares of the matrix gradients in
    // c->partials, so clip_grad_norm_ does not re-read them; valid for the gradient buffers keyed by wg_key
    bool wg_ok = false;
    int wg_slots = 0;
    const float* wg_key = nullptr;
    // which weights the W_hh images of each layer (w_img_f / w_img_b, or w_hh_h on the per-timestep path) hold
    // (DESIGN.md section 15): the raw W_hh, W_hh under the weight-drop mask of (seed, step, p), or nothing usable (the
    // update of the weight-drop mode, or the unit-level calls, left them behind p)
    enum WhhKind { kWhhRaw = 0, kWhhMasked, kWhhStale };
    struct WhhImage {
        WhhKind kind = kWhhRaw;
        uint64_t seed = 0, step = 0;
        float p = 0.f;
    } whh_img[ZRB_MAX_LAYERS];

    // ---- which fp16 images each weight matrix has: what a pack or a fused update of it must write -------------------
    zrb::WeightImages row_image(__half* img, int ld) const {
        zrb::WeightImages w;
        w.row = img; w.ld = ld;
        return w;
    }
    zrb::WeightImages w_ih_images(int l) const { return row_image(w_ih_h[l], Xp[l]); }
    zrb::WeightImages fc_w_images() const { return row_image(fc_w_h, Fp); }
    // both recurrences run in the persistent kernels: fplan.ok && bplan.ok, and bplan.ok implies fplan.ok (tc_ctx_init
    // clears bplan.ok when the forward plan is off)
    bool persistent() const { return bplan[0].ok; }
    // W_hh of layer l, recording what its images will hold.  kWhhStale asks for no image: the caller changes p and leaves
    // the images behind it.  Otherwise the slices of each persistent kernel in use, and the row image only where it is
    // read, on the per-timestep path.  row_too: the row image regardless.
    zrb::WeightImages w_hh_images(int l, const WhhImage& holds, bool row_too = false) {
        whh_img[l] = holds;
        zrb::WeightImages w = row_image(nullptr, Xp[l + 1]);
        if (holds.kind == kWhhStale) return w;
        if (row_too || !persistent()) w.row = w_hh_h[l];
        w.fwd = fplan[l].ok ? w_img_f[l] : nullptr; w.fplan = &fplan[l];
        w.bwd = bplan[l].ok ? w_img_b[l] : nullptr; w.bplan = &bplan[l];
        return w;
    }
};

namespace zrb {

// whether work may run as a programmatic dependent beside a recurrence kernel: not while zrb_prof_enable brackets the
// kernel classes with events (a record would sit between the two launches)
static bool pdl_beside_rec(const zrb_ctx* c) { return !c->prof_on; }
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

// zoneout of layer l in this call (DESIGN.md section 20): on or off, the train-mode flags zoneout_flags drew, or the
// eval-mode constants
static ZoneoutSrc zoneout_src(const zrb_ctx* c, int l) {
    ZoneoutSrc z = {};
    z.on = zoneout_on(c) ? 1 : 0;
    z.flags = c->train ? c->zflags[l] : nullptr;
    z.ec = c->z_c; z.ec1 = (float)(1.0 - (double)c->z_c);
    z.eh = c->z_h; z.eh1 = (float)(1.0 - (double)c->z_h);
    return z;
}
// train mode: every layer's flags of (seed, step): sites 3L + 3 + l (c) and 4L + 3 + l (h) over T*B*H_l, per step even in
// the variational mode
static int zoneout_draw(zrb_ctx* c, cudaStream_t s) {
    if (!zoneout_on(c) || !c->train) return ZRB_OK;
    const int L = c->cfg.layers;
    for (int l = 0; l < L; ++l) {
        const MaskSrc mc = make_mask_src(nullptr, c->seed, c->step, 3 * L + 3 + l, c->z_c, 1);
        const MaskSrc mh = make_mask_src(nullptr, c->seed, c->step, 4 * L + 3 + l, c->z_h, 1);
        ZRB_TRY(zoneout_flags(mc, mh, (int64_t)c->T * c->B * c->width[l + 1], c->zflags[l], s));
    }
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
    const int L = c->cfg.layers, V = c->cfg.vocab, Hm = c->max_width;
    const size_t N = (size_t)c->cfg.max_seq * c->cfg.max_batch, B = c->cfg.max_batch;
    for (int s = 0; s <= L; ++s) t->Xp[s] = pad64(c->width[s]);
    int G4m = 0;
    for (int l = 0; l < L; ++l) {
        t->G4p[l] = pad64(4 * c->width[l + 1]);
        if (t->G4p[l] > G4m) G4m = t->G4p[l];
    }
    t->Vp = pad64(V);
    const int K = c->experts, E = c->width[0], H = c->width[L];
    t->Fp = pad64(K ? E : H);
    for (int l = 0; l < L; ++l) {
        const size_t H = c->width[l + 1];
        ZRB_TRY(tc_alloc(c, &t->w_ih_h[l], 4 * H * t->Xp[l]));
        ZRB_TRY(tc_alloc(c, &t->w_hh_h[l], 4 * H * t->Xp[l + 1]));
        ZRB_TRY(tc_alloc(c, &t->hprev_h[l], (N + B) * t->Xp[l + 1]));
    }
    for (int l = 0; l <= L; ++l) ZRB_TRY(tc_alloc(c, &t->x_h[l], N * t->Xp[l]));
    ZRB_TRY(tc_alloc(c, &t->fc_w_h, (size_t)V * t->Fp));
    ZRB_TRY(tc_alloc(c, &t->dG_h, N * G4m));
    ZRB_TRY(tc_alloc(c, &t->dG_h_alt, N * G4m));
    ZRB_TRY(tc_alloc(c, &t->dS_h, N * (K ? K : 1) * t->Vp));
    int colsum_cols = V > 4 * Hm ? V : 4 * Hm;
    if (K) {
        t->Ua = pad64(K * E);
        t->HW = t->Ua + pad64(K);
        const size_t NK = N * K;
        if (K * E > colsum_cols) colsum_cols = K * E;
        ZRB_TRY(tc_alloc(c, &t->head_w_h, (size_t)t->HW * t->Xp[L]));
        ZRB_TRY(tc_alloc(c, &t->ua, N * t->HW));
        ZRB_TRY(tc_alloc(c, &t->lat_h, NK * pad64(E)));
        ZRB_TRY(tc_alloc(c, &t->logits, NK * V));
        ZRB_TRY(tc_alloc(c, &t->lse, NK));
        ZRB_TRY(tc_alloc(c, &t->dua_h, N * t->HW));
        ZRB_TRY(tc_alloc(c, &t->dlat, NK * E));
        ZRB_TRY(tc_alloc(c, &t->headg, (size_t)(t->Ua + K) * H));
        ZRB_TRY(tc_alloc(c, &t->vjp_s, NK));
    }
    ZRB_TRY(tc_alloc(c, &t->colsum_scratch, (size_t)colsum_h_scratch_floats(colsum_cols)));
    // one plan per layer; a direction is persistent only when every layer's plan fits (no mixed step)
    const char* force = getenv("ZRB_REC");
    bool fwd_ok = !(force && !strcmp(force, "steps")), bwd_ok = !(force && !strcmp(force, "fwdonly"));   // A/B switches
    for (int l = 0; l < L; ++l) {
        ZRB_TRY(rec_fwd_plan(c->width[l + 1], c->cfg.max_batch, &t->fplan[l]));
        ZRB_TRY(rec_bwd_plan(c->width[l + 1], c->cfg.max_batch, &t->bplan[l]));
        fwd_ok = fwd_ok && t->fplan[l].ok;
        bwd_ok = bwd_ok && t->bplan[l].ok;
    }
    for (int l = 0; l < L; ++l) {
        if (!fwd_ok) t->fplan[l].ok = 0;
        if (!fwd_ok || !bwd_ok) t->bplan[l].ok = 0;
    }
    size_t h_img = 0, g_img = 0;   // the operand images the layers run one after another share, sized for the largest
    if (fwd_ok) {
        for (int l = 0; l < L; ++l) {
            const RecPlan& fp = t->fplan[l];
            ZRB_TRY(tc_alloc(c, &t->w_img_f[l], (size_t)fp.nCTA * fp.KcS * fp.G * 64 + 16 * 64 /* M=128 over-read */));
            ZRB_TRY(tc_alloc(c, &t->h0_img[l], (size_t)fp.Kc * fp.GBi * 64));
            const size_t n = (size_t)(c->cfg.max_seq + 1) * fp.Kc * fp.GBi * 64;
            if (n > h_img) h_img = n;
        }
        ZRB_TRY(tc_alloc(c, &t->h_img, h_img));
        unsigned int* words = nullptr;
        ZRB_TRY(tc_alloc(c, &words, 64));
        t->fwd_bar.word = words;
        t->bwd_bar.word = words + 32;
    }
    if (getenv("ZRB_REC_TRACE")) ZRB_TRY(tc_alloc(c, &t->trace, (size_t)2 * (8 + c->cfg.max_seq * 8)));
    if (t->bplan[0].ok) {
        for (int l = 0; l < L; ++l) {
            const RecPlan& bp = t->bplan[l];
            ZRB_TRY(tc_alloc(c, &t->w_img_b[l], (size_t)bp.nCTA * bp.KcS * bp.G * 64 + 16 * 64));
            const size_t n = (size_t)2 * 4 * bp.Kc * bp.GBi * 64;
            if (n > g_img) g_img = n;
        }
        ZRB_TRY(tc_alloc(c, &t->g_img, g_img));
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

// the W_hh images layer l's call needs: raw outside the weight-drop mode and in eval mode, else masked with this step's
// mask (DESIGN.md section 15)
static zrb_tc_state::WhhImage whh_wanted(const zrb_ctx* c, int l) {
    zrb_tc_state::WhhImage w;
    if (wd_mask(c, l).active) {
        w.kind = zrb_tc_state::kWhhMasked;
        w.seed = c->wd_seed; w.step = c->step; w.p = c->p_wd;
    }
    return w;
}
static bool whh_current(const zrb_ctx* c, int l) {
    const zrb_tc_state::WhhImage &have = c->tc->whh_img[l], want = whh_wanted(c, l);
    if (have.kind != want.kind) return false;
    return want.kind == zrb_tc_state::kWhhRaw || (have.seed == want.seed && have.step == want.step && have.p == want.p);
}

// build layer l's W_hh images from W with the mask the call needs; row_image: also the row image w_hh_h when the
// persistent kernels do not need it (it is read only on the per-timestep path)
static int tc_pack_whh(zrb_ctx* c, const float* W, int l, bool row_image, cudaStream_t s) {
    const int H = c->width[l + 1];
    const MaskSrc m = wd_mask(c, l);
    const WeightImages w = c->tc->w_hh_images(l, whh_wanted(c, l), row_image);
    if (w.row) ZRB_TRY(convert_pad_f16(W, H, w.row, w.ld, 4 * H, H, 1.f, s, m));
    if (w.fwd) ZRB_TRY(pack_whh_fwd(W, w.fwd, H, *w.fplan, s, m));
    if (w.bwd) ZRB_TRY(pack_whh_bwd(W, w.bwd, H, *w.bplan, s, m));
    return ZRB_OK;
}

// rebuild the fp16 weight images when parameter values changed (main.py:116-117 / zrb_clip_sgd)
// the zrb_params a context reads: zrb_mos_params with experts (DESIGN.md section 19)
static size_t params_bytes(const zrb_ctx* c) { return c->experts ? sizeof(zrb_mos_params) : sizeof(zrb_params); }
static void note_packed(zrb_ctx* c, const zrb_params* p) {
    zrb_tc_state* t = c->tc;
    t->packed_version = c->weights_version;
    memcpy(&t->packed_params, p, params_bytes(c));
}

static int tc_pack_weights(zrb_ctx* c, const zrb_params* p, cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    if (t->packed_version == c->weights_version && !memcmp(&t->packed_params, p, params_bytes(c))) return ZRB_OK;
    ProfScope ps(c, ZRB_PROF_PACK, s);
    const int L = c->cfg.layers, V = c->cfg.vocab;
    for (int l = 0; l < L; ++l) {
        const int In = c->width[l], H = c->width[l + 1];
        ZRB_TRY(convert_pad_f16(p->w_ih[l], In, t->w_ih_h[l], t->Xp[l], 4 * H, In, 1.f, s));
        ZRB_TRY(tc_pack_whh(c, p->w_hh[l], l, true, s));
    }
    const int F = c->experts ? c->width[0] : c->width[L];
    ZRB_TRY(convert_pad_f16(p->fc_w, F, t->fc_w_h, t->Fp, V, F, 1.f, s));
    if (c->experts) {
        const int K = c->experts, H = c->width[L];
        const zrb_mos_params* mp = mos_of(p);
        ZRB_TRY(convert_pad_f16(mp->latent_w, H, t->head_w_h, t->Xp[L], K * c->width[0], H, 1.f, s));
        ZRB_TRY(convert_pad_f16(mp->prior_w, H, t->head_w_h + (size_t)t->Ua * t->Xp[L], t->Xp[L], K, H, 1.f, s));
    }
    note_packed(c, p);
    return ZRB_OK;
}

// One weight matrix of a param_list()-ordered TensorList: its index there, its shape, and the lazy-update item it belongs
// to (layer l, or L for fc.W; see zrb_tc_state::upd_pending).
struct WeightMatrix {
    int i, rows, cols, item;
    enum { kWih, kWhh, kFcW, kPrior, kLatent } kind;
};
struct WeightMatrices {
    WeightMatrix m[2 * ZRB_MAX_LAYERS + 3];
    int n = 0;
    const WeightMatrix* begin() const { return m; }
    const WeightMatrix* end() const { return m + n; }
    const WeightMatrix& fc_w() const { return m[n - 1]; }
};
// The matrices in the order the update launches them: W_ih then W_hh per layer, the head's prior.W and latent.W, then
// fc.W.  This is the one place that knows where param_list() (api.cu) puts them: embed, (w_ih, w_hh, b_ih, b_hh) x L,
// fc_w, fc_b (tied: embed has n = 0, E is fc_w), then with experts prior_w, latent_w, latent_b; and the one place of the
// update path that knows their shapes: W_ih [4H_l, In_l], W_hh [4H_l, H_l], fc.W [V, H_{L-1}] ([V, E] with experts),
// prior.W [K, H_{L-1}], latent.W [K*E, H_{L-1}].  The head's matrices belong to lazy item L with fc.W.
static WeightMatrices tc_matrices(const zrb_ctx* c) {
    const int L = c->cfg.layers, V = c->cfg.vocab, K = c->experts;
    WeightMatrices ms;
    for (int l = 0; l < L; ++l) {
        const int In = c->width[l], H = c->width[l + 1];
        ms.m[ms.n++] = {1 + 4 * l, 4 * H, In, l, WeightMatrix::kWih};
        ms.m[ms.n++] = {2 + 4 * l, 4 * H, H, l, WeightMatrix::kWhh};
    }
    if (K) {
        ms.m[ms.n++] = {3 + 4 * L, K, c->width[L], L, WeightMatrix::kPrior};
        ms.m[ms.n++] = {4 + 4 * L, K * c->width[0], c->width[L], L, WeightMatrix::kLatent};
    }
    ms.m[ms.n++] = {1 + 4 * L, V, K ? c->width[0] : c->width[L], L, WeightMatrix::kFcW};
    return ms;
}
// the images a fused update of m writes; whh: what W_hh's will hold afterwards (zrb_tc_state::w_hh_images)
static WeightImages tc_images(zrb_ctx* c, const WeightMatrix& m, const zrb_tc_state::WhhImage& whh) {
    zrb_tc_state* t = c->tc;
    switch (m.kind) {
        case WeightMatrix::kWhh: return t->w_hh_images(m.item, whh);
        case WeightMatrix::kWih: return t->w_ih_images(m.item);
        case WeightMatrix::kFcW: return t->fc_w_images();
        case WeightMatrix::kPrior: return t->row_image(t->head_w_h + (size_t)t->Ua * t->Xp[m.item], t->Xp[m.item]);
        default: return t->row_image(t->head_w_h, t->Xp[m.item]);
    }
}
// tl for the list kernels once the tile kernels have taken the matrices: their lengths set to 0, which every list
// kernel skips
static TensorList tc_without_matrices(const zrb_ctx* c, const TensorList& tl) {
    TensorList rest = tl;
    for (const WeightMatrix& m : tc_matrices(c)) rest.n[m.i] = 0;
    return rest;
}
// after a fused update of every matrix (applied or pending): the images are current, the next forward needs no pack
static void tc_images_current(zrb_ctx* c, const zrb_params* p) {
    zrb_tc_state* t = c->tc;
    t->wg_ok = false;
    c->weights_version++;
    note_packed(c, p);
}

// st's update of one matrix, with the tile kernels of its rule: update_pack (SGD), update_pack_avg (which also averages
// the new p, DESIGN.md section 16), update_pack_adam (section 21), update_pack_dyn (section 14) or swap_pack.  All
// rebuild the matrix's fp16 images from registers, so the next forward needs no pack.  The exception is W_hh under a
// train-step rule in the weight-drop mode: p (and g) only, and the next forward packs the images with its own mask.
// Dynamic evaluation and the swap leave the raw weights in the W_hh images: evaluation applies no weight drop.
static int tc_update_matrix(zrb_ctx* c, const WeightMatrix& m, const UpdateStep& st, int pdl_smem, cudaStream_t s) {
    zrb_tc_state::WhhImage whh;
    if (st.train() && c->p_wd > 0.f) whh.kind = zrb_tc_state::kWhhStale;
    const WeightImages img = tc_images(c, m, whh);
    float *p = st.tl.p[m.i], *g = st.tl.g[m.i];
    switch (st.kind) {
        case UpdateStep::kSgd:
            return update_pack(p, g, m.rows, m.cols, st.lr, c->scalars, img, c->keep_clipped, s, pdl_smem);
        case UpdateStep::kSgdAvg:
            return update_pack_avg(p, g, st.avg.a[m.i], st.avg.mu, st.avg.first, m.rows, m.cols, st.lr, c->scalars, img,
                                   c->keep_clipped, s, pdl_smem);
        case UpdateStep::kAdam:
            return update_pack_adam(p, g, st.adam.m[m.i], st.adam.v[m.i], st.adam.k, m.rows, m.cols, c->scalars, img,
                                    c->keep_clipped, s, pdl_smem);
        case UpdateStep::kDyn:
            return update_pack_dyn(p, g, st.tg[m.i], st.r[m.i], m.rows, m.cols, st.dyn, img, s);
        case UpdateStep::kSwap:
            return swap_pack(p, st.avg.a[m.i], m.rows, m.cols, img, s);
    }
    return ZRB_E_INVALID;
}

// apply deferred update item `item` (see zrb_tc_state::upd_pending); pdl_smem > 0: as a programmatic dependent of the
// forward recurrence kernel just enqueued on `s`, requesting its plan's beside_smem
static int tc_issue_update(zrb_ctx* c, int item, int pdl_smem, cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    if (!(t->upd_pending & (1u << item))) return ZRB_OK;
    t->upd_pending &= ~(1u << item);
    for (const WeightMatrix& m : tc_matrices(c))
        if (m.item == item) ZRB_TRY(tc_update_matrix(c, m, t->upd, pdl_smem, s));
    return ZRB_OK;
}

int tc_flush_updates(zrb_ctx* c, cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    if (!t || !t->upd_pending) return ZRB_OK;
    ProfScope ps(c, ZRB_PROF_CLIP_SGD, s);
    for (int item = 1; item <= c->cfg.layers; ++item) ZRB_TRY(tc_issue_update(c, item, 0, s));
    return ZRB_OK;
}

// The Mixture-of-Softmaxes head (DESIGN.md section 19) over the last `rows` tokens of the window: [u | a] in one GEMM,
// c and the dropped latent image, the N*K logits rows with fc.b, their LSEs, and (logp non-null) log p [rows, V].
static int tc_mos_head(zrb_ctx* c, const zrb_params* p, int rows, float* logp, cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    const int L = c->cfg.layers, V = c->cfg.vocab, K = c->experts, E = c->width[0], H = c->width[L];
    const int N = c->T * c->B, Xl = t->Xp[L], Ep = pad64(E);
    ProfScope ps(c, ZRB_PROF_PROJ_FWD, s);
    Gemm head;
    head.A = {t->x_h[L] + (size_t)(N - rows) * Xl, Xl}; head.B = {t->head_w_h, Xl};
    head.C = t->ua; head.ldc = t->HW; head.M = rows; head.N = t->Ua + K; head.K = H;
    ZRB_TRY(gemm_f16_tc(head, s));
    ZRB_TRY(mos_latent_fwd(t->ua, t->HW, mos_of(p)->latent_b, t->lat_h, Ep, rows, K, E, N - rows, mos_mask(c), s));
    Gemm logits;
    logits.A = {t->lat_h, Ep}; logits.B = {t->fc_w_h, t->Fp};
    logits.C = t->logits; logits.ldc = V; logits.M = rows * K; logits.N = V; logits.K = E; logits.bias = p->fc_b;
    ZRB_TRY(gemm_f16_tc(logits, s));
    ZRB_TRY(mos_lse(t->logits, rows * K, V, t->lse, s));
    if (logp) ZRB_TRY(mos_logp(t->logits, t->lse, t->ua, t->HW, t->Ua, rows, K, V, logp, V, s));
    return ZRB_OK;
}

int tc_forward(zrb_ctx* c, const zrb_params* p, const int64_t* x, const zrb_states* in, const zrb_states* out,
               float* scores, cudaStream_t s, bool last_only) {
    zrb_tc_state* t = c->tc;
    const int L = c->cfg.layers, V = c->cfg.vocab, T = c->T, B = c->B, N = T * B;
    // deferred updates ride beside the forward recurrences of a fused train step; any other forward applies them first
    const bool ride = t->upd_pending && t->in_train_step && t->fplan[0].ok && pdl_beside_rec(c);
    if (t->upd_pending && !ride) ZRB_TRY(tc_flush_updates(c, s));
    ZRB_TRY(tc_pack_weights(c, p, s));
    {   // state copies (in / out may be the same buffers), fp16 h0 rows and images, saved tokens: one launch
        FwdPrep fp = {};
        for (int l = 0; l < L; ++l) {
            fp.in_h[l] = in->h[l]; fp.in_c[l] = in->c[l]; fp.h0s[l] = c->h0s[l]; fp.c0s[l] = c->c0s[l];
            fp.hprev_h[l] = t->hprev_h[l]; fp.h0_img[l] = t->fplan[l].ok ? t->h0_img[l] : nullptr;
            fp.rm[l] = rec_mask(c, l);
            fp.H[l] = c->width[l + 1]; fp.Hp[l] = t->Xp[l + 1]; fp.GB[l] = t->fplan[l].GBi; fp.Kc[l] = t->fplan[l].Kc;
        }
        fp.x = x; fp.x_saved = c->x_saved;
        fp.L = L; fp.B = B; fp.N = N;
        ZRB_TRY(fwd_prep(fp, s));
    }
    ZRB_TRY(zoneout_draw(c, s));
    {
        ProfScope ps(c, ZRB_PROF_EMBED_FWD, s);
        // tied: E's update (item L) is still deferred -> gather through it; the update itself rides beside the last
        // recurrence, before the projection reads fc_w_h
        const bool through = ride && c->tied && (t->upd_pending & (1u << L));
        ZRB_TRY(embed_dropout_fwd(p->embed_w, x, nullptr, t->x_h[0], t->Xp[0], N, c->width[0], V, site_mask(c, 0), ed_mask(c), s,
                                  through ? t->upd.tl.g[tc_matrices(c).fc_w().i] : nullptr, t->upd.lr, c->scalars));
    }
    for (int l = 0; l < L; ++l) {
        const int In = c->width[l], H = c->width[l + 1], Xi = t->Xp[l], Hp = t->Xp[l + 1];
        const size_t bh = (size_t)B * H * sizeof(float);
        const RecPlan& fplan = t->fplan[l];
        float* G = c->gates[l];
        if (!whh_current(c, l)) {
            // weight drop (DESIGN.md section 15): this step's masked images, or the raw ones after a masked step.  After
            // the layer's deferred update (enqueued beside the previous recurrence), before its input GEMM: never between
            // that GEMM and its programmatic-dependent recurrence
            ProfScope ps(c, ZRB_PROF_PACK, s);
            ZRB_TRY(tc_pack_whh(c, p->w_hh[l], l, false, s));
        }
        {
            ProfScope ps(c, ZRB_PROF_GEMM_IN, s);
            Gemm xw;
            xw.A = {t->x_h[l], Xi}; xw.B = {t->w_ih_h[l], Xi};
            xw.C = G; xw.ldc = 4 * H; xw.M = N; xw.N = 4 * H; xw.K = In; xw.bias = p->b_ih[l]; xw.bias2 = p->b_hh[l];
            ZRB_TRY(gemm_f16_tc(xw, s));
        }
        MaskSrc m = site_mask(c, l + 1), rm = rec_mask(c, l);
        const ZoneoutSrc zo = zoneout_src(c, l);
        // AR / TAR (DESIGN.md section 17) reads the last layer's fp32 h (the per-timestep path always writes it)
        const bool reg_h = t->in_train_step && reg_on(c) && l == L - 1;
        ProfScope ps(c, ZRB_PROF_REC_FWD, s);
        if (fplan.ok) {
            ZRB_TRY(t->fwd_bar.claim(T, fplan.nCTA, s, [&](unsigned int* word, unsigned int base) {
                RecFwdArgs a = {};
                a.w_img = t->w_img_f[l]; a.h0_img = t->h0_img[l]; a.h_img = t->h_img; a.gates = G; a.c0 = c->c0s[l];
                a.cst = c->cst[l]; a.h_last = out->h[l]; a.c_last = out->c[l]; a.hprev_h = t->hprev_h[l];
                a.y_h = t->x_h[l + 1]; a.h_f32 = reg_h ? c->hraw[l] : nullptr; a.counter = word; a.base = base;
                a.T = T; a.B = B; a.H = H; a.Hp = Hp; a.m = m; a.rm = rm; a.trace = t->trace;
                a.zo = zo; a.h0 = c->h0s[l]; a.ctil = c->ctil[l];
                return lstm_rec_fwd(fplan, tc_watchdog(c), a, s);
            }));
            // deferred update of the NEXT layer's matrices (or of fc.W after the last layer): on the idle SMs, beside
            // this recurrence; their consumers (the next input GEMM / the projection) are enqueued behind them
            if (ride) ZRB_TRY(tc_issue_update(c, l + 1, fplan.beside_smem, s));
            continue;
        }
        for (int tt = 0; tt < T; ++tt) {
            const float* c_prev = tt ? c->cst[l] + (size_t)(tt - 1) * B * H : c->c0s[l];
            float* Gt = G + (size_t)tt * B * 4 * H;
            Gemm hw;
            hw.A = {t->hprev_h[l] + (size_t)tt * B * Hp, Hp}; hw.B = {t->w_hh_h[l], Hp};
            hw.C = Gt; hw.ldc = 4 * H; hw.M = B; hw.N = 4 * H; hw.K = H; hw.accumulate = true;
            ZRB_TRY(gemm_f16_tc(hw, s));
            const float* h_prev = tt ? c->hraw[l] + (size_t)(tt - 1) * B * H : c->h0s[l];
            ZRB_TRY(lstm_cell_fwd_tc(Gt, c_prev, c->cst[l] + (size_t)tt * B * H, c->hraw[l] + (size_t)tt * B * H,
                                     t->hprev_h[l] + (size_t)(tt + 1) * B * Hp, t->x_h[l + 1] + (size_t)tt * B * Hp, Hp, B,
                                     H, (int64_t)tt * B * H, (int64_t)N * H, m, rm, s, zo.on ? &zo : nullptr, h_prev,
                                     zo.on ? c->ctil[l] + (size_t)tt * B * H : nullptr));
        }
        ZRB_CUDA(cudaMemcpyAsync(out->h[l], c->hraw[l] + (size_t)(T - 1) * B * H, bh, cudaMemcpyDeviceToDevice, s));
        ZRB_CUDA(cudaMemcpyAsync(out->c[l], c->cst[l] + (size_t)(T - 1) * B * H, bh, cudaMemcpyDeviceToDevice, s));
    }
    if (scores && c->experts) return tc_mos_head(c, p, last_only ? B : N, t->head_loss_only ? nullptr : scores, s);
    if (scores) {
        ProfScope ps(c, ZRB_PROF_PROJ_FWD, s);
        const int rows = last_only ? B : N;
        const int Xl = t->Xp[L];
        Gemm proj;
        proj.A = {t->x_h[L] + (size_t)(N - rows) * Xl, Xl}; proj.B = {t->fc_w_h, Xl};
        proj.C = scores; proj.ldc = V; proj.M = rows; proj.N = V; proj.K = c->width[L]; proj.bias = p->fc_b;
        ZRB_TRY(gemm_f16_tc(proj, s));
    }
    return ZRB_OK;
}

const __half* tc_last_layer_image(const zrb_ctx* c) { return c->tc->x_h[c->cfg.layers]; }

// next block of n sum-of-squares slots, or null when the step does not fuse the norm
static float* wgrad_slots(zrb_ctx* c, int n) {
    zrb_tc_state* t = c->tc;
    if (!t->wg_ok) return nullptr;
    if (t->wg_slots + n > kNormGemm) {
        t->wg_ok = false;   // does not fit: the update takes the norm over the whole buffers instead
        return nullptr;
    }
    float* out = c->partials + norm_partials_base() + kNormExtra + t->wg_slots;
    t->wg_slots += n;
    return out;
}
// ... for the weight gradient the GEMM d writes
static float* wgrad_sumsq(zrb_ctx* c, const Gemm& d) { return wgrad_slots(c, gemm_f16_tc_sumsq_slots(d).first); }

// Mixture-of-Softmaxes head backward from dS_h (N*K rows) and the da columns of dua_h: fc.W / fc.b over the N*K rows,
// dc^ -> du, then dh = [du | da] [latent.W; prior.W] into dY and the head's weight gradients in one GEMM
static int tc_mos_backward(zrb_ctx* c, const zrb_params* g, float* dY, cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    const int L = c->cfg.layers, V = c->cfg.vocab, N = c->T * c->B, H = c->width[L], K = c->experts, E = c->width[0];
    const int NK = N * K, Xl = t->Xp[L], Vp = t->Vp, Ep = pad64(E);
    const float inv = 1.f / kGradScale;
    ProfScope ps(c, ZRB_PROF_PROJ_BWD, s);
    t->wg_ok = c->fused_norm;
    t->wg_slots = 0;
    t->wg_key = g->fc_w;
    t->pending = 0;
    // dc^[NK,E] = dS[NK,V] * W[V,E]; dW[V,E] = dS^T * c^ (contraction over the N*K rows); fc.b = column sums
    Gemm dlat;
    dlat.A = {t->dS_h, Vp}; dlat.B = {t->fc_w_h, t->Fp, true};
    dlat.C = t->dlat; dlat.ldc = E; dlat.M = NK; dlat.N = E; dlat.K = V; dlat.alpha = inv;
    ZRB_TRY(gemm_f16_tc(dlat, s));
    ZRB_TRY(colsum_h(t->dS_h, Vp, g->fc_b, nullptr, NK, V, inv, t->colsum_scratch, s));
    Gemm dfc;
    dfc.A = {t->dS_h, Vp, true}; dfc.B = {t->lat_h, Ep, true};
    dfc.C = g->fc_w; dfc.ldc = E; dfc.M = V; dfc.N = E; dfc.K = NK; dfc.alpha = inv;
    dfc.sumsq = wgrad_sumsq(c, dfc);
    ZRB_TRY(gemm_f16_tc(dfc, s));
    ZRB_TRY(mos_latent_bwd(t->dlat, t->ua, t->HW, t->dua_h, t->HW, N, K, E, mos_mask(c), s));
    const int M = t->Ua + K;   // [du | da] columns, zero between K*E and Ua
    Gemm dh;
    dh.A = {t->dua_h, t->HW}; dh.B = {t->head_w_h, Xl, true};
    dh.C = dY; dh.ldc = H; dh.M = N; dh.N = H; dh.K = M; dh.alpha = inv;
    ZRB_TRY(gemm_f16_tc(dh, s));
    Gemm dhead;
    dhead.A = {t->dua_h, t->HW, true}; dhead.B = {t->x_h[L], Xl, true};
    dhead.C = t->headg; dhead.ldc = H; dhead.M = M; dhead.N = H; dhead.K = N; dhead.alpha = inv;
    dhead.sumsq = wgrad_sumsq(c, dhead);   // the rows between K*E and Ua are zero: the slots sum both tensors
    ZRB_TRY(gemm_f16_tc(dhead, s));
    const zrb_mos_params* gm = mos_of(g);
    ZRB_CUDA(cudaMemcpyAsync(gm->latent_w, t->headg, (size_t)K * E * H * sizeof(float), cudaMemcpyDeviceToDevice, s));
    ZRB_CUDA(cudaMemcpyAsync(gm->prior_w, t->headg + (size_t)t->Ua * H, (size_t)K * H * sizeof(float),
                             cudaMemcpyDeviceToDevice, s));
    return colsum_h(t->dua_h, t->HW, gm->latent_b, nullptr, N, K * E, inv, t->colsum_scratch, s);
}

// fc.W's weight gradient dW[V,H] = dS^T[V,N] * A[N,H] (both operands MN-major: contraction over tokens), with its norm
// slots: claimed here, so call it where the GEMM is launched
static Gemm fc_w_wgrad(zrb_ctx* c, const zrb_params* g) {
    const zrb_tc_state* t = c->tc;
    const int L = c->cfg.layers, H = c->width[L];
    Gemm d;
    d.A = {t->dS_h, t->Vp, true}; d.B = {t->x_h[L], t->Xp[L], true};
    d.C = g->fc_w; d.ldc = H; d.M = c->cfg.vocab; d.N = H; d.K = c->T * c->B; d.alpha = 1.f / kGradScale;
    d.sumsq = wgrad_sumsq(c, d);
    return d;
}

// backward from the scaled fp16 image dS_h already in place
// projection backward: afterwards fc.W / fc.b gradients are complete and c->bwd_dy holds d loss / d act[L]
static int tc_backward_head(zrb_ctx* c, const zrb_params* p, const zrb_params* g, cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    const int L = c->cfg.layers, V = c->cfg.vocab, N = c->T * c->B, H = c->width[L];
    const int Hp = t->Xp[L], Vp = t->Vp;
    const float inv = 1.f / kGradScale;
    float* dY = c->dy;
    c->bwd_dy = c->dy;
    c->bwd_dx = c->dx;
    c->bwd_next_layer = L - 1;
    if (c->experts) return tc_mos_backward(c, g, dY, s);
    {
        ProfScope ps(c, ZRB_PROF_PROJ_BWD, s);
        // dA[N,H] = dS[N,V] * W[V,H]       (W image read MN-major)
        Gemm dA;
        dA.A = {t->dS_h, Vp}; dA.B = {t->fc_w_h, Hp, true};
        dA.C = dY; dA.ldc = H; dA.M = N; dA.N = H; dA.K = V; dA.alpha = inv;
        ZRB_TRY(gemm_f16_tc(dA, s));
        t->wg_ok = c->fused_norm;
        t->wg_slots = 0;
        t->wg_key = g->fc_w;
        ZRB_TRY(colsum_h(t->dS_h, Vp, g->fc_b, nullptr, N, V, inv, t->colsum_scratch, s));
        // dW: nothing downstream in backward reads it: with deferral on it runs underneath the first backward
        // recurrence instead of before it.
        t->pending = 0;
        if (t->defer_wgrad && t->persistent() && pdl_beside_rec(c)) t->pending = 1;
        else ZRB_TRY(gemm_f16_tc(fc_w_wgrad(c, g), s));
    }
    return ZRB_OK;
}

// the two weight gradients of layer l from dG (scaled fp16, [N,G4p]): ONE launch, dG is the shared A operand
// Weight drop (DESIGN.md section 15): the GEMM leaves dW_eff in g->w_hh[l]; the masking pass that follows it in stream
// order makes it scale * m * dW_eff in place and writes its sums of squares into the norm slots instead of the GEMM.
static int tc_layer_wgrads(zrb_ctx* c, const zrb_params* g, int l, const __half* dG_h, bool pdl, cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    const int In = c->width[l], H = c->width[l + 1], N = c->T * c->B;
    const MaskSrc wm = wd_mask(c, l);
    Gemm dw;   // dW_ih[4H,In] = dG^T * x_l, and as the dual problem dW_hh[4H,H] = dG^T * h_prev
    dw.A = {dG_h, t->G4p[l], true}; dw.B = {t->x_h[l], t->Xp[l], true};
    dw.C = g->w_ih[l]; dw.ldc = In; dw.M = 4 * H; dw.N = In; dw.K = N; dw.alpha = 1.f / kGradScale; dw.pdl = pdl;
    dw.dual.B = t->hprev_h[l]; dw.dual.C = g->w_hh[l]; dw.dual.N = H; dw.dual.ldb = t->Xp[l + 1]; dw.dual.ldc = H;
    const GemmSlots n = gemm_f16_tc_sumsq_slots(dw);
    dw.sumsq = wgrad_slots(c, n.first);
    if (!wm.active) dw.dual.sumsq = wgrad_slots(c, n.dual);
    ZRB_TRY(gemm_f16_tc(dw, s));
    if (!wm.active) return ZRB_OK;
    return weight_drop(g->w_hh[l], g->w_hh[l], (int64_t)4 * H * H, wm, wgrad_slots(c, kWeightDropBlocks), s);
}

// launch what tc_backward_head / the previous layer deferred, as a programmatic dependent of the recurrence kernel
// that was just enqueued on `s`
static int tc_issue_pending(zrb_ctx* c, const zrb_params* g, cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    const int kind = t->pending;
    t->pending = 0;
    // (no event bracket here: an event record between the recurrence kernel and its programmatic dependent would sit
    // between the two launches; while profiling, pdl_beside_rec defers nothing)
    if (kind == 1) {
        Gemm dw = fc_w_wgrad(c, g);
        dw.pdl = true;
        return gemm_f16_tc(dw, s);
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
    const int In = c->width[l], H = c->width[l + 1], V = c->cfg.vocab, T = c->T, B = c->B, N = T * B;
    const int Xi = t->Xp[l], Hp = t->Xp[l + 1], G4p = t->G4p[l];
    const size_t bh = (size_t)B * H;
    const RecPlan& bplan = t->bplan[l];
    const float inv = 1.f / kGradScale;
    if (l != c->bwd_next_layer) {
        set_error("backward layers must be visited in order L-1..0 (expected %d, got %d)", c->bwd_next_layer, l);
        return ZRB_E_STATE;
    }
    float* dY = c->bwd_dy;
    float* dX = c->bwd_dx;
    __half* dG_h = (l & 1) ? t->dG_h_alt : t->dG_h;
    const float* r = (c->reg_use && l == c->cfg.layers - 1) ? c->reg_r : nullptr;   // AR / TAR gradient (section 17)
    {
        MaskSrc m = site_mask(c, l + 1), rm = rec_mask(c, l);
        const ZoneoutSrc zo = zoneout_src(c, l);
        if (bplan.ok) {
            ProfScope ps(c, ZRB_PROF_REC_BWD, s);
            ZRB_TRY(t->bwd_bar.claim(T, bplan.nCTA, s, [&](unsigned int* word, unsigned int base) {
                RecBwdArgs a = {};
                a.w_img = t->w_img_b[l]; a.g_img = t->g_img; a.dy = dY; a.r = r; a.gates = c->gates[l];
                a.cst = c->cst[l]; a.c0 = c->c0s[l]; a.dG_h = dG_h; a.db1 = g->b_ih[l]; a.db2 = g->b_hh[l];
                a.db_scratch = c->dG;   // [N,4H] fp32, idle on this path
                a.counter = word; a.base = base;
                a.T = T; a.B = B; a.H = H; a.G4p = G4p; a.m = m; a.rm = rm;
                a.trace = t->trace ? t->trace + 8 + (size_t)c->cfg.max_seq * 8 : nullptr;
                a.zo = zo; a.ctil = c->ctil[l];
                return lstm_rec_bwd(bplan, tc_watchdog(c), a, s);
            }));
            ZRB_TRY(tc_issue_pending(c, g, s));   // runs on the SMs the cluster kernel leaves idle
        } else {
            ProfScope ps(c, ZRB_PROF_REC_BWD, s);
            ZRB_CUDA(cudaMemsetAsync(c->dc, 0, bh * sizeof(float), s));   // (the persistent kernel keeps dc in registers)
            if (zo.on) ZRB_CUDA(cudaMemsetAsync(c->zhcarry, 0, bh * sizeof(float), s));
            for (int tt = T - 1; tt >= 0; --tt) {
                const float* c_prev = tt ? c->cst[l] + (size_t)(tt - 1) * bh : c->c0s[l];
                const float* c_t = (zo.on ? c->ctil[l] : c->cst[l]) + (size_t)tt * bh;   // (zoneout: c~_t)
                ZRB_TRY(lstm_cell_bwd_tc(dY + (size_t)tt * bh, tt == T - 1 ? nullptr : c->dh_rec, c->dc,
                                         c->gates[l] + (size_t)tt * B * 4 * H, c_t, c_prev,
                                         c->dG + (size_t)tt * B * 4 * H, dG_h + (size_t)tt * B * G4p, G4p, B, H,
                                         (int64_t)tt * bh, (int64_t)N * H, m, rm, s, r ? r + (size_t)tt * bh : nullptr,
                                         zo.on ? &zo : nullptr, c->zhcarry));
                if (tt == 0) continue;
                Gemm dh;   // dh_{t-1}[B,H] = dG_t[B,4H] * W_hh[4H,H]
                dh.A = {dG_h + (size_t)tt * B * G4p, G4p}; dh.B = {t->w_hh_h[l], Hp, true};
                dh.C = c->dh_rec; dh.ldc = H; dh.M = B; dh.N = H; dh.K = 4 * H; dh.alpha = inv;
                ZRB_TRY(gemm_f16_tc(dh, s));
            }
        }
        {
            ProfScope ps(c, ZRB_PROF_GEMM_DX, s);
            Gemm dx;
            dx.A = {dG_h, G4p}; dx.B = {t->w_ih_h[l], Xi, true};
            dx.C = dX; dx.ldc = In; dx.M = N; dx.N = In; dx.K = 4 * H; dx.alpha = inv;
            ZRB_TRY(gemm_f16_tc(dx, s));
        }
        // dW_ih, dW_hh: nothing downstream in backward reads them -> for l > 0 they run underneath the next layer's
        // recurrence (which writes the other dG buffer); the bias gradients come out of the recurrence kernel itself
        if (t->defer_wgrad && bplan.ok && l > 0 && pdl_beside_rec(c)) {
            t->pending = 2;
            t->pending_layer = l;
        } else {
            ProfScope ps(c, ZRB_PROF_GEMM_WGRAD, s);
            ZRB_TRY(tc_layer_wgrads(c, g, l, dG_h, false, s));
        }
        if (!bplan.ok) ZRB_TRY(colsum(c->dG, g->b_ih[l], g->b_hh[l], N, 4 * H, s));
        float* tmp = dY; dY = dX; dX = tmp;
    }
    c->bwd_dy = dY;
    c->bwd_dx = dX;
    c->bwd_next_layer = l - 1;
    if (l > 0) return ZRB_OK;
    ProfScope ps(c, ZRB_PROF_EMBED_BWD, s);
    const int E = In;   // dY now holds d loss / d act[0], [N, E]
    const MaskSrc m0 = site_mask(c, 0), em = ed_mask(c);
    if (c->embed_rows_out) return embed_rows(dY, c->x_saved, c->embed_rows_out, N, E, V, m0, em, s);
    if (c->tied) {
        // g->embed_w holds G_proj (the projection's wgrad GEMM overwrote every row): add the fixed-point row sums, with
        // dX (free now) as the rows buffer; the fused norm's extra slots get the correction from G_proj^2 to dE^2
        ZRB_TRY(embed_rows(dY, c->x_saved, dX, N, E, V, m0, em, s));
        return embed_scatter_rows(c->x_saved, dX, g->embed_w, N, E, V, c->emb_first, c->emb_acc, s, true,
                                  c->fused_norm ? c->partials + norm_partials_base() : nullptr, kNormExtra);
    }
    if (c->emb_sparse && c->emb_prev_grad == g->embed_w) {
        ZRB_TRY(embed_zero_rows(g->embed_w, c->emb_prev_ids, c->emb_prev_n, E, V, s));   // only last window's rows are non-zero
    } else {
        ZRB_CUDA(cudaMemsetAsync(g->embed_w, 0, (size_t)V * E * sizeof(float), s));
    }
    ZRB_TRY(embed_dropout_bwd(dY, c->x_saved, g->embed_w, N, E, V, m0, em, s));
    if (c->emb_sparse) {
        ZRB_CUDA(cudaMemcpyAsync(c->emb_prev_ids, c->x_saved, (size_t)N * sizeof(int64_t), cudaMemcpyDeviceToDevice, s));
        c->emb_prev_n = N;
        c->emb_prev_grad = g->embed_w;
    }
    return ZRB_OK;
}

static int tc_backward_from_image(zrb_ctx* c, const zrb_params* p, const zrb_params* g, cudaStream_t s) {
    c->tc->defer_wgrad = true;
    ZRB_TRY(tc_backward_head(c, p, g, s));
    for (int l = c->cfg.layers - 1; l >= 0; --l) ZRB_TRY(tc_backward_layer(c, p, g, l, s));
    return ZRB_OK;
}

int tc_backward(zrb_ctx* c, const zrb_params* p, const float* dscores, const zrb_params* g, cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    const int N = c->T * c->B, V = c->cfg.vocab;
    if (c->experts) {   // dscores = dL / d log p: the mixture's VJP (log p itself goes to the scratch c->dscores)
        ProfScope ps(c, ZRB_PROF_SOFTMAX, s);
        ZRB_TRY(mos_vjp(t->logits, t->lse, t->ua, t->HW, t->Ua, N, c->experts, V, dscores, c->dscores, t->vjp_s, t->dS_h,
                        t->Vp, t->dua_h, t->HW, s));
    } else {
        ZRB_TRY(convert_pad_f16(dscores, V, t->dS_h, t->Vp, N, V, kGradScale, s));
    }
    return tc_backward_from_image(c, p, g, s);
}

// The first half of a fused gradient step: the forward over the window, the loss, and the scaled fp16 image of dscores
// in dS_h.  train = 1: dropout on with the masks of (seed, step), pending lazy updates ride beside the forward
// recurrences, and AR / TAR is computed when it is on; train = 0: the eval-mode loss.
static int tc_step_forward(zrb_ctx* c, const zrb_params* p, const int64_t* x, const int64_t* y, int T, int B,
                           const zrb_states* in, const zrb_states* out, int train, uint64_t seed, uint64_t step,
                           float* loss, cudaStream_t s) {
    c->T = T; c->B = B; c->train = train; c->seed = seed; c->step = step;
    c->have_fwd = false;
    c->reg_use = false;
    zrb_tc_state* t = c->tc;
    t->in_train_step = train != 0;
    t->head_loss_only = true;
    const int frc = tc_forward(c, p, x, in, out, c->scores, s);
    t->in_train_step = false;   // before the return code is tested: a failed forward must not leave it set
    t->head_loss_only = false;
    ZRB_TRY(frc);
    c->have_fwd = true;
    {
        ProfScope ps(c, ZRB_PROF_SOFTMAX, s);
        if (c->experts)
            ZRB_TRY(mos_nll_grad(t->logits, t->lse, t->ua, t->HW, t->Ua, y, T * B, c->experts, c->cfg.vocab, B,
                                 c->row_loss, loss, t->dS_h, t->Vp, t->dua_h, t->HW, s));
        else
            ZRB_TRY(softmax_nll(c->scores, y, T * B, c->cfg.vocab, B, c->row_loss, loss, nullptr, nullptr, s, t->dS_h,
                                t->Vp, kGradScale));
    }
    if (train && reg_on(c)) ZRB_TRY(reg_compute(c, s));   // AR / TAR: between the softmax and the projection's backward
    return ZRB_OK;
}

int tc_train_step_grads(zrb_ctx* c, const zrb_params* p, const zrb_params* g, const int64_t* x, const int64_t* y,
                        int T, int B, const zrb_states* in, const zrb_states* out, uint64_t seed, uint64_t step,
                        float* loss, cudaStream_t s) {
    ZRB_TRY(tc_step_forward(c, p, x, y, T, B, in, out, 1, seed, step, loss, s));
    return tc_backward_from_image(c, p, g, s);
}

// the gradient of the eval-mode loss (DESIGN.md section 14): the fused gradient path with c->train = 0, so that every
// site_mask / rec_mask is off while tc_forward still keeps the activations; pending lazy updates are applied first (the
// forward runs outside a train step), and the loss has no AR / TAR.  No clip norm follows, so the wgrad epilogues write
// no sum-of-squares slots.
int tc_eval_grads(zrb_ctx* c, const zrb_params* p, const zrb_params* g, const int64_t* x, const int64_t* y, int T, int B,
                  const zrb_states* in, const zrb_states* out, float* loss, cudaStream_t s) {
    ZRB_TRY(tc_step_forward(c, p, x, y, T, B, in, out, 0, 0, 0, loss, s));
    const bool fused = c->fused_norm;
    c->fused_norm = false;
    const int rc = tc_backward_from_image(c, p, g, s);
    c->fused_norm = fused;
    c->tc->wg_ok = false;
    return rc;
}

// zrb_eval_step of a Mixture-of-Softmaxes context: the eval-mode forward through the LSEs, then the mixture's row losses
int tc_mos_eval_step(zrb_ctx* c, const zrb_params* p, const int64_t* x, const int64_t* y, const zrb_states* in,
                     const zrb_states* out, float* loss, float* tgt_prob, cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    t->head_loss_only = true;
    const int frc = tc_forward(c, p, x, in, out, c->scores, s);
    t->head_loss_only = false;
    ZRB_TRY(frc);
    return mos_nll_eval(t->logits, t->lse, t->ua, t->HW, t->Ua, y, c->T * c->B, c->experts, c->cfg.vocab, c->B,
                        c->row_loss, loss, tgt_prob, s);
}

int tc_train_step_begin(zrb_ctx* c, const zrb_params* p, const zrb_params* g, const int64_t* x, const int64_t* y,
                        int T, int B, const zrb_states* in, const zrb_states* out, uint64_t seed, uint64_t step,
                        float* loss, cudaStream_t s) {
    ZRB_TRY(tc_step_forward(c, p, x, y, T, B, in, out, 1, seed, step, loss, s));
    c->tc->defer_wgrad = false;   // phased backward: every bucket is complete when its call returns
    return tc_backward_head(c, p, g, s);
}

int tc_train_step_layer(zrb_ctx* c, const zrb_params* p, const zrb_params* g, int l, cudaStream_t s) {
    return tc_backward_layer(c, p, g, l, s);
}

void tc_rec_plans(const zrb_ctx* c, int l, int32_t* h_out) {
    const RecPlan* plans[2] = {&c->tc->fplan[l], &c->tc->bplan[l]};
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
    const int H = c->cfg.hidden, N = T * B, Hp = t->Xp[0];   // (a context of one width: every pitch is Hp)
    const RecPlan &fplan = t->fplan[0], &bplan = t->bplan[0];
    if (!fplan.ok || !bplan.ok) {
        set_error("zrb_lstm_layer_fwd needs the persistent recurrence kernels (shape H=%d B=%d does not fit them)", H, B);
        return ZRB_E_INVALID;
    }
    ZRB_TRY(tc_flush_updates(c, s));
    c->T = T; c->B = B; c->train = 0;
    t->packed_version = 0;                       // slot 0 is about to hold this call's weights
    t->whh_img[0].kind = zrb_tc_state::kWhhStale;
    ZRB_TRY(convert_pad_f16(w_ih, H, t->w_ih_h[0], Hp, 4 * H, H, 1.f, s));
    ZRB_TRY(pack_whh_fwd(w_hh, t->w_img_f[0], H, fplan, s));
    ZRB_TRY(pack_whh_bwd(w_hh, t->w_img_b[0], H, bplan, s));
    ZRB_TRY(convert_pad_f16(x, H, t->x_h[0], Hp, N, H, 1.f, s));
    FwdPrep fp = {};
    fp.in_h[0] = h0; fp.in_c[0] = c0; fp.h0s[0] = c->h0s[0]; fp.c0s[0] = c->c0s[0];
    fp.hprev_h[0] = t->hprev_h[0]; fp.h0_img[0] = t->h0_img[0];
    fp.x = nullptr; fp.x_saved = nullptr;
    fp.L = 1; fp.B = B; fp.H[0] = H; fp.Hp[0] = Hp; fp.GB[0] = fplan.GBi; fp.Kc[0] = fplan.Kc; fp.N = 0;
    ZRB_TRY(fwd_prep(fp, s));
    Gemm xw;
    xw.A = {t->x_h[0], Hp}; xw.B = {t->w_ih_h[0], Hp};
    xw.C = c->gates[0]; xw.ldc = 4 * H; xw.M = N; xw.N = 4 * H; xw.K = H; xw.bias = b_ih; xw.bias2 = b_hh;
    ZRB_TRY(gemm_f16_tc(xw, s));
    MaskSrc m = make_mask_src(nullptr, 0, 0, 0, 0.f, 0);    // no dropout at this level: the caller applies it (model.py:105,108)
    ZRB_TRY(t->fwd_bar.claim(T, fplan.nCTA, s, [&](unsigned int* word, unsigned int base) {
        RecFwdArgs a = {};
        a.w_img = t->w_img_f[0]; a.h0_img = t->h0_img[0]; a.h_img = t->h_img; a.gates = c->gates[0]; a.c0 = c->c0s[0];
        a.cst = c->cst[0]; a.h_last = hT; a.c_last = cT; a.hprev_h = t->hprev_h[0]; a.y_h = t->x_h[1]; a.h_f32 = y;
        a.counter = word; a.base = base; a.T = T; a.B = B; a.H = H; a.Hp = Hp; a.m = m; a.rm = m;
        return lstm_rec_fwd(fplan, tc_watchdog(c), a, s);
    }));
    c->have_fwd = false;                         // a model-level backward must not follow this
    c->layer_fwd_ok = true;
    return ZRB_OK;
}

int tc_layer_bwd(zrb_ctx* c, const float* dy, float* dx, float* dw_ih, float* dw_hh, float* db_ih, float* db_hh,
                 cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    const int H = c->cfg.hidden, T = c->T, B = c->B, N = T * B, Hp = t->Xp[0], G4p = t->G4p[0];
    const RecPlan& bplan = t->bplan[0];
    if (!c->layer_fwd_ok) {
        set_error("zrb_lstm_layer_bwd without a preceding zrb_lstm_layer_fwd");
        return ZRB_E_STATE;
    }
    MaskSrc m = make_mask_src(nullptr, 0, 0, 0, 0.f, 0);
    ZRB_TRY(t->bwd_bar.claim(T, bplan.nCTA, s, [&](unsigned int* word, unsigned int base) {
        RecBwdArgs a = {};
        a.w_img = t->w_img_b[0]; a.g_img = t->g_img; a.dy = dy; a.gates = c->gates[0]; a.cst = c->cst[0];
        a.c0 = c->c0s[0]; a.dG_h = t->dG_h; a.db1 = db_ih; a.db2 = db_hh; a.db_scratch = c->dG;
        a.counter = word; a.base = base;
        a.T = T; a.B = B; a.H = H; a.G4p = G4p; a.m = m; a.rm = m;
        return lstm_rec_bwd(bplan, tc_watchdog(c), a, s);
    }));
    const float inv = 1.f / kGradScale;
    if (dx) {
        Gemm dX;
        dX.A = {t->dG_h, G4p}; dX.B = {t->w_ih_h[0], Hp, true};
        dX.C = dx; dX.ldc = H; dX.M = N; dX.N = H; dX.K = 4 * H; dX.alpha = inv;
        ZRB_TRY(gemm_f16_tc(dX, s));
    }
    Gemm dw;   // dW_ih and, as the dual problem, dW_hh; never norm slots: those belong to the model-level step
    dw.A = {t->dG_h, G4p, true}; dw.B = {t->x_h[0], Hp, true};
    dw.C = dw_ih; dw.ldc = H; dw.M = 4 * H; dw.N = H; dw.K = N; dw.alpha = inv;
    dw.dual.B = t->hprev_h[0]; dw.dual.C = dw_hh; dw.dual.N = H; dw.dual.ldb = Hp; dw.dual.ldc = H;
    ZRB_TRY(gemm_f16_tc(dw, s));
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

// One update: the train step's clip + SGD (main.py:114-117), SGD with iterate averaging (every tensor's new value
// averaged in the same passes, DESIGN.md section 16) or Adam (the moments in the same passes, section 21); the
// dynamic-evaluation update (section 14); or the exchange of the weights with their average (section 16).  The
// matrices' passes also write the fp16 operand images of the new weights, so the next forward needs no pack pass.
// Adam updates the embedding densely: its moments decay in every row.  Only a train step's update is deferred.
int tc_apply_update(zrb_ctx* c, const zrb_params* p, const UpdateStep& st, float max_norm, float* norm_out,
                    cudaStream_t s) {
    zrb_tc_state* t = c->tc;
    const TensorList& tl = st.tl;
    const int E = c->width[0], V = c->cfg.vocab, L = c->cfg.layers;
    const bool adam = st.kind == UpdateStep::kAdam;
    ZRB_TRY(tc_flush_updates(c, s));   // (a second update without a forward in between)
    ProfScope ps(c, st.kind == UpdateStep::kSwap ? ZRB_PROF_PACK : ZRB_PROF_CLIP_SGD, s);
    TensorList rest = tc_without_matrices(c, tl);   // what the list kernel updates
    bool lazy = false;
    if (st.train()) {
        // rows_only: only the embedding rows of the last window can be non-zero -> norm and update over those rows
        const bool rows_only = !c->tied && c->emb_sparse && c->emb_prev_grad == tl.g[0] && c->emb_prev_n > 0;
        // gemm_norm: the matrices' sums of squares are in the wgrad epilogue slots: no read of their gradients
        const bool gemm_norm = t->wg_ok && t->wg_key == tl.g[tc_matrices(c).fc_w().i];
        if (rows_only && !adam) rest.n[0] = 0;
        TensorList dense = gemm_norm ? rest : tl;   // what the norm reads
        if (rows_only) dense.n[0] = 0;
        if (c->tied && gemm_norm) {
            // E's slots describe G_proj; the extra slots hold the merge's correction to dE (tc_backward_layer)
            ZRB_TRY(grad_norm(dense, max_norm, c->partials, c->scalars, norm_out, s, true, t->wg_slots));
        } else if (rows_only) {
            ZRB_TRY(embed_first_table(c->emb_prev_ids, c->emb_first, c->emb_prev_n, V, s));
            ZRB_TRY(embed_rows_sumsq(tl.g[0], c->emb_prev_ids, c->emb_first, c->emb_prev_n, E, V,
                                     c->partials + norm_partials_base(), kNormExtra, s));   // one token per block
            ZRB_TRY(grad_norm(dense, max_norm, c->partials, c->scalars, norm_out, s, true, gemm_norm ? t->wg_slots : 0));
            if (!adam)
                ZRB_TRY(embed_rows_update(tl.p[0], tl.g[0], c->emb_prev_ids, c->emb_first, c->emb_prev_n, E, V, st.lr,
                                          c->scalars, c->keep_clipped, s));
            if (st.kind == UpdateStep::kSgdAvg) {   // the average is dense: every row moves toward the new embedding
                TensorList e{};
                e.p[0] = tl.p[0]; e.n[0] = tl.n[0]; e.count = 1;
                ZRB_TRY(avg_apply(e, st.avg.a, st.avg.mu, st.avg.first, s));
            }
        } else {
            ZRB_TRY(grad_norm(tl, max_norm, c->partials, c->scalars, norm_out, s));
        }
        // lazy update: layer 0 (needed by the very next kernels) now; layers >= 1 and fc.W beside the forward
        // recurrences of the next step (tc_forward), or at the next call that is not a fused train step
        // (tc_flush_updates)
        lazy = c->lazy_update && t->persistent() && pdl_beside_rec(c);
        if (lazy) t->upd = st;
    }
    for (const WeightMatrix& m : tc_matrices(c)) {
        // a tied E under Adam is never deferred: the next forward's gather through a pending update (tc_forward) knows
        // only the SGD rule
        if (lazy && m.item >= 1 && !(adam && c->tied && m.item == L)) t->upd_pending |= 1u << m.item;
        else ZRB_TRY(tc_update_matrix(c, m, st, 0, s));
    }
    ZRB_TRY(update_list(c, st, rest, s));
    tc_images_current(c, p);
    return ZRB_OK;
}

}  // namespace zrb
