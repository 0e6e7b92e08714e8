// C ABI of libzaremba_b200.so: context, orchestration of the forward / backward / loss /
// update kernels.  See include/zaremba_b200.h for the contract of every entry point.
#include <math.h>
#include <cmath>
#include <stdarg.h>
#include <string.h>

#include <string>
#include <vector>

#include "engine.h"

namespace zrb {

static thread_local char t_err[1024] = "";
std::atomic<int64_t> g_launches{0};
std::atomic<int> g_live_tc_ctx[64];

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(t_err, sizeof(t_err), fmt, ap);
    va_end(ap);
}

static int dev_alloc(zrb_ctx* c, void** p, size_t bytes) {
    *p = nullptr;
    if (bytes == 0) bytes = 16;
    cudaError_t e = cudaMalloc(p, bytes);
    if (e != cudaSuccess) {
        set_error("cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
        return ZRB_E_NOMEM;
    }
    c->allocs.push_back(*p);
    c->bytes += (int64_t)bytes;
    return ZRB_OK;
}
template <typename T>
static int dalloc(zrb_ctx* c, T** p, size_t count) {
    return dev_alloc(c, (void**)p, count * sizeof(T));
}

// A persistent recurrence kernel that ran out of patience (lost wake-up, grid not co-resident) finished with garbage and
// left a code in the mapped host word: every later call on this context fails -- the CUDA context is intact, a new zrb
// context works.  Costs one host load.
static const char* const kWaitNames[] = {"?", "weight slice", "operand image", "accumulators", "partner rows", "grid barrier"};
static int watchdog_check(const zrb_ctx* c) {
    if (!c->wd_host) return ZRB_OK;
    const unsigned int code = *(volatile const unsigned int*)c->wd_host;
    if (code == 0) return ZRB_OK;
    const unsigned int kind = code & 0xFF;
    set_error("a persistent recurrence kernel gave up waiting for its %s (CTA %u, step %u): results since then are invalid and "
              "this context is unusable; the CUDA context is intact",
              kind < sizeof(kWaitNames) / sizeof(kWaitNames[0]) ? kWaitNames[kind] : "?", (code >> 8) & 0xFFF, code >> 20);
    return ZRB_E_CUDA;
}

static int check_shapes(const zrb_ctx* c, int T, int B) {
    ZRB_TRY(watchdog_check(c));
    ZRB_REQUIRE(T >= 1 && T <= c->cfg.max_seq, "T=%d outside [1,%d]", T, c->cfg.max_seq);
    ZRB_REQUIRE(B >= 1 && B <= c->cfg.max_batch, "B=%d outside [1,%d]", B, c->cfg.max_batch);
    return ZRB_OK;
}

// a tied context takes E once: fc_w must be embed_w in parameters and gradients alike
static int check_tied(const zrb_ctx* c, const zrb_params* p) {
    ZRB_REQUIRE(!c->tied || !p || p->fc_w == p->embed_w, "tied context: fc_w (%p) must equal embed_w (%p)",
                (void*)p->fc_w, (void*)p->embed_w);
    return ZRB_OK;
}

MaskSrc site_mask(const zrb_ctx* c, int site) {
    const uint8_t* ex = c->explicit_masks_set ? c->explicit_masks[site] : nullptr;
    MaskSrc m = make_mask_src(ex, c->seed, c->step, site, c->cfg.dropout, c->train);
    if (c->variational) m.period = (uint32_t)c->B * (uint32_t)c->width[site];   // element (t, b, j) reads b*W + j
    return m;
}

MaskSrc rec_mask(const zrb_ctx* c, int layer) {
    return make_mask_src(nullptr, c->seed, c->step, c->cfg.layers + 1 + layer, c->p_rec, c->train && c->variational);
}

MaskSrc wd_mask(const zrb_ctx* c, int layer) {
    return make_mask_src(nullptr, c->wd_seed, c->step, 2 * c->cfg.layers + 1 + layer, c->p_wd, c->train);
}

bool reg_on(const zrb_ctx* c) { return c->ar_alpha > 0.f || c->tar_beta > 0.f; }

int reg_compute(zrb_ctx* c, cudaStream_t s) {
    const int L = c->cfg.layers;
    ZRB_TRY(activation_reg(c->hraw[L - 1], c->reg_r, c->reg_part, c->reg_val, c->T, c->B, c->width[L], site_mask(c, L),
                           c->ar_alpha, c->tar_beta, s));
    c->reg_use = true;
    return ZRB_OK;
}

MaskSrc ed_mask(const zrb_ctx* c) {
    return make_mask_src(nullptr, c->ed_seed, c->step, 3 * c->cfg.layers + 1, c->p_ed, c->train);
}

MaskSrc mos_mask(const zrb_ctx* c) {
    MaskSrc m = make_mask_src(nullptr, c->seed, c->step, 3 * c->cfg.layers + 2, c->p_mos, c->train);
    if (c->variational) m.period = (uint32_t)c->B * (uint32_t)(c->experts * c->width[0]);   // element (t, b, j): b*K*E + j
    return m;
}

// the tensors of param_list(): 3 + 4L, and the head's three with experts
static int tensor_count(const zrb_ctx* c) { return 4 * c->cfg.layers + 3 + (c->experts ? 3 : 0); }

// ZRB_E_INVALID for an entry point a Mixture-of-Softmaxes context does not support yet
static int refuse_experts(const zrb_ctx* c, const char* what) {
    ZRB_REQUIRE(!c->experts, "%s does not support a Mixture-of-Softmaxes context (experts = %d)", what, c->experts);
    return ZRB_OK;
}

static cudaEvent_t prof_event(zrb_ctx* c) {
    if (!c->prof_pool.empty()) {
        cudaEvent_t e = c->prof_pool.back();
        c->prof_pool.pop_back();
        return e;
    }
    cudaEvent_t e = nullptr;
    cudaEventCreate(&e);
    return e;
}

ProfScope::ProfScope(zrb_ctx* ctx, int cls, cudaStream_t stream) : c(ctx), s(stream) {
    if (!c->prof_on) return;
    cudaEvent_t a = prof_event(c);
    b = prof_event(c);
    cudaEventRecord(a, s);
    c->prof_recs.push_back({cls, a, b});
}
ProfScope::~ProfScope() {
    if (b) cudaEventRecord(b, s);
}

int update_list(const zrb_ctx* c, const UpdateStep& st, const TensorList& tl, cudaStream_t s) {
    switch (st.kind) {
        case UpdateStep::kSgd: return sgd_apply(tl, st.lr, c->scalars, c->keep_clipped, s);
        case UpdateStep::kSgdAvg:
            return sgd_avg_apply(tl, st.avg.a, st.lr, c->scalars, c->keep_clipped, st.avg.mu, st.avg.first, s);
        case UpdateStep::kAdam: return adam_apply(tl, st.adam, c->scalars, c->keep_clipped, s);
        case UpdateStep::kDyn: return dyneval_apply(tl, st.tg, st.r, st.dyn, s);
        case UpdateStep::kSwap: return swap_apply(tl, st.avg.a, s);
    }
    return ZRB_E_INVALID;
}

}  // namespace zrb

using namespace zrb;

extern "C" {

const char* zrb_last_error(void) { return t_err; }
const char* zrb_version(void) { return "zaremba_b200 0.1 (sm_90a)"; }
int64_t zrb_launch_count(void) { return g_launches.load(); }

// zrb_ctx_create, zrb_ctx_create_widths and zrb_ctx_create_mos: widths[0] = E, widths[1 + l] = H_l (already checked)
static int ctx_create(const zrb_config* cfg, const int* widths, zrb_ctx** out, int experts = 0) {
    ZRB_REQUIRE(cfg->max_seq > 0 && cfg->max_batch > 0, "bad window T=%d B=%d", cfg->max_seq, cfg->max_batch);
    ZRB_REQUIRE(cfg->dropout >= 0.f && cfg->dropout < 1.f, "dropout %f outside [0,1)", cfg->dropout);
    ZRB_REQUIRE(cfg->engine == ZRB_ENGINE_SIMT || cfg->engine == ZRB_ENGINE_TC, "unknown engine %d", cfg->engine);
    ZRB_REQUIRE((cfg->flags & ~ZRB_TIED_EMBEDDING) == 0, "unknown config flags 0x%x", (unsigned)cfg->flags);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        set_error("no CUDA device: libzaremba_b200 has no CPU path");
        return ZRB_E_CUDA;
    }
    zrb_ctx* c = new zrb_ctx();
    c->cfg = *cfg;
    c->tied = (cfg->flags & ZRB_TIED_EMBEDDING) != 0;
    c->experts = experts;
    const int L = cfg->layers, V = cfg->vocab;
    bool equal = true;
    for (int s = 0; s <= L; ++s) {
        c->width[s] = widths[s];
        equal = equal && widths[s] == widths[0];
        if (widths[s] > c->max_width) c->max_width = widths[s];
    }
    c->cfg.hidden = equal ? widths[0] : 0;
    const int Hm = c->max_width;
    const size_t N = (size_t)cfg->max_seq * cfg->max_batch, B = cfg->max_batch;
    int rc = ZRB_OK;
    for (int l = 0; l <= L && rc == ZRB_OK; ++l) rc = dalloc(c, &c->act[l], N * c->width[l]);
    for (int l = 0; l < L && rc == ZRB_OK; ++l) {
        const size_t H = c->width[l + 1];
        rc = dalloc(c, &c->gates[l], N * 4 * H);
        if (rc == ZRB_OK) rc = dalloc(c, &c->cst[l], N * H);
        if (rc == ZRB_OK) rc = dalloc(c, &c->hraw[l], N * H);
        if (rc == ZRB_OK) rc = dalloc(c, &c->h0s[l], B * H);
        if (rc == ZRB_OK) rc = dalloc(c, &c->c0s[l], B * H);
    }
    if (rc == ZRB_OK) rc = dalloc(c, &c->dy, N * Hm);
    if (rc == ZRB_OK) rc = dalloc(c, &c->dx, N * Hm);
    if (rc == ZRB_OK) rc = dalloc(c, &c->dG, N * 4 * Hm);
    if (rc == ZRB_OK) rc = dalloc(c, &c->dh_rec, B * Hm);
    if (rc == ZRB_OK) rc = dalloc(c, &c->dc, B * Hm);
    if (rc == ZRB_OK) rc = dalloc(c, &c->row_loss, N);
    if (rc == ZRB_OK) rc = dalloc(c, &c->partials, 4096 + kNormGemm);
    if (rc == ZRB_OK) rc = dalloc(c, &c->scalars, 16);
    if (rc == ZRB_OK) rc = dalloc(c, &c->x_saved, N);
    if (rc == ZRB_OK) rc = dalloc(c, &c->emb_prev_ids, N);
    if (rc == ZRB_OK) c->emb_prev_cap = (int64_t)N;
    if (rc == ZRB_OK) rc = dalloc(c, &c->wd_flag, 1);
    if (rc == ZRB_OK && cudaMemset(c->wd_flag, 0, sizeof(unsigned int)) != cudaSuccess) rc = ZRB_E_CUDA;
    if (rc == ZRB_OK) {
        void* hp = nullptr;
        if (cudaHostAlloc(&hp, sizeof(unsigned int), cudaHostAllocMapped) != cudaSuccess) {
            set_error("cudaHostAlloc of the watchdog word failed");
            rc = ZRB_E_CUDA;
        } else {
            c->wd_host = (unsigned int*)hp;   // (unified addressing: the same pointer is valid on the device)
            *c->wd_host = 0;
        }
    }
    if (rc == ZRB_OK) rc = dalloc(c, &c->emb_first, (size_t)V);
    if (rc == ZRB_OK && c->tied) {   // fixed-point sums of the embedding rows, every backward
        rc = dalloc(c, &c->emb_acc, N * c->width[0]);
        c->emb_cap_rows = (int64_t)N;
    }
    if (rc == ZRB_OK) rc = dalloc(c, &c->y_dev, N);
    if (rc == ZRB_OK) rc = dalloc(c, &c->x_dev, N);
    if (rc == ZRB_OK) rc = dalloc(c, &c->scores, N * V);
    if (rc == ZRB_OK) rc = dalloc(c, &c->dscores, N * V);
    if (rc == ZRB_OK && cfg->engine == ZRB_ENGINE_TC) rc = tc_ctx_init(c);
    if (rc != ZRB_OK) {
        zrb_ctx_destroy(c);
        return rc;
    }
    *out = c;
    return ZRB_OK;
}

int zrb_ctx_create(const zrb_config* cfg, zrb_ctx** out) {
    ZRB_REQUIRE(cfg && out, "null argument");
    ZRB_REQUIRE(cfg->vocab > 0 && cfg->hidden > 0 && cfg->layers > 0 && cfg->layers <= ZRB_MAX_LAYERS,
                "bad model shape V=%d H=%d L=%d", cfg->vocab, cfg->hidden, cfg->layers);
    int widths[ZRB_MAX_LAYERS + 1];
    for (int s = 0; s <= cfg->layers; ++s) widths[s] = cfg->hidden;
    return ctx_create(cfg, widths, out);
}

int zrb_ctx_create_widths(const zrb_config* cfg, const int32_t* widths, zrb_ctx** out) {
    ZRB_REQUIRE(cfg && widths && out, "null argument");
    ZRB_REQUIRE(cfg->vocab > 0 && cfg->layers > 0 && cfg->layers <= ZRB_MAX_LAYERS, "bad model shape V=%d L=%d",
                cfg->vocab, cfg->layers);
    ZRB_REQUIRE(cfg->hidden == 0, "cfg->hidden must be 0 when the widths are given (got %d)", cfg->hidden);
    const int L = cfg->layers;
    bool equal = true;
    for (int s = 0; s <= L; ++s) {
        ZRB_REQUIRE(widths[s] > 0, "width %d of site %d must be >= 1", widths[s], s);
        equal = equal && widths[s] == widths[0];
    }
    ZRB_REQUIRE(!(cfg->flags & ZRB_TIED_EMBEDDING) || widths[0] == widths[L],
                "a tied context needs E = H_{L-1} (E = %d, H_{L-1} = %d)", widths[0], widths[L]);
    ZRB_REQUIRE(equal || cfg->engine != ZRB_ENGINE_SIMT, "the validation engine takes one width only");
    int w[ZRB_MAX_LAYERS + 1];
    for (int s = 0; s <= L; ++s) w[s] = widths[s];
    return ctx_create(cfg, w, out);
}

int zrb_ctx_create_mos(const zrb_config* cfg, const int32_t* widths, int32_t experts, zrb_ctx** out) {
    ZRB_REQUIRE(cfg && out, "null argument");
    ZRB_REQUIRE(experts >= 1 && experts <= ZRB_MAX_EXPERTS, "experts=%d outside [1, %d]", experts, ZRB_MAX_EXPERTS);
    ZRB_REQUIRE(cfg->engine == ZRB_ENGINE_TC, "a Mixture-of-Softmaxes context needs the tensor-core engine");
    ZRB_REQUIRE(cfg->vocab > 0 && cfg->layers > 0 && 4 * cfg->layers + 6 <= kMaxTensors,
                "bad model shape V=%d L=%d (a Mixture-of-Softmaxes context takes at most 3 layers)", cfg->vocab,
                cfg->layers);
    const int L = cfg->layers;
    int w[ZRB_MAX_LAYERS + 1];
    if (widths) {
        ZRB_REQUIRE(cfg->hidden == 0, "cfg->hidden must be 0 when the widths are given (got %d)", cfg->hidden);
        for (int s = 0; s <= L; ++s) {
            ZRB_REQUIRE(widths[s] > 0, "width %d of site %d must be >= 1", widths[s], s);
            w[s] = widths[s];
        }
    } else {
        ZRB_REQUIRE(cfg->hidden > 0, "bad model shape H=%d", cfg->hidden);
        for (int s = 0; s <= L; ++s) w[s] = cfg->hidden;
    }
    return ctx_create(cfg, w, out, experts);
}

int zrb_set_mos_dropout(zrb_ctx* c, float p) {
    ZRB_REQUIRE(c, "null ctx");
    ZRB_REQUIRE(c->experts > 0, "latent dropout needs a Mixture-of-Softmaxes context");
    ZRB_REQUIRE(isfinite(p) && p >= 0.f && p < 1.f, "latent-dropout p %f outside [0,1)", p);
    if (p != c->p_mos) {
        c->have_fwd = false;        // a backward must not regenerate another mask than its forward used
        c->bwd_next_layer = -1;
    }
    c->p_mos = p;
    return ZRB_OK;
}

int zrb_set_zoneout(zrb_ctx* c, float z_c, float z_h) {
    ZRB_REQUIRE(c, "null ctx");
    ZRB_REQUIRE(isfinite(z_c) && z_c >= 0.f && z_c < 1.f, "zoneout z_c %f outside [0,1)", z_c);
    ZRB_REQUIRE(isfinite(z_h) && z_h >= 0.f && z_h < 1.f, "zoneout z_h %f outside [0,1)", z_h);
    ZRB_REQUIRE(c->cfg.engine == ZRB_ENGINE_TC, "zoneout needs the tensor-core engine");
    if ((z_c > 0.f || z_h > 0.f) && !c->ctil[0]) {
        const size_t N = (size_t)c->cfg.max_seq * c->cfg.max_batch;
        for (int l = 0; l < c->cfg.layers; ++l) {
            ZRB_TRY(dalloc(c, &c->ctil[l], N * c->width[l + 1]));
            ZRB_TRY(dalloc(c, &c->zflags[l], N * c->width[l + 1]));
        }
        ZRB_TRY(dalloc(c, &c->zhcarry, (size_t)c->cfg.max_batch * c->max_width));
    }
    if (z_c != c->z_c || z_h != c->z_h) {
        c->have_fwd = false;        // a backward must not apply another rule than its forward used
        c->bwd_next_layer = -1;
    }
    c->z_c = z_c;
    c->z_h = z_h;
    return ZRB_OK;
}

void zrb_ctx_destroy(zrb_ctx* c) {
    if (!c) return;
    tc_ctx_free(c);
    for (auto& r : c->prof_recs) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
    for (cudaEvent_t e : c->prof_pool) cudaEventDestroy(e);
    for (void* p : c->allocs) cudaFree(p);
    if (c->wd_host) cudaFreeHost(c->wd_host);
    delete c;
}

int64_t zrb_ctx_workspace_bytes(const zrb_ctx* c) { return c ? c->bytes : 0; }

int zrb_params_changed(zrb_ctx* c) {
    ZRB_REQUIRE(c, "null ctx");
    c->weights_version++;
    return ZRB_OK;
}

int zrb_set_lazy_update(zrb_ctx* c, int32_t on) {
    ZRB_REQUIRE(c, "null ctx");
    c->lazy_update = on != 0;
    return ZRB_OK;
}

int zrb_check_health(zrb_ctx* c) {
    ZRB_REQUIRE(c, "null ctx");
    return watchdog_check(c);
}

int zrb_flush_updates(zrb_ctx* c, void* stream) {
    ZRB_REQUIRE(c, "null ctx");
    ZRB_TRY(watchdog_check(c));
    if (c->cfg.engine != ZRB_ENGINE_TC) return ZRB_OK;
    return tc_flush_updates(c, (cudaStream_t)stream);
}

int zrb_dropout_mask(uint64_t seed, uint64_t step, int32_t site, int64_t n, float p, uint8_t* mask_out,
                     void* stream) {
    ZRB_REQUIRE(mask_out && n >= 0, "bad args");
    MaskSrc m = make_mask_src(nullptr, seed, step, site, p, 1);
    return dropout_mask_bytes(m, n, mask_out, (cudaStream_t)stream);
}

int zrb_set_explicit_masks(zrb_ctx* c, const uint8_t* const* site_masks) {
    ZRB_REQUIRE(c, "null ctx");
    if (site_masks && c->variational) {
        set_error("explicit masks replay Zaremba's per-step masks: switch the variational mode off first");
        return ZRB_E_STATE;
    }
    c->explicit_masks_set = site_masks != nullptr;
    for (int s = 0; s <= c->cfg.layers; ++s) c->explicit_masks[s] = site_masks ? site_masks[s] : nullptr;
    return ZRB_OK;
}

int zrb_set_variational_dropout(zrb_ctx* c, int32_t on, float p_rec) {
    ZRB_REQUIRE(c, "null ctx");
    ZRB_REQUIRE(on == 0 || on == 1, "on must be 0 or 1 (got %d)", on);
    ZRB_REQUIRE(p_rec >= 0.f && p_rec < 1.f, "p_rec %f outside [0,1)", p_rec);
    ZRB_REQUIRE(on || p_rec == 0.f, "p_rec %f needs the variational mode", p_rec);
    if (c->explicit_masks_set) {
        set_error("explicit masks are set: the variational mode cannot replay them");
        return ZRB_E_STATE;
    }
    if (on && c->cfg.engine == ZRB_ENGINE_SIMT && !c->hrec[0]) {
        const size_t n = (size_t)(c->cfg.max_seq + 1) * c->cfg.max_batch * c->cfg.hidden;
        for (int l = 0; l < c->cfg.layers; ++l) ZRB_TRY(dalloc(c, &c->hrec[l], n));
    }
    if ((bool)on != c->variational || p_rec != c->p_rec) {
        c->have_fwd = false;        // a backward must not regenerate other masks than its forward used
        c->bwd_next_layer = -1;
    }
    c->variational = on != 0;
    c->p_rec = p_rec;
    return ZRB_OK;
}

int zrb_set_weight_drop(zrb_ctx* c, float p, uint64_t seed) {
    ZRB_REQUIRE(c, "null ctx");
    ZRB_REQUIRE(isfinite(p) && p >= 0.f && p < 1.f, "weight-drop p %f outside [0,1)", p);
    if (p > 0.f && c->cfg.engine == ZRB_ENGINE_SIMT && !c->whh_wd[0]) {
        const size_t n = (size_t)4 * c->cfg.hidden * c->cfg.hidden;
        for (int l = 0; l < c->cfg.layers; ++l) ZRB_TRY(dalloc(c, &c->whh_wd[l], n));
    }
    if (p != c->p_wd || seed != c->wd_seed) {
        c->have_fwd = false;        // a backward must not regenerate another mask than its forward used
        c->bwd_next_layer = -1;
    }
    c->p_wd = p;
    c->wd_seed = seed;
    return ZRB_OK;
}

int zrb_set_embed_dropout(zrb_ctx* c, float p, uint64_t seed) {
    ZRB_REQUIRE(c, "null ctx");
    ZRB_REQUIRE(isfinite(p) && p >= 0.f && p < 1.f, "embedding-dropout p %f outside [0,1)", p);
    if (p != c->p_ed || seed != c->ed_seed) {
        c->have_fwd = false;        // a backward must not regenerate another mask than its forward used
        c->bwd_next_layer = -1;
    }
    c->p_ed = p;
    c->ed_seed = seed;
    return ZRB_OK;
}

int zrb_set_activation_reg(zrb_ctx* c, float alpha, float beta) {
    ZRB_REQUIRE(c, "null ctx");
    ZRB_REQUIRE(isfinite(alpha) && alpha >= 0.f, "AR alpha %f must be finite and >= 0", alpha);
    ZRB_REQUIRE(isfinite(beta) && beta >= 0.f, "TAR beta %f must be finite and >= 0", beta);
    if ((alpha > 0.f || beta > 0.f) && !c->reg_r) {
        ZRB_TRY(dalloc(c, &c->reg_r, (size_t)c->cfg.max_seq * c->cfg.max_batch * c->width[c->cfg.layers]));
        ZRB_TRY(dalloc(c, &c->reg_part, (size_t)2 * kActRegBlocks));
        ZRB_TRY(dalloc(c, &c->reg_val, 2));
        ZRB_CUDA(cudaMemset(c->reg_val, 0, 2 * sizeof(float)));
    }
    if (alpha != c->ar_alpha || beta != c->tar_beta) {
        c->have_fwd = false;        // a phased backward must not add another step's penalty gradient
        c->bwd_next_layer = -1;
    }
    c->ar_alpha = alpha;
    c->tar_beta = beta;
    return ZRB_OK;
}

int zrb_activation_reg(zrb_ctx* c, float* out2, void* stream) {
    ZRB_REQUIRE(c && out2, "null argument");
    cudaStream_t s = (cudaStream_t)stream;
    if (!c->reg_val) {
        ZRB_CUDA(cudaMemsetAsync(out2, 0, 2 * sizeof(float), s));
        return ZRB_OK;
    }
    ZRB_CUDA(cudaMemcpyAsync(out2, c->reg_val, 2 * sizeof(float), cudaMemcpyDeviceToDevice, s));
    return ZRB_OK;
}

int zrb_forward(zrb_ctx* c, const zrb_params* p, const int64_t* x, int32_t T, int32_t B, const zrb_states* in,
                const zrb_states* out, float* scores, int32_t train, uint64_t seed, uint64_t step, void* stream) {
    ZRB_REQUIRE(c && p && x && in && out, "null argument");
    ZRB_TRY(check_shapes(c, T, B));
    ZRB_TRY(check_tied(c, p));
    cudaStream_t s = (cudaStream_t)stream;
    c->T = T; c->B = B; c->train = train ? 1 : 0; c->seed = seed; c->step = step;
    c->have_fwd = false;
    c->reg_use = false;   // AR / TAR belongs to the fused train steps (DESIGN.md section 17)
    if (c->cfg.engine == ZRB_ENGINE_TC)
        ZRB_TRY(tc_forward(c, p, x, in, out, scores, s));
    else
        ZRB_TRY(simt_forward(c, p, x, in, out, scores, s));
    c->have_fwd = true;
    return ZRB_OK;
}

int zrb_backward(zrb_ctx* c, const zrb_params* p, const float* dscores, const zrb_params* g, void* stream) {
    ZRB_REQUIRE(c && p && dscores && g, "null argument");
    ZRB_TRY(check_tied(c, p));
    ZRB_TRY(check_tied(c, g));
    if (!c->have_fwd) {
        set_error("zrb_backward without a preceding zrb_forward");
        return ZRB_E_STATE;
    }
    cudaStream_t s = (cudaStream_t)stream;
    if (c->cfg.engine == ZRB_ENGINE_TC) return tc_backward(c, p, dscores, g, s);
    return simt_backward(c, p, dscores, g, s);
}

int zrb_softmax_nll(zrb_ctx* c, const float* scores, const int64_t* y, int32_t T, int32_t B, float* loss,
                    float* dscores, float* tgt_prob, void* stream) {
    ZRB_REQUIRE(c && scores && y, "null argument");
    ZRB_TRY(check_shapes(c, T, B));
    return softmax_nll(scores, y, T * B, c->cfg.vocab, B, c->row_loss, loss, dscores, tgt_prob,
                       (cudaStream_t)stream);
}

int zrb_clip_sgd(zrb_ctx* c, int32_t n, float* const* params, float* const* grads, const int64_t* sizes, float lr,
                 float max_norm, float* norm_out, void* stream) {
    ZRB_REQUIRE(c && params && grads && sizes, "null argument");
    ZRB_REQUIRE(n >= 0 && n <= 16, "at most 16 tensors per call (got %d)", n);
    if (c->cfg.engine == ZRB_ENGINE_TC) ZRB_TRY(tc_flush_updates(c, (cudaStream_t)stream));
    TensorList tl;
    tl.count = n;
    for (int i = 0; i < n; ++i) {
        tl.p[i] = params[i]; tl.g[i] = grads[i]; tl.n[i] = sizes[i];
    }
    ZRB_TRY(clip_sgd(tl, lr, max_norm, c->partials, c->scalars, norm_out, true, (cudaStream_t)stream));
    c->weights_version++;
    return ZRB_OK;
}

static TensorList param_list(const zrb_ctx* c, const zrb_params* p, const zrb_params* g);

// ---- iterate averaging (DESIGN.md section 16) -----------------------------------------------------------------------
static bool ranges_overlap(const float* a, int64_t na, const float* b, int64_t nb) {
    if (na == 0 || nb == 0) return false;
    const uintptr_t a0 = (uintptr_t)a, a1 = a0 + (uintptr_t)na * sizeof(float);
    const uintptr_t b0 = (uintptr_t)b, b1 = b0 + (uintptr_t)nb * sizeof(float);
    return a0 < b1 && b0 < a1;
}

// ZRB_E_INVALID when an average tensor overlaps a tensor of `tl` (its p, and its g when with_g)
static int check_avg_alias(const TensorList& ta, const TensorList& tl, bool with_g) {
    for (int i = 0; i < ta.count; ++i)
        for (int j = 0; j < tl.count; ++j) {
            const bool hit = ranges_overlap(ta.p[i], ta.n[i], tl.p[j], tl.n[j]) ||
                             (with_g && ranges_overlap(ta.p[i], ta.n[i], tl.g[j], tl.n[j]));
            ZRB_REQUIRE(!hit, "average tensor %d overlaps %s tensor %d", i, with_g ? "a parameter or gradient" : "parameter",
                        j);
        }
    return ZRB_OK;
}

// ZRB_E_INVALID when a moment tensor (tm.p) overlaps a parameter or gradient of `tl`
static int check_moment_alias(const TensorList& tm, const TensorList& tl) {
    for (int i = 0; i < tm.count; ++i)
        for (int j = 0; j < tl.count; ++j)
            ZRB_REQUIRE(!ranges_overlap(tm.p[i], tm.n[i], tl.p[j], tl.n[j]) &&
                            !ranges_overlap(tm.p[i], tm.n[i], tl.g[j], tl.n[j]),
                        "moment tensor %d overlaps a parameter or gradient tensor %d", i, j);
    return ZRB_OK;
}

// ZRB_E_INVALID when a tensor of `tl` (its p or g) is not 4-byte aligned: the update kernels stream them as floats
static int check_aligned(const TensorList& tl, const char* what) {
    for (int i = 0; i < tl.count; ++i)
        ZRB_REQUIRE((((uintptr_t)tl.p[i] | (uintptr_t)tl.g[i]) & 3) == 0, "%s tensor %d is not 4-byte aligned", what, i);
    return ZRB_OK;
}

static int check_not_swapped(const zrb_ctx* c) {
    ZRB_REQUIRE(!c->avg_swapped, "the parameters hold the average (zrb_swap_average): swap back before training");
    return ZRB_OK;
}

int zrb_set_average(zrb_ctx* c, const zrb_params* avg) {
    ZRB_REQUIRE(c, "null ctx");
    ZRB_REQUIRE(!c->avg_swapped, "the parameters hold the average (zrb_swap_average): swap back first");
    ZRB_REQUIRE(!avg || !c->adam_on, "iterate averaging is an SGD scheme: switch Adam off (zrb_set_adam) first");
    if (avg) {
        ZRB_REQUIRE(avg->embed_w && avg->fc_w && avg->fc_b, "null average tensor");
        ZRB_REQUIRE(!c->experts || (mos_of(avg)->prior_w && mos_of(avg)->latent_w && mos_of(avg)->latent_b),
                    "null average tensor of the Mixture-of-Softmaxes head");
        for (int l = 0; l < c->cfg.layers; ++l)
            ZRB_REQUIRE(avg->w_ih[l] && avg->w_hh[l] && avg->b_ih[l] && avg->b_hh[l], "null average tensor of layer %d", l);
        ZRB_TRY(check_tied(c, avg));
        const TensorList ta = param_list(c, avg, avg);
        for (int i = 0; i < ta.count; ++i)
            for (int j = i + 1; j < ta.count; ++j)
                ZRB_REQUIRE(!ranges_overlap(ta.p[i], ta.n[i], ta.p[j], ta.n[j]), "average tensors %d and %d overlap", i, j);
        ZRB_TRY(check_aligned(ta, "average"));
    }
    // deferred updates belong to the steps before: they average (or not) with the n they were issued with
    if (c->cfg.engine == ZRB_ENGINE_TC) ZRB_TRY(tc_flush_updates(c, nullptr));
    c->avg_on = avg != nullptr;
    if (avg) memcpy(&c->avg, avg, c->experts ? sizeof(zrb_mos_params) : sizeof(zrb_params));
    c->avg_n = 0;
    return ZRB_OK;
}

// ---- Adam (DESIGN.md section 21) -------------------------------------------------------------------------------------
// every tensor of a zrb_params (with the head's in a context with experts) is non-null
static int check_complete(const zrb_ctx* c, const zrb_params* p, const char* what) {
    ZRB_REQUIRE(p->embed_w && p->fc_w && p->fc_b, "null %s tensor", what);
    ZRB_REQUIRE(!c->experts || (mos_of(p)->prior_w && mos_of(p)->latent_w && mos_of(p)->latent_b),
                "null %s tensor of the Mixture-of-Softmaxes head", what);
    for (int l = 0; l < c->cfg.layers; ++l)
        ZRB_REQUIRE(p->w_ih[l] && p->w_hh[l] && p->b_ih[l] && p->b_hh[l], "null %s tensor of layer %d", what, l);
    return ZRB_OK;
}

int zrb_set_adam(zrb_ctx* c, const zrb_params* m, const zrb_params* v, float beta1, float beta2, float eps,
                 int64_t step) {
    ZRB_REQUIRE(c, "null ctx");
    ZRB_REQUIRE(!c->avg_swapped, "the parameters hold the average (zrb_swap_average): swap back first");
    ZRB_REQUIRE(!m == !v, "give both moment tensors m and v, or neither");
    if (m) {
        ZRB_REQUIRE(!c->avg_on, "iterate averaging is an SGD scheme: stop it (zrb_set_average(ctx, NULL)) first");
        ZRB_REQUIRE(std::isfinite(beta1) && beta1 >= 0.f && beta1 < 1.f, "beta1 = %g outside [0, 1)", (double)beta1);
        ZRB_REQUIRE(std::isfinite(beta2) && beta2 >= 0.f && beta2 < 1.f, "beta2 = %g outside [0, 1)", (double)beta2);
        ZRB_REQUIRE(std::isfinite(eps) && eps > 0.f, "eps = %g must be finite and > 0", (double)eps);
        ZRB_REQUIRE(step >= 0, "step = %lld must be >= 0", (long long)step);
        ZRB_TRY(check_complete(c, m, "first-moment"));
        ZRB_TRY(check_complete(c, v, "second-moment"));
        ZRB_TRY(check_tied(c, m));
        ZRB_TRY(check_tied(c, v));
        const TensorList tm = param_list(c, m, v);   // p: the first moments, g: the second
        for (int i = 0; i < tm.count; ++i)
            for (int j = 0; j < tm.count; ++j) {
                ZRB_REQUIRE(j <= i || !ranges_overlap(tm.p[i], tm.n[i], tm.p[j], tm.n[j]),
                            "first-moment tensors %d and %d overlap", i, j);
                ZRB_REQUIRE(j <= i || !ranges_overlap(tm.g[i], tm.n[i], tm.g[j], tm.n[j]),
                            "second-moment tensors %d and %d overlap", i, j);
                ZRB_REQUIRE(!ranges_overlap(tm.p[i], tm.n[i], tm.g[j], tm.n[j]),
                            "first-moment tensor %d overlaps second-moment tensor %d", i, j);
            }
        ZRB_TRY(check_aligned(tm, "moment"));
    }
    // deferred updates belong to the steps before: they apply the rule (and the t) they were issued with
    if (c->cfg.engine == ZRB_ENGINE_TC) ZRB_TRY(tc_flush_updates(c, nullptr));
    c->adam_on = m != nullptr;
    if (m) {
        const size_t sz = c->experts ? sizeof(zrb_mos_params) : sizeof(zrb_params);
        memcpy(&c->adam_m, m, sz);
        memcpy(&c->adam_v, v, sz);
        c->adam_b1 = beta1; c->adam_b2 = beta2; c->adam_eps = eps;
        c->adam_t = step;
    }
    return ZRB_OK;
}

int zrb_average_count(const zrb_ctx* c, int64_t* n) {
    ZRB_REQUIRE(c && n, "null argument");
    *n = c->avg_on ? c->avg_n : 0;
    return ZRB_OK;
}

// st's update of p on either engine; on the validation engine the clip norm of a train-step kind, then the list
// kernels over every tensor.  max_norm / norm_out: the clip norm (unused by the other kinds)
static int apply_update(zrb_ctx* c, const zrb_params* p, const UpdateStep& st, float max_norm, float* norm_out,
                        cudaStream_t s) {
    if (c->cfg.engine == ZRB_ENGINE_TC) return tc_apply_update(c, p, st, max_norm, norm_out, s);
    ProfScope ps(c, st.kind == UpdateStep::kSwap ? ZRB_PROF_PACK : ZRB_PROF_CLIP_SGD, s);
    if (st.train()) ZRB_TRY(grad_norm(st.tl, max_norm, c->partials, c->scalars, norm_out, s));
    ZRB_TRY(update_list(c, st, st.tl, s));
    c->weights_version++;
    return ZRB_OK;
}

int zrb_swap_average(zrb_ctx* c, const zrb_params* p, void* stream) {
    ZRB_REQUIRE(c && p, "null argument");
    ZRB_TRY(watchdog_check(c));
    ZRB_TRY(check_tied(c, p));
    ZRB_REQUIRE(c->avg_on && c->avg_n > 0, "no average to swap in: no train step has been averaged since zrb_set_average");
    UpdateStep st;
    st.kind = UpdateStep::kSwap;
    st.tl = param_list(c, p, p);
    const TensorList ta = param_list(c, &c->avg.base, &c->avg.base);
    ZRB_TRY(check_avg_alias(ta, st.tl, false));
    for (int i = 0; i < ta.count; ++i) st.avg.a[i] = ta.p[i];
    ZRB_TRY(apply_update(c, p, st, 0.f, nullptr, (cudaStream_t)stream));
    c->avg_swapped = !c->avg_swapped;
    return ZRB_OK;
}

static TensorList param_list(const zrb_ctx* c, const zrb_params* p, const zrb_params* g) {
    TensorList tl;
    const int64_t V = c->cfg.vocab;
    int k = 0;
    tl.p[k] = p->embed_w; tl.g[k] = g->embed_w; tl.n[k++] = V * c->width[0];
    for (int l = 0; l < c->cfg.layers; ++l) {
        const int64_t In = c->width[l], H = c->width[l + 1];
        tl.p[k] = p->w_ih[l]; tl.g[k] = g->w_ih[l]; tl.n[k++] = 4 * H * In;
        tl.p[k] = p->w_hh[l]; tl.g[k] = g->w_hh[l]; tl.n[k++] = 4 * H * H;
        tl.p[k] = p->b_ih[l]; tl.g[k] = g->b_ih[l]; tl.n[k++] = 4 * H;
        tl.p[k] = p->b_hh[l]; tl.g[k] = g->b_hh[l]; tl.n[k++] = 4 * H;
    }
    const int64_t H = c->width[c->cfg.layers], E = c->width[0], K = c->experts;
    tl.p[k] = p->fc_w; tl.g[k] = g->fc_w; tl.n[k++] = V * (K ? E : H);
    if (c->tied) tl.n[0] = 0;   // E once, at fc.W's slot (zero-length entries are skipped by the norm and the update)
    tl.p[k] = p->fc_b; tl.g[k] = g->fc_b; tl.n[k++] = V;
    if (K) {   // the Mixture-of-Softmaxes head (zrb_mos_params)
        const zrb_mos_params *pm = mos_of(p), *gm = mos_of(g);
        tl.p[k] = pm->prior_w; tl.g[k] = gm->prior_w; tl.n[k++] = K * H;
        tl.p[k] = pm->latent_w; tl.g[k] = gm->latent_w; tl.n[k++] = K * E * H;
        tl.p[k] = pm->latent_b; tl.g[k] = gm->latent_b; tl.n[k++] = K * E;
    }
    tl.count = k;
    return tl;
}

int zrb_train_step_grads(zrb_ctx* c, const zrb_params* p, const zrb_params* g, const int64_t* x, const int64_t* y,
                         int32_t T, int32_t B, const zrb_states* in, const zrb_states* out, uint64_t seed,
                         uint64_t step, float* loss, void* stream) {
    ZRB_REQUIRE(c && p && g && x && y && in && out, "null argument");
    ZRB_REQUIRE(tensor_count(c) <= kMaxTensors, "fused step supports at most 3 layers");
    ZRB_TRY(check_not_swapped(c));
    cudaStream_t s = (cudaStream_t)stream;
    ZRB_TRY(check_shapes(c, T, B));
    ZRB_TRY(check_tied(c, p));
    ZRB_TRY(check_tied(c, g));
    if (c->cfg.engine == ZRB_ENGINE_TC) return tc_train_step_grads(c, p, g, x, y, T, B, in, out, seed, step, loss, s);
    ZRB_TRY(zrb_forward(c, p, x, T, B, in, out, c->scores, 1, seed, step, stream));
    {
        ProfScope ps(c, ZRB_PROF_SOFTMAX, s);
        ZRB_TRY(softmax_nll(c->scores, y, T * B, c->cfg.vocab, B, c->row_loss, loss, c->dscores, nullptr, s));
    }
    if (reg_on(c)) ZRB_TRY(reg_compute(c, s));
    ZRB_TRY(zrb_backward(c, p, c->dscores, g, stream));
    return ZRB_OK;
}

// Phased variant of zrb_train_step_grads for overlapping the data-parallel all-reduce with backward.
int zrb_train_step_begin(zrb_ctx* c, const zrb_params* p, const zrb_params* g, const int64_t* x, const int64_t* y,
                         int32_t T, int32_t B, const zrb_states* in, const zrb_states* out, uint64_t seed,
                         uint64_t step, float* loss, void* stream) {
    ZRB_REQUIRE(c && p && g && x && y && in && out, "null argument");
    ZRB_TRY(check_not_swapped(c));
    ZRB_TRY(check_shapes(c, T, B));
    ZRB_TRY(check_tied(c, p));
    ZRB_TRY(check_tied(c, g));
    if (c->cfg.engine == ZRB_ENGINE_TC)
        return tc_train_step_begin(c, p, g, x, y, T, B, in, out, seed, step, loss, (cudaStream_t)stream);
    ZRB_TRY(zrb_train_step_grads(c, p, g, x, y, T, B, in, out, seed, step, loss, stream));   // validation engine: all at once
    c->bwd_next_layer = c->cfg.layers - 1;
    return ZRB_OK;
}

int zrb_train_step_layer(zrb_ctx* c, const zrb_params* p, const zrb_params* g, int32_t layer, void* stream) {
    ZRB_REQUIRE(c && p && g, "null argument");
    ZRB_REQUIRE(layer >= 0 && layer < c->cfg.layers, "layer %d out of range", layer);
    ZRB_TRY(check_not_swapped(c));
    ZRB_TRY(check_tied(c, p));
    ZRB_TRY(check_tied(c, g));
    if (c->cfg.engine == ZRB_ENGINE_TC) return tc_train_step_layer(c, p, g, layer, (cudaStream_t)stream);
    if (layer != c->bwd_next_layer) {
        set_error("backward layers must be visited in order L-1..0");
        return ZRB_E_STATE;
    }
    c->bwd_next_layer = layer - 1;
    return ZRB_OK;
}

int zrb_set_keep_clipped_grads(zrb_ctx* c, int32_t on) {
    ZRB_REQUIRE(c, "null ctx");
    c->keep_clipped = on != 0;
    return ZRB_OK;
}

int zrb_set_embed_sparse(zrb_ctx* c, int32_t on) {
    ZRB_REQUIRE(c, "null ctx");
    ZRB_REQUIRE(on >= 0 && on <= 2, "mode must be 0, 1 or 2");
    c->emb_sparse = on != 0;
    c->fused_norm = on == 1;
    c->emb_prev_grad = nullptr;
    return ZRB_OK;
}

int zrb_rec_plans(const zrb_ctx* c, int32_t* h_out) {
    ZRB_REQUIRE(c && h_out, "null argument");
    ZRB_REQUIRE(c->cfg.engine == ZRB_ENGINE_TC && c->tc, "recurrence plans exist only in tensor-core contexts");
    tc_rec_plans(c, 0, h_out);
    return ZRB_OK;
}

int zrb_rec_plans_layer(const zrb_ctx* c, int32_t layer, int32_t* h_out) {
    ZRB_REQUIRE(c && h_out, "null argument");
    ZRB_REQUIRE(c->cfg.engine == ZRB_ENGINE_TC && c->tc, "recurrence plans exist only in tensor-core contexts");
    ZRB_REQUIRE(layer >= 0 && layer < c->cfg.layers, "layer %d outside [0, %d)", layer, c->cfg.layers);
    tc_rec_plans(c, layer, h_out);
    return ZRB_OK;
}

int zrb_set_embed_rows_out(zrb_ctx* c, float* rows) {
    ZRB_REQUIRE(c, "null ctx");
    ZRB_TRY(refuse_experts(c, "zrb_set_embed_rows_out (data parallel)"));
    c->embed_rows_out = rows;
    return ZRB_OK;
}

int zrb_embed_scatter_rows(zrb_ctx* c, float* grad_embed, const int64_t* ids, const float* rows, int64_t n_rows,
                           void* stream) {
    ZRB_REQUIRE(c && grad_embed && ids && rows && n_rows >= 0, "bad arguments");
    cudaStream_t s = (cudaStream_t)stream;
    if (n_rows > c->emb_cap_rows) {
        ZRB_TRY(dalloc(c, &c->emb_acc, (size_t)n_rows * c->width[0]));   // (a previous, smaller one is kept until destroy)
        c->emb_cap_rows = n_rows;
    }
    ProfScope ps(c, ZRB_PROF_EMBED_BWD, s);
    const int H = c->width[0], V = c->cfg.vocab;
    // tied: grad_embed holds the reduced projection gradient, every row of it non-zero and updated densely
    if (c->tied) return embed_scatter_rows(ids, rows, grad_embed, (int)n_rows, H, V, c->emb_first, c->emb_acc, s, true);
    if (c->emb_sparse && c->emb_prev_grad == grad_embed) {
        ZRB_TRY(embed_zero_rows(grad_embed, c->emb_prev_ids, c->emb_prev_n, H, V, s));   // only the last step's rows are non-zero
    } else {
        ZRB_CUDA(cudaMemsetAsync(grad_embed, 0, (size_t)V * H * sizeof(float), s));
    }
    ZRB_TRY(embed_scatter_rows(ids, rows, grad_embed, (int)n_rows, H, V, c->emb_first, c->emb_acc, s));
    if (c->emb_sparse) {   // zrb_train_step_update then takes the norm over / updates these rows only
        if (n_rows > c->emb_prev_cap) {
            ZRB_TRY(dalloc(c, &c->emb_prev_ids, (size_t)n_rows));
            c->emb_prev_cap = n_rows;
        }
        ZRB_CUDA(cudaMemcpyAsync(c->emb_prev_ids, ids, (size_t)n_rows * sizeof(int64_t), cudaMemcpyDeviceToDevice, s));
        c->emb_prev_n = (int)n_rows;
        c->emb_prev_grad = grad_embed;
    }
    return ZRB_OK;
}

int zrb_train_step_update(zrb_ctx* c, const zrb_params* p, const zrb_params* g, float lr, float max_norm,
                          float* norm_out, void* stream) {
    ZRB_REQUIRE(c && p && g, "null argument");
    ZRB_TRY(watchdog_check(c));
    ZRB_REQUIRE(tensor_count(c) <= kMaxTensors, "fused step supports at most 3 layers");
    ZRB_TRY(check_tied(c, p));
    ZRB_TRY(check_tied(c, g));
    ZRB_TRY(check_not_swapped(c));
    UpdateStep st;
    st.tl = param_list(c, p, g);
    st.lr = lr;
    if (c->avg_on) {
        // iterate averaging: this update is number n = avg_n + 1, mu = fp32(1 / n) rounded once from double
        st.kind = UpdateStep::kSgdAvg;
        const TensorList ta = param_list(c, &c->avg.base, &c->avg.base);
        ZRB_TRY(check_avg_alias(ta, st.tl, true));
        for (int i = 0; i < ta.count; ++i) st.avg.a[i] = ta.p[i];
        st.avg.mu = (float)(1.0 / (double)(c->avg_n + 1));
        st.avg.first = c->avg_n == 0;
    } else if (c->adam_on) {
        // Adam: this update is number t = adam_t + 1; each scalar computed in double and rounded once to fp32
        st.kind = UpdateStep::kAdam;
        const TensorList tm = param_list(c, &c->adam_m.base, &c->adam_v.base);
        TensorList tv = tm;
        for (int i = 0; i < tm.count; ++i) tv.p[i] = tm.g[i];
        ZRB_TRY(check_moment_alias(tm, st.tl));
        ZRB_TRY(check_moment_alias(tv, st.tl));
        AdamStep& ad = st.adam;
        for (int i = 0; i < tm.count; ++i) { ad.m[i] = tm.p[i]; ad.v[i] = tm.g[i]; }
        const double b1 = c->adam_b1, b2 = c->adam_b2, t = (double)(c->adam_t + 1);
        ad.k.beta1 = c->adam_b1; ad.k.beta2 = c->adam_b2; ad.k.eps = c->adam_eps;
        ad.k.omb1 = (float)(1.0 - b1);
        ad.k.omb2 = (float)(1.0 - b2);
        ad.k.step_size = (float)((double)lr / (1.0 - std::pow(b1, t)));
        ad.k.bc2s = (float)std::sqrt(1.0 - std::pow(b2, t));
    }
    ZRB_TRY(apply_update(c, p, st, max_norm, norm_out, (cudaStream_t)stream));
    if (st.kind == UpdateStep::kSgdAvg) c->avg_n++;
    if (st.kind == UpdateStep::kAdam) c->adam_t++;
    return ZRB_OK;
}

int zrb_eval_step(zrb_ctx* c, const zrb_params* p, const int64_t* x, const int64_t* y, int32_t T, int32_t B,
                  const zrb_states* in, const zrb_states* out, float* loss, float* tgt_prob, void* stream) {
    ZRB_REQUIRE(c && p && x && y && in && out, "null argument");
    ZRB_TRY(check_shapes(c, T, B));
    ZRB_TRY(check_tied(c, p));
    if (c->experts) {
        c->T = T; c->B = B; c->train = 0; c->seed = 0; c->step = 0;
        c->have_fwd = false;  // eval keeps nothing for backward
        c->reg_use = false;
        return tc_mos_eval_step(c, p, x, y, in, out, loss, tgt_prob, (cudaStream_t)stream);
    }
    ZRB_TRY(zrb_forward(c, p, x, T, B, in, out, c->scores, 0, 0, 0, stream));
    c->have_fwd = false;  // eval keeps nothing for backward
    return softmax_nll(c->scores, y, T * B, c->cfg.vocab, B, c->row_loss, loss, nullptr, tgt_prob,
                       (cudaStream_t)stream);
}

// ---- dynamic evaluation (DESIGN.md section 14) ----------------------------------------------------------------------
// g = the gradient of the eval-mode window loss at p: the fused gradient path with no dropout (c->train = 0)
static int eval_grads(zrb_ctx* c, const zrb_params* p, const zrb_params* g, const int64_t* x, const int64_t* y, int T,
                      int B, const zrb_states* in, const zrb_states* out, float* loss, cudaStream_t s) {
    if (c->cfg.engine == ZRB_ENGINE_TC) return tc_eval_grads(c, p, g, x, y, T, B, in, out, loss, s);
    ZRB_TRY(zrb_forward(c, p, x, T, B, in, out, c->scores, 0, 0, 0, s));
    {
        ProfScope ps(c, ZRB_PROF_SOFTMAX, s);
        ZRB_TRY(softmax_nll(c->scores, y, T * B, c->cfg.vocab, B, c->row_loss, loss, c->dscores, nullptr, s));
    }
    return simt_backward(c, p, c->dscores, g, s);
}

int zrb_grad_stats_step(zrb_ctx* c, const zrb_params* p, const zrb_params* g, const zrb_params* ms, const int64_t* x,
                        const int64_t* y, int32_t T, int32_t B, const zrb_states* in, const zrb_states* out, float* loss,
                        void* stream) {
    ZRB_REQUIRE(c && p && g && ms && x && y && in && out, "null argument");
    ZRB_REQUIRE(tensor_count(c) <= kMaxTensors, "gradient statistics support at most 3 layers");
    ZRB_TRY(refuse_experts(c, "gradient statistics"));
    ZRB_TRY(check_shapes(c, T, B));
    ZRB_TRY(check_tied(c, p));
    ZRB_TRY(check_tied(c, g));
    ZRB_TRY(check_tied(c, ms));
    cudaStream_t s = (cudaStream_t)stream;
    ZRB_TRY(eval_grads(c, p, g, x, y, T, B, in, out, loss, s));
    return sq_accumulate(param_list(c, ms, g), s);
}

int zrb_grad_stats_finish(zrb_ctx* c, const zrb_params* ms, int64_t windows, float* rms_mean, void* stream) {
    ZRB_REQUIRE(c && ms && rms_mean, "null argument");
    ZRB_REQUIRE(windows >= 1, "windows=%lld must be >= 1", (long long)windows);
    ZRB_REQUIRE(tensor_count(c) <= kMaxTensors, "gradient statistics support at most 3 layers");
    ZRB_TRY(refuse_experts(c, "gradient statistics"));
    ZRB_TRY(check_tied(c, ms));
    if (!c->stats_partials) ZRB_TRY(dalloc(c, &c->stats_partials, kStatsPartials));
    return stats_finish(param_list(c, ms, ms), windows, c->stats_partials, rms_mean, (cudaStream_t)stream);
}

int zrb_dyneval_step(zrb_ctx* c, const zrb_params* p, const zrb_params* g, const zrb_params* global,
                     const zrb_params* rms, const float* rms_mean, const int64_t* x, const int64_t* y, int32_t T,
                     int32_t B, const zrb_states* in, const zrb_states* out, float lr, float lambda, float eps,
                     float* loss, void* stream) {
    ZRB_REQUIRE(c && p && g && global && x && y && in && out, "null argument");
    ZRB_REQUIRE(tensor_count(c) <= kMaxTensors, "dynamic evaluation supports at most 3 layers");
    ZRB_TRY(refuse_experts(c, "dynamic evaluation"));
    ZRB_REQUIRE(isfinite(lr) && lr >= 0.f, "lr %f must be finite and >= 0", lr);
    ZRB_REQUIRE(isfinite(lambda) && lambda >= 0.f, "lambda %f must be finite and >= 0", lambda);
    ZRB_REQUIRE(!rms || rms_mean, "the RMS rule needs rms_mean");
    ZRB_REQUIRE(!rms || (isfinite(eps) && eps > 0.f), "eps %f must be finite and > 0 under the RMS rule", eps);
    ZRB_TRY(check_shapes(c, T, B));
    ZRB_TRY(check_tied(c, p));
    ZRB_TRY(check_tied(c, g));
    ZRB_TRY(check_tied(c, global));
    ZRB_TRY(check_tied(c, rms));
    UpdateStep st;
    st.kind = UpdateStep::kDyn;
    st.tl = param_list(c, p, g);
    const TensorList tg = param_list(c, global, global);
    ZRB_TRY(check_aligned(tg, "theta_g"));
    for (int i = 0; i < tg.count; ++i) st.tg[i] = tg.p[i];
    if (rms) {
        const TensorList tr = param_list(c, rms, rms);
        ZRB_TRY(check_aligned(tr, "RMS statistic"));
        for (int i = 0; i < tr.count; ++i) st.r[i] = tr.p[i];
    }
    st.dyn.lr = lr; st.dyn.lam = lambda; st.dyn.eps = eps; st.dyn.rbar = rms ? rms_mean : nullptr;
    cudaStream_t s = (cudaStream_t)stream;
    ZRB_TRY(eval_grads(c, p, g, x, y, T, B, in, out, loss, s));
    return apply_update(c, p, st, 0.f, nullptr, s);
}

int zrb_sample(const float* scores, int64_t ld, int32_t B, int32_t V, const zrb_sampling* cfg, uint64_t pos,
               int64_t* tokens, float* logprobs, void* stream) {
    return sample_rows(scores, ld, B, V, cfg, pos, tokens, logprobs, (cudaStream_t)stream);
}

// eval-mode forward of a [c->T, B] window; only the last step's B rows are projected (scores NULL: none)
static int forward_last_rows(zrb_ctx* c, const zrb_params* p, const int64_t* x, const zrb_states* in,
                             const zrb_states* out, float* scores, cudaStream_t s) {
    if (c->cfg.engine == ZRB_ENGINE_TC) return tc_forward(c, p, x, in, out, scores, s, true);
    return simt_forward(c, p, x, in, out, scores, s, true);
}

int zrb_generate(zrb_ctx* c, const zrb_params* p, const int64_t* prompt, int32_t T0, int32_t B, const zrb_states* in,
                 const zrb_states* out, int32_t n_new, const zrb_sampling* cfg, uint64_t pos0, int64_t* tokens,
                 float* logprobs, void* stream) {
    ZRB_REQUIRE(c && p && prompt && in && out && tokens, "null argument");
    ZRB_REQUIRE(T0 >= 1 && n_new >= 1, "T0=%d and n_new=%d must be >= 1", T0, n_new);
    ZRB_TRY(check_shapes(c, 1, B));
    ZRB_TRY(sample_check(cfg, B, c->cfg.vocab));
    ZRB_TRY(check_tied(c, p));
    cudaStream_t s = (cudaStream_t)stream;
    const int V = c->cfg.vocab, S = c->cfg.max_seq;
    c->B = B; c->train = 0; c->seed = 0; c->step = 0;
    c->have_fwd = false;
    // prefill in windows of at most max_seq steps; only the last window projects (its last step)
    const zrb_states* src = in;
    for (int t0 = 0; t0 < T0; t0 += S) {
        c->T = T0 - t0 < S ? T0 - t0 : S;
        ZRB_TRY(forward_last_rows(c, p, prompt + (size_t)t0 * B, src, out, t0 + c->T == T0 ? c->scores : nullptr, s));
        src = out;
    }
    // decode: sample from the scores of position pos0 + k, feed the token back as the next T = 1 window
    c->T = 1;
    for (int k = 0; k < n_new; ++k) {
        int64_t* tok = tokens + (size_t)k * B;
        ZRB_TRY(sample_rows(c->scores, V, B, V, cfg, pos0 + (uint64_t)k, tok, logprobs ? logprobs + (size_t)k * B : nullptr,
                            s));
        if (k + 1 < n_new) ZRB_TRY(forward_last_rows(c, p, tok, out, out, c->scores, s));
    }
    return ZRB_OK;
}

int zrb_beam_step(const float* scores, int64_t ld, int32_t B, int32_t K_in, int32_t K, int32_t V, const float* cum_in,
                  const int64_t* tok_in, int32_t eos, int64_t* tokens, int32_t* parents, float* cum_out, float* logprobs,
                  void* stream) {
    ZRB_TRY(beam_check(B, K, V, eos));
    ZRB_REQUIRE(K_in >= 1 && K_in <= ZRB_MAX_BEAMS, "K_in=%d outside [1,%d]", K_in, ZRB_MAX_BEAMS);
    cudaStream_t s = (cudaStream_t)stream;
    BeamCand* cands = nullptr;   // stream-ordered scratch: no context here, and no synchronisation
    ZRB_CUDA(cudaMallocAsync((void**)&cands, (size_t)B * K_in * K * sizeof(BeamCand), s));
    const int rc = beam_step(scores, ld, B, K_in, K, V, cum_in, tok_in, eos, cands, tokens, parents, cum_out, logprobs,
                             nullptr, nullptr, 0, LayerWidths{}, s);
    ZRB_CUDA(cudaFreeAsync(cands, s));
    return rc;
}

// zrb_beam_search's scratch (engine.h): the fixed part once, the per-step arrays grown to `entries`
static int beam_scratch(zrb_ctx* c, int64_t entries) {
    if (!c->beam_cand) {
        size_t total = 0;
        for (int l = 0; l < c->cfg.layers; ++l) total += 4 * (size_t)c->cfg.max_batch * c->width[l + 1];
        float* st = nullptr;
        ZRB_TRY(dalloc(c, &st, total));
        for (int l = 0; l < c->cfg.layers; ++l) {
            const size_t BH = (size_t)c->cfg.max_batch * c->width[l + 1];
            for (int k = 0; k < 2; ++k) {
                c->beam_st[k].h[l] = st + 2 * k * BH;
                c->beam_st[k].c[l] = st + (2 * k + 1) * BH;
            }
            st += 4 * BH;
        }
        ZRB_TRY(dalloc(c, &c->beam_cum, (size_t)c->cfg.max_batch));
        ZRB_TRY(dalloc(c, &c->beam_cand, (size_t)c->cfg.max_batch * ZRB_MAX_BEAMS));
    }
    if (entries > c->beam_cap) {   // (previous, smaller ones are kept until destroy)
        ZRB_TRY(dalloc(c, &c->beam_tok, (size_t)entries));
        ZRB_TRY(dalloc(c, &c->beam_par, (size_t)entries));
        ZRB_TRY(dalloc(c, &c->beam_lp, (size_t)entries));
        c->beam_cap = entries;
    }
    return ZRB_OK;
}

int zrb_beam_search(zrb_ctx* c, const zrb_params* p, const int64_t* prompt, int32_t T0, int32_t B, const zrb_states* in,
                    const zrb_states* out, int32_t n_new, int32_t K, int32_t eos, int64_t* tokens, float* logprobs,
                    float* scores, void* stream) {
    ZRB_REQUIRE(c && p && prompt && in && out && tokens, "null argument");
    ZRB_REQUIRE(T0 >= 1 && n_new >= 1, "T0=%d and n_new=%d must be >= 1", T0, n_new);
    ZRB_TRY(beam_check(B, K, c->cfg.vocab, eos));
    ZRB_REQUIRE((int64_t)B * K <= c->cfg.max_batch, "B*K=%lld above the context's max_batch %d", (long long)B * K,
                c->cfg.max_batch);
    ZRB_TRY(check_shapes(c, 1, B * K));
    ZRB_TRY(check_tied(c, p));
    cudaStream_t s = (cudaStream_t)stream;
    const int V = c->cfg.vocab, S = c->cfg.max_seq, L = c->cfg.layers, BK = B * K;
    LayerWidths hw{};
    for (int l = 0; l < L; ++l) hw.h[l] = c->width[l + 1];
    ZRB_TRY(beam_scratch(c, (int64_t)n_new * BK));
    const zrb_states* fwd_out = &c->beam_st[0];   // the forward's output rows: B after the prefill, then B*K
    const zrb_states* gathered = &c->beam_st[1];  // rows reordered by parent, the next forward's input
    c->B = B; c->train = 0; c->seed = 0; c->step = 0;
    c->have_fwd = false;
    const zrb_states* src = in;
    for (int t0 = 0; t0 < T0; t0 += S) {
        c->T = T0 - t0 < S ? T0 - t0 : S;
        ZRB_TRY(forward_last_rows(c, p, prompt + (size_t)t0 * B, src, fwd_out, t0 + c->T == T0 ? c->scores : nullptr, s));
        src = fwd_out;
    }
    // step k: select from the scores of B*K_in rows, gather the parents' states; unless k = n_new - 1, a T = 1 forward
    // of the new tokens.  The last gather goes straight to `out`.
    c->T = 1;
    c->B = BK;
    for (int k = 0; k < n_new; ++k) {
        const int K_in = k ? K : 1;
        const size_t at = (size_t)k * BK;
        const bool last = k + 1 == n_new;
        ZRB_TRY(beam_step(c->scores, V, B, K_in, K, V, k ? c->beam_cum : nullptr, k ? c->beam_tok + at - BK : nullptr, eos,
                          c->beam_cand, c->beam_tok + at, c->beam_par + at, c->beam_cum, c->beam_lp + at, fwd_out,
                          last ? out : gathered, L, hw, s));
        if (!last) ZRB_TRY(forward_last_rows(c, p, c->beam_tok + at, gathered, fwd_out, c->scores, s));
    }
    return beam_backtrack(c->beam_tok, c->beam_par, c->beam_lp, c->beam_cum, n_new, BK, K, tokens, logprobs, scores, s);
}

int zrb_train_step_host(zrb_ctx* c, const zrb_params* p, const zrb_params* g, const int64_t* h_x,
                        const int64_t* h_y, int32_t T, int32_t B, const zrb_states* in, const zrb_states* out,
                        uint64_t seed, uint64_t step, float lr, float max_norm, float* h_loss, float* h_norm,
                        void* stream) {
    ZRB_REQUIRE(c && h_x && h_y && h_loss, "null argument");
    ZRB_TRY(check_shapes(c, T, B));
    ZRB_TRY(check_tied(c, p));
    ZRB_TRY(check_tied(c, g));
    cudaStream_t s = (cudaStream_t)stream;
    size_t nb = (size_t)T * B * sizeof(int64_t);
    ZRB_CUDA(cudaMemcpyAsync(c->x_dev, h_x, nb, cudaMemcpyHostToDevice, s));
    ZRB_CUDA(cudaMemcpyAsync(c->y_dev, h_y, nb, cudaMemcpyHostToDevice, s));
    float* d_loss = c->scalars + 4;
    float* d_norm = c->scalars + 5;
    ZRB_TRY(zrb_train_step_grads(c, p, g, c->x_dev, c->y_dev, T, B, in, out, seed, step, d_loss, stream));
    ZRB_TRY(zrb_train_step_update(c, p, g, lr, max_norm, d_norm, stream));
    ZRB_CUDA(cudaMemcpyAsync(h_loss, d_loss, sizeof(float), cudaMemcpyDeviceToHost, s));
    if (h_norm) ZRB_CUDA(cudaMemcpyAsync(h_norm, d_norm, sizeof(float), cudaMemcpyDeviceToHost, s));
    ZRB_CUDA(cudaStreamSynchronize(s));
    return watchdog_check(c);   // this step's kernels have finished: report a give-up now, not at the next call
}

int zrb_lstm_layer_fwd(zrb_ctx* c, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                       const float* x, int32_t T, int32_t B, const float* h0, const float* c0, float* y, float* hT,
                       float* cT, void* stream) {
    ZRB_REQUIRE(c && w_ih && w_hh && b_ih && b_hh && x && h0 && c0 && y, "null argument");
    ZRB_TRY(check_shapes(c, T, B));
    ZRB_REQUIRE(c->cfg.engine == ZRB_ENGINE_TC, "zrb_lstm_layer_fwd is an entry point of the tensor-core engine");
    ZRB_REQUIRE(c->cfg.hidden > 0, "zrb_lstm_layer_fwd needs a context of one width");
    ZRB_REQUIRE(h0 != hT && c0 != cT, "the unit-level entry point does not alias states");
    ZRB_REQUIRE(!zoneout_on(c), "zrb_lstm_layer_fwd has no zoneout: switch it off (zrb_set_zoneout(ctx, 0, 0)) first");
    return tc_layer_fwd(c, w_ih, w_hh, b_ih, b_hh, x, T, B, h0, c0, y, hT, cT, (cudaStream_t)stream);
}

int zrb_lstm_layer_bwd(zrb_ctx* c, const float* dy, float* dx, float* dw_ih, float* dw_hh, float* db_ih, float* db_hh,
                       void* stream) {
    ZRB_REQUIRE(c && dy && dw_ih && dw_hh && db_ih && db_hh, "null argument");
    ZRB_REQUIRE(c->cfg.engine == ZRB_ENGINE_TC, "zrb_lstm_layer_bwd is an entry point of the tensor-core engine");
    ZRB_REQUIRE(c->cfg.hidden > 0, "zrb_lstm_layer_bwd needs a context of one width");
    ZRB_REQUIRE(!zoneout_on(c), "zrb_lstm_layer_bwd has no zoneout: switch it off (zrb_set_zoneout(ctx, 0, 0)) first");
    return tc_layer_bwd(c, dy, dx, dw_ih, dw_hh, db_ih, db_hh, (cudaStream_t)stream);
}

int zrb_prof_enable(zrb_ctx* c, int32_t on) {
    ZRB_REQUIRE(c, "null ctx");
    c->prof_on = on != 0;
    return ZRB_OK;
}

int zrb_prof_read(zrb_ctx* c, float* h_ms, int64_t* h_counts) {
    ZRB_REQUIRE(c && h_ms && h_counts, "null argument");
    ZRB_CUDA(cudaDeviceSynchronize());
    for (int i = 0; i < ZRB_PROF_COUNT; ++i) { h_ms[i] = 0.f; h_counts[i] = 0; }
    for (auto& r : c->prof_recs) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) { h_ms[r.cls] += ms; h_counts[r.cls]++; }
        c->prof_pool.push_back(r.a);
        c->prof_pool.push_back(r.b);
    }
    c->prof_recs.clear();
    return ZRB_OK;
}

int zrb_prof_rec_trace(zrb_ctx* c, int64_t* h_out, int32_t max_entries) {
    ZRB_REQUIRE(c && h_out, "null argument");
    if (c->cfg.engine != ZRB_ENGINE_TC) { set_error("recurrence trace needs the tensor-core engine"); return ZRB_E_STATE; }
    return tc_rec_trace(c, (long long*)h_out, max_entries);
}

int zrb_gemm_f32(const float* A, const float* B, float* C, int32_t M, int32_t N, int32_t K, int32_t transA,
                 int32_t transB, float alpha, float beta, void* stream) {
    ZRB_REQUIRE(A && B && C && M >= 0 && N >= 0 && K >= 0, "bad gemm args");
    return gemm_f32(A, B, C, M, N, K, transA, transB, alpha, beta, (cudaStream_t)stream);
}

}  // extern "C"
