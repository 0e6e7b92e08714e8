// Context layout and the two engines' entry points (internal).
#pragma once
#include <vector>

#include "kernels.h"

struct zrb_tc_state;  // tensor-core engine private data (engine_tc.cu)

struct zrb_ctx {
    zrb_config cfg{};              // cfg.hidden = 0 when the layers' widths differ (zrb_ctx_create_widths)
    // width of dropout site s (DESIGN.md section 18): width[0] = E, width[l + 1] = H_l; layer l reads width[l] and
    // writes width[l + 1].  Every entry is cfg.hidden in a context of one width.
    int width[ZRB_MAX_LAYERS + 1] = {};
    int max_width = 0;
    int experts = 0;                       // zrb_ctx_create_mos: K softmaxes in the head (DESIGN.md section 19), 0 = plain
    float p_mos = 0.f;                     // zrb_set_mos_dropout: latent dropout of the head
    float z_c = 0.f, z_h = 0.f;            // zrb_set_zoneout: zoneout of the cell and hidden states (DESIGN.md section 20)
    float* ctil[ZRB_MAX_LAYERS] = {};      // ... [N,H_l] c~_t of the last forward, allocated when first switched on
    uint8_t* zflags[ZRB_MAX_LAYERS] = {};  // ... [N,H_l] train-mode flags of the last forward (zoneout_flags)
    float* zhcarry = nullptr;              // ... [B,max width] the per-timestep backward's carried zh * dh
    std::vector<void*> allocs;
    int64_t bytes = 0;

    // activations kept between forward and backward (fp32, token-major [N, .])
    float* act[ZRB_MAX_LAYERS + 1] = {};   // act[0] = dropout(embed(x)); act[l+1] = dropout(h of layer l)
    float* gates[ZRB_MAX_LAYERS] = {};     // [N,4H] activated (i,f,g,o)
    float* cst[ZRB_MAX_LAYERS] = {};       // [N,H]  c_t
    float* hraw[ZRB_MAX_LAYERS] = {};      // [N,H]  h_t before dropout
    float* h0s[ZRB_MAX_LAYERS] = {};       // [B,H]  state entering the window
    float* c0s[ZRB_MAX_LAYERS] = {};
    // backward scratch
    float* dy = nullptr;                   // [N,H]
    float* dx = nullptr;                   // [N,H]
    float* dG = nullptr;                   // [N,4H]
    float* dh_rec = nullptr;               // [B,H]
    float* dc = nullptr;                   // [B,H]
    // loss / optimiser scratch
    float* row_loss = nullptr;             // [N]
    float* partials = nullptr;
    float* scalars = nullptr;
    int64_t* x_saved = nullptr;            // [N] token ids of the last forward
    int64_t* x_dev = nullptr;              // staging for host-buffer entry points
    int64_t* y_dev = nullptr;
    float* scores = nullptr;               // [N,V] used by the fused step / eval
    float* dscores = nullptr;              // [N,V]

    int T = 0, B = 0, train = 0;
    uint64_t seed = 0, step = 0;
    bool have_fwd = false;
    bool layer_fwd_ok = false;             // zrb_lstm_layer_fwd ran and its activations are still in slot 0
    bool explicit_masks_set = false;
    const uint8_t* explicit_masks[ZRB_MAX_LAYERS + 1] = {};
    bool variational = false;              // zrb_set_variational_dropout: masks fixed over the window, recurrent sites
    float p_rec = 0.f;
    float* hrec[ZRB_MAX_LAYERS] = {};      // validation engine, variational mode: [(T+1)*B, H] h_{t-1} * recurrent mask
                                           // (block 0: the state entering the window); allocated when first switched on
    float p_wd = 0.f;                      // zrb_set_weight_drop: DropConnect on W_hh (DESIGN.md section 15)
    uint64_t wd_seed = 0;
    float* whh_wd[ZRB_MAX_LAYERS] = {};    // validation engine, weight drop: [4H, H] fp32(W_hh * mask * scale) of the
                                           // last train-mode forward; allocated when first switched on
    float p_ed = 0.f;                      // zrb_set_embed_dropout: whole word types dropped (DESIGN.md section 17)
    uint64_t ed_seed = 0;
    float ar_alpha = 0.f, tar_beta = 0.f;  // zrb_set_activation_reg: AR / TAR on the last layer (DESIGN.md section 17)
    bool reg_use = false;                  // this train step's backward adds reg_r (set by the fused train steps only)
    float* reg_r = nullptr;                // [max_seq * max_batch, H] the penalties' gradient wrt h of the last layer
    double* reg_part = nullptr;            // kActRegBlocks x 2 partial sums
    float* reg_val = nullptr;              // [2] the last train step's alpha-weighted AR and beta-weighted TAR
    int64_t weights_version = 1;          // bumped whenever parameter values change
    bool avg_on = false;                   // zrb_set_average: iterate averaging into `avg` (DESIGN.md section 16)
    zrb_mos_params avg{};                  // (the head tensors only in a context with experts)
    int64_t avg_n = 0;                     // train-step updates averaged so far
    bool avg_swapped = false;              // zrb_swap_average: the parameters hold the average
    bool adam_on = false;                  // zrb_set_adam: Adam in place of SGD, moments in adam_m / adam_v (section 21)
    zrb_mos_params adam_m{}, adam_v{};     // (the head tensors only in a context with experts)
    float adam_b1 = 0.f, adam_b2 = 0.f, adam_eps = 0.f;
    int64_t adam_t = 0;                    // updates applied so far: the next train-step update is number adam_t + 1
    float* bwd_dy = nullptr;               // phased backward: grad wrt the next layer's output / scratch
    float* bwd_dx = nullptr;
    int bwd_next_layer = -1;
    int* emb_first = nullptr;              // workspace of zrb_embed_scatter_rows (allocated on first use)
    long long* emb_acc = nullptr;
    int64_t emb_cap_rows = 0;
    bool keep_clipped = true;              // zrb_train_step_update writes coef * g back into the gradient buffers
    bool emb_sparse = false;               // touch only the rows of the embedding gradient that can be non-zero
    bool lazy_update = false;              // zrb_set_lazy_update: upper-layer / fc weight updates run beside the next forward
    bool fused_norm = false;               // single process: matrices' part of the clip norm from the wgrad GEMM epilogues
    bool tied = false;                     // ZRB_TIED_EMBEDDING: embed_w == fc_w in every zrb_params (DESIGN.md section 13)
    int64_t emb_prev_cap = 0;              // capacity of emb_prev_ids (tokens)
    unsigned int* wd_flag = nullptr;       // watchdog of the persistent kernels (rec_common.cuh): device word
    unsigned int* wd_host = nullptr;       // ... and the mapped host word the host polls (watchdog_check)
    int64_t* emb_prev_ids = nullptr;       // token ids whose gradient rows are non-zero in emb_prev_grad
    int emb_prev_n = 0;
    float* emb_prev_grad = nullptr;
    float* embed_rows_out = nullptr;       // if set: backward emits the embedding gradient as N masked rows here
                                           // instead of scattering into the dense table gradient (data parallel)

    // zrb_beam_search scratch, allocated on first use; the per-step arrays grow with n_new * B * K
    zrb::BeamCand* beam_cand = nullptr;    // [max_batch * ZRB_MAX_BEAMS] candidates of one step
    float* beam_cum = nullptr;             // [max_batch] cumulative scores S
    zrb_states beam_st[2] = {};            // [max_batch, H] per layer: the forward's output states / the gathered ones
    int64_t* beam_tok = nullptr;           // [n_new, B*K] per-step tokens, parents and logprobs
    int32_t* beam_par = nullptr;
    float* beam_lp = nullptr;
    int64_t beam_cap = 0;                  // entries of beam_tok / _par / _lp

    double* stats_partials = nullptr;      // zrb_grad_stats_finish: kStatsPartials fp64 block sums (allocated on first use)

    zrb_tc_state* tc = nullptr;

    // optional per-class event timing (zrb_prof_*)
    bool prof_on = false;
    struct ProfRec { int cls; cudaEvent_t a, b; };
    std::vector<ProfRec> prof_recs;
    std::vector<cudaEvent_t> prof_pool;
};

namespace zrb {

MaskSrc site_mask(const zrb_ctx* c, int site);   // dropout site 0..L (period B*H in the variational mode)
MaskSrc rec_mask(const zrb_ctx* c, int layer);   // recurrent site L+1+layer of the variational mode (inactive otherwise)
MaskSrc wd_mask(const zrb_ctx* c, int layer);    // weight-drop site 2L+1+layer over W_hh's 4H*H elements (inactive:
                                                 // eval mode or p_wd = 0)
bool reg_on(const zrb_ctx* c);                   // AR / TAR is switched on (alpha > 0 or beta > 0)
inline bool zoneout_on(const zrb_ctx* c) { return c->z_c > 0.f || c->z_h > 0.f; }   // DESIGN.md section 20
// AR / TAR of the last forward (train mode): r into reg_r and the two values into reg_val, then reg_use = true
int reg_compute(zrb_ctx* c, cudaStream_t s);
MaskSrc ed_mask(const zrb_ctx* c);               // embedding-dropout site 3L+1 over the V vocabulary rows (inactive:
                                                 // eval mode or p_ed = 0)
MaskSrc mos_mask(const zrb_ctx* c);              // latent-dropout site 3L+2 over N*K*E (period B*K*E in the variational
                                                 // mode; inactive: eval mode or p_mos = 0)
// the head tensors of a zrb_params that a context with experts was given (zrb_mos_params, its base first)
inline const zrb_mos_params* mos_of(const zrb_params* p) { return reinterpret_cast<const zrb_mos_params*>(p); }

// RAII bracket: records an event pair around the launches of one kernel class
struct ProfScope {
    zrb_ctx* c; cudaStream_t s; cudaEvent_t b = nullptr;
    ProfScope(zrb_ctx* ctx, int cls, cudaStream_t stream);
    ~ProfScope();
};

// last_only: project only the last timestep's B rows into scores [B,V] (the decode loop of zrb_generate)
int simt_forward(zrb_ctx* c, const zrb_params* p, const int64_t* x, const zrb_states* in, const zrb_states* out,
                 float* scores, cudaStream_t s, bool last_only = false);
int simt_backward(zrb_ctx* c, const zrb_params* p, const float* dscores, const zrb_params* g, cudaStream_t s);

int tc_ctx_init(zrb_ctx* c);
void tc_ctx_free(zrb_ctx* c);
int tc_forward(zrb_ctx* c, const zrb_params* p, const int64_t* x, const zrb_states* in, const zrb_states* out,
               float* scores, cudaStream_t s, bool last_only = false);
int tc_backward(zrb_ctx* c, const zrb_params* p, const float* dscores, const zrb_params* g, cudaStream_t s);
int tc_train_step_grads(zrb_ctx* c, const zrb_params* p, const zrb_params* g, const int64_t* x, const int64_t* y,
                        int T, int B, const zrb_states* in, const zrb_states* out, uint64_t seed, uint64_t step,
                        float* loss, cudaStream_t s);
int tc_mos_eval_step(zrb_ctx* c, const zrb_params* p, const int64_t* x, const int64_t* y, const zrb_states* in,
                     const zrb_states* out, float* loss, float* tgt_prob, cudaStream_t s);
int tc_train_step_begin(zrb_ctx* c, const zrb_params* p, const zrb_params* g, const int64_t* x, const int64_t* y,
                        int T, int B, const zrb_states* in, const zrb_states* out, uint64_t seed, uint64_t step,
                        float* loss, cudaStream_t s);
int tc_train_step_layer(zrb_ctx* c, const zrb_params* p, const zrb_params* g, int l, cudaStream_t s);
int tc_rec_trace(zrb_ctx* c, long long* h_out, int max_entries);
int tc_flush_updates(zrb_ctx* c, cudaStream_t s);   // apply deferred weight updates now (zrb_set_lazy_update)
const __half* tc_last_layer_image(const zrb_ctx* c);   // x_h[L]: fp16 last-layer output of the last forward, pitch
                                                       // pad64(H_{L-1})
// zrb_rec_plans_layer: layer l's 2 x {ok, KS, U, G, nCTA, GBi, Kc, KcS}
void tc_rec_plans(const zrb_ctx* c, int l, int32_t* h_out);
int tc_layer_fwd(zrb_ctx* c, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, const float* x,
                 int T, int B, const float* h0, const float* c0, float* y, float* hT, float* cT, cudaStream_t s);
int tc_layer_bwd(zrb_ctx* c, const float* dy, float* dx, float* dw_ih, float* dw_hh, float* db_ih, float* db_hh,
                 cudaStream_t s);   // the persistent backward recurrence kernel is in use for this context
// st's update of p (st.tl = param_list() over p): the matrices fused with their fp16 image rebuild, the other tensors
// by the list kernels.  max_norm / norm_out: the clip norm of a train-step kind (unused otherwise)
int tc_apply_update(zrb_ctx* c, const zrb_params* p, const UpdateStep& st, float max_norm, float* norm_out,
                    cudaStream_t s);
// st's rule by the list kernels over tl (st.tl, or the part of it without an fp16 image), no norm: it reads the clip
// coefficient in c->scalars[1]
int update_list(const zrb_ctx* c, const UpdateStep& st, const TensorList& tl, cudaStream_t s);
// dynamic evaluation (DESIGN.md section 14): eval-mode gradients
int tc_eval_grads(zrb_ctx* c, const zrb_params* p, const zrb_params* g, const int64_t* x, const int64_t* y, int T, int B,
                  const zrb_states* in, const zrb_states* out, float* loss, cudaStream_t s);

}  // namespace zrb
