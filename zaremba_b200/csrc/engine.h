// Context layout and the two engines' entry points (internal).
#pragma once
#include <vector>

#include "kernels.h"

struct zrb_tc_state;  // tensor-core engine private data (engine_tc.cu)

struct zrb_ctx {
    zrb_config cfg{};
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
    int64_t weights_version = 1;           // bumped whenever parameter values change
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
    unsigned int* resident_flag = nullptr; // written by the backward recurrence kernel once all its CTAs are resident
    unsigned int resident_seq = 0;         // value the last launch publishes there
    unsigned int* wd_flag = nullptr;       // watchdog of the persistent kernels (rec_common.cuh): device word, = resident_flag + 2
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
int tc_train_step_begin(zrb_ctx* c, const zrb_params* p, const zrb_params* g, const int64_t* x, const int64_t* y,
                        int T, int B, const zrb_states* in, const zrb_states* out, uint64_t seed, uint64_t step,
                        float* loss, cudaStream_t s);
int tc_train_step_layer(zrb_ctx* c, const zrb_params* p, const zrb_params* g, int l, cudaStream_t s);
int tc_rec_trace(zrb_ctx* c, long long* h_out, int max_entries);
int tc_flush_updates(zrb_ctx* c, cudaStream_t s);   // apply deferred weight updates now (zrb_set_lazy_update)
bool tc_persistent_bwd(const zrb_ctx* c);
const __half* tc_last_layer_image(const zrb_ctx* c);   // x_h[L]: fp16 last-layer output of the last forward, pitch pad64(H)
void tc_rec_plans(const zrb_ctx* c, int32_t* h_out);   // zrb_rec_plans: 2 x {ok, KS, U, G, nCTA, GBi, Kc, KcS}
int tc_layer_fwd(zrb_ctx* c, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, const float* x,
                 int T, int B, const float* h0, const float* c0, float* y, float* hT, float* cT, cudaStream_t s);
int tc_layer_bwd(zrb_ctx* c, const float* dy, float* dx, float* dw_ih, float* dw_hh, float* db_ih, float* db_hh,
                 cudaStream_t s);   // the persistent backward recurrence kernel is in use for this context
int tc_update(zrb_ctx* c, const zrb_params* p, const TensorList& tl, float lr, float max_norm, float* norm_out,
              cudaStream_t s);
// dynamic evaluation (DESIGN.md section 14): eval-mode gradients, and the update with the dynamic rule
int tc_eval_grads(zrb_ctx* c, const zrb_params* p, const zrb_params* g, const int64_t* x, const int64_t* y, int T, int B,
                  const zrb_states* in, const zrb_states* out, float* loss, cudaStream_t s);
int tc_dyneval_update(zrb_ctx* c, const zrb_params* p, const TensorList& tl, float* const* tg, float* const* r,
                      const DynArgs& a, cudaStream_t s);

}  // namespace zrb
