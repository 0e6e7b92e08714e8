/*
 * zaremba_b200.h -- C ABI of libzaremba_b200.so: the H100 (sm_90a) implementation of
 * the LSTM language-model hot path of ahmetumutdurmus/zaremba.
 *
 * The reference has no native boundary (it is three Python files calling PyTorch), so
 * the entry points below are what a binding for this path would bind; each one cites
 * the reference lines it replaces (paths relative to /root/reference).  INTEGRATION.md
 * shows the ctypes stub a maintainer adds to `model.py`.
 *
 * Conventions
 *   - plain C types only; every pointer is a DEVICE pointer unless its name starts with
 *     `h_` (host).  The caller owns all buffers it passes; the library owns only the
 *     context it creates (activation workspace, low-precision weight images).
 *   - every function returns 0 on success or a negative ZRB_E_* code;
 *     zrb_last_error() returns a thread-local message for the last failure.
 *   - kernels are enqueued on `stream` (a cudaStream_t passed as void*); nothing
 *     synchronises unless documented.  One context per thread / stream.
 *   - tokens n = t*B + b (t-major), exactly how `x.view(-1, H)` / `y.reshape(-1)`
 *     flatten [T,B] in model.py:67 and main.py:81.
 *   - gate row blocks follow torch.nn.LSTM: (i, f, g, o).
 */
#ifndef ZAREMBA_B200_H
#define ZAREMBA_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ZRB_OK            0
#define ZRB_E_INVALID    -1   /* bad argument / unsupported shape            */
#define ZRB_E_CUDA       -2   /* a CUDA runtime / driver call failed         */
#define ZRB_E_STATE      -3   /* call order (e.g. backward without forward)  */
#define ZRB_E_NOMEM      -4

#define ZRB_MAX_LAYERS    8

/* engines: how the dense contractions are executed */
#define ZRB_ENGINE_SIMT   0   /* fp32 CUDA-core GEMMs; validation engine                    */
#define ZRB_ENGINE_TC     1   /* wgmma tensor cores, fp16 operands, fp32 accumulation       */

typedef struct zrb_ctx zrb_ctx;   /* opaque */

/* Shape of the model, i.e. the constructor arguments of `Model` (model.py:76) plus the
 * largest [T,B] window the context must hold activations for. */
typedef struct {
    int32_t vocab;        /* V  */
    int32_t hidden;       /* H  */
    int32_t layers;       /* L  (<= ZRB_MAX_LAYERS) */
    int32_t max_seq;      /* T  upper bound */
    int32_t max_batch;    /* B  upper bound */
    int32_t engine;       /* ZRB_ENGINE_*   */
    float   dropout;      /* p of nn.Dropout (model.py:87) */
    int32_t flags;        /* ZRB_TIED_EMBEDDING or 0; any other bit: ZRB_E_INVALID */
} zrb_config;

/* Tied embedding and softmax weights (Press & Wolf, "Using the Output Embedding to Improve Language Models", EACL 2017;
 * DESIGN.md section 13).  One matrix E [V,H] is both embed.W and fc.W: every zrb_params passed to a tied context, for
 * parameters and for gradients, must have fc_w == embed_w (ZRB_E_INVALID, before anything is launched, otherwise).
 * Forward: x0 = E[x], scores = A_L E^T + b.  Gradient: dE = G_proj + G_emb, where G_proj = dS^T A_L is the projection's
 * weight gradient and, per distinct token id r of the window, e_r = the 2^-40 fixed-point sum of its dropout-masked
 * embedding-gradient rows converted to fp32 once; dE[r] = fp32(G_proj[r] + e_r) (no float atomics: bit-reproducible).
 * The clip norm and the update take E once.  zrb_embed_scatter_rows ADDS its sums into the (reduced) gradient. */
#define ZRB_TIED_EMBEDDING 1

/* The 11 (= 3 + 4L) parameter tensors in the reference's registration order
 * (model.py:83-86; SURVEY 8b): fp32, row-major, contiguous.  Shapes for one width H; a context of per-layer widths
 * (zrb_ctx_create_widths: embedding E, layer l of width H_l and input width In_l = E for l = 0, H_{l-1} after) takes
 * embed_w [V,E], w_ih[l] [4H_l,In_l], w_hh[l] [4H_l,H_l], b_ih[l] / b_hh[l] [4H_l], fc_w [V,H_{L-1}]. */
typedef struct {
    float* embed_w;                       /* [V,H]   embed.W              model.py:11 */
    float* w_ih[ZRB_MAX_LAYERS];          /* [4H,H]  rnns.l.weight_ih_l0  model.py:84 */
    float* w_hh[ZRB_MAX_LAYERS];          /* [4H,H]  rnns.l.weight_hh_l0              */
    float* b_ih[ZRB_MAX_LAYERS];          /* [4H]    rnns.l.bias_ih_l0                */
    float* b_hh[ZRB_MAX_LAYERS];          /* [4H]    rnns.l.bias_hh_l0                */
    float* fc_w;                          /* [V,H]   fc.W                 model.py:62 */
    float* fc_b;                          /* [V]     fc.b                 model.py:63 */
} zrb_params;

/* Mixture of Softmaxes (Yang, Dai, Salakhutdinov & Cohen, "Breaking the Softmax Bottleneck", ICLR 2018; DESIGN.md
 * section 19 states it bit for bit).  A context created by zrb_ctx_create_mos with K = experts takes, wherever an entry
 * point takes a `const zrb_params*`, a pointer to the `base` of a zrb_mos_params (parameters, gradients and averages
 * alike): the three head tensors follow the 3 + 4L of zrb_params, which keeps its size for every other context.
 * With h [N, H_{L-1}] the last layer's output after its dropout (site L), E the embedding width and W = fc_w [V,E]:
 *   u = h latent_w^T + latent_b [N, K*E];  c = tanh(u);  c^ = c * m / (1 - p_l), m = latent dropout, Philox site 3L + 2,
 *       element (t, b, j) = stream element t*B*K*E + b*K*E + j (variational mode: b*K*E + j), the other sites' seed
 *       and step, no mask in eval mode;
 *   a = h prior_w^T [N, K] (no bias), pi = softmax(a);  z_k = c^_k W^T + fc_b [V], q_k = softmax(z_k);
 *   p = sum_k pi_k q_k, and log p[y] = logsumexp_k(log pi_k + z_k[y] - LSE(z_k)).
 * The loss is zrb_softmax_nll's unit, B/N * sum_n -log p_n[y_n]. */
#define ZRB_MAX_EXPERTS  32
typedef struct {
    zrb_params base;
    float* prior_w;                       /* [K, H_{L-1}]    prior.W  */
    float* latent_w;                      /* [K*E, H_{L-1}]  latent.W */
    float* latent_b;                      /* [K*E]           latent.b */
} zrb_mos_params;

/* (h, c) entering / leaving the BPTT window: model.py:94-98.  [B,H] fp32 each (the
 * pytorch path's [1,B,H] has the same bytes); [B,H_l] for layer l of a context of per-layer widths. */
typedef struct {
    float* h[ZRB_MAX_LAYERS];
    float* c[ZRB_MAX_LAYERS];
} zrb_states;

const char* zrb_last_error(void);
const char* zrb_version(void);
/* number of kernels this library has launched in the calling process (bench.py's gpu_launches) */
int64_t     zrb_launch_count(void);

int  zrb_ctx_create(const zrb_config* cfg, zrb_ctx** out);
/* Layers of unequal width (AWD-LSTM's 400-1150-1150-400 model; DESIGN.md section 18): widths[0] = E, the embedding
 * width, and widths[1 + l] = H_l, the width of layer l, for l < cfg->layers; cfg->hidden must be 0.  Layer l's input
 * width is E (l = 0) or H_{l-1}; the projection reads H_{L-1}.  Every per-site rule takes its site's width: dropout
 * site 0 is over E and site l+1 over H_l (element t*B*W + b*W + j; variational: b*W + j), recurrent site L+1+l over
 * B*H_l, weight drop of layer l over 4*H_l*H_l, AR / TAR normalised by H_{L-1}, explicit masks [T*B*W] per site.  With
 * every width equal to H this is zrb_ctx_create with cfg->hidden = H, bit for bit.  ZRB_E_INVALID for a width < 1,
 * cfg->hidden != 0, a tied context with E != H_{L-1}, and ZRB_ENGINE_SIMT with unequal widths; zrb_lstm_layer_fwd /
 * _bwd return ZRB_E_INVALID on a context of unequal widths.  The neural cache takes H = H_{L-1}.  zrb_ctx_create's
 * other rules apply. */
int  zrb_ctx_create_widths(const zrb_config* cfg, const int32_t* widths, zrb_ctx** out);
/* A Mixture-of-Softmaxes context (zrb_mos_params above) of K = experts softmaxes, 1 <= K <= ZRB_MAX_EXPERTS.  widths as
 * zrb_ctx_create_widths (cfg->hidden = 0), or NULL for one width cfg->hidden.  fc_w is [V,E]; a tied context needs
 * nothing beyond that (E = H_{L-1} is not required).  In such a context zrb_forward writes log p into scores [N,V] and
 * zrb_backward takes dL / d log p; the fused train steps (_grads / _begin / _layer / _host / _update, the lazy update),
 * zrb_eval_step, averaging and swapping, zrb_generate, zrb_beam_step and zrb_beam_search work as documented, and the
 * variational mode, weight drop, embedding dropout and AR / TAR act below the head.  Its score workspace holds N*K
 * logits rows (zrb_ctx_workspace_bytes reports it).  ZRB_E_INVALID, before anything is launched, for K outside
 * [1, ZRB_MAX_EXPERTS], ZRB_ENGINE_SIMT, more layers than the fused step's tensor list holds (L <= 3), and -- follow-ups
 * not built yet -- zrb_eval_step_cache, zrb_grad_stats_step / _finish, zrb_dyneval_step and zrb_set_embed_rows_out
 * (data parallel) on such a context. */
int  zrb_ctx_create_mos(const zrb_config* cfg, const int32_t* widths, int32_t experts, zrb_ctx** out);
/* Latent dropout p_l of a Mixture-of-Softmaxes context (0 by default; train mode only).  ZRB_E_INVALID for p outside
 * [0, 1) or not finite and for a context without experts.  A change invalidates the saved forward. */
int  zrb_set_mos_dropout(zrb_ctx* ctx, float p);
/* Zoneout (Krueger et al. 2017; DESIGN.md section 20 states it bit for bit): each unit keeps its previous c with
 * probability z_c and its previous h with probability z_h, instead of taking the new ones.  Off by default (z_c = z_h =
 * 0 changes nothing).  Layer l, step t, row b, unit j: c~ and h~ are the LSTM cell's values.  Train mode: c_t = c_{t-1}
 * where the dropped flag of element t*B*H_l + b*H_l + j of zrb_dropout_mask(seed, step, 3L + 3 + l, T*B*H_l, z_c) is
 * set, else c~ (a select, no scaling); h_t likewise with site 4L + 3 + l and z_h.  `seed` is the activation-mask seed
 * of the call; the flags are drawn per step in the variational mode too.  Eval mode (zrb_eval_step, the drop-in calls
 * with train = 0, generation, beam search, the neural cache, dynamic evaluation): c_t = fma(fp32(z_c), c_{t-1},
 * fp32(1 - z_c) * c~) and h_t likewise.  The layer output and the carried states are the zoned h and c; the states
 * entering the window stay detached.  ZRB_E_INVALID for a value outside [0, 1) or not finite and for ZRB_ENGINE_SIMT;
 * zrb_lstm_layer_fwd / _bwd have no zoneout and return ZRB_E_INVALID while it is on.  The first switch-on allocates
 * 9 bytes per (t, b, j) and layer (zrb_ctx_workspace_bytes reports them).  A change invalidates the saved forward. */
int  zrb_set_zoneout(zrb_ctx* ctx, float z_c, float z_h);
void zrb_ctx_destroy(zrb_ctx* ctx);
/* bytes of device memory the context holds */
int64_t zrb_ctx_workspace_bytes(const zrb_ctx* ctx);

/* Tell the context that parameter values changed outside the library (main.py:116-117
 * updates them in place), so low-precision weight images must be rebuilt on next use. */
int  zrb_params_changed(zrb_ctx* ctx);

/* Dropout: keep-masks are a pure function of (seed, step, site, element) through
 * Philox4x32-10, so backward regenerates them.  `site` 0 = after the embedding,
 * l+1 = after layer l (the three call sites of model.py:105,108).
 * zrb_dropout_mask writes the keep-mask (1 = keep) the kernels will use, so a test can
 * hand the same mask to the oracle. */
int  zrb_dropout_mask(uint64_t seed, uint64_t step, int32_t site, int64_t n, float p,
                      uint8_t* mask_out, void* stream);
/* Optional: force explicit keep-masks instead of Philox (L+1 sites, each [T*B*H] bytes,
 * 1 = keep).  Pass NULL to return to Philox.  Used to replay the reference's masks. */
int  zrb_set_explicit_masks(zrb_ctx* ctx, const uint8_t* const* site_masks);
/* Variational dropout (Gal & Ghahramani, "A Theoretically Grounded Application of Dropout in Recurrent Neural
 * Networks", NeurIPS 2016; DESIGN.md section 11 states it bit for bit).  Opt-in; off (the default) the masks are
 * exactly the ones above.  With on = 1, in train mode:
 *   - sites 0..L keep their (seed, step, site, p) but element (t, b, j) takes the flag of element b*H + j: the mask of
 *     time step 0 held fixed over the window;
 *   - with p_rec > 0, layer l's recurrent operand at every step t (t = 0 included) is m_l * h_{t-1} / (1 - p_rec), one
 *     mask per layer shared by the four gates, site L + 1 + l, element b*H + j.  The layer's output, the carried (h, c)
 *     and c are not masked.
 * Eval mode applies no mask.  zrb_dropout_mask(seed, step, site, B*H, p) gives every mask of the mode.
 * ZRB_E_INVALID for on not 0 / 1, p_rec outside [0, 1), p_rec > 0 with on = 0; ZRB_E_STATE while explicit masks are
 * set (and zrb_set_explicit_masks with non-NULL masks returns ZRB_E_STATE while the mode is on).  A change of the mode
 * invalidates the saved forward: zrb_backward / zrb_train_step_layer then need a new forward first. */
int  zrb_set_variational_dropout(zrb_ctx* ctx, int32_t on, float p_rec);
/* Weight-dropped LSTM (Merity, Keskar & Socher, "Regularizing and Optimizing LSTM Language Models", ICLR 2018;
 * DESIGN.md section 15 states it bit for bit): DropConnect on the hidden-to-hidden matrices.  Opt-in; p = 0 (the
 * default) changes nothing.  In a train-mode call with step s, layer l uses W_eff = fp32(W_hh * m_l * scale) in place of
 * W_hh at every time step and batch row, scale = float32(1 / (1 - p)), m_l = zrb_dropout_mask(seed, s, 2L + 1 + l,
 * 4H*H, p) with element r*H + k = W_hh[r, k].  The gradient is dW_hh = fp32(scale * m_l * dW_eff) (0 where the mask
 * drops); the clip norm is taken over it.  `seed` holds no rank: every data-parallel rank draws the same mask.  Eval mode
 * and zrb_lstm_layer_fwd / _bwd use the raw W_hh.  ZRB_E_INVALID for p outside [0, 1) or not finite.  A change of the
 * mode invalidates the saved forward, as zrb_set_variational_dropout does. */
int  zrb_set_weight_drop(zrb_ctx* ctx, float p, uint64_t seed);
/* Embedding dropout (Merity, Keskar & Socher 2018, AWD-LSTM's `embedded_dropout`; DESIGN.md section 17 states it bit
 * for bit): whole word types are dropped in the gather of model.py:13-14 / :104, before the dropout of :105.  Opt-in; p = 0 (the default) changes nothing.  In a
 * train-mode call with step s, vocabulary row v is gathered as fp32(fp32(W[v, j] * s_e(v)) * s_0) with s_e(v) = 0 or
 * float32(1 / (1 - p)) from m = zrb_dropout_mask(seed, s, 3L + 1, V, p), element v = row v, and s_0 the site-0
 * multiplier; each occurrence of v adds fp32(fp32(dA * s_0) * s_e(v)) to dE (dense scatter, rows-only update,
 * zrb_set_embed_rows_out rows and the tied merge alike).  Tied: only the lookup is masked, the projection uses the raw
 * E.  `seed` holds no rank: every data-parallel rank draws the same mask.  Eval mode (generation, beam search, the
 * neural cache, dynamic evaluation) applies no mask.  ZRB_E_INVALID for p outside [0, 1) or not finite.  A change of
 * (p, seed) invalidates the saved forward, as zrb_set_weight_drop does. */
int  zrb_set_embed_dropout(zrb_ctx* ctx, float p, uint64_t seed);
/* Activation regularization, AR and TAR (Merity, Keskar & Socher 2018, AWD-LSTM main.py's `alpha * dropped_rnn_hs
 * .pow(2).mean()` and `beta * (rnn_hs[1:] - rnn_hs[:-1]).pow(2).mean()`; DESIGN.md section 17 states it bit for bit).
 * Opt-in; alpha = beta = 0 (the default) changes nothing.  Every fused train step (zrb_train_step_grads / _begin /
 * _host) differentiates NLL + R, in the unit of the loss of main.py:77-84 (B x the token mean):
 *   R = alpha / (T*H) * sum_{t,b,j} y^2 + beta / ((T-1)*H) * sum_{t>=1,b,j} (h_t - h_{t-1})^2   (TAR = 0 when T = 1)
 * with h the last layer's raw output and y = h * (its dropout multiplier, site L).  The gradient r_t = dR/dh_t enters
 * the last layer's backward after the output mask: dh_t = fp32(m * s * dY_t) + r_t + the recurrent term.  The clip
 * norm and the gradients include it.  The returned loss stays the NLL.  zrb_forward / zrb_backward, eval calls and the
 * eval-mode gradient of dynamic evaluation ignore it.  ZRB_E_INVALID for negative or non-finite alpha, beta.  A change
 * invalidates the saved forward. */
int  zrb_set_activation_reg(zrb_ctx* ctx, float alpha, float beta);
/* Enqueue on `stream` a copy of the last train step's alpha-weighted AR and beta-weighted TAR values into out2[0..1]
 * (device memory; zeros before the first step with the mode on).  No host synchronisation. */
int  zrb_activation_reg(zrb_ctx* ctx, float* out2, void* stream);

/* Model.forward (model.py:103-110): embedding gather, dropout, L x (LSTM layer,
 * dropout), vocabulary projection.
 *   x        [T,B] int64 token ids, t-major contiguous
 *   in/out   states entering / leaving the window (may alias)
 *   scores   [T*B, V] fp32 (model.py:109), or NULL to skip the projection
 *   train    nonzero = nn.Dropout active (module in .train()), activations kept for backward
 */
int  zrb_forward(zrb_ctx* ctx, const zrb_params* p, const int64_t* x, int32_t T, int32_t B,
                 const zrb_states* in, const zrb_states* out, float* scores,
                 int32_t train, uint64_t seed, uint64_t step, void* stream);

/* What autograd derives for model.py:103-110 given d loss / d scores (main.py:113).
 *   dscores  [T*B, V] fp32
 *   grads    dense gradients, same shapes as the parameters; OVERWRITTEN (not accumulated)
 */
int  zrb_backward(zrb_ctx* ctx, const zrb_params* p, const float* dscores,
                  const zrb_params* grads, void* stream);

/* nll_loss (main.py:77-84) and its gradient in one pass over the scores:
 *   loss      1 float: mean_n(-log softmax(scores)[n, y_n]) * B
 *   dscores   [N,V] fp32 (softmax - onehot) * B / N, or NULL
 *   tgt_prob  [N] fp32 softmax(scores)[n, y_n], or NULL (ensemble.py:100-106 needs it)
 */
int  zrb_softmax_nll(zrb_ctx* ctx, const float* scores, const int64_t* y, int32_t T, int32_t B,
                     float* loss, float* dscores, float* tgt_prob, void* stream);

/* clip_grad_norm_ + SGD (main.py:114-117) over n tensors:
 *   norm = sqrt(sum ||g||^2); coef = min(1, max_norm / (norm + 1e-6)); g *= coef; p -= lr*g
 *   norm_out  1 float (pre-clip norm, main.py:115) */
int  zrb_clip_sgd(zrb_ctx* ctx, int32_t n, float* const* params, float* const* grads,
                  const int64_t* sizes, float lr, float max_norm, float* norm_out, void* stream);

/* One whole iteration of main.py:109-117 without leaving the library (the data-parallel
 * hook sits between the two halves: gradients are complete after _grads, the caller may
 * all-reduce them, then _update clips on the global norm and applies SGD).
 *   y [T,B] int64; loss / norm: 1 float each */
int  zrb_train_step_grads(zrb_ctx* ctx, const zrb_params* p, const zrb_params* grads,
                          const int64_t* x, const int64_t* y, int32_t T, int32_t B,
                          const zrb_states* in, const zrb_states* out,
                          uint64_t seed, uint64_t step, float* loss, void* stream);
/* The same gradients in phases, so that a data-parallel caller can start reducing a bucket while
 * the rest of backward still runs: after _begin (forward, loss, projection backward) the gradients of
 * fc.W / fc.b are complete; after _layer(l), called for l = L-1 .. 0 in that order, those of layer l
 * (and, for l = 0, of embed.W) are complete.  _begin + all _layer calls == zrb_train_step_grads. */
int  zrb_train_step_begin(zrb_ctx* ctx, const zrb_params* p, const zrb_params* grads,
                          const int64_t* x, const int64_t* y, int32_t T, int32_t B,
                          const zrb_states* in, const zrb_states* out,
                          uint64_t seed, uint64_t step, float* loss, void* stream);
int  zrb_train_step_layer(zrb_ctx* ctx, const zrb_params* p, const zrb_params* grads, int32_t layer,
                          void* stream);
/* Sparse form of the embedding gradient for data parallelism.  The gradient of embed.W (model.py:14) is
 * non-zero only in the rows of this window's tokens.  With a rows buffer set, backward writes the N = T*B
 * dropout-masked gradient rows [N,H] there INSTEAD of scattering them into the dense table gradient; ranks
 * all-gather ids and rows (4 MB each instead of a 60 MB all-reduce) and zrb_embed_scatter_rows builds the
 * dense gradient: rows with equal id are summed in index order by the first occurrence, without atomics, so
 * all ranks get identical bits.  Pass NULL to return to the dense scatter.  In a ZRB_TIED_EMBEDDING context the
 * dense gradient already holds the (reduced) projection gradient: zrb_embed_scatter_rows adds the sums of the
 * ids' rows into it (dE[r] = fp32(G_proj[r] + e_r)) instead of clearing and writing. */
int  zrb_set_embed_rows_out(zrb_ctx* ctx, float* rows);
/* Single-process fused step (zrb_train_step_grads/_update with the SAME grads buffers every step): touch only
 * this window's rows of the dense embedding gradient (clear the previous window's rows instead of zero-filling
 * 60 MB, take the norm over and update only the rows that can be non-zero).  The dense buffer stays exactly
 * what the full version would produce.  The same promise -- zrb_train_step_update sees the gradient buffers exactly
 * as zrb_train_step_grads left them -- lets the tensor-core engine take the matrices' part of the clip norm from
 * sums of squares its wgrad GEMM epilogues emitted (no second read of the gradients).  Not for data parallel runs
 * that all-reduce the gradient buffers between the two calls. */
int  zrb_set_embed_sparse(zrb_ctx* ctx, int32_t on);
/* on = 2: the rows-only half alone, for data-parallel steps that all-reduce the gradient buffers between _grads and
 * _update (the epilogue sums of squares describe the LOCAL gradients, so the norm is taken over the reduced buffers):
 * zrb_embed_scatter_rows then clears only the rows the previous step touched and remembers this step's ids (all
 * ranks' tokens), and zrb_train_step_update takes the norm over / updates only those rows of embed.W. */
/* clip_grad_norm_ (main.py:115) scales the gradients in place, so after main.py:117 `.grad` holds coef * g.
 * on = 1 (default): zrb_train_step_update stores coef * g back like the reference.  on = 0: the update still
 * applies p -= lr * coef * g but leaves the gradient buffers as backward wrote them (the scaled gradients are
 * dead values -- main.py:109 zeroes them before the next use -- and storing them is 4 of the ~16 bytes per
 * parameter the update moves).  zrb_clip_sgd always stores them. */
int  zrb_set_keep_clipped_grads(zrb_ctx* ctx, int32_t on);
/* Lazy update (opt-in, tensor-core engine with the persistent recurrence kernels).  The SGD update of main.py:116-117 is
 * HBM-bound work with no consumer until the next forward reaches the layer it belongs to.  With on = 1,
 * zrb_train_step_update applies the clip norm, the embedding, layer 0 and all biases at once and DEFERS the matrices of
 * layers >= 1 and fc.W: the next fused train step launches them as programmatic dependents of its forward recurrence
 * kernels (layer l+1's update beside layer l's recurrence, fc.W's beside the last), on the ~23 SMs those leave idle.
 * Every other entry point that reads parameters (zrb_forward, zrb_eval_step, zrb_clip_sgd, a second _update) applies
 * what is pending first, so results never change -- but the CALLER's own reads of those parameter buffers between two
 * steps must be preceded by zrb_flush_updates(ctx, stream).  Same arithmetic, same order per element. */
int  zrb_set_lazy_update(zrb_ctx* ctx, int32_t on);
int  zrb_flush_updates(zrb_ctx* ctx, void* stream);

/* Iterate averaging (NT-ASGD of Merity, Keskar & Socher 2018; DESIGN.md section 16 states it bit for bit).  Opt-in;
 * off, nothing changes.  zrb_set_average(ctx, avg) with avg non-NULL starts averaging into the tensors of `avg` (laid
 * out like the parameters; tied: avg->fc_w == avg->embed_w) with n = 0 and leaves their contents alone; NULL stops it.
 * Every zrb_train_step_update (and zrb_train_step_host) while it is on sets n = n + 1, applies the SGD update exactly as
 * without averaging, then for every element of every parameter: a = p' at n = 1, else a = a + (p' - a) * mu with
 * mu = fp32(1 / n) and fp32 operations in that order (torch.optim.ASGD(lambd=0, t0=0) created at the start).  The
 * average is dense under the rows-only embedding update too, and it is taken of the raw W_hh under weight drop.  The
 * parameters are never changed by it.  zrb_clip_sgd, zrb_dyneval_step and every eval call leave n alone.  Pending lazy
 * updates are applied first (on the legacy default stream), with the averaging of the steps they belong to.
 * ZRB_E_INVALID for a NULL tensor, average tensors that overlap each other, an untied pair in a tied context, and while
 * swapped; zrb_train_step_update returns ZRB_E_INVALID, before anything is launched, when an average tensor overlaps a
 * parameter or gradient it was given. */
int  zrb_set_average(zrb_ctx* ctx, const zrb_params* avg);
/* n: the number of train-step updates averaged since zrb_set_average (0 while averaging is off). */
int  zrb_average_count(const zrb_ctx* ctx, int64_t* n);
/* Exchange the parameters p and the average bit for bit, and write the fp16 weight images of the values now in p in
 * the same pass (the W_hh images hold the raw weights), so that eval calls need no pack.  The context records that it is
 * swapped; a second call swaps back exactly.  While swapped every zrb_train_step_* call returns ZRB_E_INVALID (training
 * the average and swapping back would corrupt both).  ZRB_E_INVALID when n = 0 and when an average tensor overlaps p. */
int  zrb_swap_average(zrb_ctx* ctx, const zrb_params* p, void* stream);

/* Adam (Kingma & Ba 2015; DESIGN.md section 21 states it bit for bit).  Opt-in; off (the default, and m = NULL),
 * nothing changes.  zrb_set_adam(ctx, m, v, beta1, beta2, eps, step) with m and v non-NULL (laid out like the
 * parameters; tied: m->fc_w == m->embed_w, likewise v; a context with experts takes a zrb_mos_params base) makes every
 * zrb_train_step_update (and zrb_train_step_host) apply Adam after the global-norm clip, in place of SGD.  step = the
 * updates already applied, so the next is number t = step + 1; the context counts on.  Each update computes on the host,
 * in double and rounded once to fp32, step_size = lr / (1 - beta1^t), bc2s = sqrt(1 - beta2^t), omb1 = 1 - beta1 and
 * omb2 = 1 - beta2, then for every element of every parameter, with g' = coef * g (clip_grad_norm_'s scaled gradient)
 * and every fp32 operation rounded on its own in this order:
 *     m = beta1 * m + omb1 * g';  v = beta2 * v + omb2 * (g' * g');  denom = sqrt(v) / bc2s + eps;
 *     p = p - step_size * (m / denom)
 * (torch.optim.Adam with weight_decay = 0, amsgrad = False).  The embedding is updated densely (its moments decay in
 * every row); the rows-only norm and gradient clearing of zrb_set_embed_sparse stay.  g' is stored back as by SGD when
 * zrb_set_keep_clipped_grads is on.  Under lazy update the deferred matrices apply the scalars of their own step (a tied
 * E is applied at once).  zrb_clip_sgd, zrb_dyneval_step, the gradient statistics and every eval call leave m, v and t
 * alone.  Pending lazy updates are applied first (on the legacy default stream).  ZRB_E_INVALID, before anything is
 * launched, for beta1 or beta2 outside [0, 1) or not finite, eps <= 0 or not finite, step < 0, exactly one of m and v,
 * a NULL tensor, moment tensors that overlap each other, an untied pair in a tied context, and while averaging is on or
 * swapped; zrb_set_average refuses to start while Adam is on; zrb_train_step_update returns ZRB_E_INVALID when a
 * moment tensor overlaps a parameter or gradient it was given. */
int  zrb_set_adam(zrb_ctx* ctx, const zrb_params* m, const zrb_params* v, float beta1, float beta2, float eps,
                  int64_t step);

/* Watchdog of the persistent recurrence kernels.  Every wait inside them is bounded (~3 s; ZRB_SPIN_CYCLES overrides).  A
 * wait that runs out -- a lost wake-up, or a grid that never became co-resident -- does not trap: the kernel stops
 * waiting everywhere, finishes with garbage in its outputs and leaves a code in a host-mapped word.  The next call on
 * the context that launches or synchronises (zrb_forward / _eval_step / _train_step_* / _flush_updates; immediately for
 * zrb_train_step_host, which synchronises itself) returns ZRB_E_CUDA with the wait, CTA and step in zrb_last_error();
 * the zrb context stays failed, the CUDA context and the process are unharmed.  zrb_check_health reads that word
 * (one host load, no synchronisation) -- for callers that keep everything on the device and want to poll. */
int  zrb_check_health(zrb_ctx* ctx);
int  zrb_embed_scatter_rows(zrb_ctx* ctx, float* grad_embed, const int64_t* ids, const float* rows,
                            int64_t n_rows, void* stream);
int  zrb_train_step_update(zrb_ctx* ctx, const zrb_params* p, const zrb_params* grads,
                           float lr, float max_norm, float* norm_out, void* stream);

/* ---- data-parallel gradient all-reduce over NVLink peer memory, copy engines only (dp_ce.cu) ----------
 * One process per GPU.  zrb_dp_create allocates the flat gradient buffer (use zrb_dp_grad_buffer as the
 * `grads` storage) and a flag block and exports them through CUDA IPC: exchange the 128-byte blobs of all
 * ranks on the host (rank order) and hand them to zrb_dp_import.  Per step: zrb_dp_begin_step before the
 * first gradient write; after each bucket of the flat buffer is complete on `stream`
 * (zrb_train_step_begin / _layer) call zrb_dp_allreduce_bucket -- same bucket sequence on every rank, SUM
 * semantics, the last bucket with last = 1 makes `stream` wait for the whole reduction.  No SM is used for
 * the transport (cuStreamWaitValue32 / cuStreamWriteValue32 flags + peer cudaMemcpyAsync), so it overlaps
 * with the persistent recurrence kernels, which NCCL's channels do not. */
typedef struct zrb_dp zrb_dp;
int    zrb_dp_create(int32_t rank, int32_t world, int64_t n_grad, zrb_dp** out);
void   zrb_dp_destroy(zrb_dp* dp);
float* zrb_dp_grad_buffer(zrb_dp* dp);
int    zrb_dp_export(zrb_dp* dp, void* h_blob128);
int    zrb_dp_import(zrb_dp* dp, const void* h_blobs);
int    zrb_dp_begin_step(zrb_dp* dp, void* stream);
int    zrb_dp_allreduce_bucket(zrb_dp* dp, int32_t bucket, int64_t lo, int64_t hi, int32_t last, void* stream);
/* join: `stream` waits for all bucket reductions enqueued in this step (alternative to last = 1) */
int    zrb_dp_finish_step(zrb_dp* dp, void* stream);

/* The plans the persistent recurrence kernels of a tensor-core context run with, chosen at creation for its max_batch
 * (so a smaller window reuses them) from the shape and the device's SM count.  h_out[0..7] = forward, h_out[8..15] =
 * backward, each {ok, KS, U, G, nCTA, GBi, Kc, KcS}: ok = 0 means that direction takes the per-timestep path (the other
 * seven are then 0); KS = CTAs sharing one set of gate rows, each holding 1/KS of the contraction (K-split); U = hidden
 * units per CTA; G = 8-row groups of a CTA's weight slice; nCTA = grid size; GBi = 8-row batch groups of the operand
 * images (the MMA's N is 8 * GBi); Kc = 8-element chunks of the contraction; KcS = Kc / KS.  ZRB_E_INVALID for a
 * validation-engine context.  Host only, no synchronisation.  A context of per-layer widths plans every layer for its
 * own width and reports layer 0 here; either direction runs persistent only when every layer's plan fits. */
int  zrb_rec_plans(const zrb_ctx* ctx, int32_t* h_out);
/* zrb_rec_plans for layer `layer` (0 <= layer < L, else ZRB_E_INVALID). */
int  zrb_rec_plans_layer(const zrb_ctx* ctx, int32_t layer, int32_t* h_out);

/* perplexity's inner step (main.py:91-94) without materialising scores for the caller:
 * forward in eval mode + loss (+ per-token target probabilities for the ensemble). */
int  zrb_eval_step(zrb_ctx* ctx, const zrb_params* p, const int64_t* x, const int64_t* y,
                   int32_t T, int32_t B, const zrb_states* in, const zrb_states* out,
                   float* loss, float* tgt_prob, void* stream);

/* ---- text generation (not in the reference: what a user of a trained model calls next) ----------------
 * Sampling configuration: Gumbel-max over a kept set (DESIGN.md section 9 states it bit for bit).
 *   temperature  tau >= 0; 0 = greedy: argmax of the scores, lowest index on ties, no uniforms drawn
 *   top_k        keep the entries >= the k-th largest score (boundary ties kept); 0 or >= V = no filter
 *   top_p        in (0, 1]: over the top-k set with p = softmax(z / tau), keep the entries >= v*, the largest score
 *                whose set {z >= v*} holds at least top_p of the mass (boundary ties kept); 1 = no filter
 *   seed         with (position, row, entry) the key and counter of the Philox4x32-10 uniforms */
typedef struct {
    float    temperature;
    int32_t  top_k;
    float    top_p;
    int32_t  reserved;   /* 0 */
    uint64_t seed;
} zrb_sampling;

/* One token per row of scores [B, ld] fp32 (row b at scores + b*ld, V used entries, finite -- not checked):
 * tokens [B] int64, logprobs [B] fp32 = log softmax(scores[b])[token] at temperature 1 over all V entries (NULL: not
 * written).  A pure function of (scores, cfg, pos, row): the uniforms of row b at position pos are fixed.  One CTA
 * per row, no synchronisation.  ZRB_E_INVALID for temperature < 0, top_p <= 0, top_k < 0, B < 1, V < 1, V > 2^27, ld < V. */
int  zrb_sample(const float* scores, int64_t ld, int32_t B, int32_t V, const zrb_sampling* cfg, uint64_t pos,
                int64_t* tokens, float* logprobs, void* stream);

/* Continue B prompts by n_new sampled tokens without leaving the device (no host synchronisation):
 *   prefill  eval-mode forward of prompt [T0,B] int64 from `in` into `out`, in windows of at most max_seq steps;
 *            only the last step's B rows are projected
 *   step k   tokens[k] (and logprobs[k]) = zrb_sample of those scores at position pos0 + k; unless k = n_new - 1,
 *            a T = 1 eval forward of tokens[k] (read on the device) carries out -> out
 *   tokens [n_new,B] int64, logprobs [n_new,B] fp32 or NULL; in / out may alias.
 * On return `out` is the state BEFORE the last sampled token is consumed: a second call with prompt = tokens[n_new-1],
 * in = out and pos0 + n_new continues the same stream exactly.  Pending lazy weight updates are applied first; no
 * dropout; nothing is kept for zrb_backward.  Both engines; B <= the context's max_batch, any T0. */
int  zrb_generate(zrb_ctx* ctx, const zrb_params* p, const int64_t* prompt, int32_t T0, int32_t B,
                  const zrb_states* in, const zrb_states* out, int32_t n_new, const zrb_sampling* cfg,
                  uint64_t pos0, int64_t* tokens, float* logprobs, void* stream);

/* ---- beam search (DESIGN.md section 10 states it bit for bit) ------------------------------------------
 * Rows and slots: prompt b has K live hypotheses, slot k at row b*K + k; slot 0 is the best.  Per row r with scores z
 * and cumulative score S_r: m = max z, L = logf(sum_j expf(z_j - m)) (zrb_sample's reductions), logp_j = (z_j - m) - L,
 * candidate cand_j = S_r + logp_j (float32).  A row whose last token is eos (>= 0) is finished: its one candidate is
 * j = eos with logp 0 and cand S_r.  The K best candidates of a prompt -- cand descending, ties by the lower flat index
 * i*V + j, i the row's slot -- become the new slots 0..K-1 in that order. */
#define ZRB_MAX_BEAMS    32

/* One selection step: scores [B*K_in, ld] fp32 (finite, V used entries per row), cum_in [B*K_in] (NULL: all 0),
 * tok_in [B*K_in] int64 the rows' last tokens (NULL: none finished).  K_in = K, or K_in = 1 with tok_in = NULL (step 0).
 * Writes, per new slot (row b*K + k): tokens int64, parents int32 (the slot i it extends), cum_out (S) and logprobs
 * (logp) fp32.  cum_in and cum_out may alias.  No synchronisation (the candidate scratch is stream-ordered).
 * ZRB_E_INVALID for B < 1, V < 1, V > 2^26, K < 1, K > ZRB_MAX_BEAMS, K > V, eos outside [-1, V), ld < V, another K_in. */
int  zrb_beam_step(const float* scores, int64_t ld, int32_t B, int32_t K_in, int32_t K, int32_t V, const float* cum_in,
                   const int64_t* tok_in, int32_t eos, int64_t* tokens, int32_t* parents, float* cum_out,
                   float* logprobs, void* stream);

/* The K most likely continuations of B prompts by n_new tokens, without leaving the device (no host synchronisation):
 *   prefill  eval-mode forward of prompt [T0,B] int64 from `in` (B rows) as zrb_generate, last step projected
 *   step k   zrb_beam_step on those scores (step 0: B rows, S = 0), then row b*K + k takes its parent's (h, c) of every
 *            layer; unless k = n_new - 1, a T = 1 eval forward of the B*K new tokens
 *   tokens [n_new,B,K] int64, logprobs [n_new,B,K] fp32 (or NULL): the hypothesis in final slot k, traced back through
 *   the parents (eos and 0 after an eos); scores [B,K] fp32 (or NULL): its S, the float32 sum of its logprobs in order.
 * `out` (B*K rows) holds the states BEFORE each hypothesis's last token is consumed; in / out may alias.  Pending lazy
 * weight updates are applied first; no dropout; nothing is kept for zrb_backward.  Both engines, any T0.
 * ZRB_E_INVALID as zrb_beam_step, and for B*K above the context's max_batch, n_new < 1, T0 < 1. */
int  zrb_beam_search(zrb_ctx* ctx, const zrb_params* p, const int64_t* prompt, int32_t T0, int32_t B,
                     const zrb_states* in, const zrb_states* out, int32_t n_new, int32_t K, int32_t eos,
                     int64_t* tokens, float* logprobs, float* scores, void* stream);

/* ---- neural-cache evaluation (Grave, Joulin & Usunier, "Improving Neural Language Models with a Continuous Cache",
 * ICLR 2017; DESIGN.md section 12 states it bit for bit) ---------------------------------------------------------
 * Per stream b (batch row) the cache holds pairs (k_i, y_i), i the stream's position (tokens fed since the last
 * reset, counted across calls): k_i = half_rn(h_i), the last layer's output at i, and y_i the target at i.  A query at
 * position t with target y_t, cache size W, temperature theta >= 0 and weight lambda in [0, 1):
 *   C_t = { i : max(0, t - W) <= i < t }   (earlier calls and earlier rows of this window; never t itself)
 *   s_i = theta * <half(h_t), k_i>,  p_cache = sum_{i in C_t, y_i = y_t} exp(s_i - m) / sum_{i in C_t} exp(s_i - m)
 *   p = (1 - lambda) p_model + lambda p_cache, row loss = -logaddexp(log(1 - lambda) - r, log(lambda) + log(p_cache))
 *   with r = -log p_model the eval step's row loss; C_t empty (a stream's first token): p = p_model, p_cache = 0.
 * The window loss reduces the row losses as zrb_eval_step does (summed over the batch, averaged over time); lambda = 0
 * gives zrb_eval_step's loss bit for bit.  The handle is independent of any context; its position counter lives on the
 * host (no synchronisation) and a reset only zeroes it.  hidden <= 1536 (the query tile stays in shared memory).
 * ZRB_E_INVALID for hidden outside [1, 1536], batch, size or max_seq < 1. */
typedef struct zrb_cache zrb_cache;   /* opaque */
int  zrb_cache_create(int32_t hidden, int32_t batch, int32_t size, int32_t max_seq, zrb_cache** out);
int  zrb_cache_reset(zrb_cache* cache);
void zrb_cache_destroy(zrb_cache* cache);
/* The unit on its own, with no model: append h [T,B,H] fp32 (rounded to fp16) and targets y [T,B] int64 to the cache,
 * then cache_prob [T*B] fp32 = p_cache of every row.  ZRB_E_INVALID (handle unchanged) for theta < 0 or not finite,
 * B other than the cache's, T outside [1, max_seq], and a current device other than the one the cache was created on. */
int  zrb_cache_step(zrb_cache* cache, const float* h, const int64_t* y, int32_t T, int32_t B, float theta,
                    float* cache_prob, void* stream);
/* zrb_eval_step with the cache: the same eval-mode forward (pending lazy updates applied first, no dropout) and row
 * losses, then the window's last-layer outputs and targets are appended to the cache and every row attends over it.
 * loss: the window loss of the mixed p; tgt_prob [T*B] (or NULL): p_model, zrb_eval_step's tgt_prob; cache_prob [T*B]
 * (or NULL): p_cache.  With both, a caller can sweep lambda on the host.  Two launches more than zrb_eval_step (append,
 * attend and combine; the combine does the loss reduction).
 * ZRB_E_INVALID (handle unchanged) as zrb_cache_step, for lambda outside [0, 1), and for an H other than the cache's. */
int  zrb_eval_step_cache(zrb_ctx* ctx, const zrb_params* p, const int64_t* x, const int64_t* y, int32_t T, int32_t B,
                         const zrb_states* in, const zrb_states* out, zrb_cache* cache, float theta, float lambda,
                         float* loss, float* tgt_prob, float* cache_prob, void* stream);

/* ---- dynamic evaluation (Krause, Kahembwe, Murray & Renals, "Dynamic Evaluation of Neural Sequence Models", ICML 2018;
 * DESIGN.md section 14 states it bit for bit) --------------------------------------------------------------------------
 * theta = the P distinct parameter elements (a tied E once), theta_g = `global`, a snapshot taken when the pass starts.
 * Per window s ([T,B], states carried as in perplexity):
 *   1. score: the eval-mode forward at theta_s (no dropout, whatever the context's dropout / variational / explicit-mask
 *      settings); loss = zrb_eval_step's window loss, bit for bit.
 *   2. gradient: g_s = d loss / d theta of that same eval-mode function, entering states detached -- bit for bit what
 *      zrb_train_step_grads writes in a context created with dropout = 0 from the same weights, window and states.
 *   3. update: theta += a * (theta_g - theta) - lr * u, elementwise, in the fp32 order of DESIGN.md section 14:
 *        RMS rule (rms given):  u = g / (r + eps), a = min(1, lambda * r / rbar)
 *        SGD rule (rms NULL):   u = g,             a = min(1, lambda)
 *      r = the RMS statistic, rbar = *rms_mean (device), the mean of r over all P elements.  An element with r = 0 gets
 *      a = 0 and u = g / eps.  The clip of a at 1 (a parameter never moves past theta_g) is this library's choice.
 * Statistics: MS = (1/K) sum_k g_k^2 over K windows, each g_k as in step 2 at theta_g with no update, states carried from
 * zero.  zrb_grad_stats_step: the window's g into `grads` and ms += g*g (fp32, one fma; p unchanged).
 * zrb_grad_stats_finish: r = sqrtf(ms / K) in place and *rms_mean = fp32(fixed-order fp64 sum of r / P): bit-reproducible.
 * zrb_dyneval_step: steps 1-3 in one call; afterwards `grads` holds the raw g_s and the fp16 weight images are current.
 * All zrb_params of a tied context must have fc_w == embed_w; loss may be NULL.  Pending lazy updates are applied first.
 * ZRB_E_INVALID, before anything is launched and with every buffer unchanged, for lr or lambda negative or not finite,
 * eps <= 0 or not finite under the RMS rule, rms_mean NULL with rms given, windows < 1, and the tied rule. */
int  zrb_grad_stats_step(zrb_ctx* ctx, const zrb_params* p, const zrb_params* grads, const zrb_params* ms,
                         const int64_t* x, const int64_t* y, int32_t T, int32_t B, const zrb_states* in,
                         const zrb_states* out, float* loss, void* stream);
int  zrb_grad_stats_finish(zrb_ctx* ctx, const zrb_params* ms, int64_t windows, float* rms_mean, void* stream);
int  zrb_dyneval_step(zrb_ctx* ctx, const zrb_params* p, const zrb_params* grads, const zrb_params* global,
                      const zrb_params* rms, const float* rms_mean, const int64_t* x, const int64_t* y, int32_t T,
                      int32_t B, const zrb_states* in, const zrb_states* out, float lr, float lambda, float eps,
                      float* loss, void* stream);

/* Same as zrb_train_step_grads + zrb_train_step_update but with HOST token buffers
 * (pinned or pageable) and a host loss: the H2D copies of x, y and the D2H copy of the
 * loss are issued on `stream` inside the call; the call returns after the loss landed. */
int  zrb_train_step_host(zrb_ctx* ctx, const zrb_params* p, const zrb_params* grads,
                         const int64_t* h_x, const int64_t* h_y, int32_t T, int32_t B,
                         const zrb_states* in, const zrb_states* out,
                         uint64_t seed, uint64_t step, float lr, float max_norm,
                         float* h_loss, float* h_norm, void* stream);

/* Per-kernel-class timing with CUDA events recorded on the launching stream (bench.py's
 * `roofline` leg).  While enabled, every kernel class below is bracketed by an event pair.
 * zrb_prof_read synchronises, writes total milliseconds and launch-group counts per class
 * (arrays of ZRB_PROF_COUNT) and resets the accumulators. */
#define ZRB_PROF_EMBED_FWD    0   /* embedding gather + dropout                       */
#define ZRB_PROF_GEMM_IN      1   /* input-to-hidden GEMM  X * W_ih^T (all T at once)  */
#define ZRB_PROF_REC_FWD      2   /* recurrence over T: h * W_hh^T + cell pointwise    */
#define ZRB_PROF_PROJ_FWD     3   /* vocabulary projection                             */
#define ZRB_PROF_SOFTMAX      4   /* softmax-NLL fwd+bwd                               */
#define ZRB_PROF_PROJ_BWD     5   /* projection dgrad + wgrad + bias grad              */
#define ZRB_PROF_REC_BWD      6   /* reverse recurrence: cell bwd + dG * W_hh          */
#define ZRB_PROF_GEMM_DX      7   /* dG * W_ih                                         */
#define ZRB_PROF_GEMM_WGRAD   8   /* dW_ih, dW_hh, bias grads                          */
#define ZRB_PROF_EMBED_BWD    9   /* embedding scatter-add                             */
#define ZRB_PROF_CLIP_SGD    10   /* grad norm + clip + SGD (+ weight image refresh)   */
#define ZRB_PROF_PACK        11   /* low-precision weight image build                  */
#define ZRB_PROF_COUNT       12
int  zrb_prof_enable(zrb_ctx* ctx, int32_t on);
int  zrb_prof_read(zrb_ctx* ctx, float* h_ms, int64_t* h_counts);
/* Phase timeline of the persistent recurrence kernels (clock64 stamps of CTA 0, 8 per step:
 * grid barrier seen, MMA chain start, accumulators out, accumulators seen by the cell warps, partial sums landed,
 * cell math done, before / after the arrival; tools/rec_trace.py), preceded per kernel by 8 launch slots: CTA 0's clock64 at kernel entry / exit, its %globaltimer (ns)
 * at entry / exit, -(earliest CTA entry ns), latest CTA exit ns, 2 spare.  Needs ZRB_REC_TRACE=1 in the environment
 * at context creation.  Returns the number of entries written ([fwd|bwd][8 + T*8]) or a negative error. */
int  zrb_prof_rec_trace(zrb_ctx* ctx, int64_t* h_out, int32_t max_entries);

/* ---- building blocks, exported for unit tests and profiling ------------------------ */

/* ONE recurrent layer over the window through the persistent recurrence kernels alone (model.py:48-55, the nn.LSTM(H,H)
 * call of model.py:107; SURVEY 8b's zrb_lstm_layer_fwd / _bwd): input GEMM + weight-stationary recurrence, no dropout
 * (the caller applies it, as model.py:105,108 do).  Tensor-core engine only, shapes the persistent kernels accept
 * (B <= 32).  Gate row blocks (i, f, g, o).
 *   x [T*B,H] fp32 layer input; h0, c0 [B,H]; y [T*B,H] fp32 = h_t; hT, cT [B,H] final state (may be NULL)
 * The activations stay in the context for zrb_lstm_layer_bwd:
 *   dy [T*B,H] = d loss / d y (no gradient flows into hT / cT: the reference detaches the carried state, main.py:110)
 *   dx [T*B,H] (or NULL), dw_ih, dw_hh [4H,H], db_ih, db_hh [4H] : OVERWRITTEN
 * These calls borrow the context's layer-0 workspace: model-level weight images are rebuilt at the next model-level call. */
int  zrb_lstm_layer_fwd(zrb_ctx* ctx, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                        const float* x, int32_t T, int32_t B, const float* h0, const float* c0, float* y, float* hT,
                        float* cT, void* stream);
int  zrb_lstm_layer_bwd(zrb_ctx* ctx, const float* dy, float* dx, float* dw_ih, float* dw_hh, float* db_ih,
                        float* db_hh, void* stream);


/* C[M,N] = alpha * A[M,K] * op(B) + beta * C  in fp32 on CUDA cores.
 * transB != 0: B is [N,K] (C = A * B^T);  transB == 0: B is [K,N].
 * transA != 0: A is stored [K,M]. */
int  zrb_gemm_f32(const float* A, const float* B, float* C, int32_t M, int32_t N, int32_t K,
                  int32_t transA, int32_t transB, float alpha, float beta, void* stream);

/* C[M,N] (fp32) = alpha * A * B^T (+ bias[N]) (+ C if accumulate) on wgmma tensor cores,
 * fp16 operands, fp32 accumulation.  a_mn_major == 0: A is [M,K] with K contiguous (pitch lda);
 * != 0: A is stored [K,M] with M contiguous (pitch lda).  Same for B with N.  Pitches are in
 * elements and must be multiples of 8 (16 bytes); bases 16-byte aligned. */
int  zrb_gemm_f16(const void* A, int64_t lda, int32_t a_mn_major, const void* B, int64_t ldb,
                  int32_t b_mn_major, float* C, int64_t ldc, int32_t M, int32_t N, int32_t K,
                  float alpha, const float* bias, int32_t accumulate, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ZAREMBA_B200_H */
