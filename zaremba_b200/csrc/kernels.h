// Internal launcher declarations (host side).  All take a cudaStream_t and return ZRB_*.
#pragma once
#include "common.cuh"

namespace zrb {

// ---- pointwise.cu -----------------------------------------------------------------------
// out[n, :] = W[idx[n], :] * dropout   (model.py:13-14 + :105)
// pend_g (or null): gather sgd_elem(W, scalars[1] * pend_g, lr), W's deferred update (tied embedding, lazy update)
int embed_dropout_fwd(const float* W, const int64_t* idx, float* out, __half* out_h, int64_t ld_h,
                      int N, int H, int V, MaskSrc m, cudaStream_t s, const float* pend_g = nullptr, float lr = 0.f,
                      const float* scalars = nullptr);
// dW[idx[n], :] += dA[n, :] * dropout   (dW pre-zeroed)
int embed_dropout_bwd(const float* dA, const int64_t* idx, float* dW, int N, int H, int V, MaskSrc m,
                      cudaStream_t s);
// pre [B,4H] holds x-part + h-part pre-activations (+bias already added); overwritten with
// activated gates (i,f,g,o).  c_prev/c_out/h_raw/y_out [B,H]; y_out = dropout(h).
// h_rec [B,H] (or null): h * the recurrent mask rm of element b*H + j (variational mode: the next step's operand)
int lstm_cell_fwd(float* pre, const float* c_prev, float* c_out, float* h_raw, float* y_out, float* h_rec,
                  int B, int H, int64_t elem_off, int64_t n_total, MaskSrc m, MaskSrc rm, cudaStream_t s);
// dG [B,4H] out; dc [B,H] in/out carry; dh_rec [B,H] in (may be null = 0), multiplied by the recurrent mask rm;
// dy_post [B,H] upstream grad on the post-dropout output
int lstm_cell_bwd(const float* dy_post, const float* dh_rec, float* dc, const float* gates, const float* c_t,
                  const float* c_prev, float* dG, int B, int H, int64_t elem_off, int64_t n_total, MaskSrc m,
                  MaskSrc rm, cudaStream_t s);
// y[e] = x[e] * (mask multiplier of element e), e < n
int dropout_copy(const float* x, float* y, int64_t n, MaskSrc m, cudaStream_t s);
// C[n, j] += bias1[j] + bias2[j]
int add_bias2(float* C, const float* b1, const float* b2, int N, int M, cudaStream_t s);
int add_bias1(float* C, const float* b1, int N, int M, cudaStream_t s);
// out[j] = sum_n A[n, j]
int colsum(const float* A, float* out, float* out2, int N, int M, cudaStream_t s);
// softmax NLL fwd(+bwd); row_loss [N] scratch
// optional ds_h: scaled fp16 image of the gradient (pitch ld_s) for the tensor-core engine
int softmax_nll(const float* scores, const int64_t* y, int N, int V, int B, float* row_loss, float* loss,
                float* dscores, float* tgt_prob, cudaStream_t s, __half* ds_h = nullptr, int64_t ld_s = 0,
                float h_scale = 1.f);
int embed_rows(const float* dA, float* rows, int N, int H, MaskSrc m, cudaStream_t s);
// add: dW[id] += the id's sum instead of dW[id] = (tied embedding); sumsq: see embed_finish_add_kernel
int embed_scatter_rows(const int64_t* ids, const float* rows, float* dW, int n_rows, int H, int V, int* first,
                       long long* acc, cudaStream_t s, bool add = false, float* sumsq = nullptr, int nblocks = 0);
int embed_zero_rows(float* dW, const int64_t* ids, int n, int H, int V, cudaStream_t s);
int embed_first_table(const int64_t* ids, int* first, int n, int V, cudaStream_t s);
int embed_rows_sumsq(const float* dW, const int64_t* ids, const int* first, int n, int H, int V, float* partial,
                     int nblocks, cudaStream_t s);
int embed_rows_update(float* W, float* dW, const int64_t* ids, const int* first, int n, int H, int V, float lr,
                      const float* scalars, bool write_g, cudaStream_t s);
int dropout_mask_bytes(MaskSrc m, int64_t n, uint8_t* out, cudaStream_t s);

// ---- optim.cu ----------------------------------------------------------------------------
struct TensorList {
    float* p[16];
    float* g[16];
    int64_t n[16];
    int count;
};
// partials: >= 1024 floats scratch; scalars: >= 4 floats (norm, coef)
constexpr int kNormGemm = 16384;  // then: per-(tile, epilogue warp) sums of squares written by the wgrad GEMMs (tensor-core engine)
constexpr int kNormExtra = 1024;   // extra partial slots after the kNormBlocks ones (embedding rows' sum of squares)
int norm_partials_base();        // index of the first extra slot
// extra_used: the caller filled partials[norm_partials_base() .. +kNormExtra) itself (else they are zeroed here)
// n_gemm: that many slots after the extra ones hold sums of squares of tensors NOT in `tl` (gemm_f16_tc sumsq_out)
int grad_norm(const TensorList& tl, float max_norm, float* partials, float* scalars, float* norm_out,
              cudaStream_t s, bool extra_used = false, int n_gemm = 0);
// write_g: store coef * g back (clip_grad_norm_ scales .grad in place); false leaves the raw gradient
int sgd_apply(const TensorList& tl, float lr, const float* scalars, bool write_g, cudaStream_t s);
int clip_sgd(const TensorList& tl, float lr, float max_norm, float* partials, float* scalars, float* norm_out,
             bool write_g, cudaStream_t s);
// Dynamic evaluation (DESIGN.md section 14) over tensors with no fp16 image: tl.p / tl.g as above, tg / r the same
// tensors of theta_g and of the RMS statistic (r ignored under the SGD rule, a.rbar null).  Zero-length entries are skipped.
int dyneval_apply(const TensorList& tl, float* const* tg, float* const* r, const DynArgs& a, cudaStream_t s);
// ms += g * g (one fma per element) over the list: tl.p = ms, tl.g = the window's gradient
int sq_accumulate(const TensorList& tl, cudaStream_t s);
// r = sqrt(ms / windows) in place over the list (tl.p), and rbar = fp32(fixed-order fp64 sum of r / P): one partial per
// block in `partials` (>= kStatsPartials doubles), then one final reduce.  Bit-reproducible run to run.
constexpr int kStatsPartials = 2048;
int stats_finish(const TensorList& tl, int64_t windows, double* partials, float* rbar, cudaStream_t s);

// ---- sample.cu ---------------------------------------------------------------------------
// ZRB_E_INVALID for the arguments zrb_sample rejects (checked before anything is enqueued)
int sample_check(const zrb_sampling* cfg, int B, int V);
// tokens[b] (and logprobs[b]) from row b of scores [B, ld]: one CTA per row
int sample_rows(const float* scores, int64_t ld, int B, int V, const zrb_sampling* cfg, uint64_t pos, int64_t* tokens,
                float* logprobs, cudaStream_t s);

// ---- beam.cu -----------------------------------------------------------------------------
// one candidate of a beam step: cand = S + logp, flat = i*V + j (slot i of the previous step, token j)
struct BeamCand {
    float cand, logp;
    uint32_t flat;
};
// ZRB_E_INVALID for the arguments zrb_beam_step / zrb_beam_search reject (B, beam width K, vocabulary V, eos)
int beam_check(int B, int K, int V, int eos);
// One selection step (DESIGN.md section 10) over B prompts of K_in rows of scores [B*K_in, ld]: cum_in [B*K_in] (NULL:
// all 0), tok_in [B*K_in] (NULL: no row finished); outputs [B*K].  cands: B*K_in*K entries of scratch.  With L > 0 the
// (h, c) rows of every layer are gathered from src (row b*K_in + parent) to dst (row b*K + k); src and dst must not
// alias.  Two launches.
int beam_step(const float* scores, int64_t ld, int B, int K_in, int K, int V, const float* cum_in, const int64_t* tok_in,
              int eos, BeamCand* cands, int64_t* tokens, int32_t* parents, float* cum_out, float* logprobs,
              const zrb_states* src, const zrb_states* dst, int L, int H, cudaStream_t s);
// per-step [n_new, BK] tokens / parents / logprobs -> the hypotheses [n_new, B, K] of each final slot; scores = cum
int beam_backtrack(const int64_t* step_tok, const int32_t* step_par, const float* step_lp, const float* cum, int n_new,
                   int BK, int K, int64_t* tokens, float* logprobs, float* scores, cudaStream_t s);

// ---- gemm_simt.cu ------------------------------------------------------------------------
int gemm_f32(const float* A, const float* B, float* C, int M, int N, int K, int transA, int transB, float alpha,
             float beta, cudaStream_t s);

}  // namespace zrb
