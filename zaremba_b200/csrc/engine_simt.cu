// ZRB_ENGINE_SIMT: the path in fp32 on CUDA cores, one GEMM + one pointwise launch per
// timestep.  Slow by construction; it exists to validate every other piece (ABI, dropout
// replay, loss, optimiser, autograd glue) and as the on-device fp32 yardstick for the
// tensor-core engine.
#include "engine.h"

namespace zrb {

int simt_forward(zrb_ctx* c, const zrb_params* p, const int64_t* x, const zrb_states* in, const zrb_states* out,
                 float* scores, cudaStream_t s, bool last_only) {
    const int H = c->cfg.hidden, L = c->cfg.layers, V = c->cfg.vocab, T = c->T, B = c->B, N = T * B;
    const size_t bh = (size_t)B * H * sizeof(float);
    ZRB_CUDA(cudaMemcpyAsync(c->x_saved, x, (size_t)N * sizeof(int64_t), cudaMemcpyDeviceToDevice, s));
    for (int l = 0; l < L; ++l) {  // `in` may alias `out`: snapshot first (also needed by backward)
        ZRB_CUDA(cudaMemcpyAsync(c->h0s[l], in->h[l], bh, cudaMemcpyDeviceToDevice, s));
        ZRB_CUDA(cudaMemcpyAsync(c->c0s[l], in->c[l], bh, cudaMemcpyDeviceToDevice, s));
    }
    // model.py:104-105
    {
        ProfScope ps(c, ZRB_PROF_EMBED_FWD, s);
        ZRB_TRY(embed_dropout_fwd(p->embed_w, x, c->act[0], nullptr, 0, N, H, V, site_mask(c, 0), ed_mask(c), s));
    }
    for (int l = 0; l < L; ++l) {  // model.py:106-108
        float* G = c->gates[l];
        {
            ProfScope ps(c, ZRB_PROF_GEMM_IN, s);
            ZRB_TRY(gemm_f32(c->act[l], p->w_ih[l], G, N, 4 * H, H, 0, 1, 1.f, 0.f, s));
            ZRB_TRY(add_bias2(G, p->b_ih[l], p->b_hh[l], N, 4 * H, s));
        }
        MaskSrc m = site_mask(c, l + 1), rm = rec_mask(c, l), wm = wd_mask(c, l);
        ProfScope ps(c, ZRB_PROF_REC_FWD, s);
        // variational mode: the recurrent operand is hrec (block t = h_{t-1} * mask), also read by the dW_hh GEMM
        float* hrec = rm.active ? c->hrec[l] : nullptr;
        if (hrec) ZRB_TRY(dropout_copy(c->h0s[l], hrec, (int64_t)B * H, rm, s));
        // weight drop: the recurrent matrix is whh_wd = fp32(W_hh * mask * scale), also read by the backward
        const float* w_hh = wm.active ? c->whh_wd[l] : p->w_hh[l];
        if (wm.active) ZRB_TRY(weight_drop(p->w_hh[l], c->whh_wd[l], (int64_t)4 * H * H, wm, nullptr, s));
        for (int t = 0; t < T; ++t) {
            const float* h_prev = hrec ? hrec + (size_t)t * B * H : t ? c->hraw[l] + (size_t)(t - 1) * B * H : c->h0s[l];
            const float* c_prev = t ? c->cst[l] + (size_t)(t - 1) * B * H : c->c0s[l];
            float* Gt = G + (size_t)t * B * 4 * H;
            ZRB_TRY(gemm_f32(h_prev, w_hh, Gt, B, 4 * H, H, 0, 1, 1.f, 1.f, s));
            ZRB_TRY(lstm_cell_fwd(Gt, c_prev, c->cst[l] + (size_t)t * B * H, c->hraw[l] + (size_t)t * B * H,
                                  c->act[l + 1] + (size_t)t * B * H, hrec ? hrec + (size_t)(t + 1) * B * H : nullptr, B, H,
                                  (int64_t)t * B * H, (int64_t)N * H, m, rm, s));
        }
        ZRB_CUDA(cudaMemcpyAsync(out->h[l], c->hraw[l] + (size_t)(T - 1) * B * H, bh, cudaMemcpyDeviceToDevice, s));
        ZRB_CUDA(cudaMemcpyAsync(out->c[l], c->cst[l] + (size_t)(T - 1) * B * H, bh, cudaMemcpyDeviceToDevice, s));
    }
    if (scores) {  // model.py:109
        ProfScope ps(c, ZRB_PROF_PROJ_FWD, s);
        const int rows = last_only ? B : N;
        ZRB_TRY(gemm_f32(c->act[L] + (size_t)(N - rows) * H, p->fc_w, scores, rows, V, H, 0, 1, 1.f, 0.f, s));
        ZRB_TRY(add_bias1(scores, p->fc_b, rows, V, s));
    }
    return ZRB_OK;
}

int simt_backward(zrb_ctx* c, const zrb_params* p, const float* dscores, const zrb_params* g, cudaStream_t s) {
    const int H = c->cfg.hidden, L = c->cfg.layers, V = c->cfg.vocab, T = c->T, B = c->B, N = T * B;
    const size_t bh = (size_t)B * H;
    // fc: dA = dS * W ; dW = dS^T * A ; db = colsum(dS)
    float* dY = c->dy;
    float* dX = c->dx;
    {
        ProfScope ps(c, ZRB_PROF_PROJ_BWD, s);
        ZRB_TRY(gemm_f32(dscores, p->fc_w, dY, N, H, V, 0, 0, 1.f, 0.f, s));
        ZRB_TRY(gemm_f32(dscores, c->act[L], g->fc_w, V, H, N, 1, 0, 1.f, 0.f, s));
        ZRB_TRY(colsum(dscores, g->fc_b, nullptr, N, V, s));
    }
    for (int l = L - 1; l >= 0; --l) {
        MaskSrc m = site_mask(c, l + 1), rm = rec_mask(c, l), wm = wd_mask(c, l);
        const float* w_hh = wm.active ? c->whh_wd[l] : p->w_hh[l];
        const float* r = (c->reg_use && l == L - 1) ? c->reg_r : nullptr;   // AR / TAR gradient (DESIGN.md section 17)
        ZRB_CUDA(cudaMemsetAsync(c->dc, 0, bh * sizeof(float), s));
        {
        ProfScope ps(c, ZRB_PROF_REC_BWD, s);
        for (int t = T - 1; t >= 0; --t) {
            const float* c_prev = t ? c->cst[l] + (size_t)(t - 1) * bh : c->c0s[l];
            float* dGt = c->dG + (size_t)t * B * 4 * H;
            ZRB_TRY(lstm_cell_bwd(dY + (size_t)t * bh, t == T - 1 ? nullptr : c->dh_rec, c->dc,
                                  c->gates[l] + (size_t)t * B * 4 * H, c->cst[l] + (size_t)t * bh, c_prev, dGt, B, H,
                                  (int64_t)t * bh, (int64_t)N * H, m, rm, s, r ? r + (size_t)t * bh : nullptr));
            if (t > 0) ZRB_TRY(gemm_f32(dGt, w_hh, c->dh_rec, B, H, 4 * H, 0, 0, 1.f, 0.f, s));
        }
        }
        {
            ProfScope ps(c, ZRB_PROF_GEMM_DX, s);
            ZRB_TRY(gemm_f32(c->dG, p->w_ih[l], dX, N, H, 4 * H, 0, 0, 1.f, 0.f, s));
        }
        ProfScope ps(c, ZRB_PROF_GEMM_WGRAD, s);
        ZRB_TRY(gemm_f32(c->dG, c->act[l], g->w_ih[l], 4 * H, H, N, 1, 0, 1.f, 0.f, s));
        // dW_hh = sum_t dG_t^T h_{t-1}: t = 0 pairs with the entering state, t >= 1 with hraw[t-1]; in the
        // variational mode the masked operands hrec, one GEMM over all N rows
        if (rm.active) {
            ZRB_TRY(gemm_f32(c->dG, c->hrec[l], g->w_hh[l], 4 * H, H, N, 1, 0, 1.f, 0.f, s));
        } else {
            ZRB_TRY(gemm_f32(c->dG, c->h0s[l], g->w_hh[l], 4 * H, H, B, 1, 0, 1.f, 0.f, s));
        }
        if (T > 1 && !rm.active)
            ZRB_TRY(gemm_f32(c->dG + (size_t)B * 4 * H, c->hraw[l], g->w_hh[l], 4 * H, H, N - B, 1, 0, 1.f, 1.f, s));
        if (wm.active) ZRB_TRY(weight_drop(g->w_hh[l], g->w_hh[l], (int64_t)4 * H * H, wm, nullptr, s));   // scale * m * dW_eff
        ZRB_TRY(colsum(c->dG, g->b_ih[l], g->b_hh[l], N, 4 * H, s));
        float* tmp = dY; dY = dX; dX = tmp;
    }
    ProfScope ps(c, ZRB_PROF_EMBED_BWD, s);
    const MaskSrc m0 = site_mask(c, 0), em = ed_mask(c);
    if (c->embed_rows_out) return embed_rows(dY, c->x_saved, c->embed_rows_out, N, H, V, m0, em, s);
    if (c->tied) {   // g->embed_w holds G_proj: add the row sums (the tensor-core engine's fixed-point merge)
        ZRB_TRY(embed_rows(dY, c->x_saved, dX, N, H, V, m0, em, s));
        return embed_scatter_rows(c->x_saved, dX, g->embed_w, N, H, V, c->emb_first, c->emb_acc, s, true);
    }
    ZRB_CUDA(cudaMemsetAsync(g->embed_w, 0, (size_t)V * H * sizeof(float), s));
    ZRB_TRY(embed_dropout_bwd(dY, c->x_saved, g->embed_w, N, H, V, m0, em, s));
    return ZRB_OK;
}

}  // namespace zrb
