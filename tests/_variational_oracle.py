"""Numpy restatement of the variational dropout mode (DESIGN.md section 11)  --  TEST INFRASTRUCTURE ONLY.

Extends `oracle.lstm_lm_oracle` (whose functions it reuses unchanged) by the recurrent masks of Gal & Ghahramani
(2016), and `oracle.philox` by the masks of the mode:
  - sites 0..L: the mask of time step 0 (elements b*H + j of the site's stream) reused at every t, i.e. a tiled
    [T, B, H] mask, which the oracle's `model_fwd` already accepts;
  - recurrent site L + 1 + l with p_rec: the operand multiplying W_hh at every step t (t = 0 included) is
    m_l * h_{t-1} / (1 - p_rec); the layer's output, the carried (h, c) and c are not masked.
With `rmasks=None` every function here computes exactly what the oracle computes.
"""
from __future__ import annotations

import numpy as np

from oracle import lstm_lm_oracle as O
from oracle import philox as PH


# ---- masks --------------------------------------------------------------------------------------------------------
def variational_masks(seed, step, L, T, B, H, p, p_rec):
    """(site masks: L + 1 bool [T, B, H], the step-0 mask of each site tiled over T;
        recurrent masks: L bool [B, H] of sites L + 1 + l with p_rec, or None when p_rec == 0)."""
    sites = [np.broadcast_to(PH.keep_mask(seed, step, s, B * H, p).reshape(1, B, H), (T, B, H)).copy()
             for s in range(L + 1)]
    rec = None
    if float(np.float32(p_rec)) > 0.0:
        rec = [PH.keep_mask(seed, step, L + 1 + l, B * H, p_rec).reshape(B, H) for l in range(L)]
    return sites, rec


def _rec_op(h, rmask, p_rec):
    """m * h / (1 - p_rec), or h when there is no recurrent mask."""
    return h if rmask is None else O.apply_dropout(h, rmask, p_rec)


# ---- one layer ----------------------------------------------------------------------------------------------------
def lstm_layer_fwd(x, h0, c0, W_ih, W_hh, b_ih, b_hh, rmask=None, p_rec=0.0):
    """O.lstm_layer_fwd with the recurrent operand m * h_{t-1} * scale(p_rec).  The cache keeps that operand."""
    T = x.shape[0]
    h, c = h0, c0
    ys, cache = [], []
    for t in range(T):
        h_op, c_prev = _rec_op(h, rmask, p_rec), c
        h, c, (i, f, g, o) = O.lstm_cell_fwd(x[t], h_op, c, W_ih, W_hh, b_ih, b_hh)
        ys.append(h)
        cache.append((h_op, c_prev, i, f, g, o, c))
    return np.stack(ys), h, c, cache


def lstm_layer_bwd(dy, cache, x, W_ih, W_hh, rmask=None, p_rec=0.0):
    """O.lstm_layer_bwd with dh_{t-1} += scale * m * (dG_t W_hh); dW_hh pairs dG_t with the masked operand."""
    T, B, H = dy.shape
    dt = dy.dtype
    dW_ih = np.zeros_like(W_ih)
    dW_hh = np.zeros_like(W_hh)
    db = np.zeros(4 * H, dtype=dt)
    dx = np.zeros_like(x)
    dh_rec = np.zeros((B, H), dtype=dt)
    dc = np.zeros((B, H), dtype=dt)
    for t in range(T - 1, -1, -1):
        h_op, c_prev, i, f, g, o, c = cache[t]
        dh = dy[t] + dh_rec
        tc = np.tanh(c)
        do = dh * tc
        dc = dc + dh * o * (1.0 - tc * tc)
        dG = np.concatenate([dc * g * i * (1.0 - i), dc * c_prev * f * (1.0 - f),
                             dc * i * (1.0 - g * g), do * o * (1.0 - o)], axis=1)
        dc = dc * f
        dx[t] = dG @ W_ih
        dh_rec = _rec_op(dG @ W_hh, rmask, p_rec)
        dW_ih += dG.T @ x[t]
        dW_hh += dG.T @ h_op
        db += dG.sum(axis=0)
    return dx, dW_ih, dW_hh, db


# ---- the model ----------------------------------------------------------------------------------------------------
def model_fwd(params, x, states, layer_num, dropout=0.0, masks=None, rmasks=None, p_rec=0.0):
    """O.model_fwd plus per-layer recurrent masks `rmasks` (list of L bool [B, H], or None)."""
    dt = params["embed.W"].dtype
    a = O.apply_dropout(O.embed_fwd(params["embed.W"], x), None if masks is None else masks[0], dropout)
    new_states, layer_cache, layer_in = [], [], []
    for l in range(layer_num):
        layer_in.append(a)
        h0, c0 = states[l]
        y, h, c, cache = lstm_layer_fwd(
            a, h0.astype(dt), c0.astype(dt),
            params[f"rnns.{l}.weight_ih_l0"], params[f"rnns.{l}.weight_hh_l0"],
            params[f"rnns.{l}.bias_ih_l0"], params[f"rnns.{l}.bias_hh_l0"],
            None if rmasks is None else rmasks[l], p_rec)
        new_states.append((h, c))
        layer_cache.append(cache)
        a = O.apply_dropout(y, None if masks is None else masks[l + 1], dropout)
    scores = O.linear_fwd(a, params["fc.W"], params["fc.b"])
    cache = {"x": np.asarray(x), "layer_in": layer_in, "layer_cache": layer_cache, "fc_in": a, "masks": masks,
             "dropout": dropout, "rmasks": rmasks, "p_rec": p_rec}
    return scores, new_states, cache


def model_bwd(params, cache, dscores, layer_num):
    p, masks, rmasks, p_rec = cache["dropout"], cache["masks"], cache["rmasks"], cache["p_rec"]
    fc_in = cache["fc_in"]
    T, B, H = fc_in.shape
    grads = {"fc.W": dscores.T @ fc_in.reshape(-1, H), "fc.b": dscores.sum(axis=0)}
    da = (dscores @ params["fc.W"]).reshape(T, B, H)
    for l in range(layer_num - 1, -1, -1):
        da = O.apply_dropout(da, None if masks is None else masks[l + 1], p)
        dx, dWi, dWh, db = lstm_layer_bwd(da, cache["layer_cache"][l], cache["layer_in"][l],
                                          params[f"rnns.{l}.weight_ih_l0"], params[f"rnns.{l}.weight_hh_l0"],
                                          None if rmasks is None else rmasks[l], p_rec)
        grads[f"rnns.{l}.weight_ih_l0"] = dWi
        grads[f"rnns.{l}.weight_hh_l0"] = dWh
        grads[f"rnns.{l}.bias_ih_l0"] = db
        grads[f"rnns.{l}.bias_hh_l0"] = db.copy()
        da = dx
    da = O.apply_dropout(da, None if masks is None else masks[0], p)
    dE = np.zeros_like(params["embed.W"])
    np.add.at(dE, cache["x"].reshape(-1), da.reshape(-1, H))
    grads["embed.W"] = dE
    return grads


def train_step(params, x, y, states, layer_num, lr, max_norm, dropout=0.0, masks=None, rmasks=None, p_rec=0.0):
    """O.train_step with recurrent masks: forward, loss, backward, clip + SGD (in place)."""
    scores, new_states, cache = model_fwd(params, x, states, layer_num, dropout, masks, rmasks, p_rec)
    loss = O.nll_loss(scores, y)
    grads = model_bwd(params, cache, O.nll_loss_bwd(scores, y), layer_num)
    norm = O.clip_sgd(params, grads, lr, max_norm, O.param_names(layer_num))
    return loss, norm, new_states, scores, grads
