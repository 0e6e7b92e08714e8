"""Numpy restatement of embedding dropout and AR/TAR (DESIGN.md section 17)  --  TEST INFRASTRUCTURE ONLY.

Extends `tests._weight_drop_oracle` (and through it the variational restatement and `oracle.lstm_lm_oracle`, reused
unchanged) by AWD-LSTM's embedding dropout (Merity, Keskar & Socher 2018), with the mask of `oracle.philox`:
  - the keep flag of vocabulary row v is element v of site 3L + 1 at the step, seed `ed_seed`, over V elements;
  - the lookup reads W * s_e (s_e(v) = flag / (1 - p_e)) before the site-0 dropout; the gradient of W is s_e * dW_eff;
  - tied: only the lookup is masked, the projection uses the raw E, so dE = G_proj + s_e * G_emb.
  - AR/TAR on the last layer's raw output h (y = h * s, s its output mask's multiplier):
    R = alpha/(T*H) * sum y^2 + beta/((T-1)*H) * sum_{t>=1} (h_t - h_{t-1})^2, and r_t = dR/dh_t enters the last
    layer's backward after its output mask (the returned loss stays the NLL).
With `ed_mask=None`, `tied=False` and alpha = beta = 0 every function here computes exactly what the weight-drop oracle
computes.
"""
from __future__ import annotations

import numpy as np

from oracle import lstm_lm_oracle as O
from oracle import philox as PH
from tests import _tied_oracle as TO
from tests import _variational_oracle as VO
from tests import _weight_drop_oracle as WO


def embed_mask(ed_seed, step, L, V, p_e):
    """bool [V] keep flags of the mode, or None when p_e == 0."""
    if float(np.float32(p_e)) <= 0.0:
        return None
    return PH.keep_mask(ed_seed, step, 3 * L + 1, V, p_e)


def _view(params, ed_mask, p_e, tied):
    """The untied parameter dict the forward reads: embed.W masked row by row, fc.W the raw E when tied."""
    p = dict(params)
    if tied:
        p["fc.W"] = params["embed.W"]
    if ed_mask is not None:
        p["embed.W"] = O.apply_dropout(params["embed.W"], ed_mask[:, None], p_e)
    return p


def model_fwd(params, x, states, L, dropout=0.0, masks=None, rmasks=None, p_rec=0.0, wd_masks=None, p_wd=0.0,
              ed_mask=None, p_e=0.0, tied=False):
    return WO.model_fwd(_view(params, ed_mask, p_e, tied), x, states, L, dropout, masks, rmasks, p_rec, wd_masks, p_wd)


def last_layer_h(cache, L):
    """[T, B, H] raw output of the last layer, from the forward cache (h_t = o * tanh(c_t))."""
    return np.stack([o * np.tanh(c) for (_, _, _, _, _, o, c) in cache["layer_cache"][L - 1]])


def activation_reg(cache, L, alpha, beta):
    """(alpha-weighted AR, beta-weighted TAR, r [T, B, H] = dR/dh) of the forward in `cache`."""
    h = last_layer_h(cache, L)
    T, _, H = h.shape
    masks = cache["masks"]
    s = O.apply_dropout(np.ones_like(h), None if masks is None else masks[L], cache["dropout"])
    y = h * s
    wa = alpha / (T * H)
    wb = beta / ((T - 1) * H) if T > 1 else 0.0
    d = h[1:] - h[:-1]
    dp = np.concatenate([np.zeros_like(h[:1]), d])
    dn = np.concatenate([d, np.zeros_like(h[:1])])
    r = 2 * wa * y * s + 2 * wb * (dp - dn)
    return wa * float((y * y).sum()), wb * float((d * d).sum()), r


def _reg_grads(eff, cache, r, L):
    """The gradients that r (added after layer L-1's output mask) contributes, through the layers and the embedding."""
    p, masks, rmasks, p_rec = cache["dropout"], cache["masks"], cache["rmasks"], cache["p_rec"]
    T, B, H = r.shape
    grads = {"fc.W": np.zeros_like(eff["fc.W"]), "fc.b": np.zeros_like(eff["fc.b"])}
    da = r
    for l in range(L - 1, -1, -1):
        if l < L - 1:
            da = O.apply_dropout(da, None if masks is None else masks[l + 1], p)
        dx, dWi, dWh, db = VO.lstm_layer_bwd(da, cache["layer_cache"][l], cache["layer_in"][l],
                                             eff[f"rnns.{l}.weight_ih_l0"], eff[f"rnns.{l}.weight_hh_l0"],
                                             None if rmasks is None else rmasks[l], p_rec)
        grads[f"rnns.{l}.weight_ih_l0"] = dWi
        grads[f"rnns.{l}.weight_hh_l0"] = dWh
        grads[f"rnns.{l}.bias_ih_l0"] = db
        grads[f"rnns.{l}.bias_hh_l0"] = db.copy()
        da = dx
    da = O.apply_dropout(da, None if masks is None else masks[0], p)
    dE = np.zeros_like(eff["embed.W"])
    np.add.at(dE, cache["x"].reshape(-1), da.reshape(-1, H))
    grads["embed.W"] = dE
    return grads


def model_bwd(params, cache, dscores, L, wd_masks=None, p_wd=0.0, ed_mask=None, p_e=0.0, tied=False, r=None):
    """Gradients of NLL (+ the penalties whose dR/dh is r, when given)."""
    view = _view(params, ed_mask, p_e, tied)
    grads = WO.model_bwd(view, cache, dscores, L, wd_masks, p_wd)
    if r is not None:
        g2 = _reg_grads(WO.effective_params(view, L, wd_masks, p_wd), cache, r, L)
        if wd_masks is not None:
            for l in range(L):
                k = f"rnns.{l}.weight_hh_l0"
                g2[k] = O.apply_dropout(g2[k], wd_masks[l], p_wd)
        for k in g2:
            grads[k] = grads[k] + g2[k]
    if ed_mask is not None:
        grads["embed.W"] = O.apply_dropout(grads["embed.W"], ed_mask[:, None], p_e)
    if tied:
        grads["embed.W"] = grads["embed.W"] + grads.pop("fc.W")
    return grads


def train_step(params, x, y, states, L, lr, max_norm, dropout=0.0, masks=None, rmasks=None, p_rec=0.0, wd_masks=None,
               p_wd=0.0, ed_mask=None, p_e=0.0, tied=False, alpha=0.0, beta=0.0):
    """forward, loss, backward of NLL + R, clip + SGD of the raw parameters (in place; tied: over the 2 + 4L distinct
    tensors).  Returns (NLL, norm, states, scores, raw gradients, (AR, TAR))."""
    scores, new_states, cache = model_fwd(params, x, states, L, dropout, masks, rmasks, p_rec, wd_masks, p_wd, ed_mask,
                                          p_e, tied)
    loss = O.nll_loss(scores, y)
    reg = (0.0, 0.0)
    r = None
    if alpha > 0 or beta > 0:
        ar, tar, r = activation_reg(cache, L, alpha, beta)
        reg = (ar, tar)
    grads = model_bwd(params, cache, O.nll_loss_bwd(scores, y), L, wd_masks, p_wd, ed_mask, p_e, tied, r)
    raw = {k: v.copy() for k, v in grads.items()}
    norm = O.clip_sgd(params, grads, lr, max_norm, TO.param_names(L) if tied else O.param_names(L))
    return loss, norm, new_states, scores, raw, reg
