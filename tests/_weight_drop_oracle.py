"""Numpy restatement of the weight-dropped LSTM (DESIGN.md section 15)  --  TEST INFRASTRUCTURE ONLY.

Extends `tests._variational_oracle` (and through it `oracle.lstm_lm_oracle`, reused unchanged) by DropConnect on the
hidden-to-hidden matrices (Merity, Keskar & Socher 2018), with the masks of `oracle.philox`:
  - layer l's mask is the keep flags of site 2L + 1 + l at the step, seed `wd_seed`, over the 4H*H elements of W_hh
    (element r*H + k = W_hh[r, k]);
  - the forward uses W_eff = W_hh * m_l * scale(p_wd) at every time step; the gradient is scale * m_l * dW_eff.
With `wd_masks=None` every function here computes exactly what the variational oracle computes.
"""
from __future__ import annotations

import numpy as np

from oracle import lstm_lm_oracle as O
from oracle import philox as PH
from tests import _variational_oracle as VO


def weight_drop_masks(wd_seed, step, L, H, p_wd):
    """L bool [4H, H] keep-masks of the mode, or None when p_wd == 0."""
    if float(np.float32(p_wd)) <= 0.0:
        return None
    return [PH.keep_mask(wd_seed, step, 2 * L + 1 + l, 4 * H * H, p_wd).reshape(4 * H, H) for l in range(L)]


def _key(l):
    return f"rnns.{l}.weight_hh_l0"


def effective_params(params, L, wd_masks, p_wd):
    """params with every W_hh replaced by W_hh * m_l * scale (a shallow copy; the others are shared)."""
    if wd_masks is None:
        return params
    out = dict(params)
    for l in range(L):
        out[_key(l)] = O.apply_dropout(params[_key(l)], wd_masks[l], p_wd)
    return out


def model_fwd(params, x, states, L, dropout=0.0, masks=None, rmasks=None, p_rec=0.0, wd_masks=None, p_wd=0.0):
    return VO.model_fwd(effective_params(params, L, wd_masks, p_wd), x, states, L, dropout, masks, rmasks, p_rec)


def model_bwd(params, cache, dscores, L, wd_masks=None, p_wd=0.0):
    grads = VO.model_bwd(effective_params(params, L, wd_masks, p_wd), cache, dscores, L)
    if wd_masks is not None:
        for l in range(L):
            grads[_key(l)] = O.apply_dropout(grads[_key(l)], wd_masks[l], p_wd)
    return grads


def train_step(params, x, y, states, L, lr, max_norm, dropout=0.0, masks=None, rmasks=None, p_rec=0.0, wd_masks=None,
               p_wd=0.0):
    """forward, loss, backward, clip + SGD of the raw parameters (in place)."""
    scores, new_states, cache = model_fwd(params, x, states, L, dropout, masks, rmasks, p_rec, wd_masks, p_wd)
    loss = O.nll_loss(scores, y)
    grads = model_bwd(params, cache, O.nll_loss_bwd(scores, y), L, wd_masks, p_wd)
    raw = {k: v.copy() for k, v in grads.items()}
    norm = O.clip_sgd(params, grads, lr, max_norm, O.param_names(L))
    return loss, norm, new_states, scores, raw
