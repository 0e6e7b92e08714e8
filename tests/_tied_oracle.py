"""Numpy restatement of the tied embedding mode (DESIGN.md section 13)  --  TEST INFRASTRUCTURE ONLY.

Extends `oracle.lstm_lm_oracle` (through the variational restatement, which computes exactly what the oracle computes
when it is given no recurrent masks) by tying the embedding and softmax weights (Press & Wolf 2017):
  - a tied parameter dict has one matrix "embed.W" = E and no "fc.W"; the forward uses fc.W = E;
  - the gradient of E is the sum of the oracle's two [V,H] gradients (projection + embedding);
  - the clip norm and the SGD update run over the 2 + 4L distinct tensors, E counted once.
Nothing under oracle/ changes.
"""
from __future__ import annotations

from oracle import lstm_lm_oracle as O
from tests import _variational_oracle as VO


def param_names(layer_num):
    """The distinct tensors in registration order: embed.W, the LSTM tensors, fc.b."""
    return [n for n in O.param_names(layer_num) if n != "fc.W"]


def _untied_view(params):
    p = dict(params)
    p["fc.W"] = p["embed.W"]
    return p


def model_fwd(params, x, states, layer_num, dropout=0.0, masks=None, rmasks=None, p_rec=0.0):
    return VO.model_fwd(_untied_view(params), x, states, layer_num, dropout, masks, rmasks, p_rec)


def model_bwd(params, cache, dscores, layer_num):
    """The oracle's gradients with the two [V,H] gradients summed into "embed.W" (no "fc.W" entry)."""
    g = VO.model_bwd(_untied_view(params), cache, dscores, layer_num)
    g["embed.W"] = g["embed.W"] + g.pop("fc.W")
    return g


def train_step(params, x, y, states, layer_num, lr, max_norm, dropout=0.0, masks=None, rmasks=None, p_rec=0.0):
    """One tied step: forward, loss, backward, clip over the distinct tensors + SGD (params updated in place)."""
    scores, new_states, cache = model_fwd(params, x, states, layer_num, dropout, masks, rmasks, p_rec)
    loss = O.nll_loss(scores, y)
    grads = model_bwd(params, cache, O.nll_loss_bwd(scores, y), layer_num)
    norm = O.clip_sgd(params, grads, lr, max_norm, param_names(layer_num))
    return loss, norm, new_states, scores, grads
