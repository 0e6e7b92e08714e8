"""Float64 restatement of dynamic evaluation (DESIGN.md section 14)  --  TEST INFRASTRUCTURE ONLY.

Built on `oracle.lstm_lm_oracle` (untied) and `tests/_model_oracle.py` (tied); nothing under oracle/ changes.
  - the window loss and its gradient are the oracle's eval-mode (no dropout) loss and backward, entering states detached;
  - the update is theta += a * (theta_g - theta) - lr * u with the RMS rule (u = g / (r + eps), a = min(1, lam r / rbar))
    or the SGD rule (u = g, a = min(1, lam));
  - the statistics are MS = mean over K windows of g^2 at theta_g, states carried from zero, r = sqrt(MS), rbar = the
    mean of r over all distinct parameter elements.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import lstm_lm_oracle as O
from tests import _model_oracle as MO


def names(layer_num, tied=False):
    """The distinct parameter tensors (a tied E once, as "embed.W")."""
    return MO.names(layer_num, tied)


def window_grads(params, x, y, states, layer_num, tied=False):
    """(loss, grads, new states) of the eval-mode window loss at params."""
    if tied:
        loss, _, grads, _, new_states, _ = MO.train_step(
            {k: torch.as_tensor(v) for k, v in params.items()}, torch.as_tensor(x), torch.as_tensor(y),
            [(torch.as_tensor(h), torch.as_tensor(c)) for h, c in states], layer_num, True, 0.0, float("inf"))
        return (loss, {k: g.numpy() for k, g in grads.items()},
                [(h.numpy(), c.numpy()) for h, c in new_states])
    scores, new_states, cache = O.model_fwd(params, x, states, layer_num)
    loss = O.nll_loss(scores, y)
    grads = O.model_bwd(params, cache, O.nll_loss_bwd(scores, y), layer_num)
    return loss, grads, new_states


def update(params, grads, theta_g, lr, lam, rms=None, rbar=None, eps=2e-5):
    """In place over the keys of theta_g."""
    for k in theta_g:
        p, g = params[k], grads[k]
        if rms is None:
            u, a = g, min(1.0, lam)
        else:
            u = g / (rms[k] + eps)
            a = np.minimum(1.0, lam * rms[k] / rbar)
        params[k] = p + (a * (theta_g[k] - p) - lr * u)


def grad_stats(params, batches, layer_num, batch, hidden, tied=False):
    """(r per tensor, rbar, MS per tensor) over the windows, at params, states carried from zero."""
    states = O.zero_states(layer_num, batch, hidden, np.float64)
    ms = None
    for x, y in batches:
        _, g, states = window_grads(params, x, y, states, layer_num, tied)
        sq = {k: g[k] ** 2 for k in names(layer_num, tied)}
        ms = sq if ms is None else {k: ms[k] + sq[k] for k in ms}
    ms = {k: v / len(batches) for k, v in ms.items()}
    r = {k: np.sqrt(v) for k, v in ms.items()}
    P = sum(v.size for v in r.values())
    rbar = sum(float(v.sum()) for v in r.values()) / P
    return r, rbar, ms


def dynamic_pass(params, batches, layer_num, states, lr, lam, rms=None, rbar=None, eps=2e-5, tied=False):
    """Per-window losses and the final parameters of a pass from `states`; theta_g = params as given."""
    theta_g = {k: params[k].copy() for k in names(layer_num, tied)}
    P = {k: v.copy() for k, v in theta_g.items()}
    losses = []
    for x, y in batches:
        loss, g, states = window_grads(P, x, y, states, layer_num, tied)
        losses.append(loss)
        update(P, g, theta_g, lr, lam, rms, rbar, eps)
    return losses, P, states


def dynamic_perplexity(params, batches, layer_num, batch, hidden, lr, lam, rms=None, rbar=None, eps=2e-5, tied=False):
    """exp(mean over windows of loss / B) from zero states: `perplexity`'s formula."""
    states = O.zero_states(layer_num, batch, hidden, np.float64)
    losses, _, _ = dynamic_pass(params, batches, layer_num, states, lr, lam, rms, rbar, eps, tied)
    return float(np.exp(np.mean([l / batch for l in losses])))
