"""fp64 restatement of a train / eval step of a model with per-layer widths (DESIGN.md section 18), written directly in
torch float64: embedding [V,E], layer l an LSTM from In_l to H_l (gate rows i, f, g, o), projection [V,H_{L-1}] (tied:
the embedding itself), the loss main.py computes (mean over tokens of -log p, times B), clip_grad_norm_ and SGD.

Every mode, with the masks of `oracle.philox` over each site's own width (`Modes`, `mode_masks`):
  - dropout site s (0: after the embedding, l+1: after layer l) of width W_s: element (t, b, j) is stream element
    t*B*W_s + b*W_s + j; variational: b*W_s + j, the same at every t;
  - recurrent site L+1+l (variational, p_rec): layer l's operand of W_hh is h_{t-1} * m / (1 - p_rec), m over B*H_l;
  - weight drop: layer l's W_hh is W_hh * m / (1 - p_wd), m = site 2L+1+l over 4*H_l*H_l, seed wd_seed;
  - embedding dropout: row v of the lookup is E[v] * m_v / (1 - p_e), m = site 3L+1 over V, seed ed_seed; tied: the
    projection reads the raw E;
  - AR/TAR on the last layer: alpha/(T*H) * sum (h*s)^2 + beta/((T-1)*H) * sum_{t>=1} (h_t - h_{t-1})^2, H = H_{L-1}
    and s the multiplier of site L's mask, added to the loss that is differentiated (the returned loss stays the NLL).
Gradients come from torch autograd.

params: dict name -> float64 tensor in the Model's names ("embed.W", "rnns.l.weight_ih_l0", ..., "fc.W", "fc.b"; tied:
no "fc.W").  states: list of (h [B,H_l], c [B,H_l]) float64.
"""
from dataclasses import dataclass

import numpy as np
import torch

from oracle import philox as PH


@dataclass
class Modes:
    seed: int = 0            # dropout and recurrent masks (the Trainer's seed)
    step: int = 0
    p: float = 0.0
    variational: bool = False
    p_rec: float = 0.0
    wd_seed: int = 0
    p_wd: float = 0.0
    ed_seed: int = 0
    p_e: float = 0.0
    alpha: float = 0.0
    beta: float = 0.0


def site_masks(seed, step, widths, T, B, p, variational=False):
    """bool [T, B, W_s] keep flags of every dropout site s (widths[s] = W_s); with equal widths and variational off
    this is oracle.philox.site_masks"""
    out = []
    for s, W in enumerate(widths):
        if variational:
            m = PH.keep_mask(seed, step, s, B * W, p).reshape(1, B, W)
            out.append(np.broadcast_to(m, (T, B, W)).copy())
        else:
            out.append(PH.keep_mask(seed, step, s, T * B * W, p).reshape(T, B, W))
    return out


def mode_masks(md, widths, T, B, V):
    """(site masks or None, recurrent masks or None, weight-drop masks or None, embedding mask or None) of a step"""
    L = len(widths) - 1
    sites = site_masks(md.seed, md.step, widths, T, B, md.p, md.variational) if md.p > 0 else None
    rec = None
    if md.variational and md.p_rec > 0:
        rec = [PH.keep_mask(md.seed, md.step, L + 1 + l, B * H, md.p_rec).reshape(B, H) for l, H in
               enumerate(widths[1:])]
    wd = None
    if md.p_wd > 0:
        wd = [PH.keep_mask(md.wd_seed, md.step, 2 * L + 1 + l, 4 * H * H, md.p_wd).reshape(4 * H, H) for l, H in
              enumerate(widths[1:])]
    ed = PH.keep_mask(md.ed_seed, md.step, 3 * L + 1, V, md.p_e) if md.p_e > 0 else None
    return sites, rec, wd, ed


def _drop(a, mask, p):
    if mask is None:
        return a
    return a * torch.as_tensor(mask, device=a.device).to(a.dtype) * (1.0 / (1.0 - p))


def names(L, tied):
    out = ["embed.W"]
    for l in range(L):
        out += [f"rnns.{l}.weight_ih_l0", f"rnns.{l}.weight_hh_l0", f"rnns.{l}.bias_ih_l0", f"rnns.{l}.bias_hh_l0"]
    return out + (["fc.b"] if tied else ["fc.W", "fc.b"])


def forward(params, x, states, L, tied, md=None):
    """scores [T*B, V], the new states and the AR/TAR value (0 without md or with alpha = beta = 0); x [T,B] int64"""
    T, B = x.shape
    V = params["fc.b"].shape[0]
    widths = [params["embed.W"].shape[1]] + [params[f"rnns.{l}.weight_hh_l0"].shape[1] for l in range(L)]
    md = md or Modes()
    sites, rec, wd, ed = mode_masks(md, widths, T, B, V)
    E_look = _drop(params["embed.W"], None if ed is None else ed[:, None], md.p_e)
    inp = _drop(E_look[x.reshape(-1)].reshape(T, B, -1), None if sites is None else sites[0], md.p)
    new_states = []
    h_last = None
    for l in range(L):
        w_ih = params[f"rnns.{l}.weight_ih_l0"]
        w_hh = _drop(params[f"rnns.{l}.weight_hh_l0"], None if wd is None else wd[l], md.p_wd)
        b = params[f"rnns.{l}.bias_ih_l0"] + params[f"rnns.{l}.bias_hh_l0"]
        h, c = states[l]
        pre_x = inp @ w_ih.t() + b
        outs = []
        for t in range(T):
            g = pre_x[t] + _drop(h, None if rec is None else rec[l], md.p_rec) @ w_hh.t()
            i, f, gg, o = g.chunk(4, 1)
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
            h = torch.sigmoid(o) * torch.tanh(c)
            outs.append(h)
        h_last = torch.stack(outs)
        inp = _drop(h_last, None if sites is None else sites[l + 1], md.p)
        new_states.append((h, c))
    W = params["embed.W"] if tied else params["fc.W"]
    scores = inp.reshape(T * B, -1) @ W.t() + params["fc.b"]
    reg = 0.0
    if md.alpha > 0 or md.beta > 0:
        H = widths[-1]
        reg = md.alpha / (T * H) * (inp * inp).sum()
        if T > 1:
            reg = reg + md.beta / ((T - 1) * H) * ((h_last[1:] - h_last[:-1]) ** 2).sum()
    return scores, new_states, reg


def loss_of(scores, y):
    B = y.shape[1]
    return torch.nn.functional.cross_entropy(scores, y.reshape(-1), reduction="mean") * B


def train_step(params, x, y, states, L, tied, lr, max_norm, md=None):
    """(NLL, norm, raw grads, params after, states after, AR + TAR); params is not modified"""
    ps = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
    scores, new_states, reg = forward(ps, x, [(h.detach(), c.detach()) for h, c in states], L, tied, md)
    loss = loss_of(scores, y)
    (loss + reg).backward()
    grads = {k: ps[k].grad.detach().clone() for k in ps}
    norm = torch.sqrt(sum((g * g).sum() for g in grads.values()))
    coef = min(1.0, max_norm / (float(norm) + 1e-6))
    after = {k: (ps[k].detach() - lr * coef * grads[k]) for k in ps}
    return (loss.item(), float(norm), grads, after, [(h.detach(), c.detach()) for h, c in new_states],
            float(reg.detach()) if torch.is_tensor(reg) else float(reg))


def eval_loss(params, x, y, states, L, tied):
    with torch.no_grad():
        scores, new_states, _ = forward(params, x, states, L, tied)
        return float(loss_of(scores, y)), new_states
