"""fp64 restatement of a train / eval step of a Mixture-of-Softmaxes model (Yang et al. 2018; DESIGN.md section 19) on
top of `_widths_oracle`: the same embedding, LSTM stack and modes, then the head

  u = h latent.W^T + latent.b [N, K*E],  c = tanh(u),  c^ = c * m / (1 - p_l)  (m: oracle.philox site 3L + 2, element
  t*B*K*E + b*K*E + j; variational: b*K*E + j),  a = h prior.W^T,  pi = softmax(a),  z_k = c^_k W^T + fc.b,
  log p = logsumexp_k(log pi_k + log_softmax(z_k))

with h the last layer's output after its dropout and W = fc.W [V, E] (tied: embed.W).  The loss is main.py's unit
(mean over tokens of -log p[y], times B).  Gradients come from torch autograd.
"""
import numpy as np
import torch

from oracle import philox as PH
from tests import _widths_oracle as WO

Modes = WO.Modes


def names(L, tied):
    return WO.names(L, tied) + ["prior.W", "latent.W", "latent.b"]


def latent_mask(md, L, T, B, KE, p_l):
    """bool [T, B, K*E] keep flags of the latent dropout of an L-layer model, or None"""
    if p_l <= 0:
        return None
    site = 3 * L + 2
    if md.variational:
        m = PH.keep_mask(md.seed, md.step, site, B * KE, p_l).reshape(1, B, KE)
        return np.broadcast_to(m, (T, B, KE)).copy()
    return PH.keep_mask(md.seed, md.step, site, T * B * KE, p_l).reshape(T, B, KE)


def head_logp(h, params, tied, K, lmask=None, p_l=0.0):
    """log p [N, V] of the head over h [N, H] (lmask: [N, K*E] keep flags or None)"""
    W = params["embed.W"] if tied else params["fc.W"]
    E = W.shape[1]
    c = torch.tanh(h @ params["latent.W"].t() + params["latent.b"])
    if lmask is not None:
        c = c * torch.as_tensor(lmask, device=c.device).to(c.dtype) * (1.0 / (1.0 - p_l))
    z = c.reshape(-1, K, E) @ W.t() + params["fc.b"]                    # [N, K, V]
    log_pi = torch.log_softmax(h @ params["prior.W"].t(), dim=-1)       # [N, K]
    return torch.logsumexp(log_pi[:, :, None] + torch.log_softmax(z, dim=-1), dim=1)


def forward(params, x, states, L, tied, md=None, p_l=0.0):
    """log p [T*B, V], the new states and the AR/TAR value"""
    T, B = x.shape
    V = params["fc.b"].shape[0]
    K = params["prior.W"].shape[0]
    widths = [params["embed.W"].shape[1]] + [params[f"rnns.{l}.weight_hh_l0"].shape[1] for l in range(L)]
    md = md or Modes()
    sites, rec, wd, ed = WO.mode_masks(md, widths, T, B, V)
    E_look = WO._drop(params["embed.W"], None if ed is None else ed[:, None], md.p_e)
    inp = WO._drop(E_look[x.reshape(-1)].reshape(T, B, -1), None if sites is None else sites[0], md.p)
    new_states = []
    h_last = None
    for l in range(L):
        w_ih = params[f"rnns.{l}.weight_ih_l0"]
        w_hh = WO._drop(params[f"rnns.{l}.weight_hh_l0"], None if wd is None else wd[l], md.p_wd)
        b = params[f"rnns.{l}.bias_ih_l0"] + params[f"rnns.{l}.bias_hh_l0"]
        h, c = states[l]
        pre_x = inp @ w_ih.t() + b
        outs = []
        for t in range(T):
            g = pre_x[t] + WO._drop(h, None if rec is None else rec[l], md.p_rec) @ w_hh.t()
            i, f, gg, o = g.chunk(4, 1)
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
            h = torch.sigmoid(o) * torch.tanh(c)
            outs.append(h)
        h_last = torch.stack(outs)
        inp = WO._drop(h_last, None if sites is None else sites[l + 1], md.p)
        new_states.append((h, c))
    E = widths[0]
    lm = latent_mask(md, L, T, B, K * E, p_l)
    logp = head_logp(inp.reshape(T * B, -1), params, tied, K, None if lm is None else lm.reshape(T * B, -1), p_l)
    reg = 0.0
    if md.alpha > 0 or md.beta > 0:
        H = widths[-1]
        reg = md.alpha / (T * H) * (inp * inp).sum()
        if T > 1:
            reg = reg + md.beta / ((T - 1) * H) * ((h_last[1:] - h_last[:-1]) ** 2).sum()
    return logp, new_states, reg


def loss_of(logp, y):
    B = y.shape[1]
    return -logp.gather(1, y.reshape(-1, 1)).mean() * B


def train_step(params, x, y, states, L, tied, lr, max_norm, md=None, p_l=0.0):
    """(NLL, norm, raw grads, params after, states after, AR + TAR); params is not modified"""
    ps = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
    logp, new_states, reg = forward(ps, x, [(h.detach(), c.detach()) for h, c in states], L, tied, md, p_l)
    loss = loss_of(logp, y)
    (loss + reg).backward()
    grads = {k: ps[k].grad.detach().clone() for k in ps}
    norm = torch.sqrt(sum((g * g).sum() for g in grads.values()))
    coef = min(1.0, max_norm / (float(norm) + 1e-6))
    after = {k: (ps[k].detach() - lr * coef * grads[k]) for k in ps}
    return (loss.item(), float(norm), grads, after, [(h.detach(), c.detach()) for h, c in new_states],
            float(reg.detach()) if torch.is_tensor(reg) else float(reg))


def eval_loss(params, x, y, states, L, tied):
    with torch.no_grad():
        logp, new_states, _ = forward(params, x, states, L, tied)
        return float(loss_of(logp, y)), new_states


def vjp(logp, z, log_pi, G):
    """the drop-in backward's formulas: (dz [N, K, V], da [N, K]) for upstream G = dL / d log p [N, V], with
    rho = pi q / p, s_k = sum_v G rho, dz = rho G - q s, da = s - pi sum_v G"""
    q = torch.softmax(z, dim=-1)
    rho = torch.exp(log_pi[:, :, None] + torch.log_softmax(z, dim=-1) - logp[:, None, :])
    s = (G[:, None, :] * rho).sum(-1)
    dz = rho * G[:, None, :] - q * s[:, :, None]
    da = s - torch.exp(log_pi) * G.sum(-1, keepdim=True)
    return dz, da
