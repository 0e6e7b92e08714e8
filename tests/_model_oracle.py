"""fp64 restatement of a train / eval step of the model in every mode, written directly in torch float64: embedding
[V,E], layer l an LSTM from In_l to H_l (gate rows i, f, g, o), projection [V,H_{L-1}] (tied: the embedding itself), the
loss main.py computes (mean over tokens of -log p, times B), clip_grad_norm_ and SGD.  Layer widths (DESIGN.md section
18) and the number of MoS experts come from the parameter shapes.

Every mode, with the masks of `oracle.philox` over each site's own width (`Modes`, `mode_masks`):
  - dropout site s (0: after the embedding, l+1: after layer l) of width W_s: element (t, b, j) is stream element
    t*B*W_s + b*W_s + j; variational: b*W_s + j, the same at every t;
  - recurrent site L+1+l (variational, p_rec): layer l's operand of W_hh is h_{t-1} * m / (1 - p_rec), m over B*H_l;
  - weight drop: layer l's W_hh is W_hh * m / (1 - p_wd), m = site 2L+1+l over 4*H_l*H_l, seed wd_seed;
  - embedding dropout: row v of the lookup is E[v] * m_v / (1 - p_e), m = site 3L+1 over V, seed ed_seed; tied: the
    projection reads the raw E;
  - AR/TAR on the last layer: alpha/(T*H) * sum (h*s)^2 + beta/((T-1)*H) * sum_{t>=1} (h_t - h_{t-1})^2, H = H_{L-1}
    and s the multiplier of site L's mask, added to the loss that is differentiated (the returned loss stays the NLL);
  - zoneout (Krueger et al. 2017; section 20): unit (t, b, j) of layer l computes c~ = f c_{t-1} + i g and
    h~ = o tanh(c~) (h~ reads c~, not the zoned c_t), then
      train:  c_t = c_{t-1} where flagged, else c~;   h_t = h_{t-1} where flagged, else h~,
      eval:   c_t = z_c c_{t-1} + (1 - z_c) c~;      h_t = z_h h_{t-1} + (1 - z_h) h~,
    with the flags the dropped flags of site 3L+3+l (c, rate z_c) and 4L+3+l (h, rate z_h) over T*B*H_l;
  - Mixture of Softmaxes (Yang et al. 2018; section 19), when params hold "prior.W" [K, H_{L-1}]: with h the last
    layer's output after its dropout and W = fc.W [V, E] (tied: embed.W)
      u = h latent.W^T + latent.b [N, K*E],  c = tanh(u),  c^ = c * m / (1 - p_l)  (m: site 3L+2, element
      t*B*K*E + b*K*E + j; variational: b*K*E + j),  a = h prior.W^T,  pi = softmax(a),  z_k = c^_k W^T + fc.b,
      log p = logsumexp_k(log pi_k + log_softmax(z_k)),
    and `forward` returns log p in place of the scores.
Eval mode draws no mask and applies zoneout by its expectation.  Gradients come from torch autograd.

params: dict name -> float64 tensor in the Model's names ("embed.W", "rnns.l.weight_ih_l0", ..., "fc.W", "fc.b"; tied:
no "fc.W"; MoS: then "prior.W", "latent.W", "latent.b").  states: list of (h [B,H_l], c [B,H_l]) float64.
"""
from dataclasses import dataclass

import numpy as np
import torch

from oracle import philox as PH


@dataclass
class Modes:
    seed: int = 0            # dropout, recurrent, zoneout and latent masks (the Trainer's seed)
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
    z_c: float = 0.0
    z_h: float = 0.0
    p_l: float = 0.0


@dataclass
class Masks:
    """the bool masks of a step, None where the mode is off: keep flags, except zc / zh (True = the unit keeps its
    previous value)"""
    sites: list = None       # per dropout site s: [T, B, W_s]
    rec: list = None         # per layer: [B, H_l]
    wd: list = None          # per layer: [4*H_l, H_l]
    ed: np.ndarray = None    # [V]
    zc: list = None          # per layer: [T, B, H_l]
    zh: list = None          # per layer: [T, B, H_l]
    latent: np.ndarray = None  # [T, B, K*E]


def _stream(seed, step, site, T, B, W, p, variational=False):
    """bool [T, B, W] keep flags of a site: element (t, b, j) is t*B*W + b*W + j; variational: b*W + j at every t"""
    if variational:
        return np.broadcast_to(PH.keep_mask(seed, step, site, B * W, p).reshape(1, B, W), (T, B, W)).copy()
    return PH.keep_mask(seed, step, site, T * B * W, p).reshape(T, B, W)


def mode_masks(md, widths, T, B, V, K=0):
    """every mask of a step of the model with widths [E, H_0, ..., H_{L-1}] and K experts (0: no MoS head)"""
    L = len(widths) - 1
    Hs = widths[1:]
    m = Masks()
    if md.p > 0:
        m.sites = [_stream(md.seed, md.step, s, T, B, W, md.p, md.variational) for s, W in enumerate(widths)]
    if md.variational and md.p_rec > 0:
        m.rec = [PH.keep_mask(md.seed, md.step, L + 1 + l, B * H, md.p_rec).reshape(B, H) for l, H in enumerate(Hs)]
    if md.p_wd > 0:
        m.wd = [PH.keep_mask(md.wd_seed, md.step, 2 * L + 1 + l, 4 * H * H, md.p_wd).reshape(4 * H, H)
                for l, H in enumerate(Hs)]
    if md.p_e > 0:
        m.ed = PH.keep_mask(md.ed_seed, md.step, 3 * L + 1, V, md.p_e)
    if md.z_c > 0:
        m.zc = [~_stream(md.seed, md.step, 3 * L + 3 + l, T, B, H, md.z_c) for l, H in enumerate(Hs)]
    if md.z_h > 0:
        m.zh = [~_stream(md.seed, md.step, 4 * L + 3 + l, T, B, H, md.z_h) for l, H in enumerate(Hs)]
    if K and md.p_l > 0:
        m.latent = _stream(md.seed, md.step, 3 * L + 2, T, B, K * widths[0], md.p_l, md.variational)
    return m


def _drop(a, mask, p):
    if mask is None:
        return a
    return a * torch.as_tensor(mask, device=a.device).to(a.dtype) * (1.0 / (1.0 - p))


def _zone(prev, new, flags, z, train):
    """one step of zoneout: the flags select prev (train), the expectation (eval); new when the mode is off"""
    if train:
        return new if flags is None else torch.where(flags, prev, new)
    return new if z == 0 else z * prev + (1 - z) * new


def names(L, tied, experts=False):
    out = ["embed.W"]
    for l in range(L):
        out += [f"rnns.{l}.weight_ih_l0", f"rnns.{l}.weight_hh_l0", f"rnns.{l}.bias_ih_l0", f"rnns.{l}.bias_hh_l0"]
    out += ["fc.b"] if tied else ["fc.W", "fc.b"]
    return out + (["prior.W", "latent.W", "latent.b"] if experts else [])


def head_logp(h, params, tied, K, lmask=None, p_l=0.0):
    """log p [N, V] of the MoS head over h [N, H] (lmask: [N, K*E] keep flags or None)"""
    W = params["embed.W"] if tied else params["fc.W"]
    E = W.shape[1]
    c = _drop(torch.tanh(h @ params["latent.W"].t() + params["latent.b"]), lmask, p_l)
    z = c.reshape(-1, K, E) @ W.t() + params["fc.b"]                    # [N, K, V]
    log_pi = torch.log_softmax(h @ params["prior.W"].t(), dim=-1)       # [N, K]
    return torch.logsumexp(log_pi[:, :, None] + torch.log_softmax(z, dim=-1), dim=1)


def forward(params, x, states, L, tied, md=None, masks=None, train=True):
    """scores [T*B, V] (MoS: log p), the new states and the AR/TAR value (0 without md or with alpha = beta = 0);
    x [T,B] int64.  masks: those mode_masks draws from md unless given; train=False: eval mode"""
    T, B = x.shape
    V = params["fc.b"].shape[0]
    K = params["prior.W"].shape[0] if "prior.W" in params else 0
    widths = [params["embed.W"].shape[1]] + [params[f"rnns.{l}.weight_hh_l0"].shape[1] for l in range(L)]
    md = md or Modes()
    if masks is None:
        masks = mode_masks(md, widths, T, B, V, K) if train else Masks()
    sites, rec, wd, ed = masks.sites, masks.rec, masks.wd, masks.ed
    E_look = _drop(params["embed.W"], None if ed is None else ed[:, None], md.p_e)
    inp = _drop(E_look[x.reshape(-1)].reshape(T, B, -1), None if sites is None else sites[0], md.p)
    new_states = []
    h_last = None
    for l in range(L):
        w_ih = params[f"rnns.{l}.weight_ih_l0"]
        w_hh = _drop(params[f"rnns.{l}.weight_hh_l0"], None if wd is None else wd[l], md.p_wd)
        b = params[f"rnns.{l}.bias_ih_l0"] + params[f"rnns.{l}.bias_hh_l0"]
        zc, zh = (None if f is None else torch.as_tensor(f[l], device=w_ih.device) for f in (masks.zc, masks.zh))
        h, c = states[l]
        pre_x = inp @ w_ih.t() + b
        outs = []
        for t in range(T):
            g = pre_x[t] + _drop(h, None if rec is None else rec[l], md.p_rec) @ w_hh.t()
            i, f, gg, o = g.chunk(4, 1)
            c_new = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
            h_new = torch.sigmoid(o) * torch.tanh(c_new)
            c = _zone(c, c_new, None if zc is None else zc[t], md.z_c, train)
            h = _zone(h, h_new, None if zh is None else zh[t], md.z_h, train)
            outs.append(h)
        h_last = torch.stack(outs)
        inp = _drop(h_last, None if sites is None else sites[l + 1], md.p)
        new_states.append((h, c))
    if K:
        lm = None if masks.latent is None else masks.latent.reshape(T * B, -1)
        out = head_logp(inp.reshape(T * B, -1), params, tied, K, lm, md.p_l)
    else:
        W = params["embed.W"] if tied else params["fc.W"]
        out = inp.reshape(T * B, -1) @ W.t() + params["fc.b"]
    reg = 0.0
    if md.alpha > 0 or md.beta > 0:
        H = widths[-1]
        reg = md.alpha / (T * H) * (inp * inp).sum()
        if T > 1:
            reg = reg + md.beta / ((T - 1) * H) * ((h_last[1:] - h_last[:-1]) ** 2).sum()
    return out, new_states, reg


def loss_of(out, y, logp=False):
    """main.py's loss of forward's output: scores, or log p (logp=True: the MoS head)"""
    B = y.shape[1]
    if logp:
        return -out.gather(1, y.reshape(-1, 1)).mean() * B
    return torch.nn.functional.cross_entropy(out, y.reshape(-1), reduction="mean") * B


def train_step(params, x, y, states, L, tied, lr, max_norm, md=None, masks=None):
    """(NLL, norm, raw grads, params after, states after, AR + TAR); params is not modified"""
    ps = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
    out, new_states, reg = forward(ps, x, [(h.detach(), c.detach()) for h, c in states], L, tied, md, masks)
    loss = loss_of(out, y, "prior.W" in ps)
    (loss + reg).backward()
    grads = {k: ps[k].grad.detach().clone() for k in ps}
    norm = torch.sqrt(sum((g * g).sum() for g in grads.values()))
    coef = min(1.0, max_norm / (float(norm) + 1e-6))
    after = {k: (ps[k].detach() - lr * coef * grads[k]) for k in ps}
    return (loss.item(), float(norm), grads, after, [(h.detach(), c.detach()) for h, c in new_states],
            float(reg.detach()) if torch.is_tensor(reg) else float(reg))


def eval_loss(params, x, y, states, L, tied, md=None):
    """the eval-mode window loss and the states it leaves (md: the zoneout rates; no mask is drawn)"""
    with torch.no_grad():
        out, new_states, _ = forward(params, x, states, L, tied, md, train=False)
        return float(loss_of(out, y, "prior.W" in params)), new_states


def vjp(logp, z, log_pi, G):
    """the MoS drop-in backward's formulas: (dz [N, K, V], da [N, K]) for upstream G = dL / d log p [N, V], with
    rho = pi q / p, s_k = sum_v G rho, dz = rho G - q s, da = s - pi sum_v G"""
    q = torch.softmax(z, dim=-1)
    rho = torch.exp(log_pi[:, :, None] + torch.log_softmax(z, dim=-1) - logp[:, None, :])
    s = (G[:, None, :] * rho).sum(-1)
    dz = rho * G[:, None, :] - q * s[:, :, None]
    da = s - torch.exp(log_pi) * G.sum(-1, keepdim=True)
    return dz, da
