"""Float64 restatement of zoneout (Krueger et al. 2017; DESIGN.md section 20) on top of oracle/lstm_lm_oracle.py.

One layer, unit (t, b, j):  c~ = f c_{t-1} + i g,  h~ = o tanh(c~), then
  train mode:  c_t = c_{t-1} where zc, else c~;   h_t = h_{t-1} where zh, else h~   (zc, zh: boolean flags [T,B,H])
  eval mode:   c_t = z_c c_{t-1} + (1 - z_c) c~;  h_t = z_h h_{t-1} + (1 - z_h) h~
The backward is written out by hand (the CPU tests check it against torch autograd of an LSTMCell loop):
  dh_t = dy_t + (dG_{t+1} W_hh) + hcarry;  dh~ = (1 - zh) dh_t;  dc~ = (1 - zc) dc_t + dh~ o (1 - tanh^2 c~);
  gate gradients from dc~ and dh~;  dc_{t-1} = zc dc_t + f dc~;  hcarry <- zh dh_t.
(h~ reads c~, not the zoned c_t: the h~ path reaches c~ whatever zc is.)
The flags of layer l are the dropped flags of sites 3L + 3 + l (c) and 4L + 3 + l (h) over T*B*H (flags()).
"""
import numpy as np

from oracle import lstm_lm_oracle as O
from oracle import philox


def flags(seed, step, L, l, T, B, H, z_c, z_h):
    """(zc, zh) of layer l, boolean [T,B,H]: True = the unit keeps its previous value"""
    zc = ~philox.keep_mask(seed, step, 3 * L + 3 + l, T * B * H, z_c).reshape(T, B, H) if z_c > 0 else \
        np.zeros((T, B, H), bool)
    zh = ~philox.keep_mask(seed, step, 4 * L + 3 + l, T * B * H, z_h).reshape(T, B, H) if z_h > 0 else \
        np.zeros((T, B, H), bool)
    return zc, zh


def _mults(z, flag, t, train):
    """(keep, take) multipliers of step t: the flags in train mode, (z, 1 - z) in eval mode"""
    if train:
        k = flag[t].astype(np.float64)
        return k, 1.0 - k
    return z, 1.0 - z


def layer_fwd(x, h0, c0, W_ih, W_hh, b_ih, b_hh, z_c, z_h, zc=None, zh=None):
    """x [T,B,In]; zc / zh None: eval mode.  Returns y [T,B,H], h_T, c_T, cache"""
    train = zc is not None
    h, c = h0, c0
    ys, cache = [], []
    for t in range(x.shape[0]):
        h_prev, c_prev = h, c
        h_new, c_new, (i, f, g, o) = O.lstm_cell_fwd(x[t], h, c, W_ih, W_hh, b_ih, b_hh)
        kc, tc = _mults(z_c, zc, t, train)
        kh, th = _mults(z_h, zh, t, train)
        c = kc * c_prev + tc * c_new
        h = kh * h_prev + th * h_new
        ys.append(h)
        cache.append((h_prev, c_prev, i, f, g, o, c_new, kc, tc, kh, th))
    return np.stack(ys), h, c, cache


def layer_bwd(dy, cache, x, W_ih, W_hh):
    """dy [T,B,H] on the layer's outputs; the entering states are detached.  Returns dx, dW_ih, dW_hh, db"""
    T, B, H = dy.shape
    dW_ih, dW_hh = np.zeros_like(W_ih), np.zeros_like(W_hh)
    db = np.zeros(4 * H)
    dx = np.zeros_like(x)
    dh_rec = np.zeros((B, H))
    hcarry = np.zeros((B, H))
    dc = np.zeros((B, H))
    for t in range(T - 1, -1, -1):
        h_prev, c_prev, i, f, g, o, ct, kc, tc_, kh, th = cache[t]
        dh = dy[t] + dh_rec + hcarry
        dht = th * dh
        hcarry = kh * dh
        tc = np.tanh(ct)
        dct = tc_ * dc + dht * o * (1.0 - tc * tc)
        dG = np.concatenate([dct * g * i * (1.0 - i), dct * c_prev * f * (1.0 - f),
                             dct * i * (1.0 - g * g), dht * tc * o * (1.0 - o)], axis=1)
        dc = kc * dc + f * dct
        dx[t] = dG @ W_ih
        dh_rec = dG @ W_hh
        dW_ih += dG.T @ x[t]
        dW_hh += dG.T @ h_prev
        db += dG.sum(axis=0)
    return dx, dW_ih, dW_hh, db


def model_fwd(params, x, states, L, z_c, z_h, zflags=None, dropout=0.0, masks=None):
    """lstm_lm_oracle.model_fwd with zoneout in every layer; zflags = [(zc, zh)] * L (train) or None (eval)"""
    p64 = {k: np.asarray(v, np.float64) for k, v in params.items()}
    a = O.apply_dropout(O.embed_fwd(p64["embed.W"], x), None if masks is None else masks[0], dropout)
    new_states, caches, layer_in = [], [], []
    for l in range(L):
        layer_in.append(a)
        h0, c0 = (np.asarray(s, np.float64) for s in states[l])
        zc, zh = zflags[l] if zflags is not None else (None, None)
        y, h, c, cache = layer_fwd(a, h0, c0, p64[f"rnns.{l}.weight_ih_l0"], p64[f"rnns.{l}.weight_hh_l0"],
                                   p64[f"rnns.{l}.bias_ih_l0"], p64[f"rnns.{l}.bias_hh_l0"], z_c, z_h, zc, zh)
        new_states.append((h, c))
        caches.append(cache)
        a = O.apply_dropout(y, None if masks is None else masks[l + 1], dropout)
    scores = O.linear_fwd(a, p64["fc.W"], p64["fc.b"])
    return scores, new_states, {"x": np.asarray(x), "layer_in": layer_in, "caches": caches, "fc_in": a, "p64": p64,
                                "masks": masks, "dropout": dropout}


def model_bwd(cache, dscores, L):
    p64, masks, p = cache["p64"], cache["masks"], cache["dropout"]
    fc_in = cache["fc_in"]
    T, B, H = fc_in.shape
    grads = {"fc.W": dscores.T @ fc_in.reshape(-1, H), "fc.b": dscores.sum(axis=0)}
    da = (dscores @ p64["fc.W"]).reshape(T, B, H)
    for l in range(L - 1, -1, -1):
        da = O.apply_dropout(da, None if masks is None else masks[l + 1], p)
        dx, dWi, dWh, db = layer_bwd(da, cache["caches"][l], cache["layer_in"][l], p64[f"rnns.{l}.weight_ih_l0"],
                                     p64[f"rnns.{l}.weight_hh_l0"])
        grads[f"rnns.{l}.weight_ih_l0"], grads[f"rnns.{l}.weight_hh_l0"] = dWi, dWh
        grads[f"rnns.{l}.bias_ih_l0"], grads[f"rnns.{l}.bias_hh_l0"] = db, db.copy()
        da = dx
    da = O.apply_dropout(da, None if masks is None else masks[0], p)
    dE = np.zeros_like(p64["embed.W"])
    np.add.at(dE, cache["x"].reshape(-1), da.reshape(-1, da.shape[-1]))
    grads["embed.W"] = dE
    return grads


def train_step(params, x, y, states, L, lr, max_norm, z_c, z_h, zflags, dropout=0.0, masks=None):
    """one fused step (main.py:109-117) in float64; params (float64 copies) are updated in place.
    Returns loss, norm, new states, raw gradients"""
    scores, new_states, cache = model_fwd(params, x, states, L, z_c, z_h, zflags, dropout, masks)
    loss = O.nll_loss(scores, y)
    grads = model_bwd(cache, O.nll_loss_bwd(scores, y), L)
    raw = {k: v.copy() for k, v in grads.items()}
    for k in params:
        params[k] = np.asarray(params[k], np.float64)
    norm = O.clip_sgd(params, grads, lr, max_norm, O.param_names(L))
    return loss, norm, new_states, raw


def eval_loss(params, x, y, states, L, z_c, z_h):
    """the eval-mode window loss (the expectation) and the states it leaves"""
    scores, new_states, _ = model_fwd(params, x, states, L, z_c, z_h)
    return O.nll_loss(scores, y), new_states
