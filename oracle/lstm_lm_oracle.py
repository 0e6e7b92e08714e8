"""CPU oracle for the Zaremba LSTM-LM hot path  --  TEST INFRASTRUCTURE ONLY.

This file is a plain-numpy restatement of the arithmetic that the reference
(`ahmetumutdurmus/zaremba`) performs on its hot path.  It exists so that the
CUDA kernels in `zaremba_b200/csrc` can be checked against an independent
implementation on a machine where `/root/reference` is absent (the GPU box).

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline /
`--impl reference` legs may import this module.  The product path
(`zaremba_b200/`) never does and fails loudly without its CUDA library.

Parity pin: the reference has no tests / golden vectors of its own
(SURVEY.md section 4), so this oracle is pinned against OUTPUTS OF THE
REFERENCE ITSELF: `tests/golden/make_golden.py` imports
`/root/reference/model.py`, runs `Model` (both `lstm_type`s) + `main.py`'s
`nll_loss` / clip / SGD lines and stores inputs and outputs as fixtures under
`tests/golden/`; `tests/test_oracle_golden.py` checks every function below
against them.

Reference lines restated (all in /root/reference):
  Embed.forward            model.py:13-14     -> embed_fwd
  LSTM.lstm_step           model.py:34-45     -> lstm_cell_fwd   (gate order i,f,o,n)
  nn.LSTM (pytorch path)   model.py:84        -> same cell, gate order i,f,g,o
  LSTM.forward             model.py:48-55     -> lstm_layer_fwd
  Linear.forward           model.py:65-68     -> linear_fwd
  Model.forward            model.py:103-110   -> model_fwd (3 dropout sites)
  nll_loss                 main.py:77-84      -> nll_loss, nll_loss_bwd
  clip + SGD               main.py:114-117    -> clip_sgd
  perplexity               main.py:86-95      -> perplexity
  ensemble_nll_loss        ensemble.py:97-109 -> ensemble_nll_loss

Conventions: parameters use the reference's `--lstm_type pytorch` names and
gate order (i,f,g,o); `custom_to_pytorch_gates` converts the custom path's
(i,f,o,n) row blocks.  `dtype` is float32 for "what the reference computes"
and float64 for a tight bound on rounding noise.
"""
from __future__ import annotations

import numpy as np

GATES_PYTORCH = "ifgo"   # torch.nn.LSTM row-block order (rnn.py docs)
GATES_CUSTOM = "ifog"    # model.py:37-42 chunk order (i, f, o, n)


# ----------------------------------------------------------------------------
# parameter helpers
# ----------------------------------------------------------------------------
def param_names(layer_num: int):
    """Registration order of the reference's parameters (model.py:83-86)."""
    names = ["embed.W"]
    for l in range(layer_num):
        names += [f"rnns.{l}.weight_ih_l0", f"rnns.{l}.weight_hh_l0",
                  f"rnns.{l}.bias_ih_l0", f"rnns.{l}.bias_hh_l0"]
    names += ["fc.W", "fc.b"]
    return names


def param_shapes(vocab: int, hidden: int, layer_num: int):
    shp = {"embed.W": (vocab, hidden), "fc.W": (vocab, hidden), "fc.b": (vocab,)}
    for l in range(layer_num):
        shp[f"rnns.{l}.weight_ih_l0"] = (4 * hidden, hidden)
        shp[f"rnns.{l}.weight_hh_l0"] = (4 * hidden, hidden)
        shp[f"rnns.{l}.bias_ih_l0"] = (4 * hidden,)
        shp[f"rnns.{l}.bias_hh_l0"] = (4 * hidden,)
    return shp


def custom_to_pytorch_gates(a: np.ndarray) -> np.ndarray:
    """Row blocks (i,f,o,n) of the custom cell -> (i,f,g,o) of nn.LSTM."""
    i, f, o, n = np.split(a, 4, axis=0)
    return np.concatenate([i, f, n, o], axis=0)


def custom_state_dict_to_pytorch(sd: dict) -> dict:
    """Map `--lstm_type custom` parameter names/gate order to the pytorch path's."""
    out = {}
    for k, v in sd.items():
        v = np.asarray(v)
        if ".W_x" in k:
            out[k.replace("W_x", "weight_ih_l0")] = custom_to_pytorch_gates(v)
        elif ".W_h" in k:
            out[k.replace("W_h", "weight_hh_l0")] = custom_to_pytorch_gates(v)
        elif ".b_x" in k:
            out[k.replace("b_x", "bias_ih_l0")] = custom_to_pytorch_gates(v)
        elif ".b_h" in k:
            out[k.replace("b_h", "bias_hh_l0")] = custom_to_pytorch_gates(v)
        else:
            out[k] = v
    return out


def init_params(vocab, hidden, layer_num, winit, seed, dtype=np.float32):
    """U(-winit, winit) on every parameter (model.py:90-92); numpy RNG, so the
    values differ from torch's for the same seed -- use for self-contained tests."""
    rng = np.random.default_rng(seed)
    shp = param_shapes(vocab, hidden, layer_num)
    return {n: rng.uniform(-winit, winit, size=shp[n]).astype(dtype)
            for n in param_names(layer_num)}


def _sigmoid(z):
    return 1.0 / (1.0 + np.exp(-z))


# ----------------------------------------------------------------------------
# forward pieces
# ----------------------------------------------------------------------------
def embed_fwd(W, x):
    """model.py:13-14  `self.W[x]` : x [T,B] int -> [T,B,H]."""
    return W[np.asarray(x)]


def apply_dropout(a, mask, p):
    """nn.Dropout in train mode (model.py:87,105,108): keep-mask / (1-p).
    `mask` None (eval mode or p == 0) is the identity."""
    if mask is None:
        return a
    return a * (mask.astype(a.dtype) * a.dtype.type(1.0 / (1.0 - p)))


def lstm_cell_fwd(x, h, c, W_ih, W_hh, b_ih, b_hh):
    """model.py:34-45 with nn.LSTM's (i,f,g,o) row blocks.
    x,h,c [B,H]; returns h', c' and the activated gates (for backward)."""
    gates = (x @ W_ih.T + b_ih) + (h @ W_hh.T + b_hh)
    zi, zf, zg, zo = np.split(gates, 4, axis=1)
    i, f, o = _sigmoid(zi), _sigmoid(zf), _sigmoid(zo)
    g = np.tanh(zg)
    c2 = f * c + i * g
    h2 = o * np.tanh(c2)
    return h2, c2, (i, f, g, o)


def lstm_layer_fwd(x, h0, c0, W_ih, W_hh, b_ih, b_hh):
    """model.py:48-55: sequential loop over T.  x [T,B,H]; h0,c0 [B,H]."""
    T = x.shape[0]
    h, c = h0, c0
    ys, cache = [], []
    for t in range(T):
        h_prev, c_prev = h, c
        h, c, (i, f, g, o) = lstm_cell_fwd(x[t], h, c, W_ih, W_hh, b_ih, b_hh)
        ys.append(h)
        cache.append((h_prev, c_prev, i, f, g, o, c))
    return np.stack(ys), h, c, cache


def linear_fwd(x, W, b):
    """model.py:65-68: addmm(b, x.view(-1,H), W.t()) -> [T*B, V]."""
    return x.reshape(-1, x.shape[-1]) @ W.T + b


def model_fwd(params, x, states, layer_num, dropout=0.0, masks=None):
    """model.py:103-110.  `states` = list of (h[B,H], c[B,H]) (the pytorch
    path's leading 1 is squeezed).  `masks` = None (eval) or a list of
    layer_num+1 boolean keep-masks [T,B,H], one per dropout site in call
    order (after embed, after each layer).  Returns scores [T*B,V], new
    states, cache."""
    dt = params["embed.W"].dtype
    a = embed_fwd(params["embed.W"], x)
    site = 0
    acts = {"emb": a}
    a = apply_dropout(a, None if masks is None else masks[site], dropout)
    new_states, layer_cache, layer_in = [], [], []
    for l in range(layer_num):
        layer_in.append(a)
        h0, c0 = states[l]
        y, h, c, cache = lstm_layer_fwd(
            a, h0.astype(dt), c0.astype(dt),
            params[f"rnns.{l}.weight_ih_l0"], params[f"rnns.{l}.weight_hh_l0"],
            params[f"rnns.{l}.bias_ih_l0"], params[f"rnns.{l}.bias_hh_l0"])
        new_states.append((h, c))
        layer_cache.append(cache)
        site += 1
        a = apply_dropout(y, None if masks is None else masks[site], dropout)
    scores = linear_fwd(a, params["fc.W"], params["fc.b"])
    cache = {"x": np.asarray(x), "layer_in": layer_in, "layer_cache": layer_cache,
             "fc_in": a, "masks": masks, "dropout": dropout}
    return scores, new_states, cache


# ----------------------------------------------------------------------------
# loss
# ----------------------------------------------------------------------------
def nll_loss(scores, y):
    """main.py:77-84: naive softmax (no max subtraction), target prob,
    mean(-log p * batch_size).  y [T,B], flattened t-major."""
    B = y.shape[1]
    e = np.exp(scores)
    p = e / e.sum(axis=1, keepdims=True)
    yy = np.asarray(y).reshape(-1)
    ans = p[np.arange(yy.shape[0]), yy]
    return np.mean(-np.log(ans) * B)


def nll_loss_bwd(scores, y):
    """d loss / d scores = (softmax - onehot) * B / N  (= /T)."""
    B = y.shape[1]
    yy = np.asarray(y).reshape(-1)
    N = yy.shape[0]
    m = scores.max(axis=1, keepdims=True)
    e = np.exp(scores - m)
    p = e / e.sum(axis=1, keepdims=True)
    p[np.arange(N), yy] -= 1.0
    return p * scores.dtype.type(B / N)


def target_probs(scores, y):
    """softmax(scores)[n, y_n] -- what the ensemble path averages
    (ensemble.py:100-106: mean of probabilities, then index)."""
    yy = np.asarray(y).reshape(-1)
    m = scores.max(axis=1, keepdims=True)
    e = np.exp(scores - m)
    return e[np.arange(yy.shape[0]), yy] / e.sum(axis=1)


def ensemble_nll_loss(scores_list, y):
    """ensemble.py:97-109: mean over models of softmax probabilities, NLL."""
    B = y.shape[1]
    pbar = np.mean([target_probs(s, y) for s in scores_list], axis=0)
    return np.mean(-np.log(pbar) * B)


# ----------------------------------------------------------------------------
# backward (what autograd derives for model.py:103-110; SURVEY.md section 8a)
# ----------------------------------------------------------------------------
def lstm_layer_bwd(dy, cache, x, W_ih, W_hh, record=None):
    """dy [T,B,H] upstream grad on the layer's outputs.  States entering the
    window are detached (model.py:100-101) so no grad flows past t=0.
    Returns dx, dW_ih, dW_hh, db (db_ih == db_hh).  `record` (a dict or None)
    receives "dG": the gate gradients d loss / d preactivation [T,B,4H]."""
    T, B, H = dy.shape
    dt = dy.dtype
    dW_ih = np.zeros_like(W_ih)
    dW_hh = np.zeros_like(W_hh)
    db = np.zeros(4 * H, dtype=dt)
    dx = np.zeros_like(x)
    dh_rec = np.zeros((B, H), dtype=dt)
    dc = np.zeros((B, H), dtype=dt)
    if record is not None:
        record["dG"] = np.zeros((T, B, 4 * H), dtype=dt)
    for t in range(T - 1, -1, -1):
        h_prev, c_prev, i, f, g, o, c = cache[t]
        dh = dy[t] + dh_rec
        tc = np.tanh(c)
        do = dh * tc
        dc = dc + dh * o * (1.0 - tc * tc)
        di = dc * g
        dg = dc * i
        df = dc * c_prev
        dG = np.concatenate([di * i * (1.0 - i), df * f * (1.0 - f),
                             dg * (1.0 - g * g), do * o * (1.0 - o)], axis=1)
        if record is not None:
            record["dG"][t] = dG
        dc = dc * f
        dx[t] = dG @ W_ih
        dh_rec = dG @ W_hh
        dW_ih += dG.T @ x[t]
        dW_hh += dG.T @ h_prev
        db += dG.sum(axis=0)
    return dx, dW_ih, dW_hh, db


def model_bwd(params, cache, dscores, layer_num, record=None):
    """Gradients of every parameter given d loss / d scores [T*B,V].  `record`
    (a dict or None) receives, per layer l, record[l] = {"dy": the gradient
    reaching the layer's outputs [T,B,H], "dG": its gate gradients [T,B,4H]}."""
    p = cache["dropout"]
    masks = cache["masks"]
    fc_in = cache["fc_in"]
    T, B, H = fc_in.shape
    grads = {}
    flat = fc_in.reshape(-1, H)
    grads["fc.W"] = dscores.T @ flat
    grads["fc.b"] = dscores.sum(axis=0)
    da = (dscores @ params["fc.W"]).reshape(T, B, H)
    for l in range(layer_num - 1, -1, -1):
        da = apply_dropout(da, None if masks is None else masks[l + 1], p)
        rec = None
        if record is not None:
            rec = record[l] = {"dy": da}
        dx, dWi, dWh, db = lstm_layer_bwd(
            da, cache["layer_cache"][l], cache["layer_in"][l],
            params[f"rnns.{l}.weight_ih_l0"], params[f"rnns.{l}.weight_hh_l0"], rec)
        grads[f"rnns.{l}.weight_ih_l0"] = dWi
        grads[f"rnns.{l}.weight_hh_l0"] = dWh
        grads[f"rnns.{l}.bias_ih_l0"] = db
        grads[f"rnns.{l}.bias_hh_l0"] = db.copy()
        da = dx
    da = apply_dropout(da, None if masks is None else masks[0], p)
    dE = np.zeros_like(params["embed.W"])
    np.add.at(dE, cache["x"].reshape(-1), da.reshape(-1, H))
    grads["embed.W"] = dE
    return grads


# ----------------------------------------------------------------------------
# optimizer step (caller side of the hot path)
# ----------------------------------------------------------------------------
def global_grad_norm(grads, names):
    tot = 0.0
    for n in names:
        tot += float(np.sum(grads[n].astype(np.float64) ** 2))
    return np.sqrt(tot)


def clip_sgd(params, grads, lr, max_norm, names):
    """main.py:114-117: clip_grad_norm_ (coef = max_norm/(norm+1e-6), clamped
    to 1) over all parameters, then p -= lr * g.  In place; returns the norm."""
    norm = global_grad_norm(grads, names)
    coef = min(1.0, max_norm / (norm + 1e-6))
    for n in names:
        dt = params[n].dtype
        grads[n] = (grads[n] * dt.type(coef)).astype(dt)
        params[n] -= dt.type(lr) * grads[n]
    return norm


def train_step(params, x, y, states, layer_num, lr, max_norm, dropout=0.0, masks=None):
    """One iteration of main.py:109-117 (zero_grad, detach, fwd, loss, bwd, clip, SGD)."""
    names = param_names(layer_num)
    scores, new_states, cache = model_fwd(params, x, states, layer_num, dropout, masks)
    loss = nll_loss(scores, y)
    dscores = nll_loss_bwd(scores, y)
    grads = model_bwd(params, cache, dscores, layer_num)
    norm = clip_sgd(params, grads, lr, max_norm, names)
    return loss, norm, new_states, scores, grads


def zero_states(layer_num, batch, hidden, dtype=np.float32):
    """model.py:94-98 (leading 1 of the pytorch layout squeezed)."""
    return [(np.zeros((batch, hidden), dtype), np.zeros((batch, hidden), dtype))
            for _ in range(layer_num)]


def perplexity(params, batches, layer_num, batch_size, hidden):
    """main.py:86-95: eval mode, fresh zero state carried across batches,
    exp(mean_batches(loss / B))."""
    dt = params["embed.W"].dtype
    states = zero_states(layer_num, batch_size, hidden, dt)
    losses = []
    for x, y in batches:
        scores, states, _ = model_fwd(params, x, states, layer_num)
        losses.append(nll_loss(scores, y) / batch_size)
    return float(np.exp(np.mean(losses)))


def minibatch(data, batch_size, seq_length):
    """main.py:61-74: corpus [n] -> list of (x[T,B], y[T,B]); a trailing
    window is kept only if a full target window follows it."""
    data = np.asarray(data).reshape(-1)
    nb = data.shape[0] // batch_size
    d = data[: nb * batch_size].reshape(batch_size, -1)
    out = []
    L = d.shape[1]
    for i in range(0, L - 1, seq_length):
        seqlen = min(seq_length, L - 1 - i)
        if seqlen < L - 1 - i:
            out.append((d[:, i:i + seqlen].T, d[:, i + 1:i + seqlen + 1].T))
    return out
