"""A Medium model trained for one epoch on the Penn Treebank ids, and the comparisons of the kernels against the fp64
oracle at its weights  --  TEST INFRASTRUCTURE (tests/test_gpu_trained_regime.py, tools/measure_trained_error.py).

At init the gates sit near 0.5, |c| stays below ~1 and the softmax is almost flat.  A trained model saturates its gates,
lets |c| reach several units to tens and puts most of the vocabulary below 1e-6: the regime where the fixed-scale fp16
gradient images (kGradScale = 1024: dS and dG held as 1024 * value) go subnormal and the SFU activations of the
persistent kernels differ most from expf / tanhf.  Every function here returns plain numbers so that the test asserts
them and the tool prints them.
"""
from __future__ import annotations

import ctypes as C
import os
import time

import numpy as np
import torch

from oracle import lstm_lm_oracle as O
from tests._golden import GOLDEN
from tests._rounded_oracle import rounded_operand_fwd

MEDIUM = dict(V=10000, H=650, L=2, T=35, B=20, p=0.5, winit=0.05, lr=1.0, clip=5.0)    # bench.py CONFIGS["medium"]
SMALL = dict(V=10000, H=200, L=2, T=20, B=20, p=0.0, winit=0.1, lr=1.0, clip=5.0)      # bench.py CONFIGS["small"]
GRAD_SCALE = 1024.0          # tc_kernels.h kGradScale
F16_MAX = 65504.0
F16_MIN_NORMAL = 2.0 ** -14
CARRY = 3                    # valid windows run before the compared one, so that the incoming (h, c) are not zero
LONG_T = 140                 # the unit-level long window: four valid windows back to back
DEV = "cuda:0"


def ptb_splits():
    z = np.load(os.path.join(GOLDEN, "ptb_ids.npz"))
    return z["train"].astype(np.int64).reshape(-1, 1), z["valid"].astype(np.int64).reshape(-1, 1)


def _model(c, engine, params=None, V=None):
    import zaremba_b200
    m = zaremba_b200.Model(V or c["V"], c["H"], c["L"], c["p"], c["winit"], engine=engine)
    if params is not None:
        m.load_state_dict({k: torch.tensor(v) for k, v in params.items()})
    return m.to(DEV)


def train(c, engine="tc", steps=None, seed=0, lazy=True):
    """`steps` fused train steps (None: one epoch) over the train split from init (torch seed `seed`), the way bench.py
    runs them.  Returns the flushed fp32 weights, valid perplexity at init and after, the per-step losses and seconds."""
    import zaremba_b200
    trn, vld = ptb_splits()
    B, T = c["B"], c["T"]
    torch.manual_seed(seed)
    m = _model(c, engine)
    tr = zaremba_b200.Trainer(m, B, T, lazy_update=lazy)
    vb = zaremba_b200.minibatch(vld, B, T)
    m.eval()
    ppl0 = tr.perplexity(vb)
    tb = zaremba_b200.minibatch(trn, B, T)
    n = len(tb) if steps is None else steps
    X = torch.stack([x for x, _ in tb[:n]]).contiguous().to(DEV)
    Y = torch.stack([y for _, y in tb[:n]]).contiguous().to(DEV)
    m.train()
    tr.reset_states()
    losses = torch.zeros(n, device=DEV)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(n):
        loss, _ = tr.train_step(X[i], Y[i], c["lr"], c["clip"])
        losses[i] = loss / B
    tr.flush()
    torch.cuda.synchronize()
    secs = time.perf_counter() - t0
    m.eval()
    ppl1 = tr.perplexity(vb)
    params = {k: v.detach().cpu().numpy().copy() for k, v in m.named_parameters()}
    return dict(params=params, ppl_init=ppl0, ppl=ppl1, steps=n, seconds=secs, losses=losses.cpu().numpy())


class Point:
    """The trained weights, the compared valid window (after CARRY carried ones), its incoming states, and the fp64
    oracle's eval-mode and train-mode (explicit masks) passes over it."""

    def __init__(self, params, c=MEDIUM, seed=1):
        import zaremba_b200
        self.c, self.params = c, params
        self.p64 = {k: v.astype(np.float64) for k, v in params.items()}
        V, H, L, T, B = (c[k] for k in "VHLTB")
        _, vld = ptb_splits()
        vb = zaremba_b200.minibatch(vld, B, T)
        # carry: the tensor-core engine's eval steps from zero states
        m = _model(c, "tc", params)
        m.eval()
        tr = zaremba_b200.Trainer(m, B, T)
        for x, y in vb[:CARRY]:
            tr.eval_step(x.to(DEV).contiguous(), y.to(DEV).contiguous())
        self.states = [(h.reshape(B, H).cpu().numpy().copy(), cc.reshape(B, H).cpu().numpy().copy())
                       for h, cc in tr.states]
        del tr, m
        self.x, self.y = (a.numpy().copy() for a in vb[CARRY])
        self.x_long = np.concatenate([vb[CARRY + i][0].numpy() for i in range(LONG_T // T)])
        self.y_long = np.concatenate([vb[CARRY + i][1].numpy() for i in range(LONG_T // T)])
        st64 = [(h.astype(np.float64), cc.astype(np.float64)) for h, cc in self.states]
        # eval mode
        self.scores, self.states_out, self.cache = O.model_fwd(self.p64, self.x, st64, L)
        self.loss = O.nll_loss(self.scores, self.y)
        self.tp = O.target_probs(self.scores, self.y)
        self.dS = O.nll_loss_bwd(self.scores, self.y)
        self.grads = O.model_bwd(self.p64, self.cache, self.dS, L)
        self.rec = layer_grads(self.p64, self.cache, self.dS, L)
        # train mode, explicit keep-masks
        rng = np.random.default_rng(seed)
        self.masks = [rng.random((T, B, H)) >= c["p"] for _ in range(L + 1)]
        sc, _, cache = O.model_fwd(self.p64, self.x, st64, L, c["p"], self.masks)
        self.train_loss = O.nll_loss(sc, self.y)
        self.train_dS = O.nll_loss_bwd(sc, self.y)
        self.train_grads = O.model_bwd(self.p64, cache, self.train_dS, L)
        self.train_rec = layer_grads(self.p64, cache, self.train_dS, L)
        # long window (unit-level layers): eval mode over LONG_T steps from the same incoming states
        sc, _, cache = O.model_fwd(self.p64, self.x_long, st64, L)
        self.long_rec = layer_grads(self.p64, cache, O.nll_loss_bwd(sc, self.y_long), L)
        self.long_cache = cache

    def regime(self):
        """How far from init the point is: each number is a floor of the test."""
        L, T = self.c["L"], self.c["T"]
        sat = []
        cmax = 0.0
        for l in range(L):
            for (_, _, i, f, g, o, cc) in self.cache["layer_cache"][l]:
                s5, t5 = 1.0 / (1.0 + np.exp(-5.0)), np.tanh(5.0)     # |z| > 5 <=> sigma(z) outside (s(-5), s(5))
                sat += [np.abs(a - 0.5) > s5 - 0.5 for a in (i, f, o)] + [np.abs(g) > t5]
                cmax = max(cmax, float(np.abs(cc).max()))
        sat = np.concatenate([a.reshape(-1) for a in sat])
        e = np.exp(self.scores - self.scores.max(axis=1, keepdims=True))
        p = e / e.sum(axis=1, keepdims=True)
        dG = np.concatenate([self.rec[l]["dG"].reshape(-1) for l in range(L)] +
                            [self.train_rec[l]["dG"].reshape(-1) for l in range(L)])
        img = np.abs(dG) * GRAD_SCALE
        dsub = F16_MIN_NORMAL * T / GRAD_SCALE                    # p below this: the dS image is subnormal
        return {"frac_preact_gt5": float(sat.mean()), "max_abs_c": cmax,
                "median_target_prob": float(np.median(self.tp)),
                "frac_softmax_dS_subnormal": float((p < dsub).mean()),
                "frac_dG_image_subnormal": float(((img < F16_MIN_NORMAL) & (img > 0)).mean()),
                "max_dS_image": float(max(np.abs(self.dS).max(), np.abs(self.train_dS).max()) * GRAD_SCALE),
                "max_dG_image": float(img.max())}


def gate_grads(dy, layer_cache, W_hh):
    """d loss / d pre-activation [T,B,4H] of one layer (gate order i,f,g,o) given the gradient dy [T,B,H] reaching its
    outputs: the recurrence of O.lstm_layer_bwd, restated for the quantity it does not return."""
    T, B, H = dy.shape
    dG = np.zeros((T, B, 4 * H))
    dh_rec, dc = np.zeros((B, H)), np.zeros((B, H))
    for t in range(T - 1, -1, -1):
        _, c_prev, i, f, g, o, c = layer_cache[t]
        dh = dy[t] + dh_rec
        tc = np.tanh(c)
        dc = dc + dh * o * (1.0 - tc * tc)
        dG[t] = np.concatenate([dc * g * i * (1.0 - i), dc * c_prev * f * (1.0 - f), dc * i * (1.0 - g * g),
                                dh * tc * o * (1.0 - o)], axis=1)
        dc = dc * f
        dh_rec = dG[t] @ W_hh
    return dG


def layer_grads(p64, cache, dS, L):
    """Per layer l: {"dy": the gradient reaching its outputs (after its output dropout), "dG": its gate gradients}, for
    the oracle pass `cache` (O.model_fwd) and d loss / d scores `dS` -- what O.model_bwd passes down the stack."""
    T, B, H = cache["fc_in"].shape
    masks, p = cache["masks"], cache["dropout"]
    da = (dS @ p64["fc.W"]).reshape(T, B, H)
    out = {}
    for l in range(L - 1, -1, -1):
        da = O.apply_dropout(da, None if masks is None else masks[l + 1], p)
        dG = gate_grads(da, cache["layer_cache"][l], p64[f"rnns.{l}.weight_hh_l0"])
        out[l] = {"dy": da, "dG": dG}
        da = dG @ p64[f"rnns.{l}.weight_ih_l0"]
    return out


def rel(got, want):
    """(max-abs error / max-abs reference, ||error||_2 / ||reference||_2)."""
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=np.float64)
    d = got - want
    return (float(np.abs(d).max() / max(np.abs(want).max(), 1e-30)),
            float(np.linalg.norm(d) / max(np.linalg.norm(want), 1e-30)))


def row_rel(got, want, floor=1e-3):
    """Largest ||error_r|| / ||reference_r|| over the rows whose reference norm is at least `floor` of the largest row's."""
    got = np.asarray(got, dtype=np.float64).reshape(want.shape[0], -1)
    want = np.asarray(want, dtype=np.float64).reshape(want.shape[0], -1)
    nr = np.linalg.norm(want, axis=1)
    keep = nr >= floor * nr.max()
    return float((np.linalg.norm(got - want, axis=1)[keep] / nr[keep]).max()), int(keep.sum())


def _dev_states(pt, shape):
    return [(torch.tensor(h).view(shape).to(DEV), torch.tensor(cc).view(shape).to(DEV)) for h, cc in pt.states]


def eval_forward(pt, engine):
    """Eval mode at the trained point: logits (drop-in forward), loss, target probabilities and final states (the
    fused eval step), each against the fp64 oracle."""
    import zaremba_b200
    c = pt.c
    V, H, L, T, B = (c[k] for k in "VHLTB")
    x, y = torch.tensor(pt.x).to(DEV).contiguous(), torch.tensor(pt.y).to(DEV).contiguous()
    m = _model(c, engine, pt.params)
    m.eval()
    with torch.no_grad():
        scores, _ = m(x, _dev_states(pt, (1, B, H)))
    out = {"logits": rel(scores.cpu().numpy(), pt.scores)}
    m2 = _model(c, engine, pt.params)
    m2.eval()
    tr = zaremba_b200.Trainer(m2, B, T)
    for l, (h, cc) in enumerate(pt.states):
        tr.states[l][0].copy_(torch.tensor(h).view_as(tr.states[l][0]))
        tr.states[l][1].copy_(torch.tensor(cc).view_as(tr.states[l][1]))
    loss, tp = tr.eval_step(x, y, want_probs=True)
    out["loss"] = abs(loss.item() - pt.loss) / pt.loss
    tpd = tp.cpu().numpy().astype(np.float64)
    out["target_probs"] = rel(tpd, pt.tp)
    out["target_probs_elementwise"] = float((np.abs(tpd - pt.tp) / pt.tp).max())
    for l in range(L):
        out[f"h{l}"] = rel(tr.states[l][0].reshape(B, H).cpu().numpy(), pt.states_out[l][0])
        out[f"c{l}"] = rel(tr.states[l][1].reshape(B, H).cpu().numpy(), pt.states_out[l][1])
    return out


def _grad_errors(got, want):
    out = {k: rel(got[k], want[k]) for k in want}
    for k in ("fc.W", "embed.W"):
        out[f"{k} rows"] = row_rel(got[k], want[k])
    return out


def train_grads(pt, engine):
    """One fused train step's gradients (zrb_train_step_grads, the softmax kernel writes the dS image) with explicit
    dropout masks, against the oracle's train-mode pass.  Returns (loss error, {tensor: errors})."""
    import zaremba_b200
    from zaremba_b200 import _lib
    lib = _lib.load()
    c = pt.c
    T, B = c["T"], c["B"]
    m = _model(c, engine, pt.params)
    m.train()
    tr = zaremba_b200.Trainer(m, B, T)
    m.set_explicit_dropout_masks([torch.tensor(mk.astype(np.uint8)).to(DEV) for mk in pt.masks])
    for l, (h, cc) in enumerate(pt.states):
        tr.states[l][0].copy_(torch.tensor(h).view_as(tr.states[l][0]))
        tr.states[l][1].copy_(torch.tensor(cc).view_as(tr.states[l][1]))
    x, y = torch.tensor(pt.x).to(DEV).contiguous(), torch.tensor(pt.y).to(DEV).contiguous()
    _lib.check(lib.zrb_train_step_grads(tr.ctx, C.byref(tr._ps), C.byref(tr._gs), _lib.ptr(x), _lib.ptr(y), T, B,
                                        C.byref(tr._st), C.byref(tr._st), tr.seed, tr.step, _lib.ptr(tr.loss),
                                        tr._stream()))
    torch.cuda.synchronize()
    got = {k: p.grad.detach().cpu().numpy() for k, p in m.named_parameters()}
    return abs(tr.loss.item() - pt.train_loss) / pt.train_loss, _grad_errors(got, pt.train_grads)


def eval_grads(pt, engine):
    """The eval-mode gradient through the drop-in Model (zrb_forward + zrb_backward: the caller's dscores are converted
    into the dS image), against the oracle's eval-mode pass."""
    from tests.test_gpu_parity import _caller_nll_loss
    c = pt.c
    H, B = c["H"], c["B"]
    m = _model(c, engine, pt.params)
    m.eval()
    scores, _ = m(torch.tensor(pt.x), _dev_states(pt, (1, B, H)))
    _caller_nll_loss(scores, torch.tensor(pt.y)).backward()
    got = {k: p.grad.detach().cpu().numpy() for k, p in m.named_parameters()}
    return _grad_errors(got, pt.grads)


def layer_unit(pt, T):
    """Each trained layer alone through zrb_lstm_layer_fwd / _bwd (a context created for max_seq = LONG_T) on its real
    input activations and incoming states over the first T steps of the long window, against O.lstm_layer_fwd / _bwd.
    dy is the real gradient reaching the layer over the long window (its first T steps)."""
    import zaremba_b200
    from zaremba_b200 import _lib
    lib = _lib.load()
    c = pt.c
    H, L, B = c["H"], c["L"], c["B"]
    m = zaremba_b200.Model(16, H, 1, 0.0, 0.05, engine="tc").to(DEV)
    ctx = m._context(LONG_T, B)
    out = {}
    for l in range(L):
        W_ih, W_hh = pt.params[f"rnns.{l}.weight_ih_l0"], pt.params[f"rnns.{l}.weight_hh_l0"]
        b_ih, b_hh = pt.params[f"rnns.{l}.bias_ih_l0"], pt.params[f"rnns.{l}.bias_hh_l0"]
        x = pt.long_cache["layer_in"][l][:T]
        dy = pt.long_rec[l]["dy"][:T]
        h0, c0 = pt.states[l]
        out.update({f"l{l} {k}": v for k, v in layer_against_oracle(lib, ctx, W_ih, W_hh, b_ih, b_hh, x, h0, c0, dy).items()})
    return out


def layer_against_oracle(lib, ctx, W_ih, W_hh, b_ih, b_hh, x, h0, c0, dy):
    """zrb_lstm_layer_fwd + _bwd on ctx; errors (rel) of y, hT, cT, dx, dW_ih, dW_hh, db against the fp64 oracle on the
    fp32 values the device received."""
    from zaremba_b200 import _lib
    T, B, H = x.shape
    f32 = lambda a: np.asarray(a).astype(np.float32)
    dev = lambda a: torch.tensor(f32(a)).contiguous().to(DEV)
    d = {k: dev(v) for k, v in dict(W_ih=W_ih, W_hh=W_hh, b_ih=b_ih, b_hh=b_hh, x=x, h0=h0, c0=c0, dy=dy).items()}
    y, hT, cT = (torch.empty(n, H, device=DEV) for n in (T * B, B, B))
    _lib.check(lib.zrb_lstm_layer_fwd(ctx, _lib.ptr(d["W_ih"]), _lib.ptr(d["W_hh"]), _lib.ptr(d["b_ih"]),
                                      _lib.ptr(d["b_hh"]), _lib.ptr(d["x"]), T, B, _lib.ptr(d["h0"]), _lib.ptr(d["c0"]),
                                      _lib.ptr(y), _lib.ptr(hT), _lib.ptr(cT), None))
    g = lambda a: f32(a).astype(np.float64)
    ys, h_ref, c_ref, cache = O.lstm_layer_fwd(g(x), g(h0), g(c0), g(W_ih), g(W_hh), g(b_ih), g(b_hh))
    dx, dWi, dWh = torch.empty(T * B, H, device=DEV), torch.empty(4 * H, H, device=DEV), torch.empty(4 * H, H, device=DEV)
    dbi, dbh = torch.empty(4 * H, device=DEV), torch.empty(4 * H, device=DEV)
    _lib.check(lib.zrb_lstm_layer_bwd(ctx, _lib.ptr(d["dy"]), _lib.ptr(dx), _lib.ptr(dWi), _lib.ptr(dWh), _lib.ptr(dbi),
                                      _lib.ptr(dbh), None))
    dx_r, dWi_r, dWh_r, db_r = O.lstm_layer_bwd(g(dy), cache, g(x), g(W_ih), g(W_hh))
    rec = {"dG": gate_grads(g(dy), cache, g(W_hh))}
    torch.cuda.synchronize()
    yd, cd = y.cpu().numpy().reshape(T, B, H).astype(np.float64), cT.cpu().numpy().astype(np.float64)
    y_r, c_r, zmax = rounded_operand_fwd(g(x), g(h0), g(c0), g(W_ih), g(W_hh), g(b_ih), g(b_hh), yd)
    return {"rounded-operand y": float(np.abs(yd - y_r).max()),
            "rounded-operand cT": float(np.abs(cd - c_r).max() / max(np.abs(c_r).max(), 1.0)),
            "max_abs_preact": zmax, "y": rel(y.cpu().numpy().reshape(T, B, H), ys), "hT": rel(hT.cpu().numpy(), h_ref),
            "cT": rel(cT.cpu().numpy(), c_ref), "grad dx": rel(dx.cpu().numpy().reshape(T, B, H), dx_r),
            "grad dW_ih": rel(dWi.cpu().numpy(), dWi_r), "grad dW_hh": rel(dWh.cpu().numpy(), dWh_r),
            "grad db": rel(dbi.cpu().numpy(), db_r), "db_ih == db_hh": float(torch.equal(dbi, dbh)),
            "max_abs_c": float(max(np.abs(e[6]).max() for e in cache)),
            "max_dG_image": float(np.abs(rec["dG"]).max() * GRAD_SCALE),
            "frac_dG_image_subnormal": float(((np.abs(rec["dG"]) * GRAD_SCALE < F16_MIN_NORMAL)
                                              & (rec["dG"] != 0)).mean())}


def softmax_nll(pt, V):
    """zrb_softmax_nll at the trained logits (the oracle's, rounded to fp32) on the first V columns: V % 4 == 0 takes the
    register-resident kernel, otherwise the scalar one.  Targets at or beyond V are moved to column 0."""
    import zaremba_b200
    from zaremba_b200 import _lib
    lib = _lib.load()
    T, B = pt.c["T"], pt.c["B"]
    s = pt.scores[:, :V].astype(np.float32)
    y = np.where(pt.y < V, pt.y, 0)
    m = zaremba_b200.Model(V, 8, 1, 0.0, 0.1, engine="simt").to(DEV)
    ctx = m._context(T, B)
    sd, yd = torch.tensor(s).to(DEV), torch.tensor(y).to(DEV)
    loss = torch.zeros((), device=DEV)
    ds = torch.empty_like(sd)
    tp = torch.empty(T * B, device=DEV)
    _lib.check(lib.zrb_softmax_nll(ctx, _lib.ptr(sd), _lib.ptr(yd), T, B, _lib.ptr(loss), _lib.ptr(ds), _lib.ptr(tp),
                                   None))
    s64 = s.astype(np.float64)
    want = O.nll_loss(s64, y)
    want_tp = O.target_probs(s64, y)
    tpd = tp.cpu().numpy().astype(np.float64)
    return {"loss": abs(loss.item() - want) / want, "dscores": rel(ds.cpu().numpy(), O.nll_loss_bwd(s64, y)),
            "dscores rows": row_rel(ds.cpu().numpy(), O.nll_loss_bwd(s64, y), 0.0),
            "target_probs": rel(tpd, want_tp), "target_probs_elementwise": float((np.abs(tpd - want_tp) / want_tp).max())}


def sampler(pt, rows=200, seed=0x0123456789ABCDEF, pos=2 ** 32 + 7):
    """zrb_sample at the trained logits against oracle/sampling.py (top-p 0.9 / 0.95, top-k 40; temperature 1).
    Returns per setting: rows, token mismatches outside the oracle's tie / boundary margins, near-tie mismatches, the
    worst logprob error (relative beyond 1) and how many rows keep at most two entries."""
    from oracle import sampling as S
    from zaremba_b200 import _lib
    from zaremba_b200.sampling import sampling_config
    lib = _lib.load()
    V = pt.c["V"]
    z = pt.scores[:rows].astype(np.float32)
    buf = torch.tensor(z).to(DEV)
    u = [S.uniforms(seed, pos, b, V) for b in range(rows)]
    out = {}
    for top_k, top_p in ((0, 0.9), (0, 0.95), (40, 1.0)):
        cfg = sampling_config(1.0, top_k, top_p, seed)
        tok = torch.empty(rows, dtype=torch.int64, device=DEV)
        lp = torch.empty(rows, dtype=torch.float32, device=DEV)
        _lib.check(lib.zrb_sample(_lib.ptr(buf), V, rows, V, C.byref(cfg), pos, _lib.ptr(tok), _lib.ptr(lp), None))
        tok, lp = tok.cpu().numpy(), lp.cpu().numpy()
        bad = near = small = 0
        worst = 0.0
        for b in range(rows):
            want, want_lp, info = S.sample_row(z[b], 1.0, top_k, top_p, seed, pos, b, u=u[b])
            small += int(S.kept(z[b], 1.0, top_k, top_p)[0].sum() <= 2)
            if tok[b] != want:
                p32 = float(np.float32(top_p))
                tie = info["gap"] < 1e-5 * (1 + abs(info["smax"]))
                edge = any(mm is not None and abs(mm - p32) < 1e-5 for mm in info["boundary"])
                near += int(tie or edge)
                bad += int(not (tie or edge))
                want_lp = S.log_softmax_at(z[b], int(tok[b]))
            worst = max(worst, abs(float(lp[b]) - want_lp) / max(1.0, abs(want_lp)))
        out[f"top_k={top_k} top_p={top_p}"] = {"rows": rows, "bad": bad, "near": near, "logprob_err": worst,
                                               "rows_keeping_le2": small}
    return out


def trajectory(steps, seed=0):
    """Part C: the Small recipe (dropout 0) trained from one init with the tensor-core engine (lazy update, as bench.py)
    and with the fp32 validation engine on the same PTB windows.  Returns both runs' last-50-step mean loss, valid
    perplexity and seconds."""
    out = {}
    for engine in ("tc", "simt"):
        r = train(SMALL, engine, steps=steps, seed=seed, lazy=engine == "tc")
        out[engine] = {"last50_loss": float(r["losses"][-50:].mean()), "first_loss": float(r["losses"][0]),
                       "ppl": r["ppl"], "ppl_init": r["ppl_init"], "seconds": r["seconds"]}
    out["last50_loss_rel_gap"] = abs(out["tc"]["last50_loss"] - out["simt"]["last50_loss"]) / out["simt"]["last50_loss"]
    out["ppl_rel_gap"] = abs(out["tc"]["ppl"] - out["simt"]["ppl"]) / out["simt"]["ppl"]
    return out
