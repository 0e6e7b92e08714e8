"""Layers of unequal width (DESIGN.md section 18) through the tensor-core engine, against the fp64 restatement in
tests/_model_oracle.py, and the equal-width path through zrb_ctx_create_widths against zrb_ctx_create, bit for bit.

Shapes: AWD-LSTM's PTB model (E = 400, 1150-1150-400, tied), a growing stack (E = 200, 650-1500), the recurrence-plan
branches (H < 256 unsplit, K-split, pitches that are not multiples of 64), the per-timestep path (B = 40) and one layer
with E != H_0.  Every weight-gradient launch of these shapes is a dual GEMM whose two problems differ in N (dW_ih is
[4H_l, In_l], dW_hh [4H_l, H_l]), so the raw gradients and the fused clip norm check that launch against fp64.
"""
import numpy as np
import pytest
import torch

from tests import _model_oracle as O
from tests.test_gpu_parity import NORM_TOL, TOL

pytestmark = pytest.mark.gpu

SHAPES = {   # V, E, layer widths, T, B, tied
    "awd": (10000, 400, (1150, 1150, 400), 70, 20, True),
    "growing": (10000, 200, (650, 1500), 35, 20, False),
    "branches": (500, 72, (40, 200, 300), 5, 8, False),
    "steps": (500, 48, (64, 96), 5, 40, False),
    "one_layer": (500, 100, (200,), 5, 4, False),
}
LR, MAX_NORM, WINIT = 1.0, 0.25, 0.1
# states after a window: the error of the fp16 recurrent operand accumulates over the window's steps, and the second
# window starts from parameters that already differ within TOL["tc"]["grad"].  TOL["tc"] was set at T <= 35 with Large's
# winit = 0.04; here winit = 0.1 at widths up to 1500 (pre-activations 2.5x larger) and AWD's window is T = 70
STATE_TOL = {35: 5e-3, 70: 5e-3}


def _close(got, want, rel, what):
    got = torch.as_tensor(got).double().cpu()
    want = torch.as_tensor(want).double().cpu()
    scale = max(float(want.abs().max()), 1e-6)
    err = float((got - want).abs().max())
    assert err <= rel * scale, f"{what}: max abs err {err:.3e} vs scale {scale:.3e} (rel {err / scale:.2e} > {rel:.1e})"


def _model(name, winit=WINIT, **kw):
    import zaremba_b200
    V, E, sizes, T, B, tied = SHAPES[name]
    torch.manual_seed(7)
    m = zaremba_b200.Model(V, sizes[0], len(sizes), kw.pop("dropout", 0.0), winit, tied=tied, embed_size=E,
                           layer_sizes=sizes, **kw).cuda()
    return m


def _data(name, steps, seed=11):
    V, E, sizes, T, B, tied = SHAPES[name]
    g = torch.Generator().manual_seed(seed)
    xs = [torch.randint(0, V, (T, B), generator=g).cuda() for _ in range(steps)]
    ys = [torch.randint(0, V, (T, B), generator=g).cuda() for _ in range(steps)]
    return xs, ys


def _params64(m):
    return {k: v.detach().double().clone() for k, v in m.named_parameters()}


def _random_states(tr, seed=5):
    g = torch.Generator().manual_seed(seed)
    for h, c in tr.states:
        h.copy_(0.2 * torch.randn(h.shape, generator=g).cuda())
        c.copy_(0.2 * torch.randn(c.shape, generator=g).cuda())


@pytest.mark.parametrize("name", list(SHAPES))
def test_fused_steps_match_oracle(name):
    """Two carried fused train steps: loss, clip norm, parameters and states after; then eval_step and the plans."""
    import zaremba_b200
    V, E, sizes, T, B, tied = SHAPES[name]
    m = _model(name)
    m.train()
    tr = zaremba_b200.Trainer(m, B, T)
    _random_states(tr)
    params = _params64(m)
    states = [(h.detach().double().reshape(B, -1).clone(), c.detach().double().reshape(B, -1).clone())
              for h, c in tr.states]
    assert [s[0].shape[1] for s in states] == list(sizes)
    xs, ys = _data(name, 3)
    tol = TOL["tc"]
    for s in range(2):
        loss, norm = tr.train_step(xs[s], ys[s], LR, MAX_NORM)
        tr.flush()
        torch.cuda.synchronize()
        want_loss, want_norm, grads, params, states, _ = O.train_step(params, xs[s], ys[s], states, len(sizes), tied,
                                                                     LR, MAX_NORM)
        assert abs(loss.item() - want_loss) <= tol["loss"] * max(1.0, abs(want_loss)), (name, s, loss.item(), want_loss)
        assert abs(norm.item() - want_norm) <= max(tol["grad"], NORM_TOL) * want_norm, (name, s, norm.item(), want_norm)
        for k, v in m.named_parameters():   # .grad: the raw gradient (keep_clipped_grads off)
            _close(v.grad, grads[k], tol["grad"], f"{name} s{s} grad {k}")
            _close(v, params[k], tol["grad"], f"{name} s{s} param {k}")
        st_tol = STATE_TOL.get(T, tol["fwd"])
        for l, (h, c) in enumerate(tr.states):
            _close(h.reshape(B, -1), states[l][0], st_tol, f"{name} s{s} h{l}")
            _close(c.reshape(B, -1), states[l][1], st_tol, f"{name} s{s} c{l}")
    loss = tr.eval_step(xs[2], ys[2])
    want, _ = O.eval_loss(params, xs[2], ys[2], states, len(sizes), tied)
    assert abs(float(loss) - want) <= tol["loss"] * max(1.0, abs(want)), (name, float(loss), want)
    batches = list(zip(xs, ys))
    ppl = tr.perplexity(batches)
    st = [(torch.zeros(B, H, dtype=torch.float64, device="cuda"),) * 2 for H in sizes]
    logs = []
    for x, y in batches:
        lw, st = O.eval_loss(params, x, y, st, len(sizes), tied)
        logs.append(lw / B)
    want = float(np.mean(logs))
    assert abs(np.log(ppl) - want) <= tol["loss"] * max(1.0, want), (name, ppl, np.exp(want))
    for l in range(len(sizes)):
        plans = zaremba_b200._lib.rec_plans(m._ctx, l)
        # one branch for the whole step: every layer persistent, or every layer on the per-timestep path
        assert plans["fwd"]["ok"] == (0 if name == "steps" else 1), (name, l, plans)
        assert plans["bwd"]["ok"] == plans["fwd"]["ok"], (name, l, plans)
        if plans["fwd"]["ok"]:   # planned for the layer's own width: the contraction covers H_l, and equal widths plan alike
            assert 8 * plans["fwd"]["Kc"] >= sizes[l] and 8 * plans["bwd"]["Kc"] >= sizes[l], (name, l, plans)
            if l and sizes[l] == sizes[l - 1]:
                assert plans == zaremba_b200._lib.rec_plans(m._ctx, l - 1), (name, l, plans)
    if name == "branches":   # H = 40 runs the unsplit forward kernel, H = 300 the K-split one
        assert zaremba_b200._lib.rec_plans(m._ctx, 0)["fwd"]["KS"] == 1
        assert zaremba_b200._lib.rec_plans(m._ctx, 2)["fwd"]["KS"] > 1
    assert zaremba_b200._lib.rec_plans(m._ctx) == zaremba_b200._lib.rec_plans(m._ctx, 0)
    tr.close()


@pytest.mark.parametrize("name", list(SHAPES))
def test_dropin_forward_backward_matches_oracle(name):
    """zrb_forward / zrb_backward through Model.__call__ and autograd."""
    V, E, sizes, T, B, tied = SHAPES[name]
    m = _model(name)
    m.train()
    params = _params64(m)
    states = m.state_init(B)
    xs, ys = _data(name, 1)
    scores, new_states = m(xs[0], states)
    loss = torch.nn.functional.cross_entropy(scores, ys[0].reshape(-1)) * B
    loss.backward()
    ps = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    z = [(torch.zeros(B, H, dtype=torch.float64, device="cuda"),) * 2 for H in sizes]
    want_scores, want_states, _ = O.forward(ps, xs[0], z, len(sizes), tied)
    O.loss_of(want_scores, ys[0]).backward()
    tol = TOL["tc"]
    _close(scores.detach(), want_scores.detach(), tol["fwd"], f"{name} scores")
    for l, (h, c) in enumerate(new_states):
        assert tuple(h.shape) == (1, B, sizes[l])
        _close(h.reshape(B, -1), want_states[l][0].detach(), STATE_TOL.get(T, tol["fwd"]), f"{name} h{l}")
    for k, v in m.named_parameters():
        _close(v.grad, ps[k].grad, tol["grad"], f"{name} grad {k}")


def _trained_flat(V, H, L, T, B, steps, widths):
    """flat parameters, gradients, losses, norms and states after `steps` fused steps (lazy update on)"""
    import zaremba_b200
    torch.manual_seed(3)
    kw = dict(embed_size=H, layer_sizes=(H,) * L) if widths else {}
    m = zaremba_b200.Model(V, H, L, 0.5, 0.05, **kw).cuda()
    m.train()
    tr = zaremba_b200.Trainer(m, B, T, lazy_update=True)
    g = torch.Generator().manual_seed(1)
    out = []
    for _ in range(steps):
        x = torch.randperm(V, generator=g)[:T * B].view(T, B).cuda()
        y = torch.randint(0, V, (T, B), generator=g).cuda()
        loss, norm = tr.train_step(x, y, 1.0, 5.0)
        out += [loss.clone(), norm.clone()]
    tr.flush()
    torch.cuda.synchronize()
    out += [tr.flat_p.clone(), tr.flat_g.clone()] + [t.clone() for st in tr.states for t in st]
    tr.close()
    return out


@pytest.mark.parametrize("cfg", [(10000, 200, 2, 20, 20), (10000, 1500, 2, 35, 20)], ids=["small", "large"])
def test_equal_widths_bit_identical_to_one_width(cfg):
    a = _trained_flat(*cfg, steps=2, widths=False)
    b = _trained_flat(*cfg, steps=2, widths=True)
    bad = [i for i, (u, v) in enumerate(zip(a, b)) if not torch.equal(u, v)]
    assert not bad, f"entries {bad} differ between zrb_ctx_create and zrb_ctx_create_widths"


def _awd_all_modes(lazy):
    """AWD's model with every mode on: variational (+ recurrent) dropout, weight drop, embedding dropout, AR/TAR,
    NT-ASGD averaging; returns what three steps leave behind"""
    import zaremba_b200
    V, E, sizes, T, B, tied = SHAPES["awd"]
    m = _model("awd", dropout=0.4, variational=True, recurrent_dropout=0.25, weight_drop=0.5, embed_dropout=0.1)
    m.train()
    tr = zaremba_b200.Trainer(m, B, T, lazy_update=lazy, ar=2.0, tar=1.0)
    xs, ys = _data("awd", 3)
    out = []
    for s in range(3):
        if s == 1:
            tr.start_averaging()
        loss, norm = tr.train_step(xs[s], ys[s], 1.0, 0.25)
        out += [loss.clone(), norm.clone(), tr.activation_reg.clone()]
    tr.flush()
    torch.cuda.synchronize()
    out += [tr.flat_p.clone(), tr.flat_avg.clone()] + [t.clone() for st in tr.states for t in st]
    tr.close()
    return out


def test_awd_all_modes_lazy_equals_strict_and_repeats():
    lazy = _awd_all_modes(True)
    strict = _awd_all_modes(False)
    again = _awd_all_modes(True)
    assert all(torch.isfinite(t).all() for t in lazy)
    assert float(lazy[1]) > 0 and float(lazy[2].sum()) > 0
    bad = [i for i, (u, v) in enumerate(zip(lazy, strict)) if not torch.equal(u, v)]
    assert not bad, f"lazy differs from strict at {bad}"
    bad = [i for i, (u, v) in enumerate(zip(lazy, again)) if not torch.equal(u, v)]
    assert not bad, f"a repeated run differs at {bad}"


def test_awd_decode_cache_and_dynamic_evaluation():
    """Per-layer state shapes through generate, beam_search, the neural cache (H = H_{L-1}) and dynamic evaluation."""
    import zaremba_b200
    V, E, sizes, T, B, tied = SHAPES["awd"]
    m = _model("awd")
    m.eval()
    prompt = torch.randint(0, V, (6, 3), generator=torch.Generator().manual_seed(2)).cuda()
    toks, lps, st = m.generate(prompt, 5, top_k=1, seed=1)
    assert [tuple(h.shape) for h, _ in st] == [(1, 3, H) for H in sizes]
    btoks, blps, bscores, bst = m.beam_search(prompt, 5, 1)
    assert torch.equal(btoks[:, :, 0], toks), "beam_search with K = 1 differs from greedy decoding"
    # generate replayed through forward: the greedy token is the argmax of the scores of the last position
    with torch.no_grad():
        states = m.state_init(3)
        scores, states = m(prompt, states)
        assert torch.equal(scores.view(6, 3, V)[-1].argmax(1), toks[0])
    tr = zaremba_b200.Trainer(m, B, T)
    xs, ys = _data("awd", 2)
    batches = list(zip(xs, ys))
    base = float(tr.eval_step(*batches[0]))
    tr.reset_states()
    ppl = tr.perplexity(batches)
    cache = zaremba_b200.NeuralCache(hidden=sizes[-1], batch=B, size=100, max_seq=T)
    tr.reset_states()
    ppl_cache = tr.perplexity(batches, cache=cache, theta=0.5, lam=0.0)
    assert abs(ppl_cache - ppl) <= 1e-5 * ppl, (ppl_cache, ppl)
    tr.reset_states()
    ppl_dyn = tr.dynamic_perplexity(batches, lr=0.0, lam=0.0)
    assert abs(ppl_dyn - ppl) <= 1e-5 * ppl, (ppl_dyn, ppl)
    assert np.isfinite(base)
    tr.close()


# shape, Model keywords, Trainer keywords.  AWD's shape at Large's winit = 0.04: at 0.1, 1150-wide layers with W_hh
# doubled by weight drop over a 70-step window saturate the gates, and the step is chaotic (an fp16 rounding flips the
# NLL by whole percent; at T = 5 the same modes agree with the oracle to TOL["tc"])
MODES = {
    "awd_all": ("awd", dict(winit=0.04, dropout=0.4, variational=True, recurrent_dropout=0.25, weight_drop=0.5, embed_dropout=0.1),
                dict(ar=2.0, tar=1.0)),
    "branches_all": ("branches", dict(dropout=0.3, variational=True, recurrent_dropout=0.2, weight_drop=0.4,
                                      embed_dropout=0.2), dict(ar=2.0, tar=1.0)),
    "branches_zaremba": ("branches", dict(dropout=0.3, weight_drop=0.4, embed_dropout=0.2), dict(ar=1.0, tar=0.5)),
}


@pytest.mark.parametrize("case", list(MODES))
def test_modes_match_oracle(case):
    """Every width-dependent mask and normaliser against the fp64 restatement at unequal widths: dropout sites over E
    and each H_l (per step, or variational with period B*W), recurrent masks over B*H_l, weight drop over 4*H_l*H_l,
    embedding dropout over V, AR/TAR over H_{L-1}.  Two carried fused steps, NT-ASGD averaging on from the second."""
    import zaremba_b200
    name, mkw, tkw = MODES[case]
    V, E, sizes, T, B, tied = SHAPES[name]
    m = _model(name, **mkw)
    m.train()
    tr = zaremba_b200.Trainer(m, B, T, **tkw)
    p_rec = mkw.get("recurrent_dropout", mkw["dropout"] if mkw.get("variational") else 0.0)
    _random_states(tr)
    key = int(torch.initial_seed()) & 0xFFFFFFFFFFFFFFFF
    params = _params64(m)
    states = [(h.detach().double().reshape(B, -1).clone(), c.detach().double().reshape(B, -1).clone())
              for h, c in tr.states]
    xs, ys = _data(name, 2)
    tol = TOL["tc"]
    st_tol = STATE_TOL.get(T, tol["fwd"])
    avg = None
    for s in range(2):
        md = O.Modes(seed=tr.seed, step=tr.step, p=mkw["dropout"], variational=mkw.get("variational", False),
                     p_rec=p_rec, wd_seed=key, p_wd=mkw["weight_drop"], ed_seed=key,
                     p_e=mkw["embed_dropout"], alpha=tkw["ar"], beta=tkw["tar"])
        if s == 1:
            tr.start_averaging()
        loss, norm = tr.train_step(xs[s], ys[s], LR, MAX_NORM)
        reg = tr.activation_reg.clone()
        torch.cuda.synchronize()
        want_loss, want_norm, grads, params, states, want_reg = O.train_step(params, xs[s], ys[s], states, len(sizes),
                                                                             tied, LR, MAX_NORM, md)
        assert abs(loss.item() - want_loss) <= tol["loss"] * max(1.0, abs(want_loss)), (case, s, loss.item(), want_loss)
        assert abs(float(reg.sum()) - want_reg) <= tol["loss"] * max(1e-3, want_reg), (case, s, reg, want_reg)
        assert abs(norm.item() - want_norm) <= tol["grad"] * want_norm, (case, s, norm.item(), want_norm)
        for k, v in m.named_parameters():
            _close(v.grad, grads[k], tol["grad"], f"{case} s{s} grad {k}")
            _close(v, params[k], tol["grad"], f"{case} s{s} param {k}")
        for l, (h, c) in enumerate(tr.states):
            _close(h.reshape(B, -1), states[l][0], st_tol, f"{case} s{s} h{l}")
            _close(c.reshape(B, -1), states[l][1], st_tol, f"{case} s{s} c{l}")
        if s == 1:
            avg = {k: v.clone() for k, v in params.items()}   # the average of one step is that step's weights
    got = tr.average_state_dict()
    for k in avg:
        _close(got[k], avg[k], tol["grad"], f"{case} average {k}")
    tr.close()


def test_explicit_masks_take_each_sites_width():
    """zrb_set_explicit_masks with [T, B, W_s] masks per site equals the Philox masks they were drawn from, bit for bit"""
    import zaremba_b200
    V, E, sizes, T, B, tied = SHAPES["branches"]
    out = []
    for explicit in (False, True):
        m = _model("branches", dropout=0.3)
        m.train()
        tr = zaremba_b200.Trainer(m, B, T)
        if explicit:
            masks = O.mode_masks(O.Modes(seed=tr.seed, step=tr.step, p=0.3), [E, *sizes], T, B, V).sites
            m.set_explicit_dropout_masks([torch.as_tensor(mk).cuda() for mk in masks])
        xs, ys = _data("branches", 1)
        loss, norm = tr.train_step(xs[0], ys[0], LR, MAX_NORM)
        torch.cuda.synchronize()
        out.append([loss.clone(), norm.clone(), tr.flat_p.clone(), tr.flat_g.clone()])
        tr.close()
    assert all(torch.equal(a, b) for a, b in zip(*out))
