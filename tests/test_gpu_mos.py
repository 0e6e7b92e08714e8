"""Mixture of Softmaxes (DESIGN.md section 19) through the tensor-core engine, against the fp64 restatement in
tests/_model_oracle.py.

Shapes: MoS's PTB model (E = 280, 960-960-620, K = 15, T = 70, B = 12, tied), the recurrence-plan branches of
test_gpu_widths.py with K = 3, the per-timestep path (B = 40), a vocabulary that is not a multiple of 4 (the scalar
path of the mixture kernel) with one width, and one expert.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import philox as PH
from tests import _model_oracle as O
from tests.test_gpu_parity import TOL

pytestmark = pytest.mark.gpu

SHAPES = {   # V, E, layer widths (None: one width E), T, B, tied, K
    "mos_ptb": (10000, 280, (960, 960, 620), 70, 12, True, 15),
    "branches": (500, 72, (40, 200, 300), 5, 8, False, 3),
    "steps": (500, 48, (64, 96), 5, 40, False, 2),
    "v_odd_one_width": (499, 64, None, 5, 6, True, 4),
    "one_expert": (500, 32, (48, 40), 5, 4, False, 1),
}
LR, MAX_NORM, WINIT = 1.0, 0.25, 0.1
# About 3x the largest error measured against fp64 on an H100 80GB HBM3 (700 W) over every shape and mode of this file
# (relative to the largest magnitude of the compared tensor; DESIGN.md section 19): loss 2.3e-7, clip norm 7.5e-5,
# raw gradients 1.5e-3 (the prior's and the last layer's: the fp16 gradient images of the head), parameters after a
# step 1.0e-4, NT-ASGD average 8.3e-5, drop-in log p 2.2e-5, states 1.4e-3 (as test_gpu_widths.py, the fp16 recurrent
# operand's error grows over a window).  The drop-in backward under a random upstream gradient: prior.W 3.3e-3 (da =
# s - pi sum G cancels before its fp16 rounding), every other tensor within the gradient bound.
MOS_TOL = dict(loss=1e-6, norm=2.5e-4, grad=5e-3, param=3e-4, logp=7e-5, state=5e-3, random_prior=1e-2)
EVAL_TOL = TOL["tc"]["loss"]   # eval_step / perplexity, as test_gpu_widths.py
STATE_TOL = MOS_TOL["state"]


def _close(got, want, rel, what):
    got = torch.as_tensor(got).detach().double().cpu()
    want = torch.as_tensor(want).detach().double().cpu()
    scale = max(float(want.abs().max()), 1e-6)
    err = float((got - want).abs().max())
    print(f"ERR {what}: {err / scale:.2e}")
    assert err <= rel * scale, f"{what}: max abs err {err:.3e} vs scale {scale:.3e} (rel {err / scale:.2e} > {rel:.1e})"


def _widths(name):
    V, E, sizes, T, B, tied, K = SHAPES[name]
    return sizes or (E, E)


def _model(name, winit=WINIT, **kw):
    import zaremba_b200
    V, E, sizes, T, B, tied, K = SHAPES[name]
    tied = kw.pop("tied", tied)
    torch.manual_seed(7)
    wk = dict(embed_size=E, layer_sizes=sizes) if sizes else {}
    L = len(_widths(name))
    return zaremba_b200.Model(V, _widths(name)[0], L, kw.pop("dropout", 0.0), winit, tied=tied, experts=K, **wk,
                              **kw).cuda()


def _data(name, steps, seed=11):
    V, E, sizes, T, B, tied, K = SHAPES[name]
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


def _states64(tr, B):
    return [(h.detach().double().reshape(B, -1).clone(), c.detach().double().reshape(B, -1).clone())
            for h, c in tr.states]


@pytest.mark.parametrize("name", list(SHAPES))
def test_fused_steps_match_oracle(name):
    """Two carried fused train steps: loss, clip norm, raw gradients (the head's included), parameters and states; then
    eval_step and perplexity."""
    import zaremba_b200
    V, E, sizes, T, B, tied, K = SHAPES[name]
    L = len(_widths(name))
    m = _model(name)
    m.train()
    tr = zaremba_b200.Trainer(m, B, T)
    _random_states(tr)
    params = _params64(m)
    states = _states64(tr, B)
    xs, ys = _data(name, 3)
    tol = MOS_TOL
    for s in range(2):
        loss, norm = tr.train_step(xs[s], ys[s], LR, MAX_NORM)
        torch.cuda.synchronize()
        want_loss, want_norm, grads, params, states, _ = O.train_step(params, xs[s], ys[s], states, L, tied, LR,
                                                                     MAX_NORM)
        print(f"ERR {name} s{s} loss: {abs(loss.item() - want_loss) / abs(want_loss):.2e} "
              f"norm: {abs(norm.item() - want_norm) / want_norm:.2e}")
        assert abs(loss.item() - want_loss) <= tol["loss"] * abs(want_loss), (name, s, loss.item(), want_loss)
        assert abs(norm.item() - want_norm) <= tol["norm"] * want_norm, (name, s, norm.item(), want_norm)
        for k, v in m.named_parameters():
            _close(v.grad, grads[k], tol["grad"], f"{name} s{s} grad {k}")
            _close(v, params[k], tol["param"], f"{name} s{s} param {k}")
        for l, (h, c) in enumerate(tr.states):
            _close(h.reshape(B, -1), states[l][0], STATE_TOL, f"{name} s{s} h{l}")
            _close(c.reshape(B, -1), states[l][1], STATE_TOL, f"{name} s{s} c{l}")
    loss = tr.eval_step(xs[2], ys[2])
    want, _ = O.eval_loss(params, xs[2], ys[2], states, L, tied)
    assert abs(float(loss) - want) <= EVAL_TOL * max(1.0, abs(want)), (name, float(loss), want)
    batches = list(zip(xs, ys))
    ppl = tr.perplexity(batches)
    st = [(torch.zeros(B, H, dtype=torch.float64, device="cuda"),) * 2 for H in _widths(name)]
    logs = []
    for x, y in batches:
        lw, st = O.eval_loss(params, x, y, st, L, tied)
        logs.append(lw / B)
    want = float(np.mean(logs))
    assert abs(np.log(ppl) - want) <= EVAL_TOL * max(1.0, want), (name, ppl, np.exp(want))
    tr.close()


def _run(name, lazy, steps=3, **mkw):
    """flat parameters, gradients, average, losses and norms after `steps` fused steps, averaging from the second"""
    import zaremba_b200
    V, E, sizes, T, B, tied, K = SHAPES[name]
    m = _model(name, **mkw)
    m.train()
    tr = zaremba_b200.Trainer(m, B, T, lazy_update=lazy)
    xs, ys = _data(name, steps)
    out = []
    for s in range(steps):
        if s == 1:
            tr.start_averaging()
        loss, norm = tr.train_step(xs[s], ys[s], LR, MAX_NORM)
        out += [loss.clone(), norm.clone()]
    tr.flush()
    torch.cuda.synchronize()
    out += [tr.flat_p.clone(), tr.flat_g.clone(), tr.flat_avg.clone()] + [t.clone() for st in tr.states for t in st]
    tr.close()
    return out


# Tied, so that every gradient is bit-reproducible (an untied embedding's gradient is a scatter with fp32 atomics, whose
# last bits vary run to run); the per-timestep path ("steps") defers nothing: the lazy update needs the persistent kernels
@pytest.mark.parametrize("name", [n for n in SHAPES if n != "steps"])
def test_lazy_update_equals_strict(name):
    lazy = _run(name, True, dropout=0.3, mos_dropout=0.2, tied=True)
    strict = _run(name, False, dropout=0.3, mos_dropout=0.2, tied=True)
    assert all(torch.isfinite(t).all() for t in lazy)
    bad = [i for i, (u, v) in enumerate(zip(lazy, strict)) if not torch.equal(u, v)]
    assert not bad, f"lazy differs from strict at {bad}"


@pytest.mark.parametrize("name", list(SHAPES))
def test_dropin_forward_backward_matches_oracle(name):
    """zrb_forward writes log p; zrb_backward takes dL / d log p: the CE loss on log p and a random upstream gradient"""
    V, E, sizes, T, B, tied, K = SHAPES[name]
    L = len(_widths(name))
    tol = MOS_TOL
    for upstream in ("nll", "random"):
        m = _model(name)
        m.train()
        params = _params64(m)
        xs, ys = _data(name, 1)
        logp, new_states = m(xs[0], m.state_init(B))
        ps = {k: v.clone().requires_grad_(True) for k, v in params.items()}
        z = [(torch.zeros(B, H, dtype=torch.float64, device="cuda"),) * 2 for H in _widths(name)]
        want_logp, want_states, _ = O.forward(ps, xs[0], z, L, tied)
        if upstream == "nll":
            (torch.nn.functional.cross_entropy(logp, ys[0].reshape(-1)) * B).backward()
            O.loss_of(want_logp, ys[0], logp=True).backward()
        else:
            G = torch.randn(T * B, V, generator=torch.Generator().manual_seed(3)).cuda()
            (logp * G).sum().backward()
            (want_logp * G.double()).sum().backward()
        _close(logp.detach(), want_logp.detach(), tol["logp"], f"{name} log p")
        assert torch.allclose(logp.detach().exp().sum(1), torch.ones(T * B, device="cuda"), atol=1e-4)
        for l, (h, c) in enumerate(new_states):
            _close(h.reshape(B, -1), want_states[l][0].detach(), STATE_TOL, f"{name} h{l}")
        for k, v in m.named_parameters():
            rel = tol["random_prior"] if (upstream, k) == ("random", "prior.W") else tol["grad"]
            _close(v.grad, ps[k].grad, rel, f"{name} {upstream} grad {k}")


@pytest.mark.parametrize("name", list(SHAPES))
def test_greedy_generate_equals_beam_of_one_and_oracle(name):
    V, E, sizes, T, B, tied, K = SHAPES[name]
    L = len(_widths(name))
    m = _model(name)
    m.eval()
    prompt = torch.randint(0, V, (4, 3), generator=torch.Generator().manual_seed(2)).cuda()
    toks, lps, _ = m.generate(prompt, 3, top_k=1, seed=1)
    btoks, blps, _, _ = m.beam_search(prompt, 3, 1)
    assert torch.equal(btoks[:, :, 0], toks), "beam_search with K = 1 differs from greedy decoding"
    # the oracle's log p along the greedy continuation
    params = _params64(m)
    seq = torch.cat([prompt, toks[:-1]], 0)
    z = [(torch.zeros(3, H, dtype=torch.float64, device="cuda"),) * 2 for H in _widths(name)]
    want, _, _ = O.forward(params, seq, z, L, tied)
    want = want.view(seq.shape[0], 3, V)[prompt.shape[0] - 1:]
    _close(lps, want.gather(2, toks[:, :, None]).squeeze(2), MOS_TOL["logp"], f"{name} generate logprobs")
    _close(blps[:, :, 0], lps, 1e-6, f"{name} beam logprobs")


def test_latent_mask_is_zrb_dropout_mask_at_site_3L_plus_2():
    import zaremba_b200
    from zaremba_b200 import _lib
    L, n, p = 3, 12 * 15 * 280 + 5, 0.3
    got = torch.empty(n, dtype=torch.uint8, device="cuda")
    _lib.check(_lib.load().zrb_dropout_mask(99, 4, 3 * L + 2, n, p, _lib.ptr(got), None))
    assert np.array_equal(got.cpu().numpy().astype(bool), PH.keep_mask(99, 4, 3 * L + 2, n, p))
    assert zaremba_b200 is not None


# shape, Model keywords, Trainer keywords (MoS PTB at Large's winit = 0.04, as test_gpu_widths.py does for AWD)
MODES = {
    "mos_ptb_all": ("mos_ptb", dict(winit=0.04, dropout=0.4, variational=True, recurrent_dropout=0.25, weight_drop=0.5,
                                    embed_dropout=0.1, mos_dropout=0.3), dict(ar=2.0, tar=1.0)),
    "branches_all": ("branches", dict(dropout=0.3, variational=True, recurrent_dropout=0.2, weight_drop=0.4,
                                      embed_dropout=0.2, mos_dropout=0.25), dict(ar=2.0, tar=1.0)),
    "branches_zaremba": ("branches", dict(dropout=0.3, weight_drop=0.4, embed_dropout=0.2, mos_dropout=0.25),
                         dict(ar=1.0, tar=0.5)),
}


@pytest.mark.parametrize("case", list(MODES))
def test_modes_match_oracle(case):
    """Latent dropout (per step, and variational with period B*K*E) with every other mode, two carried fused steps,
    NT-ASGD averaging from the second"""
    import zaremba_b200
    name, mkw, tkw = MODES[case]
    V, E, sizes, T, B, tied, K = SHAPES[name]
    L = len(_widths(name))
    m = _model(name, **mkw)
    m.train()
    tr = zaremba_b200.Trainer(m, B, T, **tkw)
    p_rec = mkw.get("recurrent_dropout", mkw["dropout"] if mkw.get("variational") else 0.0)
    _random_states(tr)
    key = int(torch.initial_seed()) & 0xFFFFFFFFFFFFFFFF
    params = _params64(m)
    states = _states64(tr, B)
    xs, ys = _data(name, 2)
    tol = MOS_TOL
    avg = None
    for s in range(2):
        md = O.Modes(seed=tr.seed, step=tr.step, p=mkw["dropout"], variational=mkw.get("variational", False),
                     p_rec=p_rec, wd_seed=key, p_wd=mkw["weight_drop"], ed_seed=key, p_e=mkw["embed_dropout"],
                     alpha=tkw["ar"], beta=tkw["tar"], p_l=mkw["mos_dropout"])
        if s == 1:
            tr.start_averaging()
        loss, norm = tr.train_step(xs[s], ys[s], LR, MAX_NORM)
        torch.cuda.synchronize()
        want_loss, want_norm, grads, params, states, _ = O.train_step(params, xs[s], ys[s], states, L, tied, LR,
                                                                     MAX_NORM, md)
        print(f"ERR {case} s{s} loss: {abs(loss.item() - want_loss) / abs(want_loss):.2e} "
              f"norm: {abs(norm.item() - want_norm) / want_norm:.2e}")
        assert abs(loss.item() - want_loss) <= tol["loss"] * abs(want_loss), (case, s, loss.item(), want_loss)
        assert abs(norm.item() - want_norm) <= tol["norm"] * want_norm, (case, s, norm.item(), want_norm)
        for k, v in m.named_parameters():
            _close(v.grad, grads[k], tol["grad"], f"{case} s{s} grad {k}")
            _close(v, params[k], tol["param"], f"{case} s{s} param {k}")
        for l, (h, c) in enumerate(tr.states):
            _close(h.reshape(B, -1), states[l][0], STATE_TOL, f"{case} s{s} h{l}")
        if s == 1:
            avg = {k: v.clone() for k, v in params.items()}   # the average of one step is that step's weights
    got = tr.average_state_dict()
    for k in avg:
        _close(got[k], avg[k], tol["param"], f"{case} average {k}")
    tr.close()


def test_refusals():
    import zaremba_b200
    from zaremba_b200 import _lib
    lib = _lib.load()
    V, E, sizes, T, B, tied, K = SHAPES["branches"]
    h = C.c_void_p()
    for experts, engine, layers in ((0, _lib.ENGINE_TC, 2), (33, _lib.ENGINE_TC, 2), (2, _lib.ENGINE_SIMT, 2),
                                    (2, _lib.ENGINE_TC, 4)):
        cfg = _lib.ZrbConfig(V, 64, layers, T, B, engine, 0.0, 0)
        assert lib.zrb_ctx_create_mos(C.byref(cfg), None, experts, C.byref(h)) == -1, (experts, engine, layers)
    m = _model("branches")
    tr = zaremba_b200.Trainer(m, B, T)
    ctx = tr.ctx
    assert lib.zrb_set_embed_rows_out(ctx, None) == -1
    assert lib.zrb_set_mos_dropout(ctx, 1.0) == -1 and lib.zrb_set_mos_dropout(ctx, -0.1) == -1
    xs, ys = _data("branches", 2)
    batches = list(zip(xs, ys))
    with pytest.raises(ValueError, match="Mixture-of-Softmaxes"):
        tr.eval_step(xs[0], ys[0], cache=zaremba_b200.NeuralCache(hidden=sizes[-1], batch=B, size=10, max_seq=T))
    with pytest.raises(ValueError, match="Mixture-of-Softmaxes"):
        tr.dynamic_perplexity(batches, lr=0.0)
    with pytest.raises(ValueError, match="Mixture-of-Softmaxes"):
        tr.gradient_stats(batches)
    # the C entry points refuse before anything is launched
    x, y = xs[0], ys[0]
    assert lib.zrb_grad_stats_step(ctx, C.byref(tr._ps), C.byref(tr._gs), C.byref(tr._gs), _lib.ptr(x), _lib.ptr(y), T,
                                   B, C.byref(tr._st), C.byref(tr._st), None, None) == -1
    assert lib.zrb_dyneval_step(ctx, C.byref(tr._ps), C.byref(tr._gs), C.byref(tr._ps), None, None, _lib.ptr(x),
                                _lib.ptr(y), T, B, C.byref(tr._st), C.byref(tr._st), 0.0, 0.0, 1.0, None, None) == -1
    plain = zaremba_b200.Model(V, 64, 2, 0.0, 0.1).cuda()
    pc = plain._context(T, B)
    assert lib.zrb_set_mos_dropout(pc, 0.1) == -1
    tr.close()
