"""Zoneout (DESIGN.md section 20) on the GPU against the fp64 restatement of tests/_model_oracle.py, with the flags
fetched through zrb_dropout_mask.

  * two carried fused steps, alone and under Zaremba dropout: loss, clip norm, the raw gradient of every tensor (each
    relative to its own largest magnitude), parameters and states, at both forward plans (K split or not), both backward
    cluster sizes, Large's width and the per-timestep path (B = 40).  Every comparison is also made against the oracle
    without zoneout and against the oracle with the next step's flags, and both of those must fail the tolerance by a
    wide margin: a kernel that ignored zoneout or drew the wrong stream cannot pass;
  * eval mode (the expectation): the drop-in forward and backward, `eval_step` and `perplexity`, and the raw gradient of
    a dynamic-evaluation step, against the oracle, with the same discrimination checks;
  * every mode together (variational with recurrent dropout, weight drop, embedding dropout, AR/TAR, tied, unequal
    widths, NT-ASGD), and a Mixture-of-Softmaxes head: lazy equals strict bit for bit, rates of 0 after a switch-on are
    the mode off bit for bit, and the mode changes the result;
  * rates of 0 are the mode off and lazy equals strict, bit for bit, at every shape; greedy `generate` equals
    `beam_search` with one beam; the refusals.
Windows hold distinct tokens, so the embedding scatter is deterministic.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import lstm_lm_oracle as O
from oracle import philox
from tests import _model_oracle as MO

pytestmark = pytest.mark.gpu

L, LR, MAX_NORM = 2, 1.0, 0.25
# about 3x the largest error measured on an NVIDIA H100 80GB HBM3 over every test below (DESIGN.md section 20)
TOL_LOSS = 1e-6       # loss, relative (measured 2.4e-7)
TOL_PPL = 4e-6        # perplexity, relative (measured 1.2e-6)
TOL_NORM = 4e-4       # clip norm, relative (measured 1.2e-4)
TOL_GRAD = 2.5e-3     # raw gradient of a tensor, relative to its largest magnitude (measured 7.7e-4)
TOL_PARAM = 8e-4      # parameters after a step, relative to the tensor's largest magnitude (measured 2.4e-4)
TOL_STATE = 6e-4      # carried states, relative to their largest magnitude (measured 1.8e-4)
TOL_SCORE = 8e-4      # eval-mode scores, relative to their largest magnitude (measured 2.4e-4)
MARGIN = 5.0          # a wrong reference must miss by at least this many tolerances somewhere
# (V, H, T, B): the fixture shape (K split, S = 2), Small's H (no K split, S = 1), Medium's H, Large's H, the
# per-timestep path
SHAPES = [(211, 256, 7, 5), (500, 200, 12, 20), (500, 650, 10, 20), (1000, 1500, 8, 20), (300, 128, 6, 40)]
IDS = ["fixture", "small", "medium", "large", "per_timestep"]


def _dev():
    return torch.device("cuda:0")


def _model(V, H, z=(0.0, 0.0), p=0.0, **kw):
    import zaremba_b200
    torch.manual_seed(5)
    m = zaremba_b200.Model(V, H, L, p, min(0.1, 1.0 / np.sqrt(H)), zoneout_cell=z[0], zoneout_hidden=z[1],
                           **kw).to(_dev())
    m.train()
    return m


def _lib_flags(seed, step, l, T, B, H, z_c, z_h, Lm=L):
    """layer l's (zc, zh) [T,B,H] from zrb_dropout_mask at sites 3L + 3 + l and 4L + 3 + l: True = zoned"""
    from zaremba_b200 import _lib
    out = []
    for site, z in ((3 * Lm + 3 + l, z_c), (4 * Lm + 3 + l, z_h)):
        m = torch.empty(T * B * H, dtype=torch.uint8, device=_dev())
        _lib.check(_lib.load().zrb_dropout_mask(seed, step, site, T * B * H, z, _lib.ptr(m), None))
        out.append((m == 0).view(T, B, H).cpu().numpy() if z > 0 else np.zeros((T, B, H), bool))
    return tuple(out)


def _tokens(V, T, B, seed):
    rng = np.random.default_rng(seed)
    return torch.tensor(rng.permutation(V)[:T * B].reshape(T, B)), torch.tensor(rng.integers(0, V, (T, B)))


def _rel(got, want):
    """largest error relative to the reference tensor's largest magnitude"""
    got = np.asarray(got, np.float64).reshape(np.shape(want))
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-30))


def _np(t):
    return t.detach().cpu().double().numpy()


def _t64(states):
    return [(torch.tensor(h), torch.tensor(c)) for h, c in states]


def _oracle_step(params, x, y, states, md, masks):
    """one fp64 train step of the oracle on numpy params (updated in place) and states: loss, norm, states after, raw
    gradients"""
    loss, norm, grads, after, st, _ = MO.train_step({k: torch.tensor(v) for k, v in params.items()}, x, y, _t64(states),
                                                    L, False, LR, MAX_NORM, md, masks)
    params.update({k: v.numpy() for k, v in after.items()})
    return loss, norm, [(h.numpy(), c.numpy()) for h, c in st], {k: v.numpy() for k, v in grads.items()}


def _eval_oracle(params, x, y, states, z, G):
    """the oracle in eval mode at rates z, as numpy: scores, states, the gradients of sum(G * scores) and of the
    loss, and the loss"""
    grads = []
    for upstream in (G, None):
        ps = {k: torch.tensor(v, requires_grad=True) for k, v in params.items()}
        scores, st, _ = MO.forward(ps, x, _t64(states), L, False, MO.Modes(z_c=z[0], z_h=z[1]), train=False)
        loss = MO.loss_of(scores, y)
        (loss if upstream is None else (scores * torch.tensor(upstream)).sum()).backward()
        grads.append({k: v.grad.numpy() for k, v in ps.items()})
    return (scores.detach().numpy(), [(h.detach().numpy(), c.detach().numpy()) for h, c in st], grads[0], grads[1],
            loss.item())


def fused_errors(shape, p, steps=2):
    """the fused Trainer's errors against the oracle with the right flags, without zoneout, and with the next step's
    flags: {check: [err_right, err_no_zoneout, err_wrong_flags]} (the largest over the steps)"""
    import zaremba_b200
    V, H, T, B = shape
    z_c, z_h = 0.5, 0.05
    m = _model(V, H, (z_c, z_h), p)
    tr = zaremba_b200.Trainer(m, B, T)
    refs = [{k: _np(v).copy() for k, v in m.named_parameters()} for _ in range(3)]
    states = [O.zero_states(L, B, H, np.float64) for _ in range(3)]
    errs = {}

    def note(key, vals):
        old = errs.get(key, [0.0, 0.0, 0.0])
        errs[key] = [max(a, b) for a, b in zip(old, vals)]

    for it in range(steps):
        x, y = _tokens(V, T, B, it)
        right = [_lib_flags(tr.seed, tr.step, l, T, B, H, z_c, z_h) for l in range(L)]
        wrong = [_lib_flags(tr.seed, tr.step + 1, l, T, B, H, z_c, z_h) for l in range(L)]
        none = [(np.zeros((T, B, H), bool),) * 2 for _ in range(L)]
        masks = philox.site_masks(tr.seed, tr.step, L, T, B, H, p) if p > 0 else None
        assert any(f.any() for f in right[0])
        loss, norm = tr.train_step(x.to(_dev()), y.to(_dev()), LR, MAX_NORM)
        got_g = {k: _np(v.grad) for k, v in m.named_parameters()}
        got_p = {k: _np(v) for k, v in m.named_parameters()}
        rows = []
        for r, zf in enumerate((right, none, wrong)):
            mk = MO.Masks(sites=masks, zc=[f[0] for f in zf], zh=[f[1] for f in zf])
            want_loss, want_norm, states[r], raw = _oracle_step(refs[r], x, y, states[r],
                                                                MO.Modes(p=p, z_c=z_c, z_h=z_h), mk)
            rows.append((want_loss, want_norm, raw))
        note("loss", [abs(loss.item() - w[0]) / w[0] for w in rows])
        note("norm", [abs(norm.item() - w[1]) / w[1] for w in rows])
        for k in got_g:
            note("grad " + k, [_rel(got_g[k], w[2][k]) for w in rows])
            note("param " + k, [_rel(got_p[k], refs[r][k]) for r in range(3)])
        for l, (h, c) in enumerate(tr.states):
            note("state h", [_rel(_np(h), states[r][l][0]) for r in range(3)])
            note("state c", [_rel(_np(c), states[r][l][1]) for r in range(3)])
    return errs


def _tol(key):
    return {"loss": TOL_LOSS, "norm": TOL_NORM}.get(key) or (
        TOL_GRAD if key.startswith("grad") else TOL_PARAM if key.startswith("param") else TOL_STATE)


def _check(errs, tol=_tol):
    bad = {k: v[0] for k, v in errs.items() if v[0] >= tol(k)}
    assert not bad, bad
    for r, what in ((1, "the oracle without zoneout"), (2, "the oracle with another step's flags")):
        worst = max(v[r] / tol(k) for k, v in errs.items())
        assert worst > MARGIN, f"{what} is within {worst:.1f} tolerances: the comparison cannot tell them apart"


@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_fused_steps_against_the_oracle(shape):
    _check(fused_errors(shape, 0.0))


@pytest.mark.parametrize("shape", [SHAPES[0], SHAPES[2], SHAPES[4]], ids=[IDS[0], IDS[2], IDS[4]])
def test_fused_steps_under_zaremba_dropout(shape):
    _check(fused_errors(shape, 0.3))


def eval_errors(shape):
    """eval mode against the oracle's expectation, and against the oracle without zoneout:
    {check: [err_right, err_no_zoneout]}"""
    import zaremba_b200
    V, H, T, B = shape
    z_c, z_h = 0.3, 0.2
    m = _model(V, H, (z_c, z_h))
    params = {k: _np(v) for k, v in m.named_parameters()}
    x, y = _tokens(V, T, B, 9)
    zeros = O.zero_states(L, B, H, np.float64)
    errs = {}
    # the drop-in forward and backward (a fixed upstream gradient)
    m.eval()
    st = m.state_init(B)
    scores, st = m(x.to(_dev()), st)
    G = torch.randn(scores.shape, generator=torch.Generator().manual_seed(3)).to(_dev())
    scores.backward(G)
    refs = [_eval_oracle(params, x, y, zeros, z, _np(G)) for z in ((z_c, z_h), (0.0, 0.0))]
    errs["dropin scores"] = [_rel(_np(scores), r[0]) for r in refs]
    errs["dropin state c"] = [max(_rel(_np(st[l][1]), r[1][l][1]) for l in range(L)) for r in refs]
    errs["dropin state h"] = [max(_rel(_np(st[l][0]), r[1][l][0]) for l in range(L)) for r in refs]
    for k, v in m.named_parameters():
        errs["dropin grad " + k] = [_rel(_np(v.grad), r[2][k]) for r in refs]
    # eval_step, perplexity and the raw gradient of a dynamic-evaluation step (lr = 0: the weights stay put)
    m.zero_grad(set_to_none=True)
    tr = zaremba_b200.Trainer(m, B, T)
    want = [r[4] for r in refs]
    errs["eval_step"] = [abs(tr.eval_step(x.to(_dev()), y.to(_dev())).item() - w) / w for w in want]
    ppl = tr.perplexity([(x, y)])
    errs["perplexity"] = [abs(ppl - math.exp(w / B)) / math.exp(w / B) for w in want]
    tr.reset_states()
    tr.dynamic_eval_step(x.to(_dev()), y.to(_dev()), tr.flat_p.clone(), 0.0)
    for k, v in m.named_parameters():
        errs["dyneval grad " + k] = [_rel(_np(v.grad), r[3][k]) for r in refs]
    return errs


def _eval_tol(key):
    return TOL_SCORE if "scores" in key else TOL_STATE if "state" in key else TOL_LOSS if key == "eval_step" else \
        TOL_PPL if key == "perplexity" else TOL_GRAD


@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_eval_mode_against_the_oracle(shape):
    errs = eval_errors(shape)
    bad = {k: v[0] for k, v in errs.items() if v[0] >= _eval_tol(k)}
    assert not bad, bad
    worst = max(v[1] / _eval_tol(k) for k, v in errs.items())
    assert worst > MARGIN, f"the oracle without zoneout is within {worst:.1f} tolerances"


def _run(make, steps=3, lazy=False, set_zero=False, avg=True):
    """three fused steps of a Trainer over make()'s model; losses, norms and parameters (and the average)"""
    import zaremba_b200
    from zaremba_b200 import _lib
    m, T, B = make()
    tr = zaremba_b200.Trainer(m, B, T, lazy_update=lazy, ar=1.0, tar=1.0)
    if set_zero:
        _lib.check(_lib.load().zrb_set_zoneout(tr.ctx, 0.5, 0.5))
        _lib.check(_lib.load().zrb_set_zoneout(tr.ctx, 0.0, 0.0))
    if avg:
        tr.start_averaging()
    res = []
    for it in range(steps):
        x, y = _tokens(m.vocab_size, T, B, it)
        loss, norm = tr.train_step(x.to(_dev()), y.to(_dev()), LR, MAX_NORM)
        res += [loss.item(), norm.item()]
    tr.flush()
    res += [v.detach().cpu().clone() for v in m.parameters()]
    if avg:
        res.append(tr.flat_avg.detach().cpu().clone())
    tr.close()
    return res


def _same(a, b):
    assert len(a) == len(b)
    for i, (u, v) in enumerate(zip(a, b)):
        assert (u == v) if isinstance(u, float) else torch.equal(u, v), i


def _all_modes(z, experts=None):
    """variational dropout with recurrent dropout, weight drop, embedding dropout, tied, unequal widths (AWD's
    400-1150-1150-400 shape scaled down), and optionally a Mixture-of-Softmaxes head"""
    def make():
        import zaremba_b200
        torch.manual_seed(7)
        sizes = (96, 96, 40) if experts else (192, 192, 64)
        m = zaremba_b200.Model(400, sizes[0], 3, 0.3, 0.08, variational=True, recurrent_dropout=0.2, tied=True,
                               weight_drop=0.3, embed_dropout=0.1, embed_size=32 if experts else 64, layer_sizes=sizes,
                               experts=experts, zoneout_cell=z[0], zoneout_hidden=z[1]).to(_dev())
        m.train()
        return m, 9, 12
    return make


@pytest.mark.parametrize("experts", [None, 3], ids=["awd", "mos"])
def test_every_mode_together(experts):
    on = _run(_all_modes((0.5, 0.05), experts))
    assert all(math.isfinite(v) for v in on[:6])
    _same(on, _run(_all_modes((0.5, 0.05), experts), lazy=True))
    off = _run(_all_modes((0.0, 0.0), experts))
    _same(off, _run(_all_modes((0.0, 0.0), experts), set_zero=True))
    assert on[0] != off[0]


@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_zero_rates_are_the_mode_off(shape):
    """zrb_set_zoneout(ctx, 0, 0) after a switch-on runs the mode-off kernels: bit for bit the plain model"""
    V, H, T, B = shape
    _same(_run(lambda: (_model(V, H), T, B), steps=2, avg=False),
          _run(lambda: (_model(V, H), T, B), steps=2, set_zero=True, avg=False))


@pytest.mark.parametrize("shape", SHAPES[1:4], ids=IDS[1:4])
def test_lazy_equals_strict(shape):
    V, H, T, B = shape
    _same(_run(lambda: (_model(V, H, (0.4, 0.1)), T, B)), _run(lambda: (_model(V, H, (0.4, 0.1)), T, B), lazy=True))


def test_generate_equals_beam_search_with_one_beam():
    V, H, T, B = SHAPES[1]
    m = _model(V, H, (0.5, 0.05))
    m.eval()
    x, _ = _tokens(V, 4, 3, 1)
    toks, _, _ = m.generate(x, 6, temperature=1e-6, seed=1)
    btoks, _, _, _ = m.beam_search(x, 6, 1)
    assert torch.equal(toks, btoks[:, :, 0])


def test_refusals():
    from zaremba_b200 import _lib
    lib = _lib.load()
    E_INVALID = -1
    cfg = _lib.ZrbConfig(50, 64, 1, 4, 4, _lib.ENGINE_TC, 0.0, 0)
    h = C.c_void_p()
    _lib.check(lib.zrb_ctx_create(C.byref(cfg), C.byref(h)))
    try:
        for bad in (1.0, -0.1, float("nan"), float("inf")):
            assert lib.zrb_set_zoneout(h, bad, 0.0) == E_INVALID
            assert lib.zrb_set_zoneout(h, 0.0, bad) == E_INVALID
        assert lib.zrb_set_zoneout(None, 0.1, 0.1) == E_INVALID
        before = lib.zrb_ctx_workspace_bytes(h)
        _lib.check(lib.zrb_set_zoneout(h, 0.5, 0.05))
        assert lib.zrb_ctx_workspace_bytes(h) > before      # the c~ buffers and flags are reported
        x = torch.zeros(4, 4, 64, device=_dev())
        w = torch.zeros(256, 64, device=_dev())
        b = torch.zeros(256, device=_dev())
        s0 = torch.zeros(4, 64, device=_dev())
        y = torch.zeros(16, 64, device=_dev())
        assert lib.zrb_lstm_layer_fwd(h, _lib.ptr(w), _lib.ptr(w), _lib.ptr(b), _lib.ptr(b), _lib.ptr(x), 4, 4,
                                      _lib.ptr(s0), _lib.ptr(s0), _lib.ptr(y), None, None, None) == E_INVALID
        assert lib.zrb_lstm_layer_bwd(h, _lib.ptr(y), None, _lib.ptr(w), _lib.ptr(w), _lib.ptr(b), _lib.ptr(b),
                                      None) == E_INVALID
    finally:
        lib.zrb_ctx_destroy(h)
    cfg = _lib.ZrbConfig(50, 64, 1, 4, 4, _lib.ENGINE_SIMT, 0.0, 0)
    _lib.check(lib.zrb_ctx_create(C.byref(cfg), C.byref(h)))
    try:
        assert lib.zrb_set_zoneout(h, 0.5, 0.0) == E_INVALID
    finally:
        lib.zrb_ctx_destroy(h)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_devices_in_one_process():
    """the zoneout kernels' shared-memory limit belongs to each device's context: a model per device both train"""
    import zaremba_b200
    V, H, T, B = SHAPES[2]
    x, y = _tokens(V, T, B, 0)
    for d in (0, 1):
        dev = torch.device(f"cuda:{d}")
        torch.manual_seed(5)
        m = zaremba_b200.Model(V, H, L, 0.0, 0.05, zoneout_cell=0.5, zoneout_hidden=0.05).to(dev)
        m.train()
        tr = zaremba_b200.Trainer(m, B, T)
        loss, _ = tr.train_step(x.to(dev), y.to(dev), LR, MAX_NORM)
        assert math.isfinite(loss.item())
        tr.close()
