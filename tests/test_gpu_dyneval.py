"""Dynamic evaluation on the GPU (DESIGN.md section 14): the gradient is the eval-mode one bit for bit, the update is
exact and leaves current fp16 images, whole passes match the float64 restatement tests/_dyneval_oracle.py, the identities
with perplexity / eval_step / lazy update, the statistics, and the rejected arguments.

Tolerances are test_gpu_parity's TOL per engine."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import _dyneval_oracle as DO
from tests._golden import StepCase
from tests.test_gpu_parity import ENGINES, TOL, _prof_counts, _record, _scale_close

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
# name -> (V, H, L, T, B, winit): the exact Small / Medium / Large shapes, B = 1, B = 40 (per-timestep recurrence),
# odd H = 257 (the update's one-column path, K-split), and the reference fixture's shape.  The update kernels take 4
# columns per thread when H % 4 == 0 (Large, B = 40), 2 when H % 4 == 2 (Medium) and 1 when H is odd
SHAPES = {
    "fixture": None,
    "small": (10000, 200, 2, 20, 20, 0.1),
    "medium": (10000, 650, 2, 35, 20, 0.05),
    "large": (10000, 1500, 2, 35, 20, 0.04),
    "small_b1": (10000, 200, 2, 5, 1, 0.1),
    "steps_b40": (400, 64, 2, 4, 40, 0.1),
    "odd_h": (300, 257, 2, 5, 9, 0.1),
}


def _shape(name):
    if name == "fixture":
        c = StepCase("tiny_dropout")
        return c.V, c.H, c.L, c.T, c.B, c.winit
    return SHAPES[name]


def _model(name, engine, p=0.0, tied=False, seed=1, **kw):
    import zaremba_b200
    V, H, L, T, B, winit = _shape(name)
    torch.manual_seed(seed)
    m = zaremba_b200.Model(V, H, L, p, winit, engine=engine, tied=tied, **kw)
    if name == "fixture" and not tied:
        params = StepCase("tiny_dropout").params0()
        m.load_state_dict({k: torch.tensor(v) for k, v in params.items()})
    return m.to(DEV)


def _trainer(m, name, states_seed=None, **kw):
    import zaremba_b200
    V, H, L, T, B, _ = _shape(name)
    tr = zaremba_b200.Trainer(m, B, T, **kw)
    if states_seed is not None:
        g = torch.Generator().manual_seed(states_seed)
        for h, c in tr.states:
            h.copy_(torch.rand(h.shape, generator=g) * 0.6 - 0.3)
            c.copy_(torch.rand(c.shape, generator=g) - 0.5)
    return tr


def _windows(name, n, seed=2):
    """n windows [T,B] whose tokens occur at most twice each (the untied embedding gradient is a scatter with fp32
    atomics: three rows of one token may sum in either order, two always give the same bits)."""
    V, H, L, T, B, _ = _shape(name)
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        ids = torch.cat([torch.randperm(V, generator=g), torch.randperm(V, generator=g)])[:T * B]
        x = ids[torch.randperm(T * B, generator=g)].view(T, B).contiguous().to(DEV)
        y = torch.randint(0, V, (T, B), generator=g).to(DEV)
        out.append((x, y))
    return out


def _copy_weights(dst, src):
    with torch.no_grad():
        for a, b in zip(dst.ordered_parameters(), src.ordered_parameters()):
            a.copy_(b)


GRAD_CASES = [("fixture", e, v) for e in ENGINES for v in (False, True)] + \
             [(n, e, False) for n in ("small", "medium", "large", "small_b1", "steps_b40") for e in ENGINES] + \
             [("large", "tc", True)]


@pytest.mark.parametrize("name,engine,variational", GRAD_CASES)
def test_gradient_is_the_eval_mode_gradient(name, engine, variational):
    """g of zrb_dyneval_step in a p = 0.65 context (also variational) = zrb_train_step_grads's g in a p = 0 context."""
    from zaremba_b200 import _lib
    lib = _lib.load()
    kw = dict(variational=True) if variational else {}
    m1 = _model(name, engine, p=0.65, **kw)
    m2 = _model(name, engine, p=0.0)
    _copy_weights(m2, m1)
    tr1, tr2 = _trainer(m1, name, states_seed=5), _trainer(m2, name, states_seed=5)
    (x, y), = _windows(name, 1)
    T, B = x.shape
    loss1 = tr1.dynamic_eval_step(x, y, tr1.flat_p.clone(), lr=0.1, lam=0.2).clone()
    loss2 = torch.zeros((), device=DEV)
    _lib.check(lib.zrb_train_step_grads(tr2.ctx, C.byref(tr2._ps), C.byref(tr2._gs), _lib.ptr(x), _lib.ptr(y), T, B,
                                        C.byref(tr2._st), C.byref(tr2._st), 99, 7, _lib.ptr(loss2), tr2._stream()))
    torch.cuda.synchronize()
    assert torch.equal(tr1.flat_g, tr2.flat_g), "the dynamic step's gradient is not the eval-mode gradient"
    assert torch.equal(loss1, loss2), (loss1.item(), loss2.item())
    for (h1, c1), (h2, c2) in zip(tr1.states, tr2.states):
        assert torch.equal(h1, h2) and torch.equal(c1, c2)


def _ulp32(x):
    x = np.abs(np.asarray(x, dtype=np.float32))
    return np.spacing(x).astype(np.float64)


@pytest.mark.parametrize("rule", ["rms", "sgd"])
@pytest.mark.parametrize("name,tied", [("large", False), ("large", True), ("medium", False), ("medium", True),
                                       ("odd_h", False), ("odd_h", True), ("steps_b40", False)])
def test_update_is_exact_and_images_are_current(name, tied, rule):
    """Every element of theta_{s+1} against the float64 formula on the same fp32 inputs (theta_s, g read back, theta_g,
    r, r-bar), held to ulp(theta_{s+1}) + 4 ulp(S), S = |a d| + |lr u|: to first order the roundings of d, a, u and
    lr * u stay within 3 ulp(S), the FMA's within ulp(S) and the final add's within ulp(theta_{s+1}).  Then the fp16
    images the update wrote equal what a fresh pack of the same fp32 weights builds (no repack in the adapted context,
    bit-identical eval outputs)."""
    import zaremba_b200
    from zaremba_b200 import _lib
    lib = _lib.load()
    m = _model(name, "tc", p=0.5, tied=tied)
    tr = _trainer(m, name, states_seed=3)
    wins = _windows(name, 4)
    stats = tr.gradient_stats(wins[:2]) if rule == "rms" else None
    # the scalars as the kernels hold them: the float64 formula runs on the same fp32 inputs
    lr, lam, eps = (float(np.float32(v)) for v in ((2e-4, 0.2, 2e-5) if rule == "rms" else (0.5, 0.05, 2e-5)))
    theta_g = tr.flat_p.clone()
    tr.dynamic_eval_step(*wins[2], theta_g, lr, lam, stats, eps)       # theta_1 != theta_g
    p0 = tr.flat_p.double()
    tr.dynamic_eval_step(*wins[3], theta_g, lr, lam, stats, eps)
    torch.cuda.synchronize()
    g = tr.flat_g.double()
    tg = theta_g.double()
    d = tg - p0
    if rule == "rms":
        r, rbar = stats.rms.double(), float(stats.mean)
        u = g / (r + eps)
        a = torch.clamp(lam * r / rbar, max=1.0)
        assert (lam * r / rbar > 1).any(), "some elements must reach the clip of a"
    else:
        u, a = g, min(1.0, lam)
    want = (p0 + (a * d - lr * u)).cpu().numpy()
    got = tr.flat_p.double().cpu().numpy()
    terms = (a * d).abs() + lr * u.abs()
    ulp_s = _ulp32(terms.cpu().numpy())
    tol = _ulp32(want) + 4 * ulp_s
    err = np.abs(got - want)
    _record("dyneval_update_err_over_tol", float((err / tol).max()))
    bad = np.nonzero(err > tol)[0]
    assert bad.size == 0, (f"{bad.size} elements off, first {bad[:5]}: got {got[bad[:5]]} want {want[bad[:5]]}, "
                           f"err / ulp(S) {err[bad[:5]] / ulp_s[bad[:5]]}, err / ulp(want) {err[bad[:5]] / _ulp32(want)[bad[:5]]}")
    assert (np.abs(got - p0.cpu().numpy()) > 0).mean() > 0.3, "the parameters must move"

    # images: the adapted context against a fresh one packed from the same fp32 weights
    m2 = _model(name, "tc", p=0.5, tied=tied)
    _copy_weights(m2, m)
    tr2 = _trainer(m2, name)
    for (h1, c1), (h2, c2) in zip(tr.states, tr2.states):
        h2.copy_(h1); c2.copy_(c1)
    x, y = _windows(name, 1, seed=9)[0]
    out = []
    for t in (tr, tr2):
        _lib.check(lib.zrb_prof_enable(t.ctx, 1))
        loss, tp = t.eval_step(x, y, want_probs=True)
        out.append((loss.clone(), tp.clone(), [s.clone() for st in t.states for s in st], _prof_counts(lib, t.ctx)))
    pack = _lib.PROF_CLASSES.index("pack")
    assert out[0][3][pack] == 0, "the adapted context repacked: its images were not marked current"
    assert out[1][3][pack] >= 1
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1]), "stale fp16 images"
    for a_, b_ in zip(out[0][2], out[1][2]):
        assert torch.equal(a_, b_), "stale recurrent images"
    assert isinstance(stats, (zaremba_b200.GradStats, type(None)))


def _oracle_params(m):
    return {k: v.detach().double().cpu().numpy() for k, v in m.named_parameters() if not (m.tied and k == "fc.W")}


@pytest.mark.parametrize("rule", ["rms", "sgd"])
@pytest.mark.parametrize("tied", [False, True], ids=["untied", "tied"])
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", ["fixture", "small"])
def test_whole_pass_matches_the_restatement(name, engine, tied, rule):
    V, H, L, T, B, _ = _shape(name)
    tol = TOL[engine]
    m = _model(name, engine, p=0.5, tied=tied)
    tr = _trainer(m, name)
    wins = _windows(name, 5, seed=4)
    P0 = _oracle_params(m)
    stats = tr.gradient_stats(wins) if rule == "rms" else None
    # eps = r-bar keeps u = g / (r + eps) within |g| / r-bar, so that the engines' gradient error is not amplified by
    # elements whose r is tiny
    lr, lam = (1e-3, 0.05) if rule == "rms" else (0.5, 0.05)
    eps = float(stats.mean) if stats is not None else 2e-5
    rms = rbar = None
    if stats is not None:       # the restatement takes the device's r (the statistics are checked on their own below)
        base = tr.flat_p.data_ptr()
        rms = {k: stats.rms[(q.data_ptr() - base) // 4:][:q.numel()].double().view_as(q).cpu().numpy()
               for k, q in m.named_parameters() if not (tied and k == "fc.W")}
        rbar = float(stats.mean)
    got = []
    tr.reset_states()
    theta_g = tr.flat_p.clone()
    for x, y in wins:
        got.append(tr.dynamic_eval_step(x, y, theta_g, lr, lam, stats, eps).item())
    batches = [(x.cpu().numpy(), y.cpu().numpy()) for x, y in wins]
    from oracle import lstm_lm_oracle as O
    want, Pw, _ = DO.dynamic_pass(P0, batches, L, O.zero_states(L, B, H, np.float64), lr, lam, rms, rbar, eps,
                                tied)
    for s, (a, b) in enumerate(zip(got, want)):
        _record("loss", abs(a - b) / max(1.0, abs(b)))
        assert abs(a - b) <= tol["loss"] * max(1.0, abs(b)), (s, a, b)
    for k, q in m.named_parameters():
        if tied and k == "fc.W":
            continue
        _scale_close(q.detach().cpu().numpy(), Pw[k], tol["grad"], f"{name} param {k}")
    assert got[0] != got[-1]


@pytest.mark.parametrize("engine", ENGINES)
def test_identities(engine):
    """lr = lam = 0 is perplexity() exactly with theta bit-unchanged; window 0 is zrb_eval_step's loss at lr > 0;
    restore=True puts theta_g back bit for bit."""
    m = _model("small", engine, p=0.5)
    tr = _trainer(m, "small")
    wins = _windows("small", 4, seed=6)
    p0 = tr.flat_p.clone()
    want = tr.perplexity([(x.cpu(), y.cpu()) for x, y in wins])
    stats = tr.gradient_stats(wins[:2])
    for st in (None, stats):
        got = tr.dynamic_perplexity([(x.cpu(), y.cpu()) for x, y in wins], 0.0, 0.0, st, restore=False)
        assert got == want, (got, want)
        assert torch.equal(tr.flat_p, p0)
    tr.reset_states()
    l0 = tr.eval_step(*wins[0]).clone()
    tr.reset_states()
    l1 = tr.dynamic_eval_step(*wins[0], p0, 0.5, 0.1).clone()
    assert torch.equal(l0, l1), (l0.item(), l1.item())
    assert not torch.equal(tr.flat_p, p0)
    tr.flat_p.copy_(p0)
    tr.params_changed()
    adapted = tr.dynamic_perplexity([(x.cpu(), y.cpu()) for x, y in wins], 0.5, 0.02)
    assert adapted != want
    assert torch.equal(tr.flat_p, p0)
    assert tr.perplexity([(x.cpu(), y.cpu()) for x, y in wins]) == want


@pytest.mark.parametrize("tied", [False, True], ids=["untied", "tied"])
def test_lazy_update_with_pending_updates_equals_strict(tied):
    res = {}
    for lazy in (False, True):
        m = _model("small", "tc", p=0.5, tied=tied)
        tr = _trainer(m, "small", lazy_update=lazy)
        tr.seed = 11
        for x, y in _windows("small", 2, seed=8):
            tr.train_step(x, y, 1.0, 0.5)
        wins = [(x.cpu(), y.cpu()) for x, y in _windows("small", 3, seed=10)]
        stats = tr.gradient_stats(wins[:2])
        ppl = tr.dynamic_perplexity(wins, 2e-4, 0.05, stats, restore=False)
        torch.cuda.synchronize()
        res[lazy] = (ppl, stats.rms.clone(), stats.mean.clone(), tr.flat_p.clone())
    assert res[False][0] == res[True][0]
    for a, b in zip(res[False][1:], res[True][1:]):
        assert torch.equal(a, b)


@pytest.mark.parametrize("tied", [False, True], ids=["untied", "tied"])
@pytest.mark.parametrize("engine", ENGINES)
def test_statistics(engine, tied):
    """r and r-bar over K = 6 windows against float64 from the per-window gradients (relative 1e-6); two runs are
    bit-identical; a tied model counts E once."""
    m = _model("small", engine, p=0.5, tied=tied)
    tr = _trainer(m, "small")
    wins = _windows("small", 6, seed=12)
    p0 = tr.flat_p.clone()
    tr.reset_states()
    ms = torch.zeros_like(tr.flat_p, dtype=torch.float64)
    for x, y in wins:           # per-window gradients at theta_g, states carried from zero
        tr.dynamic_eval_step(x, y, p0, 0.0, 0.0)
        ms += tr.flat_g.double() ** 2
    assert torch.equal(tr.flat_p, p0)
    r64 = (ms / len(wins)).sqrt()
    s1 = tr.gradient_stats(wins)
    s2 = tr.gradient_stats(wins)
    assert torch.equal(s1.rms, s2.rms) and torch.equal(s1.mean, s2.mean), "the statistics must be bit-reproducible"
    assert s1.windows == len(wins)
    assert s1.rms.numel() == sum(q.numel() for q in m.parameters()) == tr.flat_p.numel()
    err = ((s1.rms.double() - r64).abs() / r64.clamp_min(1e-9 * r64.max().item())).max().item()
    _record("stats_rel", err)
    assert err <= 1e-6, err
    rbar64 = r64.sum().item() / r64.numel()
    assert abs(float(s1.mean) - rbar64) <= 1e-6 * rbar64
    assert torch.equal(tr.flat_p, p0)


def test_rejections_leave_everything_unchanged():
    from zaremba_b200 import _lib
    lib = _lib.load()
    for tied in (False, True):
        m = _model("steps_b40", "tc", p=0.5, tied=tied)
        tr = _trainer(m, "steps_b40", states_seed=1)
        (x, y), = _windows("steps_b40", 1)
        T, B = x.shape
        stats = tr.gradient_stats([(x, y)])
        tr.flat_g.fill_(0.25)
        before = [tr.flat_p.clone(), tr.flat_g.clone()] + [t.clone() for st in tr.states for t in st]
        gl = tr._flat_params_struct(tr.flat_p.clone())
        keep = tr.flat_p.clone()
        rms = tr._flat_params_struct(stats.rms)
        nan, inf = float("nan"), float("inf")
        bad = [dict(lr=-1.0), dict(lr=nan), dict(lr=inf), dict(lam=-0.1), dict(lam=nan), dict(lam=inf),
               dict(eps=0.0), dict(eps=-1.0), dict(eps=nan), dict(eps=inf), dict(mean=None)]
        for kw in bad:
            a = dict(lr=0.1, lam=0.1, eps=2e-5, mean=_lib.ptr(stats.mean))
            a.update(kw)
            rc = lib.zrb_dyneval_step(tr.ctx, C.byref(tr._ps), C.byref(tr._gs), C.byref(gl), C.byref(rms), a["mean"],
                                      _lib.ptr(x), _lib.ptr(y), T, B, C.byref(tr._st), C.byref(tr._st), a["lr"],
                                      a["lam"], a["eps"], _lib.ptr(tr.loss), tr._stream())
            assert rc == -1, kw
        ms = tr._flat_params_struct(torch.zeros_like(tr.flat_p))
        assert lib.zrb_grad_stats_finish(tr.ctx, C.byref(ms), 0, _lib.ptr(stats.mean), tr._stream()) == -1
        assert lib.zrb_grad_stats_finish(tr.ctx, C.byref(ms), -3, _lib.ptr(stats.mean), tr._stream()) == -1
        if tied:   # a zrb_params whose fc_w != embed_w
            for which in ("grads", "global", "rms", "ms"):
                structs = {"grads": tr._gs, "global": gl, "rms": rms, "ms": ms}
                s = _lib.ZrbParams.from_buffer_copy(structs[which])
                s.fc_w = s.fc_b
                structs[which] = s
                if which == "ms":
                    rc = lib.zrb_grad_stats_step(tr.ctx, C.byref(tr._ps), C.byref(tr._gs), C.byref(s), _lib.ptr(x),
                                                 _lib.ptr(y), T, B, C.byref(tr._st), C.byref(tr._st), None,
                                                 tr._stream())
                    assert rc == -1
                    assert lib.zrb_grad_stats_finish(tr.ctx, C.byref(s), 1, _lib.ptr(stats.mean), tr._stream()) == -1
                    continue
                rc = lib.zrb_dyneval_step(tr.ctx, C.byref(tr._ps), C.byref(structs["grads"]), C.byref(structs["global"]),
                                          C.byref(structs["rms"]), _lib.ptr(stats.mean), _lib.ptr(x), _lib.ptr(y), T, B,
                                          C.byref(tr._st), C.byref(tr._st), 0.1, 0.1, 2e-5, _lib.ptr(tr.loss),
                                          tr._stream())
                assert rc == -1, which
        torch.cuda.synchronize()
        after = [tr.flat_p, tr.flat_g] + [t for st in tr.states for t in st]
        for a_, b_ in zip(before, after):
            assert torch.equal(a_, b_), "a rejected call changed a buffer"
        # the context is still usable, and the SGD rule needs neither eps nor rms_mean
        tr.dynamic_eval_step(x, y, keep, 0.1, 0.1, None, eps=-1.0)
        tr.dynamic_eval_step(x, y, keep, 2e-4, 0.1, stats)
        torch.cuda.synchronize()
        assert torch.isfinite(tr.flat_p).all() and not torch.equal(tr.flat_p, keep)


def test_data_parallel_is_refused():
    m = _model("steps_b40", "tc")
    tr = _trainer(m, "steps_b40")
    tr.world = 2
    (x, y), = _windows("steps_b40", 1)
    with pytest.raises(ValueError, match="data_parallel=False"):
        tr.dynamic_eval_step(x, y, tr.flat_p.clone(), 0.1)
    with pytest.raises(ValueError):
        tr.gradient_stats([(x, y)])
    with pytest.raises(ValueError):
        tr.dynamic_perplexity([(x, y)], 0.1)


def test_trainer_rejects_mismatched_arguments():
    """theta_g / statistics of the wrong size, dtype or device are refused on every call (also after a valid call has
    cached the pointer structs), and so is a window wider than the Trainer's states."""
    m = _model("steps_b40", "tc")
    tr = _trainer(m, "steps_b40")
    (x, y), = _windows("steps_b40", 1)
    theta_g = tr.flat_p.clone()
    tr.dynamic_eval_step(x, y, theta_g, 0.1)
    stats = tr.gradient_stats([(x, y)])
    for bad in (theta_g[:-1], theta_g.double(), theta_g.cpu(), torch.empty(2 * theta_g.numel(), device=DEV)[::2]):
        with pytest.raises(ValueError):
            tr.dynamic_eval_step(x, y, bad, 0.1)
    import zaremba_b200
    for bad in (zaremba_b200.GradStats(stats.rms[:-1], stats.mean, 1), zaremba_b200.GradStats(stats.rms, stats.rms, 1)):
        with pytest.raises(ValueError):
            tr.dynamic_eval_step(x, y, theta_g, 1e-4, 0.1, bad)
    wide = [torch.cat([t, t], dim=1).contiguous() for t in (x, y)]       # [T, 2B]
    tr.gradient_stats([tuple(wide)])                                      # grows the model's context to 2B ...
    with pytest.raises(ValueError, match="exceeds the Trainer's batch"):
        tr.dynamic_eval_step(*wide, theta_g, 0.1)                        # ... but the Trainer's states hold B rows
    tr.dynamic_eval_step(x, y, theta_g, 0.1)
    torch.cuda.synchronize()
    assert torch.isfinite(tr.flat_p).all()
