"""GPU tests of Adam in the fused train step (DESIGN.md section 21) at the recurrence-plan branches of
tests/test_gpu_dropout.py and at the Small / Medium / Large shapes.

  * bit for bit per step: with keep_clipped_grads=True `.grad` holds the exact g' after a step, and p, m and v equal
    the fp32 restatement of tests/_adam_oracle.py applied to the previous p, m, v and that g' -- rows-only and dense
    embedding, tied, weight drop, variational dropout, train_step_host, lazy update, the validation engine and a
    Mixture-of-Softmaxes head (K = 3);
  * keep_clipped_grads=False gives the same p, m, v bit for bit;
  * the whole run against fp64: K carried steps against tests/_model_oracle.py's gradients with fp64 Adam -- loss,
    clip norm, parameters, m and v -- on both engines, rows-only and tied;
  * lazy equals strict bit for bit, also with evaluation, generation and flush() between steps while updates pend;
  * dynamic evaluation, gradient statistics (also for windows that make the model re-create its context),
    perplexity and zrb_clip_sgd leave m, v and t alone, and training continues like an untouched twin;
  * torch interop: the drop-in Model + clip_grad_norm_ + torch.optim.Adam tracks the fused Trainer;
    optimizer_state_dict() loads into torch.optim.Adam and back; 2 steps, save, load into a fresh Trainer with the
    default betas, 2 steps equals 4 straight steps bit for bit (untied, tied, MoS head);
  * every refusal of zrb_set_adam / zrb_set_average / zrb_train_step_update / the Trainer;
  * two GPUs (skipped otherwise): every rank's p, m and v are identical.
Windows hold distinct tokens, so the embedding scatter is deterministic and twins can be compared bit for bit.
"""
import ctypes as C
import gc
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import _adam_oracle as AO
from tests.test_gpu_asgd import SHAPES, _dev, _row
from tests.test_gpu_dropout import L, P_DROP, ROW_IDS
from tests.test_gpu_parity import ENGINES, _caller_nll_loss

pytestmark = pytest.mark.gpu

LR, MAX_NORM = 2e-3, 0.25
BETAS, EPS = (0.9, 0.999), 1e-8
K = 4                    # train steps per run

# feature -> (Model kwargs, Trainer kwargs, host steps, dense embedding)
FEATURES = {
    "rows_only": ({}, {}, False, False),
    "dense_embed": ({}, {}, False, True),
    "tied": ({"tied": True}, {}, False, False),
    "weight_drop": ({"weight_drop": 0.5}, {}, False, False),
    "variational": ({"variational": True}, {}, False, False),
    "host": ({}, {}, True, False),
    "lazy": ({}, {"lazy_update": True}, False, False),
    "lazy_tied_wd": ({"tied": True, "weight_drop": 0.5}, {"lazy_update": True}, False, False),
    "mos": ({"experts": 3}, {}, False, False),
    "melis": ({}, {"betas": (0.0, 0.999), "eps": 1e-9}, False, False),
}
FEATURE_ROW = [r for r in ("tc_h48", "simt_h48") if r in ROW_IDS]
CASES = ([(r, "rows_only") for r in ROW_IDS]
         + [(r, f) for r in FEATURE_ROW for f in FEATURES if f != "rows_only" and not (f == "mos" and "simt" in r)]
         + ([(s, "rows_only") for s in SHAPES] + [("medium", "lazy"), ("large", "lazy"), ("small", "mos")]
            if "tc" in ENGINES else []))


def _winit(row):
    return min(row.winit, 1.3 / np.sqrt(row.H))


def _model(row, **kw):
    import zaremba_b200
    torch.manual_seed(row.torch_seed)
    m = zaremba_b200.Model(row.V, row.H, L, P_DROP, _winit(row), engine=row.engine, **kw).to(_dev())
    m.train()
    return m


def _trainer(row, feature, monkeypatch, **extra):
    import zaremba_b200
    mkw, tkw, _, dense = FEATURES[feature]
    monkeypatch.setenv("ZRB_EMBED_SPARSE", "0" if dense else "1")
    m = _model(row, **mkw)
    kw = dict(optimizer="adam", betas=BETAS, eps=EPS)
    kw.update(tkw)
    kw.update(extra)
    tr = zaremba_b200.Trainer(m, row.B, row.T, **kw)
    for (h, c), (h0, c0) in zip(tr.states, row.states()):
        h.copy_(h0)
        c.copy_(c0)
    row.check_branch(tr.ctx)
    return m, tr


def _step(tr, row, s, host):
    x, y = row.x[s % 2], row.y[s % 2]
    if host:
        loss, norm = tr.train_step_host(x, y, LR, MAX_NORM)
        return torch.tensor(loss), torch.tensor(norm)
    loss, norm = tr.train_step(x.to(_dev()), y.to(_dev()), LR, MAX_NORM)
    return loss.clone(), norm.clone()


def _snap(tr):
    tr.flush()
    torch.cuda.synchronize()
    return dict(p=tr.flat_p.cpu(), g=tr.flat_g.cpu(), m=tr.flat_m.cpu(), v=tr.flat_v.cpu(), t=tr.adam_step)


def _run(row, feature, monkeypatch, keep=True, between=None, **extra):
    """K steps; the state before the first and after every step.  between(tr, s): called before step s >= 1."""
    m, tr = _trainer(row, feature, monkeypatch, keep_clipped_grads=keep, **extra)
    host = FEATURES[feature][2]
    out = [_snap(tr)]
    for s in range(K):
        if between is not None and s >= 1:
            between(tr, s)
        loss, norm = _step(tr, row, s, host)
        snap = _snap(tr)
        snap.update(loss=loss.cpu(), norm=norm.cpu())
        out.append(snap)
    tr.close()
    del tr, m
    gc.collect()
    return out


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def _betas(feature):
    tkw = FEATURES[feature][1]
    return tkw.get("betas", BETAS), tkw.get("eps", EPS)


def _oracle_check(run, feature, what):
    (b1, b2), eps = _betas(feature)
    for s in range(1, len(run)):
        prev, cur = run[s - 1], run[s]
        assert cur["t"] == s
        p, _, m, v = AO.adam_fp32(prev["p"].numpy(), cur["g"].numpy(), prev["m"].numpy(), prev["v"].numpy(), 1.0, LR,
                                  b1, b2, eps, s)
        for name, want in (("p", p), ("m", m), ("v", v)):
            got = cur[name].numpy()
            bad = np.flatnonzero(got.view(np.int32) != want.view(np.int32))
            assert bad.size == 0, (what, s, name, bad.size, bad[:4], got[bad[:4]], want[bad[:4]])


@pytest.mark.parametrize("row_id,feature", CASES, ids=[f"{r}-{f}" for r, f in CASES])
def test_every_step_is_the_restatement_and_keep_clipped_does_not_matter(row_id, feature, monkeypatch):
    row = _row(row_id)
    kept = _run(row, feature, monkeypatch, keep=True)
    _oracle_check(kept, feature, f"{row_id}/{feature}")
    assert any(s["m"].abs().max() > 0 for s in kept[1:]) and float(kept[-1]["norm"]) > 0
    plain = _run(_row(row_id), feature, monkeypatch, keep=False)
    for s, (a, b) in enumerate(zip(kept, plain)):
        for name in ("p", "m", "v"):
            assert _bits_equal(a[name], b[name]), (row_id, feature, s, name)


# ---- the whole run against fp64 ---------------------------------------------------------------------------------------
# Largest error measured on an H100 (DESIGN.md section 21), and the tolerances per engine, about 3x those: loss and clip
# norm relative; m and v as max |error| over max |reference| per tensor; p as the L2 error of the displacement p - p_0
# over the reference displacement's L2 norm per tensor (an element whose true gradient is tiny may take the opposite
# sign from fp16 operands, and Adam turns that into a whole step of the other sign, so p is judged as a direction of
# travel; the carried steps then start from slightly different weights, which the later m and v inherit).  The fp64
# Adam takes the betas as the library does, rounded to fp32 (the C ABI's type).
TOL64 = {"tc": {"loss": 3e-6, "norm": 2e-4, "p": 7e-2, "m": 4.5e-2, "v": 6e-2},
         "simt": {"loss": 2.5e-7, "norm": 2e-7, "p": 7.5e-5, "m": 2e-6, "v": 3e-6}}
ORACLE_CASES = [(r, f) for r in ("tc_h48", "odd_h", "simt_h48") if r in ROW_IDS for f in ("rows_only", "tied")
                if not (r == "odd_h" and f == "tied")]


def _adam64(P, M, V, grads, coef, t, betas, eps):
    for k in P:
        P[k], _, M[k], V[k] = (torch.as_tensor(a) for a in AO.adam_fp64(P[k].numpy(), grads[k].numpy(), M[k].numpy(),
                                                                        V[k].numpy(), coef, LR, betas[0], betas[1],
                                                                        eps, t))


@pytest.mark.parametrize("row_id,feature", ORACLE_CASES, ids=[f"{r}-{f}" for r, f in ORACLE_CASES])
def test_the_run_against_fp64_adam(row_id, feature, monkeypatch):
    """K carried steps against tests/_model_oracle.py's fp64 gradients (the Trainer's Philox masks, states carried)
    with fp64 Adam on the oracle's own p, m and v: loss, clip norm, parameters, m and v after every step."""
    from tests import _model_oracle as MO
    row = _row(row_id)
    m, tr = _trainer(row, feature, monkeypatch, keep_clipped_grads=False)
    tied = feature == "tied"
    names = [k for k, _ in m.named_parameters()]
    assert names == MO.names(L, tied)
    P = {k: q.detach().cpu().double() for k, q in m.named_parameters()}
    P0 = {k: v.clone() for k, v in P.items()}
    M = {k: torch.zeros_like(v) for k, v in P.items()}
    V = {k: torch.zeros_like(v) for k, v in P.items()}
    st = [(h.double().reshape(row.B, row.H), c.double().reshape(row.B, row.H)) for h, c in row.states()]
    st = [(h.cpu(), c.cpu()) for h, c in st]
    tol = TOL64[row.engine]
    betas = tuple(float(np.float32(b)) for b in BETAS)
    worst = {k: (0.0, "") for k in tol}
    for s in range(K):
        x, y = row.x[s % 2], row.y[s % 2]
        md = MO.Modes(seed=tr.seed, step=tr.step, p=P_DROP)
        loss64, norm64, grads, _, st, _ = MO.train_step(P, x, y, st, L, tied, LR, MAX_NORM, md)
        _adam64(P, M, V, grads, min(1.0, MAX_NORM / (norm64 + 1e-6)), s + 1, betas, EPS)
        loss, norm = _step(tr, row, s, False)
        got = _snap(tr)
        errs = {"loss": abs(float(loss) - loss64) / abs(loss64), "norm": abs(float(norm) - norm64) / norm64}
        params = dict(m.named_parameters())
        base = tr.flat_p.data_ptr()
        for k, q in params.items():
            off, n = (q.data_ptr() - base) // 4, q.numel()
            gp, gm, gv = (got[w][off:off + n].view(q.shape).double() for w in ("p", "m", "v"))
            d_ref = P[k] - P0[k]
            errs[f"p {k}"] = float((gp - P[k]).norm() / d_ref.norm())
            errs[f"m {k}"] = float((gm - M[k]).abs().max() / M[k].abs().max())
            errs[f"v {k}"] = float((gv - V[k]).abs().max() / V[k].abs().max())
        for name, e in errs.items():
            cls = name.split()[0]
            if e > worst[cls][0]:
                worst[cls] = (e, f"step {s} {name}")
    tr.close()
    print(f"fp64 run {row_id}/{feature}: " + ", ".join(f"{k} {v[0]:.2e} ({v[1]})" for k, v in worst.items()))
    for cls, (e, where) in worst.items():
        assert e <= tol[cls], (row_id, feature, where, e)


LAZY_SHAPES = [s for s in ("tc_h48", "small", "medium", "large") if "tc" in ENGINES and (s in SHAPES or s in ROW_IDS)]


def _base_row_id():
    return FEATURE_ROW[0] if FEATURE_ROW else ROW_IDS[0]


@pytest.mark.parametrize("shape", LAZY_SHAPES)
def test_lazy_equals_strict(shape, monkeypatch):
    """6 steps without a flush of the test's own: steps 2 and 4 take the previous step's deferred updates beside their
    forward recurrences; before steps 1, 3 and 5 an evaluation, a generation and a flush() apply them."""
    def run(feature):
        row = _row(shape)
        m, tr = _trainer(row, feature, monkeypatch, keep_clipped_grads=True)
        losses = []
        for s in range(6):
            if s == 1:
                tr.eval_step(row.x[0].to(_dev()), row.y[0].to(_dev()))
            elif s == 3:
                tr.model.generate(row.x[1][:2].to(_dev()), 3, seed=5)
            elif s == 5:
                tr.flush()
            loss, norm = _step(tr, row, s, False)
            losses += [loss, norm]
        out = _snap(tr)
        out["ln"] = torch.stack(losses).cpu()
        tr.close()
        del tr, m
        gc.collect()
        return out
    strict, lazy = run("rows_only"), run("lazy")
    for name in ("p", "g", "m", "v", "ln"):
        assert _bits_equal(strict[name], lazy[name]), (shape, name)
    assert strict["t"] == lazy["t"] == 6


# ---- other entry points leave the moments alone ---------------------------------------------------------------------
def _clip_sgd(tr):
    """zrb_clip_sgd on copies of the parameters (the weights stay as they are)"""
    from zaremba_b200 import _lib
    params = list(tr.model.ordered_parameters())
    n = len(params)
    copies = [p.detach().clone() for p in params]
    grads = [torch.full_like(p, 0.5) for p in params]
    norm = torch.zeros((), device=_dev())
    _lib.check(_lib.load().zrb_clip_sgd(tr.ctx, n, (C.c_void_p * n)(*[q.data_ptr() for q in copies]),
                                        (C.c_void_p * n)(*[g.data_ptr() for g in grads]),
                                        (C.c_int64 * n)(*[p.numel() for p in params]), 0.5, 0.25,
                                        C.c_void_p(norm.data_ptr()), None))


def test_other_entry_points_leave_the_moments_alone(monkeypatch):
    """A twin resets its states between steps; the other one also runs dynamic evaluation and perplexity, gradient
    statistics (the second over windows twice as long, which re-create the model's context), and zrb_clip_sgd."""
    def others(row):
        def f(tr, s):
            saved = tr.flat_p.clone()
            wins = [(row.x[0], row.y[0])]
            if s == 1:
                tr.dynamic_perplexity(wins, lr=0.1)
                tr.perplexity(wins)
            elif s == 2:
                tr.gradient_stats(wins)
                serial = tr.model._ctx_serial
                tr.gradient_stats([(torch.cat([row.x[0], row.x[1]]), torch.cat([row.y[0], row.y[1]]))])
                assert tr.model._ctx_serial != serial
            else:
                _clip_sgd(tr)
            torch.cuda.synchronize()
            assert _bits_equal(tr.flat_p, saved)
            tr.reset_states()
        return f
    r1, r2 = _row(_base_row_id()), _row(_base_row_id())
    twin = _run(r1, "rows_only", monkeypatch, between=lambda tr, s: tr.reset_states())
    got = _run(r2, "rows_only", monkeypatch, between=others(r2))
    for s, (a, b) in enumerate(zip(twin, got)):
        assert a["t"] == b["t"] == s
        for name in ("p", "m", "v"):
            assert _bits_equal(a[name], b[name]), (s, name)


# ---- torch interop --------------------------------------------------------------------------------------------------
def test_dropin_with_torch_adam_tracks_the_trainer(monkeypatch):
    """dropout 0: the drop-in Model under autograd + clip_grad_norm_ + torch.optim.Adam against the fused step.  The
    gradients come from the same kernels; the updates differ by torch's rounding, its fp64 betas (tests/test_adam_cpu.py)
    and its own clip norm, and Adam's normalised step amplifies that only where |g| is near eps."""
    import zaremba_b200
    row = _row(_base_row_id())
    monkeypatch.setenv("ZRB_EMBED_SPARSE", "1")
    torch.manual_seed(row.torch_seed)
    m = zaremba_b200.Model(row.V, row.H, L, 0.0, _winit(row), engine=row.engine).to(_dev())
    ref = {k: v.detach().clone() for k, v in m.state_dict().items()}
    tr = zaremba_b200.Trainer(m, row.B, row.T, optimizer="adam", betas=BETAS, eps=EPS)
    for s in range(K):
        tr.train_step(row.x[s % 2].to(_dev()), row.y[s % 2].to(_dev()), LR, MAX_NORM)
    tr.flush()
    fused = {k: p.detach().clone() for k, p in m.named_parameters()}
    tr.close()
    del tr, m
    gc.collect()
    d = zaremba_b200.Model(row.V, row.H, L, 0.0, _winit(row), engine=row.engine).to(_dev())
    d.load_state_dict(ref)
    opt = torch.optim.Adam(d.parameters(), lr=LR, betas=BETAS, eps=EPS)
    states = d.state_init(row.B)
    for s in range(K):
        opt.zero_grad(set_to_none=True)
        scores, states = d(row.x[s % 2], states)
        _caller_nll_loss(scores, row.y[s % 2]).backward()
        torch.nn.utils.clip_grad_norm_(d.parameters(), MAX_NORM)
        opt.step()
        states = d.detach(states)
    for k, p in d.named_parameters():
        moved = (fused[k] - ref[k]).abs().max().item()
        err = (p.detach() - fused[k]).abs().max().item()
        assert moved > 0, k
        assert err <= 0.05 * moved, (k, err, moved)


SAVED_BETAS, SAVED_EPS = (0.5, 0.99), 1e-7      # not the Trainer's defaults: the resumed Trainer must take them


@pytest.mark.parametrize("feature", ["rows_only", "tied"] + (["mos"] if "tc" in ENGINES else []))
def test_state_dict_round_trip_and_resume(feature, monkeypatch):
    """2 steps with non-default betas and eps, optimizer_state_dict() through torch.optim.Adam's load_state_dict /
    state_dict, then a Trainer created with the defaults on the saved weights and states loads it and trains 2 more:
    the same p, m, v as 4 straight steps, bit for bit.  Tied (E sits next to fc.b in the flat layout) and the MoS head
    (its tensors laid out last) check the state's indices against model.parameters(); the embedding's moments must be
    zero exactly in the rows of tokens no window holds."""
    import zaremba_b200
    rid = _base_row_id() if feature != "mos" else "tc_h48"
    hyper = dict(betas=SAVED_BETAS, eps=SAVED_EPS)
    straight = _run(_row(rid), feature, monkeypatch, **hyper)
    row = _row(rid)
    m, tr = _trainer(row, feature, monkeypatch, keep_clipped_grads=True, **hyper)
    for s in range(2):
        _step(tr, row, s, False)
    sd = tr.optimizer_state_dict()
    params = {k: v.detach().clone() for k, v in m.state_dict().items()}
    states = [(h.clone(), c.clone()) for h, c in tr.states]
    plist = list(m.parameters())
    assert sorted(sd["state"]) == list(range(len(plist)))
    for i, p in enumerate(plist):
        assert sd["state"][i]["exp_avg"].shape == p.shape and sd["state"][i]["exp_avg_sq"].shape == p.shape, i
    seen = torch.zeros(row.V, dtype=torch.bool)
    seen[torch.cat([row.x[0].reshape(-1), row.x[1].reshape(-1)])] = True
    emb = [i for i, p in enumerate(plist) if p is m.embed.W]
    assert len(emb) == 1
    rows_nonzero = sd["state"][emb[0]]["exp_avg_sq"].cpu().abs().sum(1) > 0
    if feature == "tied":          # E is also the projection: every row has a gradient
        assert rows_nonzero.all()
    else:
        assert torch.equal(rows_nonzero, seen)
    opt = torch.optim.Adam(m.parameters(), lr=1.0)
    opt.load_state_dict(sd)
    assert opt.param_groups[0]["betas"] == SAVED_BETAS and opt.param_groups[0]["eps"] == SAVED_EPS
    assert all(float(opt.state[p]["step"]) == 2.0 for p in m.parameters())
    sd2 = opt.state_dict()
    tr.close()
    del tr, m, opt
    gc.collect()
    m2 = _model(row, **FEATURES[feature][0])     # seeds torch as before: the Trainer's dropout seed
    m2.load_state_dict(params)
    tr2 = zaremba_b200.Trainer(m2, row.B, row.T, keep_clipped_grads=True, optimizer="adam")
    assert tr2._betas == BETAS and tr2._eps == EPS
    tr2.load_optimizer_state_dict(sd2)
    assert tr2.adam_step == 2 and tr2._betas == SAVED_BETAS and tr2._eps == SAVED_EPS
    tr2.step = 2                             # the dropout masks of steps 3 and 4
    for (h, c), (h0, c0) in zip(tr2.states, states):
        h.copy_(h0)
        c.copy_(c0)
    for s in range(2, 4):
        _step(tr2, row, s, False)
    got = _snap(tr2)
    assert got["t"] == 4
    for name in ("p", "m", "v"):
        assert _bits_equal(got[name], straight[4][name]), name
    tr2.close()


# ---- refusals -------------------------------------------------------------------------------------------------------
def test_refusals(monkeypatch):
    from zaremba_b200 import _lib
    lib = _lib.load()
    row = _row(_base_row_id())
    m, tr = _trainer(row, "rows_only", monkeypatch)
    ctx = tr.ctx
    ms, vs = tr._m_s, tr._v_s
    E = -1

    def set_adam(m_, v_, b1=0.9, b2=0.999, eps=1e-8, step=0):
        return lib.zrb_set_adam(ctx, None if m_ is None else C.byref(m_), None if v_ is None else C.byref(v_), b1, b2,
                                eps, step)
    for b in (-0.1, 1.0, 1.5, float("nan"), float("inf")):
        assert set_adam(ms, vs, b1=b) == E and set_adam(ms, vs, b2=b) == E, b
    for e in (0.0, -1e-8, float("nan"), float("inf")):
        assert set_adam(ms, vs, eps=e) == E, e
    assert set_adam(ms, vs, step=-1) == E
    assert set_adam(ms, None) == E and set_adam(None, vs) == E
    assert set_adam(ms, ms) == E                     # m and v overlap
    # a moment tensor that is not 4-byte aligned (in a buffer of its own, so it overlaps nothing); never left installed
    spare = torch.zeros(tr.flat_m.numel() + 1, device=_dev())
    odd = _lib.ZrbParams.from_buffer_copy(ms)
    odd.w_hh[0] = spare.data_ptr() + 2
    try:
        assert set_adam(odd, vs) == E
    finally:
        set_adam(None, None)
    # moments that alias the parameters pass zrb_set_adam but stop the train step before anything is launched
    assert set_adam(tr._ps, vs) == 0
    before = tr.flat_p.clone()
    with pytest.raises(_lib.ZrbError):
        tr.train_step(row.x[0].to(_dev()), row.y[0].to(_dev()), LR, MAX_NORM)
    assert set_adam(tr._gs, vs) == 0
    with pytest.raises(_lib.ZrbError):
        tr.train_step(row.x[0].to(_dev()), row.y[0].to(_dev()), LR, MAX_NORM)
    torch.cuda.synchronize()
    assert _bits_equal(tr.flat_p, before)
    assert set_adam(ms, vs) == 0
    # averaging and Adam exclude each other
    avg = torch.zeros_like(tr.flat_p)
    avg_s = tr._flat_params_struct(avg)
    assert lib.zrb_set_average(ctx, C.byref(avg_s)) == E
    with pytest.raises(ValueError):
        tr.start_averaging()
    assert set_adam(None, None) == 0
    assert lib.zrb_set_average(ctx, C.byref(avg_s)) == 0
    assert set_adam(ms, vs) == E
    assert lib.zrb_set_average(ctx, None) == 0
    assert set_adam(ms, vs) == 0
    tr.close()
    del tr, m
    gc.collect()
    # a tied context refuses an untied pair of moments
    m, tr = _trainer(row, "tied", monkeypatch)
    bad = _lib.ZrbParams.from_buffer_copy(tr._m_s)
    bad.fc_w = tr.flat_v.data_ptr()
    assert lib.zrb_set_adam(tr.ctx, C.byref(bad), C.byref(tr._v_s), 0.9, 0.999, 1e-8, 0) == E
    tr.close()
    # the Trainer without Adam has no Adam state
    import zaremba_b200
    sgd = zaremba_b200.Trainer(_model(row), row.B, row.T)
    with pytest.raises(ValueError):
        sgd.optimizer_state_dict()
    sgd.close()


def test_no_adam_while_swapped(monkeypatch):
    import zaremba_b200
    from zaremba_b200 import _lib
    row = _row(_base_row_id())
    monkeypatch.setenv("ZRB_EMBED_SPARSE", "1")
    m = _model(row)
    tr = zaremba_b200.Trainer(m, row.B, row.T)
    tr.start_averaging()
    tr.train_step(row.x[0].to(_dev()), row.y[0].to(_dev()), 1.0, MAX_NORM)
    mm, vv = torch.zeros_like(tr.flat_p), torch.zeros_like(tr.flat_p)
    ms, vs = tr._flat_params_struct(mm), tr._flat_params_struct(vv)
    with tr.averaged_weights():
        assert _lib.load().zrb_set_adam(tr.ctx, C.byref(ms), C.byref(vs), 0.9, 0.999, 1e-8, 0) == -1
    tr.close()


# ---- two GPUs -------------------------------------------------------------------------------------------------------
_DP_SCRIPT = r"""
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, os.environ["ZRB_TEST_ROOT"])
import zaremba_b200
dist.init_process_group("nccl")
r = dist.get_rank(); torch.cuda.set_device(r)
torch.manual_seed(11)
m = zaremba_b200.Model(1000, 256, 2, 0.1, 0.05).cuda()
tr = zaremba_b200.Trainer(m, 8, 10, optimizer="adam")
g = torch.Generator().manual_seed(3)
for s in range(3):
    x = torch.randint(0, 1000, (10, 8 * dist.get_world_size()), generator=g)[:, 8 * r:8 * r + 8].contiguous().cuda()
    y = torch.randint(0, 1000, (10, 8 * dist.get_world_size()), generator=g)[:, 8 * r:8 * r + 8].contiguous().cuda()
    tr.train_step(x, y, 1e-3, 0.25)
tr.flush(); torch.cuda.synchronize()
out = os.environ["ZRB_TEST_OUT"]
torch.save({"p": tr.flat_p.cpu(), "m": tr.flat_m.cpu(), "v": tr.flat_v.cpu(), "t": tr.adam_step}, f"{out}/rank{r}.pt")
tr.close(); dist.destroy_process_group()
"""


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_keep_identical_moments(tmp_path):
    script = tmp_path / "dp.py"
    script.write_text(_DP_SCRIPT)
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    env = dict(os.environ, ZRB_TEST_ROOT=os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
               ZRB_TEST_OUT=str(tmp_path))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc_per_node=2",
                        f"--master_port={port}", str(script)], env=env, timeout=600,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    a, b = torch.load(tmp_path / "rank0.pt"), torch.load(tmp_path / "rank1.pt")
    assert a["t"] == b["t"] == 3
    for name in ("p", "m", "v"):
        assert _bits_equal(a[name], b[name]), name
