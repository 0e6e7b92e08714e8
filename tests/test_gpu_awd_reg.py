"""GPU tests of embedding dropout and AR/TAR (DESIGN.md section 17) at every recurrence-plan branch: the rows of
tests/test_gpu_dropout.py (every plan branch, the per-timestep path at B = 40, the validation engine).

  * equivalence, bit for bit: a step with the mode on equals a mode-off context whose embed.W holds fp32(W * s_e)
    (loss, scores, states and every other gradient), and dE = fp32(s_e * dE_off) -- on the fused Trainer and on the
    drop-in Model, alone and with the variational mode and weight drop;
  * two carried steps of the fused Trainer (and the drop-in Model) against the fp64 restatement of
    tests/_model_oracle.py with masks computed by oracle/philox.py, alone and with everything on (variational,
    weight drop, tied);
  * AR/TAR: alpha = beta = 0 is the mode off bit for bit; with alpha, beta > 0 the returned loss and the states are
    bit-identical to the mode off, R matches the fp64 oracle, and the penalties' own gradient contribution (gradients
    with alpha, beta minus gradients without) matches the oracle's;
  * everything on (p_e = 0.1, alpha = 2, beta = 1, variational, weight drop; untied and tied) against the oracle for two
    carried steps, also at the Small, Medium and Large shapes;
  * lazy equals strict (clipped gradients kept or not); eval untouched; p = 0 is the mode off; rejected arguments and
    call orders; two GPUs.
Windows hold distinct tokens, so the embedding scatter is deterministic.
"""
import ctypes as C
import dataclasses
import gc
import math
import os

import numpy as np
import pytest
import torch

from tests import _model_oracle as MO
from tests.test_gpu_dropout import L, P_DROP, ROW_IDS, Row
from tests.test_gpu_parity import ENGINES, TOL, _caller_nll_loss, _scale_close

pytestmark = pytest.mark.gpu

LR, MAX_NORM = 1.0, 0.25
STEP = 3          # a step other than 0, so that a mask keyed on the wrong word shows
P_E = 0.3         # (0.1 in the everything-on runs: AWD's setting)


def _dev():
    return torch.device("cuda:0")


def _winit(row):
    """The recipes' init scale, as tests/test_gpu_variational.py uses it (winit * sqrt(H) <= 1.3)."""
    return min(row.winit, 1.3 / math.sqrt(row.H))


def _model(row, p_e=0.0, **kw):
    import zaremba_b200
    torch.manual_seed(row.torch_seed)
    m = zaremba_b200.Model(row.V, row.H, L, P_DROP, _winit(row), engine=row.engine, embed_dropout=p_e, **kw).to(_dev())
    m.train()
    return m


def _lib_mask(seed, step, V, p):
    """the keep flags [V] as zrb_dropout_mask draws them (its equality with oracle/philox.py is pinned by
    test_gpu_dropout.test_dropout_mask_equals_reference)"""
    from zaremba_b200 import _lib
    out = torch.empty(V, dtype=torch.uint8, device=_dev())
    _lib.check(_lib.load().zrb_dropout_mask(seed, step, 3 * L + 1, V, p, _lib.ptr(out), None))
    return out.bool()


def _mul(mask, p):
    """the multiplier 0 / float32(1 / (1 - p)) of each row, as a [V, 1] column"""
    return (mask.float() * float(np.float32(1.0 / (1.0 - float(np.float32(p)))))).view(-1, 1)


def _offsets(model, tr):
    """{name: (offset, numel)} of every parameter in the Trainer's flat buffers (tied: E does not sit first)"""
    base = tr.flat_p.data_ptr()
    return {n: ((p.data_ptr() - base) // 4, p.numel()) for n, p in model.named_parameters()}


# ---- equivalence with a masked embedding, bit for bit -------------------------------------------------------------
def _trainer_grads(row, p_e, mul=None, **kw):
    """One fused step at STEP: loss, norm, states, {name: raw gradient}; mul: replace embed.W by embed.W * mul."""
    import zaremba_b200
    m = _model(row, p_e, **kw)
    if mul is not None:
        with torch.no_grad():
            m.embed.W.mul_(mul)
    tr = zaremba_b200.Trainer(m, row.B, row.T)
    for (h, c), (h0, c0) in zip(tr.states, row.states()):
        h.copy_(h0)
        c.copy_(c0)
    row.check_branch(tr.ctx)
    tr.step = STEP
    loss, norm = tr.train_step(row.x[0].to(_dev()), row.y[0].to(_dev()), LR, MAX_NORM)
    tr.flush()
    torch.cuda.synchronize()
    grads = {n: p.grad.detach().clone() for n, p in m.named_parameters()}
    out = dict(loss=loss.clone(), norm=norm.clone(), states=[t.clone() for st in tr.states for t in st], grads=grads)
    tr.close()
    del tr, m
    gc.collect()
    return out


def _dropin_grads(row, p_e, mul=None, **kw):
    """Drop-in Model at dropout step 0: forward, the caller's loss, backward."""
    m = _model(row, p_e, **kw)
    if mul is not None:
        with torch.no_grad():
            m.embed.W.mul_(mul)
    row.check_branch(m._context(row.T, row.B))
    scores, states = m(row.x[0], row.states())
    _caller_nll_loss(scores, row.y[0]).backward()
    out = dict(scores=scores.detach().clone(), states=[t.clone() for st in states for t in st],
               grads={n: p.grad.detach().clone() for n, p in m.named_parameters()})
    del m
    gc.collect()
    return out


def _assert_equivalent(got, ref, mul, what):
    for k in ("loss", "scores"):
        if k in got:
            assert torch.equal(got[k], ref[k]), f"{what}: {k} differs"
    bad = [i for i, (a, b) in enumerate(zip(got["states"], ref["states"])) if not torch.equal(a, b)]
    assert not bad, f"{what}: states {bad} differ"
    for n, g in got["grads"].items():
        if n == "embed.W":
            assert torch.equal(g, ref["grads"][n] * mul), f"{what}: embed.W is not s_e * dE_off"
            assert (g[mul.view(-1) == 0] == 0).all()
        else:
            assert torch.equal(g, ref["grads"][n]), f"{what}: gradient {n} differs"


@pytest.mark.parametrize("row", ROW_IDS)
def test_equals_masked_embedding_bit_for_bit(row):
    r = Row(row)
    seed = r.torch_seed                      # torch.initial_seed() after _model's manual_seed: the mode's seed
    keep = _lib_mask(seed, STEP, r.V, P_E)
    x0 = r.x[0].to(_dev()).view(-1)
    if x0.numel() >= 20:
        assert keep[x0].any() and not keep[x0].all(), "the window should hold dropped and kept word types"
    mul = _mul(keep, P_E)
    got = _trainer_grads(r, P_E)
    ref = _trainer_grads(r, 0.0, mul=mul)
    _assert_equivalent(got, ref, mul, f"{row} trainer")
    mul0 = _mul(_lib_mask(seed, 0, r.V, P_E), P_E)
    got = _dropin_grads(r, P_E)
    ref = _dropin_grads(r, 0.0, mul=mul0)
    _assert_equivalent(got, ref, mul0, f"{row} drop-in")


@pytest.mark.parametrize("mode", ["variational", "weight_drop"])
def test_composes_with_variational_and_weight_drop(mode):
    """The equivalence above with variational=True (p_rec 0.5) or weight_drop=0.5, on a persistent-plan row, the
    per-timestep row and the validation engine."""
    for row in [r for r in ("odd_h", "steps_b40", "simt_h48") if r in ROW_IDS]:
        r = Row(row)
        kw = dict(variational=True, recurrent_dropout=0.5) if mode == "variational" else dict(weight_drop=0.5)
        mul = _mul(_lib_mask(r.torch_seed, STEP, r.V, P_E), P_E)
        got = _trainer_grads(r, P_E, **kw)
        ref = _trainer_grads(r, 0.0, mul=mul, **kw)
        _assert_equivalent(got, ref, mul, f"{row} {mode}")


# ---- against the fp64 oracle --------------------------------------------------------------------------------------
_oracle_cache = {}


def _oracle_steps(row, tied, lr, modes):
    """two carried fp64 steps from the row's model and states, as numpy: loss, norm, scores, states, raw grads,
    params after and (AR, TAR) per step; modes(s) gives step s's Modes"""
    m = _model(row, tied=tied)
    params = {k: v.detach().cpu().double() for k, v in m.named_parameters()}
    del m
    states = [(h.double(), c.double()) for h, c in row.h0]
    out = []
    for s in range(2):
        md = modes(s)
        with torch.no_grad():
            sc, _, ar = MO.forward(params, row.x[s], states, L, tied, dataclasses.replace(md, beta=0.0))
            tar = MO.forward(params, row.x[s], states, L, tied, dataclasses.replace(md, alpha=0.0))[2]
        loss, norm, grads, params, states, _ = MO.train_step(params, row.x[s], row.y[s], states, L, tied, lr,
                                                             MAX_NORM, md)
        out.append(dict(loss=loss, norm=norm, scores=sc.numpy(), states=[(h.numpy(), c.numpy()) for h, c in states],
                        grads={k: v.numpy() for k, v in grads.items()},
                        params={k: v.numpy() for k, v in params.items()}, reg=(float(ar), float(tar))))
    return out


def _oracle(row, seed, p_e, variational=False, p_wd=0.0, tied=False, alpha=0.0, beta=0.0):
    key = (row.name, seed, p_e, variational, p_wd, tied, alpha, beta)
    if key not in _oracle_cache:
        out = _oracle_steps(row, tied, LR, lambda s: MO.Modes(
            seed=seed, step=s, p=P_DROP, variational=variational, p_rec=P_DROP if variational else 0.0,
            wd_seed=row.torch_seed, p_wd=p_wd, ed_seed=row.torch_seed, p_e=p_e, alpha=alpha, beta=beta))
        _oracle_cache.clear()
        _oracle_cache[key] = out
    return _oracle_cache[key]


def _trainer_run(row, p_e, lazy=False, keep=False, eval_between=False, ar=0.0, tar=0.0, lr=LR, **kw):
    import zaremba_b200
    m = _model(row, p_e, **kw)
    tr = zaremba_b200.Trainer(m, row.B, row.T, lazy_update=lazy, keep_clipped_grads=keep, ar=ar, tar=tar)
    for (h, c), (h0, c0) in zip(tr.states, row.states()):
        h.copy_(h0)
        c.copy_(c0)
    row.check_branch(tr.ctx)
    out = []
    for s in range(2):
        loss, norm = tr.train_step(row.x[s].to(_dev()), row.y[s].to(_dev()), lr, MAX_NORM)
        loss, norm = loss.clone(), norm.clone()   # (eval_step writes the same loss buffer)
        reg = tr.activation_reg.clone()
        if eval_between and s == 0:
            saved = [t.clone() for st in tr.states for t in st]
            m.eval()
            tr.eval_step(row.x[1].to(_dev()), row.y[1].to(_dev()))
            m.train()
            for t, v in zip([t for st in tr.states for t in st], saved):
                t.copy_(v)
        tr.flush()
        torch.cuda.synchronize()
        out.append(dict(loss=loss.clone(), norm=norm.clone(), states=[t.clone() for st in tr.states for t in st],
                        flat_g=tr.flat_g.clone(), flat_p=tr.flat_p.clone(), reg=reg))
    seed = tr.seed
    offs = _offsets(m, tr)
    tr.close()
    del tr, m
    gc.collect()
    return out, seed, offs


def _dropin_run(row, p_e, **kw):
    m = _model(row, p_e, **kw)
    row.check_branch(m._context(row.T, row.B))
    states = row.states()
    out = []
    for s in range(2):
        m.zero_grad(set_to_none=True)
        scores, states = m(row.x[s], states)
        loss = _caller_nll_loss(scores, row.y[s])
        loss.backward()
        grads = {k: p.grad.clone() for k, p in m.named_parameters()}
        torch.nn.utils.clip_grad_norm_(m.parameters(), MAX_NORM)
        with torch.no_grad():
            for p in m.parameters():
                p -= LR * p.grad
        states = m.detach(states)
        out.append(dict(loss=loss.detach().clone(), scores=scores.detach().clone(),
                        states=[t.clone() for st in states for t in st], grads=grads,
                        params={k: p.detach().clone() for k, p in m.named_parameters()}))
    seed = m._seed
    del m
    gc.collect()
    return out, seed


def _check_against_oracle(row, got, ref, tag, offs=None):
    tol = TOL[row.engine]
    for s, (g, r) in enumerate(zip(got, ref)):
        t = f"{tag} step {s}"
        assert abs(g["loss"].item() - r["loss"]) <= tol["loss"] * abs(r["loss"]), (t, g["loss"].item(), r["loss"])
        for l in range(L):
            _scale_close(g["states"][2 * l].reshape(row.B, row.H).cpu().numpy(), r["states"][l][0], tol["fwd"], f"{t} h{l}")
            _scale_close(g["states"][2 * l + 1].reshape(row.B, row.H).cpu().numpy(), r["states"][l][1], tol["fwd"],
                         f"{t} c{l}")
        if "scores" in g:
            _scale_close(g["scores"].cpu().numpy(), r["scores"], tol["fwd"], f"{t} scores")
        if "reg" in g:   # the alpha-weighted AR and beta-weighted TAR of the step, held like the loss
            for i, what in enumerate(("AR", "TAR")):
                got_v, want_v = g["reg"][i].item(), r["reg"][i]
                assert abs(got_v - want_v) <= tol["loss"] * abs(want_v) + 1e-30, (t, what, got_v, want_v)
        if "flat_g" in g:
            grads = {k: g["flat_g"][o:o + n] for k, (o, n) in offs.items()}
            params = {k: g["flat_p"][o:o + n] for k, (o, n) in offs.items()}
        else:
            grads, params = g["grads"], g["params"]
        assert sorted(grads) == sorted(r["grads"]), t
        for k in r["grads"]:
            _scale_close(grads[k].cpu().numpy().reshape(r["grads"][k].shape), r["grads"][k], tol["grad"], f"{t} grad {k}")
            _scale_close(params[k].cpu().numpy().reshape(r["params"][k].shape), r["params"][k], tol["grad"],
                         f"{t} param {k}")


@pytest.mark.parametrize("row", ROW_IDS)
def test_trainer_and_dropin_against_fp64_oracle(row):
    r = Row(row)
    got, seed, offs = _trainer_run(r, P_E)
    ref = _oracle(r, seed, P_E)
    _check_against_oracle(r, got, ref, f"{row} trainer", offs)
    got, seed2 = _dropin_run(r, P_E)
    assert seed2 == seed
    _check_against_oracle(r, got, ref, f"{row} drop-in")


ALL_ON = dict(variational=True, weight_drop=0.5)
AR, TAR = 2.0, 1.0   # AWD-LSTM's values


@pytest.mark.parametrize("tied", [False, True], ids=["untied", "tied"])
@pytest.mark.parametrize("row", [r for r in ("odd_h", "b8_padded", "steps_b40", "simt_h48") if r in ROW_IDS])
def test_everything_on_against_fp64_oracle(row, tied):
    """p_e = 0.1 and AR/TAR (2, 1) with the variational mode (p_rec = p) and weight drop 0.5, untied and tied
    (projection unmasked)."""
    r = Row(row)
    got, seed, offs = _trainer_run(r, 0.1, tied=tied, ar=AR, tar=TAR, **ALL_ON)
    ref = _oracle(r, seed, 0.1, variational=True, p_wd=0.5, tied=tied, alpha=AR, beta=TAR)
    _check_against_oracle(r, got, ref, f"{row} all-on {'tied' if tied else 'untied'} trainer", offs)
    if tied:   # the projection's gradient reaches every row: dropped rows are not zero
        keep = _lib_mask(r.torch_seed, 0, r.V, 0.1)
        o, n = offs["embed.W"]
        g = got[0]["flat_g"][o:o + n].view(r.V, r.H)
        assert (g[~keep] != 0).any()


class _Shape(Row):
    """A recipe's shape (tools/bench_weight_drop.py's CONFIGS: V, H, T, B) with Row's windows of distinct tokens,
    states and masks; the plan is whatever the device picks."""

    def __init__(self, config):
        import sys
        sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
        from bench_weight_drop import CONFIGS
        V, H, _, T, B, _ = CONFIGS[config]
        self.name, self.engine, self.H, self.T, self.B, self.branch = config, "tc", H, T, B, None
        self.V = V
        self.winit = 0.04 if H >= 1000 else 0.1
        self.torch_seed = 2000 + ["small", "medium", "large"].index(config)
        g = torch.Generator().manual_seed(self.torch_seed)
        N = T * B
        self.x = [torch.randperm(V, generator=g)[:N].view(T, B) for _ in range(2)]
        self.y = [torch.randint(0, V, (T, B), generator=g) for _ in range(2)]
        self.h0 = [(torch.rand(B, H, generator=g) - 0.5, torch.rand(B, H, generator=g) * 2 - 1) for _ in range(L)]


@pytest.mark.parametrize("tied", [False, True], ids=["untied", "tied"])
@pytest.mark.parametrize("config", ["small", "medium", "large"])
def test_everything_on_at_recipe_shapes(config, tied):
    """Two carried steps with everything on at the Small, Medium and Large shapes, against the fp64 oracle."""
    if "tc" not in ENGINES:
        pytest.skip("tensor-core engine not selected")
    r = _Shape(config)
    got, seed, offs = _trainer_run(r, 0.1, tied=tied, ar=AR, tar=TAR, **ALL_ON)
    ref = _oracle(r, seed, 0.1, variational=True, p_wd=0.5, tied=tied, alpha=AR, beta=TAR)
    _check_against_oracle(r, got, ref, f"{config} all-on {'tied' if tied else 'untied'}", offs)


# ---- AR / TAR -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("row", ROW_IDS)
def test_activation_reg_leaves_the_nll_and_adds_its_gradient(row):
    """alpha = beta = 0 is the mode off bit for bit.  With alpha = 2, beta = 1 (lr = 0, so both steps see the same
    weights): the returned loss and the carried states are bit-identical to the mode off, R matches the oracle within
    the loss tolerance, and the penalties' gradient contribution g(2, 1) - g(0, 0) matches the oracle's within
    2 * TOL["grad"] of the scale of the whole gradient (the difference inherits the rounding of both gradients)."""
    r = Row(row)
    off, seed, offs = _trainer_run(r, 0.0, lr=0.0)
    zero = _trainer_run(r, 0.0, lr=0.0, ar=0.0, tar=0.0)[0]
    _assert_runs_equal(zero, off, f"{row} alpha=beta=0")
    on = _trainer_run(r, 0.0, lr=0.0, ar=AR, tar=TAR)[0]
    tol = TOL[r.engine]
    for s in range(2):
        assert torch.equal(on[s]["loss"], off[s]["loss"]), f"{row} step {s}: the returned loss is not the NLL"
        assert all(torch.equal(a, b) for a, b in zip(on[s]["states"], off[s]["states"])), f"{row} step {s}: states"
        assert torch.equal(off[s]["reg"], torch.zeros(2, device=_dev()))
    ref_on = _oracle_lr0(r, seed, AR, TAR)
    ref_off = _oracle_lr0(r, seed, 0.0, 0.0)
    for s in range(2):
        for i, what in enumerate(("AR", "TAR")):
            got_v, want_v = on[s]["reg"][i].item(), ref_on[s]["reg"][i]
            assert want_v > 0 or (what == "TAR" and r.T == 1)
            assert abs(got_v - want_v) <= tol["loss"] * abs(want_v) + 1e-30, (row, s, what, got_v, want_v)
        for k, (o, n) in offs.items():
            d = (on[s]["flat_g"][o:o + n] - off[s]["flat_g"][o:o + n]).double().cpu().numpy()
            want = (ref_on[s]["grads"][k] - ref_off[s]["grads"][k]).reshape(-1)
            scale = np.abs(ref_on[s]["grads"][k]).max()
            err = np.abs(d - want).max()
            assert err <= 2 * tol["grad"] * scale, (row, s, k, err, scale, np.abs(want).max())


_oracle_lr0_cache = {}


def _oracle_lr0(row, seed, alpha, beta):
    """Two steps of the fp64 restatement at lr = 0 (the weights stay put; the states carry)."""
    key = (row.name, seed, alpha, beta)
    if key not in _oracle_lr0_cache:
        out = _oracle_steps(row, False, 0.0, lambda s: MO.Modes(seed=seed, step=s, p=P_DROP, alpha=alpha, beta=beta))
        if len(_oracle_lr0_cache) > 2:
            _oracle_lr0_cache.clear()
        _oracle_lr0_cache[key] = out
    return _oracle_lr0_cache[key]


# ---- schedules, eval, p = 0 ---------------------------------------------------------------------------------------
def _assert_runs_equal(a, b, what):
    for s, (u, v) in enumerate(zip(a, b)):
        bad = [k for k in u if not (torch.equal(u[k], v[k]) if torch.is_tensor(u[k])
                                    else all(torch.equal(p, q) for p, q in zip(u[k], v[k])))]
        assert not bad, f"{what} step {s}: {bad} differ"


@pytest.mark.parametrize("keep", [False, True], ids=["raw_grads", "clipped_grads"])
def test_lazy_update_equals_strict(keep):
    """Including the tied lazy gather that applies E's deferred update on the fly."""
    if "tc" not in ENGINES:
        pytest.skip("tensor-core engine not selected")
    for row, kw in (("odd_h", dict(ar=AR, tar=TAR)), ("b8_padded", dict(tied=True, ar=AR, tar=TAR, **ALL_ON))):
        r = Row(row)
        got = _trainer_run(r, P_E, lazy=True, keep=keep, **kw)[0]
        want = _trainer_run(r, P_E, keep=keep, **kw)[0]
        _assert_runs_equal(got, want, f"{row} lazy")


@pytest.mark.parametrize("row", [r for r in ("odd_h", "steps_b40", "simt_h48") if r in ROW_IDS])
def test_train_eval_train_equals_train_train(row):
    r = Row(row)
    got = _trainer_run(r, P_E, eval_between=True)[0]
    want = _trainer_run(r, P_E)[0]
    _assert_runs_equal(got, want, f"{row} train-eval-train")


@pytest.mark.parametrize("row", [r for r in ("odd_h", "steps_b40", "simt_h48") if r in ROW_IDS])
def test_eval_is_untouched(row):
    """After two steps with embedding dropout and AR/TAR: eval_step, perplexity, generate, beam_search and
    dynamic_eval_step equal a mode-off model holding the same weights, bit for bit."""
    import zaremba_b200
    r = Row(row)
    res = []
    weights = None
    for p_e in (P_E, 0.0):
        m = _model(r, p_e)
        if weights is None:
            tr = zaremba_b200.Trainer(m, r.B, r.T, ar=AR, tar=TAR)
            for s in range(2):
                tr.train_step(r.x[s].to(_dev()), r.y[s].to(_dev()), LR, MAX_NORM)
            tr.flush()
            weights = {k: v.detach().clone() for k, v in m.state_dict().items()}
        else:
            m.load_state_dict(weights)
            tr = zaremba_b200.Trainer(m, r.B, r.T)
        m.eval()
        tr.reset_states()
        loss = tr.eval_step(r.x[0].to(_dev()), r.y[0].to(_dev())).clone()
        ppl = tr.perplexity([(r.x[0], r.y[0]), (r.x[1], r.y[1])])
        tok, lp, _ = m.generate(r.x[0][:, :1], 3, temperature=1.0, seed=9)
        bt, blp, bsc, _ = m.beam_search(r.x[0][:, :1], 3, 3)
        theta = tr.flat_p.clone()
        tr.reset_states()
        dl = tr.dynamic_eval_step(r.x[1].to(_dev()), r.y[1].to(_dev()), theta, 0.1, 0.01).clone()
        torch.cuda.synchronize()
        res.append([loss, torch.tensor(ppl), tok, lp, bt, blp, bsc, dl, tr.flat_p.clone(), tr.flat_g.clone()])
        tr.close()
        del tr, m
        gc.collect()
    for i, (a, b) in enumerate(zip(*res)):
        assert torch.equal(a, b), f"output {i} differs"


@pytest.mark.parametrize("row", [r for r in ("odd_h", "simt_h48") if r in ROW_IDS])
def test_p0_equals_mode_off(row):
    from zaremba_b200 import _lib
    r = Row(row)
    want = _trainer_run(r, 0.0)[0]
    import zaremba_b200
    m = _model(r)
    tr = zaremba_b200.Trainer(m, r.B, r.T)
    _lib.check(_lib.load().zrb_set_embed_dropout(tr.ctx, 0.0, 12345))
    for (h, c), (h0, c0) in zip(tr.states, r.states()):
        h.copy_(h0)
        c.copy_(c0)
    got = []
    for s in range(2):
        loss, norm = tr.train_step(r.x[s].to(_dev()), r.y[s].to(_dev()), LR, MAX_NORM)
        torch.cuda.synchronize()
        got.append(dict(loss=loss.clone(), norm=norm.clone(), states=[t.clone() for st in tr.states for t in st],
                        flat_g=tr.flat_g.clone(), flat_p=tr.flat_p.clone()))
    tr.close()
    _assert_runs_equal(got, want, f"{row} p=0")


def test_rejected_arguments_and_call_order():
    import zaremba_b200
    from zaremba_b200 import _lib
    lib = _lib.load()
    E_INVALID, E_STATE = -1, -3
    r = Row("tc_h48" if "tc" in ENGINES else "simt_h48")
    m = _model(r)
    tr = zaremba_b200.Trainer(m, r.B, r.T)
    ctx = tr.ctx
    for p in (-0.1, 1.0, 1.5, float("nan"), float("inf"), -float("inf")):
        assert lib.zrb_set_embed_dropout(ctx, p, 1) == E_INVALID, p
    assert lib.zrb_set_embed_dropout(None, 0.1, 1) == E_INVALID
    for a, b in ((-1.0, 0.0), (0.0, -1.0), (float("nan"), 1.0), (1.0, float("inf"))):
        assert lib.zrb_set_activation_reg(ctx, a, b) == E_INVALID, (a, b)
    assert lib.zrb_set_activation_reg(None, 1.0, 1.0) == E_INVALID
    assert lib.zrb_activation_reg(ctx, None, None) == E_INVALID
    x, y = r.x[0].to(_dev()), r.y[0].to(_dev())
    stream = tr._stream()
    scores = torch.empty(r.T * r.B, r.V, device=_dev())
    _lib.check(lib.zrb_forward(ctx, C.byref(tr._ps), _lib.ptr(x), r.T, r.B, C.byref(tr._st), C.byref(tr._st),
                               _lib.ptr(scores), 1, tr.seed, 0, stream))
    _lib.check(lib.zrb_set_embed_dropout(ctx, 0.1, 7))
    assert lib.zrb_backward(ctx, C.byref(tr._ps), _lib.ptr(scores), C.byref(tr._gs), stream) == E_STATE
    _lib.check(lib.zrb_train_step_begin(ctx, C.byref(tr._ps), C.byref(tr._gs), _lib.ptr(x), _lib.ptr(y), r.T, r.B,
                                        C.byref(tr._st), C.byref(tr._st), tr.seed, 1, _lib.ptr(tr.loss), stream))
    _lib.check(lib.zrb_set_embed_dropout(ctx, 0.1, 8))          # another seed is another mode
    assert lib.zrb_train_step_layer(ctx, C.byref(tr._ps), C.byref(tr._gs), L - 1, stream) == E_STATE
    _lib.check(lib.zrb_train_step_begin(ctx, C.byref(tr._ps), C.byref(tr._gs), _lib.ptr(x), _lib.ptr(y), r.T, r.B,
                                        C.byref(tr._st), C.byref(tr._st), tr.seed, 2, _lib.ptr(tr.loss), stream))
    _lib.check(lib.zrb_set_embed_dropout(ctx, 0.1, 8))          # the same mode again keeps the saved forward
    for l in range(L - 1, -1, -1):
        _lib.check(lib.zrb_train_step_layer(ctx, C.byref(tr._ps), C.byref(tr._gs), l, stream))
    torch.cuda.synchronize()
    tr.close()


# ---- two GPUs -----------------------------------------------------------------------------------------------------
def _dp_worker(rank, world, port, q, transport):
    import torch.distributed as dist
    import zaremba_b200
    from zaremba_b200 import _lib
    from tests.test_gpu_multi import B, H, STEPS, T, V
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank), ZRB_DP_TRANSPORT=transport)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    lib = _lib.load()
    g = torch.Generator().manual_seed(3)
    data = torch.randint(0, V, (B * world, STEPS * T + 1), generator=g)
    torch.manual_seed(7)
    m = zaremba_b200.Model(V, H, L, P_DROP, 0.1, embed_dropout=P_E).to(dev)
    m.train()
    tr = zaremba_b200.Trainer(m, B, T)
    assert tr.transport == transport
    rows = slice(rank * B, (rank + 1) * B)
    seeds = []
    for i in range(STEPS):
        x = data[rows, i * T:(i + 1) * T].t().contiguous().to(dev)
        y = data[rows, i * T + 1:(i + 1) * T + 1].t().contiguous().to(dev)
        seeds.append((tr.seed, tr.step))
        tr.train_step(x, y, 1.0, 0.25)
    tr.flush()
    dp_p = tr.flat_p.clone()
    bits = dp_p.view(torch.int32).to(torch.int64)
    chk = torch.stack([bits.sum(), (bits * (torch.arange(bits.numel(), device=dev) % 8191 + 1)).sum()])
    hi, lo = chk.clone(), chk.clone()
    dist.all_reduce(hi, op=dist.ReduceOp.MAX); dist.all_reduce(lo, op=dist.ReduceOp.MIN)
    res = {"identical": bool((hi == lo).all().item())}
    n = T * B * H
    masks = torch.empty(STEPS, L + 1, n, dtype=torch.uint8, device=dev)
    for i, (seed, step) in enumerate(seeds):
        for site in range(L + 1):
            _lib.check(lib.zrb_dropout_mask(seed, step, site, n, P_DROP, _lib.ptr(masks[i, site]), None))
    allm = [torch.empty_like(masks) for _ in range(world)]
    dist.all_gather(allm, masks)
    if rank == 0:
        torch.manual_seed(7)
        m2 = zaremba_b200.Model(V, H, L, P_DROP, 0.1, embed_dropout=P_E).to(dev)
        m2.train()
        tr2 = zaremba_b200.Trainer(m2, B * world, T, data_parallel=False)
        for i in range(STEPS):
            x = data[:, i * T:(i + 1) * T].t().contiguous().to(dev)
            y = data[:, i * T + 1:(i + 1) * T + 1].t().contiguous().to(dev)
            full = [torch.cat([allm[r][i, site].view(T, B, H) for r in range(world)], dim=1).contiguous()
                    for site in range(L + 1)]
            m2.set_explicit_dropout_masks(full)
            tr2.train_step(x, y, 1.0, 0.25)
        tr2.flush()
        res["err"] = (dp_p - tr2.flat_p).abs().max().item() / tr2.flat_p.abs().max().item()
        tr2.close()
    dist.barrier()
    tr.close()
    dist.destroy_process_group()
    q.put((rank, res))


@pytest.mark.parametrize("transport", ["ce", "nccl"])
def test_dp_step_equals_single_process(transport):
    """World 2 against one process at 2B replaying the ranks' activation masks: the embedding mask is common to the
    ranks (no rank in its seed), so both train the same weights."""
    from tests.test_gpu_multi import _need_two, _spawn
    _need_two()
    out = _spawn(_dp_worker, 2, transport)
    assert out[0]["identical"] and out[1]["identical"], "replicas diverged across ranks"
    assert out[0]["err"] < 2e-3, out[0]
