"""GPU tests of the variational dropout mode (DESIGN.md section 11) at every kernel and recurrence-plan branch that
applies a mask: the rows of tests/test_gpu_dropout.py (every plan branch, the per-timestep path at B = 40, both
embedding paths, the validation engine).

  * two carried train steps through the fused Trainer and the drop-in Model against the fp64 restatement of
    tests/_model_oracle.py, with masks computed by oracle/philox.py, never by the library;
  * with p_rec = 0 the mode is bit for bit Zaremba's path fed the step-0 masks tiled over the window (the
    fixed-over-window indexing of every kernel and branch, the rows-out embedding gradient included);
  * a lazy-update Trainer equals a strict one bit for bit; inference is untouched by the mode;
  * the rejected arguments and call orders.
Windows hold distinct tokens, so the embedding scatter is deterministic.
"""
import ctypes as C
import gc
import math

import numpy as np
import pytest
import torch

from oracle import lstm_lm_oracle as O
from tests import _model_oracle as MO
from tests.test_gpu_dropout import L, P_DROP, ROW_IDS, Row
from tests.test_gpu_parity import ENGINES, TOL, _caller_nll_loss, _scale_close

pytestmark = pytest.mark.gpu

LR, MAX_NORM = 1.0, 0.25


def _dev():
    return torch.device("cuda:0")


def _winit(row):
    """The README recipes' init scale, winit * sqrt(H) <= 1.3 (Medium: 0.05 at H = 650).  The dropout rows' 0.1 at
    H = 650 puts the recurrence at p_rec = 0.65 in a chaotic regime: measured on an H100, the tensor-core engine's fp16
    operand rounding grew to 7e-3 (step 0) and 2e-2 (step 1) of the states' scale there, while the fp32 engine agrees
    with the fp64 oracle to 5e-7 at every row."""
    return min(row.winit, 1.3 / math.sqrt(row.H))


def _model(row, variational=True, p_rec=None):
    import zaremba_b200
    torch.manual_seed(row.torch_seed)
    kw = dict(variational=True, recurrent_dropout=p_rec) if variational else {}
    m = zaremba_b200.Model(row.V, row.H, L, P_DROP, _winit(row), engine=row.engine, **kw).to(_dev())
    m.train()
    return m


_oracle_cache = {}


def _tiled_masks(seed, step, T, B, H):
    """the variational mode's site masks: the step-0 mask of every site tiled over the window"""
    return MO.mode_masks(MO.Modes(seed=seed, step=step, p=P_DROP, variational=True), [H] * (L + 1), T, B, 0).sites


def _oracle(row, seed, p_rec):
    """fp64 oracle of two carried steps: per step loss, norm, states, unclipped grads, updated params (numpy)."""
    key = (row.name, seed, p_rec)
    if key not in _oracle_cache:
        m = _model(row, False)
        params = {k: v.detach().cpu().double() for k, v in m.named_parameters()}
        del m
        states = [(h.double(), c.double()) for h, c in row.h0]
        out = []
        for s in range(2):
            md = MO.Modes(seed=seed, step=s, p=P_DROP, variational=True, p_rec=p_rec)
            with torch.no_grad():
                sc = MO.forward(params, row.x[s], states, L, False, md)[0]
            loss, norm, grads, params, states, _ = MO.train_step(params, row.x[s], row.y[s], states, L, False, LR,
                                                                 MAX_NORM, md)
            out.append(dict(loss=loss, norm=norm, scores=sc.numpy(), states=[(h.numpy(), c.numpy()) for h, c in states],
                            grads={k: v.numpy() for k, v in grads.items()},
                            params={k: v.numpy() for k, v in params.items()}))
        _oracle_cache.clear()
        _oracle_cache[key] = out
    return _oracle_cache[key]


def _sizes(row):
    return [int(np.prod(O.param_shapes(row.V, row.H, L)[k])) for k in O.param_names(L)]


def _trainer_run(row, variational=True, p_rec=None, explicit=False, lazy=False):
    import zaremba_b200
    m = _model(row, variational, p_rec)
    tr = zaremba_b200.Trainer(m, row.B, row.T, lazy_update=lazy)
    for (h, c), (h0, c0) in zip(tr.states, row.states()):
        h.copy_(h0)
        c.copy_(c0)
    row.check_branch(tr.ctx)
    out = []
    for s in range(2):
        if explicit:
            masks = _tiled_masks(tr.seed, s, row.T, row.B, row.H)
            m.set_explicit_dropout_masks([torch.tensor(mk).to(_dev()) for mk in masks])
        loss, norm = tr.train_step(row.x[s].to(_dev()), row.y[s].to(_dev()), LR, MAX_NORM)
        tr.flush()
        torch.cuda.synchronize()
        out.append(dict(loss=loss.clone(), norm=norm.clone(), states=[t.clone() for st in tr.states for t in st],
                        flat_g=tr.flat_g.clone(), flat_p=tr.flat_p.clone()))
    seed = tr.seed
    tr.close()
    del tr, m
    gc.collect()
    return out, seed


def _dropin_run(row, variational=True, p_rec=None, explicit=False):
    """Drop-in Model: forward, caller's loss, backward, caller's clip + SGD; states carried into step 1."""
    m = _model(row, variational, p_rec)
    row.check_branch(m._context(row.T, row.B))
    seed = int(torch.initial_seed()) & 0xFFFFFFFFFFFFFFFF
    states = row.states()
    out = []
    for s in range(2):
        if explicit:
            masks = _tiled_masks(seed, s, row.T, row.B, row.H)
            m.set_explicit_dropout_masks([torch.tensor(mk).to(_dev()) for mk in masks])
        m.zero_grad(set_to_none=True)
        scores, states = m(row.x[s], states)
        loss = _caller_nll_loss(scores, row.y[s])
        loss.backward()
        grads = {k: p.grad.clone() for k, p in m.named_parameters()}
        norm = torch.nn.utils.clip_grad_norm_(m.parameters(), MAX_NORM)
        with torch.no_grad():
            for p in m.parameters():
                p -= LR * p.grad
        states = m.detach(states)
        out.append(dict(loss=loss.detach().clone(), norm=norm.detach().clone(), scores=scores.detach().clone(),
                        states=[t.clone() for st in states for t in st], grads=grads,
                        params={k: p.detach().clone() for k, p in m.named_parameters()}))
    assert m._seed == seed and m._drop_step == 2
    del m
    gc.collect()
    return out, seed


def _check_against_oracle(row, got, ref, tag):
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
        if "flat_g" in g:
            grads = dict(zip(O.param_names(L), g["flat_g"].split(_sizes(row))))
            params = dict(zip(O.param_names(L), g["flat_p"].split(_sizes(row))))
        else:
            grads, params = g["grads"], g["params"]
        for k in O.param_names(L):
            _scale_close(grads[k].cpu().numpy().reshape(r["grads"][k].shape), r["grads"][k], tol["grad"], f"{t} grad {k}")
            _scale_close(params[k].cpu().numpy().reshape(r["params"][k].shape), r["params"][k], tol["grad"],
                         f"{t} param {k}")


@pytest.mark.parametrize("p_rec", [0.65, 0.3])
@pytest.mark.parametrize("row", ROW_IDS)
def test_trainer_and_dropin_against_fp64_oracle(row, p_rec):
    """Two carried steps, fused Trainer and drop-in Model (forward, backward, the caller's clip + SGD), against the fp64
    oracle fed oracle/philox.py's masks of the mode: scores, states, loss, gradients and updated parameters."""
    r = Row(row)
    got, seed = _trainer_run(r, p_rec=p_rec)
    ref = _oracle(r, seed, p_rec)
    _check_against_oracle(r, got, ref, f"{row} trainer")
    got, seed2 = _dropin_run(r, p_rec=p_rec)
    assert seed2 == seed
    _check_against_oracle(r, got, ref, f"{row} drop-in")


def _assert_bits_equal(a, b, what):
    for s, (u, v) in enumerate(zip(a, b)):
        for k in u:
            x, y = u[k], v[k]
            if isinstance(x, dict):
                bad = [n for n in x if not torch.equal(x[n], y[n])]
            elif isinstance(x, list):
                bad = [i for i, (p, q) in enumerate(zip(x, y)) if not torch.equal(p, q)]
            else:
                bad = [] if torch.equal(x, y) else [k]
            assert not bad, f"{what} step {s}: {k} differs ({bad})"


@pytest.mark.parametrize("row", ROW_IDS)
def test_without_recurrent_dropout_equals_tiled_explicit_masks(row):
    """variational=True, recurrent_dropout=0 against Zaremba's path fed the step-0 masks tiled over T through
    set_explicit_dropout_masks: fused Trainer and drop-in Model, two steps, bit for bit."""
    r = Row(row)
    got, _ = _trainer_run(r, p_rec=0.0)
    want, _ = _trainer_run(r, variational=False, explicit=True)
    _assert_bits_equal(got, want, f"{row} trainer")
    got, _ = _dropin_run(r, p_rec=0.0)
    want, _ = _dropin_run(r, variational=False, explicit=True)
    _assert_bits_equal(got, want, f"{row} drop-in")


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("H", [48, 257])
def test_embed_rows_out_fixed_over_window(H, engine):
    """zrb_set_embed_rows_out in the variational mode (p_rec = 0) equals Zaremba's path fed the tiled masks, bit for
    bit, and its zeros are exactly the dropped elements of the site-0 mask of step 0, repeated at every t."""
    import zaremba_b200
    from zaremba_b200 import _lib
    lib = _lib.load()
    V, T, B = 400, 5, 9
    g = torch.Generator().manual_seed(5)
    x = torch.randperm(V, generator=g)[:T * B].view(T, B).to(_dev())
    y = torch.randint(0, V, (T, B), generator=g).to(_dev())
    out = []
    for variational in (True, False):
        torch.manual_seed(41 + H)
        kw = dict(variational=True, recurrent_dropout=0.0) if variational else {}
        m = zaremba_b200.Model(V, H, L, P_DROP, 0.1, engine=engine, **kw).to(_dev())
        m.train()
        tr = zaremba_b200.Trainer(m, B, T)
        if not variational:
            masks = _tiled_masks(tr.seed, tr.step, T, B, H)
            m.set_explicit_dropout_masks([torch.tensor(mk).to(_dev()) for mk in masks])
        rows = torch.full((T * B, H), float("nan"), device=_dev())
        _lib.check(lib.zrb_set_embed_rows_out(tr.ctx, _lib.ptr(rows)))
        try:
            _lib.check(lib.zrb_train_step_grads(tr.ctx, C.byref(tr._ps), C.byref(tr._gs), _lib.ptr(x), _lib.ptr(y), T, B,
                                                C.byref(tr._st), C.byref(tr._st), tr.seed, tr.step, _lib.ptr(tr.loss),
                                                tr._stream()))
            torch.cuda.synchronize()
        finally:
            _lib.check(lib.zrb_set_embed_rows_out(tr.ctx, None))
        out.append(rows.clone())
        keep = _tiled_masks(tr.seed, tr.step, T, B, H)[0].reshape(T * B, H)
        tr.close()
        del tr, m
        gc.collect()
    assert torch.equal(out[0], out[1])
    rw = out[0].cpu().numpy()
    assert np.isfinite(rw).all() and (rw[~keep] == 0).all() and (rw[keep] != 0).all()


def test_lazy_update_equals_strict():
    """A lazy-update Trainer with the mode on equals a strict one, bit for bit, over two steps."""
    if "tc" not in ENGINES:
        pytest.skip("tensor-core engine not selected")
    r = Row("odd_h")
    got, _ = _trainer_run(r, p_rec=0.65, lazy=True)
    want, _ = _trainer_run(r, p_rec=0.65)
    _assert_bits_equal(got, want, "lazy")


@pytest.mark.parametrize("row", [r for r in ("odd_h", "steps_b40", "simt_h48") if r in ROW_IDS])
def test_inference_is_untouched(row):
    """eval forward / perplexity, generate and beam_search of a model in the mode equal the same weights without it."""
    r = Row(row)
    res = []
    for variational in (True, False):
        m = _model(r, variational, 0.5 if variational else None)
        m.eval()
        with torch.no_grad():
            sc, st = m(r.x[0], r.states())
        tok, lp, _ = m.generate(r.x[0][:, :4], 3, temperature=1.0, seed=9)
        bt, blp, bsc, _ = m.beam_search(r.x[0][:, :1], 3, 3)   # (1 prompt x 3 beams fits every row's max_batch)
        import zaremba_b200
        tr = zaremba_b200.Trainer(m, r.B, r.T)
        ppl = tr.perplexity([(r.x[0], r.y[0]), (r.x[1], r.y[1])])
        res.append([sc, *[t for s in st for t in s], tok, lp, bt, blp, bsc, torch.tensor(float(ppl))])
        tr.close()
        del tr, m
        gc.collect()
    for i, (a, b) in enumerate(zip(*res)):
        assert torch.equal(a, b), f"output {i} differs"


def test_rejected_arguments_and_call_order():
    import zaremba_b200
    from zaremba_b200 import _lib
    lib = _lib.load()
    E_INVALID, E_STATE = -1, -3
    with pytest.raises(ValueError):
        zaremba_b200.Model(50, 16, L, 0.5, 0.1, recurrent_dropout=0.2)
    with pytest.raises(ValueError):
        zaremba_b200.Model(50, 16, L, 0.5, 0.1, variational=True, recurrent_dropout=-0.1)
    r = Row("tc_h48" if "tc" in ENGINES else "simt_h48")
    m = _model(r, False)
    tr = zaremba_b200.Trainer(m, r.B, r.T)
    ctx = tr.ctx
    for on, p in ((2, 0.0), (-1, 0.0), (1, -0.1), (1, 1.0), (1, 1.5), (0, 0.3)):
        assert lib.zrb_set_variational_dropout(ctx, on, p) == E_INVALID, (on, p)
    keep = torch.ones(r.T * r.B * r.H, dtype=torch.uint8, device=_dev())
    mk = (C.c_void_p * (L + 1))(*[keep.data_ptr()] * (L + 1))
    _lib.check(lib.zrb_set_explicit_masks(ctx, mk))
    assert lib.zrb_set_variational_dropout(ctx, 1, 0.3) == E_STATE
    _lib.check(lib.zrb_set_explicit_masks(ctx, None))
    _lib.check(lib.zrb_set_variational_dropout(ctx, 1, 0.3))
    assert lib.zrb_set_explicit_masks(ctx, mk) == E_STATE
    _lib.check(lib.zrb_set_explicit_masks(ctx, None))          # NULL is always accepted
    x, y = r.x[0].to(_dev()), r.y[0].to(_dev())
    stream = tr._stream()
    # a mode change between forward and backward: zrb_backward refuses
    scores = torch.empty(r.T * r.B, r.V, device=_dev())
    _lib.check(lib.zrb_forward(ctx, C.byref(tr._ps), _lib.ptr(x), r.T, r.B, C.byref(tr._st), C.byref(tr._st),
                               _lib.ptr(scores), 1, tr.seed, 0, stream))
    _lib.check(lib.zrb_set_variational_dropout(ctx, 1, 0.2))
    assert lib.zrb_backward(ctx, C.byref(tr._ps), _lib.ptr(scores), C.byref(tr._gs), stream) == E_STATE
    # ... and between the phases of a train step: zrb_train_step_layer refuses
    _lib.check(lib.zrb_train_step_begin(ctx, C.byref(tr._ps), C.byref(tr._gs), _lib.ptr(x), _lib.ptr(y), r.T, r.B,
                                        C.byref(tr._st), C.byref(tr._st), tr.seed, 1, _lib.ptr(tr.loss), stream))
    _lib.check(lib.zrb_set_variational_dropout(ctx, 0, 0.0))
    assert lib.zrb_train_step_layer(ctx, C.byref(tr._ps), C.byref(tr._gs), L - 1, stream) == E_STATE
    # setting the same mode again keeps the saved forward
    _lib.check(lib.zrb_train_step_begin(ctx, C.byref(tr._ps), C.byref(tr._gs), _lib.ptr(x), _lib.ptr(y), r.T, r.B,
                                        C.byref(tr._st), C.byref(tr._st), tr.seed, 2, _lib.ptr(tr.loss), stream))
    _lib.check(lib.zrb_set_variational_dropout(ctx, 0, 0.0))
    for l in range(L - 1, -1, -1):
        _lib.check(lib.zrb_train_step_layer(ctx, C.byref(tr._ps), C.byref(tr._gs), l, stream))
    torch.cuda.synchronize()
    mv = _model(r, True, 0.3)
    with pytest.raises(ValueError):
        mv.set_explicit_dropout_masks([keep.view(r.T, r.B, r.H)] * (L + 1))
    tr.close()
