"""The variational dropout mode without a GPU: the fp64 restatement (tests/_model_oracle.py) against an independent
float64 torch-autograd restatement, its agreement with the oracle when there is no recurrent mask, and the new C entry
point in the header and the ctypes binding."""
import os
import re

import numpy as np
import torch

from oracle import lstm_lm_oracle as O
from oracle import philox as PH
from tests import _model_oracle as MO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V, H, L, T, B = 23, 8, 2, 5, 3
P, P_REC = 0.4, 0.3


def _setup(seed=7):
    rng = np.random.default_rng(seed)
    params = O.init_params(V, H, L, 0.3, seed, dtype=np.float64)
    x = rng.integers(0, V, size=(T, B))
    y = rng.integers(0, V, size=(T, B))
    states = [(rng.uniform(-0.5, 0.5, (B, H)), rng.uniform(-1, 1, (B, H))) for _ in range(L)]   # non-zero entering
    mk = _masks(P_REC)
    return params, x, y, states, mk.sites, mk.rec


def _masks(p_rec):
    return MO.mode_masks(MO.Modes(seed=12345, step=3, p=P, variational=True, p_rec=p_rec), [H] * (L + 1), T, B, V)


def _oracle(params, x, y, states, masks, rmasks, p_rec):
    """_model_oracle's loss, scores, states and raw gradients (autograd) as numpy"""
    ps = {k: torch.tensor(v, requires_grad=True) for k, v in params.items()}
    sc, st, _ = MO.forward(ps, torch.tensor(x), [(torch.tensor(h), torch.tensor(c)) for h, c in states], L, False,
                           MO.Modes(p=P, variational=True, p_rec=p_rec), MO.Masks(sites=masks, rec=rmasks))
    loss = MO.loss_of(sc, torch.tensor(y))
    loss.backward()
    return (loss.item(), sc.detach().numpy(), [(h.detach().numpy(), c.detach().numpy()) for h, c in st],
            {k: v.grad.numpy() for k, v in ps.items()})


def _torch_restatement(params, x, y, states, masks, rmasks):
    """model.py:103-110 as an explicit per-step loop in float64 torch with both kinds of mask; autograd for the
    gradients.  Returns (loss, scores, states, grads)."""
    tp = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in params.items()}
    s, sr = 1.0 / (1.0 - P), 1.0 / (1.0 - P_REC)
    m = [torch.tensor(mk, dtype=torch.float64) * s for mk in masks]
    rm = [torch.tensor(mk, dtype=torch.float64) * sr for mk in rmasks]
    a = tp["embed.W"][torch.tensor(x)] * m[0]
    out_states = []
    for l in range(L):
        h, c = (torch.tensor(v, dtype=torch.float64) for v in states[l])
        Wi, Wh = tp[f"rnns.{l}.weight_ih_l0"], tp[f"rnns.{l}.weight_hh_l0"]
        bi, bh = tp[f"rnns.{l}.bias_ih_l0"], tp[f"rnns.{l}.bias_hh_l0"]
        ys = []
        for t in range(T):
            z = a[t] @ Wi.T + bi + (h * rm[l]) @ Wh.T + bh        # the recurrent operand is masked, h itself is not
            i, f, g, o = z.chunk(4, dim=1)
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
            h = torch.sigmoid(o) * torch.tanh(c)
            ys.append(h)
        out_states.append((h.detach().numpy(), c.detach().numpy()))
        a = torch.stack(ys) * m[l + 1]
    scores = a.reshape(-1, H) @ tp["fc.W"].T + tp["fc.b"]
    logp = torch.log_softmax(scores, dim=1)
    loss = -logp[torch.arange(T * B), torch.tensor(y).reshape(-1)].mean() * B
    loss.backward()
    return loss.item(), scores.detach().numpy(), out_states, {k: v.grad.numpy() for k, v in tp.items()}


def test_variational_oracle_matches_torch_autograd():
    params, x, y, states, masks, rmasks = _setup()
    assert rmasks is not None and not all(m.all() for m in rmasks)
    loss, sc, st, grads = _oracle(params, x, y, states, masks, rmasks, P_REC)
    t_loss, t_sc, t_st, t_grads = _torch_restatement(params, x, y, states, masks, rmasks)
    np.testing.assert_allclose(loss, t_loss, rtol=1e-12)
    np.testing.assert_allclose(sc, t_sc, rtol=1e-11, atol=1e-12)
    for l in range(L):
        np.testing.assert_allclose(st[l][0], t_st[l][0], rtol=1e-11, atol=1e-12)
        np.testing.assert_allclose(st[l][1], t_st[l][1], rtol=1e-11, atol=1e-12)
    assert sorted(grads) == sorted(t_grads) and len(grads) == 3 + 4 * L
    for k in grads:
        np.testing.assert_allclose(grads[k], t_grads[k], rtol=1e-9, atol=1e-12, err_msg=k)


def test_recurrent_masks_change_the_result():
    """The recurrent masks are not a no-op (guards the torch comparison above against a restatement that ignores them)."""
    params, x, y, states, masks, rmasks = _setup()
    a = _oracle(params, x, y, states, masks, rmasks, P_REC)[1]
    b = _oracle(params, x, y, states, masks, None, 0.0)[1]
    assert np.abs(a - b).max() > 1e-3


def test_without_recurrent_masks_equals_the_oracle_with_tiled_masks():
    params, x, y, states, masks, _ = _setup()
    """p_rec = 0: the numpy oracle given the tiled masks, to 1e-12 relative (two separate implementations)"""
    params, x, y, states, masks, _ = _setup()
    mk = _masks(0.0)
    masks0 = mk.sites
    assert mk.rec is None
    for s in range(L + 1):   # the step-0 slice of the site's per-step mask, reused for every t
        want = PH.keep_mask(12345, 3, s, T * B * H, P).reshape(T, B, H)[0]
        assert all(np.array_equal(masks0[s][t], want) for t in range(T))
    loss, sc, st, _ = _oracle(params, x, y, states, masks0, None, 0.0)
    tp = {k: torch.tensor(v) for k, v in params.items()}
    _, norm, grads, after, _, _ = MO.train_step(tp, torch.tensor(x), torch.tensor(y),
                                                [(torch.tensor(h), torch.tensor(c)) for h, c in states], L, False, 1.0,
                                                0.25, MO.Modes(p=P, variational=True), MO.Masks(sites=masks0))
    p2 = {k: v.copy() for k, v in params.items()}
    want = O.train_step(p2, x, y, states, L, 1.0, 0.25, P, masks0)
    np.testing.assert_allclose(loss, want[0], rtol=1e-12)
    np.testing.assert_allclose(norm, want[1], rtol=1e-12)
    np.testing.assert_allclose(sc, want[3], rtol=1e-12)
    for (h, c), (h2, c2) in zip(st, want[2]):
        np.testing.assert_allclose(h, h2, rtol=1e-12)
        np.testing.assert_allclose(c, c2, rtol=1e-12)
    coef = min(1.0, 0.25 / (norm + 1e-6))
    for k in p2:
        np.testing.assert_allclose(grads[k].numpy() * coef, want[4][k], rtol=1e-12, err_msg=k)
        np.testing.assert_allclose(after[k].numpy(), p2[k], rtol=1e-12, err_msg=k)


def test_entry_point_declared_and_bound():
    from zaremba_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "zaremba_b200.h")).read()
    assert re.search(r"int\s+zrb_set_variational_dropout\(zrb_ctx\* ctx, int32_t on, float p_rec\);", hdr)
    import ctypes as C
    res, args = _lib._SIGNATURES["zrb_set_variational_dropout"]
    assert res is C.c_int and args == [C.c_void_p, C.c_int32, C.c_float]
    assert "zrb_set_variational_dropout" in _lib.exported_symbols()


def test_model_rejects_recurrent_dropout_without_the_mode():
    import pytest
    import zaremba_b200
    with pytest.raises(ValueError):
        zaremba_b200.Model(V, H, L, P, 0.1, recurrent_dropout=0.3)
    with pytest.raises(ValueError):
        zaremba_b200.Model(V, H, L, P, 0.1, variational=True, recurrent_dropout=1.0)
    m = zaremba_b200.Model(V, H, L, P, 0.1, variational=True)
    assert m.p_rec == P                           # None: Gal's setting, the same p as dropout
    assert zaremba_b200.Model(V, H, L, P, 0.1, variational=True, recurrent_dropout=0.0).p_rec == 0.0
    with pytest.raises(ValueError):
        m.set_explicit_dropout_masks([torch.ones(T, B, H, dtype=torch.uint8)] * (L + 1))
