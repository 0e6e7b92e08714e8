"""The variational dropout mode without a GPU: its numpy restatement (tests/_variational_oracle.py) against an
independent float64 torch-autograd restatement, its reduction to the oracle when there is no recurrent mask, and the
new C entry point in the header and the ctypes binding."""
import os
import re

import numpy as np
import torch

from oracle import lstm_lm_oracle as O
from oracle import philox as PH
from tests import _variational_oracle as VO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V, H, L, T, B = 23, 8, 2, 5, 3
P, P_REC = 0.4, 0.3


def _setup(seed=7):
    rng = np.random.default_rng(seed)
    params = O.init_params(V, H, L, 0.3, seed, dtype=np.float64)
    x = rng.integers(0, V, size=(T, B))
    y = rng.integers(0, V, size=(T, B))
    states = [(rng.uniform(-0.5, 0.5, (B, H)), rng.uniform(-1, 1, (B, H))) for _ in range(L)]   # non-zero entering
    masks, rmasks = VO.variational_masks(12345, 3, L, T, B, H, P, P_REC)
    return params, x, y, states, masks, rmasks


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
    sc, st, cache = VO.model_fwd(params, x, states, L, P, masks, rmasks, P_REC)
    grads = VO.model_bwd(params, cache, O.nll_loss_bwd(sc, y), L)
    loss = O.nll_loss(sc, y)
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
    a, _, _ = VO.model_fwd(params, x, states, L, P, masks, rmasks, P_REC)
    b, _, _ = VO.model_fwd(params, x, states, L, P, masks, None, 0.0)
    assert np.abs(a - b).max() > 1e-3


def test_without_recurrent_masks_equals_the_oracle_with_tiled_masks():
    params, x, y, states, masks, _ = _setup()
    masks0, rm0 = VO.variational_masks(12345, 3, L, T, B, H, P, 0.0)
    assert rm0 is None
    for s in range(L + 1):   # the step-0 slice of the site's per-step mask, reused for every t
        want = PH.keep_mask(12345, 3, s, T * B * H, P).reshape(T, B, H)[0]
        assert all(np.array_equal(masks0[s][t], want) for t in range(T))
    p1 = {k: v.copy() for k, v in params.items()}
    p2 = {k: v.copy() for k, v in params.items()}
    got = VO.train_step(p1, x, y, states, L, 1.0, 0.25, P, masks0, None, 0.0)
    want = O.train_step(p2, x, y, states, L, 1.0, 0.25, P, masks0)
    assert got[0] == want[0] and got[1] == want[1]
    np.testing.assert_array_equal(got[3], want[3])
    for (h, c), (h2, c2) in zip(got[2], want[2]):
        np.testing.assert_array_equal(h, h2)
        np.testing.assert_array_equal(c, c2)
    for k in p1:
        np.testing.assert_array_equal(got[4][k], want[4][k])
        np.testing.assert_array_equal(p1[k], p2[k])


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
