"""The weight-dropped LSTM without a GPU: the fp64 restatement (tests/_model_oracle.py) against an independent
float64 torch-autograd restatement with a masked W_hh, with Zaremba's dropout and with the variational mode; the masks'
definition; the new C entry point in the header and the ctypes binding; Model(weight_drop=) argument checks."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from oracle import lstm_lm_oracle as O
from oracle import philox as PH
from tests import _model_oracle as MO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V, H, L, T, B = 23, 8, 2, 5, 3
P, P_REC, P_WD = 0.4, 0.3, 0.5
WD_SEED, STEP = 987654321, 3


def _setup(variational, seed=7):
    rng = np.random.default_rng(seed)
    params = O.init_params(V, H, L, 0.3, seed, dtype=np.float64)
    x = rng.integers(0, V, size=(T, B))
    y = rng.integers(0, V, size=(T, B))
    states = [(rng.uniform(-0.5, 0.5, (B, H)), rng.uniform(-1, 1, (B, H))) for _ in range(L)]   # non-zero entering
    mk = MO.mode_masks(_modes(variational, P_WD), [H] * (L + 1), T, B, V)
    return params, x, y, states, mk.sites, mk.rec, mk.wd


def _modes(variational, p_wd):
    return MO.Modes(seed=12345, step=STEP, p=P, variational=variational, p_rec=P_REC if variational else 0.0,
                    wd_seed=WD_SEED, p_wd=p_wd)


def _oracle(params, x, y, states, masks, rmasks, wd, variational):
    """_model_oracle's loss, scores, states and raw gradients (autograd) as numpy"""
    ps = {k: torch.tensor(v, requires_grad=True) for k, v in params.items()}
    sc, st, _ = MO.forward(ps, torch.tensor(x), [(torch.tensor(h), torch.tensor(c)) for h, c in states], L, False,
                           _modes(variational, P_WD), MO.Masks(sites=masks, rec=rmasks, wd=wd))
    loss = MO.loss_of(sc, torch.tensor(y))
    loss.backward()
    return (loss.item(), sc.detach().numpy(), [(h.detach().numpy(), c.detach().numpy()) for h, c in st],
            {k: v.grad.numpy() for k, v in ps.items()})


def _torch_restatement(params, x, y, states, masks, rmasks, wd):
    """model.py:103-110 as an explicit per-step loop in float64 torch, W_hh replaced by W_hh * m * scale inside the
    graph (AWD-LSTM's WeightDrop); autograd for the gradients.  Returns (loss, scores, states, grads)."""
    tp = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in params.items()}
    s, sr, sw = 1.0 / (1.0 - P), 1.0 / (1.0 - P_REC), 1.0 / (1.0 - P_WD)
    m = [torch.tensor(mk, dtype=torch.float64) * s for mk in masks]
    rm = [torch.tensor(mk, dtype=torch.float64) * sr for mk in rmasks] if rmasks is not None else [1.0] * L
    a = tp["embed.W"][torch.tensor(x)] * m[0]
    out_states = []
    for l in range(L):
        h, c = (torch.tensor(v, dtype=torch.float64) for v in states[l])
        Wi, bi, bh = tp[f"rnns.{l}.weight_ih_l0"], tp[f"rnns.{l}.bias_ih_l0"], tp[f"rnns.{l}.bias_hh_l0"]
        Wh = tp[f"rnns.{l}.weight_hh_l0"] * (torch.tensor(wd[l], dtype=torch.float64) * sw)
        ys = []
        for t in range(T):
            z = a[t] @ Wi.T + bi + (h * rm[l]) @ Wh.T + bh
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


@pytest.mark.parametrize("variational", [False, True])
def test_weight_drop_oracle_matches_torch_autograd(variational):
    params, x, y, states, masks, rmasks, wd = _setup(variational)
    assert wd is not None and all(not w.all() and w.any() for w in wd)
    loss, sc, st, grads = _oracle(params, x, y, states, masks, rmasks, wd, variational)
    t_loss, t_sc, t_st, t_grads = _torch_restatement(params, x, y, states, masks, rmasks, wd)
    np.testing.assert_allclose(loss, t_loss, rtol=1e-12)
    np.testing.assert_allclose(sc, t_sc, rtol=1e-11, atol=1e-12)
    for l in range(L):
        np.testing.assert_allclose(st[l][0], t_st[l][0], rtol=1e-11, atol=1e-12)
        np.testing.assert_allclose(st[l][1], t_st[l][1], rtol=1e-11, atol=1e-12)
    assert sorted(grads) == sorted(t_grads) and len(grads) == 3 + 4 * L
    for k in grads:
        np.testing.assert_allclose(grads[k], t_grads[k], rtol=1e-9, atol=1e-12, err_msg=k)
    for l in range(L):   # exactly 0 where the mask drops
        assert (grads[f"rnns.{l}.weight_hh_l0"][~wd[l]] == 0).all()


def test_weight_drop_changes_the_result_and_p0_is_the_identity():
    """p_wd = 0 is the numpy oracle, to 1e-12 relative (two separate implementations)"""
    params, x, y, states, masks, _, wd = _setup(False)
    a = _oracle(params, x, y, states, masks, None, wd, False)[1]
    b = _oracle(params, x, y, states, masks, None, None, False)[1]
    assert np.abs(a - b).max() > 1e-3
    assert MO.mode_masks(_modes(False, 0.0), [H] * (L + 1), T, B, V).wd is None
    tp = {k: torch.tensor(v) for k, v in params.items()}
    loss, norm, _, after, _, _ = MO.train_step(tp, torch.tensor(x), torch.tensor(y),
                                               [(torch.tensor(h), torch.tensor(c)) for h, c in states], L, False, 1.0,
                                               0.25, _modes(False, 0.0), MO.Masks(sites=masks))
    p2 = {k: v.copy() for k, v in params.items()}
    want = O.train_step(p2, x, y, states, L, 1.0, 0.25, P, masks)
    np.testing.assert_allclose(loss, want[0], rtol=1e-12)
    np.testing.assert_allclose(norm, want[1], rtol=1e-12)
    for k in p2:
        np.testing.assert_allclose(after[k].numpy(), p2[k], rtol=1e-12, err_msg=k)


def test_masks_are_site_2L_plus_1_plus_l_over_w_hh():
    """The mask of layer l is zrb_dropout_mask(wd_seed, step, 2L + 1 + l, 4H*H, p) read in W_hh's row-major order; the
    sites follow the variational mode's recurrent ones and stay far from the sampler's counter word 0xFFFFFFFF."""
    wd = MO.mode_masks(_modes(False, P_WD), [H] * (L + 1), T, B, V).wd
    for l in range(L):
        want = PH.keep_mask(WD_SEED, STEP, 2 * L + 1 + l, 4 * H * H, P_WD).reshape(4 * H, H)
        np.testing.assert_array_equal(wd[l], want)
    assert not np.array_equal(wd[0], wd[1])
    assert 0.3 < 1 - np.mean(np.concatenate([w.ravel() for w in wd])) < 0.7
    assert 3 * 8 < 0xFFFFFFFF   # largest site with ZRB_MAX_LAYERS = 8: 2L + 1 + (L - 1) = 3L


def test_entry_point_declared_and_bound():
    from zaremba_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "zaremba_b200.h")).read()
    assert re.search(r"int\s+zrb_set_weight_drop\(zrb_ctx\* ctx, float p, uint64_t seed\);", hdr)
    res, args = _lib._SIGNATURES["zrb_set_weight_drop"]
    assert res is C.c_int and args == [C.c_void_p, C.c_float, C.c_uint64]
    assert "zrb_set_weight_drop" in _lib.exported_symbols()


def test_model_rejects_bad_weight_drop():
    import zaremba_b200
    for bad in (-0.1, 1.0, 1.5, float("nan"), float("inf"), True, "0.5", None):
        with pytest.raises(ValueError):
            zaremba_b200.Model(V, H, L, P, 0.1, weight_drop=bad)
    with pytest.raises(ValueError):
        zaremba_b200.Model(V, H, L, P, 0.1, "custom", weight_drop=0.5)
    with pytest.raises(TypeError):
        zaremba_b200.Model(V, H, L, P, 0.1, "pytorch", "tc", False, None, False, 0.5)   # keyword-only
    assert zaremba_b200.Model(V, H, L, P, 0.1, weight_drop=0.5).weight_drop == 0.5
    assert zaremba_b200.Model(V, H, L, P, 0.1, "custom", weight_drop=0.0).weight_drop == 0.0
    assert zaremba_b200.Model(V, H, L, P, 0.1).weight_drop == 0.0
    m = zaremba_b200.Model(V, H, L, P, 0.1, weight_drop=0.5, variational=True, tied=True)
    assert sorted(m.state_dict()) == sorted(zaremba_b200.Model(V, H, L, P, 0.1, tied=True).state_dict())
