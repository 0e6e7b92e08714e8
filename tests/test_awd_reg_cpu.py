"""Embedding dropout and AR/TAR without a GPU: their numpy restatement (tests/_awd_reg_oracle.py) against an
independent float64 torch-autograd loop written as AWD-LSTM writes it (`F.embedding(x, W * mask / (1 - p))`, then
`alpha * y.pow(2).mean()` and `beta * (h[1:] - h[:-1]).pow(2).mean()`, times B), with Zaremba's dropout, the variational
mode, weight drop, tied weights and T = 1; the mask's site; the C entry points in the header and the ctypes binding;
Model(embed_dropout=) and Trainer(ar=, tar=) argument checks."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import lstm_lm_oracle as O
from oracle import philox as PH
from tests import _awd_reg_oracle as AO
from tests import _variational_oracle as VO
from tests import _weight_drop_oracle as WO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V, H, L, B = 23, 8, 2, 3
P, P_REC, P_WD, P_E = 0.4, 0.3, 0.5, 0.3
SEED, STEP = 987654321, 3
ALPHA, BETA = 2.0, 1.0


def _setup(T, variational, weight_drop, tied, seed=7):
    rng = np.random.default_rng(seed)
    params = O.init_params(V, H, L, 0.3, seed, dtype=np.float64)
    if tied:
        del params["fc.W"]
    x = rng.integers(0, V, size=(T, B))
    y = rng.integers(0, V, size=(T, B))
    states = [(rng.uniform(-0.5, 0.5, (B, H)), rng.uniform(-1, 1, (B, H))) for _ in range(L)]   # non-zero entering
    if variational:
        masks, rmasks = VO.variational_masks(12345, STEP, L, T, B, H, P, P_REC)
    else:
        masks, rmasks = PH.site_masks(12345, STEP, L, T, B, H, P), None
    wd = WO.weight_drop_masks(SEED, STEP, L, H, P_WD) if weight_drop else None
    em = AO.embed_mask(SEED, STEP, L, V, P_E)
    return params, x, y, states, masks, rmasks, wd, em


def _torch_restatement(params, x, y, states, masks, rmasks, wd, em, tied, alpha=0.0, beta=0.0):
    """model.py:103-110 as an explicit per-step loop in float64 torch with AWD-LSTM's embedded_dropout
    (F.embedding(x, W * mask / (1 - p))), the projection reading the raw E when tied; autograd for the gradients.
    The backward differentiates NLL + AR + TAR (AWD's main.py terms times B, the unit of the NLL).
    Returns (NLL, scores, states, grads, (AR, TAR))."""
    tp = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in params.items()}
    T = x.shape[0]
    s, sr, sw = 1.0 / (1.0 - P), 1.0 / (1.0 - P_REC), 1.0 / (1.0 - P_WD)
    m = [torch.tensor(mk, dtype=torch.float64) * s for mk in masks]
    rm = [torch.tensor(mk, dtype=torch.float64) * sr for mk in rmasks] if rmasks is not None else [1.0] * L
    E = tp["embed.W"]
    emask = torch.tensor(em, dtype=torch.float64)[:, None]
    a = F.embedding(torch.tensor(x), E * emask / (1.0 - P_E)) * m[0]
    out_states = []
    for l in range(L):
        h, c = (torch.tensor(v, dtype=torch.float64) for v in states[l])
        Wi, bi, bh = tp[f"rnns.{l}.weight_ih_l0"], tp[f"rnns.{l}.bias_ih_l0"], tp[f"rnns.{l}.bias_hh_l0"]
        Wh = tp[f"rnns.{l}.weight_hh_l0"]
        if wd is not None:
            Wh = Wh * (torch.tensor(wd[l], dtype=torch.float64) * sw)
        ys = []
        for t in range(T):
            z = a[t] @ Wi.T + bi + (h * rm[l]) @ Wh.T + bh
            i, f, g, o = z.chunk(4, dim=1)
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
            h = torch.sigmoid(o) * torch.tanh(c)
            ys.append(h)
        out_states.append((h.detach().numpy(), c.detach().numpy()))
        hs = torch.stack(ys)
        a = hs * m[l + 1]
    fcW = E if tied else tp["fc.W"]
    scores = a.reshape(-1, H) @ fcW.T + tp["fc.b"]
    logp = torch.log_softmax(scores, dim=1)
    loss = -logp[torch.arange(T * B), torch.tensor(y).reshape(-1)].mean() * B
    ar = alpha * a.pow(2).mean() * B
    tar = beta * (hs[1:] - hs[:-1]).pow(2).mean() * B if T > 1 else torch.zeros((), dtype=torch.float64)
    (loss + ar + tar).backward()
    return (loss.item(), scores.detach().numpy(), out_states, {k: v.grad.numpy() for k, v in tp.items()},
            (ar.item(), tar.item()))


CASES = {   # name -> (T, variational, weight_drop, tied)
    "zaremba": (5, False, False, False),
    "variational": (5, True, False, False),
    "weight_drop": (5, False, True, False),
    "tied": (5, False, False, True),
    "all": (5, True, True, True),
    "t1": (1, False, False, False),
}


@pytest.mark.parametrize("case", list(CASES))
def test_embed_dropout_oracle_matches_torch_autograd(case):
    T, variational, weight_drop, tied = CASES[case]
    params, x, y, states, masks, rmasks, wd, em = _setup(T, variational, weight_drop, tied)
    assert not em.all() and em.any()
    assert (~em[x]).any() and em[x].any(), "the window should hold dropped and kept word types"
    p_rec = P_REC if variational else 0.0
    sc, st, cache = AO.model_fwd(params, x, states, L, P, masks, rmasks, p_rec, wd, P_WD, em, P_E, tied)
    grads = AO.model_bwd(params, cache, O.nll_loss_bwd(sc, y), L, wd, P_WD, em, P_E, tied)
    loss = O.nll_loss(sc, y)
    t_loss, t_sc, t_st, t_grads, _ = _torch_restatement(params, x, y, states, masks, rmasks, wd, em, tied)
    np.testing.assert_allclose(loss, t_loss, rtol=1e-12)
    np.testing.assert_allclose(sc, t_sc, rtol=1e-11, atol=1e-12)
    for l in range(L):
        np.testing.assert_allclose(st[l][0], t_st[l][0], rtol=1e-11, atol=1e-12)
        np.testing.assert_allclose(st[l][1], t_st[l][1], rtol=1e-11, atol=1e-12)
    assert sorted(grads) == sorted(t_grads) and len(grads) == (2 if tied else 3) + 4 * L
    for k in grads:
        np.testing.assert_allclose(grads[k], t_grads[k], rtol=1e-9, atol=1e-12, err_msg=k)
    if not tied:   # exactly 0 on every dropped row; tied: the projection's gradient reaches every row
        assert (grads["embed.W"][~em] == 0).all()
        assert (grads["embed.W"][np.unique(x[em[x]])] != 0).any(axis=1).all()


@pytest.mark.parametrize("case", list(CASES))
def test_activation_reg_oracle_matches_torch_autograd(case):
    """AR/TAR (alpha = 2, beta = 1, AWD's values) on top of every case above, embedding dropout included: the NLL,
    scores and states are those without the penalties; R and all gradients match the loop's."""
    T, variational, weight_drop, tied = CASES[case]
    params, x, y, states, masks, rmasks, wd, em = _setup(T, variational, weight_drop, tied)
    p_rec = P_REC if variational else 0.0
    sc, st, cache = AO.model_fwd(params, x, states, L, P, masks, rmasks, p_rec, wd, P_WD, em, P_E, tied)
    ar, tar, r = AO.activation_reg(cache, L, ALPHA, BETA)
    grads = AO.model_bwd(params, cache, O.nll_loss_bwd(sc, y), L, wd, P_WD, em, P_E, tied, r)
    t_loss, t_sc, t_st, t_grads, (t_ar, t_tar) = _torch_restatement(params, x, y, states, masks, rmasks, wd, em, tied,
                                                                    ALPHA, BETA)
    np.testing.assert_allclose(O.nll_loss(sc, y), t_loss, rtol=1e-12)
    np.testing.assert_allclose(sc, t_sc, rtol=1e-11, atol=1e-12)
    assert ar > 0 and (tar > 0) == (T > 1)
    np.testing.assert_allclose(ar, t_ar, rtol=1e-12)
    np.testing.assert_allclose(tar, t_tar, rtol=1e-12, atol=1e-300)
    for k in grads:
        np.testing.assert_allclose(grads[k], t_grads[k], rtol=1e-9, atol=1e-12, err_msg=k)
    # the penalties reach units whose output was dropped: r is not 0 everywhere the last site's mask drops
    if T > 1:
        dropped = ~np.broadcast_to(masks[L], r.shape)
        assert (r[dropped] != 0).any()
    # the full train step carries the values
    p1 = {k: v.copy() for k, v in params.items()}
    out = AO.train_step(p1, x, y, states, L, 1.0, 0.25, P, masks, rmasks, p_rec, wd, P_WD, em, P_E, tied, ALPHA, BETA)
    assert out[0] == O.nll_loss(sc, y) and out[5] == (ar, tar)


def test_tied_projection_is_unmasked():
    """Tied: dE = G_proj + s_e * G_emb, with the projection reading the raw E."""
    params, x, y, states, masks, _, _, em = _setup(5, False, False, True)
    sc, _, cache = AO.model_fwd(params, x, states, L, P, masks, ed_mask=em, p_e=P_E, tied=True)
    untied = dict(params, **{"fc.W": params["embed.W"].copy()})
    sc2, _, cache2 = AO.model_fwd(untied, x, states, L, P, masks, ed_mask=em, p_e=P_E)
    np.testing.assert_array_equal(sc, sc2)
    g = AO.model_bwd(params, cache, O.nll_loss_bwd(sc, y), L, ed_mask=em, p_e=P_E, tied=True)
    g2 = AO.model_bwd(untied, cache2, O.nll_loss_bwd(sc2, y), L, ed_mask=em, p_e=P_E)
    np.testing.assert_allclose(g["embed.W"], g2["embed.W"] + g2["fc.W"], rtol=1e-13, atol=1e-15)


def test_p0_is_the_weight_drop_oracle():
    params, x, y, states, masks, _, wd, _ = _setup(5, False, True, False)
    assert AO.embed_mask(SEED, STEP, L, V, 0.0) is None
    p1 = {k: v.copy() for k, v in params.items()}
    p2 = {k: v.copy() for k, v in params.items()}
    got = AO.train_step(p1, x, y, states, L, 1.0, 0.25, P, masks, None, 0.0, wd, P_WD)
    want = WO.train_step(p2, x, y, states, L, 1.0, 0.25, P, masks, None, 0.0, wd, P_WD)
    assert got[0] == want[0] and got[1] == want[1] and got[5] == (0.0, 0.0)
    for k in p1:
        np.testing.assert_array_equal(p1[k], p2[k])


def test_mask_is_site_3L_plus_1_over_the_vocabulary():
    """The keep flag of word v is element v of zrb_dropout_mask(seed, step, 3L + 1, V, p): the site after the
    weight-drop ones (2L + 1 .. 3L), far from the sampler's counter word 0xFFFFFFFF."""
    em = AO.embed_mask(SEED, STEP, L, V, P_E)
    np.testing.assert_array_equal(em, PH.keep_mask(SEED, STEP, 3 * L + 1, V, P_E))
    wd_sites = {2 * L + 1 + l for l in range(L)}
    assert 3 * L + 1 not in wd_sites and 3 * L + 1 > max(wd_sites)
    big = AO.embed_mask(SEED, STEP, L, 100000, P_E)
    assert abs((1 - big.mean()) - P_E) < 0.01
    assert not np.array_equal(big, AO.embed_mask(SEED, STEP + 1, L, 100000, P_E))
    assert 3 * 8 + 1 < 0xFFFFFFFF   # largest site with ZRB_MAX_LAYERS = 8


@pytest.mark.parametrize("name,decl,argtypes", [
    ("zrb_set_embed_dropout", r"zrb_set_embed_dropout\(zrb_ctx\* ctx, float p, uint64_t seed\);",
     [C.c_void_p, C.c_float, C.c_uint64]),
    ("zrb_set_activation_reg", r"zrb_set_activation_reg\(zrb_ctx\* ctx, float alpha, float beta\);",
     [C.c_void_p, C.c_float, C.c_float]),
    ("zrb_activation_reg", r"zrb_activation_reg\(zrb_ctx\* ctx, float\* out2, void\* stream\);",
     [C.c_void_p, C.c_void_p, C.c_void_p]),
])
def test_entry_point_declared_and_bound(name, decl, argtypes):
    from zaremba_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "zaremba_b200.h")).read()
    assert re.search(r"int\s+" + decl, hdr)
    res, args = _lib._SIGNATURES[name]
    assert res is C.c_int and args == argtypes
    assert name in _lib.exported_symbols()
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    assert re.search(r"^\|[^|\n]*`" + name + "`", doc, re.M), f"INTEGRATION.md's ABI table has no row for {name}"


def test_model_rejects_bad_embed_dropout():
    import zaremba_b200
    for bad in (-0.1, 1.0, 1.5, float("nan"), float("inf"), True, "0.1", None):
        with pytest.raises(ValueError):
            zaremba_b200.Model(V, H, L, P, 0.1, embed_dropout=bad)
    with pytest.raises(TypeError):
        zaremba_b200.Model(V, H, L, P, 0.1, "pytorch", "tc", False, None, False, 0.0, 0.1)   # keyword-only
    assert zaremba_b200.Model(V, H, L, P, 0.1, embed_dropout=0.1).embed_dropout == 0.1
    assert zaremba_b200.Model(V, H, L, P, 0.1, "custom", embed_dropout=0.1).embed_dropout == 0.1
    assert zaremba_b200.Model(V, H, L, P, 0.1).embed_dropout == 0.0
    m = zaremba_b200.Model(V, H, L, P, 0.1, embed_dropout=0.1, weight_drop=0.5, variational=True, tied=True)
    assert sorted(m.state_dict()) == sorted(zaremba_b200.Model(V, H, L, P, 0.1, tied=True).state_dict())


def test_trainer_rejects_bad_ar_tar():
    """Trainer(ar=, tar=) is keyword-only and checked before anything touches a device."""
    import inspect

    import zaremba_b200
    sig = inspect.signature(zaremba_b200.Trainer.__init__)
    assert sig.parameters["ar"].kind is inspect.Parameter.KEYWORD_ONLY and sig.parameters["ar"].default == 0.0
    assert sig.parameters["tar"].kind is inspect.Parameter.KEYWORD_ONLY and sig.parameters["tar"].default == 0.0
    m = zaremba_b200.Model(V, H, L, P, 0.1)
    for kw in (dict(ar=-1.0), dict(tar=-0.5), dict(ar=float("nan")), dict(tar=float("inf")), dict(ar=True),
               dict(tar="1")):
        with pytest.raises(ValueError):
            zaremba_b200.Trainer(m, B, 5, **kw)
