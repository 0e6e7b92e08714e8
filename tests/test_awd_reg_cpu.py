"""Embedding dropout and AR/TAR without a GPU: the fp64 restatement (tests/_model_oracle.py) against an
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
from tests import _model_oracle as MO

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
    mk = MO.mode_masks(_modes(variational, weight_drop), [H] * (L + 1), T, B, V)
    return params, x, y, states, mk.sites, mk.rec, mk.wd, mk.ed


def _modes(variational, weight_drop, alpha=0.0, beta=0.0, p_e=P_E):
    return MO.Modes(seed=12345, step=STEP, p=P, variational=variational, p_rec=P_REC if variational else 0.0,
                    wd_seed=SEED, p_wd=P_WD if weight_drop else 0.0, ed_seed=SEED, p_e=p_e, alpha=alpha, beta=beta)


def _embed_mask(step, V, p_e):
    return MO.mode_masks(MO.Modes(ed_seed=SEED, step=step, p_e=p_e), [H] * (L + 1), 1, 1, V).ed


def _tensors(params, x, y, states):
    return ({k: torch.tensor(v) for k, v in params.items()}, torch.tensor(x), torch.tensor(y),
            [(torch.tensor(h), torch.tensor(c)) for h, c in states])


def _oracle(params, x, y, states, masks, rmasks, wd, em, md, tied):
    """_model_oracle's NLL, scores, states, raw gradients of NLL + AR + TAR (autograd) and AR + TAR, as numpy"""
    ps, x, y, states = _tensors(params, x, y, states)
    ps = {k: v.requires_grad_(True) for k, v in ps.items()}
    sc, st, reg = MO.forward(ps, x, states, L, tied, md, MO.Masks(sites=masks, rec=rmasks, wd=wd, ed=em))
    loss = MO.loss_of(sc, y)
    (loss + reg).backward()
    return (loss.item(), sc.detach().numpy(), [(h.detach().numpy(), c.detach().numpy()) for h, c in st],
            {k: v.grad.numpy() for k, v in ps.items()}, torch.as_tensor(reg).item())


def _torch_restatement(params, x, y, states, masks, rmasks, wd, em, tied, alpha=0.0, beta=0.0):
    """model.py:103-110 as an explicit per-step loop in float64 torch with AWD-LSTM's embedded_dropout
    (F.embedding(x, W * mask / (1 - p))), the projection reading the raw E when tied; autograd for the gradients.
    The backward differentiates NLL + AR + TAR (AWD's main.py terms times B, the unit of the NLL).
    Returns (NLL, scores, states, grads, (AR, TAR), r = d(AR + TAR) / dh of the last layer's raw output)."""
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
    r = torch.autograd.grad(ar + tar, hs, retain_graph=True)[0] if alpha > 0 or beta > 0 else None
    (loss + ar + tar).backward()
    return (loss.item(), scores.detach().numpy(), out_states, {k: v.grad.numpy() for k, v in tp.items()},
            (ar.item(), tar.item()), r)


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
    loss, sc, st, grads, _ = _oracle(params, x, y, states, masks, rmasks, wd, em, _modes(variational, weight_drop),
                                     tied)
    t_loss, t_sc, t_st, t_grads, _, _ = _torch_restatement(params, x, y, states, masks, rmasks, wd, em, tied)
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
    args = (params, x, y, states, masks, rmasks, wd, em)
    nll, sc, st, grads, reg = _oracle(*args, _modes(variational, weight_drop, ALPHA, BETA), tied)
    ar = _oracle(*args, _modes(variational, weight_drop, ALPHA, 0.0), tied)[4]
    tar = _oracle(*args, _modes(variational, weight_drop, 0.0, BETA), tied)[4]
    t_loss, t_sc, t_st, t_grads, (t_ar, t_tar), r = _torch_restatement(*args, tied, ALPHA, BETA)
    np.testing.assert_allclose(nll, t_loss, rtol=1e-12)
    np.testing.assert_allclose(sc, t_sc, rtol=1e-11, atol=1e-12)
    assert ar > 0 and (tar > 0) == (T > 1)
    np.testing.assert_allclose(ar, t_ar, rtol=1e-12)
    np.testing.assert_allclose(tar, t_tar, rtol=1e-12, atol=1e-300)
    for k in grads:
        np.testing.assert_allclose(grads[k], t_grads[k], rtol=1e-9, atol=1e-12, err_msg=k)
    # the penalties reach units whose output was dropped (r is not 0 everywhere the last site's mask drops), so the
    # gradients above tell TAR on the raw h from TAR on the masked output
    if T > 1:
        dropped = ~np.broadcast_to(masks[L], r.shape)
        assert (r.numpy()[dropped] != 0).any()
    # the full train step carries the values
    out = MO.train_step(*_tensors(params, x, y, states), L, tied, 1.0, 0.25,
                        _modes(variational, weight_drop, ALPHA, BETA), MO.Masks(sites=masks, rec=rmasks, wd=wd, ed=em))
    assert out[0] == nll and out[5] == reg == ar + tar


def test_tied_projection_is_unmasked():
    """Tied: dE = G_proj + s_e * G_emb, with the projection reading the raw E."""
    params, x, y, states, masks, _, _, em = _setup(5, False, False, True)
    md = _modes(False, False)
    _, sc, _, g, _ = _oracle(params, x, y, states, masks, None, None, em, md, True)
    untied = dict(params, **{"fc.W": params["embed.W"].copy()})
    _, sc2, _, g2, _ = _oracle(untied, x, y, states, masks, None, None, em, md, False)
    np.testing.assert_array_equal(sc, sc2)
    np.testing.assert_allclose(g["embed.W"], g2["embed.W"] + g2["fc.W"], rtol=1e-13, atol=1e-15)


def test_p0_is_the_weight_drop_oracle():
    """p_e = 0 draws no mask and is the weight-drop step, bit for bit"""
    params, x, y, states, masks, _, wd, _ = _setup(5, False, True, False)
    assert _embed_mask(STEP, V, 0.0) is None
    got = MO.train_step(*_tensors(params, x, y, states), L, False, 1.0, 0.25, _modes(False, True, p_e=0.0))
    want = MO.train_step(*_tensors(params, x, y, states), L, False, 1.0, 0.25,
                         MO.Modes(p=P, p_wd=P_WD), MO.Masks(sites=masks, wd=wd))
    assert got[0] == want[0] and got[1] == want[1] and got[5] == 0.0
    for k in params:
        assert torch.equal(got[3][k], want[3][k]), k


def test_mask_is_site_3L_plus_1_over_the_vocabulary():
    """The keep flag of word v is element v of zrb_dropout_mask(seed, step, 3L + 1, V, p): the site after the
    weight-drop ones (2L + 1 .. 3L), far from the sampler's counter word 0xFFFFFFFF."""
    em = _embed_mask(STEP, V, P_E)
    np.testing.assert_array_equal(em, PH.keep_mask(SEED, STEP, 3 * L + 1, V, P_E))
    wd_sites = {2 * L + 1 + l for l in range(L)}
    assert 3 * L + 1 not in wd_sites and 3 * L + 1 > max(wd_sites)
    big = _embed_mask(STEP, 100000, P_E)
    assert abs((1 - big.mean()) - P_E) < 0.01
    assert not np.array_equal(big, _embed_mask(STEP + 1, 100000, P_E))
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
