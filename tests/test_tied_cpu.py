"""The tied embedding mode without a GPU: the float64 restatement (tests/_model_oracle.py) against torch autograd over a
genuinely shared nn.Parameter, the host side of Model(tied=True), and the flag in the header and the ctypes binding."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch
from torch import nn

from oracle import lstm_lm_oracle as O
from oracle import philox as PH
from tests import _model_oracle as MO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V, H, L, T, B = 23, 8, 2, 5, 3
P = 0.4


def _setup(seed=7):
    rng = np.random.default_rng(seed)
    params = O.init_params(V, H, L, 0.3, seed, dtype=np.float64)
    del params["fc.W"]
    x = rng.integers(0, V, size=(T, B))
    x[1, 0] = x[3, 2] = x[0, 1]                       # a repeated token: its rows sum in the embedding part
    y = rng.integers(0, V, size=(T, B))
    states = [(rng.uniform(-0.5, 0.5, (B, H)), rng.uniform(-1, 1, (B, H))) for _ in range(L)]   # non-zero entering
    masks = [PH.keep_mask(99, 1, s, T * B * H, P).reshape(T, B, H) for s in range(L + 1)]
    return params, x, y, states, masks


def _oracle(params, x, y, states, masks, lr=0.0, max_norm=float("inf")):
    """_model_oracle's tied step as numpy: (NLL, norm, raw grads, params after, states after, scores)"""
    ps = {k: torch.tensor(v) for k, v in params.items()}
    x, y = torch.tensor(x), torch.tensor(y)
    states = [(torch.tensor(h), torch.tensor(c)) for h, c in states]
    md, mk = MO.Modes(p=P), MO.Masks(sites=masks)
    loss, norm, grads, after, st, _ = MO.train_step(ps, x, y, states, L, True, lr, max_norm, md, mk)
    sc = MO.forward(ps, x, states, L, True, md, mk)[0]
    return (loss, norm, {k: v.numpy() for k, v in grads.items()}, {k: v.numpy() for k, v in after.items()},
            [(h.numpy(), c.numpy()) for h, c in st], sc.numpy())


class _TorchTied(nn.Module):
    """model.py:103-110 in float64 torch with fc.W and embed.W ONE nn.Parameter."""

    def __init__(self, params):
        super().__init__()
        self.E = nn.Parameter(torch.tensor(params["embed.W"]))
        self.lstm = nn.ParameterList()
        for l in range(L):
            for k in ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0"):
                self.lstm.append(nn.Parameter(torch.tensor(params[f"rnns.{l}.{k}"])))
        self.b = nn.Parameter(torch.tensor(params["fc.b"]))

    def forward(self, x, y, states, masks):
        s = 1.0 / (1.0 - P)
        m = [torch.tensor(mk, dtype=torch.float64) * s for mk in masks]
        a = self.E[torch.tensor(x)] * m[0]
        out = []
        for l in range(L):
            Wi, Wh, bi, bh = self.lstm[4 * l:4 * l + 4]
            h, c = (torch.tensor(v) for v in states[l])
            ys = []
            for t in range(T):
                i, f, g, o = (a[t] @ Wi.T + bi + h @ Wh.T + bh).chunk(4, dim=1)
                c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
                h = torch.sigmoid(o) * torch.tanh(c)
                ys.append(h)
            out.append((h.detach().numpy(), c.detach().numpy()))
            a = torch.stack(ys) * m[l + 1]
        scores = a.reshape(-1, H) @ self.E.T + self.b          # the SAME parameter projects
        logp = torch.log_softmax(scores, dim=1)
        loss = -logp[torch.arange(T * B), torch.tensor(y).reshape(-1)].mean() * B
        return loss, scores, out

    def named(self):
        names = MO.names(L, True)
        return dict(zip(names, [self.E, *self.lstm, self.b]))


def test_tied_oracle_matches_torch_autograd_with_a_shared_parameter():
    params, x, y, states, masks = _setup()
    lr, max_norm = 0.9, 0.05
    tm = _TorchTied(params)
    t_loss, t_sc, t_st = tm(x, y, states, masks)
    t_loss.backward()
    t_grads = {k: p.grad.numpy().copy() for k, p in tm.named().items()}

    loss, norm, grads, p_or, st, sc = _oracle(params, x, y, states, masks, lr, max_norm)
    np.testing.assert_allclose(loss, t_loss.item(), rtol=1e-12)
    np.testing.assert_allclose(sc, t_sc.detach().numpy(), rtol=1e-11, atol=1e-12)
    for l in range(L):
        np.testing.assert_allclose(st[l][0], t_st[l][0], rtol=1e-11, atol=1e-12)
        np.testing.assert_allclose(st[l][1], t_st[l][1], rtol=1e-11, atol=1e-12)
    assert sorted(t_grads) == sorted(MO.names(L, True)) and len(t_grads) == 2 + 4 * L

    t_norm = torch.nn.utils.clip_grad_norm_(tm.parameters(), max_norm).item()
    np.testing.assert_allclose(norm, t_norm, rtol=1e-12)
    coef = min(1.0, max_norm / (norm + 1e-6))
    assert coef < 1.0, "the clip must be active"
    for k in MO.names(L, True):
        np.testing.assert_allclose(grads[k], t_grads[k], rtol=1e-10, atol=1e-13, err_msg=k)
    with torch.no_grad():
        for p in tm.parameters():
            p -= lr * p.grad
    for k, p in tm.named().items():
        np.testing.assert_allclose(p_or[k], p.detach().numpy(), rtol=1e-12, atol=1e-14, err_msg=k)


def test_tied_gradient_is_the_sum_of_the_untied_pair():
    """against the numpy oracle's untied pair, to 1e-12 relative (two separate implementations)"""
    params, x, y, states, masks = _setup(3)
    untied = dict(params, **{"fc.W": params["embed.W"].copy()})
    sc, _, cache = O.model_fwd(untied, x, states, L, P, masks)
    g_u = O.model_bwd(untied, cache, O.nll_loss_bwd(sc, y), L)
    _, _, g_t, _, _, sc_t = _oracle(params, x, y, states, masks)
    np.testing.assert_allclose(sc_t, sc, rtol=1e-12)
    np.testing.assert_allclose(g_t["embed.W"], g_u["embed.W"] + g_u["fc.W"], rtol=1e-12)
    assert "fc.W" not in g_t


def _names(m):
    return [n for n, _ in m.named_parameters()]


def test_model_tied_on_the_host():
    import zaremba_b200
    torch.manual_seed(3)
    m = zaremba_b200.Model(V, H, L, 0.5, 0.1, tied=True)
    assert m.fc.W is m.embed.W
    assert len(list(m.parameters())) == 2 + 4 * L
    assert _names(m) == MO.names(L, True)
    assert [id(p) for p in m.ordered_parameters()] == [id(p) for p in m.parameters()]
    assert sum(p.numel() for p in m.parameters()) == V * H + 4 * L * (2 * H * H + 2 * H) + V
    sd = m.state_dict()
    assert sorted(sd) == sorted(O.param_names(L)) and len(sd) == 3 + 4 * L
    assert torch.equal(sd["embed.W"], sd["fc.W"])
    # a tied checkpoint loads into an untied model, and back into a tied one
    u = zaremba_b200.Model(V, H, L, 0.5, 0.1)
    u.load_state_dict(sd)
    assert torch.equal(u.fc.W, m.embed.W) and u.fc.W is not u.embed.W
    t2 = zaremba_b200.Model(V, H, L, 0.5, 0.1, tied=True)
    t2.load_state_dict(sd)
    assert torch.equal(t2.embed.W, m.embed.W) and t2.fc.W is t2.embed.W


def test_model_tied_rejects_mismatched_checkpoint_and_non_bool():
    import zaremba_b200
    torch.manual_seed(4)
    u = zaremba_b200.Model(V, H, L, 0.5, 0.1)
    m = zaremba_b200.Model(V, H, L, 0.5, 0.1, tied=True)
    before = m.embed.W.detach().clone()
    with pytest.raises(ValueError, match="embed.W and fc.W"):
        m.load_state_dict(u.state_dict())
    assert torch.equal(m.embed.W, before), "a refused checkpoint leaves the model unchanged"
    for bad in (1, 0, "yes", None, 1.0):
        with pytest.raises(ValueError, match="tied"):
            zaremba_b200.Model(V, H, L, 0.5, 0.1, tied=bad)
    with pytest.raises(TypeError):
        zaremba_b200.Model(V, H, L, 0.5, 0.1, "pytorch", "tc", False, None, True)   # keyword only


def test_tied_init_is_seed_for_seed_the_untied_one():
    """reset_parameters walks parameters(): E and the LSTM tensors equal an untied model's embed.W and LSTM tensors,
    and fc.b is drawn where the untied model draws fc.W."""
    import zaremba_b200
    torch.manual_seed(11)
    u = zaremba_b200.Model(V, H, L, 0.5, 0.1)
    torch.manual_seed(11)
    t = zaremba_b200.Model(V, H, L, 0.5, 0.1, tied=True)
    su, st = u.state_dict(), t.state_dict()
    for k in MO.names(L, True)[:-1]:
        assert torch.equal(su[k], st[k]), k
    # replay Model's draws: the LSTM constructors (as nn.LSTM's), then reset_parameters up to where fc.W would be drawn
    torch.manual_seed(11)
    for _ in range(L):
        zaremba_b200.model.LSTM(H, H)
    nn.init.uniform_(torch.empty(V, H), -0.1, 0.1)
    for _ in range(L):
        for shape in ((4 * H, H), (4 * H, H), (4 * H,), (4 * H,)):
            nn.init.uniform_(torch.empty(shape), -0.1, 0.1)
    assert torch.equal(t.fc.b.detach(), nn.init.uniform_(torch.empty(V), -0.1, 0.1))
    assert not torch.equal(t.fc.b.detach(), u.fc.b.detach())


def test_model_without_the_keyword_is_unchanged():
    import zaremba_b200
    torch.manual_seed(5)
    a = zaremba_b200.Model(V, H, L, 0.5, 0.1)
    torch.manual_seed(5)
    b = zaremba_b200.Model(V, H, L, 0.5, 0.1, "pytorch", tied=False)
    assert a.tied is False and a.fc.W is not a.embed.W
    assert len(list(a.parameters())) == 3 + 4 * L and _names(a) == O.param_names(L)
    assert len(a.ordered_parameters()) == 3 + 4 * L
    for (ka, va), (kb, vb) in zip(a.state_dict().items(), b.state_dict().items()):
        assert ka == kb and torch.equal(va, vb)


def test_header_documents_the_flag_and_the_binding_has_it():
    from zaremba_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "zaremba_b200.h")).read()
    assert re.search(r"#define\s+ZRB_TIED_EMBEDDING\s+1\b", hdr)
    assert re.search(r"int32_t\s+flags;", hdr) and "reserved;\n} zrb_config" not in hdr
    assert _lib.TIED_EMBEDDING == 1
    assert _lib.ZrbConfig.flags.offset == 28 and C.sizeof(_lib.ZrbConfig) == 32
