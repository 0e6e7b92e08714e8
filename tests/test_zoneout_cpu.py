"""Zoneout (DESIGN.md section 20) without a GPU: the fp64 restatement of tests/_model_oracle.py against torch autograd of
a literal transcription of Krueger et al.'s LSTM equations, its flags, the Model's arguments, the ABI, and what ptxas
makes of the zoneout instantiations of the persistent recurrence kernels."""
import os
import re

import numpy as np
import pytest
import torch

from oracle import lstm_lm_oracle as O
from oracle import philox
from tests import _model_oracle as MO
from tests.test_rec_codegen_cpu import _stack_frames, ptxas_logs  # noqa: F401  (the module fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V, H, L, T, B = 23, 6, 2, 5, 3


def _params(seed=0):
    return O.init_params(V, H, L, 0.3, seed, dtype=np.float64)


def _masks(seed, step, z_c, z_h, Lm=L):
    return MO.mode_masks(MO.Modes(seed=seed, step=step, z_c=z_c, z_h=z_h), [H] * (Lm + 1), T, B, V)


def _oracle(params, x, y, states, z_c, z_h, train):
    """_model_oracle's loss, states and gradients (autograd) as numpy, flags of seed 7 at step 3 in train mode"""
    P = {k: torch.tensor(v, requires_grad=True) for k, v in params.items()}
    scores, st, _ = MO.forward(P, torch.as_tensor(x), [tuple(torch.tensor(v) for v in s) for s in states], L, False,
                               MO.Modes(seed=7, step=3, z_c=z_c, z_h=z_h), train=train)
    loss = MO.loss_of(scores, torch.as_tensor(y))
    loss.backward()
    return (loss.item(), scores.detach().numpy(), [(h.detach().numpy(), c.detach().numpy()) for h, c in st],
            {k: v.grad.numpy() for k, v in P.items()})


def _krueger(params, x, y, states, z_c, z_h, zflags):
    """Krueger et al. 2017 (section 3): an LSTMCell loop, c_t = d^c c_{t-1} + (1 - d^c) c~ and h_t likewise, with the
    masks d = the flags in train mode and d = z in eval mode; the loss of main.py:77-84.  Autograd gives the gradients."""
    P = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in params.items()}
    a = P["embed.W"][torch.as_tensor(x)]
    new_states = []
    for l in range(L):
        cell = torch.nn.LSTMCell(H, H).double()
        h, c = (torch.tensor(s, dtype=torch.float64) for s in states[l])
        ys = []
        for t in range(T):
            h_new, c_new = torch.func.functional_call(cell, {
                "weight_ih": P[f"rnns.{l}.weight_ih_l0"], "weight_hh": P[f"rnns.{l}.weight_hh_l0"],
                "bias_ih": P[f"rnns.{l}.bias_ih_l0"], "bias_hh": P[f"rnns.{l}.bias_hh_l0"]}, (a[t], (h, c)))
            if zflags is None:
                dc, dh = z_c, z_h
            else:
                dc = 0.0 if zflags.zc is None else torch.tensor(zflags.zc[l][t], dtype=torch.float64)
                dh = 0.0 if zflags.zh is None else torch.tensor(zflags.zh[l][t], dtype=torch.float64)
            c = dc * c + (1 - dc) * c_new
            h = dh * h + (1 - dh) * h_new
            ys.append(h)
        new_states.append((h.detach().numpy(), c.detach().numpy()))
        a = torch.stack(ys)
    scores = a.reshape(-1, H) @ P["fc.W"].T + P["fc.b"]
    p = torch.softmax(scores, 1)[torch.arange(T * B), torch.as_tensor(y).reshape(-1)]
    loss = torch.mean(-torch.log(p) * B)
    loss.backward()
    return loss.item(), new_states, {k: v.grad.numpy() for k, v in P.items()}


@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("z", [(0.5, 0.05), (0.3, 0.4), (0.0, 0.2)])
def test_oracle_equals_autograd_of_krueger(train, z):
    z_c, z_h = z
    rng = np.random.default_rng(1)
    x, y = rng.integers(0, V, (T, B)), rng.integers(0, V, (T, B))
    states = [(rng.standard_normal((B, H)) * 0.5, rng.standard_normal((B, H))) for _ in range(L)]
    params = _params()
    zflags = _masks(7, 3, z_c, z_h) if train else None
    want_loss, want_states, want = _krueger(params, x, y, states, z_c, z_h, zflags)
    loss, _, got_states, got = _oracle(params, x, y, states, z_c, z_h, train)
    assert abs(loss - want_loss) < 1e-12
    for (h, c), (wh, wc) in zip(got_states, want_states):
        np.testing.assert_allclose(h, wh, atol=1e-13)
        np.testing.assert_allclose(c, wc, atol=1e-13)
    for k in O.param_names(L):
        np.testing.assert_allclose(got[k], want[k], atol=1e-12, err_msg=k)


def test_zero_rates_are_the_plain_lstm():
    """against the numpy oracle, to 1e-12 relative (two separate implementations)"""
    rng = np.random.default_rng(2)
    x, y = rng.integers(0, V, (T, B)), rng.integers(0, V, (T, B))
    states = O.zero_states(L, B, H, np.float64)
    params = _params()
    _, scores, _, got = _oracle(params, x, y, states, 0.0, 0.0, True)
    want_scores, _, want_cache = O.model_fwd(params, x, states, L)
    np.testing.assert_allclose(scores, want_scores, rtol=1e-12)
    want = O.model_bwd(params, want_cache, O.nll_loss_bwd(want_scores, y), L)
    for k in O.param_names(L):
        np.testing.assert_allclose(got[k], want[k], rtol=1e-12, atol=1e-15, err_msg=k)


def test_flags_take_their_own_sites():
    """c's flags are site 3L + 3 + l and h's 4L + 3 + l, the dropped flags of the site's stream; none collides with the
    sites before them (0 .. 3L + 2) or with each other"""
    Lm = 3
    sites = {(3 * Lm + 3 + l) for l in range(Lm)} | {(4 * Lm + 3 + l) for l in range(Lm)}
    assert len(sites) == 2 * Lm and min(sites) == 3 * Lm + 3 and max(sites) == 5 * Lm + 2
    mk = _masks(11, 4, 0.5, 0.25, Lm)
    zc, zh = mk.zc[1], mk.zh[1]
    np.testing.assert_array_equal(zc.reshape(-1), ~philox.keep_mask(11, 4, 3 * Lm + 4, T * B * H, 0.5))
    np.testing.assert_array_equal(zh.reshape(-1), ~philox.keep_mask(11, 4, 4 * Lm + 4, T * B * H, 0.25))
    assert 0.3 < zc.mean() < 0.7 and 0.05 < zh.mean() < 0.5
    mk0 = _masks(11, 4, 0.0, 0.0, Lm)
    assert mk0.zc is None and mk0.zh is None          # no flag: no unit is zoned


@pytest.mark.parametrize("kw, msg", [
    ({"zoneout_cell": 1.0}, "zoneout_cell"), ({"zoneout_hidden": -0.1}, "zoneout_hidden"),
    ({"zoneout_cell": True}, "zoneout_cell"), ({"zoneout_hidden": "0.1"}, "zoneout_hidden"),
    ({"zoneout_cell": 0.5, "lstm_type": "custom"}, "lstm_type"), ({"zoneout_hidden": 0.1, "engine": "simt"}, "engine"),
])
def test_model_refuses(kw, msg):
    import zaremba_b200
    with pytest.raises(ValueError, match=msg):
        zaremba_b200.Model(V, H, L, 0.0, 0.1, **kw)


def test_model_arguments_and_checkpoint():
    import zaremba_b200
    torch.manual_seed(0)
    plain = zaremba_b200.Model(V, H, L, 0.0, 0.1)
    torch.manual_seed(0)
    m = zaremba_b200.Model(V, H, L, 0.0, 0.1, zoneout_cell=0.5, zoneout_hidden=0.05)
    assert (m.zoneout_cell, m.zoneout_hidden) == (0.5, 0.05)
    sd, want = m.state_dict(), plain.state_dict()
    assert list(sd) == list(want) and all(torch.equal(sd[k], want[k]) for k in sd)
    with pytest.raises(TypeError):
        zaremba_b200.Model(V, H, L, 0.0, 0.1, "pytorch", "tc", False, None, 0.5)   # keyword-only


def test_abi_declares_zrb_set_zoneout():
    from zaremba_b200 import _lib
    with open(os.path.join(ROOT, "include", "zaremba_b200.h")) as f:
        hdr = f.read()
    assert re.search(r"int\s+zrb_set_zoneout\(zrb_ctx\* ctx, float z_c, float z_h\);", hdr)
    res, args = _lib._SIGNATURES["zrb_set_zoneout"]
    assert len(args) == 3
    with open(os.path.join(ROOT, "zaremba_b200", "csrc", "api.cu")) as f:
        api = f.read()
    body = api[api.index("int zrb_set_zoneout("):]
    body = body[:body.index("\n}\n")]
    # refusals before anything is allocated or launched
    assert body.index("ZRB_ENGINE_TC") < body.index("dalloc") and "isfinite(z_c)" in body and "isfinite(z_h)" in body
    for entry in ("zrb_lstm_layer_fwd", "zrb_lstm_layer_bwd"):
        fn = api[api.index(f"int {entry}("):]
        fn = fn[:fn.index("\n}\n")]
        assert "!zoneout_on(c)" in fn, entry
    with open(os.path.join(ROOT, "INTEGRATION.md")) as f:
        assert "zrb_set_zoneout" in f.read()


def test_zoneout_instantiations_use_no_local_memory(ptxas_logs):  # noqa: F811
    log = ptxas_logs["lstm_rec_zoneout.cu"]
    frames = _stack_frames(log)
    kernels = {f: b for f, b in frames.items() if re.search(r"lstm_rec_(fwd|bwd)_kernel", f)}
    assert len(kernels) == 4 and all(re.search(r"Lb1EE", f) for f in kernels), frames
    assert all(b == 0 for b in kernels.values()), kernels
    assert not re.search(r"[1-9]\d* bytes spill", "\n".join(
        ln for ln in log.splitlines() if "spill" in ln)), "a zoneout instantiation spills"


def test_mode_off_instantiations_stay_where_they_were(ptxas_logs):  # noqa: F811
    """lstm_rec_fwd.cu / lstm_rec_bwd.cu hold only the mode-off instantiations (ZO = false)"""
    for name in ("lstm_rec_fwd.cu", "lstm_rec_bwd.cu"):
        kernels = [f for f in _stack_frames(ptxas_logs[name]) if re.search(r"lstm_rec_(fwd|bwd)_kernel", f)]
        assert len(kernels) == 2 and all(f.endswith("Lb0EEEvNS_10RecFwdArgsE") or f.endswith("Lb0EEEvNS_10RecBwdArgsE")
                                         for f in kernels), kernels
