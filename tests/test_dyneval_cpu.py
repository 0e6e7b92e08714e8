"""The float64 restatement of dynamic evaluation (tests/_dyneval_oracle.py, DESIGN.md section 14) against an independent
torch-autograd float64 loop, its identities, and the new entry points' declarations and bindings."""
import os
import re

import numpy as np
import pytest
import torch

from oracle import lstm_lm_oracle as O
from tests import _dyneval_oracle as DO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V, H, L, T, B = 23, 6, 2, 4, 3
WINDOWS = 4
LR, LAM, EPS = 0.3, 0.02, 2e-5
LR_RMS = 3e-3     # u = g / (r + eps) is O(1) per element: a step the size of the SGD rule's


def _setup(tied, seed=11):
    rng = np.random.default_rng(seed)
    params = O.init_params(V, H, L, 0.3, seed, np.float64)
    if tied:
        params.pop("fc.W")
    data = rng.integers(0, V, size=(B, WINDOWS * T + 1))
    data[0, 2] = data[1, 5] = data[2, 1] = data[0, 6] = 7          # a token repeated inside a window and across them
    batches = [(data[:, s * T:(s + 1) * T].T.copy(), data[:, s * T + 1:(s + 1) * T + 1].T.copy()) for s in range(WINDOWS)]
    states = [(rng.uniform(-0.5, 0.5, (B, H)), rng.uniform(-0.5, 0.5, (B, H))) for _ in range(L)]
    return params, batches, states


def _torch_window(P, x, y, states, tied):
    """Eval-mode loss of one window with torch ops over float64 leaves (an independent restatement of model.py)."""
    E = P["embed.W"]
    Wfc = E if tied else P["fc.W"]
    a = E[torch.as_tensor(x)]
    new = []
    for l in range(L):
        h, c = (torch.as_tensor(s) for s in states[l])
        Wi, Wh = P[f"rnns.{l}.weight_ih_l0"], P[f"rnns.{l}.weight_hh_l0"]
        bi, bh = P[f"rnns.{l}.bias_ih_l0"], P[f"rnns.{l}.bias_hh_l0"]
        outs = []
        for t in range(a.shape[0]):
            i, f, g, o = (a[t] @ Wi.T + bi + h @ Wh.T + bh).chunk(4, dim=1)
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
            h = torch.sigmoid(o) * torch.tanh(c)
            outs.append(h)
        a = torch.stack(outs)
        new.append((h.detach().numpy(), c.detach().numpy()))
    scores = a.reshape(-1, H) @ Wfc.T + P["fc.b"]
    logp = torch.log_softmax(scores, dim=1)[torch.arange(scores.shape[0]), torch.as_tensor(y).reshape(-1)]
    return -logp.mean() * B, new


def _torch_grads(P, x, y, states, tied):
    for v in P.values():
        v.grad = None
    loss, new = _torch_window(P, x, y, states, tied)
    loss.backward()
    return loss.item(), {k: v.grad.detach().clone() for k, v in P.items()}, new


def _torch_reference(params, batches, states, tied, rule):
    P = {k: torch.tensor(v, requires_grad=True) for k, v in params.items()}
    # statistics at theta_g, states carried from zero
    ms = {k: torch.zeros_like(v) for k, v in P.items()}
    st = [(np.zeros((B, H)), np.zeros((B, H))) for _ in range(L)]
    for x, y in batches:
        _, g, st = _torch_grads(P, x, y, st, tied)
        for k in ms:
            ms[k] += g[k] ** 2
    r = {k: (v / len(batches)).sqrt() for k, v in ms.items()}
    rbar = sum(v.sum() for v in r.values()) / sum(v.numel() for v in r.values())
    theta_g = {k: v.detach().clone() for k, v in P.items()}
    losses, st = [], states
    for x, y in batches:
        loss, g, st = _torch_grads(P, x, y, st, tied)
        losses.append(loss)
        with torch.no_grad():
            for k, p in P.items():
                if rule == "rms":
                    u, a, lr = g[k] / (r[k] + EPS), torch.clamp(LAM * r[k] / rbar, max=1.0), LR_RMS
                else:
                    u, a, lr = g[k], min(1.0, LAM), LR
                p += a * (theta_g[k] - p) - lr * u
    return losses, {k: v.detach().numpy() for k, v in P.items()}, {k: v.numpy() for k, v in ms.items()}, r, rbar.item()


@pytest.mark.parametrize("rule", ["rms", "sgd"])
@pytest.mark.parametrize("tied", [False, True], ids=["untied", "tied"])
def test_restatement_matches_torch_autograd(tied, rule):
    params, batches, states = _setup(tied)
    want_losses, want_params, want_ms, want_r, want_rbar = _torch_reference(params, batches, states, tied, rule)
    r, rbar, ms = DO.grad_stats(params, batches, L, B, H, tied)
    assert sorted(r) == sorted(want_r) == sorted(DO.names(L, tied))
    for k in r:
        np.testing.assert_allclose(ms[k], want_ms[k] / len(batches), rtol=1e-12, atol=1e-15)
        np.testing.assert_allclose(r[k], want_r[k].numpy(), rtol=1e-12, atol=1e-15)
    assert abs(rbar - want_rbar) <= 1e-12 * want_rbar
    losses, final, _ = DO.dynamic_pass(params, batches, L, states, LR_RMS if rule == "rms" else LR, LAM,
                                       r if rule == "rms" else None,
                                       rbar if rule == "rms" else None, EPS, tied)
    np.testing.assert_allclose(losses, want_losses, rtol=1e-12)
    for k in final:
        np.testing.assert_allclose(final[k], want_params[k], rtol=1e-10, atol=1e-12)
    assert all(np.isfinite(v).all() for v in final.values())
    moved = max(np.abs(final[k] - params[k]).max() for k in final)
    assert moved > 1e-3, "the pass must adapt the weights"
    assert abs(losses[-1] - DO.dynamic_pass(params, batches, L, states, 0.0, 0.0, tied=tied)[0][-1]) > 1e-6


@pytest.mark.parametrize("tied", [False, True], ids=["untied", "tied"])
def test_zero_rates_reproduce_perplexity(tied):
    params, batches, _ = _setup(tied)
    full = dict(params)
    if tied:
        full["fc.W"] = full["embed.W"]
    want = O.perplexity(full, batches, L, B, H)
    r, rbar, _ = DO.grad_stats(params, batches, L, B, H, tied)
    for rms, rb in ((None, None), (r, rbar)):
        assert DO.dynamic_perplexity(params, batches, L, B, H, 0.0, 0.0, rms, rb, EPS, tied) == pytest.approx(want,
                                                                                                              rel=1e-14)


def test_first_window_loss_does_not_depend_on_the_rates():
    params, batches, states = _setup(False)
    r, rbar, _ = DO.grad_stats(params, batches, L, B, H)
    first = {DO.dynamic_pass(params, batches, L, states, lr, lam, rms, rb)[0][0]
             for lr, lam in ((0.0, 0.0), (0.05, 0.0), (0.01, 0.7)) for rms, rb in ((None, None), (r, rbar))}
    assert len(first) == 1


def test_zero_statistic_gives_no_decay_and_a_step_of_g_over_eps():
    p = {"w": np.array([1.0, 2.0])}
    DO.update(p, {"w": np.array([0.5, 0.5])}, {"w": np.array([0.0, 0.0])}, 0.1, 10.0,
              rms={"w": np.array([0.0, 1.0])}, rbar=0.5, eps=0.25)
    # element 0: r = 0 -> a = 0, u = g / eps = 2; element 1: a = min(1, 10 * 1 / 0.5) = 1 (clipped), u = 0.5 / 1.25
    np.testing.assert_allclose(p["w"], [1.0 - 0.1 * 2.0, 0.0 - 0.1 * 0.4])


def test_entry_points_are_declared_and_bound():
    from zaremba_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "zaremba_b200.h")).read(), flags=re.S)
    for name in ("zrb_grad_stats_step", "zrb_grad_stats_finish", "zrb_dyneval_step"):
        assert re.search(rf"\b{name}\s*\(", src), name
        assert name in _lib.exported_symbols(), name
    import zaremba_b200
    assert zaremba_b200.GradStats is zaremba_b200.dyneval.GradStats
    for m in ("gradient_stats", "dynamic_eval_step", "dynamic_perplexity"):
        assert callable(getattr(zaremba_b200.Trainer, m))
