"""The float64 restatement of the neural-cache evaluation (tests/_neural_cache_oracle.py, DESIGN.md section 12) against
an independent brute-force loop, and the properties the definition implies.  No GPU."""
import numpy as np
import pytest
import torch

from tests._neural_cache_oracle import NeuralCache, half_round, mix_row_loss


def _brute(windows, W, theta):
    """p_cache of every row of every window: an explicit per-stream history list and a torch float64 softmax."""
    B = windows[0][0].shape[1]
    hist = [[] for _ in range(B)]
    out = []
    for h, y in windows:
        T = h.shape[0]
        pc = np.zeros((T, B))
        for t in range(T):
            for b in range(B):
                q = torch.tensor(half_round(h[t, b]), dtype=torch.float64)
                past = hist[b][-W:]
                if past:
                    keys = torch.tensor(np.stack([k for k, _ in past]), dtype=torch.float64)
                    p = torch.softmax(theta * (keys @ q), dim=0)
                    pc[t, b] = float(sum(p[i] for i, (_, tok) in enumerate(past) if tok == y[t, b]))
                hist[b].append((half_round(h[t, b]), int(y[t, b])))
        out.append(pc.reshape(-1))
    return out


def _stream(T, B, H, V, seed):
    rng = np.random.default_rng(seed)
    h = rng.normal(size=(T, B, H)) * 0.5
    y = rng.integers(0, V, size=(T, B))
    return h, y


@pytest.mark.parametrize("W", [1, 5, 100])
@pytest.mark.parametrize("theta", [0.0, 0.7, 6.0])
def test_oracle_against_brute_force(W, theta):
    h, y = _stream(23, 3, 16, 5, W)
    windows = [(h[:9], y[:9]), (h[9:10], y[9:10]), (h[10:], y[10:])]
    want = _brute(windows, W, theta)
    c = NeuralCache(W, 3)
    for (hw, yw), w in zip(windows, want):
        got = c.step(hw, yw, theta)["p_cache"]
        np.testing.assert_allclose(got, w, rtol=1e-12, atol=1e-14)


@pytest.mark.parametrize("W", [1, 5, 100])
@pytest.mark.parametrize("chunk", [1, 7, 35])
def test_windows_of_any_length_give_the_same_p_cache(W, chunk):
    T, B = 70, 2
    h, y = _stream(T, B, 12, 4, 11)
    whole = NeuralCache(W, B).step(h, y, 1.3)["p_cache"].reshape(T, B)
    c = NeuralCache(W, B)
    parts = [c.step(h[t:t + chunk], y[t:t + chunk], 1.3)["p_cache"].reshape(-1, B) for t in range(0, T, chunk)]
    np.testing.assert_allclose(np.concatenate(parts), whole, rtol=1e-12, atol=1e-15)


def test_lambda_zero_is_the_plain_nll_and_theta_zero_is_uniform():
    T, B, W = 30, 3, 8
    h, y = _stream(T, B, 10, 3, 5)
    r = np.random.default_rng(1).uniform(0.5, 9.0, size=T * B)
    out = NeuralCache(W, B).step(h, y, 2.0, lam=0.0, row_loss=r)
    np.testing.assert_array_equal(out["row_loss"], r)
    assert out["loss"] == pytest.approx(r.mean() * B, rel=1e-15)
    uni = NeuralCache(W, B).step(h, y, 0.0)["p_cache"].reshape(T, B)
    for t in range(T):
        for b in range(B):
            past = y[max(0, t - W):t, b]
            assert uni[t, b] == pytest.approx((past == y[t, b]).mean() if len(past) else 0.0, abs=1e-15)


def test_first_token_after_reset_and_absent_targets():
    T, B, W, lam = 6, 2, 4, 0.25
    h, _ = _stream(T, B, 8, 3, 2)
    y = np.arange(T * B).reshape(T, B) + 100          # no target is ever in the cache
    r = np.full(T * B, 3.0)
    c = NeuralCache(W, B)
    c.step(h, (y % 3), 1.0)                           # fill it, then reset
    c.reset()
    out = c.step(h, y, 1.0, lam=lam, row_loss=r)
    assert out["empty"][:B].all() and not out["empty"][B:].any()
    np.testing.assert_array_equal(out["p_cache"], 0.0)
    np.testing.assert_array_equal(out["row_loss"][:B], r[:B])                 # C_t empty: p = p_model
    np.testing.assert_allclose(out["row_loss"][B:], 3.0 - np.log1p(-lam), rtol=1e-15)   # p = (1 - lam) p_model


def test_log_add_exp_form_needs_no_exp_of_the_row_loss():
    r = np.array([2000.0, 1.0])                       # p_model = exp(-2000) underflows float64
    got = mix_row_loss(r, np.array([0.5, 0.5]), np.array([False, False]), 0.1)
    assert np.isfinite(got).all()
    assert got[0] == pytest.approx(-np.log(0.1 * 0.5), rel=1e-12)
    assert got[1] == pytest.approx(-np.log(0.9 * np.exp(-1.0) + 0.05), rel=1e-12)


def test_entry_points_are_declared_and_bound():
    from zaremba_b200 import _lib
    names = set(_lib.exported_symbols())
    assert {"zrb_cache_create", "zrb_cache_reset", "zrb_cache_destroy", "zrb_cache_step",
            "zrb_eval_step_cache"} <= names
    import zaremba_b200
    assert zaremba_b200.NeuralCache and zaremba_b200.cache_step
