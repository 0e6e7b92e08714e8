"""GPU tests of the neural-cache evaluation (zrb_cache_step, zrb_eval_step_cache, Trainer.perplexity(cache=)).

  * the attend kernel alone (zrb_cache_step) against the float64 restatement fed the same fp16 keys, over H, B and W,
    over calls that wrap the ring, with duplicated tokens, exact-tie logits and temperatures where one key dominates;
  * lambda = 0 against zrb_eval_step bit for bit, lambda > 0 against the fp64 model plus the restatement over carried
    windows, on both engines;
  * reproducibility, a lazy-update Trainer, rejected arguments and the launch count.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import lstm_lm_oracle as O
from tests._neural_cache_oracle import NeuralCache as CacheOracle
from tests.test_gpu_parity import ENGINES, TOL

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
# Largest |p_cache - oracle| of zrb_cache_step over test_cache_step_against_oracle, fp32 accumulation of fp16 products
# against float64: 8.8e-5 (H = 1500, B = 20, W = 2000, at the temperatures where one key dominates; H100 80GB HBM3,
# 400 W power limit).  Held at about 3x (DESIGN.md sections 5 and 12).
P_TOL = 2.5e-4


def _bits(t):
    return t.detach().contiguous().view(torch.int32).cpu().numpy()


def _keys(T, B, H, rng, kind):
    """Last-layer-like outputs (|h| < 1); `ties` repeats rows so that logits tie exactly."""
    h = np.tanh(rng.normal(size=(T, B, H)) * 0.8).astype(np.float32)
    if kind == "ties":
        h[1::3] = h[0:T - 1:3][: len(h[1::3])]
    return h


CASES = [  # (H, B, W, T, calls): every H, B and W of the issue; the last calls wrap the ring (cap = W + T rounded to 64)
    (40, 1, 1, 7, 12),
    (40, 20, 35, 35, 6),
    (200, 40, 500, 35, 20),
    (200, 1, 2000, 64, 40),
    (650, 20, 35, 35, 5),
    (650, 1, 500, 35, 20),
    (1500, 20, 2000, 100, 24),
    (1500, 40, 35, 35, 4),
    (1500, 1, 1, 3, 5),
]


@pytest.mark.parametrize("H,B,W,T,calls", CASES)
def test_cache_step_against_oracle(H, B, W, T, calls):
    import zaremba_b200
    rng = np.random.default_rng(H * 7 + B * 3 + W)
    cache = zaremba_b200.NeuralCache(H, B, W, T)
    oracle = CacheOracle(W, B)
    worst = 0.0
    fed = 0
    for k in range(calls):
        Tk = T if k % 3 else max(1, T - 2)              # windows shorter than max_seq too
        kind = "ties" if k % 2 else "plain"
        h = _keys(Tk, B, H, rng, kind)
        y = rng.integers(0, 4 if k % 2 else 50, size=(Tk, B))   # few distinct tokens: many duplicates
        theta = [0.0, 0.3, 3.0, 40.0][k % 4] * 8.0 / np.sqrt(H)   # up to one key dominating
        got = zaremba_b200.cache_step(cache, torch.from_numpy(h), torch.from_numpy(y), theta).cpu().numpy()
        fed += Tk
        check = fed > W + T or k < 2 or k == calls - 1            # every call once the ring has wrapped
        want = oracle.step(h, y, theta, compute=check)
        if not check:
            continue
        err = np.abs(got.astype(np.float64) - want["p_cache"]).max()
        worst = max(worst, err)
        assert err <= P_TOL, f"call {k} theta {theta}: |p_cache - oracle| = {err}"
        assert (got[want["empty"]] == 0).all()
    assert fed > W + T or W > 500, "the ring never wrapped"
    print(f"H={H} B={B} W={W}: worst |p_cache - oracle| {worst:.3g}")


def test_cache_step_is_bit_reproducible_and_reset_forgets():
    import zaremba_b200
    rng = np.random.default_rng(0)
    H, B, W, T = 650, 20, 500, 35
    hs = [torch.from_numpy(_keys(T, B, H, rng, "ties")) for _ in range(4)]
    ys = [torch.from_numpy(rng.integers(0, 20, size=(T, B))) for _ in range(4)]
    cache = zaremba_b200.NeuralCache(H, B, W, T)
    runs = []
    for _ in range(2):
        cache.reset()
        runs.append([_bits(zaremba_b200.cache_step(cache, h, y, 1.5)) for h, y in zip(hs, ys)])
    for a, b in zip(*runs):
        assert np.array_equal(a, b)


def _model(engine, V=300, H=200, L=2, seed=0):
    import zaremba_b200
    torch.manual_seed(seed)
    return zaremba_b200.Model(V, H, L, 0.0, 1.3 / np.sqrt(H), engine=engine).to(DEV)


def _windows(V, T, B, n, seed):
    rng = np.random.default_rng(seed)
    data = rng.integers(0, V // 6, size=(n * T + 1) * B)      # a small working vocabulary: the cache has something to find
    data = data.reshape(B, -1)
    return [(torch.from_numpy(data[:, i * T:(i + 1) * T].T.copy()).to(DEV),
             torch.from_numpy(data[:, i * T + 1:(i + 1) * T + 1].T.copy()).to(DEV)) for i in range(n)]


@pytest.mark.parametrize("engine", ENGINES)
def test_lambda_zero_is_eval_step_bit_for_bit(engine):
    import zaremba_b200
    T, B = 35, 20
    m = _model(engine)
    tr = zaremba_b200.Trainer(m, B, T)
    cache = zaremba_b200.NeuralCache(200, B, 100, T)
    wins = _windows(300, T, B, 4, 1)
    plain = []
    tr.reset_states()
    for x, y in wins:
        loss, p = tr.eval_step(x, y, want_probs=True)
        plain.append((_bits(loss.reshape(1)), _bits(p)))
    tr.reset_states()
    cache.reset()
    for (x, y), (lb, pb) in zip(wins, plain):
        loss, p, pc = tr.eval_step(x, y, want_probs=True, cache=cache, theta=1.0, lam=0.0)
        assert np.array_equal(_bits(loss.reshape(1)), lb)
        assert np.array_equal(_bits(p), pb)
    assert tr.perplexity([(x.cpu(), y.cpu()) for x, y in wins], cache=cache, theta=1.0, lam=0.0) == \
        tr.perplexity([(x.cpu(), y.cpu()) for x, y in wins])


@pytest.mark.parametrize("engine", ENGINES)
def test_lambda_positive_against_fp64_oracle(engine):
    import zaremba_b200
    V, H, L, T, B, W, theta, lam = 300, 200, 2, 35, 20, 50, 2.0, 0.3
    m = _model(engine, V, H, L)
    params = {k: v.detach().cpu().numpy().astype(np.float64) for k, v in m.named_parameters()}
    tr = zaremba_b200.Trainer(m, B, T)
    cache = zaremba_b200.NeuralCache(H, B, W, T)
    oracle = CacheOracle(W, B)
    states = O.zero_states(L, B, H, dtype=np.float64)
    tol = TOL[engine]
    tr.reset_states()
    for x, y in _windows(V, T, B, 4, 2):
        loss, p, pc = tr.eval_step(x, y, want_probs=True, cache=cache, theta=theta, lam=lam)
        scores, states, fc = O.model_fwd(params, x.cpu().numpy(), states, L)
        pm = O.target_probs(scores, y.cpu().numpy())
        want = oracle.step(fc["fc_in"], y.cpu().numpy(), theta, lam, -np.log(pm))
        assert abs(loss.item() - want["loss"]) <= tol["loss"] * abs(want["loss"]), (loss.item(), want["loss"])
        np.testing.assert_allclose(p.cpu().numpy(), pm, rtol=tol["fwd"] * 10, atol=1e-7)
        np.testing.assert_allclose(pc.cpu().numpy(), want["p_cache"], atol=tol["fwd"] * 10)
    assert want["p_cache"].mean() > 0.01     # the cache found something


def test_lazy_update_trainer_equals_flushed():
    import zaremba_b200
    T, B = 35, 20
    out = []
    for flush in (False, True):
        m = _model("tc", seed=4)
        tr = zaremba_b200.Trainer(m, B, T, lazy_update=True)
        wins = _windows(300, T, B, 3, 3)
        tr.train_step(wins[0][0], wins[0][1], 1.0, 5.0)
        if flush:
            tr.flush()
        cache = zaremba_b200.NeuralCache(200, B, 100, T)
        tr.reset_states()
        res = [[_bits(t.reshape(-1)) for t in tr.eval_step(x, y, want_probs=True, cache=cache, theta=1.0, lam=0.2)]
               for x, y in wins[1:]]
        out.append(res)
    for a, b in zip(*out):
        for u, v in zip(a, b):
            assert np.array_equal(u, v)


def test_rejected_arguments_leave_the_handle_unchanged():
    import zaremba_b200
    from zaremba_b200 import _lib
    lib = _lib.load()
    T, B, H, W = 35, 20, 200, 100
    h_out = C.c_void_p()
    for args in ((0, B, W, T), (1537, B, W, T), (H, 0, W, T), (H, B, 0, T), (H, B, W, 0)):
        assert lib.zrb_cache_create(*args, C.byref(h_out)) == -1
    m = _model("tc")
    tr = zaremba_b200.Trainer(m, B, T)
    wins = _windows(300, T, B, 3, 5)
    ref = zaremba_b200.NeuralCache(H, B, W, T)
    want = [[_bits(t.reshape(-1)) for t in tr.eval_step(x, y, want_probs=True, cache=ref, theta=1.0, lam=0.2)]
            for x, y in wins]
    cache = zaremba_b200.NeuralCache(H, B, W, T)
    other = zaremba_b200.NeuralCache(H + 8, B, W, T)
    tr.reset_states()
    x, y = wins[0]
    st = torch.cuda.current_stream().cuda_stream
    loss = torch.zeros((), device=DEV)
    bad = [(cache.handle, -1.0, 0.2, x, y), (cache.handle, float("inf"), 0.2, x, y), (cache.handle, float("nan"), 0.2, x, y),
           (cache.handle, 1.0, -0.1, x, y), (cache.handle, 1.0, 1.0, x, y), (other.handle, 1.0, 0.2, x, y),
           (cache.handle, 1.0, 0.2, x[:, :B - 1].contiguous(), y[:, :B - 1].contiguous())]
    for hdl, th, lam, xx, yy in bad:
        rc = lib.zrb_eval_step_cache(tr.ctx, C.byref(tr._ps), _lib.ptr(xx), _lib.ptr(yy), xx.shape[0], xx.shape[1],
                                     C.byref(tr._st), C.byref(tr._st), hdl, th, lam, _lib.ptr(loss), None, None, st)
        assert rc == -1, (th, lam)
    small = zaremba_b200.NeuralCache(H, B, W, 10)
    rc = lib.zrb_eval_step_cache(tr.ctx, C.byref(tr._ps), _lib.ptr(x), _lib.ptr(y), T, B, C.byref(tr._st),
                                 C.byref(tr._st), small.handle, 1.0, 0.2, _lib.ptr(loss), None, None, st)
    assert rc == -1
    hs = torch.zeros(T, B, H, device=DEV)
    out = torch.zeros(T * B, device=DEV)
    for th, bb in ((-1.0, B), (float("nan"), B), (1.0, B + 1)):
        assert lib.zrb_cache_step(cache.handle, _lib.ptr(hs), _lib.ptr(y), T, bb, th, _lib.ptr(out), st) == -1
    assert lib.zrb_cache_step(cache.handle, _lib.ptr(hs), _lib.ptr(y), T + 1, B, 1.0, _lib.ptr(out), st) == -1
    tr.reset_states()
    got = [[_bits(t.reshape(-1)) for t in tr.eval_step(xx, yy, want_probs=True, cache=cache, theta=1.0, lam=0.2)]
           for xx, yy in wins]
    for g, w in zip(got, want):
        for u, v in zip(g, w):
            assert np.array_equal(u, v)
    with pytest.raises(ValueError):
        zaremba_b200.cache_step(cache, hs, y, -1.0)


@pytest.mark.parametrize("engine", ENGINES)
def test_launch_count(engine):
    import zaremba_b200
    from zaremba_b200 import _lib
    lib = _lib.load()
    T, B = 35, 20
    m = _model(engine)
    tr = zaremba_b200.Trainer(m, B, T)
    cache = zaremba_b200.NeuralCache(200, B, 2000, T)
    x, y = _windows(300, T, B, 1, 6)[0]
    tr.eval_step(x, y)
    tr.eval_step(x, y, cache=cache, theta=1.0, lam=0.1)
    n0 = lib.zrb_launch_count()
    tr.eval_step(x, y)
    n1 = lib.zrb_launch_count()
    tr.eval_step(x, y, cache=cache, theta=1.0, lam=0.1)
    n2 = lib.zrb_launch_count()
    assert n2 - n1 <= (n1 - n0) + 3, (n1 - n0, n2 - n1)


def test_a_narrower_cache_created_later_leaves_a_wider_one_working():
    """The attend kernels' shared-memory limit is a device-wide attribute: a handle of small H created after one of
    large H must not lower it under the first."""
    import zaremba_b200
    rng = np.random.default_rng(9)
    T, B, W = 35, 20, 500
    wins = [(torch.from_numpy(_keys(T, B, 1500, rng, "plain")), torch.from_numpy(rng.integers(0, 30, size=(T, B))))
            for _ in range(3)]
    wide = zaremba_b200.NeuralCache(1500, B, W, T)
    want = [_bits(zaremba_b200.cache_step(wide, h, y, 0.2)) for h, y in wins]
    narrow = zaremba_b200.NeuralCache(40, B, W, T)
    zaremba_b200.cache_step(narrow, torch.from_numpy(_keys(T, B, 40, rng, "plain")), wins[0][1], 0.2)
    wide.reset()
    for (h, y), w in zip(wins, want):
        assert np.array_equal(_bits(zaremba_b200.cache_step(wide, h, y, 0.2)), w)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs a second GPU")
def test_a_cache_is_refused_on_another_device():
    import zaremba_b200
    from zaremba_b200 import _lib
    lib = _lib.load()
    T, B, H = 35, 4, 64
    cache = zaremba_b200.NeuralCache(H, B, 100, T, device="cuda:1")
    h = torch.zeros(T, B, H, device=DEV)
    y = torch.zeros(T, B, dtype=torch.int64, device=DEV)
    out = torch.zeros(T * B, device=DEV)
    with torch.cuda.device(0):
        assert lib.zrb_cache_step(cache.handle, _lib.ptr(h), _lib.ptr(y), T, B, 1.0, _lib.ptr(out), None) == -1
        assert b"device" in lib.zrb_last_error()


def test_cache_eval_reads_custom_layout_checkpoints(tmp_path):
    """tools/cache_eval.py on a custom-layout checkpoint and on the same weights saved in the pytorch layout."""
    import json
    import os
    import subprocess
    import sys
    import zaremba_b200
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    torch.manual_seed(0)
    custom = zaremba_b200.Model(10000, 64, 2, 0.0, 0.1, "custom")
    plain = zaremba_b200.Model(10000, 64, 2, 0.0, 0.1)
    with torch.no_grad():
        for p, w in zip(plain.ordered_parameters(), custom._lib_weights()):
            p.copy_(w)
    res = []
    for name, m in (("custom", custom), ("pytorch", plain)):
        ck, js = tmp_path / f"{name}.pt", tmp_path / f"{name}.json"
        torch.save(m.state_dict(), ck)
        subprocess.run([sys.executable, os.path.join(root, "tools", "cache_eval.py"), str(ck), "--size", "50",
                        "--thetas", "0.5", "--lambdas", "0.1", "--json", str(js)], check=True, cwd=root,
                       stdout=subprocess.DEVNULL)
        res.append(json.load(open(js)))
    assert res[0]["layers"] == 2
    assert res[0]["no_cache"] == res[1]["no_cache"] and res[0]["cache"] == res[1]["cache"]
