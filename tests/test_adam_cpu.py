"""Adam in the fused train step (DESIGN.md section 21) without a GPU.

- The fp32 restatement (tests/_adam_oracle.py) and its fp64 twin against torch.optim.Adam (weight_decay=0,
  amsgrad=False, the single-tensor path), several steps with clip coefficients < 1.  fp64: the same values to 1e-12
  relative (torch's m is a lerp, the documented rule a sum of products).  fp32: torch rounds the lerp and its scalar
  products differently, and the C ABI takes the betas as fp32, so 1 - beta2 is 1 - fp32(0.999) = 0.000999987 where
  torch uses 0.001 (v then differs by 1.3e-5 relative).  The parameters agree to TOL_P32 of the largest |p|, m to
  1e-6 of the largest |m|, v to 2e-5 relative.
- The flat <-> torch.optim.Adam state-dict conversion of the Trainer, both directions.
- The C ABI: header prototype, ctypes binding, refusals that need no context; the Trainer's argument refusals.
"""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest
import torch

from tests import _adam_oracle as AO
from zaremba_b200.trainer import adam_state_from_torch, adam_state_to_torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL_P32 = 4e-7      # |p_restatement - p_torch| / max|p| over 6 fp32 steps (measured: at most 1.3e-7)


def _torch_run(dtype, seed, betas, eps, lr, coefs):
    """torch.optim.Adam over one tensor with gradients g_k * coef_k; returns the per-step (p, m, v) and the raw g."""
    g = torch.Generator().manual_seed(seed)
    p = torch.nn.Parameter(torch.randn(4096, generator=g, dtype=torch.float64).to(dtype))
    opt = torch.optim.Adam([p], lr=lr, betas=betas, eps=eps, weight_decay=0.0, amsgrad=False, foreach=False)
    p0 = p.detach().clone()
    grads, out = [], []
    for k, coef in enumerate(coefs):
        raw = (torch.randn(4096, generator=g, dtype=torch.float64) * (1.0 + k)).to(dtype)
        grads.append(raw.clone())
        p.grad = raw * torch.tensor(coef, dtype=dtype)
        opt.step()
        st = opt.state[p]
        out.append((p.detach().clone(), st["exp_avg"].clone(), st["exp_avg_sq"].clone()))
    return p0, grads, out


CASES = [((0.9, 0.999), 1e-8, 1e-3), ((0.0, 0.999), 1e-9, 2e-3), ((0.5, 0.99), 1e-6, 0.1)]


@pytest.mark.parametrize("betas,eps,lr", CASES)
def test_fp64_restatement_equals_torch_adam(betas, eps, lr):
    coefs = [1.0, 0.5, 0.25, 0.9, 1.0, 0.125]
    p0, grads, out = _torch_run(torch.float64, 0, betas, eps, lr, coefs)
    p, m, v = p0.numpy(), np.zeros(p0.shape), np.zeros(p0.shape)
    for t, (raw, coef, (tp, tm, tv)) in enumerate(zip(grads, coefs, out), start=1):
        p, _, m, v = AO.adam_fp64(p, raw.numpy(), m, v, coef, lr, betas[0], betas[1], eps, t)
        np.testing.assert_allclose(p, tp.numpy(), rtol=0, atol=1e-12 * np.abs(p).max())
        np.testing.assert_allclose(m, tm.numpy(), rtol=0, atol=1e-12 * np.abs(m).max())
        np.testing.assert_allclose(v, tv.numpy(), rtol=0, atol=1e-12 * np.abs(v).max())


@pytest.mark.parametrize("betas,eps,lr", CASES)
def test_fp32_restatement_tracks_torch_adam(betas, eps, lr):
    coefs = [1.0, 0.5, 0.25, 0.9, 1.0, 0.125]
    p0, grads, out = _torch_run(torch.float32, 1, betas, eps, lr, coefs)
    p, m, v = p0.numpy(), np.zeros(p0.shape, np.float32), np.zeros(p0.shape, np.float32)
    for t, (raw, coef, (tp, tm, tv)) in enumerate(zip(grads, coefs, out), start=1):
        # torch clips in place: its .grad is the fp32 product raw * coef, the kernels' g'
        p, gs, m, v = AO.adam_fp32(p, raw.numpy(), m, v, coef, lr, betas[0], betas[1], eps, t)
        assert gs.tobytes() == (raw * torch.tensor(coef)).numpy().tobytes()
        assert np.abs(p - tp.numpy()).max() <= TOL_P32 * np.abs(p).max(), t
        assert np.abs(m - tm.numpy()).max() <= 1e-6 * np.abs(m).max(), t
        np.testing.assert_allclose(v, tv.numpy(), rtol=2e-5, atol=0)


def test_scalars_are_rounded_once_from_double():
    for t in (1, 2, 10, 1000, 10 ** 6):
        b1, b2, omb1, omb2, eps, step_size, bc2s = AO.scalars(1e-3, 0.9, 0.999, 1e-8, t)
        B1, B2 = float(np.float32(0.9)), float(np.float32(0.999))
        assert (b1, b2, eps) == (np.float32(0.9), np.float32(0.999), np.float32(1e-8))
        assert omb1 == np.float32(1.0 - B1) and omb2 == np.float32(1.0 - B2)
        assert step_size == np.float32(float(np.float32(1e-3)) / (1.0 - B1 ** t))
        assert bc2s == np.float32(math.sqrt(1.0 - B2 ** t))


def test_restatement_order_is_the_documented_one():
    """One element worked by hand in the documented order, each product and sum rounded on its own."""
    f = np.float32
    p, g, m, v, coef = f(0.75), f(3.0), f(0.125), f(0.5), f(0.5)
    b1, b2, omb1, omb2, eps, step_size, bc2s = AO.scalars(0.01, 0.9, 0.999, 1e-8, 3)
    gs = f(g * coef)
    m1 = f(f(b1 * m) + f(omb1 * gs))
    v1 = f(f(b2 * v) + f(omb2 * f(gs * gs)))
    d = f(f(np.sqrt(v1) / bc2s) + eps)
    p1 = f(p - f(step_size * f(m1 / d)))
    out = AO.adam_fp32(np.array([p]), np.array([g]), np.array([m]), np.array([v]), coef, 0.01, 0.9, 0.999, 1e-8, 3)
    assert [o[0] for o in out] == [p1, gs, m1, v1]


# ---- the state-dict conversion --------------------------------------------------------------------------------------
def _layout(shapes):
    out, off = [], 0
    for i, s in enumerate(shapes):
        out.append((i, s, off))
        off += math.prod(s)
    return out, off


def test_state_dict_round_trip_through_torch_adam():
    """flat moments -> torch format -> loaded into a torch.optim.Adam -> its state_dict() -> flat again: bit for bit,
    and the torch optimiser steps on from the same t."""
    shapes = [(7, 3), (12,), (5, 4, 2)]
    layout, n = _layout(shapes)
    g = torch.Generator().manual_seed(3)
    flat_m, flat_v = torch.randn(n, generator=g), torch.rand(n, generator=g)
    sd = adam_state_to_torch(flat_m, flat_v, 5, layout, 0.002, (0.0, 0.999), 1e-9)
    params = [torch.nn.Parameter(torch.randn(s, generator=g)) for s in shapes]
    opt = torch.optim.Adam(params, lr=1.0)
    opt.load_state_dict(sd)
    assert opt.param_groups[0]["lr"] == 0.002 and opt.param_groups[0]["betas"] == (0.0, 0.999)
    assert opt.param_groups[0]["eps"] == 1e-9
    back_m, back_v = torch.full((n,), float("nan")), torch.full((n,), float("nan"))
    step, betas, eps, lr = adam_state_from_torch(opt.state_dict(), layout, back_m, back_v)
    assert (step, betas, eps, lr) == (5, (0.0, 0.999), 1e-9, 0.002)
    assert torch.equal(back_m, flat_m) and torch.equal(back_v, flat_v)
    for p in params:
        p.grad = torch.ones_like(p)
    opt.step()
    assert all(float(opt.state[p]["step"]) == 6.0 for p in params)


def test_state_dict_of_a_fresh_optimizer():
    layout, n = _layout([(4,), (2, 2)])
    sd = adam_state_to_torch(torch.zeros(n), torch.zeros(n), 0, layout, 1e-3, (0.9, 0.999), 1e-8)
    assert sd["state"] == {}
    params = [torch.nn.Parameter(torch.zeros(s)) for _, s, _ in layout]
    fresh = torch.optim.Adam(params).state_dict()
    m, v = torch.ones(n), torch.ones(n)
    assert adam_state_from_torch(fresh, layout, m, v)[0] == 0
    assert not m.any() and not v.any()


@pytest.mark.parametrize("change,match", [
    (lambda sd: sd["param_groups"][0].update(weight_decay=0.1), "weight_decay"),
    (lambda sd: sd["param_groups"][0].update(amsgrad=True), "amsgrad"),
    (lambda sd: sd["param_groups"][0].update(betas=(1.0, 0.999)), "beta1"),
    (lambda sd: sd["param_groups"][0].update(eps=0.0), "eps"),
    (lambda sd: sd["param_groups"][0].update(params=[1, 0]), "param group"),
    (lambda sd: sd["state"][1].update(step=torch.tensor(4.0)), "common step"),
    (lambda sd: sd["state"].pop(0), "common step"),
    (lambda sd: sd["state"][0].update(exp_avg=torch.zeros(3)), "shape"),
])
def test_state_dict_refusals(change, match):
    layout, n = _layout([(4,), (2, 2)])
    sd = adam_state_to_torch(torch.ones(n), torch.ones(n), 3, layout, 1e-3, (0.9, 0.999), 1e-8)
    change(sd)
    with pytest.raises(ValueError, match=match):
        adam_state_from_torch(sd, layout, torch.zeros(n), torch.zeros(n))


# ---- C ABI and the Trainer's arguments ------------------------------------------------------------------------------
def test_header_and_binding():
    from zaremba_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "zaremba_b200.h")).read()
    assert re.search(r"int\s+zrb_set_adam\(zrb_ctx\* ctx, const zrb_params\* m, const zrb_params\* v, float beta1, "
                     r"float beta2, float eps,\s+int64_t step\);", hdr)
    P = C.POINTER(_lib.ZrbParams)
    assert _lib._SIGNATURES["zrb_set_adam"] == (C.c_int, [C.c_void_p, P, P, C.c_float, C.c_float, C.c_float,
                                                          C.c_int64])
    import zaremba_b200
    for m in ("optimizer_state_dict", "load_optimizer_state_dict"):
        assert callable(getattr(zaremba_b200.Trainer, m)), m


def test_null_context_is_refused():
    from zaremba_b200 import _lib
    try:
        lib = _lib.load()
    except Exception as e:   # no library and no nvcc: nothing to call
        pytest.skip(f"library unavailable: {e}")
    ps = _lib.ZrbParams()
    assert lib.zrb_set_adam(None, C.byref(ps), C.byref(ps), 0.9, 0.999, 1e-8, 0) == -1
    assert lib.zrb_set_adam(None, None, None, 0.9, 0.999, 1e-8, 0) == -1


@pytest.mark.parametrize("kw,match", [
    ({"optimizer": "adamw"}, "optimizer"),
    ({"optimizer": "adam", "betas": (0.9, 1.0)}, "beta2"),
    ({"optimizer": "adam", "betas": (-0.1, 0.999)}, "beta1"),
    ({"optimizer": "adam", "betas": (float("nan"), 0.999)}, "beta1"),
    ({"optimizer": "adam", "eps": 0.0}, "eps"),
    ({"optimizer": "adam", "eps": float("inf")}, "eps"),
    ({"optimizer": "adam", "betas": (0.9,)}, "betas"),
])
def test_trainer_refuses_bad_arguments_before_touching_a_device(kw, match):
    import zaremba_b200
    m = zaremba_b200.Model(10, 8, 1, 0.0, 0.1)
    with pytest.raises(ValueError, match=match):
        zaremba_b200.Trainer(m, 2, 3, **kw)
