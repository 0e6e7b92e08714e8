"""The fused weight update's image rebuild at the Large and Small shapes, compared bit for bit with a fresh pack.

tests/test_gpu_parity.py::test_fused_update_rebuilds_what_a_fresh_pack_builds covers every plan branch at small H.
The update kernels (optim_tc.cu) map their grid straight onto 8-row tiles, so the shapes of the train-step configs
reach cases those H do not: H = 1500 (the Large plan: K-split forward pairs, 8-CTA backward clusters, a last tile of
4 rows since H % 8 = 4, column tiles that end inside a warp) and H = 200 (Small: the unsplit forward plan).  Each case
runs three clipped, dropout'ed train steps on the strict or the lazy schedule, with clipped gradients kept or not (the
kernels' write-back of coef * g), and then checks that the trained context computes exactly what a fresh context
packed from the same fp32 weights computes: eval loss, target probabilities and states, and one gradient pass.
"""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

V, L, T, LR, MAX_NORM = 256, 2, 5, 1.0, 0.05


def _dev():
    return torch.device("cuda:0")


def _plan_reached(plans, case):
    fp, bp = plans["fwd"], plans["bwd"]
    if case == "large":
        return fp["ok"] and fp["KS"] == 2 and bp["ok"] and bp["KS"] == 2   # backward clusters of 4 * KS = 8 CTAs
    return fp["ok"] and fp["KS"] == 1 and bp["ok"]


@pytest.mark.parametrize("keep", [False, True], ids=["drop_clipped", "keep_clipped"])
@pytest.mark.parametrize("lazy", [False, True], ids=["strict", "lazy"])
@pytest.mark.parametrize("H,case", [(1500, "large"), (200, "small")])
def test_update_images_equal_a_fresh_pack(H, case, lazy, keep):
    import zaremba_b200
    from zaremba_b200 import _lib
    lib = _lib.load()
    B = 20
    torch.manual_seed(H + int(lazy) + 2 * int(keep))
    m1 = zaremba_b200.Model(V, H, L, 0.3, 0.1).to(_dev())
    m1.train()
    tr1 = zaremba_b200.Trainer(m1, B, T, lazy_update=lazy, keep_clipped_grads=keep)
    plans = _lib.rec_plans(tr1.ctx)
    if not _plan_reached(plans, case):
        pytest.skip(f"H={H} B={B} gets plans {plans} on this device, not the {case} ones")
    g = torch.Generator().manual_seed(3)
    data = torch.randint(0, V, (B, 3 * T + 1), generator=g)
    for s in range(3):
        x = data[:, s * T:(s + 1) * T].t().contiguous().to(_dev())
        y = data[:, s * T + 1:(s + 1) * T + 1].t().contiguous().to(_dev())
        _, norm = tr1.train_step(x, y, LR, MAX_NORM)
        assert norm.item() > 2 * MAX_NORM, "the clip must be active"
    tr1.flush()
    torch.cuda.synchronize()
    if keep:   # the kept gradients are the clipped ones: their norm is max_norm (up to fp32 rounding)
        kept = tr1.flat_g.double().norm().item()
        assert abs(kept - MAX_NORM) < 1e-4 * MAX_NORM, (kept, MAX_NORM)

    m2 = zaremba_b200.Model(V, H, L, 0.3, 0.1).to(_dev())
    with torch.no_grad():
        for p2, p1 in zip(m2.ordered_parameters(), m1.ordered_parameters()):
            p2.copy_(p1)
    m2.train()
    tr2 = zaremba_b200.Trainer(m2, B, T, lazy_update=lazy)
    for (h1, c1), (h2, c2) in zip(tr1.states, tr2.states):
        h2.copy_(h1)
        c2.copy_(c1)
    assert torch.equal(tr1.flat_p, tr2.flat_p)

    perm = torch.randperm(V, generator=g)[:T * B]          # distinct tokens: no colliding atomics in the scatter
    x = perm.view(T, B).contiguous().to(_dev())
    y = torch.randint(0, V, (T, B), generator=g).to(_dev())
    out = []
    pack = _lib.PROF_CLASSES.index("pack")
    for tr in (tr1, tr2):
        _lib.check(lib.zrb_prof_enable(tr.ctx, 1))
        loss, tp = tr.eval_step(x, y, want_probs=True)
        ev = (loss.clone(), tp.clone(), [t.clone() for st in tr.states for t in st])
        gl = torch.zeros((), device=_dev())
        _lib.check(lib.zrb_train_step_grads(tr.ctx, C.byref(tr._ps), C.byref(tr._gs), _lib.ptr(x), _lib.ptr(y), T, B,
                                            C.byref(tr._st), C.byref(tr._st), 7, 1000, _lib.ptr(gl), tr._stream()))
        ms, counts = (C.c_float * len(_lib.PROF_CLASSES))(), (C.c_int64 * len(_lib.PROF_CLASSES))()
        _lib.check(lib.zrb_prof_read(tr.ctx, ms, counts))
        _lib.check(lib.zrb_prof_enable(tr.ctx, 0))
        out.append((ev, gl, tr.flat_g.clone(), [t.clone() for st in tr.states for t in st], counts[pack]))
    (ev1, gl1, g1, st1, packs1), (ev2, gl2, g2, st2, packs2) = out
    assert packs1 == 0, "the trained context repacked its weights: the comparison would be vacuous"
    assert packs2 >= 1, "the fresh context must have packed (profiling sanity)"
    assert torch.equal(ev1[0], ev2[0]), (ev1[0].item(), ev2[0].item())
    assert torch.equal(ev1[1], ev2[1]), "eval target probabilities differ"
    for a, b in zip(ev1[2], ev2[2]):
        assert torch.equal(a, b), "eval states differ"
    assert torch.equal(gl1, gl2), (gl1.item(), gl2.item())
    for a, b in zip(st1, st2):
        assert torch.equal(a, b), "train-step states differ"
    if not torch.equal(g1, g2):
        sizes = [p.numel() for p in m1.ordered_parameters()]
        names = ["embed"] + [f"{k}{l}" for l in range(L) for k in ("w_ih", "w_hh", "b_ih", "b_hh")] + ["fc_w", "fc_b"]
        bad = [n for n, a, b in zip(names, g1.split(sizes), g2.split(sizes)) if not torch.equal(a, b)]
        raise AssertionError(f"gradients differ in {bad}")
