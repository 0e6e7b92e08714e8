"""The rounded-operand restatement (tests/_rounded_oracle.py) that tests/test_gpu_rec_bwd_images.py holds the
recurrence kernels to, checked without a GPU: against the exact fp64 oracle, its magnitudes, its mutations, and the
exactness the GPU test's probe relies on."""
import numpy as np
import pytest
import torch

from oracle import lstm_lm_oracle as O
from tests import _rounded_oracle as RO


def _layer_data(H, T, B, seed, w=0.3):
    rng = np.random.default_rng(seed)
    W_ih, W_hh = rng.uniform(-w, w, size=(4 * H, H)), rng.uniform(-w, w, size=(4 * H, H))
    b_ih, b_hh = rng.uniform(-w, w, size=4 * H), rng.uniform(-w, w, size=4 * H)
    x = rng.normal(size=(T, B, H))
    h0, c0 = rng.uniform(-0.5, 0.5, size=(B, H)), rng.uniform(-1.0, 1.0, size=(B, H))
    dy = rng.normal(size=(T, B, H)) * 0.1
    return dict(x=x, h0=h0, c0=c0, W_ih=W_ih, W_hh=W_hh, b_ih=b_ih, b_hh=b_hh, dy=dy)


@pytest.mark.parametrize("H,T,B", [(8, 1, 1), (12, 5, 3), (24, 9, 10)])
def test_unrounded_restatement_is_the_exact_oracle(H, T, B):
    """Without rounding, forward and backward forced on their own exact values equal O.lstm_layer_fwd / _bwd."""
    d = _layer_data(H, T, B, H + T)
    t = {k: torch.tensor(v) for k, v in d.items()}
    fw, dG, E, dx, dWi, dWh, db = RO.layer(t["x"], t["h0"], t["c0"], t["W_ih"], t["W_hh"], t["b_ih"], t["b_hh"],
                                           t["dy"], rounded=False)
    ys, _, cT, cache = O.lstm_layer_fwd(d["x"], d["h0"], d["c0"], d["W_ih"], d["W_hh"], d["b_ih"], d["b_hh"])
    rec = {}
    want = O.lstm_layer_bwd(d["dy"], cache, d["x"], d["W_ih"], d["W_hh"], record=rec)
    close = lambda a, b: np.testing.assert_allclose(np.asarray(a), b, rtol=1e-12, atol=1e-12 * np.abs(b).max())
    close(torch.stack(fw["h"]), ys)
    close(fw["c"][-1].v, cT)
    close(dG, rec["dG"])
    for got, w in zip((dx, dWi, dWh, db), want):
        close(got, w)
    assert (E >= dG.abs()).all()


@pytest.mark.parametrize("H,T,B", [(12, 5, 3), (24, 9, 10)])
def test_rounded_restatement_within_its_magnitude_bound(H, T, B):
    """With fp16 operands and fp16 dG images (forced on its own images) the restatement departs from the exact one by
    fp16 rounding: at most a few units of 2^-11 times the magnitude E, element by element."""
    d = {k: torch.tensor(v) for k, v in _layer_data(H, T, B, 3 * H + T).items()}
    args = [d[k] for k in ("x", "h0", "c0", "W_ih", "W_hh", "b_ih", "b_hh", "dy")]
    _, dG_r, E, *_ = RO.layer(*args, rounded=True)
    _, dG_x, _, *_ = RO.layer(*args, rounded=False)
    ratio = float(((dG_r - dG_x).abs() / E).max())
    assert 0.0 < ratio <= 8 * 2.0 ** -11, ratio


def test_teacher_forced_backward_and_mutations():
    """Forced on images it made itself, the backward gives back its own images; each mutation of the kernel's kind
    moves the result."""
    H, T, B = 16, 6, 10
    d = {k: torch.tensor(v) for k, v in _layer_data(H, T, B, 5).items()}
    fw, dG, E, *_ = RO.layer(*[d[k] for k in ("x", "h0", "c0", "W_ih", "W_hh", "b_ih", "b_hh", "dy")])
    img = RO.image(dG)
    Wr = RO.r16(d["W_hh"])
    again, _ = RO.backward(fw, d["dy"], Wr, d["c0"], img=img)
    assert torch.equal(RO.image(again), img)
    geometry = (torch.arange(H), torch.arange(H - 4, H))
    q = torch.tensor(np.random.default_rng(1).integers(0, 2, size=(B, H)) * 2.0)
    zh = torch.tensor(np.random.default_rng(2).random((T, B, H)) < 0.5)
    for mut in RO.MUTATIONS:
        kw = dict(q=q) if mut == "multiplier_on_dy" else dict(zh=zh) if mut == "drop_hcarry" else {}
        ref, _ = RO.backward(fw, d["dy"], Wr, d["c0"], img=img, **kw)
        if mut == "flush_subnormal":
            img_s = img.clone()
            img_s[2, 0, :4] = 2.0 ** -20
            ref, _ = RO.backward(fw, d["dy"], Wr, d["c0"], img=img_s)
            got, _ = RO.backward(fw, d["dy"], Wr, d["c0"], img=img_s, mutate=mut, geometry=geometry)
        else:
            got, _ = RO.backward(fw, d["dy"], Wr, d["c0"], img=img, mutate=mut, geometry=geometry, **kw)
        # (a flushed subnormal image moves its products by about 2^-30: the GPU test resolves that against its bound)
        floor = 0.0 if mut == "flush_subnormal" else 1e-3 * float(ref.abs().max())
        assert (got - ref).abs().max() > floor, mut


def test_probe_is_exact_for_every_fp16_value():
    """The GPU test reads each dG image through dE = (img * 1 * 2^-10) * 2 (identity W_ih, then the site-0 multiplier
    2) and passes dy in as dS = img * 2^-10 times the site-L multiplier 2: every finite fp16 value survives both in
    fp32 and comes back unchanged."""
    bits = np.arange(0, 2 ** 16, dtype=np.uint32).astype(np.uint16)
    v = bits.view(np.float16)
    v = v[np.isfinite(v)].astype(np.float32)
    dx = (v * np.float32(1.0)) * np.float32(2.0 ** -10)
    dE = dx * np.float32(2.0)
    back = np.float32(1024.0) * dE / np.float32(2.0)
    assert np.array_equal(back, v)
    assert np.array_equal(back.astype(np.float16).astype(np.float32), v)
    assert np.array_equal((dx * np.float32(2.0)).astype(np.float64), v.astype(np.float64) * 2.0 ** -9)


def test_rescaled_images_bracket_the_true_image():
    """rescale_image: from y = r(h) the image r(2h), and from y = r(2h) the image r(h), to within the stated
    uncertainty, and exactly where it states none; tiny and subnormal h included."""
    rng = np.random.default_rng(0)
    h = np.concatenate([rng.normal(size=20000) * 10.0 ** rng.uniform(-9, 0, size=20000),
                        np.arange(-300, 300) * 2.0 ** -26]).astype(np.float32).astype(np.float64)
    h = torch.tensor(h)
    for k, y, want in ((2, RO.r16(h), RO.r16(2 * h)), (0.5, RO.r16(2 * h), RO.r16(h))):
        best, amb = RO.rescale_image(y, k)
        assert ((want - best).abs() <= amb).all(), k
        assert torch.equal(want[amb == 0], best[amb == 0]), k
        assert (amb > 0).any() and (amb == 0).any(), k
