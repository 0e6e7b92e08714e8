"""The GEMM's default epilogue (staggered consumer warpgroups, paired stores, the 132-SM tile plan) against
ZRB_GEMM_EPI=direct (lockstep warpgroups, one store per element, the earlier plan): outputs must be BIT-IDENTICAL.

  * every zrb_gemm_f16 call shape of the Small / Medium / Large train steps (input GEMM with bias, projection with
    bias, the dgrads with split-K, the weight gradients), plus the odd shapes and ldc > N cases of test_gpu_gemm.py,
    poisoned as there: operand padding NaN, C NaN before a plain store, a sentinel in the ldc padding and the row after;
  * one fused Trainer step at Large from the same seeded weights and states, lazy update on (which reaches the modes
    zrb_gemm_f16 cannot: bias2, the dual weight-gradient launch with sum-of-squares slots, the programmatic-dependent
    launches), followed by a second step that runs on the rebuilt fp16 images and an eval pass: loss, clip norm,
    states, every parameter and gradient.

The switch is read at every launch, so both sides run in this one process.
"""
import gc
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

SENTINEL = 12345.0


def _steps_shapes():
    """(name, M, N, K, a_mn, b_mn, bias) of every zrb_gemm_f16-reachable GEMM of the three bench configurations."""
    out = []
    for cfg, H, T, B in (("small", 200, 20, 20), ("medium", 650, 35, 20), ("large", 1500, 35, 20)):
        V, Nt = 10000, T * B
        out += [
            (f"{cfg}-gemm_in", Nt, 4 * H, H, 0, 0, True),
            (f"{cfg}-proj_fwd", Nt, V, H, 0, 0, True),
            (f"{cfg}-proj_dgrad", Nt, H, V, 0, 1, False),
            (f"{cfg}-gemm_dx", Nt, H, 4 * H, 0, 1, False),
            (f"{cfg}-wgrad_fc", V, H, Nt, 1, 1, False),
            (f"{cfg}-wgrad_ih", 4 * H, H, Nt, 1, 1, False),
        ]
    return out


ODD = [(700, 1500, 6000, 0), (20, 6000, 1500, 0), (1, 1, 1500, 0), (1921, 1900, 100, 0), (2047, 1800, 8, 0),
       (1985, 2000, 1500, 16), (191, 200, 1500, 24), (64, 72, 100, 0), (65, 130, 1, 0), (1, 1, 8, 0),
       (127, 300, 1500, 8), (700, 6000, 1500, 0), (700, 6000, 1500, 8), (700, 6001, 1500, 0)]

CASES = [(n, M, N, K, a, b, bias, 0) for n, M, N, K, a, b, bias in _steps_shapes()]
CASES += [(f"odd-{M}x{N}x{K}-pad{p}-{a}{b}", M, N, K, a, b, i % 2 == 0, p)
          for i, (M, N, K, p) in enumerate(ODD) for a, b in ((0, 0), (1, 1), (0, 1))]


def _operand(logical, mn_major):
    rows, K = logical.shape
    inner, outer = (rows, K) if mn_major else (K, rows)
    ld = (inner + 7) // 8 * 8 + 8
    buf = torch.full((outer + 8, ld), float("nan"), dtype=torch.float16, device="cuda")
    buf[:outer, :inner] = logical.t() if mn_major else logical
    return buf, ld


def _run(lib, side, A, lda, a_mn, Bm, ldb, b_mn, M, N, K, ldc, alpha, bias, acc, C0=None):
    from zaremba_b200 import _lib
    c = torch.full((M + 1, ldc), SENTINEL, device="cuda")
    c[:M, :N] = float("nan") if C0 is None else C0
    old = os.environ.pop("ZRB_GEMM_EPI", None)
    try:
        if side == "direct":
            os.environ["ZRB_GEMM_EPI"] = "direct"
        _lib.check(lib.zrb_gemm_f16(_lib.ptr(A), lda, a_mn, _lib.ptr(Bm), ldb, b_mn, _lib.ptr(c), ldc, M, N, K, alpha,
                                    _lib.ptr(bias), acc, None))
        torch.cuda.synchronize()
    finally:
        os.environ.pop("ZRB_GEMM_EPI", None)
        if old is not None:
            os.environ["ZRB_GEMM_EPI"] = old
    return c


@pytest.mark.parametrize("name,M,N,K,a_mn,b_mn,use_bias,ldc_pad", CASES, ids=[c[0] for c in CASES])
def test_gemm_epilogue_bit_identical(name, M, N, K, a_mn, b_mn, use_bias, ldc_pad):
    from zaremba_b200 import _lib
    lib = _lib.load()
    g = torch.Generator(device="cuda").manual_seed(M * 7919 + N * 31 + K)
    A = torch.randn(M, K, device="cuda", generator=g).half()
    Bm = torch.randn(N, K, device="cuda", generator=g).half()
    bias = torch.randn(N, device="cuda", generator=g) if use_bias else None
    Ab, lda = _operand(A, a_mn)
    Bb, ldb = _operand(Bm, b_mn)
    ldc = N + ldc_pad
    new = _run(lib, "new", Ab, lda, a_mn, Bb, ldb, b_mn, M, N, K, ldc, 0.75, bias, 0)
    old = _run(lib, "direct", Ab, lda, a_mn, Bb, ldb, b_mn, M, N, K, ldc, 0.75, bias, 0)
    assert not torch.isnan(new[:M, :N]).any(), f"{name}: NaN in the output"
    assert (new[:M, N:] == SENTINEL).all() and (new[M] == SENTINEL).all(), f"{name}: write outside [M, N]"
    assert torch.equal(new, old), f"{name}: {(new != old).sum().item()} elements differ from ZRB_GEMM_EPI=direct"
    if ldc_pad == 0 and M * N <= 4_000_000:
        C0 = torch.randn(M, N, device="cuda", generator=g)
        acc_bias = torch.randn(N, device="cuda", generator=g)
        new = _run(lib, "new", Ab, lda, a_mn, Bb, ldb, b_mn, M, N, K, ldc, -0.5, acc_bias, 1, C0)
        old = _run(lib, "direct", Ab, lda, a_mn, Bb, ldb, b_mn, M, N, K, ldc, -0.5, acc_bias, 1, C0)
        assert torch.equal(new, old), f"{name}: accumulate = 1 differs from ZRB_GEMM_EPI=direct"


def _large_steps(side):
    import zaremba_b200
    os.environ.pop("ZRB_GEMM_EPI", None)
    if side == "direct":
        os.environ["ZRB_GEMM_EPI"] = "direct"
    try:
        V, H, L, T, B = 10000, 1500, 2, 35, 20
        torch.manual_seed(1234)
        m = zaremba_b200.Model(V, H, L, 0.65, 0.04).cuda()
        m.train()
        tr = zaremba_b200.Trainer(m, B, T, lazy_update=True)
        g = torch.Generator().manual_seed(99)
        for h, c in tr.states:
            h.copy_(0.1 * torch.randn(h.shape, generator=g).cuda())
            c.copy_(0.1 * torch.randn(c.shape, generator=g).cuda())
        # distinct input tokens per window: the embedding gradient is a scatter-add with fp32 atomics, and a token
        # seen three or more times sums its rows in whatever order they land (DESIGN §6), GEMMs or not
        xs = [torch.randperm(V, generator=g)[:T * B].view(T, B).contiguous().cuda() for _ in range(2)]
        ys = [torch.randint(0, V, (T, B), generator=g).cuda() for _ in range(2)]
        out = {}
        for s in range(2):
            x, y = xs[s], ys[s]
            loss, norm = tr.train_step(x, y, 1.0, 5.0)
            tr.flush()
            torch.cuda.synchronize()
            out[f"loss{s}"], out[f"norm{s}"] = loss.clone(), norm.clone()
            out[f"flat_g{s}"], out[f"flat_p{s}"] = tr.flat_g.clone(), tr.flat_p.clone()
            for i, t in enumerate(t for st in tr.states for t in st):
                out[f"state{s}.{i}"] = t.clone()
        loss, probs = tr.eval_step(xs[0], ys[0], want_probs=True)
        torch.cuda.synchronize()
        out["eval_loss"], out["eval_probs"] = loss.clone(), probs.clone()
        tr.close()
        del tr, m
        gc.collect()
        return out
    finally:
        os.environ.pop("ZRB_GEMM_EPI", None)


def test_large_trainer_step_bit_identical():
    """Two fused Large steps (the second one on the fp16 images the first one's update rebuilt) and an eval pass."""
    new = _large_steps("new")
    old = _large_steps("direct")
    assert new["norm0"].item() > 0 and torch.isfinite(new["loss0"]).all()
    bad = [k for k in new if not torch.equal(new[k], old[k])]
    assert not bad, f"differ from ZRB_GEMM_EPI=direct: {bad}"
