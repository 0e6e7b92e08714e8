"""The split-K GEMM plan in CTA pairs (gemm_tc.cu gemm_f16_tc_pair_kernel: 64-row work items, two per 2-CTA cluster,
the B tile multicast to both) against ZRB_GEMM_EPI=direct (the 128-row split plan): outputs must be BIT-IDENTICAL.

  * every split-K call shape of the Small / Medium / Large train steps (the dgrads dS*W_fc and dG*W_ih; Large takes the
    pair plan, Small and Medium, with 128-wide tiles, keep the 128-row one);
  * odd shapes that take the pair plan (on a 132-SM H100): M in {65, 127} (one 128-row tile, two 64-row items) and
    {700, 701} (64-row blocks odd in number: the last ones pair along N without sharing B), N not a multiple of 256
    (5 N blocks: one item left over, paired with a copy of itself), odd K-block counts (K halves of unequal length),
    all four operand layouts, with and without bias;
  * poisoned as in test_gpu_gemm.py: operand padding NaN, C NaN before the call, a sentinel in the row after M;
  * a torch.profiler run of the Large dS*W_fc call: the pair kernel ran on 132 CTAs (66 clusters of 2 -- it is only
    launched in 2-CTA clusters).
"""
import json
import os
import tempfile

import pytest
import torch

pytestmark = pytest.mark.gpu

SENTINEL = 12345.0
V = 10000


def _config_shapes():
    out = []
    for cfg, H, T, B in (("small", 200, 20, 20), ("medium", 650, 35, 20), ("large", 1500, 35, 20)):
        out += [(f"{cfg}-proj_dgrad", T * B, H, V, 0, 1, False), (f"{cfg}-gemm_dx", T * B, H, 4 * H, 0, 1, False)]
    return out


# (M, N, K): 65 / 127 rows = one 128-row tile, two 64-row items (N wide enough for 256-wide split tiles); 700 / 701 =
# 11 64-row blocks; N = 1300 / 1200 not multiples of 256, 1200 giving 5 N blocks (11 x 5 items per K half: one left
# over); K = 6080 / 6050 odd K-block counts (95)
ODD = [(65, 6600, 1500), (127, 7000, 2000), (700, 1500, 6080), (701, 1300, 6000), (700, 1200, 10000),
       (701, 1200, 6050)]


def _pair_plan(M, N, K, nsm=132):
    """gemm_tc.cu's choice restated: split K over 256-wide tiles, more 64-row items than 128-row tiles, and all the
    pairs resident at once (66 clusters of 2 on a 132-SM H100)."""
    cdiv = lambda a, b: (a + b - 1) // b
    tm, tm64, tn, kb = cdiv(M, 128), cdiv(M, 64), cdiv(N, 256), cdiv(K, 64)
    split256 = 2 * tm * tn <= nsm and 2 * tm * tn >= (nsm * 4) // 10 and kb // 2 >= 8
    pairs = 2 * ((tm64 // 2) * tn + ((tn + 1) // 2 if tm64 % 2 else 0))
    return split256 and tm64 > tm and pairs <= nsm // 2


assert all(_pair_plan(M, N, K) for M, N, K in ODD)

CASES = [(n, M, N, K, a, b, bias) for n, M, N, K, a, b, bias in _config_shapes()]
CASES += [(f"odd-{M}x{N}x{K}-{a}{b}", M, N, K, a, b, i % 2 == 1)
          for i, (M, N, K) in enumerate(ODD) for a, b in ((0, 0), (0, 1), (1, 0), (1, 1))]


def _operand(logical, mn_major):
    rows, K = logical.shape
    inner, outer = (rows, K) if mn_major else (K, rows)
    ld = (inner + 7) // 8 * 8 + 8
    buf = torch.full((outer + 8, ld), float("nan"), dtype=torch.float16, device="cuda")
    buf[:outer, :inner] = logical.t() if mn_major else logical
    return buf, ld


def _run(lib, side, A, lda, a_mn, Bm, ldb, b_mn, M, N, K, bias):
    from zaremba_b200 import _lib
    c = torch.full((M + 1, N), SENTINEL, device="cuda")
    c[:M] = float("nan")
    old = os.environ.pop("ZRB_GEMM_EPI", None)
    try:
        if side == "direct":
            os.environ["ZRB_GEMM_EPI"] = "direct"
        _lib.check(lib.zrb_gemm_f16(_lib.ptr(A), lda, a_mn, _lib.ptr(Bm), ldb, b_mn, _lib.ptr(c), N, M, N, K, 0.75,
                                    _lib.ptr(bias), 0, None))
        torch.cuda.synchronize()
    finally:
        os.environ.pop("ZRB_GEMM_EPI", None)
        if old is not None:
            os.environ["ZRB_GEMM_EPI"] = old
    return c


def _inputs(M, N, K, a_mn, b_mn, use_bias):
    g = torch.Generator(device="cuda").manual_seed(M * 7919 + N * 31 + K)
    A = torch.randn(M, K, device="cuda", generator=g).half()
    Bm = torch.randn(N, K, device="cuda", generator=g).half()
    bias = torch.randn(N, device="cuda", generator=g) if use_bias else None
    Ab, lda = _operand(A, a_mn)
    Bb, ldb = _operand(Bm, b_mn)
    return A, Bm, Ab, lda, Bb, ldb, bias


@pytest.mark.parametrize("name,M,N,K,a_mn,b_mn,use_bias", CASES, ids=[c[0] for c in CASES])
def test_pair_plan_bit_identical(name, M, N, K, a_mn, b_mn, use_bias):
    from zaremba_b200 import _lib
    lib = _lib.load()
    A, Bm, Ab, lda, Bb, ldb, bias = _inputs(M, N, K, a_mn, b_mn, use_bias)
    new = _run(lib, "new", Ab, lda, a_mn, Bb, ldb, b_mn, M, N, K, bias)
    old = _run(lib, "direct", Ab, lda, a_mn, Bb, ldb, b_mn, M, N, K, bias)
    assert not torch.isnan(new[:M]).any(), f"{name}: NaN in the output"
    assert (new[M] == SENTINEL).all(), f"{name}: write past row M"
    assert torch.equal(new, old), f"{name}: {(new != old).sum().item()} elements differ from ZRB_GEMM_EPI=direct"
    # and the product itself (bit identity alone would pass two equally wrong plans)
    ref = 0.75 * (A.double() @ Bm.double().t()) + (bias.double() if use_bias else 0.0)
    scale = 0.75 * (A.double().abs() @ Bm.double().abs().t()) + (bias.double().abs() if use_bias else 0.0)
    err = ((new[:M].double() - ref).abs() / scale.clamp_min(1e-30)).max().item()
    assert err < 3e-6, f"{name}: error {err:.3g} of the summed magnitude"


def test_pair_plan_runs_at_large():
    """The Large dS*W_fc dgrad (700 x 1500 x 10000) runs as the pair kernel on 66 clusters of 2 CTAs."""
    from torch.profiler import ProfilerActivity, profile
    from zaremba_b200 import _lib
    lib = _lib.load()
    M, N, K = 700, 1500, V
    _, _, Ab, lda, Bb, ldb, _ = _inputs(M, N, K, 0, 1, False)
    c = torch.empty(M, N, device="cuda")
    os.environ.pop("ZRB_GEMM_EPI", None)

    def call():
        _lib.check(lib.zrb_gemm_f16(_lib.ptr(Ab), lda, 0, _lib.ptr(Bb), ldb, 1, _lib.ptr(c), N, M, N, K, 1.0,
                                    None, 0, None))
    call()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    assert torch.cuda.get_device_properties(0).multi_processor_count == 132
    with tempfile.TemporaryDirectory() as d:   # kernel events carry their grid in the exported trace
        prof.export_chrome_trace(os.path.join(d, "trace.json"))
        with open(os.path.join(d, "trace.json")) as f:
            trace = json.load(f)
    kernels = {e["name"]: e["args"]["grid"] for e in trace["traceEvents"] if e.get("cat") == "kernel"}
    pair = [g for n, g in kernels.items() if "gemm_f16_tc_pair_kernel" in n]
    assert pair == [[132, 1, 1]], f"the pair plan did not run on 132 CTAs: {kernels}"
