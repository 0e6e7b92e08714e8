"""The K-split recurrence plans at N = pad8(B): the operand and dG images hold the real 8-row batch groups, two at B <= 8
(rec_split_groups), so B = 17..24 runs at N = 24, an odd group count the plans used to pad to 32.

  - a CPU restatement of rec_fwd_plan / rec_bwd_plan at 132 SMs, asserting which branch and which U each shape gets;
  - on the GPU, the restatement against the device's plans (on a 132-SM device), and one layer through the persistent
    kernels against the fp64 oracle (test_gpu_parity._layer_against_oracle) and element by element through the dG
    images (test_gpu_rec_bwd_images) at N = 24: B = 20 at H = 1500, and B = 17 with a partly filled last CTA and cluster.
"""
import pytest
import torch

# restated from lstm_rec_fwd.cu / lstm_rec_bwd.cu / rec_common.cuh
EPI_THREADS, MAX_CELL, SMEM_MAX = 256, 2, 227 * 1024
NSM = 132                 # H100 SXM
MAX_CLUSTERS8 = 15        # cudaOccupancyMaxActiveClusters for 8-CTA clusters at one CTA per SM on a 132-SM H100
FIELDS = ("ok", "KS", "U", "G", "nCTA", "GBi", "Kc", "KcS")


def smem_bytes(Kc, G, GB):
    return Kc * G * 128 + Kc * GB * 128 + 2 * 64 * (GB * 8 + 1) * 4 + 256


def split_groups(GB):
    return max(GB, 2)


def _fits(U, KcS, GBi):
    """Shared memory, and the receive area for the 8U rows a CTA receives."""
    return smem_bytes(KcS, U, GBi) <= SMEM_MAX and 8 * U * (GBi * 8 + 4) <= 128 * (GBi * 8 + 1)


def _plan(KS, U, G, nCTA, GBi, Kc, KcS):
    return dict(ok=1, KS=KS, U=U, G=G, nCTA=nCTA, GBi=GBi, Kc=Kc, KcS=KcS)


def _first_choice(U, B, nCTA, nsm):
    """The split plans' first choice: one (unit, batch) cell per epilogue thread, and at least an eighth of the SMs
    left for the work launched beside the recurrence."""
    return U * B <= EPI_THREADS and nCTA <= nsm - nsm // 8


def fwd_plan(H, B, nsm=NSM):
    GB = (B + 7) // 8
    if GB * 8 > 32:
        return dict.fromkeys(FIELDS, 0)
    if H >= 256:
        Kc = (H + 31) // 32 * 32 // 8
        KcS = Kc // 2
        for first in (True, False):
            for U in range(16, 0, -1):
                npair = -(-H // (2 * U))
                if 2 * npair > nsm:
                    break
                if U * B > MAX_CELL * EPI_THREADS or (first and not _first_choice(U, B, 2 * npair, nsm)):
                    continue
                if _fits(U, KcS, split_groups(GB)):
                    return _plan(2, U, U, 2 * npair, split_groups(GB), Kc, KcS)
    Kc = (H + 15) // 16 * 16 // 8
    for U in range(16, 0, -1):
        n = -(-H // U)
        if n > nsm:
            break
        G = (4 * U + 7) // 8
        if smem_bytes(Kc, G, GB) <= SMEM_MAX and U * B <= MAX_CELL * EPI_THREADS:
            return _plan(1, U, G, n, GB, Kc, Kc)
    return dict.fromkeys(FIELDS, 0)


def bwd_plan(H, B, nsm=NSM, max_clusters8=MAX_CLUSTERS8):
    GB = (B + 7) // 8
    if GB * 8 > 32:
        return dict.fromkeys(FIELDS, 0)
    if H >= 256:
        Kc = (H + 31) // 32 * 32 // 8
        KcS = Kc // 2
        for first in (True, False):
            for U in range(16, 0, -1):
                ncl = -(-H // (8 * U))
                if 8 * U > 128:
                    continue
                if 8 * ncl > nsm:
                    break
                if U * B > MAX_CELL * EPI_THREADS or (first and not _first_choice(U, B, 8 * ncl, nsm)):
                    continue
                if _fits(U, KcS, split_groups(GB)) and ncl <= max_clusters8:
                    return _plan(2, U, U, 8 * ncl, split_groups(GB), Kc, KcS)
    Kc = (H + 15) // 16 * 16 // 8
    for U in range(16, 0, -1):
        if (4 * U) % 8:
            continue
        ncl = -(-H // (4 * U))
        if ncl > (nsm - 16) // 4:
            break
        if smem_bytes(Kc, U // 2, GB) <= SMEM_MAX and U * B <= MAX_CELL * EPI_THREADS:
            return _plan(1, U, U // 2, 4 * ncl, GB, Kc, Kc)
    return dict.fromkeys(FIELDS, 0)


# (H, B) -> (forward U, nCTA), (backward U, nCTA), GBi at 132 SMs
EXPECTED = {
    (1500, 20): ((14, 108), (14, 112), 3),   # Large: both grids leave SMs for the deferred update / weight gradients
    (650, 20): ((12, 56), (12, 56), 3),      # Medium: the first choice
    (300, 17): ((14, 22), (14, 24), 3),      # N = 24, the last CTA and the last cluster partly filled
    (1500, 1): ((13, 116), (13, 120), 2),    # B <= 8 keeps N = 16: at N = 8 the receive area limits U to 12
    (300, 8): ((13, 24), (13, 24), 2),
    (1500, 32): ((13, 116), (13, 120), 4),   # N = 32: the plans the even pad gave
}


@pytest.mark.parametrize("H,B", list(EXPECTED))
def test_restated_plans_at_132_sms(H, B):
    (fu, fn), (bu, bn), gbi = EXPECTED[(H, B)]
    fp, bp = fwd_plan(H, B), bwd_plan(H, B)
    assert (fp["KS"], fp["U"], fp["nCTA"], fp["GBi"]) == (2, fu, fn, gbi), fp
    assert (bp["KS"], bp["U"], bp["nCTA"], bp["GBi"]) == (2, bu, bn, gbi), bp
    assert fp["GBi"] == bp["GBi"] == max((B + 7) // 8, 2)


def test_restated_b17_case_is_partly_filled():
    fp, bp = fwd_plan(300, 17), bwd_plan(300, 17)
    assert 0 < 300 - (fp["nCTA"] - 1) * fp["U"] < fp["U"]      # the last forward CTA owns fewer than U units
    assert 300 % (8 * bp["U"]) != 0                              # the last backward cluster is partly empty


def _device_plans(H, T, B):
    import zaremba_b200
    from zaremba_b200 import _lib
    m = zaremba_b200.Model(16, H, 1, 0.0, 0.05, engine="tc").to("cuda:0")
    return m, _lib.rec_plans(m._context(T, B))


@pytest.mark.gpu
@pytest.mark.parametrize("H,B", list(EXPECTED) + [(200, 20), (255, 32), (257, 9), (96, 7)])
def test_device_plans_match_the_restatement(H, B):
    if torch.cuda.get_device_properties(0).multi_processor_count != NSM:
        pytest.skip("the restatement is for 132 SMs")
    _, plans = _device_plans(H, 2, B)
    for kind, want in (("fwd", fwd_plan(H, B)), ("bwd", bwd_plan(H, B))):
        assert {k: plans[kind][k] for k in FIELDS} == want, (kind, plans[kind], want)


# (H, T, B): one layer through the persistent kernels at an odd batch-group count (N = 24)
ODD_GB = [(300, 6, 17), (1500, 35, 20)]


@pytest.mark.gpu
@pytest.mark.parametrize("H,T,B", ODD_GB)
def test_layer_at_odd_group_count_against_oracle(H, T, B):
    from tests.test_gpu_parity import _layer_against_oracle
    from zaremba_b200 import _lib
    m, plans = _device_plans(H, T, B)
    fp, bp = plans["fwd"], plans["bwd"]
    assert fp["ok"] and bp["ok"] and fp["KS"] == 2 and bp["KS"] == 2, plans
    assert fp["GBi"] == bp["GBi"] == 3, plans
    _layer_against_oracle(_lib.load(), m._context(T, B), H, T, B, H + T)


@pytest.mark.gpu
@pytest.mark.parametrize("H,T,B", ODD_GB)
def test_backward_images_at_odd_group_count(H, T, B, monkeypatch):
    from tests import test_gpu_rec_bwd_images as BI
    name = f"odd_gb_H{H}_T{T}_B{B}"
    monkeypatch.setitem(BI.CASES, name, (H, T, B, "init", "zaremba", None, None))
    BI.test_backward_images_against_rounded_operand_oracle(name)
