"""The backward recurrence element by element: every dG image the kernels store, at every step, against the
rounded-operand restatement (tests/_rounded_oracle.py) teacher-forced on the device's own images.

The other backward tests compare dx, dW and db with the exact fp64 oracle as a fraction of each tensor's largest
element, which cannot see an error confined to small elements or diluted by the sum over T * B.  The images dG_t
themselves are not outputs, so this file makes them observable, bit for bit, with a probe model:

  - one layer whose input width is the gate width (Model(embed_size=4H)) and W_ih = I: the input GEMM hands the layer
    the pre-activation r(x) exactly, and the dgrad GEMM dx = dG_h W_ih_img 2^-10 has one non-zero product per output,
    so dx is the image divided by 1024;
  - distinct tokens for every (t, b), embedding rows holding the layer inputs: each dense-scatter row of dE receives
    one exact addition, so dE gives back dx times the site-0 multiplier;
  - fc.W = [I_H; 0], fc.b = 0, dscores with 1024 dS fp16-exact: the projection dgrad hands the layer dy = dS exactly,
    and the forward's scores[:, :H] are the fp16 image of the layer output;
  - Zaremba dropout p = 0.5 by explicit masks: site 0 all ones (multiplier 2, exact); a first forward with site L all
    ones reads r(2h), the second, with a random site-L mask, is the one differentiated.  The variational and zoneout
    modes refuse explicit masks and run at p = 0 (variational: p_rec = 0.5, multiplier 2).

Checks per case: each dG image against the restatement within half an fp16 ulp plus TAU * 1024 * E (E: the
restatement's magnitude of the element), with the clamp at 65504; dW_ih and dW_hh as GEMMs on the device's own images
at the GEMM test's tolerance; db against the sum of the restatement's dG; the forward's h images against the
teacher-forced forward.  And resolution: deliberate mutations of the restatement of the kind these kernels could get
wrong must land at least RESOLUTION times outside the bound on some element, or the case is vacuous.
"""

import numpy as np
import pytest
import torch

from oracle import philox as PH
from tests import _rounded_oracle as RO
from tests.test_gpu_gemm import TOL as GEMM_TOL
from tests.test_gpu_parity import LAYER_CASES, _plan_branch, _record
from tests.test_gpu_trained_regime import ACT_TOL, ACT_TOL_PER_H, _saturated

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
# Measured on an H100 80GB HBM3 at a 700 W power limit over CASES: a dG image lies at most 2.0e-5 * 1024 E beyond half
# an fp16 ulp of the restatement (zoneout at S = 2; 4e-6 .. 1.3e-5 elsewhere, 3.4e-6 .. 4.5e-6 saturated), db at most
# 7.4e-8 of its summed magnitudes.  TAU is three times the largest.
TAU = 6e-5
# dW_ih / dW_hh per element over sum |img| |operand| / 1024: at most 1.0e-6 where the images span a few decades (held to
# the GEMM test's TOL), 3.9e-6 where saturation spreads them over nine (K = T * B products whose running sum sits at the
# few dominant ones, so each addition rounds at the scale of the whole sum): held to three times that
DW_TOL = dict(saturated=1.2e-5)
RESOLUTION = 100.0
ZONEOUT = (0.3, 0.4)          # zoneout_cell, zoneout_hidden

# name -> (H, T, B, data, mode, plan branch of test_gpu_parity._plan_branch or None, context window or None)
CASES = {f"{c}_H{H}_T{T}_B{B}": (H, T, B, "init", "zaremba", c, None) for (H, T, B), c in LAYER_CASES.items()}
CASES.update({
    "long_H650_T140_B20": (650, 140, 20, "init", "zaremba", None, None),
    "ctx35x32_run3x5_H650": (650, 3, 5, "init", "zaremba", None, (35, 32)),
    "saturated_H650_T35_B20": (650, 35, 20, "saturated", "zaremba", None, None),
    "saturated_H1500_T35_B32": (1500, 35, 32, "saturated", "zaremba", "two_cells_n32", None),
    "exploding_H650_T35_B20": (650, 35, 20, "exploding", "zaremba", None, None),
    "variational_H650_T35_B20": (650, 35, 20, "init", "variational", None, None),
    "zoneout_S1_H255_T4_B32": (255, 4, 32, "init", "zoneout", "nosplit_n32", None),
    "zoneout_S2_H650_T35_B32": (650, 35, 32, "init", "zoneout", "one_tile_n32", None),
    "per_timestep_H650_T35_B40": (650, 35, 40, "saturated", "zaremba", "per_timestep", None),
})


def _data(kind, H, T, B, seed):
    """numpy fp64: xr [T,B,4H] (the fp16-exact pre-activation the input GEMM hands the layer), W_hh, b_ih, b_hh, h0, c0
    (fp32 values) and dy [T,B,H] with 1024 dy fp16-exact."""
    rng = np.random.default_rng(seed)
    f32 = lambda a: np.asarray(a).astype(np.float32).astype(np.float64)
    r16 = lambda a: np.asarray(a).astype(np.float16).astype(np.float64)
    if kind == "saturated":
        a = _saturated(H, T, B, seed)
        x, W_ih, W_hh, b_ih, b_hh, h0, c0, dy = (a[k] for k in ("x", "W_ih", "W_hh", "b_ih", "b_hh", "h0", "c0", "dy"))
    elif kind == "init":
        w = 0.04 if H >= 1000 else 0.08
        W_ih, W_hh = rng.uniform(-w, w, size=(4 * H, H)), rng.uniform(-w, w, size=(4 * H, H))
        b_ih, b_hh = rng.uniform(-w, w, size=4 * H), rng.uniform(-w, w, size=4 * H)
        x = rng.normal(size=(T, B, H)) * 0.5
        h0, c0 = rng.uniform(-0.5, 0.5, size=(B, H)), rng.uniform(-1.0, 1.0, size=(B, H))
        dy = rng.normal(size=(T, B, H)) * 0.1
    else:
        # exploding: a large-norm W_hh (few gates beyond |z| = 5) with an upstream gradient near the fp16 image's
        # limit: dh grows backwards until a few percent of the images reach the clamp
        W_ih = rng.normal(size=(4 * H, H)) * 0.5 / np.sqrt(H)
        W_hh = rng.normal(size=(4 * H, H)) * 0.6
        b_ih, b_hh = np.zeros(4 * H), np.zeros(4 * H)
        b_hh[3 * H:] = -2.5
        x = rng.normal(size=(T, B, H))
        h0, c0 = rng.uniform(-0.05, 0.05, size=(B, H)), rng.uniform(-1.0, 1.0, size=(B, H))
        dy = np.clip(rng.normal(size=(T, B, H)) * 30.0, -60.0, 60.0)
    return dict(xr=r16(f32(x) @ f32(W_ih).T), W_hh=f32(W_hh), b_ih=f32(b_ih), b_hh=f32(b_hh), h0=f32(h0), c0=f32(c0),
                dy=r16(1024.0 * dy) / 1024.0)


def _probe(name):
    """Runs the probe model for case `name`; returns the device's images and gradients and what the oracle needs."""
    import zaremba_b200
    from zaremba_b200 import _lib
    H, T, B, data, mode, branch, ctx_tb = CASES[name]
    V = max(T * B, H)
    p = 0.5 if mode == "zaremba" else 0.0
    kw = dict(variational=True, recurrent_dropout=0.5) if mode == "variational" else \
        dict(zoneout_cell=ZONEOUT[0], zoneout_hidden=ZONEOUT[1]) if mode == "zoneout" else {}
    torch.manual_seed(0)
    m = zaremba_b200.Model(V, H, 1, p, 0.05, engine="tc", embed_size=4 * H, layer_sizes=[H], **kw).to(DEV)
    plans = _lib.rec_plans(m._context(*(ctx_tb or (T, B))))
    fp, bp = plans["fwd"], plans["bwd"]
    if branch == "per_timestep":
        assert not fp["ok"] and not bp["ok"], plans
    elif branch in (None, "baseline"):
        assert fp["ok"] and bp["ok"], plans
    else:
        if not (fp["ok"] and bp["ok"]):
            pytest.skip(f"H={H} B={B} does not fit the persistent kernels on this device: {plans}")
        if not _plan_branch(branch, H, B, fp, bp):
            pytest.skip(f"on {torch.cuda.get_device_properties(0).multi_processor_count} SMs H={H} B={B} gets {plans}, "
                        f"not the {branch} branch this case is for")
    d = _data(data, H, T, B, 7 * H + T)
    rng = np.random.default_rng(H + 3 * T + B)
    s0 = 2.0 if mode == "zaremba" else 1.0
    tok = rng.permutation(V)[:T * B].reshape(T, B)
    emb = np.zeros((V, 4 * H))
    emb[tok.reshape(-1)] = d["xr"].reshape(-1, 4 * H) / s0
    fc = np.zeros((V, H))
    fc[:H] = np.eye(H)
    dev = lambda a: torch.as_tensor(a, dtype=torch.float32, device=DEV)
    m.load_state_dict({"embed.W": dev(emb), "rnns.0.weight_ih_l0": torch.eye(4 * H, device=DEV),
                       "rnns.0.weight_hh_l0": dev(d["W_hh"]), "rnns.0.bias_ih_l0": dev(d["b_ih"]),
                       "rnns.0.bias_hh_l0": dev(d["b_hh"]), "fc.W": dev(fc), "fc.b": torch.zeros(V, device=DEV)})
    m.train()
    states = lambda: [(dev(d["h0"]).view(1, B, H), dev(d["c0"]).view(1, B, H))]
    xt = torch.as_tensor(tok)
    dS = torch.zeros(T * B, V, device=DEV)
    dS[:, :H] = dev(d["dy"].reshape(T * B, H))
    maskL = None
    if mode == "zaremba":
        maskL = rng.random((T, B, H)) >= 0.5
        ones0 = torch.ones(T, B, 4 * H, dtype=torch.uint8, device=DEV)
        m.set_explicit_dropout_masks([ones0, torch.ones(T, B, H, dtype=torch.uint8, device=DEV)])
        with torch.no_grad():
            s1, st1 = m(xt, states())
        m.set_explicit_dropout_masks([ones0, torch.as_tensor(maskL.astype(np.uint8), device=DEV)])
        s2, st2 = m(xt, states())
        assert torch.equal(st1[0][0], st2[0][0]) and torch.equal(st1[0][1], st2[0][1]), "the two forwards differ"
    else:
        s2, st2 = m(xt, states())
        s1 = s2.detach()
    s2.backward(dS)
    torch.cuda.synchronize()
    g = {k: v.grad.detach().to(torch.float64) for k, v in m.named_parameters()}
    f64 = lambda a: torch.as_tensor(a, dtype=torch.float64, device=DEV)
    # the probe works as stated
    s1 = s1.detach().to(torch.float64)
    assert torch.equal(s1[:, H:], torch.zeros_like(s1[:, H:])), "scores beyond the first H columns"
    Y = s1[:, :H].reshape(T, B, H)
    assert torch.equal(RO.r16(Y), Y), "scores[:, :H] are not fp16 images"
    dE = g["embed.W"]
    used = torch.zeros(V, dtype=torch.bool, device=DEV)
    used[f64(tok.reshape(-1)).long()] = True
    assert torch.equal(dE[~used], torch.zeros_like(dE[~used])), "unused embedding rows received gradient"
    img = (RO.GRAD_SCALE * dE[f64(tok.reshape(-1)).long()] / s0).reshape(T, B, 4 * H)
    assert torch.equal(RO.r16(img), img), "1024 dE / s0 is not an fp16 image"
    out = dict(H=H, T=T, B=B, mode=mode, bp=bp, persistent=bool(bp["ok"]), img=img, Y=Y, g=g,
               hT=st2[0][0].detach().reshape(B, H).to(torch.float64), cT=st2[0][1].detach().reshape(B, H).to(torch.float64),
               **{k: f64(v) for k, v in d.items()})
    out["sy"] = s0                                  # Y = r(sy h)
    out["dyv"] = out["dy"] * (2.0 * f64(maskL) if maskL is not None else 1.0)
    seed, step = m._seed, m._drop_step - 1
    out["q"] = None
    if mode == "variational":
        out["q"] = 2.0 * f64(PH.keep_mask(seed, step, 2, B * H, 0.5).reshape(B, H))
    out["zc"] = out["zh"] = None
    if mode == "zoneout":
        out["zc"], out["zh"] = (torch.as_tensor(~PH.keep_mask(seed, step, site, T * B * H, z).reshape(T, B, H),
                                                device=DEV) for site, z in ((6, ZONEOUT[0]), (7, ZONEOUT[1])))
    del m
    return out


def _operands(r):
    """The recurrent operand each step multiplied (the device's image of q h_{t-1}; h_{-1} = h0) and its uncertainty
    where it is known only through the image of another multiple of h (RO.rescale_image)."""
    q = 1.0 if r["q"] is None else r["q"]
    a0 = RO.r16(q * r["h0"])
    Y = r["Y"][:-1]
    if r["sy"] == 2.0:
        a, amb = RO.rescale_image(Y, 0.5)
    elif r["q"] is not None:
        a, amb = RO.rescale_image(Y, 2)
        a, amb = a * (r["q"] / 2.0), amb * (r["q"] / 2.0)
    else:
        a, amb = Y, torch.zeros_like(Y)
    return torch.cat([a0[None], a]), torch.cat([torch.zeros_like(a0)[None], amb])


def _exceed(img, dG, E, tau):
    """Per element: how far the device image lies beyond half an fp16 ulp of the clamped reference, in units of
    tau * 1024 * E."""
    ref = (RO.GRAD_SCALE * dG).clamp(-RO.F16_MAX, RO.F16_MAX)
    return ((img - ref).abs() - 0.5 * RO.ulp16(img)) / (tau * RO.GRAD_SCALE * E)


@pytest.mark.parametrize("name", list(CASES))
def test_backward_images_against_rounded_operand_oracle(name):
    r = _probe(name)
    H, T, B = r["H"], r["T"], r["B"]
    img, Y = r["img"], r["Y"]
    N = T * B
    a, amb = _operands(r)
    Wr = RO.r16(r["W_hh"])
    pre = RO.M(r["xr"] + r["b_ih"] + r["b_hh"], r["xr"].abs() + r["b_ih"].abs() + r["b_hh"].abs())
    fw = RO.forward(pre, Wr, r["c0"], a=a, zc=r["zc"], zh=r["zh"])
    bad, rep = [], {}

    # forward: the device's h images against the teacher-forced forward
    h_ref = torch.stack([h.v for h in fw["hn"]])
    err = ((Y - r["sy"] * h_ref).abs() - 0.5 * RO.ulp16(Y)) / r["sy"]
    if r["zh"] is not None:
        prev = torch.cat([RO.r16(r["sy"] * r["h0"])[None], Y[:-1]])
        assert torch.equal(Y[r["zh"]], prev[r["zh"]]), "a zoned-out h is not its predecessor"
        err = torch.where(r["zh"], 0.0, err)
    rep["fwd y (abs)"] = float(err.max())
    if rep["fwd y (abs)"] > ACT_TOL_PER_H * H:
        bad.append(f"forward h: {rep['fwd y (abs)']:.2e} > {ACT_TOL_PER_H * H:.1e}")
    assert torch.equal(RO.r16(r["sy"] * r["hT"]), Y[-1]), "hT is not the last step's h"
    c_ref = fw["c"][-1].v
    rep["fwd cT"] = float((r["cT"] - c_ref).abs().max() / max(float(c_ref.abs().max()), 1.0))
    if rep["fwd cT"] > ACT_TOL["fwd"]:
        bad.append(f"cT: {rep['fwd cT']:.2e} > {ACT_TOL['fwd']:.1e}")

    # backward: every image of every step
    assert torch.isfinite(img).all(), "inf / NaN among the dG images"
    dG, E = RO.backward(fw, r["dyv"], Wr, r["c0"], img=img, q=r["q"], zc=r["zc"], zh=r["zh"])
    ex = _exceed(img, dG, E, 1.0)   # (in units of 1024 E: the measured tau)
    rep["dG image / (1024 E)"] = float(ex.max())   # tau of this case
    if rep["dG image / (1024 E)"] > TAU:
        t, b, k = np.unravel_index(int(ex.argmax()), ex.shape)
        bad.append(f"dG image at t={t} b={b} gate={k // H} unit={k % H}: {float(img[t, b, k])} vs "
                   f"{float(RO.GRAD_SCALE * dG[t, b, k])}, {rep['dG image / (1024 E)']:.2e} of 1024 E > TAU {TAU:.1e}")
    big = (RO.GRAD_SCALE * dG).abs() > 1.001 * (RO.F16_MAX + 16.0)
    assert torch.equal(img[big].abs(), torch.full_like(img[big], RO.F16_MAX)), "a clearly clamped image is not 65504"

    # dW_ih, dW_hh: GEMMs on the device's images, per element against sum |img| |operand| / 1024
    G = img.reshape(N, 4 * H)
    X = r["xr"].reshape(N, 4 * H)
    s = G.abs().T @ X.abs() / RO.GRAD_SCALE
    e = (r["g"]["rnns.0.weight_ih_l0"] - G.T @ X / RO.GRAD_SCALE).abs()
    rep["dW_ih / s"] = float((e / s.clamp(min=1e-300)).max())
    assert torch.equal(e[s == 0], torch.zeros_like(e[s == 0]))
    del s, e
    A, Aamb = a.reshape(N, H), amb.reshape(N, H)
    slack = G.abs().T @ Aamb / RO.GRAD_SCALE
    s = G.abs().T @ (A.abs() + Aamb) / RO.GRAD_SCALE
    e = ((r["g"]["rnns.0.weight_hh_l0"] - G.T @ A / RO.GRAD_SCALE).abs() - slack).clamp(min=0.0)
    rep["dW_hh / s"] = float((e / s.clamp(min=1e-300)).max())
    dw_tol = DW_TOL.get(CASES[name][3], GEMM_TOL)
    for k in ("dW_ih / s", "dW_hh / s"):
        if rep[k] > dw_tol:
            bad.append(f"{k}: {rep[k]:.2e} > {dw_tol:.1e}")

    # db: the sum of the restatement's dG, within TAU of the summed magnitudes; both bias gradients one tensor
    assert torch.equal(r["g"]["rnns.0.bias_ih_l0"], r["g"]["rnns.0.bias_hh_l0"])
    e = (r["g"]["rnns.0.bias_ih_l0"] - dG.sum((0, 1))).abs()
    rep["db / sum E"] = float((e / E.sum((0, 1)).clamp(min=1e-300)).max())
    if rep["db / sum E"] > TAU:
        bad.append(f"db: {rep['db / sum E']:.2e} of the summed magnitudes > TAU {TAU:.1e}")

    # the regime a case is for
    sub = ((img != 0) & (img.abs() < RO.F16_MIN_NORMAL))
    rep["subnormal images"] = float(sub.double().mean())
    rep["clamped images"] = float((img.abs() == RO.F16_MAX).double().mean())
    if "saturated" in name:
        assert sub.any(), "no subnormal dG image"
    if "exploding" in name:
        assert rep["clamped images"] > 0, "no clamped dG image"

    # resolution: mutations of the restatement land far outside the bound
    muts = []
    if T > 1:
        muts += ["stale_slot", "shift_column"] + (["drop_partial"] if r["persistent"] else [])
        if "saturated" in name:
            muts.append("flush_subnormal")
        if r["q"] is not None:
            muts.append("multiplier_on_dy")
        if r["zh"] is not None:
            muts.append("drop_hcarry")
    geometry = None
    if r["persistent"]:
        bp = r["bp"]
        # the partial of the g gate's rows (their products carry tanh' <= 1, not sigmoid' <= 1/4: at T = 2, B = 1 a
        # missing i-gate half lands only ~90 times outside the bound), the whole block at S = 1, its first K half at S = 2
        rows = 2 * H + torch.arange(H if bp["KS"] == 1 else min(8 * bp["KcS"], H), device=DEV)
        uc = 4 * bp["KS"] * bp["U"]   # units of a cluster: the last one's are partly filled unless uc divides H
        geometry = (rows, torch.arange((H - 1) // uc * uc, H, device=DEV))
    for mut in muts:
        dGm, _ = RO.backward(fw, r["dyv"], Wr, r["c0"], img=img, q=r["q"], zc=r["zc"], zh=r["zh"], mutate=mut,
                             geometry=geometry)
        rep[f"resolution {mut}"] = float(_exceed(img, dGm, E, TAU).max())
        if rep[f"resolution {mut}"] < RESOLUTION:
            bad.append(f"mutation {mut} lands {rep[f'resolution {mut}']:.1f} x the bound, < {RESOLUTION}: vacuous")
    for k, v in rep.items():
        _record(k, v)
    print(f"\n{name}: bwd plan {r['bp']}\n  " + "\n  ".join(f"{k}: {v:.3e}" for k, v in rep.items()))
    assert not bad, bad
