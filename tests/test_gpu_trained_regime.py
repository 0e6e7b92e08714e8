"""The kernels at a trained model's operating point, against the fp64 oracle.

Every other GPU comparison runs at init weights, where the gates sit near 0.5, |c| stays below ~1 and the softmax is
almost flat.  Here:

  A. A Medium model (V = 10000, H = 650, L = 2, T = 35, B = 20, p = 0.5, lr 1, clip 5) trained for one epoch of the
     Penn Treebank train split with the fused Trainer (tensor-core engine, lazy update, as bench.py runs it).  At its
     weights, on a valid window with carried states: the regime itself is asserted (saturated gates, large |c|, peaked
     softmax, subnormal dS / dG images), then eval forward and gradients of both engines, clamp headroom of the fp16
     gradient images, each trained layer alone at T = 35 and T = 140, zrb_softmax_nll and zrb_sample at the trained
     logits.  Gradients are held to two metrics: the error relative to the tensor's max-abs value, and
     ||g - g*|| / ||g*|| per tensor and per row of fc.W and the embedding (rows down to 1e-3 of the largest row's
     norm), the one that sees subnormal tails of the dS / dG images.
  B. Synthetic saturation (pre-activations of std ~8, forget bias +4, inputs N(0, 2^2), dy spanning nine decades so that
     the dG image runs from fp16 subnormals up to 8 * 1024) at every recurrence-plan branch of
     test_lstm_layer_unit_abi_against_oracle and at two long windows, and once at B = 40 through the per-timestep path
     (tc_cell.cu's expf / tanhf instead of the persistent kernels' SFU activations).  A few units per case are pinned
     at |z| > 40, where __expf overflows or exceeds 2^126; the forward is also held, tightly, to an oracle fed the same
     fp16-rounded operands, which isolates fp32 accumulation and the activation functions.
  C. The Small recipe trained from one init with both engines on the same PTB windows: the loss curves' tails and the
     valid perplexities agree.

Part A's trained point is what one epoch reaches, not a converged model: few gates are saturated and |c| stays below
about 12, so the saturation coverage is Part B's.  What Part A adds is the peaked softmax (subnormal dS images), real
activations and gradients of a trained model, and the sampler's top-p boundary on one or two entries.

The training is not bit-reproducible, so Part A's bounds and floors come from twelve independent trainings; every
tolerance is about three times the largest value measured on an H100 80GB HBM3 (TOL below; DESIGN.md section 5 lists
the measurements and the power limit), every floor about a third of the smallest.
ZRB_ERROR_REPORT2=<path> dumps every measured value.
"""
import numpy as np
import pytest
import torch

from oracle import lstm_lm_oracle as O
from tests import _trained_regime as R
from tests.test_gpu_parity import LAYER_CASES, MEASURED, _plan_branch, _record

pytestmark = pytest.mark.gpu

ENGINES = ["tc", "simt"]
# The trained fixture is not bit-reproducible (the embedding-gradient scatter adds with fp32 atomics, so every run trains
# slightly different weights): each bound below is about three times the largest value over TWELVE independent trainings
# (torch seeds 0..11, `python tools/measure_trained_error.py --runs 12`) on an H100 80GB HBM3 at a 700 W power limit,
# and each floor about a third of the smallest.  fwd / grad = max-abs error over the tensor's max-abs value;
# l2 = ||g - g*|| / ||g*||; rows = worst row of fc.W / embed.W by the same L2 ratio.
#   tc    logits and states <= 4.3e-4, loss 2.8e-6, target probs 2.2e-4, gradients 8.7e-4 (l2 4.7e-4), rows 1.95e-3
#   simt  logits and states <= 1.3e-6, loss 1.0e-7, target probs 3.8e-6, gradients 2.1e-5 (l2 3.4e-6), rows 1.9e-5;
#         held to the suite's stated validation-engine tolerance (tests/test_gpu_parity.py TOL["simt"]: it differs from
#         fp32 by summation order only), which is above three times these and away from fp32 rounding level
TOL = {"tc": dict(fwd=1.3e-3, loss=1e-5, tp=7e-4, grad=2.6e-3, l2=1.5e-3, rows=6e-3),
       "simt": dict(fwd=5e-5, loss=2e-5, tp=5e-5, grad=1e-4, l2=1e-4, rows=1e-4)}
# one trained layer alone, T = 35 and 140: measured y / states <= 6.5e-4, gradients <= 5.2e-4 (l2 2.9e-4)
LAYER_TOL = dict(fwd=2e-3, grad=1.6e-3, l2=9e-4)
# synthetic saturation (part B), persistent kernels and the B = 40 per-timestep path alike, against the exact-operand
# oracle: measured y / states <= 1.34e-2, gradients <= 8.6e-3 (l2 4.1e-3).  This is the fp16 rounding of the operands
# (|dz| ~ 2^-12 |z|, and |z| is ten times init's); the activations are isolated by ACT_TOL below.
SAT_TOL = dict(fwd=4e-2, grad=2.6e-2, l2=1.2e-2)
# the forward against an oracle fed the same fp16-rounded operands and the device's own h_{t-1} (R.rounded_operand_fwd):
# what remains is fp32 accumulation, which grows with H, and the activation functions (lstm_cell.cuh: the SFU FastAct in
# the persistent kernels, expf / tanhf in the per-timestep path), with pre-activations up to |z| = 122.  Measured y
# (absolute) <= 3.3e-8 * H over every case (1.2e-7 at H = 40, 4.1e-5 at H = 1500), c_T <= 1.5e-6 of max(|c|, 1)
ACT_TOL_PER_H = 1e-7
ACT_TOL = dict(fwd=4.5e-6)
# loss 8.8e-8, dscores 5.4e-7 of the scale (held to the suite's 2e-6 / 2e-5), worst dscores row 2.6e-3 (rows whose
# target probability is near 1: p - 1 cancels in fp32), target probabilities 6.8e-7 element by element (a few fp32 ulp)
SOFTMAX_TOL = dict(loss=2e-6, dscores=2e-5, rows=8e-3, tp=5e-6)
# part C, relative gaps between the two engines after TRAJ_STEPS steps, largest of twelve seeds: 3.1e-3 (loss) and 6.0e-2
# (perplexity).  The trajectories drift apart like any two summation orders of one training run: each engine alone
# (atomics in the embedding scatter) ends at valid perplexities a few percent apart from run to run
TRAJ_TOL = dict(loss=1e-2, ppl=0.18)
TRAJ_STEPS = 500
# the regime floors (part A): about a third of the smallest value over the twelve trainings (range in brackets), so that
# a training run that silently failed (weights near init, where each of these is about zero) cannot pass
FLOORS = dict(frac_preact_gt5=1.2e-3,            # (3.7e-3 .. 4.3e-3)
              max_abs_c=1.5,                      # (4.7 .. 12.2)
              median_target_prob=2.4e-3,          # (7.3e-3 .. 8.8e-3; 1e-4 at init)
              frac_softmax_dS_subnormal=1.5e-2,   # (4.7e-2 .. 5.8e-2)
              frac_dG_image_subnormal=4e-3)       # (1.20e-2 .. 1.29e-2)
PPL_DROP = 15.0             # valid perplexity after the epoch at least this many times below its value at init (>= 43)
SAMPLER_PEAKED_ROWS = 1     # rows of 200 whose top-p 0.9 set holds at most two entries (3 .. 5)
CLAMP_MARGIN = 8.0          # max |dS| * 1024 and max |dG| * 1024 stay below 65504 / CLAMP_MARGIN


def _check(what, errs, tol, kind):
    """errs: (max-abs rel, l2 rel) or a float; records and returns the failures as strings."""
    bad = []
    if isinstance(errs, tuple) and len(errs) == 2 and isinstance(errs[1], int):      # row_rel: (worst, rows)
        _record(f"{what} (rows)", errs[0])
        if errs[0] > tol["rows"]:
            bad.append(f"{what}: worst row {errs[0]:.2e} > {tol['rows']:.1e} over {errs[1]} rows")
    elif isinstance(errs, tuple):
        _record(f"{what}", errs[0])
        _record(f"{what} (l2)", errs[1])
        if errs[0] > tol[kind]:
            bad.append(f"{what}: {errs[0]:.2e} of its scale > {tol[kind]:.1e}")
        if "l2" in tol and kind != "fwd" and errs[1] > tol["l2"]:
            bad.append(f"{what}: ||err|| / ||ref|| {errs[1]:.2e} > {tol['l2']:.1e}")
    else:
        _record(what, errs)
        if errs > tol[kind]:
            bad.append(f"{what}: {errs:.2e} > {tol[kind]:.1e}")
    return bad


# ---------------------------------------------------------------------------------------------------------------------
# A. a model trained on the fly
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def trained():
    return R.train(R.MEDIUM)


@pytest.fixture(scope="module")
def point(trained):
    return R.Point(trained["params"])


def test_trained_point_is_in_the_trained_regime(trained, point):
    """Non-vacuity: training worked, and the point reaches what init never does."""
    _record("ppl_init", trained["ppl_init"])
    _record("ppl", trained["ppl"])
    _record("train_seconds", trained["seconds"])
    st = point.regime()
    for k, v in st.items():
        _record(k, v)
    print(f"\n{trained['steps']} steps in {trained['seconds']:.1f} s: valid ppl {trained['ppl_init']:.0f} -> "
          f"{trained['ppl']:.1f}; {st}")
    assert trained["ppl"] * PPL_DROP < trained["ppl_init"], (trained["ppl"], trained["ppl_init"])
    low = {k: (st[k], f) for k, f in FLOORS.items() if not st[k] > f}
    assert not low, f"below the regime floors (measured, floor): {low}"


def test_gradient_images_keep_clamp_headroom(point):
    """max |dS| * 1024 and max |dG| * 1024 of the trained point (oracle, eval and train mode) stay well inside fp16."""
    st = point.regime()
    _record("max_dS_image", st["max_dS_image"])
    _record("max_dG_image", st["max_dG_image"])
    assert st["max_dS_image"] * CLAMP_MARGIN < R.F16_MAX, st
    assert st["max_dG_image"] * CLAMP_MARGIN < R.F16_MAX, st


@pytest.mark.parametrize("engine", ENGINES)
def test_trained_eval_forward_against_oracle(point, engine):
    """Eval mode: logits (drop-in forward), loss, target probabilities and final states (fused eval step)."""
    tol = TOL[engine]
    out = R.eval_forward(point, engine)
    bad = []
    for k, v in out.items():
        kind = {"loss": "loss", "target_probs": "tp"}.get(k, "fwd")
        if k == "target_probs_elementwise":
            _record(k, v)
            continue
        bad += _check(f"{engine} {k}", v, tol, kind)
    assert not bad, bad


@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("engine", ENGINES)
def test_trained_gradients_against_oracle(point, engine, mode):
    """train: one fused step's gradients (zrb_train_step_grads) with explicit dropout masks; eval: the drop-in Model's
    eval-mode backward.  Every tensor by its max-abs scale and by L2; fc.W and embed.W also row by row."""
    tol = TOL[engine]
    bad = []
    if mode == "train":
        loss_err, errs = R.train_grads(point, engine)
        bad += _check(f"{engine} train loss", loss_err, tol, "loss")
    else:
        errs = R.eval_grads(point, engine)
    for k, v in errs.items():
        bad += _check(f"{engine} {mode} grad {k}", v, tol, "grad")
    assert not bad, bad


@pytest.mark.parametrize("T", [35, R.LONG_T])
def test_trained_layers_unit_level(point, T):
    """Each trained layer through zrb_lstm_layer_fwd / _bwd (context for max_seq = 140) on its real inputs, incoming
    states and output gradients, T = 35 and T = 140, against O.lstm_layer_fwd / _bwd."""
    from zaremba_b200 import _lib
    import zaremba_b200
    m = zaremba_b200.Model(16, R.MEDIUM["H"], 1, 0.0, 0.05, engine="tc").to(R.DEV)
    plans = _lib.rec_plans(m._context(R.LONG_T, R.MEDIUM["B"]))
    assert plans["fwd"]["ok"] and plans["bwd"]["ok"], plans
    out = R.layer_unit(point, T)
    bad = []
    for k, v in out.items():
        if k.endswith("db_ih == db_hh"):
            assert v == 1.0, k
        elif isinstance(v, tuple):
            bad += _check(f"T={T} {k}", v, LAYER_TOL, "grad" if "grad" in k else "fwd")
        elif "rounded-operand" in k:
            H = R.MEDIUM["H"]
            bad += _check(f"T={T} {k}", v, dict(fwd=ACT_TOL_PER_H * H) if k.endswith(" y") else ACT_TOL, "fwd")
        else:
            _record(f"T={T} {k}", v)
    assert not bad, bad


@pytest.mark.parametrize("V", [10000, 9999], ids=["register", "scalar"])
def test_trained_softmax_nll(point, V):
    """zrb_softmax_nll at the trained logits: loss, dscores (by scale and row by row) and target probabilities (by
    scale and element by element, down to the smallest)."""
    out = R.softmax_nll(point, V)
    bad = []
    bad += _check(f"V={V} loss", out["loss"], SOFTMAX_TOL, "loss")
    _record(f"V={V} dscores", out["dscores"][0])
    _record(f"V={V} dscores (l2)", out["dscores"][1])
    if out["dscores"][0] > SOFTMAX_TOL["dscores"]:
        bad.append(f"dscores {out['dscores']}")
    bad += _check(f"V={V} dscores", out["dscores rows"], SOFTMAX_TOL, "rows")
    _record(f"V={V} target_probs", out["target_probs"][0])
    _record(f"V={V} target_probs_elementwise", out["target_probs_elementwise"])
    if out["target_probs_elementwise"] > SOFTMAX_TOL["tp"]:
        bad.append(f"target probs {out['target_probs_elementwise']:.2e}")
    assert not bad, bad


def test_trained_sampler_at_peaked_rows(point):
    """zrb_sample at the trained logits, top-p 0.9 / 0.95 and top-k 40, against oracle/sampling.py.  Peaked rows put the
    top-p boundary on one or two entries; that must happen on some rows for the check to mean anything."""
    out = R.sampler(point)
    for k, v in out.items():
        for kk in ("logprob_err", "rows_keeping_le2", "near"):
            _record(f"{k} {kk}", v[kk])
    print(f"\n{out}")
    for k, v in out.items():
        assert v["bad"] == 0, (k, v)
        assert v["near"] <= max(2, v["rows"] // 100), (k, v)
        assert v["logprob_err"] <= 1e-5, (k, v)
    assert out["top_k=0 top_p=0.9"]["rows_keeping_le2"] >= SAMPLER_PEAKED_ROWS, out


# ---------------------------------------------------------------------------------------------------------------------
# B. synthetic saturation at every recurrence-plan branch
# ---------------------------------------------------------------------------------------------------------------------
SAT_CASES = dict(LAYER_CASES)
SAT_CASES.update({(650, 140, 20): "long", (1500, 120, 20): "long"})
DG_MAX = 8.0                # the largest |dG| of a case: its image is 8 * 1024, 8x below the fp16 clamp
PLANTED = 8                 # units per case whose four pre-activations are pinned beyond +-40


def _saturated(H, T, B, seed):
    """Weights whose gate pre-activations have std ~8 (|x| ~ 2 and |h| ~ 0.7 per element), forget bias +4, inputs
    N(0, 2^2), c0 ~ N(0, 5^2), PLANTED units pinned at |z| > 40; dy rows of magnitudes 10^U(-8, 0), rescaled by a power of two so that max |dG| = DG_MAX."""
    rng = np.random.default_rng(seed)
    sw = np.sqrt(64.0 / (4.5 * H))
    W_ih, W_hh = rng.normal(size=(4 * H, H)) * sw, rng.normal(size=(4 * H, H)) * sw
    b_ih, b_hh = rng.normal(size=4 * H), np.zeros(4 * H)
    b_hh[H:2 * H] = 4.0
    # planted units: every gate of PLANTED units driven to |z| in 48..92, where __expf overflows or its result exceeds
    # 2^126 (the large-denominator rule of __fdividef) in FastAct's sigmoid / tanh (lstm_cell.cuh)
    j = rng.choice(H, size=min(PLANTED, H), replace=False)
    for k in range(4):
        b_ih[k * H + j] = rng.choice([-1.0, 1.0], size=j.size) * rng.uniform(48.0, 92.0, size=j.size)
    x = rng.normal(size=(T, B, H)) * 2.0
    h0, c0 = rng.uniform(-1.0, 1.0, size=(B, H)), rng.normal(size=(B, H)) * 5.0
    dy = rng.normal(size=(T, B, H)) * 10.0 ** rng.uniform(-8, 0, size=(T, B, 1))
    f = lambda a: a.astype(np.float32).astype(np.float64)
    arr = dict(W_ih=f(W_ih), W_hh=f(W_hh), b_ih=f(b_ih), b_hh=f(b_hh), x=f(x), h0=f(h0), c0=f(c0))
    _, _, _, cache = O.lstm_layer_fwd(arr["x"], arr["h0"], arr["c0"], arr["W_ih"], arr["W_hh"], arr["b_ih"], arr["b_hh"])
    dG = R.gate_grads(f(dy), cache, arr["W_hh"])
    arr["dy"] = f(dy) * 2.0 ** np.floor(np.log2(DG_MAX / np.abs(dG).max()))
    return arr


@pytest.mark.parametrize("H,T,B", list(SAT_CASES))
def test_saturated_layer_at_every_plan_branch(H, T, B):
    """zrb_lstm_layer_fwd / _bwd with saturated gates and |c| in the tens, at the shapes (and plan-branch predicate) of
    test_lstm_layer_unit_abi_against_oracle plus two long windows; skips when this device's SM count leads elsewhere."""
    import zaremba_b200
    from zaremba_b200 import _lib
    lib = _lib.load()
    m = zaremba_b200.Model(16, H, 1, 0.0, 0.05, engine="tc").to(R.DEV)
    ctx = m._context(T, B)
    case = SAT_CASES[(H, T, B)]
    plans = _lib.rec_plans(ctx)
    fp, bp = plans["fwd"], plans["bwd"]
    if case not in ("baseline", "long") and not (fp["ok"] and bp["ok"]):
        pytest.skip(f"H={H} B={B} does not fit the persistent kernels on this device: {plans}")
    assert fp["ok"] and bp["ok"], plans
    if case != "long" and not _plan_branch(case, H, B, fp, bp):
        pytest.skip(f"on {torch.cuda.get_device_properties(0).multi_processor_count} SMs H={H} B={B} gets {plans}, "
                    f"not the {case} branch this case is for")
    a = _saturated(H, T, B, 7 * H + T)
    out = R.layer_against_oracle(lib, ctx, a["W_ih"], a["W_hh"], a["b_ih"], a["b_hh"], a["x"], a["h0"], a["c0"], a["dy"])
    bad = []
    for k, v in out.items():
        if k == "db_ih == db_hh":
            assert v == 1.0
        elif isinstance(v, tuple):
            bad += _check(k, v, SAT_TOL, "grad" if "grad" in k else "fwd")
        elif k.startswith("rounded-operand"):
            bad += _check(k, v, dict(fwd=ACT_TOL_PER_H * H) if k.endswith(" y") else ACT_TOL, "fwd")
        else:
            _record(k, v)
    assert out["max_abs_preact"] > 40.0, out                 # the planted units reach the SFU edge cases
    print(f"\n{case} H={H} T={T} B={B}: max|c| {out['max_abs_c']:.1f}, max dG image {out['max_dG_image']:.0f}, "
          f"subnormal dG images {out['frac_dG_image_subnormal']:.3f}")
    assert out["max_abs_c"] > 8.0 and out["frac_dG_image_subnormal"] > 0.01, out       # the regime is reached
    assert not bad, bad


def test_saturated_per_timestep_path_b40():
    """The same saturation at B = 40, which the persistent kernels do not take: one GEMM + one cell launch per step
    (tc_cell.cu, expf / tanhf).  A one-layer model whose embedding rows are the inputs (one token per (t, b)), eval
    forward and backward from a chosen dscores, against the fp64 oracle."""
    import zaremba_b200
    from zaremba_b200 import _lib
    H, T, B = 650, 35, 40
    V = T * B
    a = _saturated(H, T, B, 11)
    rng = np.random.default_rng(12)
    tok = rng.permutation(V).reshape(T, B)
    emb = np.zeros((V, H))
    emb[tok.reshape(-1)] = a["x"].reshape(-1, H)
    params = {"embed.W": emb, "rnns.0.weight_ih_l0": a["W_ih"], "rnns.0.weight_hh_l0": a["W_hh"],
              "rnns.0.bias_ih_l0": a["b_ih"], "rnns.0.bias_hh_l0": a["b_hh"],
              "fc.W": rng.normal(size=(V, H)) * 0.1, "fc.b": rng.normal(size=V)}
    params = {k: v.astype(np.float32).astype(np.float64) for k, v in params.items()}
    m = zaremba_b200.Model(V, H, 1, 0.0, 0.05, engine="tc")
    m.load_state_dict({k: torch.tensor(v, dtype=torch.float32) for k, v in params.items()})
    m = m.to(R.DEV).eval()
    assert not _lib.rec_plans(m._context(T, B))["fwd"]["ok"], "B = 40 should not fit the persistent kernels"
    st0 = [(a["h0"], a["c0"])]
    sc, st, cache = O.model_fwd(params, tok, st0, 1)
    dS = rng.normal(size=(T * B, V)) * 10.0 ** rng.uniform(-8, 0, size=(T * B, 1))
    dG = R.layer_grads(params, cache, dS, 1)[0]["dG"]
    dS = (dS * 2.0 ** np.floor(np.log2(DG_MAX / np.abs(dG).max()))).astype(np.float32).astype(np.float64)
    assert np.abs(dS).max() * R.GRAD_SCALE * CLAMP_MARGIN < R.F16_MAX
    grads = O.model_bwd(params, cache, dS, 1)
    dG = R.layer_grads(params, cache, dS, 1)[0]["dG"]
    states = [(torch.tensor(a["h0"], dtype=torch.float32).view(1, B, H).to(R.DEV),
               torch.tensor(a["c0"], dtype=torch.float32).view(1, B, H).to(R.DEV))]
    scores, states = m(torch.tensor(tok), states)
    scores.backward(torch.tensor(dS, dtype=torch.float32, device=R.DEV))
    bad = _check("B=40 scores", R.rel(scores.detach().cpu().numpy(), sc), SAT_TOL, "fwd")
    bad += _check("B=40 hT", R.rel(states[0][0].reshape(B, H).cpu().numpy(), st[0][0]), SAT_TOL, "fwd")
    bad += _check("B=40 cT", R.rel(states[0][1].reshape(B, H).cpu().numpy(), st[0][1]), SAT_TOL, "fwd")
    for k, p in m.named_parameters():
        bad += _check(f"B=40 grad {k}", R.rel(p.grad.cpu().numpy(), grads[k]), SAT_TOL, "grad")
    img = np.abs(dG) * R.GRAD_SCALE
    _record("B=40 frac_dG_image_subnormal", ((img < R.F16_MIN_NORMAL) & (img > 0)).mean())
    _record("B=40 max_abs_c", max(np.abs(e[6]).max() for e in cache["layer_cache"][0]))
    assert not bad, bad


def test_per_timestep_activations_against_rounded_operands():
    """One step at B = 40 (the per-timestep path: tc_cell.cu's expf / tanhf) with the saturated weights and the planted
    units, against the rounded-operand oracle: the activation implementations are compared where they differ."""
    import zaremba_b200
    from zaremba_b200 import _lib
    H, T, B = 650, 1, 40
    V = T * B
    a = _saturated(H, T, B, 13)
    tok = np.arange(V).reshape(T, B)
    params = {"embed.W": a["x"].reshape(V, H), "rnns.0.weight_ih_l0": a["W_ih"], "rnns.0.weight_hh_l0": a["W_hh"],
              "rnns.0.bias_ih_l0": a["b_ih"], "rnns.0.bias_hh_l0": a["b_hh"], "fc.W": np.zeros((V, H)), "fc.b": np.zeros(V)}
    m = zaremba_b200.Model(V, H, 1, 0.0, 0.05, engine="tc")
    m.load_state_dict({k: torch.tensor(v, dtype=torch.float32) for k, v in params.items()})
    m = m.to(R.DEV).eval()
    assert not _lib.rec_plans(m._context(T, B))["fwd"]["ok"], "B = 40 should not fit the persistent kernels"
    states = [(torch.tensor(a["h0"], dtype=torch.float32).view(1, B, H).to(R.DEV),
               torch.tensor(a["c0"], dtype=torch.float32).view(1, B, H).to(R.DEV))]
    with torch.no_grad():
        _, states = m(torch.tensor(tok), states)
    hd = states[0][0].reshape(1, B, H).cpu().numpy().astype(np.float64)
    cd = states[0][1].reshape(B, H).cpu().numpy().astype(np.float64)
    y_r, c_r, zmax = R.rounded_operand_fwd(a["x"], a["h0"], a["c0"], a["W_ih"], a["W_hh"], a["b_ih"], a["b_hh"], hd)
    bad = _check("B=40 rounded-operand y", float(np.abs(hd - y_r).max()), dict(fwd=ACT_TOL_PER_H * H), "fwd")
    bad += _check("B=40 rounded-operand cT", float(np.abs(cd - c_r).max() / max(np.abs(c_r).max(), 1.0)), ACT_TOL, "fwd")
    assert zmax > 40.0, zmax
    assert not bad, bad


# ---------------------------------------------------------------------------------------------------------------------
# C. short training-trajectory parity
# ---------------------------------------------------------------------------------------------------------------------
def test_small_training_trajectory_engines_agree():
    """The Small recipe (dropout 0: no masks to share) for TRAJ_STEPS fused steps from one init on the same PTB windows,
    tensor-core engine (lazy update) against the fp32 validation engine: mean loss of the last 50 steps and valid
    perplexity."""
    out = R.trajectory(TRAJ_STEPS)
    for e in ("tc", "simt"):
        for k, v in out[e].items():
            _record(f"{e} {k}", v)
    _record("last50_loss_rel_gap", out["last50_loss_rel_gap"])
    _record("ppl_rel_gap", out["ppl_rel_gap"])
    print(f"\n{out}")
    assert out["tc"]["ppl"] * 5 < out["tc"]["ppl_init"], out          # the run learned something
    assert out["last50_loss_rel_gap"] <= TRAJ_TOL["loss"], out
    assert out["ppl_rel_gap"] <= TRAJ_TOL["ppl"], out


def test_zz_write_measured_errors():
    """Not a check: dumps what every GPU test of the session measured, these included (ZRB_ERROR_REPORT2=path)."""
    import json
    import os
    out = os.environ.get("ZRB_ERROR_REPORT2")
    if out and MEASURED:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        json.dump(MEASURED, open(out, "w"), indent=1, default=float)
