"""GPU parity at the EXACT shapes of BASELINE.json configs[0..2] (README.md:20-27 recipes, V = 10000):
Small 2x200 / T=20, Medium 2x650 / T=35 / p=0.5, Large 2x1500 / T=35 / p=0.65, B=20.

The fixtures `tests/golden/{small,medium,large}_cfg_summary.npz` were minted by tests/golden/make_golden.py
from the UNMODIFIED reference (`Model(..., "pytorch")` on CPU fp32, two carried train steps of main.py:109-117,
train mode, the reference's own dropout masks recorded bit-packed).  They hold summaries (the tensors are up to
60 MB each): loss, clip norm, 8 score rows x 64 columns, per-tensor gradient L2 norms and the first 32 gradient
elements, per-tensor sums and first 32 elements of the parameters AFTER the update, and the full (h, c) states.
Initial weights are re-derived from the seed (seed-for-seed construction is itself checked).

H=650 pads to Hp=704 / Kc=82 and H=200 to Hp=256 / Kc=26: other recurrence plans (units per CTA, CTA count) than
H=1500's, which is the shape class a plan bug would hide in.

Tolerances (relative to the compared quantity's own scale), ~3x what was measured on an H100
(ZRB_ERROR_REPORT=<path> writes the measurements):
  simt (fp32 CUDA cores)                         loss 2e-5, scores/states 5e-5, gradient norms 1e-4
  tc   (wgmma, fp16 operands, fp32 accumulate)    loss 3e-4, scores/states 1.5e-3, gradient norms 1.5e-3,
                                                 gradient heads 1e-2 of the head's max
The reference's OWN `clip_grad_norm_` on CPU is only good to ~1e-3 at Large (fp32 accumulation over 66 M
squares: the per-tensor L2 norms recomputed in fp64 from the same gradients give 1.8734, torch reported 1.8715),
so the clip norm is compared with the norm recomputed from the fixture's per-tensor L2s; the reference's own figure
is held to 2.5e-3.  No config clips in these steps (norm < max_norm), so the parameter update does not depend on it.
"""
import os

import numpy as np
import pytest
import torch

from oracle import lstm_lm_oracle as O
from tests._golden import GOLDEN

pytestmark = pytest.mark.gpu

ENGINES = os.environ.get("ZRB_TEST_ENGINES", "simt,tc").split(",")
CASES = ["small_cfg_summary", "medium_cfg_summary", "large_cfg_summary"]
TOL = {"simt": dict(loss=2e-5, fwd=5e-5, l2=1e-4, head=2e-3, psum=2e-6),
       "tc": dict(loss=3e-4, fwd=1.5e-3, l2=1.5e-3, head=1e-2, psum=1e-4)}
MEASURED = {}      # filled while the tests run; written by the last test (ZRB_ERROR_REPORT)


def _dev():
    return torch.device("cuda:0")


def _rel(got, want, scale=None):
    got = np.asarray(got, dtype=np.float64); want = np.asarray(want, dtype=np.float64)
    scale = max(np.abs(want).max(), 1e-30) if scale is None else scale
    return float(np.abs(got - want).max() / scale)


class Summary:
    def __init__(self, name):
        self.z = z = np.load(os.path.join(GOLDEN, name + ".npz"))
        self.V, self.H, self.L, self.T, self.B, self.steps = [int(v) for v in z["meta"]]
        self.p, self.lr, self.max_norm = float(z["dropout"]), float(z["lr"]), float(z["max_norm"])
        self.winit, self.seed = float(z["winit"]), int(z["seed"])
        self.names = O.param_names(self.L)

    def model(self, engine):
        import zaremba_b200
        torch.manual_seed(self.seed)
        m = zaremba_b200.Model(self.V, self.H, self.L, self.p, self.winit, engine=engine)
        for k, v in m.named_parameters():       # seed-for-seed with the reference (model.py:76-92)
            a = v.detach().numpy().astype(np.float64)
            np.testing.assert_allclose([a.sum(), np.abs(a).sum(), (a * a).sum()], self.z["param0_sum/" + k], rtol=1e-12)
        m = m.to(_dev())
        m.train() if self.p > 0 else m.eval()
        return m

    def xy(self, s):
        return torch.tensor(self.z[f"s{s}/x"]), torch.tensor(self.z[f"s{s}/y"])

    def masks(self, s):
        if self.p == 0:
            return None
        n = self.T * self.B * self.H
        return [torch.tensor(np.unpackbits(self.z[f"s{s}/mask/{i}"])[:n].reshape(self.T, self.B, self.H)).to(_dev())
                for i in range(self.L + 1)]

    def norm_from_l2(self, s):
        return float(np.sqrt(sum(float(self.z[f"s{s}/grad_l2/" + k]) ** 2 for k in self.names)))


def _check_states(c, s, states, tol, tag, rec):
    for l in range(c.L):
        for j, nm in enumerate("hc"):
            e = _rel(states[l][j].reshape(c.B, c.H).cpu().numpy(), c.z[f"s{s}/{nm}/{l}"])
            rec[f"s{s}/{nm}{l}"] = e
            assert e <= tol["fwd"], f"{tag} s{s} {nm}{l}: {e:.2e}"


def _check_params_after(c, s, m, tol, tag, rec):
    for k, prm in m.named_parameters():
        a = prm.detach().cpu().numpy()
        head = c.z[f"s{s}/param_head/" + k]
        e = _rel(a.reshape(-1)[:32], head, max(np.abs(head).max(), c.winit))
        sums = c.z[f"s{s}/param_sum/" + k]
        a64 = a.astype(np.float64)
        e2 = abs(np.abs(a64).sum() - sums[1]) / sums[1]
        rec[f"s{s}/param/{k}"] = max(e, e2)
        assert e <= tol["head"] * 0.1 and e2 <= tol["psum"], f"{tag} s{s} param {k}: head {e:.2e} |sum| {e2:.2e}"


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", CASES)
def test_dropin_loop_at_baseline_shapes(name, engine):
    """main.py:109-117 verbatim (eager loss, clip_grad_norm_, per-parameter SGD) on the drop-in Model."""
    from tests.test_gpu_parity import _caller_nll_loss
    c = Summary(name)
    tol = TOL[engine]
    m = c.model(engine)
    rec = MEASURED.setdefault(f"dropin/{name}/{engine}", {})
    states = m.state_init(c.B)
    N = c.T * c.B
    for s in range(c.steps):
        x, y = c.xy(s)
        x, y = x.t().contiguous().t(), y.t().contiguous().t()     # non-contiguous CPU views like main.py:71-72
        if c.p > 0:
            m.set_explicit_dropout_masks(c.masks(s))
        m.zero_grad()
        states = m.detach(states)
        scores, states = m(x, states)
        loss = _caller_nll_loss(scores, y)
        loss.backward()
        want = float(c.z[f"s{s}/loss"])
        rec[f"s{s}/loss"] = abs(loss.item() - want) / want
        assert rec[f"s{s}/loss"] <= tol["loss"], (loss.item(), want)
        sc = scores.detach().cpu().numpy()
        e = _rel(sc[:: max(1, N // 8)][:, :64], c.z[f"s{s}/scores_rows"])
        rec[f"s{s}/scores_rows"] = e
        assert e <= tol["fwd"], f"{name} s{s} score rows {e:.2e}"
        asum = np.abs(sc.astype(np.float64)).sum()
        assert abs(asum - c.z[f"s{s}/scores_sum"][1]) <= tol["fwd"] * c.z[f"s{s}/scores_sum"][1]
        for k, prm in m.named_parameters():
            g = prm.grad.detach().cpu().numpy()
            l2, ref = float(np.sqrt((g.astype(np.float64) ** 2).sum())), float(c.z[f"s{s}/grad_l2/" + k])
            head = c.z[f"s{s}/grad_head/" + k]
            eh = _rel(g.reshape(-1)[:32], head, max(np.abs(head).max(), ref / np.sqrt(g.size)))
            rec[f"s{s}/grad_l2/{k}"] = abs(l2 - ref) / ref
            rec[f"s{s}/grad_head/{k}"] = eh
            assert abs(l2 - ref) <= tol["l2"] * ref, f"{name} s{s} |grad {k}| {l2} vs {ref}"
            assert eh <= tol["head"], f"{name} s{s} grad head {k}: {eh:.2e}"
        with torch.no_grad():
            norm = float(torch.nn.utils.clip_grad_norm_(m.parameters(), c.max_norm))
            for prm in m.parameters():
                prm -= c.lr * prm.grad
        assert norm < c.max_norm                       # these steps do not clip
        rec[f"s{s}/norm_vs_l2"] = abs(norm - c.norm_from_l2(s)) / c.norm_from_l2(s)
        assert rec[f"s{s}/norm_vs_l2"] <= tol["l2"] + 1e-3   # + torch's own fp32 foreach-norm accuracy on the GPU side
        _check_params_after(c, s, m, tol, name, rec)
        _check_states(c, s, states, tol, name, rec)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", CASES)
def test_fused_trainer_at_baseline_shapes(name, engine):
    """The fused step (zrb_train_step_grads + zrb_train_step_update: epilogue-fed clip norm, rows-only embedding
    update, fp16 image rebuild) over the same two carried steps, train mode, the reference's masks."""
    import zaremba_b200
    c = Summary(name)
    tol = TOL[engine]
    m = c.model(engine)
    tr = zaremba_b200.Trainer(m, c.B, c.T)
    rec = MEASURED.setdefault(f"trainer/{name}/{engine}", {})
    for s in range(c.steps):
        x, y = c.xy(s)
        if c.p > 0:
            m.set_explicit_dropout_masks(c.masks(s))
        loss, norm = tr.train_step(x.to(_dev()).contiguous(), y.to(_dev()).contiguous(), c.lr, c.max_norm)
        want = float(c.z[f"s{s}/loss"])
        rec[f"s{s}/loss"] = abs(loss.item() - want) / want
        assert rec[f"s{s}/loss"] <= tol["loss"], (loss.item(), want)
        nref = c.norm_from_l2(s)
        rec[f"s{s}/norm_vs_l2"] = abs(norm.item() - nref) / nref
        rec[f"s{s}/norm_vs_reference_clip_grad_norm"] = abs(norm.item() - float(c.z[f"s{s}/norm"])) / nref
        assert rec[f"s{s}/norm_vs_l2"] <= tol["l2"], (norm.item(), nref)
        assert rec[f"s{s}/norm_vs_reference_clip_grad_norm"] <= 2.5e-3
        _check_params_after(c, s, m, tol, name, rec)
        _check_states(c, s, tr.states, tol, name, rec)


@pytest.mark.parametrize("engine", ENGINES)
def test_large_fused_trainer_philox_step_against_fp64_oracle(engine):
    """BASELINE configs[2], train mode at p=0.65 with the library's own Philox masks (the fp64 oracle gets the same
    masks from the independent generator oracle/philox.py): loss, clip norm and every UPDATED weight tensor of the
    fused `Trainer` step, with a max_norm that makes the clip active."""
    import zaremba_b200
    from oracle import philox as PH
    V, H, L, T, B, p = 10000, 1500, 2, 35, 20, 0.65
    torch.manual_seed(1)
    m = zaremba_b200.Model(V, H, L, p, 0.04, engine=engine).to(_dev())
    m.train()
    params = {k: v.detach().cpu().numpy().astype(np.float64) for k, v in m.named_parameters()}
    tr = zaremba_b200.Trainer(m, B, T)
    g = torch.Generator().manual_seed(2)
    data = torch.randint(0, V, (B, T + 1), generator=g)
    x, y = data[:, :T].t().contiguous(), data[:, 1:].t().contiguous()
    max_norm, lr = 1.0, 1.0                            # the step's norm is ~1.9: coef ~0.53
    seed, step = tr.seed, tr.step
    loss, norm = tr.train_step(x.to(_dev()), y.to(_dev()), lr, max_norm)
    masks = PH.site_masks(seed, step, L, T, B, H, p)
    assert abs(np.mean([mk.mean() for mk in masks]) - (1 - p)) < 2e-3
    sc, st, cache = O.model_fwd(params, x.numpy(), O.zero_states(L, B, H, np.float64), L, p, masks)
    want_loss = O.nll_loss(sc, y.numpy())
    grads = O.model_bwd(params, cache, O.nll_loss_bwd(sc, y.numpy()), L)
    want_norm = O.clip_sgd(params, grads, lr, max_norm, O.param_names(L))     # updates `params` in place
    assert want_norm > 1.5 * max_norm
    tol = dict(loss=3e-4, norm=1.5e-3, upd=2e-3) if engine == "tc" else dict(loss=2e-5, norm=1e-4, upd=1e-4)
    rec = MEASURED.setdefault(f"philox_large/{engine}", {})
    rec["loss"] = abs(loss.item() - want_loss) / want_loss
    rec["norm"] = abs(norm.item() - want_norm) / want_norm
    assert rec["loss"] <= tol["loss"] and rec["norm"] <= tol["norm"], (loss.item(), want_loss, norm.item(), want_norm)
    coef = max_norm / (want_norm + 1e-6)
    for k, prm in m.named_parameters():
        # error of the UPDATE (new - old) relative to the largest update element of the tensor
        upd_scale = lr * coef * np.abs(grads[k]).max()
        e = _rel(prm.detach().cpu().numpy(), params[k], upd_scale)
        rec[f"updated/{k}"] = e
        assert e <= tol["upd"], f"updated {k}: {e:.2e} of the largest update"
    for l in range(L):
        assert _rel(tr.states[l][0].reshape(B, H).cpu().numpy(), st[l][0]) <= (1.5e-3 if engine == "tc" else 5e-5)


def test_zz_write_measured_errors():
    """Not a check: dumps the errors the tests above measured (ZRB_ERROR_REPORT=path)."""
    import json
    out = os.environ.get("ZRB_ERROR_REPORT")
    if out and MEASURED:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        worst = {k: {"max": max(v.values()), "worst_key": max(v, key=v.get), "all": v} for k, v in MEASURED.items() if v}
        json.dump(worst, open(out, "w"), indent=1)
