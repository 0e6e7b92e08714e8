"""GPU parity tests: the CUDA path (through the C ABI, via zaremba_b200.Model / Trainer and
direct ctypes calls) against the reference fixtures and the numpy oracle.

Tolerances (stated per engine):
  simt  fp32 CUDA-core engine: differs from the fp32 reference only by summation order
        -> 5e-5 relative to the tensor's scale.
  tc    tensor-core engine: fp16 operands (11-bit significand, the same as the TF32 the
        reference's own cuDNN path uses on GPU), fp32 accumulation -> 1.2e-3 relative to the
        tensor's scale on logits/states, 4e-3 on gradients and updated parameters: about three times
        the largest error measured over the fixture cases (see DESIGN.md, "Numerics").
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import lstm_lm_oracle as O
from tests._golden import GOLDEN, STEP_CASES, StepCase

pytestmark = pytest.mark.gpu

ENGINES = os.environ.get("ZRB_TEST_ENGINES", "simt,tc").split(",")
# tc: ~3x the largest error measured over all fixture cases on an H100 (ZRB_ERROR_REPORT2=<path> writes them:
# logits/states <= 3.6e-4, gradients / updated parameters <= 1.3e-3 of the tensor's scale)
TOL = {"simt": dict(fwd=5e-5, grad=1e-4, loss=2e-5), "tc": dict(fwd=1.2e-3, grad=4e-3, loss=1e-3)}


def _dev():
    return torch.device("cuda:0")


MEASURED = {}      # what -> largest relative error seen (dumped by test_zz_write_measured_errors)


def _scale_close(got, want, rel, what):
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=np.float64)
    scale = max(np.abs(want).max(), 1e-6)
    err = np.abs(got - want).max()
    key = os.environ.get("PYTEST_CURRENT_TEST", "?").split("::")[-1].split(" ")[0]
    kind = "grad" if ("grad" in what or "param" in what) else "fwd"
    MEASURED.setdefault(key, {}).setdefault(kind, 0.0)
    MEASURED[key][kind] = max(MEASURED[key][kind], float(err / scale))
    assert err <= rel * scale, f"{what}: max abs err {err:.3e} vs scale {scale:.3e} (rel {err / scale:.2e} > {rel:.1e})"


def _caller_nll_loss(scores, y):
    """what main.py:77-84 does with our scores (torch ops on the CALLER's side of the boundary)."""
    B = y.size(1)
    e = scores.exp()
    p = e / e.sum(1, keepdim=True)
    yy = y.reshape(-1).to(scores.device)
    return torch.mean(-torch.log(p[torch.arange(yy.numel(), device=scores.device), yy]) * B)


def _model_from_case(c, engine, lstm_type=None):
    import zaremba_b200
    lstm_type = lstm_type or c.lstm_type
    m = zaremba_b200.Model(c.V, c.H, c.L, c.dropout, c.winit, lstm_type, engine=engine)
    raw = {k[len("param0/"):]: c.z[k] for k in c.z.files if k.startswith("param0/")}
    sd = m.state_dict()
    assert sorted(sd) == sorted(raw), (sorted(sd), sorted(raw))
    m.load_state_dict({k: torch.tensor(v) for k, v in raw.items()})
    return m.to(_dev())


def _states_to_model(c, m):
    sts = []
    for h, cc in c.states0():
        shape = (c.B, c.H) if m.lstm_type == "custom" else (1, c.B, c.H)
        sts.append((torch.tensor(h).view(shape).to(_dev()), torch.tensor(cc).view(shape).to(_dev())))
    return sts


def _grads_pytorch_order(c, m):
    g = {k: p.grad.detach().cpu().numpy() for k, p in m.named_parameters()}
    return O.custom_state_dict_to_pytorch(g) if c.lstm_type == "custom" else g


def _params_pytorch_order(c, m):
    g = {k: p.detach().cpu().numpy() for k, p in m.named_parameters()}
    return O.custom_state_dict_to_pytorch(g) if c.lstm_type == "custom" else g


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", STEP_CASES)
def test_dropin_train_steps_match_reference(name, engine):
    """The reference's own loop (main.py:109-117) run against the drop-in Model, compared
    with what the reference recorded for the same weights, tokens, states and dropout masks."""
    c = StepCase(name)
    tol = TOL[engine]
    m = _model_from_case(c, engine)
    m.train() if c.dropout > 0 else m.eval()
    states = _states_to_model(c, m)
    for s in range(c.steps):
        x = torch.tensor(c.x(s)).t().contiguous().t()      # non-contiguous CPU view like main.py:71
        y = torch.tensor(c.y(s)).t().contiguous().t()
        if c.dropout > 0:
            m.set_explicit_dropout_masks([torch.tensor(mk).to(_dev()) for mk in c.masks(s)])
        m.zero_grad()
        states = m.detach(states)
        scores, states = m(x, states)
        loss = _caller_nll_loss(scores, y)
        loss.backward()
        _scale_close(scores.detach().cpu().numpy(), c.scores(s), tol["fwd"], f"{name} s{s} scores")
        assert abs(loss.item() - c.loss(s)) <= tol["loss"] * max(1.0, abs(c.loss(s)))
        grads = _grads_pytorch_order(c, m)
        ref_grads = c.grads(s)
        for k in c.names:
            _scale_close(grads[k], ref_grads[k], tol["grad"], f"{name} s{s} grad {k}")
        with torch.no_grad():
            norm = torch.nn.utils.clip_grad_norm_(m.parameters(), c.max_norm)
            for p in m.parameters():
                p -= c.lr * p.grad
        assert abs(float(norm) - c.norm(s)) <= tol["grad"] * max(1.0, c.norm(s))
        after = _params_pytorch_order(c, m)
        ref_after = c.params_after(s)
        for k in c.names:
            _scale_close(after[k], ref_after[k], tol["grad"], f"{name} s{s} param {k}")
        for l, (h, cc) in enumerate(c.states_after(s)):
            _scale_close(states[l][0].reshape(c.B, c.H).cpu().numpy(), h, tol["fwd"], f"{name} s{s} h{l}")
            _scale_close(states[l][1].reshape(c.B, c.H).cpu().numpy(), cc, tol["fwd"], f"{name} s{s} c{l}")


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", ["tiny_pytorch", "tiny_dropout", "tiny_carry3", "mid_H72", "edge_T1_B1_L1"])
def test_fused_trainer_matches_reference(name, engine):
    """zrb_train_step_grads + zrb_train_step_update (one library call per half step)."""
    import zaremba_b200
    c = StepCase(name)
    tol = TOL[engine]
    m = _model_from_case(c, engine)
    m.train()
    tr = zaremba_b200.Trainer(m, c.B, c.T)
    for l, (h, cc) in enumerate(c.states0()):
        tr.states[l][0].copy_(torch.tensor(h).view_as(tr.states[l][0]))
        tr.states[l][1].copy_(torch.tensor(cc).view_as(tr.states[l][1]))
    for s in range(c.steps):
        x = torch.tensor(c.x(s)).to(_dev()).contiguous()
        y = torch.tensor(c.y(s)).to(_dev()).contiguous()
        if c.dropout > 0:
            m.set_explicit_dropout_masks([torch.tensor(mk).to(_dev()) for mk in c.masks(s)])
        loss, norm = tr.train_step(x, y, c.lr, c.max_norm)
        assert abs(loss.item() - c.loss(s)) <= tol["loss"] * max(1.0, abs(c.loss(s)))
        assert abs(norm.item() - c.norm(s)) <= tol["grad"] * max(1.0, c.norm(s))
        after = _params_pytorch_order(c, m)
        ref_after = c.params_after(s)
        for k in c.names:
            _scale_close(after[k], ref_after[k], tol["grad"], f"{name} s{s} param {k}")
        for l, (h, cc) in enumerate(c.states_after(s)):
            _scale_close(tr.states[l][0].reshape(c.B, c.H).cpu().numpy(), h, tol["fwd"], f"{name} s{s} h{l}")


@pytest.mark.parametrize("engine", ENGINES)
def test_keep_clipped_grads_option(engine):
    """clip_grad_norm_ (main.py:115) leaves coef * g in .grad.  keep_clipped_grads=True reproduces that;
    the default skips the dead store: same weights, loss and norm, .grad = the raw gradients."""
    import zaremba_b200
    c = StepCase("mid_H72")
    x = torch.tensor(c.x(0)).to(_dev()).contiguous()
    y = torch.tensor(c.y(0)).to(_dev()).contiguous()
    max_norm = 0.5 * c.norm(0)                      # make sure the clip is active (coef = 0.5)
    res = []
    for keep in (True, False):
        m = _model_from_case(c, engine)
        m.eval()                                    # no dropout: both runs see the same gradients
        tr = zaremba_b200.Trainer(m, c.B, c.T, keep_clipped_grads=keep)
        loss, norm = tr.train_step(x, y, c.lr, max_norm)
        res.append((loss.item(), norm.item(), tr.flat_p.clone(), tr.flat_g.clone()))
    (l1, n1, p1, g1), (l0, n0, p0, g0) = res
    # two separate runs: atomics in the embedding scatter may order differently -> last-bit tolerance
    assert abs(l1 - l0) <= 1e-6 * abs(l0) and abs(n1 - n0) <= 1e-6 * n0, (l1, l0, n1, n0)
    torch.testing.assert_close(p1, p0, rtol=1e-6, atol=1e-7)
    coef = min(1.0, max_norm / (n1 + 1e-6))
    assert coef < 0.75
    scale = g0.abs().max().item()
    assert (g1 - g0 * coef).abs().max().item() <= 1e-5 * scale, "kept gradients are coef * raw gradients"
    assert (g0 - g1).abs().max().item() > 0.1 * scale, "default leaves the raw gradients"


def test_lazy_update_equals_strict_update():
    """Trainer(lazy_update=True) defers the upper-layer / fc weight updates to run beside the next step's forward
    recurrences: after flush() the parameters must equal the strict schedule's (same arithmetic per element), eval in
    between must see the updated weights without an explicit flush, and an un-flushed read shows what the docstring
    says (fc.W still holding the previous step's values)."""
    import zaremba_b200
    c = StepCase("mid_H72")
    res = {}
    for lazy in (False, True):
        m = _model_from_case(c, "tc")
        m.train()
        tr = zaremba_b200.Trainer(m, c.B, c.T, lazy_update=lazy)
        x = torch.tensor(c.x(0)).to(_dev()).contiguous()
        y = torch.tensor(c.y(0)).to(_dev()).contiguous()
        fc_before = m.fc.W.detach().clone()
        losses = []
        for s in range(3):
            loss, norm = tr.train_step(x, y, c.lr, 0.5 * c.norm(0))
            losses.append(loss.item())
            if s == 0 and lazy:
                torch.cuda.synchronize()
                assert torch.equal(m.fc.W.detach(), fc_before), "fc.W update should still be pending"
            if s == 1:
                m.eval()
                ev = tr.eval_step(x, y).item()          # applies what is pending first
                m.train()
        tr.flush()
        torch.cuda.synchronize()
        res[lazy] = (losses, ev, tr.flat_p.clone())
    for a, b in zip(res[False][0], res[True][0]):
        assert abs(a - b) <= 1e-6 * abs(a), (res[False][0], res[True][0])
    assert abs(res[False][1] - res[True][1]) <= 1e-6 * abs(res[False][1])
    torch.testing.assert_close(res[True][2], res[False][2], rtol=1e-6, atol=1e-7)


def test_recurrence_launch_modes_agree():
    """The persistent recurrence kernels are launched as programmatic dependents of the GEMM before them while ONE
    tensor-core context is alive on the device, and cooperatively as soon as a second one exists (tc_common.cuh,
    rec_launch_programmatic): both launches must give the same bits.  H = 256 takes the K-split (cluster) kernels.
    Every window holds distinct tokens: a token that occurs three times would make the embedding scatter's fp32
    atomics round differently from run to run, whatever the launch mode."""
    import gc
    import zaremba_b200
    V, H, L, T, B = 500, 256, 2, 9, 8
    g = torch.Generator().manual_seed(11)
    xs = [torch.randperm(V, generator=g)[:T * B].view(T, B) for _ in range(3)]
    ys = [torch.randint(0, V, (T, B), generator=g) for _ in range(3)]

    def run(tr):
        out = []
        for i in range(3):
            x = xs[i].contiguous().to(_dev())
            y = ys[i].contiguous().to(_dev())
            loss, norm = tr.train_step(x, y, 1.0, 0.25)
            out.append((loss.item(), norm.item()))
        tr.flush()
        torch.cuda.synchronize()
        return out, tr.flat_p.clone()

    def make():
        torch.manual_seed(5)
        m = zaremba_b200.Model(V, H, L, 0.0, 0.1).to(_dev())
        m.train()
        return m, zaremba_b200.Trainer(m, B, T)

    gc.collect()
    m1, t1 = make()
    alone = run(t1)                 # (programmatic if no context of an earlier test is still alive)
    t1.close(); del m1, t1
    gc.collect()
    m2, t2 = make()
    m3, t3 = make()                 # a second live context: both now launch cooperatively
    both = run(t2)
    assert alone[0] == both[0], (alone[0], both[0])
    assert torch.equal(alone[1], both[1])


@pytest.mark.parametrize("engine", ENGINES)
def test_host_buffer_step_equals_device_step(engine):
    """zrb_train_step_host (H2D/D2H inside) == device-token step, bit for bit in eval of loss."""
    import zaremba_b200
    c = StepCase("mid_H72")
    outs = []
    for mode in ("dev", "host"):
        m = _model_from_case(c, engine)
        m.train()
        tr = zaremba_b200.Trainer(m, c.B, c.T)
        x, y = torch.tensor(c.x(0)), torch.tensor(c.y(0))
        if mode == "dev":
            loss, norm = tr.train_step(x.to(_dev()).contiguous(), y.to(_dev()).contiguous(), c.lr, c.max_norm)
            outs.append((loss.item(), norm.item(), tr.flat_p.clone()))
        else:
            loss, norm = tr.train_step_host(x.t().contiguous().t(), y.t().contiguous().t(), c.lr, c.max_norm)
            outs.append((loss, norm, tr.flat_p.clone()))
    assert abs(outs[0][0] - outs[1][0]) <= 1e-6 * abs(outs[0][0])
    assert abs(outs[0][1] - outs[1][1]) <= 1e-5 * abs(outs[0][1])
    assert torch.allclose(outs[0][2], outs[1][2], rtol=0, atol=1e-6)


def test_gemm_f32_matches_numpy():
    from zaremba_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(0)
    for (M, N, K, ta, tb) in [(5, 7, 3, 0, 1), (64, 64, 16, 0, 0), (70, 130, 33, 1, 0), (20, 6000, 1500, 0, 1),
                              (1, 1, 1, 1, 1), (129, 65, 257, 1, 1)]:
        A = rng.normal(size=(K, M) if ta else (M, K)).astype(np.float32)
        Bm = rng.normal(size=(N, K) if tb else (K, N)).astype(np.float32)
        C0 = rng.normal(size=(M, N)).astype(np.float32)
        a, b, c = (torch.tensor(v).cuda() for v in (A, Bm, C0))
        _lib.check(lib.zrb_gemm_f32(_lib.ptr(a), _lib.ptr(b), _lib.ptr(c), M, N, K, ta, tb, 0.5, 2.0, None))
        want = 0.5 * ((A.T if ta else A).astype(np.float64) @ (Bm.T if tb else Bm).astype(np.float64)) + 2.0 * C0
        _scale_close(c.cpu().numpy(), want, 2e-6 * max(1, K ** 0.5), f"gemm {M}x{N}x{K}")


@pytest.mark.parametrize("T,B,V", [(35, 20, 10000), (7, 3, 97), (5, 4, 5004), (3, 2, 16384), (2, 2, 16388)])
def test_softmax_nll_against_oracle_and_properties(T, B, V):
    """zrb_softmax_nll vs main.py:77-84 restated; gradient rows sum to ~0; target prob in (0,1].
    V % 4 == 0 and V <= 16384 take the register-resident kernel (2..8 chunks per thread), the rest the scalar one."""
    from zaremba_b200 import _lib
    import zaremba_b200
    lib = _lib.load()
    m = zaremba_b200.Model(V, 8, 1, 0.0, 0.1, engine="simt").to(_dev())
    ctx = m._context(T, B)
    rng = np.random.default_rng(3)
    s = (rng.normal(size=(T * B, V)) * 3).astype(np.float32)
    y = rng.integers(0, V, size=(T, B))
    sd, yd = torch.tensor(s).cuda(), torch.tensor(y).cuda()
    loss = torch.zeros((), device="cuda"); ds = torch.empty_like(sd); tp = torch.empty(T * B, device="cuda")
    _lib.check(lib.zrb_softmax_nll(ctx, _lib.ptr(sd), _lib.ptr(yd), T, B, _lib.ptr(loss), _lib.ptr(ds), _lib.ptr(tp), None))
    want = O.nll_loss(s.astype(np.float64), y)
    assert abs(loss.item() - want) < 2e-6 * want
    _scale_close(ds.cpu().numpy(), O.nll_loss_bwd(s.astype(np.float64), y), 2e-5, "dscores")
    _scale_close(tp.cpu().numpy(), O.target_probs(s.astype(np.float64), y), 2e-5, "target probs")
    assert ds.sum(1).abs().max().item() < 1e-6
    assert (tp > 0).all() and (tp <= 1).all()


def test_clip_sgd_matches_oracle():
    from zaremba_b200 import _lib
    import zaremba_b200
    lib = _lib.load()
    m = zaremba_b200.Model(11, 8, 1, 0.0, 0.1, engine="simt").to(_dev())
    ctx = m._context(2, 2)
    rng = np.random.default_rng(5)
    sizes = [1, 7, 1000003, 64, 12345]
    for max_norm in (1e9, 3.0):
        ps = [rng.normal(size=n).astype(np.float32) for n in sizes]
        gs = [rng.normal(size=n).astype(np.float32) * 0.01 for n in sizes]
        pd = [torch.tensor(v).cuda() for v in ps]; gd = [torch.tensor(v).cuda() for v in gs]
        names = [str(i) for i in range(len(sizes))]
        pp = dict(zip(names, [v.copy() for v in ps])); gg = dict(zip(names, [v.copy() for v in gs]))
        want_norm = O.clip_sgd(pp, gg, 0.7, max_norm, names)
        arr_p = (C.c_void_p * len(sizes))(*[t.data_ptr() for t in pd])
        arr_g = (C.c_void_p * len(sizes))(*[t.data_ptr() for t in gd])
        arr_n = (C.c_int64 * len(sizes))(*sizes)
        norm = torch.zeros((), device="cuda")
        _lib.check(lib.zrb_clip_sgd(ctx, len(sizes), arr_p, arr_g, arr_n, 0.7, max_norm, _lib.ptr(norm), None))
        assert abs(norm.item() - want_norm) < 1e-5 * want_norm
        for i, n in enumerate(names):
            np.testing.assert_allclose(pd[i].cpu().numpy(), pp[n], rtol=1e-5, atol=1e-7)
            np.testing.assert_allclose(gd[i].cpu().numpy(), gg[n], rtol=1e-5, atol=1e-9)


@pytest.mark.parametrize("engine", ENGINES)
def test_large_config_against_fp64_oracle(engine):
    """BASELINE.json configs[2] shape (2x1500, T=35, B=20, V=10000), eval mode: logits, loss and
    final states vs the fp64 oracle; plus size-independent properties (determinism,
    linearity of backward in dscores)."""
    import zaremba_b200
    V, H, L, T, B = 10000, 1500, 2, 35, 20
    torch.manual_seed(1)
    m = zaremba_b200.Model(V, H, L, 0.65, 0.04, engine=engine).to(_dev())
    m.eval()
    g = torch.Generator().manual_seed(2)
    data = torch.randint(0, V, (B, T + 1), generator=g)
    x, y = data[:, :T].t(), data[:, 1:].t()
    with torch.no_grad():
        scores_a, _ = m(x, m.state_init(B))
        scores_b, _ = m(x, m.state_init(B))
    assert torch.equal(scores_a, scores_b), "forward is not deterministic"
    scores, states = m(x, m.state_init(B))
    assert torch.equal(scores, scores_a)
    params = {k: v.detach().cpu().numpy().astype(np.float64) for k, v in m.named_parameters()}
    sc, st, cache = O.model_fwd(params, x.numpy(), O.zero_states(L, B, H, np.float64), L)
    # measured at this config (tools/measure_error.py): tc 3.4e-4 logits / <= 5.7e-4 grads of each tensor's
    # scale; the reference's own cuDNN-TF32 path 1.7e-4 / <= 4.7e-4.  Held to ~3x the measurement here.
    tol = dict(TOL[engine], fwd=1.2e-3, grad=2e-3) if engine == "tc" else TOL[engine]
    _scale_close(scores.detach().cpu().numpy(), sc, tol["fwd"], "L logits")
    for l in range(L):
        _scale_close(states[l][0].reshape(B, H).cpu().numpy(), st[l][0], tol["fwd"], f"L h{l}")
        _scale_close(states[l][1].reshape(B, H).cpu().numpy(), st[l][1], tol["fwd"], f"L c{l}")
    loss = _caller_nll_loss(scores, y)
    want = O.nll_loss(sc, y.numpy())
    assert abs(loss.item() - want) < tol["loss"] * want
    # backward: linear in dscores
    loss.backward()
    g1 = {k: p.grad.clone() for k, p in m.named_parameters()}
    m.zero_grad()
    scores, _ = m(x, m.state_init(B))
    (2.0 * _caller_nll_loss(scores, y)).backward()
    lin = 2e-5 if engine == "simt" else 2e-3   # fp16 images round differently near the subnormal range
    for k, p in m.named_parameters():
        _scale_close(p.grad.cpu().numpy(), 2.0 * g1[k].cpu().numpy(), lin, f"linearity {k}")
    grads = O.model_bwd(params, cache, O.nll_loss_bwd(sc, y.numpy()), L)
    for k in grads:
        _scale_close(g1[k].cpu().numpy(), grads[k], tol["grad"], f"L grad {k}")


@pytest.mark.parametrize("engine", ENGINES)
def test_perplexity_and_ensemble_on_ptb_slice(engine):
    """main.py:86-95 and ensemble.py:97-109 through Trainer.perplexity / eval_step."""
    import zaremba_b200
    z = np.load(os.path.join(GOLDEN, "perplexity_ptb_slice.npz"))
    V, H, L, T, B = [int(v) for v in z["meta"]]
    ms = []
    for pre in ("param/", "param2/"):
        m = zaremba_b200.Model(V, H, L, 0.0, 0.1, engine=engine)
        m.load_state_dict({k[len(pre):]: torch.tensor(z[k]) for k in z.files if k.startswith(pre)})
        ms.append(m.to(_dev()).eval())
    ds = zaremba_b200.minibatch(z["ids"], B, T)
    assert len(ds) == int(z["n_batches"])
    tr = zaremba_b200.Trainer(ms[0], B, T)
    ppl = tr.perplexity(ds)
    assert abs(ppl - float(z["ppl"])) < TOL[engine]["loss"] * float(z["ppl"])
    x, y = ds[0]
    probs = []
    for m in ms:
        t = zaremba_b200.Trainer(m, B, T)
        _, tp = t.eval_step(x.to(_dev()).contiguous(), y.to(_dev()).contiguous(), want_probs=True)
        probs.append(tp.clone())
    ens = torch.mean(-torch.log(torch.stack(probs).mean(0)) * B).item()
    assert abs(ens - float(z["ens_loss"])) < TOL[engine]["loss"] * abs(float(z["ens_loss"]))


def _plan_branch(case, H, B, fp, bp):
    """Whether the plans (zrb_rec_plans) reach the branch a unit-level case exists for.  nCTA depends on the
    SM count and is never pinned; what is asserted is the branch.  A K-split CTA pair (forward) owns 2U units = 8U gate
    rows, a backward CTA of an 8-CTA cluster 8U rows: U <= 8 means ONE M = 64 tile per CTA.  The MMA's N is 8 GBi.  The
    256 epilogue threads own U*B (unit, batch) cells: more than 256 means two cells per thread."""
    both = (fp, bp)
    if case == "one_tile_n32":
        return all(p["KS"] == 2 and p["U"] <= 8 and p["GBi"] == 4 for p in both)
    if case == "two_cells_n32":
        return fp["KS"] == 2 and fp["U"] * B > 256 and fp["GBi"] == 4
    if case == "b8_padded":
        # GB = 1 padded to two batch groups; the last CTA (and the last backward cluster) only partly populated
        return (all(p["KS"] == 2 and p["GBi"] == 2 for p in both) and 0 < H - (fp["nCTA"] - 1) * fp["U"] < fp["U"]
                and H % (8 * bp["U"]) != 0)
    if case == "odd_h":
        return all(p["KS"] == 2 for p in both) and H % (8 * bp["U"]) != 0
    if case == "nosplit_n32":
        return all(p["KS"] == 1 and p["GBi"] == 4 for p in both) and fp["U"] * B > 256
    if case == "b1_split":
        return all(p["KS"] == 2 and p["GBi"] == 2 for p in both)
    if case in ("t1", "baseline"):
        return True
    raise AssertionError(case)


# (H, T, B) -> what the case covers.  The baseline rows are the exact per-layer shapes of BASELINE configs[0..2]; the
# rest reach the plan branches those never take (by a 132-SM restatement of rec_fwd_plan / rec_bwd_plan)
LAYER_CASES = {
    (1500, 35, 20): "baseline", (650, 35, 20): "baseline", (200, 20, 20): "baseline", (96, 5, 7): "baseline",
    (650, 35, 32): "one_tile_n32",     # forward and backward K-split with U = 8: one M = 64 tile; N = 32
    (1500, 35, 32): "two_cells_n32",   # K-split, U = 13: 416 cells on 256 epilogue threads; N = 32
    (300, 6, 8): "b8_padded",          # K-split at B <= 8; H % 32 != 0; the last CTA owns 1 unit
    (257, 5, 9): "odd_h",              # odd H on the split path; the last cluster partly empty
    (255, 4, 32): "nosplit_n32",       # largest H without the K-split; N = 32; two cells per thread
    (1500, 2, 1): "b1_split",          # K-split at B = 1
    (40, 1, 1): "t1",                  # T = 1: the backward kernel has no recurrent term
}


def _layer_against_oracle(lib, ctx, H, T, B, seed):
    """One zrb_lstm_layer_fwd + _bwd on ctx against the fp64 oracle; returns the outputs' device tensors."""
    from zaremba_b200 import _lib
    rng = np.random.default_rng(seed)
    w = 0.04 if H >= 1000 else 0.08
    W_ih, W_hh = rng.uniform(-w, w, size=(4 * H, H)), rng.uniform(-w, w, size=(4 * H, H))
    b_ih, b_hh = rng.uniform(-w, w, size=4 * H), rng.uniform(-w, w, size=4 * H)
    x = rng.normal(size=(T, B, H)) * 0.5
    h0, c0 = rng.uniform(-0.5, 0.5, size=(B, H)), rng.uniform(-1.0, 1.0, size=(B, H))
    dy = rng.normal(size=(T, B, H)) * 0.1
    dev = lambda a: torch.tensor(a, dtype=torch.float32).contiguous().to(_dev())
    d = {k: dev(v) for k, v in dict(W_ih=W_ih, W_hh=W_hh, b_ih=b_ih, b_hh=b_hh, x=x, h0=h0, c0=c0, dy=dy).items()}
    y, hT, cT = torch.empty(T * B, H, device=_dev()), torch.empty(B, H, device=_dev()), torch.empty(B, H, device=_dev())
    _lib.check(lib.zrb_lstm_layer_fwd(ctx, _lib.ptr(d["W_ih"]), _lib.ptr(d["W_hh"]), _lib.ptr(d["b_ih"]), _lib.ptr(d["b_hh"]),
                                      _lib.ptr(d["x"]), T, B, _lib.ptr(d["h0"]), _lib.ptr(d["c0"]), _lib.ptr(y), _lib.ptr(hT),
                                      _lib.ptr(cT), None))
    f32 = lambda a: a.astype(np.float32).astype(np.float64)          # the values the device actually received
    ys, h_ref, c_ref, cache = O.lstm_layer_fwd(f32(x), f32(h0), f32(c0), f32(W_ih), f32(W_hh), f32(b_ih), f32(b_hh))
    tag = f"layer H={H} T={T} B={B}"
    _scale_close(y.cpu().numpy().reshape(T, B, H), ys, 2e-3, f"{tag} y")
    _scale_close(hT.cpu().numpy(), h_ref, 2e-3, f"{tag} hT")
    _scale_close(cT.cpu().numpy(), c_ref, 2e-3, f"{tag} cT")
    dx, dWi, dWh = torch.empty(T * B, H, device=_dev()), torch.empty(4 * H, H, device=_dev()), torch.empty(4 * H, H, device=_dev())
    dbi, dbh = torch.empty(4 * H, device=_dev()), torch.empty(4 * H, device=_dev())
    _lib.check(lib.zrb_lstm_layer_bwd(ctx, _lib.ptr(d["dy"]), _lib.ptr(dx), _lib.ptr(dWi), _lib.ptr(dWh), _lib.ptr(dbi),
                                      _lib.ptr(dbh), None))
    dx_r, dWi_r, dWh_r, db_r = O.lstm_layer_bwd(f32(dy), cache, f32(x), f32(W_ih), f32(W_hh))
    _scale_close(dx.cpu().numpy().reshape(T, B, H), dx_r, 2.5e-3, f"{tag} grad dx")
    _scale_close(dWi.cpu().numpy(), dWi_r, 2.5e-3, f"{tag} grad dW_ih")
    _scale_close(dWh.cpu().numpy(), dWh_r, 2.5e-3, f"{tag} grad dW_hh")
    _scale_close(dbi.cpu().numpy(), db_r, 2.5e-3, f"{tag} grad db_ih")
    assert torch.equal(dbi, dbh)
    return d, (dx, dWi, dWh, dbi, dbh)


@pytest.mark.parametrize("H,T,B", list(LAYER_CASES))
def test_lstm_layer_unit_abi_against_oracle(H, T, B):
    """zrb_lstm_layer_fwd / zrb_lstm_layer_bwd: ONE recurrent layer through the persistent recurrence kernels alone
    (SURVEY 8b's unit-level entry points), against the fp64 restatement of model.py:48-55 and of its autograd (oracle
    lstm_layer_fwd / lstm_layer_bwd), at the per-layer shapes of BASELINE configs[0..2] and at shapes that reach the
    other branches of the recurrence plans (see LAYER_CASES; the case asserts the branch through zrb_rec_plans and skips
    when this device's SM count does not lead there).  Non-zero incoming state.
    Tolerance: 2e-3 of each tensor's scale forward, 2.5e-3 backward (largest measured on an H100 over these cases with
    these N(0, 0.5) inputs: see DESIGN.md section 5)."""
    import zaremba_b200
    from zaremba_b200 import _lib
    lib = _lib.load()
    m = zaremba_b200.Model(16, H, 1, 0.0, 0.05, engine="tc").to(_dev())
    ctx = m._context(T, B)
    case = LAYER_CASES[(H, T, B)]
    plans = _lib.rec_plans(ctx)
    fp, bp = plans["fwd"], plans["bwd"]
    if case != "baseline" and not (fp["ok"] and bp["ok"]):   # (the baseline shapes must run the persistent kernels)
        pytest.skip(f"H={H} B={B} does not fit the persistent kernels on this device: {plans}")
    if not _plan_branch(case, H, B, fp, bp):
        pytest.skip(f"on {torch.cuda.get_device_properties(0).multi_processor_count} SMs H={H} B={B} gets {plans}, "
                    f"not the {case} branch this case is for")
    print(f"\n{case} H={H} T={T} B={B}: fwd {fp} bwd {bp}")
    d, (dx, dWi, dWh, dbi, dbh) = _layer_against_oracle(lib, ctx, H, T, B, H + T)
    # call order is enforced, and the model-level path still works after the unit-level calls borrowed its workspace
    assert lib.zrb_lstm_layer_bwd(ctx, _lib.ptr(d["dy"]), _lib.ptr(dx), _lib.ptr(dWi), _lib.ptr(dWh), _lib.ptr(dbi),
                                  _lib.ptr(dbh), None) == -3
    xtok = torch.zeros(T, B, dtype=torch.long)
    with torch.no_grad():
        s1, _ = m(xtok, m.state_init(B))
        s2, _ = m(xtok, m.state_init(B))
    assert torch.equal(s1, s2) and torch.isfinite(s1).all()


def test_lstm_layer_context_reused_for_a_smaller_window():
    """Model._context keeps a context for every window up to the one it was built for, so the recurrence plans and the
    padded operand images belong to the LARGER batch: a context built for (T=35, B=32) runs the full window and then
    (T=3, B=5) -- 5 batch rows in images laid out for 32 -- and both runs must match the oracle."""
    import zaremba_b200
    from zaremba_b200 import _lib
    lib = _lib.load()
    H = 650
    m = zaremba_b200.Model(16, H, 1, 0.0, 0.05, engine="tc").to(_dev())
    ctx = m._context(35, 32)
    plans = _lib.rec_plans(ctx)
    if not (plans["fwd"]["ok"] and plans["bwd"]["ok"]):
        pytest.skip(f"H={H} B=32 does not fit the persistent kernels on this device: {plans}")
    assert plans["fwd"]["GBi"] == 4 and plans["bwd"]["GBi"] == 4, plans
    _layer_against_oracle(lib, ctx, H, 35, 32, 1)
    assert m._context(3, 5).value == ctx.value, "the model should reuse its context for a smaller window"
    _layer_against_oracle(lib, ctx, H, 3, 5, 2)
    assert _lib.rec_plans(ctx) == plans


def test_error_paths():
    """Reference-like error behaviour: bad shapes / call order raise instead of corrupting memory."""
    import zaremba_b200
    from zaremba_b200 import _lib
    m = zaremba_b200.Model(13, 8, 1, 0.0, 0.1, engine="simt")
    with pytest.raises(RuntimeError):
        m(torch.zeros(2, 2, dtype=torch.long), m.state_init(2))        # CPU model: no fallback
    m = m.to(_dev())
    lib = _lib.load()
    ctx = m._context(2, 2)
    ps, _ = m._params_struct(m.ordered_parameters())
    rc = lib.zrb_backward(ctx, C.byref(ps), C.c_void_p(1), C.byref(ps), None)
    assert rc == -3 and b"forward" in lib.zrb_last_error()
    assert lib.zrb_rec_plans(ctx, (C.c_int32 * 16)()) == -1        # the validation engine has no recurrence plans
    cfg = _lib.ZrbConfig(0, 8, 1, 2, 2, 0, 0.0, 0)
    h = C.c_void_p()
    assert lib.zrb_ctx_create(C.byref(cfg), C.byref(h)) == -1


@pytest.mark.parametrize("engine", ENGINES)
def test_phased_backward_equals_monolithic(engine):
    """zrb_train_step_begin + zrb_train_step_layer(L-1..0) produce the gradients of zrb_train_step_grads
    (the data-parallel trainer reduces buckets between the phases); out-of-order layers are refused."""
    import zaremba_b200
    from zaremba_b200 import _lib
    lib = _lib.load()
    c = StepCase("mid_H72")
    grads = []
    for phased in (False, True):
        m = _model_from_case(c, engine)
        m.train()
        tr = zaremba_b200.Trainer(m, c.B, c.T)
        x = torch.tensor(c.x(0)).to(_dev()).contiguous()
        y = torch.tensor(c.y(0)).to(_dev()).contiguous()
        if not phased:
            _lib.check(lib.zrb_train_step_grads(tr.ctx, C.byref(tr._ps), C.byref(tr._gs), _lib.ptr(x), _lib.ptr(y),
                                                c.T, c.B, C.byref(tr._st), C.byref(tr._st), 1, 0, _lib.ptr(tr.loss), None))
        else:
            _lib.check(lib.zrb_train_step_begin(tr.ctx, C.byref(tr._ps), C.byref(tr._gs), _lib.ptr(x), _lib.ptr(y),
                                                c.T, c.B, C.byref(tr._st), C.byref(tr._st), 1, 0, _lib.ptr(tr.loss), None))
            assert lib.zrb_train_step_layer(tr.ctx, C.byref(tr._ps), C.byref(tr._gs), 0, None) == -3   # wrong order
            for l in range(c.L - 1, -1, -1):
                _lib.check(lib.zrb_train_step_layer(tr.ctx, C.byref(tr._ps), C.byref(tr._gs), l, None))
        torch.cuda.synchronize()
        grads.append(tr.flat_g.clone())
        lo, hi = tr._buckets[0]
        assert hi == tr.flat_g.numel() and tr._buckets[-1][0] == 0
        assert sum(b - a for a, b in tr._buckets) == tr.flat_g.numel()
    assert torch.allclose(grads[0], grads[1], rtol=1e-5, atol=1e-7 * float(grads[0].abs().max()) + 1e-9)


def test_sparse_embedding_gradient_rows_and_scatter():
    """Data-parallel form of the embedding gradient: zrb_set_embed_rows_out + zrb_embed_scatter_rows == the dense
    scatter (np.add.at), with duplicate tokens, and bit-identical across repeated runs (integer accumulation)."""
    import zaremba_b200
    from zaremba_b200 import _lib
    lib = _lib.load()
    V, H, n = 211, 48, 700
    m = zaremba_b200.Model(V, H, 1, 0.0, 0.1, engine="simt").to(_dev())
    ctx = m._context(7, 5)
    rng = np.random.default_rng(9)
    ids = rng.integers(0, 40, size=n)          # few distinct ids: many duplicates
    rows = (rng.normal(size=(n, H)) * 10.0 ** rng.integers(-6, 2, size=(n, 1))).astype(np.float32)
    want = np.zeros((V, H), dtype=np.float64)
    np.add.at(want, ids, rows.astype(np.float64))
    idt, rt = torch.tensor(ids).cuda(), torch.tensor(rows).cuda()
    outs = []
    for rep in range(2):
        g = torch.full((V, H), 7.0, device="cuda")
        _lib.check(lib.zrb_embed_scatter_rows(ctx, _lib.ptr(g), _lib.ptr(idt), _lib.ptr(rt), n, None))
        outs.append(g.clone())
    assert torch.equal(outs[0], outs[1])
    np.testing.assert_allclose(outs[0].cpu().numpy(), want, rtol=2e-6, atol=1e-9)


def test_per_timestep_fallback_for_wide_batches():
    """B > 32 does not fit the persistent recurrence kernels (accumulator / staging sized for N <= 32):
    the tensor-core engine must fall back to one GEMM + one cell launch per timestep and still match the oracle."""
    import zaremba_b200
    V, H, L, T, B = 83, 64, 2, 4, 40
    torch.manual_seed(4)
    m = zaremba_b200.Model(V, H, L, 0.0, 0.2, engine="tc").to(_dev())
    m.train()
    rng = np.random.default_rng(6)
    x = torch.tensor(rng.integers(0, V, size=(T, B))); y = torch.tensor(rng.integers(0, V, size=(T, B)))
    scores, _ = m(x, m.state_init(B))
    _caller_nll_loss(scores, y).backward()
    params = {k: v.detach().cpu().numpy().astype(np.float64) for k, v in m.named_parameters()}
    sc, _, cache = O.model_fwd(params, x.numpy(), O.zero_states(L, B, H, np.float64), L)
    grads = O.model_bwd(params, cache, O.nll_loss_bwd(sc, y.numpy()), L)
    _scale_close(scores.detach().cpu().numpy(), sc, TOL["tc"]["fwd"], "scores (B=40)")
    for k, prm in m.named_parameters():
        _scale_close(prm.grad.cpu().numpy(), grads[k], TOL["tc"]["grad"], f"grad {k} (B=40)")


def _record(what, value):
    key = os.environ.get("PYTEST_CURRENT_TEST", "?").split("::")[-1].split(" ")[0]
    MEASURED.setdefault(key, {})[what] = max(MEASURED.get(key, {}).get(what, 0.0), float(value))


def _prof_counts(lib, ctx):
    """Launch-group counts per profiling class since zrb_prof_enable(ctx, 1); turns profiling off again."""
    from zaremba_b200 import _lib
    ms, counts = (C.c_float * 12)(), (C.c_int64 * 12)()
    _lib.check(lib.zrb_prof_read(ctx, ms, counts))
    _lib.check(lib.zrb_prof_enable(ctx, 0))
    return list(counts)


@pytest.mark.parametrize("lazy", [False, True], ids=["strict", "lazy"])
@pytest.mark.parametrize("H,B,branch", [(72, 20, "nosplit"), (256, 8, "vec4"), (650, 20, "vec2"), (257, 9, "vec1"),
                                        (64, 40, "steps")])
def test_fused_update_rebuilds_what_a_fresh_pack_builds(H, B, branch, lazy):
    """zrb_train_step_update rewrites the fp16 operand images of the new weights from registers (optim_tc.cu: the row
    images, and update_pack_whh_kernel's K-split forward slices and 8-CTA backward slices, 4 / 2 / 1 columns per thread
    as H % 4 and alignment allow) and then declares them current, so nothing repacks them.  A stale or misplaced element
    would shift the next step by about lr * g of one weight, far below any oracle tolerance -- so compare bits instead:
    after three clipped, dropout'ed steps (strict or lazy schedule, flushed) the trained context must compute exactly
    what a FRESH context packed from the same fp32 weights computes: eval loss, target probabilities and states, and
    one gradient pass (same tokens -- all distinct, so the embedding scatter has no colliding atomics -- same dropout
    masks, sparse embedding on).  Branches: 72 = no K-split; 256 / 650 / 257 = K-split with 4 / 2 / 1 columns per
    thread; B = 40 = per-timestep path (row image of W_hh)."""
    import zaremba_b200
    from zaremba_b200 import _lib
    lib = _lib.load()
    V, L, T, lr, max_norm = 256, 2, 5, 1.0, 0.05
    torch.manual_seed(H + B)
    m1 = zaremba_b200.Model(V, H, L, 0.3, 0.1).to(_dev())
    m1.train()
    tr1 = zaremba_b200.Trainer(m1, B, T, lazy_update=lazy)
    fp = _lib.rec_plans(tr1.ctx)["fwd"]
    reached = {"nosplit": fp["ok"] and fp["KS"] == 1, "steps": not fp["ok"]}.get(branch, fp["ok"] and fp["KS"] == 2)
    if not reached:
        pytest.skip(f"H={H} B={B} gets forward plan {fp} on this device, not the {branch} branch")
    g = torch.Generator().manual_seed(3)
    data = torch.randint(0, V, (B, 3 * T + 1), generator=g)
    for s in range(3):
        x = data[:, s * T:(s + 1) * T].t().contiguous().to(_dev())
        y = data[:, s * T + 1:(s + 1) * T + 1].t().contiguous().to(_dev())
        _, norm = tr1.train_step(x, y, lr, max_norm)
        assert norm.item() > 2 * max_norm, "the clip must be active"
    tr1.flush()
    torch.cuda.synchronize()

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

    perm = torch.randperm(V, generator=g)[:T * B]          # distinct tokens
    x = perm.view(T, B).contiguous().to(_dev())
    y = torch.randint(0, V, (T, B), generator=g).to(_dev())
    out = []
    for tr in (tr1, tr2):
        _lib.check(lib.zrb_prof_enable(tr.ctx, 1))
        loss, tp = tr.eval_step(x, y, want_probs=True)
        ev = (loss.clone(), tp.clone(), [t.clone() for st in tr.states for t in st])
        gl = torch.zeros((), device=_dev())
        _lib.check(lib.zrb_train_step_grads(tr.ctx, C.byref(tr._ps), C.byref(tr._gs), _lib.ptr(x), _lib.ptr(y), T, B,
                                            C.byref(tr._st), C.byref(tr._st), 7, 1000, _lib.ptr(gl),
                                            tr._stream()))
        counts = _prof_counts(lib, tr.ctx)
        out.append((ev, gl, tr.flat_g.clone(), [t.clone() for st in tr.states for t in st], counts))
    (ev1, gl1, g1, st1, counts1), (ev2, gl2, g2, st2, counts2) = out
    pack = _lib.PROF_CLASSES.index("pack")
    assert counts1[pack] == 0, "the trained context repacked its weights: the comparison would be vacuous"
    assert counts2[pack] >= 1, "the fresh context must have packed (profiling sanity)"
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


def _tile_width(M, N, nsm):
    """gemm_tc.cu choose_tiles for a weight-gradient GEMM (never split: its epilogue writes sum-of-squares slots)."""
    cdiv = lambda a, b: (a + b - 1) // b
    return 256 if cdiv(M, 128) * cdiv(N, 256) >= (nsm * 9) // 10 else 128


NORM_TOL = 1.2e-7    # 2^-23: one ulp of the fp32 norm at worst


@pytest.mark.parametrize("sparse", [1, 0], ids=["sparse", "dense"])
@pytest.mark.parametrize("shape", ["large", "small"])
def test_fused_step_norm_and_update_are_exact(shape, sparse):
    """The clip norm of the fused step against the fp64 norm of the gradients it left in flat_g, and the update
    against fp32(p - lr * fp32(coef * g)) with coef rebuilt from the returned norm as norm_finalize_kernel (optim.cu)
    computes it.  With the sparse embedding on (zrb_set_embed_sparse 1) the matrices' part of the norm comes from
    sums of squares the wgrad GEMM epilogues leave, one slot per (tile, consumer warp) = one 16 x (tile width) block of
    a weight gradient.  NORM_TOL is about 3x the largest error measured on an H100 80GB HBM3 (400 W limit): 4.7e-8 at
    Large, 1.6e-8 at the small shape.  It is checked to be below the norm change that losing the median slot (6.1e-6 at
    Large, 2.2e-4 small) or tile 0 of any one weight gradient (>= 1.2e-5 / 7.6e-4) would cause, so a lost or
    double-counted slot fails; at Large 90% of all single slots are resolved.  The update may use an FMA, so it is held to one ulp of
    max(|p|, |p_new|).  Two steps, the second one reusing the gradient buffers (rows of the previous window cleared
    instead of a full memset)."""
    import zaremba_b200
    from zaremba_b200 import _lib
    lib = _lib.load()
    # init 0.1 / 0.3 rather than the configs' 0.04: with 0.04 and dropout 0.65 the lower layer's gradient blocks are so
    # small that losing one of them moves the norm by less than one fp32 ulp, which no check of an fp32 norm can see
    V, H, L, T, B, p, winit = (10000, 1500, 2, 35, 20, 0.65, 0.1) if shape == "large" else (300, 256, 2, 9, 8, 0.3, 0.3)
    lr, max_norm = 0.7, 0.25
    torch.manual_seed(17)
    m = zaremba_b200.Model(V, H, L, p, winit).to(_dev())
    m.train()
    tr = zaremba_b200.Trainer(m, B, T)                       # keep_clipped_grads=False: flat_g keeps the raw g
    _lib.check(lib.zrb_set_embed_sparse(tr.ctx, sparse))
    tr._embed_sparse = sparse
    sizes = [p.numel() for p in m.ordered_parameters()]
    offs = np.cumsum([0] + sizes)
    mats = [(int(offs[1 + 4 * l + k]), 4 * H, H) for l in range(L) for k in (0, 1)] + [(int(offs[1 + 4 * L]), V, H)]
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    g = torch.Generator().manual_seed(5)
    data = torch.randint(0, V, (B, 2 * T + 1), generator=g)
    for s in range(2):
        x = data[:, s * T:(s + 1) * T].t().contiguous().to(_dev())
        y = data[:, s * T + 1:(s + 1) * T + 1].t().contiguous().to(_dev())
        p_old = tr.flat_p.clone()
        _, norm = tr.train_step(x, y, lr, max_norm)
        torch.cuda.synchronize()
        n = norm.item()
        g64 = tr.flat_g.double()
        ref = g64.pow(2).sum().sqrt().item()
        rel = abs(n - ref) / ref
        _record("norm", rel)
        # what one dropped sum-of-squares slot would do to the norm: slot (tile, w) holds rows [16w, 16w + 16) of the
        # tile x its columns, i.e. one 16 x bn block of a weight gradient
        slots, tile0 = [], []
        for o, M, N in mats:
            bn = _tile_width(M, N, nsm)
            gm = g64[o:o + M * N].view(M, N)
            gm = torch.nn.functional.pad(gm, (0, -N % bn, 0, -M % 16))
            ss = gm.pow(2).view(gm.shape[0] // 16, 16, gm.shape[1] // bn, bn).sum(dim=(1, 3))
            slots.append(ss.flatten())
            tile0.append(ss[:8, 0].sum())
        slots = torch.cat(slots)
        effect = (ref - torch.sqrt(ref ** 2 - slots)) / ref
        tile0_effect = min((ref - torch.sqrt(ref ** 2 - t)).item() / ref for t in tile0)
        median = effect.median().item()
        _record("median_one_slot_effect", median)
        _record("slots_resolved_fraction", (effect > NORM_TOL).double().mean().item())
        _record("tile0_effect", tile0_effect)
        assert rel <= NORM_TOL, f"step {s}: norm {n!r} vs fp64 {ref!r} (rel {rel:.2e} > {NORM_TOL:.1e})"
        if sparse:      # the bound resolves one lost slot of a typical block and the loss of tile 0 of any weight gradient
            assert NORM_TOL < median and NORM_TOL < tile0_effect, (NORM_TOL, median, tile0_effect)
        coef = np.float32(max_norm) / (np.float32(n) + np.float32(1e-6))
        assert coef < 1, "the clip must be active"
        gc = tr.flat_g * torch.tensor(float(coef), dtype=torch.float32, device=_dev())   # fp32(coef * g)
        want = (p_old.double() - float(np.float32(lr)) * gc.double()).float()
        big = torch.maximum(p_old.abs(), want.abs())
        ulp = torch.nextafter(big, torch.full_like(big, float("inf"))) - big
        diff = (tr.flat_p - want).abs()
        _record("update_ulps", (diff / ulp).max().item())
        bad = (diff > ulp).nonzero()
        assert bad.numel() == 0, f"step {s}: {bad.numel()} parameters off by more than 1 ulp, first at {bad[0].item()}"


def test_zz_write_measured_errors():
    """Not a check: dumps the largest relative errors the tests above measured (ZRB_ERROR_REPORT2=path)."""
    import json
    out = os.environ.get("ZRB_ERROR_REPORT2")
    if out and MEASURED:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        json.dump(MEASURED, open(out, "w"), indent=1)
