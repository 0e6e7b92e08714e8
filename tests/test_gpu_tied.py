"""Tied embedding and softmax weights on the GPU (DESIGN.md section 13): Model(tied=True) and the fused Trainer against
the float64 restatement tests/_model_oracle.py, the fused clip norm and update, bit-reproducibility, lazy = strict, tied
against untied with equal weights, the variational mode, rejected arguments and the data-parallel step.

Tolerances are test_gpu_parity's (TOL per engine, NORM_TOL for the fused norm)."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from oracle import philox as PH
from tests import _model_oracle as MO
from tests._golden import StepCase
from tests.test_gpu_parity import ENGINES, NORM_TOL, TOL, _caller_nll_loss, _record, _scale_close

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
LR, MAX_NORM = 1.0, 5.0
# name -> (V, H, L, T, B, p, winit): the exact Small / Medium / Large shapes (with dropout, so that Philox masks apply),
# the per-timestep path (B = 40 does not fit the persistent recurrence kernels) and the reference fixture's shape
SHAPES = {
    "small": (10000, 200, 2, 20, 20, 0.5, 0.1),
    "medium": (10000, 650, 2, 35, 20, 0.5, 0.05),
    "large": (10000, 1500, 2, 35, 20, 0.65, 0.04),
    "steps_b40": (400, 64, 2, 4, 40, 0.5, 0.1),
    "fixture": "tiny_dropout",
}


@functools.lru_cache(maxsize=None)
def _case(name):
    """(V, H, L, T, B, p, float32 params {tied names}, [x], [y], states0, [masks per step] or None, explicit?)"""
    spec = SHAPES[name]
    if isinstance(spec, str):
        c = StepCase(spec)
        params = {k: v.astype(np.float32) for k, v in c.params0().items()}
        params.pop("fc.W")
        states = [(h.astype(np.float32), cc.astype(np.float32)) for h, cc in c.states0()]
        return (c.V, c.H, c.L, c.T, c.B, c.dropout, params, [c.x(s) for s in range(2)], [c.y(s) for s in range(2)],
                states, [[m.astype(bool) for m in c.masks(s)] for s in range(2)], True)
    V, H, L, T, B, p, winit = spec
    torch.manual_seed(1)
    import zaremba_b200
    m = zaremba_b200.Model(V, H, L, p, winit, tied=True)
    params = {k: v.detach().numpy().copy() for k, v in m.named_parameters()}
    rng = np.random.default_rng(2)
    xs = [rng.integers(0, V, size=(T, B)) for _ in range(2)]
    ys = [rng.integers(0, V, size=(T, B)) for _ in range(2)]
    states = [(rng.uniform(-0.3, 0.3, (B, H)).astype(np.float32), rng.uniform(-0.5, 0.5, (B, H)).astype(np.float32))
              for _ in range(L)]
    return V, H, L, T, B, p, params, xs, ys, states, None, False


SEED = 4242


def _masks(name, s, seed=SEED):
    V, H, L, T, B, p, _, _, _, _, masks, _ = _case(name)
    return masks[s] if masks is not None else PH.site_masks(seed, s, L, T, B, H, p)


@functools.lru_cache(maxsize=None)
def _oracle(name):
    """Two carried tied steps in float64: per step (loss, norm, raw grads, params after, states after), as numpy."""
    V, H, L, T, B, p, params, xs, ys, states, _, _ = _case(name)
    P = {k: _t64(v) for k, v in params.items()}
    st = [(_t64(h), _t64(c)) for h, c in states]
    out = []
    for s in range(2):
        loss, norm, raw, P, st, _ = MO.train_step(P, _tok(xs[s]), _tok(ys[s]), st, L, True, LR, MAX_NORM,
                                                  MO.Modes(p=p), MO.Masks(sites=_masks(name, s)))
        out.append((loss, norm, _np(raw), _np(P), [(h.numpy(), c.numpy()) for h, c in st]))
    return out


def _t64(a):
    return torch.tensor(a, dtype=torch.float64)


def _tok(a):
    return torch.as_tensor(a, dtype=torch.int64)


def _np(d):
    return {k: v.numpy() for k, v in d.items()}


def _tied_model(name, engine, **kw):
    import zaremba_b200
    V, H, L, T, B, p, params, *_ = _case(name)
    m = zaremba_b200.Model(V, H, L, p, 0.1, engine=engine, tied=True, **kw)
    m.load_state_dict({**{k: torch.tensor(v) for k, v in params.items()}, "fc.W": torch.tensor(params["embed.W"])})
    return m.to(DEV)


CASE_IDS = [(n, e) for n in SHAPES for e in ENGINES]


@pytest.mark.parametrize("name,engine", CASE_IDS)
def test_dropin_tied_steps_match_oracle(name, engine):
    """main.py's loop (forward, loss in torch, backward, clip_grad_norm_ + SGD in torch) on Model(tied=True)."""
    V, H, L, T, B, p, _, xs, ys, states, _, explicit = _case(name)
    tol = TOL[engine]
    m = _tied_model(name, engine)
    m.train()
    m._seed, m._drop_step = SEED, 0
    sts = [(torch.tensor(h).view(1, B, H).to(DEV), torch.tensor(c).view(1, B, H).to(DEV)) for h, c in states]
    for s, (loss_w, norm_w, grads_w, params_w, st_w) in enumerate(_oracle(name)):
        if explicit:
            m.set_explicit_dropout_masks([torch.tensor(mk).to(DEV) for mk in _masks(name, s)])
        m.zero_grad()
        sts = m.detach(sts)
        scores, sts = m(torch.tensor(xs[s]), sts)
        loss = _caller_nll_loss(scores, torch.tensor(ys[s]))
        loss.backward()
        assert abs(loss.item() - loss_w) <= tol["loss"] * max(1.0, abs(loss_w)), (loss.item(), loss_w)
        got = {k: q.grad.detach().cpu().numpy() for k, q in m.named_parameters()}
        assert sorted(got) == sorted(grads_w)
        for k in grads_w:
            _scale_close(got[k], grads_w[k], tol["grad"], f"{name} s{s} grad {k}")
        with torch.no_grad():
            norm = torch.nn.utils.clip_grad_norm_(m.parameters(), MAX_NORM)
            for q in m.parameters():
                q -= LR * q.grad
        assert abs(float(norm) - norm_w) <= tol["grad"] * max(1.0, norm_w)
        for k, q in m.named_parameters():
            _scale_close(q.detach().cpu().numpy(), params_w[k], tol["grad"], f"{name} s{s} param {k}")
        for l in range(L):
            _scale_close(sts[l][0].reshape(B, H).cpu().numpy(), st_w[l][0], tol["fwd"], f"{name} s{s} h{l}")
    assert m.fc.W is m.embed.W


@pytest.mark.parametrize("name,engine", CASE_IDS)
def test_fused_trainer_tied_matches_oracle(name, engine):
    import zaremba_b200
    V, H, L, T, B, p, _, xs, ys, states, _, explicit = _case(name)
    tol = TOL[engine]
    m = _tied_model(name, engine)
    m.train()
    tr = zaremba_b200.Trainer(m, B, T)
    tr.seed = SEED
    assert tr.flat_p.numel() == sum(q.numel() for q in m.parameters())
    for l, (h, c) in enumerate(states):
        tr.states[l][0].copy_(torch.tensor(h).view_as(tr.states[l][0]))
        tr.states[l][1].copy_(torch.tensor(c).view_as(tr.states[l][1]))
    for s, (loss_w, norm_w, _, params_w, st_w) in enumerate(_oracle(name)):
        if explicit:
            m.set_explicit_dropout_masks([torch.tensor(mk).to(DEV) for mk in _masks(name, s)])
        loss, norm = tr.train_step(torch.tensor(xs[s]).to(DEV), torch.tensor(ys[s]).to(DEV), LR, MAX_NORM)
        assert abs(loss.item() - loss_w) <= tol["loss"] * max(1.0, abs(loss_w)), (loss.item(), loss_w)
        assert abs(norm.item() - norm_w) <= tol["grad"] * max(1.0, norm_w), (norm.item(), norm_w)
        for k, q in m.named_parameters():
            _scale_close(q.detach().cpu().numpy(), params_w[k], tol["grad"], f"{name} s{s} param {k}")
        for l in range(L):
            _scale_close(tr.states[l][0].reshape(B, H).cpu().numpy(), st_w[l][0], tol["fwd"], f"{name} s{s} h{l}")


@pytest.mark.parametrize("sparse", [1, 0], ids=["sparse", "dense"])
@pytest.mark.parametrize("shape", ["large", "small"])
def test_tied_fused_step_norm_and_update_are_exact(shape, sparse):
    """test_gpu_parity.test_fused_step_norm_and_update_are_exact for a tied model: sparse = the wgrad epilogue slots
    (which describe G_proj) plus the merge's correction in the extra slots, dense = the full read of the buffers."""
    import zaremba_b200
    from zaremba_b200 import _lib
    lib = _lib.load()
    V, H, L, T, B, p, winit = (10000, 1500, 2, 35, 20, 0.65, 0.1) if shape == "large" else (300, 256, 2, 9, 8, 0.3, 0.3)
    lr, max_norm = 0.7, 0.25
    torch.manual_seed(17)
    m = zaremba_b200.Model(V, H, L, p, winit, tied=True).to(DEV)
    m.train()
    tr = zaremba_b200.Trainer(m, B, T)
    _lib.check(lib.zrb_set_embed_sparse(tr.ctx, sparse))
    tr._embed_sparse = sparse
    g = torch.Generator().manual_seed(5)
    data = torch.randint(0, V, (B, 2 * T + 1), generator=g)
    for s in range(2):
        x = data[:, s * T:(s + 1) * T].t().contiguous().to(DEV)
        y = data[:, s * T + 1:(s + 1) * T + 1].t().contiguous().to(DEV)
        p_old = tr.flat_p.clone()
        _, norm = tr.train_step(x, y, lr, max_norm)
        torch.cuda.synchronize()
        n = norm.item()
        ref = tr.flat_g.double().pow(2).sum().sqrt().item()      # E is in flat_g once
        _record("norm", abs(n - ref) / ref)
        assert abs(n - ref) / ref <= NORM_TOL, f"step {s}: norm {n!r} vs fp64 {ref!r}"
        coef = np.float32(max_norm) / (np.float32(n) + np.float32(1e-6))
        assert coef < 1, "the clip must be active"
        gc = tr.flat_g * torch.tensor(float(coef), dtype=torch.float32, device=DEV)
        want = (p_old.double() - float(np.float32(lr)) * gc.double()).float()
        big = torch.maximum(p_old.abs(), want.abs())
        ulp = torch.nextafter(big, torch.full_like(big, float("inf"))) - big
        _record("update_ulps", ((tr.flat_p - want).abs() / ulp).max().item())
        bad = ((tr.flat_p - want).abs() > ulp).nonzero()
        assert bad.numel() == 0, f"step {s}: {bad.numel()} parameters off by more than 1 ulp"


def _philox_trainer(name="small", **kw):
    import zaremba_b200
    V, H, L, T, B, p, params, xs, ys, states, _, _ = _case(name)
    m = _tied_model(name, "tc")
    m.train()
    tr = zaremba_b200.Trainer(m, B, T, **kw)
    tr.seed = SEED
    return m, tr, [torch.tensor(x).to(DEV) for x in xs], [torch.tensor(y).to(DEV) for y in ys]


def test_tied_step_gradient_is_bit_reproducible():
    m, tr, xs, ys = _philox_trainer()
    p0 = tr.flat_p.clone()
    runs = []
    for _ in range(2):
        tr.flat_p.copy_(p0)
        tr.params_changed()
        tr.reset_states()
        tr.step = 0
        tr.train_step(xs[0], ys[0], LR, MAX_NORM)
        torch.cuda.synchronize()
        runs.append((tr.flat_g.clone(), tr.flat_p.clone()))
    assert torch.equal(runs[0][0], runs[1][0]), "the tied gradient must not depend on the run"
    assert torch.equal(runs[0][1], runs[1][1])


@pytest.mark.parametrize("keep", [True, False], ids=["keep_clipped", "raw_grads"])
def test_tied_lazy_update_equals_strict_bit_for_bit(keep):
    res = {}
    for lazy in (False, True):
        m, tr, xs, ys = _philox_trainer(lazy_update=lazy, keep_clipped_grads=keep)
        out = []
        for s in range(3):
            loss, norm = tr.train_step(xs[s % 2], ys[s % 2], LR, 0.5)
            out.append((loss.clone(), norm.clone()))
        tr.flush()
        torch.cuda.synchronize()
        res[lazy] = (out, tr.flat_p.clone(), tr.flat_g.clone())
    for (l0, n0), (l1, n1) in zip(res[False][0], res[True][0]):
        assert torch.equal(l0, l1) and torch.equal(n0, n1), (l0.item(), l1.item(), n0.item(), n1.item())
    assert torch.equal(res[False][1], res[True][1]), "weights"
    assert torch.equal(res[False][2], res[True][2]), "gradient buffers"


def test_tied_equals_untied_with_equal_weights():
    """Inference of a tied model is that of an untied model holding E in both matrices, bit for bit; one train step's
    tied gradient is the untied pair's sum up to fp32 reassociation."""
    import zaremba_b200
    V, H, L, T, B = 2000, 256, 2, 12, 8
    torch.manual_seed(9)
    t = zaremba_b200.Model(V, H, L, 0.5, 0.1, tied=True).to(DEV)
    u = zaremba_b200.Model(V, H, L, 0.5, 0.1).to(DEV)
    u.load_state_dict(t.state_dict())
    for mm in (t, u):
        mm.eval()
    g = torch.Generator().manual_seed(1)
    data = torch.randint(0, V, (B, 4 * T + 1), generator=g)
    batches = [(data[:, i * T:(i + 1) * T].t().contiguous(), data[:, i * T + 1:(i + 1) * T + 1].t().contiguous())
               for i in range(4)]
    tt, tu = zaremba_b200.Trainer(t, B, T), zaremba_b200.Trainer(u, B, T)
    x, y = batches[0][0].to(DEV), batches[0][1].to(DEV)
    lt, pt = tt.eval_step(x, y, want_probs=True)
    lu, pu = tu.eval_step(x, y, want_probs=True)
    assert torch.equal(lt, lu) and torch.equal(pt, pu)
    assert tt.perplexity(batches) == tu.perplexity(batches)
    ct, cu = zaremba_b200.NeuralCache(H, B, 50, T), zaremba_b200.NeuralCache(H, B, 50, T)
    assert tt.perplexity(batches, cache=ct, theta=0.3, lam=0.1) == tu.perplexity(batches, cache=cu, theta=0.3, lam=0.1)
    prompt = batches[1][0][:5, :3]
    a, b = t.generate(prompt, 6, seed=3, temperature=0.9), u.generate(prompt, 6, seed=3, temperature=0.9)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    a, b = t.beam_search(prompt, 4, 2), u.beam_search(prompt, 4, 2)
    assert all(torch.equal(p, q) for p, q in zip(a[:3], b[:3]))
    # one train step: tied dE vs untied embed.W + fc.W gradients
    for mm in (t, u):
        mm.train()
    tu.seed = tt.seed
    tt.train_step(x, y, LR, MAX_NORM)
    tu.train_step(x, y, LR, MAX_NORM)
    torch.cuda.synchronize()
    want = (u.embed.W.grad + u.fc.W.grad).cpu().numpy()
    _scale_close(t.embed.W.grad.cpu().numpy(), want, 1e-6, "tied dE vs untied sum")
    for (k, q), (_, r) in zip([kv for kv in t.named_parameters() if kv[0] != "embed.W"],
                              [kv for kv in u.named_parameters() if kv[0] not in ("embed.W", "fc.W")]):
        _scale_close(q.grad.cpu().numpy(), r.grad.cpu().numpy(), 1e-6, f"grad {k}")


def test_tied_variational_against_oracle():
    import zaremba_b200
    V, H, L, T, B, p, p_rec = 500, 256, 2, 8, 8, 0.5, 0.3
    torch.manual_seed(21)
    m = zaremba_b200.Model(V, H, L, p, 0.08, variational=True, recurrent_dropout=p_rec, tied=True).to(DEV)
    m.train()
    m._seed, m._drop_step = SEED, 0
    P = {k: q.detach().cpu().double() for k, q in m.named_parameters()}
    rng = np.random.default_rng(4)
    st = [(_t64(rng.uniform(-0.3, 0.3, (B, H))), _t64(rng.uniform(-0.5, 0.5, (B, H)))) for _ in range(L)]
    sts = [(h.float().view(1, B, H).to(DEV), c.float().view(1, B, H).to(DEV)) for h, c in st]
    tol = TOL["tc"]
    for s in range(2):
        x, y = rng.integers(0, V, size=(T, B)), rng.integers(0, V, size=(T, B))
        md = MO.Modes(seed=SEED, step=s, p=p, variational=True, p_rec=p_rec)
        loss_w, norm_w, raw_w, P, st, _ = MO.train_step(P, _tok(x), _tok(y), st, L, True, LR, MAX_NORM, md)
        coef = min(1.0, MAX_NORM / (norm_w + 1e-6))
        m.zero_grad()
        sts = m.detach(sts)
        scores, sts = m(torch.tensor(x), sts)
        loss = _caller_nll_loss(scores, torch.tensor(y))
        loss.backward()
        assert abs(loss.item() - loss_w) <= tol["loss"] * max(1.0, abs(loss_w))
        with torch.no_grad():
            norm = torch.nn.utils.clip_grad_norm_(m.parameters(), MAX_NORM)
            for q in m.parameters():
                q -= LR * q.grad
        assert abs(float(norm) - norm_w) <= tol["grad"] * max(1.0, norm_w)
        for k, q in m.named_parameters():
            _scale_close(q.grad.cpu().numpy(), raw_w[k].numpy() * coef, tol["grad"], f"s{s} clipped grad {k}")
            _scale_close(q.detach().cpu().numpy(), P[k].numpy(), tol["grad"], f"s{s} param {k}")


def test_tied_rejected_arguments_leave_the_context_usable():
    import zaremba_b200
    from zaremba_b200 import _lib
    lib = _lib.load()
    for flags in (2, 3, -1):
        cfg = _lib.ZrbConfig(100, 64, 1, 4, 4, _lib.ENGINE_TC, 0.0, flags)
        h = C.c_void_p()
        assert lib.zrb_ctx_create(C.byref(cfg), C.byref(h)) == -1 and b"flags" in lib.zrb_last_error()
    m, tr, xs, ys = _philox_trainer()
    T, B = xs[0].shape
    other = torch.zeros_like(m.embed.W)
    bad_p, _ = m._params_struct(m.ordered_parameters())
    bad_p.fc_w = other.data_ptr()
    bad_g, _ = m._params_struct([q.grad for q in m.ordered_parameters()])
    bad_g.fc_w = other.data_ptr()
    st = C.byref(tr._st)
    lib_calls = [
        lambda: lib.zrb_forward(tr.ctx, C.byref(bad_p), _lib.ptr(xs[0]), T, B, st, st, None, 1, 0, 0, None),
        lambda: lib.zrb_eval_step(tr.ctx, C.byref(bad_p), _lib.ptr(xs[0]), _lib.ptr(ys[0]), T, B, st, st,
                                  _lib.ptr(tr.loss), None, None),
        lambda: lib.zrb_train_step_grads(tr.ctx, C.byref(tr._ps), C.byref(bad_g), _lib.ptr(xs[0]), _lib.ptr(ys[0]),
                                         T, B, st, st, 0, 0, _lib.ptr(tr.loss), None),
        lambda: lib.zrb_train_step_grads(tr.ctx, C.byref(bad_p), C.byref(tr._gs), _lib.ptr(xs[0]), _lib.ptr(ys[0]),
                                         T, B, st, st, 0, 0, _lib.ptr(tr.loss), None),
        lambda: lib.zrb_train_step_update(tr.ctx, C.byref(tr._ps), C.byref(bad_g), 1.0, 1.0, None, None),
        lambda: lib.zrb_backward(tr.ctx, C.byref(tr._ps), _lib.ptr(other), C.byref(bad_g), None),
    ]
    p0 = tr.flat_p.clone()
    for i, call in enumerate(lib_calls):
        assert call() == -1, i
        assert b"tied" in lib.zrb_last_error(), i
    torch.cuda.synchronize()
    assert torch.equal(tr.flat_p, p0) and not other.any()
    loss, norm = tr.train_step(xs[0], ys[0], LR, MAX_NORM)
    assert np.isfinite(loss.item()) and norm.item() > 0


# ---- data parallel (two GPUs) -------------------------------------------------------------------------------------
def _dp_tied_worker(rank, world, port, q, transport):
    import os
    import torch.distributed as dist
    import zaremba_b200
    from zaremba_b200 import _lib
    from tests.test_gpu_multi import B as MB, H as MH, L as ML, P_DROP, STEPS, T as MT, V as MV
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank), ZRB_DP_TRANSPORT=transport)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    lib = _lib.load()
    g = torch.Generator().manual_seed(3)
    data = torch.randint(0, MV, (MB * world, STEPS * MT + 1), generator=g)
    torch.manual_seed(7)
    m = zaremba_b200.Model(MV, MH, ML, P_DROP, 0.1, tied=True).to(dev)
    m.train()
    tr = zaremba_b200.Trainer(m, MB, MT)
    assert tr.transport == transport
    rows = slice(rank * MB, (rank + 1) * MB)
    seeds, out = [], []
    for i in range(STEPS):
        x = data[rows, i * MT:(i + 1) * MT].t().contiguous().to(dev)
        y = data[rows, i * MT + 1:(i + 1) * MT + 1].t().contiguous().to(dev)
        seeds.append((tr.seed, tr.step))
        loss, norm = tr.train_step(x, y, 1.0, 0.25)
        out.append((loss.item(), norm.item()))
    dp_p = tr.flat_p.clone()
    allp = [torch.empty_like(dp_p) for _ in range(world)]
    dist.all_gather(allp, dp_p)
    identical = all(torch.equal(allp[0], a) for a in allp)
    n = MT * MB * MH
    masks = torch.empty(STEPS, ML + 1, n, dtype=torch.uint8, device=dev)
    for i, (seed, step) in enumerate(seeds):
        for site in range(ML + 1):
            _lib.check(lib.zrb_dropout_mask(seed, step, site, n, P_DROP, _lib.ptr(masks[i, site]), None))
    allm = [torch.empty_like(masks) for _ in range(world)]
    dist.all_gather(allm, masks)
    losses = torch.tensor([o[0] for o in out], device=dev, dtype=torch.float64)
    dist.all_reduce(losses)
    res = {"identical": identical, "norms": [o[1] for o in out], "loss_sum": losses.tolist()}
    if rank == 0:
        torch.manual_seed(7)
        m2 = zaremba_b200.Model(MV, MH, ML, P_DROP, 0.1, tied=True).to(dev)
        m2.train()
        tr2 = zaremba_b200.Trainer(m2, MB * world, MT, data_parallel=False)
        ref = []
        for i in range(STEPS):
            x = data[:, i * MT:(i + 1) * MT].t().contiguous().to(dev)
            y = data[:, i * MT + 1:(i + 1) * MT + 1].t().contiguous().to(dev)
            full = [torch.cat([allm[r][i, site].view(MT, MB, MH) for r in range(world)], dim=1).contiguous()
                    for site in range(ML + 1)]
            m2.set_explicit_dropout_masks(full)
            loss, norm = tr2.train_step(x, y, 1.0, 0.25)
            ref.append((loss.item(), norm.item()))
        res.update(err=(dp_p - tr2.flat_p).abs().max().item() / tr2.flat_p.abs().max().item(), ref=ref)
    dist.barrier()
    tr.close()
    dist.destroy_process_group()
    q.put((rank, res))


@pytest.mark.parametrize("transport", ["ce", "nccl"])
def test_tied_dp_step_equals_single_process(transport):
    from tests.test_gpu_multi import _need_two, _spawn
    _need_two()
    out = _spawn(_dp_tied_worker, 2, transport)
    r0 = out[0]
    assert out[0]["identical"] and out[1]["identical"], "replicas diverged across ranks"
    assert r0["err"] < 2e-3, r0
    for (l_ref, n_ref), l_dp, n_dp in zip(r0["ref"], r0["loss_sum"], r0["norms"]):
        assert abs(l_dp - l_ref) < 2e-3 * abs(l_ref) and abs(n_dp - n_ref) < 3e-3 * n_ref, r0
