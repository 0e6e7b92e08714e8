"""GPU tests of the weight-dropped LSTM (DESIGN.md section 15) at every recurrence-plan branch: the rows of
tests/test_gpu_dropout.py (every plan branch, the per-timestep path at B = 40, the validation engine).

  * equivalence, bit for bit: the gradient half of a step with the mode on equals a mode-off context whose W_hh holds
    fp32(W_hh * m * scale) (loss, scores, states and every other gradient), and dW_hh = fp32(scale * m * dW_eff) -- this
    pins the masked fp16 images and the gradient mask with no tolerance; the fused clip norm against the fp64 norm;
  * two carried steps of the fused Trainer and the drop-in Model against the fp64 restatement of
    tests/_model_oracle.py with masks computed by oracle/philox.py;
  * lazy equals strict; eval untouched; p = 0 is the mode off; rejected arguments and call orders; two GPUs.
Windows hold distinct tokens, so the embedding scatter is deterministic.
"""
import ctypes as C
import gc
import math
import os

import numpy as np
import pytest
import torch

from oracle import lstm_lm_oracle as O
from tests import _model_oracle as MO
from tests.test_gpu_dropout import L, P_DROP, ROW_IDS, Row
from tests.test_gpu_parity import ENGINES, NORM_TOL, TOL, _caller_nll_loss, _scale_close

pytestmark = pytest.mark.gpu

LR, MAX_NORM = 1.0, 0.25
STEP = 3          # a step other than 0, so that a mask keyed on the wrong word shows


def _dev():
    return torch.device("cuda:0")


def _winit(row):
    """The recipes' init scale, as tests/test_gpu_variational.py uses it (winit * sqrt(H) <= 1.3)."""
    return min(row.winit, 1.3 / math.sqrt(row.H))


def _model(row, p_wd=0.0, **kw):
    import zaremba_b200
    torch.manual_seed(row.torch_seed)
    m = zaremba_b200.Model(row.V, row.H, L, P_DROP, _winit(row), engine=row.engine, weight_drop=p_wd, **kw).to(_dev())
    m.train()
    return m


def _lib_mask(seed, step, l, H, p):
    """layer l's keep-mask [4H, H] as zrb_dropout_mask draws it (its equality with oracle/philox.py is pinned by
    test_gpu_dropout.test_dropout_mask_equals_reference)."""
    from zaremba_b200 import _lib
    out = torch.empty(4 * H * H, dtype=torch.uint8, device=_dev())
    _lib.check(_lib.load().zrb_dropout_mask(seed, step, 2 * L + 1 + l, 4 * H * H, p, _lib.ptr(out), None))
    return out.view(4 * H, H).bool()


def _mul(mask, p):
    """the multiplier 0 / float32(1 / (1 - p)) of each element"""
    return mask.float() * float(np.float32(1.0 / (1.0 - float(np.float32(p)))))


def _whh_names():
    return [f"rnns.{l}.weight_hh_l0" for l in range(L)]


def _sizes(model):
    return [p.numel() for p in model.ordered_parameters()]


def _names(model):
    ids = {id(p): n for n, p in model.named_parameters()}
    return [ids[id(p)] for p in model.ordered_parameters()]


# ---- equivalence with masked weights, bit for bit -----------------------------------------------------------------
def _trainer_grads(row, p_wd, masked_whh=None, **kw):
    """One fused step at STEP: loss, norm, states, {name: raw gradient}; masked_whh: replace W_hh by W_hh * mul."""
    import zaremba_b200
    m = _model(row, p_wd, **kw)
    if masked_whh is not None:
        with torch.no_grad():
            for l, mul in enumerate(masked_whh):
                m.rnns[l].weight_hh_l0.mul_(mul)
    tr = zaremba_b200.Trainer(m, row.B, row.T)
    for (h, c), (h0, c0) in zip(tr.states, row.states()):
        h.copy_(h0)
        c.copy_(c0)
    row.check_branch(tr.ctx)
    tr.step = STEP
    loss, norm = tr.train_step(row.x[0].to(_dev()), row.y[0].to(_dev()), LR, MAX_NORM)
    tr.flush()
    torch.cuda.synchronize()
    grads = {n: p.grad.detach().clone() for n, p in m.named_parameters()}
    out = dict(loss=loss.clone(), norm=norm.clone(), states=[t.clone() for st in tr.states for t in st], grads=grads)
    tr.close()
    del tr, m
    gc.collect()
    return out


def _dropin_grads(row, p_wd, masked_whh=None, **kw):
    """Drop-in Model at dropout step 0: forward, the caller's loss, backward."""
    m = _model(row, p_wd, **kw)
    if masked_whh is not None:
        with torch.no_grad():
            for l, mul in enumerate(masked_whh):
                m.rnns[l].weight_hh_l0.mul_(mul)
    row.check_branch(m._context(row.T, row.B))
    scores, states = m(row.x[0], row.states())
    _caller_nll_loss(scores, row.y[0]).backward()
    out = dict(scores=scores.detach().clone(), states=[t.clone() for st in states for t in st],
               grads={n: p.grad.detach().clone() for n, p in m.named_parameters()})
    del m
    gc.collect()
    return out


def _assert_equivalent(got, ref, muls, what):
    for k in ("loss", "scores"):
        if k in got:
            assert torch.equal(got[k], ref[k]), f"{what}: {k} differs"
    bad = [i for i, (a, b) in enumerate(zip(got["states"], ref["states"])) if not torch.equal(a, b)]
    assert not bad, f"{what}: states {bad} differ"
    whh = _whh_names()
    for n, g in got["grads"].items():
        if n in whh:
            mul = muls[whh.index(n)]
            want = ref["grads"][n] * mul
            assert torch.equal(g, want), f"{what}: {n} is not scale * m * dW_eff"
            assert (g[mul == 0] == 0).all()
        else:
            assert torch.equal(g, ref["grads"][n]), f"{what}: gradient {n} differs"


@pytest.mark.parametrize("row", ROW_IDS)
def test_equals_masked_weights_bit_for_bit(row):
    r = Row(row)
    p_wd = 0.5
    seed = r.torch_seed                      # torch.initial_seed() after _model's manual_seed: the mode's seed
    muls = [_mul(_lib_mask(seed, STEP, l, r.H, p_wd), p_wd) for l in range(L)]
    got = _trainer_grads(r, p_wd)
    ref = _trainer_grads(r, 0.0, masked_whh=muls)
    _assert_equivalent(got, ref, muls, f"{row} trainer")
    # the clip norm is the norm of the masked gradient buffers (tensor-core engine: fused, W_hh's part summed by the
    # masking pass; validation engine: one pass over the buffers)
    want = math.sqrt(sum(float((g.double() ** 2).sum()) for g in got["grads"].values()))
    tol = NORM_TOL if r.engine == "tc" else 1e-6
    assert abs(got["norm"].item() - want) <= tol * want, (got["norm"].item(), want)
    muls0 = [_mul(_lib_mask(seed, 0, l, r.H, p_wd), p_wd) for l in range(L)]
    got = _dropin_grads(r, p_wd)
    ref = _dropin_grads(r, 0.0, masked_whh=muls0)
    _assert_equivalent(got, ref, muls0, f"{row} drop-in")


@pytest.mark.parametrize("mode", ["variational", "tied"])
def test_composes_with_variational_and_tied(mode):
    """The equivalence above with variational=True (p_rec 0.5) or tied=True, on a persistent-plan row and the
    per-timestep row."""
    for row in [r for r in ("odd_h", "steps_b40", "simt_h48") if r in ROW_IDS]:
        r = Row(row)
        kw = dict(variational=True, recurrent_dropout=0.5) if mode == "variational" else dict(tied=True)
        muls = [_mul(_lib_mask(r.torch_seed, STEP, l, r.H, 0.5), 0.5) for l in range(L)]
        got = _trainer_grads(r, 0.5, **kw)
        ref = _trainer_grads(r, 0.0, masked_whh=muls, **kw)
        _assert_equivalent(got, ref, muls, f"{row} {mode}")


# ---- against the fp64 oracle --------------------------------------------------------------------------------------
_oracle_cache = {}


def _oracle(row, seed, p_wd, variational):
    key = (row.name, seed, p_wd, variational)
    if key not in _oracle_cache:
        m = _model(row)
        params = {k: v.detach().cpu().double() for k, v in m.named_parameters()}
        del m
        states = [(h.double(), c.double()) for h, c in row.h0]
        out = []
        for s in range(2):
            md = MO.Modes(seed=seed, step=s, p=P_DROP, variational=variational,
                          p_rec=P_DROP if variational else 0.0, wd_seed=row.torch_seed, p_wd=p_wd)
            with torch.no_grad():
                sc = MO.forward(params, row.x[s], states, L, False, md)[0]
            loss, norm, grads, params, states, _ = MO.train_step(params, row.x[s], row.y[s], states, L, False, LR,
                                                                 MAX_NORM, md)
            out.append(dict(loss=loss, norm=norm, scores=sc.numpy(), states=[(h.numpy(), c.numpy()) for h, c in states],
                            grads={k: v.numpy() for k, v in grads.items()},
                            params={k: v.numpy() for k, v in params.items()}))
        _oracle_cache.clear()
        _oracle_cache[key] = out
    return _oracle_cache[key]


def _trainer_run(row, p_wd, lazy=False, keep=False, eval_between=False, **kw):
    import zaremba_b200
    m = _model(row, p_wd, **kw)
    tr = zaremba_b200.Trainer(m, row.B, row.T, lazy_update=lazy, keep_clipped_grads=keep)
    for (h, c), (h0, c0) in zip(tr.states, row.states()):
        h.copy_(h0)
        c.copy_(c0)
    row.check_branch(tr.ctx)
    out = []
    for s in range(2):
        loss, norm = tr.train_step(row.x[s].to(_dev()), row.y[s].to(_dev()), LR, MAX_NORM)
        loss, norm = loss.clone(), norm.clone()   # (eval_step writes the same loss buffer)
        if eval_between and s == 0:
            saved = [t.clone() for st in tr.states for t in st]
            m.eval()
            tr.eval_step(row.x[1].to(_dev()), row.y[1].to(_dev()))
            m.train()
            for t, v in zip([t for st in tr.states for t in st], saved):
                t.copy_(v)
        tr.flush()
        torch.cuda.synchronize()
        out.append(dict(loss=loss.clone(), norm=norm.clone(), states=[t.clone() for st in tr.states for t in st],
                        flat_g=tr.flat_g.clone(), flat_p=tr.flat_p.clone()))
    seed = tr.seed
    names, sizes = _names(m), _sizes(m)
    tr.close()
    del tr, m
    gc.collect()
    return out, seed, names, sizes


def _dropin_run(row, p_wd, **kw):
    m = _model(row, p_wd, **kw)
    row.check_branch(m._context(row.T, row.B))
    states = row.states()
    out = []
    for s in range(2):
        m.zero_grad(set_to_none=True)
        scores, states = m(row.x[s], states)
        loss = _caller_nll_loss(scores, row.y[s])
        loss.backward()
        grads = {k: p.grad.clone() for k, p in m.named_parameters()}
        torch.nn.utils.clip_grad_norm_(m.parameters(), MAX_NORM)
        with torch.no_grad():
            for p in m.parameters():
                p -= LR * p.grad
        states = m.detach(states)
        out.append(dict(loss=loss.detach().clone(), scores=scores.detach().clone(),
                        states=[t.clone() for st in states for t in st], grads=grads,
                        params={k: p.detach().clone() for k, p in m.named_parameters()}))
    seed = m._seed
    del m
    gc.collect()
    return out, seed


def _check_against_oracle(row, got, ref, tag, names=None, sizes=None):
    tol = TOL[row.engine]
    for s, (g, r) in enumerate(zip(got, ref)):
        t = f"{tag} step {s}"
        assert abs(g["loss"].item() - r["loss"]) <= tol["loss"] * abs(r["loss"]), (t, g["loss"].item(), r["loss"])
        for l in range(L):
            _scale_close(g["states"][2 * l].reshape(row.B, row.H).cpu().numpy(), r["states"][l][0], tol["fwd"], f"{t} h{l}")
            _scale_close(g["states"][2 * l + 1].reshape(row.B, row.H).cpu().numpy(), r["states"][l][1], tol["fwd"],
                         f"{t} c{l}")
        if "scores" in g:
            _scale_close(g["scores"].cpu().numpy(), r["scores"], tol["fwd"], f"{t} scores")
        if "flat_g" in g:
            grads = dict(zip(names, g["flat_g"].split(sizes)))
            params = dict(zip(names, g["flat_p"].split(sizes)))
        else:
            grads, params = g["grads"], g["params"]
        for k in O.param_names(L):
            _scale_close(grads[k].cpu().numpy().reshape(r["grads"][k].shape), r["grads"][k], tol["grad"], f"{t} grad {k}")
            _scale_close(params[k].cpu().numpy().reshape(r["params"][k].shape), r["params"][k], tol["grad"],
                         f"{t} param {k}")


# p = 0.5 at every row; p = 0.2 (another threshold of the same draws) at a persistent, a padded, the per-timestep and
# a validation-engine row
ORACLE_CASES = [(row, 0.5) for row in ROW_IDS] + \
    [(row, 0.2) for row in ("odd_h", "b8_padded", "steps_b40", "simt_h257") if row in ROW_IDS]


@pytest.mark.parametrize("row,p_wd", ORACLE_CASES)
def test_trainer_and_dropin_against_fp64_oracle(row, p_wd):
    r = Row(row)
    got, seed, names, sizes = _trainer_run(r, p_wd)
    ref = _oracle(r, seed, p_wd, False)
    _check_against_oracle(r, got, ref, f"{row} trainer", names, sizes)
    got, seed2 = _dropin_run(r, p_wd)
    assert seed2 == seed
    _check_against_oracle(r, got, ref, f"{row} drop-in")


@pytest.mark.parametrize("row", [r for r in ("odd_h", "simt_h48") if r in ROW_IDS])
def test_variational_against_fp64_oracle(row):
    r = Row(row)
    got, seed, names, sizes = _trainer_run(r, 0.5, variational=True)
    _check_against_oracle(r, got, _oracle(r, seed, 0.5, True), f"{row} variational trainer", names, sizes)


# ---- schedules, eval, p = 0 ---------------------------------------------------------------------------------------
def _assert_runs_equal(a, b, what):
    for s, (u, v) in enumerate(zip(a, b)):
        bad = [k for k in u if not (torch.equal(u[k], v[k]) if torch.is_tensor(u[k])
                                    else all(torch.equal(p, q) for p, q in zip(u[k], v[k])))]
        assert not bad, f"{what} step {s}: {bad} differ"


@pytest.mark.parametrize("keep", [False, True], ids=["raw_grads", "clipped_grads"])
def test_lazy_update_equals_strict(keep):
    if "tc" not in ENGINES:
        pytest.skip("tensor-core engine not selected")
    for row, kw in (("odd_h", {}), ("b8_padded", dict(variational=True, tied=True))):
        r = Row(row)
        got = _trainer_run(r, 0.5, lazy=True, keep=keep, **kw)[0]
        want = _trainer_run(r, 0.5, keep=keep, **kw)[0]
        _assert_runs_equal(got, want, f"{row} lazy")


@pytest.mark.parametrize("row", [r for r in ("odd_h", "steps_b40", "simt_h48") if r in ROW_IDS])
def test_train_eval_train_equals_train_train(row):
    r = Row(row)
    got = _trainer_run(r, 0.5, eval_between=True)[0]
    want = _trainer_run(r, 0.5)[0]
    _assert_runs_equal(got, want, f"{row} train-eval-train")


@pytest.mark.parametrize("row", [r for r in ("odd_h", "steps_b40", "simt_h48") if r in ROW_IDS])
def test_eval_is_untouched(row):
    """After two weight-dropped steps: eval_step, perplexity, generate, beam_search and dynamic_eval_step equal a
    mode-off model holding the same weights, bit for bit."""
    import zaremba_b200
    r = Row(row)
    res = []
    weights = None
    for p_wd in (0.5, 0.0):
        m = _model(r, p_wd)
        if weights is None:
            tr = zaremba_b200.Trainer(m, r.B, r.T)
            for s in range(2):
                tr.train_step(r.x[s].to(_dev()), r.y[s].to(_dev()), LR, MAX_NORM)
            tr.flush()
            weights = {k: v.detach().clone() for k, v in m.state_dict().items()}
        else:
            m.load_state_dict(weights)
            tr = zaremba_b200.Trainer(m, r.B, r.T)
        m.eval()
        tr.reset_states()
        loss = tr.eval_step(r.x[0].to(_dev()), r.y[0].to(_dev())).clone()
        ppl = tr.perplexity([(r.x[0], r.y[0]), (r.x[1], r.y[1])])
        tok, lp, _ = m.generate(r.x[0][:, :1], 3, temperature=1.0, seed=9)
        bt, blp, bsc, _ = m.beam_search(r.x[0][:, :1], 3, 3)
        theta = tr.flat_p.clone()
        tr.reset_states()
        dl = tr.dynamic_eval_step(r.x[1].to(_dev()), r.y[1].to(_dev()), theta, 0.1, 0.01).clone()
        torch.cuda.synchronize()
        res.append([loss, torch.tensor(ppl), tok, lp, bt, blp, bsc, dl, tr.flat_p.clone(), tr.flat_g.clone()])
        tr.close()
        del tr, m
        gc.collect()
    for i, (a, b) in enumerate(zip(*res)):
        assert torch.equal(a, b), f"output {i} differs"


@pytest.mark.parametrize("row", [r for r in ("odd_h", "simt_h48") if r in ROW_IDS])
def test_p0_equals_mode_off(row):
    from zaremba_b200 import _lib
    r = Row(row)
    want = _trainer_run(r, 0.0)[0]
    import zaremba_b200
    m = _model(r)
    tr = zaremba_b200.Trainer(m, r.B, r.T)
    _lib.check(_lib.load().zrb_set_weight_drop(tr.ctx, 0.0, 12345))
    for (h, c), (h0, c0) in zip(tr.states, r.states()):
        h.copy_(h0)
        c.copy_(c0)
    got = []
    for s in range(2):
        loss, norm = tr.train_step(r.x[s].to(_dev()), r.y[s].to(_dev()), LR, MAX_NORM)
        torch.cuda.synchronize()
        got.append(dict(loss=loss.clone(), norm=norm.clone(), states=[t.clone() for st in tr.states for t in st],
                        flat_g=tr.flat_g.clone(), flat_p=tr.flat_p.clone()))
    tr.close()
    _assert_runs_equal(got, want, f"{row} p=0")


def test_rejected_arguments_and_call_order():
    import zaremba_b200
    from zaremba_b200 import _lib
    lib = _lib.load()
    E_INVALID, E_STATE = -1, -3
    r = Row("tc_h48" if "tc" in ENGINES else "simt_h48")
    m = _model(r)
    tr = zaremba_b200.Trainer(m, r.B, r.T)
    ctx = tr.ctx
    for p in (-0.1, 1.0, 1.5, float("nan"), float("inf"), -float("inf")):
        assert lib.zrb_set_weight_drop(ctx, p, 1) == E_INVALID, p
    assert lib.zrb_set_weight_drop(None, 0.5, 1) == E_INVALID
    x, y = r.x[0].to(_dev()), r.y[0].to(_dev())
    stream = tr._stream()
    scores = torch.empty(r.T * r.B, r.V, device=_dev())
    _lib.check(lib.zrb_forward(ctx, C.byref(tr._ps), _lib.ptr(x), r.T, r.B, C.byref(tr._st), C.byref(tr._st),
                               _lib.ptr(scores), 1, tr.seed, 0, stream))
    _lib.check(lib.zrb_set_weight_drop(ctx, 0.5, 7))
    assert lib.zrb_backward(ctx, C.byref(tr._ps), _lib.ptr(scores), C.byref(tr._gs), stream) == E_STATE
    _lib.check(lib.zrb_train_step_begin(ctx, C.byref(tr._ps), C.byref(tr._gs), _lib.ptr(x), _lib.ptr(y), r.T, r.B,
                                        C.byref(tr._st), C.byref(tr._st), tr.seed, 1, _lib.ptr(tr.loss), stream))
    _lib.check(lib.zrb_set_weight_drop(ctx, 0.5, 8))            # another seed is another mode
    assert lib.zrb_train_step_layer(ctx, C.byref(tr._ps), C.byref(tr._gs), L - 1, stream) == E_STATE
    _lib.check(lib.zrb_train_step_begin(ctx, C.byref(tr._ps), C.byref(tr._gs), _lib.ptr(x), _lib.ptr(y), r.T, r.B,
                                        C.byref(tr._st), C.byref(tr._st), tr.seed, 2, _lib.ptr(tr.loss), stream))
    _lib.check(lib.zrb_set_weight_drop(ctx, 0.5, 8))            # the same mode again keeps the saved forward
    for l in range(L - 1, -1, -1):
        _lib.check(lib.zrb_train_step_layer(ctx, C.byref(tr._ps), C.byref(tr._gs), l, stream))
    torch.cuda.synchronize()
    tr.close()


# ---- two GPUs -----------------------------------------------------------------------------------------------------
def _dp_worker(rank, world, port, q, transport):
    import torch.distributed as dist
    import zaremba_b200
    from zaremba_b200 import _lib
    from tests.test_gpu_multi import B, H, STEPS, T, V
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank), ZRB_DP_TRANSPORT=transport)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    lib = _lib.load()
    p_wd = 0.5
    g = torch.Generator().manual_seed(3)
    data = torch.randint(0, V, (B * world, STEPS * T + 1), generator=g)
    torch.manual_seed(7)
    m = zaremba_b200.Model(V, H, L, P_DROP, 0.1, weight_drop=p_wd).to(dev)
    m.train()
    tr = zaremba_b200.Trainer(m, B, T)
    assert tr.transport == transport
    rows = slice(rank * B, (rank + 1) * B)
    seeds = []
    for i in range(STEPS):
        x = data[rows, i * T:(i + 1) * T].t().contiguous().to(dev)
        y = data[rows, i * T + 1:(i + 1) * T + 1].t().contiguous().to(dev)
        seeds.append((tr.seed, tr.step))
        tr.train_step(x, y, 1.0, 0.25)
    tr.flush()
    dp_p = tr.flat_p.clone()
    bits = dp_p.view(torch.int32).to(torch.int64)
    chk = torch.stack([bits.sum(), (bits * (torch.arange(bits.numel(), device=dev) % 8191 + 1)).sum()])
    hi, lo = chk.clone(), chk.clone()
    dist.all_reduce(hi, op=dist.ReduceOp.MAX); dist.all_reduce(lo, op=dist.ReduceOp.MIN)
    res = {"identical": bool((hi == lo).all().item())}
    # the weight-drop masks each rank's images were built from: the mode's seed is torch's, with no rank in it
    wd_seed = torch.tensor([int(torch.initial_seed())], dtype=torch.int64, device=dev)
    seeds_all = [torch.empty_like(wd_seed) for _ in range(world)]
    dist.all_gather(seeds_all, wd_seed)
    res["same_wd_seed"] = all(int(s.item()) == int(wd_seed.item()) for s in seeds_all)
    n = T * B * H
    masks = torch.empty(STEPS, L + 1, n, dtype=torch.uint8, device=dev)
    for i, (seed, step) in enumerate(seeds):
        for site in range(L + 1):
            _lib.check(lib.zrb_dropout_mask(seed, step, site, n, P_DROP, _lib.ptr(masks[i, site]), None))
    allm = [torch.empty_like(masks) for _ in range(world)]
    dist.all_gather(allm, masks)
    if rank == 0:
        torch.manual_seed(7)
        m2 = zaremba_b200.Model(V, H, L, P_DROP, 0.1, weight_drop=p_wd).to(dev)
        m2.train()
        tr2 = zaremba_b200.Trainer(m2, B * world, T, data_parallel=False)
        for i in range(STEPS):
            x = data[:, i * T:(i + 1) * T].t().contiguous().to(dev)
            y = data[:, i * T + 1:(i + 1) * T + 1].t().contiguous().to(dev)
            full = [torch.cat([allm[r][i, site].view(T, B, H) for r in range(world)], dim=1).contiguous()
                    for site in range(L + 1)]
            m2.set_explicit_dropout_masks(full)
            tr2.train_step(x, y, 1.0, 0.25)
        tr2.flush()
        res["err"] = (dp_p - tr2.flat_p).abs().max().item() / tr2.flat_p.abs().max().item()
        tr2.close()
    dist.barrier()
    tr.close()
    dist.destroy_process_group()
    q.put((rank, res))


@pytest.mark.parametrize("transport", ["ce", "nccl"])
def test_dp_step_equals_single_process(transport):
    """World 2 against one process at 2B replaying the ranks' activation masks: the weight-drop mask is common to the
    ranks, so both train the same weights."""
    from tests.test_gpu_multi import _need_two, _spawn
    _need_two()
    out = _spawn(_dp_worker, 2, transport)
    assert out[0]["identical"] and out[1]["identical"], "replicas diverged across ranks"
    assert out[0]["same_wd_seed"] and out[1]["same_wd_seed"]
    assert out[0]["err"] < 2e-3, out[0]
