"""The state a tensor-core context carries from one call to the next, against a cold twin, bit for bit.

A context keeps fp16 weight images (packed_version / packed_params / weights_version decide when they are rebuilt),
what each layer's W_hh images hold (raw, weight-drop masked, stale: DESIGN.md section 15), the lazy update's deferred
items, the average's state (section 16), the sparse-embedding bookkeeping and the modes.  Each entry point must leave
all of it right for whichever entry point comes next.  Two Model + Trainer pairs with the same seed, weights, states
and modes run the same seeded operation sequence (tests/_call_sequences.py):

  * warm: the configuration under test, lazy update on, caches left alone;
  * cold: strict update, and trainer.params_changed() before every operation (a flush, a version bump and a full
    repack from fp32), so it carries no image or deferred state from one call to the next.

The fused update writes what a fresh pack writes, lazy equals strict, and windows hold distinct tokens (the embedding
scatter is then deterministic), so after every operation everything it returns, the Trainer's states and the average's
count must be torch.equal between the twins, and after every operation that reads the weights (which applies pending
updates) so must flat_p, flat_g and flat_avg.  A failure prints the sequence; ZRB_SEQ=<seed> replays that seed alone.
A profiled replay of the warm twin checks that the comparison is not vacuous: evaluations after a fused update take the
cached images (no pack), and lazy items are pending when evaluations, decoding, swaps and dynamic evaluation arrive.

Plus the context re-creation regressions: a re-created context applies the old one's deferred updates, keeps the
Trainer's modes even at a reused address, and never silently loses the average.
"""
import ctypes as C
import gc
import math
import os

import pytest
import torch

from tests import _call_sequences as S
from tests.test_gpu_parity import _caller_nll_loss

pytestmark = pytest.mark.gpu

LR = 1.0


def _dev():
    return torch.device("cuda:0")


def _lib():
    from zaremba_b200 import _lib
    return _lib


class Row:
    def __init__(self, name):
        self.name = name
        self.H, self.T, self.B, self.plan, self.tied = S.ROWS[name]
        self.V = S.vocab(self.T, self.B)
        self.torch_seed = 4200 + list(S.ROWS).index(name)

    def windows(self, seed, T=None):
        """Four [T,B] windows of distinct tokens and their targets (CPU)."""
        T = T or self.T
        g = torch.Generator().manual_seed(seed)
        xs = [torch.randperm(self.V, generator=g)[:T * self.B].view(T, self.B) for _ in range(4)]
        ys = [torch.randint(0, self.V, (T, self.B), generator=g) for _ in range(4)]
        return xs, ys

    def check_plans(self, ctx):
        plans = _lib().rec_plans(ctx)
        fp, bp = plans["fwd"], plans["bwd"]
        want = {"persistent": (1, 1), "steps": (0, 0), "fwdonly": (1, 0)}[self.plan]
        if (bool(fp["ok"]), bool(bp["ok"])) != tuple(map(bool, want)):
            pytest.skip(f"H={self.H} B={self.B} gets {plans} on "
                        f"{torch.cuda.get_device_properties(0).multi_processor_count} SMs, not the {self.plan} plan")


class Twin:
    """One Model + Trainer of a row, with the per-twin objects a sequence needs."""

    def __init__(self, row, seed, warm, initial_wd):
        import zaremba_b200
        self.row, self.warm = row, warm
        torch.manual_seed(row.torch_seed)
        self.m = zaremba_b200.Model(row.V, row.H, S.L, S.P_DROP, 0.1, tied=row.tied, weight_drop=initial_wd).to(_dev())
        self.m.train()
        self.tr = zaremba_b200.Trainer(self.m, row.B, row.T, lazy_update=warm)
        g = torch.Generator().manual_seed(seed)
        for h, c in self.tr.states:
            h.copy_(torch.rand(h.shape, generator=g) - 0.5)
            c.copy_(torch.rand(c.shape, generator=g) * 2 - 1)
        self.xs, self.ys = row.windows(seed)
        self.cache = zaremba_b200.NeuralCache(row.H, row.B, 50, row.T)
        self.theta_g = self.tr.flat_p.clone()
        self.stats = None
        self.cm = None

    def close(self):
        if self.cm is not None:
            _leave(self)
        self.cache.close()
        self.tr.close()


def _leave(tw):
    cm, tw.cm = tw.cm, None
    if cm == "abi":
        _lib().check(_lib().load().zrb_swap_average(tw.tr.ctx, C.byref(tw.tr._ps), tw.tr._stream()))
        tw.tr._swapped = False
    else:
        cm.__exit__(None, None, None)


def _states(tr):
    return [t.clone() for st in tr.states for t in st]


def _wide(tw, T, seed):
    xs, ys = tw.row.windows(seed, T)
    return xs[0], ys[0]


def _dev_w(tw, w):
    return tw.xs[w].to(_dev()).contiguous(), tw.ys[w].to(_dev()).contiguous()


def _train_phased(tr, x, y, max_norm):
    """zrb_train_step_begin / _layer (L-1..0) / _update driven directly, with the Trainer's bookkeeping."""
    lib = _lib().load()
    T, B = x.shape
    tr._check_not_swapped()
    tr._check_versions()
    _lib().check(lib.zrb_train_step_begin(tr.ctx, C.byref(tr._ps), C.byref(tr._gs), _lib().ptr(x), _lib().ptr(y), T, B,
                                          C.byref(tr._st), C.byref(tr._st), tr.seed, tr.step, _lib().ptr(tr.loss),
                                          tr._stream()))
    for l in range(S.L - 1, -1, -1):
        _lib().check(lib.zrb_train_step_layer(tr.ctx, C.byref(tr._ps), C.byref(tr._gs), l, tr._stream()))
    _lib().check(lib.zrb_train_step_update(tr.ctx, C.byref(tr._ps), C.byref(tr._gs), LR, max_norm, _lib().ptr(tr.norm),
                                           tr._stream()))
    tr.step += 1
    tr._pending = True
    return tr.loss, tr.norm


def _dropin_grads(tw, x, y):
    """Model.forward in train mode and autograd backward; the gradients are returned, .grad is left alone."""
    m = tw.m
    states = [(h.clone(), c.clone()) for h, c in tw.tr.states]
    scores, states = m(x, states)
    params = m.ordered_parameters()
    grads = torch.autograd.grad(_caller_nll_loss(scores, y), params)
    return scores.detach(), params, grads, [t for st in states for t in st]


def _unit(tw, seed):
    """zrb_lstm_layer_fwd / _bwd on the model's own context: one random layer of the model's width."""
    lib, H, T, B = _lib().load(), tw.row.H, tw.row.T, tw.row.B
    g = torch.Generator().manual_seed(seed)
    mk = lambda *s, a=0.08: ((torch.rand(*s, generator=g) * 2 - 1) * a).to(_dev())
    w_ih, w_hh, b_ih, b_hh = mk(4 * H, H), mk(4 * H, H), mk(4 * H), mk(4 * H)
    x, h0, c0, dy = mk(T * B, H, a=1.0), mk(B, H, a=0.5), mk(B, H, a=1.0), mk(T * B, H, a=0.1)
    y, hT, cT = torch.empty(T * B, H, device=_dev()), torch.empty(B, H, device=_dev()), torch.empty(B, H, device=_dev())
    P = _lib().ptr
    _lib().check(lib.zrb_lstm_layer_fwd(tw.tr.ctx, P(w_ih), P(w_hh), P(b_ih), P(b_hh), P(x), T, B, P(h0), P(c0), P(y),
                                        P(hT), P(cT), None))
    dx, dwi, dwh = torch.empty_like(x), torch.empty_like(w_ih), torch.empty_like(w_hh)
    dbi, dbh = torch.empty_like(b_ih), torch.empty_like(b_hh)
    _lib().check(lib.zrb_lstm_layer_bwd(tw.tr.ctx, P(dy), P(dx), P(dwi), P(dwh), P(dbi), P(dbh), None))
    return dict(y=y, hT=hT, cT=cT, dx=dx, dwi=dwi, dwh=dwh, dbi=dbi, dbh=dbh)


def _refuse(tw, kind, seed):
    tr, m, row = tw.tr, tw.m, tw.row
    x, y = _dev_w(tw, 0)
    if kind == "train_in_avg":
        with pytest.raises(RuntimeError):
            tr.train_step(x, y, LR, 0.25)
    elif kind == "start_in_avg":
        with pytest.raises(RuntimeError):
            tr.start_averaging()
    elif kind == "dyneval_wide":
        xw = torch.arange(row.T * (row.B + 1), device=_dev()).view(row.T, row.B + 1) % row.V
        with pytest.raises(ValueError):
            tr.dynamic_eval_step(xw, xw, tw.theta_g, 0.05)
    elif kind == "generate_wide":
        with pytest.raises(ValueError):
            m.generate(torch.zeros(2, m._ctx_key[1] + 1, dtype=torch.int64), 2, seed=1)
    elif kind == "unit_no_plan":
        with pytest.raises(_lib().ZrbError):
            _unit(tw, seed)
    elif kind == "enter_n0":
        with pytest.raises(_lib().ZrbError):
            with tr.averaged_weights():
                pass
    elif kind == "stats_wide_avg":
        with pytest.raises(ValueError):
            tr.gradient_stats([_wide(tw, m._ctx_key[0] + S.GROW, seed)])
    elif kind == "fwd_wide_avg":
        xw, _ = _wide(tw, m._ctx_key[0] + S.GROW, seed)
        with pytest.raises(RuntimeError), torch.no_grad():
            m(xw, [(h.clone(), c.clone()) for h, c in tr.states])
    else:
        raise AssertionError(kind)
    return {}


def run_op(tw, op, a):
    """Run one operation on a twin; returns what it computed (tensors and numbers to compare)."""
    lib, tr, m = _lib().load(), tw.tr, tw.m
    P = _lib().ptr
    if op in ("train_clip", "train_noclip"):
        x, y = _dev_w(tw, a["w"])
        loss, norm = tr.train_step(x, y, LR, 0.05 if op == "train_clip" else 1e9)
        return dict(loss=loss.clone(), norm=norm.clone())
    if op == "train_host":
        loss, norm = tr.train_step_host(tw.xs[a["w"]], tw.ys[a["w"]], LR, 0.25)
        return dict(loss=loss, norm=norm)
    if op == "train_phased":
        x, y = _dev_w(tw, a["w"])
        loss, norm = _train_phased(tr, x, y, 0.25)
        return dict(loss=loss.clone(), norm=norm.clone())
    if op == "eval":
        loss, tp = tr.eval_step(*_dev_w(tw, a["w"]), want_probs=True)
        return dict(loss=loss.clone(), tp=tp.clone())
    if op == "ppl":
        return dict(ppl=tr.perplexity([(tw.xs[a["w"]], tw.ys[a["w"]]), (tw.xs[a["w2"]], tw.ys[a["w2"]])]))
    if op == "eval_cache":
        loss, pm, pc = tr.eval_step(*_dev_w(tw, a["w"]), want_probs=True, cache=tw.cache, theta=0.3, lam=0.1)
        return dict(loss=loss.clone(), pm=pm.clone(), pc=pc.clone())
    if op == "fwd_eval":
        m.eval()
        try:
            with torch.no_grad():
                scores, st = m(tw.xs[a["w"]], [(h.clone(), c.clone()) for h, c in tr.states])
        finally:
            m.train()
        return dict(scores=scores, states=[t for s in st for t in s])
    if op == "generate":
        g = torch.Generator().manual_seed(a["seed"])
        prompt = torch.randint(0, tw.row.V, (3, a["Bp"]), generator=g)
        tok, lp, st = m.generate(prompt, a["n_new"], seed=a["seed"])
        return dict(tok=tok, lp=lp, states=[t for s in st for t in s])
    if op == "beam":
        g = torch.Generator().manual_seed(a["seed"])
        prompt = torch.randint(0, tw.row.V, (2, a["Bp"]), generator=g)
        tok, lp, sc, st = m.beam_search(prompt, a["n_new"], a["K"])
        return dict(tok=tok, lp=lp, sc=sc, states=[t for s in st for t in s])
    if op in ("fwd_clip_sgd", "fwd_torch_sgd"):
        scores, params, grads, st = _dropin_grads(tw, *_dev_w(tw, a["w"]))
        if op == "fwd_clip_sgd":      # the library's clip + SGD, as tests/test_gpu_parity.py calls it
            n = len(params)
            norm = torch.zeros((), device=_dev())
            _lib().check(lib.zrb_clip_sgd(tr.ctx, n, (C.c_void_p * n)(*[p.data_ptr() for p in params]),
                                          (C.c_void_p * n)(*[g.data_ptr() for g in grads]),
                                          (C.c_int64 * n)(*[p.numel() for p in params]), 0.5, 0.25, P(norm), None))
        else:                          # a torch SGD step: the parameters' versions change outside the library
            tr.flush()
            norm = torch.zeros(())
            with torch.no_grad():
                for p, g in zip(params, grads):
                    p.add_(g, alpha=-0.5)
        return dict(scores=scores, grads=list(grads), states=st, norm=norm)
    if op == "grad_stats":
        tw.stats = tr.gradient_stats([(tw.xs[a["w"]], tw.ys[a["w"]]), (tw.xs[a["w2"]], tw.ys[a["w2"]])])
        return dict(rms=tw.stats.rms.clone(), mean=tw.stats.mean.clone())
    if op in ("dyneval_sgd", "dyneval_rms"):
        if op == "dyneval_rms" and tw.stats is None:
            tw.stats = tr.gradient_stats([(tw.xs[0], tw.ys[0])])
        x, y = _dev_w(tw, a["w"])
        if op == "dyneval_sgd":
            loss = tr.dynamic_eval_step(x, y, tw.theta_g, 0.05, lam=0.01)
        else:
            loss = tr.dynamic_eval_step(x, y, tw.theta_g, 0.002, lam=0.01, stats=tw.stats)
        return dict(loss=loss.clone())
    if op == "avg_start":
        tr.start_averaging()
        return {}
    if op == "avg_stop":
        tr.stop_averaging()
        return {}
    if op == "avg_enter":
        if a["abi"]:                   # zrb_swap_average itself must apply pending updates first
            _lib().check(lib.zrb_swap_average(tr.ctx, C.byref(tr._ps), tr._stream()))
            tr._swapped, tw.cm = True, "abi"
        else:
            tw.cm = tr.averaged_weights()
            tw.cm.__enter__()
        return {}
    if op == "avg_leave":
        _leave(tw)
        return {}
    if op == "wd":
        m.weight_drop = a["p"]
        _lib().check(lib.zrb_set_weight_drop(tr.ctx, a["p"], a["seed"]))
        return {}
    if op == "ed":
        m.embed_dropout = a["p"]
        _lib().check(lib.zrb_set_embed_dropout(tr.ctx, a["p"], a["seed"]))
        return {}
    if op == "var":
        m.variational, m.p_rec = a["on"], a["p_rec"]
        _lib().check(lib.zrb_set_variational_dropout(tr.ctx, 1 if a["on"] else 0, a["p_rec"]))
        return {}
    if op == "artar":
        tr._ar, tr._tar = a["ar"], a["tar"]
        _lib().check(lib.zrb_set_activation_reg(tr.ctx, a["ar"], a["tar"]))
        return {}
    if op == "keep_clipped":
        tr._keep_clipped = a["on"]
        _lib().check(lib.zrb_set_keep_clipped_grads(tr.ctx, 1 if a["on"] else 0))
        return {}
    if op == "lazy":
        if tw.warm:                    # the cold twin stays strict
            tr._lazy = a["on"]
            _lib().check(lib.zrb_set_lazy_update(tr.ctx, 1 if a["on"] else 0))
        return {}
    if op == "edit":
        tr.flush()
        with torch.no_grad():
            m.ordered_parameters()[a["i"]].add_(a["delta"])
        return {}
    if op == "flush":
        tr.flush()
        return {}
    if op == "unit":
        return _unit(tw, a["seed"])
    if op in ("grow_fwd", "grow_stats"):
        if a["refused"]:
            return _refuse(tw, "fwd_wide_avg" if op == "grow_fwd" else "stats_wide_avg", a["seed"])
        x, y = _wide(tw, a["T"], a["seed"])
        if op == "grow_stats":
            tw.stats = tr.gradient_stats([(x, y)])
            return dict(rms=tw.stats.rms.clone(), mean=tw.stats.mean.clone())
        if not a["train"]:
            m.eval()
        try:
            with torch.no_grad():
                scores, st = m(x, [(h.clone(), c.clone()) for h, c in tr.states])
        finally:
            m.train()
        return dict(scores=scores, states=[t for s in st for t in s])
    if op == "refuse":
        return _refuse(tw, a["kind"], a["seed"])
    raise AssertionError(op)


def _flat(v):
    if isinstance(v, (list, tuple)):
        return [u for x in v for u in _flat(x)]
    return [v]


def _diff(a, b):
    """Names of the entries of two op results that are not bit-identical."""
    bad = []
    for k in a:
        for i, (u, v) in enumerate(zip(_flat(a[k]), _flat(b[k]))):
            same = torch.equal(u.cpu(), v.cpu()) if isinstance(u, torch.Tensor) else u == v
            if not same:
                bad.append(f"{k}[{i}]")
    return bad


def _full_state(tw):
    tr = tw.tr
    out = dict(flat_p=tr.flat_p.clone(), flat_g=tr.flat_g.clone(), n=tr.averaged_steps, states=_states(tr))
    if getattr(tr, "flat_avg", None) is not None:
        out["flat_avg"] = tr.flat_avg.clone()
    return out


def _seeds():
    only = os.environ.get("ZRB_SEQ")
    return [int(only)] if only else S.SEEDS


def _run_sequence(row, seed, monkeypatch):
    seq = S.sequence(row.name, seed)
    if row.plan == "fwdonly":          # for every context of the sequence, re-created ones too
        monkeypatch.setenv("ZRB_REC", "fwdonly")
    twins = [Twin(row, seed, warm, seq[0]["initial_wd"]) for warm in (True, False)]
    warm, cold = twins
    where = lambda i, what: (f"{row.name} seed {seed}: after op {i} ({seq[i]['op']} {seq[i]['args']}) the warm and "
                             f"cold twins differ in {what}\nreplay with ZRB_SEQ={seed}\n{S.describe(seq)}")
    try:
        row.check_plans(warm.tr.ctx)
        for i, s in enumerate(seq):
            cold.tr.params_changed()
            res = [run_op(tw, s["op"], s["args"]) for tw in twins]
            torch.cuda.synchronize()
            bad = _diff(*res)
            assert not bad, where(i, bad)
            full = [_full_state(tw) for tw in twins]
            keys = ["n", "states"] + (["flat_p", "flat_g", "flat_avg"] if S.flushes(s["op"], s["args"]) else [])
            bad = _diff({k: full[0].get(k, []) for k in keys}, {k: full[1].get(k, []) for k in keys})
            assert not bad, where(i, bad)
    finally:
        for tw in twins:
            tw.close()
        del twins, warm, cold
        gc.collect()


@pytest.mark.parametrize("row", list(S.ROWS))
def test_warm_context_equals_cold_twin(row, monkeypatch):
    r = Row(row)
    for seed in _seeds():
        _run_sequence(r, seed, monkeypatch)


# ---- the comparison is not vacuous ------------------------------------------------------------------------------------
def _profiled_replay(row, seed, monkeypatch):
    """The warm twin alone, zrb_prof_enable on around every operation that is not a Trainer train step (profiling
    turns the lazy riding off).  Per operation: (op, previous op, launch-group counts per class, or None)."""
    lib = _lib().load()
    seq = S.sequence(row.name, seed)
    if row.plan == "fwdonly":
        monkeypatch.setenv("ZRB_REC", "fwdonly")
    tw = Twin(row, seed, True, seq[0]["initial_wd"])
    out = []
    try:
        row.check_plans(tw.tr.ctx)
        for s in seq:
            prof = s["op"] not in S.TRAIN
            serial = tw.m._ctx_serial
            if prof:
                _lib().check(lib.zrb_prof_enable(tw.m._ctx, 1))
            run_op(tw, s["op"], s["args"])
            counts = None
            if prof and tw.m._ctx_serial == serial:
                ms, cnt = (C.c_float * 12)(), (C.c_int64 * 12)()
                _lib().check(lib.zrb_prof_read(tw.m._ctx, ms, cnt))
                _lib().check(lib.zrb_prof_enable(tw.m._ctx, 0))
                counts = dict(zip(_lib().PROF_CLASSES, cnt))
            out.append((s["op"], s["prev"], counts))
    finally:
        tw.close()
        del tw
        gc.collect()
    return out


@pytest.mark.parametrize("row", list(S.ROWS))
def test_sequences_exercise_cached_images_and_pending_updates(row, monkeypatch):
    """Per row: some evaluation right after a fused update took the images the update wrote (no pack), and on the
    persistent rows lazy items were pending when an evaluation, decode, swap or dynamic evaluation arrived.  Decoding
    and dynamic evaluation after an update may repack legitimately (a model-level call's first version check, W_hh after
    a weight-dropped step), so their cached path is asserted over all rows together, once every row has run."""
    r = Row(row)
    runs = [_profiled_replay(r, seed, monkeypatch) for seed in _seeds()]
    after_update = [(op, c) for run in runs for op, prev, c in run if prev in S.TRAIN and c is not None]
    cached = {op for op, c in after_update if c["pack"] == 0}
    _CACHED_ANYWHERE.update(cached)
    _ROWS_SEEN.add(row)
    assert cached & set(S.EVAL), f"no evaluation after a fused update took the cached images: {after_update}"
    if len(_ROWS_SEEN) == len(S.ROWS) and not os.environ.get("ZRB_SEQ"):
        assert _CACHED_ANYWHERE & {"generate", "beam", "dyneval_sgd", "dyneval_rms"}, \
            "no generate / beam / dyneval after a fused update took the cached images on any row"
    print(f"\n{row}: cached images after an update in {sorted(cached)}")
    if r.plan != "persistent":
        return                          # the lazy update defers only where both persistent kernels run
    flushed = set()
    for run in runs:
        for op, prev, c in run:
            # a deferred item is applied under the clip_sgd class; dynamic evaluation's own update is one more group
            if c is not None and c["clip_sgd"] >= (2 if op in ("dyneval_sgd", "dyneval_rms") else 1):
                flushed.add(op)
    kinds = set(S.EVAL) | set(S.DECODE) | {"avg_enter", "dyneval_sgd", "dyneval_rms"}
    assert flushed & kinds, "lazy items were never pending when an evaluation, decode, swap or dyneval arrived"
    print(f"{row}: pending lazy items applied by {sorted(flushed)}")


_CACHED_ANYWHERE, _ROWS_SEEN = set(), set()


# ---- context re-creation ------------------------------------------------------------------------------------------------
def _pair(row, seed=7, **tkw):
    import zaremba_b200
    out = []
    for warm in (True, False):
        torch.manual_seed(row.torch_seed)
        m = zaremba_b200.Model(row.V, row.H, S.L, S.P_DROP, 0.1).to(_dev())
        m.train()
        out.append((m, zaremba_b200.Trainer(m, row.B, row.T, lazy_update=warm, **tkw)))
    row.check_plans(out[0][1].ctx)
    return out


def test_context_growth_applies_pending_lazy_updates():
    """A lazy step defers the update of layers >= 1 and fc.W; model(x) with a longer window then re-creates the
    context.  The new context must start from the updated weights: the forward's scores and, after a flush, flat_p equal
    the strict twin's bit for bit."""
    r = Row("persistent-untied")
    xs, ys = r.windows(11)
    xw, _ = r.windows(12, r.T + S.GROW)
    res = []
    for m, tr in _pair(r):
        tr.train_step(xs[0].to(_dev()), ys[0].to(_dev()), LR, 0.25)
        with torch.no_grad():
            scores, _ = m(xw[0], m.state_init(r.B))
        assert m._ctx_key[0] == r.T + S.GROW, "the window must have re-created the context"
        tr.flush()
        torch.cuda.synchronize()
        res.append((scores.clone(), tr.flat_p.clone()))
        tr.close()
    (s1, p1), (s2, p2) = res
    assert torch.equal(p1, p2), "the lazy step's deferred update was lost when the context was re-created"
    assert torch.equal(s1, s2), "the re-created context did not compute with the updated weights"


def test_context_growth_keeps_the_average():
    """With averaging on, a window longer than the context is refused before anything changes -- gradient_stats
    with ValueError, Model.forward with RuntimeError, inside averaged_weights() too -- and averaging goes on: the count,
    the average and the weights equal a twin that never asked, bit for bit."""
    r = Row("persistent-untied")
    xs, ys = r.windows(21)
    xw, yw = r.windows(22, r.T + S.GROW)
    res = []
    for k, (m, tr) in enumerate(_pair(r)):
        tr.start_averaging()
        for s in range(2):
            tr.train_step(xs[s].to(_dev()), ys[s].to(_dev()), LR, 0.25)
        if k == 0:
            try:
                tr.gradient_stats([(xw[0], yw[0])])
            except ValueError as e:
                assert "average" in str(e), e
            else:
                pytest.fail(f"gradient_stats re-created the context while averaging: averaged_steps now reads "
                            f"{tr.averaged_steps} instead of 2, the average was lost")
            step = m._drop_step
            with pytest.raises(RuntimeError, match="average"), torch.no_grad():
                m(xw[0], m.state_init(r.B))
            assert m._drop_step == step, "a refused forward consumed a dropout step"
            with tr.averaged_weights():
                with pytest.raises(ValueError, match="average"):
                    tr.gradient_stats([(xw[0], yw[0])])
            assert m._ctx_key[0] == r.T, "the context was re-created"
        assert tr.averaged_steps == 2, "the average was lost"
        tr.train_step(xs[2].to(_dev()), ys[2].to(_dev()), LR, 0.25)
        tr.flush()
        torch.cuda.synchronize()
        res.append((tr.averaged_steps, tr.flat_p.clone(), tr.flat_avg.clone()))
        tr.close()
    (n1, p1, a1), (n2, p2, a2) = res
    assert n1 == n2 == 3, (n1, n2)
    assert torch.equal(p1, p2) and torch.equal(a1, a2), "the refusals changed the weights or the average"


def test_trainer_modes_survive_context_growth():
    """gradient_stats on longer windows re-creates the context (averaging off).  The Trainer must hand the new context
    its modes -- AR / TAR, keep_clipped_grads, the lazy update, the sparse embedding -- even when the new context reuses
    the old one's address: the next train step equals that of a Trainer whose context was created at the longer shape
    from the start, bit for bit (loss, norm, AR / TAR values, weights, gradients)."""
    import zaremba_b200
    r = Row("persistent-untied")
    xs, ys = r.windows(31)
    xw, yw = r.windows(32, r.T + S.GROW)
    res = []
    for grown in (True, False):
        torch.manual_seed(r.torch_seed)
        m = zaremba_b200.Model(r.V, r.H, S.L, S.P_DROP, 0.1).to(_dev())
        m.train()
        if not grown:
            m._context(r.T + S.GROW, r.B)
        tr = zaremba_b200.Trainer(m, r.B, r.T, lazy_update=True, keep_clipped_grads=True, ar=2.0, tar=1.0)
        r.check_plans(tr.ctx)
        before = tr.ctx.value
        tr.gradient_stats([(xw[0], yw[0])])
        if grown:
            print(f"\nre-created context at the {'same' if tr.ctx.value == before else 'another'} address")
        for s in range(2):
            loss, norm = tr.train_step(xs[s].to(_dev()), ys[s].to(_dev()), LR, 0.05)
        reg = tr.activation_reg.clone()
        tr.flush()
        torch.cuda.synchronize()
        res.append((loss.clone(), norm.clone(), reg, tr.flat_p.clone(), tr.flat_g.clone()))
        tr.close()
    assert res[1][2].abs().sum() > 0
    for name, a, b in zip(("loss", "norm", "activation_reg", "flat_p", "flat_g"), *res):
        assert torch.equal(a, b), f"{name} differs after the context was re-created"


def test_leaving_averaged_weights_after_the_context_was_dropped():
    """If the context goes while the average is swapped in (here: dropped by hand), leaving averaged_weights() still
    restores the weights and the average bit for bit, by copies, and reports the lost average with RuntimeError;
    training then goes on with averaging off."""
    r = Row("persistent-untied")
    xs, ys = r.windows(41)
    (m, tr), _ = _pair(r)
    tr.start_averaging()
    for s in range(2):
        tr.train_step(xs[s].to(_dev()), ys[s].to(_dev()), LR, 0.25)
    tr.flush()
    torch.cuda.synchronize()
    p0, a0 = tr.flat_p.clone(), tr.flat_avg.clone()
    with pytest.raises(RuntimeError, match="average"):
        with tr.averaged_weights():
            m._destroy_ctx()
    torch.cuda.synchronize()
    assert torch.equal(tr.flat_p, p0) and torch.equal(tr.flat_avg, a0), "leaving did not restore weights and average"
    assert tr.averaged_steps == 0 and m._ctx_pinned is None
    loss, _ = tr.train_step(xs[2].to(_dev()), ys[2].to(_dev()), LR, 0.25)
    assert math.isfinite(loss.item())
    tr.close()
