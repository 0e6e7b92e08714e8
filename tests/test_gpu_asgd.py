"""GPU tests of iterate averaging (NT-ASGD, DESIGN.md section 16) at the recurrence-plan branches of
tests/test_gpu_dropout.py and at the Small / Medium / Large shapes.

  * with averaging on for k steps, loss, clip norm, the weights and `.grad` are bit-identical to a twin with it off, and
    the average equals the fp32 restatement of tests/_asgd_oracle.py applied to the twin's weights after every step,
    bit for bit -- dense and rows-only embedding, tied, weight drop, variational dropout, keep_clipped_grads,
    train_step_host, the validation engine, and the lazy update (also with start_averaging() and averaged_weights()
    between steps while updates are pending);
  * zrb_swap_average: two swaps restore weights and average bit for bit; perplexity inside averaged_weights() equals
    that of a fresh Trainer loaded from average_state_dict(), and that of a full repack of the swapped-in weights (the
    fp16 images the swap wrote are the pack's); under weight drop an eval after the swap reads the raw weights;
  * refusals: a swap with n = 0, a train step while swapped, averages that alias the parameters;
  * two GPUs (skipped otherwise): every rank's average is identical and is the restatement over its weights.
Windows hold distinct tokens, so the embedding scatter is deterministic and twins can be compared bit for bit.
"""
import ctypes as C
import gc
import math

import numpy as np
import pytest
import torch

from tests import _asgd_oracle as AO
from tests.test_gpu_dropout import L, P_DROP, ROW_IDS, Row
from tests.test_gpu_parity import ENGINES

pytestmark = pytest.mark.gpu

LR, MAX_NORM = 1.0, 0.25
K = 4                    # train steps per run


def _dev():
    return torch.device("cuda:0")


def _winit(row):
    return min(row.winit, 1.3 / math.sqrt(row.H))


class Shape:
    """A recipe's model shape with two windows of distinct tokens (Row's interface, no plan branch)."""

    def __init__(self, name, engine, V, H, T, B, seed):
        self.name, self.engine, self.V, self.H, self.T, self.B, self.branch = name, engine, V, H, T, B, None
        self.winit, self.torch_seed = 0.05, seed
        g = torch.Generator().manual_seed(seed)
        self.x = [torch.randperm(V, generator=g)[:T * B].view(T, B) for _ in range(2)]
        self.y = [torch.randint(0, V, (T, B), generator=g) for _ in range(2)]
        self.h0 = [(torch.zeros(B, H), torch.zeros(B, H)) for _ in range(L)]

    def states(self):
        return [(h.view(1, self.B, self.H).to(_dev()), c.view(1, self.B, self.H).to(_dev())) for h, c in self.h0]

    def check_branch(self, ctx):
        pass


SHAPES = {"small": (10000, 200, 20, 20), "medium": (10000, 650, 35, 20), "large": (10000, 1500, 35, 20)}


def _row(name):
    if name in SHAPES:
        return Shape(name, "tc", *SHAPES[name], seed=77)
    return Row(name)


# feature -> (Model kwargs, Trainer kwargs, host steps, dense embedding)
FEATURES = {
    "rows_only": ({}, {}, False, False),
    "dense_embed": ({}, {}, False, True),
    "tied": ({"tied": True}, {}, False, False),
    "weight_drop": ({"weight_drop": 0.5}, {}, False, False),
    "variational": ({"variational": True}, {}, False, False),
    "keep_clipped": ({}, {"keep_clipped_grads": True}, False, False),
    "host": ({}, {}, True, False),
    "lazy": ({}, {"lazy_update": True}, False, False),
    "lazy_tied_wd": ({"tied": True, "weight_drop": 0.5}, {"lazy_update": True}, False, False),
}
FEATURE_ROW = [r for r in ("tc_h48", "simt_h48") if r in ROW_IDS]
CASES = ([(r, "rows_only") for r in ROW_IDS] + [(r, f) for r in FEATURE_ROW for f in FEATURES if f != "rows_only"]
         + ([(s, "rows_only") for s in SHAPES] + [("medium", "lazy"), ("large", "lazy")] if "tc" in ENGINES else []))


def _model(row, **kw):
    import zaremba_b200
    torch.manual_seed(row.torch_seed)
    m = zaremba_b200.Model(row.V, row.H, L, P_DROP, _winit(row), engine=row.engine, **kw).to(_dev())
    m.train()
    return m


def _trainer(row, feature, monkeypatch):
    import zaremba_b200
    mkw, tkw, _, dense = FEATURES[feature]
    monkeypatch.setenv("ZRB_EMBED_SPARSE", "0" if dense else "1")
    m = _model(row, **mkw)
    tr = zaremba_b200.Trainer(m, row.B, row.T, **tkw)
    for (h, c), (h0, c0) in zip(tr.states, row.states()):
        h.copy_(h0)
        c.copy_(c0)
    row.check_branch(tr.ctx)
    return m, tr


def _step(tr, row, s, host):
    x, y = row.x[s % 2], row.y[s % 2]
    if host:
        loss, norm = tr.train_step_host(x, y, LR, MAX_NORM)
        return torch.tensor(loss), torch.tensor(norm)
    loss, norm = tr.train_step(x.to(_dev()), y.to(_dev()), LR, MAX_NORM)
    return loss.clone(), norm.clone()


def _run(row, feature, monkeypatch, avg_from):
    """K steps, averaging started before step avg_from (None: off); per step loss, norm, flat_p, flat_g, flat_avg, n."""
    m, tr = _trainer(row, feature, monkeypatch)
    host = FEATURES[feature][2]
    out = []
    for s in range(K):
        if avg_from is not None and s == avg_from:
            tr.start_averaging()
        loss, norm = _step(tr, row, s, host)
        tr.flush()
        torch.cuda.synchronize()
        out.append(dict(loss=loss.cpu(), norm=norm.cpu(), p=tr.flat_p.cpu(), g=tr.flat_g.cpu(),
                        a=tr.flat_avg.cpu() if avg_from is not None and s >= avg_from else None,
                        n=tr.averaged_steps))
    tr.close()
    del tr, m
    gc.collect()
    return out


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def _oracle_check(on, off, avg_from, what):
    av = AO.Averager()
    for s, (a, b) in enumerate(zip(on, off)):
        for k in ("loss", "norm", "p", "g"):
            assert _bits_equal(a[k], b[k]), f"{what} step {s}: {k} differs from the mode-off twin"
        if s < avg_from:
            assert a["n"] == 0
            continue
        want = av.update(b["p"].numpy())
        assert a["n"] == av.n, (a["n"], av.n)
        got = a["a"].numpy()
        if got.tobytes() != want.tobytes():
            bad = np.flatnonzero(got.view(np.int32) != want.view(np.int32))
            raise AssertionError(f"{what} step {s}: {bad.size} averaged elements differ, first at {bad[0]}: "
                                 f"{got[bad[0]]!r} vs {want[bad[0]]!r}")


@pytest.mark.parametrize("row,feature", CASES, ids=[f"{r}-{f}" for r, f in CASES])
def test_average_is_the_restatement_and_weights_are_untouched(row, feature, monkeypatch):
    r = _row(row)
    avg_from = 1                      # a step other than the first: the average starts from the weights of that step
    on = _run(r, feature, monkeypatch, avg_from)
    off = _run(r, feature, monkeypatch, None)
    _oracle_check(on, off, avg_from, f"{row}/{feature}")


@pytest.mark.parametrize("row", [r for r in ("tc_h48", "two_cells_n32", "medium") if r in ROW_IDS or r in SHAPES])
def test_lazy_with_pending_updates_equals_strict(row, monkeypatch):
    """Lazy update, no flush between steps: start_averaging() and an averaged_weights() block (with an eval inside)
    entered while updates are pending; the final weights and average equal the strict run's bit for bit."""
    if "tc" not in ENGINES:
        pytest.skip("the lazy update is a tensor-core engine schedule")
    r = _row(row)
    res = {}
    for feature in ("lazy", "rows_only"):
        m, tr = _trainer(r, feature, monkeypatch)
        for s in range(K):
            if s == 1:
                tr.start_averaging()
            if s == 3:
                saved = [t.clone() for st in tr.states for t in st]
                with tr.averaged_weights():
                    tr.eval_step(r.x[0].to(_dev()), r.y[0].to(_dev()))
                for t, v in zip([t for st in tr.states for t in st], saved):
                    t.copy_(v)
            _step(tr, r, s, False)
        tr.flush()
        torch.cuda.synchronize()
        res[feature] = (tr.flat_p.cpu(), tr.flat_avg.cpu(), tr.averaged_steps)
        tr.close()
        del tr, m
        gc.collect()
    (p1, a1, n1), (p2, a2, n2) = res["lazy"], res["rows_only"]
    assert n1 == n2 == K - 1
    assert _bits_equal(p1, p2), "lazy weights differ from strict"
    assert _bits_equal(a1, a2), "lazy average differs from strict"


def _ppl(tr, row):
    return tr.perplexity([(row.x[0], row.y[0]), (row.x[1], row.y[1])])


@pytest.mark.parametrize("row,feature", [(r, f) for r in FEATURE_ROW + ["two_cells_n32"] if r in ROW_IDS
                                         for f in ("rows_only", "tied", "weight_drop", "lazy")
                                         if not (f == "lazy" and r.startswith("simt"))])
def test_swap(row, feature, monkeypatch):
    import zaremba_b200
    r = _row(row)
    m, tr = _trainer(r, feature, monkeypatch)
    tr.start_averaging()
    for s in range(3):
        _step(tr, r, s, False)
    tr.flush()
    torch.cuda.synchronize()
    p0, a0 = tr.flat_p.clone(), tr.flat_avg.clone()
    ref_sd = tr.average_state_dict()
    with tr.averaged_weights():
        assert _bits_equal(tr.flat_p, a0) and _bits_equal(tr.flat_avg, p0), "the swap is not an exchange"
        ppl_swapped = _ppl(tr, r)
        with pytest.raises(RuntimeError):
            _step(tr, r, 3, False)
        # the library refuses too, whatever the caller checks
        from zaremba_b200 import _lib
        assert _lib.load().zrb_train_step_update(tr.ctx, C.byref(tr._ps), C.byref(tr._gs), LR, MAX_NORM,
                                                 _lib.ptr(tr.norm), None) == -1
        sd_inside = tr.average_state_dict()
        tr.params_changed()               # a full repack of the swapped-in weights
        ppl_repacked = _ppl(tr, r)
        n_inside = tr.averaged_steps
    torch.cuda.synchronize()
    assert _bits_equal(tr.flat_p, p0) and _bits_equal(tr.flat_avg, a0), "two swaps do not restore"
    assert n_inside == tr.averaged_steps == 3, "eval must not advance n"
    assert ppl_swapped == ppl_repacked, (ppl_swapped, ppl_repacked)
    for k, v in ref_sd.items():
        assert _bits_equal(v, sd_inside[k]), k
    # a fresh Trainer whose model holds the average
    mkw = FEATURES[feature][0]
    m2 = _model(r, **mkw)
    m2.load_state_dict(ref_sd)
    tr2 = zaremba_b200.Trainer(m2, r.B, r.T)
    ppl_fresh = _ppl(tr2, r)
    assert ppl_swapped == ppl_fresh, (ppl_swapped, ppl_fresh)
    if mkw.get("weight_drop"):
        # eval reads the raw weights: the same model without weight drop scores the same
        m3 = _model(r, **{k: v for k, v in mkw.items() if k != "weight_drop"})
        m3.load_state_dict(ref_sd)
        tr3 = zaremba_b200.Trainer(m3, r.B, r.T)
        assert _ppl(tr3, r) == ppl_swapped
        tr3.close()
    tr2.close()
    tr.close()
    del tr, tr2, m, m2
    gc.collect()


def test_refusals(monkeypatch):
    from zaremba_b200 import _lib
    row = FEATURE_ROW[0] if FEATURE_ROW else ROW_IDS[0]
    r = _row(row)
    m, tr = _trainer(r, "rows_only", monkeypatch)
    lib = _lib.load()
    assert tr.averaged_steps == 0
    tr.start_averaging()
    with pytest.raises(_lib.ZrbError):           # n = 0: nothing to swap in
        with tr.averaged_weights():
            pass
    assert not getattr(tr, "_swapped", False)
    _step(tr, r, 0, False)
    assert tr.averaged_steps == 1
    tr.start_averaging()                          # restart
    assert tr.averaged_steps == 0
    _step(tr, r, 1, False)
    assert tr.averaged_steps == 1
    tr.stop_averaging()
    assert tr.averaged_steps == 0
    p_before = tr.flat_p.clone()
    # averages that alias the parameters / gradients: refused before anything is launched
    for alias in (tr._ps, tr._gs):
        assert lib.zrb_set_average(tr.ctx, C.byref(alias)) == 0
        rc = lib.zrb_train_step_update(tr.ctx, C.byref(tr._ps), C.byref(tr._gs), LR, MAX_NORM, _lib.ptr(tr.norm), None)
        assert rc == -1, rc
        assert "overlaps" in lib.zrb_last_error().decode()
    assert lib.zrb_set_average(tr.ctx, None) == 0
    torch.cuda.synchronize()
    assert _bits_equal(tr.flat_p, p_before)
    # average tensors that overlap each other
    bad = _lib.ZrbParams()
    C.memmove(C.byref(bad), C.byref(tr._avg_s), C.sizeof(bad))
    bad.b_hh[0] = bad.b_ih[0]
    assert lib.zrb_set_average(tr.ctx, C.byref(bad)) == -1
    # an average tensor that is not 4-byte aligned (in a buffer of its own, so it overlaps nothing); never left installed
    spare = torch.zeros(tr.flat_avg.numel() + 1, device=_dev())
    odd = _lib.ZrbParams()
    C.memmove(C.byref(odd), C.byref(tr._avg_s), C.sizeof(odd))
    odd.w_hh[0] = spare.data_ptr() + 2
    try:
        assert lib.zrb_set_average(tr.ctx, C.byref(odd)) == -1
    finally:
        lib.zrb_set_average(tr.ctx, None)
    tr.close()
    del tr, m
    gc.collect()


def test_clip_sgd_and_dyneval_do_not_advance_n(monkeypatch):
    row = FEATURE_ROW[0] if FEATURE_ROW else ROW_IDS[0]
    r = _row(row)
    m, tr = _trainer(r, "rows_only", monkeypatch)
    tr.start_averaging()
    _step(tr, r, 0, False)
    a = tr.flat_avg.clone()
    tr.dynamic_perplexity([(r.x[0], r.y[0])], lr=0.1)
    torch.cuda.synchronize()
    assert tr.averaged_steps == 1 and _bits_equal(tr.flat_avg, a)
    tr.close()


# ---- two GPUs -------------------------------------------------------------------------------------------------------
def _dp_worker(rank, world, port, q, transport):
    import os
    import torch.distributed as dist
    import zaremba_b200
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank), ZRB_DP_TRANSPORT=transport)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    V, H, T, B, STEPS = 1000, 256, 12, 8, 4
    g = torch.Generator().manual_seed(3)
    data = torch.randint(0, V, (B * world, STEPS * T + 1), generator=g)
    torch.manual_seed(7)
    m = zaremba_b200.Model(V, H, L, 0.0, 0.1).to(dev)
    m.train()
    tr = zaremba_b200.Trainer(m, B, T)
    rows = slice(rank * B, (rank + 1) * B)
    av = AO.Averager()
    ok = True
    for i in range(STEPS):
        if i == 1:
            tr.start_averaging()
        x = data[rows, i * T:(i + 1) * T].t().contiguous().to(dev)
        y = data[rows, i * T + 1:(i + 1) * T + 1].t().contiguous().to(dev)
        tr.train_step(x, y, 1.0, 0.25)
        tr.flush()
        if i >= 1:
            ok = ok and tr.flat_avg.cpu().numpy().tobytes() == av.update(tr.flat_p.cpu().numpy()).tobytes()
    bits = tr.flat_avg.view(torch.int32).to(torch.int64)
    chk = torch.stack([bits.sum(), (bits * (torch.arange(bits.numel(), device=dev) % 8191 + 1)).sum()])
    hi, lo = chk.clone(), chk.clone()
    dist.all_reduce(hi, op=dist.ReduceOp.MAX)
    dist.all_reduce(lo, op=dist.ReduceOp.MIN)
    res = {"identical": bool((hi == lo).all().item()), "oracle": ok}
    dist.barrier()
    tr.close()
    dist.destroy_process_group()
    q.put((rank, res))


@pytest.mark.parametrize("transport", ["ce", "nccl"])
def test_dp_average_is_identical_on_every_rank(transport):
    from tests.test_gpu_multi import _need_two, _spawn
    _need_two()
    out = _spawn(_dp_worker, 2, transport)
    for r in (0, 1):
        assert out[r]["identical"], "averages diverged across ranks"
        assert out[r]["oracle"], f"rank {r}: the average is not the restatement over its weights"
