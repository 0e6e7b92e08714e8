"""GPU tests of the in-kernel dropout masks against the independent Philox4x32-10 of oracle/philox.py.

Keep flags are never stored: every kernel that applies a dropout site regenerates them from (seed, step, site,
element).  Three kinds of check, all against masks computed in numpy from the written definition (DESIGN.md
section 3), never against masks the library reports about itself:
  * zrb_dropout_mask equals the reference bit for bit over ragged n, sites, both words of the step, seeds and p;
  * a fused `Trainer` and the drop-in `Model` running their own Philox masks give exactly the bits of the same runs
    fed the reference masks through set_explicit_dropout_masks, at two steps and at shapes that reach every kernel
    and recurrence-plan branch that applies a mask (a wrong generator, a stale step or a mask-index slip in one
    branch changes some bits);
  * step 0 of each shape against the fp64 oracle with the reference masks (an index slip reads the same wrong
    element from both mask sources, so only the oracle sees it), and the rows-out embedding gradient on one GPU.
Bit equality needs deterministic runs: every window holds distinct tokens, so the embedding scatter adds one
atomic per element.
"""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

from oracle import lstm_lm_oracle as O
from oracle import philox as PH
from tests.test_gpu_parity import ENGINES, TOL, _caller_nll_loss, _plan_branch, _record, _scale_close

pytestmark = pytest.mark.gpu

P_DROP, L = 0.65, 2


def _dev():
    return torch.device("cuda:0")


@pytest.mark.parametrize("seed", ["zero", "high", "initial"])
def test_dropout_mask_equals_reference(seed):
    """zrb_dropout_mask against oracle.philox.keep_mask, bit for bit: n in {1, 2, 3, 5, 1023, 3 * 2^20 + 3} (partial
    last group), sites 0, 1, 2, 7, steps 0, 1, 2^32 - 1, 2^32, 2^32 + 5 (the step's high word is part of the key),
    p in {0, 0.5, float32(0.65), 1e-7, 0.999}.  Nothing past element n - 1 is written."""
    from zaremba_b200 import _lib
    lib = _lib.load()
    seed = {"zero": 0, "high": 2 ** 63 + 12345, "initial": int(torch.initial_seed())}[seed]
    ns = [1, 2, 3, 5, 1023, 3 * 2 ** 20 + 3]
    pad = 13
    buf = torch.empty(ns[-1] + pad, dtype=torch.uint8, device=_dev())
    for site in (0, 1, 2, 7):
        for step in (0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 5):
            r = PH.draws(seed, step, site, ns[-1])
            for p in (0.0, 0.5, float(np.float32(0.65)), 1e-7, 0.999):
                want = PH.keep_mask(seed, step, site, ns[-1], p) if p == 0 else r >= np.uint32(PH.threshold(p))
                for n in ns:
                    buf.fill_(0xA5)
                    _lib.check(lib.zrb_dropout_mask(seed, step, site, n, p, _lib.ptr(buf[:n]), None))
                    got = buf[:n + pad].cpu().numpy()
                    tag = f"seed={seed} step={step} site={site} p={p} n={n}"
                    assert (got[n:] == 0xA5).all(), f"{tag}: wrote past the end"
                    if not np.array_equal(got[:n], want[:n]):
                        bad = np.flatnonzero(got[:n] != want[:n])
                        raise AssertionError(f"{tag}: {bad.size} flags differ, first at element {bad[0]}")


# name -> (engine, H, T, B, branch).  The tc rows are the recurrence-plan branch shapes of test_gpu_parity's
# LAYER_CASES (two layers here, so the forward epilogue applies masks of site 1 and 2 and the backward epilogue reads
# them), the per-timestep path at B > 32 and a small shape; the simt rows run the validation engine's cell kernels.
# H % 4 == 0 (1500, 300, 40, 64, 48) takes the embedding's quad path, H % 4 != 0 (650, 257, 255) the per-element one.
ROWS = {
    "one_tile_n32": ("tc", 650, 35, 32, "one_tile_n32"),
    "two_cells_n32": ("tc", 1500, 35, 32, "two_cells_n32"),
    "b8_padded": ("tc", 300, 6, 8, "b8_padded"),
    "odd_h": ("tc", 257, 5, 9, "odd_h"),
    "nosplit_n32": ("tc", 255, 4, 32, "nosplit_n32"),
    "b1_split": ("tc", 1500, 2, 1, "b1_split"),
    "t1": ("tc", 40, 1, 1, "t1"),
    "steps_b40": ("tc", 64, 4, 40, "steps"),
    "tc_h48": ("tc", 48, 6, 5, None),
    "simt_h48": ("simt", 48, 6, 5, None),
    "simt_h257": ("simt", 257, 5, 9, None),
}
ROW_IDS = [r for r in ROWS if ROWS[r][0] in ENGINES]


class Row:
    """Shape, weights (seeded torch init), two windows of distinct tokens and the incoming states of one row."""

    def __init__(self, name):
        self.name = name
        self.engine, self.H, self.T, self.B, self.branch = ROWS[name]
        self.V = max(97, self.T * self.B + 13)          # V >= T * B: each window can hold distinct tokens
        self.winit = 0.04 if self.H >= 1000 else 0.1
        self.torch_seed = 1000 + list(ROWS).index(name)
        g = torch.Generator().manual_seed(self.torch_seed)
        N = self.T * self.B
        self.x = [torch.randperm(self.V, generator=g)[:N].view(self.T, self.B) for _ in range(2)]
        self.y = [torch.randint(0, self.V, (self.T, self.B), generator=g) for _ in range(2)]
        self.h0 = [(torch.rand(self.B, self.H, generator=g) - 0.5, torch.rand(self.B, self.H, generator=g) * 2 - 1)
                   for _ in range(L)]

    def model(self):
        import zaremba_b200
        torch.manual_seed(self.torch_seed)               # same weights every call; Philox seed = torch.initial_seed()
        m = zaremba_b200.Model(self.V, self.H, L, P_DROP, self.winit, engine=self.engine).to(_dev())
        m.train()
        return m

    def states(self):
        return [(h.view(1, self.B, self.H).to(_dev()), c.view(1, self.B, self.H).to(_dev())) for h, c in self.h0]

    def masks(self, seed, step):
        return PH.site_masks(seed, step, L, self.T, self.B, self.H, P_DROP)

    def check_branch(self, ctx):
        """Skip when this device's SM count leads the row's shape to another plan branch."""
        from zaremba_b200 import _lib
        if self.engine != "tc" or self.branch is None:
            return
        plans = _lib.rec_plans(ctx)
        fp, bp = plans["fwd"], plans["bwd"]
        if self.branch == "steps":
            assert not fp["ok"] and not bp["ok"], f"B={self.B} should take the per-timestep path: {plans}"
            return
        if not (fp["ok"] and bp["ok"]) or not _plan_branch(self.branch, self.H, self.B, fp, bp):
            pytest.skip(f"on {torch.cuda.get_device_properties(0).multi_processor_count} SMs H={self.H} B={self.B} "
                        f"gets {plans}, not the {self.branch} branch")
        print(f"\n{self.name}: fwd {fp} bwd {bp}")

    _oracle_cache = {}

    def oracle_step0(self, seed):
        """fp64 oracle of step 0 (window 0, the row's weights and states, the reference masks of step 0)."""
        key = (self.name, seed)
        if key not in self._oracle_cache:
            m = self.model()
            params = {k: v.detach().cpu().numpy().astype(np.float64) for k, v in m.named_parameters()}
            del m
            masks = self.masks(seed, 0)
            st0 = [(h.numpy().astype(np.float64), c.numpy().astype(np.float64)) for h, c in self.h0]
            x, y = self.x[0].numpy(), self.y[0].numpy()
            sc, st, cache = O.model_fwd(params, x, st0, L, P_DROP, masks)
            grads = O.model_bwd(params, cache, O.nll_loss_bwd(sc, y), L)
            self._oracle_cache.clear()
            self._oracle_cache[key] = dict(scores=sc, states=st, loss=O.nll_loss(sc, y), grads=grads)
        return self._oracle_cache[key]


def _first_diff(pairs):
    return [name for name, a, b in pairs if not torch.equal(a, b)]


def _trainer_run(row, explicit, lazy=False, host=False):
    """Two fused train steps; returns per step (loss, norm, states, flat_g, flat_p) and the Trainer's seed."""
    import zaremba_b200
    m = row.model()
    tr = zaremba_b200.Trainer(m, row.B, row.T, lazy_update=lazy)
    for (h, c), (h0, c0) in zip(tr.states, row.states()):
        h.copy_(h0)
        c.copy_(c0)
    row.check_branch(tr.ctx)
    out = []
    for s in range(2):
        if explicit:
            m.set_explicit_dropout_masks([torch.tensor(mk).to(_dev()) for mk in row.masks(tr.seed, s)])
        if host:
            loss, norm = tr.train_step_host(row.x[s], row.y[s], 1.0, 0.25)
            loss, norm = torch.tensor(loss), torch.tensor(norm)
        else:
            loss, norm = tr.train_step(row.x[s].to(_dev()), row.y[s].to(_dev()), 1.0, 0.25)
        tr.flush()
        torch.cuda.synchronize()
        out.append(dict(loss=loss.clone(), norm=norm.clone(), states=[t.clone() for st in tr.states for t in st],
                        flat_g=tr.flat_g.clone(), flat_p=tr.flat_p.clone()))
    assert tr.step == 2
    seed = tr.seed
    tr.close()
    del tr, m
    gc.collect()
    return out, seed


def _compare_steps(philox, explicit, sizes=None):
    names = ["embed"] + [f"{k}{l}" for l in range(L) for k in ("w_ih", "w_hh", "b_ih", "b_hh")] + ["fc_w", "fc_b"]
    for s, (a, b) in enumerate(zip(philox, explicit)):
        pairs = [(k, a[k], b[k]) for k in a if k not in ("states", "grads")]
        pairs += [(f"state{i}", u, v) for i, (u, v) in enumerate(zip(a["states"], b["states"]))]
        if "grads" in a:
            pairs += [(f"grad {k}", a["grads"][k], b["grads"][k]) for k in a["grads"]]
        for big in ("flat_g", "flat_p"):
            if big in a and sizes is not None and not torch.equal(a[big], b[big]):
                pairs += [(f"{big} {n}", u, v) for n, u, v in zip(names, a[big].split(sizes), b[big].split(sizes))]
        bad = _first_diff(pairs)
        assert not bad, f"step {s}: Philox and explicit reference masks differ in {bad}"


@pytest.mark.parametrize("row", ROW_IDS)
def test_trainer_philox_equals_reference_masks(row):
    """Fused Trainer, two steps: its own Philox masks against a fresh Trainer (same weights and states) fed
    oracle.philox masks of steps 0 and 1 -- loss, clip norm, states, flat_g and flat_p bit for bit.  Step 0 also
    against the fp64 oracle with those masks (loss, states, every gradient) within the engine's tolerance."""
    r = Row(row)
    got, seed = _trainer_run(r, explicit=False)
    want, seed2 = _trainer_run(r, explicit=True)
    assert seed == seed2 == int(torch.initial_seed()) & 0xFFFFFFFFFFFFFFFF
    sizes = [int(np.prod(O.param_shapes(r.V, r.H, L)[k])) for k in O.param_names(L)]
    _compare_steps(got, want, sizes)
    ref = r.oracle_step0(seed)
    tol = TOL[r.engine]
    g0 = got[0]
    assert abs(g0["loss"].item() - ref["loss"]) <= tol["loss"] * abs(ref["loss"]), (g0["loss"].item(), ref["loss"])
    _record("loss", abs(g0["loss"].item() - ref["loss"]) / abs(ref["loss"]))
    for l in range(L):
        _scale_close(g0["states"][2 * l].reshape(r.B, r.H).cpu().numpy(), ref["states"][l][0], tol["fwd"], f"{row} h{l}")
        _scale_close(g0["states"][2 * l + 1].reshape(r.B, r.H).cpu().numpy(), ref["states"][l][1], tol["fwd"], f"{row} c{l}")
    for k, g in zip(O.param_names(L), g0["flat_g"].split(sizes)):
        _scale_close(g.cpu().numpy().reshape(ref["grads"][k].shape), ref["grads"][k], tol["grad"], f"{row} grad {k}")


def _dropin_run(row, explicit):
    """Drop-in Model: train forward + backward (step 0), an eval forward, train forward + backward (step 1)."""
    m = row.model()
    row.check_branch(m._context(row.T, row.B))
    out = []
    for s in range(2):
        if explicit:
            m.set_explicit_dropout_masks([torch.tensor(mk).to(_dev()) for mk in row.masks(int(torch.initial_seed()), s)])
        m.zero_grad(set_to_none=True)
        states = row.states()
        scores, states = m(row.x[s], states)
        _caller_nll_loss(scores, row.y[s]).backward()
        out.append(dict(scores=scores.detach().clone(), states=[t.clone() for st in states for t in st],
                        grads={k: p.grad.clone() for k, p in m.named_parameters()}))
        if s == 0 and not explicit:
            m.eval()
            with torch.no_grad():
                m(row.x[1], row.states())                # must not consume a dropout step
            m.train()
    seed, steps = m._seed, m._drop_step
    del m
    gc.collect()
    return out, seed, steps


@pytest.mark.parametrize("row", ROW_IDS)
def test_dropin_philox_equals_reference_masks(row):
    """The drop-in Model (train step, eval forward, train step) against the explicit replay of oracle.philox masks
    of steps 0 and 1, bit for bit (scores, states, every gradient): the eval pass between must not consume a step.
    Step 0 also against the fp64 oracle (scores, states, every gradient)."""
    r = Row(row)
    got, seed, steps = _dropin_run(r, explicit=False)
    assert seed == int(torch.initial_seed()) & 0xFFFFFFFFFFFFFFFF and steps == 2
    want, _, _ = _dropin_run(r, explicit=True)
    _compare_steps(got, want)
    ref = r.oracle_step0(seed)
    tol = TOL[r.engine]
    g0 = got[0]
    _scale_close(g0["scores"].cpu().numpy(), ref["scores"], tol["fwd"], f"{row} scores")
    for l in range(L):
        _scale_close(g0["states"][2 * l].reshape(r.B, r.H).cpu().numpy(), ref["states"][l][0], tol["fwd"], f"{row} h{l}")
        _scale_close(g0["states"][2 * l + 1].reshape(r.B, r.H).cpu().numpy(), ref["states"][l][1], tol["fwd"], f"{row} c{l}")
    for k in O.param_names(L):
        _scale_close(g0["grads"][k].cpu().numpy(), ref["grads"][k], tol["grad"], f"{row} grad {k}")


@pytest.mark.parametrize("mode", ["host", "lazy"])
def test_host_and_lazy_steps_philox_equal_reference_masks(mode):
    """train_step_host (tokens from host memory, step number passed through zrb_train_step_host) and the lazy update
    schedule: two Philox steps equal the explicit replay of the reference masks of steps 0 and 1, bit for bit."""
    if "tc" not in ENGINES:
        pytest.skip("tensor-core engine not selected")
    r = Row("odd_h")
    kw = dict(host=True) if mode == "host" else dict(lazy=True)
    got, seed = _trainer_run(r, explicit=False, **kw)
    want, _ = _trainer_run(r, explicit=True, **kw)
    sizes = [int(np.prod(O.param_shapes(r.V, r.H, L)[k])) for k in O.param_names(L)]
    _compare_steps(got, want, sizes)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("H", [48, 257])
def test_embed_rows_out_single_gpu(H, engine):
    """zrb_set_embed_rows_out on one GPU: backward leaves the embedding gradient as N dropout-masked rows (the
    data-parallel form).  Rows are exactly 0 where the reference site-0 mask drops, non-zero where it keeps, every
    element is written, and scattered by token id they equal the fp64 oracle's embedding gradient."""
    import zaremba_b200
    from zaremba_b200 import _lib
    lib = _lib.load()
    V, T, B = 400, 5, 9
    torch.manual_seed(31 + H)
    m = zaremba_b200.Model(V, H, L, P_DROP, 0.1, engine=engine).to(_dev())
    m.train()
    params = {k: v.detach().cpu().numpy().astype(np.float64) for k, v in m.named_parameters()}
    tr = zaremba_b200.Trainer(m, B, T)
    g = torch.Generator().manual_seed(4)
    x = torch.randint(0, V // 4, (T, B), generator=g)      # repeated tokens: the scatter sums rows
    y = torch.randint(0, V, (T, B), generator=g)
    xd, yd = x.to(_dev()), y.to(_dev())
    rows = torch.full((T * B, H), float("nan"), device=_dev())
    _lib.check(lib.zrb_set_embed_rows_out(tr.ctx, _lib.ptr(rows)))
    try:
        _lib.check(lib.zrb_train_step_grads(tr.ctx, C.byref(tr._ps), C.byref(tr._gs), _lib.ptr(xd), _lib.ptr(yd), T, B,
                                            C.byref(tr._st), C.byref(tr._st), tr.seed, tr.step, _lib.ptr(tr.loss),
                                            tr._stream()))
        torch.cuda.synchronize()
    finally:
        _lib.check(lib.zrb_set_embed_rows_out(tr.ctx, None))
    rw = rows.cpu().numpy()
    keep = PH.keep_mask(tr.seed, tr.step, 0, T * B * H, P_DROP).reshape(T * B, H)
    assert np.isfinite(rw).all(), "rows left unwritten"
    assert (rw[~keep] == 0).all(), f"{int((rw[~keep] != 0).sum())} dropped elements carry a gradient"
    assert (rw[keep] != 0).all(), f"{int((rw[keep] == 0).sum())} kept elements carry no gradient"
    dE = np.zeros((V, H))
    np.add.at(dE, x.numpy().reshape(-1), rw.astype(np.float64))
    masks = PH.site_masks(tr.seed, tr.step, L, T, B, H, P_DROP)
    sc, _, cache = O.model_fwd(params, x.numpy(), O.zero_states(L, B, H, np.float64), L, P_DROP, masks)
    grads = O.model_bwd(params, cache, O.nll_loss_bwd(sc, y.numpy()), L)
    _scale_close(dE, grads["embed.W"], TOL[engine]["grad"], f"rows-out embedding grad H={H}")
