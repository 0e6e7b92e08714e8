"""GPU tests of the beam search (zrb_beam_step, zrb_beam_search, Model.beam_search).

  * the step kernels against the float64 restatement of oracle/beam.py over V, K and B, on rows with exact ties,
    identical rows with equal S, finished rows and a wide range of S;
  * the search's wiring, bit for bit: it equals an explicit loop of T = 1 `Model.forward` calls on states reordered in
    torch by the parents, followed by `zaremba_b200.beam_step`, on both recurrence paths;
  * K = 1 against greedy `generate`; an exhaustive search against all V^2 continuations scored by the fp64 oracle;
  * logprobs against the fp64 oracle's teacher-forced ones (chunked prefill), scores as float32 sums;
  * the interplay with a lazy-update Trainer and the context, the launch count per token.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import beam as BM
from oracle import lstm_lm_oracle as O
from tests.test_gpu_parity import ENGINES, TOL

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
SHAPES = {"small": 200, "medium": 650, "large": 1500}    # BASELINE shapes: V = 10000, L = 2
V_PTB, L = 10000, 2


def _bits(t):
    return t.detach().contiguous().view(torch.int32).cpu().numpy() if t.dtype == torch.float32 else t.cpu().numpy()


def _rows(V, R, rng):
    """Score rows with exact ties and a wide dynamic range (row scale 0.01 .. 50, offsets up to +-100)."""
    z = np.empty((R, V), dtype=np.float32)
    for r in range(R):
        scale = [0.01, 0.3, 1.0, 4.0, 50.0][r % 5]
        row = rng.normal(size=V) * scale + [0.0, 100.0, -100.0][r % 3]
        if r % 4 == 1:
            row = np.round(row * 4) / 4                        # many exact ties
        if r % 4 == 2 and V > 3:
            row[rng.choice(V, 3, replace=False)] = row.max()   # a tied maximum
        z[r] = row
    return z


def _step_dev(lib, _lib, buf, ld, B, K_in, K, V, cum, last, eos, pad=5):
    """zrb_beam_step with outputs padded by `pad` sentinel entries, which must survive."""
    n = B * K
    outs = [torch.full((n + pad,), -7, dtype=torch.int64, device=DEV), torch.full((n + pad,), -7, dtype=torch.int32, device=DEV),
            torch.full((n + pad,), 1234.5, device=DEV), torch.full((n + pad,), 1234.5, device=DEV)]
    _lib.check(lib.zrb_beam_step(_lib.ptr(buf), ld, B, K_in, K, V, _lib.ptr(cum), _lib.ptr(last), eos,
                                 *[_lib.ptr(o) for o in outs], None))
    res = [o.cpu().numpy() for o in outs]
    for o, fill in zip(res, (-7, -7, 1234.5, 1234.5)):
        assert (o[n:] == fill).all(), "wrote past the outputs"
    return [o[:n] for o in res]


@pytest.mark.parametrize("V", [33, 10000, 10001, 50000])
def test_beam_step_against_oracle(V):
    from zaremba_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(V)
    near = picks = 0
    worst = 0.0
    for K in [k for k in (1, 2, 5, 8, 32) if k <= V]:
        for B in (1, 3):
            for form in ("first", "next", "finished", "identical"):
                K_in = 1 if form == "first" else K
                R = B * K_in
                z = _rows(V, R, rng)
                cum = last = None
                eos = -1
                if form != "first":
                    cum = (rng.normal(size=R) * [1.0, 30.0, 300.0][K % 3]).astype(np.float32)   # S over a wide range
                if form == "finished":
                    eos = int(rng.integers(V))
                    last = rng.integers(0, V, size=R)
                    last[::2] = eos                            # every other row finished
                if form == "identical":                         # identical rows of a prompt with equal S
                    for b in range(B):
                        z[b * K:(b + 1) * K] = z[b * K]
                        cum[b * K:(b + 1) * K] = cum[b * K]
                ld = V + 3 if B == 3 else V
                buf = torch.full((R, ld), float("nan"), device=DEV)
                buf[:, :V] = torch.from_numpy(z)
                cum_d = None if cum is None else torch.from_numpy(cum).to(DEV)
                last_d = None if last is None else torch.from_numpy(last).to(DEV)
                got = _step_dev(lib, _lib, buf, ld, B, K_in, K, V, cum_d, last_d, eos)
                again = _step_dev(lib, _lib, buf, ld, B, K_in, K, V, cum_d, last_d, eos)
                tag = f"V={V} K={K} B={B} {form}"
                for a, b in zip(got, again):
                    assert np.array_equal(a.view(np.int32) if a.dtype == np.float32 else a,
                                          b.view(np.int32) if b.dtype == np.float32 else b), f"{tag}: two runs differ"
                tok, par, S, lp = got
                wtok, wpar, wS, wlp, _ = BM.step(z, K, None if cum is None else cum.astype(np.float64), last, eos)
                lsm = BM.log_softmax(z)
                for b in range(B):
                    for k in range(K):
                        r = b * K + k
                        picks += 1
                        i = b * K_in + int(par[r])
                        finished = last is not None and eos >= 0 and last[i] == eos
                        assert 0 <= par[r] < K_in and 0 <= tok[r] < V
                        want_lp = 0.0 if finished else lsm[i, tok[r]]
                        assert not finished or tok[r] == eos
                        want_S = (0.0 if cum is None else float(cum[i])) + want_lp
                        if (tok[r], par[r]) != (wtok[r], wpar[r]):
                            # only where the two candidates lie within float32 rounding of each other
                            assert abs(want_S - wS[r]) <= 1e-5 * max(1.0, abs(wS[r])), \
                                f"{tag} slot {r}: ({par[r]},{tok[r]}) != ({wpar[r]},{wtok[r]}): {want_S} vs {wS[r]}"
                            near += 1
                        for g, w in ((lp[r], want_lp), (S[r], want_S)):
                            err = abs(float(g) - w) / max(1.0, abs(w))
                            worst = max(worst, err)
                            assert err <= 1e-5, f"{tag} slot {r}: {g} vs {w}"
                    assert np.all(np.diff(S[b * K:(b + 1) * K]) <= 0), f"{tag}: S not descending"
                    flat = par[b * K:(b + 1) * K].astype(np.int64) * V + tok[b * K:(b + 1) * K]
                    assert len(set(flat.tolist())) == K, f"{tag}: a candidate chosen twice"
    # S up to +-300 (float32 spacing 3e-5) on rows of scale 0.01 with up to 50 000 entries puts neighbouring candidates
    # within one rounding of each other: about 1 % of the picks swap there (each such pick is checked above)
    assert near <= max(4, picks // 40), f"{near} of {picks} picks differ from the oracle within float32 rounding"
    print(f"V={V}: {picks} picks, {near} near-tie differences, worst relative error {worst:.2e}")


def test_beam_step_rejects_bad_arguments():
    from zaremba_b200 import _lib
    lib = _lib.load()
    z = torch.zeros(64, 40, device=DEV)
    o64 = torch.zeros(64 * 33, dtype=torch.int64, device=DEV)
    o32 = torch.zeros(64 * 33, dtype=torch.int32, device=DEV)
    f = torch.zeros(64 * 33, device=DEV)
    last = torch.zeros(64, dtype=torch.int64, device=DEV)

    def call(B=2, K_in=1, K=4, V=40, ld=40, eos=-1, tok_in=None):
        return lib.zrb_beam_step(_lib.ptr(z), ld, B, K_in, K, V, None, _lib.ptr(tok_in), eos, _lib.ptr(o64),
                                 _lib.ptr(o32), _lib.ptr(f), _lib.ptr(f), None)
    assert call() == 0
    torch.cuda.synchronize()
    for kw in (dict(K=0), dict(K=33), dict(V=3, ld=40), dict(eos=-2), dict(eos=40), dict(B=0), dict(ld=39),
               dict(K_in=2), dict(tok_in=last)):
        assert call(**kw) == -1, kw
    m = _model(64, "tc", V=40)
    with pytest.raises(ValueError, match="beams"):
        m.beam_search(torch.zeros(1, 1, dtype=torch.int64), 2, 33)
    m._context(1, 8)
    with pytest.raises(ValueError, match="max_batch 8"):
        m.beam_search(torch.zeros(1, 3, dtype=torch.int64), 2, 3)
    from zaremba_b200 import _lib as Lb
    ps, keep = m._params_struct(m._lib_weights())
    st = m.state_init(8)
    sin, k1 = m._states_struct(st)
    x = torch.zeros(1, 2, dtype=torch.int64, device=DEV)
    tok = torch.zeros(64, dtype=torch.int64, device=DEV)
    for T0, B, n_new, K, eos in ((0, 2, 2, 2, -1), (1, 2, 0, 2, -1), (1, 2, 2, 5, -1), (1, 2, 2, 2, 40),
                                 (1, 2, 2, 0, -1)):
        assert lib.zrb_beam_search(m._ctx, C.byref(ps), Lb.ptr(x), T0, B, C.byref(sin), C.byref(sin), n_new, K, eos,
                                   Lb.ptr(tok), None, None, None) == -1, (T0, B, n_new, K, eos)


def _model(H, engine, V=V_PTB, seed=11, lstm_type="pytorch"):
    import zaremba_b200
    torch.manual_seed(seed)
    return zaremba_b200.Model(V, H, L, 0.5, 0.1 if H < 1000 else 0.05, lstm_type, engine=engine).to(DEV)


def _prompt(T0, B, V=V_PTB, seed=3):
    return torch.randint(0, V, (T0, B), generator=torch.Generator().manual_seed(seed))


def _replay(m, prompt, n_new, K, eos):
    """The search spelled out: Model.forward at T = 1, beam_step, states reordered in torch, then the backtrack."""
    import zaremba_b200
    T0, B = prompt.shape
    m.eval()
    states = m.state_init(B)
    with torch.no_grad():
        scores, states = m(prompt.to(DEV), states)
        scores = scores.view(T0, B, -1)[-1]
        cum = last = None
        steps = []
        for k in range(n_new):
            K_in = 1 if cum is None else K
            tok, par, cum, lp = zaremba_b200.beam_step(scores, K, cum, last, eos)
            src = (torch.arange(B, device=DEV).repeat_interleave(K) * K_in + par.long())
            states = [(h.index_select(1, src), c.index_select(1, src)) for h, c in states]
            steps.append((tok, par, lp))
            if k + 1 < n_new:
                scores, states = m(tok.view(1, B * K), states)
                last = tok
    tokens = torch.empty(n_new, B * K, dtype=torch.int64, device=DEV)
    logprobs = torch.empty(n_new, B * K, device=DEV)
    slot = torch.arange(B * K, device=DEV)
    base = slot - slot % K
    slot = slot % K
    for k in range(n_new - 1, -1, -1):
        tok, par, lp = steps[k]
        tokens[k], logprobs[k] = tok[base + slot], lp[base + slot]
        slot = par[base + slot].long()
    return tokens.view(n_new, B, K), logprobs.view(n_new, B, K), cum.view(B, K), states


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("BK", [(2, 4), (1, 32), (5, 8)], ids=["bk8", "bk32", "bk40"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_beam_search_equals_forward_and_beam_step_replay(shape, BK, engine):
    B, K = BK
    n_new = 20
    m = _model(SHAPES[shape], engine)
    m._context(1, B * K)                                       # both runs use the plans of a B*K-row context
    prompt = _prompt(1, B)
    m.eval()
    with torch.no_grad():
        first, _ = m(prompt.to(DEV), m.state_init(B))
    for eos in (-1, int(first[0].argmax())):                   # with eos: prompt 0's best first token finishes at once
        m.train()                                              # beam_search ignores .training
        tokens, logprobs, scores, st = m.beam_search(prompt, n_new, K, eos=None if eos < 0 else eos)
        rt, rl, rs, rst = _replay(m, prompt, n_new, K, eos)
        tag = f"{shape} B={B} K={K} eos={eos}"
        assert np.array_equal(_bits(tokens), _bits(rt)), f"{tag}: tokens differ"
        assert np.array_equal(_bits(logprobs), _bits(rl)), f"{tag}: logprobs differ"
        assert np.array_equal(_bits(scores), _bits(rs)), f"{tag}: scores differ"
        for (h, c), (h2, c2) in zip(st, rst):
            assert h.shape == (1, B * K, m.hidden_size)
            assert np.array_equal(_bits(h), _bits(h2)) and np.array_equal(_bits(c), _bits(c2)), f"{tag}: states differ"
        if eos >= 0:
            t = tokens.cpu().numpy()
            assert t[0, 0, 0] == eos and (t[:, 0, 0] == eos).all(), f"{tag}: the finished beam must stay eos"
            assert (logprobs[1:, 0, 0] == 0).all()
            hit = t == eos
            after = np.cumsum(hit, 0) > 0
            assert (t[after] == eos).all() and (logprobs.cpu().numpy()[1:][after[:-1]] == 0).all()


@pytest.mark.parametrize("engine", ENGINES)
def test_k1_equals_greedy_generate(engine):
    B, n_new = 20, 40
    m = _model(650, engine).eval()
    prompt = _prompt(3, B)
    gt, gl, _ = m.generate(prompt, n_new, temperature=0.0, seed=0)
    bt, bl, bs, _ = m.beam_search(prompt, n_new, 1)
    gt, gl, bt, bl = gt.cpu().numpy(), gl.cpu().numpy(), bt[:, :, 0].cpu().numpy(), bl[:, :, 0].cpu().numpy()
    diverged = 0
    for b in range(B):
        d = np.nonzero(gt[:, b] != bt[:, b])[0]
        k = d[0] if d.size else n_new
        assert np.array_equal(gl[:k, b].view(np.int32), bl[:k, b].view(np.int32)), f"row {b}: logprobs differ"
        if k < n_new:
            # a rounding tie: replay the greedy prefix and check that the two tokens' candidates meet in float32
            diverged += 1
            x = torch.cat([prompt[:, b:b + 1], torch.from_numpy(gt[:k, b:b + 1])]).to(DEV)
            with torch.no_grad():
                z = m(x, m.state_init(1))[0][-1].double().cpu().numpy()
            S = float(np.sum(bl[:k, b].astype(np.float32), dtype=np.float32))
            gap = z[gt[k, b]] - z[bt[k, b]]
            lse = np.log(np.exp(z - z.max()).sum())
            mag = abs(S) + abs(z[bt[k, b]] - z.max()) + lse
            assert 0 <= gap <= 2 * np.spacing(np.float32(max(mag, 1.0))), \
                f"row {b} step {k}: tokens {gt[k, b]} / {bt[k, b]} differ by {gap} in score"
    assert diverged <= 2, f"{diverged} rows left greedy decoding"
    assert np.array_equal(_bits(bs[:, 0]), _bits(torch.from_numpy(np.cumsum(bl, 0, dtype=np.float32)[-1])))


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("B", [1, 2], ids=["persistent", "per_timestep"])
def test_exhaustive_on_device(engine, B):
    V, H, K, n_new = 32, 64, 32, 2
    m = _model(H, engine, V=V, seed=5)
    with torch.no_grad():
        m.fc.W.mul_(8.0)                                       # a peaked distribution: the ranking means something
    m._context(2, B * K)
    if engine == "tc":
        from zaremba_b200 import _lib
        assert bool(_lib.rec_plans(m._ctx)["fwd"]["ok"]) == (B == 1), "B = 1: persistent, B = 2: per-timestep path"
    prompt = _prompt(2, B, V=V)
    tokens, logprobs, scores, _ = m.beam_search(prompt, n_new, K)
    params = {k: v.detach().double().cpu().numpy() for k, v in m.named_parameters()}
    tol = 0.0
    for b in range(B):
        seqs = np.array([(i, j) for i in range(V) for j in range(V)])
        x = np.concatenate([np.repeat(prompt[:, b:b + 1].numpy(), V * V, 1), seqs[:, :1].T])
        sc, _, _ = O.model_fwd(params, x, O.zero_states(L, V * V, H, np.float64), L)
        sc = sc.reshape(3, V * V, V)
        lp = BM.log_softmax(sc[1])[np.arange(V * V), seqs[:, 0]] + BM.log_softmax(sc[2])[np.arange(V * V), seqs[:, 1]]
        tol = 2 * n_new * 2 * TOL[engine]["fwd"] * np.abs(sc).max()
        order = np.argsort(-lp, kind="stable")
        want = lp[order[:K]]
        got = tokens[:, b, :].cpu().numpy().T
        got_lp = lp[got[:, 0] * V + got[:, 1]]
        assert len({tuple(g) for g in got}) == K, "hypotheses must be distinct"
        # the k-th returned hypothesis scores like the k-th best of all 1024, up to swaps within the engine's tolerance
        assert np.all(np.abs(got_lp - want) <= tol), (np.abs(got_lp - want).max(), tol)
        assert np.all(got_lp >= want[-1] - tol)
    print(f"{engine} B={B}: tolerance {tol:.2e}")


def _oracle_logprobs(m, prompt, tokens):
    """Teacher-forced fp64 log-probabilities of tokens[k] after prompt + tokens[:k], columns b*K + k."""
    n_new, B, K = tokens.shape
    params = {k: v.detach().double().cpu().numpy() for k, v in m.named_parameters()}
    tk = tokens.reshape(n_new, B * K).cpu().numpy()
    x = np.concatenate([np.repeat(prompt.numpy(), K, 1), tk[:-1]])
    T = x.shape[0]
    scores, _, _ = O.model_fwd(params, x, O.zero_states(L, B * K, m.hidden_size, np.float64), L)
    sc = scores.reshape(T, B * K, -1)[prompt.shape[0] - 1:]
    want = np.take_along_axis(BM.log_softmax(sc), tk[..., None], -1)[..., 0]
    return want.reshape(n_new, B, K), np.abs(sc).max()


@pytest.mark.parametrize("engine", ENGINES)
def test_beam_logprobs_against_oracle_chunked(engine):
    B, K, T0, n_new = 4, 5, 35, 12
    m = _model(650, engine)
    m._context(8, B * K)                                       # max_seq 8 < T0: prefill in five windows
    prompt = _prompt(T0, B)
    tokens, logprobs, scores, _ = m.beam_search(prompt, n_new, K)
    assert m._ctx_key[:2] == (8, B * K), "beam_search must keep the existing context"
    want, scale = _oracle_logprobs(m, prompt, tokens)
    lp = logprobs.cpu().numpy()
    err = np.abs(lp - want).max()
    tol = 2 * TOL[engine]["fwd"] * scale
    assert err <= tol, f"{engine}: logprob error {err:.3e} > {tol:.3e}"
    sums = np.zeros((B, K), dtype=np.float32)
    for k in range(n_new):
        sums = (sums + lp[k]).astype(np.float32)
    assert np.array_equal(sums.view(np.int32), _bits(scores)), "scores must be the float32 sums of the logprobs"
    s = scores.cpu().numpy()
    assert np.all(np.diff(s, axis=1) <= 0), "scores must not increase across k"
    t = tokens.cpu().numpy()
    for b in range(B):
        assert len({tuple(t[:, b, k]) for k in range(K)}) == K, "hypotheses must be distinct"
    print(f"{engine}: logprob error {err:.2e} (scale {scale:.2f})")


def test_beam_search_after_lazy_trainer_step():
    import zaremba_b200
    B, T, K = 20, 35, 4
    m = _model(650, "tc")
    m.train()
    tr = zaremba_b200.Trainer(m, B, T, lazy_update=True)
    g = torch.Generator().manual_seed(4)
    x = torch.randint(0, V_PTB, (T, B), generator=g).to(DEV)
    y = torch.randint(0, V_PTB, (T, B), generator=g).to(DEV)
    tr.train_step(x, y, 1.0, 5.0)
    step, drop = tr.step, m._drop_step
    prompt = _prompt(3, B // K)
    a = m.beam_search(prompt, 8, K, eos=7)                     # weight updates still pending in the context
    tr.flush()
    b = m.beam_search(prompt, 8, K, eos=7)
    for u, v in zip(a[:3], b[:3]):
        assert np.array_equal(_bits(u), _bits(v))
    for (h, c), (h2, c2) in zip(a[3], b[3]):
        assert np.array_equal(_bits(h), _bits(h2)) and np.array_equal(_bits(c), _bits(c2))
    assert tr.step == step and m._drop_step == drop, "beam_search must not advance the dropout step"
    ctx = m._ctx.value
    with pytest.raises(ValueError, match="max_batch 20"):
        m.beam_search(_prompt(1, B // K + 1), 2, K)
    assert m._ctx.value == ctx, "the context must not be replaced"
    tr.train_step(x, y, 1.0, 5.0)                              # the Trainer still works on the same context


def test_launch_count_per_beam_token():
    """Persistent path: per token the unchanged forward (state prep, embedding, one input GEMM and one recurrence per
    layer, projection: 2L + 3) and the two beam kernels: 2L + 5."""
    from zaremba_b200 import _lib
    lib = _lib.load()
    m = _model(650, "tc")
    m._context(1, 20)
    prompt = _prompt(1, 4)
    m.beam_search(prompt, 3, 5)                                # packs the weight images, allocates the scratch
    assert _lib.rec_plans(m._ctx)["fwd"]["ok"], "B*K = 20 should run the persistent recurrence"
    counts = []
    for n in (5, 25):
        torch.cuda.synchronize()
        c0 = lib.zrb_launch_count()
        m.beam_search(prompt, n, 5)
        counts.append(lib.zrb_launch_count() - c0)
    per_token = (counts[1] - counts[0]) / 20
    assert per_token == 2 * L + 5, (counts, per_token)
