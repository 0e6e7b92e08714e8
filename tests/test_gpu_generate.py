"""GPU tests of on-device sampling (zrb_sample) and the decode loop (zrb_generate, Model.generate).

  * the sampler against the float64 restatement of oracle/sampling.py over a grid of V, B, temperature, top-k and
    top-p, on rows with exact ties and a wide dynamic range;
  * the loop's wiring, bit for bit: a generation equals an explicit replay of T = 1 `Model.forward` calls followed by
    `zaremba_b200.sample` at position k (feedback token, carried state and position counter);
  * the generated log-probabilities against the fp64 oracle's teacher-forced ones, also with a prompt longer than the
    context's max_seq (chunked prefill);
  * chaining two calls, the custom layout, the interplay with a lazy-update Trainer, the launch count per token.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import lstm_lm_oracle as O
from oracle import sampling as S
from tests.test_gpu_parity import ENGINES, TOL

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
SEED = 0x0123456789ABCDEF
SHAPES = {"small": 200, "medium": 650, "large": 1500}    # BASELINE shapes: V = 10000, L = 2
V_PTB, L = 10000, 2


def _rows(V, B, rng):
    """Score rows with exact ties and a wide dynamic range (row scale 0.01 .. 50, offsets up to +-100)."""
    z = np.empty((B, V), dtype=np.float32)
    for b in range(B):
        scale = [0.01, 0.3, 1.0, 4.0, 50.0][b % 5]
        row = rng.normal(size=V) * scale + [0.0, 100.0, -100.0][b % 3]
        if b % 4 == 1:
            row = np.round(row * 4) / 4                        # many exact ties
        if b % 4 == 2 and V > 3:
            row[rng.choice(V, 3, replace=False)] = row.max()   # a tied maximum
        z[b] = row
    return z


def _sample_dev(lib, _lib, scores_dev, ld, B, V, cfg, pos, pad):
    tokens = torch.full((B + pad,), -7, dtype=torch.int64, device=DEV)
    logprobs = torch.full((B + pad,), 1234.5, dtype=torch.float32, device=DEV)
    _lib.check(lib.zrb_sample(_lib.ptr(scores_dev), ld, B, V, C.byref(cfg), pos, _lib.ptr(tokens), _lib.ptr(logprobs),
                              None))
    t, lp = tokens.cpu().numpy(), logprobs.cpu().numpy()
    assert (t[B:] == -7).all() and (lp[B:] == 1234.5).all(), "wrote past row B - 1"
    return t[:B], lp[:B]


@pytest.mark.parametrize("V", [1, 33, 10000, 10001, 50000])
def test_sampler_against_oracle(V):
    from zaremba_b200 import _lib
    from zaremba_b200.sampling import sampling_config
    lib = _lib.load()
    rng = np.random.default_rng(V)
    pos = 2 ** 32 + 7                                          # the position's high word is part of the key
    near, drawn, worst_lp = 0, 0, 0.0
    for B in (1, 20, 40):
        z = _rows(V, B, rng)
        ld = V + 3 if B == 20 else V                           # a row pitch above V
        buf = torch.full((B, ld), float("nan"), device=DEV)
        buf[:, :V] = torch.from_numpy(z)
        u = [S.uniforms(SEED, pos, b, V) for b in range(B)]
        for tau in (0.0, 0.7, 1.0, 1.5):
            for top_k in (0, 1, 40, V):
                for top_p in (1.0, 0.9, 0.3, 1e-6):
                    cfg = sampling_config(tau, top_k, top_p, SEED)
                    tok, lp = _sample_dev(lib, _lib, buf, ld, B, V, cfg, pos, 5)
                    tok2, lp2 = _sample_dev(lib, _lib, buf, ld, B, V, cfg, pos, 5)
                    tag = f"V={V} B={B} tau={tau} top_k={top_k} top_p={top_p}"
                    assert np.array_equal(tok, tok2) and np.array_equal(lp.view(np.uint32), lp2.view(np.uint32)), \
                        f"{tag}: two runs differ"
                    for b in range(B):
                        want, want_lp, info = S.sample_row(z[b], tau, top_k, top_p, SEED, pos, b, u=u[b])
                        if tau == 0.0:
                            assert tok[b] == want, f"{tag} row {b}: greedy {tok[b]} != {want}"
                        else:
                            drawn += 1
                            if tok[b] != want:
                                p32 = float(np.float32(top_p))
                                tie = info["gap"] < 1e-5 * (1 + abs(info["smax"]))
                                edge = any(m is not None and abs(m - p32) < 1e-5 for m in info["boundary"])
                                assert tie or edge, f"{tag} row {b}: token {tok[b]} != {want} ({info})"
                                near += 1
                                want_lp = S.log_softmax_at(z[b], int(tok[b]))
                        err = abs(float(lp[b]) - want_lp)
                        worst_lp = max(worst_lp, err / max(1.0, abs(want_lp)))
                        # float32 spacing at |logprob| ~ 400 is 3e-5: the bound is relative beyond 1
                        assert err <= 1e-5 * max(1.0, abs(want_lp)), f"{tag} row {b}: logprob {lp[b]} vs {want_lp}"
    assert near <= max(2, drawn // 200), f"{near} of {drawn} draws differ from the oracle within the tie margins"
    print(f"V={V}: {drawn} draws, {near} near-tie differences, worst logprob error {worst_lp:.2e}")


def test_sampler_rejects_bad_arguments():
    from zaremba_b200 import _lib
    from zaremba_b200.sampling import sampling_config
    lib = _lib.load()
    z = torch.zeros(2, 5, device=DEV)
    tok = torch.zeros(2, dtype=torch.int64, device=DEV)
    for cfg, B, V, ld in ((sampling_config(-0.1), 2, 5, 5), (sampling_config(top_p=0.0), 2, 5, 5),
                          (sampling_config(top_k=-1), 2, 5, 5), (sampling_config(), 0, 5, 5),
                          (sampling_config(), 2, 0, 5), (sampling_config(), 2, 5, 4)):
        assert lib.zrb_sample(_lib.ptr(z), ld, B, V, C.byref(cfg), 0, _lib.ptr(tok), None, None) == -1


def _model(H, B, engine, lstm_type="pytorch", V=V_PTB, seed=11):
    import zaremba_b200
    torch.manual_seed(seed)
    m = zaremba_b200.Model(V, H, L, 0.5, 0.1 if H < 1000 else 0.05, lstm_type, engine=engine).to(DEV)
    return m


def _prompt(T0, B, V=V_PTB, seed=3):
    return torch.randint(0, V, (T0, B), generator=torch.Generator().manual_seed(seed))


def _bits(t):
    return t.detach().contiguous().view(torch.int32).cpu().numpy() if t.dtype == torch.float32 else t.cpu().numpy()


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("B", [1, 20, 40])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_generate_equals_forward_and_sample_replay(shape, B, engine):
    import zaremba_b200
    H, n_new = SHAPES[shape], 40
    m = _model(H, B, engine)
    m.train()                                                  # generate ignores .training
    prompt = _prompt(1, B)
    kw = dict(temperature=0.9, top_k=50, top_p=0.95, seed=SEED)
    tokens, logprobs, st = m.generate(prompt, n_new, **kw)
    m.eval()
    states = m.state_init(B)
    x = prompt.to(DEV)
    with torch.no_grad():
        for k in range(n_new):
            scores, states = m(x, states)
            t, lp = zaremba_b200.sample(scores, pos=k, **kw)
            assert np.array_equal(_bits(t), _bits(tokens[k])), f"step {k}: tokens differ"
            assert np.array_equal(_bits(lp), _bits(logprobs[k])), f"step {k}: logprobs differ"
            x = tokens[k].view(1, B)
    # after n_new forwards the replay has consumed the prompt and tokens[0 .. n_new-2]: the state generate returns
    for (h, c), (h2, c2) in zip(st, states):
        assert np.array_equal(_bits(h), _bits(h2)) and np.array_equal(_bits(c), _bits(c2)), "final states differ"
    assert len(set(tokens.flatten().tolist())) > 5, "a sampled stream should not collapse"


def _oracle_logprobs(m, prompt, tokens):
    """Teacher-forced fp64 log-probabilities of tokens[k] after prompt + tokens[:k]."""
    params = {k: v.detach().double().cpu().numpy() for k, v in m.named_parameters()}
    x = torch.cat([prompt, tokens[:-1].cpu()]).numpy()
    T, B = x.shape
    scores, _, _ = O.model_fwd(params, x, O.zero_states(L, B, m.hidden_size, np.float64), L)
    T0 = prompt.shape[0]
    sc = scores.reshape(T, B, -1)[T0 - 1:]
    mx = sc.max(-1, keepdims=True)
    lse = (mx + np.log(np.exp(sc - mx).sum(-1, keepdims=True)))[..., 0]
    want = np.take_along_axis(sc, tokens.cpu().numpy()[..., None], -1)[..., 0] - lse
    return want, np.abs(sc).max()


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("chunked", [False, True], ids=["one_window", "chunked_prefill"])
def test_generate_logprobs_against_oracle(engine, chunked):
    H, B, T0, n_new = 650, 20, 35, 40
    m = _model(H, B, engine)
    if chunked:
        m._context(8, B)                                       # max_seq 8 < T0: prefill in five windows
    prompt = _prompt(T0, B)
    tokens, logprobs, _ = m.generate(prompt, n_new, temperature=1.0, top_k=0, top_p=1.0, seed=SEED)
    if chunked:
        assert m._ctx_key[0] == 8, "generate must keep the existing context"
    want, scale = _oracle_logprobs(m, prompt, tokens)
    err = np.abs(logprobs.cpu().numpy() - want).max()
    # log softmax(z)[t] moves by at most twice the largest score error: the engine's forward tolerance of the scores
    tol = 2 * TOL[engine]["fwd"] * scale
    assert err <= tol, f"{engine}: logprob error {err:.3e} > {tol:.3e} (scores' scale {scale:.2f})"
    print(f"{engine} {'chunked' if chunked else 'one window'}: logprob error {err:.2e} (scale {scale:.2f})")


@pytest.mark.parametrize("engine", ENGINES)
def test_generate_chains(engine):
    m = _model(650, 20, engine)
    prompt = _prompt(5, 20)
    kw = dict(temperature=1.2, top_k=0, top_p=0.8, seed=SEED)
    t10, lp10, st10 = m.generate(prompt, 10, **kw)
    t4, lp4, st4 = m.generate(prompt, 4, **kw)
    t6, lp6, st6 = m.generate(t4[-1:], 6, states=st4, pos=4, **kw)
    assert np.array_equal(_bits(t10), _bits(torch.cat([t4, t6])))
    assert np.array_equal(_bits(lp10), _bits(torch.cat([lp4, lp6])))
    for (h, c), (h2, c2) in zip(st10, st6):
        assert np.array_equal(_bits(h), _bits(h2)) and np.array_equal(_bits(c), _bits(c2))


@pytest.mark.parametrize("engine", ENGINES)
def test_custom_layout_equals_permuted_pytorch_layout(engine):
    from zaremba_b200.model import _ifon_to_ifgo
    mc = _model(300, 8, engine, lstm_type="custom")
    mp = _model(300, 8, engine, seed=99)
    with torch.no_grad():
        mp.embed.W.copy_(mc.embed.W); mp.fc.W.copy_(mc.fc.W); mp.fc.b.copy_(mc.fc.b)
        for rc, rp in zip(mc.rnns, mp.rnns):
            for src, dst in zip(rc.tensors(), rp.tensors()):
                dst.copy_(_ifon_to_ifgo(src))
    prompt = _prompt(6, 8)
    kw = dict(temperature=0.8, top_k=20, top_p=1.0, seed=SEED)
    tc, lc, sc = mc.generate(prompt, 12, **kw)
    tp, lp, sp = mp.generate(prompt, 12, **kw)
    assert np.array_equal(_bits(tc), _bits(tp)) and np.array_equal(_bits(lc), _bits(lp))
    for (h, c), (h2, c2) in zip(sc, sp):
        assert h.shape == (8, 300) and h2.shape == (1, 8, 300)
        assert np.array_equal(_bits(h), _bits(h2.view(8, 300))) and np.array_equal(_bits(c), _bits(c2.view(8, 300)))


def test_generate_after_lazy_trainer_step():
    import zaremba_b200
    B, T = 20, 35
    m = _model(650, B, "tc")
    m.train()
    tr = zaremba_b200.Trainer(m, B, T, lazy_update=True)
    g = torch.Generator().manual_seed(4)
    x = torch.randint(0, V_PTB, (T, B), generator=g).to(DEV)
    y = torch.randint(0, V_PTB, (T, B), generator=g).to(DEV)
    tr.train_step(x, y, 1.0, 5.0)
    step, drop = tr.step, m._drop_step
    prompt = _prompt(3, B)
    kw = dict(temperature=1.0, top_k=40, top_p=0.9, seed=SEED)
    ta, la, sa = m.generate(prompt, 8, **kw)                   # weight updates still pending in the context
    tr.flush()
    tb, lb, sb = m.generate(prompt, 8, **kw)
    assert np.array_equal(_bits(ta), _bits(tb)) and np.array_equal(_bits(la), _bits(lb))
    for (h, c), (h2, c2) in zip(sa, sb):
        assert np.array_equal(_bits(h), _bits(h2)) and np.array_equal(_bits(c), _bits(c2))
    assert tr.step == step and m._drop_step == drop, "generate must not advance the dropout step"
    ctx = m._ctx.value
    with pytest.raises(ValueError, match="max_batch 20"):
        m.generate(_prompt(1, B + 1), 2)
    assert m._ctx.value == ctx, "the context must not be replaced"
    tr.train_step(x, y, 1.0, 5.0)                              # the Trainer still works on the same context


def test_launch_count_per_decode_token():
    """Persistent path: per token the sampler plus the unchanged forward -- state prep, embedding, one input GEMM and
    one recurrence per layer, projection: 2L + 4 kernels (the split-K GEMMs' zero-fill is a memset, not a kernel)."""
    from zaremba_b200 import _lib
    lib = _lib.load()
    m = _model(650, 20, "tc")
    prompt = _prompt(1, 20)
    m.generate(prompt, 3, seed=1)                              # packs the weight images
    assert _lib.rec_plans(m._ctx)["fwd"]["ok"], "B = 20 should run the persistent recurrence"
    counts = []
    for n in (5, 25):
        torch.cuda.synchronize()
        c0 = lib.zrb_launch_count()
        m.generate(prompt, n, seed=1)
        counts.append(lib.zrb_launch_count() - c0)
    per_token = (counts[1] - counts[0]) / 20
    assert per_token == 2 * L + 4, (counts, per_token)
