"""The beam-search oracle (oracle/beam.py) on toy models, without a GPU: it is what the GPU tests hold the kernels to.

  * exhaustive: with K >= V^(n_new-1) the search returns exactly the brute-force top K of all V^n_new continuations;
  * K = 1 is greedy decoding;
  * ties: equal candidates come out in flat-index order (slot, then token);
  * finished beams keep their score, emit only eos at log-probability 0 and stay in the ranking.
"""
import itertools

import numpy as np

from oracle import beam as BM


def _table_model(V, B, seed):
    """Scores of the next token from (prompt, last token, position): a random table model."""
    rng = np.random.default_rng(seed)
    first = rng.normal(size=(B, V)) * 2
    trans = rng.normal(size=(V, V)) * 2
    pos = rng.normal(size=(8, V)) * 0.5

    def next_scores(rows):
        return np.stack([first[b] if not p else trans[p[-1]] + pos[len(p)] for b, p in rows])
    return next_scores


def _brute_force(next_scores, b, V, n_new):
    out = []
    for seq in itertools.product(range(V), repeat=n_new):
        lp = [BM.log_softmax(next_scores([(b, seq[:t])])[0])[seq[t]] for t in range(n_new)]
        out.append((sum(lp), seq))
    out.sort(key=lambda e: -e[0])
    return out


def test_exhaustive_search_equals_brute_force():
    for V, n_new, seed in ((4, 3, 0), (5, 2, 1), (3, 4, 2)):
        B, K = 2, V ** (n_new - 1)
        f = _table_model(V, B, seed)
        hyps = BM.search(f, B, n_new, K)
        for b in range(B):
            want = _brute_force(f, b, V, n_new)[:K]
            got = hyps[b]
            assert [h[0] for h in got] == [w[1] for w in want], f"V={V} n_new={n_new} prompt {b}"
            assert np.allclose([h[2] for h in got], [w[0] for w in want], rtol=0, atol=1e-12)
            for tok, lps, score in got:
                assert abs(sum(lps) - score) < 1e-12


def test_k1_is_greedy():
    V, B, n_new = 7, 3, 6
    f = _table_model(V, B, 5)
    hyps = BM.search(f, B, n_new, 1)
    for b in range(B):
        seq = ()
        for _ in range(n_new):
            seq += (int(np.argmax(f([(b, seq)])[0])),)
        assert hyps[b][0][0] == seq


def test_ties_come_out_in_flat_index_order():
    z = np.array([0.5, 2.0, 2.0, -1.0, 2.0, 0.0])
    tok, par, *_ = BM.step(z[None], 3)                          # the first step: one row, three tied maxima
    assert tok.tolist() == [1, 2, 4] and par.tolist() == [0, 0, 0]
    z1 = np.array([0.5, 2.0, 1.0, -1.0])
    tok, par, cum, _, _ = BM.step(np.stack([z1, z1]), 2, cum=np.array([-1.25, -1.25]))   # identical rows, equal S
    assert tok.tolist() == [1, 1] and par.tolist() == [0, 1] and cum[0] == cum[1]


def test_finished_beam_keeps_score_and_competes():
    V, eos = 4, 0
    # after eos the table makes every continuation expensive, so the finished hypothesis overtakes live ones
    first = np.array([3.0, 2.9, -5.0, -5.0])
    trans = np.full((V, V), -8.0)
    trans[1] = [-3.0, -3.0, -3.0, -3.0]

    def f(rows):
        return np.stack([first if not p else trans[p[-1]] for _, p in rows])
    hyps = BM.search(f, 1, 4, 2, eos=eos)[0]
    best_tok, best_lp, best_score = hyps[0]
    assert best_tok == (0, 0, 0, 0), hyps
    assert best_lp[1:] == (0.0, 0.0, 0.0)
    assert best_score == best_lp[0] == BM.log_softmax(first)[0]
    assert hyps[1][0][0] == 1 and eos not in hyps[1][0][:1]
    # the step form: a finished row offers exactly one candidate, eos at logp 0 with its own S
    scores = np.array([[9.0, 1.0, 0.0, 0.0], [0.0, 5.0, 0.0, 0.0]])
    tok, par, cum, lp, _ = BM.step(scores, 2, cum=np.array([-1.0, -2.0]), last=np.array([eos, 1]), eos=eos)
    assert (tok[0], par[0], cum[0], lp[0]) == (eos, 0, -1.0, 0.0)
    assert (tok[1], par[1]) == (1, 1)
