"""Independent numpy restatement of the library's beam search (zrb_beam_step, zrb_beam_search)  --  TEST
INFRASTRUCTURE ONLY.

States DESIGN.md section 10 in float64 from its written definition, so that tests can check the kernels' choices and
scores without asking the library about itself.

Definition, for K beams over a vocabulary of V entries:
  row r       slot i of a prompt, cumulative score S_r, last token t_r (none before the first step)
  logp        logp_rj = z_rj - logsumexp(z_r); candidate cand_rj = S_r + logp_rj
  finished    t_r == eos (eos >= 0): the row's only candidate is j = eos with logp 0 and cand S_r
  order       cand descending, then flat index i*V + j ascending
  selection   the K best candidates of a prompt become its slots 0..K-1 in that order; slot k' records parent i,
              token j, S = cand, logp
  first step  one row per prompt (the prompt's last position), S = 0, never finished
  output      the hypothesis in final slot k traced back through the parents; its score is its final S
"""
from __future__ import annotations

import numpy as np


def log_softmax(z):
    z = np.asarray(z, dtype=np.float64)
    m = z.max(-1, keepdims=True)
    return z - m - np.log(np.exp(z - m).sum(-1, keepdims=True))


def candidates(scores, cum, last, eos):
    """All candidates of one prompt's rows: (cand, flat, logp) float64 / int64 / float64 arrays, flat = i*V + j."""
    scores = np.asarray(scores, dtype=np.float64)
    R, V = scores.shape
    lp = log_softmax(scores)
    cand, flat, logp = [], [], []
    for i in range(R):
        if last is not None and eos is not None and eos >= 0 and last[i] == eos:
            cand.append([cum[i]]); flat.append([i * V + eos]); logp.append([0.0])
        else:
            cand.append(cum[i] + lp[i]); flat.append(i * V + np.arange(V)); logp.append(lp[i])
    return np.concatenate(cand), np.concatenate(flat).astype(np.int64), np.concatenate(logp)


def select(cand, flat, K):
    """Indices of the K best (all of them when there are fewer), best first: cand descending, flat ascending."""
    order = np.lexsort((flat, -cand))
    return order[:K]


def step(scores, K, cum=None, last=None, eos=-1):
    """One step over B prompts, as zrb_beam_step.  scores [B*K_in, V]; cum None = the first step (K_in = 1, S = 0).
    Returns (tokens, parents, cum_out, logprobs) [B*K] and, per prompt, the float64 margin between its K-th and
    (K+1)-th candidates (inf when there is no (K+1)-th)."""
    scores = np.asarray(scores, dtype=np.float64)
    V = scores.shape[1]
    K_in = 1 if cum is None else K
    B = scores.shape[0] // K_in
    cum = np.zeros(B * K_in) if cum is None else np.asarray(cum, dtype=np.float64)
    out = [np.empty(B * K, np.int64), np.empty(B * K, np.int64), np.empty(B * K), np.empty(B * K)]
    margins = []
    for b in range(B):
        rows = slice(b * K_in, (b + 1) * K_in)
        c, f, lp = candidates(scores[rows], cum[rows], None if last is None else np.asarray(last)[rows], eos)
        order = np.lexsort((f, -c))
        pick = order[:K]
        out[0][b * K:(b + 1) * K] = f[pick] % V
        out[1][b * K:(b + 1) * K] = f[pick] // V
        out[2][b * K:(b + 1) * K] = c[pick]
        out[3][b * K:(b + 1) * K] = lp[pick]
        margins.append(c[order[K - 1]] - c[order[K]] if order.size > K else np.inf)
    return (*out, np.array(margins))


def search(next_scores, B, n_new, K, eos=-1):
    """A whole search over B prompts.  next_scores(rows) -> float64 [len(rows), V] gives the scores of the next token
    for each row (b, prefix): prompt b continued by the tuple of tokens `prefix` (() at the first step).

    Keeps all candidates when a prompt has fewer than K (so K >= V^(n_new-1) enumerates every sequence).  Returns
    per prompt a list of (tokens tuple, logprobs tuple, score), best first."""
    hyps = [[((), (), 0.0)] for _ in range(B)]
    for _ in range(n_new):
        rows = [(b, h[0]) for b in range(B) for h in hyps[b]]
        sc = np.asarray(next_scores(rows), dtype=np.float64)
        at = 0
        for b in range(B):
            live = hyps[b]
            z = sc[at:at + len(live)]
            at += len(live)
            last = [h[0][-1] if h[0] else -1 for h in live]
            c, f, _ = candidates(z, [h[2] for h in live], last, eos)
            lp_rows = log_softmax(z)
            V = z.shape[1]
            new = []
            for e in select(c, f, K):
                i, j = divmod(int(f[e]), V)
                tok, lps, _ = live[i]
                lp = 0.0 if (eos >= 0 and last[i] == eos) else float(lp_rows[i, j])
                new.append((tok + (j,), lps + (lp,), float(c[e])))
            hyps[b] = new
    return hyps
