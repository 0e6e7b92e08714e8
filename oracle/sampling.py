"""Independent numpy restatement of the library's sampler (zrb_sample)  --  TEST INFRASTRUCTURE ONLY.

States DESIGN.md section 9 in float64 from its written definition, with oracle/philox.py's generator, so that tests
can check the kernel's tokens and log-probabilities without asking the library about itself.

Definition, for row b of a [B,V] score matrix z at position pos (temperature tau, top_k, top_p taken as the float32
values the config holds; seed and pos 64-bit unsigned):
  uniforms   key (seed lo32, seed hi32 XOR pos hi32); counter (j // 4, b, 0xFFFFFFFF, pos lo32); word r[j % 4];
             u_j = ((r >> 9) + 0.5) * 2^-23, strictly inside (0, 1)
  greedy     tau == 0: argmax_j z_j, lowest index on ties; nothing else applies
  top-k      0 < top_k < V: keep j with z_j >= the top_k-th largest z (ties at the boundary kept)
  top-p      top_p < 1: p = softmax(z / tau) over the top-k set; v* = the largest score such that the mass of
             {kept j : z_j >= v*} is >= top_p; keep z_j >= v* (ties kept)
  draw       token = argmax over kept j of z_j / tau + g_j, g_j = -log(-log u_j), lowest index on ties
  logprob    log softmax(z)[token] at temperature 1 over all V entries
"""
from __future__ import annotations

import numpy as np

from oracle import philox as PH

_LO = 0xFFFFFFFF


def uniforms(seed, pos, b, V):
    """float64 [V] (or [len(pos), V] for an array of positions): u_j of row b."""
    seed = int(seed) & (2 ** 64 - 1)
    pos_arr = np.atleast_1d(np.asarray(pos, dtype=np.uint64))
    G = (int(V) + 3) // 4
    ctr = np.empty((pos_arr.size, G, 4), dtype=np.uint64)
    ctr[..., 0] = np.arange(G, dtype=np.uint64)
    ctr[..., 1] = int(b) & _LO
    ctr[..., 2] = _LO
    ctr[..., 3] = (pos_arr & np.uint64(_LO))[:, None]
    key = np.empty((pos_arr.size, 1, 2), dtype=np.uint64)
    key[..., 0] = seed & _LO
    key[..., 1] = ((np.uint64(seed >> 32) ^ (pos_arr >> np.uint64(32))) & np.uint64(_LO))[:, None]
    r = PH.philox4x32_10(ctr, key).reshape(pos_arr.size, -1)[:, :V]
    u = ((r >> np.uint32(9)).astype(np.float64) + 0.5) * 2.0 ** -23
    return u if np.ndim(pos) else u[0]


def _f32(v):
    return float(np.float32(v))


def kept(z, temperature, top_k, top_p):
    """bool [V]: the kept set of one row (temperature > 0).  Also returns the top-p boundary's cumulative masses
    (mass of {z > v*}, mass of {z >= v*}; both None without the filter)."""
    z = np.asarray(z, dtype=np.float64)
    V = z.size
    tau, top_p = _f32(temperature), _f32(top_p)
    keep = np.ones(V, dtype=bool)
    if 0 < top_k < V:
        kth = np.sort(z)[::-1][top_k - 1]
        keep = z >= kth
    if top_p >= 1.0:
        return keep, (None, None)
    zs = z[keep]
    w = np.exp((zs - zs.max()) / tau)
    w /= w.sum()
    vals, inv = np.unique(zs, return_inverse=True)         # ascending distinct scores
    mass = np.bincount(inv.reshape(-1), weights=w, minlength=vals.size)[::-1]
    cum = np.cumsum(mass)                                   # mass of {z >= vals[::-1][i]}
    i = int(np.argmax(cum >= top_p)) if (cum >= top_p).any() else vals.size - 1
    v_star = vals[::-1][i]
    return keep & (z >= v_star), (cum[i] - mass[i], cum[i])


def log_softmax_at(z, j):
    z = np.asarray(z, dtype=np.float64)
    m = z.max()
    return z[j] - m - np.log(np.exp(z - m).sum())


def sample_row(z, temperature, top_k, top_p, seed, pos, b, u=None):
    """(token, logprob, info) of row b at position pos.  info: 'gap' = distance between the two largest perturbed
    scores over the kept set (inf for greedy or a single kept entry), 'boundary' = the top-p boundary masses.
    u: the row's uniforms(seed, pos, b, V) when the caller already has them."""
    z = np.asarray(z, dtype=np.float64)
    tau = _f32(temperature)
    if tau == 0.0:
        tok = int(np.argmax(z))
        return tok, log_softmax_at(z, tok), {"gap": np.inf, "boundary": (None, None)}
    keep, boundary = kept(z, temperature, top_k, top_p)
    g = -np.log(-np.log(uniforms(seed, pos, b, z.size) if u is None else u))
    s = np.where(keep, z / tau + g, -np.inf)
    tok = int(np.argmax(s))
    sk = s[keep]
    top2 = np.partition(sk, sk.size - 2)[-2:] if sk.size > 1 else None
    gap = np.inf if top2 is None else top2.max() - top2.min()
    return tok, log_softmax_at(z, tok), {"gap": gap, "boundary": boundary, "smax": s[tok]}


def sample(scores, temperature=1.0, top_k=0, top_p=1.0, seed=0, pos=0):
    """Rows of scores [B,V]: tokens [B] int64, logprobs [B] float64, per-row info."""
    out = [sample_row(row, temperature, top_k, top_p, seed, pos, b) for b, row in enumerate(np.asarray(scores))]
    return (np.array([o[0] for o in out], dtype=np.int64), np.array([o[1] for o in out]), [o[2] for o in out])


def filtered_probs(z, temperature, top_k, top_p):
    """The distribution a draw follows: softmax(z / tau) renormalised over the kept set (Gumbel-max)."""
    z = np.asarray(z, dtype=np.float64)
    keep, _ = kept(z, temperature, top_k, top_p)
    w = np.where(keep, np.exp((z - z[keep].max()) / _f32(temperature)), 0.0)
    return w / w.sum()
