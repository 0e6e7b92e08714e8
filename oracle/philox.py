"""Independent numpy restatement of the library's dropout keep-masks  --  TEST INFRASTRUCTURE ONLY.

The CUDA kernels never store a dropout mask: every kernel that applies a dropout site regenerates the keep flags
from a counter-based generator (zaremba_b200/csrc/common.cuh).  This module states the same masks from their
written definition (DESIGN.md section 3), so that tests can check the kernels' masks bit for bit without asking
the library for them.

Definition (all words are 32-bit unsigned; seed and step are 64-bit unsigned):
  generator  Philox4x32-10 (Salmon et al., SC'11; the Random123 constants): ten rounds of
               (c0, c1, c2, c3) <- (hi(M1*c2) ^ c1 ^ k0, lo(M1*c2), hi(M0*c0) ^ c3 ^ k1, lo(M0*c0))
             with M0 = 0xD2511F53, M1 = 0xCD9E8D57, the key bumped by (0x9E3779B9, 0xBB67AE85) after each round
  key        (k0, k1) = (seed lo32, seed hi32 XOR step hi32)
  counter    (g lo32, g hi32, site, step lo32) for the group g = e // 4 of element e
  lane       e % 4: element e reads word r[e % 4] of its group's output
  keep       iff (r[lane] >> 8) >= round-half-up(p * 2^24), p being the float32 value the config holds
  scale      float32(1 / (1 - p)), the multiplier of a kept element
  identity   p = 0 or eval mode keeps every element with multiplier 1

Elements are numbered row-major over the site's [T, B, H] activation (e = (t * B + b) * H + j); sites are 0 for the
embedding output and l + 1 for the output of recurrent layer l.
"""
from __future__ import annotations

import numpy as np

M0, M1 = 0xD2511F53, 0xCD9E8D57
W0, W1 = 0x9E3779B9, 0xBB67AE85
_LO = np.uint64(0xFFFFFFFF)
_32 = np.uint64(32)


def philox4x32_10(ctr, key):
    """Philox4x32-10 of counters `ctr` (uint32-valued, shape [..., 4]) under keys `key` ([..., 2], broadcast against
    the counters).  Returns uint32 [..., 4]."""
    ctr = np.asarray(ctr, dtype=np.uint64)
    key = np.asarray(key, dtype=np.uint64)
    c0, c1, c2, c3 = (ctr[..., i] & _LO for i in range(4))
    k0, k1 = key[..., 0] & _LO, key[..., 1] & _LO
    for _ in range(10):
        p0 = np.uint64(M0) * c0            # < 2^64: exact in uint64
        p1 = np.uint64(M1) * c2
        c0, c1, c2, c3 = (p1 >> _32) ^ c1 ^ k0, p1 & _LO, (p0 >> _32) ^ c3 ^ k1, p0 & _LO
        k0 = (k0 + np.uint64(W0)) & _LO
        k1 = (k1 + np.uint64(W1)) & _LO
    return np.stack([c0, c1, c2, c3], axis=-1).astype(np.uint32)


def threshold(p):
    """Keep iff (r >> 8) >= threshold(p): round-half-up of float32(p) * 2^24 (exact in float64)."""
    return int(np.floor(float(np.float32(p)) * 16777216.0 + 0.5))


def scale(p):
    """Multiplier of a kept element: float32(1 / (1 - p)) with p the float32 value."""
    return np.float32(1.0 / (1.0 - float(np.float32(p))))


def key_words(seed, step):
    seed, step = int(seed) & (2 ** 64 - 1), int(step) & (2 ** 64 - 1)
    return seed & 0xFFFFFFFF, (seed >> 32) ^ (step >> 32)


def draws(seed, step, site, n):
    """uint32[n]: the 24-bit draw r[e % 4] >> 8 of elements 0..n-1 (independent of p)."""
    n = int(n)
    G = (n + 3) // 4
    g = np.arange(G, dtype=np.uint64)
    ctr = np.empty((G, 4), dtype=np.uint64)
    ctr[:, 0] = g & _LO
    ctr[:, 1] = g >> _32
    ctr[:, 2] = int(site) & 0xFFFFFFFF
    ctr[:, 3] = int(step) & 0xFFFFFFFF
    r = philox4x32_10(ctr, np.array(key_words(seed, step), dtype=np.uint64))
    return r.reshape(-1)[:n] >> np.uint32(8)


def keep_mask(seed, step, site, n, p):
    """bool[n]: the keep flags of elements 0..n-1 of dropout site `site` at training step `step`."""
    if float(np.float32(p)) <= 0.0:
        return np.ones(int(n), dtype=bool)
    return draws(seed, step, site, n) >= np.uint32(threshold(p))


def site_masks(seed, step, L, T, B, H, p):
    """The L + 1 keep-masks of one training step, [T, B, H] each, in the oracle's site order."""
    return [keep_mask(seed, step, site, T * B * H, p).reshape(T, B, H) for site in range(L + 1)]
