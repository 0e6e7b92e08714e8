"""The sampler's definition, checked without a GPU.

oracle/sampling.py states zrb_sample in float64 from its written definition (DESIGN.md section 9).  Here it is pinned
on hand-built rows (ties at every boundary), shown to draw from the renormalised filtered softmax by a seeded
chi-square test, and -- when nvcc is available -- the library's own host-side key / counter / uniform rule
(common.cuh: make_sample_src, sample_words, sample_uniform) is compiled into a small host program and compared with the
oracle's uniforms bit for bit.
"""
import ctypes as C
import subprocess

import numpy as np
import pytest
from scipy import stats

from oracle import philox as PH
from oracle import sampling as S


def test_greedy_ties_go_to_the_lowest_index():
    z = np.array([0.5, 2.0, -1.0, 2.0, 2.0], dtype=np.float32)
    for seed in (0, 7):
        tok, lp, _ = S.sample_row(z, 0.0, 0, 1.0, seed, 3, 0)
        assert tok == 1
        assert np.isclose(lp, 2.0 - np.log(np.exp(z.astype(np.float64)).sum()))
    # greedy ignores the filters
    assert S.sample_row(z, 0.0, 1, 1e-6, 0, 0, 0)[0] == 1


def test_top_k_and_top_p_keep_boundary_ties():
    z = np.array([3.0, 1.0, 2.0, 2.0, 0.0, 2.0, -5.0])
    keep, _ = S.kept(z, 1.0, 2, 1.0)                      # 2nd largest is 2.0: all three 2.0 entries stay
    assert keep.tolist() == [True, False, True, True, False, True, False]
    keep, _ = S.kept(z, 1.0, 4, 1.0)
    assert keep.tolist() == [True, False, True, True, False, True, False]
    keep, _ = S.kept(z, 1.0, 5, 1.0)
    assert keep.tolist() == [True, True, True, True, False, True, False]
    # top-p: the max alone holds p0 = e^3 / sum; asking for a bit more must take all three 2.0 ties together
    w = np.exp(z - 3.0) / np.exp(z - 3.0).sum()
    keep, (above, incl) = S.kept(z, 1.0, 0, float(w[0]) * 1.01)
    assert keep.tolist() == [True, False, True, True, False, True, False]
    assert np.isclose(above, w[0]) and np.isclose(incl, w[0] + 3 * w[2])
    # top-p over the top-k set: renormalised over the kept four
    keep, _ = S.kept(z, 1.0, 2, 0.999)
    assert keep.tolist() == [True, False, True, True, False, True, False]


def test_tiny_top_p_keeps_only_the_maximum_and_top_k_1_is_greedy():
    rng = np.random.default_rng(0)
    for _ in range(20):
        z = rng.normal(size=37).astype(np.float32)
        want = int(np.argmax(z))
        keep, _ = S.kept(z, 0.7, 0, 1e-6)
        assert keep.sum() == 1 and keep[want]
        for seed, pos in ((0, 0), (1, 2 ** 40 + 3)):
            assert S.sample_row(z, 1.3, 0, 1e-6, seed, pos, 5)[0] == want
            assert S.sample_row(z, 1.3, 1, 1.0, seed, pos, 5)[0] == want


def _chi2(z, tau, top_k, top_p, n=40000, seed=1234):
    q = S.filtered_probs(z, tau, top_k, top_p)
    u = S.uniforms(seed, np.arange(n), 0, z.size)           # n positions of one row
    keep, _ = S.kept(z, tau, top_k, top_p)
    s = np.where(keep, z.astype(np.float64) / np.float32(tau) - np.log(-np.log(u)), -np.inf)
    tok = np.argmax(s, axis=1)
    # the vectorised draw is the row-wise definition
    for p in (0, 1, 17, n - 1):
        assert tok[p] == S.sample_row(z, tau, top_k, top_p, seed, p, 0)[0]
    counts = np.bincount(tok, minlength=z.size)
    assert counts[q == 0].sum() == 0, "drew a filtered entry"
    k = q > 0
    return stats.chisquare(counts[k], q[k] * n).pvalue, int(k.sum())


def test_draws_follow_the_filtered_softmax():
    z = np.random.default_rng(5).normal(size=50).astype(np.float32)
    p, kept_n = _chi2(z, 0.8, 20, 0.9)
    assert 1 < kept_n < 20, kept_n                         # both filters bite
    assert p > 1e-3, p
    p, kept_n = _chi2(z, 0.8, 0, 1.0)
    assert kept_n == 50 and p > 1e-3, p


_HOST_PROGRAM = r"""
#include <cstdio>
#include <cstring>
#include "common.cuh"
// stdin lines:  "U seed pos b g"  -> the four words of zrb::sample_words and the bits of their four uniforms
//               "W r"              -> the bits of zrb::sample_uniform(r)
int main() {
    char kind[4];
    while (scanf("%3s", kind) == 1) {
        if (!strcmp(kind, "U")) {
            unsigned long long seed, pos;
            unsigned b, g;
            if (scanf("%llu %llu %u %u", &seed, &pos, &b, &g) != 4) return 1;
            zrb::Philox4 r = zrb::sample_words(zrb::make_sample_src(seed, pos), g, b);
            for (int i = 0; i < 4; ++i) {
                float u = zrb::sample_uniform(r.v[i]);
                unsigned bits;
                memcpy(&bits, &u, 4);
                printf("%u %u ", r.v[i], bits);
            }
            printf("\n");
        } else {
            unsigned r;
            if (scanf("%u", &r) != 1) return 1;
            float u = zrb::sample_uniform(r);
            unsigned bits;
            memcpy(&bits, &u, 4);
            printf("%u\n", bits);
        }
    }
    return 0;
}
"""


def test_library_host_uniforms_match_the_oracle(tmp_path):
    from zaremba_b200 import build as zb
    try:
        nvcc = zb._nvcc()
    except RuntimeError:
        pytest.skip("nvcc is not available")
    src = tmp_path / "sample_host.cu"
    src.write_text(_HOST_PROGRAM)
    exe = tmp_path / "sample_host"
    subprocess.run([nvcc, *zb.ARCH, "-std=c++17", "-I", zb.CSRC, str(src), "-o", str(exe)], check=True,
                   capture_output=True, text=True)
    V = 4 * 6 + 3
    cases = [(s, p, b) for s in (0, 2 ** 63 + 12345, 0xFFFFFFFFFFFFFFFF) for p in (0, 1, 2 ** 32 - 1, 2 ** 32 + 5)
             for b in (0, 1, 39)]
    lines = [f"U {s} {p} {b} {g}" for s, p, b in cases for g in range((V + 3) // 4)]
    words = [0, 1, 511, 512, 0x7FFFFFFF, 0xFFFFFDFF, 0xFFFFFE00, 0xFFFFFFFF]
    lines += [f"W {r}" for r in words]
    out = subprocess.run([str(exe)], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True,
                         timeout=60).stdout.split("\n")
    i = 0
    for s, p, b in cases:
        want = S.uniforms(s, p, b, V)
        got_w, got_u = [], []
        for g in range((V + 3) // 4):
            v = [int(t) for t in out[i].split()]
            got_w += v[0::2]
            got_u += v[1::2]
            i += 1
        got_u = np.array(got_u[:V], dtype=np.uint32).view(np.float32)
        assert np.array_equal(got_u.astype(np.float64), want), (s, p, b)
        # the words are Philox4x32-10 under the stated key and counter
        k = ((s & 0xFFFFFFFF), ((s >> 32) ^ (p >> 32)) & 0xFFFFFFFF)
        ctr = [(g, b, 0xFFFFFFFF, p & 0xFFFFFFFF) for g in range((V + 3) // 4)]
        ref = PH.philox4x32_10(np.array(ctr, dtype=np.uint64), np.array(k, dtype=np.uint64)).reshape(-1)
        assert [int(w) for w in ref] == got_w, (s, p, b)
    for r, line in zip(words, out[i:]):
        u = float(np.array([int(line)], dtype=np.uint32).view(np.float32)[0])
        assert u == ((r >> 9) + 0.5) * 2.0 ** -23, (r, u)
        assert 0.0 < u < 1.0
    lo = float(np.array([int(out[i])], dtype=np.uint32).view(np.float32)[0])
    hi = float(np.array([int(out[i + len(words) - 1])], dtype=np.uint32).view(np.float32)[0])
    assert lo == 2.0 ** -24 and hi == 1.0 - 2.0 ** -24


def test_sampling_struct_layout():
    from zaremba_b200 import _lib
    assert C.sizeof(_lib.ZrbSampling) == 24
    assert [getattr(_lib.ZrbSampling, f).offset for f in ("temperature", "top_k", "top_p", "reserved", "seed")] == \
        [0, 4, 8, 12, 16]
