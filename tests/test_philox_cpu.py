"""The dropout masks' generator, checked without a GPU.

oracle/philox.py states the keep-masks from their written definition (DESIGN.md section 3).  Here it is pinned to the
published Philox4x32-10 known-answer vectors (Random123's kat_vectors), to a plain one-counter restatement of the round
function, and to the definition's threshold and identity rules.  When nvcc is available, the library's own host-side
generator and key derivation (common.cuh: philox4x32_10, make_mask_src) are compiled into a small host program and
checked against the same vectors and the same definition.
"""
import os
import subprocess

import numpy as np
import pytest

from oracle import philox as P

# Random123 kat_vectors, philox4x32 with 10 rounds: counter, key -> output
KAT = [
    ((0x00000000, 0x00000000, 0x00000000, 0x00000000), (0x00000000, 0x00000000),
     (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff, 0xffffffff, 0xffffffff, 0xffffffff), (0xffffffff, 0xffffffff),
     (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
]


def _philox_scalar(ctr, key):
    """One counter, Python integers: the round function exactly as Salmon et al. state it."""
    c0, c1, c2, c3 = ctr
    k0, k1 = key
    for _ in range(10):
        hi0, lo0 = divmod(0xD2511F53 * c0, 1 << 32)
        hi1, lo1 = divmod(0xCD9E8D57 * c2, 1 << 32)
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return c0, c1, c2, c3


def _keep_scalar(seed, step, site, e, p):
    k = (seed & 0xFFFFFFFF, ((seed >> 32) ^ (step >> 32)) & 0xFFFFFFFF)
    g = e // 4
    r = _philox_scalar((g & 0xFFFFFFFF, g >> 32, site, step & 0xFFFFFFFF), k)
    return (r[e % 4] >> 8) >= P.threshold(p)


@pytest.mark.parametrize("ctr,key,want", KAT)
def test_known_answer_vectors(ctr, key, want):
    assert _philox_scalar(ctr, key) == want
    got = P.philox4x32_10(np.array([ctr], dtype=np.uint64), np.array(key, dtype=np.uint64))
    assert got.dtype == np.uint32 and tuple(int(v) for v in got[0]) == want


def test_vectorised_equals_scalar():
    rng = np.random.default_rng(0)
    ctr = rng.integers(0, 2 ** 32, size=(64, 4), dtype=np.uint64)
    key = rng.integers(0, 2 ** 32, size=(64, 2), dtype=np.uint64)
    got = P.philox4x32_10(ctr, key)
    for i in range(64):
        assert tuple(int(v) for v in got[i]) == _philox_scalar(tuple(int(v) for v in ctr[i]), tuple(int(v) for v in key[i]))
    # masks: element by element, over both key words, a non-zero site, the step's high word and a ragged n
    for seed, step, site, p in [(0, 0, 0, 0.5), (2 ** 63 + 12345, 2 ** 32 + 5, 7, 0.65), (0xDEADBEEF12345678, 1, 2, 0.999),
                                (5, 2 ** 32 - 1, 1, 1e-7)]:
        n = 1023
        mask = P.keep_mask(seed, step, site, n, p)
        assert mask.shape == (n,) and mask.dtype == bool
        assert [bool(v) for v in mask] == [_keep_scalar(seed, step, site, e, p) for e in range(n)]
        assert np.array_equal(P.keep_mask(seed, step, site, 5, p), mask[:5]), "a mask must not depend on n"


def test_identity_threshold_and_scale():
    assert P.keep_mask(123, 4, 1, 1001, 0.0).all()
    assert P.threshold(np.float32(0.65)) == 10905190          # float32(0.65) * 2^24 = 10905189.6
    assert P.threshold(0.65) == P.threshold(np.float32(0.65)), "p is the float32 value the config holds"
    assert P.threshold(0.5) == 1 << 23 and P.threshold(1e-7) == 2
    assert P.scale(0.65) == np.float32(1.0 / (1.0 - float(np.float32(0.65))))
    assert P.scale(0.5) == np.float32(2.0)
    # distinct sites, steps and seeds draw distinct masks; the keep rate is about 1 - p
    a = P.keep_mask(1, 0, 0, 40000, 0.65)
    for other in (P.keep_mask(1, 0, 1, 40000, 0.65), P.keep_mask(1, 1, 0, 40000, 0.65), P.keep_mask(2, 0, 0, 40000, 0.65)):
        assert not np.array_equal(a, other)
    assert abs(a.mean() - 0.35) < 0.01


_HOST_PROGRAM = r"""
#include <cstdio>
#include <cstring>
#include "common.cuh"
// stdin lines:  "P c0 c1 c2 c3 k0 k1"  -> the four output words of zrb::philox4x32_10
//               "M seed step site p"   -> the fields of zrb::make_mask_src (train mode)
int main() {
    char kind[4];
    while (scanf("%3s", kind) == 1) {
        if (!strcmp(kind, "P")) {
            unsigned c0, c1, c2, c3, k0, k1;
            if (scanf("%u %u %u %u %u %u", &c0, &c1, &c2, &c3, &k0, &k1) != 6) return 1;
            zrb::Philox4 r = zrb::philox4x32_10(c0, c1, c2, c3, k0, k1);
            printf("%u %u %u %u\n", r.v[0], r.v[1], r.v[2], r.v[3]);
        } else {
            unsigned long long seed, step;
            int site;
            float p;
            if (scanf("%llu %llu %d %a", &seed, &step, &site, &p) != 4) return 1;
            zrb::MaskSrc m = zrb::make_mask_src(nullptr, seed, step, site, p, 1);
            unsigned sbits;
            memcpy(&sbits, &m.scale, 4);
            printf("%u %u %u %u %u %u %d\n", m.k0, m.k1, m.c2, m.c3, m.thresh, sbits, m.active);
        }
    }
    return 0;
}
"""


def test_library_host_generator_matches_reference(tmp_path):
    """common.cuh's philox4x32_10 and make_mask_src, compiled for the host, against the known answers and the
    definition (key derivation, counter words, threshold, scale, identity at p = 0)."""
    from zaremba_b200 import build as zb
    try:
        nvcc = zb._nvcc()
    except RuntimeError:
        pytest.skip("nvcc is not available")
    src = tmp_path / "philox_host.cu"
    src.write_text(_HOST_PROGRAM)
    exe = tmp_path / "philox_host"
    subprocess.run([nvcc, *zb.ARCH, "-std=c++17", "-I", zb.CSRC, str(src), "-o", str(exe)], check=True,
                   capture_output=True, text=True)
    rng = np.random.default_rng(1)
    vec = [(c, k) for c, k, _ in KAT] + [(tuple(int(v) for v in rng.integers(0, 2 ** 32, 4)),
                                          tuple(int(v) for v in rng.integers(0, 2 ** 32, 2))) for _ in range(16)]
    cases = [(s, t, site, p) for s in (0, 2 ** 63 + 12345, 0xFFFFFFFFFFFFFFFF) for t in (0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 5)
             for site, p in ((0, 0.65), (7, 0.5), (2, 1e-7), (1, 0.999), (1, 0.0))]
    lines = [f"P {' '.join(map(str, c))} {' '.join(map(str, k))}" for c, k in vec]
    lines += [f"M {s} {t} {site} {float(np.float32(p)).hex()}" for s, t, site, p in cases]
    out = subprocess.run([str(exe)], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True,
                         timeout=60).stdout.split("\n")
    for (c, k), line in zip(vec, out):
        assert tuple(int(v) for v in line.split()) == _philox_scalar(c, k), (c, k, line)
    for (s, t, site, p), line in zip(cases, out[len(vec):]):
        k0, k1, c2, c3, thresh, sbits, active = (int(v) for v in line.split())
        assert (k0, k1) == P.key_words(s, t), (s, t, line)
        assert (c2, c3) == (site, t & 0xFFFFFFFF), (s, t, line)
        assert active == (1 if p > 0 else 0)
        if p > 0:
            assert thresh == P.threshold(p), (p, thresh)
            assert np.array([sbits], dtype=np.uint32).view(np.float32)[0] == P.scale(p), (p, sbits)
