"""CPU model of the MSM's signed-digit recoding (csrc/msm.cu), run on the digit-boundary corpus of msm_corpus.py.

The recoding exists twice: in k_digits (the histogram pass, and the index scatter) and in k_scatter_records (the cursors of
the record scatter).  The histogram sizes every bucket and the scatter fills it, so the two must give the same digits; a
disagreement writes records past a bucket's range.  The model below restates their loop statement by statement, with the
32-bit arithmetic of the device, and test_model_matches_both_recodings_in_the_source checks that both kernels still contain
exactly those statements.  No GPU needed."""
import re
import os

import numpy as np
import pytest

from oracle import bls12_377 as py

import msm_corpus as mc

HERE = os.path.dirname(os.path.abspath(__file__))
MSM_CU = os.path.join(HERE, "..", "snarkvm_b200", "csrc", "msm.cu")
M32 = 0xFFFFFFFF


def recode(s: int, c: int):
    """The digit loop of k_digits / k_scatter_records on the 8 little-endian words of s.
    Returns [(raw, neg, mag)] per window and the carry left after the last window."""
    words = [(s >> (32 * k)) & M32 for k in range(8)]
    nwin = 253 // c + 1
    half = (1 << (c - 1)) & M32
    carry = 0
    out = []
    for w in range(nwin):
        bit = w * c
        wi, sh = bit >> 5, bit & 31
        lo = hi = 0
        for k in range(8):                                  # for (k < 8) { if (k == wi) lo = s[k]; if (k == wi + 1) hi = s[k]; }
            if k == wi:
                lo = words[k]
            if k == wi + 1:
                hi = words[k]
        funnel = (((hi << 32) | lo) >> sh) & M32            # __funnelshift_r(lo, hi, sh)
        raw = ((funnel & (((1 << c) - 1) & M32)) + carry) & M32
        neg = 1 if raw > half else 0
        mag = (((1 << c) - raw) & M32) if neg else raw
        carry = neg
        out.append((raw, neg, mag))
    return out, carry


def test_model_matches_both_recodings_in_the_source():
    """both device loops consist of the statements the model restates"""
    src = open(MSM_CU).read()
    stmts = {
        "half": r"(?:const )?uint32_t half = 1u << \(c - 1\);",
        "raw": r"(?:const )?uint32_t raw = \(__funnelshift_r\(lo, hi, sh\) & \(\(1u << c\) - 1u\)\) \+ carry;",
        "neg": r"(?:const )?uint32_t neg = raw > half \? 1u : 0u;",
        "mag": r"(?:const )?uint32_t mag = neg \? \(1u << c\) - raw : raw;",
        "carry": r"carry = neg;",
        "select": r"for \(int k = 0; k < 8; k\+\+\) \{ if \(k == wi\) lo = s\[k\]; if \(k == wi \+ 1\) hi = s\[k\]; \}",
        "nwin": r"p\.nwin = 253 / c \+ 1;",
    }
    bodies = {}
    for kernel in ("k_digits", "k_scatter_records"):
        m = re.search(r"__global__ void __launch_bounds__\(256\) " + kernel + r"\(.*?\n\}\n", src, re.S)
        assert m, kernel
        bodies[kernel] = m.group(0)
    for name, pat in stmts.items():
        if name == "nwin":
            assert len(re.findall(pat, src)) == 2, "msm_make_plan and msm_make_plan_precomputed"
            continue
        for kernel, body in bodies.items():
            assert len(re.findall(pat, body)) == 1, (kernel, name)
    # the bucket slot: window w of the plain path feeds bucket set w, bucket mag − 1
    assert "(flat ? 0u : (uint32_t)w * nbuckets) + (mag - 1u)" in bodies["k_digits"]
    assert "(FLAT ? 0u : (uint32_t)w * nbuckets) + (mag - 1u)" in bodies["k_scatter_records"]


@pytest.mark.parametrize("c", list(range(2, 25)))
def test_recoding_is_exact_and_in_range(c):
    """Σ d_w·2^{cw} = s, |d_w| ≤ 2^{c−1}, bucket index mag − 1 < nbuckets, no carry out of the top window — on the digit-boundary
    corpus for this c, the corpora of two neighbouring window sizes and random scalars"""
    nbuckets = 1 << (c - 1)
    rng = np.random.default_rng(c)
    corpus = mc.digit_boundary_scalars(c)
    corpus += mc.digit_boundary_scalars(c - 1 if c > 2 else 3, seed=1) + mc.digit_boundary_scalars(c + 1 if c < 24 else 23, seed=2)
    corpus += [int(rng.integers(0, 1 << 62)) << 191 | int(rng.integers(0, 1 << 62)) for _ in range(200)]
    corpus = [s % py.R_MOD for s in corpus]
    for s in corpus:
        digits, carry = recode(s, c)
        assert carry == 0, (c, s)
        total = 0
        for w, (raw, neg, mag) in enumerate(digits):
            assert 0 <= mag <= nbuckets, (c, s, w)
            if mag:
                assert mag - 1 < nbuckets
            total += (-mag if neg else mag) << (c * w)
        assert total == s, (c, s)


@pytest.mark.parametrize("c", list(range(2, 25)))
def test_corpus_reaches_the_boundaries(c):
    """raw == half, raw == half + 1 and raw == 2^c (carry only) in every window that can hold them below r; the carry-only
    top window where c divides 253 (c = 11, 23)"""
    half = 1 << (c - 1)
    nwin = mc.nwin_of(c)
    seen = set()
    top_carry_only = False
    for s in mc.digit_boundary_scalars(c):
        digits, _ = recode(s, c)
        for w, (raw, neg, mag) in enumerate(digits):
            seen.add((w, raw))
        field_top = s >> ((nwin - 1) * c)
        if field_top == 0 and digits[-1][0] == 1:
            top_carry_only = True

    def reachable(w, t):
        # some field f < 2^c and incoming carry cin with f + cin = t and a scalar below r that has them
        for cin in (0, 1):
            f = t - cin
            if not 0 <= f < (1 << c) or (cin and w == 0):
                continue
            lowest = (f << (w * c)) + (((half + 1) << ((w - 1) * c)) if cin else 0)
            if lowest < py.R_MOD:
                return True
        return False

    missing = [(w, t) for w in range(nwin) for t in (half, half + 1, 1 << c) if reachable(w, t) and (w, t) not in seen]
    assert not missing, missing
    # every window below the top two holds all three (window 0 has no incoming carry, so no raw == 2^c)
    for w in range(nwin - 2):
        assert all((w, t) in seen for t in (half, half + 1) + ((1 << c,) if w else ())), w
    if 253 % c == 0:
        assert top_carry_only
