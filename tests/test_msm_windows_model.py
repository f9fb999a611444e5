"""CPU model of the MSM's mixed window layouts (MsmPlan: nwin − 1 windows of c bits and a c_top-bit top window whose buckets
span several bucket sets), on the digit-boundary corpus of msm_corpus.py.  No GPU needed.

The digit loop of k_digits / k_scatter_records is the uniform one (test_msm_digits_model.py) with the window width chosen per
window; the model restates it with the device's 32-bit arithmetic and checks that the digits sum back to s, that every digit
indexes a bucket inside its own window's sets, and that the top digit of a scalar below 2^253 is never negative."""
import os
import re

import numpy as np
import pytest

from oracle import bls12_377 as py

import msm_corpus as mc

HERE = os.path.dirname(os.path.abspath(__file__))
MSM_CU = os.path.join(HERE, "..", "snarkvm_b200", "csrc", "msm.cu")
M32 = 0xFFFFFFFF

# (c, nwin, c_top): the 2^24 plan and the small layouts the GPU path table forces onto small inputs
LAYOUTS = [(18, 14, 20), (12, 21, 14), (8, 32, 10), (15, 17, 14)]


def recode(s: int, c_low: int, nwin: int, c_top: int):
    words = [(s >> (32 * k)) & M32 for k in range(8)]
    carry = 0
    out = []
    for w in range(nwin):
        c = c_top if w == nwin - 1 else c_low
        bit = w * c_low
        wi, sh = bit >> 5, bit & 31
        lo = words[wi] if wi < 8 else 0
        hi = words[wi + 1] if wi + 1 < 8 else 0
        funnel = (((hi << 32) | lo) >> sh) & M32
        half = (1 << (c - 1)) & M32
        raw = ((funnel & (((1 << c) - 1) & M32)) + carry) & M32
        neg = 1 if raw > half else 0
        mag = (((1 << c) - raw) & M32) if neg else raw
        carry = neg
        out.append((raw, neg, mag))
    return out, carry


def top_sets(c, c_top):
    return 1 << (c_top - c) if c_top > c else 1


def test_both_kernels_pick_the_width_per_window():
    src = open(MSM_CU).read()
    for kernel in ("k_digits", "k_scatter_records"):
        m = re.search(r"__global__ void __launch_bounds__\(256\) " + kernel + r"\(.*?\n\}\n", src, re.S)
        assert m, kernel
        body = m.group(0)
        assert re.search(r"const int c = w == nwin - 1 \? c_top : c_low;", body), kernel
        assert re.search(r"(?:const )?int bit = w \* c_low", body), kernel
    assert 'parse_window_widths("18*13,20", p)' in src


def check_layout(c, nwin, c_top, corpus):
    nb = 1 << (c - 1)
    for s in corpus:
        digits, carry = recode(s, c, nwin, c_top)
        total = 0
        for w, (raw, neg, mag) in enumerate(digits):
            sets = top_sets(c, c_top) if w == nwin - 1 else 1
            cap = 1 << ((c_top if w == nwin - 1 else c) - 1)
            assert 0 <= mag <= cap, (s, w)
            if mag:
                slot = w * nb + mag - 1                                   # (uint32_t)w * nbuckets + (mag - 1u)
                assert w * nb <= slot < (w + sets) * nb, (s, w)
            total += (-mag if neg else mag) << (c * w)
        if s < 1 << 253:
            assert carry == 0 and digits[-1][1] == 0, s                 # no carry out, top digit ≥ 0
            assert total == s, s


@pytest.mark.parametrize("c,nwin,c_top", LAYOUTS)
def test_mixed_recoding_is_exact_and_in_range(c, nwin, c_top):
    rng = np.random.default_rng(c)
    corpus = mc.digit_boundary_scalars(c) + mc.digit_boundary_scalars(c_top, seed=1)
    corpus += [int(rng.integers(0, 1 << 62)) << 191 | int(rng.integers(0, 1 << 62)) for _ in range(200)]
    corpus = [v % py.R_MOD for v in corpus]
    # scalars in [r, 2^253) are accepted and must stay exact; bits 253..255 are flagged, but their digits must stay in range
    corpus += [(1 << 253) - 1, py.R_MOD, py.R_MOD + 12345, (1 << 253) - (1 << 200)]
    corpus += [(1 << 256) - 1, (7 << 253) | 5, 1 << 253]
    check_layout(c, nwin, c_top, corpus)


def test_layout_parameters():
    for c, nwin, c_top in LAYOUTS:
        assert (nwin - 1) * c < 253 <= (nwin - 1) * c + c_top - 1           # the top window absorbs the last carry
    # the 2^24 plan: 14 windows, every bucket set 2^17 buckets, the top window in four sets
    assert top_sets(18, 20) == 4 and 13 * 18 == 234


def test_corpus_reaches_the_top_digits():
    """the corpus for c = 18 reaches the top window's largest digit below r, (r − 1) >> 234, and a carry into the top window"""
    c, nwin, c_top = LAYOUTS[0]
    top_max = (py.R_MOD - 1) >> ((nwin - 1) * c)
    seen_max = False
    seen_carry = False
    for s in mc.digit_boundary_scalars(c):
        digits, _ = recode(s, c, nwin, c_top)
        raw_top = digits[-1][0]
        field = s >> ((nwin - 1) * c)
        seen_max |= raw_top == top_max
        seen_carry |= raw_top == field + 1
    assert seen_max and seen_carry
    assert top_max == 305881
