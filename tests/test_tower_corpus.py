"""CPU: the tower operand corpus (tests/tower_corpus.py) is what it claims to be, and its word layout is the GT image of
tests/pairing_oracle.py."""
import random

import numpy as np
import pytest

import pairing_oracle as po
import tower_corpus as tc

Q = tc.Q
WRAPS = {Q - 1, Q, Q + 1, 2 * Q - 2}


@pytest.fixture(scope="module")
def cyclotomic():
    return tc.cyclotomic_elements()


def test_cyclotomic_inputs_lie_in_the_cyclotomic_subgroup(cyclotomic):
    """g^(q⁴ − q² + 1) = 1, i.e. g^(q⁴)·g = g^(q²), for every input; and literally, by the power, for two of them.  Elements that
    differ by a factor in Fq6 share their image, so there are fewer inputs than corpus elements."""
    assert cyclotomic[0] == po.F12_ONE and len(cyclotomic) > 50
    for g in cyclotomic:
        assert po.f12_mul(po.f12_frob(g, 4), g) == po.f12_frob(g, 2)
    for g in cyclotomic[1:3]:
        assert po.f12_pow(g, Q**4 - Q**2 + 1) == po.F12_ONE


def test_frobenius_rows_agree_with_repeated_q_powers():
    """the oracle's f6_frob / f12_frob(·, k) against k applications of the q-power map (pinned to f^q in test_pairing_oracle.py),
    so every row of the coefficient tables is checked by its definition, not by its own table"""
    rng = random.Random(7)
    f = tuple(tuple((rng.randrange(Q), rng.randrange(Q)) for _ in range(3)) for _ in range(2))
    g = f
    for k in range(12):
        assert po.f12_frob(f, k) == g, k
        assert po.f6_frob(f[0], k % 6) == g[0], k
        g = po.f12_frob(g, 1)


@pytest.mark.parametrize("kind,slots", [("f6", 3), ("f12", 6)])
def test_every_family_is_present(kind, slots):
    els = tc.elements(kind)
    fams = {f for f, _ in els}
    want = {"zero", "one", "minus_one", "in_fq2", "all_q_minus_1", "shaped", "boundary", "uniform"}
    want |= {f"slot{i}" for i in range(slots)} | {f"fq{j}" for j in range(2 * slots)}
    if kind == "f12":
        want |= {"in_fq6", "in_w"}
    assert fams == want
    for f, e in els:
        comps = tc.flat(e)
        nz = [i for i, v in enumerate(comps) if v]
        if f.startswith("slot"):
            i = int(f[4:])
            assert nz and set(nz) <= {2 * i, 2 * i + 1}, f
        elif f.startswith("fq"):
            assert nz == [int(f[2:])], f
        elif f == "in_fq2":
            assert nz and set(nz) <= {0, 1}
        elif f == "in_fq6":
            assert nz and max(nz) < 6
        elif f == "in_w":
            assert nz and min(nz) >= 6
        elif f == "all_q_minus_1":
            imgs = {v * tc.fc.QR % Q for v in comps}
            assert comps == [Q - 1] * len(comps) or imgs == {Q - 1}


@pytest.mark.parametrize("kind", ["f6", "f12"])
def test_shaped_families_reach_the_wrap_points(kind):
    """boundary elements put image sums of matching components on q − 1, q, q + 1 and 2q − 2, and the product pairs include
    m_all_ones pairs (a·b ≡ q mod 2^384 component by component)"""
    seen = set()
    for f, e in tc.elements(kind):
        if f != "boundary":
            continue
        imgs = [v * tc.fc.QR % Q for v in tc.flat(e)]
        hits = {imgs[i] + imgs[j] for i in range(len(imgs)) for j in range(i % 2, i, 2)} & WRAPS
        assert hits, e
        seen |= hits
    assert seen == WRAPS
    m_all_ones = 0
    for a, b in tc.pairs(kind):
        ia = [v * tc.fc.QR % Q for v in tc.flat(a)]
        ib = [v * tc.fc.QR % Q for v in tc.flat(b)]
        m_all_ones += all(x * y % (1 << 384) == Q for x, y in zip(ia, ib))
    assert m_all_ones >= 20


def test_sparse_coefficients_have_zero_and_q_minus_1_parts():
    for n in (2, 3):
        co = tc.sparse_coefficients(n)
        for i in range(n):
            parts = {c[i] for c in co}
            assert {(0, 0), (Q - 1, 0), (Q - 1, Q - 1), (tc.plain(Q - 1), tc.plain(Q - 1))} <= parts


def test_is_one_perturbations_cover_every_word():
    cases = tc.is_one_cases()
    assert [c[1] for c in cases].count(True) == 1
    perturbed = [w for _, _, w in cases if w is not None]
    assert sorted(set(perturbed)) == list(range(144)) and len(perturbed) == 288
    one = tc.words([po.F12_ONE])[0]
    for e, want, w in cases:
        row = tc.words([e])[0]
        if w is not None:
            assert [i for i in range(144) if row[i] != one[i]] == [w]
        assert (row == one).all() == want
    raw1 = tc.words([cases[3][0]])[0]
    assert raw1[0] == 1 and not raw1[1:].any()


def test_final_exponentiation_cases():
    cases = tc.final_exp_cases()
    fams = [f for f, _ in cases]
    assert fams.count("zero") == 1 and fams.count("in_fq6") >= 8 and fams.count("general") >= 4 and len(cases) <= 40
    for f, e in cases:
        assert (e == po.F12_ONE or e[1] == po.F6_ZERO) if f in ("zero", "in_fq6") else e[1] != po.F6_ZERO


def test_line_step_operands_reach_zero_and_q_minus_1():
    states = tc.line_states()
    comps = {v for s in states for v in tc.flat(s)}
    assert {0, 1, Q - 1, tc.plain(Q - 1)} <= comps
    assert any(s[2] == (0, 0) for s in states) and any(s[1] == (0, 0) for s in states)
    assert len(tc.addition_cases()) > len(states)


@pytest.mark.parametrize("kind", ["f6", "f12"])
def test_word_layout_is_the_gt_image(kind):
    """words() writes the reference's Fp12 image: it round-trips through pairing_oracle.gt_bytes / gt_from_bytes"""
    els = [e for _, e in tc.elements(kind)]
    w = tc.words(els)
    assert w.dtype == np.uint32 and w.shape == (len(els), 72 if kind == "f6" else 144)
    assert tc.from_words(w, kind) == els
    if kind == "f12":
        for e, row in zip(els, w):
            assert row.tobytes() == po.gt_bytes(e)
            assert po.gt_from_bytes(row.tobytes()) == e
    else:
        for e, row in zip(els, w):
            full = (e, po.F6_ZERO)
            assert row.tobytes() == po.gt_bytes(full)[:288]
