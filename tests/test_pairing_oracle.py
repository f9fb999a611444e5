"""CPU: the big-int pairing restatement (tests/pairing_oracle.py) against the reference's constants and the pairing's algebra, and the
device tables (tower.cuh, pairing.cu) against the restatement.  The Python pairing takes ~0.1 s, so the pairings are few."""
import json
import os
import random
import re

import pytest

from oracle import bls12_377 as py
from oracle import g2 as og2

import pairing_oracle as po

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
Q, R = po.Q, py.R_MOD


@pytest.fixture(scope="module")
def pairing_golden():
    with open(os.path.join(HERE, "golden", "pairing_constants.json")) as f:
        return json.load(f)


def _limbs(v):
    return [(v >> (64 * i)) & (2**64 - 1) for i in range(6)]


def _rand_f12(rng):
    return tuple(tuple((rng.randrange(Q), rng.randrange(Q)) for _ in range(3)) for _ in range(2))


def test_frobenius_coefficients_equal_the_reference(pairing_golden):
    for name, table in (("FROBENIUS_COEFF_FP6_C1", po.FP6_C1), ("FROBENIUS_COEFF_FP6_C2", po.FP6_C2), ("FROBENIUS_COEFF_FP12_C1", po.FP12_C1)):
        want = pairing_golden[name]
        assert len(want) == len(table)
        for c, w in zip(table, want):
            assert [_limbs(py.fq_to_mont(c[0])), _limbs(py.fq_to_mont(c[1]))] == w, name


def test_frobenius_map_is_the_q_power():
    rng = random.Random(1)
    f = _rand_f12(rng)
    assert po.f12_frob(f, 1) == po.f12_pow(f, Q)
    assert po.f12_frob(f, 2) == po.f12_frob(po.f12_frob(f, 1), 1)
    assert po.f12_frob(f, 3) == po.f12_frob(po.f12_frob(f, 2), 1)
    assert po.f12_frob(f, 12) == f


def _header_table(src, name, rows):
    m = re.search(r"uint32_t " + name + r"\[" + str(rows) + r"\]\[12\] = \{(.*?)\};", src, re.S)
    assert m, name
    vals = [int(x, 16) for x in re.findall(r"0x([0-9a-f]{8})u", m.group(1))]
    assert len(vals) == rows * 12
    return [sum(vals[12 * r + i] << (32 * i) for i in range(12)) for r in range(rows)]


def test_device_tables_equal_the_oracle():
    with open(os.path.join(ROOT, "snarkvm_b200", "csrc", "tower.cuh")) as f:
        src = f.read()
    for name, table in (("FROB_FP6_C1", po.FP6_C1), ("FROB_FP6_C2", po.FP6_C2), ("FROB_FP12_C1", po.FP12_C1)):
        assert all(c[1] == 0 for c in table), name                       # the tables keep c0 only
        assert _header_table(src, name, len(table)) == [py.fq_to_mont(c[0]) for c in table], name
    with open(os.path.join(ROOT, "snarkvm_b200", "csrc", "pairing.cu")) as f:
        src = f.read()
    m = re.search(r"G2_B1\[12\] = \{(.*?)\};", src, re.S)
    vals = [int(x, 16) for x in re.findall(r"0x([0-9a-f]{8})u", m.group(1))]
    assert og2.G2_B[0] == 0 and sum(v << (32 * i) for i, v in enumerate(vals)) == py.fq_to_mont(og2.G2_B[1])


def test_mul_by_034_equals_the_full_product():
    rng = random.Random(2)
    for _ in range(3):
        f = _rand_f12(rng)
        c0, c3, c4 = ((rng.randrange(Q), rng.randrange(Q)) for _ in range(3))
        sparse = ((c0, og2.F2_ZERO, og2.F2_ZERO), (c3, c4, og2.F2_ZERO))
        assert po.mul_by_034(f, c0, c3, c4) == po.f12_mul(f, sparse)


def test_cyclotomic_square_equals_squaring_after_the_easy_part():
    rng = random.Random(3)
    for _ in range(3):
        f = _rand_f12(rng)
        g = po.f12_mul(po.f12_conj(f), po.f12_inv(f))                  # f^(q⁶ − 1)
        g = po.f12_mul(po.f12_frob(g, 2), g)                            # … (q² + 1)
        assert po.cyclotomic_square(g) == po.f12_sqr(g)
        assert po.cyclotomic_exp(g, 0xB5) == po.f12_pow(g, 0xB5)
        assert po.f12_mul(f, po.f12_inv(f)) == po.F12_ONE


def test_prepare_has_69_triples():
    coeffs, inf = po.g2_prepare(og2.G2_GEN)
    assert not inf and len(coeffs) == 69 == 63 + bin(po.X)[3:].count("1")
    assert po.g2_prepare(None) == ([], True)
    assert len(po.prepared_bytes(po.g2_prepare(og2.G2_GEN))) == po.PREPARED_BYTES == len(po.prepared_bytes(po.g2_prepare(None)))


@pytest.fixture(scope="module")
def e_gen():
    return po.pairing(py.G1_GENERATOR, og2.G2_GEN)


def test_bilinearity(e_gen):
    """bls12_377/tests.rs test_bilinearity: e(sP, Q) = e(P, sQ) = e(P, Q)^s ≠ 1"""
    rng = random.Random(4)
    P = py.g1_mul(py.G1_GENERATOR, rng.randrange(1, R))
    Qp = og2.g2_mul(og2.G2_GEN, rng.randrange(1, R))
    s = rng.randrange(1, R)
    a1 = po.pairing(py.g1_mul(P, s), Qp)
    a2 = po.pairing(P, og2.g2_mul(Qp, s))
    a3 = po.f12_pow(po.pairing(P, Qp), s)
    assert a1 == a2 == a3 and a1 != po.F12_ONE


def test_generator_pairing_has_order_r(e_gen):
    assert e_gen != po.F12_ONE
    assert po.f12_pow(e_gen, R) == po.F12_ONE
    assert po.pairing(None, og2.G2_GEN) == po.F12_ONE == po.pairing(py.G1_GENERATOR, None)


def test_final_exponentiation_multiple():
    """final_exponentiation(f) = f^(m·(q¹² − 1)/r) with m = 3: read off the formula and checked on a Miller value"""
    lam = po.final_exponentiation_exponent()
    hard = (Q**4 - Q**2 + 1) // R
    assert (Q**4 - Q**2 + 1) % R == 0 and lam % hard == 0 and lam // hard == po.FINAL_EXP_MULTIPLE == 3
    f = po.miller_loop([(py.G1_GENERATOR, po.g2_prepare(og2.G2_GEN))])
    assert po.final_exponentiation(f) == po.f12_pow(f, po.FINAL_EXP_MULTIPLE * (Q**12 - 1) // R)


def test_separate_miller_loops_multiply_to_the_shared_loop():
    rng = random.Random(5)
    pairs = [(py.g1_mul(py.G1_GENERATOR, rng.randrange(1, R)), po.g2_prepare(og2.g2_mul(og2.G2_GEN, rng.randrange(1, R)))) for _ in range(3)]
    pairs.append((None, pairs[0][1]))
    pairs.append((pairs[1][0], po.g2_prepare(None)))
    shared = po.miller_loop(pairs)
    prod = po.F12_ONE
    for p in pairs:
        prod = po.f12_mul(prod, po.miller_loop([p]))
    assert shared == prod


def test_gt_image_round_trip():
    f = _rand_f12(random.Random(6))
    b = po.gt_bytes(f)
    assert len(b) == po.GT_BYTES and po.gt_from_bytes(b) == f


def test_real_srs_beta_h():
    """e(β·G, H) = e(G, β·H) on the mainnet setup: powers[1] of powers-of-beta-15 against beta-h.usrs"""
    with open(os.path.join(HERE, "golden", "beta_h.usrs"), "rb") as f:
        beta_h = po.usrs_g2_point(f.read())
    assert og2.g2_is_on_curve(beta_h)
    with open(os.path.join(HERE, "golden", "powers_of_beta_15_first512.usrs"), "rb") as f:
        powers = py.parse_usrs_points(f.read(), 2)
    assert powers[0] == py.G1_GENERATOR
    assert po.product_of_pairings([(powers[1], og2.G2_GEN), (py.g1_neg(powers[0]), beta_h)]) == po.F12_ONE
    assert po.product_of_pairings([(powers[0], og2.G2_GEN), (py.g1_neg(powers[1]), beta_h)]) != po.F12_ONE
