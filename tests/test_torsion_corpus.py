"""CPU: the torsion and square-root corpora of torsion_corpus.py are what they claim.  Every G1 torsion point is on the curve with
the order it claims, E[7] and E[13] get a point on each of their lines, the reference's formula [x²]·φ(P) + P = O agrees with the
definition [r]·P = O on every entry (x² ≡ 1 modulo the torsion exponent, so (φ + 1)(T) = −φ²(T) ≠ O on torsion), and the traced
chain reaches O mid-chain, the doubling and cancelling branches and acc = P at the final addition.  The Fq values reach every
Tonelli–Shanks depth and long loops, the Fq2 values both arms of (a0 ± n)/2 and both a1 = 0 branches; the restatements return roots
that square back.  The G2 x values have a real x³ + B', and h2 is odd with no factor below 10^6."""
import random

import g2_bytes_oracle as o2
import torsion_corpus as tc
import varuna_bytes_oracle as vb
from oracle import bls12_377 as py
from oracle import g2 as og2

Q, R = tc.Q, tc.R


def test_group_orders_and_phi():
    assert tc.N1 == Q - tc.X                                      # #E(Fq) = q + 1 − t, t = x + 1
    assert tc.EXPONENT % 2 ** 46 == 0 and tc.H1 % (tc.EXPONENT // 2 ** 46) == 0
    assert pow(tc.PHI, 3, Q) == 1 and tc.PHI != 1
    assert tc.X2 % tc.EXPONENT == 1 and tc.X2 % (2 * tc.EXPONENT) == 1
    rng = random.Random(1)
    p = tc.random_point(rng)
    assert py.g1_mul(p, tc.N1) is None and py.g1_mul(p, R * tc.EXPONENT) is None    # E(Fq)'s exponent is r·EXPONENT


def test_torsion_points_have_their_orders():
    tor = tc.g1_torsion()
    for name, t, n in tor:
        assert py.g1_is_on_curve(t), name
        assert tc.order(t, n) == n, name
        assert tc.EXPONENT % n == 0 and tc.definition_status(t) == tc.NOT_IN_SUBGROUP, name
    orders = {n for _name, _t, n in tor}
    assert {2, 4, 8, 2 ** 16, 2 ** 45, 2 ** 46, 3, 7, 13, 499, tc.EXPONENT} <= orders
    assert {t for _n, t, o in tor if o == 2} == {(Q - 1, 0), ((-tc.PHI) % Q, 0), ((-tc.PHI * tc.PHI) % Q, 0)}
    assert {t for _n, t, o in tor if o == 3} == {(0, 1), (0, Q - 1)}
    for ell in (7, 13):                                          # one point on each of the ℓ + 1 lines of E[ℓ]
        pts = [t for _n, t, o in tor if o == ell]
        spans = {tc._subgroup_of(t, ell) for t in pts}
        assert len(pts) == ell + 1 and len(spans) == ell + 1


def test_formula_agrees_with_the_definition_and_reaches_every_branch():
    entries = tc.g1_entries()
    seen = set()
    for name, p, definition, formula, events in entries:
        assert definition == formula, name
        seen |= events
    assert {"O mid-chain", "doubling branch", "cancelling branch", "acc = P at the final addition"} <= seen
    statuses = {d for _n, _p, d, _f, _e in entries}
    assert statuses == {tc.VALID, tc.NOT_ON_CURVE, tc.NOT_IN_SUBGROUP}
    # on torsion the formula gives −φ²(T)
    for name, t, _n in tc.g1_torsion():
        assert py.g1_add(py.g1_mul(tc.phi(t), tc.X2), t) == py.g1_neg(tc.phi(tc.phi(t))), name
    # acc = P at the final addition happens exactly where φ(T) = T: the order-3 points
    for name, p, _d, _f, events in entries:
        if "acc = P at the final addition" in events:
            assert p[0] == 0 and tc.phi(p) == p, name


def test_fq_values_reach_every_depth_and_long_loops():
    vals = tc.fq_values()
    depths, rounds = set(), 0
    for a in vals:
        root, ks = tc.fq_sqrt_trace(a)
        assert root == vb.sqrt(a)[0]                              # the bytes oracle's restatement returns the same root
        assert (root is not None) == tc.is_square(a), a
        if root is not None:
            assert root * root % Q == a % Q
            depths.add(ks[0] if ks else 0)
            rounds = max(rounds, len(ks))
        else:
            assert ks == [tc.TWO_ADICITY]
    assert depths == set(range(tc.TWO_ADICITY))
    assert rounds >= 40
    assert {0, 1, Q - 1} <= set(vals) and sum(not tc.is_square(a) for a in vals) >= 5


def test_fq2_values_reach_both_arms_and_both_real_branches():
    vals = tc.fq2_values()
    branches, norm_depths, t_depths = set(), set(), set()
    for a in vals:
        root, branch = tc.fq2_sqrt_trace(a)
        assert root == o2.fq2_sqrt(a)
        assert (root is not None) == tc.fq2_is_square(a), a
        branches.add(branch)
        if root is not None:
            assert og2.f2_sqr(root) == (a[0] % Q, a[1] % Q)
        if a[1] and root is not None:
            ks = tc.fq_sqrt_trace(tc.norm(a))[1]
            norm_depths.add(ks[0] if ks else 0)
            ks = tc.fq_sqrt_trace(root[0] * root[0])[1]
            t_depths.add(ks[0] if ks else 0)
    assert branches == {"a1 = 0, real", "a1 = 0, imaginary", "(a0 + n)/2", "(a0 − n)/2", "no norm root"}
    assert (0, 0) in vals
    assert {0, 1, 2, 3, 5, 8, 13, 21, 34, 45} <= norm_depths and {0, 1, 2, 7, 19, 45} <= t_depths


def test_g2_inputs():
    xs = tc.g2_real_rhs_x()
    assert sum(tc.is_square(a0) for _x, a0 in xs) == sum(not tc.is_square(a0) for _x, a0 in xs) > 0
    for x, a0 in xs:
        assert o2.rhs(x) == (a0, 0)
        y = o2.fq2_sqrt(o2.rhs(x))
        assert y is not None and og2.f2_sqr(y) == (a0, 0)
    for name, p in tc.g2_mixed_points():
        assert og2.g2_is_on_curve(p), name
        assert tc.g2_mul_raw(p, tc.H2 * R) is None, name
        assert o2.check(p) == o2.NOT_IN_SUBGROUP, name


def test_h2_is_odd_without_small_factors():
    h2 = tc.H2
    assert abs(Q * Q + 1 - h2 * R) <= 2 * Q                      # Hasse
    assert tc.g2_mul_raw(o2.G2_GEN, R) is None
    assert h2 % 2 == 1
    sieve = bytearray([1]) * 1_000_000
    sieve[0:2] = b"\0\0"
    for i in range(2, 1000):
        if sieve[i]:
            sieve[i * i::i] = bytearray(len(sieve[i * i::i]))
    assert not [p for p in range(3, 1_000_000, 2) if sieve[p] and h2 % p == 0]
