"""TEST INFRASTRUCTURE — Python big-int restatement of the BLS12-377 pairing, on top of oracle/g2.py.

Restates, as plain mathematics on Python integers:
  * Fq6 = Fq2[v]/(v³ − u), Fq12 = Fq6[w]/(w² − v)   — fields/src/fp6_3over2.rs, fp12_2over3over2.rs; curves/src/bls12_377/fq6.rs
                                                       (NONRESIDUE = u), fq12.rs.  Elements are tuples: Fq6 = (c0, c1, c2) of Fq2,
                                                       Fq12 = (c0, c1) of Fq6.
  * Frobenius coefficients          — computed here from their definitions: u^((q^k − 1)/3), u^((2q^k − 2)/3) for Fq6 and
                                       u^((q^k − 1)/6) for Fq12 (tests/test_pairing_oracle.py pins them to the reference's numbers).
  * mul_by_034, cyclotomic_square, cyclotomic_exp — fp12_2over3over2.rs
  * G2Prepared::from_affine         — templates/bls12/g2.rs (doubling_step, addition_step, twist type D): 63 doubling and 6 addition
                                       steps for X = 0x8508c00000000001, so 69 coefficient triples
  * miller_loop, final_exponentiation — templates/bls12/bls12.rs (X not negative; eprint 2016/130, Table 1)

What the final exponentiation computes: final_exponentiation(f) = f^(m·(q¹² − 1)/r) with m = FINAL_EXP_MULTIPLE = 3 (the Table 1
formula raises to 3·(q⁴ − q² + 1)/r after the easy part (q⁶ − 1)(q² + 1); tests/test_pairing_oracle.py derives m from the formula's
exponent and checks it on a field element).  m is prime to r, so e(P, Q) = 1 exactly when the m = 1 pairing is one.

Byte images: a prepared point is 69 × 3 Fq2 (c0.c0 c0.c1 c1.c0 … c2.c1, Montgomery, 48 B LE each: 19872 B), then the infinity flag
as a little-endian u32 and 28 zero bytes (19904 B; an infinity point has zero coefficients).  A GT value is twelve Montgomery Fq in
the order c0.c0.c0, c0.c0.c1, c0.c1.c0, … c1.c2.c1: 576 B.  Only tests/ may import this module.
"""
from __future__ import annotations

from oracle.bls12_377 import Q_MOD, R_MOD, fq_from_mont, fq_to_mont
from oracle.g2 import F2_ONE, F2_ZERO, G2_B, NONRESIDUE, f2_add, f2_inv, f2_mul, f2_neg, f2_sqr, f2_sub

Q = Q_MOD
X = 0x8508C00000000001
FINAL_EXP_MULTIPLE = 3
PREPARED_BYTES = 19904
COEFF_TRIPLES = 69
GT_BYTES = 576
U = (0, 1)                                           # the Fq6 non-residue u


def f2_pow(a, e: int):
    acc = F2_ONE
    for bit in bin(e)[2:] if e else "":
        acc = f2_sqr(acc)
        if bit == "1":
            acc = f2_mul(acc, a)
    return acc


def f2_mul_fp(a, s: int): return (a[0] * s % Q, a[1] * s % Q)
def f2_nr(a): return (NONRESIDUE * a[1] % Q, a[0])   # a·u, u² = −5
def f2_dbl(a): return f2_add(a, a)


FP2_C1 = [1, Q - 1]                                  # −5^((q^k − 1)/2): Frobenius of Fq2 conjugates
FP6_C1 = [f2_pow(U, (Q ** k - 1) // 3) for k in range(6)]
FP6_C2 = [f2_pow(U, (2 * Q ** k - 2) // 3) for k in range(6)]
FP12_C1 = [f2_pow(U, (Q ** k - 1) // 6) for k in range(12)]


def f2_frob(a, k): return (a[0], a[1] * FP2_C1[k % 2] % Q)


# ---- Fq6 ----
F6_ZERO, F6_ONE = (F2_ZERO, F2_ZERO, F2_ZERO), (F2_ONE, F2_ZERO, F2_ZERO)
def f6_add(a, b): return tuple(f2_add(x, y) for x, y in zip(a, b))
def f6_sub(a, b): return tuple(f2_sub(x, y) for x, y in zip(a, b))
def f6_neg(a): return tuple(f2_neg(x) for x in a)
def f6_nr(a): return (f2_nr(a[2]), a[0], a[1])       # a·v, v³ = u


def f6_mul(a, b):
    a0, a1, a2 = a
    b0, b1, b2 = b
    return (f2_add(f2_mul(a0, b0), f2_nr(f2_add(f2_mul(a1, b2), f2_mul(a2, b1)))),
            f2_add(f2_add(f2_mul(a0, b1), f2_mul(a1, b0)), f2_nr(f2_mul(a2, b2))),
            f2_add(f2_add(f2_mul(a0, b2), f2_mul(a1, b1)), f2_mul(a2, b0)))


def f6_inv(a):
    a0, a1, a2 = a
    t0 = f2_sub(f2_sqr(a0), f2_nr(f2_mul(a1, a2)))
    t1 = f2_sub(f2_nr(f2_sqr(a2)), f2_mul(a0, a1))
    t2 = f2_sub(f2_sqr(a1), f2_mul(a0, a2))
    n = f2_inv(f2_add(f2_mul(a0, t0), f2_nr(f2_add(f2_mul(a2, t1), f2_mul(a1, t2)))))
    return (f2_mul(t0, n), f2_mul(t1, n), f2_mul(t2, n))


def f6_frob(a, k):
    return (f2_frob(a[0], k), f2_mul(f2_frob(a[1], k), FP6_C1[k % 6]), f2_mul(f2_frob(a[2], k), FP6_C2[k % 6]))


# ---- Fq12 ----
F12_ONE = (F6_ONE, F6_ZERO)


def f12_mul(a, b):
    return (f6_add(f6_mul(a[0], b[0]), f6_nr(f6_mul(a[1], b[1]))), f6_add(f6_mul(a[0], b[1]), f6_mul(a[1], b[0])))


def f12_sqr(a): return f12_mul(a, a)
def f12_conj(a): return (a[0], f6_neg(a[1]))


def f12_inv(a):
    t = f6_inv(f6_sub(f6_mul(a[0], a[0]), f6_nr(f6_mul(a[1], a[1]))))
    return (f6_mul(a[0], t), f6_neg(f6_mul(a[1], t)))


def f12_frob(a, k):
    c1 = f6_frob(a[1], k)
    return (f6_frob(a[0], k), tuple(f2_mul(x, FP12_C1[k % 12]) for x in c1))


def f12_pow(a, e: int):
    acc = F12_ONE
    for bit in bin(e)[2:] if e else "":
        acc = f12_sqr(acc)
        if bit == "1":
            acc = f12_mul(acc, a)
    return acc


def mul_by_034(f, c0, c3, c4):
    """f · ((c0, 0, 0) + (c3, c4, 0)·w), with the reference's three-product schedule"""
    a = tuple(f2_mul(x, c0) for x in f[0])
    b = f6_mul(f[1], (c3, c4, F2_ZERO))
    e = f6_mul(f6_add(f[0], f[1]), (f2_add(c0, c3), c4, F2_ZERO))
    return (f6_add(a, f6_nr(b)), f6_sub(e, f6_add(a, b)))


def cyclotomic_square(f):
    """fp12_2over3over2.rs cyclotomic_square (Granger–Scott): the square of an element of the cyclotomic subgroup"""
    z0, z4, z3 = f[0]
    z2, z1, z5 = f[1]

    def sq(a, b):
        t = f2_mul(a, b)
        return f2_sub(f2_sub(f2_mul(f2_add(a, b), f2_add(a, f2_nr(b))), t), f2_nr(t)), f2_dbl(t)
    t0, t1 = sq(z0, z1)
    t2, t3 = sq(z2, z3)
    t4, t5 = sq(z4, z5)
    r00 = f2_add(f2_dbl(f2_sub(t0, z0)), t0)
    r11 = f2_add(f2_dbl(f2_add(t1, z1)), t1)
    tmp = f2_nr(t5)
    r10 = f2_add(f2_dbl(f2_add(tmp, z2)), tmp)
    r02 = f2_add(f2_dbl(f2_sub(t4, z3)), t4)
    r01 = f2_add(f2_dbl(f2_sub(t2, z4)), t2)
    r12 = f2_add(f2_dbl(f2_add(t3, z5)), t3)
    return ((r00, r01, r02), (r10, r11, r12))


def cyclotomic_exp(f, e: int):
    res, found = F12_ONE, False
    for bit in bin(e)[2:]:
        if not found:
            if bit == "0":
                continue
            found = True
        res = cyclotomic_square(res)
        if bit == "1":
            res = f12_mul(res, f)
    return res


def exp_by_x(f): return cyclotomic_exp(f, X)        # X is not negative: no conjugation


# ---- G2Prepared ----
TWO_INV = (Q + 1) // 2


def _doubling_step(r):
    x, y, z = r
    a = f2_mul_fp(f2_mul(x, y), TWO_INV)
    b = f2_sqr(y)
    c = f2_sqr(z)
    e = f2_mul(G2_B, f2_add(f2_dbl(c), c))
    f = f2_add(f2_dbl(e), e)
    g = f2_mul_fp(f2_add(b, f), TWO_INV)
    h = f2_sub(f2_sqr(f2_add(y, z)), f2_add(b, c))
    i = f2_sub(e, b)
    j = f2_sqr(x)
    e_sq = f2_sqr(e)
    nr = (f2_mul(a, f2_sub(b, f)), f2_sub(f2_sqr(g), f2_add(f2_dbl(e_sq), e_sq)), f2_mul(b, h))
    return nr, (f2_neg(h), f2_add(f2_dbl(j), j), i)


def _addition_step(r, q):
    x, y, z = r
    qx, qy = q
    theta = f2_sub(y, f2_mul(qy, z))
    lam = f2_sub(x, f2_mul(qx, z))
    c = f2_sqr(theta)
    d = f2_sqr(lam)
    e = f2_mul(lam, d)
    f = f2_mul(z, c)
    g = f2_mul(x, d)
    h = f2_sub(f2_add(e, f), f2_dbl(g))
    nr = (f2_mul(lam, h), f2_sub(f2_mul(theta, f2_sub(g, h)), f2_mul(e, y)), f2_mul(z, e))
    j = f2_sub(f2_mul(theta, qx), f2_mul(lam, qy))
    return nr, (lam, f2_neg(theta), j)


def g2_prepare(q):
    """G2Prepared::from_affine → (coefficient triples, infinity)"""
    if q is None:
        return [], True
    r = (q[0], q[1], F2_ONE)
    coeffs = []
    for bit in bin(X)[3:]:
        r, c = _doubling_step(r)
        coeffs.append(c)
        if bit == "1":
            r, c = _addition_step(r, q)
            coeffs.append(c)
    assert len(coeffs) == COEFF_TRIPLES
    return coeffs, False


# ---- Miller loop, final exponentiation ----
def _ell(f, c, p):
    return mul_by_034(f, f2_mul_fp(c[0], p[1]), f2_mul_fp(c[1], p[0]), c[2])


def miller_loop(pairs):
    """the reference's shared-squaring loop over [(G1 affine or None, prepared)]; pairs with infinity contribute nothing"""
    live = [(p, iter(q[0])) for p, q in pairs if p is not None and not q[1]]
    f = F12_ONE
    for bit in bin(X)[3:]:
        f = f12_sqr(f)
        for p, it in live:
            f = _ell(f, next(it), p)
        if bit == "1":
            for p, it in live:
                f = _ell(f, next(it), p)
    return f


def final_exponentiation(f):
    f1 = f12_conj(f)
    f2 = f12_inv(f)
    r = f12_mul(f1, f2)
    f2 = r
    r = f12_frob(r, 2)
    r = f12_mul(r, f2)
    y0 = f12_conj(cyclotomic_square(r))
    y5 = exp_by_x(r)
    y1 = cyclotomic_square(y5)
    y3 = f12_mul(y0, y5)
    y0 = exp_by_x(y3)
    y2 = exp_by_x(y0)
    y4 = f12_mul(exp_by_x(y2), y1)
    y1 = exp_by_x(y4)
    y3 = f12_conj(y3)
    y1 = f12_mul(f12_mul(y1, y3), r)
    y3 = f12_conj(r)
    y0 = f12_frob(f12_mul(y0, r), 3)
    y4 = f12_frob(f12_mul(y4, y3), 1)
    y5 = f12_frob(f12_mul(y5, y2), 2)
    return f12_mul(f12_mul(f12_mul(y5, y0), y4), y1)


def final_exponentiation_exponent() -> int:
    """the exponent λ with final_exponentiation(f) = g^λ, g = f^((q⁶ − 1)(q² + 1)), read off the formula above: a product adds
    exponents, conjugation negates them (g is in the cyclotomic subgroup), frobenius_map(k) multiplies by q^k, exp_by_x by X and a
    cyclotomic square by two"""
    r = 1
    y0 = -2 * r
    y5 = X * r
    y1 = 2 * y5
    y3 = y0 + y5
    y0 = X * y3
    y2 = X * y0
    y4 = X * y2 + y1
    y1 = X * y4
    y3 = -y3
    y1 = y1 + y3 + r
    y3 = -r
    y0 = (y0 + r) * Q ** 3
    y4 = (y4 + y3) * Q
    y5 = (y5 + y2) * Q ** 2
    return y5 + y0 + y4 + y1


def pairing(p, q):
    return final_exponentiation(miller_loop([(p, g2_prepare(q))]))


def product_of_pairings(pairs):
    """PairingEngine::product_of_pairings over [(G1 affine or None, G2 affine or None)]"""
    return final_exponentiation(miller_loop([(p, g2_prepare(q)) for p, q in pairs]))


# ---- byte images ----
def _fq(v: int) -> bytes: return fq_to_mont(v).to_bytes(48, "little")
def _f2(a) -> bytes: return _fq(a[0]) + _fq(a[1])


def gt_bytes(f) -> bytes:
    return b"".join(_f2(c) for c6 in f for c in c6)


def gt_from_bytes(b: bytes):
    v = [fq_from_mont(int.from_bytes(b[48 * i: 48 * i + 48], "little")) for i in range(12)]
    c = [(v[2 * i], v[2 * i + 1]) for i in range(6)]
    return ((c[0], c[1], c[2]), (c[3], c[4], c[5]))


def prepared_bytes(prep) -> bytes:
    coeffs, inf = prep
    body = b"".join(_f2(c) for t in coeffs for c in t) if not inf else b"\0" * (COEFF_TRIPLES * 288)
    return body + (1 if inf else 0).to_bytes(4, "little") + b"\0" * 28


def usrs_g2_point(blob: bytes):
    """a 192-byte uncompressed G2 point (x.c0, x.c1, y.c0, y.c1, 48 B LE each; bit 6 of the last byte = infinity, bit 7 = y's sign)
    → ((x0, x1), (y0, y1)) or None"""
    assert len(blob) == 192
    last = bytearray(blob)
    flags = last[191] & 0xC0
    last[191] &= 0x3F
    if flags & 0x40:
        return None
    v = [int.from_bytes(bytes(last[48 * i: 48 * i + 48]), "little") for i in range(4)]
    return ((v[0], v[1]), (v[2], v[3]))


__all__ = ["Q", "R_MOD", "X"]
