"""Seeded big-integer corpora for the rare paths of the point readers' device functions (verify.cu): small-order G1 points for
g1_check, Fq and Fq2 values for every branch of fq_sqrt and fq2_sqrt, and G2 inputs for the real-right-hand-side decodes and g2_check.

    G1 torsion   E(Fq) has order h1·r, h1 = 2^92·3·7²·13²·499², and its cofactor torsion is (Z/2^46)² × Z/3 × (Z/7)² × (Z/13)² ×
                 (Z/499)²: points of exact order 2, 4, 8, 2^16, 2^45, 2^46, the three order-2 points (−1, 0), (−PHI, 0), (−PHI², 0),
                 both order-3 points (0, ±1), order 7 and 13 with one point on each of the ℓ + 1 lines of E[ℓ], order 499, and one
                 point of the torsion exponent 2^46·3·7·13·499; each made as [n1/d]·(random point) with its order checked.  Every
                 torsion point T comes with −T, φ(T), T + S (S in G1) and T with y moved off the curve.  Each entry carries its status
                 by the definition (Affine::check as [r]·P = O) and by the reference's formula [x²]·φ(P) + P = O, traced through the
                 device's XYZZ chain with its branches recorded.
    Fq roots     0, 1, q − 1 and values next to q; squares at every Tonelli–Shanks depth 0 … 45 (ω^(2^(46−k))·s², ω the 2-adic root
                 of unity, s of odd order); squares whose loop runs many rounds (ω^j·s², j even with many bits set); non-squares.
    Fq2 roots    a1 = 0 with a0 a square, a non-square and 0; a1 ≠ 0 as c² for a root c whose norm and c0² sit at chosen depths, so
                 that both arms of (a0 ± n)/2 run; non-squares (a non-square norm).
    G2           compressed x whose x³ + B' is real (3·x0² = 1/(5·x1) + 5·x1²), its real part a square or not; points T2 + S2 with
                 T2 = [r]·R2 (the G2 cofactor h2 is odd with no small factor, so G2 has no small-order points to build).

The square-root restatements follow verify.cu statement by statement, so they return the root the device returns."""
import functools
import math
import random

import g2_bytes_oracle as o2
import varuna_bytes_oracle as vb
from oracle import bls12_377 as py
from oracle import g2 as og2

Q, R = py.Q_MOD, py.R_MOD
VALID, NOT_ON_CURVE, NOT_IN_SUBGROUP = vb.VALID, vb.NOT_ON_CURVE, vb.NOT_IN_SUBGROUP
X = 0x8508C00000000001                                  # the BLS parameter
X2 = X * X
H1 = 2 ** 92 * 3 * 7 ** 2 * 13 ** 2 * 499 ** 2          # #E(Fq) / r
N1 = H1 * R
EXPONENT = 2 ** 46 * 3 * 7 * 13 * 499                   # the exponent of E(Fq)'s cofactor torsion
TWO_ADICITY, OMEGA = vb.TWO_ADICITY, vb.TWO_ADIC_ROOT
_T = (Q - 1) >> TWO_ADICITY
B1 = o2.B1                                              # G2's B' = (0, b1), b1 = −1/5


def _cube_roots_of_unity():
    w, _k = vb.sqrt(Q - 3)
    half = pow(2, -1, Q)
    return [(-1 + w) * half % Q, (-1 - w) * half % Q]


def _phi_formula(p, phi):
    return py.g1_add(py.g1_mul((phi * p[0] % Q, p[1]), X2), p)


# PHI of the reference: the primitive cube root of unity for which [x²]·φ(G) + G = O on the G1 generator
PHI = next(w for w in _cube_roots_of_unity() if _phi_formula(py.G1_GENERATOR, w) is None)


def phi(p):
    return None if p is None else (PHI * p[0] % Q, p[1])


# --------------------------------------------------------------------------------------------------------------------------------
# G1: the definition and the device's chain
# --------------------------------------------------------------------------------------------------------------------------------
def definition_status(p) -> int:
    """Affine::check by the definition: the curve, then [r]·P = O"""
    if p is None:
        return VALID
    if not py.g1_is_on_curve(p):
        return NOT_ON_CURVE
    return VALID if py.g1_mul(p, R) is None else NOT_IN_SUBGROUP


def _madd(acc, q, events: set, final: bool):
    """XyzzT::add_affine's branches on affine values: acc = O takes q, acc = q doubles, acc = −q cancels"""
    if acc is None:
        events.add("final from O" if final else "add to O")
        return q
    if acc[0] == q[0]:
        if acc[1] == q[1]:
            events.add("acc = P at the final addition" if final else "doubling branch")
            return py.g1_add(q, q)
        events.add("cancelling branch at the final addition" if final else "cancelling branch")
        return None
    return py.g1_add(acc, q)


def formula_trace(p):
    """g1_check's chain on an on-curve point p ≠ O: acc = φ(P), then per bit of x² below the leading one a doubling and, for a set
    bit, a mixed addition of φ(P); then a mixed addition of P → (status, the branches taken)"""
    q = phi(p)
    acc, events = q, set()
    for b in range(X2.bit_length() - 2, -1, -1):
        if acc is not None:
            acc = py.g1_add(acc, acc)
            if acc is None:
                events.add("O mid-chain")
        if (X2 >> b) & 1:
            acc = _madd(acc, q, events, False)
            if acc is None:
                events.add("O mid-chain")
    acc = _madd(acc, p, events, True)
    return (VALID if acc is None else NOT_IN_SUBGROUP), frozenset(events)


def formula_status(p) -> int:
    if p is None:
        return VALID
    if not py.g1_is_on_curve(p):
        return NOT_ON_CURVE
    return formula_trace(p)[0]


def _factor(d: int) -> list:
    return [p for p in (2, 3, 7, 13, 499) if d % p == 0]


def order(p, multiple: int) -> int:
    """the exact order of p, given a multiple of it whose primes are those of h1"""
    assert py.g1_mul(p, multiple) is None
    n = multiple
    for f in _factor(multiple):
        while n % f == 0 and py.g1_mul(p, n // f) is None:
            n //= f
    return n


def random_point(rng):
    while True:
        x = rng.randrange(Q)
        y, _k = vb.sqrt(x ** 3 + 1)
        if y is not None:
            return (x, y if rng.random() < 0.5 else (Q - y) % Q)


def _part(n: int, primes) -> int:
    """the part of n made of the given primes"""
    out = 1
    for f in primes:
        while n % f == 0:
            n, out = n // f, out * f
    return out


def torsion_point(rng, d: int):
    """[n1/d']·(random point) for d | EXPONENT, retried until its order is exactly d: d' is d times the part of h1 / EXPONENT on
    d's primes (the ℓ-torsion is (Z/ℓ^a)², so n1/ℓ^a alone would leave a factor ℓ^a of the component)"""
    primes = _factor(d)
    m = N1 // _part(H1, primes) * (_part(EXPONENT, primes) // d)
    while True:
        t = py.g1_mul(random_point(rng), m)
        if t is not None and order(t, d) == d:
            return t


def _subgroup_of(p, ell):
    return frozenset(x for x in (py.g1_mul(p, k) for k in range(1, ell)))


def lines(rng, ell: int) -> list:
    """one point on each of the ℓ + 1 lines (order-ℓ subgroups) of E[ℓ] ≅ (Z/ℓ)²: A, then B + [k]·A for k < ℓ"""
    a = torsion_point(rng, ell)
    span = _subgroup_of(a, ell)
    while True:
        b = torsion_point(rng, ell)
        if b not in span:
            break
    return [a] + [py.g1_add(b, py.g1_mul(a, k)) for k in range(ell)]


@functools.lru_cache(maxsize=None)
def g1_torsion(seed: int = 0x7045):
    """[(name, T, its order)]"""
    rng = random.Random(seed)
    out = []
    t46 = torsion_point(rng, 2 ** 46)
    for e in (1, 2, 3, 16, 45, 46):
        out.append((f"order 2^{e}", py.g1_mul(t46, 2 ** (46 - e)), 2 ** e))
    for k, x in enumerate((Q - 1, (-PHI) % Q, (-PHI * PHI) % Q)):
        out.append((f"order 2, x = −PHI^{k}", (x, 0), 2))
    out += [("order 3, y = 1", (0, 1), 3), ("order 3, y = −1", (0, Q - 1), 3)]
    for ell in (7, 13):
        out += [(f"order {ell}, line {k}", p, ell) for k, p in enumerate(lines(rng, ell))]
    out.append(("order 499", torsion_point(rng, 499), 499))
    out.append(("order 2^46·3·7·13·499", torsion_point(rng, EXPONENT), EXPONENT))
    return out


@functools.lru_cache(maxsize=None)
def g1_entries(seed: int = 0x7045):
    """[(name, point or None, definition status, formula status, branches of the formula's chain)]: every torsion point T with
    −T, φ(T), T + S and T off the curve; subgroup points and infinity as controls"""
    rng = random.Random(seed + 1)
    pts = [("infinity", None), ("G", py.G1_GENERATOR)]
    pts += [(f"S{k}", py.g1_mul(py.G1_GENERATOR, rng.randrange(1, R))) for k in range(3)]
    for name, t, _n in g1_torsion(seed):
        s = py.g1_mul(py.G1_GENERATOR, rng.randrange(1, R))
        pts += [(name, t), (f"−({name})", py.g1_neg(t)), (f"φ({name})", phi(t)), (f"{name} + S", py.g1_add(t, s)),
                (f"{name}, y + 1", (t[0], (t[1] + 1) % Q))]
    out = []
    for name, p in pts:
        events = formula_trace(p)[1] if p is not None and py.g1_is_on_curve(p) else frozenset()
        out.append((name, p, definition_status(p), formula_status(p), events))
    return out


# --------------------------------------------------------------------------------------------------------------------------------
# Fq: Tonelli–Shanks as fq_sqrt runs it
# --------------------------------------------------------------------------------------------------------------------------------
def fq_sqrt_trace(a: int):
    """fq_sqrt of verify.cu → (root or None, [k of each round]); k = 46 in the first round marks a non-square"""
    a %= Q
    if a == 0:
        return 0, []
    w = pow(a, (_T - 1) // 2, Q)
    x = a * w % Q
    b = x * w % Q
    z, v, ks = OMEGA, TWO_ADICITY, []
    while b != 1:
        k, b2k = 0, b
        while b2k != 1 and k < v:
            b2k, k = b2k * b2k % Q, k + 1
        ks.append(k)
        if k == v:
            return None, ks
        c = z
        for _ in range(v - k - 1):
            c = c * c % Q
        z = c * c % Q
        b, x, v = b * z % Q, x * c % Q, k
    return x, ks


def is_square(a: int) -> bool:
    """Euler's criterion"""
    return pow(a % Q, (Q - 1) // 2, Q) in (0, 1)


def _odd_order(rng) -> int:
    while True:
        s = pow(rng.randrange(1, Q), 1 << TWO_ADICITY, Q)
        if s != 1:
            return s


def at_depth(rng, k: int) -> int:
    """a square whose a^t has order 2^k (k ≤ 45): ω^(2^(46−k))·s², s of odd order"""
    return pow(OMEGA, 1 << (TWO_ADICITY - k), Q) * pow(_odd_order(rng), 2, Q) % Q


def _omega_j(rng, j: int) -> int:
    return pow(OMEGA, j, Q) * pow(_odd_order(rng), 2, Q) % Q


# j even with many bits set: every bit 1 … 45, every odd bit, every even bit from 2, and random even j
MANY_ROUNDS_J = [(1 << 46) - 2, sum(1 << i for i in range(1, 46, 2)), sum(1 << i for i in range(2, 46, 2))]
NON_SQUARE_J = [1, 3, (1 << 46) - 1, (1 << 45) + 1, 0x2AAAAAAAAAAB]


@functools.lru_cache(maxsize=None)
def fq_values(seed: int = 0x5A):
    rng = random.Random(seed)
    vals = [0, 1, Q - 1, 2, 3, 5]
    vals += [Q - k for k in range(2, 9)]
    for k in range(TWO_ADICITY):
        vals += [at_depth(rng, k) for _ in range(2)]
    vals += [_omega_j(rng, j) for j in MANY_ROUNDS_J]
    vals += [_omega_j(rng, 2 * rng.randrange(1 << 44) | sum(1 << i for i in range(1, 46, 3))) for _ in range(6)]
    vals += [_omega_j(rng, j) for j in NON_SQUARE_J]
    vals += [rng.randrange(Q) for _ in range(16)]
    return vals


# --------------------------------------------------------------------------------------------------------------------------------
# Fq2 = Fq[u]/(u² + 5): fq2_sqrt as verify.cu runs it
# --------------------------------------------------------------------------------------------------------------------------------
def fq2_sqrt_trace(a):
    """fq2_sqrt of verify.cu → (root or None, branch): "a1 = 0, real" (√a0), "a1 = 0, imaginary" (√(a0·b1)·u), "(a0 + n)/2" or
    "(a0 − n)/2" (the arm whose t was a square), or "no norm root" / "no t root" when it returns false"""
    a0, a1 = a[0] % Q, a[1] % Q
    if a1 == 0:
        r, _ks = fq_sqrt_trace(a0)
        if r is not None:
            return (r, 0), "a1 = 0, real"
        r, _ks = fq_sqrt_trace(a0 * B1)
        return (None, "no root") if r is None else ((0, r), "a1 = 0, imaginary")
    n, _ks = fq_sqrt_trace(a0 * a0 + 5 * a1 * a1)
    if n is None:
        return None, "no norm root"
    half = pow(2, -1, Q)
    for arm, t in (("(a0 + n)/2", (a0 + n) * half), ("(a0 − n)/2", (a0 - n) * half)):
        c0, _ks = fq_sqrt_trace(t)
        if c0 is not None:
            return (c0, a1 * pow(2 * c0, -1, Q) % Q), arm
    return None, "no t root"


def norm(a) -> int:
    return (a[0] * a[0] + 5 * a[1] * a[1]) % Q


def fq2_is_square(a) -> bool:
    """a is a square in Fq2 iff its norm is one in Fq"""
    return is_square(norm(a))


def _from_root(rng, kt: int, kn: int):
    """c² for c = c0 + c1·u with c0² at Tonelli–Shanks depth kt and the norm N(c) = c0² + 5·c1² chosen so that N(c)² = a0² + 5·a1²
    sits at depth kn (N(c) = ω^(2^(45−kn))·s; c1² = (N − c0²)/5 must be a non-zero square)"""
    c0 = pow(OMEGA, 1 << (TWO_ADICITY - 1 - kt), Q) * _odd_order(rng) % Q
    while True:
        n = pow(OMEGA, 1 << (TWO_ADICITY - 1 - kn), Q) * _odd_order(rng) % Q
        c1, _ks = fq_sqrt_trace((n - c0 * c0) * pow(5, -1, Q))
        if c1:
            break
    c = (c0, c1 if rng.random() < 0.5 else Q - c1)
    return og2.f2_sqr(c)


DEPTH_PAIRS = [(kt, kn) for kt in (0, 1, 2, 7, 19, 45) for kn in (0, 1, 2, 3, 5, 8, 13, 21, 34, 45)]


@functools.lru_cache(maxsize=None)
def fq2_values(seed: int = 0x5B):
    rng = random.Random(seed)
    vals = [(0, 0), (1, 0), (Q - 1, 0), (5, 0), (Q - 5, 0)]
    vals += [(at_depth(rng, k), 0) for k in (0, 1, 2, 9, 30, 45)]                          # a1 = 0, a0 a square
    vals += [(_omega_j(rng, j), 0) for j in NON_SQUARE_J]                                  # a1 = 0, a0 a non-square
    vals += [_from_root(rng, kt, kn) for kt, kn in DEPTH_PAIRS]
    vals += [(0, rng.randrange(1, Q)) for _ in range(3)]                                   # norm 5·a1²: a non-square
    while sum(not fq2_is_square(v) for v in vals) < 16:
        v = (rng.randrange(Q), rng.randrange(Q))
        if not fq2_is_square(v):
            vals.append(v)
    vals += [(rng.randrange(Q), rng.randrange(Q)) for _ in range(16)]
    return vals


# --------------------------------------------------------------------------------------------------------------------------------
# G2
# --------------------------------------------------------------------------------------------------------------------------------
def _h2() -> int:
    """#E'(Fq2)/r: of the six sextic-twist orders q² + 1 − T (T = ±t2, (±t2 ± 3f)/2, t2 = t² − 2q, t = x + 1 the trace over Fq,
    t2² − 4q² = −3f²) the one r divides and E(Fq2)'s own order q² + 1 − t2 is not"""
    t2 = (X + 1) ** 2 - 2 * Q
    f = math.isqrt((4 * Q * Q - t2 * t2) // 3)
    assert 3 * f * f == 4 * Q * Q - t2 * t2
    orders = [Q * Q + 1 - T for T in (-t2, (t2 + 3 * f) // 2, (t2 - 3 * f) // 2, (-t2 + 3 * f) // 2, (-t2 - 3 * f) // 2)]
    (n,) = [n for n in orders if n % R == 0]
    return n // R


H2 = _h2()


def g2_mul_raw(p, k: int):
    """[k]·P by double-and-add over k's bits, the scalar not reduced mod r"""
    acc = og2.J_INF
    for bit in bin(k)[2:]:
        acc = og2._jdbl(acc)
        if bit == "1":
            acc = og2._jadd_affine(acc, p)
    return og2._jaff(acc)


def g2_random_point(rng):
    while True:
        x = (rng.randrange(Q), rng.randrange(Q))
        y = o2.fq2_sqrt(o2.rhs(x))
        if y is not None:
            return (x, y)


@functools.lru_cache(maxsize=None)
def g2_real_rhs_x(seed: int = 0x62, each: int = 12):
    """[(x, real part of x³ + B')]: `each` x whose x³ + B' is real with a square real part and `each` with a non-square one.  The
    u-part 3·x0²·x1 − 5·x1³ + b1 vanishes iff 3·x0² = 1/(5·x1) + 5·x1²"""
    rng = random.Random(seed)
    sq, non = [], []
    inv3 = pow(3, -1, Q)
    while len(sq) < each or len(non) < each:
        x1 = rng.randrange(1, Q)
        x0, _ks = fq_sqrt_trace((pow(5 * x1, -1, Q) + 5 * x1 * x1) * inv3)
        if x0 is None:
            continue
        x = (x0 if rng.random() < 0.5 else (Q - x0) % Q, x1)
        a = o2.rhs(x)
        assert a[1] == 0
        (sq if is_square(a[0]) else non).append((x, a[0]))
    return sq[:each] + non[:each]


@functools.lru_cache(maxsize=None)
def g2_mixed_points(seed: int = 0x63, count: int = 3):
    """[(name, point)]: T2 = [r]·R2 for random R2 on E'(Fq2) (of order dividing h2), T2 + S2 and −(T2 + S2) with S2 in G2"""
    rng = random.Random(seed)
    out = []
    for k in range(count):
        t2 = g2_mul_raw(g2_random_point(rng), R)
        s2 = og2.g2_mul(o2.G2_GEN, rng.randrange(1, R))
        ts = og2.g2_add(t2, s2)
        out += [(f"T2_{k}", t2), (f"T2_{k} + S2", ts), (f"−(T2_{k} + S2)", og2.g2_neg(ts))]
    return out
