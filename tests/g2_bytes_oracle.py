"""Big-integer restatement of the byte forms and validation of G2 points, and of kzg10::VerifierKey's byte form, for the tests.

    Affine<G2>   curves/src/templates/macros.rs:67-144 (CanonicalSerialize / CanonicalDeserialize), Fp2 with flags of
                 fields/src/fp2.rs:427-457 (c0 without flags, then c1 with them), SWFlags of utilities/src/serialize/flags.rs
    order on Fp2 fields/src/fp2.rs:241-250: c1 is compared first, then c0
    check        Valid for Affine<G2>: is_on_curve and [r]·P = O (curves/src/bls12_377/g2.rs:120-124), by the definition
    VerifierKey  algorithms/src/polycommit/kzg10/data_structures.rs:200-232: g, γ·G, h, β·h

A point is ((x0, x1), (y0, y1)) of canonical integers, or None for infinity.  Statuses follow include/snarkvm_b200.h (the G1 values,
shared by both groups)."""
from oracle import g2 as og2
from oracle.bls12_377 import Q_MOD as Q, R_MOD as R

import varuna_bytes_oracle as vb

VALID, NOT_CANONICAL, NOT_ON_CURVE, NOT_IN_SUBGROUP, BAD_FLAGS = vb.VALID, vb.NOT_CANONICAL, vb.NOT_ON_CURVE, vb.NOT_IN_SUBGROUP, vb.BAD_FLAGS
POSITIVE_Y, INFINITY = vb.POSITIVE_Y, vb.INFINITY
B1 = og2.G2_B[1]
assert B1 == (-pow(5, -1, Q)) % Q
G2_GEN = og2.G2_GEN


def rhs(x):
    """x³ + B'"""
    return og2.f2_add(og2.f2_mul(og2.f2_sqr(x), x), og2.G2_B)


def fq2_sqrt(a):
    """a square root of a in Fq2 = Fq[u]/(u² + 5), or None: a is a square iff a0² + 5·a1² is one in Fq; with a1 ≠ 0 exactly one
    of t = (a0 ± √(a0² + 5·a1²))/2 is a square, and (√t + a1/(2√t)·u)² = a; with a1 = 0 the root is √a0 or √(−a0/5)·u"""
    a0, a1 = a[0] % Q, a[1] % Q
    if a1 == 0:
        r, _k = vb.sqrt(a0)
        if r is not None:
            return (r, 0)
        r, _k = vb.sqrt(a0 * B1)
        return None if r is None else (0, r)
    n, _k = vb.sqrt(a0 * a0 + 5 * a1 * a1)
    if n is None:
        return None
    half = pow(2, -1, Q)
    for t in ((a0 + n) * half, (a0 - n) * half):
        c0, _k = vb.sqrt(t)
        if c0 is not None:
            return (c0, a1 * pow(2 * c0, -1, Q) % Q)
    return None


def greater(a, b) -> bool:
    """a > b in the reference's order on Fp2"""
    return (a[1], a[0]) > (b[1], b[0])


def mul_by_r(p):
    """[r]·P by double-and-add over r's bits, without reducing the scalar mod r (oracle.g2.g2_mul does)"""
    acc = og2.J_INF
    for bit in bin(R)[2:]:
        acc = og2._jdbl(acc)
        if bit == "1":
            acc = og2._jadd_affine(acc, p)
    return og2._jaff(acc)


def check(p) -> int:
    """Valid for Affine<G2> of a decoded point; coordinates are canonical here"""
    if p is None:
        return VALID
    if not og2.g2_is_on_curve(p):
        return NOT_ON_CURVE
    return VALID if mul_by_r(p) is None else NOT_IN_SUBGROUP


def decode(b: bytes, compressed: bool, validate: bool):
    """→ (status, point or None); a point only when the bytes decode to one"""
    ncoords = 2 if compressed else 4
    assert len(b) == 48 * ncoords
    flags = b[-1] & 0xC0
    c = []
    for k in range(ncoords):
        raw = bytearray(b[48 * k: 48 * k + 48])
        last = k == ncoords - 1
        if (flags == 0xC0) if last else (raw[47] & 0x80):
            return BAD_FLAGS, None
        if last:
            raw[47] &= 0x3F
        v = int.from_bytes(raw, "little")
        if v >= Q:
            return NOT_CANONICAL, None
        c.append(v)
    if flags == INFINITY:
        return VALID, None
    x = (c[0], c[1])
    if compressed:
        y = fq2_sqrt(rhs(x))
        if y is None:
            return NOT_ON_CURVE, None
        neg = og2.f2_neg(y)
        y = neg if greater(y, neg) != (flags == POSITIVE_Y) else y
        p = (x, y)
    else:
        p = (x, (c[2], c[3]))
    return (check(p) if validate else VALID), p


def image(b: bytes, compressed: bool, validate: bool) -> tuple:
    """→ (status, the 200-byte Affine<G2> image device.g2_deserialize writes): the decoded point's (infinity: Affine::zero()),
    all zero bytes when the bytes decode to no point"""
    s, p = decode(b, compressed, validate)
    return s, og2.g2_affine_bytes(p) if p is not None or s == VALID else bytes(200)


def encode(p, compressed: bool) -> bytes:
    if p is None:
        x, y, flags = (0, 0), (1, 0), INFINITY
    else:
        x, y = p
        flags = POSITIVE_Y if compressed and greater(y, og2.f2_neg(y)) else 0
    coords = [x[0], x[1]] if compressed else [x[0], x[1], y[0], y[1]]
    out = bytearray(b"".join(v.to_bytes(48, "little") for v in coords))
    out[-1] |= flags
    return bytes(out)


def verifier_key_bytes(g, gamma_g, h, beta_h, compressed: bool = True) -> bytes:
    """CanonicalSerialize of kzg10::VerifierKey: g, γ·G (G1, varuna_bytes_oracle.encode_g1), h, β·h"""
    return vb.encode_g1(g, compressed) + vb.encode_g1(gamma_g, compressed) + encode(h, compressed) + encode(beta_h, compressed)
