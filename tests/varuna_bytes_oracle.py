"""Big-integer restatement of the byte forms of G1 points, Varuna proofs, verifying keys and certificates, for the tests.

    G1 points   curves/src/templates/macros.rs:67-144 (Affine<P> CanonicalSerialize / CanonicalDeserialize), SWFlags of
                utilities/src/serialize/flags.rs, from_x_coordinate of short_weierstrass_jacobian/affine.rs:140-150
    Proof       snark/varuna/data_structures/proof.rs:305-368
    VK          circuit_verifying_key.rs (derived): CircuitInfo (six u64), Vec<Commitment> (u64 length), the 32-byte id
    Certificate certificate.rs (derived): BatchLCProof, a Vec<KZGProof> of (w, Option<Fr> random_v)

A point is (x, y) of canonical integers, or None for infinity.  Statuses follow include/snarkvm_b200.h."""
import json
import os
import struct

from oracle import bls12_377 as py

Q, R = py.Q_MOD, py.R_MOD
VALID, NOT_CANONICAL, NOT_ON_CURVE, NOT_IN_SUBGROUP, BAD_FLAGS = 0, 1, 2, 3, 4
POSITIVE_Y, INFINITY = 0x80, 0x40

with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_constants.json")) as _f:
    _FQ = json.load(_f)["fq"]
TWO_ADICITY = _FQ["TWO_ADICITY"]
_T = (Q - 1) >> TWO_ADICITY
# TWO_ADIC_ROOT_OF_UNITY is stored as Montgomery limbs
TWO_ADIC_ROOT = py.fq_from_mont(sum(v << (64 * i) for i, v in enumerate(_FQ["TWO_ADIC_ROOT_OF_UNITY"])))
assert pow(TWO_ADIC_ROOT, 1 << (TWO_ADICITY - 1), Q) == Q - 1


def sqrt(a: int):
    """Tonelli–Shanks over Fq → (a root or None, k of the first round: the order of a^t is 2^k)"""
    a %= Q
    if a == 0:
        return 0, 0
    x, b, z, v = pow(a, (_T + 1) // 2, Q), pow(a, _T, Q), TWO_ADIC_ROOT, TWO_ADICITY
    first = None
    while b != 1:
        k, b2k = 0, b
        while b2k != 1 and k < v:
            b2k, k = b2k * b2k % Q, k + 1
        first = k if first is None else first
        if k == v:
            return None, first
        c = pow(z, 1 << (v - k - 1), Q)
        z, v = c * c % Q, k
        b, x = b * z % Q, x * c % Q
    return x, first or 0


def in_subgroup(p) -> bool:
    return p is None or py.g1_mul(p, R) is None


def decode_g1(b: bytes, compressed: bool, validate: bool):
    """→ (status, point or None); a point only when the bytes decode to one"""
    b = bytearray(b)
    if compressed:
        flags = b[47] & 0xC0
        b[47] &= 0x3F
        x = int.from_bytes(b, "little")
        if flags == 0xC0:
            return BAD_FLAGS, None
        if x >= Q:
            return NOT_CANONICAL, None
        if flags == INFINITY:
            return VALID, None
        y, _k = sqrt(x * x * x + 1)
        if y is None:
            return NOT_ON_CURVE, None
        neg = (Q - y) % Q
        y = y if (y < neg) ^ (flags == POSITIVE_Y) else neg
        p = (x, y)
    else:
        if b[47] & 0x80:
            return BAD_FLAGS, None
        x = int.from_bytes(b[:48], "little")
        if x >= Q:
            return NOT_CANONICAL, None
        flags = b[95] & 0xC0
        if flags == 0xC0:
            return BAD_FLAGS, None
        b[95] &= 0x3F
        y = int.from_bytes(b[48:], "little")
        if y >= Q:
            return NOT_CANONICAL, None
        if flags == INFINITY:
            return VALID, None
        p = (x, y)
        if validate and not py.g1_is_on_curve(p):
            return NOT_ON_CURVE, p
    if validate and not in_subgroup(p):
        return NOT_IN_SUBGROUP, p
    return VALID, p


def image(b: bytes, compressed: bool, validate: bool) -> tuple:
    """→ (status, the 104-byte Affine image device.g1_deserialize writes): the decoded point's (infinity: Affine::zero()), all
    zero bytes when the bytes decode to no point"""
    s, p = decode_g1(b, compressed, validate)
    return s, py.affine_bytes(p) if p is not None or s == VALID else bytes(104)


def encode_g1(p, compressed: bool) -> bytes:
    if p is None:
        x, y, flags = 0, 1, INFINITY
    else:
        x, y = p
        flags = POSITIVE_Y if compressed and y > (Q - y) % Q else 0
    if compressed:
        out = bytearray(x.to_bytes(48, "little"))
    else:
        out = bytearray(x.to_bytes(48, "little") + y.to_bytes(48, "little"))
    out[-1] |= flags
    return bytes(out)


class Reader:
    """a blob walked as the reference reads it: every failure raises ValueError"""

    def __init__(self, blob: bytes, offset: int, compressed: bool, validate: bool = False):
        self.b, self.o, self.c, self.v = blob, offset, compressed, validate

    def take(self, n: int) -> bytes:
        if self.o + n > len(self.b):
            raise ValueError("truncated")
        self.o += n
        return self.b[self.o - n: self.o]

    def u64(self) -> int:
        return struct.unpack("<Q", self.take(8))[0]

    def tag(self) -> bool:
        t = self.take(1)[0]
        if t > 1:
            raise ValueError("bad option tag")
        return t == 1

    def fr(self) -> int:
        v = int.from_bytes(self.take(32), "little")
        if v >= R:
            raise ValueError("Fr not below r")
        return v

    def point(self):
        s, p = decode_g1(self.take(48 if self.c else 96), self.c, self.v)
        if s != VALID:
            raise ValueError(f"point status {s}")
        return p

    def batch_lc(self) -> list:
        return [(self.point(), self.fr() if self.tag() else None) for _ in range(self.u64())]


def read_proof(r: Reader) -> dict:
    K = r.u64()
    if 8 * K > len(r.b) - r.o:
        raise ValueError("truncated")
    sizes = [r.u64() for _ in range(K)]
    if sum(sizes) * 48 > len(r.b):
        raise ValueError("truncated")
    p = {"batch_sizes": sizes, "w": [r.point() for _ in range(sum(sizes))]}
    p["mask_poly"] = r.point() if r.tag() else None
    for n in ("h_0", "g_1", "h_1"):
        p[n] = r.point()
    for m in "abc":
        p[f"g_{m}"] = [r.point() for _ in range(K)]
    p["h_2"] = r.point()
    p["g_1_eval"] = r.fr()
    for m in "abc":
        p[f"g_{m}_evals"] = [r.fr() for _ in range(K)]
    p["third_sums"] = [[[r.fr() for _ in range(3)] for _ in range(b)] for b in sizes]
    p["fourth_sums"] = [[r.fr() for _ in range(3)] for _ in range(K)]
    p["pc_proof"] = r.batch_lc()
    return p


def write_proof(p: dict, compressed: bool = True) -> bytes:
    g = lambda pt: encode_g1(pt, compressed)                                    # noqa: E731
    fr = lambda v: v.to_bytes(32, "little")                                     # noqa: E731
    out = [struct.pack(f"<{1 + len(p['batch_sizes'])}Q", len(p["batch_sizes"]), *p["batch_sizes"])]
    out += [g(w) for w in p["w"]]
    out += [b"\x00"] if p["mask_poly"] is None else [b"\x01", g(p["mask_poly"])]
    out += [g(p[n]) for n in ("h_0", "g_1", "h_1")]
    out += [g(x) for m in "abc" for x in p[f"g_{m}"]] + [g(p["h_2"]), fr(p["g_1_eval"])]
    out += [fr(v) for m in "abc" for v in p[f"g_{m}_evals"]]
    out += [fr(v) for sums in p["third_sums"] for t in sums for v in t] + [fr(v) for t in p["fourth_sums"] for v in t]
    return b"".join(out) + write_batch_lc(p["pc_proof"], compressed)


def write_batch_lc(pc: list, compressed: bool = True) -> bytes:
    out = [struct.pack("<Q", len(pc))]
    for w, v in pc:
        out += [encode_g1(w, compressed)] + ([b"\x00"] if v is None else [b"\x01", v.to_bytes(32, "little")])
    return b"".join(out)


def read_verifying_key(r: Reader) -> dict:
    info = [r.u64() for _ in range(6)]
    n = r.u64()
    if n != 12:
        raise ValueError("not twelve commitments")
    return {"info": info, "commitments": [r.point() for _ in range(n)], "id": r.take(32)}


def write_verifying_key(vk: dict, compressed: bool = True) -> bytes:
    return (struct.pack("<7Q", *vk["info"], len(vk["commitments"])) + b"".join(encode_g1(p, compressed) for p in vk["commitments"])
            + vk["id"])
