"""Big-integer restatement of the byte form of Varuna proving keys, for the tests: CircuitProvingKey ToBytes / FromBytes
(circuit_proving_key.rs:42-57) = the verifying key (compressed, as varuna_bytes_oracle writes it), the Circuit (CanonicalSerialize:
ahp/indexer/circuit.rs:158-237, ahp/matrices.rs:101-112, fft/evaluations.rs, fft/domain.rs:82-98) and the CommitterKey (ToBytes:
polycommit/sonic_pc/data_structures.rs:65-265, points as Affine ToBytes, affine.rs:293-313).  A ToBytes point is (x, y, infinity)
with canonical x, y: FromBytes keeps them as read.  Statuses follow include/snarkvm_b200.h."""
import hashlib
import struct

from oracle import bls12_377 as py
from varuna_bytes_oracle import (BAD_FLAGS, NOT_CANONICAL, NOT_IN_SUBGROUP, NOT_ON_CURVE, VALID, Q, R, Reader, in_subgroup,
                                 read_verifying_key, write_verifying_key)


FR_GENERATOR = 22                                                               # fr.rs: GENERATOR
DOMAIN_BYTES, VK_BYTES, POINT97 = 172, 8 * 7 + 12 * 48 + 32, 97


def domain_size(n: int) -> int:
    return 1 if n <= 1 else 1 << (n - 1).bit_length()


def domain_bytes(size: int) -> bytes:
    """EvaluationDomain::new(size) serialized: u64 size, u32 log size, size, 1/size, ω, 1/ω, 1/GENERATOR"""
    w = py.fr_root_of_unity(size)
    vals = (size % R, pow(size, -1, R), w, pow(w, -1, R), pow(FR_GENERATOR, -1, R))
    return struct.pack("<QI", size, size.bit_length() - 1) + b"".join(v.to_bytes(32, "little") for v in vals)


def encode_point97(p) -> bytes:
    x, y, inf = p
    return x.to_bytes(48, "little") + y.to_bytes(48, "little") + bytes([int(inf)])


def decode_point97(b: bytes, validate: bool):
    """→ (status, (x, y, infinity) or None): below q, an infinity byte of 0 or 1, `infinity != (x == 0) && y == 1` refused"""
    x, y, inf = int.from_bytes(b[:48], "little"), int.from_bytes(b[48:96], "little"), b[96]
    if x >= Q or y >= Q:
        return NOT_CANONICAL, None
    if inf > 1 or ((inf == 1) != (x == 0) and y == 1):
        return BAD_FLAGS, None
    if validate and not inf:
        if not py.g1_is_on_curve((x, y)):
            return NOT_ON_CURVE, (x, y, False)
        if not in_subgroup((x, y)):
            return NOT_IN_SUBGROUP, (x, y, False)
    return VALID, (x, y, bool(inf))


def proving_key_size(info, zk: bool = True, hiding_bound: int = 1) -> int:
    """the byte length of a proving key set up for CircuitInfo `info` (six counts): trimmed to AHPForR1CS::max_degree with the
    deduplicated degree bounds of g_1, g_a, g_b, g_c, no Lagrange bases"""
    npub, nvar, ncons, *nnz = info
    z = 1 if zk else 0
    r, v, k = domain_size(ncons), domain_size(nvar), domain_size(max(nnz))
    max_degree = max(2 * r + 2 * z - 2, 2 * v + 2 * z - 2, v + 3 if zk else 0, v, r, k - 1)
    bounds = sorted({domain_size(n) - 2 for n in [nvar] + nnz})
    circuit = 48 + sum(8 + 8 * ncons + 40 * n for n in nnz) + sum(3 * (8 + 32 * domain_size(n) + DOMAIN_BYTES) + 1 for n in nnz)
    g = hiding_bound + 2
    ck = (4 + POINT97 * (max_degree + 1) + 4 + 4 + POINT97 * g + 1 + 4 + POINT97 * (bounds[-1] + 1)
          + 1 + 4 + len(bounds) * (8 + POINT97 * g) + 1 + 4 + 4 * len(bounds) + 32)
    return VK_BYTES + circuit + ck


def write_committer_key(ck: dict) -> bytes:
    pts = lambda ps: b"".join(encode_point97(p) for p in ps)                    # noqa: E731
    out = [struct.pack("<I", len(ck["powers"])), pts(ck["powers"]), struct.pack("<I", len(ck["lagrange"]))]
    for size in sorted(ck["lagrange"]):
        out += [struct.pack("<I", size), pts(ck["lagrange"][size])]
    out += [struct.pack("<I", len(ck["gamma"])), pts(ck["gamma"])]
    out += [b"\x00"] if ck["shifted"] is None else [b"\x01", struct.pack("<I", len(ck["shifted"])), pts(ck["shifted"])]
    if ck["shifted_gamma"] is None:
        out.append(b"\x00")
    else:
        out += [b"\x01", struct.pack("<I", len(ck["shifted_gamma"]))]
        for b in sorted(ck["shifted_gamma"]):
            out += [struct.pack("<II", b, len(ck["shifted_gamma"][b])), pts(ck["shifted_gamma"][b])]
    out += [b"\x00"] if ck["bounds"] is None else [b"\x01", struct.pack(f"<I{len(ck['bounds'])}I", len(ck["bounds"]), *ck["bounds"])]
    h = hashlib.sha256(pts(ck["powers"]) + pts(ck["gamma"]) + (pts(ck["shifted"]) if ck["shifted"] is not None else b"")
                       + b"".join(pts(ck["shifted_gamma"][b]) for b in sorted(ck["shifted_gamma"] or {})))
    return b"".join(out) + h.digest()


def write_proving_key(pk: dict) -> bytes:
    """pk: {"vk": verifying key dict, "matrices": three lists of rows of (value, column), "arith": three dicts of "row", "col",
    "row_col_val" value lists, "ck": {"powers", "lagrange" {size: points}, "gamma", "shifted" or None, "shifted_gamma" {bound:
    points} or None, "bounds" or None}}"""
    fr = lambda vs: b"".join(v.to_bytes(32, "little") for v in vs)             # noqa: E731
    out = [write_verifying_key(pk["vk"]), struct.pack("<6Q", *pk["vk"]["info"])]
    for rows in pk["matrices"]:
        out.append(struct.pack("<Q", len(rows)))
        for row in rows:
            out.append(struct.pack("<Q", len(row)) + b"".join(v.to_bytes(32, "little") + struct.pack("<Q", c) for v, c in row))
    for a in pk["arith"]:
        for name in ("row", "col", "row_col", "row_col_val"):
            if name == "row_col":
                out.append(b"\x00")
                continue
            vs = a[name]
            out += [struct.pack("<Q", len(vs)), fr(vs), domain_bytes(len(vs))]
    return b"".join(out) + write_committer_key(pk["ck"])


class KeyReader(Reader):
    """a proving key walked as the reference reads it, plus the hash check; u32 counts for the committer key"""

    def u32(self) -> int:
        return struct.unpack("<I", self.take(4))[0]

    def point97(self):
        s, p = decode_point97(self.take(POINT97), self.v)
        if s != VALID:
            raise ValueError(f"point status {s}")
        return p

    def points(self, n: int) -> list:
        if n * POINT97 > len(self.b) - self.o:
            raise ValueError("truncated")
        return [self.point97() for _ in range(n)]


def read_committer_key(r: KeyReader) -> dict:
    ck = {"powers": r.points(r.u32()), "lagrange": {}}
    for _ in range(r.u32()):
        size = r.u32()
        ck["lagrange"][size] = r.points(size)
    ck["gamma"] = r.points(r.u32())
    ck["shifted"] = r.points(r.u32()) if r.tag() else None
    ck["shifted_gamma"] = None
    if r.tag():
        ck["shifted_gamma"] = {}
        for _ in range(r.u32()):
            b = r.u32()
            ck["shifted_gamma"][b] = r.points(r.u32())
    ck["bounds"] = [r.u32() for _ in range(r.u32())] if r.tag() else None
    want = write_committer_key(ck)[-32:]
    if r.take(32) != want:
        raise ValueError("Mismatching group elements")
    return ck


def read_proving_key(r: KeyReader) -> dict:
    saved, r.c = r.c, True
    vk = read_verifying_key(r)
    r.c = saved
    info = [r.u64() for _ in range(6)]
    matrices = []
    for _ in range(3):
        rows = []
        for _ in range(r.u64()):
            n = r.u64()
            if 40 * n > len(r.b) - r.o:
                raise ValueError("truncated")
            row = []
            for _ in range(n):
                v = r.fr()
                row.append((v, r.u64()))
            rows.append(row)
        matrices.append(rows)
    arith = []
    for _ in range(3):
        a = {}
        for name in ("row", "col", "row_col", "row_col_val"):
            if name == "row_col" and not r.tag():
                continue
            n = r.u64()
            if 32 * n > len(r.b) - r.o:
                raise ValueError("truncated")
            a[name] = [r.fr() for _ in range(n)]
            r.take(DOMAIN_BYTES)
        arith.append(a)
    return {"vk": vk, "info": info, "matrices": matrices, "arith": arith, "ck": read_committer_key(r)}
