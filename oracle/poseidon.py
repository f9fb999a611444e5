"""TEST INFRASTRUCTURE ONLY — CPU restatement (Python big integers) of snarkVM's Poseidon duplex sponge and of the transcript of a
verifying-key certificate.

    algorithms/src/crypto_hash/poseidon.rs:120-208      PoseidonSponge<F, RATE, 1>: AlgebraicSponge     → Sponge
    algorithms/src/crypto_hash/poseidon.rs:211-255      apply_ark / apply_s_box / apply_mds / permute   → Sponge.permute
    algorithms/src/crypto_hash/poseidon.rs:258-333      absorb_internal / squeeze_internal              → Sponge._absorb_internal / _squeeze_internal
    algorithms/src/crypto_hash/poseidon.rs:436-492      get_bits / get_fe                               → Sponge.get_bits / get_fe
    algorithms/src/traits/algebraic_sponge.rs:47-68     absorb_bytes                                    → Sponge.absorb_bytes
    algorithms/src/snark/varuna/varuna.rs:155-165       init_sponge_for_certificate                     → certificate_elements
    algorithms/src/snark/varuna/varuna.rs:248, 293      squeeze_nonnative_field_elements(12)            → certificate_challenges
    algorithms/src/polycommit/sonic_pc/mod.rs:277, 329  prover: combine_for_open's challenge, then `_randomizer`
    algorithms/src/polycommit/sonic_pc/mod.rs:602, 405  verifier: accumulate_elems' curr_challenge, then the next randomizer

Values are canonical integers (not Montgomery).  The parameters (ark, mds, α, round counts) are an argument: the tests build them
with snarkvm_b200/poseidon.py, whose generator is pinned to the reference's own snapshots.  This module shares no code with the
device path.
"""
from __future__ import annotations

RATE = 2
SHORT_BITS = 168
FR_MOD = 8444461749428370424248824938781546531375899335154063827935233455917409239041
FR_BITS = 253

# VarunaSNARK::PROTOCOL_NAME (varuna.rs:68).  init_sponge_for_certificate absorbs `to_bytes_le![&Self::PROTOCOL_NAME]`: the macro
# (utilities/src/bytes.rs:35-52) calls ToBytes::write_le on `&&[u8]`, which is `impl ToBytes for &T` (bytes.rs:452-457) around
# `impl ToBytes for &[T]` (bytes.rs:442-450): every byte written in turn, no length prefix.  So the certificate absorbs the same
# eleven raw bytes as init_sponge (varuna.rs:142).
PROTOCOL_NAME = b"VARUNA-2023"


class Sponge:
    """PoseidonSponge<F, RATE, 1> over the prime `modulus` of `bits` bits (F::size_in_bits()).  `mode` is ("absorbing", i) or
    ("squeezing", i) like DuplexSpongeMode; state[0] is the capacity element, state[1:] the rate."""

    def __init__(self, modulus: int, bits: int, params: tuple, rate: int = RATE):
        self.p, self.bits, self.rate = modulus, bits, rate
        self.alpha, self.full_rounds, self.partial_rounds, self.ark, self.mds = params
        self.state = [0] * (rate + 1)
        self.mode = ("absorbing", 0)
        self.permutations = 0

    # ---- the permutation (poseidon.rs:211-255) ----
    def permute(self):
        p = self.p
        half = self.full_rounds // 2
        for i in range(self.full_rounds + self.partial_rounds):
            s = [(x + k) % p for x, k in zip(self.state, self.ark[i])]
            if half <= i < half + self.partial_rounds:
                s[0] = pow(s[0], self.alpha, p)
            else:
                s = [pow(x, self.alpha, p) for x in s]
            self.state = [sum(a * b for a, b in zip(s, row)) % p for row in self.mds]
        self.permutations += 1

    # ---- absorb_internal / squeeze_internal (poseidon.rs:258-333) ----
    def _absorb_internal(self, rate_start: int, elements: list):
        chunks = [elements[: self.rate - rate_start]]
        rest = elements[self.rate - rate_start:]
        chunks += [rest[i: i + self.rate] for i in range(0, len(rest), self.rate)]
        for i, chunk in enumerate(chunks):
            for j, e in enumerate(chunk):
                self.state[1 + rate_start + j] = (self.state[1 + rate_start + j] + e) % self.p
            if i == len(chunks) - 1:
                self.mode = ("absorbing", rate_start + len(chunk))
                return
            self.permute()
            rate_start = 0

    def _squeeze_internal(self, rate_start: int, count: int) -> list:
        out = []
        sizes = [min(self.rate - rate_start, count)]
        rest = count - sizes[0]
        sizes += [min(self.rate, rest - i) for i in range(0, rest, self.rate)]
        for i, size in enumerate(sizes):
            out += self.state[1 + rate_start: 1 + rate_start + size]
            if i == len(sizes) - 1:
                self.mode = ("squeezing", rate_start + size)
                return out
            self.permute()
            rate_start = 0
        return out

    # ---- AlgebraicSponge (poseidon.rs:148-208) ----
    def absorb_native_field_elements(self, elements):
        elements = [int(e) for e in elements]
        if any(not 0 <= e < self.p for e in elements):
            raise ValueError("an absorbed element is not below the modulus")
        if not elements:
            return
        kind, index = self.mode
        if kind == "absorbing":
            if index == self.rate:
                self.permute()
                index = 0
            self._absorb_internal(index, elements)
        else:
            self.permute()
            self._absorb_internal(0, elements)

    def squeeze_native_field_elements(self, count: int) -> list:
        if count == 0:
            return []
        kind, index = self.mode
        if kind == "absorbing":
            self.permute()
            return self._squeeze_internal(0, count)
        if index == self.rate:
            self.permute()
            index = 0
        return self._squeeze_internal(index, count)

    def absorb_bytes(self, data: bytes):
        """algebraic_sponge.rs:47-68, bit by bit: each byte most significant bit first, chunks of size_in_bits − 1 bits, each chunk
        read as a big-endian integer (BigInteger::from_bits_be, utilities/src/biginteger/bigint_384.rs:265-276)"""
        cap = self.bits - 1
        bits = [(byte >> (7 - k)) & 1 for byte in data for k in range(8)]
        elements = []
        for i in range(0, len(bits), cap):
            v = 0
            for b in bits[i: i + cap]:
                v = (v << 1) | b
            elements.append(v)
        self.absorb_native_field_elements(elements)

    # ---- get_bits / get_fe (poseidon.rs:436-492) ----
    def get_bits(self, num_bits: int) -> list:
        """each squeezed element's canonical big-endian bits after the top REPR_SHAVE_BITS + 1: its low size_in_bits − 1 bits"""
        per = self.bits - 1
        out = []
        for e in self.squeeze_native_field_elements(-(-num_bits // per)):
            out += [(e >> (per - 1 - k)) & 1 for k in range(per)]
        return out[:num_bits]

    def get_fe(self, count: int, short: bool) -> list:
        width = SHORT_BITS if short else FR_BITS - 1
        bits = self.get_bits(width * count)
        out = []
        for i in range(count):
            v = 0
            for k, b in enumerate(reversed(bits[i * width: (i + 1) * width])):
                if b:
                    v = (v + (1 << k)) % FR_MOD
            out.append(v)
        return out

    def squeeze_nonnative_field_elements(self, count: int) -> list:
        return self.get_fe(count, False)

    def squeeze_short_nonnative_field_elements(self, count: int) -> list:
        return self.get_fe(count, True)


def affine_field_elements(point) -> list:
    """SWAffine::to_field_elements (curves/src/templates/to_field_vec.rs:52-64): x, y, then the infinity flag as 0 / 1
    (fields/src/to_field_vec.rs:26-30).  `point` is (x, y) of canonical integers, or None for the point at infinity, whose
    reference image is (0, 1, true) (short_weierstrass_jacobian/affine.rs:57-59)."""
    if point is None:
        return [0, 1, 1]
    return [point[0], point[1], 0]


def certificate_sponge(modulus: int, bits: int, params: tuple, circuit_info_bytes: bytes, commitments: list, circuit_id: bytes) -> Sponge:
    """init_sponge_for_certificate (varuna.rs:155-165): the protocol name, CircuitInfo::to_bytes_le, the twelve commitments as
    field elements (KZGCommitment → its G1Affine, kzg10/data_structures.rs:305-309), the id bytes"""
    s = Sponge(modulus, bits, params)
    s.absorb_bytes(PROTOCOL_NAME)
    s.absorb_bytes(circuit_info_bytes)
    s.absorb_native_field_elements([e for c in commitments for e in affine_field_elements(c)])
    s.absorb_bytes(circuit_id)
    return s


def certificate_challenges(sponge: Sponge, num_commitments: int = 12) -> tuple:
    """after init_sponge_for_certificate: the num_commitments nonnative challenges (varuna.rs:248, 293), then the two short squeezes
    of the opening — ξ (combine_for_open's challenge / accumulate_elems' curr_challenge) and the randomizer (batch_open's
    `_randomizer` / batch_check's next randomizer)"""
    challenges = sponge.squeeze_nonnative_field_elements(num_commitments)
    xi = sponge.squeeze_short_nonnative_field_elements(1)[0]
    randomizer = sponge.squeeze_short_nonnative_field_elements(1)[0]
    return challenges, (xi, randomizer)
