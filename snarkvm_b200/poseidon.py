"""Poseidon parameters of PoseidonSponge<F, RATE, 1> and the host side of the device sponge (csrc/poseidon.cu).

The parameters are snarkVM's `default_poseidon_parameters` (fields/src/traits/poseidon_default.rs:42-110): a Grain LFSR
(fields/src/traits/poseidon_grain_lfsr.rs) seeded with the field's bit size, the state width, the full and partial round counts
gives the additive round keys by rejection sampling, then two vectors x, y reduced mod p, and the MDS matrix is the Cauchy
matrix 1 / (x_i + y_j).  The round counts come from the `PoseidonDefaultParametersEntry` tables of curves/src/bls12_377/fr.rs:196-204
and fq.rs:180-188.  Snarkvm's Fiat–Shamir sponge is PoseidonSponge<Fq, 2, 1> (console/network/src/lib.rs:65): α = 17, 8 full and
31 partial rounds.  The reference pins only Fr's parameters; tests/test_poseidon_oracle.py checks this generator against them,
which is what pins Fq's too.

Everything here is host work: parameters are computed once per process and uploaded once per device; `bytes_to_field_elements`,
`nonnative_field_elements` and the Montgomery conversions are the O(|input|) encodings a caller does before a
`device.poseidon_transcripts` call; `fresh_states` makes the state records a resumable transcript starts from.
"""
from __future__ import annotations

import functools

import numpy as np
import torch

R_MOD = 8444461749428370424248824938781546531375899335154063827935233455917409239041   # curves/src/bls12_377/fr.rs
Q_MOD = 258664426012969094010652733694893533536393512754914660539884262666720468348340822774968888139573360124440321458177  # fq.rs

FIELD_FR, FIELD_FQ = 0, 1          # SNARKVM_B200_FIELD_FR / _FQ
# field → (modulus, MODULUS_BITS, 32-bit limbs of the in-memory image)
FIELDS = {FIELD_FR: (R_MOD, 253, 8), FIELD_FQ: (Q_MOD, 377, 12)}

# PARAMS_OPT_FOR_CONSTRAINTS: rate → (alpha, full_rounds, partial_rounds, skip_matrices)
DEFAULT_PARAMETERS = {
    FIELD_FR: {2: (17, 8, 31, 0), 3: (17, 8, 31, 0), 4: (17, 8, 31, 0), 5: (17, 8, 31, 0), 6: (17, 8, 31, 0), 7: (17, 8, 31, 0),
               8: (17, 8, 31, 0)},
    FIELD_FQ: {2: (17, 8, 31, 0), 3: (5, 8, 56, 0), 4: (5, 8, 56, 0), 5: (5, 8, 57, 0), 6: (5, 8, 57, 0), 7: (5, 8, 57, 0),
               8: (5, 8, 57, 0)},
}

# the device sponge's shape: rate 2, capacity 1, α = 17, 8 full and 31 partial rounds (the same for Fr and Fq)
RATE = 2

# operation kinds of a transcript (SNARKVM_B200_POSEIDON_*)
OP_ABSORB, OP_SQUEEZE, OP_SQUEEZE_NONNATIVE, OP_SQUEEZE_SHORT_NONNATIVE = 0, 1, 2, 3


class GrainLFSR:
    """PoseidonGrainLFSR (poseidon_grain_lfsr.rs:23-217)"""

    def __init__(self, field_size_in_bits: int, state_len: int, full_rounds: int, partial_rounds: int, sbox_is_inverse: bool = False):
        state = [False] * 80
        state[1] = True                                     # b0, b1: the field (prime)
        state[5] = sbox_is_inverse                          # b2 … b5: the S-box
        for lo, hi, value in ((6, 17, field_size_in_bits), (18, 29, state_len), (30, 39, full_rounds), (40, 49, partial_rounds)):
            for i in range(hi, lo - 1, -1):
                state[i] = bool(value & 1)
                value >>= 1
        for i in range(50, 80):
            state[i] = True
        self.bits, self.state, self.head = field_size_in_bits, state, 0
        for _ in range(160):
            self._next_bit()

    def _next_bit(self) -> bool:
        s, h = self.state, self.head
        b = s[(h + 62) % 80] ^ s[(h + 51) % 80] ^ s[(h + 38) % 80] ^ s[(h + 23) % 80] ^ s[(h + 13) % 80] ^ s[h]
        s[h] = b
        self.head = (h + 1) % 80
        return b

    def _bits(self, n: int):
        """LFSRIter: a bit is kept only when the bit before it is one"""
        for _ in range(n):
            while not self._next_bit():
                self._next_bit()
            yield self._next_bit()

    def _integer(self) -> int:
        """field_size_in_bits bits, most significant first"""
        v = 0
        for b in self._bits(self.bits):
            v = (v << 1) | b
        return v

    def field_elements_rejection_sampling(self, modulus: int, count: int) -> list:
        out = []
        for _ in range(count):
            while True:
                v = self._integer()
                if v < modulus:
                    out.append(v)
                    break
        return out

    def field_elements_mod_p(self, modulus: int, count: int) -> list:
        return [self._integer() % modulus for _ in range(count)]


@functools.cache
def parameters(field: int, rate: int = RATE) -> tuple:
    """default_poseidon_parameters::<rate>() of the field → (alpha, full_rounds, partial_rounds, ark, mds) with canonical integers:
    ark[round][i] for the rate + 1 state elements, mds[i][j]"""
    p, bits, _n = FIELDS[field]
    alpha, full, partial, skip = DEFAULT_PARAMETERS[field][rate]
    lfsr = GrainLFSR(bits, rate + 1, full, partial)
    ark = [lfsr.field_elements_rejection_sampling(p, rate + 1) for _ in range(full + partial)]
    for _ in range(skip):
        lfsr.field_elements_mod_p(p, 2 * (rate + 1))
    xs = lfsr.field_elements_mod_p(p, rate + 1)
    ys = lfsr.field_elements_mod_p(p, rate + 1)
    mds = [[pow((x + y) % p, -1, p) for y in ys] for x in xs]
    return alpha, full, partial, ark, mds


def to_mont_words(field: int, values) -> np.ndarray:
    """canonical integers → their Montgomery images as [len, limbs] uint32 (the device layout)"""
    p, _bits, n = FIELDS[field]
    r = (1 << (32 * n)) % p
    blob = b"".join((int(v) * r % p).to_bytes(4 * n, "little") for v in values)
    return np.frombuffer(blob, dtype=np.uint32).reshape(-1, n).copy()


def from_mont_words(field: int, words: np.ndarray) -> list:
    """Montgomery images [m, limbs] (any unsigned or signed integer dtype of the same bytes) → canonical integers"""
    p, _bits, n = FIELDS[field]
    rinv = pow((1 << (32 * n)) % p, -1, p)
    raw = np.ascontiguousarray(words).view(np.uint8).reshape(-1, 4 * n)
    return [int.from_bytes(row.tobytes(), "little") * rinv % p for row in raw]


def device_parameters(field: int, dev) -> torch.Tensor:
    """ark (39 × 3) then mds (3 × 3) of PoseidonSponge<F, 2, 1>, Montgomery, as one int64 CUDA tensor on `dev`; uploaded once per
    device and field"""
    dev = torch.device(dev)
    if dev.type == "cuda" and dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    key = (field, dev)
    if key not in _uploaded:
        _alpha, _full, _partial, ark, mds = parameters(field, RATE)
        words = to_mont_words(field, [v for row in ark for v in row] + [v for row in mds for v in row])
        _uploaded[key] = torch.from_numpy(words.view(np.int64)).to(dev)
    return _uploaded[key]


_uploaded: dict = {}


def state_words(field: int) -> int:
    """32-bit words of one state record of a resumable transcript: the three state elements, the mode, the index, two zero words"""
    return 3 * FIELDS[field][2] + 4


def fresh_states(field: int, count: int, dev) -> torch.Tensor:
    """`count` state records of a new sponge (state zero, absorbing at index 0) as the int64 CUDA tensor device.poseidon_transcripts
    resumes from and updates"""
    return torch.zeros((count, state_words(field) // 2), dtype=torch.int64, device=dev)


def bytes_to_field_elements(data: bytes, field: int) -> list:
    """AlgebraicSponge::absorb_bytes's packing (algorithms/src/traits/algebraic_sponge.rs:47-68): the bytes' bits, most significant
    bit of each byte first, cut into chunks of size_in_bits − 1 bits; each chunk (the last one may be shorter) is read as a
    big-endian integer.  No bytes give no element."""
    _p, bits, _n = FIELDS[field]
    cap = bits - 1
    total = 8 * len(data)
    v = int.from_bytes(data, "big")
    out = []
    for start in range(0, total, cap):
        width = min(cap, total - start)
        out.append((v >> (total - start - width)) & ((1 << width) - 1))
    return out



# OptimizationType (algorithms/src/traits/algebraic_sponge.rs:156-163)
OPT_CONSTRAINTS, OPT_WEIGHT = 0, 1


def find_parameters(base_field_prime_length: int, target_field_prime_bit_length: int, optimization_type: int) -> tuple:
    """nonnative_params::find_parameters (algebraic_sponge.rs:166-229): the limb count and limb size of least cost → (num_limbs,
    bits_per_limb)"""
    surfeit = 10
    max_limb_size = min((base_field_prime_length - 1 - surfeit - 1) // 2 - 1, target_field_prime_bit_length)
    best = None
    for limb_size in range(1, max_limb_size + 1):
        num_of_limbs = (target_field_prime_bit_length + limb_size - 1) // limb_size
        group_size = (base_field_prime_length - 1 - surfeit - 1 - 1 - limb_size + limb_size - 1) // limb_size
        num_of_groups = (2 * num_of_limbs - 1 + group_size - 1) // group_size
        t = target_field_prime_bit_length
        if optimization_type == OPT_CONSTRAINTS:
            cost = 2 * num_of_limbs - 1 + t + t + num_of_limbs + num_of_groups + (num_of_groups - 1) * (limb_size * 2 + surfeit) + 1
        else:
            cost = (6 * num_of_limbs * num_of_limbs + 4 * t + 4 * t + num_of_limbs + num_of_limbs * num_of_limbs + 2 * (2 * num_of_limbs - 1)
                    + num_of_limbs + num_of_groups + 6 * num_of_groups + (num_of_groups - 1) * (2 * limb_size + surfeit) * 4 + 2)
        if best is None or cost < best[0]:
            best = (cost, num_of_limbs, limb_size)
    return best[1], best[2]


def overhead(x: int) -> int:
    """the `overhead!` macro (algebraic_sponge.rs:105-134) on a non-zero integer: its bit length, plus one unless it is a power of two"""
    return x.bit_length() + (0 if x & (x - 1) == 0 else 1)


# absorb_nonnative_field_elements::<Fr> into the Fq sponge (poseidon.rs:168, 337-432): get_params(253, 377, Weight)
NONNATIVE_LIMBS, NONNATIVE_LIMB_BITS = find_parameters(FIELDS[FIELD_FQ][1], FIELDS[FIELD_FR][1], OPT_WEIGHT)
assert (NONNATIVE_LIMBS, NONNATIVE_LIMB_BITS) == (5, 51)
# every limb is pushed with noise one, so each carries a budget of bits_per_limb + overhead!(1 + 1) bits; two consecutive limbs merge
# when their budgets fit in the Fq sponge's capacity, size_in_bits − 1
_LIMB_BUDGET = NONNATIVE_LIMB_BITS + overhead(2)
_MERGE = 2 * _LIMB_BUDGET <= FIELDS[FIELD_FQ][1] - 1


def nonnative_field_elements(values) -> list:
    """the Fq elements one absorb_nonnative_field_elements call of Fr values absorbs natively (push_elements_to_sponge, poseidon.rs:
    412-432): each value (canonical, < r) split into NONNATIVE_LIMBS limbs of NONNATIVE_LIMB_BITS bits, big limb first
    (get_limbs_representations), then compress_elements (:343-377) over the whole stream: a limb and the next merge as
    first · 2^budget + second while two budgets fit in the capacity; a last odd limb stays alone.  No values give no element."""
    mask = (1 << NONNATIVE_LIMB_BITS) - 1
    limbs = []
    for v in values:
        v = int(v)
        if not 0 <= v < R_MOD:
            raise ValueError("a nonnative value is not below r")
        limbs += [(v >> (NONNATIVE_LIMB_BITS * i)) & mask for i in reversed(range(NONNATIVE_LIMBS))]
    if not _MERGE:
        return limbs
    out = [(limbs[i] << _LIMB_BUDGET) + limbs[i + 1] for i in range(0, len(limbs) - 1, 2)]
    if len(limbs) % 2:
        out.append(limbs[-1])
    return out
