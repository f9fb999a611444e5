"""TEST INFRASTRUCTURE ONLY — CPU restatement (Python big integers) of the nonnative absorption of snarkVM's Poseidon sponge and of
the Fiat–Shamir transcript of VarunaSNARK::prove_batch, as a verifier recomputes it from a proof and the verifying keys.

    algorithms/src/traits/algebraic_sponge.rs:105-134   overhead!                                   → overhead
    algorithms/src/traits/algebraic_sponge.rs:148-229   get_params / find_parameters                → find_parameters
    algorithms/src/crypto_hash/poseidon.rs:168, 337-432 absorb_nonnative_field_elements, compress_elements,
                                                        get_limbs_representations                   → PoseidonSponge
    algorithms/src/snark/varuna/varuna.rs:136-194       init_sponge, absorb, absorb_with_sums       → prove_batch_transcript
    algorithms/src/snark/varuna/ahp/verifier/verifier.rs:39-197   the verifier's squeezes           → prove_batch_transcript
    algorithms/src/polycommit/sonic_pc/mod.rs:259-342   the opening challenges                      → prove_batch_transcript

It works bit by bit where the reference does (write_bits_be, from_bits_be) and shares no code with snarkvm_b200/poseidon.py.
"""
from __future__ import annotations

from oracle.poseidon import PROTOCOL_NAME, Sponge, affine_field_elements

Q = 258664426012969094010652733694893533536393512754914660539884262666720468348340822774968888139573360124440321458177
R = 8444461749428370424248824938781546531375899335154063827935233455917409239041
Q_BITS, R_BITS = 377, 253
WEIGHT = "weight"


def find_parameters(base_bits: int, target_bits: int, optimization_type: str = WEIGHT) -> tuple:
    surfeit = 10
    max_limb_size = (base_bits - 1 - surfeit - 1) // 2 - 1
    if max_limb_size > target_bits:
        max_limb_size = target_bits
    found, min_cost, min_size, min_limbs = False, 0, 0, 0
    limb_size = 1
    while limb_size <= max_limb_size:
        n = (target_bits + limb_size - 1) // limb_size
        group_size = (base_bits - 1 - surfeit - 1 - 1 - limb_size + limb_size - 1) // limb_size
        groups = (2 * n - 1 + group_size - 1) // group_size
        cost = 0
        if optimization_type == WEIGHT:
            cost += 6 * n * n
            cost += target_bits * 3 + target_bits
            cost += target_bits * 3 + target_bits + n
            cost += n * n + 2 * (2 * n - 1)
            cost += n + groups + 6 * groups + (groups - 1) * (2 * limb_size + surfeit) * 4 + 2
        else:
            cost += 2 * n - 1
            cost += target_bits
            cost += target_bits + n
            cost += groups + (groups - 1) * (limb_size * 2 + surfeit) + 1
        if not found or cost < min_cost:
            found, min_cost, min_size, min_limbs = True, cost, limb_size, n
        limb_size += 1
    return min_limbs, min_size


def bits_be(x: int, width: int) -> list:
    return [(x >> (width - 1 - i)) & 1 for i in range(width)]


def overhead(x: int) -> int:
    """the macro on an Fq value: its 384 big-endian bits, leading zeros skipped, one more unless a power of two"""
    bits = bits_be(x, 384)
    skipped = 0
    for b in bits:
        if b:
            break
        skipped += 1
    power_of_2 = not any(bits[skipped + 1:])
    return len(bits) - skipped if power_of_2 else len(bits) - skipped + 1


def limbs(value: int, num_limbs: int, bits_per_limb: int) -> list:
    """get_limbs_representations: the low bits_per_limb bits of cur (write_bits_be of the 256-bit integer, then from_bits_be of the
    tail), cur >>= bits_per_limb, num_limbs times; then reversed (big limb first)"""
    out, cur = [], value
    for _ in range(num_limbs):
        tail = bits_be(cur, 256)[256 - bits_per_limb:]
        v = 0
        for b in tail:
            v = (v << 1) | b
        out.append(v)
        cur >>= bits_per_limb
    return out[::-1]


def compress(src: list, bits_per_limb: int) -> list:
    """compress_elements over (limb, noise = 1) pairs with a peekable iterator"""
    capacity = Q_BITS - 1
    table = [pow(2, i, Q) for i in range(capacity)]
    out, i = [], 0
    while i < len(src):
        first = src[i]
        i += 1
        first_max = bits_per_limb + overhead(1 + 1)
        if i < len(src):
            second_max = bits_per_limb + overhead(1 + 1)
            if first_max + second_max <= capacity:
                out.append((first * table[second_max] + src[i]) % Q)
                i += 1
                continue
        out.append(first)
    return out


class PoseidonSponge(Sponge):
    """oracle.poseidon.Sponge over Fq with absorb_nonnative_field_elements of Fr values"""

    def absorb_nonnative_field_elements(self, values):
        num_limbs, bits_per_limb = find_parameters(Q_BITS, R_BITS, WEIGHT)
        src = [limb for v in values for limb in limbs(int(v) % R, num_limbs, bits_per_limb)]
        self.absorb_native_field_elements(compress(src, bits_per_limb))


def affine_of_image(words) -> tuple | None:
    """a normalised projective image (18 u64: X, Y, Z Montgomery Fq) → canonical affine (x, y), None at infinity"""
    limbs_ = [int(w) for w in words]
    if not any(limbs_[12:18]):
        return None
    rinv = pow(1 << 384, -1, Q)
    x = sum(v << (64 * i) for i, v in enumerate(limbs_[0:6])) * rinv % Q
    y = sum(v << (64 * i) for i, v in enumerate(limbs_[6:12])) * rinv % Q
    return (x, y)


def prove_batch_transcript(params: tuple, batch_sizes: list, public_inputs: list, vk_commitments: list, view: dict):
    """the verifier's transcript of one prove_batch proof → (challenges dict, log).  Circuits in id order.  public_inputs: per circuit,
    per instance, the padded public input (canonical); vk_commitments: per circuit its twelve commitments as affine (x, y) / None.
    view: 'w' (per instance, circuit by circuit), 'mask' (None outside the hiding mode), 'h_0', 'g_1', 'h_1', 'g_a', 'g_b', 'g_c'
    (per circuit), 'h_2' as affine points; 'third_sums' (per circuit, per instance, three), 'fourth_sums' (per circuit, three),
    'evaluations' (Evaluations::to_field_elements).  log: (operation, count) in the order the transcript runs them."""
    sponge = PoseidonSponge(Q, Q_BITS, params)
    log = []

    def absorb_points(points):
        log.append(("absorb_native", 3 * len(points)))
        sponge.absorb_native_field_elements([e for p in points for e in affine_field_elements(p)])

    def absorb_nonnative(values):
        log.append(("absorb_nonnative", len(values)))
        sponge.absorb_nonnative_field_elements(values)

    def squeeze(n, short=False):
        log.append(("squeeze_short" if short else "squeeze", n))
        return sponge.squeeze_short_nonnative_field_elements(n) if short else sponge.squeeze_nonnative_field_elements(n)

    log.append(("absorb_bytes", len(PROTOCOL_NAME)))
    sponge.absorb_bytes(PROTOCOL_NAME)
    for b, inputs in zip(batch_sizes, public_inputs):
        log.append(("absorb_bytes", 8))
        sponge.absorb_bytes(b.to_bytes(8, "little"))
        for x in inputs:
            absorb_nonnative(x)
    for comms in vk_commitments:
        absorb_points(comms)
    absorb_points(list(view["w"]) + ([view["mask"]] if view.get("mask") is not None else []))
    combiners = []
    for i, b in enumerate(batch_sizes):
        e = squeeze(b - 1 + (1 if i else 0))
        combiners.append((e[b - 1] if i else 1, [1] + e[: b - 1]))
    absorb_points([view["h_0"]])
    alpha, eta_b, eta_c = squeeze(3)
    absorb_points([view["g_1"], view["h_1"]])
    for sums in view["third_sums"]:
        for s in sums:
            absorb_nonnative(s)
    beta = squeeze(1)[0]
    absorb_points([p for k in range(len(batch_sizes)) for p in (view["g_a"][k], view["g_b"][k], view["g_c"][k])])
    for s in view["fourth_sums"]:
        absorb_nonnative(s)
    deltas = [[1] + squeeze(2)] + [squeeze(3) for _ in batch_sizes[1:]]
    absorb_points([view["h_2"]])
    gamma = squeeze(1)[0]
    absorb_nonnative(view["evaluations"])
    # the query set's points by name: α opens rowcheck_zerocheck; β g_1 and lineval_sumcheck; γ every g_M and matrix_sumcheck
    opening = []
    for count in (1, 2, 3 * len(batch_sizes) + 1):
        opening += [squeeze(1, True)[0] for _ in range(count + 1)]
    challenges = {"batch_combiners": combiners, "alpha": alpha, "eta_b": eta_b, "eta_c": eta_c, "beta": beta, "deltas": deltas,
                  "gamma": gamma, "opening": opening}
    return challenges, log, sponge
