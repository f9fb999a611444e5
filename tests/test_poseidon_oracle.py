"""CPU tests of the Poseidon parameters (snarkvm_b200/poseidon.py) and of the big-integer sponge (oracle/poseidon.py), against the
reference's own snapshots (tests/golden/poseidon_vectors.json, extracted by make_poseidon_golden.py), and of the host encoding of a
verifying-key certificate's transcript (varuna._certificate_transcripts) against the oracle's transcript."""
import copy
import json
import os
import random

import numpy as np
import pytest

from oracle import poseidon as op
from snarkvm_b200 import poseidon as ps

HERE = os.path.dirname(os.path.abspath(__file__))
R, Q = ps.R_MOD, ps.Q_MOD


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(HERE, "golden", "poseidon_vectors.json")) as f:
        return json.load(f)


def _sponge(field):
    p, bits, _n = ps.FIELDS[field]
    return op.Sponge(p, bits, ps.parameters(field, 2))


def test_grain_lfsr_samples(golden):
    lfsr = ps.GrainLFSR(253, 3, 8, 31)
    assert lfsr.field_elements_rejection_sampling(R, 1) == golden["grain_first_sample"]
    assert lfsr.field_elements_rejection_sampling(R, 1) == golden["grain_second_sample"]


@pytest.mark.parametrize("rate", range(2, 9))
def test_fr_ark_and_mds(golden, rate):
    alpha, full, partial, ark, mds = ps.parameters(ps.FIELD_FR, rate)
    assert (alpha, full, partial) == (17, 8, 31)
    assert ark == golden["ark"][str(rate)]
    assert mds == golden["mds"][str(rate)]


def test_fq_rate_2_shape():
    """snarkVM's Fiat–Shamir parameters: no reference vector; the generator is the one the Fr snapshots pin"""
    alpha, full, partial, ark, mds = ps.parameters(ps.FIELD_FQ, 2)
    assert (alpha, full, partial) == (17, 8, 31)
    assert len(ark) == 39 and all(len(r) == 3 and all(0 <= v < Q for v in r) for r in ark)
    assert len(mds) == 3 and all(len(r) == 3 for r in mds)
    assert ark != ps.parameters(ps.FIELD_FR, 2)[3]


def test_absorb_squeeze_vectors_and_modes(golden):
    """test_poseidon_sponge_consistency (crypto_hash/tests.rs:51-71): the 100 snapshots and its mode assertions"""
    for a in range(10):
        for s in range(10):
            sp = _sponge(ps.FIELD_FR)
            sp.absorb_native_field_elements([1237812] * a)
            nai = a % 2 if a % 2 != 0 or a == 0 else 2
            assert sp.mode == ("absorbing", nai)
            assert sp.squeeze_native_field_elements(s) == golden["absorb_squeeze"][f"{a},{s}"], (a, s)
            if s == 0:
                assert sp.mode == ("absorbing", nai)
            else:
                assert sp.mode == ("squeezing", s % 2 if s % 2 != 0 else 2)


def _bits_of(data: bytes, cap: int) -> list:
    """absorb_bytes restated on a list of bits: MSB of each byte first, chunks of `cap`, each read big-endian"""
    bits = []
    for byte in data:
        for k in range(7, -1, -1):
            bits.append((byte >> k) & 1)
    out = []
    for i in range(0, len(bits), cap):
        out.append(int("".join(map(str, bits[i: i + cap])) or "0", 2))
    return out


@pytest.mark.parametrize("field", [ps.FIELD_FQ, ps.FIELD_FR])
@pytest.mark.parametrize("nbytes", [0, 1, 31, 32, 46, 47, 48, 95])
def test_absorb_bytes(field, nbytes):
    rng = random.Random(nbytes)
    data = bytes(rng.randrange(256) for _ in range(nbytes))
    cap = ps.FIELDS[field][1] - 1
    want = _bits_of(data, cap)
    assert ps.bytes_to_field_elements(data, field) == want
    sp = _sponge(field)
    sp.absorb_bytes(data)
    ref = _sponge(field)
    ref.absorb_native_field_elements(want)
    assert sp.state == ref.state and sp.mode == ref.mode
    if field == ps.FIELD_FQ:
        assert len(want) == {0: 0, 1: 1, 31: 1, 32: 1, 46: 1, 47: 1, 48: 2, 95: 3}[nbytes]


@pytest.mark.parametrize("field", [ps.FIELD_FQ, ps.FIELD_FR])
@pytest.mark.parametrize("short", [False, True])
def test_nonnative_outputs_are_the_squeezed_bits(field, short):
    rng = random.Random(7)
    p = ps.FIELDS[field][0]
    width = 168 if short else 252
    for count in (0, 1, 2, 3, 12):
        sp = _sponge(field)
        sp.absorb_native_field_elements([rng.randrange(p) for _ in range(rng.randrange(5))])
        twin = copy.deepcopy(sp)
        got = sp.get_fe(count, short)
        bits = twin.get_bits(width * count)
        assert sp.state == twin.state and sp.mode == twin.mode
        assert len(got) == count
        assert got == [int("".join(map(str, bits[i * width: (i + 1) * width])), 2) for i in range(count)]
        assert all(v < (1 << width) and v < R for v in got)
        assert twin.permutations == sp.permutations


def _known_key():
    from snarkvm_b200 import varuna as dv
    rng = random.Random(11)
    info = dv.CircuitInfo(4, 100, 70, 300, 250, 200)
    comms = np.zeros((12, 18), dtype=np.uint64)
    affine = []
    one = (1 << 384) % Q
    for i in range(12):
        if i == 5:                                                         # the point at infinity: (0, one, 0)
            comms[i, 6:12] = np.frombuffer(one.to_bytes(48, "little"), dtype=np.uint64)
            affine.append(None)
            continue
        x, y = rng.randrange(Q), rng.randrange(Q)
        comms[i, 0:6] = np.frombuffer((x * one % Q).to_bytes(48, "little"), dtype=np.uint64)
        comms[i, 6:12] = np.frombuffer((y * one % Q).to_bytes(48, "little"), dtype=np.uint64)
        comms[i, 12:18] = np.frombuffer(one.to_bytes(48, "little"), dtype=np.uint64)
        affine.append((x, y))
    ident = bytes(rng.randrange(256) for _ in range(32))
    return dv.CircuitVerifyingKey(info, comms, ident), affine


class _Logged(op.Sponge):
    def absorb_native_field_elements(self, elements):
        self.calls = getattr(self, "calls", []) + [list(elements)]
        super().absorb_native_field_elements(elements)


def test_certificate_transcript_encoding():
    """the op lists certificate_challenges sends to the device: the oracle's absorb calls, element for element, then 12 + 1 + 1
    nonnative squeezes"""
    from snarkvm_b200 import varuna as dv
    vk, affine = _known_key()
    vk2 = copy.deepcopy(vk)
    vk2.id = bytes(32)
    ops, op_start, inputs = dv._certificate_transcripts([vk, vk2])
    assert op_start.tolist() == [0, 7, 14]
    for k, key in enumerate((vk, vk2)):
        sp = _Logged(Q, 377, ps.parameters(ps.FIELD_FQ, 2))
        sp.absorb_bytes(op.PROTOCOL_NAME)
        sp.absorb_bytes(key.circuit_info.to_bytes_le())
        sp.absorb_native_field_elements([e for c in affine for e in op.affine_field_elements(c)])
        sp.absorb_bytes(key.id)
        assert [len(c) for c in sp.calls] == [1, 2, 36, 1]
        got = []
        for kind, n, off in ops[7 * k: 7 * k + 4].tolist():
            assert kind == ps.OP_ABSORB
            got.append(ps.from_mont_words(ps.FIELD_FQ, inputs[off: off + n]))
        assert got == sp.calls
        assert ops[7 * k + 4:7 * k + 7].tolist() == [[ps.OP_SQUEEZE_NONNATIVE, 12, 14 * k], [ps.OP_SQUEEZE_SHORT_NONNATIVE, 1, 14 * k + 12],
                                                     [ps.OP_SQUEEZE_SHORT_NONNATIVE, 1, 14 * k + 13]]
        # the same transcript through certificate_sponge / certificate_challenges: 19 permutations while absorbing the 40
        # elements, 5 for the nine squeezed elements of the challenges, one for the randomizer
        s2 = op.certificate_sponge(Q, 377, ps.parameters(ps.FIELD_FQ, 2), key.circuit_info.to_bytes_le(), affine, key.id)
        assert s2.state == sp.state
        ch, (xi, rand) = op.certificate_challenges(s2)
        assert len(ch) == 12 and all(0 <= c < R for c in ch) and xi < (1 << 168) and rand < (1 << 168)
        assert s2.permutations == 25
    assert sp.calls[0] == [int.from_bytes(op.PROTOCOL_NAME, "big")]


def test_a_key_without_id_is_refused():
    from snarkvm_b200 import varuna as dv
    vk, _ = _known_key()
    vk.id = None
    with pytest.raises(ValueError):
        dv._certificate_transcripts([vk])
