"""CPU: the G2 byte-form oracle (g2_bytes_oracle) and the verifier key's host checks.

The oracle's Fq2 roots square back, decode inverts encode on subgroup points and infinity in both forms, both mainnet G2 fixtures
(β·H and the 27 negative powers of β·H) are on the curve with [r]·P = O, the VerifierKey layout is 288 / 576 bytes, and
UniversalVerifier.from_bytes refuses a wrong length, trailing bytes and a g or h other than the generator before any device call."""
import os
import random

import pytest

import g2_bytes_oracle as o
import varuna_bytes_oracle as vb
from oracle import bls12_377 as py
from oracle import g2 as og2

HERE = os.path.dirname(os.path.abspath(__file__))


def _read(name):
    with open(os.path.join(HERE, "golden", name), "rb") as f:
        return f.read()


def test_roots_square_back():
    rng = random.Random(5)
    found = 0
    for k in range(200):
        a = (rng.randrange(o.Q), 0 if k % 10 == 0 else rng.randrange(o.Q))
        r = o.fq2_sqrt(a)
        if r is not None:
            assert og2.f2_sqr(r) == a
            found += 1
        sq = og2.f2_sqr(a)
        assert og2.f2_sqr(o.fq2_sqrt(sq)) == sq
    assert 50 < found < 150
    assert o.fq2_sqrt((0, 0)) == (0, 0)


@pytest.mark.parametrize("compressed", [True, False], ids=["compressed", "uncompressed"])
def test_encode_decode_invert(compressed):
    rng = random.Random(6)
    pts = [og2.g2_mul(o.G2_GEN, rng.randrange(1, o.R)) for _ in range(4)] + [o.G2_GEN, None]
    for p in pts:
        b = o.encode(p, compressed)
        assert len(b) == (96 if compressed else 192)
        assert o.decode(b, compressed, True) == (o.VALID, p)
        if p is not None:
            neg = (p[0], og2.f2_neg(p[1]))
            assert o.decode(o.encode(neg, compressed), compressed, True) == (o.VALID, neg)


def test_mainnet_fixtures_are_in_the_subgroup():
    from snarkvm_b200 import varuna as dv
    points = [_read("beta_h.usrs")] + [p for _d, p in dv._u64_map(_read("neg_powers_of_beta.usrs"), 192, "negative powers")]
    assert len(points) == 28
    for b in points:
        s, p = o.decode(b, False, True)
        assert s == o.VALID and p is not None
        assert o.encode(p, False) == b


def test_verifier_key_layout_and_host_refusals():
    from snarkvm_b200 import varuna as dv
    gen1, gen2 = py.G1_GENERATOR, o.G2_GEN
    assert dv.G1_GENERATOR == gen1 and dv.G2_GENERATOR == gen2
    gamma_g, beta_h = py.g1_mul(gen1, 7), og2.g2_mul(gen2, 11)
    for compressed, size in ((True, 288), (False, 576)):
        blob = o.verifier_key_bytes(gen1, gamma_g, gen2, beta_h, compressed)
        assert len(blob) == size
        with pytest.raises(ValueError, match="not 287"):
            dv.UniversalVerifier.from_bytes(blob[:-1] if compressed else blob[:287], compressed, device_="cpu")
        with pytest.raises(ValueError, match="trailing bytes"):
            dv.UniversalVerifier.from_bytes(blob + b"\0", compressed, device_="cpu")
        g1 = 48 if compressed else 96
        not_g = vb.encode_g1(gamma_g, compressed) + blob[g1:]
        with pytest.raises(ValueError, match="g: not the G1 generator"):
            dv.UniversalVerifier.from_bytes(not_g, compressed, device_="cpu")
        neg_g = vb.encode_g1((gen1[0], o.Q - gen1[1]), compressed) + blob[g1:]
        if compressed:                                            # −g differs only in the sign bit
            with pytest.raises(ValueError, match="g: not the G1 generator"):
                dv.UniversalVerifier.from_bytes(neg_g, compressed, device_="cpu")
        not_h = blob[:2 * g1] + o.encode(beta_h, compressed) + blob[2 * g1 + (96 if compressed else 192):]
        with pytest.raises(ValueError, match="h: not the G2 generator"):
            dv.UniversalVerifier.from_bytes(not_h, compressed, device_="cpu")
        inf_h = blob[:2 * g1] + o.encode(None, compressed) + blob[2 * g1 + (96 if compressed else 192):]
        with pytest.raises(ValueError, match="h: not the G2 generator"):
            dv.UniversalVerifier.from_bytes(inf_h, compressed, device_="cpu")
