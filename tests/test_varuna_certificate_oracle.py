"""The verifying-key certificate restatement (tests/varuna_certificate_oracle.py) checked without a GPU: the circuit id's byte stream
is the serialize_uncompressed layout, the Lagrange route of evaluate_index_polynomials equals Horner on the interpolated index
polynomials (point outside and inside K), and on a setup with a known trapdoor the certificate satisfies the pairing equation in the
exponent, lhs = β·W, which fails after any change to a commitment, W, the point or the circuit."""
import hashlib
import random
import struct

import numpy as np
import pytest

from oracle import bls12_377 as py
from oracle import sonic as osonic
from oracle import varuna as ov

import varuna_certificate_oracle as vco
import varuna_index_oracle as vio

R = ov.R
BETA, GAMMA = 0x5EED5EED1234567 % R, 0xABCDEF % R
D = 63


def test_id_stream_layout_of_a_hand_built_matrix():
    # row 0: (5, column 2), (R − 1, column 7); row 1: empty
    m = [[(5, 2), (R - 1, 7)], []]
    want = (b"\x02" + b"\0" * 7                                        # nrows = 2
            + b"\x02" + b"\0" * 7                                      # row 0 holds two entries
            + b"\x05" + b"\0" * 31 + b"\x02" + b"\0" * 7              # 5 as 32 LE bytes, column 2 as u64 LE
            + (R - 1).to_bytes(32, "little") + b"\x07" + b"\0" * 7    # r − 1, column 7
            + b"\0" * 8)                                               # row 1 holds nothing
    assert vco.id_stream(m) == want
    assert len(want) == 8 + 8 * 2 + 40 * 2
    # row r's header sits at 8 + 8·r + 40·row_ptr[r]
    assert want[8 + 8 * 1 + 40 * 2:] == b"\0" * 8


def test_circuit_id_hashes_info_then_a_b_c(golden):
    a, b = golden["varuna_circuit_0_prover"]["witness_a_b"]
    c = ov.Circuit(ov.test_circuit(a, b, 3, 7, 7))
    info = vio.circuit_info(c)
    assert vco.circuit_info_bytes(info) == struct.pack("<6Q", 4, 7, 7, 7, 7, 7)
    from snarkvm_b200 import varuna as dv
    assert dv.CircuitInfo(*info).to_bytes_le() == vco.circuit_info_bytes(info)
    stream = vco.circuit_info_bytes(info) + b"".join(vco.id_stream(m) for m in (c.a, c.b, c.c))
    assert vco.circuit_id(c) == hashlib.blake2s(stream, digest_size=32).digest()
    # one changed value changes the id
    c2 = ov.Circuit(ov.test_circuit(a, b, 3, 7, 7))
    c2.a[0][0] = (2, c2.a[0][0][1])
    assert vco.circuit_id(c2) != vco.circuit_id(c)


def _circuits(golden):
    # the TestCircuit has a last row unlike the others: with every index polynomial of degree ≤ 1 (one mul_var) the opening would
    # hold at any point, so a moved point could not be told apart
    a, b = golden["varuna_circuit_0_prover"]["witness_a_b"]
    yield "circuit_0", ov.Circuit(ov.test_circuit(a, b, 3, 7, 7))
    yield "test_circuit_2_30_21", ov.Circuit(ov.test_circuit(3, 5, 2, 30, 21))
    yield "sparse", ov.Circuit(vio.sparse_r1cs(3, 4, 40, 37, (61, 64, 33)))


@pytest.mark.parametrize("inside", [False, True])
def test_lagrange_route_equals_horner_on_the_index_polynomials(golden, inside):
    rng = random.Random(5 + inside)
    for name, c in _circuits(golden):
        polys = vio.index_polynomials(c)
        # inside: an element of the largest K (a smaller K holds it only when its index is a multiple of the size ratio)
        point = c.max_non_zero_domain.elements()[3 % c.max_non_zero_domain.size] if inside else rng.randrange(R)
        combiners = [1] + [rng.randrange(R) for _ in range(11)]
        got = vco.evaluate_index_polynomials(c, point, combiners)
        want = sum(k * ov.poly_eval(polys[n], point) for k, n in zip(combiners, vio.INDEX_ORDER)) % R
        assert got == want, (name, inside)
        evals = vco.index_evaluations_at(c, point)
        for n in vio.INDEX_ORDER:
            assert evals[n] == ov.poly_eval(polys[n], point), (name, n)


def _g(cpu):
    return np.frombuffer(py.affine_bytes(py.G1_GENERATOR), dtype=np.uint8)


@pytest.fixture(scope="module")
def srs(oracle_cpu):
    g = _g(oracle_cpu)

    def pts(scalars):
        out = np.zeros((len(scalars), 104), dtype=np.uint8)
        for i, s in enumerate(scalars):
            out[i] = np.frombuffer(py.affine_bytes(py.projective_from_bytes(oracle_cpu.g1_mul(g, osonic._scalars([s])[0]).tobytes())),
                                   dtype=np.uint8)
        return out
    return pts([pow(BETA, i, R) for i in range(D + 1)]), pts([GAMMA * pow(BETA, i, R) % R for i in range(D + 2)])


def _setup_and_certify(c, srs, rng):
    powers, gpowers = srs
    info, comms = vio.circuit_setup(c, powers, gpowers, osonic.commit)
    challenges = [rng.randrange(R) for _ in range(12)]
    xi = rng.randrange(R)
    w = vco.prove_vk(powers, gpowers, c, challenges, iter([xi, rng.randrange(R)]))
    return info, comms, challenges, xi, w


def _beta_w(cpu, w):
    return cpu.g1_mul(vco.affine(w), osonic._scalars([BETA])[0])


@pytest.mark.parametrize("name", ["circuit_0", "test_circuit_2_30_21"])
def test_certificate_satisfies_the_pairing_equation_in_the_exponent(golden, oracle_cpu, srs, name):
    c = dict(_circuits(golden))[name]
    rng = random.Random(11)
    info, comms, challenges, xi, w = _setup_and_certify(c, srs, rng)
    cid = vco.circuit_id(c)
    g = _g(oracle_cpu)
    matches, v, lhs = vco.verify_vk(c, info, cid, comms, w, g, challenges, xi)
    assert matches
    assert (lhs == _beta_w(oracle_cpu, w)).all()
    # W in closed form: ξ·(lc(β) − lc(z))/(β − z)·G
    polys = vio.index_polynomials(c)
    z, combiners = vco.point_and_combiners(challenges)
    lc = lambda x: sum(k * ov.poly_eval(polys[n], x) for k, n in zip(combiners, vio.INDEX_ORDER)) % R      # noqa: E731
    assert v == lc(z)
    assert (w == oracle_cpu.g1_mul(g, osonic._scalars([xi * (lc(BETA) - v) * pow(BETA - z, -1, R) % R])[0])).all()

    # each tampering breaks lhs = β·W
    other = oracle_cpu.g1_mul(g, osonic._scalars([12345])[0])
    bad = [x.copy() for x in comms]
    bad[4] = other
    assert not (vco.verify_vk(c, info, cid, bad, w, g, challenges, xi)[2] == _beta_w(oracle_cpu, w)).all()
    assert not (vco.verify_vk(c, info, cid, comms, other, g, challenges, xi)[2] == _beta_w(oracle_cpu, other)).all()
    moved = challenges[:-1] + [(challenges[-1] + 1) % R]
    assert not (vco.verify_vk(c, info, cid, comms, w, g, moved, xi)[2] == _beta_w(oracle_cpu, w)).all()
    tampered = _tampered_circuit(golden, name)
    matches2, _v2, lhs2 = vco.verify_vk(tampered, info, cid, comms, w, g, challenges, xi)
    assert not matches2
    assert vio.circuit_info(tampered) == info and vco.circuit_id(tampered) != cid
    assert not (lhs2 == _beta_w(oracle_cpu, w)).all()


def _tampered_circuit(golden, name):
    """the same circuit with the value of A's first entry changed, re-indexed"""
    c = dict(_circuits(golden))[name]
    val, col = c.a[0][0]
    c.a[0][0] = ((val + 1) % R, col)
    r_el, c_el = c.constraint_domain.elements(), c.variable_domain.elements()
    c.ariths[0] = ov.matrix_evals(c.a, c.non_zero_domains[0], c.variable_domain, c.input_domain, r_el, c_el)
    return c
