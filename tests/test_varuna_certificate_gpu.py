"""GPU: the verifying-key certificate on the device — the circuit id's byte stream (device.csr_serialize, Circuit.id), the one-pass
linear combination (device.fr_lincomb), the four inner products of MatrixEvals::evaluate (device.matrix_evals_dot), prove_vk and
verify_vk — against the CPU restatement (tests/varuna_certificate_oracle.py), on a synthetic SRS, on the real 2^15-point SRS and in
closed form at 2^18 constraints."""
import os
import random

import numpy as np
import pytest

from oracle import bls12_377 as py
from oracle import sonic as osonic
from oracle import varuna as ov

import varuna_certificate_oracle as vco
import varuna_index_oracle as vio
from test_varuna_setup_gpu import CASES, _device_circuit, _oracle_circuit

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
R = ov.R
BETA, GAMMA = 0x1234567890ABCDEF1234567890ABCDEF % R, 0xFEDCBA0987654321FEDCBA % R


def _mont_tensor(vals):
    import torch
    from snarkvm_b200 import varuna as dv
    a = np.array([dv._mont(v) for v in vals], dtype=np.uint64).reshape(-1, 4)
    return torch.from_numpy(a.view(np.int64)).cuda()


def _ints(t) -> list:
    from snarkvm_b200 import device
    if t.shape[0] == 0:
        return []
    h = device.fr_from_mont(t.contiguous()).cpu().numpy().view(np.uint64)
    return [int(r[0]) | int(r[1]) << 64 | int(r[2]) << 128 | int(r[3]) << 192 for r in h]


@pytest.mark.parametrize("name", list(CASES))
def test_id_stream_and_id_vs_oracle(name, golden):
    oc = _oracle_circuit(name, golden)
    dc = _device_circuit(oc)
    for m, om in zip((dc.a, dc.b, dc.c), (oc.a, oc.b, oc.c)):
        assert bytes(m.serialize().cpu().numpy()) == vco.id_stream(om), name
    assert dc.id() == vco.circuit_id(oc)
    assert dc.id() is dc.id()                                          # cached


def test_id_stream_of_bad_row_ptr_raises():
    import torch
    from snarkvm_b200 import CudaError, device
    cols = torch.tensor([0, 1, 2], dtype=torch.int32, device="cuda")
    vals = _mont_tensor([1, 2, 3])
    for ptr in ([0, 2, 1, 3], [0, 1, 2, 4], [1, 1, 2, 3]):
        with pytest.raises(CudaError):
            device.csr_serialize(torch.tensor(ptr, dtype=torch.int32, device="cuda"), cols, vals)


def test_lincomb_equals_the_axpy_sequence():
    from snarkvm_b200 import device
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import poly_axpy
    rng = random.Random(3)
    lens = [5, 300, 0, 1, 257, 64, 300, 1000, 7, 2, 999, 513]
    coeffs = [1, rng.randrange(R), 7, 0, 1, rng.randrange(R), R - 1, rng.randrange(R), 0, 1, rng.randrange(R), 2]
    polys = [_mont_tensor([rng.randrange(R) for _ in range(n)]) for n in lens]
    for k in (1, 2, 5, 12):
        got = device.fr_lincomb(polys[:k], [dv._mont(c) for c in coeffs[:k]])
        acc = None
        for c, p in zip(coeffs[:k], polys[:k]):
            acc = poly_axpy(acc, c, p)
        assert got.shape[0] == max(lens[:k])
        want = np.zeros((got.shape[0], 4), dtype=np.int64)
        want[: acc.shape[0]] = acc.cpu().numpy()
        assert (got.cpu().numpy() == want).all(), k
    with pytest.raises(ValueError):
        device.fr_lincomb(polys + polys[:1], [dv._mont(1)] * 13)


@pytest.mark.parametrize("lg", [0, 1, 5, 12])
@pytest.mark.parametrize("inside", [False, True])
def test_matrix_evals_dot_vs_oracle(lg, inside):
    from snarkvm_b200 import device
    from snarkvm_b200.algorithms import EvaluationDomain
    rng = random.Random(lg * 2 + inside)
    n = 1 << lg
    K = ov.Domain(n)
    row, col, rcv = ([rng.randrange(R) for _ in range(n)] for _ in range(3))
    point = K.elements()[n // 2 if n > 1 else 0] if inside else rng.randrange(R)
    lag = K.evaluate_all_lagrange_coefficients(point)
    want = vco.matrix_evals_dot(ov.MatrixEvals(row, col, rcv, K), lag)
    dlag = EvaluationDomain.new(n).evaluate_all_lagrange_coefficients(point)
    assert _ints(dlag) == lag
    got = device.matrix_evals_dot(_mont_tensor(row), _mont_tensor(col), _mont_tensor(rcv), dlag)
    assert [_ints_host(v) for v in got] == want


def _ints_host(limbs) -> int:
    from snarkvm_b200.algorithms import _fr_mont_to_int
    return _fr_mont_to_int(limbs)


@pytest.mark.parametrize("name", list(CASES))
def test_evaluate_index_polynomials_vs_oracle(name, golden):
    oc = _oracle_circuit(name, golden)
    dc = _device_circuit(oc)
    rng = random.Random(hash(name) & 0xFFFF)
    combiners = [1] + [rng.randrange(R) for _ in range(11)]
    for point in (rng.randrange(R), oc.max_non_zero_domain.elements()[1 % oc.max_non_zero_domain.size]):
        assert dc.evaluate_index_polynomials(point, combiners) == vco.evaluate_index_polynomials(oc, point, combiners), name


@pytest.fixture(scope="module")
def synthetic():
    from snarkvm_b200 import sonic_pc
    powers, gamma = sonic_pc.synthetic_srs(2047, BETA, GAMMA)
    return powers, gamma, powers.cpu().numpy(), gamma.cpu().numpy()


def _device_open_combinations(pk, challenges, opening):
    """the certificate through the device's general SonicKZG10.open_combinations (poly_axpy per term)"""
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import LabeledPolynomial, Randomness, SonicKZG10
    point, combiners = vco.point_and_combiners(challenges)
    polys = pk.circuit.index_polynomials()
    lc = [("circuit_check", list(zip(combiners, dv.INDEX_POLYNOMIAL_NAMES)))]
    (w, _), = SonicKZG10.open_combinations(pk.committer_key, lc, [LabeledPolynomial(n, p) for n, p in polys.items()],
                                           [Randomness()] * 12, [("circuit_check", ("challenge", point))], iter(opening))
    return w


def _check_certificate(oc, dc, powers, gamma, hp, hg, oracle_cpu, rng):
    from snarkvm_b200 import varuna as dv
    pk, vk = dv.circuit_setup(dc, powers, gamma, with_id=True)
    assert vk.id == vco.circuit_id(oc)
    challenges = [rng.randrange(R) for _ in range(12)]
    opening = [rng.randrange(R), rng.randrange(R)]
    cert = dv.prove_vk(pk, challenges, iter(opening))
    want_w = vco.prove_vk(hp, hg, oc, challenges, iter(opening))
    assert (cert.w == want_w).all()
    assert (cert.w == _device_open_combinations(pk, challenges, opening)).all()
    check = dv.verify_vk(dc, vk, cert, challenges, opening[0])
    g = np.frombuffer(py.affine_bytes(py.G1_GENERATOR), dtype=np.uint8)
    info, comms = vio.circuit_setup(oc, hp, hg, osonic.commit)
    matches, v, lhs = vco.verify_vk(oc, info, vco.circuit_id(oc), comms, want_w, g, challenges, opening[0])
    assert check.matches and matches
    assert check.evaluation == v
    assert (check.lhs == lhs).all()
    assert (check.w == cert.w).all()
    return pk, vk, cert, check, challenges, opening


@pytest.mark.parametrize("name", ["circuit_0", "test_circuit_3_100_70", "sparse_one_public", "test_circuit_2_1024_1014"])
def test_certificate_on_a_synthetic_srs(name, golden, oracle_cpu, synthetic):
    powers, gamma, hp, hg = synthetic
    oc = _oracle_circuit(name, golden)
    _pk, _vk, cert, check, _ch, _op = _check_certificate(oc, _device_circuit(oc), powers, gamma, hp, hg, oracle_cpu, random.Random(7))
    bw = oracle_cpu.g1_mul(vco.affine(cert.w), osonic._scalars([BETA])[0])
    assert (check.lhs == bw).all()                                     # e(lhs, H) = e(W, β·H) in the exponent


@pytest.fixture(scope="module")
def real_srs():
    import torch
    from helpers import affine_array
    blob = open(os.path.join(HERE, "golden", "powers_of_beta_15.usrs"), "rb").read()
    n = int.from_bytes(blob[:8], "little")
    host = affine_array(py.parse_usrs_points(blob, n))
    return host, torch.from_numpy(host).cuda()


@pytest.mark.parametrize("shape", [None, (2, 1 << 12, (1 << 12) - 10)])
def test_certificate_on_the_real_srs(shape, golden, oracle_cpu, real_srs):
    from snarkvm_b200 import varuna as dv
    host, powers = real_srs
    rng = random.Random(21)
    if shape is None:
        a, b = golden["varuna_circuit_0_prover"]["witness_a_b"]
        shape = (3, 7, 7)
    else:
        a, b = rng.randrange(2, R), rng.randrange(2, R)
    circuit, _z = dv.test_circuit_csr(a, b, *shape, "cuda")
    oc = ov.Circuit(ov.test_circuit(a, b, *shape))
    _check_certificate(oc, circuit, powers, powers, host, host, oracle_cpu, rng)


def test_certificate_closed_form_at_2_18(oracle_cpu):
    """TestCircuit with 2^18 constraints: W = ξ·(lc(β) − v)/(β − z)·G, with lc(β) by Horner on the device's index polynomials and v
    from the Lagrange route, and lhs = β·W"""
    from snarkvm_b200 import device
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.algorithms import _fr_mont_to_int
    from snarkvm_b200.sonic_pc import synthetic_srs
    n = 1 << 18
    circuit, _z = dv.test_circuit_csr(3, 5, 2, n, n - 10, "cuda")
    powers, gamma = synthetic_srs(circuit.info.max_degree(), BETA, GAMMA)
    pk, vk = dv.circuit_setup(circuit, powers, gamma, with_id=True)
    rng = random.Random(18)
    challenges = [rng.randrange(R) for _ in range(12)]
    xi = rng.randrange(R)
    cert = dv.prove_vk(pk, challenges, iter([xi, rng.randrange(R)]))
    check = dv.verify_vk(circuit, vk, cert, challenges, xi)
    z, combiners = vco.point_and_combiners(challenges)
    polys = circuit.index_polynomials()
    horner = lambda x: sum(c * _fr_mont_to_int(device.poly_evaluate(polys[name], dv._mont(x)))                # noqa: E731
                           for c, name in zip(combiners, dv.INDEX_POLYNOMIAL_NAMES)) % R
    assert check.matches and check.evaluation == horner(z)
    g = np.frombuffer(py.affine_bytes(py.G1_GENERATOR), dtype=np.uint8)
    w_scalar = xi * (horner(BETA) - check.evaluation) % R * pow(BETA - z, -1, R) % R
    assert (cert.w == oracle_cpu.g1_mul(g, osonic._scalars([w_scalar])[0])).all()
    assert (check.lhs == oracle_cpu.g1_mul(g, osonic._scalars([BETA * w_scalar % R])[0])).all()


def test_errors():
    import torch
    from snarkvm_b200 import launch_count
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import synthetic_srs
    circuit, _ = dv.test_circuit_csr(3, 5, 3, 100, 70, "cuda")
    D = circuit.info.max_degree()
    powers, gamma = synthetic_srs(D, BETA, GAMMA)
    pk, vk = dv.circuit_setup(circuit, powers, gamma, with_id=True)
    assert dv.circuit_setup(circuit, powers, gamma)[1].id is None         # the id only when asked for
    rng = random.Random(1)
    ch = [rng.randrange(R) for _ in range(12)]
    cert = dv.prove_vk(pk, ch, iter([5, 6]))
    torch.cuda.synchronize()
    before = launch_count()
    for bad in (ch[:11], ch + [1]):
        with pytest.raises(ValueError):
            dv.prove_vk(pk, bad, iter([5, 6]))
        with pytest.raises(ValueError):
            dv.verify_vk(circuit, vk, cert, bad, 5)
    with pytest.raises(ValueError):
        circuit.evaluate_index_polynomials(3, ch[:11])
    with pytest.raises(ValueError):                                       # one power short of max_degree + 1, id or not
        dv.circuit_setup(circuit, powers[:D].contiguous(), gamma, with_id=True)
    assert launch_count() == before
    # a verifying key of another circuit: the info or the id differs
    other, _ = dv.test_circuit_csr(3, 7, 3, 100, 70, "cuda")              # same shape, different witness: same matrices
    assert other.id() == circuit.id()
    assert dv.verify_vk(other, vk, cert, ch, 5).matches
    for c2 in (dv.test_circuit_csr(3, 5, 2, 100, 70, "cuda")[0], dv.test_circuit_csr(3, 5, 3, 128, 70, "cuda")[0]):
        assert c2.id() != vk.id
        assert not dv.verify_vk(c2, vk, cert, ch, 5).matches
    # the same counts and a changed value: only the id tells them apart
    one = np.tile(dv._mont(1), (100, 1))
    vals = one.copy()
    vals[0] = dv._mont(2)
    mats = [dv.Matrix(circuit.a.row_ptr.cpu().numpy(), m.cols.cpu().numpy(), v, "cuda") for m, v in ((circuit.a, vals), (circuit.b, one), (circuit.c, one))]
    changed = dv.Circuit(*mats, circuit.num_public, circuit.num_variables)
    assert changed.info == vk.circuit_info and changed.id() != vk.id
    res = dv.verify_vk(changed, vk, cert, ch, 5)
    assert not res.matches and len(vk.id) == 32
