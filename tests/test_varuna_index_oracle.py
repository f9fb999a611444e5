"""The circuit-setup restatement (tests/varuna_index_oracle.py) checked without a GPU: the index polynomials interpolate the indexer's
evaluations, they rebuild the prover's a(X) and b(X) of every matrix exactly as the verifier does (ahp/ahp.rs:416-444) — the prover
polynomials being pinned by the reference's circuit_0 vectors (tests/test_varuna_golden.py) — the label order is the reference's
string sort, max_degree / degree_bounds match hand-computed values, and on a setup with a known trapdoor every commitment is p(β)·G."""
import random

import numpy as np
import pytest

from oracle import bls12_377 as py
from oracle import varuna as ov

import varuna_index_oracle as vio

R = ov.R


def _circuit_0(golden):
    a, b = golden["varuna_circuit_0_prover"]["witness_a_b"]
    return ov.Circuit(ov.test_circuit(a, b, 3, 7, 7))


def _circuits(golden):
    yield "circuit_0", _circuit_0(golden)
    for shape in ((1, 16, 16), (3, 100, 70), (2, 50, 70)):
        yield f"test_circuit{shape}", ov.Circuit(ov.test_circuit(3, 5, *shape))
    yield "sparse", ov.Circuit(vio.sparse_r1cs(3, 4, 40, 37, (61, 64, 33)))


def test_fft_of_index_polynomials_equals_their_evaluations(golden):
    for name, circuit in _circuits(golden):
        polys, evals = vio.index_polynomials(circuit), vio.index_evaluations(circuit)
        doms = dict(zip("abc", circuit.non_zero_domains))
        assert list(polys) == list(vio.INDEX_ORDER)
        for label, p in polys.items():
            K = doms[label[-1]]
            assert len(p) <= K.size and len(evals[label]) == K.size
            assert K.fft(p) == evals[label], (name, label)
        # the padding of matrix_evals (matrices.rs:174-181): row = col = row_col = 1, row_col_val = 0 past the entries
        for m, nnz in zip("abc", vio.circuit_info(circuit)[3:]):
            for suffix, pad in (("row", 1), ("col", 1), ("row_col", 1), ("row_col_val", 0)):
                assert set(evals[f"{suffix}_{m}"][nnz:]) <= {pad}


def _prove(circuit, instances, alpha, eta_b, eta_c, beta, deltas, combs=None):
    p = ov.Prover(circuit, instances)
    p.first_round(); p.assignments(); p.second_round(1, combs)
    p.third_round(alpha, eta_b, eta_c, 1, combs)
    p.fourth_round(alpha, beta)
    p.fifth_round(deltas)
    return p


def _cases(golden):
    kat = golden["varuna_circuit_0_prover"]
    a, b = kat["witness_a_b"]
    ch = [int(x) for x in kat["challenges"]]
    alpha, _eta_a, eta_b, eta_c, beta, da, db, dc, gamma = ch
    yield "circuit_0 (KAT challenges)", _circuit_0(golden), [ov.test_circuit(a, b, 3, 7, 7)], (alpha, eta_b, eta_c, beta, [da, db, dc], gamma), None
    rng = random.Random(17)
    shape = (3, 30, 21)
    wit = [(rng.randrange(2, R), rng.randrange(2, R)) for _ in range(2)]
    r = lambda: rng.randrange(2, R)              # noqa: E731
    yield "batch of two", ov.Circuit(ov.test_circuit(wit[0][0], wit[0][1], *shape)), [ov.test_circuit(x, y, *shape) for x, y in wit], \
        (r(), r(), r(), r(), [r(), r(), r()], r()), [1, r()]


def test_index_polynomials_rebuild_the_prover_a_and_b(golden):
    """for every matrix: v_rc·row_col_val = a_poly_M and rc_size·(αβ − α·col − β·row + row_col) = b_poly_M, coefficient for coefficient"""
    for name, circuit, instances, (alpha, eta_b, eta_c, beta, deltas, _gamma), combs in _cases(golden):
        p = _prove(circuit, instances, alpha, eta_b, eta_c, beta, deltas, combs)
        polys = vio.index_polynomials(circuit)
        Rd, V = circuit.constraint_domain, circuit.variable_domain
        v_rc = Rd.evaluate_vanishing_polynomial(alpha) * V.evaluate_vanishing_polynomial(beta) % R
        for m, a_poly, b_poly in zip("abc", p.a_polys, p.b_polys):
            a, b = vio.verifier_a_b(polys, m, alpha, beta, v_rc, Rd.size * V.size)
            assert a == a_poly, (name, m)
            assert b == b_poly, (name, m)


def test_matrix_sumcheck_vanishes_with_the_verifiers_a_and_b(golden):
    """matrix_sumcheck(γ) = 0 (ahp.rs:384) when a_poly_M / b_poly_M are the verifier's combinations of the index polynomials"""
    for name, circuit, instances, (alpha, eta_b, eta_c, beta, deltas, gamma), combs in _cases(golden):
        p = _prove(circuit, instances, alpha, eta_b, eta_c, beta, deltas, combs)
        lcs, _qs = p.linear_combinations(alpha, eta_b, eta_c, beta, deltas, gamma, 1, combs)
        polys = vio.index_polynomials(circuit)
        Rd, V = circuit.constraint_domain, circuit.variable_domain
        v_rc = Rd.evaluate_vanishing_polynomial(alpha) * V.evaluate_vanishing_polynomial(beta) % R
        own = p.polynomials()
        for m in "abc":
            own[f"a_poly_{m}"], own[f"b_poly_{m}"] = vio.verifier_a_b(polys, m, alpha, beta, v_rc, Rd.size * V.size)
        terms = dict(lcs)["matrix_sumcheck"]
        assert sum(c * (1 if l is None else ov.poly_eval(own[l], gamma)) for c, l in terms) % R == 0, name
        assert any(l == "a_poly_a" for _, l in terms) and any(l == "b_poly_c" for _, l in terms)


def test_label_order_is_the_references_string_sort():
    rng = random.Random(4)
    for _ in range(3):
        cid = "".join(rng.choice("0123456789abcdef") for _ in range(64))
        labels = vio.index_labels(cid)
        assert len(set(labels)) == 12
        assert sorted(labels) == [f"circuit_{cid}_{n}" for n in vio.INDEX_ORDER]
    assert list(vio.INDEX_ORDER) == ["col_a", "col_b", "col_c", "row_a", "row_b", "row_c", "row_col_a", "row_col_b", "row_col_c",
                                     "row_col_val_a", "row_col_val_b", "row_col_val_c"]
    from snarkvm_b200 import varuna as dv
    assert dv.INDEX_POLYNOMIAL_NAMES == vio.INDEX_ORDER


@pytest.mark.parametrize("info,zk,want_degree,want_bounds", [
    # (num_public, num_variables, num_constraints, nnz_a, nnz_b, nnz_c)
    ((4, 7, 7, 7, 7, 7), False, 14, [6, 6, 6, 6]),                     # R = C = K = 8: max(2·8 − 2, 2·8 − 2, 8, 8, 7)
    ((4, 7, 7, 7, 7, 7), True, 16, [6, 6, 6, 6]),                      # + 2·zk_bound; mask v + 3 = 11
    ((2, 70, 100, 100, 100, 100), False, 254, [126, 126, 126, 126]),   # R = 128, C = 128, K = 128
    ((2, 1000, 10, 3000, 5, 3), False, 4095, [1022, 4094, 6, 2]),      # K = 4096: non_zero_domain_size − 1 beats 2·1024 − 2
    ((2, 1000, 10, 3000, 5, 3), True, 4095, [1022, 4094, 6, 2]),
    ((8, 4096, 4097, 20, 20, 20), True, 16384, [4094, 30, 30, 30]),    # R = 8192: 2·8192 + 2 − 2
    ((1, 3, 1, 2, 2, 2), True, 8, [2, 0, 0, 0]),                        # C = 4: mask v + 3 = 7 < 2·4 + 2 − 2 = 8
    ((1, 3, 1, 2, 2, 2), False, 6, [2, 0, 0, 0]),
])
def test_max_degree_and_degree_bounds(info, zk, want_degree, want_bounds):
    from snarkvm_b200 import varuna as dv
    assert vio.degree_bounds(info) == want_bounds
    assert vio.max_degree(info, zk) == want_degree
    dinfo = dv.CircuitInfo(*info)
    assert dinfo.degree_bounds() == want_bounds
    assert dinfo.max_degree(zk) == want_degree


def test_circuit_info_of_the_restated_indexer(golden):
    c0 = _circuit_0(golden)
    assert vio.circuit_info(c0) == (4, 7, 7, 7, 7, 7)                   # One + 3 public mul_vars: already a power of two
    assert vio.max_degree(vio.circuit_info(c0), False) == 14


def test_oracle_commitments_on_a_known_trapdoor(golden, oracle_cpu):
    """every commitment circuit_setup makes on (β^i·G, γβ^i·G) is p(β)·G for its index polynomial p"""
    from oracle import sonic as osonic
    beta, gamma = 0x5EED5EED1234567 % R, 0xABCDEF % R
    g = np.frombuffer(py.affine_bytes(py.G1_GENERATOR), dtype=np.uint8)
    for name, circuit in list(_circuits(golden))[:3]:
        info = vio.circuit_info(circuit)
        d = vio.max_degree(info, False)
        pts = lambda scale, n: np.stack([np.frombuffer(py.affine_bytes(py.projective_from_bytes(                    # noqa: E731
            oracle_cpu.g1_mul(g, osonic._scalars([scale * pow(beta, i, R) % R])[0]).tobytes())), dtype=np.uint8) for i in range(n)])
        powers, gpowers = pts(1, d + 1), pts(gamma, d + 2)
        got_info, comms = vio.circuit_setup(circuit, powers, gpowers, osonic.commit)
        assert got_info == info and len(comms) == 12
        polys = vio.index_polynomials(circuit)
        for label, c in zip(vio.INDEX_ORDER, comms):
            want = oracle_cpu.g1_mul(g, osonic._scalars([ov.poly_eval(polys[label], beta)])[0])
            assert (c == want).all(), (name, label)
        with pytest.raises(ValueError):
            vio.circuit_setup(circuit, powers[:d], gpowers, osonic.commit)
