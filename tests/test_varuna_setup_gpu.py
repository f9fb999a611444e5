"""GPU: Varuna circuit setup on the device — the indexer's evaluations and transposes (device.varuna_matrix_evals / csr_transpose),
the twelve index polynomials (Circuit.index_polynomials) and the verifying key's commitments (varuna.circuit_setup) — against the CPU
restatement (tests/varuna_index_oracle.py on oracle/varuna.py and oracle/sonic.py), on the real 2^15-point SRS without a trapdoor
through the prover's own a(X), b(X), and in closed form at 2^18 constraints."""
import os
import random
from collections import Counter

import numpy as np
import pytest

from oracle import bls12_377 as py
from oracle import sonic as osonic
from oracle import varuna as ov

import varuna_index_oracle as vio

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
R = ov.R
BETA, GAMMA = 0x1234567890ABCDEF1234567890ABCDEF % R, 0xFEDCBA0987654321FEDCBA % R


def _ints(t) -> list:
    """device Montgomery tensor [n, 4] → canonical ints"""
    from snarkvm_b200 import device
    if t.shape[0] == 0:
        return []
    h = device.fr_from_mont(t.contiguous()).cpu().numpy().view(np.uint64)
    return [int(r[0]) | int(r[1]) << 64 | int(r[2]) << 128 | int(r[3]) << 192 for r in h]


def _device_circuit(o_circuit):
    from snarkvm_b200 import varuna as dv
    mats = []
    for m in (o_circuit.a, o_circuit.b, o_circuit.c):
        row_ptr = np.concatenate([[0], np.cumsum([len(r) for r in m])]).astype(np.int64)
        cols = np.array([c for r in m for _, c in r], dtype=np.int64)
        vals = np.array([dv._mont(v) for r in m for v, _ in r], dtype=np.uint64).reshape(-1, 4)
        mats.append(dv.Matrix(row_ptr, cols, vals, "cuda"))
    return dv.Circuit(mats[0], mats[1], mats[2], o_circuit.num_public, o_circuit.num_variables)


def _kat_circuit(golden):
    a, b = golden["varuna_circuit_0_prover"]["witness_a_b"]
    return ov.Circuit(ov.test_circuit(a, b, 3, 7, 7))


CASES = {
    "circuit_0": None,
    # the four TestCircuit shapes of test_varuna_gpu.py
    "test_circuit_1_16_16": (1, 16, 16),
    "test_circuit_3_100_70": (3, 100, 70),
    "test_circuit_2_1024_1014": (2, 1 << 10, (1 << 10) - 10),
    "test_circuit_5_3000_4096": (5, 3000, 1 << 12),
    # random R1CS: empty rows, public columns, a public column in 300 rows of A (the long-row path of the transposed sparse_matvec),
    # nnz = 2^9 and 2^9 + 1, an empty C
    "sparse_hot_pow2_empty": ("sparse", 1, 8, 300, 400, (512, 513, 0), (5, 300)),
    "sparse_one_public": ("sparse", 2, 1, 50, 30, (64, 65, 16), (0, 0)),
    "sparse_tall": ("sparse", 3, 4, 100, 1000, (1024, 1025, 999), (0, 0)),
}


def _oracle_circuit(name, golden):
    spec = CASES[name]
    if spec is None:
        return _kat_circuit(golden)
    if spec[0] == "sparse":
        _, seed, npub, nprv, ncon, nnz, hot = spec
        return ov.Circuit(vio.sparse_r1cs(seed, npub, nprv, ncon, nnz, hot))
    return ov.Circuit(ov.test_circuit(3, 5, *spec))


@pytest.mark.parametrize("name", list(CASES))
def test_evaluations_transposes_and_index_polynomials_vs_oracle(name, golden):
    import torch
    from snarkvm_b200 import device
    oc = _oracle_circuit(name, golden)
    dc = _device_circuit(oc)
    assert [m.nnz for m in (dc.a, dc.b, dc.c)] == list(vio.circuit_info(oc)[3:])
    V = oc.variable_domain
    rng = random.Random(hash(name) & 0xFFFF)
    for m, om, arith, oarith, tm in zip("abc", (oc.a, oc.b, oc.c), dc.ariths, oc.ariths, dc.transposes):
        # matrix_evals, element by element, padding included
        assert arith.domain.size == oarith.domain.size
        assert _ints(arith.row) == oarith.row, (name, m)
        assert _ints(arith.col) == oarith.col, (name, m)
        assert _ints(arith.row_col_val) == oarith.row_col_val, (name, m)
        # transpose: the same matrix (a multiset of (value, row) per transposed row) …
        ot = ov.transpose(om, V, oc.input_domain)
        assert tm.nrows == V.size and tm.nnz == sum(len(r) for r in ot)
        ptr = tm.row_ptr.cpu().numpy().astype(np.int64)
        assert ptr[0] == 0 and (np.diff(ptr) == [len(r) for r in ot]).all(), (name, m)
        rows, vals = tm.cols.cpu().numpy(), _ints(tm.vals)
        for t, want in enumerate(ot):
            got = Counter(zip(vals[ptr[t]:ptr[t + 1]], rows[ptr[t]:ptr[t + 1]].tolist()))
            assert got == Counter(want), (name, m, t)
        # … and the same products through sparse_matvec on random vectors
        for _ in range(2):
            x = [rng.randrange(R) for _ in range(oc.num_constraints)]
            xd = torch.from_numpy(np.array([py.to_limbs(py.fr_to_mont(v), 4) for v in x], dtype=np.uint64).reshape(-1, 4).view(np.int64)).cuda()
            got = _ints(device.sparse_matvec(tm.row_ptr, tm.cols, tm.vals, xd))
            assert got == [sum(v * x[r] for v, r in col) % R for col in ot], (name, m)
    # MatrixArithmetization::new
    polys, want = dc.index_polynomials(), vio.index_polynomials(oc)
    assert list(polys) == list(vio.INDEX_ORDER)
    for label in vio.INDEX_ORDER:
        from snarkvm_b200 import varuna as dv
        assert polys[label].shape[0] == dict(zip("abc", oc.non_zero_domains))[label[-1]].size
        assert dv.trimmed(polys[label]) == want[label], (name, label)


@pytest.fixture(scope="module")
def synthetic():
    from snarkvm_b200 import sonic_pc
    D = 2047
    powers, gamma = sonic_pc.synthetic_srs(D, BETA, GAMMA)
    return powers, gamma, powers.cpu().numpy(), gamma.cpu().numpy()


@pytest.mark.parametrize("name", ["circuit_0", "test_circuit_3_100_70", "sparse_hot_pow2_empty", "sparse_one_public"])
def test_verifying_key_vs_oracle_on_a_synthetic_srs(name, golden, oracle_cpu, synthetic):
    from snarkvm_b200 import varuna as dv
    powers, gamma, hp, hg = synthetic
    oc = _oracle_circuit(name, golden)
    if name == "sparse_hot_pow2_empty":                                  # C is empty: its degree bound would be |K| − 2 = −1
        oc = ov.Circuit(vio.sparse_r1cs(1, 8, 300, 400, (512, 513, 2), (5, 300)))
    pk, vk = dv.circuit_setup(_device_circuit(oc), powers, gamma)
    info, want = vio.circuit_setup(oc, hp, hg, osonic.commit)
    assert vk.circuit_info == dv.CircuitInfo(*info)
    assert vk.circuit_commitments.shape == (12, 18)
    for label, got, w in zip(vio.INDEX_ORDER, vk.circuit_commitments, want):
        assert (got == w).all(), (name, label)
    assert pk.circuit_verifying_key is vk
    assert pk.committer_key.powers_of_beta_g.shape[0] == vio.max_degree(info, False) + 1
    assert pk.committer_key.enforced_degree_bounds == sorted(set(vio.degree_bounds(info)))


@pytest.fixture(scope="module")
def real_srs():
    import torch
    from helpers import affine_array
    blob = open(os.path.join(HERE, "golden", "powers_of_beta_15.usrs"), "rb").read()
    n = int.from_bytes(blob[:8], "little")
    host = affine_array(py.parse_usrs_points(blob, n))
    return host, torch.from_numpy(host).cuda()


def _combination(oracle_cpu, terms):
    """Σ scalar·point with the oracle's group law; points are normalised projective images (uint64[18]) or affine rows"""
    acc = None
    for scalar, point in terms:
        if point.dtype == np.uint64:
            p = py.projective_from_bytes(point.tobytes())
            if p is None or scalar % R == 0:
                continue
            point = np.frombuffer(py.affine_bytes(p), dtype=np.uint8)
        t = oracle_cpu.g1_mul(point, osonic._scalars([scalar])[0])
        acc = t if acc is None else oracle_cpu.g1_add(acc, t)
    return oracle_cpu.g1_normalise(acc) if acc is not None else osonic.INFINITY.copy()


@pytest.mark.parametrize("shape", [None, (2, 1 << 12, (1 << 12) - 10)])
def test_verifying_key_on_the_real_srs(shape, golden, oracle_cpu, real_srs):
    """the real powers of β (no trapdoor): the commitments equal the oracle's, and the prover's own a_poly_M / b_poly_M commit to the
    verifier's combinations of them (ahp.rs:430-444), v_rc·[row_col_val] and rc_size·(αβ·powers[0] − α·[col] − β·[row] + [row_col])"""
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import LabeledPolynomial, SonicKZG10
    host, powers = real_srs
    rng = random.Random(99)
    if shape is None:
        a, b = golden["varuna_circuit_0_prover"]["witness_a_b"]
        shape = (3, 7, 7)
    else:
        a, b = rng.randrange(2, R), rng.randrange(2, R)
    circuit, z = dv.test_circuit_csr(a, b, *shape, "cuda")
    oc = ov.Circuit(ov.test_circuit(a, b, *shape))
    # the gamma powers are only read by hiding commitments, which circuit setup never makes
    pk, vk = dv.circuit_setup(circuit, powers, powers)
    info, want = vio.circuit_setup(oc, host, host, osonic.commit)
    for label, got, w in zip(vio.INDEX_ORDER, vk.circuit_commitments, want):
        assert (got == w).all(), (shape, label)
    comm = dict(zip(vio.INDEX_ORDER, vk.circuit_commitments))
    alpha, beta = rng.randrange(2, R), rng.randrange(2, R)
    p = dv.Prover(circuit, [z])
    p.fourth_round(alpha, beta)
    Rd, V = circuit.constraint_domain, circuit.variable_domain
    v_rc = (pow(alpha, Rd.size, R) - 1) * (pow(beta, V.size, R) - 1) % R
    rc = Rd.size * V.size % R
    labeled = [LabeledPolynomial(f"{k}_{m}", t) for m, a_poly, b_poly in zip("abc", p.a_polys, p.b_polys) for k, t in (("a", a_poly), ("b", b_poly))]
    got, _ = SonicKZG10.commit(pk.committer_key, labeled)
    for i, m in enumerate("abc"):
        want_a = _combination(oracle_cpu, [(v_rc, comm[f"row_col_val_{m}"])])
        want_b = _combination(oracle_cpu, [(rc * alpha * beta % R, host[0]), (-rc * alpha % R, comm[f"col_{m}"]),
                                           (-rc * beta % R, comm[f"row_{m}"]), (rc, comm[f"row_col_{m}"])])
        assert (got[2 * i] == want_a).all(), (shape, "a", m)
        assert (got[2 * i + 1] == want_b).all(), (shape, "b", m)


def test_verifying_key_closed_form_at_2_18(oracle_cpu):
    """TestCircuit with 2^18 constraints: every commitment is p(β)·G with p(β) = Σ_k e_k·L_k(β) over K from the evaluations e the
    circuit's shape determines — row ω^k, col ω_C^{reindex(col)}, row_col = row_col_val = row·col (every value is one)"""
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import synthetic_srs
    n = 1 << 18
    circuit, _z = dv.test_circuit_csr(3, 5, 2, n, n - 10, "cuda")
    assert circuit.num_public == 4 and circuit.variable_domain.size == n and circuit.max_non_zero_domain.size == n
    D = circuit.info.max_degree()
    assert D == 2 * n - 2
    powers, gamma = synthetic_srs(D, BETA, GAMMA)
    _pk, vk = dv.circuit_setup(circuit, powers, gamma)
    w = py.fr_root_of_unity(n)
    elems = [1] * n
    for k in range(1, n):
        elems[k] = elems[k - 1] * w % R
    # L_k(β) = (β^n − 1)/n · ω^k / (β − ω^k), by one batch inversion
    den = [(BETA - e) % R for e in elems]
    pre = [1] * (n + 1)
    for k in range(n):
        pre[k + 1] = pre[k] * den[k] % R
    inv = pow(pre[n], -1, R)
    lag = [0] * n
    scale = (pow(BETA, n, R) - 1) * pow(n, -1, R) % R
    for k in range(n - 1, -1, -1):
        lag[k] = scale * elems[k] % R * (inv * pre[k] % R) % R
        inv = inv * den[k] % R
    # padded = 4 public variables, private a = 4, b = 5, mul_vars 1, 2 (test_circuit_csr); period = |C| / |I| = 2^16
    reindex = lambda c: c * (n // 4) if c < 4 else (c - 4) + (c - 4) // (n // 4 - 1) + 1      # noqa: E731
    cols = {"a": [4] * (n - 1) + [1], "b": [5] * n, "c": [1] * (n - 1) + [2]}
    value = {}
    value["row"] = sum(e * l for e, l in zip(elems, lag)) % R
    for m, cl in cols.items():
        ce = {c: elems[reindex(c)] for c in set(cl)}                    # ω_C = ω_K here: both domains have 2^18 elements
        value[f"col_{m}"] = sum(ce[c] * l for c, l in zip(cl, lag)) % R
        value[f"row_col_{m}"] = sum(e * ce[c] % R * l for e, c, l in zip(elems, cl, lag)) % R
    g = np.frombuffer(py.affine_bytes(py.G1_GENERATOR), dtype=np.uint8)
    assert value["row"] == BETA                                          # row evaluations are the domain itself: row(X) = X
    for label, got in zip(vio.INDEX_ORDER, vk.circuit_commitments):
        kind, m = label.rsplit("_", 1)
        v = value["row"] if kind == "row" else value[f"row_col_{m}"] if kind == "row_col_val" else value[f"{kind}_{m}"]
        assert (got == oracle_cpu.g1_mul(g, osonic._scalars([v])[0])).all(), label


def test_errors():
    import torch
    from snarkvm_b200 import CudaError, device, launch_count
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import synthetic_srs
    circuit, _ = dv.test_circuit_csr(3, 5, 3, 100, 70, "cuda")
    D = circuit.info.max_degree()
    powers, gamma = synthetic_srs(D, BETA, GAMMA)
    torch.cuda.synchronize()
    before = launch_count()
    with pytest.raises(ValueError):                                      # one power short of max_degree + 1
        dv.circuit_setup(circuit, powers[:D].contiguous(), gamma)
    assert launch_count() == before
    dv.circuit_setup(circuit, powers, gamma)                             # exactly max_degree + 1 powers is enough
    # |C| = |I|: reindex_by_subdomain has no room for the private variables
    one = np.tile(dv._mont(1), (4, 1))
    mats = [dv.Matrix(np.arange(5), np.array([0, 1, 2, 3]), one, "cuda") for _ in range(3)]
    before = launch_count()
    with pytest.raises(ValueError):
        dv.Circuit(mats[0], mats[1], mats[2], 4, 4)
    assert launch_count() == before
    # a column ≥ num_variables
    bad = dv.Matrix(np.arange(5), np.array([0, 5, 2, 8]), one, "cuda")
    with pytest.raises(CudaError):
        dv.Circuit(bad, mats[1], mats[2], 4, 8)
    with pytest.raises(CudaError):
        device.csr_transpose(bad.row_ptr, bad.cols, bad.vals, 8, 4, 3)
    with pytest.raises(CudaError):
        device.varuna_matrix_evals(bad.row_ptr, bad.cols, bad.vals, 8, 4, 2, 3, 2)
    # the same matrix with its columns in range goes through both
    ok = dv.Matrix(np.arange(5), np.array([0, 5, 2, 7]), one, "cuda")
    c = dv.Circuit(ok, mats[1], mats[2], 4, 8)
    assert _ints(c.transposes[0].vals) == [1, 1, 1, 1]
