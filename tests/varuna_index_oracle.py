"""TEST INFRASTRUCTURE ONLY — CPU restatement (Python big integers) of Varuna's circuit setup, on top of oracle/varuna.py's indexer
and oracle/sonic.py's commit.

Restates, from algorithms/src/snark/varuna:
    ahp/indexer/indexer.rs:104-115, varuna.rs:116    index_polynomial_labels_single, the label sort   → index_labels / INDEX_ORDER
    ahp/indexer/indexer.rs:169-176                  CircuitInfo                                        → circuit_info
    ahp/ahp.rs:85-107, circuit_info.rs:43-46         max_degree (zk_bound 0 or 1)                       → max_degree
    ahp/ahp.rs:110-121                              get_degree_bounds                                  → degree_bounds
    ahp/matrices.rs:211-240                         MatrixArithmetization::new                         → index_polynomials
    ahp/ahp.rs:416-444                              the verifier's a(X), b(X) from the index polynomials → verifier_a_b
    varuna.rs:72-134                                batch_circuit_setup for one circuit               → circuit_setup
Polynomials are trimmed coefficient lists of canonical integers, as in oracle/varuna.py.
"""
from __future__ import annotations

from oracle import varuna as ov

R = ov.R
MATRICES = "abc"
NAMES = ("row", "col", "row_col", "row_col_val")                   # index_polynomial_labels_single order
# the twelve polynomials in label order: circuit_{id}_ is a common prefix, so the sort only sees "{name}_{matrix}"
INDEX_ORDER = tuple(f"{n}_{m}" for n in ("col", "row", "row_col", "row_col_val") for m in MATRICES)


def index_labels(circuit_id: str) -> list:
    """every label of the index, in generation order (interpolate_matrix_evals: a, b, c; then indexer.rs:108-113 per matrix)"""
    return [f"circuit_{circuit_id}_{n}_{m}" for m in MATRICES for n in NAMES]


def circuit_info(circuit: ov.Circuit) -> tuple:
    """(num_public_inputs, num_public_and_private_variables, num_constraints, num_non_zero_a, num_non_zero_b, num_non_zero_c)"""
    nnz = [sum(len(r) for r in m) for m in (circuit.a, circuit.b, circuit.c)]
    return (circuit.num_public, circuit.num_variables, circuit.num_constraints, *nnz)


def _size(n: int) -> int:
    return ov.Domain(n).size                                        # compute_size_of_domain


def max_degree(info: tuple, zk: bool) -> int:
    _, num_variables, num_constraints, na, nb, nc = info
    zk_bound = 1 if zk else 0
    r, v, k = _size(num_constraints), _size(num_variables), _size(max(na, nb, nc))
    return max([2 * r + 2 * zk_bound - 2, 2 * v + 2 * zk_bound - 2, v + 3 if zk else 0, v, r, k - 1])


def degree_bounds(info: tuple) -> list:
    _, num_variables, _, na, nb, nc = info
    return [_size(num_variables) - 2, _size(na) - 2, _size(nb) - 2, _size(nc) - 2]


def index_evaluations(circuit: ov.Circuit) -> dict:
    """the evaluations on K each index polynomial interpolates: row, col, row_col (row·col, padding 1·1) and row_col_val"""
    out = {}
    for m, arith in zip(MATRICES, circuit.ariths):
        out[f"row_{m}"] = list(arith.row)
        out[f"col_{m}"] = list(arith.col)
        out[f"row_col_{m}"] = [r * c % R for r, c in zip(arith.row, arith.col)]
        out[f"row_col_val_{m}"] = list(arith.row_col_val)
    return out


def index_polynomials(circuit: ov.Circuit) -> dict:
    """MatrixArithmetization::new for A, B, C: name → the iFFT over that matrix's K of its evaluations"""
    evals = index_evaluations(circuit)
    doms = dict(zip(MATRICES, circuit.non_zero_domains))
    return {name: doms[name[-1]].ifft(evals[name]) for name in INDEX_ORDER}


def verifier_a_b(polys: dict, m: str, alpha: int, beta: int, v_rc: int, rc_size: int):
    """construct_matrix_linear_combinations (ahp.rs:430-444) as polynomials: a = v_rc·row_col_val,
    b = rc_size·(αβ − α·col − β·row + row_col)"""
    a = ov.poly_scale(polys[f"row_col_val_{m}"], v_rc)
    b = ov.poly_add([alpha * beta % R], ov.poly_scale(polys[f"col_{m}"], -alpha % R))
    b = ov.poly_add(b, ov.poly_scale(polys[f"row_{m}"], -beta % R))
    b = ov.poly_add(b, polys[f"row_col_{m}"])
    return a, ov.poly_scale(b, rc_size % R)


def sparse_r1cs(seed: int, num_public: int, num_private: int, num_constraints: int, nnz: tuple, hot: tuple = (0, 0)) -> ov.ConstraintSystem:
    """a constraint system whose A, B, C hold exactly nnz[0], nnz[1], nnz[2] entries at random distinct (row, variable) positions with
    random non-zero coefficients (rows without entries and public columns come naturally); hot = (variable, rows): A also uses that
    variable in its first `rows` rows.  num_public (One included) should be a power of two so padding leaves it alone.  The
    assignment is random: the system indexes, it is not satisfied."""
    import random
    rng = random.Random(seed)
    cs = ov.ConstraintSystem()
    for _ in range(num_public - 1):
        cs.alloc_input(rng.randrange(R))
    for _ in range(num_private):
        cs.alloc(rng.randrange(R))
    nv = num_public + num_private
    var = lambda v: ("pub", v) if v < num_public else ("priv", v - num_public)       # noqa: E731
    rows = []
    for k, n in enumerate(nnz):
        cells = set((r, hot[0]) for r in range(hot[1])) if k == 0 else set()
        assert n <= num_constraints * nv and len(cells) <= n
        while len(cells) < n:
            cells.add((rng.randrange(num_constraints), rng.randrange(nv)))
        m = [[] for _ in range(num_constraints)]
        for r, v in sorted(cells):
            m[r].append((rng.randrange(1, R), var(v)))
        rows.append(m)
    for a, b, c in zip(*rows):
        cs.enforce(a, b, c)
    return cs


def circuit_setup(circuit: ov.Circuit, pp_powers, pp_gamma_powers, commit, zk: bool = False):
    """batch_circuit_setup for one circuit (varuna.rs:72-134) → (circuit_info, [commitment] in INDEX_ORDER).  `commit` is
    oracle/sonic.py's commit; pp_powers / pp_gamma_powers are the SRS arrays oracle/sonic.py's CommitterKey takes."""
    from oracle import sonic as osonic
    info = circuit_info(circuit)
    d = max_degree(info, zk)
    if len(pp_powers) < d + 1:
        raise ValueError("the SRS does not support the circuit's max degree")
    ck = osonic.CommitterKey(pp_powers, pp_gamma_powers, d, (), 1, degree_bounds(info))
    polys = index_polynomials(circuit)
    comms, rands = commit(ck, [(name, polys[name], None, None, False) for name in INDEX_ORDER])
    assert all(r is None for r in rands)                            # varuna.rs:112-113: no randomness
    return info, comms
