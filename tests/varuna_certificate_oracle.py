"""TEST INFRASTRUCTURE ONLY — CPU restatement (Python big integers) of Varuna's verifying-key certificate, on top of oracle/varuna.py's
indexer, oracle/sonic.py's open_combinations and tests/varuna_index_oracle.py's index polynomials.

Restates, from algorithms/src:
    snark/varuna/ahp/indexer/circuit.rs:109-121     Circuit::hash (Blake2s-256 of CircuitInfo, A, B, C) → id_stream / circuit_id
    snark/varuna/varuna.rs:236-276                  prove_vk after the sponge                         → prove_vk
    snark/varuna/ahp/indexer/indexer.rs:232-260     evaluate_index_polynomials                        → evaluate_index_polynomials
    snark/varuna/ahp/matrices.rs:114-126            MatrixEvals::evaluate                             → matrix_evals_dot
    snark/varuna/varuna.rs:280-331 + polycommit/sonic_pc/mod.rs:344-411, 477-544, 582-635
                                                    verify_vk up to check_elems' pairing, one point   → verify_vk
The serialization follows utilities/src/serialize/impls.rs (u64 LE length prefixes, usize as u64 LE) and fields/src/macros.rs:190-245
(an Fr is its 32 canonical LE bytes with empty flags).  The sponge stays with the caller: challenges are arguments.
"""
from __future__ import annotations

import hashlib
import struct

import numpy as np

from oracle import sonic as osonic
from oracle import varuna as ov

import varuna_index_oracle as vio

R = ov.R


def id_stream(matrix) -> bytes:
    """serialize_uncompressed of a Matrix = Vec<Vec<(Fr, usize)>>: [u64 nrows], per row [u64 len][len × (32 B value, u64 column)]"""
    out = [struct.pack("<Q", len(matrix))]
    for row in matrix:
        out.append(struct.pack("<Q", len(row)))
        for val, col in row:
            out.append((val % R).to_bytes(32, "little") + struct.pack("<Q", col))
    return b"".join(out)


def circuit_info_bytes(info: tuple) -> bytes:
    """CircuitInfo: its six usize fields as u64 LE, in declaration order (circuit_info.rs:24-38)"""
    return struct.pack("<6Q", *info)


def circuit_id(circuit: ov.Circuit) -> bytes:
    h = hashlib.blake2s(digest_size=32)
    h.update(circuit_info_bytes(vio.circuit_info(circuit)))
    for m in (circuit.a, circuit.b, circuit.c):
        h.update(id_stream(m))
    return h.digest()


def point_and_combiners(challenges) -> tuple:
    """squeeze_nonnative_field_elements(12) → (point = the last, combiners = [1] + the first eleven)"""
    challenges = [int(c) % R for c in challenges]
    assert len(challenges) == 12
    return challenges[-1], [1] + challenges[:-1]


def prove_vk(pp_powers, pp_gamma_powers, circuit: ov.Circuit, challenges, opening_challenges):
    """the certificate's w: open_combinations of circuit_check = Σ c_i·p_i (label order) at the point, empty randomness, on the
    committer key circuit_setup trims"""
    point, combiners = point_and_combiners(challenges)
    info = vio.circuit_info(circuit)
    ck = osonic.CommitterKey(pp_powers, pp_gamma_powers, vio.max_degree(info, False), (), 1, vio.degree_bounds(info))
    polys = vio.index_polynomials(circuit)
    lc = [("circuit_check", [(c, name) for c, name in zip(combiners, vio.INDEX_ORDER)])]
    (w, random_v), = osonic.open_combinations(ck, lc, {name: (polys[name], None, None) for name in vio.INDEX_ORDER},
                                              [("circuit_check", ("challenge", point))], iter(opening_challenges))
    assert random_v is None
    return w


def matrix_evals_dot(arith: ov.MatrixEvals, lagrange: list) -> list:
    """MatrixEvals::evaluate: [Σ l·row, Σ l·col, Σ l·row·col, Σ l·row_col_val]"""
    return [sum(l * r for l, r in zip(lagrange, arith.row)) % R,
            sum(l * c for l, c in zip(lagrange, arith.col)) % R,
            sum(l * r % R * c for l, r, c in zip(lagrange, arith.row, arith.col)) % R,
            sum(l * v for l, v in zip(lagrange, arith.row_col_val)) % R]


def index_evaluations_at(circuit: ov.Circuit, point: int) -> dict:
    """name → p_name(point), through each K's Lagrange coefficients at the point"""
    out = {}
    for m, arith in zip(vio.MATRICES, circuit.ariths):
        lag = arith.domain.evaluate_all_lagrange_coefficients(point % R)
        for name, v in zip(vio.NAMES, matrix_evals_dot(arith, lag)):
            out[f"{name}_{m}"] = v
    return out


def evaluate_index_polynomials(circuit: ov.Circuit, point: int, combiners) -> int:
    evals = index_evaluations_at(circuit, point)
    combiners = list(combiners)
    assert len(combiners) == 12
    return sum(c * evals[name] for c, name in zip(combiners, vio.INDEX_ORDER)) % R


def affine(projective: np.ndarray) -> np.ndarray:
    """normalised projective image uint64[18] → 104-byte Affine image (x, y, infinity flag, padding)"""
    limbs = np.ascontiguousarray(projective, dtype=np.uint64).reshape(18)
    out = np.zeros(104, dtype=np.uint8)
    out[:96] = limbs[:12].view(np.uint8)
    out[96] = 0 if limbs[12:].any() else 1
    return out


def verify_vk(circuit: ov.Circuit, vk_info: tuple, vk_id: bytes, commitments, w: np.ndarray, g_affine: np.ndarray, challenges,
              opening_challenge: int):
    """→ (matches, evaluation, lhs): matches = the re-indexed circuit's info and id equal the verifying key's; lhs = ξ·Σ c_i·C_i −
    ξ·v·G + z·W, the G1 element check_elems pairs with H (randomizer one, one point; W pairs with β·H)"""
    point, combiners = point_and_combiners(challenges)
    xi = int(opening_challenge) % R
    matches = vio.circuit_info(circuit) == tuple(vk_info) and circuit_id(circuit) == vk_id
    v = evaluate_index_polynomials(circuit, point, combiners)
    bases = np.stack([affine(c) for c in commitments] + [g_affine, affine(w)])
    lhs = osonic.msm(bases, [xi * c % R for c in combiners] + [(-xi * v) % R, point])
    return matches, v, lhs
