"""Varuna AHP prover rounds with every polynomial resident in HBM (SURVEY §8 f3).

Device-side mirror of /root/reference/algorithms/src/snark/varuna for the part of `prove_batch` (varuna.rs:336-620) that is
bulk field arithmetic — the five `AHPForR1CS::prover_*_round` functions and the indexer's arithmetization:

    ahp/indexer/indexer.rs:121-200, ahp/matrices.rs:138-195, 249-270   Circuit            (domains, row / col / row_col_val on K, transposes)
    ahp/matrices.rs:211-240                        Circuit.index_polynomials (MatrixArithmetization::new)
    varuna.rs:72-134, 226-233                      circuit_setup        (the verifying key's twelve index commitments)
    ahp/indexer/circuit.rs:109-121                 Circuit.id           (Blake2s of the index counts and the serialized matrices)
    varuna.rs:155-165, 236-331                     certificate_challenges (the certificate's Poseidon transcript)
    varuna.rs:236-276                              prove_vk             (the verifying-key certificate)
    ahp/indexer/indexer.rs:232-260                 Circuit.evaluate_index_polynomials
    varuna.rs:280-331                              verify_vk            (up to the final pairing)
    varuna.rs:136-194, 336-620                     prove_batch          (the transcript, the rounds, the commitments and openings → Proof)
    ahp/verifier/verifier.rs:39-197                Transcript squeezes  (the verifier's messages the prover draws)
    ahp/prover/round_functions/mod.rs:43-192, ahp/prover/state.rs:107-178   init_prover   (z_A, z_B, z_C by sparse mat-vec, x_poly)
    ahp/prover/round_functions/first.rs:129-160    prover_first_round   (w)
    ahp/prover/round_functions/third.rs:207-234    calculate_assignments (z)
    ahp/prover/round_functions/second.rs:77-146    prover_second_round  (h_0)
    ahp/prover/round_functions/third.rs:126-326    prover_third_round   (g_1, h_1, lineval sums)
    ahp/prover/round_functions/fourth.rs:151-245   prover_fourth_round  (g_a, g_b, g_c, sums)
    ahp/prover/round_functions/fifth.rs:41-67      prover_fifth_round   (h_2)
    ahp/selectors.rs:70-123                        apply_randomized_selector

for the NON-HIDING mode (VarunaNonHidingMode), one circuit, any batch of instances.  Everything O(n) runs in this library's
kernels (NTT passes, PolyMultiplier pipeline, divide_by_vanishing_poly, batch inversion, sparse mat-vec, elementwise Fr ops);
torch only owns the buffers and does index plumbing (gathers, concatenation).  The rounds take their challenges as host scalars;
prove_batch draws them from its own Fiat–Shamir transcript (Transcript, a resumable PoseidonSponge<Fq, 2, 1> on csrc/poseidon.cu),
and certificate_challenges draws a certificate's.
Polynomials are CUDA tensors [m, 4] int64 (Montgomery Fr, low degree first, NOT trimmed: trailing zero coefficients may be present;
`trimmed()` gives the reference's canonical form on the host).
"""
from __future__ import annotations

import hashlib
import random
import struct
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass

import numpy as np
import torch

from . import device, poseidon
from ._lib import CudaError
from .algorithms import EvaluationDomain, _fr_int_to_mont, _fr_mont_to_int
from .cuda import NTTDirection, NTTType
from .sonic_pc import check_combinations_scalars

R_MOD = 8444461749428370424248824938781546531375899335154063827935233455917409239041   # curves/src/bls12_377/fr.rs:138-145


def _mont(v: int) -> np.ndarray:
    return _fr_int_to_mont(v % R_MOD)


def _zeros(n: int, dev) -> torch.Tensor:
    return torch.zeros((n, 4), dtype=torch.int64, device=dev)


def _pad(x: torch.Tensor, n: int) -> torch.Tensor:
    if x.shape[0] == n:
        return x
    out = _zeros(n, x.device)
    out[: x.shape[0]] = x[:n]
    return out


def _scale(x: torch.Tensor, k: int) -> torch.Tensor:
    if x.shape[0] == 0 or k % R_MOD == 1:
        return x
    return device.fr_vec_op(x, _mont(k), device.FR_MUL)


def _add(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """a + b for polynomials of different lengths"""
    if a.shape[0] < b.shape[0]:
        a, b = b, a
    if b.shape[0] == 0:
        return a
    out = a.clone()
    device.fr_vec_op(out[: b.shape[0]], b, device.FR_ADD, out=out[: b.shape[0]])
    return out


def _sub(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    n = max(a.shape[0], b.shape[0])
    out = _pad(a, n).clone() if a.shape[0] == n else _pad(a, n)
    if b.shape[0]:
        device.fr_vec_op(out[: b.shape[0]], b, device.FR_SUB, out=out[: b.shape[0]])
    return out


def trimmed(poly: torch.Tensor) -> list:
    """host copy as canonical integers with trailing zeros removed (DensePolynomial::from_coefficients_vec, dense.rs:61-66)"""
    h = device.fr_from_mont(poly).cpu().numpy().view(np.uint64) if poly.shape[0] else np.zeros((0, 4), dtype=np.uint64)
    vals = [sum(int(v) << (64 * i) for i, v in enumerate(row)) for row in h]
    while vals and vals[-1] == 0:
        vals.pop()
    return vals


def polymul(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """PolyMultiplier::multiply of two coefficient vectors (fft/polynomial/multiplier.rs:70-134)"""
    if a.shape[0] == 0 or b.shape[0] == 0:
        return _zeros(0, a.device)
    dom = EvaluationDomain.new(a.shape[0] + b.shape[0] - 1)
    return device.polymul([a.contiguous(), b.contiguous()], [], dom.log_size_of_group)


def divide_by_vanishing(p: torch.Tensor, domain: EvaluationDomain):
    return device.poly_divide_by_vanishing(p.contiguous(), domain.size)


def mul_by_vanishing(p: torch.Tensor, domain: EvaluationDomain) -> torch.Tensor:
    """DensePolynomial::mul_by_vanishing_poly (dense.rs:153-158): p·(x^n − 1)"""
    n, m = domain.size, p.shape[0]
    out = _zeros(n + m, p.device)
    out[n:] = p
    device.fr_vec_op(out[:m], p, device.FR_SUB, out=out[:m])       # out[:m] −= p (for m > n the shifted copy is already there)
    return out


def apply_randomized_selector(poly: torch.Tensor, combiner: int, target: EvaluationDomain, src: EvaluationDomain, remainder_witness: bool):
    """ahp/selectors.rs:70-123"""
    multiplier = combiner * src.size % R_MOD * pow(target.size, -1, R_MOD) % R_MOD
    if not remainder_witness:
        h, _rem = divide_by_vanishing(poly, src)               # the reference asserts a zero remainder; parity tests check the result
        return _scale(h, multiplier), None
    poly = _scale(poly, multiplier)
    h, xg = divide_by_vanishing(poly, src)
    if target.size != src.size:
        xg = mul_by_vanishing(xg, target)
        xg, _rem = divide_by_vanishing(xg, src)
    return h, xg


class Matrix:
    """A sparse R1CS matrix in CSR form on the device: row_ptr int32 [nrows + 1], cols int32 [nnz] (variable indices: public first,
    then private — into_matrix_helper, ahp/matrices.rs:39-63), vals [nnz, 4] int64 Montgomery.  The arrays are uploaded once; no
    host copy is kept."""

    def __init__(self, row_ptr: np.ndarray, cols: np.ndarray, vals_mont: np.ndarray, dev):
        self.nrows, self.nnz = len(row_ptr) - 1, len(cols)
        self.row_ptr = torch.from_numpy(np.ascontiguousarray(row_ptr, dtype=np.int32)).to(dev)
        self.cols = torch.from_numpy(np.ascontiguousarray(cols, dtype=np.int32)).to(dev)
        self.vals = torch.from_numpy(np.ascontiguousarray(vals_mont, dtype=np.uint64).reshape(-1, 4).view(np.int64)).to(dev)

    @classmethod
    def from_device(cls, row_ptr: torch.Tensor, cols: torch.Tensor, vals: torch.Tensor) -> "Matrix":
        m = cls.__new__(cls)
        m.nrows, m.nnz = row_ptr.numel() - 1, cols.numel()
        m.row_ptr, m.cols, m.vals = row_ptr, cols, vals
        return m

    def serialize(self) -> torch.Tensor:
        """the matrix's part of the circuit id's byte stream (serialize_uncompressed of Vec<Vec<(Fr, usize)>>), built on the device
        → CUDA uint8 tensor of 8 + 8·nrows + 40·nnz bytes.  It equals the reference's bytes when every row holds its entries as
        into_matrix_helper leaves them (ahp/matrices.rs:39-63): columns increasing, no repeats, no zero values."""
        return device.csr_serialize(self.row_ptr, self.cols, self.vals)


class MatrixEvals:
    """ahp/matrices.rs:102-136: row, col, row_col_val evaluations on the non-zero domain K"""

    def __init__(self, row, col, row_col_val, domain):
        self.row, self.col, self.row_col_val, self.domain = row, col, row_col_val, domain


_domain_size = EvaluationDomain.compute_size_of_domain            # fft/domain.rs:151-154


@dataclass(frozen=True)
class CircuitInfo:
    """ahp/indexer/circuit_info.rs: the six counts index_helper records (ahp/indexer/indexer.rs:169-176)"""
    num_public_inputs: int
    num_public_and_private_variables: int
    num_constraints: int
    num_non_zero_a: int
    num_non_zero_b: int
    num_non_zero_c: int

    def max_degree(self, zk: bool = False) -> int:
        """CircuitInfo::max_degree → AHPForR1CS::max_degree (circuit_info.rs:43-46, ahp/ahp.rs:85-107); zk_bound is 1 in the hiding
        mode, 0 otherwise"""
        zk_bound = 1 if zk else 0
        r = _domain_size(self.num_constraints)
        v = _domain_size(self.num_public_and_private_variables)
        k = _domain_size(max(self.num_non_zero_a, self.num_non_zero_b, self.num_non_zero_c))
        return max(2 * r + 2 * zk_bound - 2, 2 * v + 2 * zk_bound - 2, v + 3 if zk else 0, v, r, k - 1)

    def degree_bounds(self) -> list:
        """AHPForR1CS::get_degree_bounds (ahp/ahp.rs:110-121): the bounds of g_1, g_a, g_b, g_c"""
        return [_domain_size(n) - 2 for n in (self.num_public_and_private_variables, self.num_non_zero_a, self.num_non_zero_b,
                                               self.num_non_zero_c)]

    def to_bytes_le(self) -> bytes:
        """the six counts as u64 LE (ToBytes, circuit_info.rs:49-58; the derived serialize_uncompressed writes the same bytes)"""
        return struct.pack("<6Q", self.num_public_inputs, self.num_public_and_private_variables, self.num_constraints,
                           self.num_non_zero_a, self.num_non_zero_b, self.num_non_zero_c)


# the twelve index polynomials in the order of their labels circuit_{id}_{name}_{matrix} sorted as strings (varuna.rs:116), which
# is the same for every circuit id
INDEX_POLYNOMIAL_NAMES = tuple(f"{p}_{m}" for p in ("col", "row", "row_col", "row_col_val") for m in "abc")


class Circuit:
    """AHPForR1CS::index_helper (ahp/indexer/indexer.rs:121-200) for the non-hiding mode: the caller has already padded the public
    variables to a power of two (pad_input_for_indexer_and_prover, ahp/matrices.rs:85-100).  The evaluations on K are built on the
    device from the CSR arrays (index_circuits, which indexes many circuits in one pass; this constructor is its batch of one).  The
    transposes are prover data: they are built on first use (device.csr_transpose), so setup and certificates never pay for them."""

    def __init__(self, a: Matrix, b: Matrix, c: Matrix, num_public: int, num_variables: int):
        self._shape(a, b, c, num_public, num_variables)
        _matrix_evals([self])

    def _shape(self, a: Matrix, b: Matrix, c: Matrix, num_public: int, num_variables: int):
        """the domains and counts; no launch"""
        self.a, self.b, self.c = a, b, c
        self.num_public, self.num_variables, self.num_constraints = num_public, num_variables, a.nrows
        if num_public & (num_public - 1):
            raise ValueError("public variables must be padded to a power of two")
        self.constraint_domain = EvaluationDomain.new(self.num_constraints)
        self.variable_domain = EvaluationDomain.new(num_variables)
        self.input_domain = EvaluationDomain.new(num_public)
        if self.variable_domain.size <= self.input_domain.size:          # reindex_by_subdomain (fft/domain.rs:327-329)
            raise ValueError("other.size() must be smaller than self.size()")
        self.non_zero_domains = [EvaluationDomain.new(m.nnz) for m in (a, b, c)]
        self.max_non_zero_domain = max(self.non_zero_domains, key=lambda d: d.size)
        self.info = CircuitInfo(num_public, num_variables, self.num_constraints, a.nnz, b.nnz, c.nnz)
        self.ariths, self._transposes = [], None

    @property
    def transposes(self) -> list:
        """transpose (ahp/matrices.rs:249-270) of A, B, C over the variable domain, built on the first call"""
        if self._transposes is None:
            lg_c = self.variable_domain.log_size_of_group
            self._transposes = [Matrix.from_device(*device.csr_transpose(m.row_ptr, m.cols, m.vals, self.num_variables,
                                                                         self.input_domain.size, lg_c)) for m in (self.a, self.b, self.c)]
        return self._transposes

    def index_polynomials(self) -> dict:
        """MatrixArithmetization::new (ahp/matrices.rs:211-240) for A, B, C: the iFFT over each matrix's K of row, col, row_col
        (= row∘col, padding 1·1 = 1) and row_col_val → {name: [|K|, 4] i64 Montgomery coefficients} in INDEX_POLYNOMIAL_NAMES order"""
        return index_polynomials([self])[0]

    def id(self) -> bytes:
        """Circuit::hash (ahp/indexer/circuit.rs:109-121): Blake2s-256 of CircuitInfo and of A, B, C serialized uncompressed
        (circuit_ids for one circuit).  Computed once, then cached."""
        return circuit_ids([self])[0]

    _id = None

    def evaluate_index_polynomials(self, point: int, combiners) -> int:
        """AHPForR1CS::evaluate_index_polynomials (ahp/indexer/indexer.rs:232-260): Σ_i combiners_i·p_i(point) over the twelve index
        polynomials in INDEX_POLYNOMIAL_NAMES (= label) order, from their evaluations on K through the Lagrange coefficients of each
        matrix's K at the point (a point inside K included, fft/domain.rs:258-292); no polynomial is interpolated."""
        return evaluate_index_polynomials([self], [point], [combiners])[0]


def _device_of(circuits: list):
    """the one device every circuit lives on"""
    devs = {c.a.row_ptr.device for c in circuits}
    if len(devs) != 1:
        raise ValueError(f"the circuits live on {len(devs)} devices; a batch runs on one")
    return devs.pop()


def _bad_circuit(err: "CudaError", per_circuit: int, positions=None):
    """a segmented call's CudaError, re-raised naming the circuit (and matrix) of the first bad segment"""
    seg = getattr(err, "segment", None)
    if seg is None:
        return err
    k = seg // per_circuit if positions is None else positions[seg // per_circuit]
    return CudaError(err.code, f"circuit {k}: matrix {'abc'[seg % per_circuit]} has a column ≥ num_variables or a row_ptr "
                                           "that does not run from 0 to nnz")


def _matrix_evals(circuits: list) -> None:
    """matrix_evals (ahp/matrices.rs:138-195) of every matrix of every circuit: one launch, one synchronisation"""
    specs = []
    for c in circuits:
        lg_r, lg_c = c.constraint_domain.log_size_of_group, c.variable_domain.log_size_of_group
        for m, K in zip((c.a, c.b, c.c), c.non_zero_domains):
            specs.append((m.row_ptr, m.cols, m.vals, c.num_variables, c.input_domain.size, lg_r, lg_c, K.log_size_of_group))
    try:
        outs = device.varuna_matrix_evals_batch(specs)
    except CudaError as e:
        raise _bad_circuit(e, 3) from None
    for k, c in enumerate(circuits):
        c.ariths = [MatrixEvals(*outs[3 * k + j], K) for j, K in enumerate(c.non_zero_domains)]


def index_circuits(specs: list) -> list:
    """AHPForR1CS::index_helper for many circuits at once: `specs` holds (a, b, c, num_public, num_variables) per circuit → [Circuit]
    in input order, each equal to Circuit(*spec).  The evaluations of every matrix come from one launch and one synchronisation.  A
    malformed matrix raises CudaError naming its circuit; circuits on different devices raise ValueError."""
    if not specs:
        raise ValueError("no circuits to index")
    circuits = []
    for spec in specs:
        c = Circuit.__new__(Circuit)
        c._shape(*spec)
        circuits.append(c)
    _device_of(circuits)
    _matrix_evals(circuits)
    return circuits


def index_polynomials(circuits: list) -> list:
    """Circuit.index_polynomials of every circuit → [dict], with all 12·K interpolations in one batched iNTT (transforms of equal |K|
    share launches)"""
    polys = []
    for c in circuits:
        out = {}
        for m, arith in zip("abc", c.ariths):
            out[f"row_{m}"] = arith.row.clone()
            out[f"col_{m}"] = arith.col.clone()
            out[f"row_col_{m}"] = device.fr_vec_op(arith.row, arith.col, device.FR_MUL)
            out[f"row_col_val_{m}"] = arith.row_col_val.clone()
        polys.append({name: out[name] for name in INDEX_POLYNOMIAL_NAMES})
    device.ntt_batch_([t for p in polys for t in p.values()], NTTDirection.Inverse, NTTType.Standard)
    return polys


# Blake2s of the circuit ids runs on this many host threads: hashlib releases the GIL while it hashes a large buffer
ID_HASH_THREADS = 8


def circuit_ids(circuits: list) -> list:
    """Circuit::hash of every circuit → [32-byte id], cached on each circuit.  The byte streams of all matrices not yet hashed come
    from one launch and one synchronisation; one copy brings them to the host, where one Blake2s per circuit runs on a small thread
    pool.  A malformed row_ptr raises CudaError naming its circuit."""
    todo = [k for k, c in enumerate(circuits) if c._id is None]
    todo = [k for i, k in enumerate(todo) if all(circuits[k] is not circuits[j] for j in todo[:i])]
    if todo:
        try:
            buf, offs = device.csr_serialize_batch([(m.row_ptr, m.cols, m.vals) for k in todo for m in (circuits[k].a, circuits[k].b,
                                                                                                         circuits[k].c)])
        except CudaError as e:
            raise _bad_circuit(e, 3, todo) from None
        host = buf.cpu().numpy()

        def digest(i: int) -> bytes:
            h = hashlib.blake2s(digest_size=32)
            h.update(circuits[todo[i]].info.to_bytes_le())
            for j in range(3 * i, 3 * i + 3):
                h.update(host[offs[j]: offs[j + 1]].data)
            return h.digest()
        if len(todo) == 1:
            digests = [digest(0)]
        else:
            with ThreadPoolExecutor(min(ID_HASH_THREADS, len(todo))) as pool:
                digests = list(pool.map(digest, range(len(todo))))
        for k, d in zip(todo, digests):
            circuits[k]._id = d
    return [c._id for c in circuits]


def evaluate_index_polynomials(circuits: list, points: list, combiners: list) -> list:
    """Circuit.evaluate_index_polynomials of circuit k at points[k] with combiners[k], for every k → [int].  The Lagrange coefficients
    of all 3·K domains share one batch inversion, and the 4·3·K inner products one pass and one synchronisation."""
    combiners = [[int(c) % R_MOD for c in cs] for cs in combiners]
    for cs in combiners:
        if len(cs) != len(INDEX_POLYNOMIAL_NAMES):
            raise ValueError(f"{len(cs)} combiners for {len(INDEX_POLYNOMIAL_NAMES)} index polynomials")
    dots = device.matrix_evals_at_points([(a.row, a.col, a.row_col_val, _mont(int(p))) for c, p in zip(circuits, points) for a in c.ariths])
    out = []
    for k, cs in enumerate(combiners):
        evals = {}
        for j, m in enumerate("abc"):
            for name, v in zip(("row", "col", "row_col", "row_col_val"), dots[3 * k + j]):
                evals[f"{name}_{m}"] = _fr_mont_to_int(v)
        out.append(sum(c * evals[name] for c, name in zip(cs, INDEX_POLYNOMIAL_NAMES)) % R_MOD)
    return out


@dataclass
class CircuitVerifyingKey:
    """snark/varuna/data_structures/circuit_verifying_key.rs: the index counts, the twelve index commitments (normalised projective
    uint64[12, 18]) in INDEX_POLYNOMIAL_NAMES order and the circuit id (Circuit.id(), 32 bytes; None when setup was not asked for it)"""
    circuit_info: CircuitInfo
    circuit_commitments: np.ndarray
    id: bytes | None = None

    def to_bytes(self, compress: bool = True, device_="cuda") -> bytes:
        """the bytes of CanonicalSerialize (compressed: ToBytes), every point through one device.g1_serialize call"""
        return _to_bytes_many(_verifying_key_parts, [self], compress, device_)[0]

    @staticmethod
    def read(blob, offset: int = 0, compress: bool = True, validate: bool = True, device_="cuda"):
        """the CircuitVerifyingKey whose bytes start at `offset` of `blob` → (CircuitVerifyingKey, the offset after it); errors as verifying_keys_from_bytes"""
        objs, ends = _from_bytes_many(_walk_verifying_key, [blob], [offset], compress, validate, device_)
        return objs[0], ends[0]

    @staticmethod
    def from_bytes(blob, compress: bool = True, validate: bool = True, device_="cuda") -> "CircuitVerifyingKey":
        """the CircuitVerifyingKey at the start of `blob` (FromBytes when compressed); trailing bytes are ignored"""
        return CircuitVerifyingKey.read(blob, 0, compress, validate, device_)[0]


@dataclass
class CircuitProvingKey:
    """snark/varuna/data_structures/circuit_proving_key.rs: the verifying key, the indexed circuit and its committer key"""
    circuit_verifying_key: CircuitVerifyingKey
    circuit: Circuit
    committer_key: object

    def to_bytes(self) -> bytes:
        """ToBytes (circuit_proving_key.rs:42-49): proving_keys_to_bytes of this key"""
        return proving_keys_to_bytes([self])[0]

    @staticmethod
    def read(blob, offset: int = 0, validate: bool = True, device_="cuda"):
        """the CircuitProvingKey whose bytes start at `offset` of `blob` → (CircuitProvingKey, the offset after it); errors as
        proving_keys_from_bytes.  A snarkVM `.prover` file is a version byte (1) and then this layout: read it at offset 1."""
        pks, ends = _proving_keys_from_bytes([blob], [offset], validate, device_)
        return pks[0], ends[0]

    @staticmethod
    def from_bytes(blob, validate: bool = True, device_="cuda") -> "CircuitProvingKey":
        """the CircuitProvingKey at the start of `blob`; trailing bytes are ignored"""
        return CircuitProvingKey.read(blob, 0, validate, device_)[0]


def batch_circuit_setup(circuits: list, pp_powers_of_beta_g: torch.Tensor, pp_powers_of_beta_times_gamma_g: torch.Tensor, zk: bool = False,
                        with_id: bool = False) -> list:
    """VarunaSNARK::batch_circuit_setup (varuna.rs:72-134): for every circuit, trim the universal parameters to its max_degree and
    degree bounds and commit its twelve index polynomials (no degree bound, no hiding) → [(CircuitProvingKey, CircuitVerifyingKey)] in
    input order, each equal to circuit_setup's.  All 12·K interpolations share one batched iNTT, and all 12·K commitments one MSM pass:
    every trimmed key is a prefix of the same powers, so their bases merge into one array.  The SRS is (β^i·G, γβ^i·G) as
    sonic_pc.CommitterKey.trim takes it; an SRS too short for the largest circuit raises ValueError before any launch.  `with_id`
    also fills each verifying key's circuit id (circuit_ids)."""
    from .sonic_pc import CommitterKey
    if not circuits:
        raise ValueError("no circuits to set up")
    _device_of(circuits)
    need = max(c.info.max_degree(zk) for c in circuits) + 1
    if pp_powers_of_beta_g.shape[0] < need:                             # download_powers_for(0..max_degree), varuna.rs:85-87
        raise ValueError(f"the SRS holds {pp_powers_of_beta_g.shape[0]} powers; the largest circuit needs {need}")
    cks = [CommitterKey.trim(pp_powers_of_beta_g, pp_powers_of_beta_times_gamma_g, c.info.max_degree(zk), (), 1, c.info.degree_bounds())
           for c in circuits]
    polys = index_polynomials(circuits)
    comms = device.sonic_commit_batch([ck.powers_of_beta_g for ck in cks for _ in INDEX_POLYNOMIAL_NAMES],
                                      [t for p in polys for t in p.values()])
    ids = circuit_ids(circuits) if with_id else [None] * len(circuits)
    out = []
    for k, (c, ck) in enumerate(zip(circuits, cks)):
        vk = CircuitVerifyingKey(c.info, comms[12 * k: 12 * k + 12].copy(), ids[k])
        out.append((CircuitProvingKey(vk, c, ck), vk))
    return out


def circuit_setup(circuit: Circuit, pp_powers_of_beta_g: torch.Tensor, pp_powers_of_beta_times_gamma_g: torch.Tensor, zk: bool = False,
                  with_id: bool = False):
    """VarunaSNARK::circuit_setup (varuna.rs:226-233): batch_circuit_setup of one circuit → (CircuitProvingKey, CircuitVerifyingKey)"""
    return batch_circuit_setup([circuit], pp_powers_of_beta_g, pp_powers_of_beta_times_gamma_g, zk, with_id)[0]


@dataclass
class Certificate:
    """snark/varuna/data_structures/certificate.rs: the BatchLCProof of prove_vk, one non-hiding KZG proof `w` (normalised projective
    uint64[18]) at the one query point"""
    w: np.ndarray

    def to_bytes(self, compress: bool = True, device_="cuda") -> bytes:
        """the bytes of CanonicalSerialize (compressed: ToBytes), every point through one device.g1_serialize call"""
        return _to_bytes_many(_certificate_parts, [self], compress, device_)[0]

    @staticmethod
    def read(blob, offset: int = 0, compress: bool = True, validate: bool = True, device_="cuda"):
        """the Certificate whose bytes start at `offset` of `blob` → (Certificate, the offset after it); errors as certificates_from_bytes"""
        objs, ends = _from_bytes_many(_walk_certificate, [blob], [offset], compress, validate, device_)
        return objs[0], ends[0]

    @staticmethod
    def from_bytes(blob, compress: bool = True, validate: bool = True, device_="cuda") -> "Certificate":
        """the Certificate at the start of `blob` (FromBytes when compressed); trailing bytes are ignored"""
        return Certificate.read(blob, 0, compress, validate, device_)[0]


def _certificate_point(challenges) -> tuple:
    """the twelve values squeeze_nonnative_field_elements(12) yields → (point, combiners): the last is the point, the combiners are
    one followed by the first eleven (varuna.rs:248-255, 296-300)"""
    challenges = [int(c) % R_MOD for c in challenges]
    if len(challenges) != len(INDEX_POLYNOMIAL_NAMES):
        raise ValueError(f"{len(challenges)} challenges; a certificate takes {len(INDEX_POLYNOMIAL_NAMES)}")
    return challenges[-1], [1] + challenges[:-1]


PROTOCOL_NAME = b"VARUNA-2023"                                           # VarunaSNARK::PROTOCOL_NAME (varuna.rs:68)
_CERTIFICATE_ELEMENTS = 40          # absorbed per certificate: name 1, CircuitInfo 2, twelve commitments × (x, y, infinity) 36, id 1
_CERTIFICATE_SQUEEZES = 14          # nonnative Fr per certificate: twelve challenges, then ξ and the randomizer (short)


def _commitment_elements(comms) -> np.ndarray:
    """commitments (normalised projective uint64[k, 18]) → their SWAffine::to_field_elements (x, y, infinity flag,
    curves/src/templates/to_field_vec.rs:52-64) as Montgomery Fq words uint32[3k, 12].  A normalised projective image is (x, y, 1) or
    (0, 1, 0): its X, Y are the affine x, y of SWAffine, Affine::zero() included."""
    comms = np.ascontiguousarray(comms, dtype=np.uint64).reshape(-1, 18)
    c = np.zeros((comms.shape[0], 3, 12), dtype=np.uint32)
    c[:, 0] = comms[:, 0:6].view(np.uint32)
    c[:, 1] = comms[:, 6:12].view(np.uint32)
    c[~comms[:, 12:18].any(axis=1), 2] = poseidon.to_mont_words(poseidon.FIELD_FQ, [1])[0]
    return c.reshape(-1, 12)


def _certificate_transcripts(vks: list):
    """init_sponge_for_certificate (varuna.rs:155-165) of every key, then its squeezes, as the op lists of
    device.poseidon_transcripts → (ops, op_start, inputs) as host arrays.  Per key: absorb_bytes of the protocol name (to_bytes_le!
    of a byte slice writes the bytes without a length prefix, utilities/src/bytes.rs:442-457), of CircuitInfo::to_bytes_le and of the
    id, and absorb_native_field_elements of the twelve commitments as SWAffine::to_field_elements (x, y, infinity flag,
    curves/src/templates/to_field_vec.rs:52-64); then squeeze_nonnative_field_elements(12) (varuna.rs:248, 293) and two
    squeeze_short_nonnative_field_element calls: combine_for_open's challenge ξ and batch_open's `_randomizer` on the prover side
    (sonic_pc/mod.rs:277, 329), accumulate_elems' curr_challenge and batch_check's next randomizer on the verifier side (:602, :405)
    — the same two squeezes in the same order."""
    fq = poseidon.FIELD_FQ
    K = len(vks)
    name = poseidon.to_mont_words(fq, poseidon.bytes_to_field_elements(PROTOCOL_NAME, fq))
    inputs = np.zeros((K, _CERTIFICATE_ELEMENTS, 12), dtype=np.uint32)
    for k, vk in enumerate(vks):
        if vk.id is None:
            raise ValueError(f"verifying key {k} has no circuit id; a certificate's transcript absorbs it")
        comms = np.ascontiguousarray(vk.circuit_commitments, dtype=np.uint64).reshape(len(INDEX_POLYNOMIAL_NAMES), 18)
        info = poseidon.to_mont_words(fq, poseidon.bytes_to_field_elements(vk.circuit_info.to_bytes_le(), fq))
        ident = poseidon.to_mont_words(fq, poseidon.bytes_to_field_elements(bytes(vk.id), fq))
        if len(name) + len(info) + 3 * comms.shape[0] + len(ident) != _CERTIFICATE_ELEMENTS:
            raise ValueError(f"verifying key {k}: a 32-byte id and twelve commitments expected")
        inputs[k] = np.concatenate([name, info, _commitment_elements(comms), ident])
    base_in = np.arange(K, dtype=np.int64)[:, None] * _CERTIFICATE_ELEMENTS
    base_out = np.arange(K, dtype=np.int64)[:, None] * _CERTIFICATE_SQUEEZES
    ops = np.zeros((K, 7, 3), dtype=np.int64)
    short = poseidon.OP_SQUEEZE_SHORT_NONNATIVE
    ops[:, :, 0] = [poseidon.OP_ABSORB] * 4 + [poseidon.OP_SQUEEZE_NONNATIVE, short, short]
    ops[:, :, 1] = [1, 2, 36, 1, 12, 1, 1]
    ops[:, :4, 2] = base_in + [0, 1, 3, 39]
    ops[:, 4:, 2] = base_out + [0, 12, 13]
    op_start = np.arange(0, 7 * K + 1, 7, dtype=np.int32)
    return ops.reshape(-1, 3).astype(np.int32), op_start, inputs.reshape(-1, 12)


def certificate_challenges(vks: list, device_=None) -> list:
    """The Fiat–Shamir challenges of every key's certificate, as prove_vk and verify_vk draw them from PoseidonSponge<Fq, 2, 1>
    (init_sponge_for_certificate, varuna.rs:155-165, then varuna.rs:248 / 293 and sonic_pc/mod.rs:277, 329 / 602, 405) → [(twelve
    challenges, (ξ, randomizer))] in input order, canonical integers mod r.  The transcript depends only on the verifying key; all K
    run in one device call, one thread each.  A key without a circuit id raises ValueError (a reference key always has its id)."""
    if not vks:
        raise ValueError("no verifying keys")
    ops, op_start, inputs = _certificate_transcripts(vks)
    dev = torch.device(device_) if device_ is not None else torch.device("cuda", torch.cuda.current_device())
    _out, fr = device.poseidon_transcripts(
        poseidon.FIELD_FQ, torch.from_numpy(ops).to(dev), torch.from_numpy(op_start).to(dev),
        torch.from_numpy(inputs.view(np.int64)).to(dev), 0, _CERTIFICATE_SQUEEZES * len(vks))
    vals = [_fr_mont_to_int(row) for row in fr.cpu().numpy().view(np.uint64)]
    S = _CERTIFICATE_SQUEEZES
    return [(vals[S * k: S * k + 12], (vals[S * k + 12], vals[S * k + 13])) for k in range(len(vks))]


def prove_vk_batch(pks: list, challenges: list | None = None, opening_challenges: list | None = None) -> list:
    """VarunaSNARK::prove_vk (varuna.rs:236-276) for every proving key: open Σ c_i·p_i over its twelve index polynomials
    (c = [1] + challenges[k][:11] in label order) at z = challenges[k][11] → [Certificate] in input order.  The opening is
    SonicKZG10.batch_open of `circuit_check` with empty randomness: it consumes opening_challenges[k] (its combination challenge ξ,
    then the discarded randomizer) as open_combinations would, and scales the combination by ξ, which is folded into the
    coefficients.  Omitted challenges (None) are the sponge's: certificate_challenges of the verifying keys, which needs each key's
    id.  All interpolations share one batched iNTT, all K combinations one fr_lincomb launch, and all K witness commitments one MSM
    pass."""
    if not pks:
        raise ValueError("no proving keys")
    if challenges is None or opening_challenges is None:
        derived = certificate_challenges([pk.circuit_verifying_key for pk in pks], _device_of([pk.circuit for pk in pks]))
        challenges = [d[0] for d in derived] if challenges is None else challenges
        opening_challenges = [d[1] for d in derived] if opening_challenges is None else opening_challenges
    if len(challenges) != len(pks) or len(opening_challenges) != len(pks):
        raise ValueError("one set of challenges and opening challenges per proving key")
    points = [_certificate_point(ch) for ch in challenges]
    circuits = [pk.circuit for pk in pks]
    dev = _device_of(circuits)
    xis = []
    for oc in opening_challenges:
        it = iter(oc)
        xis.append(int(next(it)) % R_MOD)
        next(it)                                                        # `_randomizer`
    for pk, c in zip(pks, circuits):
        if c.max_non_zero_domain.size > pk.committer_key.powers_of_beta_g.shape[0]:
            raise ValueError("check_degree_is_too_large")
    polys = index_polynomials(circuits)
    combined = device.fr_lincomb_batch([(list(p.values()), [_mont(xi * c) for c in combiners])
                                        for p, xi, (_z, combiners) in zip(polys, xis, points)])
    # kzg10::open (kzg10/mod.rs:220-241): a zero ξ leaves the empty polynomial, whose witness is empty
    witnesses = [device.poly_divide_by_linear(comb, _mont(z)) if xi else _zeros(0, dev) for comb, xi, (z, _c) in zip(combined, xis, points)]
    ws = device.sonic_commit_batch([pk.committer_key.powers_of_beta_g for pk in pks], witnesses)
    return [Certificate(w.copy()) for w in ws]


def prove_vk(pk: CircuitProvingKey, challenges=None, opening_challenges=None) -> Certificate:
    """VarunaSNARK::prove_vk (varuna.rs:236-276): prove_vk_batch of one proving key (the sponge's challenges when omitted)"""
    return prove_vk_batch([pk], None if challenges is None else [challenges],
                          None if opening_challenges is None else [opening_challenges])[0]


@dataclass
class VerifyingKeyCheck:
    """verify_vk's result.  `matches`: the circuit's info and id equal the verifying key's (the reference stops with
    CircuitNotFound otherwise; the other fields are still computed here).  The certificate is valid iff `matches` and
    e(lhs, H)·e(−w, β·H) = 1.  `valid` is that verdict when verify_vk ran with a UniversalVerifier, and None without one."""
    matches: bool
    evaluation: int
    lhs: np.ndarray
    w: np.ndarray
    valid: bool | None = None


Q_MOD = 258664426012969094010652733694893533536393512754914660539884262666720468348340822774968888139573360124440321458177  # fq.rs
_FQ_R = (1 << 384) % Q_MOD
# G2_GENERATOR_{X,Y}_{C0,C1} of curves/src/bls12_377/g2.rs, out of Montgomery form
G2_GENERATOR = (
    (170590608266080109581922461902299092015242589883741236963254737235977648828052995125541529645051927918098146183295,
     83407003718128594709087171351153471074446327721872642659202721143408712182996929763094113874399921859453255070254),
    (1843833842842620867708835993770650838640642469700861403869757682057607397502738488921663703124647238454792872005,
     33145532013610981697337930729788870077912093258611421158732879580766461459275194744385880708057348608045241477209),
)
# the G1 generator of curves/src/bls12_377/g1.rs, out of Montgomery form
G1_GENERATOR = (89363714989903307245735717098563574705733591463163614225748337416674727625843187853442697973404985688481508350822,
                3702177272937190650578065972808860481433820514072818216637796320125658674906330993856598323293086021583822603349)


def _generator_bytes(coords, compressed: bool) -> bytes:
    """the byte form of a generator ((x, y) over Fq, or ((x0, x1), (y0, y1)) over Fq2) without flag bits: y's sign in the
    compressed form is compared apart"""
    x, y = coords
    x, y = (x, y) if isinstance(x, tuple) else ((x,), (y,))
    return b"".join(v.to_bytes(48, "little") for v in (x if compressed else x + y))


def _is_generator(b: bytes, coords, compressed: bool) -> bool:
    """the bytes of a point decode to the generator: the same coordinates, no Infinity bit and, compressed, the generator's
    sign (PositiveY iff y > −y; in the uncompressed form the sign bit is ignored, as the reference ignores it)"""
    y = coords[1]
    y_pos = (y[1], y[0]) > ((-y[1]) % Q_MOD, (-y[0]) % Q_MOD) if isinstance(y, tuple) else y > (-y) % Q_MOD
    flags = b[-1] & 0xC0
    body = b[:-1] + bytes([b[-1] & 0x3F])
    if flags & 0x40 or body != _generator_bytes(coords, compressed):
        return False
    return not compressed or (flags == 0x80) == y_pos


def _g2_affine(p) -> np.ndarray:
    """((x0, x1), (y0, y1)) of plain integers, or None → the 200-byte Affine<G2> image (Montgomery; Affine::zero() = (0, 1, true))"""
    coords, inf = (((0, 0), (1, 0)), 1) if p is None else (p, 0)
    out = np.zeros(200, dtype=np.uint8)
    out[:192] = np.frombuffer(b"".join((v * _FQ_R % Q_MOD).to_bytes(48, "little") for c in coords for v in c), dtype=np.uint8)
    out[192] = inf
    return out


def _g1_affine(p) -> np.ndarray:
    """(x, y) of plain integers, or None → the 104-byte Affine<G1> image (Montgomery; Affine::zero() = (0, 1, true))"""
    (x, y), inf = ((0, 1), 1) if p is None else (p, 0)
    out = np.zeros(104, dtype=np.uint8)
    out[:96] = np.frombuffer(b"".join((v * _FQ_R % Q_MOD).to_bytes(48, "little") for v in (x, y)), dtype=np.uint8)
    out[96] = inf
    return out


def _parse_g1(blob: bytes, what: str) -> np.ndarray:
    """a 96-byte uncompressed G1 point (x, y 48 B LE each; bit 6 of the last byte = infinity, bit 7 = y's sign,
    utilities/src/serialize/flags.rs) → its Affine image; a coordinate ≥ q raises ValueError"""
    b = bytearray(blob)
    infinity = bool(b[95] & 0x40)
    b[95] &= 0x3F
    v = [int.from_bytes(bytes(b[48 * i: 48 * i + 48]), "little") for i in range(2)]
    if any(x >= Q_MOD for x in v):
        raise ValueError(f"a coordinate of {what} is not below q")
    return _g1_affine(None if infinity else (v[0], v[1]))


def _parse_g2(blob: bytes, what: str) -> np.ndarray:
    """a 192-byte uncompressed G2 point (x.c0, x.c1, y.c0, y.c1, 48 B LE each; the flags in the last byte) → its Affine image; a
    coordinate ≥ q raises ValueError"""
    if len(blob) != 192:
        raise ValueError(f"a G2 point is 192 bytes, not {len(blob)}")
    b = bytearray(blob)
    infinity = bool(b[191] & 0x40)
    b[191] &= 0x3F
    v = [int.from_bytes(bytes(b[48 * i: 48 * i + 48]), "little") for i in range(4)]
    if any(x >= Q_MOD for x in v):
        raise ValueError(f"a coordinate of {what} is not below q")
    return _g2_affine(None if infinity else ((v[0], v[1]), (v[2], v[3])))


def _u64_map(blob: bytes, entry: int, what: str) -> list:
    """a serialised BTreeMap<usize, point>: a u64 count, then (u64 key, `entry` bytes) per entry → [(key, bytes)]"""
    if len(blob) < 8:
        raise ValueError(f"{what}: no entry count")
    (n,) = struct.unpack_from("<Q", blob, 0)
    if len(blob) != 8 + n * (8 + entry):
        raise ValueError(f"{what}: {len(blob)} bytes do not hold {n} entries of {8 + entry} bytes")
    out = []
    for k in range(n):
        off = 8 + k * (8 + entry)
        out.append((struct.unpack_from("<Q", blob, off)[0], blob[off + 8: off + 8 + entry]))
    return out


def parse_neg_powers(blob: bytes) -> dict:
    """`neg-powers-of-beta.usrs` (a BTreeMap<usize, G2Affine>) → {degree bound: 200-byte Affine<G2> image of β^{-(D − d)}·H}"""
    return {d: _parse_g2(p, f"the negative power for bound {d}") for d, p in _u64_map(blob, 192, "negative powers of β·H")}


def parse_gamma_powers(blob: bytes) -> dict:
    """`powers-of-beta-gamma.usrs` (a BTreeMap<usize, G1Affine>) → {i: 104-byte Affine<G1> image of γβ^i·G}"""
    return {i: _parse_g1(p, f"γβ^{i}·G") for i, p in _u64_map(blob, 96, "powers of β·γ·G")}


def _validate_g2(named: list, dev) -> None:
    """Valid for Affine<G2> of every (name, 200-byte Affine<G2> image) in one device.g2_validate launch; ValueError names the
    first that fails"""
    status = device.g2_validate(torch.from_numpy(np.stack([img for _n, img in named])).to(dev)).cpu().numpy()
    bad = np.nonzero(status)[0]
    if bad.size:
        raise ValueError(f"{named[int(bad[0])][0]}: {_G1_STATUS[int(status[bad[0]])]}")


class UniversalVerifier:
    """The pairing half of the universal verifier (kzg10/data_structures.rs UniversalParams: h, prepared_h, prepared_beta_h,
    gamma_g, prepared_negative_powers_of_beta_h; g is the first power of β·G): g and gamma_g (γ·G, None when unknown) as 104-byte
    Affine<G1> images, h (the G2 generator) and β·h as 200-byte Affine<G2> images, and `prepared`, h, β·h and then the negative
    powers of β·H in increasing degree bound, prepared once on the device ([2 + bounds, device.G2_PREPARED_BYTES]).
    `neg_index` maps each degree bound d to the row of `prepared` that holds β^{-(D − d)}·H, D the SRS's maximum degree."""

    def __init__(self, beta_h: np.ndarray, device_="cuda", gamma_g: np.ndarray | None = None, neg_powers: dict | None = None):
        dev = torch.device(device_)
        self.h = _g2_affine(G2_GENERATOR)
        self.beta_h = np.ascontiguousarray(beta_h, dtype=np.uint8).reshape(200)
        self.g = device.generator_mul(torch.from_numpy(np.array([[1, 0, 0, 0]], dtype=np.uint64).view(np.int64)).to(dev)).cpu().numpy()[0]
        self.gamma_g = None if gamma_g is None else np.ascontiguousarray(gamma_g, dtype=np.uint8).reshape(104)
        bounds = sorted(neg_powers or {})
        self.neg_index = {d: 2 + k for k, d in enumerate(bounds)}
        g2 = [self.h, self.beta_h] + [np.ascontiguousarray(neg_powers[d], dtype=np.uint8).reshape(200) for d in bounds]
        self.prepared = device.g2_prepare(torch.from_numpy(np.stack(g2)).to(dev))
        self.device = self.prepared.device

    @classmethod
    def from_usrs(cls, blob: bytes, device_="cuda", validate: bool = False) -> "UniversalVerifier":
        """β·H from the mainnet `beta-h.usrs` bytes: x.c0, x.c1, y.c0, y.c1 (48 B LE each), bit 6 of the last byte = infinity and
        bit 7 = y's sign (utilities/src/serialize/flags.rs).  A coordinate ≥ q raises ValueError.  The reference reads this file
        unchecked (deserialize_uncompressed_unchecked, parameters/src/mainnet/powers.rs:86-96); with `validate`, β·H must also pass
        Valid for Affine<G2> (device.g2_validate), or ValueError names it."""
        beta_h = _parse_g2(blob, "β·H")
        if validate:
            _validate_g2([("β·H", beta_h)], torch.device(device_))
        return cls(beta_h, device_)

    @classmethod
    def from_mainnet(cls, beta_h: bytes, neg_powers: bytes, gamma_powers: bytes, device_="cuda",
                     validate: bool = False) -> "UniversalVerifier":
        """the mainnet verifier from the bytes of `beta-h.usrs`, `neg-powers-of-beta.usrs` (every degree bound 2^k − 2 with its
        β^{-(D − d)}·H) and `powers-of-beta-gamma.usrs` (its key 0 is γ·G).  A coordinate ≥ q raises ValueError.  With `validate`,
        β·H and every negative power pass Valid for Affine<G2> in one device.g2_validate launch and γ·G passes Affine::check
        (device.g1_validate); a failure raises ValueError naming β·H, the degree bound of the negative power, or γ·G."""
        gammas = parse_gamma_powers(gamma_powers)
        if 0 not in gammas:
            raise ValueError("the powers of β·γ·G hold no γ·G")
        bh, neg = _parse_g2(beta_h, "β·H"), parse_neg_powers(neg_powers)
        if validate:
            dev = torch.device(device_)
            _validate_g2([("β·H", bh)] + [(f"the negative power for bound {d}", neg[d]) for d in sorted(neg)], dev)
            status = int(device.g1_validate(torch.from_numpy(gammas[0][None].copy()).to(dev)).cpu()[0])
            if status != device.G1_VALID:
                raise ValueError(f"γ·G: {_G1_BYTES_STATUS[status]}")
        return cls(bh, device_, gammas[0], neg)

    def to_bytes(self, compressed: bool = True) -> bytes:
        """CanonicalSerialize of kzg10::VerifierKey (kzg10/data_structures.rs:200-214): g, γ·G, h, β·h; 288 bytes compressed (the
        reference's write_le), 576 uncompressed.  The G1 points go through one device.g1_serialize call and the G2 points through
        one device.g2_serialize call.  A verifier without γ·G raises ValueError."""
        if self.gamma_g is None:
            raise ValueError("this verifier holds no γ·G, which the verifier key's bytes need")
        g1 = torch.from_numpy(_projective_limbs(np.stack([self.g, self.gamma_g])).view(np.int64)).to(self.device)
        g2 = torch.from_numpy(np.stack([self.h, self.beta_h])).to(self.device)
        b1 = device.g1_serialize(g1, compressed).cpu().numpy()
        b2 = device.g2_serialize(g2, compressed).cpu().numpy()
        return b1.tobytes() + b2.tobytes()

    @classmethod
    def from_bytes(cls, blob, compressed: bool = True, validate: bool = True, neg_powers: dict | None = None,
                   device_="cuda") -> "UniversalVerifier":
        """the inverse of to_bytes (CanonicalDeserialize of kzg10::VerifierKey, data_structures.rs:217-232; read_le is the
        compressed form, validated): g and γ·G in one device.g1_deserialize launch, h and β·h in one device.g2_deserialize launch.
        `neg_powers` ({degree bound: 200-byte Affine<G2> image}, as parse_neg_powers gives) is held as the constructor holds it.
        A wrong length or trailing bytes, or a g or h other than the G1 or G2 generator (which this verifier assumes, DESIGN §4c),
        raises ValueError on the host before any device call; a point that fails to decode (or, with `validate`, Valid) raises
        ValueError naming the field."""
        blob = bytes(blob)
        g1_size, g2_size = _g1_size(compressed), device.G2_COMPRESSED_BYTES if compressed else device.G2_UNCOMPRESSED_BYTES
        want = 2 * g1_size + 2 * g2_size
        if len(blob) != want:
            raise ValueError(f"a verifier key is {want} bytes in this form, not {len(blob)}"
                             + (" (trailing bytes)" if len(blob) > want else ""))
        if not _is_generator(blob[:g1_size], G1_GENERATOR, compressed):
            raise ValueError("g: not the G1 generator, which this verifier assumes")
        if not _is_generator(blob[2 * g1_size: 2 * g1_size + g2_size], G2_GENERATOR, compressed):
            raise ValueError("h: not the G2 generator, which this verifier assumes")
        dev = torch.device(device_)
        raw1 = torch.from_numpy(np.frombuffer(blob[:2 * g1_size], dtype=np.uint8).copy()).to(dev)
        raw2 = torch.from_numpy(np.frombuffer(blob[2 * g1_size:], dtype=np.uint8).copy()).to(dev)
        img1, st1 = device.g1_deserialize(raw1, compressed, validate)
        img2, st2 = device.g2_deserialize(raw2, compressed, validate)
        img1, st1, img2, st2 = img1.cpu().numpy(), st1.cpu().numpy(), img2.cpu().numpy(), st2.cpu().numpy()
        for name, s in zip(("g", "gamma_g", "h", "beta_h"), list(st1) + list(st2)):
            if s != device.G1_VALID:
                raise ValueError(f"{name}: {_G1_BYTES_STATUS[int(s)]}")
        return cls(img2[1], device_, img1[1], neg_powers)

    @classmethod
    def synthetic(cls, beta: int, device_="cuda", max_degree: int | None = None, gamma: int | None = None,
                  bounds=()) -> "UniversalVerifier":
        """the verifier of a setup with a known β (sonic_pc.synthetic_srs): β·H by the G2 MSM of one point; with `gamma`, γ·G; for
        each degree bound d of `bounds`, β^{-(max_degree − d)}·H by the same G2 MSM (max_degree: the SRS's highest power of β)"""
        dev = torch.device(device_)
        beta %= R_MOD

        def g2_mul(k: int) -> np.ndarray:
            scalar = torch.from_numpy(np.array([[(k >> (64 * i)) & (2**64 - 1) for i in range(4)]], dtype=np.uint64).view(np.int64)).to(dev)
            proj = device.msm_g2(torch.from_numpy(_g2_affine(G2_GENERATOR)[None]).to(dev), scalar)   # normalised: (x, y, 1) or (0, 1, 0)
            img = np.zeros(200, dtype=np.uint8)
            img[:192] = proj[:24].view(np.uint8)
            img[192] = 0 if proj[24:].any() else 1
            return img
        if bounds and max_degree is None:
            raise ValueError("negative powers of β·H need the SRS's max_degree")
        neg = {int(d): g2_mul(pow(beta, -(max_degree - int(d)), R_MOD)) for d in bounds}
        gamma_g = None
        if gamma is not None:
            k = gamma % R_MOD
            scal = torch.from_numpy(np.array([[(k >> (64 * i)) & (2**64 - 1) for i in range(4)]], dtype=np.uint64).view(np.int64)).to(dev)
            gamma_g = device.generator_mul(scal).cpu().numpy()[0]
        return cls(g2_mul(beta), device_, gamma_g, neg)


def _affine(projective: np.ndarray) -> np.ndarray:
    """normalised projective image (X, Y, Z = one or (0, one, 0)) → the 104-byte Affine image (x, y, infinity flag, padding)"""
    limbs = np.ascontiguousarray(projective, dtype=np.uint64).reshape(18)
    out = np.zeros(104, dtype=np.uint8)
    out[:96] = limbs[:12].view(np.uint8)
    out[96] = 1 if not limbs[12:].any() else 0
    return out


def _affine_neg(projective: np.ndarray) -> np.ndarray:
    """the Affine image of −P (y ↦ q − y on the Montgomery image; zero stays zero)"""
    out = _affine(projective)
    y = int.from_bytes(out[48:96].tobytes(), "little")
    out[48:96] = np.frombuffer(((Q_MOD - y) % Q_MOD).to_bytes(48, "little"), dtype=np.uint8)
    return out


def verify_vk_batch(circuits: list, vks: list, certificates: list, challenges: list | None = None, opening_challenges: list | None = None,
                    verifier: UniversalVerifier | None = None) -> list:
    """VarunaSNARK::verify_vk (varuna.rs:280-331) up to the pairing, for every (circuit, verifying key, certificate) → [VerifyingKeyCheck]
    in input order.  The circuits are already indexed (Circuit).  Omitted challenges (None) are the sponge's: certificate_challenges
    of the verifying keys (their twelve challenges and ξ), which needs each key's id.  The evaluation v comes from evaluate_index_polynomials;
    check_combinations → batch_check → accumulate_elems for one point with randomizer one (sonic_pc/mod.rs:344-411, 477-544, 582-635)
    reduces to lhs = ξ·C_lc − ξ·v·G + z·W with C_lc = Σ c_i·C_i, ξ = opening_challenges[k]: a 14-point sum over the twelve commitments,
    G and W.  check_elems' pairing equation is then e(lhs, H) = e(W, β·H).  G is the universal verifier's g, the SRS's first power,
    which is the G1 generator in the mainnet setup and in synthetic_srs.  The ids not yet cached come from one circuit_ids call, the
    K evaluations from one evaluate_index_polynomials pass, and the K sums are K jobs of one MSM pass."""
    K = len(circuits)
    if K == 0:
        raise ValueError("no circuits to verify")
    if challenges is None or opening_challenges is None:
        if len(vks) != K:
            raise ValueError("one verifying key per circuit")
        derived = certificate_challenges(vks, _device_of(circuits))
        challenges = [d[0] for d in derived] if challenges is None else challenges
        opening_challenges = [d[1][0] for d in derived] if opening_challenges is None else opening_challenges
    if not (len(vks) == len(certificates) == len(challenges) == len(opening_challenges) == K):
        raise ValueError("one verifying key, certificate, set of challenges and opening challenge per circuit")
    points = [_certificate_point(ch) for ch in challenges]
    xis = [int(x) % R_MOD for x in opening_challenges]
    dev = _device_of(circuits)
    compare = [c.info == vk.circuit_info and vk.id is not None for c, vk in zip(circuits, vks)]
    circuit_ids([c for c, k in zip(circuits, compare) if k])
    matches = [k and c.id() == vk.id for c, vk, k in zip(circuits, vks, compare)]
    evaluations = evaluate_index_polynomials(circuits, [z for z, _c in points], [c for _z, c in points])
    g = device.generator_mul(torch.from_numpy(np.array([[1, 0, 0, 0]], dtype=np.uint64).view(np.int64)).to(dev)).cpu().numpy()[0]
    bases, scalars = [], []
    for vk, cert, (z, combiners), xi, v in zip(vks, certificates, points, xis, evaluations):
        bases += [_affine(c) for c in vk.circuit_commitments] + [g, _affine(cert.w)]           # C_0 … C_11, G, W
        scalars += [_mont(xi * c) for c in combiners] + [_mont(-xi * v), _mont(z)]
    bases_d = torch.from_numpy(np.stack(bases)).to(dev)
    scalars_d = torch.from_numpy(np.stack(scalars).view(np.int64)).to(dev)
    lhs = device.sonic_commit_batch([bases_d[14 * k: 14 * k + 14] for k in range(K)], [scalars_d[14 * k: 14 * k + 14] for k in range(K)])
    checks = [VerifyingKeyCheck(m, v, lhs[k].copy(), cert.w) for k, (m, v, cert) in enumerate(zip(matches, evaluations, certificates))]
    if verifier is None:
        return checks
    if verifier.device != dev:
        raise ValueError("the verifier's prepared points live on another device than the circuits")
    # check_elems (sonic_pc/mod.rs:637-677): e(lhs, H)·e(−W, β·H) = 1, every circuit one check of one pairing-products call
    g1 = torch.from_numpy(np.stack([a for c in checks for a in (_affine(c.lhs), _affine_neg(c.w))])).to(dev)
    g2_index = torch.tensor([0, 1] * K, dtype=torch.int32, device=dev)
    check_start = torch.arange(0, 2 * K + 1, 2, dtype=torch.int32, device=dev)
    _gt, is_one = device.pairing_products(g1, g2_index, verifier.prepared, check_start)
    for c, one in zip(checks, is_one.cpu().tolist()):
        c.valid = bool(c.matches and one)
    return checks


def verify_vk(circuit: Circuit, vk: CircuitVerifyingKey, certificate: Certificate, challenges=None, opening_challenge: int | None = None,
              verifier: UniversalVerifier | None = None) -> VerifyingKeyCheck:
    """VarunaSNARK::verify_vk (varuna.rs:280-331): verify_vk_batch of one circuit (up to the pairing without a verifier; the
    sponge's challenges when omitted)"""
    return verify_vk_batch([circuit], [vk], [certificate], None if challenges is None else [challenges],
                           None if opening_challenge is None else [opening_challenge], verifier)[0]


def witness_label(circuit_id: bytes, poly: str, i: int) -> str:
    """ahp/ahp.rs:46-50: circuit_{id as hex}_{poly}_{i:08}"""
    return f"circuit_{circuit_id.hex()}_{poly}_{i:08}"


def _vanish(d: EvaluationDomain, x: int) -> int:
    return (pow(x, d.size, R_MOD) - 1) % R_MOD


def _selector(target: EvaluationDomain, src: EvaluationDomain, x: int) -> int:
    """the selector of src inside target at x (selectors.rs): v_target(x)·|src| / (v_src(x)·|target|); one when they are equal"""
    if target.size == src.size:
        return 1
    return _vanish(target, x) * src.size % R_MOD * pow(_vanish(src, x) * target.size % R_MOD, -1, R_MOD) % R_MOD


def _largest(domains) -> EvaluationDomain:
    return max(domains, key=lambda d: d.size)


class BatchProver:
    """init_prover + State::initialize and the five AHP rounds of VarunaSNARK::prove_batch (varuna.rs:336-620) for K circuits, each with
    its own batch of instances.  `program`: [(Circuit, [assignment, …])], an assignment being one CUDA tensor [num_variables, 4] per
    instance (padded public variables, the first one One, then private).  The circuits are taken in Circuit.id() order, as the
    reference keys its prover state by circuit and orders circuits by id (ahp/indexer/circuit.rs:96-100); `circuits`, and every
    per-circuit argument and attribute, follow that order, so the order of `program` changes no result.  A one-circuit batch never
    computes the id.  Challenges are arguments (the Poseidon sponge stays with the caller):
        batch_combiners: per circuit (circuit combiner, [one combiner per instance]),
        deltas:          per circuit (δ_a, δ_b, δ_c).
    Per-circuit O(n) work runs as segmented kernels: one pass for a round's mat-vecs, products, fourth-round evaluations and selector
    sums, whatever the number of circuits and instances (launches grow only with the number of distinct domain sizes)."""

    def __init__(self, program: list):
        self._setup(program)
        BatchProver._load_many([self])

    def _setup(self, program: list):
        """the checks, the circuit order and the domains: everything before the first device pass"""
        if not program:
            raise ValueError("no circuits to prove")
        for k, (c, zs) in enumerate(program):
            if not zs:
                raise ValueError(f"circuit {k}: no instances")
            for z in zs:
                if z.shape[0] != c.num_variables:                       # AHPError::InstanceDoesNotMatchIndex
                    raise ValueError(f"circuit {k}: instance does not match the index ({z.shape[0]} variables, the index has "
                                     f"{c.num_variables})")
        self.dev = _device_of([c for c, _ in program])
        if any(z.device != self.dev for _, zs in program for z in zs):
            raise ValueError("an assignment lives on another device than its circuit")
        order = [0]
        if len(program) > 1:
            ids = circuit_ids([c for c, _ in program])
            if len(set(ids)) != len(ids):
                raise ValueError("two entries of the program have equal circuit ids")
            order = sorted(range(len(program)), key=lambda k: ids[k])
        self.positions = order                                            # circuit i of the batch is program[positions[i]]
        self.circuits = [program[k][0] for k in order]
        self.z = [[z.contiguous() for z in program[k][1]] for k in order]
        self.batch = [len(zs) for zs in self.z]
        cs = self.circuits
        self.max_constraint_domain = _largest(c.constraint_domain for c in cs)
        self.max_variable_domain = _largest(c.variable_domain for c in cs)
        self.max_non_zero_domain = _largest(c.max_non_zero_domain for c in cs)
        self.mask_poly = None

    @staticmethod
    def _load_many(provers: list):
        """z_A, z_B, z_C of every instance of every prover (round_functions/mod.rs:128-152) in one mat-vec pass, each written into a
        zeroed |R|-row slot of its prover's buffer so that round 2 interpolates them without a per-instance copy; x_poly of every
        instance (state.rs:137-139) in one batched iNTT.  A bad matrix raises CudaError naming the circuit (and the prover, when
        there are several)."""
        jobs, outs, owners = [], [], []
        for n, p in enumerate(provers):
            cs = p.circuits
            slots = [(i, j, m) for i, c in enumerate(cs) for j in range(p.batch[i]) for m in range(3)]
            sizes = [cs[i].constraint_domain.size for i, _j, _m in slots]
            p._zbuf = _zeros(sum(sizes), p.dev)
            offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64).tolist()
            p._zslots = list(zip(offs, sizes))
            mine = [p._zbuf[o: o + cs[i].num_constraints] for o, (i, _j, _m) in zip(offs, slots)]
            jobs += [(mat.row_ptr, mat.cols, mat.vals, p.z[i][j]) for i, j, m in slots for mat in ((cs[i].a, cs[i].b, cs[i].c)[m],)]
            outs += mine
            owners += [(n, slot) for slot in slots]
            p.z_a, p.z_b, p.z_c = ([[None] * b for b in p.batch] for _ in range(3))
            for (i, j, m), out in zip(slots, mine):
                (p.z_a, p.z_b, p.z_c)[m][i][j] = out
        try:
            device.sparse_matvec_batch(jobs, outs)
        except CudaError as e:
            seg = getattr(e, "segment", None)
            if seg is None:
                raise
            n, (i, _j, m) = owners[seg]
            job = f"job {n}: " if len(provers) > 1 else ""
            raise CudaError(e.code, f"{job}circuit {provers[n].positions[i]}: matrix {'abc'[m]} has a column ≥ num_variables or a row_ptr "
                                    "that does not run from 0 to nnz") from None
        pubs = [z[: c.num_public] for p in provers for c, zs in zip(p.circuits, p.z) for z in zs]
        xbuf = torch.cat(pubs) if len(pubs) > 1 else pubs[0].clone()
        offs = np.concatenate([[0], np.cumsum([x.shape[0] for x in pubs])]).astype(np.int64).tolist()
        flat = [xbuf[a: b] for a, b in zip(offs, offs[1:])]
        device.ntt_batch_(flat, NTTDirection.Inverse, NTTType.Standard)
        it = iter(flat)
        for p in provers:
            p.x_polys = p._per_circuit([next(it) for _ in range(sum(p.batch))])

    def _per_circuit(self, flat: list) -> list:
        out, it = [], iter(flat)
        for b in self.batch:
            out.append([next(it) for _ in range(b)])
        return out

    def _combiners(self, batch_combiners) -> list:
        if batch_combiners is None:
            return [(1, [1] * b) for b in self.batch]
        if len(batch_combiners) != len(self.circuits):
            raise ValueError(f"{len(batch_combiners)} sets of batch combiners for {len(self.circuits)} circuits")
        out = []
        for (cc, inst), b in zip(batch_combiners, self.batch):
            if len(inst) != b:
                raise ValueError(f"{len(inst)} instance combiners for {b} instances")
            out.append((int(cc) % R_MOD, [int(x) % R_MOD for x in inst]))
        return out

    # ---- round 1: calculate_w (first.rs:129-160), per instance ----
    def first_round(self):
        self.w_polys = []
        for c, zs, xs in zip(self.circuits, self.z, self.x_polys):
            V, I = c.variable_domain, c.input_domain
            # the index plumbing of calculate_w depends only on the two domain sizes: built once per circuit and device
            cache = c.__dict__.setdefault("_w_index", {})
            if self.dev not in cache:
                ratio = V.size // I.size
                k = torch.arange(V.size, dtype=torch.int64, device=self.dev)
                mask = (k % ratio) != 0
                cache[self.dev] = (k[mask].contiguous(), (k - torch.div(k, ratio, rounding_mode="floor") - 1)[mask].contiguous())
            keep, src = cache[self.dev]
            ws = []
            for z, x_poly in zip(zs, xs):
                w_ext = _zeros(V.size - I.size, self.dev)
                prv = z[c.num_public:]
                w_ext[: prv.shape[0]] = prv
                x_evals = V.fft_in_place(_pad(x_poly, V.size).clone())
                evals = _zeros(V.size, self.dev)
                evals[keep] = device.fr_vec_op(w_ext[src].contiguous(), x_evals[keep].contiguous(), device.FR_SUB)
                w_poly, _rem = divide_by_vanishing(V.ifft_in_place(evals), I)
                ws.append(w_poly)
            self.w_polys.append(ws)
        return self.w_polys

    def set_mask_poly(self, h_1_mask_rand, g_1_mask_rand):
        """calculate_mask_poly (first.rs:102-127) for the hiding mode, over the LARGEST variable domain: rand(degree 3)·v_H plus
        rand(degree 5) with a zero constant term; the random coefficients (ints) are arguments.  A first-round oracle (no degree or
        hiding bound, first.rs:54-56) that enters h_1 / g_1 in the third round."""
        assert len(h_1_mask_rand) == 4 and len(g_1_mask_rand) == 6
        n = self.max_variable_domain.size
        mask = [0] * (n + 4)
        for i, c in enumerate(h_1_mask_rand):
            mask[n + i] = (mask[n + i] + c) % R_MOD
            mask[i] = (mask[i] - c) % R_MOD
        for i, c in enumerate(g_1_mask_rand):
            if i:
                mask[i] = (mask[i] + c) % R_MOD
        idx = sorted(set(range(6)) | set(range(n, n + 4)))              # the (at most ten) non-zero coefficients
        vals = np.array([_mont(mask[i]) for i in idx], dtype=np.uint64).reshape(-1, 4)
        self.mask_poly = _zeros(n + 4, self.dev)
        self.mask_poly[torch.tensor(idx, dtype=torch.int64, device=self.dev)] = torch.from_numpy(vals.view(np.int64)).to(self.dev)
        return self.mask_poly

    # ---- calculate_assignments (third.rs:207-234): z = w·v_I + x, one launch for every instance ----
    def assignments(self):
        return BatchProver._assignments_many([self])[0]

    @staticmethod
    def _assignments_many(provers: list) -> list:
        jobs = []
        for p in provers:
            for c, ws, xs in zip(p.circuits, p.w_polys, p.x_polys):
                I = c.input_domain.size
                for w, x in zip(ws, xs):
                    jobs.append((I + w.shape[0], [(x, _mont(1)), (w, _mont(-1)), (w, _mont(1), I)]))
        it = iter(device.fr_lincomb_terms(jobs))
        for p in provers:
            p.z_polys = p._per_circuit([next(it) for _ in range(sum(p.batch))])
        return [p.z_polys for p in provers]

    # ---- round 2: h_0 (second.rs:76-142) ----
    def second_round(self, batch_combiners=None):
        """h_0 = Σ over circuits and instances of apply_randomized_selector(comb_inst·rowcheck, comb_circuit, R_max, R_i, false).  The
        rowcheck z_A·z_B − z_C has degree < 2|R_i| and z_C degree < |R_i|, so its quotient by v_{R_i} is the upper half of z_A·z_B:
        one batched iNTT, one batched product and one selector sum for the whole batch."""
        return BatchProver._second_round_many([self], [batch_combiners])[0]

    @staticmethod
    def _second_round_many(provers: list, batch_combiners: list) -> list:
        """second_round of every prover (with its own combiners) in the same batched iNTT, product and selector-sum launch"""
        combs = [p._combiners(bc) for p, bc in zip(provers, batch_combiners)]
        abs_ = []
        for p in provers:
            evals = p._zbuf.clone()                                       # z_A, z_B of every instance, interpolated in place
            abs_.append([evals[o: o + n] for k, (o, n) in enumerate(p._zslots) if k % 3 != 2])
        device.ntt_batch_([t for ab in abs_ for t in ab], NTTDirection.Inverse, NTTType.Standard)
        prods = iter(device.polymul_batch([pair for ab in abs_ for pair in zip(ab[0::2], ab[1::2])]))
        jobs = []
        for p, comb in zip(provers, combs):
            R = p.max_constraint_domain
            terms = []
            for c, (cc, inst) in zip(p.circuits, comb):
                n = c.constraint_domain.size
                scale = cc * n % R_MOD * pow(R.size, -1, R_MOD) % R_MOD
                for comb_inst in inst:
                    terms.append((next(prods)[n:], _mont(comb_inst * scale)))
            jobs.append((max(t[0].shape[0] for t in terms), terms))
        for p, h_0 in zip(provers, device.fr_lincomb_terms(jobs)):
            p.h_0 = h_0
        return [p.h_0 for p in provers]

    # ---- evaluate_all_lagrange_coefficients (fft/domain.rs:258-292) on the device ----
    @staticmethod
    def lagrange_coefficients(domain: EvaluationDomain, tau: int, dev) -> torch.Tensor:
        return domain.evaluate_all_lagrange_coefficients(tau, dev)

    # ---- round 3: lineval sumcheck (third.rs:126-218, 280-326) ----
    def third_round(self, alpha: int, eta_b: int, eta_c: int, batch_combiners=None):
        """h_1 and g_1 over C_max (remainder witness, target C_max, source C_i) and the per-instance sums |C_i|·Σ_j coeff_{j·|C_i|}.
        M(α, ·) of every transpose is one segmented mat-vec (α is shared: one Lagrange vector per distinct |R|), their interpolation
        one batched iNTT, the 3·Σ instances products M(α)·z one batched product; the sums and both selector sums are one launch and
        the sums reach the host in one copy."""
        BatchProver._third_round_many([self], [(alpha, eta_b, eta_c)], [batch_combiners])
        return self.g_1, self.h_1

    @staticmethod
    def _third_round_many(provers: list, challenges: list, batch_combiners: list) -> None:
        """third_round of every prover with its own (α, η_b, η_c) and combiners: one Lagrange vector per (prover, distinct |R|), then
        the same mat-vec pass, iNTT, product, sum launch and copy for all of them"""
        combs = [p._combiners(bc) for p, bc in zip(provers, batch_combiners)]
        spmv, pairs, owners = [], [], []
        for p, (alpha, _eb, _ec) in zip(provers, challenges):
            lag = {}
            for c in p.circuits:
                if c.constraint_domain.size not in lag:
                    lag[c.constraint_domain.size] = p.lagrange_coefficients(c.constraint_domain, alpha, p.dev)
            spmv += [(t.row_ptr, t.cols, t.vals, lag[c.constraint_domain.size]) for c in p.circuits for t in c.transposes]
        m_evals = device.sparse_matvec_batch(spmv)
        device.ntt_batch_(m_evals, NTTDirection.Inverse, NTTType.Standard)
        base = 0
        for n, p in enumerate(provers):
            for i, _c in enumerate(p.circuits):
                for j, z_poly in enumerate(p.z_polys[i]):
                    for m in range(3):
                        pairs.append((m_evals[base + 3 * i + m], z_poly))
                        owners.append((n, i, j, m))
            base += 3 * len(p.circuits)
        prods = device.polymul_batch(pairs)
        sums_buf = _zeros(len(prods), provers[0].dev)
        sum_jobs, h_terms, xg_terms = [], [[] for _ in provers], [[] for _ in provers]
        for (n, i, j, m), z_m in zip(owners, prods):
            p, (_alpha, eta_b, eta_c), C = provers[n], challenges[n], provers[n].max_variable_domain
            nv = p.circuits[i].variable_domain.size
            # Σ_{c ∈ C_i} z_m(c) = |C_i| · Σ_j coefficient_{j·|C_i|}
            sum_jobs.append((1, [(z_m[k: k + 1], _mont(1)) for k in range(0, z_m.shape[0], nv)]))
            cc, inst = combs[n][i]
            etas = (1, eta_b % R_MOD, eta_c % R_MOD)
            mult = cc * inst[j] % R_MOD * etas[m] % R_MOD * nv % R_MOD * pow(C.size, -1, R_MOD) % R_MOD
            assert z_m.shape[0] <= 2 * nv
            lo, hi = z_m[:nv], z_m[nv:]
            h_terms[n].append((hi, _mont(mult)))
            # the remainder lo + hi times v_{C_max} / v_{C_i}: |C_max| / |C_i| copies of it, |C_i| apart
            xg_terms[n] += [(lo, _mont(mult), 0, nv, C.size // nv), (hi, _mont(mult), 0, nv, C.size // nv)]
        for n, p in enumerate(provers):
            if p.mask_poly is not None:                                   # third.rs:207-213 (hiding mode)
                h_mask, xg_mask = divide_by_vanishing(p.mask_poly, p.max_variable_domain)
                h_terms[n].append((h_mask, _mont(1)))
                xg_terms[n].append((xg_mask, _mont(1)))
        hx = [job for n, p in enumerate(provers)
              for job in ((max(t[0].shape[0] for t in h_terms[n]), h_terms[n]), (p.max_variable_domain.size, xg_terms[n]))]
        out = device.fr_lincomb_terms(sum_jobs + hx, [sums_buf[k: k + 1] for k in range(len(prods))] + [None] * len(hx))
        for n, p in enumerate(provers):
            p.h_1, xg_1 = out[len(sum_jobs) + 2 * n], out[len(sum_jobs) + 2 * n + 1]
            p.g_1 = xg_1[1:]
            p.third_sums = [[[0, 0, 0] for _ in range(b)] for b in p.batch]
        host = device.fr_from_mont(sums_buf).cpu().numpy().view(np.uint64)
        for (n, i, j, m), row in zip(owners, host):
            nv = provers[n].circuits[i].variable_domain.size
            provers[n].third_sums[i][j][m] = nv * sum(int(v) << (64 * t) for t, v in enumerate(row)) % R_MOD

    # ---- round 4: matrix sumchecks (fourth.rs:79-245) ----
    def fourth_round(self, alpha: int, beta: int):
        """per matrix of every circuit, with that circuit's v_{R_i}(α)·v_{C_i}(β) and |R_i|·|C_i|; the selector goes from K_matrix to the
        global K_max.  The evaluations of all 3K matrices are three launches, their 9K interpolations one batched iNTT, the products
        b·f one batched product, the 3K quotients one launch; the 3K sums f[0] reach the host in one copy."""
        return BatchProver._fourth_round_many([self], [(alpha, beta)])[0]

    @staticmethod
    def _fourth_round_many(provers: list, challenges: list) -> list:
        """fourth_round of every prover with its own (α, β): the matrices of all of them in the same launches, α and β per segment"""
        jobs, doms, kmax = [], [], []
        for p, (alpha, beta) in zip(provers, challenges):
            for c in p.circuits:
                Rd, V = c.constraint_domain, c.variable_domain
                v_rc = _vanish(Rd, alpha) * _vanish(V, beta) % R_MOD
                rc = Rd.size * V.size % R_MOD
                scale = v_rc * pow(Rd.size, -1, R_MOD) % R_MOD * pow(V.size, -1, R_MOD) % R_MOD
                for arith in c.ariths:
                    jobs.append((arith.row, arith.col, arith.row_col_val, _mont(v_rc), _mont(rc), _mont(scale), _mont(alpha), _mont(beta)))
                    doms.append(arith.domain)
                    kmax.append(p.max_non_zero_domain.size)
        evals = device.varuna_round4_evals_batch(jobs)
        device.ntt_batch_([t for trio in evals for t in trio], NTTDirection.Inverse, NTTType.Standard)
        bf = device.polymul_batch([(b, f) for _a, b, f in evals])
        lhs = device.fr_lincomb_terms([(d.size, [(q[d.size:], _mont(-d.size * pow(km, -1, R_MOD)))]) for q, d, km in zip(bf, doms, kmax)])
        f0 = torch.stack([f[0] for _a, _b, f in evals]).cpu().numpy().view(np.uint64)
        base = 0
        for p in provers:
            p.gs, p.lhs, p.fourth_sums, p.a_polys, p.b_polys = [], [], [], [], []
            for i in range(len(p.circuits)):
                at = base + 3 * i
                trio = evals[at: at + 3]
                p.gs.append([f[1:] for _a, _b, f in trio])
                p.lhs.append(lhs[at: at + 3])
                p.fourth_sums.append([_fr_mont_to_int(f0[at + m]) for m in range(3)])
                p.a_polys.append([a for a, _b, _f in trio])
                p.b_polys.append([b for _a, b, _f in trio])
            base += 3 * len(p.circuits)
        return [p.gs for p in provers]

    # ---- round 5 (fifth.rs:43-67): h_2 = Σ δ·lhs over all 3K matrices, one launch ----
    def fifth_round(self, deltas):
        return BatchProver._fifth_round_many([self], [deltas])[0]

    @staticmethod
    def _fifth_round_many(provers: list, deltas: list) -> list:
        for p, ds in zip(provers, deltas):
            if len(ds) != len(p.circuits) or any(len(d) != 3 for d in ds):
                raise ValueError(f"one (δ_a, δ_b, δ_c) per circuit: {len(p.circuits)} circuits")
        jobs = []
        for p, ds in zip(provers, deltas):
            terms = [(lhs, _mont(int(d) % R_MOD)) for dd, ls in zip(ds, p.lhs) for d, lhs in zip(dd, ls)]
            jobs.append((max(t[0].shape[0] for t in terms), terms))
        for p, h_2 in zip(provers, device.fr_lincomb_terms(jobs)):
            p.h_2 = h_2
        return [p.h_2 for p in provers]

    # ---- labels, oracles, linear combinations ----
    def _labels(self):
        """label(i, name, j) of circuit i's polynomial: the reference's witness_label names (ahp.rs:46-50; a_poly / b_poly as
        construct_matrix_linear_combinations names them, ahp.rs:408-409)"""
        return _label_fn(circuit_ids(self.circuits))

    def polynomials(self, label=None) -> dict:
        """label → device polynomial, everything prove_batch hands to open_combinations, in its order (varuna.rs:509-517): the a and b
        polynomials of every circuit, the first-round oracles (w of every instance, then mask_poly), h_0, g_1, h_1, every g_M, h_2"""
        label = label or self._labels()
        out = {}
        for i, ps in enumerate(self.a_polys):
            out.update({label(i, "a_poly", m): p for m, p in enumerate(ps)})
        for i, ps in enumerate(self.b_polys):
            out.update({label(i, "b_poly", m): p for m, p in enumerate(ps)})
        for i, ws in enumerate(self.w_polys):
            out.update({label(i, "w", j): w for j, w in enumerate(ws)})
        if self.mask_poly is not None:
            out["mask_poly"] = self.mask_poly
        out.update({"h_0": self.h_0, "g_1": self.g_1, "h_1": self.h_1})
        for i, gs in enumerate(self.gs):
            out.update({label(i, f"g_{m}", 0): g for m, g in zip("abc", gs)})
        out["h_2"] = self.h_2
        return out

    def oracles(self) -> dict:
        """every polynomial the prover commits to, by round (varuna.rs:387-506)"""
        first = [w for ws in self.w_polys for w in ws] + ([self.mask_poly] if self.mask_poly is not None else [])
        return {1: first, 2: [self.h_0], 3: [self.g_1, self.h_1], 4: [g for gs in self.gs for g in gs], 5: [self.h_2]}

    def labeled_oracles(self, zk: bool = False, label=None, rounds=(1, 2, 3, 4, 5)) -> dict:
        """round → [sonic_pc.LabeledPolynomial] for each of `rounds` (all computed already) with the reference's bounds (first.rs,
        third.rs, fourth.rs polynomial infos): g_1 bounded by |C_max| − 2, each circuit's g_M by its own |K_M| − 2; in the hiding mode
        (zk) w, g_1 and g_M carry hiding bound 1.  Each round's list commits in ONE SonicKZG10.commit pass, whose passes take mixed
        degree bounds as they are."""
        from .sonic_pc import LabeledPolynomial
        label = label or self._labels()
        hb = 1 if zk else None

        def fit(p, bound):                                               # device polynomials may carry trailing zeros
            return p[: bound + 1] if p.shape[0] > bound + 1 else p

        def first():
            out = [LabeledPolynomial(label(i, "w", j), w, None, hb) for i, ws in enumerate(self.w_polys) for j, w in enumerate(ws)]
            if self.mask_poly is not None:
                out.append(LabeledPolynomial("mask_poly", self.mask_poly, None, None))
            return out

        def third():
            bg1 = self.max_variable_domain.size - 2
            return [LabeledPolynomial("g_1", fit(self.g_1, bg1), bg1, hb), LabeledPolynomial("h_1", self.h_1, None, None)]

        def fourth():
            return [LabeledPolynomial(label(i, f"g_{m}", 0), fit(g, d.size - 2), d.size - 2, hb)
                    for i, (c, gs) in enumerate(zip(self.circuits, self.gs)) for m, g, d in zip("abc", gs, c.non_zero_domains)]
        build = {1: first, 2: lambda: [LabeledPolynomial("h_0", self.h_0, None, None)], 3: third, 4: fourth,
                 5: lambda: [LabeledPolynomial("h_2", self.h_2, None, None)]}
        return {r: build[r]() for r in rounds}

    @staticmethod
    def _eval(poly: torch.Tensor, point: int) -> int:
        return _fr_mont_to_int(device.poly_evaluate(poly.contiguous(), _mont(point))) if poly.shape[0] else 0

    def _eval_points(self, beta: int, gamma: int) -> list:
        """the evaluations the linear combinations and the proof need, as (polynomial, point): g_1(β), every g_M(γ), every x(β)"""
        return ([(self.g_1, beta)] + [(g, gamma) for gs in self.gs for g in gs] +
                [(x, beta) for xs in self.x_polys for x in xs])

    def _take_evals(self, vals: list) -> tuple:
        """_eval_points' values → (g_1(β), per circuit [g_a(γ), g_b(γ), g_c(γ)], per circuit per instance x(β))"""
        it = iter(vals)
        g_1 = next(it)
        gs = [[next(it) for _ in range(3)] for _ in self.gs]
        return g_1, gs, [[next(it) for _ in xs] for xs in self.x_polys]

    @staticmethod
    def _evals_many(provers: list, points: list) -> list:
        """_take_evals of every prover at its (β, γ) from one device.poly_evaluate_batch pass"""
        jobs = [p._eval_points(beta, gamma) for p, (beta, gamma) in zip(provers, points)]
        host = device.poly_evaluate_batch([(poly.contiguous(), _mont(x)) for js in jobs for poly, x in js])
        vals = iter(_fr_mont_to_int(row) for row in host)
        return [p._take_evals([next(vals) for _ in js]) for p, js in zip(provers, jobs)]

    def linear_combinations(self, alpha, eta_b, eta_c, beta, deltas, gamma, batch_combiners=None, label=None):
        """AHPForR1CS::construct_linear_combinations (ahp/ahp.rs:172-389) on the prover's side and the query set for K circuits
        (linear_combinations below), with the evaluations it needs (g_1(β), g_M(γ), x(β)) from one device Horner pass"""
        if len(deltas) != len(self.circuits) or any(len(d) != 3 for d in deltas):
            raise ValueError(f"one (δ_a, δ_b, δ_c) per circuit: {len(self.circuits)} circuits")
        g_1_at_beta, g_at_gamma, x_at_beta = BatchProver._evals_many([self], [(beta, gamma)])[0]
        return linear_combinations(self.circuits, self._combiners(batch_combiners), self.third_sums, self.fourth_sums,
                                   (alpha, eta_b, eta_c, beta, deltas, gamma), g_1_at_beta, g_at_gamma, x_at_beta,
                                   label or self._labels(), self.mask_poly is not None)


def linear_combinations(circuits: list, combs: list, third_sums: list, fourth_sums: list, challenges: tuple, g_1_at_beta: int,
                        g_at_gamma: list, x_at_beta: list, label, mask: bool):
    """AHPForR1CS::construct_linear_combinations (ahp/ahp.rs:172-389) and the verifier's query set for K circuits → (lcs, query_set):
    lcs = [(label, [(coefficient, polynomial label or None for LCTerm::One)])] in the reference's BTreeMap order, query_set =
    [(lc label, (point name, point))].  Only numbers go in, so the prover and the verifier share it: per circuit (id order) its
    domains (`circuits[i]` has constraint_domain, variable_domain, input_domain and non_zero_domains), (circuit combiner, instance
    combiners), third sums (per instance) and fourth sums; challenges = (α, η_b, η_c, β, [(δ_a, δ_b, δ_c)], γ); g_1(β); per
    circuit (g_a(γ), g_b(γ), g_c(γ)); per circuit, per instance x(β).  Each circuit's terms are scaled by the selector of its
    domain inside the max domain at α, β and γ.  The matrix sumcheck names each circuit's a_poly / b_poly (the prover's
    polynomials; the verifier expands them into index commitments, ahp.rs:408-445)."""
    alpha, eta_b, eta_c, beta, deltas, gamma = challenges
    cs = circuits
    R = _largest(c.constraint_domain for c in cs)
    C = _largest(c.variable_domain for c in cs)
    K = _largest(d for c in cs for d in c.non_zero_domains)
    lcs = {}
    const = 0
    for c, (cc, inst), sums in zip(cs, combs, third_sums):
        term = sum(comb * (s[0] * s[1] - s[2]) for comb, s in zip(inst, sums)) % R_MOD
        const = (const + cc * _selector(R, c.constraint_domain, alpha) % R_MOD * term) % R_MOD
    lcs["rowcheck_zerocheck"] = [(const, None), ((-_vanish(R, alpha)) % R_MOD, "h_0")]
    lcs["g_1"] = [(1, "g_1")]
    lineval = [(1, "mask_poly")] if mask else []
    batch_lineval_sum = 0
    for i, (c, (cc, inst)) in enumerate(zip(cs, combs)):
        sums4 = [s * d.size % R_MOD for s, d in zip(fourth_sums[i], c.non_zero_domains)]
        weight = (sums4[0] + sums4[1] * eta_b + sums4[2] * eta_c) % R_MOD
        v_x_beta, sel = _vanish(c.input_domain, beta), _selector(C, c.variable_domain, beta)
        for j, comb in enumerate(inst):
            k = cc * comb % R_MOD * sel % R_MOD
            lineval.append((k * weight % R_MOD * x_at_beta[i][j] % R_MOD, None))
            lineval.append((k * weight % R_MOD * v_x_beta % R_MOD, label(i, "w", j)))
        batch_lineval_sum += cc * sum(comb * (s[0] + eta_b * s[1] + eta_c * s[2]) for comb, s in zip(inst, third_sums[i]))
    batch_lineval_sum = batch_lineval_sum % R_MOD * pow(C.size, -1, R_MOD) % R_MOD
    lineval += [((-_vanish(C, beta)) % R_MOD, "h_1"), ((-beta * g_1_at_beta) % R_MOD, None), ((-batch_lineval_sum) % R_MOD, None)]
    lcs["lineval_sumcheck"] = lineval
    points = {"rowcheck_zerocheck": ("alpha", alpha), "g_1": ("beta", beta), "lineval_sumcheck": ("beta", beta),
              "matrix_sumcheck": ("gamma", gamma)}
    matrix = []
    for i, c in enumerate(cs):
        for m, (g_at, s, delta, d) in enumerate(zip(g_at_gamma[i], fourth_sums[i], deltas[i], c.non_zero_domains)):
            g_label = label(i, f"g_{'abc'[m]}", 0)
            lcs[g_label] = [(1, g_label)]
            points[g_label] = ("gamma", gamma)
            selector = _selector(K, d, gamma)
            b_term = (gamma * g_at + s) % R_MOD
            matrix.append((delta * selector % R_MOD, label(i, "a_poly", m)))
            matrix.append(((-delta * selector % R_MOD * b_term) % R_MOD, label(i, "b_poly", m)))
    matrix.append(((-_vanish(K, gamma)) % R_MOD, "h_2"))
    lcs["matrix_sumcheck"] = matrix
    order = sorted(lcs)
    return [(k, lcs[k]) for k in order], [(k, points[k]) for k in order]


def _short_label(_i, name, j=0):
    """the one-circuit labels: w_{j}, g_{m}, a_poly_{m}, b_poly_{m}"""
    if name in ("a_poly", "b_poly"):
        return f"{name}_{'abc'[j]}"
    return name if name.startswith("g_") else f"{name}_{j}"


class Prover:
    """BatchProver of one circuit, with the one-circuit interface: `assignments` is one CUDA tensor [num_variables, 4] per instance
    (padded public variables, the first one One, then private); attributes are the circuit's own lists, labels are short (w_{j}, g_{m},
    a_poly_{m}, b_poly_{m}).  The circuit id is never computed."""

    def __init__(self, circuit: Circuit, assignments: list):
        self._b = BatchProver([(circuit, assignments)])
        self.circuit = circuit
        self.batch = len(assignments)
        self.z = self._b.z[0]

    lagrange_coefficients = staticmethod(BatchProver.lagrange_coefficients)
    _eval = staticmethod(BatchProver._eval)

    def _combiners(self, circuit_combiner, instance_combiners):
        return [(circuit_combiner, instance_combiners or [1] * self.batch)]

    z_a = property(lambda self: self._b.z_a[0])
    z_b = property(lambda self: self._b.z_b[0])
    z_c = property(lambda self: self._b.z_c[0])
    x_polys = property(lambda self: self._b.x_polys[0])
    w_polys = property(lambda self: self._b.w_polys[0])
    z_polys = property(lambda self: self._b.z_polys[0])
    h_0 = property(lambda self: self._b.h_0)
    g_1 = property(lambda self: self._b.g_1)
    h_1 = property(lambda self: self._b.h_1)
    h_2 = property(lambda self: self._b.h_2)
    mask_poly = property(lambda self: self._b.mask_poly)
    third_sums = property(lambda self: self._b.third_sums[0])
    gs = property(lambda self: self._b.gs[0])
    lhs = property(lambda self: self._b.lhs[0])
    fourth_sums = property(lambda self: self._b.fourth_sums[0])
    a_polys = property(lambda self: self._b.a_polys[0])
    b_polys = property(lambda self: self._b.b_polys[0])

    def first_round(self):
        return self._b.first_round()[0]

    def assignments(self):
        return self._b.assignments()[0]

    def second_round(self, circuit_combiner: int = 1, instance_combiners=None):
        return self._b.second_round(self._combiners(circuit_combiner, instance_combiners))

    def third_round(self, alpha: int, eta_b: int, eta_c: int, circuit_combiner: int = 1, instance_combiners=None):
        return self._b.third_round(alpha, eta_b, eta_c, self._combiners(circuit_combiner, instance_combiners))

    def set_mask_poly(self, h_1_mask_rand, g_1_mask_rand):
        return self._b.set_mask_poly(h_1_mask_rand, g_1_mask_rand)

    def fourth_round(self, alpha: int, beta: int):
        return self._b.fourth_round(alpha, beta)[0]

    def fifth_round(self, deltas):
        return self._b.fifth_round([deltas])

    def polynomials(self) -> dict:
        """label → device polynomial, everything prove_batch hands to open_combinations (varuna.rs:509-517)"""
        return self._b.polynomials(_short_label)

    def oracles(self) -> dict:
        return self._b.oracles()

    def linear_combinations(self, alpha, eta_b, eta_c, beta, deltas, gamma, circuit_combiner: int = 1, instance_combiners=None):
        """→ (lcs, query_set) exactly as oracle/varuna.py Prover.linear_combinations"""
        return self._b.linear_combinations(alpha, eta_b, eta_c, beta, [deltas], gamma, self._combiners(circuit_combiner, instance_combiners),
                                           _short_label)


def test_circuit_csr(a: int, b: int, mul_depth: int, num_constraints: int, num_variables: int, dev):
    """TestCircuit (data_structures/test_circuit.rs:42-139) laid out directly as CSR matrices and one assignment, with the public
    variables padded to a power of two: every A, B, C row has a single unit entry.  Returns (Circuit, assignment tensor)."""
    num_public = 1 + mul_depth
    padded = 1 << (num_public - 1).bit_length() if num_public > 1 else 1
    num_private = num_variables - num_public
    nv = padded + num_private
    va, vb = padded + 0, padded + 1                                   # private variables a, b
    mul = [1 + i for i in range(mul_depth)]                            # public mul_var i
    mul_constraints = mul_depth - 1
    plain = num_constraints - mul_constraints
    a_cols = np.array([va] * plain + [mul[i] for i in range(mul_constraints)], dtype=np.int64)
    b_cols = np.full(num_constraints, vb, dtype=np.int64)
    c_cols = np.array([mul[0]] * plain + [mul[i + 1] for i in range(mul_constraints)], dtype=np.int64)
    row_ptr = np.arange(num_constraints + 1, dtype=np.int64)
    ones = np.tile(_mont(1), (num_constraints, 1))
    mats = [Matrix(row_ptr, cols, ones, dev) for cols in (a_cols, b_cols, c_cols)]
    circuit = Circuit(mats[0], mats[1], mats[2], padded, nv)
    z = np.zeros((nv, 4), dtype=np.uint64)
    z[0] = _mont(1)
    v = a % R_MOD
    for i in range(mul_depth):
        v = v * b % R_MOD
        z[1 + i] = _mont(v)
    z[padded:] = _mont(a)
    z[vb] = _mont(b)
    return circuit, torch.from_numpy(z.view(np.int64)).to(dev)


# ---- prove_batch: the prover's Fiat–Shamir transcript and the Proof (varuna.rs:136-194, 336-620; data_structures/proof.rs) ----

class TranscriptOps:
    """The operation list of one PoseidonSponge<Fq, 2, 1> transcript, queued on the host in the layout of
    device.poseidon_transcripts: absorbs take their elements from this transcript's own inputs, squeezes write this transcript's own
    outputs (offsets from zero).  `permutations` counts what running the list costs, from the mode and index alone, with the kernel's
    lazy rule (a permutation before the first element of a full rate, or of a change of direction)."""

    def __init__(self):
        self._ops, self._inputs, self._nin, self._nout = [], [], 0, 0
        self._squeezing, self._idx = False, 0
        self.permutations = 0

    def _advance(self, absorb: bool, count: int):
        if count == 0:
            return
        if absorb == self._squeezing:
            self._idx, self._squeezing = poseidon.RATE, not absorb
        first = poseidon.RATE - self._idx                                 # elements that fit before the next permutation
        if count > first:
            self.permutations += -(-(count - first) // poseidon.RATE)
            self._idx = (count - first - 1) % poseidon.RATE + 1
        else:
            self._idx += count

    def absorb_native(self, words: np.ndarray):
        """absorb_native_field_elements of Montgomery Fq words uint32[n, 12]"""
        words = np.ascontiguousarray(words, dtype=np.uint32).reshape(-1, 12)
        if words.shape[0]:
            self._ops.append((poseidon.OP_ABSORB, words.shape[0], self._nin))
            self._inputs.append(words)
            self._nin += words.shape[0]
            self._advance(True, words.shape[0])

    def absorb_bytes(self, data: bytes):
        self.absorb_native(poseidon.to_mont_words(poseidon.FIELD_FQ, poseidon.bytes_to_field_elements(data, poseidon.FIELD_FQ)))

    def absorb_nonnative(self, values):
        """absorb_nonnative_field_elements of canonical Fr values: one call, compressed over its own stream"""
        self.absorb_native(poseidon.to_mont_words(poseidon.FIELD_FQ, poseidon.nonnative_field_elements(values)))

    def absorb_commitments(self, comms):
        """absorb_native_field_elements of commitments (normalised projective uint64[k, 18])"""
        self.absorb_native(_commitment_elements(comms))

    def queue_squeeze(self, counts: list, short: bool = False):
        """one squeeze_nonnative_field_elements(n) call (squeeze_short_… when `short`) per entry of `counts`"""
        kind = poseidon.OP_SQUEEZE_SHORT_NONNATIVE if short else poseidon.OP_SQUEEZE_NONNATIVE
        width = 168 if short else 252
        for n in counts:
            self._ops.append((kind, n, self._nout))
            self._nout += n
            self._advance(False, -(-n * width // (poseidon.FIELDS[poseidon.FIELD_FQ][1] - 1)))

    def inputs(self) -> np.ndarray:
        return np.concatenate(self._inputs) if self._inputs else np.zeros((0, 12), dtype=np.uint32)


class Transcript(TranscriptOps):
    """The prover's PoseidonSponge<Fq, 2, 1>, its state kept in HBM between calls as one state record
    (device.poseidon_transcripts with `state`).  Absorbs only queue operations; `squeeze` runs everything queued and its squeezes
    in one device call, so a round costs one call.  `calls` and `permutations` count what the sponge has run.  `state`, when given,
    is the record to use (a row of a tensor whose rows are the records of several transcripts that squeeze together,
    squeeze_many)."""

    def __init__(self, dev, state: torch.Tensor | None = None):
        super().__init__()
        self.dev = torch.device(dev)
        self.state = poseidon.fresh_states(poseidon.FIELD_FQ, 1, self.dev) if state is None else state
        self.calls = 0

    def squeeze(self, counts: list, short: bool = False) -> list:
        """one squeeze_nonnative_field_elements(n) call (squeeze_short_… when `short`) per entry of `counts`, after everything
        queued, in one device call → [[canonical Fr] per call]"""
        return squeeze_many([self], [counts], self.state, short)[0]


def squeeze_many(transcripts: list, counts: list, states: torch.Tensor, short: bool = False) -> list:
    """Transcript.squeeze of every transcript with its own `counts`, all of them as transcripts of ONE device.poseidon_transcripts
    call.  `states`: the state records of the transcripts, in order, as the rows of one tensor (each transcript's `state` a view of
    its row) → per transcript [[canonical Fr] per call].  A malformed operation or record raises CudaError whose .transcript is the
    index of the lowest such transcript in `transcripts`."""
    ops_all, starts, inputs, nin, nfr, offs = [], [0], [], 0, 0, []
    for t, cs in zip(transcripts, counts):
        t.queue_squeeze(cs, short)
        ops = np.array(t._ops, dtype=np.int64).reshape(-1, 3)
        ops[:, 2] += np.where(ops[:, 0] == poseidon.OP_ABSORB, nin, nfr)
        ops_all.append(ops)
        starts.append(starts[-1] + ops.shape[0])
        inputs.append(t.inputs())
        offs.append(nfr)
        nin += t._nin
        nfr += t._nout
    dev = transcripts[0].dev
    _out, fr = device.poseidon_transcripts(poseidon.FIELD_FQ, torch.from_numpy(np.concatenate(ops_all).astype(np.int32)).to(dev),
                                           torch.tensor(starts, dtype=torch.int32, device=dev),
                                           torch.from_numpy(np.concatenate(inputs).view(np.int64)).to(dev), 0, nfr, states)
    vals = [_fr_mont_to_int(row) for row in fr.cpu().numpy().view(np.uint64)] if nfr else []
    out = []
    for t, cs, off in zip(transcripts, counts, offs):
        t.calls += 1
        t._ops, t._inputs, t._nin, t._nout = [], [], 0, 0
        mine, k = [], off
        for n in cs:
            mine.append(vals[k: k + n])
            k += n
        out.append(mine)
    return out


@dataclass
class Commitments:
    """data_structures/proof.rs Commitments: normalised projective uint64[18] each, circuits in id order"""
    witness_commitments: list                  # w of every instance, circuit by circuit
    mask_poly: np.ndarray | None               # the hiding mode only
    h_0: np.ndarray
    g_1: np.ndarray
    h_1: np.ndarray
    g_a_commitments: list
    g_b_commitments: list
    g_c_commitments: list
    h_2: np.ndarray


@dataclass
class Evaluations:
    """data_structures/proof.rs Evaluations: g_1(β) and every circuit's g_a, g_b, g_c at γ, canonical integers"""
    g_1_eval: int
    g_a_evals: list
    g_b_evals: list
    g_c_evals: list

    def to_field_elements(self) -> list:
        """the order prove_batch absorbs them in (proof.rs:212-219)"""
        return [self.g_1_eval] + list(self.g_a_evals) + list(self.g_b_evals) + list(self.g_c_evals)


@dataclass
class Proof:
    """data_structures/proof.rs Proof, in memory: per circuit (id order) its batch size; the commitments; the evaluations; the third
    round's sums (per circuit, per instance (sum_a, sum_b, sum_c)) and the fourth round's (per circuit); the BatchLCProof — one
    (w uint64[18], random_v: Montgomery Fr uint64[4] in the hiding mode, else None) per query point (α, β, γ)."""
    batch_sizes: list
    commitments: Commitments
    evaluations: Evaluations
    third_sums: list
    fourth_sums: list
    pc_proof: list

    def check_batch_sizes(self) -> None:
        """Proof::check_batch_sizes (proof.rs): every per-instance and per-circuit list matches the batch sizes; ValueError if not"""
        K, total = len(self.batch_sizes), sum(self.batch_sizes)
        c, e = self.commitments, self.evaluations
        if (len(c.witness_commitments) != total or any(b == 0 for b in self.batch_sizes)
                or not len(c.g_a_commitments) == len(c.g_b_commitments) == len(c.g_c_commitments) == K
                or not len(e.g_a_evals) == len(e.g_b_evals) == len(e.g_c_evals) == K
                or [len(s) for s in self.third_sums] != list(self.batch_sizes) or len(self.fourth_sums) != K):
            raise ValueError("InvalidBatchSize: the proof's lists do not match its batch sizes")

    def to_bytes(self, compress: bool = True, device_="cuda") -> bytes:
        """the bytes of CanonicalSerialize (compressed: ToBytes), every point through one device.g1_serialize call"""
        return _to_bytes_many(_proof_parts, [self], compress, device_)[0]

    @staticmethod
    def read(blob, offset: int = 0, compress: bool = True, validate: bool = True, device_="cuda"):
        """the Proof whose bytes start at `offset` of `blob` → (Proof, the offset after it); errors as proofs_from_bytes"""
        objs, ends = _from_bytes_many(_walk_proof, [blob], [offset], compress, validate, device_)
        return objs[0], ends[0]

    @staticmethod
    def from_bytes(blob, compress: bool = True, validate: bool = True, device_="cuda") -> "Proof":
        """the Proof at the start of `blob` (FromBytes when compressed); trailing bytes are ignored"""
        return Proof.read(blob, 0, compress, validate, device_)[0]


def _union_committer_key(cks: list):
    """CommitterUnionKey::union (sonic_pc/data_structures.rs) of committer keys trimmed from one SRS: the longest powers, every
    enforced degree bound"""
    from .sonic_pc import CommitterKey
    if len(cks) == 1:
        return cks[0]
    if all(ck.max_degree is not None for ck in cks):
        if len({ck.max_degree for ck in cks}) != 1:
            raise ValueError("the committer keys come from different universal parameters")
    else:
        # a key read from bytes does not carry its SRS's degree, but every key trimmed from one SRS ends its shifted powers on
        # the SRS's last power
        lasts = [ck.shifted_powers_of_beta_g[-1] for ck in cks if ck.shifted_powers_of_beta_g is not None and
                 ck.shifted_powers_of_beta_g.shape[0]]
        if len(lasts) != len(cks) or not all(torch.equal(lasts[0], t) for t in lasts[1:]):
            raise ValueError("the committer keys come from different universal parameters")
    max_degree = next((ck.max_degree for ck in cks if ck.max_degree is not None), None)
    longest = max(cks, key=lambda ck: ck.powers_of_beta_g.shape[0])
    bounds = sorted({b for ck in cks for b in (ck.enforced_degree_bounds or [])})
    shifted, gamma = None, {}
    for ck in cks:
        if ck.enforced_degree_bounds:
            gamma.update(ck.shifted_powers_of_beta_times_gamma_g)
            if ck.enforced_degree_bounds[-1] == bounds[-1]:
                shifted = ck.shifted_powers_of_beta_g
    return CommitterKey(longest.powers_of_beta_g, longest.powers_of_beta_times_gamma_g, {}, shifted, gamma or None, bounds or None,
                        max_degree)


def _public_inputs(prover: "BatchProver") -> list:
    """every instance's padded public input as canonical integers: per circuit (id order), per instance"""
    out = []
    for c, zs in zip(prover.circuits, prover.z):
        host = device.fr_from_mont(torch.cat([z[: c.num_public] for z in zs])).cpu().numpy().view(np.uint64)
        vals = [sum(int(v) << (64 * t) for t, v in enumerate(row)) for row in host]
        out.append([vals[j * c.num_public: (j + 1) * c.num_public] for j in range(len(zs))])
    return out


def _prove_batch(pks_to_assignments: list, zk: bool = False, rng=None):
    """prove_batch (below) → (Proof, challenges, transcript): challenges is a dict of everything the transcript yielded"""
    return _prove_batch_many([pks_to_assignments], zk, None if rng is None else [rng])[0]


def prove_batch(pks_to_assignments: list, zk: bool = False, rng=None) -> Proof:
    """VarunaSNARK::prove_batch (varuna.rs:336-620) → Proof.  `pks_to_assignments`: [(CircuitProvingKey, [assignment, …])], an
    assignment as BatchProver takes it; the circuits are proved in id order, so the order of the list changes nothing.  Every
    challenge comes from the prover's own Fiat–Shamir transcript (PoseidonSponge<Fq, 2, 1>, one device call per round):
        init_sponge      the protocol name; per circuit its batch size (u64 LE) and each instance's padded public input (nonnative);
                         every circuit's twelve vk commitments
        round 1          w of every instance (and mask_poly) → per circuit batch_size − 1 (+ 1 after the first circuit) combiners
        round 2          h_0 → α, η_b, η_c          round 3   g_1, h_1, every instance's sums → β
        round 4          every g_a, g_b, g_c, every circuit's sums → δ (two for the first circuit, three for each further one)
        round 5          h_2 → γ
        openings         the evaluations (nonnative) → per query point one short challenge per linear combination, then the randomizer
    The vanishing polynomial of the largest constraint, variable and non-zero domain must not vanish at α, β and γ (ValueError).
    The committer key is the union of the proving keys' keys.  In the hiding mode (zk) the mask polynomial (4 then 6 coefficients)
    and each hiding commitment's blinding polynomial (3 coefficients, in commitment order) are drawn from `rng` (anything with
    randrange; a SystemRandom when None).  That stream cannot equal the reference's ChaCha stream, so a hiding proof is valid but not
    the reference's bytes; a non-hiding proof is deterministic.  This is prove_batch_many with one job."""
    return _prove_batch(pks_to_assignments, zk, rng)[0]


def prove_batch_many(jobs: list, zk: bool = False, rngs: list | None = None, stats: dict | None = None) -> list:
    """prove_batch of every job in `jobs` (each a pks_to_assignments list) in one call → one Proof per job, in input order.  Proof k
    is byte for byte prove_batch(jobs[k]) when not hiding, and prove_batch(jobs[k], True, rngs[k]) in the hiding mode: job k draws
    from its own rng (`rngs`: one per job, or None for a SystemRandom each) in prove_batch's order, the mask and then the blindings
    in commitment order.  The jobs run through the rounds in lockstep and share every device call of a round:
        transcript     the queued operations of every job's sponge as transcripts of one device.poseidon_transcripts call (their
                       state records rows of one tensor), six calls in all
        rounds         each segmented pass BatchProver makes for one job (mat-vecs, batched NTTs and products, linear combinations,
                       round 4 with each job's α and β) over the segments of all jobs; the Lagrange vectors at α stay one call per
                       (job, |R|), round 1's per-instance work stays per instance
        commitments    each round's polynomials of every job in one device.sonic_commit_batch pass (SonicKZG10.commit_many)
        evaluations    g_1(β), every g_M(γ) and every x(β) of every job in one device.poly_evaluate_batch pass
        openings       every job's linear combinations in one pass (SonicKZG10.open_combinations_many)
    Every job's round polynomials are resident at once: a caller whose jobs do not fit in device memory splits the call.
    ValueError, naming the lowest job at fault, for an empty `jobs`, an empty job, an instance that does not match its index, jobs on
    different devices, committer keys of different SRSs, and a vanishing polynomial that is zero at α, β or γ; nothing is returned
    then.  A transcript's CudaError names the job.  `stats`, when given, receives the seconds of each stage ("transcript", "rounds",
    "commitments", "openings", "host" for the rest) and the counts "transcript_calls" and "commitment_passes"."""
    return [proof for proof, _ch, _t in _prove_batch_many(jobs, zk, rngs, stats)]


def _prove_batch_many(jobs: list, zk: bool = False, rngs: list | None = None, stats: dict | None = None) -> list:
    """prove_batch_many → [(Proof, challenges, transcript)] per job"""
    import time
    from .sonic_pc import LabeledPolynomial, Randomness, SonicKZG10
    clock = time.perf_counter
    t_start = clock()
    spent = {"transcript": 0.0, "rounds": 0.0, "commitments": 0.0, "openings": 0.0}
    passes = [0]
    if not jobs:
        raise ValueError("EmptyBatch: no jobs to prove")
    P = len(jobs)
    if zk:
        rngs = [random.SystemRandom() for _ in jobs] if rngs is None else list(rngs)
        if len(rngs) != P:
            raise ValueError(f"{len(rngs)} rngs for {P} jobs")
    provers, cks, pks = [], [], []
    for k, job in enumerate(jobs):
        try:
            if not job:
                raise ValueError("EmptyBatch: no circuits to prove")
            p = BatchProver.__new__(BatchProver)
            p._setup([(pk.circuit, list(zs)) for pk, zs in job])
            if k and p.dev != provers[0].dev:
                raise ValueError(f"the job is on {p.dev}, job 0 on {provers[0].dev}: every job must be on one device")
            pks.append([job[i][0] for i in p.positions])
            cks.append(_union_committer_key([pk.committer_key for pk in pks[-1]]))
        except ValueError as e:
            raise ValueError(f"job {k}: {e}") from None
        provers.append(p)
    dev = provers[0].dev

    def timed(stage, fn, *args):
        t = clock()
        out = fn(*args)
        if stats is not None and stage == "rounds":
            torch.cuda.synchronize(dev)
        spent[stage] += clock() - t
        return out

    def rand_fr(k, n):
        return [rngs[k].randrange(R_MOD) for _ in range(n)]

    timed("rounds", BatchProver._load_many, provers)
    # init_sponge (varuna.rs:136-153): one state record per job, rows of one tensor
    states = poseidon.fresh_states(poseidon.FIELD_FQ, P, dev)
    ts = [Transcript(dev, states[k: k + 1]) for k in range(P)]
    for t, p, pk in zip(ts, provers, pks):
        _init_sponge(t, p.batch, _public_inputs(p), [x.circuit_verifying_key.circuit_commitments for x in pk])

    def squeeze(counts, short=False):
        try:
            return timed("transcript", squeeze_many, ts, counts, states, short)
        except CudaError as e:
            if getattr(e, "transcript", None) is None:
                raise
            err = CudaError(e.code, f"job {e.transcript}: its transcript's operations or state record are malformed")
            err.job = e.transcript
            raise err from None

    def check_vanishing(points, domains, name):
        for k, (x, d) in enumerate(zip(points, domains)):
            if _vanish(d, x) == 0:
                raise ValueError(f"job {k}: the vanishing polynomial of the largest domain is zero at {name}")

    labels = [p._labels() for p in provers]
    rounds, rands, comms = [{} for _ in provers], [{} for _ in provers], [{} for _ in provers]

    def round_commit(r):
        items = []
        for k, p in enumerate(provers):
            rounds[k][r] = p.labeled_oracles(zk, labels[k], rounds=(r,))[r]
            blind = [None if lp.hiding_bound is None else
                     torch.from_numpy(np.array([_mont(v) for v in rand_fr(k, lp.hiding_bound + 2)], dtype=np.uint64).view(np.int64)).to(dev)
                     for lp in rounds[k][r]]
            items.append((cks[k], rounds[k][r], blind))
        passes[0] += 1
        for k, (c, rr) in enumerate(timed("commitments", SonicKZG10.commit_many, items)):
            comms[k][r], rands[k][r] = list(c), list(rr)
            ts[k].absorb_commitments(np.stack(comms[k][r]))

    # round 1
    if zk:
        for k, p in enumerate(provers):
            p.set_mask_poly(rand_fr(k, 4), rand_fr(k, 6))
    for p in provers:
        timed("rounds", p.first_round)
    timed("rounds", BatchProver._assignments_many, provers)
    round_commit(1)
    elems = squeeze([[b - 1 + (1 if i else 0) for i, b in enumerate(p.batch)] for p in provers])
    combs = [[(e[b - 1] if i else 1, [1] + e[: b - 1]) for i, (b, e) in enumerate(zip(p.batch, el))] for p, el in zip(provers, elems)]
    # round 2
    timed("rounds", BatchProver._second_round_many, provers, combs)
    round_commit(2)
    abc = [o[0] for o in squeeze([[3]] * P)]
    check_vanishing([x[0] for x in abc], [p.max_constraint_domain for p in provers], "α")
    # round 3
    timed("rounds", BatchProver._third_round_many, provers, abc, combs)
    round_commit(3)
    for t, p in zip(ts, provers):
        for sums in p.third_sums:
            for s in sums:
                t.absorb_nonnative(s)
    betas = [o[0][0] for o in squeeze([[1]] * P)]
    check_vanishing(betas, [p.max_variable_domain for p in provers], "β")
    # round 4
    timed("rounds", BatchProver._fourth_round_many, provers, [(x[0], b) for x, b in zip(abc, betas)])
    round_commit(4)
    for t, p in zip(ts, provers):
        for s in p.fourth_sums:
            t.absorb_nonnative(s)
    deltas = [[[1] + d[0]] + d[1:] for d in squeeze([[2] + [3] * (len(p.circuits) - 1) for p in provers])]
    # round 5
    timed("rounds", BatchProver._fifth_round_many, provers, deltas)
    round_commit(5)
    gammas = [o[0][0] for o in squeeze([[1]] * P)]
    check_vanishing(gammas, [p.max_non_zero_domain for p in provers], "γ")

    # the evaluations of every job in one pass, then the linear combinations and the openings
    evals = timed("openings", BatchProver._evals_many, provers, list(zip(betas, gammas)))
    lcs, evaluations, per_point = [], [], []
    for k, p in enumerate(provers):
        (alpha, eta_b, eta_c), beta, gamma = abc[k], betas[k], gammas[k]
        g_1_at_beta, g_at_gamma, x_at_beta = evals[k]
        lcs.append(linear_combinations(p.circuits, p._combiners(combs[k]), p.third_sums, p.fourth_sums,
                                       (alpha, eta_b, eta_c, beta, deltas[k], gamma), g_1_at_beta, g_at_gamma, x_at_beta, labels[k],
                                       p.mask_poly is not None))
        evaluations.append(Evaluations(g_1_at_beta, *([g[m] for g in g_at_gamma] for m in range(3))))
        ts[k].absorb_nonnative(evaluations[k].to_field_elements())
        # open_combinations: per point (by name), one short challenge per linear combination opened there, then `_randomizer`
        count = {}
        for _lc, (point_name, _x) in lcs[k][1]:
            count[point_name] = count.get(point_name, 0) + 1
        per_point.append(sum(n + 1 for n in count.values()))
    opening = [[x for [x] in o] for o in squeeze([[1] * n for n in per_point], short=True)]
    items = []
    for k, p in enumerate(provers):
        polys = p.polynomials(labels[k])
        ab = [LabeledPolynomial(key, v, None, None) for key, v in polys.items() if "_a_poly_" in key or "_b_poly_" in key]
        labeled = ab + [lp for r in sorted(rounds[k]) for lp in rounds[k][r]]
        rr = [Randomness() for _ in ab] + [x for r in sorted(rands[k]) for x in rands[k][r]]
        items.append((cks[k], lcs[k][0], labeled, rr, lcs[k][1], iter(opening[k])))
    passes[0] += 1
    pc_proofs = timed("openings", SonicKZG10.open_combinations_many, items)

    out = []
    for k, p in enumerate(provers):
        K, c = len(p.circuits), comms[k]
        nw = sum(p.batch)
        gs = [c[4][3 * i: 3 * i + 3] for i in range(K)]
        commitments = Commitments(c[1][:nw], c[1][nw] if zk else None, c[2][0], c[3][0], c[3][1], [g[0] for g in gs], [g[1] for g in gs],
                                  [g[2] for g in gs], c[5][0])
        proof = Proof(list(p.batch), commitments, evaluations[k], [[list(s) for s in sums] for sums in p.third_sums],
                      [list(s) for s in p.fourth_sums], pc_proofs[k])
        proof.check_batch_sizes()
        alpha, eta_b, eta_c = abc[k]
        challenges = {"batch_combiners": combs[k], "alpha": alpha, "eta_b": eta_b, "eta_c": eta_c, "beta": betas[k], "deltas": deltas[k],
                      "gamma": gammas[k], "opening": opening[k]}
        out.append((proof, challenges, ts[k]))
    if stats is not None:
        stats.update(spent)
        stats["host"] = clock() - t_start - sum(spent.values())
        stats["transcript_calls"] = ts[0].calls
        stats["commitment_passes"] = passes[0]
    return out


# ---- verify_batch: the verifier (varuna.rs:625-933; sonic_pc/mod.rs:344-411, 477-544, 582-677) ----

class _KeyDomains:
    """the domains of a verifying key's CircuitInfo, under Circuit's attribute names (what linear_combinations reads)"""

    def __init__(self, info: CircuitInfo):
        self.constraint_domain = EvaluationDomain.new(info.num_constraints)
        self.variable_domain = EvaluationDomain.new(info.num_public_and_private_variables)
        self.input_domain = EvaluationDomain.new(info.num_public_inputs)
        self.non_zero_domains = [EvaluationDomain.new(n) for n in (info.num_non_zero_a, info.num_non_zero_b, info.num_non_zero_c)]
        if None in [self.constraint_domain, self.variable_domain, self.input_domain] + self.non_zero_domains:
            raise ValueError("a domain of the circuit info is above the 2-adicity of Fr")


_FQ_ONE = np.frombuffer(_FQ_R.to_bytes(48, "little"), dtype=np.uint64)
_OPENING_POINTS = ("alpha", "beta", "gamma")          # the query set's point names, in the BTreeMap order batch_check walks


def _fr_value(v, what: str) -> int:
    v = int(v)
    if not 0 <= v < R_MOD:
        raise ValueError(f"{what} is not below r")
    return v


def _outside_image(comm, what: str) -> np.ndarray:
    """a normalised projective image (X, Y, one) or (·, ·, zero) from the caller → its Affine image"""
    return _affine(_normalised(comm, what))


class _ProofView:
    """one (keys_to_inputs, proof) entry after the checks verify_batch makes before the transcript: circuits in id order, their
    domains, the padded public inputs, and every G1 point taken from the caller (labels, names, Affine images)"""

    def __init__(self, keys_to_inputs: list, proof: Proof):
        if not keys_to_inputs:
            raise ValueError("EmptyBatch: no verifying keys")
        proof.check_batch_sizes()
        if len(proof.batch_sizes) != len(keys_to_inputs):
            raise ValueError(f"batch_sizes: the proof has {len(proof.batch_sizes)} circuits, the call {len(keys_to_inputs)}")
        for k, (vk, _inputs) in enumerate(keys_to_inputs):
            if vk.id is None:
                raise ValueError(f"verifying key {k} has no circuit id")
        order = sorted(range(len(keys_to_inputs)), key=lambda k: bytes(keys_to_inputs[k][0].id))
        self.vks = [keys_to_inputs[k][0] for k in order]
        self.ids = [bytes(vk.id) for vk in self.vks]
        if len(set(self.ids)) != len(self.ids):
            raise ValueError("two verifying keys have equal circuit ids")
        self.domains = [_KeyDomains(vk.circuit_info) for vk in self.vks]
        self.inputs = []
        for i, (k, b) in enumerate(zip(order, proof.batch_sizes)):
            inputs, size = keys_to_inputs[k][1], self.domains[i].input_domain.size
            if not inputs:
                raise ValueError(f"public inputs of verifying key {k}: EmptyBatch")
            if len(inputs) != b:
                raise ValueError(f"public inputs of verifying key {k}: {len(inputs)} inputs for a batch of {b}")
            padded = []
            for j, x in enumerate(inputs):
                x = [_fr_value(v, f"public input {j} of verifying key {k}") for v in x]
                if not x or x[0] != 1:
                    raise ValueError(f"public input {j} of verifying key {k}: the first element is not one")
                if len(x) > size:
                    raise ValueError(f"public input {j} of verifying key {k}: {len(x)} elements for an input domain of {size}")
                padded.append(x + [0] * (size - len(x)))
            self.inputs.append(padded)
        if len(proof.pc_proof) != len(_OPENING_POINTS) or any(len(e) != 2 for e in proof.pc_proof):
            raise ValueError(f"pc_proof: one (w, random_v) per query point ({len(_OPENING_POINTS)}) expected")
        for name, vals in (("third_sums", [s for sums in proof.third_sums for t in sums for s in t]),
                           ("fourth_sums", [s for t in proof.fourth_sums for s in t]), ("evaluations", proof.evaluations.to_field_elements())):
            for v in vals:
                _fr_value(v, name)
        if any(len(t) != 3 for sums in proof.third_sums for t in sums) or any(len(t) != 3 for t in proof.fourth_sums):
            raise ValueError("third_sums / fourth_sums: three sums per entry expected")
        self.random_v = [None if v is None else _fr_mont_to_int(v) for _w, v in proof.pc_proof]
        self.label = _label_fn(self.ids)
        c = proof.commitments
        pts = []                                                         # (label, name, commitment)
        for i, vk in enumerate(self.vks):
            comms = np.ascontiguousarray(vk.circuit_commitments, dtype=np.uint64).reshape(-1, 18)
            if comms.shape[0] != len(INDEX_POLYNOMIAL_NAMES):
                raise ValueError(f"verifying key {order[i]}: {comms.shape[0]} circuit commitments")
            pts += [(f"circuit_{self.ids[i].hex()}_{n}", f"verifying key {order[i]} commitment {n}", x)
                    for n, x in zip(INDEX_POLYNOMIAL_NAMES, comms)]
        it = iter(c.witness_commitments)
        for i, b in enumerate(proof.batch_sizes):
            pts += [(self.label(i, "w", j), f"witness_commitments[{sum(proof.batch_sizes[:i]) + j}]", next(it)) for j in range(b)]
        if c.mask_poly is not None:
            pts.append(("mask_poly", "mask_poly", c.mask_poly))
        pts += [("h_0", "h_0", c.h_0), ("g_1", "g_1", c.g_1), ("h_1", "h_1", c.h_1)]
        for i in range(len(self.vks)):
            for m in "abc":
                pts.append((self.label(i, f"g_{m}", 0), f"g_{m}_commitments[{i}]", getattr(c, f"g_{m}_commitments")[i]))
        pts.append(("h_2", "h_2", c.h_2))
        pts += [(f"w_{p}", f"pc_proof[{p}].w", w) for p, (w, _v) in enumerate(proof.pc_proof)]
        self.labels = [lab for lab, _n, _x in pts]
        self.names = [n for _l, n, _x in pts]
        self.images = [_outside_image(x, n) for _l, n, x in pts]
        self.proof = proof
        # degree bounds of the bounded commitments (third and fourth round polynomial info): g_1, every g_M
        C = _largest(d.variable_domain for d in self.domains)
        self.bounds = {"g_1": C.size - 2}
        for i, d in enumerate(self.domains):
            for m, K in zip("abc", d.non_zero_domains):
                self.bounds[self.label(i, f"g_{m}", 0)] = K.size - 2

    def transcript(self) -> TranscriptOps:
        """the verifier's sponge (varuna.rs:136-153, 770-860; verifier.rs; sonic_pc/mod.rs:405, 602), every squeeze queued: the
        same operations prove_batch runs"""
        p, c = self.proof, self.proof.commitments
        t = TranscriptOps()
        _init_sponge(t, p.batch_sizes, self.inputs, [vk.circuit_commitments for vk in self.vks])
        t.absorb_commitments(np.stack(list(c.witness_commitments) + ([c.mask_poly] if c.mask_poly is not None else [])))
        t.queue_squeeze([b - 1 + (1 if i else 0) for i, b in enumerate(p.batch_sizes)])
        t.absorb_commitments(np.stack([c.h_0]))
        t.queue_squeeze([3])
        t.absorb_commitments(np.stack([c.g_1, c.h_1]))
        for sums in p.third_sums:
            for s in sums:
                t.absorb_nonnative(s)
        t.queue_squeeze([1])
        t.absorb_commitments(np.stack([g for i in range(len(self.vks)) for g in (c.g_a_commitments[i], c.g_b_commitments[i],
                                                                                 c.g_c_commitments[i])]))
        for s in p.fourth_sums:
            t.absorb_nonnative(s)
        t.queue_squeeze([2] + [3] * (len(self.vks) - 1))
        t.absorb_commitments(np.stack([c.h_2]))
        t.queue_squeeze([1])
        t.absorb_nonnative(p.evaluations.to_field_elements())
        t.queue_squeeze([1] * (3 * len(self.vks) + 7), short=True)       # per point one per lc (1, 2, 3K + 1), then the randomizer
        return t

    def challenges(self, vals: list) -> dict:
        """the transcript's squeezes (canonical, in order) → the challenges, as _prove_batch names them"""
        it = iter(vals)
        take = lambda n: [next(it) for _ in range(n)]                     # noqa: E731
        combs = []
        for i, b in enumerate(self.proof.batch_sizes):
            e = take(b - 1 + (1 if i else 0))
            combs.append((e[b - 1] if i else 1, [1] + e[: b - 1]))
        alpha, eta_b, eta_c = take(3)
        beta = take(1)[0]
        d = [take(2)] + [take(3) for _ in self.vks[1:]]
        deltas = [[1] + d[0]] + d[1:]
        gamma = take(1)[0]
        return {"batch_combiners": combs, "alpha": alpha, "eta_b": eta_b, "eta_c": eta_c, "beta": beta, "deltas": deltas,
                "gamma": gamma, "opening": list(it)}

    def check_scalars(self, ch: dict, x_at_beta: list, zk: bool) -> dict:
        """construct_linear_combinations on the verifier's side (a_poly / b_poly expanded into the index commitments, ahp.rs:408-445),
        then check_combinations → batch_check → accumulate_elems folded into scalars: {degree bound or None: {label: scalar}}, with
        the None group minus the adjusted witness (g, each w, γ·G), and {"witness": {label: scalar}}, −Σ r_q·w_q"""
        p, ev = self.proof, self.proof.evaluations
        alpha, beta, gamma = ch["alpha"], ch["beta"], ch["gamma"]
        lcs, query_set = linear_combinations(
            self.domains, ch["batch_combiners"], p.third_sums, p.fourth_sums, (alpha, ch["eta_b"], ch["eta_c"], beta, ch["deltas"], gamma),
            ev.g_1_eval, [list(g) for g in zip(ev.g_a_evals, ev.g_b_evals, ev.g_c_evals)], x_at_beta, self.label, zk)
        expand = {}
        for i, d in enumerate(self.domains):
            v_rc = _vanish(d.constraint_domain, alpha) * _vanish(d.variable_domain, beta) % R_MOD
            rc = d.constraint_domain.size * d.variable_domain.size % R_MOD
            for j, m in enumerate("abc"):
                idx = f"circuit_{self.ids[i].hex()}_{{}}_{m}".format
                expand[self.label(i, "a_poly", j)] = [(v_rc, idx("row_col_val"))]
                expand[self.label(i, "b_poly", j)] = [(rc * alpha % R_MOD * beta % R_MOD, None), ((-rc * alpha) % R_MOD, idx("col")),
                                                      ((-rc * beta) % R_MOD, idx("row")), (rc, idx("row_col"))]
        evals = {"g_1": ev.g_1_eval}
        for i in range(len(self.vks)):
            for m, vals in zip("abc", (ev.g_a_evals, ev.g_b_evals, ev.g_c_evals)):
                evals[self.label(i, f"g_{m}", 0)] = vals[i]
        lcs = [(lc_label, [(k * k2 % R_MOD, lab2) for k, lab in lc for k2, lab2 in (expand[lab] if lab in expand else [(1, lab)])])
               for lc_label, lc in lcs]
        return check_combinations_scalars(lcs, query_set, {lab: evals.get(lab, 0) for lab, _lc in lcs}, self.bounds, self.random_v,
                                          iter(ch["opening"]))


def _label_fn(ids: list):
    """label(i, name, j) of circuit i's polynomial: the reference's witness_label names (ahp.rs:46-50; a_poly / b_poly as
    construct_matrix_linear_combinations names them, ahp.rs:408-409)"""
    def label(i, name, j=0):
        if name in ("a_poly", "b_poly"):
            return f"circuit_{ids[i].hex()}_{name}_{'abc'[j]}"
        return witness_label(ids[i], name, j)
    return label


def _init_sponge(t: TranscriptOps, batch_sizes: list, public_inputs: list, vk_commitments: list) -> None:
    """init_sponge (varuna.rs:136-153): the protocol name; per circuit (id order) its batch size (u64 LE) and each instance's padded
    public input (nonnative); every circuit's twelve vk commitments"""
    t.absorb_bytes(PROTOCOL_NAME)
    for b, inputs in zip(batch_sizes, public_inputs):
        t.absorb_bytes(struct.pack("<Q", b))
        for x in inputs:
            t.absorb_nonnative(x)
    for comms in vk_commitments:
        t.absorb_commitments(comms)


_G1_STATUS = {device.G1_NOT_CANONICAL: "a coordinate is not below q", device.G1_NOT_ON_CURVE: "not on the curve",
              device.G1_NOT_IN_SUBGROUP: "not in the prime-order subgroup"}


def verify_batch_many(verifier: UniversalVerifier, batch: list, zk: bool = False, stats: dict | None = None) -> list:
    """VarunaSNARK::verify_batch (varuna.rs:625-933) for many proofs in one call: `batch` is [(keys_to_inputs, proof)], keys_to_inputs
    [(CircuitVerifyingKey, [public input, …])] with each public input a list of canonical Fr integers, formatted (first element one)
    → one verdict per proof, in input order.  The circuits of a proof are taken in id order, so the order of keys_to_inputs changes
    nothing.  The work of all proofs shares each device call:
        validation    every vk commitment, proof commitment and opening w as Affine::check (device.g1_validate), one launch
        transcript    each proof's whole PoseidonSponge<Fq, 2, 1> operation list, built on the host because the verifier knows every
                      absorbed element up front; all proofs as transcripts of one device.poseidon_transcripts call
        x(β)          every instance's Σ x_i·L_i(β) over its input domain, one device.matrix_evals_at_points pass
        scalars       on the host: the verifier's linear combinations, and check_combinations / batch_check folded into one scalar per
                      base point for each degree-bound group (None, |C_max| − 2, every |K_M| − 2), the None group minus the adjusted
                      witness
        MSM           every group of every proof and each proof's −Σ r_q·w_q as jobs of one device.sonic_commit_batch pass
        pairing       each proof one check of one device.pairing_products call: the None group with H, each bounded group with its
                      negative power of β·H, −Σ r_q·w_q with β·H
    ValueError, naming the lowest proof at fault and the field, for what the reference returns as an error: an empty batch, the proof's
    lists not matching its batch sizes, a count of public inputs other than the batch size, an input longer than its input domain or
    not starting with one, a pc_proof without exactly one (w, random_v) per query point, a G1 point failing validation, the largest
    domains' vanishing polynomial zero at α, β or γ, a degree bound the verifier holds no negative power for, a hiding proof and a
    verifier without γ·G.  False when the proof's hiding mode is not `zk` (varuna.rs:716-727) or the pairing check fails.  `stats`,
    when given, receives the seconds of each stage and the transcripts' permutation counts."""
    import time
    clock = time.perf_counter
    t0 = clock()
    if not batch:
        raise ValueError("no proofs to verify")
    n = len(batch)
    errors, verdict, views = {}, [None] * n, [None] * n
    for k, (keys_to_inputs, proof) in enumerate(batch):
        try:
            views[k] = _ProofView(list(keys_to_inputs), proof)
        except ValueError as e:
            errors[k] = str(e)

    def live():
        return [k for k in range(n) if k not in errors and verdict[k] is None]
    dev = verifier.device
    # validation: every outside point of every proof in one launch
    todo = live()
    pts = np.stack([img for k in todo for img in views[k].images] + [verifier.g] + ([verifier.gamma_g] if verifier.gamma_g is not None else []))
    pts_dev = torch.from_numpy(pts).to(dev)
    t1 = clock()
    nout = sum(len(views[k].images) for k in todo)
    status = device.g1_validate(pts_dev[:nout]).cpu().numpy() if nout else np.zeros(0, dtype=np.int32)
    t2 = clock()
    base, row = {}, 0
    for k in todo:
        v = views[k]
        base[k] = row
        bad = np.nonzero(status[row: row + len(v.images)])[0]
        if bad.size:
            errors[k] = f"{v.names[bad[0]]}: {_G1_STATUS[int(status[row + bad[0]])]}"
        row += len(v.images)
    for k in live():
        c = views[k].proof
        hiding, mask = any(v is not None for _w, v in c.pc_proof), c.commitments.mask_poly is not None
        if not ((hiding and mask) if zk else (not hiding and not mask)):
            verdict[k] = False
    # transcripts: one thread per proof
    todo = live()
    ops_all, starts, inputs, nin, nfr, transcripts = [], [0], [], 0, 0, {}
    for k in todo:
        t = views[k].transcript()
        transcripts[k] = (t, nfr)
        ops = np.array(t._ops, dtype=np.int64).reshape(-1, 3)
        ops[:, 2] += np.where(ops[:, 0] == poseidon.OP_ABSORB, nin, nfr)
        ops_all.append(ops)
        starts.append(starts[-1] + ops.shape[0])
        inputs.append(t.inputs())
        nin += t._nin
        nfr += t._nout
    t3 = clock()
    vals = []
    if todo:
        _out, fr = device.poseidon_transcripts(
            poseidon.FIELD_FQ, torch.from_numpy(np.concatenate(ops_all).astype(np.int32)).to(dev),
            torch.tensor(starts, dtype=torch.int32, device=dev), torch.from_numpy(np.concatenate(inputs).view(np.int64)).to(dev), 0, nfr)
        vals = [_fr_mont_to_int(r) for r in fr.cpu().numpy().view(np.uint64)]
    t4 = clock()
    chs = {}
    for k in todo:
        t, off = transcripts[k]
        v = views[k]
        ch = chs[k] = v.challenges(vals[off: off + t._nout])
        for name, x, doms in (("α", ch["alpha"], [d.constraint_domain for d in v.domains]),
                              ("β", ch["beta"], [d.variable_domain for d in v.domains]),
                              ("γ", ch["gamma"], [d for dd in v.domains for d in dd.non_zero_domains])):
            if _vanish(_largest(doms), x) == 0:
                errors[k] = f"the vanishing polynomial of the largest domain is zero at {name}"
                break
    # x(β): every instance of every proof in one pass
    todo = live()
    xs = [(k, i, x) for k in todo for i, ins in enumerate(views[k].inputs) for x in ins]
    t5 = clock()
    x_at = {}
    if xs:
        flat = torch.from_numpy(np.stack([_mont(v) for _k, _i, x in xs for v in x]).view(np.int64)).to(dev)
        jobs, off = [], 0
        for k, _i, x in xs:
            sl = flat[off: off + len(x)]
            jobs.append((sl, sl, sl, _mont(chs[k]["beta"])))
            off += len(x)
        dots = device.matrix_evals_at_points(jobs)
        for (k, i, _x), d in zip(xs, dots):
            x_at.setdefault(k, [[] for _ in views[k].inputs])[i].append(_fr_mont_to_int(d[0]))
    t6 = clock()
    # scalars, then every MSM job of every proof in one pass
    jobs, pairs = [], []
    g_row, gamma_row = nout, nout + 1
    for k in todo:
        v = views[k]
        groups = v.check_scalars(chs[k], x_at[k], zk)
        for d in groups:
            if d not in (None, "witness") and d not in verifier.neg_index:
                errors[k] = f"UnsupportedDegreeBound({d}): the verifier holds no negative power of β·H for it"
        if "gamma_g" in groups[None] and verifier.gamma_g is None:
            errors[k] = "the proof is hiding and the verifier holds no γ·G"
        if k in errors:
            continue
        local = {lab: base[k] + j for j, lab in enumerate(v.labels)}
        local.update({"g": g_row, "gamma_g": gamma_row})
        for d in [None] + sorted(d for d in groups if d not in (None, "witness")) + ["witness"]:
            items = sorted(groups[d].items())
            jobs.append(([local[lab] for lab, _s in items], [s for _l, s in items]))
            pairs.append((k, 0 if d is None else 1 if d == "witness" else verifier.neg_index[d]))
    if errors:
        k = min(errors)
        raise ValueError(f"proof {k}: {errors[k]}")
    t7 = clock()
    todo = live()
    if jobs:
        idx = torch.tensor([i for rows, _s in jobs for i in rows], dtype=torch.int64, device=dev)
        bases = pts_dev[idx]
        scal = torch.from_numpy(np.stack([_mont(s) for _r, ss in jobs for s in ss]).view(np.int64)).to(dev)
        offs = np.concatenate([[0], np.cumsum([len(r) for r, _s in jobs])]).tolist()
        sums = device.sonic_commit_batch([bases[a: b] for a, b in zip(offs, offs[1:])], [scal[a: b] for a, b in zip(offs, offs[1:])])
        t8 = clock()
        g1 = torch.from_numpy(np.stack([_affine(s) for s in sums])).to(dev)
        g2_index = torch.tensor([q for _k, q in pairs], dtype=torch.int32, device=dev)
        per_proof = [sum(1 for o, _q in pairs if o == k) for k in todo]
        check_start = torch.tensor(np.concatenate([[0], np.cumsum(per_proof)]), dtype=torch.int32, device=dev)
        _gt, is_one = device.pairing_products(g1, g2_index, verifier.prepared, check_start)
        for k, one in zip(todo, is_one.cpu().tolist()):
            verdict[k] = bool(one)
    else:
        t8 = t7
    t9 = clock()
    if stats is not None:
        stats.update({"validation": t2 - t1, "transcript": t4 - t3, "x_at_beta": t6 - t5, "msm": t8 - t7, "pairing": t9 - t8,
                      "host": (t1 - t0) + (t3 - t2) + (t5 - t4) + (t7 - t6),
                      "permutations": [transcripts[k][0].permutations for k in transcripts]})
    return verdict


def verify_batch(verifier: UniversalVerifier, keys_to_inputs: list, proof: Proof, zk: bool = False) -> bool:
    """VarunaSNARK::verify_batch (varuna.rs:625-933) of one proof: verify_batch_many with one entry"""
    return verify_batch_many(verifier, [(keys_to_inputs, proof)], zk)[0]


# ---- byte forms: CanonicalSerialize / CanonicalDeserialize of Proof (data_structures/proof.rs:305-368), CircuitVerifyingKey
# (circuit_verifying_key.rs, derived) and Certificate (certificate.rs, derived), in the compressed (ToBytes) or uncompressed mode ----

_G1_BYTES_STATUS = {**_G1_STATUS, device.G1_BAD_FLAGS: "malformed flag bits"}


def _g1_size(compress: bool) -> int:
    return device.G1_COMPRESSED_BYTES if compress else device.G1_UNCOMPRESSED_BYTES


class _Walk:
    """one blob's host walk from `offset`: bounds-checked reads in the reference's field order; every G1 point's bytes are appended
    to the shared `points` list ((bytes, field)) and stand for their index there until the one device call decodes them all"""

    def __init__(self, blob, offset: int, compress: bool, points: list):
        self.b, self.o, self.psize, self.points = bytes(blob), int(offset), _g1_size(compress), points
        if not 0 <= self.o <= len(self.b):
            raise ValueError(f"offset {offset} is outside the blob")

    def need(self, n: int, field: str) -> None:
        if n > len(self.b) - self.o:
            raise ValueError(f"{field}: {len(self.b) - self.o} bytes left, at least {n} needed")

    def take(self, n: int, field: str) -> bytes:
        self.need(n, field)
        self.o += n
        return self.b[self.o - n: self.o]

    def u64(self, field: str) -> int:
        return struct.unpack("<Q", self.take(8, field))[0]

    def tag(self, field: str) -> bool:
        """an Option's tag (bool::read_le): 0 or 1"""
        t = self.take(1, field)[0]
        if t > 1:
            raise ValueError(f"{field}: option tag {t} is neither 0 nor 1")
        return t == 1

    def fr(self, field: str) -> int:
        v = int.from_bytes(self.take(32, field), "little")
        if v >= R_MOD:
            raise ValueError(f"{field}: not below r")
        return v

    def point(self, field: str) -> int:
        self.points.append((self.take(self.psize, field), field))
        return len(self.points) - 1

    def batch_lc_proof(self, field: str) -> list:
        """BatchLCProof: a u64 count of KZGProof (w, Option<Fr> random_v) → [(point index, Montgomery random_v or None)]"""
        n = self.u64(f"{field} length")
        self.need(n * (self.psize + 1), f"{field} of {n} proofs")
        out = []
        for p in range(n):
            w = self.point(f"{field}[{p}].w")
            v = self.fr(f"{field}[{p}].random_v") if self.tag(f"{field}[{p}].random_v tag") else None
            out.append((w, None if v is None else _fr_int_to_mont(v)))
        return out


def _walk_proof(w: _Walk):
    """proof.rs:344-368 → a function of the decoded points that builds the Proof.  Every count is checked against the bytes left
    before anything of its size is read, so a blob claiming 2^40 instances costs nothing."""
    P = w.psize
    K = w.u64("batch_sizes length")
    w.need(8 * K, f"batch_sizes of {K} circuits")
    sizes = [w.u64(f"batch_sizes[{i}]") for i in range(K)]
    total = sum(sizes)
    # at least: every commitment without the mask, the mask tag, every Fr, the pc_proof length
    w.need(P * (total + 4 + 3 * K) + 1 + 32 * (1 + 6 * K + 3 * total) + 8, f"the body of batch sizes {sizes}")
    wit = [w.point(f"witness_commitments[{j}]") for j in range(total)]
    mask = w.point("mask_poly") if w.tag("mask_poly tag") else None
    h_0, g_1, h_1 = (w.point(n) for n in ("h_0", "g_1", "h_1"))
    g_abc = [[w.point(f"g_{m}_commitments[{i}]") for i in range(K)] for m in "abc"]
    h_2 = w.point("h_2")
    g_1_eval = w.fr("evaluations.g_1_eval")
    evals = [[w.fr(f"evaluations.g_{m}_evals[{i}]") for i in range(K)] for m in "abc"]
    third = [[[w.fr(f"third_sums[{i}][{j}]") for _ in range(3)] for j in range(b)] for i, b in enumerate(sizes)]
    fourth = [[w.fr(f"fourth_sums[{i}]") for _ in range(3)] for i in range(K)]
    pc = w.batch_lc_proof("pc_proof")

    def build(pts):
        comms = Commitments([pts[j] for j in wit], None if mask is None else pts[mask], pts[h_0], pts[g_1], pts[h_1],
                            *[[pts[j] for j in g] for g in g_abc], pts[h_2])
        return Proof(sizes, comms, Evaluations(g_1_eval, *evals), third, fourth, [(pts[j], v) for j, v in pc])
    return build


def _walk_verifying_key(w: _Walk):
    """CircuitInfo (six u64), the commitments as a Vec (u64 length, which must be 12), the 32-byte circuit id"""
    info = CircuitInfo(*[w.u64(f"circuit_info.{f}") for f in CircuitInfo.__dataclass_fields__])
    n = w.u64("circuit_commitments length")
    if n != len(INDEX_POLYNOMIAL_NAMES):
        raise ValueError(f"circuit_commitments: {n} commitments, not {len(INDEX_POLYNOMIAL_NAMES)}")
    comms = [w.point(f"circuit_commitments[{name}]") for name in INDEX_POLYNOMIAL_NAMES]
    cid = w.take(32, "id")
    return lambda pts: CircuitVerifyingKey(info, np.stack([pts[j] for j in comms]), cid)


def _walk_certificate(w: _Walk):
    """the BatchLCProof of prove_vk: exactly one non-hiding KZG proof"""
    pc = w.batch_lc_proof("pc_proof")
    if len(pc) != 1 or pc[0][1] is not None:
        raise ValueError("pc_proof: a certificate holds exactly one non-hiding proof")
    return lambda pts: Certificate(pts[pc[0][0]])


def _from_bytes_many(walk, blobs, offsets, compress: bool, validate: bool, device_):
    """walk every blob on the host, then decode every point of every blob in one device call → (objects, end offsets).
    ValueError names the lowest blob at fault and its field.  A blob that fails the walk is reported before any device call,
    unless a blob below it holds points, which are then decoded to find whether one of them fails first."""
    points, builds, ends, starts, fail = [], [], [], [], None
    for k, blob in enumerate(blobs):
        starts.append(len(points))
        try:
            w = _Walk(blob, offsets[k], compress, points)
            builds.append(walk(w))
            ends.append(w.o)
        except ValueError as e:
            fail = (k, str(e))
            del points[starts[-1]:]
            break
    pts = []
    if points:
        raw = torch.from_numpy(np.frombuffer(b"".join(b for b, _f in points), dtype=np.uint8).copy()).to(torch.device(device_))
        images, status = device.g1_deserialize(raw, compress, validate)
        images, status = images.cpu().numpy(), status.cpu().numpy()
        bad = np.nonzero(status)[0]
        if bad.size:
            i = int(bad[0])
            k = int(np.searchsorted(starts, i, side="right")) - 1
            raise ValueError(f"blob {k}: {points[i][1]}: {_G1_BYTES_STATUS[int(status[i])]}")
        pts = list(_projective_limbs(images))
    if fail is not None:
        raise ValueError(f"blob {fail[0]}: {fail[1]}")
    return [b(pts) for b in builds], ends


def _normalised(comm, what: str) -> np.ndarray:
    """a normalised projective image (X, Y, one) or (·, ·, zero) from the caller → its uint64[18] limbs; ValueError if not"""
    limbs = np.ascontiguousarray(comm, dtype=np.uint64).reshape(-1)
    if limbs.size != 18 or not (not limbs[12:].any() or (limbs[12:] == _FQ_ONE).all()):
        raise ValueError(f"{what} is not a normalised projective image")
    return limbs


def _fr_bytes(v, what: str) -> bytes:
    return _fr_value(v, what).to_bytes(32, "little")


def _proof_parts(p: Proof) -> list:
    """proof.rs:305-317: bytes and (point, field) pairs in write order"""
    p.check_batch_sizes()
    c, e = p.commitments, p.evaluations
    parts = [struct.pack(f"<{1 + len(p.batch_sizes)}Q", len(p.batch_sizes), *p.batch_sizes)]
    parts += [(x, f"witness_commitments[{j}]") for j, x in enumerate(c.witness_commitments)]
    parts += [b"\x00"] if c.mask_poly is None else [b"\x01", (c.mask_poly, "mask_poly")]
    parts += [(c.h_0, "h_0"), (c.g_1, "g_1"), (c.h_1, "h_1")]
    for m in "abc":
        parts += [(x, f"g_{m}_commitments[{i}]") for i, x in enumerate(getattr(c, f"g_{m}_commitments"))]
    parts.append((c.h_2, "h_2"))
    parts.append(_fr_bytes(e.g_1_eval, "evaluations.g_1_eval"))
    parts += [_fr_bytes(v, "evaluations") for v in list(e.g_a_evals) + list(e.g_b_evals) + list(e.g_c_evals)]
    parts += [_fr_bytes(v, "third_sums") for sums in p.third_sums for t in sums for v in t]
    parts += [_fr_bytes(v, "fourth_sums") for t in p.fourth_sums for v in t]
    return parts + _batch_lc_parts(p.pc_proof)


def _batch_lc_parts(pc: list) -> list:
    parts = [struct.pack("<Q", len(pc))]
    for q, (w, v) in enumerate(pc):
        parts.append((w, f"pc_proof[{q}].w"))
        parts += [b"\x00"] if v is None else [b"\x01", _fr_bytes(_fr_mont_to_int(v), f"pc_proof[{q}].random_v")]
    return parts


def _verifying_key_parts(vk: CircuitVerifyingKey) -> list:
    comms = np.ascontiguousarray(vk.circuit_commitments, dtype=np.uint64).reshape(-1, 18)
    if comms.shape[0] != len(INDEX_POLYNOMIAL_NAMES) or vk.id is None or len(vk.id) != 32:
        raise ValueError("a verifying key's bytes need its twelve commitments and its 32-byte circuit id")
    return ([vk.circuit_info.to_bytes_le(), struct.pack("<Q", len(comms))]
            + [(x, f"circuit_commitments[{n}]") for n, x in zip(INDEX_POLYNOMIAL_NAMES, comms)] + [bytes(vk.id)])


def _certificate_parts(cert: Certificate) -> list:
    return _batch_lc_parts([(cert.w, None)])


def _to_bytes_many(parts_fn, objs, compress: bool, device_) -> list:
    """every object's layout on the host, every point of every object through one device.g1_serialize call → bytes per object"""
    layouts = [parts_fn(o) for o in objs]
    pts = [_normalised(x, f"object {k}: {what}") for k, parts in enumerate(layouts) for x, what in
           (q for q in parts if not isinstance(q, bytes))]
    enc = []
    if pts:
        enc = device.g1_serialize(torch.from_numpy(np.stack(pts).view(np.int64)).to(torch.device(device_)), compress).cpu().numpy()
    it = iter(enc)
    return [b"".join(q if isinstance(q, bytes) else next(it).tobytes() for q in parts) for parts in layouts]


def proofs_to_bytes(proofs: list, compress: bool = True, device_="cuda") -> list:
    """Proof::serialize_with_mode of every proof (compressed: ToBytes), all points in one device call → [bytes]"""
    return _to_bytes_many(_proof_parts, proofs, compress, device_)


def proofs_from_bytes(blobs: list, compress: bool = True, validate: bool = True, device_="cuda") -> list:
    """Proof::deserialize_with_mode of every blob (compressed: FromBytes; trailing bytes are ignored): one host walk gathers every
    G1 point, one device call decodes them (device.g1_deserialize; with `validate` each also passes Affine::check) → [Proof].
    ValueError names the lowest blob at fault and the field: bytes missing, an Option tag other than 0 or 1, an Fr not below r, a
    count the bytes left cannot hold, or a point that does not decode (or, with `validate`, fails the check)."""
    return _from_bytes_many(_walk_proof, blobs, [0] * len(blobs), compress, validate, device_)[0]


def verifying_keys_from_bytes(blobs: list, compress: bool = True, validate: bool = True, device_="cuda") -> list:
    """CircuitVerifyingKey::deserialize_with_mode of every blob, as proofs_from_bytes → [CircuitVerifyingKey]"""
    return _from_bytes_many(_walk_verifying_key, blobs, [0] * len(blobs), compress, validate, device_)[0]


def certificates_from_bytes(blobs: list, compress: bool = True, validate: bool = True, device_="cuda") -> list:
    """Certificate::deserialize_with_mode of every blob, as proofs_from_bytes → [Certificate]"""
    return _from_bytes_many(_walk_certificate, blobs, [0] * len(blobs), compress, validate, device_)[0]


# ---- byte form of CircuitProvingKey: ToBytes / FromBytes (circuit_proving_key.rs:42-57) = the verifying key (CanonicalSerialize,
# compressed), the Circuit (CanonicalSerialize, compressed: ahp/indexer/circuit.rs:158-237) and the CommitterKey (ToBytes,
# sonic_pc/data_structures.rs:65-265) ----

_FR_TWO_ADIC_ROOT = 8065159656716812877374967518403273466521432693661810619979959746626482506078   # fr.rs:110: FrParameters
_FR_GENERATOR = 22                                                                                   # fr.rs:126: GENERATOR
_DOMAIN_FIELDS = (("size", 0, 8), ("log_size_of_group", 8, 4), ("size_as_field_element", 12, 32), ("size_inv", 44, 32),
                  ("group_gen", 76, 32), ("group_gen_inv", 108, 32), ("generator_inv", 140, 32))
_DOMAIN_BYTES = 172
_VK_BYTES = 48 + 8 + 12 * device.G1_COMPRESSED_BYTES + 32


def _domain_bytes(size: int) -> bytes:
    """CanonicalSerialize of EvaluationDomain::new(size) for a power of two (fft/domain.rs:82-147): u64 size, u32 log size, then
    size, 1/size, the subgroup's generator ω (TWO_ADIC_ROOT_OF_UNITY squared down to order `size`), 1/ω and 1/GENERATOR as Fr"""
    cached = _DOMAIN_CACHE.get(size)
    if cached is None:
        lg = size.bit_length() - 1
        w = pow(_FR_TWO_ADIC_ROOT, 1 << (47 - lg), R_MOD)
        vals = (size % R_MOD, pow(size, -1, R_MOD), w, pow(w, -1, R_MOD), pow(_FR_GENERATOR, -1, R_MOD))
        cached = _DOMAIN_CACHE[size] = struct.pack("<QI", size, lg) + b"".join(v.to_bytes(32, "little") for v in vals)
    return cached


_DOMAIN_CACHE: dict = {}


@dataclass
class _KeyLayout:
    """where one proving key's sections sit in its blob (byte offsets), from the host walk"""
    info: CircuitInfo
    vk_points: int                 # the twelve compressed commitments
    vk_id: bytes
    id_span: tuple                 # (start, end): CircuitInfo and the three matrices, the bytes of the circuit id
    matrices: list                 # per matrix (offset of its u64 row count, host row_ptr int32)
    evals: list                    # per matrix {"row", "col", "row_col_val": offset of the first value}
    domains: list                  # per matrix K
    ck: object                     # sonic_pc.CommitterKeyLayout


def _walk_proving_key(r) -> _KeyLayout:
    """the headers of one proving key from r's offset, checking each count against the bytes left before anything of its size
    exists; the bulk sections are only located (a matrix's rows by the library's row walk)"""
    from .sonic_pc import walk_committer_key
    fields = CircuitInfo.__dataclass_fields__
    info = CircuitInfo(*[r.u64(f"circuit_verifying_key.circuit_info.{f}") for f in fields])
    n = r.u64("circuit_verifying_key.circuit_commitments length")
    if n != len(INDEX_POLYNOMIAL_NAMES):
        raise r.fail("circuit_verifying_key.circuit_commitments", f"{n} commitments, not {len(INDEX_POLYNOMIAL_NAMES)}")
    vk_points = r.o
    r.take(len(INDEX_POLYNOMIAL_NAMES) * device.G1_COMPRESSED_BYTES, "circuit_verifying_key.circuit_commitments")
    vk_id = bytes(r.take(32, "circuit_verifying_key.id"))
    start = r.o
    cinfo = CircuitInfo(*[r.u64(f"circuit.index_info.{f}") for f in fields])
    if cinfo != info:
        raise r.fail("circuit_verifying_key.circuit_info", "differs from the circuit's index_info")
    # the domains Circuit's read builds (circuit.rs:196-214) and those Circuit._shape needs
    counts = (info.num_constraints, info.num_public_and_private_variables, info.num_public_inputs, info.num_non_zero_a,
              info.num_non_zero_b, info.num_non_zero_c)
    doms = [EvaluationDomain.new(c) for c in counts]
    for f, d in zip(("num_constraints", "num_public_and_private_variables", "num_public_inputs", "num_non_zero_a",
                     "num_non_zero_b", "num_non_zero_c"), doms):
        if d is None:
            raise r.fail(f"circuit.index_info.{f}", "no evaluation domain holds this many elements")
    if info.num_public_inputs & (info.num_public_inputs - 1) or doms[1].size <= doms[2].size:
        raise r.fail("circuit.index_info", "public inputs not padded to a power of two below the variable domain")
    matrices = []
    for m, nnz in zip("abc", counts[3:]):
        at = r.o
        nrows = r.u64(f"circuit.{m} length")
        if nrows != info.num_constraints:
            raise r.fail(f"circuit.{m}", f"{nrows} rows, not num_constraints = {info.num_constraints}")
        r.need(8 * nrows + 40 * nnz, f"circuit.{m} of {nrows} rows and {nnz} entries")
        row_ptr, bad = device.matrix_row_walk(r.mv, r.o, nrows, nnz)
        if row_ptr is None:
            what = f"circuit.{m}[{bad}]" if 0 <= bad < nrows else f"circuit.{m}"
            raise r.fail(what, f"the row lengths overrun the matrix or disagree with num_non_zero_{m} = {nnz}")
        r.o += 8 * nrows + 40 * nnz
        matrices.append((at, row_ptr))
    id_span = (start, r.o)
    evals, ks = [], [d.size for d in doms[3:]]
    for m, K in zip("abc", ks):
        e = {}
        for name in ("row", "col", "row_col", "row_col_val"):
            fld = f"circuit.{m}_arith.{name}"
            if name == "row_col":
                if r.tag(f"{fld} tag"):
                    raise r.fail(fld, "present; a proving key holds it pruned (prune_row_col_evals)")
                continue
            n = r.u64(f"{fld} length")
            if n != K:
                raise r.fail(fld, f"{n} evaluations, not |K| = {K}")
            r.need(32 * K + _DOMAIN_BYTES, f"{fld} of {K} evaluations and its domain")
            e[name] = r.o
            r.o += 32 * K
            got, want = r.take(_DOMAIN_BYTES, f"{fld}.domain"), _domain_bytes(K)
            if got != want:
                f, _o, _n = next(x for x in _DOMAIN_FIELDS if got[x[1]: x[1] + x[2]] != want[x[1]: x[1] + x[2]])
                raise r.fail(f"{fld}.domain.{f}", f"differs from EvaluationDomain::new({K})")
        evals.append(e)
    return _KeyLayout(info, vk_points, vk_id, id_span, matrices, evals, ks, walk_committer_key(r))


def _blake2s(mv: memoryview, span: tuple) -> bytes:
    return hashlib.blake2s(mv[span[0]: span[1]], digest_size=32).digest()


def _proving_keys_from_bytes(blobs: list, offsets: list, validate: bool, device_):
    """proving_keys_from_bytes at per-blob offsets → (keys, end offsets)"""
    from .sonic_pc import POINT_BYTES, ByteReader, first_bad_point, gather_records, upload
    if not blobs:
        return [], []
    mvs = [memoryview(b).cast("B") for b in blobs]
    layouts, ends = [], []
    for k, (mv, off) in enumerate(zip(mvs, offsets)):
        r = ByteReader(mv, off, f"blob {k}")
        layouts.append(_walk_proving_key(r))
        ends.append(r.o)
    dev = torch.device(device_)
    pool = ThreadPoolExecutor(min(ID_HASH_THREADS, 2 * len(blobs)))
    try:
        # host: SHA-256 and Blake2s of the bytes as read, while the device decodes
        shas = [pool.submit(L.ck.sha256, mv) for L, mv in zip(layouts, mvs)]
        ids = [pool.submit(_blake2s, mv, L.id_span) for L, mv in zip(layouts, mvs)]
        # device: each blob's key once into one buffer; every row_ptr in one upload
        base = np.cumsum([0] + [e - o for o, e in zip(offsets, ends)]).tolist()
        d_blob = torch.empty(base[-1], dtype=torch.uint8, device=dev)
        for k, (mv, off) in enumerate(zip(mvs, offsets)):
            upload(mv[off: ends[k]], d_blob[base[k]: base[k + 1]])
        row_ptrs = torch.from_numpy(np.concatenate([rp for L in layouts for _o, rp in L.matrices])).to(dev)
        nnzs = [n for L in layouts for n in (L.info.num_non_zero_a, L.info.num_non_zero_b, L.info.num_non_zero_c)]
        vals = torch.empty((sum(nnzs), 4), dtype=torch.int64, device=dev)
        cols = torch.empty(sum(nnzs), dtype=torch.int32, device=dev)
        evals = torch.empty((3 * sum(sum(L.domains) for L in layouts), 4), dtype=torch.int64, device=dev)
        # every point of the call: the verifying keys' compressed commitments, then the committer keys' ToBytes points
        shift = [b - o for b, o in zip(base, offsets)]
        vk_raw = gather_records(d_blob, [(L.vk_points + shift[k], 12) for k, L in enumerate(layouts)], device.G1_COMPRESSED_BYTES)
        vk_images, vk_status = device.g1_deserialize(vk_raw, device.G1_COMPRESSED, validate)
        ck_runs, ck_first = [], []
        for k, L in enumerate(layouts):
            ck_first.append(sum(n for _o, n in ck_runs))
            ck_runs += [(o + shift[k], n) for o, n in L.ck.runs()]
        ck_images, ck_status = device.g1_deserialize(gather_records(d_blob, ck_runs, POINT_BYTES), device.G1_TO_BYTES, validate)
        # every Fr record of the call in one launch; its synchronisation also ends the point decodes
        segments, owners, mats, arith = [], [], [], []
        at_rp = at_nnz = at_ev = 0
        for k, L in enumerate(layouts):
            for j, (m, (o, rp)) in enumerate(zip("abc", L.matrices)):
                nnz = nnzs[3 * k + j]
                views = (row_ptrs[at_rp: at_rp + rp.size], cols[at_nnz: at_nnz + nnz], vals[at_nnz: at_nnz + nnz])
                segments.append((o + shift[k], nnz, 40, views[2], views[1], L.info.num_public_and_private_variables, views[0]))
                owners.append((k, o, f"circuit.{m}", rp))
                mats.append(views)
                at_rp += rp.size
                at_nnz += nnz
            for m, e, K in zip("abc", L.evals, L.domains):
                trio = []
                for name in ("row", "col", "row_col_val"):
                    out = evals[at_ev: at_ev + K]
                    at_ev += K
                    segments.append((e[name] + shift[k], K, 32, out, None, 0, None))
                    owners.append((k, e[name], f"circuit.{m}_arith.{name}", None))
                    trio.append(out)
                arith.append(trio)
        bad = device.fr_records_decode(d_blob, segments)
        # the first fault of the lowest blob at fault, in byte order; a hash is checked after every element
        faults = []
        for (k, o, fld, rp), b in zip(owners, bad):
            if b is not None:
                e, why = b
                if rp is not None:                                     # a matrix entry: name its row
                    row = int(np.searchsorted(rp, e, side="right")) - 1
                    fld, at = f"{fld}[{row}][{e - rp[row]}]", o + 16 + 8 * row + 40 * e
                else:
                    fld, at = f"{fld}[{e}]", o + 32 * e
                what = "not below r" if why == device.FR_RECORD_NOT_CANONICAL else \
                    "column not below num_public_and_private_variables"
                faults.append((k, 0, at, f"{fld}: {what}"))
        bad_vk = first_bad_point(vk_status, [(12 * k, 12, "circuit_verifying_key.circuit_commitments", L.vk_points)
                                             for k, L in enumerate(layouts)], device.G1_COMPRESSED_BYTES)
        if bad_vk is not None:
            faults.append((bad_vk[0] // 12, 0, bad_vk[2], bad_vk[1]))
        bad_ck = first_bad_point(ck_status, [(f, n, f"committer_key.{fld}", o) for k, L in enumerate(layouts)
                                             for f, n, fld, o in L.ck.fields(ck_first[k])], POINT_BYTES)
        if bad_ck is not None:
            faults.append((int(np.searchsorted(ck_first, bad_ck[0], side="right")) - 1, 0, bad_ck[2], bad_ck[1]))
        for k, L in enumerate(layouts):
            if shas[k].result() != bytes(mvs[k][L.ck.hash_offset: L.ck.hash_offset + 32]):
                faults.append((k, 1, L.ck.hash_offset, "committer_key.hash: the SHA-256 of the points differs"))
            if ids[k].result() != L.vk_id:
                faults.append((k, 1, L.vk_points, "circuit_verifying_key.id: differs from the circuit's id"))
        if faults:
            k, _rank, _at, what = min(faults)
            raise ValueError(f"blob {k}: {what}")
    finally:
        pool.shutdown(wait=True)
    vk_limbs = _projective_limbs(vk_images.cpu().numpy())
    out = []
    for k, L in enumerate(layouts):
        c = Circuit.__new__(Circuit)
        c._shape(*[Matrix.from_device(*mats[3 * k + j]) for j in range(3)], L.info.num_public_inputs,
                 L.info.num_public_and_private_variables)
        c.ariths = [MatrixEvals(*arith[3 * k + j], K) for j, K in enumerate(c.non_zero_domains)]
        c._id = L.vk_id
        vk = CircuitVerifyingKey(L.info, vk_limbs[12 * k: 12 * k + 12].copy(), L.vk_id)
        out.append(CircuitProvingKey(vk, c, L.ck.build(ck_images, ck_first[k])))
    return out, ends


def proving_keys_from_bytes(blobs: list, validate: bool = True, device_="cuda") -> list:
    """CircuitProvingKey::read_le (circuit_proving_key.rs:51-57) of every blob (trailing bytes are ignored) → [CircuitProvingKey].

    The host walks the headers only — counts, tags, CircuitInfo, domains, the matrices' row lengths (a bounds-checked walk in the
    library) — and checks every count against the bytes left before anything of that size exists; a header fault of any blob is
    reported before any device call.  Each key's bytes then go to the device once, and a fixed number of launches decodes every
    key of the call: one for the Fr records (matrix values and columns, evaluations), one per point form (the verifying keys'
    compressed commitments, the committer keys' 97-byte points; with `validate` each point also passes Affine::check).  One
    synchronisation precedes the reports.  The SHA-256 of each committer key's points and the Blake2s circuit id are computed from
    the bytes as read, on host threads, while the device decodes.  The loaded Circuit holds the decoded CSR arrays and
    evaluations; its id is the one computed here, and no matrix_evals pass runs.  Its committer key's max_degree is None.

    ValueError names the blob, the field and the element: everything the reference refuses (bytes missing, a tag or bool other
    than 0 or 1, an Fr not below r, a coordinate not below q, an infinity byte the reference refuses, a SHA-256 mismatch), and,
    stricter than the reference, because this prover would otherwise diverge from it silently:
      a column not below num_public_and_private_variables (an out-of-range read in the prover's mat-vecs and transposes);
      a matrix whose row count or entry count differs from CircuitInfo;
      an evaluation vector whose length is not |K|, or whose EvaluationDomain differs from EvaluationDomain::new(|K|);
      a row_col evaluation vector present (setup always prunes it);
      a CircuitInfo without the domains the prover needs (public inputs padded to a power of two below the variable domain);
      a verifying key whose circuit_info or id differs from the circuit's;
      committer-key map keys not strictly increasing;
      with `validate`, a point off the curve or outside the subgroup.
    Body faults name the lowest blob at fault and its first fault in byte order, hashes after elements."""
    return _proving_keys_from_bytes(blobs, [0] * len(blobs), validate, device_)[0]


def _projective_limbs(images: np.ndarray) -> np.ndarray:
    """Affine<G1> images [n, 104] → normalised projective limbs uint64[n, 18]"""
    limbs = np.zeros((images.shape[0], 18), dtype=np.uint64)
    limbs[:, :12] = images[:, :96].copy().view(np.uint64)
    inf = images[:, 96] != 0
    limbs[~inf, 12:] = _FQ_ONE
    limbs[inf, :12] = 0
    limbs[inf, 6:12] = _FQ_ONE                                        # (0, one, 0)
    return limbs


def proving_keys_to_bytes(pks: list) -> list:
    """CircuitProvingKey::write_le (circuit_proving_key.rs:42-49) of every key → [bytes]: the verifying key compressed (its id
    the circuit's), the circuit (CircuitInfo; A, B, C through csr_serialize; per matrix row, col, row_col = None and row_col_val
    through fr_from_mont, each with its domain), the committer key's ToBytes.  Every matrix of the call shares one launch, the
    evaluations one, and the points of each form one."""
    from .sonic_pc import committer_keys_to_bytes
    if not pks:
        return []
    circuits = [pk.circuit for pk in pks]
    buf, offs = device.csr_serialize_batch([(m.row_ptr, m.cols, m.vals) for c in circuits for m in (c.a, c.b, c.c)])
    mats = buf.cpu().numpy()
    for k, c in enumerate(circuits):
        if c._id is None:
            c._id = hashlib.blake2s(c.info.to_bytes_le() + mats[offs[3 * k]: offs[3 * k + 3]].tobytes(), digest_size=32).digest()
    ev = device.fr_from_mont(torch.cat([t for c in circuits for a in c.ariths for t in (a.row, a.col, a.row_col_val)]))
    ev = ev.cpu().numpy().view(np.uint8).reshape(-1)
    vks = [CircuitVerifyingKey(pk.circuit_verifying_key.circuit_info, pk.circuit_verifying_key.circuit_commitments, pk.circuit.id())
           for pk in pks]
    vk_bytes = _to_bytes_many(_verifying_key_parts, vks, True, circuits[0].a.row_ptr.device)
    ck_bytes = committer_keys_to_bytes([pk.committer_key for pk in pks])
    out, at = [], 0
    for k, c in enumerate(circuits):
        parts = [vk_bytes[k], c.info.to_bytes_le(), mats[offs[3 * k]: offs[3 * k + 3]].tobytes()]
        for a in c.ariths:
            K = a.domain.size
            head = struct.pack("<Q", K)
            for j in range(3):
                if j == 2:
                    parts.append(b"\x00")                                     # row_col: pruned
                parts += [head, ev[at: at + 32 * K].tobytes(), _domain_bytes(K)]
                at += 32 * K
        out.append(b"".join(parts) + ck_bytes[k])
    return out
