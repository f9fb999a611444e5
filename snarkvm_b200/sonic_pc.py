"""SonicKZG10 — the polynomial commitment layer the Varuna prover calls (SURVEY §8 f1) — on device-resident operands.

Mirror of /root/reference/algorithms/src/polycommit/sonic_pc:
    mod.rs:62-175     trim                  CommitterKey.trim
    mod.rs:177-257    commit                SonicKZG10.commit          (ONE msm_core pass for the whole round)
    mod.rs:259-284    combine_for_open      SonicKZG10.combine_for_open
    mod.rs:286-342    batch_open            SonicKZG10.batch_open
    mod.rs:413-475    open_combinations     SonicKZG10.open_combinations
    mod.rs:344-411, 477-544, 582-677   check_combinations → batch_check → accumulate_elems → check_elems' inputs as scalars
                                       check_combinations_scalars
    data_structures.rs:310-341   shifted_powers_of_beta_g / lagrange_basis
and of kzg10/mod.rs:98-156 (commit), :220-277 (open) through algorithms.KZG10.

Polynomials are CUDA tensors [m, 4] int64 of Montgomery Fr coefficients (low degree first; trailing zeros allowed); bases are CUDA
uint8 tensors [n, 104] in the reference's Affine layout; commitments and proofs come back as the normalised projective image
(uint64[18]) like every MSM of this package.  Two things the Rust code draws from generators are ARGUMENTS here, because neither
generator can be reproduced outside Rust: the blinding polynomials (`KZGRandomness::rand`, kzg10/data_structures.rs) and the
Fiat-Shamir challenges (`fs_rng.squeeze_short_nonnative_field_element`, a Poseidon sponge on the host) — the latter as an iterator
consumed in the reference's squeeze order.
"""
from __future__ import annotations

import hashlib
import struct
import warnings
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass, field

import numpy as np
import torch

from . import device
from .algorithms import KZG10, EvaluationDomain, _fr_int_to_mont, _R_MOD

STRIDE = device.AFFINE_STRIDE


# ---- small polynomial helpers on Montgomery coefficient tensors ----
def _zeros(n: int, dev) -> torch.Tensor:
    return torch.zeros((n, 4), dtype=torch.int64, device=dev)


def poly_axpy(acc: torch.Tensor | None, coeff: int, p: torch.Tensor) -> torch.Tensor:
    """acc + coeff·p (DensePolynomial `+= (coeff, &poly)`, fft/polynomial/dense.rs), acc = None is the zero polynomial"""
    coeff %= _R_MOD
    if p.shape[0] == 0 or coeff == 0:
        return acc if acc is not None else _zeros(0, p.device)
    term = p if coeff == 1 else device.fr_vec_op(p, _fr_int_to_mont(coeff), device.FR_MUL)
    if acc is None or acc.shape[0] == 0:
        return term.clone() if term is p else term
    if acc.shape[0] < term.shape[0]:
        out = term.clone() if term is p else term
        device.fr_vec_op(out[: acc.shape[0]], acc, device.FR_ADD, out=out[: acc.shape[0]])
        return out
    out = acc.clone()
    device.fr_vec_op(out[: term.shape[0]], term, device.FR_ADD, out=out[: term.shape[0]])
    return out


@dataclass
class LabeledPolynomial:
    """polycommit/data_structures.rs LabeledPolynomial / LabeledPolynomialWithBasis: `polynomial` holds monomial coefficients, or
    — with `lagrange=True` — evaluations over the domain of their count (committed against the Lagrange basis of that size)."""
    label: str
    polynomial: torch.Tensor
    degree_bound: int | None = None
    hiding_bound: int | None = None
    lagrange: bool = False


@dataclass
class Randomness:
    """KZGRandomness: the blinding polynomial of a hiding commitment (hiding_bound + 2 coefficients), None = Randomness::empty()"""
    blinding_polynomial: torch.Tensor | None = None

    def is_hiding(self) -> bool:
        return self.blinding_polynomial is not None and self.blinding_polynomial.shape[0] > 0

    def axpy(self, coeff: int, other: "Randomness") -> "Randomness":
        if not other.is_hiding():
            return self
        return Randomness(poly_axpy(self.blinding_polynomial, coeff, other.blinding_polynomial))


@dataclass
class CommitterKey:
    """sonic_pc/data_structures.rs CommitterKey / CommitterUnionKey over an SRS resident in HBM"""
    powers_of_beta_g: torch.Tensor                                   # [supported_degree + 1, 104]
    powers_of_beta_times_gamma_g: torch.Tensor                       # [supported_hiding_bound + 2, 104]
    lagrange_bases_at_beta_g: dict = field(default_factory=dict)     # size → [size, 104]
    shifted_powers_of_beta_g: torch.Tensor | None = None             # pp.powers[max_degree − highest bound …]
    shifted_powers_of_beta_times_gamma_g: dict | None = None         # bound → gamma powers of that shift
    enforced_degree_bounds: list | None = None
    max_degree: int | None = 0        # the SRS's degree; None for a key read from bytes, whose byte form does not carry it

    @classmethod
    def trim(cls, pp_powers_of_beta_g: torch.Tensor, pp_powers_of_beta_times_gamma_g: torch.Tensor, supported_degree: int,
             supported_lagrange_sizes=(), supported_hiding_bound: int = 1, enforced_degree_bounds=None) -> "CommitterKey":
        """mod.rs:62-175.  `pp_powers_of_beta_times_gamma_g` is dense here (γβ^i·G for every i the reference keeps sparsely)."""
        max_degree = pp_powers_of_beta_g.shape[0] - 1
        bounds = None
        shifted = shifted_gamma = None
        if enforced_degree_bounds is not None:
            bounds = sorted(set(int(b) for b in enforced_degree_bounds))
            if bounds:
                highest = bounds[-1]
                if highest > supported_degree:
                    raise ValueError(f"The highest enforced degree bound {highest} is larger than the supported degree {supported_degree}")
                shifted = pp_powers_of_beta_g[max_degree - highest:]
                shifted_gamma = {}
                for b in bounds:
                    shift = max_degree - b
                    shifted_gamma[b] = pp_powers_of_beta_times_gamma_g[shift: min(max_degree, shift + supported_hiding_bound) + 2]
        gamma = pp_powers_of_beta_times_gamma_g[: supported_hiding_bound + 2]
        if gamma.shape[0] != supported_hiding_bound + 2:
            raise ValueError("HidingBoundToolarge")
        bases = {}
        for size in supported_lagrange_sizes:
            if size & (size - 1):
                raise ValueError(f"The Lagrange basis size ({size}) is not a power of two")
            if size > max_degree + 1:
                raise ValueError(f"The Lagrange basis size ({size}) is larger than the supported degree ({max_degree + 1})")
            bases[size] = device.lagrange_basis(pp_powers_of_beta_g[:size].contiguous())
        return cls(pp_powers_of_beta_g[: supported_degree + 1], gamma, bases, shifted, shifted_gamma, bounds, max_degree)

    def powers(self):
        return self.powers_of_beta_g, self.powers_of_beta_times_gamma_g

    def shifted_powers(self, degree_bound: int):
        """data_structures.rs:310-331 → (powers, gamma powers) of the shift that enforces `degree_bound`"""
        if self.shifted_powers_of_beta_g is None or degree_bound not in (self.enforced_degree_bounds or []):
            raise ValueError(f"degree bound {degree_bound} is not enforced by this committer key")
        return self.shifted_powers_of_beta_g[self.enforced_degree_bounds[-1] - degree_bound:], self.shifted_powers_of_beta_times_gamma_g[degree_bound]

    def lagrange_basis(self, size: int):
        if size not in self.lagrange_bases_at_beta_g:
            raise ValueError(f"UnsupportedLagrangeBasisSize({size})")
        return self.lagrange_bases_at_beta_g[size], self.powers_of_beta_times_gamma_g

    def to_bytes(self) -> bytes:
        """ToBytes (data_structures.rs:186-265): every point in its 97-byte form through one device.g1_serialize call, then the
        SHA-256 of the point sections"""
        return committer_keys_to_bytes([self])[0]

    @staticmethod
    def read(blob, offset: int = 0, validate: bool = True, device_="cuda"):
        """FromBytes (data_structures.rs:65-184) of the key whose bytes start at `offset` of `blob` → (CommitterKey, the offset after
        it).  The host walks the headers only (no copy of `blob`); the key's bytes go to the device once and every point is decoded
        there by one device.g1_deserialize call (with `validate`, each also passes Affine::check).  ValueError names the field and
        the element: bytes missing, a bool other than 0 or 1, a coordinate not below q, an infinity byte the reference refuses, a
        SHA-256 that differs from the points', and — stricter than the reference — the keys of the Lagrange bases or of the shifted
        γ powers not strictly increasing (ToBytes writes a BTreeMap in order) and, with `validate`, a point off the curve or outside
        the subgroup.  max_degree is None: the byte form does not carry the SRS's degree."""
        mv = memoryview(blob).cast("B")
        r = ByteReader(mv, offset, "committer key")
        layout = walk_committer_key(r)
        with ThreadPoolExecutor(1) as pool:
            digest = pool.submit(layout.sha256, mv)
            d_blob = upload(mv[offset: r.o], torch.empty(r.o - offset, dtype=torch.uint8, device=torch.device(device_)))
            runs = [(o - offset, n) for o, n in layout.runs()]
            images, status = device.g1_deserialize(gather_records(d_blob, runs, POINT_BYTES), device.G1_TO_BYTES, validate)
            bad = first_bad_point(status, layout.fields(), POINT_BYTES)
            if bad is not None:
                raise ValueError(f"committer key: {bad[1]}")
            if digest.result() != bytes(mv[layout.hash_offset: layout.hash_offset + 32]):
                raise ValueError("committer key: hash: the SHA-256 of the points differs")
        return layout.build(images), r.o


def _check_degrees_and_bounds(ck: CommitterKey, p: LabeledPolynomial) -> None:
    """kzg10/mod.rs check_degrees_and_bounds: a bounded polynomial needs degree ≤ bound ≤ max_degree and an enforced bound"""
    _check_bound(ck, p.label, p.polynomial.shape[0], p.degree_bound)


def _check_bound(ck: CommitterKey, label: str, length: int, degree_bound: int | None) -> None:
    """_check_degrees_and_bounds of a polynomial of `length` coefficients"""
    if degree_bound is not None:
        if ck.enforced_degree_bounds is None or degree_bound not in ck.enforced_degree_bounds:
            raise ValueError(f"UnsupportedDegreeBound({degree_bound})")
        # a key read from bytes has no max_degree: its enforced bounds, all within its SRS, stand for it
        if length - 1 > degree_bound or (ck.max_degree is not None and degree_bound > ck.max_degree):
            raise ValueError(f"IncorrectDegreeBound for {label}")


class SonicKZG10:
    @staticmethod
    def commit(ck: CommitterKey, polynomials: list, blindings: list | None = None):
        """mod.rs:177-257 → (commitments uint64[count, 18], [Randomness]).  All MSMs of the round — plain powers, shifted powers,
        Lagrange bases, blinding terms — go through ONE device pass (device.sonic_commit_batch).  `blindings[i]`: the blinding
        polynomial of polynomial i (hiding_bound + 2 Montgomery coefficients) when it is hiding, else None."""
        return SonicKZG10.commit_many([(ck, polynomials, blindings)])[0]

    @staticmethod
    def commit_many(items: list) -> list:
        """commit of every (committer key, polynomials, blindings or None) in `items`, all of them in ONE device.sonic_commit_batch
        pass → [(commitments uint64[count, 18], [Randomness])], entry k equal to commit(*items[k])"""
        bases, gammas, polys, rands, counts = [], [], [], [], []
        for ck, polynomials, blindings in items:
            blindings = list(blindings) if blindings is not None else [None] * len(polynomials)
            for p, b in zip(polynomials, blindings):
                _check_degrees_and_bounds(ck, p)
                if p.lagrange:
                    n = p.polynomial.shape[0]
                    size = 1 << max(n - 1, 0).bit_length()
                    basis, gamma = ck.lagrange_basis(size)
                    if n == 0 or size != basis.shape[0]:
                        raise ValueError("evaluations do not match the Lagrange basis size")
                elif p.degree_bound is not None:
                    basis, gamma = ck.shifted_powers(p.degree_bound)
                else:
                    basis, gamma = ck.powers()
                if p.hiding_bound is not None:
                    if b is None or b.shape[0] != p.hiding_bound + 2:
                        raise ValueError(f"{p.label}: a hiding commitment needs a blinding polynomial of hiding_bound + 2 coefficients")
                    rands.append(Randomness(b))
                else:
                    rands.append(Randomness())
                bases.append(basis); gammas.append(gamma); polys.append(p.polynomial)
            counts.append(len(polynomials))
        any_hiding = any(r.is_hiding() for r in rands)
        out = device.sonic_commit_batch(bases, polys, gammas if any_hiding else None,
                                        [r.blinding_polynomial for r in rands] if any_hiding else None)
        offs = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64).tolist()
        return [(out[a: b], rands[a: b]) for a, b in zip(offs, offs[1:])]

    @staticmethod
    def combine_for_open(ck: CommitterKey, labeled_polynomials: list, rands: list, challenges):
        """mod.rs:259-284 + combine_polynomials :548-565: Σ challenge_i·p_i with one squeezed challenge per polynomial"""
        poly, rand = None, Randomness()
        for p, r in zip(labeled_polynomials, rands):
            _check_degrees_and_bounds(ck, p)
            ch = int(next(challenges)) % _R_MOD
            poly = poly_axpy(poly, ch, p.polynomial)
            rand = rand.axpy(ch, r)
        return (poly if poly is not None else _zeros(0, ck.powers_of_beta_g.device)), rand

    @staticmethod
    def batch_open(ck: CommitterKey, labeled_polynomials: list, query_set: list, rands: list, challenges):
        """mod.rs:286-342 → [(w uint64[18], random_v uint64[4] or None)] in the order of the point names (a BTreeMap in the reference).
        query_set: iterable of (label, (point_name, point as int)).  `challenges` yields, per point, one value per polynomial opened
        there (labels in sorted order) and then the discarded `_randomizer`, exactly the reference's squeeze sequence."""
        poly_rand = {p.label: (p, r) for p, r in zip(labeled_polynomials, rands)}
        by_point: dict = {}
        for label, (point_name, point) in query_set:
            entry = by_point.setdefault(point_name, (point, set()))
            entry[1].add(label)
        powers, gamma = ck.powers()
        witnesses, hiding_witnesses, random_vs = [], [], []
        for point_name in sorted(by_point):
            point, labels = by_point[point_name]
            qp, qr = [], []
            for label in sorted(labels):
                if label not in poly_rand:
                    raise KeyError(f"MissingPolynomial {{ label: {label} }}")
                qp.append(poly_rand[label][0]); qr.append(poly_rand[label][1])
            polynomial, rand = SonicKZG10.combine_for_open(ck, qp, qr, challenges)
            next(challenges)                                                   # `_randomizer`
            z = _fr_int_to_mont(int(point) % _R_MOD)
            if polynomial.shape[0] > powers.shape[0]:
                raise ValueError("check_degree_is_too_large")
            # kzg10::open (mod.rs:303-321): the witness polynomials now, their commitments below — all points in ONE device pass
            w, rw = KZG10.compute_witness_polynomial(polynomial, z, rand.blinding_polynomial if rand.is_hiding() else None)
            witnesses.append(w); hiding_witnesses.append(rw)
            random_vs.append(device.poly_evaluate(rand.blinding_polynomial, z) if rand.is_hiding() else None)
        k = len(witnesses)
        any_hiding = any(h is not None for h in hiding_witnesses)
        ws = device.sonic_commit_batch([powers] * k, witnesses, [gamma] * k if any_hiding else None, hiding_witnesses if any_hiding else None)
        return [(ws[i], random_vs[i]) for i in range(k)]

    @staticmethod
    def open_combinations(ck: CommitterKey, linear_combinations: list, polynomials: list, rands: list, query_set: list, challenges):
        """mod.rs:413-475.  linear_combinations: [(lc_label, [(coeff as int, polynomial label or None for the constant term)])];
        the query set names LC labels.  Returns the BatchLCProof's list of (w, random_v)."""
        return SonicKZG10.open_combinations_many([(ck, linear_combinations, polynomials, rands, query_set, challenges)])[0]

    @staticmethod
    def open_combinations_many(items: list) -> list:
        """open_combinations of every (ck, linear_combinations, polynomials, rands, query_set, challenges) in `items` in one pass →
        one BatchLCProof list of (w, random_v) per item, equal to open_combinations of that item.  Each query point's opening
        challenges are folded into its linear combinations' coefficients on the host, so every (item, point) combined polynomial, and
        its blinding polynomial, is one output of one device.fr_lincomb_terms launch; the witnesses of all of them are one
        device.poly_divide_by_linear_batch, the random_v one device.poly_evaluate_batch and the witness commitments, hiding parts
        included, one device.sonic_commit_batch pass.  The field is exact, so the reassociation gives the same bytes."""
        opened = []                                  # per (item, point): (item, z, combined polynomial job, blinding job or None)
        for k, (ck, linear_combinations, polynomials, rands, query_set, challenges) in enumerate(items):
            label_map = {p.label: (p, r) for p, r in zip(polynomials, rands)}
            lcs = {}                                 # lc label → (degree bound, [(coefficient, LabeledPolynomial, Randomness)])
            for lc_label, terms in linear_combinations:
                degree_bound, used = None, []
                for coeff, label in terms:
                    if label is None:                                          # LCTerm::One: not committed, used by the verifier directly
                        continue
                    if label not in label_map:
                        raise KeyError(f"MissingPolynomial {{ label: {label} }}")
                    cur, cur_rand = label_map[label]
                    if cur.degree_bound is not None:
                        if len(terms) != 1:
                            raise ValueError(f"EquationHasDegreeBounds({lc_label})")
                        assert int(coeff) % _R_MOD == 1, "Coefficient must be one for degree-bounded equations"
                        degree_bound = cur.degree_bound
                    used.append((int(coeff) % _R_MOD, cur, cur_rand))
                lcs[lc_label] = (degree_bound, used)
            by_point: dict = {}
            for label, (point_name, point) in query_set:
                by_point.setdefault(point_name, (point, set()))[1].add(label)
            powers = ck.powers_of_beta_g
            for point_name in sorted(by_point):
                point, labels = by_point[point_name]
                poly_terms, blind_terms = [], []
                for label in sorted(labels):
                    if label not in lcs:
                        raise KeyError(f"MissingPolynomial {{ label: {label} }}")
                    degree_bound, used = lcs[label]
                    _check_bound(ck, label, max([p.polynomial.shape[0] for c, p, _r in used if c], default=0), degree_bound)
                    ch = int(next(challenges)) % _R_MOD
                    for c, p, r in used:
                        c = c * ch % _R_MOD
                        if c == 0:
                            continue
                        if p.polynomial.shape[0]:
                            poly_terms.append((p.polynomial, _fr_int_to_mont(c)))
                        if r.is_hiding():
                            blind_terms.append((r.blinding_polynomial, _fr_int_to_mont(c)))
                next(challenges)                                                   # `_randomizer`
                n = max([t[0].shape[0] for t in poly_terms], default=0)
                if n > powers.shape[0]:
                    raise ValueError("check_degree_is_too_large")
                blind = (max(t[0].shape[0] for t in blind_terms), blind_terms) if blind_terms else None
                opened.append((k, _fr_int_to_mont(int(point) % _R_MOD), (n, poly_terms), blind))
        if not opened:
            return [[] for _ in items]
        # kzg10::open (mod.rs:303-321) of every (item, point): combined polynomials, witnesses, random_v, then ONE commitment pass
        hiding = [i for i, o in enumerate(opened) if o[3] is not None]
        combined = device.fr_lincomb_terms([o[2] for o in opened] + [opened[i][3] for i in hiding])
        witnesses = device.poly_divide_by_linear_batch([(p, o[1]) for p, o in zip(combined, opened)] +
                                                       [(b, opened[i][1]) for b, i in zip(combined[len(opened):], hiding)])
        random_vs = device.poly_evaluate_batch([(b, opened[i][1]) for b, i in zip(combined[len(opened):], hiding)])
        hiding_witnesses = [None] * len(opened)
        for j, i in enumerate(hiding):
            hiding_witnesses[i] = witnesses[len(opened) + j]
        powers = [items[o[0]][0].powers() for o in opened]
        ws = device.sonic_commit_batch([p for p, _g in powers], witnesses[: len(opened)], [g for _p, g in powers] if hiding else None,
                                       hiding_witnesses if hiding else None)
        out = [[] for _ in items]
        rv = dict(zip(hiding, random_vs))
        for i, o in enumerate(opened):
            out[o[0]].append((ws[i], rv[i].copy() if i in rv else None))
        return out


def check_combinations_scalars(linear_combinations: list, query_set: list, evaluations: dict, degree_bounds: dict, random_vs: list,
                               challenges) -> dict:
    """check_combinations (mod.rs:477-544) → batch_check (:344-411) → accumulate_elems (:582-635), with every G1 sum kept as one scalar
    per base point, so that a caller runs check_elems' MSMs (:637-677) as one pass.  linear_combinations: [(lc label, [(coefficient,
    base label or None for LCTerm::One)])]; query_set: [(lc label, (point name, point))]; evaluations: {lc label: value at its point};
    degree_bounds: {base label: bound} of the bounded commitments; random_vs: per point name in sorted order, the opening's random_v
    (canonical) or None; `challenges` yields the sponge's short squeezes in order.  The opening witness of the q-th point is the base
    "w_{q}", G is "g" and γ·G "gamma_g".  → {degree bound or None: {base label: scalar}, "witness": {base label: scalar}}: the
    None group already minus the combined adjusted witness (both pair with H), "witness" the negated combined witness (it pairs
    with β·H), each bounded group pairing with its negative power of β·H."""
    terms, values = {}, {}
    for lc_label, lc in linear_combinations:
        bounded = [lab for _k, lab in lc if lab in degree_bounds]
        if bounded and (len(lc) != 1 or lc[0][0] % _R_MOD != 1):
            raise ValueError(f"EquationHasDegreeBounds({lc_label})")
        terms[lc_label] = [(k, lab) for k, lab in lc if lab is not None]
        # LCTerm::One moves into the evaluation (mod.rs:504-510)
        values[lc_label] = (evaluations[lc_label] - sum(k for k, lab in lc if lab is None)) % _R_MOD
    by_point = {}
    for lc_label, (name, z) in query_set:
        by_point.setdefault(name, (z, []))[1].append(lc_label)
    if len(by_point) != len(random_vs):
        raise ValueError(f"{len(random_vs)} openings for {len(by_point)} query points")
    groups, witness, r = {None: {}}, {}, 1

    def add(group, label, v):
        group[label] = (group.get(label, 0) + v) % _R_MOD
    for q, name in enumerate(sorted(by_point)):
        z, labels = by_point[name]
        combined = 0
        for lc_label in sorted(labels):
            challenge = int(next(challenges))
            combined += challenge * values[lc_label]
            for k, lab in terms[lc_label]:
                add(groups.setdefault(degree_bounds.get(lab), {}), lab, r * challenge % _R_MOD * k)
        none = groups[None]
        add(none, "g", -r * combined)
        add(none, f"w_{q}", r * z)
        if random_vs[q] is not None:
            add(none, "gamma_g", -r * random_vs[q])
        witness[f"w_{q}"] = (-r) % _R_MOD
        r = int(next(challenges))
    return {**groups, "witness": witness}


def synthetic_srs(max_degree: int, beta: int, gamma: int, dev="cuda"):
    """(powers_of_beta_g, powers_of_beta_times_gamma_g) = (β^i·G, γβ^i·G) for i ≤ max_degree (+1 for the gamma powers, which the
    reference keeps one degree further, mod.rs:104-105) — a universal setup with KNOWN trapdoor for tests and benches, where every
    commitment can be checked in the scalar field: commit(p, r) = (p(β) + γ·r(β))·G.  Built on the device from the generator by
    one fixed-base pass (device.generate_powers)."""
    return device.generate_powers(max_degree + 1, beta, 1, dev), device.generate_powers(max_degree + 2, beta, gamma, dev)


# ---- byte form: ToBytes / FromBytes of CommitterKey (data_structures.rs:65-265) ----
POINT_BYTES = device.G1_TO_BYTES_BYTES
_G1_STATUS = {device.G1_NOT_CANONICAL: "a coordinate not below q", device.G1_NOT_ON_CURVE: "not on the curve",
              device.G1_NOT_IN_SUBGROUP: "not in the prime-order subgroup", device.G1_BAD_FLAGS: "an infinity byte the reference refuses"}


class ByteReader:
    """bounds-checked little-endian header reads from `offset` of a memoryview; every failure is a ValueError naming `name` and
    the field"""

    def __init__(self, mv: memoryview, offset: int, name: str):
        self.mv, self.o, self.name = mv, int(offset), name
        if not 0 <= self.o <= len(mv):
            raise ValueError(f"{name}: offset {offset} is outside the blob")

    def fail(self, field: str, what: str) -> ValueError:
        return ValueError(f"{self.name}: {field}: {what}")

    def need(self, n: int, field: str) -> None:
        if n > len(self.mv) - self.o:
            raise self.fail(field, f"{len(self.mv) - self.o} bytes left, at least {n} needed")

    def take(self, n: int, field: str) -> memoryview:
        self.need(n, field)
        self.o += n
        return self.mv[self.o - n: self.o]

    def u32(self, field: str) -> int:
        return struct.unpack("<I", self.take(4, field))[0]

    def u64(self, field: str) -> int:
        return struct.unpack("<Q", self.take(8, field))[0]

    def tag(self, field: str) -> bool:
        """bool::read_le, also an Option's tag: 0 or 1"""
        t = self.take(1, field)[0]
        if t > 1:
            raise self.fail(field, f"{t} is neither 0 nor 1")
        return t == 1


def upload(mv: memoryview, out: torch.Tensor) -> torch.Tensor:
    """one copy of host bytes into the uint8 device tensor `out` of their length, without a host copy first → out"""
    if len(mv):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")                  # a read-only buffer is only read here
            out.copy_(torch.from_numpy(np.frombuffer(mv, dtype=np.uint8)))
    return out


def gather_records(d_blob: torch.Tensor, runs: list, size: int) -> torch.Tensor:
    """the `size`-byte records of every run (byte offset in d_blob, count), concatenated in run order by one gather → uint8
    [records · size] on d_blob's device"""
    counts = np.array([n for _o, n in runs], dtype=np.int64)
    total = int(counts.sum()) if runs else 0
    if total == 0:
        return torch.empty(0, dtype=torch.uint8, device=d_blob.device)
    starts = np.array([o for o, _n in runs], dtype=np.int64)
    first = np.cumsum(counts) - counts
    offsets = np.repeat(starts - size * first, counts) + size * np.arange(total, dtype=np.int64)
    windows = d_blob.as_strided((d_blob.numel() - size + 1, size), (1, 1))     # row j: the `size` bytes from j
    return windows.index_select(0, torch.from_numpy(offsets).to(d_blob.device)).reshape(-1)


def first_bad_point(status: torch.Tensor, runs: list, size: int):
    """the first point whose status is not G1_VALID → (its index, "field[element]: reason", its byte offset), or None; `runs`
    places the points: [(first index, count, field, byte offset of the run)], `size` bytes per point"""
    bad = torch.nonzero(status).flatten()[:1].cpu().tolist()
    if not bad:
        return None
    i = bad[0]
    for first, n, fld, at in runs:
        if first <= i < first + n:
            return i, f"{fld}[{i - first}]: {_G1_STATUS[int(status[i])]}", at + size * (i - first)
    raise AssertionError("a point outside every run")


@dataclass
class CommitterKeyLayout:
    """where one committer key's sections sit in its blob: point runs as (byte offset, count), the bound keys and the hash"""
    powers: tuple
    lagrange: list                 # [(size, offset)]
    gamma: tuple
    shifted: tuple | None
    shifted_gamma: list | None     # [(bound, offset, count)]
    bounds: list | None
    hash_offset: int

    def runs(self) -> list:
        """every point run in blob order"""
        out = [self.powers] + [(o, n) for n, o in self.lagrange] + [self.gamma]
        out += [self.shifted] if self.shifted is not None else []
        return out + [(o, n) for _b, o, n in self.shifted_gamma or []]

    def fields(self, first: int = 0) -> list:
        """[(first point index, count, field, byte offset)] of the runs, points numbered from `first`"""
        names = (["powers_of_beta_g"] + [f"lagrange_bases_at_beta_g[{n}]" for n, _o in self.lagrange] + ["powers_of_beta_times_gamma_g"]
                 + (["shifted_powers_of_beta_g"] if self.shifted is not None else [])
                 + [f"shifted_powers_of_beta_times_gamma_g[{b}]" for b, _o, _n in self.shifted_gamma or []])
        out = []
        for name, (o, n) in zip(names, self.runs()):
            out.append((first, n, name, o))
            first += n
        return out

    def sha256(self, mv: memoryview) -> bytes:
        """the hash FromBytes recomputes (data_structures.rs:152-177): the bytes of every point section but the Lagrange bases, as
        read (every accepted encoding writes back to itself)"""
        h = hashlib.sha256()
        for o, n in [self.powers, self.gamma] + ([self.shifted] if self.shifted is not None else []) + \
                [(o, n) for _b, o, n in self.shifted_gamma or []]:
            h.update(mv[o: o + POINT_BYTES * n])
        return h.digest()

    def build(self, images: torch.Tensor, first: int = 0) -> CommitterKey:
        """the CommitterKey whose points are images[first:], decoded in runs() order (views, no copy)"""
        views = []
        for _o, n in self.runs():
            views.append(images[first: first + n])
            first += n
        it = iter(views)
        powers = next(it)
        lagrange = {size: next(it) for size, _o in self.lagrange}
        gamma = next(it)
        shifted = next(it) if self.shifted is not None else None
        shifted_gamma = None if self.shifted_gamma is None else {b: next(it) for b, _o, _n in self.shifted_gamma}
        return CommitterKey(powers, gamma, lagrange, shifted, shifted_gamma, None if self.bounds is None else list(self.bounds), None)


def walk_committer_key(r: ByteReader) -> CommitterKeyLayout:
    """the headers of ToBytes for CommitterKey from r's offset: u32 counts, bool tags, u32 keys and bounds; every count is checked
    against the bytes left before anything of its size exists, and the points are only located"""
    def run(field: str) -> tuple:
        n = r.u32(f"{field} length")
        r.need(POINT_BYTES * n, f"{field} of {n} points")
        r.o += POINT_BYTES * n
        return r.o - POINT_BYTES * n, n

    def increasing(keys: list, field: str) -> None:
        for i in range(1, len(keys)):
            if keys[i] <= keys[i - 1]:
                raise r.fail(f"{field}[{i}]", f"key {keys[i]} does not follow {keys[i - 1]}")

    powers = run("powers_of_beta_g")
    nl = r.u32("lagrange_bases_at_beta_g length")
    r.need(4 * nl, f"lagrange_bases_at_beta_g of {nl} bases")
    lagrange = []
    for i in range(nl):
        size = r.u32(f"lagrange_bases_at_beta_g[{i}] size")
        r.need(POINT_BYTES * size, f"lagrange_bases_at_beta_g[{i}] of {size} points")
        lagrange.append((size, r.o))
        r.o += POINT_BYTES * size
    increasing([n for n, _o in lagrange], "lagrange_bases_at_beta_g")
    gamma = run("powers_of_beta_times_gamma_g")
    shifted = run("shifted_powers_of_beta_g") if r.tag("shifted_powers_of_beta_g tag") else None
    shifted_gamma = None
    if r.tag("shifted_powers_of_beta_times_gamma_g tag"):
        nb = r.u32("shifted_powers_of_beta_times_gamma_g length")
        r.need(8 * nb, f"shifted_powers_of_beta_times_gamma_g of {nb} entries")
        shifted_gamma = []
        for i in range(nb):
            b = r.u32(f"shifted_powers_of_beta_times_gamma_g[{i}] key")
            o, n = run(f"shifted_powers_of_beta_times_gamma_g[{i}]")
            shifted_gamma.append((b, o, n))
        increasing([b for b, _o, _n in shifted_gamma], "shifted_powers_of_beta_times_gamma_g")
    bounds = None
    if r.tag("enforced_degree_bounds tag"):
        nb = r.u32("enforced_degree_bounds length")
        r.need(4 * nb, f"enforced_degree_bounds of {nb} bounds")
        bounds = list(struct.unpack(f"<{nb}I", r.take(4 * nb, "enforced_degree_bounds")))
    hash_offset = r.o
    r.take(32, "hash")
    return CommitterKeyLayout(powers, lagrange, gamma, shifted, shifted_gamma, bounds, hash_offset)


def _committer_key_parts(ck: CommitterKey) -> list:
    """ToBytes of one key in write order: bytes, and point tensors ([n, 104] Affine images) with whether the hash covers them"""
    parts = [struct.pack("<I", ck.powers_of_beta_g.shape[0]), (ck.powers_of_beta_g, True),
             struct.pack("<I", len(ck.lagrange_bases_at_beta_g))]
    for size in sorted(ck.lagrange_bases_at_beta_g):
        parts += [struct.pack("<I", size), (ck.lagrange_bases_at_beta_g[size], False)]
    parts += [struct.pack("<I", ck.powers_of_beta_times_gamma_g.shape[0]), (ck.powers_of_beta_times_gamma_g, True)]
    if ck.shifted_powers_of_beta_g is None:
        parts.append(b"\x00")
    else:
        parts += [b"\x01", struct.pack("<I", ck.shifted_powers_of_beta_g.shape[0]), (ck.shifted_powers_of_beta_g, True)]
    if ck.shifted_powers_of_beta_times_gamma_g is None:
        parts.append(b"\x00")
    else:
        parts += [b"\x01", struct.pack("<I", len(ck.shifted_powers_of_beta_times_gamma_g))]
        for b in sorted(ck.shifted_powers_of_beta_times_gamma_g):
            v = ck.shifted_powers_of_beta_times_gamma_g[b]
            parts += [struct.pack("<II", b, v.shape[0]), (v, True)]
    if ck.enforced_degree_bounds is None:
        parts.append(b"\x00")
    else:
        parts += [b"\x01", struct.pack(f"<I{len(ck.enforced_degree_bounds)}I", len(ck.enforced_degree_bounds), *ck.enforced_degree_bounds)]
    return parts


def committer_keys_to_bytes(cks: list) -> list:
    """ToBytes of every key, all points of all keys through one device.g1_serialize call (the 97-byte form) → [bytes]"""
    layouts = [_committer_key_parts(ck) for ck in cks]
    tensors = [t for parts in layouts for t, _h in (q for q in parts if not isinstance(q, bytes))]
    enc = np.zeros(0, dtype=np.uint8)
    if tensors and sum(t.shape[0] for t in tensors):
        flat = torch.cat([t.reshape(-1, STRIDE) for t in tensors])
        enc = device.g1_serialize(flat.contiguous(), device.G1_TO_BYTES).cpu().numpy().reshape(-1)
    out, at = [], 0
    for parts in layouts:
        chunks, h = [], hashlib.sha256()
        for q in parts:
            if isinstance(q, bytes):
                chunks.append(q)
                continue
            t, hashed = q
            b = enc[at: at + POINT_BYTES * t.shape[0]].tobytes()
            at += POINT_BYTES * t.shape[0]
            chunks.append(b)
            if hashed:
                h.update(b)
        out.append(b"".join(chunks) + h.digest())
    return out
