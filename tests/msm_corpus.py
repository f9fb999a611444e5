"""Seeded MSM inputs shaped to reach the rare branches of the G1 pipeline (csrc/msm.cu), and the closed form that checks them.

Scalars
  * digit_boundary_scalars(c): for every window w, the window's c-bit field takes each of 0, 1, half − 1, half, half + 1 and
    2^c − 1 (half = 2^(c−1)) with an incoming carry of 0 and of 1, so the signed-digit recoding of k_digits / k_scatter_records
    meets raw == half (largest positive digit), raw == half + 1 (negative digit, carry out) and raw == 2^c (field all ones plus
    a carry: digit 0, carry out) in every window that can hold them below r.  Plus carry chains through all windows, every
    window at half / half + 1, top windows at their maximum below r, and 0, 1, r − 1.
  * equal / half-equal / few-hot scalar families (one hot bucket per window, a hot bucket over a full background, a few
    dozen hot values).
Bases
  Builders edit a base array and keep the multipliers in step: generated bases are P_i = k_i·G, a repeated row keeps k,
  a negated row gets r − k, an ∞ row gets 0.  Torsion rows (the order-2 point (q − 1, 0), the order-3 points (0, ±1)) are
  valid curve points outside the prime-order subgroup: they have no multiplier and are tracked by kind, and
  closed_form() adds their contribution (s mod 2 or ±s mod 3 copies) with big integers.
"""
from __future__ import annotations

import random

import numpy as np

from oracle import bls12_377 as py

R = py.R_MOD
Q = py.Q_MOD
SCALAR_BITS = 253

T2 = (Q - 1, 0)              # y² = x³ + 1 at x = −1: y = 0, order 2
T3 = (0, 1)                  # x = 0: y = ±1, order 3 (2·T3 = −T3 = (0, q − 1))
T3_NEG = (0, Q - 1)
TORSION = {"t2": T2, "t3": T3, "t3neg": T3_NEG}


def nwin_of(c: int) -> int:
    return SCALAR_BITS // c + 1


# ---------------------------------------------------------------------------------------------------------------------------
# scalars
# ---------------------------------------------------------------------------------------------------------------------------
def _set_field(s: int, w: int, c: int, f: int) -> int:
    mask = ((1 << c) - 1) << (w * c)
    return (s & ~mask) | (f << (w * c))


def digit_boundary_scalars(c: int, seed: int = 0) -> list[int]:
    """Canonical scalars < r whose windows reach the recoding's boundaries (see the module docstring), deterministic in seed."""
    rng = random.Random(seed * 1000003 + c)
    nw = nwin_of(c)
    half = 1 << (c - 1)
    fields = sorted({0, 1, half - 1, half, half + 1, (1 << c) - 1})
    out: list[int] = []
    for w in range(nw):
        for f in fields:
            for cin in ((0, 1) if w > 0 else (0,)):
                for attempt in range(3):
                    if attempt == 0:
                        s = rng.getrandbits(SCALAR_BITS)                       # random background
                    elif attempt == 1:
                        s = rng.getrandbits(w * c) if w else 0                 # nothing above window w
                    else:
                        s = 0
                    s = _set_field(s, w, c, f)
                    s &= (1 << (w + 1) * c) - 1 if attempt else (1 << 256) - 1
                    if w > 0:
                        # carry into w: window w − 1 all ones (raw ≥ 2^c − 1 > half) or its least value with carry out (half + 1);
                        # no carry: window w − 1 zero (raw ≤ 1 ≤ half)
                        lower = ((1 << c) - 1 if attempt < 2 else half + 1) if cin else 0
                        s = _set_field(s, w - 1, c, lower)
                        if attempt == 2:
                            s &= ~((1 << (w - 1) * c) - 1)
                    if s < R:
                        out.append(s)
                        break
    # carry chains through every window and every window at one boundary value
    for k in range(1, SCALAR_BITS):
        if k % c == 0 or k % c == c - 1 or k in (1, 2, 252):
            out.append((1 << k) - 1)
    for f in (half, half + 1, (1 << c) - 1, half - 1):
        s = 0
        for w in range(nw):
            s = _set_field(s, w, c, f)
        s &= (1 << 256) - 1
        while s >= R:                                               # drop top windows until it fits
            s &= (1 << (s.bit_length() - 1)) - 1
        out.append(s)
    # top windows at their maximum below r: the largest value of the top windows with everything below all ones / zero
    for w in range(nw - 1, max(-1, nw - 4), -1):
        top = (R - 1) >> (w * c)
        out.append(top << (w * c))
        out.append(min(R - 1, (top << (w * c)) | ((1 << (w * c)) - 1)))
    out += [0, 1, 2, R - 1, R - 2, (R - 1) // 2, R >> 1]
    assert all(0 <= s < R for s in out)
    return out


def to_limbs(vals) -> np.ndarray:
    return np.array([py.to_limbs(v, 4) for v in vals], dtype=np.uint64).reshape(-1, 4)


def mont_limbs(vals) -> np.ndarray:
    """Montgomery images s·2^256 mod r of canonical scalars (what KZG10::commit takes)"""
    return to_limbs([py.fr_to_mont(v) for v in vals])


def scalar_family(kind: str, n: int, seed: int) -> np.ndarray:
    """uint64 [n, 4] canonical scalars of one family:
       uniform, equal (one value: one hot bucket per window), half_equal (half the rows one value over a uniform background),
       few_hot (half the rows drawn from 48 values), special (0, 1, r − 1 in runs, uniform otherwise)."""
    from helpers import random_canonical_fr
    s = random_canonical_fr(n, seed)
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        return s
    if kind == "equal":
        return np.tile(s[:1], (n, 1))
    if kind == "half_equal":
        s[rng.permutation(n)[: n // 2]] = s[0]
        return s
    if kind == "few_hot":
        hot = rng.permutation(n)[: n // 2]
        s[hot] = s[rng.integers(0, 48, size=hot.size)]
        return s
    if kind == "special":
        k = max(1, n // 16)
        s[0:k] = 0
        s[k:2 * k] = to_limbs([1])[0]
        s[2 * k:3 * k] = to_limbs([R - 1])[0]
        return s
    raise ValueError(kind)


SCALAR_FAMILIES = ("uniform", "equal", "half_equal", "few_hot", "special")


# ---------------------------------------------------------------------------------------------------------------------------
# bases
# ---------------------------------------------------------------------------------------------------------------------------
class Bases:
    """A host base array [n, 104] with what is known about each row: ks[i] = k with row i = k·G (canonical, [n, 4] limbs),
    or a torsion kind in `torsion` (row index → "t2" / "t3" / "t3neg"), whose k is then 0 and whose contribution closed_form()
    adds separately."""

    def __init__(self, rows: np.ndarray, ks: np.ndarray):
        self.rows = rows
        self.ks = ks
        self.torsion: dict[int, str] = {}

    @staticmethod
    def generated(rows: np.ndarray, seed: int) -> "Bases":
        from helpers import generated_base_multipliers
        ks = np.zeros((rows.shape[0], 4), dtype=np.uint64)
        ks[:, 0] = generated_base_multipliers(seed, rows.shape[0])
        return Bases(rows.copy(), ks)

    def copy(self) -> "Bases":
        b = Bases(self.rows.copy(), self.ks.copy())
        b.torsion = dict(self.torsion)
        return b

    def repeat(self, src: int, idx) -> "Bases":
        """rows idx := row src (same multiplier)"""
        idx = np.asarray(idx)
        self.rows[idx] = self.rows[src]
        self.ks[idx] = self.ks[src]
        for i in idx.tolist():
            self.torsion.pop(i, None)
        if src in self.torsion:
            for i in idx.tolist():
                self.torsion[i] = self.torsion[src]
        return self

    def negate(self, idx) -> "Bases":
        """rows idx := −row (y → q − y in the Montgomery image; k → r − k)"""
        for i in np.asarray(idx).reshape(-1).tolist():
            if self.rows[i, 96]:
                continue
            y = int.from_bytes(self.rows[i, 48:96].tobytes(), "little")
            self.rows[i, 48:96] = np.frombuffer(((Q - y) % Q).to_bytes(48, "little"), dtype=np.uint8)
            k = py.from_limbs(self.ks[i])
            self.ks[i] = py.to_limbs((R - k) % R, 4)
            if i in self.torsion:
                self.torsion[i] = {"t2": "t2", "t3": "t3neg", "t3neg": "t3"}[self.torsion[i]]
        return self

    def alternate(self, src: int, idx) -> "Bases":
        """rows idx := P, −P, P, −P, … with P = row src"""
        idx = np.asarray(idx)
        self.repeat(src, idx)
        self.negate(idx[1::2])
        return self

    def infinity(self, idx) -> "Bases":
        idx = np.asarray(idx)
        self.rows[idx] = np.frombuffer(py.affine_bytes(None), dtype=np.uint8)
        self.ks[idx] = 0
        for i in idx.reshape(-1).tolist():
            self.torsion.pop(i, None)
        return self

    def torsion_points(self, idx, kind: str) -> "Bases":
        idx = np.asarray(idx)
        self.rows[idx] = np.frombuffer(py.affine_bytes(TORSION[kind]), dtype=np.uint8)
        self.ks[idx] = 0
        for i in idx.reshape(-1).tolist():
            self.torsion[i] = kind
        return self


def closed_form(cpu, b: Bases, scal: np.ndarray) -> np.ndarray:
    """Σ s_i·row_i as the normalised projective image (uint64 [18]): (Σ s_i·k_i mod r)·G from the oracle's dot product and
    scalar multiplication, plus the torsion rows' part with big integers (an order-2 point counts s mod 2 times, (0, 1) counts
    Σ ±s mod 3 times)."""
    n = scal.shape[0]
    g = np.frombuffer(py.affine_bytes(py.G1_GENERATOR), dtype=np.uint8)
    main = cpu.g1_mul(g, cpu.fr_dot_canonical(scal, b.ks[:n]))
    t2 = t3 = 0
    for i, kind in b.torsion.items():
        if i >= n:
            continue
        s = py.from_limbs(scal[i])
        if kind == "t2":
            t2 += s
        else:
            t3 += s if kind == "t3" else -s
    if t2 % 2 == 0 and t3 % 3 == 0:
        return main
    p = py.projective_from_bytes(main.tobytes())
    if t2 % 2:
        p = py.g1_add(p, T2)
    if t3 % 3:
        p = py.g1_add(p, T3 if t3 % 3 == 1 else T3_NEG)
    return np.frombuffer(py.projective_bytes_normalised(p), dtype=np.uint64)
