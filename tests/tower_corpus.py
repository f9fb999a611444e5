"""Operand corpus for the element-wise tests of the pairing's extension tower and G2 line steps (tower.cuh, pairing.cu).

Elements are the oracle's tuples of plain Fq integers (tests/pairing_oracle.py): Fq2 = (c0, c1), Fq6 = (c0, c1, c2) of Fq2,
Fq12 = (c0, c1) of Fq6.  The device reads their Montgomery images in the GT word order, which `words` writes.  The shaped families
are chosen in image space, where the carries happen: components whose images are the values of tests/field_corpus.py (next to q
and to 2^{32k}, mostly-all-ones limbs), pairs of elements whose matching components are m_all_ones pairs (every reduction
multiplier of their products 2^32 − 1), and elements whose components, added as the Karatsuba / CH-SQR2 / mul_by_01 sums add them,
land on q − 1, q, q + 1 and 2q − 2.  The structured families are the cases where a formula that skips a component or a table row
still looks right on random inputs: zero, one, −1, one non-zero Fq2 (and one non-zero Fq) per slot, elements of Fq2 and of Fq6,
every component q − 1.  Everything is deterministic (seeded); tests/test_tower_corpus.py checks that each family is present.
"""
from __future__ import annotations

import random

import numpy as np

import field_corpus as fc
import pairing_oracle as po

Q = fc.Q
F2_ZERO, F2_ONE = (0, 0), (1, 0)
MINUS_ONE = Q - 1


# ---- images and words ------------------------------------------------------------------------------------------------------------
def plain(img: int) -> int:
    """the Fq element whose Montgomery image is img"""
    return img * fc.QR_INV % Q


def flat(x) -> list[int]:
    """plain Fq components of an Fq / Fq2 / Fq6 / Fq12 element (or a tuple of them) in memory order"""
    return [x] if isinstance(x, int) else [v for c in x for v in flat(c)]


def unflat(vals: list[int], kind: str):
    """inverse of flat for one element of kind "f2", "f6", "f12" or "f2x3" (a line-step state or a coefficient triple)"""
    f2 = [(vals[2 * i], vals[2 * i + 1]) for i in range(len(vals) // 2)]
    if kind == "f2":
        return f2[0]
    if kind in ("f6", "f2x3"):
        return tuple(f2[:3])
    assert kind == "f12"
    return (tuple(f2[:3]), tuple(f2[3:6]))


def words(elems) -> np.ndarray:
    """[len(elems), 12·components] uint32: the Montgomery images of every element's components, limbs little-endian"""
    rows = [[v * fc.QR % Q for v in flat(e)] for e in elems]
    n = len(rows[0])
    return fc.to_limbs([v for r in rows for v in r], 12).reshape(len(rows), 12 * n)


def from_words(arr: np.ndarray, kind: str) -> list:
    """device words → elements; asserts that every component image is below q"""
    imgs = fc.from_limbs(np.ascontiguousarray(arr, dtype=np.uint32).reshape(-1, 12))
    assert all(v < Q for v in imgs), "unreduced component"
    per = arr.shape[1] // 12
    return [unflat([plain(v) for v in imgs[i * per:(i + 1) * per]], kind) for i in range(arr.shape[0])]


# ---- component pools -------------------------------------------------------------------------------------------------------------
def _image_pool(rng: random.Random) -> list[int]:
    return fc.fixed_values(Q, 12) + fc.mostly_ones(rng, Q, 12, 40) + fc.uniform(rng, Q, 24)


def _boundary(rng: random.Random, v: int) -> int:
    """an image w < q with v + w ∈ {q − 1, q, q + 1, 2q − 2} (q − 1 − v always qualifies)"""
    return rng.choice([s - v for s in (Q - 1, Q, Q + 1, 2 * Q - 2) if 0 <= s - v < Q])


def _shaped(rng: random.Random, pool: list[int], ncomp: int, boundary: bool) -> list[int]:
    """ncomp plain components whose images come from the pool; with `boundary`, the second Fq2 slot and most later ones are chosen
    so that each of their components sums with the matching component of an earlier slot (or of the other Fq6 half) to a wrap
    point (the first slot is often q − 1, from which 2q − 2 is reachable)"""
    imgs: list[int] = []
    for i in range(ncomp):
        if boundary and i >= 2 and (i < 4 or rng.random() < 0.8):
            imgs.append(_boundary(rng, imgs[rng.randrange(i % 2, i, 2)]))    # same component (c0 / c1) of an earlier Fq2 slot
        elif boundary and i < 2 and rng.random() < 0.25:
            imgs.append(Q - 1)
        else:
            imgs.append(rng.choice(pool))
    return [plain(v) for v in imgs]


def fq2_values(seed: int = 0) -> list[tuple[int, int]]:
    """Fq2 values for slots and coefficients: 0, 1, u, −1, (q − 1, q − 1) in both plain and image form, shaped, random"""
    rng = random.Random(f"tower-fq2:{seed}")
    pool = _image_pool(rng)
    vals = [F2_ZERO, F2_ONE, (0, 1), (MINUS_ONE, 0), (MINUS_ONE, MINUS_ONE), (plain(Q - 1), plain(Q - 1)), (plain(1), 0)]
    vals += [tuple(_shaped(rng, pool, 2, False)) for _ in range(10)]
    vals += [(rng.randrange(Q), rng.randrange(Q)) for _ in range(3)]
    return vals


# ---- elements --------------------------------------------------------------------------------------------------------------------
def _f6(c) -> tuple: return (c[0], c[1], c[2])
def _f12(c) -> tuple: return ((c[0], c[1], c[2]), (c[3], c[4], c[5]))


def _build(slots: int, f2s: list) -> tuple:
    return _f6(f2s) if slots == 3 else _f12(f2s)


def elements(kind: str, seed: int = 0) -> list[tuple[str, tuple]]:
    """(family, element) for kind "f6" or "f12".  Families: zero, one, minus_one, slot<i> (one non-zero Fq2 in slot i), fq<j> (one
    non-zero Fq component j), in_fq2, in_fq6 (f12: c1 = 0), in_w (f12: c0 = 0), all_q_minus_1 (plain and image), shaped, boundary,
    uniform"""
    slots = 3 if kind == "f6" else 6
    rng = random.Random(f"tower-{kind}:{seed}")
    pool = _image_pool(rng)
    f2v = fq2_values(seed)
    zero = [F2_ZERO] * slots
    out = [("zero", _build(slots, zero)), ("one", _build(slots, [F2_ONE] + zero[1:])),
           ("minus_one", _build(slots, [(MINUS_ONE, 0)] + zero[1:]))]
    for i in range(slots):
        for v in rng.sample(f2v[1:], 4):
            s = list(zero)
            s[i] = v
            out.append((f"slot{i}", _build(slots, s)))
    for j in range(2 * slots):
        for v in (1, MINUS_ONE, rng.choice([plain(x) for x in pool if x])):
            comps = [0] * (2 * slots)
            comps[j] = v
            out.append((f"fq{j}", unflat(comps, kind)))
    for v in f2v[1:8]:
        out.append(("in_fq2", _build(slots, [v] + zero[1:])))
    if kind == "f12":
        for _ in range(6):
            out.append(("in_fq6", _f12(list(unflat(_shaped(rng, pool, 6, True), "f6")) + [F2_ZERO] * 3)))
            out.append(("in_w", _f12([F2_ZERO] * 3 + list(unflat(_shaped(rng, pool, 6, True), "f6")))))
    out.append(("all_q_minus_1", unflat([MINUS_ONE] * (2 * slots), kind)))
    out.append(("all_q_minus_1", unflat([plain(Q - 1)] * (2 * slots), kind)))
    for _ in range(24):
        out.append(("shaped", unflat(_shaped(rng, pool, 2 * slots, False), kind)))
    for _ in range(24):
        out.append(("boundary", unflat(_shaped(rng, pool, 2 * slots, True), kind)))
    for _ in range(8):
        out.append(("uniform", unflat([rng.randrange(Q) for _ in range(2 * slots)], kind)))
    return out


def pairs(kind: str, seed: int = 0) -> list[tuple[tuple, tuple]]:
    """operand pairs for the products: every element against a few partners (itself, one, −1, a shaped and a uniform element),
    element pairs whose matching components are m_all_ones pairs, and boundary elements against each other"""
    rng = random.Random(f"tower-pairs-{kind}:{seed}")
    fam_els = elements(kind, seed)
    els = [e for _, e in fam_els]
    fam = dict(fam_els)
    partners = [fam["one"], fam["minus_one"], fam["all_q_minus_1"]] + [e for f, e in fam_els if f == "shaped"][:2]
    out = [(a, a) for a in els] + [(a, rng.choice(partners)) for a in els] + [(rng.choice(els), a) for a in els]
    ncomp = 6 if kind == "f6" else 12
    for _ in range(24):
        ab = fc.m_all_ones_pairs(rng, Q, 12, ncomp)
        out.append((unflat([plain(a) for a, _ in ab], kind), unflat([plain(b) for _, b in ab], kind)))
    bnd = [e for f, e in fam_els if f == "boundary"]
    out += list(zip(bnd, bnd[1:] + bnd[:1]))
    return out


def sparse_coefficients(n: int, seed: int = 0) -> list[tuple]:
    """n Fq2 tuples for mul_by_01 (n = 2) or mul_by_034 / a line triple (n = 3): every part zero, 1, −1 or q − 1 in both forms in
    turn, then shaped and uniform parts"""
    rng = random.Random(f"tower-coeffs-{n}:{seed}")
    f2v = fq2_values(seed)
    special = f2v[:7]
    out = []
    for i in range(n):                                   # one part special, the others not
        for v in special:
            t = [rng.choice(f2v[7:]) for _ in range(n)]
            t[i] = v
            out.append(tuple(t))
    for v in special:
        out.append(tuple([v] * n))
    for _ in range(30):
        out.append(tuple(rng.choice(f2v) for _ in range(n)))
    return out


def mul_by_01_cases(seed: int = 0) -> list[tuple[tuple, tuple]]:
    els = [e for _, e in elements("f6", seed)]
    co = sparse_coefficients(2, seed)
    rng = random.Random(f"tower-01:{seed}")
    return [(e, co[i % len(co)]) for i, e in enumerate(els)] + [(rng.choice(els), c) for c in co]


def mul_by_034_cases(seed: int = 0) -> list[tuple[tuple, tuple]]:
    els = [e for _, e in elements("f12", seed)]
    co = sparse_coefficients(3, seed)
    rng = random.Random(f"tower-034:{seed}")
    return [(e, co[i % len(co)]) for i, e in enumerate(els)] + [(rng.choice(els), c) for c in co]


def ell_cases(seed: int = 0) -> list[tuple[tuple, tuple, tuple[int, int]]]:
    """(f, coefficient triple, G1 point (x, y)): the point's coordinates from the shaped pool, 0, 1 and −1 among them"""
    rng = random.Random(f"tower-ell:{seed}")
    pool = [plain(v) for v in _image_pool(rng)] + [0, 1, MINUS_ONE]
    return [(f, c, (rng.choice(pool), rng.choice(pool))) for f, c in mul_by_034_cases(seed)[::2]]


def easy_part(f):
    """f^((q⁶ − 1)(q² + 1)), which lies in the cyclotomic subgroup"""
    g = po.f12_mul(po.f12_conj(f), po.f12_inv(f))
    return po.f12_mul(po.f12_frob(g, 2), g)


def cyclotomic_elements(seed: int = 0) -> list[tuple]:
    """one, and the easy-part image of every non-zero element of the Fq12 corpus (duplicates dropped)"""
    out = [po.F12_ONE]
    for f, e in elements("f12", seed):
        if f != "zero":
            g = easy_part(e)
            if g not in out:
                out.append(g)
    return out


def is_one_cases() -> list[tuple[tuple, bool, int | None]]:
    """(element, is it one, the word that was changed or None): zero, one, −1, raw 1 (image 1, not one), then one with a single
    word changed at each of the 144 word positions, by its low bit and by a high bit that keeps the component below q"""
    one_img = [fc.QR] + [0] * 11
    cases = [(unflat([0] * 12, "f12"), False, None), (po.F12_ONE, True, None), (unflat([MINUS_ONE] + [0] * 11, "f12"), False, None),
             (unflat([plain(1)] + [0] * 11, "f12"), False, None)]
    for w in range(144):
        fi, li = divmod(w, 12)
        for bit in (0, 31 if li < 11 else 24):
            imgs = list(one_img)
            imgs[fi] ^= 1 << (32 * li + bit)
            assert imgs[fi] < Q
            cases.append((unflat([plain(v) for v in imgs], "f12"), False, w))
    return cases


def final_exp_cases(seed: int = 0) -> list[tuple[str, tuple]]:
    """(family, element) for the final exponentiation, without the device Miller values (the GPU test adds them): zero, which the
    device maps to zero; non-zero elements of Fq6, which go to one; a few general elements"""
    rng = random.Random(f"tower-fe:{seed}")
    f12 = elements("f12", seed)
    in6 = [e for f, e in f12 if f in ("one", "minus_one", "in_fq2", "in_fq6")
           or (f.startswith("slot") and int(f[4:]) < 3) or (f.startswith("fq") and f[2:].isdigit() and int(f[2:]) < 6)]
    out = [("zero", f12[0][1])] + [("in_fq6", e) for e in rng.sample(in6, 12)]
    general = [e for f, e in f12 if f in ("in_w", "boundary", "all_q_minus_1") or (f.startswith("slot") and int(f[4:]) >= 3)]
    out += [("general", e) for e in rng.sample(general, 8)]
    return out


def line_states(seed: int = 0) -> list[tuple]:
    """(X, Y, Z) over Fq2 for the line steps: every coordinate from fq2_values (zeros and q − 1 among them), and the affine images
    (x, y, 1) of a few G2 points"""
    rng = random.Random(f"tower-line:{seed}")
    f2v = fq2_values(seed)
    out = [(a, b, c) for a in f2v[:7] for b in f2v[:7] for c in f2v[:7] if rng.random() < 0.25]
    out += [tuple(rng.choice(f2v) for _ in range(3)) for _ in range(60)]
    out += [(p[0], p[1], F2_ONE) for p in fc.g2_points(4, seed)]
    return out


def addition_cases(seed: int = 0) -> list[tuple[tuple, tuple]]:
    """(state, affine Q) pairs: Q from fq2_values and real G2 points, with states equal to Q's affine image among them"""
    rng = random.Random(f"tower-add:{seed}")
    f2v = fq2_values(seed)
    pts = fc.g2_points(4, seed)
    out = [(s, (rng.choice(f2v), rng.choice(f2v))) for s in line_states(seed)]
    out += [((p[0], p[1], F2_ONE), p) for p in pts]
    out += [((pts[i][0], pts[i][1], F2_ONE), pts[(i + 1) % len(pts)]) for i in range(len(pts))]
    return out
