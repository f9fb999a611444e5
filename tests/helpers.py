"""Shared input generators for the parity tests (seeded, deterministic)."""
from __future__ import annotations

import numpy as np

from oracle import bls12_377 as py

R_LIMBS = np.array(py.to_limbs(py.R_MOD, 4), dtype=np.uint64)


def random_canonical_fr(n: int, seed: int) -> np.ndarray:
    """Uniform integers in [0, r) as uint64 [n, 4]: draw 4 limbs, clear the top REPR_SHAVE_BITS = 3 bits,
    reject ≥ r — the reference's own sampler (fields/src/macros.rs:40-56)."""
    rng = np.random.default_rng(seed)
    out = np.empty((n, 4), dtype=np.uint64)
    todo = np.arange(n)
    while todo.size:
        x = rng.integers(0, 2**64, size=(todo.size, 4), dtype=np.uint64)
        x[:, 3] &= np.uint64((1 << 61) - 1)
        ok = _less_than_r(x)
        out[todo[ok]] = x[ok]
        todo = todo[~ok]
    return out


def _less_than_r(x: np.ndarray) -> np.ndarray:
    lt = np.zeros(x.shape[0], dtype=bool)
    eq = np.ones(x.shape[0], dtype=bool)
    for i in (3, 2, 1, 0):
        lt |= eq & (x[:, i] < R_LIMBS[i])
        eq &= x[:, i] == R_LIMBS[i]
    return lt


def random_fr_mont(n: int, seed: int) -> np.ndarray:
    """Random field elements as Montgomery limb images.  Any canonical value < r is a valid Montgomery
    image of some element, so uniform canonical draws are uniform Fr images."""
    return random_canonical_fr(n, seed)


NEAR_R = np.array([py.to_limbs(py.R_MOD - 1, 4), py.to_limbs(py.R_MOD - 2, 4)], dtype=np.uint64)


def put_near_r(x):
    """The first and last min(4, n) rows of x ← r − 1, r − 2, r − 2, r − 1: the largest canonical limbs, which uniform draws
    never reach, at even and odd indices.  x: uint64 [n, 4] array or int64 [n, 4] tensor, modified in place → x."""
    k = min(4, x.shape[0])
    v = NEAR_R[[0, 1, 1, 0][:k]]
    if not isinstance(x, np.ndarray):
        import torch
        v = torch.from_numpy(v.view(np.int64)).to(x.device)
    x[:k] = v
    x[x.shape[0] - k:] = v
    return x


def fr_ints_to_mont_array(vals) -> np.ndarray:
    return np.array([py.to_limbs(py.fr_to_mont(v), 4) for v in vals], dtype=np.uint64).reshape(-1, 4)


def mont_array_to_fr_ints(arr) -> list:
    return [py.fr_from_mont(py.from_limbs(r)) for r in np.asarray(arr).reshape(-1, 4)]


def affine_array(points) -> np.ndarray:
    """list of (x, y) / None → uint8 [n, 104] reference images"""
    return np.frombuffer(b"".join(py.affine_bytes(p) for p in points), dtype=np.uint8).reshape(len(points), 104).copy()


def oracle_bases(cpu, n: int, seed: int) -> np.ndarray:
    """n distinct subgroup points on the CPU: P_i = (s + i)·G built by doubling blocks with the oracle's
    batched affine addition (no square roots, every point in the prime-order subgroup)."""
    s = 1 + (seed * 7919) % 1000003
    first = py.g1_mul(py.G1_GENERATOR, s)
    bases = np.zeros((n, 104), dtype=np.uint8)
    bases[0] = np.frombuffer(py.affine_bytes(first), dtype=np.uint8)
    cur = 1
    while cur < n:
        m = min(cur, n - cur)
        step = np.frombuffer(py.affine_bytes(py.g1_mul(py.G1_GENERATOR, cur)), dtype=np.uint8)
        bases[cur:cur + m] = cpu.batch_affine_add(bases[:m], np.tile(step, (m, 1)))
        cur += m
    return bases


def scalars_from_ints(vals) -> np.ndarray:
    return np.array([py.to_limbs(v, 4) for v in vals], dtype=np.uint64).reshape(-1, 4)


def splitmix64(x: int) -> int:
    m = (1 << 64) - 1
    x = (x + 0x9E3779B97F4A7C15) & m
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & m
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & m
    return x ^ (x >> 31)


def generated_base_multiplier(seed: int, i: int) -> int:
    """The 64-bit multiplier k with P_i = k·G used by snarkvm_b200_generate_bases_device (msm.cu)."""
    k = splitmix64((seed & ((1 << 64) - 1)) ^ splitmix64(i))
    return k if k else 1


def generated_base_multipliers(seed: int, n: int) -> np.ndarray:
    """Vectorised generated_base_multiplier for i in [0, n): uint64 [n]."""
    def sm(x):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return x ^ (x >> np.uint64(31))
    with np.errstate(over="ignore"):
        k = sm(np.uint64(seed & ((1 << 64) - 1)) ^ sm(np.arange(n, dtype=np.uint64)))
    k[k == 0] = 1
    return k
