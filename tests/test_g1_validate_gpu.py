"""GPU: device.g1_validate (k_g1_validate) — Affine::check of G1 points taken from outside — against the statuses the big-integer
restatement in oracle/bls12_377.py gives: random subgroup points and infinity (valid), coordinate images at q and above, off-curve
points, on-curve points outside the prime-order subgroup (a random x with x³ + 1 square), and those points times the cofactor
(valid again)."""
import random

import numpy as np
import pytest

from oracle import bls12_377 as py

pytestmark = pytest.mark.gpu
Q, R = py.Q_MOD, py.R_MOD
COFACTOR = 0x170b5d44300000000000000000000000          # (q − x) / r, x the BLS parameter: the order of E(Fq) over r


def _sqrt(a: int):
    """a square root of a mod q (Tonelli–Shanks), None when a is not a square"""
    a %= Q
    if a == 0:
        return 0
    if pow(a, (Q - 1) // 2, Q) != 1:
        return None
    s, t = 0, Q - 1
    while t % 2 == 0:
        s, t = s + 1, t // 2
    z = next(z for z in range(2, 1000) if pow(z, (Q - 1) // 2, Q) == Q - 1)
    m, c, x, b = s, pow(z, t, Q), pow(a, (t + 1) // 2, Q), pow(a, t, Q)
    while b != 1:
        i, b2 = 0, b
        while b2 != 1:
            b2, i = b2 * b2 % Q, i + 1
        e = pow(c, 1 << (m - i - 1), Q)
        m, c, x, b = i, e * e % Q, x * e % Q, b * e * e % Q
    return x


def _raw(x_img: int, y_img: int) -> bytes:
    """an Affine image with the given raw (Montgomery-image) coordinates, not at infinity"""
    return x_img.to_bytes(48, "little") + y_img.to_bytes(48, "little") + b"\0" * 8


def _expected(p) -> int:
    """the oracle's status of a canonical point (None = infinity)"""
    if p is None:
        return 0
    if not py.g1_is_on_curve(p):
        return 2
    return 0 if py.g1_mul(p, R) is None else 3


def test_statuses_equal_the_oracle():
    import torch
    from snarkvm_b200 import device
    rng = random.Random(2024)
    images, want = [], []

    def add(p):
        images.append(py.affine_bytes(p))
        want.append(_expected(p))
    for _ in range(8):                                                  # subgroup points, infinity
        add(py.g1_mul(py.G1_GENERATOR, rng.randrange(1, R)))
    add(None)
    add(py.g1_mul(py.G1_GENERATOR, R - 1))
    outside = []
    while len(outside) < 6:                                             # on the curve, outside the subgroup
        x = rng.randrange(Q)
        y = _sqrt(x ** 3 + 1)
        if y is not None and py.g1_mul((x, y), R) is not None:
            outside.append((x, y))
    for p in outside:
        add(p)
        add(py.g1_mul(p, COFACTOR))                                     # cleared into the subgroup
        add((p[0], (p[1] + 1) % Q))                                     # off the curve
    good = py.g1_mul(py.G1_GENERATOR, 12345)
    gx, gy = py.fq_to_mont(good[0]), py.fq_to_mont(good[1])
    for x_img, y_img in ((Q, gy), (gx, Q), (Q + 1, gy), (gx, (1 << 384) - 1), ((1 << 381) + 5, gy)):
        images.append(_raw(x_img, y_img))                               # a coordinate image at q or above
        want.append(1)
    assert sorted(set(want)) == [0, 1, 2, 3]
    pts = torch.from_numpy(np.frombuffer(b"".join(images), dtype=np.uint8).reshape(-1, 104).copy()).cuda()
    assert device.g1_validate(pts).cpu().tolist() == want
    # a wider stride reads the same points
    wide = torch.zeros((pts.shape[0], 136), dtype=torch.uint8, device="cuda")
    wide[:, :104] = pts
    assert device.g1_validate(wide, stride=136).cpu().tolist() == want
    assert device.g1_validate(pts[:0]).numel() == 0
