"""GPU: the BLS12-377 pairing on the device (device.g2_prepare, device.pairing_products) against the big-int restatement
(tests/pairing_oracle.py), the whole mainnet SRS checked by pairings, and verify_vk_batch's verdict with a UniversalVerifier."""
import os
import random

import numpy as np
import pytest

from oracle import bls12_377 as py
from oracle import g2 as og2

import pairing_oracle as po
from helpers import affine_array

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
R = py.R_MOD
BETA, GAMMA = 0x1234567890ABCDEF1234567890ABCDEF % R, 0xFEDCBA0987654321FEDCBA % R


def _g2_images(points):
    import torch
    return torch.from_numpy(np.frombuffer(b"".join(og2.g2_affine_bytes(p) for p in points), dtype=np.uint8).reshape(-1, 200).copy()).cuda()


def _i32(v):
    import torch
    return torch.tensor(v, dtype=torch.int32, device="cuda")


def _g1(points):
    import torch
    return torch.from_numpy(affine_array(points)).cuda()


def _rows(t):
    return [bytes(r) for r in t.cpu().numpy()]


def test_prepare_vs_oracle():
    from snarkvm_b200 import device
    rng = random.Random(1)
    pts = [og2.G2_GEN, None] + [og2.g2_mul(og2.G2_GEN, rng.randrange(1, R)) for _ in range(3)] + [None]
    got = _rows(device.g2_prepare(_g2_images(pts)))
    assert got == [po.prepared_bytes(po.g2_prepare(p)) for p in pts]


def test_miller_values_and_gt_vs_oracle():
    from snarkvm_b200 import device
    rng = random.Random(2)
    g2s = [og2.G2_GEN, og2.g2_mul(og2.G2_GEN, rng.randrange(1, R)), None]
    prepared = device.g2_prepare(_g2_images(g2s))
    g1s = [py.G1_GENERATOR, py.g1_mul(py.G1_GENERATOR, rng.randrange(1, R)), None, py.g1_mul(py.G1_GENERATOR, rng.randrange(1, R))]
    pairs = [(0, 0), (1, 1), (2, 0), (3, 2), (3, 1), (1, 0)]             # (G1, G2) indices; G1 #2 and G2 #2 are at infinity
    checks = [[0], [1], [2], [3], [0, 1, 2, 3, 4, 5], [4, 5], []]
    order = [p for c in checks for p in c]
    starts = np.cumsum([0] + [len(c) for c in checks]).tolist()
    gt, is_one, miller = device.pairing_products(_g1([g1s[pairs[i][0]] for i in order]), _i32([pairs[i][1] for i in order]), prepared,
                                                 _i32(starts), miller=True)
    preps = [po.g2_prepare(q) for q in g2s]
    want_miller = [po.miller_loop([(g1s[pairs[i][0]], preps[pairs[i][1]])]) for i in order]
    assert _rows(miller) == [po.gt_bytes(f) for f in want_miller]
    want_gt = []
    for c in checks:
        want_gt.append(po.final_exponentiation(po.miller_loop([(g1s[pairs[i][0]], preps[pairs[i][1]]) for i in c])))
    assert _rows(gt) == [po.gt_bytes(f) for f in want_gt]
    assert is_one.cpu().tolist() == [f == po.F12_ONE for f in want_gt] == [False, False, True, True, False, False, True]
    assert want_gt[0] == po.pairing(py.G1_GENERATOR, og2.G2_GEN)


def test_mixed_batch_of_checks_is_bilinear():
    """40 checks of 1–16 pairs Σ e(s_i·G, t_j·H): one exactly when Σ s_i·t_j ≡ 0 (mod r).  Pairs at infinity on either side are mixed
    in, and one check has nothing else — about 350 device pairings."""
    import torch
    from snarkvm_b200 import device
    rng = random.Random(3)
    ts = [rng.randrange(1, R) for _ in range(6)]
    prepared = device.g2_prepare(_g2_images([og2.g2_mul(og2.G2_GEN, t) for t in ts] + [None]))
    INF = len(ts)
    scalars, g2_index, starts, want = [], [], [0], []
    for c in range(40):
        n = 1 + c % 16
        js = [rng.randrange(len(ts)) for _ in range(n)]
        ss = [rng.randrange(R) for _ in range(n - 1)]
        acc = sum(s * ts[j] for s, j in zip(ss, js)) % R
        last = -acc * pow(ts[js[-1]], -1, R) % R
        one = c % 3 != 1
        ss.append(last if one else (last + 1) % R)
        if c == 7:                                                        # nothing but infinity
            js, ss, one = [INF, 0], [5, 0], True
        elif c % 5 == 0:                                                  # an extra pair at infinity on each side
            js, ss = js + [INF, 1], ss + [rng.randrange(1, R), 0]
        scalars += ss
        g2_index += js
        starts.append(len(scalars))
        want.append(one)
    limbs = np.array([[(s >> (64 * i)) & (2**64 - 1) for i in range(4)] for s in scalars], dtype=np.uint64)
    g1 = device.generator_mul(torch.from_numpy(limbs.view(np.int64)).cuda())
    gt, is_one = device.pairing_products(g1, _i32(g2_index), prepared, _i32(starts))
    assert is_one.cpu().tolist() == want
    assert len(scalars) > 300
    ones = [bytes(r) for r, w in zip(gt.cpu().numpy(), want) if w]
    assert set(ones) == {po.gt_bytes(po.F12_ONE)}


@pytest.fixture(scope="module")
def real_srs():
    blob = open(os.path.join(HERE, "golden", "powers_of_beta_15.usrs"), "rb").read()
    return py.parse_usrs_points(blob, int.from_bytes(blob[:8], "little"))


def _beta_h():
    with open(os.path.join(HERE, "golden", "beta_h.usrs"), "rb") as f:
        return po.usrs_g2_point(f.read())


def _srs_checks(powers):
    """check i: e(powers[i+1], H)·e(−powers[i], β·H)"""
    n = len(powers) - 1
    pts = [p for i in range(n) for p in (powers[i + 1], py.g1_neg(powers[i]))]
    return _g1(pts), _i32([0, 1] * n), _i32(list(range(0, 2 * n + 1, 2)))


def test_the_whole_mainnet_srs(real_srs):
    from snarkvm_b200 import device
    prepared = device.g2_prepare(_g2_images([og2.G2_GEN, _beta_h()]))
    g1, idx, starts = _srs_checks(real_srs)
    _gt, is_one = device.pairing_products(g1, idx, prepared, starts)
    assert is_one.numel() == (1 << 15) - 1 and bool(is_one.all())
    swapped = list(real_srs)
    swapped[100], swapped[200] = swapped[200], swapped[100]
    g1, idx, starts = _srs_checks(swapped)
    _gt, is_one = device.pairing_products(g1, idx, prepared, starts)
    assert [i for i, v in enumerate(is_one.cpu().tolist()) if not v] == [99, 100, 199, 200]


def test_bad_inputs_are_rejected():
    import torch
    from snarkvm_b200 import CudaError, device
    imgs = _g2_images([og2.G2_GEN, og2.G2_GEN, og2.G2_GEN])
    bad = imgs.clone()
    q = torch.from_numpy(np.frombuffer(py.Q_MOD.to_bytes(48, "little"), dtype=np.uint8).copy()).cuda()
    bad[1, 48:96] = q                                                     # x.c1 = q
    bad[2, 144:192] = q
    with pytest.raises(CudaError) as ei:
        device.g2_prepare(bad)
    assert ei.value.point == 1
    prepared = device.g2_prepare(imgs)
    g1 = _g1([py.G1_GENERATOR] * 4)
    g1b = g1.clone()
    g1b[2, 0:48] = q
    with pytest.raises(CudaError) as ei:
        device.pairing_products(g1b, _i32([0, 1, 2, 0]), prepared, _i32([0, 2, 4]))
    assert ei.value.check == 1
    with pytest.raises(CudaError) as ei:
        device.pairing_products(g1, _i32([0, 1, 2, 3]), prepared, _i32([0, 1, 2, 3, 4]))     # G2 index out of range
    assert ei.value.check == 3
    with pytest.raises(CudaError):
        device.pairing_products(g1, _i32([0, 1, 2, 0]), prepared, _i32([0, 3, 2, 4]))
    with pytest.raises(CudaError):
        device.pairing_products(g1, _i32([0, 1, 2, 0]), prepared, _i32([0, 2, 3]))           # does not end at the last pair


# ---- verify_vk with a verdict ----
def _program(powers, gamma, shapes, rng):
    from snarkvm_b200 import varuna as dv
    circuits = [dv.test_circuit_csr(rng.randrange(2, R), rng.randrange(2, R), *s, "cuda")[0] for s in shapes]
    setups = dv.batch_circuit_setup(circuits, powers, gamma, with_id=True)
    pks, vks = [s[0] for s in setups], [s[1] for s in setups]
    challenges = [[rng.randrange(R) for _ in range(12)] for _ in circuits]
    openings = [[rng.randrange(R), rng.randrange(R)] for _ in circuits]
    certs = dv.prove_vk_batch(pks, challenges, openings)
    return circuits, vks, certs, challenges, [o[0] for o in openings]


def _same(a, b):
    return (a.matches == b.matches and a.evaluation == b.evaluation and (a.lhs == b.lhs).all() and (a.w == b.w).all()
            and a.valid == b.valid)


SHAPES = [(3, 7, 7), (3, 100, 70), (2, 1024, 1014), (4, 300, 250)]


def _check_program(verifier, powers, gamma, shapes, rng):
    from snarkvm_b200 import varuna as dv
    circuits, vks, certs, ch, xi = _program(powers, gamma, shapes, rng)
    res = dv.verify_vk_batch(circuits, vks, certs, ch, xi, verifier=verifier)
    assert all(r.matches and r.valid is True for r in res)
    plain = dv.verify_vk_batch(circuits, vks, certs, ch, xi)
    assert all(p.valid is None for p in plain)
    assert all(_same(dv.VerifyingKeyCheck(p.matches, p.evaluation, p.lhs, p.w, r.valid), r) for p, r in zip(plain, res))
    loop = [dv.verify_vk(c, vk, cert, chk, x, verifier) for c, vk, cert, chk, x in zip(circuits, vks, certs, ch, xi)]
    assert all(_same(a, b) for a, b in zip(loop, res))
    return circuits, vks, certs, ch, xi


def test_verify_vk_verdict_on_a_synthetic_srs():
    from snarkvm_b200 import device
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import synthetic_srs
    rng = random.Random(4)
    powers, gamma = synthetic_srs(4095, BETA, GAMMA)
    verifier = dv.UniversalVerifier.synthetic(BETA)
    assert bytes(verifier.beta_h) == og2.g2_affine_bytes(og2.g2_mul(og2.G2_GEN, BETA))
    assert bytes(verifier.h) == og2.g2_affine_bytes(og2.G2_GEN)
    circuits, vks, certs, ch, xi = _check_program(verifier, powers, gamma, SHAPES, rng)
    K = len(circuits)
    # w perturbed: G in place of W
    import torch
    g = device.generator_mul(torch.tensor([[1, 0, 0, 0]], dtype=torch.int64, device="cuda")).cpu().numpy()[0]
    other = np.zeros(18, dtype=np.uint64)
    other[:12] = g[:96].view(np.uint64)
    other[12:18] = np.frombuffer(((1 << 384) % py.Q_MOD).to_bytes(48, "little"), dtype=np.uint64)
    bad_certs = list(certs)
    bad_certs[1] = dv.Certificate(other)
    res = dv.verify_vk_batch(circuits, vks, bad_certs, ch, xi, verifier=verifier)
    assert [r.valid for r in res] == [k != 1 for k in range(K)] and all(r.matches for r in res)
    # the challenges differ
    bad_ch = [list(c) for c in ch]
    bad_ch[2][11] = (bad_ch[2][11] + 1) % R
    res = dv.verify_vk_batch(circuits, vks, certs, bad_ch, xi, verifier=verifier)
    assert [r.valid for r in res] == [k != 2 for k in range(K)] and all(r.matches for r in res)
    bad_xi = list(xi)
    bad_xi[0] = (bad_xi[0] + 1) % R
    assert [r.valid for r in dv.verify_vk_batch(circuits, vks, certs, ch, bad_xi, verifier=verifier)] == [k != 0 for k in range(K)]
    # two circuits' verifying keys swapped
    vks2 = [vks[1], vks[0]] + vks[2:]
    res = dv.verify_vk_batch(circuits, vks2, certs, ch, xi, verifier=verifier)
    assert [r.valid for r in res] == [False, False] + [True] * (K - 2)
    # another circuit against the verifying key: matches is false as well
    wrong = dv.test_circuit_csr(3, 5, 3, 128, 70, "cuda")[0]
    res = dv.verify_vk(wrong, vks[1], certs[1], ch[1], xi[1], verifier)
    assert not res.matches and res.valid is False


def test_verify_vk_verdict_on_the_real_srs(real_srs):
    import torch
    from snarkvm_b200 import varuna as dv
    rng = random.Random(5)
    powers = torch.from_numpy(affine_array(real_srs)).cuda()
    with open(os.path.join(HERE, "golden", "beta_h.usrs"), "rb") as f:
        verifier = dv.UniversalVerifier.from_usrs(f.read())
    assert bytes(verifier.beta_h) == og2.g2_affine_bytes(_beta_h())
    assert (verifier.g == affine_array(real_srs[:1])[0]).all()
    circuits, vks, certs, ch, xi = _check_program(verifier, powers, powers, [(3, 7, 7), (2, 1 << 12, (1 << 12) - 10)], rng)
    res = dv.verify_vk_batch(circuits, vks, certs[::-1], ch, xi, verifier=verifier)
    assert [r.valid for r in res] == [False, False]
