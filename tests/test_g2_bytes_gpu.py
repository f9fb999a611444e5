"""GPU: G2 points from and to their bytes, G2 validation, and the verifier key's byte form.

device.g2_deserialize / g2_validate (k_g2_deserialize, k_g2_validate) against the big-integer restatement (g2_bytes_oracle) on a
corpus of subgroup points of both signs, infinity in both forms, on-curve points off the subgroup (random x with a root, and their
sums with subgroup points), off-curve points, each coordinate at or above q, every bad flag combination, compressed x without a
root and 400 random squares; device.g2_serialize's sign rule on images whose y has c1 = 0.  The mainnet β·H and negative powers
decode validated and re-serialise; UniversalVerifier.from_mainnet(validate=True) accepts them and names a replaced entry;
UniversalVerifier.to_bytes / from_bytes round-trip and the rebuilt verifier gives the same verify_vk and verify_batch verdicts."""
import copy
import os
import random

import numpy as np
import pytest
import torch

import g2_bytes_oracle as o
import varuna_bytes_oracle as vb
from oracle import bls12_377 as py
from oracle import g2 as og2

pytestmark = pytest.mark.gpu
Q, R = o.Q, o.R
HERE = os.path.dirname(os.path.abspath(__file__))


def _read(name):
    with open(os.path.join(HERE, "golden", name), "rb") as f:
        return f.read()


def _neg(p):
    return (p[0], og2.f2_neg(p[1]))


def _raw(coords, flags=0):
    b = bytearray(b"".join(v.to_bytes(48, "little") for v in coords))
    b[-1] |= flags
    return bytes(b)


@pytest.fixture(scope="module")
def corpus():
    """{compressed: [bytes]}"""
    rng = random.Random(0x62B7E5)
    sub = [og2.g2_mul(o.G2_GEN, rng.randrange(1, R)) for _ in range(8)] + [o.G2_GEN]
    off, squares, non = [], [], []
    while len(squares) < 400 or len(non) < 8:
        x = (rng.randrange(Q), rng.randrange(Q))
        (squares if o.fq2_sqrt(o.rhs(x)) is not None else non).append(x)
    for x in squares[:6]:
        p = (x, o.fq2_sqrt(o.rhs(x)))
        assert o.check(p) == o.NOT_IN_SUBGROUP
        off.append(p)
    off += [og2.g2_add(p, s) for p, s in zip(off[:3], sub)]
    # x with c1 = 0: x³ + B' has c0 = x0³, c1 = b1, so these reach the a1 ≠ 0 branch with small norms
    for c0 in range(1, 40):
        if o.fq2_sqrt(o.rhs((c0, 0))) is not None:
            squares.append((c0, 0))
    comp, unc = [], []
    for p in sub + off:
        for q in (p, _neg(p)):
            comp.append(o.encode(q, True))
            unc.append(o.encode(q, False))
    comp += [o.encode(None, True), _raw((5, 7), o.INFINITY)]
    unc += [o.encode(None, False), _raw((1, 2, 3, 4), o.INFINITY)]
    comp += [_raw(x, f) for x in squares for f in (0, o.POSITIVE_Y)][:800]
    comp += [_raw(x, f) for x in non for f in (0, o.POSITIVE_Y)]
    # off-curve uncompressed points: a subgroup point with one coordinate moved
    g = sub[0]
    unc += [_raw((g[0][0], g[0][1], (g[1][0] + 1) % Q, g[1][1])), _raw(((g[0][0] + 1) % Q, g[0][1], g[1][0], g[1][1]))]
    # every coordinate at q and above
    for k in range(2):
        for v in (Q, Q + 1, (1 << 382) - 1):
            c = [g[0][0], g[0][1]]
            c[k] = v
            comp.append(_raw(c))
    for k in range(4):
        for v in (Q, Q + 1):
            c = [g[0][0], g[0][1], g[1][0], g[1][1]]
            c[k] = v
            unc.append(_raw(c))
    # every flag combination: bit 7 / bit 6 of each coordinate's last byte
    for size, base in ((2, [g[0][0], g[0][1]]), (4, [g[0][0], g[0][1], g[1][0], g[1][1]])):
        good = _raw(base)
        for k in range(size):
            for f in (0x40, 0x80, 0xC0):
                b = bytearray(good)
                b[48 * k + 47] |= f
                (comp if size == 2 else unc).append(bytes(b))
    return {True: comp, False: unc}


@pytest.mark.parametrize("compressed", [True, False], ids=["compressed", "uncompressed"])
@pytest.mark.parametrize("validate", [True, False], ids=["validate", "unchecked"])
def test_deserialize_equals_the_oracle(corpus, compressed, validate):
    from snarkvm_b200 import device
    blobs = corpus[compressed]
    raw = torch.from_numpy(np.frombuffer(b"".join(blobs), dtype=np.uint8).copy()).cuda()
    images, status = device.g2_deserialize(raw, compressed, validate)
    images, status = images.cpu().numpy(), status.cpu().numpy()
    want = [o.image(b, compressed, validate) for b in blobs]
    for k, (b, (s, img)) in enumerate(zip(blobs, want)):
        assert int(status[k]) == s, (k, b.hex())
        assert images[k].tobytes() == img, (k, b.hex())
    seen = set(int(v) for v in status)
    assert {o.VALID, o.NOT_CANONICAL, o.BAD_FLAGS} <= seen
    if compressed:
        assert o.NOT_ON_CURVE in seen
    if validate:
        assert o.NOT_IN_SUBGROUP in seen and (compressed or o.NOT_ON_CURVE in seen)


def test_validate_equals_the_oracle(corpus):
    """g2_validate on the images of every uncompressed point that decodes, and on images with a coordinate ≥ q, strided"""
    from snarkvm_b200 import device
    pts = [p for b in corpus[False] for s, p in [o.decode(b, False, False)] if s == o.VALID]
    imgs = [og2.g2_affine_bytes(p) for p in pts]
    bad = bytearray(og2.g2_affine_bytes(o.G2_GEN))
    bad[96:144] = Q.to_bytes(48, "little")                        # y.c0 = q as a raw image
    imgs.append(bytes(bad))
    want = [o.check(p) for p in pts] + [o.NOT_CANONICAL]
    stride = 208
    buf = np.zeros((len(imgs), stride), dtype=np.uint8)
    buf[:, :200] = np.frombuffer(b"".join(imgs), dtype=np.uint8).reshape(-1, 200)
    status = device.g2_validate(torch.from_numpy(buf).cuda(), stride).cpu().numpy()
    assert [int(s) for s in status] == want
    assert {o.VALID, o.NOT_ON_CURVE, o.NOT_IN_SUBGROUP, o.NOT_CANONICAL} <= set(want)


def test_serialize_inverts_deserialize_and_signs_by_fp2_order(corpus):
    from snarkvm_b200 import device
    for compressed in (True, False):
        blobs = [b for b in corpus[compressed] if o.decode(b, compressed, False)[0] == o.VALID]
        pts = [o.decode(b, compressed, False)[1] for b in blobs]
        imgs = torch.from_numpy(np.frombuffer(b"".join(og2.g2_affine_bytes(p) for p in pts), dtype=np.uint8).copy()).cuda()
        out = device.g2_serialize(imgs, compressed).cpu().numpy()
        assert [bytes(r) for r in out] == [o.encode(p, compressed) for p in pts]
    # synthetic images whose y has c1 = 0: c0 alone decides the sign
    rng = random.Random(9)
    ys = [(rng.randrange(Q), 0) for _ in range(16)] + [((Q - 1) // 2, 0), ((Q + 1) // 2, 0), (0, 0), (1, 0), (Q - 1, 0),
                                                        (5, 1), (5, Q - 1), (0, (Q - 1) // 2), (0, (Q + 1) // 2)]
    pts = [((rng.randrange(Q), rng.randrange(Q)), y) for y in ys]
    imgs = torch.from_numpy(np.frombuffer(b"".join(og2.g2_affine_bytes(p) for p in pts), dtype=np.uint8).copy()).cuda()
    out = device.g2_serialize(imgs, True).cpu().numpy()
    assert [bytes(r) for r in out] == [o.encode(p, True) for p in pts]
    assert len({bool(r[-1] & 0x80) for r in out}) == 2


def test_mainnet_fixtures():
    from snarkvm_b200 import device
    from snarkvm_b200 import varuna as dv
    beta_h, neg = _read("beta_h.usrs"), _read("neg_powers_of_beta.usrs")
    pts = [beta_h] + [p for _d, p in dv._u64_map(neg, 192, "negative powers")]
    raw = torch.from_numpy(np.frombuffer(b"".join(pts), dtype=np.uint8).copy()).cuda()
    images, status = device.g2_deserialize(raw, False, True)
    assert (status.cpu().numpy() == device.G1_VALID).all()
    assert device.g2_serialize(images, False).cpu().numpy().tobytes() == b"".join(pts)
    assert (device.g2_validate(images).cpu().numpy() == device.G1_VALID).all()
    comp = device.g2_serialize(images, True)
    assert [bytes(r) for r in comp.cpu().numpy()] == [o.encode(o.decode(b, False, False)[1], True) for b in pts]
    back, st = device.g2_deserialize(comp.reshape(-1).contiguous(), True, True)
    assert (st.cpu().numpy() == device.G1_VALID).all() and torch.equal(back, images)
    # the prepared points of a validated load equal today's unchecked load
    gamma = _read("powers_of_beta_gamma.usrs")
    plain = dv.UniversalVerifier.from_mainnet(beta_h, neg, gamma)
    checked = dv.UniversalVerifier.from_mainnet(beta_h, neg, gamma, validate=True)
    assert torch.equal(plain.prepared, checked.prepared) and plain.neg_index == checked.neg_index
    assert dv.UniversalVerifier.from_usrs(beta_h, validate=True).beta_h.tobytes() == plain.beta_h.tobytes()


def _replace_neg_power(blob, index, point_bytes):
    off = 8 + index * 200 + 8
    return blob[:off] + point_bytes + blob[off + 192:]


def test_mainnet_validation_names_the_entry():
    from snarkvm_b200 import varuna as dv
    beta_h, neg, gamma = _read("beta_h.usrs"), _read("neg_powers_of_beta.usrs"), _read("powers_of_beta_gamma.usrs")
    entries = dv._u64_map(neg, 192, "negative powers")
    x = (3, 0)
    while o.fq2_sqrt(o.rhs(x)) is None:
        x = (x[0] + 1, 0)
    off_sub = o.encode((x, o.fq2_sqrt(o.rhs(x))), False)
    g = o.decode(beta_h, False, False)[1]
    off_curve = o.encode((g[0], (g[1][0], (g[1][1] + 1) % Q)), False)
    d5 = entries[5][0]
    for bad, reason in ((off_curve, "not on the curve"), (off_sub, "not in the prime-order subgroup")):
        with pytest.raises(ValueError, match=rf"β·H: {reason}"):
            dv.UniversalVerifier.from_mainnet(bad, neg, gamma, validate=True)
        with pytest.raises(ValueError, match=rf"β·H: {reason}"):
            dv.UniversalVerifier.from_usrs(bad, validate=True)
        with pytest.raises(ValueError, match=rf"the negative power for bound {d5}: {reason}"):
            dv.UniversalVerifier.from_mainnet(beta_h, _replace_neg_power(neg, 5, bad), gamma, validate=True)
        # without validation the load behaves as before: it takes the point
        v = dv.UniversalVerifier.from_mainnet(beta_h, _replace_neg_power(neg, 5, bad), gamma)
        assert v.neg_index[d5] == 2 + 5


def _same_verifier(a, b):
    return (a.g.tobytes() == b.g.tobytes() and a.gamma_g.tobytes() == b.gamma_g.tobytes() and a.h.tobytes() == b.h.tobytes()
            and a.beta_h.tobytes() == b.beta_h.tobytes() and torch.equal(a.prepared, b.prepared) and a.neg_index == b.neg_index)


def test_verifier_key_round_trip_and_verdicts():
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import synthetic_srs
    import test_varuna_verify_gpu as tv
    # the mainnet verifier: bytes equal the oracle's, and both forms round-trip
    beta_h, neg, gamma = _read("beta_h.usrs"), _read("neg_powers_of_beta.usrs"), _read("powers_of_beta_gamma.usrs")
    main = dv.UniversalVerifier.from_mainnet(beta_h, neg, gamma)
    gamma_pt = vb.decode_g1(gamma[16:112], False, False)[1]
    for compressed in (True, False):
        blob = main.to_bytes(compressed)
        assert len(blob) == (288 if compressed else 576)
        assert blob == o.verifier_key_bytes(py.G1_GENERATOR, gamma_pt, o.G2_GEN, o.decode(beta_h, False, False)[1], compressed)
        back = dv.UniversalVerifier.from_bytes(blob, compressed, neg_powers=dv.parse_neg_powers(neg))
        assert _same_verifier(back, main) and back.to_bytes(compressed) == blob
    with pytest.raises(ValueError, match="holds no γ·G"):
        dv.UniversalVerifier.from_usrs(beta_h).to_bytes()
    # a flipped x bit of β·h: the field is named
    blob = main.to_bytes()
    bad = bytearray(blob)
    bad[2 * 48 + 96] ^= 0x01
    with pytest.raises(ValueError, match="beta_h: "):
        dv.UniversalVerifier.from_bytes(bytes(bad))
    # a synthetic verifier with γ and negative powers: the rebuilt one gives the same verdicts
    program, kti, D = tv._program("one", False)
    verifier = tv._verifier(D)
    blob = verifier.to_bytes()
    neg_imgs = {d: np.frombuffer(og2.g2_affine_bytes(og2.g2_mul(o.G2_GEN, pow(tv.BETA, -(D - d), R))), dtype=np.uint8)
                for d in tv._bounds(D)}
    rebuilt = dv.UniversalVerifier.from_bytes(blob, neg_powers=neg_imgs)
    assert _same_verifier(rebuilt, verifier)
    assert dv.UniversalVerifier.from_bytes(verifier.to_bytes(False), False, neg_powers=neg_imgs).to_bytes() == blob
    proof = dv.prove_batch(program, False)
    tampered = copy.deepcopy(proof)
    tampered.evaluations.g_1_eval = (tampered.evaluations.g_1_eval + 1) % R
    for v in (verifier, rebuilt):
        assert dv.verify_batch_many(v, [(kti, proof), (kti, tampered)], False) == [True, False]
    # certificates under verify_vk
    rng = random.Random(3)
    circuits = [dv.test_circuit_csr(rng.randrange(2, R), rng.randrange(2, R), 2, 64, 60, "cuda")[0]]
    powers, gpowers = synthetic_srs(8191, tv.BETA, tv.GAMMA)
    (pk, vk), = dv.batch_circuit_setup(circuits, powers, gpowers, with_id=True)
    cert = dv.prove_vk_batch([pk])[0]
    cb = bytearray(cert.to_bytes())
    cb[8 + 47] ^= 0x80                                            # −w
    bad_cert = dv.Certificate.from_bytes(bytes(cb))
    for v in (verifier, rebuilt):
        assert [r.valid for r in dv.verify_vk_batch(circuits * 2, [vk, vk], [cert, bad_cert], verifier=v)] == [True, False]
