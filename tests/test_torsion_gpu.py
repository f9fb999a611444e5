"""GPU: the point readers' device functions on the torsion and square-root corpora of torsion_corpus.py.

g1_validate (k_g1_validate) on every G1 corpus image, at strides 104 and 136, gives the oracle's statuses: small-order points and
their −T, φ(T), T + S are refused, whatever branch the chain takes.  g1_deserialize in the compressed (both flags), uncompressed and
97-byte forms, with and without validation, equals varuna_bytes_oracle / varuna_pk_bytes_oracle in status and image, and
g1_serialize inverts it (y = 0 under PositiveY, y = (q ± 1)/2).  snarkvm_b200_test_sqrt_device runs the decoders' fq_sqrt and
fq2_sqrt element-wise: the ok flag is Euler's criterion (of the norm for Fq2), each root is canonical, squares back and is the root
the Python restatement predicts, so every depth, the long loops and every fq2_sqrt branch run on the device.  g2_deserialize of x
with a real x³ + B' and g2_validate of T2 + S2 equal g2_bytes_oracle.  Each reader refuses a torsion point, or one plus a subgroup
point, with a ValueError naming the blob and field and "not in the prime-order subgroup"."""
import copy
import os
import random

import numpy as np
import pytest
import torch

import g2_bytes_oracle as o2
import torsion_corpus as tc
import varuna_bytes_oracle as vb
import varuna_pk_bytes_oracle as vpk
from oracle import bls12_377 as py
from oracle import g2 as og2

pytestmark = pytest.mark.gpu
Q, R = tc.Q, tc.R
FIELD_FQ, FIELD_FQ2 = 1, 2                                       # SNARKVM_B200_FIELD_FQ / FQ2
HERE = os.path.dirname(os.path.abspath(__file__))
REFUSED = "not in the prime-order subgroup"


def _read(*path):
    with open(os.path.join(HERE, "golden", *path), "rb") as f:
        return f.read()


def _cuda(data: bytes) -> torch.Tensor:
    return torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).cuda()


def _x_bytes(x, flags=0):
    b = bytearray(x.to_bytes(48, "little"))
    b[47] |= flags
    return bytes(b)


@pytest.fixture(scope="module")
def entries():
    return tc.g1_entries()


def test_g1_validate_on_torsion(entries):
    from snarkvm_b200 import device
    want = [d for _n, _p, d, _f, _e in entries]
    assert want == [f for _n, _p, _d, f, _e in entries]
    pts = _cuda(b"".join(py.affine_bytes(p) for _n, p, _d, _f, _e in entries)).reshape(-1, 104)
    got = device.g1_validate(pts).cpu().tolist()
    assert got == want, [n for (n, *_r), g, w in zip(entries, got, want) if g != w]
    wide = torch.zeros((pts.shape[0], 136), dtype=torch.uint8, device="cuda")
    wide[:, :104] = pts
    assert device.g1_validate(wide, stride=136).cpu().tolist() == want


def _blobs(entries, form):
    """every corpus point in `form`: compressed x under both flags (points on the curve), uncompressed and 97-byte as they are"""
    out = []
    for _n, p, _d, _f, _e in entries:
        if form == "compressed":
            if p is not None and py.g1_is_on_curve(p):
                out += [_x_bytes(p[0]), _x_bytes(p[0], vb.POSITIVE_Y)]
        elif form == "uncompressed":
            out.append(vb.encode_g1(p, False))
        elif p is not None:
            out.append(vpk.encode_point97((p[0], p[1], False)))
    return out


def _image97(b, validate):
    s, p = vpk.decode_point97(b, validate)
    if p is None:
        return s, bytes(104)
    x, y, inf = p
    return s, py.fq_to_mont(x).to_bytes(48, "little") + py.fq_to_mont(y).to_bytes(48, "little") + bytes([int(inf)]) + bytes(7)


@pytest.mark.parametrize("form", ["compressed", "uncompressed", "to_bytes"])
@pytest.mark.parametrize("validate", [False, True], ids=["unchecked", "validated"])
def test_g1_deserialize_on_torsion(entries, form, validate):
    from snarkvm_b200 import device
    blobs = _blobs(entries, form)
    mode = {"compressed": True, "uncompressed": False, "to_bytes": device.G1_TO_BYTES}[form]
    images, status = device.g1_deserialize(_cuda(b"".join(blobs)), mode, validate)
    images, status = images.cpu().numpy(), status.cpu().tolist()
    want = [_image97(b, validate) if form == "to_bytes" else vb.image(b, form == "compressed", validate) for b in blobs]
    assert status == [s for s, _i in want]
    for k, (_s, img) in enumerate(want):
        assert images[k].tobytes() == img, k
    if validate:
        assert vb.NOT_IN_SUBGROUP in status and (form == "compressed" or vb.NOT_ON_CURVE in status)


def test_g1_serialize_inverts_on_torsion(entries):
    from snarkvm_b200 import device
    blobs = _blobs(entries, "compressed")
    images, status = device.g1_deserialize(_cuda(b"".join(blobs)), True, False)
    assert (status == 0).all()
    points = [vb.decode_g1(b, True, False)[1] for b in blobs]
    order2 = {(Q - 1, 0), ((-tc.PHI) % Q, 0), ((-tc.PHI * tc.PHI) % Q, 0)}
    assert {p for p in points if p[1] == 0} == order2                     # y = 0, each under both flags
    assert {b for b in blobs if b[47] & vb.POSITIVE_Y and vb.decode_g1(b, True, False)[1] in order2}
    rng = random.Random(5)
    extra = [(rng.randrange(Q), (Q - 1) // 2), (rng.randrange(Q), (Q + 1) // 2), (0, (Q + 1) // 2)]
    proj = _cuda(b"".join(py.projective_bytes_normalised(p) for p in points + extra)).view(torch.int64).reshape(-1, 18)
    for mode in (True, False):
        out = device.g1_serialize(proj, mode).cpu().numpy()
        assert [r.tobytes() for r in out] == [vb.encode_g1(p, mode) for p in points + extra]
        back, st = device.g1_deserialize(_cuda(out[:len(points)].tobytes()), mode, False)
        assert (st == 0).all() and torch.equal(back, images)
    flags = [vb.encode_g1(p, True)[47] & 0xC0 for p in extra]
    assert flags == [0, vb.POSITIVE_Y, vb.POSITIVE_Y]


def _device_sqrt(field, vals):
    from snarkvm_b200 import _lib
    if field == FIELD_FQ:
        data = b"".join(py.fq_to_mont(a).to_bytes(48, "little") for a in vals)
    else:
        data = b"".join(py.fq_to_mont(c).to_bytes(48, "little") for a in vals for c in a)
    inp = _cuda(data)
    out = torch.zeros_like(inp)
    ok = torch.full((len(vals),), -1, dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib().snarkvm_b200_test_sqrt_device(field, out.data_ptr(), ok.data_ptr(), inp.data_ptr(), len(vals),
                                                        torch.cuda.current_stream().cuda_stream))
    raw = out.cpu().numpy().tobytes()
    imgs = [int.from_bytes(raw[48 * i: 48 * i + 48], "little") for i in range(len(raw) // 48)]
    return imgs, ok.cpu().tolist()


def test_fq_sqrt_on_every_depth():
    vals = tc.fq_values()
    imgs, ok = _device_sqrt(FIELD_FQ, vals)
    assert ok == [int(tc.is_square(a)) for a in vals]
    for a, img, good in zip(vals, imgs, ok):
        assert img < Q, a                                         # canonical image
        root = py.fq_from_mont(img)
        if good:
            assert root * root % Q == a % Q and root == tc.fq_sqrt_trace(a)[0], a
        else:
            assert img == 0


def test_fq2_sqrt_on_every_branch():
    vals = tc.fq2_values()
    imgs, ok = _device_sqrt(FIELD_FQ2, vals)
    assert ok == [int(tc.fq2_is_square(a)) for a in vals]
    branches = set()
    for k, (a, good) in enumerate(zip(vals, ok)):
        c = (imgs[2 * k], imgs[2 * k + 1])
        assert c[0] < Q and c[1] < Q, a
        root = (py.fq_from_mont(c[0]), py.fq_from_mont(c[1]))
        want, branch = tc.fq2_sqrt_trace(a)
        branches.add(branch)
        if good:
            assert og2.f2_sqr(root) == (a[0] % Q, a[1] % Q) and root == want, (a, branch)
        else:
            assert c == (0, 0)
    assert {"a1 = 0, real", "a1 = 0, imaginary", "(a0 + n)/2", "(a0 − n)/2"} <= branches


@pytest.mark.parametrize("validate", [False, True], ids=["unchecked", "validated"])
def test_g2_deserialize_real_rhs(validate):
    from snarkvm_b200 import device
    blobs = [_x_bytes(x[0]) + _x_bytes(x[1], f) for x, _a0 in tc.g2_real_rhs_x() for f in (0, o2.POSITIVE_Y)]
    images, status = device.g2_deserialize(_cuda(b"".join(blobs)), True, validate)
    images, status = images.cpu().numpy(), status.cpu().tolist()
    want = [o2.image(b, True, validate) for b in blobs]
    assert status == [s for s, _i in want]
    for k, (_s, img) in enumerate(want):
        assert images[k].tobytes() == img, k
    # the real root (y.c1 = 0) and the imaginary one (y.c0 = 0) both occur, under both signs
    ys = [o2.decode(b, True, False)[1][1] for b in blobs]
    assert any(y[1] == 0 and y[0] for y in ys) and any(y[0] == 0 and y[1] for y in ys)


def test_g2_validate_and_decode_mixed_points():
    from snarkvm_b200 import device
    pts = tc.g2_mixed_points()
    imgs = b"".join(og2.g2_affine_bytes(p) for _n, p in pts)
    got = device.g2_validate(_cuda(imgs).reshape(-1, 200)).cpu().tolist()
    assert got == [o2.check(p) for _n, p in pts] == [o2.NOT_IN_SUBGROUP] * len(pts)
    for compressed in (True, False):
        blobs = [o2.encode(p, compressed) for _n, p in pts]
        images, status = device.g2_deserialize(_cuda(b"".join(blobs)), compressed, True)
        want = [o2.image(b, compressed, True) for b in blobs]
        assert status.cpu().tolist() == [s for s, _i in want]
        assert [r.tobytes() for r in images.cpu().numpy()] == [i for _s, i in want]


@pytest.fixture(scope="module")
def bad_points():
    """(name, point) outside the subgroup: a point of order 2^46 and one of order 7 plus a subgroup point"""
    tor = {name: t for name, t, _n in tc.g1_torsion()}
    s = py.g1_mul(py.G1_GENERATOR, 0xC0FFEE)
    return [("T", tor["order 2^46"]), ("T + S", py.g1_add(tor["order 7, line 3"], s))]


def test_proofs_and_certificates_refuse_torsion(bad_points):
    from snarkvm_b200 import varuna as dv
    blob = _read("varuna_bytes", "genesis_proof_0.bin")
    K = int.from_bytes(blob[:8], "little")
    at = 8 + 8 * K                                                # the first witness commitment
    good_cert = vb.write_batch_lc([(py.G1_GENERATOR, None)])
    for _name, p in bad_points:
        bad = blob[:at] + vb.encode_g1(p, True) + blob[at + 48:]
        with pytest.raises(ValueError, match=rf"blob 1: witness_commitments\[0\]: {REFUSED}"):
            dv.proofs_from_bytes([blob, bad])
        assert len(dv.proofs_from_bytes([bad], validate=False)) == 1
        with pytest.raises(ValueError, match=rf"blob 1: pc_proof\[0\]\.w: {REFUSED}"):
            dv.certificates_from_bytes([good_cert, vb.write_batch_lc([(p, None)])])
        with pytest.raises(ValueError, match=rf"blob 0: pc_proof\[0\]\.w: {REFUSED}"):
            dv.certificates_from_bytes([vb.write_batch_lc([(p, None)], False)], False)


def test_proving_keys_refuse_torsion(bad_points):
    import test_varuna_pk_bytes_gpu as tpk
    from snarkvm_b200 import varuna as dv
    _n, _zk, pks, _a, _d, blobs = tpk._keyed("one", False)
    blob = blobs[0]
    first = len(blob) - len(pks[0].committer_key.to_bytes()) + 4
    for _name, p in bad_points:
        at = first + 97                                           # powers_of_beta_g[1]
        bad = blob[:at] + vpk.encode_point97((p[0], p[1], False)) + blob[at + 97:]
        with pytest.raises(ValueError, match=rf"blob 1: committer_key\.powers_of_beta_g\[1\]: {REFUSED}"):
            dv.proving_keys_from_bytes([blob, bad])


def test_universal_verifier_refuses_torsion(bad_points):
    from snarkvm_b200 import varuna as dv
    beta_h, neg, gamma = _read("beta_h.usrs"), _read("neg_powers_of_beta.usrs"), _read("powers_of_beta_gamma.usrs")
    main = dv.UniversalVerifier.from_mainnet(beta_h, neg, gamma)
    for compressed in (True, False):
        blob = main.to_bytes(compressed)
        size = 48 if compressed else 96
        for _name, p in bad_points:
            bad = blob[:size] + vb.encode_g1(p, compressed) + blob[2 * size:]
            with pytest.raises(ValueError, match=rf"gamma_g: {REFUSED}"):
                dv.UniversalVerifier.from_bytes(bad, compressed, neg_powers=dv.parse_neg_powers(neg))
    for _name, p in bad_points:
        bad = gamma[:16] + vb.encode_g1(p, False) + gamma[112:]       # key 0 of powers-of-beta-gamma: γ·G
        with pytest.raises(ValueError, match=rf"γ·G: {REFUSED}"):
            dv.UniversalVerifier.from_mainnet(beta_h, neg, bad, validate=True)


def _refused(call, *words):
    with pytest.raises(ValueError) as e:
        call()
    for w in words + (REFUSED,):
        assert w in str(e.value), (w, str(e.value))


def test_verify_batch_many_refuses_torsion(bad_points):
    import test_varuna_verify_gpu as tv
    from snarkvm_b200 import varuna as dv
    program, kti, D = tv._program("one", False)
    proof = dv.prove_batch(program, False)
    verifier = tv._verifier(D)
    for _name, p in bad_points:
        img = np.frombuffer(py.projective_bytes_normalised(p), dtype=np.uint64).copy()
        bad = copy.deepcopy(proof)
        bad.commitments.h_1 = img
        _refused(lambda: dv.verify_batch_many(verifier, [(kti, proof), (kti, bad)], False), "proof 1", "h_1")
        bad = copy.deepcopy(proof)
        bad.pc_proof[0] = (img, bad.pc_proof[0][1])
        _refused(lambda: dv.verify_batch_many(verifier, [(kti, bad)], False), "proof 0", "pc_proof[0].w")
