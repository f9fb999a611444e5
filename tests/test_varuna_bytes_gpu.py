"""GPU: G1 points, Varuna proofs, verifying keys and certificates from and to their bytes.

device.g1_deserialize (k_g1_deserialize) against the big-integer restatement (varuna_bytes_oracle) on a corpus of subgroup points
of both signs, x = 0, x = −1 (the order-2 point), non-residue x, coordinates at q and above, both flags, infinity with a nonzero x,
on-curve points off the subgroup and random squares whose Tonelli–Shanks runs its longest first round, compressed and uncompressed,
with and without validation; device.g1_serialize inverts it.  The mainnet verifying keys and the genesis proofs parse with
validation, in one batch and one by one, and re-serialise to their bytes.  prove_batch's proofs (synthetic and mainnet SRS, both
modes, one and three circuits) and prove_vk_batch's certificates round-trip in every compress / validate mode, their compressed
bytes equal the oracle's, the decoded objects verify, a flipped sign bit decodes to the negation and fails verification, and a
flipped x bit is refused naming the blob and the field."""
import glob
import os
import random

import numpy as np
import pytest
import torch

import varuna_bytes_oracle as vb
from oracle import bls12_377 as py

pytestmark = pytest.mark.gpu
Q, R = vb.Q, vb.R
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "varuna_bytes")
KEYS = sorted(os.path.basename(f)[: -len(".verifier")] for f in glob.glob(os.path.join(GOLDEN, "*.verifier")))


def _read(name):
    with open(os.path.join(GOLDEN, name), "rb") as f:
        return f.read()


def _x_bytes(x, flags=0):
    b = bytearray(x.to_bytes(48, "little"))
    b[47] |= flags
    return bytes(b)


def _points(rng):
    """(subgroup points, on-curve points off the subgroup, residue x, non-residue x)"""
    sub = [py.g1_mul(py.G1_GENERATOR, rng.randrange(1, R)) for _ in range(16)]
    off, squares, non = [], [], []
    while len(squares) < 400 or len(non) < 8:
        x = rng.randrange(Q)
        y, _k = vb.sqrt(x ** 3 + 1)
        (squares if y is not None else non).append(x)
    for x in squares[:8]:
        p = (x, vb.sqrt(x ** 3 + 1)[0])
        assert not vb.in_subgroup(p)
        off.append(p)
    return sub, off, squares, non[:8]


@pytest.fixture(scope="module")
def corpus():
    rng = random.Random(0xB17E5)
    sub, off, squares, non = _points(rng)
    comp = []
    for p in sub + off:
        comp += [vb.encode_g1(p, True), vb.encode_g1((p[0], Q - p[1]), True)]
    comp += [_x_bytes(0), _x_bytes(0, 0x80), _x_bytes(Q - 1), _x_bytes(Q - 1, 0x80)]          # (0, ±1), (−1, 0) under both flags
    comp += [_x_bytes(x, f) for x in non for f in (0, 0x80)]
    comp += [_x_bytes(v, f) for v in (Q, Q + 1, (1 << 377) - 1, 1 << 377, (1 << 382) - 1) for f in (0, 0x80, 0x40)]
    comp += [_x_bytes(v, 0xC0) for v in (0, 5, Q - 1)]
    comp += [_x_bytes(v, 0x40) for v in (1, 12345, Q - 1)]                                    # infinity with x ≠ 0
    comp += [_x_bytes(x, 0x80 * (k & 1)) for k, x in enumerate(squares)]
    firsts = [vb.sqrt(x ** 3 + 1)[1] for x in squares]
    assert max(firsts) == vb.TWO_ADICITY - 1                                                 # the longest first round ran
    unc = []
    for p in sub + off + [(0, 1), (Q - 1, 0)]:
        unc.append(vb.encode_g1(p, False))
    x, y = sub[0]
    unc += [vb.encode_g1((x, (y + 1) % Q), False)]                                            # off the curve
    unc += [x.to_bytes(48, "little") + _x_bytes(v, f) for v in (Q, 1 << 377) for f in (0, 0x40)]
    unc += [_x_bytes(x, 0x80) + y.to_bytes(48, "little"), _x_bytes(Q) + y.to_bytes(48, "little")]
    unc += [x.to_bytes(48, "little") + _x_bytes(y, 0xC0), _x_bytes(7) + _x_bytes(9, 0x40), _x_bytes(x) + _x_bytes(y, 0x80)]
    return comp, unc


def _decode(blobs, compressed, validate):
    from snarkvm_b200 import device
    raw = torch.from_numpy(np.frombuffer(b"".join(blobs), dtype=np.uint8).copy()).cuda()
    images, status = device.g1_deserialize(raw, compressed, validate)
    return images.cpu().numpy(), status.cpu().numpy()


@pytest.mark.parametrize("compressed", [True, False], ids=["compressed", "uncompressed"])
@pytest.mark.parametrize("validate", [False, True], ids=["unchecked", "validated"])
def test_deserialize_equals_the_oracle(corpus, compressed, validate):
    blobs = corpus[0] if compressed else corpus[1]
    images, status = _decode(blobs, compressed, validate)
    want = [vb.image(b, compressed, validate) for b in blobs]
    assert status.tolist() == [s for s, _i in want]
    for k, (_s, img) in enumerate(want):
        assert images[k].tobytes() == img, k
    seen = set(status.tolist())
    assert {vb.VALID, vb.NOT_CANONICAL, vb.BAD_FLAGS} <= seen
    if compressed or validate:
        assert vb.NOT_ON_CURVE in seen
    if validate:
        assert vb.NOT_IN_SUBGROUP in seen
    if compressed:                                     # the order-2 point (−1, 0): accepted unchecked, off the subgroup checked
        k = blobs.index(_x_bytes(Q - 1))
        assert status[k] == (vb.NOT_IN_SUBGROUP if validate else vb.VALID) == status[k + 1]


@pytest.mark.parametrize("compressed", [True, False], ids=["compressed", "uncompressed"])
def test_serialize_inverts_deserialize(corpus, compressed):
    from snarkvm_b200 import device
    blobs = corpus[0] if compressed else corpus[1]
    images, status = _decode(blobs, compressed, False)
    ok = np.nonzero(status == vb.VALID)[0]
    proj = np.zeros((ok.size, 18), dtype=np.uint64)
    proj[:, :12] = images[ok, :96].copy().view(np.uint64)
    one = np.frombuffer(((1 << 384) % Q).to_bytes(48, "little"), dtype=np.uint64)
    inf = images[ok, 96] != 0
    proj[~inf, 12:] = one
    proj[inf, :12] = 0
    proj[inf, 6:12] = one
    for mode in (True, False):
        out = device.g1_serialize(torch.from_numpy(proj.view(np.int64)).cuda(), mode).cpu().numpy()
        for row, k in zip(out, ok):
            _s, p = vb.decode_g1(blobs[k], compressed, False)
            assert row.tobytes() == vb.encode_g1(p, mode), k
        back, st = _decode([r.tobytes() for r in out], mode, False)
        # compressed bytes keep x and a sign only: a point off the curve (accepted unchecked from 96 bytes) comes back on it
        keep = [not mode or vb.decode_g1(blobs[k], compressed, True)[0] != vb.NOT_ON_CURVE for k in ok]
        assert (st == 0).all() and (back[keep] == images[ok][keep]).all()


def test_mainnet_keys_and_genesis_proofs():
    from snarkvm_b200 import varuna as dv
    blobs = [_read(f"{n}.verifier")[1:] for n in KEYS]
    vks = dv.verifying_keys_from_bytes(blobs)
    for blob, vk in zip(blobs, vks):
        ref = vb.read_verifying_key(vb.Reader(blob, 0, compressed=True))
        one = dv.CircuitVerifyingKey.from_bytes(blob)
        assert vk.id == one.id == ref["id"] and vk.circuit_info == one.circuit_info
        assert list(vk.circuit_info.to_bytes_le()) == list(blob[:48])
        assert (vk.circuit_commitments == one.circuit_commitments).all()
        assert [py.projective_from_bytes(c.tobytes()) for c in vk.circuit_commitments] == ref["commitments"]
        assert vk.to_bytes() == blob[:664]
        d = dv._KeyDomains(vk.circuit_info)
        assert d.constraint_domain.size >= vk.circuit_info.num_constraints
    proofs = [_read(f"genesis_proof_{k}.bin") for k in range(8)]
    got = dv.proofs_from_bytes(proofs)
    assert dv.proofs_to_bytes(got) == proofs
    for blob, p in zip(proofs, got):
        q, end = dv.Proof.read(blob + b"trailing")
        assert end == len(blob) and _same_proof(p, q)
        assert q.to_bytes() == blob
    # every point of every key and proof passes Affine::check
    pts = [blob[56 + 48 * i: 104 + 48 * i] for blob in blobs for i in range(12)]
    assert (_decode(pts, True, True)[1] == 0).all()


def _same_proof(a, b):
    from snarkvm_b200.algorithms import _fr_mont_to_int
    ca, cb = a.commitments, b.commitments
    eq = lambda x, y: (np.asarray(x, dtype=np.uint64) == np.asarray(y, dtype=np.uint64)).all()   # noqa: E731
    same = (list(a.batch_sizes) == list(b.batch_sizes) and len(ca.witness_commitments) == len(cb.witness_commitments)
            and all(eq(x, y) for x, y in zip(ca.witness_commitments, cb.witness_commitments))
            and (ca.mask_poly is None) == (cb.mask_poly is None) and (ca.mask_poly is None or eq(ca.mask_poly, cb.mask_poly))
            and all(eq(getattr(ca, n), getattr(cb, n)) for n in ("h_0", "g_1", "h_1", "h_2"))
            and all(eq(x, y) for m in "abc" for x, y in zip(getattr(ca, f"g_{m}_commitments"), getattr(cb, f"g_{m}_commitments")))
            and a.evaluations.to_field_elements() == b.evaluations.to_field_elements()
            and [[list(t) for t in s] for s in a.third_sums] == [[list(t) for t in s] for s in b.third_sums]
            and [list(t) for t in a.fourth_sums] == [list(t) for t in b.fourth_sums] and len(a.pc_proof) == len(b.pc_proof))
    for (wa, va), (wb, vbb) in zip(a.pc_proof, b.pc_proof):
        same = same and eq(wa, wb) and (None if va is None else _fr_mont_to_int(va)) == (None if vbb is None else _fr_mont_to_int(vbb))
    return bool(same)


def _point(limbs):
    return py.projective_from_bytes(np.asarray(limbs, dtype=np.uint64).tobytes())


def _oracle_proof(p) -> dict:
    from snarkvm_b200.algorithms import _fr_mont_to_int
    c, e = p.commitments, p.evaluations
    return {"batch_sizes": list(p.batch_sizes), "w": [_point(w) for w in c.witness_commitments],
            "mask_poly": None if c.mask_poly is None else _point(c.mask_poly),
            **{n: _point(getattr(c, n)) for n in ("h_0", "g_1", "h_1", "h_2")},
            **{f"g_{m}": [_point(x) for x in getattr(c, f"g_{m}_commitments")] for m in "abc"},
            "g_1_eval": e.g_1_eval, "g_a_evals": list(e.g_a_evals), "g_b_evals": list(e.g_b_evals), "g_c_evals": list(e.g_c_evals),
            "third_sums": p.third_sums, "fourth_sums": p.fourth_sums,
            "pc_proof": [(_point(w), None if v is None else _fr_mont_to_int(v)) for w, v in p.pc_proof]}


def _flip(blob, off, mask):
    b = bytearray(blob)
    b[off] ^= mask
    return bytes(b)


def _mainnet_program(name, zk):
    """the committer keys test_varuna_verify_gpu.test_mainnet_srs builds from the mainnet powers"""
    import test_varuna_verify_gpu as tv
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import CommitterKey
    powers, shifted, gammas = tv._mainnet_srs()
    gamma_dense = torch.from_numpy(np.stack([gammas[i] for i in range(3)])).cuda()
    program, kti, _D = tv._program(name, zk, (powers, gamma_dense))
    top, keyed = shifted.shape[0], []
    for pk, zs in program:
        bounds = sorted(set(pk.circuit.info.degree_bounds()))
        ck = CommitterKey(pk.committer_key.powers_of_beta_g, gamma_dense, {}, shifted[top - 1 - bounds[-1]:],
                          {d: torch.from_numpy(np.stack([gammas[tv.MAINNET_D - d + i] for i in range(3)])).cuda() for d in bounds},
                          bounds, tv.MAINNET_D)
        keyed.append((dv.CircuitProvingKey(pk.circuit_verifying_key, pk.circuit, ck), zs))
    return keyed, kti, tv._mainnet_verifier()


@pytest.mark.parametrize("setup", ["synthetic", "mainnet"])
@pytest.mark.parametrize("name", ["one", "three"])
@pytest.mark.parametrize("zk", [False, True], ids=["plain", "zk"])
def test_generated_proofs_round_trip(setup, name, zk):
    import test_varuna_verify_gpu as tv
    from snarkvm_b200 import varuna as dv
    if setup == "synthetic":
        program, kti, D = tv._program(name, zk)
        verifier = tv._verifier(D)
    else:
        program, kti, verifier = _mainnet_program(name, zk)
    proof = dv.prove_batch(program, zk, random.Random(11) if zk else None)
    for compress in (True, False):
        blob = proof.to_bytes(compress)
        for validate in (True, False):
            assert _same_proof(dv.Proof.from_bytes(blob, compress, validate), proof), (compress, validate)
    blob = proof.to_bytes()
    assert blob == vb.write_proof(_oracle_proof(proof))
    back = dv.Proof.from_bytes(blob)
    assert dv.verify_batch(verifier, kti, back, zk) is True
    # h_0, g_1, h_1 follow the batch sizes, the witness commitments and the mask; take the first that is not infinity
    K, total = len(proof.batch_sizes), sum(proof.batch_sizes)
    name, at = next((n, 8 + 8 * K + 48 * total + 1 + (48 if zk else 0) + 48 * j) for j, n in enumerate(("h_0", "g_1", "h_1"))
                    if np.asarray(getattr(proof.commitments, n))[12:].any())
    neg = dv.Proof.from_bytes(_flip(blob, at + 47, 0x80))
    a, b = (np.asarray(getattr(p.commitments, name), dtype=np.uint64) for p in (back, neg))
    assert int.from_bytes(b[6:12].tobytes(), "little") == Q - int.from_bytes(a[6:12].tobytes(), "little") and (a[:6] == b[:6]).all()
    assert dv.verify_batch(verifier, kti, neg, zk) is False
    with pytest.raises(ValueError, match=rf"blob 1: {name}: "):
        dv.proofs_from_bytes([blob, _flip(blob, at, 0x01)])


def test_certificates_round_trip():
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import synthetic_srs
    import test_varuna_verify_gpu as tv
    rng = random.Random(3)
    circuits = [dv.test_circuit_csr(rng.randrange(2, R), rng.randrange(2, R), 2 + k, 64 * (k + 1), 60 * (k + 1), "cuda")[0]
                for k in range(3)]
    powers, gamma = synthetic_srs(8191, tv.BETA, tv.GAMMA)
    setups = dv.batch_circuit_setup(circuits, powers, gamma, with_id=True)
    pks, vks = [s[0] for s in setups], [s[1] for s in setups]
    certs = dv.prove_vk_batch(pks)
    verifier = dv.UniversalVerifier.synthetic(tv.BETA)
    for compress in (True, False):
        for validate in (True, False):
            vk2 = dv.verifying_keys_from_bytes([vk.to_bytes(compress) for vk in vks], compress, validate)
            c2 = dv.certificates_from_bytes([c.to_bytes(compress) for c in certs], compress, validate)
            assert all((a.circuit_commitments == b.circuit_commitments).all() and a.circuit_info == b.circuit_info and a.id == b.id
                       for a, b in zip(vks, vk2))
            assert all((a.w == b.w).all() for a, b in zip(certs, c2))
    blobs = [c.to_bytes() for c in certs]
    assert blobs == [vb.write_batch_lc([(_point(c.w), None)]) for c in certs]
    vk_blobs = [vk.to_bytes() for vk in vks]
    assert vk_blobs == [vb.write_verifying_key({"info": _info_counts(vk), "commitments": [_point(x) for x in vk.circuit_commitments],
                                                "id": vk.id}) for vk in vks]
    back = dv.certificates_from_bytes(blobs)
    res = dv.verify_vk_batch(circuits, dv.verifying_keys_from_bytes(vk_blobs), back, verifier=verifier)
    assert all(r.matches and r.valid is True for r in res)
    w_at = 8
    neg = dv.certificates_from_bytes([_flip(b, w_at + 47, 0x80) for b in blobs])
    assert [r.valid for r in dv.verify_vk_batch(circuits, vks, neg, verifier=verifier)] == [False] * 3
    with pytest.raises(ValueError, match=r"blob 2: pc_proof\[0\]\.w: "):
        dv.certificates_from_bytes(blobs[:2] + [_flip(blobs[2], w_at, 0x01)])


def _info_counts(vk):
    i = vk.circuit_info
    return [i.num_public_inputs, i.num_public_and_private_variables, i.num_constraints, i.num_non_zero_a, i.num_non_zero_b,
            i.num_non_zero_c]
