"""GPU: the byte form of Varuna proving keys — varuna.proving_keys_to_bytes / proving_keys_from_bytes, CircuitProvingKey and
sonic_pc.CommitterKey to_bytes / read — against the big-integer restatement (varuna_pk_bytes_oracle).

The 97-byte ToBytes form of k_g1_deserialize / k_g1_serialize and k_fr_records match the oracle on corpora of edge cases, with and
without validation.  Keys from batch_circuit_setup (one circuit, three of different R, C and K; both modes) write the oracle's
bytes and read back to equal CSR arrays, evaluations, committer-key images and verifying keys, with the circuit id of a fresh
csr_serialize.  Loaded keys prove byte-identically (non-hiding) and their hiding proofs verify.  A committer key trimmed from the
mainnet 2^15 powers round-trips and holds the .usrs points.  Many keys per call equal one-by-one reads, at offsets and with trailing
bytes; malformed bodies raise ValueError naming blob, field and element."""
import functools
import hashlib
import os
import random
import struct

import numpy as np
import pytest
import torch

import varuna_bytes_oracle as vb
import varuna_pk_bytes_oracle as vpk
from helpers import affine_array
from oracle import bls12_377 as py

pytestmark = pytest.mark.gpu
R, Q = vb.R, vb.Q
BETA, GAMMA = 0x1234567890ABCDEF % R, 0xFEDCBA09 % R
HERE = os.path.dirname(os.path.abspath(__file__))
# (constraints, variables, mul_depth) per circuit
SHAPES = {"one": [(64, 60, 2)], "three": [(64, 60, 2), (200, 300, 3), (1000, 700, 5)]}


def _image97(p) -> bytes:
    x, y, inf = p
    return py.fq_to_mont(x).to_bytes(48, "little") + py.fq_to_mont(y).to_bytes(48, "little") + bytes([int(inf)]) + bytes(7)


def _non_subgroup_point():
    x = 2
    while True:
        y, _k = vb.sqrt(x ** 3 + 1)
        if y is not None and not vb.in_subgroup((x, y)):
            return x, y
        x += 1


def test_to_bytes_point_corpus_matches_the_oracle():
    from snarkvm_b200 import device
    g = [py.g1_mul((py.G1_GEN_X, py.G1_GEN_Y), k) for k in (1, 2, 3, 12345, R - 1)]
    ox, oy = _non_subgroup_point()
    recs = [vpk.encode_point97((x, y, False)) for x, y in g]
    recs += [vpk.encode_point97(p) for p in [(0, 1, True), (0, 1, False), (5, 1, True), (5, 1, False), (0, 0, True), (0, 7, True),
                                            (g[0][0], g[0][1], True), (g[1][0], 1, True), (0, 0, False)]]
    recs += [x.to_bytes(48, "little") + y.to_bytes(48, "little") + b"\x00"
             for x, y in [(Q, g[0][1]), (g[0][0], Q), (Q + 1, g[0][1]), (2**384 - 1, g[0][1]), (g[0][0], 2**384 - 1)]]
    recs += [vpk.encode_point97((g[0][0], g[0][1], False))[:96] + b"\x02", vpk.encode_point97((0, 1, True))[:96] + b"\x02"]
    recs += [vpk.encode_point97((g[0][0], (g[0][1] + 1) % Q, False)), vpk.encode_point97((ox, oy, False))]
    raw = torch.from_numpy(np.frombuffer(b"".join(recs), dtype=np.uint8).copy()).cuda()
    for validate in (False, True):
        images, status = device.g1_deserialize(raw, device.G1_TO_BYTES, validate)
        images, status = images.cpu().numpy(), status.cpu().numpy()
        seen = set()
        for i, b in enumerate(recs):
            s, p = vpk.decode_point97(b, validate)
            seen.add(s)
            assert status[i] == s, (i, validate)
            want = _image97(p) if p is not None and s == vb.VALID else (bytes(104) if p is None else None)
            if want is not None:
                assert images[i].tobytes() == want, (i, validate)
        assert seen == ({vb.VALID, vb.NOT_CANONICAL, vb.BAD_FLAGS, vb.NOT_ON_CURVE, vb.NOT_IN_SUBGROUP} if validate else
                        {vb.VALID, vb.NOT_CANONICAL, vb.BAD_FLAGS})
        # every accepted point writes back to its own bytes, infinity included
        ok = np.nonzero(status == 0)[0]
        out = device.g1_serialize(torch.from_numpy(images[ok].copy()).cuda(), device.G1_TO_BYTES).cpu().numpy()
        assert [r.tobytes() for r in out] == [recs[i] for i in ok]


def test_fr_record_corpus_matches_the_oracle():
    from snarkvm_b200 import device
    vals = [0, R - 1, R, 2**256 - 1, 12345]
    nvars = 1000
    cols = [nvars - 1, nvars, 2**31, 2**63, 0]
    ev = b"".join(v.to_bytes(32, "little") for v in vals)
    # a matrix of five rows, one entry each except an empty row 1 (entries of rows 0, 2, 3, 4, 4)
    rows = [[0], [], [1], [2], [3, 4]]
    mat = struct.pack("<Q", len(rows)) + b"".join(struct.pack("<Q", len(r)) + b"".join(
        vals[e].to_bytes(32, "little") + struct.pack("<Q", cols[e]) for e in r) for r in rows)
    blob = b"\x07" + ev + mat + b"\x00"                                    # odd offsets: no alignment
    d = torch.from_numpy(np.frombuffer(blob, dtype=np.uint8).copy()).cuda()
    out_e = torch.empty((5, 4), dtype=torch.int64, device="cuda")
    out_m = torch.empty((5, 4), dtype=torch.int64, device="cuda")
    out_c = torch.empty(5, dtype=torch.int32, device="cuda")
    rp = torch.tensor([0, 1, 1, 2, 3, 5], dtype=torch.int32, device="cuda")
    # the same values as plain 40-byte runs of the matrix's last row, whose two entries are adjacent
    out_r = torch.empty((2, 4), dtype=torch.int64, device="cuda")
    out_rc = torch.empty(2, dtype=torch.int32, device="cuda")
    last = 1 + len(ev) + len(mat) - 80
    bad = device.fr_records_decode(d, [(1, 5, 32, out_e, None, 0, None), (1 + len(ev), 5, 40, out_m, out_c, nvars, rp),
                                       (last, 2, 40, out_r, out_rc, nvars, None)])
    assert bad == [(2, device.FR_RECORD_NOT_CANONICAL), (1, device.FR_RECORD_BAD_COLUMN), (0, device.FR_RECORD_NOT_CANONICAL)]

    def ints(t):
        h = t.cpu().numpy().view(np.uint64)
        return [py.fr_from_mont(sum(int(v) << (64 * i) for i, v in enumerate(row))) for row in h]
    got = ints(out_e)
    assert got[0] == 0 and got[1] == R - 1 and got[4] == 12345
    got = ints(out_m)
    assert got[0] == 0 and got[1] == R - 1 and got[4] == 12345
    assert out_c.cpu().tolist()[0] == nvars - 1 and out_c.cpu().tolist()[4] == 0
    assert ints(out_r)[1] == 12345 and out_rc.cpu().tolist()[1] == 0
    from snarkvm_b200._lib import CudaError
    with pytest.raises(CudaError):                                        # a segment that leaves the blob
        device.fr_records_decode(d, [(len(blob) - 31, 1, 32, out_e[:1], None, 0, None)])


def _keys(name, zk, srs=None):
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import synthetic_srs
    rng = random.Random(len(SHAPES[name]))
    made = [dv.test_circuit_csr(rng.randrange(2, R), rng.randrange(2, R), depth, nc, nv, "cuda") for nc, nv, depth in SHAPES[name]]
    circuits = [c for c, _z in made]
    D = max(c.info.max_degree(zk) for c in circuits) + 8
    powers, gpowers = srs or synthetic_srs(D, BETA, GAMMA)
    keys = dv.batch_circuit_setup(circuits, powers, gpowers, zk, with_id=True)
    return [pk for pk, _vk in keys], [[z] for _c, z in made], D


def _fr_ints(t):
    from snarkvm_b200 import device
    if t.shape[0] == 0:
        return []
    h = device.fr_from_mont(t.contiguous()).cpu().numpy().view(np.uint64)
    return [sum(int(v) << (64 * i) for i, v in enumerate(row)) for row in h]


def _points97(t):
    out = []
    for img in t.cpu().numpy():
        b = img.tobytes()
        out.append((py.fq_from_mont(int.from_bytes(b[:48], "little")), py.fq_from_mont(int.from_bytes(b[48:96], "little")), b[96] != 0))
    return out


def _oracle_dict(pk):
    """the key's contents as the oracle's integers"""
    c, ck, vk = pk.circuit, pk.committer_key, pk.circuit_verifying_key
    matrices = []
    for m in (c.a, c.b, c.c):
        rp, cols, vals = m.row_ptr.cpu().tolist(), m.cols.cpu().tolist(), _fr_ints(m.vals)
        matrices.append([[(vals[e], cols[e]) for e in range(rp[i], rp[i + 1])] for i in range(m.nrows)])
    arith = [{n: _fr_ints(getattr(a, n)) for n in ("row", "col", "row_col_val")} for a in c.ariths]
    comms = [py.projective_from_bytes(np.ascontiguousarray(x, dtype=np.uint64).tobytes()) for x in vk.circuit_commitments]
    return {"vk": {"info": list(struct.unpack("<6Q", vk.circuit_info.to_bytes_le())),
                   "commitments": comms, "id": c.id()},
            "matrices": matrices, "arith": arith,
            "ck": {"powers": _points97(ck.powers_of_beta_g), "lagrange": {}, "gamma": _points97(ck.powers_of_beta_times_gamma_g),
                   "shifted": None if ck.shifted_powers_of_beta_g is None else _points97(ck.shifted_powers_of_beta_g),
                   "shifted_gamma": None if ck.shifted_powers_of_beta_times_gamma_g is None else
                   {b: _points97(v) for b, v in ck.shifted_powers_of_beta_times_gamma_g.items()},
                   "bounds": ck.enforced_degree_bounds}}


def _same_key(a, b):
    """equal CSR arrays, evaluations, committer-key images and verifying key"""
    for m, n in zip((a.circuit.a, a.circuit.b, a.circuit.c), (b.circuit.a, b.circuit.b, b.circuit.c)):
        assert torch.equal(m.row_ptr, n.row_ptr) and torch.equal(m.cols, n.cols) and torch.equal(m.vals, n.vals)
    for x, y in zip(a.circuit.ariths, b.circuit.ariths):
        assert x.domain.size == y.domain.size
        for name in ("row", "col", "row_col_val"):
            assert torch.equal(getattr(x, name), getattr(y, name))
    ca, cb = a.committer_key, b.committer_key
    for name in ("powers_of_beta_g", "powers_of_beta_times_gamma_g", "shifted_powers_of_beta_g"):
        assert torch.equal(getattr(ca, name), getattr(cb, name))
    assert ca.shifted_powers_of_beta_times_gamma_g.keys() == cb.shifted_powers_of_beta_times_gamma_g.keys()
    for k in ca.shifted_powers_of_beta_times_gamma_g:
        assert torch.equal(ca.shifted_powers_of_beta_times_gamma_g[k], cb.shifted_powers_of_beta_times_gamma_g[k])
    assert ca.enforced_degree_bounds == cb.enforced_degree_bounds and ca.lagrange_bases_at_beta_g == cb.lagrange_bases_at_beta_g == {}
    va, vb_ = a.circuit_verifying_key, b.circuit_verifying_key
    assert va.circuit_info == vb_.circuit_info and va.id == vb_.id and (va.circuit_commitments == vb_.circuit_commitments).all()
    assert a.circuit.info == b.circuit.info and a.circuit.id() == b.circuit.id()


@functools.lru_cache(maxsize=None)
def _keyed(name, zk):
    from snarkvm_b200 import varuna as dv
    pks, assignments, D = _keys(name, zk)
    return name, zk, pks, assignments, D, dv.proving_keys_to_bytes(pks)


@pytest.fixture(scope="module", params=[("one", False), ("one", True), ("three", False), ("three", True)],
                ids=lambda p: f"{p[0]}-{'zk' if p[1] else 'plain'}")
def keyed(request):
    return _keyed(*request.param)


def test_round_trip_matches_the_oracle(keyed):
    from snarkvm_b200 import device
    from snarkvm_b200 import varuna as dv
    name, zk, pks, _a, _d, blobs = keyed
    loaded = dv.proving_keys_from_bytes(blobs)
    coinciding = 0
    for pk, blob, back in zip(pks, blobs, loaded):
        assert blob == vpk.write_proving_key(_oracle_dict(pk))
        assert len(blob) == vpk.proving_key_size(struct.unpack("<6Q", pk.circuit.info.to_bytes_le()), zk)
        _same_key(pk, back)
        fresh = hashlib.blake2s(pk.circuit.info.to_bytes_le() + b"".join(
            device.csr_serialize(m.row_ptr, m.cols, m.vals).cpu().numpy().tobytes() for m in (back.circuit.a, back.circuit.b,
                                                                                           back.circuit.c)), digest_size=32).digest()
        assert back.circuit.id() == fresh == back.circuit_verifying_key.id
        assert back.committer_key.max_degree is None
        assert back.to_bytes() == blob
        coinciding += len(pk.committer_key.enforced_degree_bounds) < 4
    assert coinciding >= 1                                                 # a key whose degree bounds coincide


def test_loaded_keys_prove_as_the_originals(keyed):
    from snarkvm_b200 import varuna as dv
    name, zk, pks, assignments, D, blobs = keyed
    loaded = dv.proving_keys_from_bytes(blobs)
    if not zk:
        want = dv.prove_batch(list(zip(pks, assignments)), zk)
        got = dv.prove_batch(list(zip(loaded, assignments)), zk)
        assert dv.proofs_to_bytes([got]) == dv.proofs_to_bytes([want])
        mixed = dv.prove_batch(list(zip([loaded[0]] + pks[1:], assignments)), zk)      # a loaded key with setup-made ones
        assert dv.proofs_to_bytes([mixed]) == dv.proofs_to_bytes([want])
    else:
        proof = dv.prove_batch(list(zip(loaded, assignments)), zk, random.Random(3))
        bounds = [(1 << k) - 2 for k in range(1, D.bit_length() + 1) if (1 << k) - 2 <= D]
        verifier = dv.UniversalVerifier.synthetic(BETA, max_degree=D, gamma=GAMMA, bounds=bounds)
        kti = [(pk.circuit_verifying_key, [_fr_ints(z[: pk.circuit.num_public]) for z in zs]) for pk, zs in zip(loaded, assignments)]
        assert dv.verify_batch_many(verifier, [(kti, proof)], zk) == [True]


def test_many_per_call_offsets_and_trailing_bytes():
    from snarkvm_b200 import varuna as dv
    _n, _zk, pks, _a, _d, blobs = _keyed("three", False)
    many = dv.proving_keys_from_bytes(blobs + blobs[:1])
    ones = [dv.CircuitProvingKey.from_bytes(b) for b in blobs + blobs[:1]]
    for a, b in zip(many, ones):
        _same_key(a, b)
    prefix = b"\x01" + bytes(range(40))
    got, end = dv.CircuitProvingKey.read(bytearray(prefix + blobs[1] + b"trailing"), len(prefix))
    assert end == len(prefix) + len(blobs[1])
    _same_key(got, pks[1])
    ck, end = type(pks[0].committer_key).read(memoryview(b"xyz" + pks[0].committer_key.to_bytes() + b"!"), 3)
    assert end == 3 + len(pks[0].committer_key.to_bytes())
    assert torch.equal(ck.powers_of_beta_g, pks[0].committer_key.powers_of_beta_g)


def _layout(pk):
    """byte offsets inside a key's blob: matrix sections, evaluation vectors, domain of A's row, the committer key"""
    c = pk.circuit
    o = {"a": vpk.VK_BYTES + 48}
    o["b"] = o["a"] + 8 + 8 * c.num_constraints + 40 * c.a.nnz
    o["c"] = o["b"] + 8 + 8 * c.num_constraints + 40 * c.b.nnz
    at = o["c"] + 8 + 8 * c.num_constraints + 40 * c.c.nnz
    o["row_a"] = at + 8
    o["dom_a"] = at + 8 + 32 * c.ariths[0].domain.size
    o["col_b"] = at + 3 * (8 + 32 * c.ariths[0].domain.size + 172) + 1 + 8 + 32 * c.ariths[1].domain.size + 172 + 8
    return o


def test_malformed_bodies_are_refused():
    from snarkvm_b200 import varuna as dv
    _n, _zk, pks, _a, _d, blobs = _keyed("three", True)
    pk, blob = pks[1], blobs[1]
    o = _layout(pk)
    r_bytes = R.to_bytes(32, "little")

    def refused(edit, pattern):
        bad = bytearray(blob)
        edit(bad)
        with pytest.raises(ValueError, match=pattern):
            dv.proving_keys_from_bytes([blobs[0], bytes(bad)])

    rp = pk.circuit.a.row_ptr.cpu().tolist()
    row = next(i for i in range(len(rp) - 1) if rp[i + 1] > rp[i])
    e = rp[row]
    entry = o["a"] + 16 + 8 * row + 40 * e
    refused(lambda b: b.__setitem__(slice(entry, entry + 32), r_bytes), rf"blob 1: circuit\.a\[{row}\]\[0\]: not below r")
    refused(lambda b: b.__setitem__(slice(o["row_a"] + 64, o["row_a"] + 96), b"\xff" * 32),
            r"blob 1: circuit\.a_arith\.row\[2\]: not below r")
    nv = pk.circuit.num_variables
    refused(lambda b: b.__setitem__(slice(entry + 32, entry + 40), struct.pack("<Q", nv)),
            rf"blob 1: circuit\.a\[{row}\]\[0\]: column not below")
    refused(lambda b: b.__setitem__(o["dom_a"] + 76, b[o["dom_a"] + 76] ^ 1), r"blob 1: circuit\.a_arith\.row\.domain\.group_gen: differs")
    refused(lambda b: b.__setitem__(len(b) - 1, b[-1] ^ 1), r"blob 1: committer_key\.hash: the SHA-256")
    # a point byte flipped so that the point still decodes (no validation): only the hash breaks
    first_power = len(blob) - len(pk.committer_key.to_bytes()) + 4
    bad = bytearray(blob)
    bad[first_power + 5] ^= 1
    with pytest.raises(ValueError, match=r"blob 0: committer_key\.hash"):
        dv.proving_keys_from_bytes([bytes(bad)], validate=False)
    with pytest.raises(ValueError, match=r"blob 0: committer_key\.powers_of_beta_g\[0\]: not on the curve"):
        dv.proving_keys_from_bytes([bytes(bad)])
    # a matrix value changed to another canonical value: the circuit id no longer matches the verifying key's
    refused(lambda b: b.__setitem__(entry, b[entry] ^ 1), r"blob 1: circuit_verifying_key\.id: differs")
    # a verifying key of another circuit
    refused(lambda b: b.__setitem__(slice(0, vpk.VK_BYTES), blobs[2][: vpk.VK_BYTES]),
            r"blob 1: circuit_verifying_key\.circuit_info: differs")


def test_committer_key_of_the_mainnet_powers_round_trips():
    from snarkvm_b200 import sonic_pc
    blob = open(os.path.join(HERE, "golden", "powers_of_beta_15.usrs"), "rb").read()
    n = int.from_bytes(blob[:8], "little")
    pts = py.parse_usrs_points(blob, n)
    powers = torch.from_numpy(affine_array(pts)).cuda()
    gammas = sonic_pc.synthetic_srs(n, BETA, GAMMA)[1]                    # any γ powers: the hash covers them as they are
    ck = sonic_pc.CommitterKey.trim(powers, gammas, n - 1 - 100, (), 1, [30, 126, n - 1 - 100])
    raw = ck.to_bytes()
    assert raw[4: 4 + 97 * (n - 100)] == b"".join(vpk.encode_point97((x, y, False)) for x, y in pts[: n - 100])
    assert raw == vpk.write_committer_key({"powers": _points97(ck.powers_of_beta_g), "lagrange": {},
                                          "gamma": _points97(ck.powers_of_beta_times_gamma_g),
                                          "shifted": _points97(ck.shifted_powers_of_beta_g),
                                          "shifted_gamma": {b: _points97(v) for b, v in ck.shifted_powers_of_beta_times_gamma_g.items()},
                                          "bounds": ck.enforced_degree_bounds})
    back, end = sonic_pc.CommitterKey.read(raw)
    assert end == len(raw) and back.max_degree is None
    assert torch.equal(back.powers_of_beta_g, ck.powers_of_beta_g) and torch.equal(back.shifted_powers_of_beta_g, ck.shifted_powers_of_beta_g)
    assert back.enforced_degree_bounds == ck.enforced_degree_bounds
    assert torch.equal(back.shifted_powers_of_beta_g[-1], powers[-1])     # shifted powers end on the SRS's last power
