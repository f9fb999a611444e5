"""CPU: the byte forms of Varuna proofs and verifying keys on real data and on malformed blobs.

The mainnet verifying keys and the genesis block's proofs (tests/golden/varuna_bytes, copied by make_bytes_golden.py) match the
metadata checksums and re-encode byte for byte through the big-integer restatement (varuna_bytes_oracle), compressed and
uncompressed.  varuna.proofs_from_bytes and its siblings refuse malformed blobs — truncated, an Option tag other than 0 or 1, an Fr
not below r, a count the bytes cannot hold — during the host walk, before any device call, naming the lowest blob at fault."""
import glob
import hashlib
import json
import os
import struct

import numpy as np
import pytest
import torch

import varuna_bytes_oracle as vb

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "varuna_bytes")
KEYS = sorted(os.path.basename(f)[: -len(".verifier")] for f in glob.glob(os.path.join(GOLDEN, "*.verifier")))
VK_BYTES = 664


def _read(name):
    with open(os.path.join(GOLDEN, name), "rb") as f:
        return f.read()


def _proofs():
    return [_read(f"genesis_proof_{k}.bin") for k in range(8)]


def test_fixtures_match_the_metadata_checksums():
    assert len(KEYS) == 16
    with_num_variables = 0
    for name in KEYS:
        blob = _read(f"{name}.verifier")
        meta = json.loads(_read(f"{name}.metadata"))
        assert hashlib.sha256(blob).hexdigest() == meta["verifier_checksum"]
        assert len(blob) == meta["verifier_size"] and blob[0] == 1 and len(blob) in (1 + VK_BYTES, 1 + VK_BYTES + 8)
        with_num_variables += len(blob) == 1 + VK_BYTES + 8
    assert with_num_variables == 14


def test_oracle_reencodes_the_mainnet_keys():
    flags = set()
    for name in KEYS:
        blob = _read(f"{name}.verifier")[1:]
        r = vb.Reader(blob, 0, compressed=True)
        vk = vb.read_verifying_key(r)
        assert r.o == VK_BYTES
        assert vb.write_verifying_key(vk) == blob[:VK_BYTES]
        flags |= {blob[6 * 8 + 8 + 48 * i + 47] >> 7 for i in range(12)}
        unc = vb.write_verifying_key(vk, compressed=False)
        assert vb.read_verifying_key(vb.Reader(unc, 0, compressed=False)) == vk
    assert flags == {0, 1}                                                  # both signs occur


def test_oracle_reencodes_the_genesis_proofs():
    for blob in _proofs():
        assert len(blob) == 956
        r = vb.Reader(blob, 0, compressed=True)
        p = vb.read_proof(r)
        assert r.o == len(blob)
        assert p["batch_sizes"] == [1] and p["mask_poly"] is not None
        assert [v is not None for _w, v in p["pc_proof"]] == [False, True, False]   # random_v at β only
        assert vb.write_proof(p) == blob
        unc = vb.write_proof(p, compressed=False)
        assert len(unc) == len(blob) + 48 * 12                         # twelve points
        assert vb.read_proof(vb.Reader(unc, 0, compressed=False)) == p


def test_oracle_square_root():
    q = vb.Q
    for a in (0, 1, 4, q - 1, 12345678901234567890):
        y, _k = vb.sqrt(a)
        assert (y is None) == (pow(a, (q - 1) // 2, q) == q - 1)
        if y is not None:
            assert y * y % q == a % q


@pytest.fixture
def no_device(monkeypatch):
    """fails the test if a G1 point reaches the device"""
    from snarkvm_b200 import device

    def refuse(*_a, **_k):
        raise AssertionError("a malformed blob reached the device")
    monkeypatch.setattr(device, "g1_deserialize", refuse)


def _raises(fn, blobs, *words):
    with pytest.raises(ValueError) as ei:
        fn(blobs)
    for w in words:
        assert w in str(ei.value), (w, str(ei.value))


def _with(blob, off, new):
    return blob[:off] + new + blob[off + len(new):]


# offsets in a genesis proof (compressed, one circuit, one instance, hiding)
MASK_TAG = 8 + 8 + 48
G1_EVAL = MASK_TAG + 1 + 48 + 3 * 48 + 3 * 48 + 48
PC_LEN = G1_EVAL + 32 * 4 + 32 * 3 + 32 * 3


def test_malformed_proofs_are_refused_on_the_host(no_device):
    from snarkvm_b200 import varuna as dv
    good = _proofs()[0]
    fn = dv.proofs_from_bytes
    _raises(fn, [good[:500]], "blob 0", "the body of batch sizes [1]")          # below the least size one circuit can take
    _raises(fn, [good[:PC_LEN + 20]], "blob 0", "pc_proof of 3 proofs")
    _raises(fn, [good[:-1]], "blob 0", "pc_proof")
    _raises(fn, [good[:4]], "blob 0", "batch_sizes length")
    _raises(fn, [_with(good, MASK_TAG, b"\x02")], "blob 0", "mask_poly tag", "neither 0 nor 1")
    _raises(fn, [_with(good, PC_LEN + 8 + 48, b"\x07")], "blob 0", "pc_proof[0].random_v tag")
    _raises(fn, [_with(good, G1_EVAL, vb.R.to_bytes(32, "little"))], "blob 0", "evaluations.g_1_eval", "not below r")
    _raises(fn, [_with(good, G1_EVAL, b"\xff" * 32)], "blob 0", "g_1_eval", "not below r")
    _raises(fn, [_with(good, 0, struct.pack("<Q", 1 << 40))], "blob 0", "batch_sizes")
    _raises(fn, [_with(good, 8, struct.pack("<Q", 1 << 40))], "blob 0", "batch sizes [1099511627776]")
    _raises(fn, [_with(good, PC_LEN, struct.pack("<Q", 1 << 40))], "blob 0", "pc_proof")
    # trailing bytes are not an error, but a missing one is — in any blob of a batch, and the first bad blob is named
    with pytest.raises(ValueError, match="blob 0"):
        fn([good[:100], good[:50]])


def test_malformed_keys_and_certificates_are_refused_on_the_host(no_device):
    from snarkvm_b200 import varuna as dv
    vk = _read(f"{KEYS[0]}.verifier")[1:]
    _raises(dv.verifying_keys_from_bytes, [vk[:600]], "blob 0", "circuit_commitments")
    _raises(dv.verifying_keys_from_bytes, [vk[:650]], "blob 0", "id")
    _raises(dv.verifying_keys_from_bytes, [_with(vk, 48, struct.pack("<Q", 11))], "blob 0", "11 commitments")
    cert = struct.pack("<Q", 1) + bytes(47) + b"\x40" + b"\x00"
    _raises(dv.certificates_from_bytes, [cert[:-1]], "blob 0", "pc_proof of 1 proofs")
    _raises(dv.certificates_from_bytes, [cert[:-1] + b"\x02"], "blob 0", "pc_proof[0].random_v tag")
    _raises(dv.certificates_from_bytes, [cert[:-1] + b"\x01" + bytes(32)], "blob 0", "non-hiding")
    _raises(dv.certificates_from_bytes, [struct.pack("<Q", 2) + cert[8:] * 2], "blob 0", "exactly one")


def test_the_lowest_blob_at_fault_is_named(monkeypatch):
    """the points of the blobs before a malformed one are decoded (here by a stand-in that accepts every point) to learn whether
    one of them fails first; the malformed blob's own points are not"""
    from snarkvm_b200 import device
    from snarkvm_b200 import varuna as dv
    seen = []

    def accept(raw, compressed, validate):
        n = raw.numel() // 48
        seen.append(n)
        return torch.zeros((n, 104), dtype=torch.uint8), torch.zeros(n, dtype=torch.int32)
    monkeypatch.setattr(device, "g1_deserialize", accept)
    good = _proofs()[0]
    _raises(lambda b: dv.proofs_from_bytes(b, device_="cpu"), [good, good + b"tail", good[:900], good[:10]], "blob 2", "pc_proof")
    assert seen == [24]                                                    # twelve points in each of the first two

    def reject_last(raw, compressed, validate):
        n = raw.numel() // 48
        status = torch.zeros(n, dtype=torch.int32)
        status[-1] = device.G1_NOT_IN_SUBGROUP
        return torch.zeros((n, 104), dtype=torch.uint8), status
    monkeypatch.setattr(device, "g1_deserialize", reject_last)
    _raises(lambda b: dv.proofs_from_bytes(b, device_="cpu"), [good, good, good[:10]], "blob 1", "pc_proof[2].w",
            "not in the prime-order subgroup")


def test_proofs_read_from_an_offset(monkeypatch):
    """Proof.read walks from `offset` and returns where the proof ends; the decoded objects carry the layout's counts"""
    from snarkvm_b200 import device
    from snarkvm_b200 import varuna as dv

    def accept(raw, compressed, validate):
        n = raw.numel() // 48
        return torch.zeros((n, 104), dtype=torch.uint8), torch.zeros(n, dtype=torch.int32)
    monkeypatch.setattr(device, "g1_deserialize", accept)
    good = _proofs()[3]
    p, end = dv.Proof.read(b"\x01" + good + b"next", 1, device_="cpu")
    assert end == 1 + len(good)
    assert p.batch_sizes == [1] and len(p.commitments.witness_commitments) == 1 and p.commitments.mask_poly is not None
    assert [v is None for _w, v in p.pc_proof] == [True, False, True]
    ref = vb.read_proof(vb.Reader(good, 0, compressed=True))
    assert p.evaluations.g_1_eval == ref["g_1_eval"] and p.third_sums == ref["third_sums"] and p.fourth_sums == ref["fourth_sums"]
    from snarkvm_b200.algorithms import _fr_mont_to_int
    assert _fr_mont_to_int(p.pc_proof[1][1]) == ref["pc_proof"][1][1]
    assert all(np.asarray(w).shape == (18,) for w in p.commitments.witness_commitments)
