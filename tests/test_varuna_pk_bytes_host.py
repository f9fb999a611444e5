"""CPU: the byte form of Varuna proving keys (CircuitProvingKey ToBytes / FromBytes) on the mainnet key sizes and on malformed
headers.

The layout, applied to the CircuitInfo of each of the 16 mainnet verifying keys (tests/golden/varuna_bytes), predicts the
`prover_size` of its metadata exactly.  The big-integer writer and reader (varuna_pk_bytes_oracle) round-trip a small
hand-built key, and varuna._domain_bytes equals the oracle's EvaluationDomain::new.  varuna.proving_keys_from_bytes refuses
malformed headers — truncation anywhere, a bool or Option tag of 2, a count claiming 2^40 elements, a row-length chain that
overruns its matrix — during the host walk, before any device call, naming the blob and the field."""
import glob
import json
import os
import random
import struct

import pytest

import varuna_bytes_oracle as vb
import varuna_pk_bytes_oracle as vpk
from oracle import bls12_377 as py

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "varuna_bytes")
KEYS = sorted(os.path.basename(f)[: -len(".verifier")] for f in glob.glob(os.path.join(GOLDEN, "*.verifier")))


def _read(name):
    with open(os.path.join(GOLDEN, name), "rb") as f:
        return f.read()


def test_size_formula_predicts_every_mainnet_prover_size():
    assert len(KEYS) == 16
    for name in KEYS:
        blob = _read(f"{name}.verifier")
        info = struct.unpack("<6Q", blob[1:49])
        meta = json.loads(_read(f"{name}.metadata"))
        assert 1 + vpk.proving_key_size(info) == meta["prover_size"], name        # the version byte, then the key
    assert 1 + vpk.proving_key_size(struct.unpack("<6Q", _read("inclusion.verifier")[1:49])) == 233812212


def _point(k):
    x, y = py.g1_mul((py.G1_GEN_X, py.G1_GEN_Y), k)
    return x, y, False


def small_key(seed=1):
    """a hand-built key: 2 public of 6 variables, 3 constraints, A/B/C with 3/2/4 entries, a committer key of a few points"""
    rng = random.Random(seed)
    info = [2, 6, 3, 3, 2, 4]
    shapes = [[[0, 2], [1], []], [[5], [], [3]], [[0], [1, 4], [2]]]
    matrices = [[[(rng.randrange(1, vb.R), c) for c in row] for row in m] for m in shapes]
    arith = [{n: [rng.randrange(vb.R) for _ in range(vpk.domain_size(nnz))] for n in ("row", "col", "row_col_val")}
             for nnz in info[3:]]
    pts = [_point(k) for k in range(1, 12)]
    ck = {"powers": pts[:5], "lagrange": {}, "gamma": pts[5:8], "shifted": pts[2:5], "shifted_gamma": {1: pts[8:11], 2: pts[5:8]},
          "bounds": [1, 2]}
    vk = {"info": info, "commitments": [py.g1_mul((py.G1_GEN_X, py.G1_GEN_Y), k + 20) for k in range(12)], "id": bytes(range(32))}
    return {"vk": vk, "matrices": matrices, "arith": arith, "ck": ck}


def test_oracle_round_trips_a_small_key():
    pk = small_key()
    blob = vpk.write_proving_key(pk)
    r = vpk.KeyReader(blob, 0, compressed=False, validate=True)
    back = vpk.read_proving_key(r)
    assert r.o == len(blob)
    assert back["vk"] == pk["vk"] and back["matrices"] == pk["matrices"] and back["ck"] == pk["ck"]
    assert [{n: a[n] for n in ("row", "col", "row_col_val")} for a in back["arith"]] == pk["arith"]
    assert vpk.write_proving_key(back) == blob
    bad = bytearray(blob)
    bad[-40] ^= 1                                                               # the last bound: the hash still holds
    vpk.read_proving_key(vpk.KeyReader(bytes(bad), 0, False))
    bad[-33 - 4 * 2 - 4 - 1 - 10] ^= 1                                          # a byte of a shifted γ point: it does not
    with pytest.raises(ValueError, match="Mismatching"):
        vpk.read_proving_key(vpk.KeyReader(bytes(bad), 0, False))


def test_domain_bytes_match_the_oracle():
    from snarkvm_b200 import varuna as dv
    for lg in range(0, 21):
        assert dv._domain_bytes(1 << lg) == vpk.domain_bytes(1 << lg)


@pytest.fixture
def no_device(monkeypatch):
    """any device work during these tests is a failure: the host walk must refuse first"""
    from snarkvm_b200 import device, sonic_pc

    def refuse(*_a, **_k):
        raise AssertionError("a device call before the host walk finished")
    for mod, name in ((device, "g1_deserialize"), (device, "fr_records_decode"), (sonic_pc, "upload")):
        monkeypatch.setattr(mod, name, refuse)


def _offsets(pk):
    """byte offsets of the small key's sections: the circuit, each matrix, each evaluation vector, the committer key"""
    out = {"circuit": vpk.VK_BYTES, "a": vpk.VK_BYTES + 48}
    out["b"] = out["a"] + 8 + 8 * 3 + 40 * 3
    out["c"] = out["b"] + 8 + 8 * 3 + 40 * 2
    out["arith"] = out["c"] + 8 + 8 * 3 + 40 * 4
    at, ev = out["arith"], []
    for nnz in (3, 2, 4):
        K = vpk.domain_size(nnz)
        ev.append(at)
        at += 3 * (8 + 32 * K + vpk.DOMAIN_BYTES) + 1
    out["ev"], out["ck"] = ev, at
    return out


def test_every_truncation_is_refused_by_the_host_walk(no_device):
    from snarkvm_b200 import varuna as dv
    blob = vpk.write_proving_key(small_key())
    for n in range(len(blob)):
        with pytest.raises(ValueError, match="blob 0: .*bytes left"):
            dv.proving_keys_from_bytes([blob[:n]])


def test_tags_of_two_are_refused(no_device):
    from snarkvm_b200 import varuna as dv
    pk = small_key()
    blob = vpk.write_proving_key(pk)
    o = _offsets(pk)
    K = vpk.domain_size(3)
    row_col = o["ev"][0] + 2 * (8 + 32 * K + vpk.DOMAIN_BYTES)
    ck = o["ck"]
    shifted = ck + 4 + 97 * 5 + 4 + 4 + 97 * 3
    shifted_gamma = shifted + 1 + 4 + 97 * 3
    bounds = shifted_gamma + 1 + 4 + 2 * (8 + 97 * 3)
    for at, field in ((row_col, "circuit.a_arith.row_col tag"), (shifted, "shifted_powers_of_beta_g tag"),
                      (shifted_gamma, "shifted_powers_of_beta_times_gamma_g tag"), (bounds, "enforced_degree_bounds tag")):
        assert blob[at] == 1 or field.startswith("circuit")
        bad = bytearray(blob)
        bad[at] = 2
        with pytest.raises(ValueError, match=f"blob 1: {field}: 2 is neither 0 nor 1"):
            dv.proving_keys_from_bytes([blob, bytes(bad)])


def test_huge_counts_are_refused_before_allocation(no_device):
    from snarkvm_b200 import varuna as dv
    pk = small_key()
    blob = vpk.write_proving_key(pk)
    o = _offsets(pk)
    # 2^40 constraints in both infos and in the row count of A
    bad = bytearray(blob)
    for at in (16, o["circuit"] + 16, o["a"]):
        bad[at: at + 8] = struct.pack("<Q", 1 << 40)
    with pytest.raises(ValueError, match=r"blob 0: circuit\.a of 1099511627776 rows .*bytes left"):
        dv.proving_keys_from_bytes([bytes(bad)])
    # an evaluation vector of 2^40 values
    bad = bytearray(blob)
    bad[o["ev"][1]: o["ev"][1] + 8] = struct.pack("<Q", 1 << 40)
    with pytest.raises(ValueError, match=r"blob 0: circuit\.b_arith\.row: 1099511627776 evaluations, not \|K\| = 2"):
        dv.proving_keys_from_bytes([bytes(bad)])
    # 2^32 − 1 powers of β·G
    bad = bytearray(blob)
    bad[o["ck"]: o["ck"] + 4] = struct.pack("<I", 2**32 - 1)
    with pytest.raises(ValueError, match=r"blob 0: powers_of_beta_g of 4294967295 points: .*bytes left"):
        dv.proving_keys_from_bytes([bytes(bad)])


def test_row_chains_that_overrun_or_disagree_are_refused(no_device):
    from snarkvm_b200 import varuna as dv
    pk = small_key()
    blob = vpk.write_proving_key(pk)
    o = _offsets(pk)
    row1 = o["b"] + 8 + 8 + 40                                       # B's second row header (B's rows hold 1, 0, 1 entries)
    assert struct.unpack("<Q", blob[row1: row1 + 8])[0] == 0
    for length, row in ((1 << 40, 1), (1, 2)):          # far past the section; then row 2 carries the count past num_non_zero_b
        bad = bytearray(blob)
        bad[row1: row1 + 8] = struct.pack("<Q", length)
        with pytest.raises(ValueError, match=rf"blob 0: circuit\.b\[{row}\]: the row lengths overrun"):
            dv.proving_keys_from_bytes([bytes(bad)])
    bad = bytearray(blob)
    row2 = row1 + 8
    bad[row2: row2 + 8] = struct.pack("<Q", 0)                     # the last row loses its entry: the rows hold too few
    with pytest.raises(ValueError, match=r"blob 0: circuit\.b: the row lengths"):
        dv.proving_keys_from_bytes([bytes(bad)])


def test_a_verifying_key_of_another_circuit_is_refused(no_device):
    from snarkvm_b200 import varuna as dv
    blob = bytearray(vpk.write_proving_key(small_key()))
    blob[8: 16] = struct.pack("<Q", 8)                               # the vk's num_public_and_private_variables
    with pytest.raises(ValueError, match=r"blob 0: circuit_verifying_key\.circuit_info: differs"):
        dv.proving_keys_from_bytes([bytes(blob)])
