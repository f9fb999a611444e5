"""Self-contained verifying-key certificates: prove_vk / verify_vk drawing their challenges from the device Poseidon sponge
(varuna.certificate_challenges) — against the big-integer sponge (oracle/poseidon.py) for a mixed 32-circuit program, byte for byte
against the same calls given the oracle's challenges, and with the pairing's verdict on a synthetic setup and on the mainnet 2^15 SRS."""
import copy
import dataclasses
import os
import random

import numpy as np
import pytest

from helpers import affine_array
from oracle import bls12_377 as py
from oracle import poseidon as op
from snarkvm_b200 import poseidon as ps

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
R, Q = py.R_MOD, py.Q_MOD
BETA, GAMMA = 0x1234567890ABCDEF1234567890ABCDEF % R, 0xFEDCBA0987654321FEDCBA % R
# (mul_depth, constraints, variables) of 32 test circuits from 2^3 to 2^12 constraints: distinct matrices, so distinct ids
SHAPES = [(2 + k % 3, 7 + 125 * k, 7 + 120 * k) for k in range(32)]


def _oracle_challenges(vk):
    qinv = pow((1 << 384) % Q, -1, Q)
    affine = []
    for row in np.ascontiguousarray(vk.circuit_commitments, dtype=np.uint64).reshape(12, 18):
        x, y = (int.from_bytes(row[6 * i: 6 * i + 6].tobytes(), "little") * qinv % Q for i in range(2))
        affine.append((x, y) if row[12:].any() else None)
    s = op.certificate_sponge(Q, 377, ps.parameters(ps.FIELD_FQ, 2), vk.circuit_info.to_bytes_le(), affine, vk.id)
    return op.certificate_challenges(s)


def _program(powers, gamma, count, seed):
    from snarkvm_b200 import varuna as dv
    rng = random.Random(seed)
    circuits = [dv.test_circuit_csr(rng.randrange(2, R), rng.randrange(2, R), *SHAPES[k], "cuda")[0] for k in range(count)]
    setups = dv.batch_circuit_setup(circuits, powers, gamma, with_id=True)
    return circuits, [s[0] for s in setups], [s[1] for s in setups]


@pytest.fixture(scope="module")
def synthetic():
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import synthetic_srs
    powers, gamma = synthetic_srs(8191, BETA, GAMMA)
    return _program(powers, gamma, 32, 1), dv.UniversalVerifier.synthetic(BETA)


def test_derived_challenges_equal_the_oracle(synthetic):
    from snarkvm_b200 import varuna as dv
    (_circuits, _pks, vks), _v = synthetic
    got = dv.certificate_challenges(vks)
    assert len({tuple(g[0]) for g in got}) == len(vks)
    for vk, g in zip(vks, got):
        assert g == _oracle_challenges(vk)


def test_prove_with_derived_challenges_equals_given(synthetic):
    from snarkvm_b200 import varuna as dv
    (_circuits, pks, vks), _v = synthetic
    want = [_oracle_challenges(vk) for vk in vks]
    derived = dv.prove_vk_batch(pks)
    given = dv.prove_vk_batch(pks, [w[0] for w in want], [w[1] for w in want])
    assert all(a.w.tobytes() == b.w.tobytes() for a, b in zip(derived, given))
    assert dv.prove_vk(pks[3]).w.tobytes() == derived[3].w.tobytes()


def _same(a, b):
    return (a.matches == b.matches and a.evaluation == b.evaluation and (a.lhs == b.lhs).all() and (a.w == b.w).all()
            and a.valid == b.valid)


def test_verify_with_derived_challenges(synthetic):
    from snarkvm_b200 import varuna as dv
    (circuits, pks, vks), verifier = synthetic
    certs = dv.prove_vk_batch(pks)
    res = dv.verify_vk_batch(circuits, vks, certs, verifier=verifier)
    assert all(r.matches and r.valid is True for r in res)
    want = [_oracle_challenges(vk) for vk in vks]
    given = dv.verify_vk_batch(circuits, vks, certs, [w[0] for w in want], [w[1][0] for w in want], verifier=verifier)
    assert all(_same(a, b) for a, b in zip(res, given))
    assert _same(dv.verify_vk(circuits[5], vks[5], certs[5], verifier=verifier), res[5])
    assert _same(dv.verify_vk_batch(circuits[5:6], vks[5:6], certs[5:6], verifier=verifier)[0], res[5])
    # one commitment, the circuit info, the id or W changed: that circuit alone is invalid
    K = len(circuits)
    for k, change in [(1, "commitment"), (2, "info"), (4, "id"), (6, "w")]:
        vks2, certs2 = list(vks), list(certs)
        vk = copy.deepcopy(vks[k])
        if change == "commitment":
            vk.circuit_commitments[7] = vks[k].circuit_commitments[8]
        elif change == "info":
            vk.circuit_info = dataclasses.replace(vk.circuit_info, num_non_zero_a=vk.circuit_info.num_non_zero_a + 1)
        elif change == "id":
            vk.id = bytes([vk.id[0] ^ 1]) + vk.id[1:]
        else:
            certs2[k] = dv.Certificate(certs[k - 1].w.copy())
        vks2[k] = vk
        out = dv.verify_vk_batch(circuits, vks2, certs2, verifier=verifier)
        assert [r.valid for r in out] == [i != k for i in range(K)], change
        assert out[k].matches == (change in ("commitment", "w")), change
    vk = copy.deepcopy(vks[0])
    vk.id = None
    with pytest.raises(ValueError):
        dv.verify_vk_batch(circuits[:1], [vk], certs[:1], verifier=verifier)
    with pytest.raises(ValueError):
        dv.prove_vk_batch([dataclasses.replace(pks[0], circuit_verifying_key=vk)])


def test_mainnet_srs():
    import torch
    from snarkvm_b200 import varuna as dv
    blob = open(os.path.join(HERE, "golden", "powers_of_beta_15.usrs"), "rb").read()
    powers = torch.from_numpy(affine_array(py.parse_usrs_points(blob, int.from_bytes(blob[:8], "little")))).cuda()
    with open(os.path.join(HERE, "golden", "beta_h.usrs"), "rb") as f:
        verifier = dv.UniversalVerifier.from_usrs(f.read())
    circuits, pks, vks = _program(powers, powers, 5, 2)
    certs = dv.prove_vk_batch(pks)
    assert all(r.matches and r.valid is True for r in dv.verify_vk_batch(circuits, vks, certs, verifier=verifier))
    assert [r.valid for r in dv.verify_vk_batch(circuits, vks, certs[::-1], verifier=verifier)] == [False, False, True, False, False]
