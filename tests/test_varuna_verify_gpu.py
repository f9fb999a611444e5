"""GPU: varuna.verify_batch / verify_batch_many on proofs varuna.prove_batch made — one circuit, and three circuits of different
domains with 1, 2 and 3 instances, in both modes — on a known-trapdoor setup: every honest proof is accepted; one changed commitment,
w, vk commitment, sum, evaluation, random_v or public input, or a mismatched mode, is rejected; each malformed input raises
ValueError naming the proof and the field; one verify_batch_many call over every variant gives the verdicts of one-at-a-time calls,
and the order of keys_to_inputs changes none.  On the mainnet SRS (no trapdoor): each negative power of β·H pairs with its shifted
power of β·G, and proofs made with a committer key of the mainnet powers verify under UniversalVerifier.from_mainnet."""
import copy
import os
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
R = 8444461749428370424248824938781546531375899335154063827935233455917409239041
BETA, GAMMA = 0x1234567890ABCDEF % R, 0xFEDCBA09 % R
# (constraints, variables, mul_depth) per circuit; instances per circuit
SHAPES = {"one": ([(64, 60, 2)], [1]), "three": ([(64, 60, 2), (200, 300, 3), (1000, 700, 5)], [1, 2, 3])}
VARIANTS = [("one", False), ("one", True), ("three", False), ("three", True)]
HERE = os.path.dirname(os.path.abspath(__file__))


def _ints(t):
    from snarkvm_b200 import device
    h = device.fr_from_mont(t).cpu().numpy().view(np.uint64)
    return [sum(int(v) << (64 * i) for i, v in enumerate(row)) for row in h]


def _program(name, zk, srs=None, D=None):
    """[(proving key, assignments)] and keys_to_inputs, set up on the known-trapdoor SRS of max degree D (by default the program's
    max_degree + 8; or on `srs`: (β powers, γβ powers)) → (program, keys_to_inputs, D)"""
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import synthetic_srs
    shapes, batch = SHAPES[name]
    rng = random.Random(len(shapes))
    circuits, assignments = [], []
    for (nc, nv, depth), b in zip(shapes, batch):
        zs = [dv.test_circuit_csr(rng.randrange(2, R), rng.randrange(2, R), depth, nc, nv, "cuda") for _ in range(b)]
        circuits.append(zs[0][0])
        assignments.append([z for _c, z in zs])
    D = D or max(c.info.max_degree(zk) for c in circuits) + 8
    powers, gpowers = srs or synthetic_srs(D, BETA, GAMMA)
    keys = dv.batch_circuit_setup(circuits, powers, gpowers, zk, with_id=True)
    program = [(pk, zs) for (pk, _vk), zs in zip(keys, assignments)]
    keys_to_inputs = [(vk, [_ints(z[: c.num_public]) for z in zs]) for (_pk, vk), c, zs in zip(keys, circuits, assignments)]
    return program, keys_to_inputs, D


def _bounds(D):
    return [(1 << k) - 2 for k in range(1, D.bit_length() + 1) if (1 << k) - 2 <= D]


@pytest.fixture(scope="module")
def proved():
    """variant → (keys_to_inputs, proof, zk, D): every variant set up on the same known-trapdoor SRS of max degree D"""
    from snarkvm_b200 import varuna as dv
    D = _program("three", True)[2]                    # the largest max_degree: one SRS, so proofs of every variant share a verifier
    out = {}
    for name, zk in VARIANTS:
        program, kti, _d = _program(name, zk, D=D)
        out[(name, zk)] = (kti, dv.prove_batch(program, zk, random.Random(7) if zk else None), zk, D)
    return out


def _verifier(D):
    from snarkvm_b200 import varuna as dv
    return dv.UniversalVerifier.synthetic(BETA, max_degree=D, gamma=GAMMA, bounds=_bounds(D))


@pytest.mark.parametrize("variant", VARIANTS, ids=lambda v: f"{v[0]}-{'zk' if v[1] else 'plain'}")
def test_honest_proofs_pass(proved, variant):
    from snarkvm_b200 import varuna as dv
    kti, proof, zk, D = proved[variant]
    verifier = _verifier(D)
    assert dv.verify_batch(verifier, kti, proof, zk) is True
    assert dv.verify_batch(verifier, kti[::-1], proof, zk) is True              # keys_to_inputs in any order
    assert dv.verify_batch(verifier, kti, proof, not zk) is False               # the other mode


def _tampered(kti, proof, zk):
    """(description, keys_to_inputs, proof) variants each of which the verifier must reject"""
    out = []
    c = proof.commitments
    other = c.h_1                                                              # a valid G1 point that is not the one in place

    def with_commitment(field, value, index=None):
        p = copy.deepcopy(proof)
        if index is None:
            setattr(p.commitments, field, value)
        else:
            getattr(p.commitments, field)[index] = value
        return p
    out.append(("h_0", kti, with_commitment("h_0", other)))
    out.append(("g_1", kti, with_commitment("g_1", c.h_0)))
    out.append(("h_1", kti, with_commitment("h_1", c.h_0)))
    out.append(("h_2", kti, with_commitment("h_2", other)))
    out.append(("witness_commitments[-1]", kti, with_commitment("witness_commitments", other, -1)))
    out.append(("g_a_commitments[0]", kti, with_commitment("g_a_commitments", other, 0)))
    out.append(("g_c_commitments[-1]", kti, with_commitment("g_c_commitments", other, -1)))
    if zk:
        out.append(("mask_poly", kti, with_commitment("mask_poly", other)))
    for q in range(3):
        p = copy.deepcopy(proof)
        p.pc_proof[q] = (other, p.pc_proof[q][1])
        out.append((f"pc_proof[{q}].w", kti, p))
        if p.pc_proof[q][1] is not None:
            from snarkvm_b200 import varuna as dv
            p = copy.deepcopy(proof)
            p.pc_proof[q] = (p.pc_proof[q][0], dv._mont(dv._fr_mont_to_int(p.pc_proof[q][1]) + 1))
            out.append((f"pc_proof[{q}].random_v", kti, p))
    k2 = copy.deepcopy(kti)
    k2[-1][0].circuit_commitments[3] = kti[0][0].circuit_commitments[7] if len(kti) == 1 else kti[0][0].circuit_commitments[3]
    out.append(("vk commitment", k2, proof))
    for field, path in (("third_sums", (-1, -1, 2)), ("third_sums", (0, 0, 0)), ("fourth_sums", (-1, 1))):
        p = copy.deepcopy(proof)
        t = getattr(p, field)
        for i in path[:-1]:
            t = t[i]
        t[path[-1]] = (t[path[-1]] + 1) % R
        out.append((f"{field}{list(path)}", kti, p))
    for field in ("g_1_eval", "g_a_evals", "g_c_evals"):
        p = copy.deepcopy(proof)
        if field == "g_1_eval":
            p.evaluations.g_1_eval = (p.evaluations.g_1_eval + 1) % R
        else:
            getattr(p.evaluations, field)[-1] = (getattr(p.evaluations, field)[-1] + 1) % R
        out.append((field, kti, p))
    k3 = copy.deepcopy(kti)
    k3[-1][1][-1][1] = (k3[-1][1][-1][1] + 1) % R
    out.append(("public input", k3, proof))
    return out


@pytest.mark.parametrize("variant", VARIANTS, ids=lambda v: f"{v[0]}-{'zk' if v[1] else 'plain'}")
def test_tampering_flips_the_verdict_and_batched_equals_single(proved, variant):
    """every tampered variant is rejected one at a time; one verify_batch_many call over the honest proof and every variant (and
    the honest proof with keys_to_inputs reversed) gives the same verdicts"""
    from snarkvm_b200 import varuna as dv
    kti, proof, zk, D = proved[variant]
    verifier = _verifier(D)
    cases = _tampered(kti, proof, zk)
    singles = []
    for what, k, p in cases:
        v = dv.verify_batch(verifier, k, p, zk)
        assert v is False, what
        singles.append(v)
    batch = [(kti, proof)] + [(k, p) for _w, k, p in cases] + [(kti[::-1], proof)]
    assert dv.verify_batch_many(verifier, batch, zk) == [True] + singles + [True]


def test_all_variants_in_one_call(proved):
    """proofs of different programs in one verify_batch_many call, each mode in its own call, interleaved with rejected ones"""
    from snarkvm_b200 import varuna as dv
    D = max(v[3] for v in proved.values())
    verifier = _verifier(D)
    for zk in (False, True):
        entries = [(kti, proof) for (name, z), (kti, proof, _zk, _d) in proved.items() if z == zk]
        other = [(kti, proof) for (name, z), (kti, proof, _zk, _d) in proved.items() if z != zk]
        batch = entries + other + entries[::-1]
        want = [dv.verify_batch(verifier, k, p, zk) for k, p in batch]
        assert want == [True] * len(entries) + [False] * len(other) + [True] * len(entries)
        assert dv.verify_batch_many(verifier, batch, zk) == want


def _raises(verifier, batch, zk, *words):
    from snarkvm_b200 import varuna as dv
    with pytest.raises(ValueError) as e:
        dv.verify_batch_many(verifier, batch, zk)
    for w in words:
        assert w in str(e.value), (w, str(e.value))


def test_malformed_inputs_raise_naming_proof_and_field(proved):
    from snarkvm_b200 import varuna as dv
    kti, proof, zk, D = proved[("three", False)]
    verifier = _verifier(D)
    good = (kti, proof)
    with pytest.raises(ValueError):
        dv.verify_batch_many(verifier, [], zk)
    _raises(verifier, [good, ([], proof)], zk, "proof 1", "EmptyBatch")
    p = copy.deepcopy(proof)
    p.commitments.witness_commitments.pop()
    _raises(verifier, [good, (kti, p)], zk, "proof 1", "InvalidBatchSize")
    k = copy.deepcopy(kti)
    k[0] = (k[0][0], k[0][1] + k[0][1])
    _raises(verifier, [good, good, (k, proof)], zk, "proof 2", "public inputs", "inputs for a batch")
    k = copy.deepcopy(kti)
    k[1][1][0] = k[1][1][0] + [0] * 8
    _raises(verifier, [(k, proof)], zk, "proof 0", "public input 0", "input domain")
    k = copy.deepcopy(kti)
    k[1][1][0][0] = 2
    _raises(verifier, [(k, proof)], zk, "proof 0", "first element is not one")
    p = copy.deepcopy(proof)
    p.pc_proof = p.pc_proof[:2]
    _raises(verifier, [good, (kti, p)], zk, "proof 1", "pc_proof")
    # a G1 point that fails validation: off the curve, and a coordinate image ≥ q
    p = copy.deepcopy(proof)
    h = np.array(p.commitments.h_1, dtype=np.uint64).copy()
    h[6] ^= np.uint64(1)
    p.commitments.h_1 = h
    _raises(verifier, [good, (kti, p)], zk, "proof 1", "h_1", "not on the curve")
    p = copy.deepcopy(proof)
    w = np.array(p.pc_proof[2][0], dtype=np.uint64).copy()
    w[:6] = np.frombuffer((dv.Q_MOD + 3).to_bytes(48, "little"), dtype=np.uint64)
    p.pc_proof[2] = (w, p.pc_proof[2][1])
    _raises(verifier, [(kti, p), good], zk, "proof 0", "pc_proof[2].w", "not below q")
    k = copy.deepcopy(kti)
    c = np.array(k[2][0].circuit_commitments, dtype=np.uint64).copy()
    c[4, 6] ^= np.uint64(1)
    k[2][0].circuit_commitments = c
    _raises(verifier, [good, (k, proof)], zk, "proof 1", "verifying key 2", "row_b")
    # the lowest proof at fault is named, whichever stage finds it
    _raises(verifier, [good, (kti, p), ([], proof)], zk, "proof 1")


def _mainnet_verifier():
    from snarkvm_b200 import varuna as dv

    def read(name):
        with open(os.path.join(HERE, "golden", name), "rb") as f:
            return f.read()
    return dv.UniversalVerifier.from_mainnet(read("beta_h.usrs"), read("neg_powers_of_beta.usrs"), read("powers_of_beta_gamma.usrs"))


def _mainnet_srs():
    """(powers of β·G from the 2^15 file, the top 1024 powers of the 2^28 SRS, {i: γβ^i·G}) as device / host arrays"""
    import torch
    from helpers import affine_array
    from oracle import bls12_377 as py
    from snarkvm_b200 import varuna as dv

    def points(name):
        with open(os.path.join(HERE, "golden", name), "rb") as f:
            blob = f.read()
        return torch.from_numpy(affine_array(py.parse_usrs_points(blob, int.from_bytes(blob[:8], "little")))).cuda()
    with open(os.path.join(HERE, "golden", "powers_of_beta_gamma.usrs"), "rb") as f:
        gammas = dv.parse_gamma_powers(f.read())
    return points("powers_of_beta_15.usrs"), points("shifted_powers_of_beta_top1024.usrs"), gammas


MAINNET_D = (1 << 28) - 1


def test_mainnet_negative_powers_pair_with_the_shifted_powers():
    """for every bound d the fixture's top 1024 powers reach: e(β^{D−d}·G, β^{-(D−d)}·H)·e(−G, H) = 1, and a neighbouring power fails"""
    import torch
    from snarkvm_b200 import device
    from snarkvm_b200 import varuna as dv
    verifier = _mainnet_verifier()
    _powers, shifted, _g = _mainnet_srs()
    assert sorted(verifier.neg_index) == [(1 << k) - 2 for k in range(1, 28)]
    top = shifted.shape[0]
    g1, idx = [], []
    bounds = [d for d in sorted(verifier.neg_index) if d < top - 1]
    neg_g = verifier.g.copy()                                                  # −G: y ↦ q − y on the Montgomery image
    neg_g[48:96] = np.frombuffer((dv.Q_MOD - int.from_bytes(neg_g[48:96].tobytes(), "little")).to_bytes(48, "little"), dtype=np.uint8)
    for d in bounds:
        for off in (0, 1):
            g1 += [shifted[top - 1 - d - off].cpu().numpy(), neg_g]
            idx += [verifier.neg_index[d], 0]
    starts = torch.arange(0, len(g1) + 1, 2, dtype=torch.int32, device="cuda")
    _gt, ones = device.pairing_products(torch.from_numpy(np.stack(g1)).cuda(), torch.tensor(idx, dtype=torch.int32, device="cuda"),
                                        verifier.prepared, starts)
    assert ones.cpu().tolist() == [True, False] * len(bounds)


@pytest.mark.parametrize("name", ["one", "three"])
@pytest.mark.parametrize("zk", [False, True], ids=["plain", "zk"])
def test_mainnet_srs(name, zk):
    """a committer key of the mainnet powers (the 2^15 prefix, the shifts of the 2^28 SRS for every enforced bound, the γ map):
    prove_batch's proofs verify under UniversalVerifier.from_mainnet; a tampered g_1 and a tampered g_a are rejected"""
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import CommitterKey
    powers, shifted, gammas = _mainnet_srs()
    import torch
    gamma_dense = torch.from_numpy(np.stack([gammas[i] for i in range(3)])).cuda()
    program, kti, _D = _program(name, zk, (powers, gamma_dense))
    top = shifted.shape[0]
    keyed = []
    for pk, zs in program:
        bounds = sorted(set(pk.circuit.info.degree_bounds()))
        highest = bounds[-1]
        ck = CommitterKey(pk.committer_key.powers_of_beta_g, gamma_dense, {}, shifted[top - 1 - highest:],
                          {d: torch.from_numpy(np.stack([gammas[MAINNET_D - d + i] for i in range(3)])).cuda() for d in bounds},
                          bounds, MAINNET_D)
        keyed.append((dv.CircuitProvingKey(pk.circuit_verifying_key, pk.circuit, ck), zs))
    proof = dv.prove_batch(keyed, zk, random.Random(5) if zk else None)
    verifier = _mainnet_verifier()
    bad_g1, bad_ga = copy.deepcopy(proof), copy.deepcopy(proof)
    bad_g1.commitments.g_1 = proof.commitments.h_1
    bad_ga.commitments.g_a_commitments[0] = proof.commitments.h_0
    assert dv.verify_batch_many(verifier, [(kti, proof), (kti, bad_g1), (kti, bad_ga)], zk) == [True, False, False]
