"""CPU: the verifier's scalar side in snarkvm_b200/varuna.py (linear_combinations with a_poly / b_poly expanded, and check_combinations
→ batch_check → accumulate_elems folded into one scalar per base point of each degree-bound group) equals the literal big-integer
restatement in tests/varuna_verifier_oracle.py, on seeded proof numbers and challenges for one circuit and for three circuits with
1, 2 and 3 instances, in both modes.  The mainnet fixtures the verifier reads hold the SHA-256 values of the reference's metadata (the
shifted powers: a pinned 1024-point slice), the degree bounds 2^k − 2 for k = 1 … 27 and 84 powers of β·γ·G."""
import hashlib
import os
import random

import numpy as np
import pytest

import varuna_verifier_oracle as vo

R = vo.R
HERE = os.path.dirname(os.path.abspath(__file__))
# (num_public, num_variables, num_constraints, nnz_a, nnz_b, nnz_c) per circuit
INFOS = {"one": [(4, 64, 64, 64, 64, 64)], "three": [(4, 64, 64, 64, 64, 64), (4, 304, 200, 200, 200, 200), (8, 708, 1000, 1000, 1000, 997)]}
BATCH = {"one": [1], "three": [1, 2, 3]}


def _image(rng):
    """a normalised projective image with arbitrary x, y and z = one: the scalar side never reads the coordinates"""
    from snarkvm_b200 import varuna as dv
    out = np.zeros(18, dtype=np.uint64)
    out[:12] = np.frombuffer(rng.randrange(dv.Q_MOD).to_bytes(48, "little") + rng.randrange(dv.Q_MOD).to_bytes(48, "little"), dtype=np.uint64)
    out[12:] = dv._FQ_ONE
    return out


def _case(name, zk, seed):
    from snarkvm_b200 import varuna as dv
    rng = random.Random(seed)
    fr = lambda: rng.randrange(R)                                              # noqa: E731
    infos = [dv.CircuitInfo(*i) for i in INFOS[name]]
    batch = BATCH[name]
    kti = []
    for k, (info, b) in enumerate(zip(infos, batch)):
        vk = dv.CircuitVerifyingKey(info, np.stack([_image(rng) for _ in range(12)]), bytes([0x30 + 7 * k]) + bytes(rng.randrange(256) for _ in range(31)))
        kti.append((vk, [[1] + [fr() for _ in range(info.num_public_inputs - 1)] for _ in range(b)]))
    K = len(infos)
    comms = dv.Commitments([_image(rng) for _ in range(sum(batch))], _image(rng) if zk else None, _image(rng), _image(rng), _image(rng),
                           [_image(rng) for _ in range(K)], [_image(rng) for _ in range(K)], [_image(rng) for _ in range(K)], _image(rng))
    proof = dv.Proof(batch, comms, dv.Evaluations(fr(), [fr() for _ in range(K)], [fr() for _ in range(K)], [fr() for _ in range(K)]),
                     [[[fr(), fr(), fr()] for _ in range(b)] for b in batch], [[fr(), fr(), fr()] for _ in range(K)],
                     [(_image(rng), dv._mont(fr()) if zk and q else None) for q in range(3)])
    combs = [(1 if i == 0 else fr(), [1] + [fr() for _ in range(b - 1)]) for i, b in enumerate(batch)]
    ch = {"batch_combiners": combs, "alpha": fr(), "eta_b": fr(), "eta_c": fr(), "beta": fr(),
          "deltas": [[1, fr(), fr()]] + [[fr(), fr(), fr()] for _ in range(K - 1)], "gamma": fr(),
          "opening": [fr() >> 85 for _ in range(3 * K + 7)]}
    return kti, proof, ch


@pytest.mark.parametrize("name", ["one", "three"])
@pytest.mark.parametrize("zk", [False, True], ids=["plain", "zk"])
@pytest.mark.parametrize("seed", [1, 2])
def test_scalars_equal_the_oracle(name, zk, seed):
    from snarkvm_b200 import varuna as dv
    kti, proof, ch = _case(name, zk, seed)
    view = dv._ProofView(kti, proof)
    # the verifier's x(β), from the oracle's Lagrange coefficients (the device pass is checked by the GPU tests)
    x_at_beta = [[sum(x * l for x, l in zip(inp, vo.lagrange_coefficients(d.input_domain.size, ch["beta"]))) % R for inp in ins]
                 for d, ins in zip(view.domains, view.inputs)]
    got = view.check_scalars(ch, x_at_beta, zk)

    # the oracle, from the reference's labels and its own restatement
    circuits = [{"id": vid.hex(), "info": tuple(vars(vk.circuit_info).values())} for vid, vk in zip(view.ids, view.vks)]
    ev = proof.evaluations
    evals = {"g_1": ev.g_1_eval}
    for i, c in enumerate(circuits):
        for m, vals in zip("abc", (ev.g_a_evals, ev.g_b_evals, ev.g_c_evals)):
            evals[f"circuit_{c['id']}_g_{m}_{0:08}"] = vals[i]
    lcs = vo.construct_linear_combinations(circuits, view.inputs, evals, proof.third_sums, proof.fourth_sums, ch, zk)
    C_max = max(vo.size_of(c["info"][1]) for c in circuits)
    commitments = {lab: ({lab: 1}, None) for lab in view.labels}
    commitments["g_1"] = ({"g_1": 1}, C_max - 2)
    for c in circuits:
        for m, nnz in zip("abc", c["info"][3:]):
            lab = f"circuit_{c['id']}_g_{m}_{0:08}"
            commitments[lab] = ({lab: 1}, vo.size_of(nnz) - 2)
    points = {"alpha": ch["alpha"], "beta": ch["beta"], "gamma": ch["gamma"]}
    where = {"rowcheck_zerocheck": "alpha", "g_1": "beta", "lineval_sumcheck": "beta", "matrix_sumcheck": "gamma"}
    query_set = [(lab, (where.get(lab, "gamma"), points[where.get(lab, "gamma")])) for lab in lcs]
    values = {(lab, x): (evals.get(lab, 0)) for lab, (_n, x) in query_set}
    rv = [None if v is None else dv._fr_mont_to_int(v) for _w, v in proof.pc_proof]
    groups, witness, adjusted = vo.check_combinations(lcs, commitments, query_set, values, [(f"w_{q}", rv[q]) for q in range(3)],
                                                      iter(ch["opening"]))
    # check_elems pairs −adjusted with H like the None group: the verifier merges the two
    merged = dict(groups.get(None, {}))
    for k, v in adjusted.items():
        merged[k] = (merged.get(k, 0) - v) % R
    want = {d: {k: v for k, v in g.items() if v} for d, g in groups.items() if d is not None}
    want[None] = {k: v for k, v in merged.items() if v}
    want["witness"] = {k: (-v) % R for k, v in witness.items()}
    assert {d: {k: v for k, v in g.items() if v} for d, g in got.items()} == want
    assert sorted(d for d in got if d not in (None, "witness")) == sorted({C_max - 2} | {vo.size_of(n) - 2 for c in circuits for n in c["info"][3:]})


def test_malformed_proofs_raise_before_any_launch():
    from snarkvm_b200 import varuna as dv
    kti, proof, _ch = _case("three", False, 3)
    dv._ProofView(kti, proof)
    with pytest.raises(ValueError, match="EmptyBatch"):
        dv._ProofView([], proof)
    bad = [(vk, ins[:-1] if k == 2 else ins) for k, (vk, ins) in enumerate(kti)]
    with pytest.raises(ValueError, match="public inputs of verifying key 2"):
        dv._ProofView(bad, proof)
    proof.third_sums[0][0][1] = R
    with pytest.raises(ValueError, match="third_sums is not below r"):
        dv._ProofView(kti, proof)


def _read(name):
    with open(os.path.join(HERE, "golden", name), "rb") as f:
        return f.read()


def test_mainnet_fixtures():
    """the SHA-256 values listed in the reference's .metadata files (and that of the shifted powers' slice), and what the parsers
    read"""
    from snarkvm_b200 import varuna as dv
    sha = {"neg_powers_of_beta.usrs": "ded57ae81c510f8fd50c8f3ec3387e8397ffdde71acfcc639ff1a2728a0848cd",
           "powers_of_beta_gamma.usrs": "03fd7fc81234b014e1e260c797e9b716b5587429871026f17a455cd0938d8be1",
           # the last 1024 points of shifted-powers-of-beta-15.usrs (SHA-256 7c732bfa…a7ed49) under a count of 1024
           "shifted_powers_of_beta_top1024.usrs": "3b318bbd72b8ebc62c99f88990851a10ad8c41bb5779ad595a14dcd194a869c0"}
    for name, digest in sha.items():
        assert hashlib.sha256(_read(name)).hexdigest() == digest, name
    top = _read("shifted_powers_of_beta_top1024.usrs")
    assert int.from_bytes(top[:8], "little") == 1024 and len(top) == 8 + 1024 * 96
    assert sorted(dv.parse_neg_powers(_read("neg_powers_of_beta.usrs"))) == [(1 << k) - 2 for k in range(1, 28)]
    gammas = dv.parse_gamma_powers(_read("powers_of_beta_gamma.usrs"))
    assert len(gammas) == 84 and 0 in gammas
    blob = bytearray(_read("neg_powers_of_beta.usrs"))
    blob[16: 16 + 48] = (dv.Q_MOD + 1).to_bytes(48, "little")
    with pytest.raises(ValueError, match="not below q"):
        dv.parse_neg_powers(bytes(blob))
    with pytest.raises(ValueError, match="entries"):
        dv.parse_gamma_powers(_read("powers_of_beta_gamma.usrs")[:-1])
