"""GPU: varuna.prove_batch — the prover's Fiat–Shamir transcript on the resumable device sponge — for one circuit with one instance
and for three circuits of different domains with 1, 2 and 3 instances, in both modes, on a known-trapdoor setup.  Every challenge
equals tests/varuna_transcript_oracle.py recomputed from the Proof's fields, the verifying keys and the public inputs alone; a
BatchProver driven by those challenges reproduces every commitment, evaluation and opening; the three AHP identities vanish; each
opening has its closed form, blinding included; the input order does not change the proof; a changed public input or vk commitment
changes every later challenge.  On the mainnet 2^15 SRS, in both modes, the α opening passes the pairing check."""
import random

import numpy as np
import pytest

import varuna_transcript_oracle as vto

pytestmark = pytest.mark.gpu
R = vto.R
BETA, GAMMA = 0x1234567890ABCDEF % R, 0xFEDCBA09 % R
# (constraints, variables, mul_depth) per circuit; instances per circuit
SHAPES = {"one": ([(64, 60, 2)], [1]), "three": ([(64, 60, 2), (200, 300, 3), (1000, 700, 5)], [1, 2, 3])}


def _program(name, zk, srs=None):
    """the program's proving keys and assignments, set up on a known-trapdoor SRS (or on `srs`: (β powers, γβ powers))"""
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import synthetic_srs
    shapes, batch = SHAPES[name]
    rng = random.Random(len(shapes))
    circuits, assignments = [], []
    for (nc, nv, depth), b in zip(shapes, batch):
        zs = [dv.test_circuit_csr(rng.randrange(2, R), rng.randrange(2, R), depth, nc, nv, "cuda") for _ in range(b)]
        circuits.append(zs[0][0])
        assignments.append([z for _c, z in zs])
    D = max(c.info.max_degree(zk) for c in circuits) + 8
    powers, gpowers = srs or synthetic_srs(D, BETA, GAMMA)
    keys = dv.batch_circuit_setup(circuits, powers, gpowers, zk)
    return [(pk, zs) for (pk, _vk), zs in zip(keys, assignments)]


def _ints(t):
    from snarkvm_b200 import device
    h = device.fr_from_mont(t).cpu().numpy().view(np.uint64)
    return [sum(int(v) << (64 * i) for i, v in enumerate(row)) for row in h]


def _oracle(proof, program, order, change=None):
    """the verifier's transcript from the proof, the verifying keys and the public inputs (circuits in id order)"""
    from snarkvm_b200 import poseidon
    aff = vto.affine_of_image
    c = proof.commitments
    public = [[_ints(z[: program[k][0].circuit.num_public]) for z in program[k][1]] for k in order]
    vks = [[aff(x) for x in program[k][0].circuit_verifying_key.circuit_commitments] for k in order]
    if change == "public":
        public[-1][-1][1] = (public[-1][-1][1] + 1) % R
    elif change == "vk":
        vks[0][5] = vto.affine_of_image(program[order[1 % len(order)]][0].circuit_verifying_key.circuit_commitments[5]) \
            if len(order) > 1 else None
    view = {"w": [aff(x) for x in c.witness_commitments], "mask": None if c.mask_poly is None else aff(c.mask_poly),
            "h_0": aff(c.h_0), "g_1": aff(c.g_1), "h_1": aff(c.h_1), "g_a": [aff(x) for x in c.g_a_commitments],
            "g_b": [aff(x) for x in c.g_b_commitments], "g_c": [aff(x) for x in c.g_c_commitments], "h_2": aff(c.h_2),
            "third_sums": proof.third_sums, "fourth_sums": proof.fourth_sums, "evaluations": proof.evaluations.to_field_elements()}
    return vto.prove_batch_transcript(poseidon.parameters(poseidon.FIELD_FQ), proof.batch_sizes, public, vks, view)


def _flat(ch):
    """every challenge in transcript order"""
    out = [x for cc, inst in ch["batch_combiners"] for x in inst[1:] + ([cc] if cc != 1 else [])]
    out += [ch["alpha"], ch["eta_b"], ch["eta_c"], ch["beta"]] + [d for ds in ch["deltas"] for d in ds][1:] + [ch["gamma"]]
    return out + ch["opening"]


@pytest.fixture(scope="module", params=[("one", False), ("one", True), ("three", False), ("three", True)],
                ids=lambda p: f"{p[0]}-{'zk' if p[1] else 'plain'}")
def proved(request):
    from snarkvm_b200 import varuna as dv
    name, zk = request.param
    program = _program(name, zk)
    proof, ch, transcript = dv._prove_batch(program, zk, random.Random(7) if zk else None)
    order = dv.BatchProver([(pk.circuit, zs) for pk, zs in program]).positions
    return name, zk, program, order, proof, ch, transcript


def test_challenges_equal_the_verifiers_transcript(proved):
    _name, _zk, program, order, proof, ch, transcript = proved
    want, log, sponge = _oracle(proof, program, order)
    assert ch == want
    assert transcript.calls == 6 and transcript.permutations == sponge.permutations       # five rounds, openings
    for d in ("alpha", "beta", "gamma"):
        assert ch[d] != 0


def test_a_changed_input_changes_every_later_challenge(proved):
    _name, _zk, program, order, proof, ch, _t = proved
    base = _flat(ch)
    for change in ("public", "vk"):
        other = _flat(_oracle(proof, program, order, change)[0])
        assert len(other) == len(base)
        assert all(a != b for a, b in zip(base, other)), change


def _replay(program, ch, zk, rng):
    """a BatchProver driven by the given challenges: the rounds, one commit pass per round, the linear combinations, the openings.  In
    the hiding mode it draws from `rng` what prove_batch draws, in the same order: the mask polynomial (4, then 6 coefficients), then
    three blinding coefficients per hiding commitment in commitment order.  → (prover, commitments per round, blinding coefficients
    by label, lcs, query set, openings)"""
    import torch
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import LabeledPolynomial, Randomness, SonicKZG10
    p = dv.BatchProver([(pk.circuit, zs) for pk, zs in program])
    ck = dv._union_committer_key([program[k][0].committer_key for k in p.positions])
    combs = ch["batch_combiners"]
    draw = lambda n: [rng.randrange(R) for _ in range(n)]          # noqa: E731
    if zk:
        p.set_mask_poly(draw(4), draw(6))
    p.first_round(); p.assignments(); p.second_round(combs)
    p.third_round(ch["alpha"], ch["eta_b"], ch["eta_c"], combs)
    p.fourth_round(ch["alpha"], ch["beta"])
    p.fifth_round(ch["deltas"])
    rounds = p.labeled_oracles(zk)
    comms, rands, blind = {}, [], {}
    to_dev = lambda v: torch.from_numpy(np.array([dv._mont(x) for x in v], dtype=np.uint64).view(np.int64)).cuda()   # noqa: E731
    for r in sorted(rounds):
        for lp in rounds[r]:
            if lp.hiding_bound is not None:
                blind[lp.label] = draw(lp.hiding_bound + 2)
        c, rr = SonicKZG10.commit(ck, rounds[r], [to_dev(blind[lp.label]) if lp.label in blind else None for lp in rounds[r]])
        comms[r] = list(c)
        rands += rr
    lcs, qs = p.linear_combinations(ch["alpha"], ch["eta_b"], ch["eta_c"], ch["beta"], ch["deltas"], ch["gamma"], combs)
    polys = p.polynomials()
    ab = [LabeledPolynomial(k, v, None, None) for k, v in polys.items() if "_a_poly_" in k or "_b_poly_" in k]
    opened = SonicKZG10.open_combinations(ck, lcs, ab + [lp for r in sorted(rounds) for lp in rounds[r]],
                                          [Randomness() for _ in ab] + rands, qs, iter(ch["opening"]))
    return p, comms, blind, lcs, qs, opened


def _same(a, b) -> bool:
    return (a is None and b is None) or (a is not None and b is not None and bool((np.asarray(a) == np.asarray(b)).all()))


def _host_eval(coeffs, x):
    return sum(c * pow(x, i, R) for i, c in enumerate(coeffs)) % R


def test_replay_reproduces_the_proof_identities_and_openings(proved):
    """in both modes: the replay's commitments, sums, evaluations and openings equal the proof's; the three identities vanish at the
    derived challenges; every opening has its closed form on the known trapdoor, blinding included"""
    import torch
    from snarkvm_b200 import device
    from snarkvm_b200 import varuna as dv
    _name, zk, program, order, proof, ch, _t = proved
    p, comms, blind, lcs, qs, opened = _replay(program, ch, zk, random.Random(7))
    c = proof.commitments
    nw = sum(proof.batch_sizes)
    assert len(comms[1]) == nw + zk and all(_same(a, b) for a, b in zip(comms[1], c.witness_commitments))
    assert _same(comms[1][nw] if zk else None, c.mask_poly)
    assert _same(comms[2][0], c.h_0) and _same(comms[3][0], c.g_1) and _same(comms[3][1], c.h_1) and _same(comms[5][0], c.h_2)
    for i in range(len(order)):
        for m, got in enumerate((c.g_a_commitments, c.g_b_commitments, c.g_c_commitments)):
            assert _same(comms[4][3 * i + m], got[i])
    assert proof.third_sums == p.third_sums and proof.fourth_sums == p.fourth_sums
    assert proof.evaluations.g_1_eval == dv.BatchProver._eval(p.g_1, ch["beta"])
    assert [proof.evaluations.g_a_evals, proof.evaluations.g_b_evals, proof.evaluations.g_c_evals] == \
        [[dv.BatchProver._eval(gs[m], ch["gamma"]) for gs in p.gs] for m in range(3)]
    assert len(opened) == len(proof.pc_proof) == 3
    for (w, v), (pw, pv) in zip(opened, proof.pc_proof):
        assert _same(w, pw) and _same(v, pv)
    # the three AHP identities vanish at the derived challenges
    polys, points = p.polynomials(), dict(qs)
    for name in ("rowcheck_zerocheck", "lineval_sumcheck", "matrix_sumcheck"):
        x = points[name][1]
        assert sum(k * (1 if lab is None else dv.BatchProver._eval(polys[lab], x)) for k, lab in dict(lcs)[name]) % R == 0, name
    # each opening's closed form on the known trapdoor: w = ((p(β) − p(z)) + γ·(r(β) − r(z))) / (β − z) · G with p = Σ ξ_i·lc_i over
    # the point's linear combinations (labels in order), r = Σ ξ_i·(the lc's combination of blinding polynomials), ξ the opening
    # challenges; random_v = r(z)
    it = iter(ch["opening"])
    by_point = {}
    for lc, (pname, z) in qs:
        by_point.setdefault(pname, (z, []))[1].append(lc)
    ev = lambda terms, x: sum(k * dv.BatchProver._eval(polys[lab], x) for k, lab in terms if lab is not None) % R   # noqa: E731
    ev_r = lambda terms, x: sum(k * _host_eval(blind[lab], x) for k, lab in terms if lab in blind) % R             # noqa: E731
    hiding_points = 0
    for (pname, (z, labels)), (w, v) in zip(sorted(by_point.items()), proof.pc_proof):
        xis = [next(it) for _ in labels]
        next(it)
        terms = [dict(lcs)[lab] for lab in sorted(labels)]
        s = sum(xi * (ev(t, BETA) - ev(t, z)) for xi, t in zip(xis, terms)) % R
        r_z = sum(xi * ev_r(t, z) for xi, t in zip(xis, terms)) % R
        s = (s + GAMMA * sum(xi * (ev_r(t, BETA) - ev_r(t, z)) for xi, t in zip(xis, terms))) * pow(BETA - z, -1, R) % R
        scal = torch.from_numpy(np.array([[(s >> (64 * i)) & (2**64 - 1) for i in range(4)]], dtype=np.uint64).view(np.int64)).cuda()
        want = device.generator_mul(scal).cpu().numpy()[0]
        assert (dv._affine(w)[:97] == want[:97]).all(), pname
        if v is not None:
            hiding_points += 1
            assert dv._fr_mont_to_int(v) == r_z, pname
    # α opens only rowcheck_zerocheck (h_0, not hiding); β and γ open the hiding g_1 and g_M
    assert [v is not None for _w, v in proof.pc_proof] == [False, zk, zk] and hiding_points == 2 * zk


def _proof_equal(a, b) -> bool:
    ca, cb = a.commitments, b.commitments
    singles = ("mask_poly", "h_0", "g_1", "h_1", "h_2")
    lists = ("witness_commitments", "g_a_commitments", "g_b_commitments", "g_c_commitments")
    return (a.batch_sizes == b.batch_sizes and a.evaluations == b.evaluations and a.third_sums == b.third_sums
            and a.fourth_sums == b.fourth_sums and all(_same(getattr(ca, f), getattr(cb, f)) for f in singles)
            and all(len(getattr(ca, f)) == len(getattr(cb, f)) and all(_same(x, y) for x, y in zip(getattr(ca, f), getattr(cb, f)))
                    for f in lists)
            and len(a.pc_proof) == len(b.pc_proof) and all(_same(wa, wb) and _same(va, vb) for (wa, va), (wb, vb) in zip(a.pc_proof, b.pc_proof)))


def test_input_order_does_not_change_the_proof(proved):
    """the whole proof and every challenge, in both modes (the rng is drawn in commitment order, which follows the circuit ids)"""
    from snarkvm_b200 import varuna as dv
    name, zk, program, _order, proof, ch, _t = proved
    if name == "one":
        pytest.skip("a program of one circuit has one order")
    again, ch_again, _tr = dv._prove_batch(program[::-1], zk, random.Random(7) if zk else None)
    assert ch_again == ch and _proof_equal(again, proof)
    if zk:                                                                    # another blinding stream gives another proof
        assert not _proof_equal(again, dv.prove_batch(program, zk, random.Random(8)))


def _rowcheck_constant(proof, program, order, ch):
    """the constant term of rowcheck_zerocheck as a verifier forms it from the proof's third-round sums and the circuits' constraint
    domains: Σ_circuits cc · s_{R_i}(α) · Σ_j comb_j·(s_a·s_b − s_c), s_{R_i} the selector of R_i inside the largest R"""
    size = lambda n: 1 << max(n - 1, 0).bit_length()          # noqa: E731
    alpha = ch["alpha"]
    sizes = [size(program[k][0].circuit.num_constraints) for k in order]
    big = max(sizes)
    v = lambda n: (pow(alpha, n, R) - 1) % R                  # noqa: E731
    const = 0
    for n, (cc, inst), sums in zip(sizes, ch["batch_combiners"], proof.third_sums):
        sel = 1 if n == big else v(big) * n * pow(v(n) * big, -1, R) % R
        const += cc * sel * sum(comb * (s[0] * s[1] - s[2]) for comb, s in zip(inst, sums))
    return const % R, (-v(big)) % R


@pytest.mark.parametrize("name", ["one", "three"])
@pytest.mark.parametrize("zk", [False, True], ids=["plain", "zk"])
def test_mainnet_srs(name, zk):
    """on the mainnet 2^15 SRS (its β powers also stand in for the γ powers, which the fixture lacks): the challenges equal the
    verifier's transcript, and the α opening — rowcheck_zerocheck, which holds no degree-bounded or hiding polynomial — satisfies
    e(lhs, H) = e(w, β·H) with lhs = ξ·(c_h0·C_h0 + c·G) + α·w, where the verifier forms c and c_h0 from the proof's sums and the
    domains; a wrong constant fails the same check"""
    import os
    import torch
    from helpers import affine_array
    from oracle import bls12_377 as py
    from snarkvm_b200 import device
    from snarkvm_b200 import varuna as dv
    here = os.path.dirname(os.path.abspath(__file__))
    blob = open(os.path.join(here, "golden", "powers_of_beta_15.usrs"), "rb").read()
    powers = torch.from_numpy(affine_array(py.parse_usrs_points(blob, int.from_bytes(blob[:8], "little")))).cuda()
    with open(os.path.join(here, "golden", "beta_h.usrs"), "rb") as f:
        verifier = dv.UniversalVerifier.from_usrs(f.read())
    program = _program(name, zk, (powers, powers))
    proof, ch, _t = dv._prove_batch(program, zk, random.Random(5) if zk else None)
    order = dv.BatchProver([(pk.circuit, zs) for pk, zs in program]).positions
    assert _oracle(proof, program, order)[0] == ch
    const, c_h0 = _rowcheck_constant(proof, program, order, ch)
    xi, alpha = ch["opening"][0], ch["alpha"]
    w = proof.pc_proof[0][0]
    checks = []
    for c in (const, const + 1):
        bases = torch.from_numpy(np.stack([dv._affine(proof.commitments.h_0), verifier.g, dv._affine(w)])).cuda()
        scalars = torch.from_numpy(np.stack([dv._mont(xi * c_h0), dv._mont(xi * c), dv._mont(alpha)]).view(np.int64)).cuda()
        lhs = device.sonic_commit_batch([bases], [scalars])[0]
        checks += [dv._affine(lhs), dv._affine_neg(w)]
    g1 = torch.from_numpy(np.stack(checks)).cuda()
    _gt, is_one = device.pairing_products(g1, torch.tensor([0, 1, 0, 1], dtype=torch.int32, device="cuda"), verifier.prepared,
                                          torch.tensor([0, 2, 4], dtype=torch.int32, device="cuda"))
    assert is_one.cpu().tolist() == [True, False]
