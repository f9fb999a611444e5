"""GPU: varuna.prove_batch_many — many independent Varuna proofs per call, sharing each round's transcript call, commitment pass and
segmented kernels — and the three segmented entry points it adds: device.poly_evaluate_batch, device.poly_divide_by_linear_batch
and device.varuna_round4_evals_batch (round 4 with each segment's own α and β).

Kernels are checked against the one-polynomial calls and against big-integer Horner evaluation and division.  Proofs are checked
byte for byte against prove_batch of each job, non-hiding and hiding (seeded rngs), their challenges against
tests/varuna_transcript_oracle.py, the call counts in `stats`, and one verify_batch_many call over all of them."""
import random

import numpy as np
import pytest
import torch

import varuna_transcript_oracle as vto

pytestmark = pytest.mark.gpu
R = vto.R
BETA, GAMMA = 0x1234567890ABCDEF % R, 0xFEDCBA09 % R
# (constraints, variables, mul_depth) of the three circuits the jobs draw on
SHAPES = [(64, 60, 2), (200, 300, 3), (1000, 700, 5)]


def _mont_rows(vals):
    from snarkvm_b200 import varuna as dv
    return torch.from_numpy(np.array([dv._mont(v) for v in vals], dtype=np.uint64).reshape(-1, 4).view(np.int64)).cuda()


def _ints(t):
    from snarkvm_b200 import device
    if t.shape[0] == 0:
        return []
    h = device.fr_from_mont(t.contiguous()).cpu().numpy().view(np.uint64)
    return [sum(int(v) << (64 * i) for i, v in enumerate(row)) for row in h]


def _int(row):
    from snarkvm_b200.algorithms import _fr_mont_to_int
    return _fr_mont_to_int(row)


def _horner(coeffs, z):
    acc = 0
    for c in reversed(coeffs):
        acc = (acc * z + c) % R
    return acc


def _divide(coeffs, z):
    """(p − p(z)) / (x − z) by synthetic division → quotient coefficients, low degree first"""
    q, acc = [0] * max(len(coeffs) - 1, 0), 0
    for i in range(len(coeffs) - 1, 0, -1):
        acc = (acc * z + coeffs[i]) % R
        q[i - 1] = acc
    return q


LENGTHS = [0, 1, 2, 3, 15, 16, 17, 63, 64, 65, 255, 257, 4095, 4097, 16383, 16385, 1 << 20]


def _points():
    """a random point, zero, and points inside every domain of two or more elements (1 and −1)"""
    return [random.Random(3).randrange(R), 0, 1, R - 1]


@pytest.fixture(scope="module")
def polys():
    rng = random.Random(11)
    vals = {n: [rng.randrange(R) for _ in range(n)] for n in LENGTHS}
    return vals, {n: _mont_rows(v) for n, v in vals.items()}


def test_poly_evaluate_batch(polys):
    from snarkvm_b200 import device, varuna as dv
    vals, dev = polys
    jobs = [(dev[n], dv._mont(z), n, z) for z in _points() for n in LENGTHS]
    rng = random.Random(5)
    rng.shuffle(jobs)                                                      # a mix of lengths and points in one call
    got = device.poly_evaluate_batch([(t, zm) for t, zm, _n, _z in jobs])
    assert got.shape == (len(jobs), 4)
    for row, (t, zm, n, z) in zip(got, jobs):
        assert (row == device.poly_evaluate(t, zm)).all()
        assert _int(row) == _horner(vals[n], z), (n, z)
    assert device.poly_evaluate_batch([]).shape == (0, 4)
    assert (device.poly_evaluate_batch([(dev[0], dv._mont(5))]) == 0).all()


def test_poly_divide_by_linear_batch(polys):
    from snarkvm_b200 import device, varuna as dv
    vals, dev = polys
    jobs = [(dev[n], dv._mont(z), n, z) for z in _points() for n in LENGTHS]
    random.Random(6).shuffle(jobs)
    got = device.poly_divide_by_linear_batch([(t, zm) for t, zm, _n, _z in jobs])
    for q, (t, zm, n, z) in zip(got, jobs):
        assert q.shape == (max(n - 1, 0), 4)
        assert torch.equal(q, device.poly_divide_by_linear(t, zm))
        if n <= 4097:
            assert _ints(q) == _divide(vals[n], z), (n, z)
    # q·(x − z) + p(z) = p on a sample
    for q, (t, zm, n, z) in zip(got, jobs):
        if n in (2, 65, 1 << 20):
            qs, p = _ints(q), vals[n]
            pz = _horner(p, z)
            for i in random.Random(n).sample(range(n), min(n, 64)):
                lhs = ((qs[i - 1] if i >= 1 else 0) - z * (qs[i] if i < n - 1 else 0) + (pz if i == 0 else 0)) % R
                assert lhs == p[i], (n, i)
    assert device.poly_divide_by_linear_batch([]) == []


def test_round4_per_segment_challenges():
    """segments of three circuits, each with its own (α, β), equal varuna_round4_evals run per (α, β) group"""
    from snarkvm_b200 import device, varuna as dv
    rng = random.Random(21)
    circuits = [dv.test_circuit_csr(rng.randrange(2, R), rng.randrange(2, R), d, nc, nv, "cuda")[0] for nc, nv, d in SHAPES]
    groups = []
    for c in circuits:
        for _rep in range(2):
            alpha, beta = rng.randrange(R), rng.randrange(R)
            jobs = [(a.row, a.col, a.row_col_val, dv._mont(rng.randrange(R)), dv._mont(rng.randrange(R)), dv._mont(rng.randrange(R)))
                    for a in c.ariths]
            groups.append((jobs, alpha, beta))
    flat = [j + (dv._mont(a), dv._mont(b)) for jobs, a, b in groups for j in jobs]
    got = device.varuna_round4_evals_batch(flat)
    k = 0
    for jobs, a, b in groups:
        want = device.varuna_round4_evals(jobs, dv._mont(a), dv._mont(b))
        for trio_w in want:
            for x, y in zip(got[k], trio_w):
                assert torch.equal(x, y)
            k += 1
    # the shared-challenge entry point is a call of the same kernel: its results equal the old formula on the host
    jobs, a, b = groups[0]
    (ta, tb, tf), = device.varuna_round4_evals(jobs[:1], dv._mont(a), dv._mont(b))
    row, col, rcv = _ints(jobs[0][0]), _ints(jobs[0][1]), _ints(jobs[0][2])
    v_rc, rc, sc = (_int(np.asarray(x, dtype=np.uint64)) for x in jobs[0][3:6])
    for i in random.Random(1).sample(range(len(row)), 16):
        d = (row[i] - a) * (col[i] - b) % R
        assert _ints(ta[i: i + 1])[0] == v_rc * rcv[i] % R
        assert _ints(tb[i: i + 1])[0] == rc * d % R
        assert _ints(tf[i: i + 1])[0] == (sc * rcv[i] * pow(d, -1, R) % R if d else 0)


# ---- proofs ----

def _setup(zk):
    """three circuits set up on one known-trapdoor SRS (their committer keys trimmed to different degrees) and three assignments
    of each → (pks, assignments, D)"""
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import synthetic_srs
    rng = random.Random(len(SHAPES))
    circuits, assignments = [], []
    for nc, nv, depth in SHAPES:
        zs = [dv.test_circuit_csr(rng.randrange(2, R), rng.randrange(2, R), depth, nc, nv, "cuda") for _ in range(3)]
        circuits.append(zs[0][0])
        assignments.append([z for _c, z in zs])
    D = max(c.info.max_degree(True) for c in circuits) + 8
    powers, gpowers = synthetic_srs(D, BETA, GAMMA)
    keys = dv.batch_circuit_setup(circuits, powers, gpowers, zk, with_id=True)
    return [pk for pk, _vk in keys], [vk for _pk, vk in keys], assignments, D


def _jobs(pks, zs):
    """eight jobs: one circuit and several circuits per job, several instances, different constraint sizes, a job given twice"""
    A, B, C = pks
    return [[(A, [zs[0][0]])],
            [(A, zs[0][:2]), (B, zs[1][:1]), (C, zs[2])],
            [(C, zs[2][:1])],
            [(A, [zs[0][0]])],
            [(B, zs[1][:2])],
            [(B, zs[1][2:]), (A, zs[0][2:])],
            [(C, zs[2][1:])],
            [(A, zs[0][:2]), (B, zs[1][:1]), (C, zs[2])]]


@pytest.fixture(scope="module", params=[False, True], ids=["plain", "zk"])
def setup(request):
    zk = request.param
    pks, vks, zs, D = _setup(zk)
    return zk, pks, vks, zs, D, _jobs(pks, zs)


def _oracle(job, proof):
    """the verifier's transcript of one proof from its fields, the verifying keys and the public inputs (circuits in id order)"""
    from snarkvm_b200 import poseidon, varuna as dv
    order = dv.BatchProver([(pk.circuit, zs) for pk, zs in job]).positions
    aff = vto.affine_of_image
    c = proof.commitments
    public = [[_ints(z[: job[k][0].circuit.num_public]) for z in job[k][1]] for k in order]
    vks = [[aff(x) for x in job[k][0].circuit_verifying_key.circuit_commitments] for k in order]
    view = {"w": [aff(x) for x in c.witness_commitments], "mask": None if c.mask_poly is None else aff(c.mask_poly),
            "h_0": aff(c.h_0), "g_1": aff(c.g_1), "h_1": aff(c.h_1), "g_a": [aff(x) for x in c.g_a_commitments],
            "g_b": [aff(x) for x in c.g_b_commitments], "g_c": [aff(x) for x in c.g_c_commitments], "h_2": aff(c.h_2),
            "third_sums": proof.third_sums, "fourth_sums": proof.fourth_sums, "evaluations": proof.evaluations.to_field_elements()}
    return vto.prove_batch_transcript(poseidon.parameters(poseidon.FIELD_FQ), proof.batch_sizes, public, vks, view)[0]


@pytest.mark.parametrize("P", [1, 3, 8])
def test_proofs_equal_prove_batch(setup, P):
    from snarkvm_b200 import varuna as dv
    zk, _pks, _vks, _zs, _D, jobs = setup
    pick = {1: [1], 3: [0, 1, 2], 8: list(range(8))}[P]
    chosen = [jobs[k] for k in pick]
    stats = {}
    rngs = [random.Random(100 + k) for k in pick] if zk else None
    many = dv._prove_batch_many(chosen, zk, rngs, stats)
    assert len(many) == P
    assert stats["transcript_calls"] == 6 and stats["commitment_passes"] == 6
    for key in ("transcript", "rounds", "commitments", "openings"):
        assert stats[key] >= 0
    for k, job, (proof, ch, transcript) in zip(pick, chosen, many):
        want = dv.prove_batch(job, zk, random.Random(100 + k) if zk else None)
        assert proof.to_bytes() == want.to_bytes(), k
        assert ch == _oracle(job, proof)
        assert transcript.calls == 6
    assert [p.to_bytes() for p in dv.prove_batch_many(chosen, zk, [random.Random(100 + k) for k in pick] if zk else None)] == \
        [p.to_bytes() for p, _c, _t in many]


def test_one_verify_batch_many_accepts_every_proof(setup):
    from snarkvm_b200 import varuna as dv
    zk, _pks, vks, zs, D, jobs = setup
    proofs = dv.prove_batch_many(jobs, zk, [random.Random(7 + k) for k in range(len(jobs))] if zk else None)
    vk_of = {id(pk): vk for pk, vk in zip(_pks, vks)}
    batch = [([(vk_of[id(pk)], [_ints(z[: pk.circuit.num_public]) for z in assignments]) for pk, assignments in job], proof)
             for job, proof in zip(jobs, proofs)]
    bounds = [(1 << k) - 2 for k in range(1, D.bit_length() + 1) if (1 << k) - 2 <= D]
    verifier = dv.UniversalVerifier.synthetic(BETA, max_degree=D, gamma=GAMMA, bounds=bounds)
    assert dv.verify_batch_many(verifier, batch, zk) == [True] * len(jobs)


def test_errors_name_the_lowest_job(setup, monkeypatch):
    from snarkvm_b200 import varuna as dv
    zk, pks, _vks, zs, _D, jobs = setup
    with pytest.raises(ValueError, match="EmptyBatch"):
        dv.prove_batch_many([])
    with pytest.raises(ValueError, match="job 2: EmptyBatch"):
        dv.prove_batch_many([jobs[0], jobs[1], [], []])
    bad = [(pks[1], [zs[0][0]])]                                           # circuit B with an assignment of circuit A
    with pytest.raises(ValueError, match="job 1: circuit 0: instance does not match the index"):
        dv.prove_batch_many([jobs[0], bad, jobs[2], bad])
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError, match="job 1: .*one device"):
            dv.prove_batch_many([jobs[0], [(pks[0], [zs[0][0].to("cuda:1")])]])
    # a challenge inside its domain: the squeezes of α, then β, then γ give job 1 (and job 2) the value one
    real = dv.squeeze_many
    for call, name in ((2, "α"), (3, "β"), (5, "γ")):
        seen = [0]

        def fake(ts, counts, states, short=False, call=call):
            out = real(ts, counts, states, short)
            seen[0] += 1
            if seen[0] == call:
                for k in (1, 2):
                    out[k][0][0] = 1
            return out
        monkeypatch.setattr(dv, "squeeze_many", fake)
        with pytest.raises(ValueError, match=f"job 1: the vanishing polynomial of the largest domain is zero at {name}"):
            dv.prove_batch_many(jobs[:3], zk, [random.Random(k) for k in range(3)] if zk else None)
    monkeypatch.setattr(dv, "squeeze_many", real)
