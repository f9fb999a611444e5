"""GPU: Varuna setup and verifying-key certificates for many circuits per call — index_circuits, batch_circuit_setup, prove_vk_batch
and verify_vk_batch — against the one-circuit functions byte for byte, against the CPU restatements, with a torch.profiler trace
that shows the shared launches, and the batched NTT (device.ntt_batch_) against ntt_ transform by transform."""
import os
import random
from collections import Counter

import numpy as np
import pytest

from oracle import bls12_377 as py
from oracle import sonic as osonic
from oracle import varuna as ov

import varuna_certificate_oracle as vco
import varuna_index_oracle as vio
from test_varuna_setup_gpu import _device_circuit, _oracle_circuit

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
R = ov.R
BETA, GAMMA = 0x1234567890ABCDEF1234567890ABCDEF % R, 0xFEDCBA0987654321FEDCBA % R

# a "program": TestCircuits from 2^4 to 2^12 constraints, circuit_0, random sparse R1CS (a different |K| per matrix; empty rows and a
# hot public column), and one circuit twice
PROGRAM = ["test_circuit_1_16_16", "test_circuit_3_100_70", "circuit_0", "sparse_one_public", "sparse_hot", "test_circuit_2_1024_1014",
           "test_circuit_5_3000_4096", "test_circuit_3_100_70"]


def _oracle(name, golden):
    if name == "sparse_hot":                                             # C not empty: its degree bound |K| − 2 must exist
        return ov.Circuit(vio.sparse_r1cs(1, 8, 300, 400, (512, 513, 2), (5, 300)))
    return _oracle_circuit(name, golden)


def _specs(circuits):
    return [(c.a, c.b, c.c, c.num_public, c.num_variables) for c in circuits]


@pytest.fixture(scope="module")
def program(golden):
    ocs = [_oracle(n, golden) for n in PROGRAM]
    return ocs, [_device_circuit(oc) for oc in ocs]


def _traced(fn, expected):
    """(fn(), Counter of the CUDA kernels it launched by name without namespace or parameters).  A profiling session can lose the
    first kernels launched after it starts (test_msm_paths_gpu.py meets the same), so every session runs the (deterministic) call
    once in a warm-up step, with the activity collection already on, and keeps only the second, active step.  A trace that still
    lacks any of the `expected` kernels is taken again."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile, schedule
    for _ in range(4):
        kept = []
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], schedule=schedule(wait=0, warmup=1, active=1),
                     on_trace_ready=lambda p: kept.append(list(p.events()))) as prof:
            fn()
            torch.cuda.synchronize()
            prof.step()                                                  # end of the warm-up step: nothing of it is kept
            out = fn()
            torch.cuda.synchronize()
            prof.step()                                                  # end of the active step: its trace is kept
        names = Counter()
        for e in (kept[-1] if kept else []):
            if e.device_type == DeviceType.CUDA:
                n = e.name.split("(")[0].strip()
                names[(n[5:] if n.startswith("void ") else n).replace("b200::", "")] += 1
        if all(names[k] for k in expected):
            break
    return out, names


def _batch_equals_loop(singles, powers, gamma, seed):
    """every batched result against the one-circuit functions; returns the batched (pks, vks, certs, checks, challenges, xis)"""
    import torch
    from snarkvm_b200 import varuna as dv
    batch = dv.index_circuits(_specs(singles))
    for c, s in zip(batch, singles):
        for a, b in zip(c.ariths, s.ariths):
            assert a.domain.size == b.domain.size
            for x, y in ((a.row, b.row), (a.col, b.col), (a.row_col_val, b.row_col_val)):
                assert torch.equal(x, y)
    polys = dv.index_polynomials(batch)
    for p, s in zip(polys, singles):
        want = s.index_polynomials()
        assert list(p) == list(want)
        assert all(torch.equal(p[k], want[k]) for k in want)
    keys = dv.batch_circuit_setup(batch, powers, gamma, with_id=True)
    rng = random.Random(seed)
    challenges = [[rng.randrange(R) for _ in range(12)] for _ in batch]
    openings = [[rng.randrange(R), rng.randrange(R)] for _ in batch]
    certs = dv.prove_vk_batch([pk for pk, _ in keys], challenges, [iter(o) for o in openings])
    checks = dv.verify_vk_batch(batch, [vk for _, vk in keys], certs, challenges, [o[0] for o in openings])
    for k, s in enumerate(singles):
        pk1, vk1 = dv.circuit_setup(s, powers, gamma, with_id=True)
        pk, vk = keys[k]
        assert pk.circuit is batch[k] and pk.circuit_verifying_key is vk
        assert vk.circuit_info == vk1.circuit_info and vk.id == vk1.id == s.id() and len(vk.id) == 32
        assert (vk.circuit_commitments == vk1.circuit_commitments).all(), k
        assert pk.committer_key.powers_of_beta_g.shape == pk1.committer_key.powers_of_beta_g.shape
        assert pk.committer_key.enforced_degree_bounds == pk1.committer_key.enforced_degree_bounds
        cert1 = dv.prove_vk(pk1, challenges[k], iter(openings[k]))
        assert (certs[k].w == cert1.w).all(), k
        check1 = dv.verify_vk(s, vk1, cert1, challenges[k], openings[k][0])
        assert checks[k].matches and check1.matches
        assert checks[k].evaluation == check1.evaluation
        assert (checks[k].lhs == check1.lhs).all() and (checks[k].w == certs[k].w).all()
    return batch, keys, certs, checks, challenges, openings


def test_batch_equals_loop_on_a_synthetic_srs(program, oracle_cpu):
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import synthetic_srs
    ocs, singles = program
    D = max(s.info.max_degree() for s in singles)
    powers, gamma = synthetic_srs(D, BETA, GAMMA)
    batch, keys, certs, checks, challenges, openings = _batch_equals_loop(singles, powers, gamma, 5)
    # the same Circuit object twice in one call, and a circuit whose id is already cached
    again = dv.batch_circuit_setup([batch[0], batch[0], batch[1]], powers, gamma, with_id=True)
    assert all((a[1].circuit_commitments == keys[k][1].circuit_commitments).all() and a[1].id == keys[k][1].id
               for a, k in zip(again, (0, 0, 1)))
    # lhs = β·W: e(lhs, H) = e(W, β·H) in the exponent
    for cert, check in zip(certs, checks):
        assert (check.lhs == oracle_cpu.g1_mul(vco.affine(cert.w), osonic._scalars([BETA])[0])).all()


def test_batch_against_the_oracles(program, oracle_cpu):
    """one batch of the smaller circuits: the commitments against varuna_index_oracle, W, the evaluations and lhs against
    varuna_certificate_oracle"""
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import synthetic_srs
    ocs, singles = program
    pick = [0, 1, 2, 3, 4, 7]
    powers, gamma = synthetic_srs(2047, BETA, GAMMA)
    hp, hg = powers.cpu().numpy(), gamma.cpu().numpy()
    batch = dv.index_circuits(_specs([singles[i] for i in pick]))
    keys = dv.batch_circuit_setup(batch, powers, gamma, with_id=True)
    rng = random.Random(11)
    challenges = [[rng.randrange(R) for _ in range(12)] for _ in pick]
    openings = [[rng.randrange(R), rng.randrange(R)] for _ in pick]
    certs = dv.prove_vk_batch([pk for pk, _ in keys], challenges, openings)
    checks = dv.verify_vk_batch(batch, [vk for _, vk in keys], certs, challenges, [o[0] for o in openings])
    g = np.frombuffer(py.affine_bytes(py.G1_GENERATOR), dtype=np.uint8)
    for k, i in enumerate(pick):
        oc = ocs[i]
        info, comms = vio.circuit_setup(oc, hp, hg, osonic.commit)
        assert keys[k][1].circuit_info == dv.CircuitInfo(*info)
        for got, want in zip(keys[k][1].circuit_commitments, comms):
            assert (got == want).all(), PROGRAM[i]
        assert keys[k][1].id == vco.circuit_id(oc)
        want_w = vco.prove_vk(hp, hg, oc, challenges[k], iter(openings[k]))
        assert (certs[k].w == want_w).all(), PROGRAM[i]
        matches, v, lhs = vco.verify_vk(oc, info, vco.circuit_id(oc), comms, want_w, g, challenges[k], openings[k][0])
        assert matches and checks[k].matches
        assert checks[k].evaluation == v
        assert (checks[k].lhs == lhs).all()
        assert (checks[k].lhs == oracle_cpu.g1_mul(vco.affine(certs[k].w), osonic._scalars([BETA])[0])).all()


def test_batch_equals_loop_on_the_real_srs(program):
    import torch
    from helpers import affine_array
    blob = open(os.path.join(HERE, "golden", "powers_of_beta_15.usrs"), "rb").read()
    powers = torch.from_numpy(affine_array(py.parse_usrs_points(blob, int.from_bytes(blob[:8], "little")))).cuda()
    _batch_equals_loop(program[1], powers, powers, 15)


def test_evaluations_with_points_inside_k(program):
    """evaluate_index_polynomials for a whole batch, with points inside each circuit's largest K (and outside), equals the loop"""
    from snarkvm_b200 import varuna as dv
    singles = program[1]
    rng = random.Random(4)
    combiners = [[1] + [rng.randrange(R) for _ in range(11)] for _ in singles]
    for inside in (False, True):
        points = []
        for s in singles:
            K = s.max_non_zero_domain
            w = py.fr_root_of_unity(K.size) if K.size > 1 else 1
            points.append(pow(w, rng.randrange(K.size), R) if inside else rng.randrange(R))
        got = dv.evaluate_index_polynomials(singles, points, combiners)
        assert got == [s.evaluate_index_polynomials(p, c) for s, p, c in zip(singles, points, combiners)]


def test_shared_work_is_shared(program):
    import torch
    from snarkvm_b200 import _lib, launch_count
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import synthetic_srs
    singles = program[1]
    K = len(singles)
    powers, gamma = synthetic_srs(max(s.info.max_degree() for s in singles), BETA, GAMMA)
    torch.cuda.synchronize()
    before = launch_count()
    dv.index_circuits(_specs(singles))
    assert launch_count() - before == 1                                  # the evaluations of all 3·K matrices, nothing else
    rng = random.Random(8)
    ch = [[rng.randrange(R) for _ in range(12)] for _ in range(K)]
    setup = lambda: dv.batch_circuit_setup(dv.index_circuits(_specs(singles)), powers, gamma, with_id=True)     # noqa: E731
    keys = setup()
    prove = lambda: dv.prove_vk_batch([pk for pk, _ in keys], ch, [[3, 4]] * K)             # noqa: E731
    certs = prove()
    verify = lambda: dv.verify_vk_batch([pk.circuit for pk, _ in keys], [vk for _, vk in keys], certs, ch, [3] * K)  # noqa: E731

    def deploy_and_verify():
        """a deployment and its verification: index, setup with ids, certificates, checks"""
        circuits = dv.index_circuits(_specs(singles))
        pks = [pk for pk, _ in dv.batch_circuit_setup(circuits, powers, gamma, with_id=True)]
        cs = dv.prove_vk_batch(pks, ch, [[3, 4]] * K)
        return dv.verify_vk_batch(circuits, [pk.circuit_verifying_key for pk in pks], cs, ch, [3] * K)
    checks, kern = _traced(deploy_and_verify, ["k_matrix_evals", "k_csr_serialize", "k_fr_lincomb", "k_lagrange_denominators"])
    assert all(c.matches for c in checks)
    assert kern["k_matrix_evals"] == 1 and kern["k_csr_transpose_scatter"] == 0, kern     # one launch for all 3·K matrices
    assert kern["k_csr_serialize"] == 1, kern                            # all ids at setup; verify finds them cached
    sizes = {s.non_zero_domains[j].size for s in singles for j in range(3)}
    # setup and prove_vk each interpolate all 12·K index polynomials: one launch per pass per size
    assert kern["k_ntt_pass<true>"] == 2 * sum(1 if n <= 1 << 11 else 2 for n in sizes) and kern["k_ntt_pass<false>"] == 0, kern
    assert kern["k_fr_lincomb"] == 1, kern
    assert kern["k_lagrange_denominators"] == 1 and kern["k_fr_batch_inverse"] == 1, kern
    assert kern["k_matrix_evals_dot"] == 1 and kern["k_fr_sum_segments"] == 1, kern
    # one MSM pass each: the bucket sort's profiling scope is recorded once per pass
    _lib.profile_enable(True)
    try:
        for fn in (setup, prove, verify):
            _lib.profile_collect(_lib.PROF_MSM_SORT)
            fn()
            assert _lib.profile_collect(_lib.PROF_MSM_SORT)[1] == 1
    finally:
        _lib.profile_enable(False)


def test_errors(program):
    import torch
    from snarkvm_b200 import CudaError, launch_count
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import synthetic_srs
    singles = program[1]
    D = max(s.info.max_degree() for s in singles)
    powers, gamma = synthetic_srs(D, BETA, GAMMA)
    torch.cuda.synchronize()
    before = launch_count()
    for fn in (lambda: dv.index_circuits([]), lambda: dv.batch_circuit_setup([], powers, gamma),
               lambda: dv.prove_vk_batch([], [], []), lambda: dv.verify_vk_batch([], [], [], [], []),
               lambda: dv.batch_circuit_setup(singles, powers[:D].contiguous(), gamma, with_id=True)):     # short for the largest only
        with pytest.raises(ValueError):
            fn()
    assert launch_count() == before
    small = dv.batch_circuit_setup(singles[:2], powers[: singles[1].info.max_degree() + 1].contiguous(), gamma)
    assert len(small) == 2
    # a bad column in matrix B of circuit 3 (of five), then a bad row_ptr in matrix C of circuit 2: the message names the circuit
    one = np.tile(dv._mont(1), (4, 1))
    ok = [dv.Matrix(np.arange(5), np.array([0, 1, 2, 3]), one, "cuda") for _ in range(3)]
    bad_col = dv.Matrix(np.arange(5), np.array([0, 5, 2, 8]), one, "cuda")
    specs = [(ok[0], ok[1], ok[2], 4, 8)] * 3 + [(ok[0], bad_col, ok[2], 4, 8)] + [(ok[0], ok[1], ok[2], 4, 8)]
    with pytest.raises(CudaError, match="circuit 3: matrix b"):
        dv.index_circuits(specs)
    circuits = dv.index_circuits([(ok[0], ok[1], ok[2], 4, 8)] * 4)
    bad_ptr = dv.Matrix(np.array([0, 1, 2, 1, 4]), np.array([0, 1, 2, 3]), one, "cuda")
    circuits[2] = dv.Circuit(ok[0], ok[1], ok[2], 4, 8)
    circuits[2].c = bad_ptr                                              # same evaluations' shape, a row_ptr that goes backwards
    with pytest.raises(CudaError, match="circuit 2: matrix c"):
        dv.circuit_ids(circuits)
    # a batch of one is the one-circuit function
    pk, vk = dv.batch_circuit_setup([singles[2]], powers, gamma, with_id=True)[0]
    pk1, vk1 = dv.circuit_setup(singles[2], powers, gamma, with_id=True)
    assert (vk.circuit_commitments == vk1.circuit_commitments).all() and vk.id == vk1.id
    # circuits on two devices
    if torch.cuda.device_count() > 1:
        c1 = dv.Circuit(*(dv.Matrix(np.arange(5), np.array([0, 1, 2, 3]), one, "cuda:1") for _ in range(3)), 4, 8)
        with pytest.raises(ValueError):
            dv.batch_circuit_setup([singles[0], c1], powers, gamma)


@pytest.mark.parametrize("direction", ["forward", "inverse"])
@pytest.mark.parametrize("ntt_type", ["standard", "coset"])
def test_ntt_batch_equals_ntt(direction, ntt_type):
    import torch
    from snarkvm_b200 import device
    from snarkvm_b200.cuda import NTTDirection, NTTType
    d = NTTDirection.Forward if direction == "forward" else NTTDirection.Inverse
    t = NTTType.Standard if ntt_type == "standard" else NTTType.Coset
    g = torch.Generator(device="cuda").manual_seed(7)

    def rand(lg):
        x = torch.randint(-2**63, 2**63 - 1, (1 << lg, 4), dtype=torch.int64, device="cuda", generator=g)
        x[:, 3] &= (1 << 60) - 1                                           # < r
        return x
    # 70 000 transforms of one size take two grid rows of at most 65 535
    for lgs in (list(range(21)) + [12, 0, 4, 20, 11, 13], [4] * 1000, [1] * 70000):
        xs = [rand(lg) for lg in lgs]
        want = [device.ntt_(x.clone(), d, t) for x in xs]
        got = device.ntt_batch_([x.clone() for x in xs], d, t)
        for lg, a, b in zip(lgs, got, want):
            assert torch.equal(a, b), lg
