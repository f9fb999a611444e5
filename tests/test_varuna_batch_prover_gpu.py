"""GPU: varuna.BatchProver — several circuits in one proof — round by round against the CPU restatement
(tests/varuna_batch_prover_oracle.py) in both modes, its commitments and openings against oracle/sonic.py, the three identities and
every degree bound at 2^18 constraints, launches that do not grow with the number of circuits, its errors, and each new kernel
against its one-job counterpart."""
import copy
import random

import numpy as np
import pytest

from oracle import varuna as ov

import varuna_batch_prover_oracle as bpo
from test_varuna_batch_gpu import _traced
from test_varuna_setup_gpu import _device_circuit

pytestmark = pytest.mark.gpu
R = ov.R


def _z(cs):
    """the device assignment of a (padded) constraint system"""
    import torch
    from snarkvm_b200 import varuna as dv
    cs = copy.deepcopy(cs)
    ov.pad_input_for_indexer_and_prover(cs)
    return torch.from_numpy(np.array([dv._mont(v) for v in cs.public + cs.private], dtype=np.uint64).reshape(-1, 4).view(np.int64)).cuda()


def _test_circuit(rng, shape, batch):
    wit = [(rng.randrange(2, R), rng.randrange(2, R)) for _ in range(batch)]
    return ov.Circuit(ov.test_circuit(*wit[0], *shape)), [ov.test_circuit(a, b, *shape) for a, b in wit]


# a mixed program: TestCircuits of 2^4 to 2^12 constraints with 1–3 instances, circuit_0, satisfied sparse R1CS with a different |K|
# per matrix and a hot column (B's transpose has a row over 256 entries)
def _program(seed=1):
    rng = random.Random(seed)
    out = [_test_circuit(rng, (1, 16, 16), 1), _test_circuit(rng, (3, 7, 7), 2), _test_circuit(rng, (2, 1 << 10, (1 << 10) - 10), 3),
           _test_circuit(rng, (5, 3000, 1 << 12), 1)]
    for s, shape in ((5, (4, 60, 40)), (6, (8, 300, 600))):
        cs = bpo.satisfied_sparse_r1cs(s, *shape)
        out.append((ov.Circuit(copy.deepcopy(cs)), [copy.deepcopy(cs), copy.deepcopy(cs)]))
    return out


def _challenges(rng, n, batch):
    r = lambda: rng.randrange(2, R)          # noqa: E731
    return (r(), r(), r(), r(), r()), [(r(), [r() for _ in range(b)]) for b in batch], [[r(), r(), r()] for _ in range(n)]


def _run_device(dp, ch, combs, deltas, mask=None):
    alpha, eta_b, eta_c, beta, gamma = ch
    if mask is not None:
        dp.set_mask_poly(*mask)
    dp.first_round(); dp.assignments(); dp.second_round(combs)
    dp.third_round(alpha, eta_b, eta_c, combs)
    dp.fourth_round(alpha, beta)
    dp.fifth_round(deltas)
    return dp.linear_combinations(alpha, eta_b, eta_c, beta, deltas, gamma, combs)


@pytest.fixture(scope="module")
def mixed():
    from snarkvm_b200 import varuna as dv
    prog = _program()
    circuits = [_device_circuit(oc) for oc, _ in prog]
    ids = dv.circuit_ids(circuits)
    return prog, circuits, ids


@pytest.mark.parametrize("zk", [False, True])
def test_mixed_program_vs_restatement(mixed, zk):
    """every round polynomial (trimmed), every sum and every linear combination equal the restatement's; then one SonicKZG10.commit
    pass per round with the reference's bounds and open_combinations equal oracle/sonic.py on a known-trapdoor SRS"""
    import torch
    from oracle import sonic as osonic
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import CommitterKey, SonicKZG10, synthetic_srs
    prog, circuits, ids = mixed
    device_program = [(c, [_z(cs) for cs in inst]) for c, (_oc, inst) in zip(circuits, prog)]
    order = sorted(range(len(prog)), key=lambda k: ids[k])
    rng = random.Random(3 + zk)
    ch, combs, deltas = _challenges(rng, len(prog), [len(prog[k][1]) for k in order])
    mask = ([rng.randrange(R) for _ in range(4)], [rng.randrange(R) for _ in range(6)]) if zk else None
    dp = dv.BatchProver(device_program[::-1])                            # the input order does not matter
    assert dp.positions == [len(prog) - 1 - k for k in order]
    got_lcs, got_qs = _run_device(dp, ch, combs, deltas, mask)
    op, want_lcs, want_qs = bpo.run([(ids[k], oc, copy.deepcopy(inst)) for k, (oc, inst) in enumerate(prog)], ch, combs, deltas, mask)
    for i in range(len(prog)):
        assert [dv.trimmed(w) for w in dp.w_polys[i]] == op.w_polys[i]
        assert [dv.trimmed(z) for z in dp.z_polys[i]] == op.z_polys[i]
        assert [dv.trimmed(g) for g in dp.gs[i]] == op.gs[i], i
        assert [dv.trimmed(x) for x in dp.lhs[i]] == op.lhs[i], i
        assert dp.third_sums[i] == op.third_sums[i] and dp.fourth_sums[i] == op.fourth_sums[i], i
    for name in ("h_0", "g_1", "h_1", "h_2"):
        assert dv.trimmed(getattr(dp, name)) == getattr(op, name), name
    assert got_lcs == want_lcs and got_qs == want_qs
    dpolys, opolys = dp.polynomials(), op.polynomials()
    assert sorted(dpolys) == sorted(opolys)
    for k in opolys:
        assert dv.trimmed(dpolys[k]) == opolys[k], k
    # commitments: one pass per round with the reference's bounds, then the openings
    D = 2 * dp.max_constraint_domain.size + 16
    BETA, GAMMA = 0x1234567890ABCDEF % R, 0xFEDCBA09 % R
    powers, gpowers = synthetic_srs(D, BETA, GAMMA)
    rounds = dp.labeled_oracles(zk)
    labeled = [lp for r in sorted(rounds) for lp in rounds[r]]
    bounds = sorted({lp.degree_bound for lp in labeled if lp.degree_bound is not None})
    ck = CommitterKey.trim(powers, gpowers, supported_degree=D, supported_hiding_bound=1, enforced_degree_bounds=bounds)
    ock = osonic.CommitterKey(powers.cpu().numpy(), gpowers.cpu().numpy(), D, (), 1, bounds)
    to_dev = lambda v: torch.from_numpy(np.array([dv._mont(x) for x in v], dtype=np.uint64).reshape(-1, 4).view(np.int64)).cuda()   # noqa: E731
    blind = {lp.label: ([rng.randrange(R) for _ in range(3)] if lp.hiding_bound else None) for lp in labeled}
    comms, rands = [], []
    for r in sorted(rounds):
        c, rr = SonicKZG10.commit(ck, rounds[r], [None if blind[lp.label] is None else to_dev(blind[lp.label]) for lp in rounds[r]])
        comms += list(c); rands += list(rr)
    want, _ = osonic.commit(ock, [(lp.label, opolys[lp.label], lp.degree_bound, lp.hiding_bound, False) for lp in labeled],
                            [blind[lp.label] for lp in labeled])
    for i, lp in enumerate(labeled):
        assert (comms[i] == want[i]).all(), lp.label
    # the a / b polynomials are opened too (prove_batch gathers them first): committed here without bounds
    extra = _ab_labeled(dp, dpolys)
    _c, extra_rands = SonicKZG10.commit(ck, extra, [None] * len(extra))
    all_labeled = labeled + extra
    all_rands = rands + list(extra_rands)
    chal = [rng.randrange(1 << 128) for _ in range(len(got_lcs) + 3)]
    got = SonicKZG10.open_combinations(ck, got_lcs, all_labeled, all_rands, got_qs, iter(chal))
    want_open = osonic.open_combinations(ock, want_lcs, {k: (opolys[k], blind.get(k), next((lp.degree_bound for lp in labeled if lp.label == k), None))
                                                         for k in opolys}, want_qs, iter(chal))
    assert len(got) == len(want_open) == 3
    for (gw, gv), (ww, wv) in zip(got, want_open):
        assert (gw == ww).all()
        assert (gv is None) == (wv is None)


def _ab_labeled(dp, dpolys):
    from snarkvm_b200.sonic_pc import LabeledPolynomial
    return [LabeledPolynomial(k, v, None, None) for k, v in dpolys.items() if "_a_poly_" in k or "_b_poly_" in k]


def test_at_scale_identities_and_degree_bounds():
    """a TestCircuit of 2^18 constraints with two instances, one of 2^16 and a satisfied sparse R1CS of 2^14 (B's transpose holds a
    row of every constraint, cut into many segments): the three identities vanish, evaluated on the device, and every degree bound
    holds"""
    from snarkvm_b200 import varuna as dv
    rng = random.Random(18)
    c18a, z18a = dv.test_circuit_csr(rng.randrange(2, R), rng.randrange(2, R), 3, 1 << 18, 1 << 17, "cuda")
    _c, z18b = dv.test_circuit_csr(rng.randrange(2, R), rng.randrange(2, R), 3, 1 << 18, 1 << 17, "cuda")
    c16, z16 = dv.test_circuit_csr(rng.randrange(2, R), rng.randrange(2, R), 2, 1 << 16, 1 << 16, "cuda")
    cs = bpo.satisfied_sparse_r1cs(14, 8, 1 << 13, 1 << 14)
    c14 = _device_circuit(ov.Circuit(copy.deepcopy(cs)))
    dp = dv.BatchProver([(c14, [_z(cs)]), (c18a, [z18a, z18b]), (c16, [z16])])
    ch, combs, deltas = _challenges(rng, 3, dp.batch)
    lcs, qs = _run_device(dp, ch, combs, deltas)
    polys, points = dp.polynomials(), dict(qs)
    for name in ("rowcheck_zerocheck", "lineval_sumcheck", "matrix_sumcheck"):
        x = points[name][1]
        assert sum(coeff * (1 if lab is None else dv.BatchProver._eval(polys[lab], x)) for coeff, lab in dict(lcs)[name]) % R == 0, name
    deg = lambda p: len(dv.trimmed(p)) - 1          # noqa: E731
    Rm, Cm, Km = dp.max_constraint_domain.size, dp.max_variable_domain.size, dp.max_non_zero_domain.size
    assert deg(dp.h_0) <= 2 * Rm - 2 and deg(dp.g_1) <= Cm - 2 and deg(dp.h_1) <= 2 * Cm - 2 and deg(dp.h_2) <= Km - 2
    for c, gs in zip(dp.circuits, dp.gs):
        for g, d in zip(gs, c.non_zero_domains):
            assert deg(g) <= d.size - 2


def _same_size_program(n):
    """n different TestCircuits with equal domain sizes (R = C = K = 128)"""
    from snarkvm_b200 import varuna as dv
    rng = random.Random(n)
    out = []
    for k in range(n):
        c, z = dv.test_circuit_csr(rng.randrange(2, R), rng.randrange(2, R), 2, 100 + k, 90, "cuda")
        out.append((c, [z]))
    return out


def test_launches_do_not_grow_with_circuits():
    """kernel launches per round, by kernel name, are the same for 2 and for 8 circuits of the same domain sizes"""
    from snarkvm_b200 import launch_count
    from snarkvm_b200 import varuna as dv
    import torch
    expected = {2: ["k_polymul_load", "k_polymul_pointwise", "k_fr_lincomb"],
                3: ["k_sparse_matvec", "k_spmv_long_rows", "k_polymul_load", "k_fr_lincomb", "k_fr_convert"],
                4: ["k_round4_evals", "k_round4_f", "k_polymul_load", "k_fr_lincomb"], 5: ["k_fr_lincomb"]}
    counts = []
    for n in (2, 8):
        prog = _same_size_program(n)
        dv.circuit_ids([c for c, _ in prog])
        rng = random.Random(5)
        ch, combs, deltas = _challenges(rng, n, [1] * n)
        alpha, eta_b, eta_c, beta, _gamma = ch
        dp = dv.BatchProver(prog)
        dp.first_round(); dp.assignments()
        rounds = {2: lambda: dp.second_round(combs), 3: lambda: dp.third_round(alpha, eta_b, eta_c, combs),
                  4: lambda: dp.fourth_round(alpha, beta), 5: lambda: dp.fifth_round(deltas)}
        per = {}
        pad = torch.zeros(1, device="cuda")
        for r, fn in rounds.items():
            fn()                                                         # builds the cached transposes
            before = launch_count()
            fn()
            n_launch = launch_count() - before
            # a profiling session can lose the first kernels of its active step: a few torch launches go first
            _out, names = _traced(lambda: ([pad.add_(1) for _ in range(4)], fn()), expected[r])
            per[r] = (n_launch, {k: v for k, v in names.items() if k.startswith("k_")})
        counts.append(per)
    assert counts[0] == counts[1]


def test_errors_name_the_circuit(mixed):
    import torch
    from snarkvm_b200 import CudaError, launch_count
    from snarkvm_b200 import varuna as dv
    prog, circuits, _ids = mixed
    z0 = _z(prog[0][1][0])
    before = launch_count()
    with pytest.raises(ValueError, match="equal circuit ids"):
        dv.BatchProver([(circuits[0], [z0]), (circuits[0], [z0])])
    with pytest.raises(ValueError, match="circuit 1: instance does not match"):
        dv.BatchProver([(circuits[0], [z0]), (circuits[2], [z0])])
    assert launch_count() == before
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError, match="devices"):
            c1 = copy.copy(circuits[1])
            c1.a = copy.copy(c1.a)
            c1.a.row_ptr = c1.a.row_ptr.to("cuda:1")
            dv.BatchProver([(circuits[0], [z0]), (c1, [z0])])
    bad = _device_circuit(prog[4][0])
    bad.b.cols[3] = bad.num_variables + 7
    with pytest.raises(CudaError, match="circuit 1: matrix b"):
        dv.BatchProver([(circuits[0], [z0]), (bad, [_z(prog[4][1][0])])])


def test_kernels_match_their_one_job_counterparts(mixed):
    import torch
    from snarkvm_b200 import device
    from snarkvm_b200 import varuna as dv
    prog, circuits, _ids = mixed
    # segmented mat-vec (the transposes include long rows that cross segments) = sparse_matvec
    jobs = []
    for c, (_oc, inst) in zip(circuits, prog):
        z = _z(inst[0])
        jobs += [(m.row_ptr, m.cols, m.vals, z) for m in (c.a, c.b, c.c)]
        x = torch.randint(0, 1 << 62, (c.num_constraints, 4), dtype=torch.int64, device="cuda")
        x[:, 3] = 0
        jobs += [(t.row_ptr, t.cols, t.vals, x) for t in c.transposes]
    for out, (rp, cols, vals, x) in zip(device.sparse_matvec_batch(jobs), jobs):
        assert torch.equal(out, device.sparse_matvec(rp, cols, vals, x))
    # batched products = polymul, mixed sizes
    g = torch.Generator(device="cuda").manual_seed(1)
    rand = lambda n: torch.cat([torch.randint(0, 1 << 62, (n, 3), dtype=torch.int64, device="cuda", generator=g),      # noqa: E731
                                torch.zeros((n, 1), dtype=torch.int64, device="cuda")], 1)
    pairs = [(rand(a), rand(b)) for a, b in ((1, 1), (3, 5), (16, 16), (1000, 24), (4096, 4096), (7, 1))]
    for out, (a, b) in zip(device.polymul_batch(pairs), pairs):
        assert torch.equal(out, dv.polymul(a, b))
    # the uncapped lincomb (20 terms, offset views, repeated copies) = the axpy sequence
    polys = [rand(n) for n in (5, 64, 17, 1, 33) * 4]
    coeffs = [random.Random(k).randrange(R) for k in range(20)]
    terms, want = [], torch.zeros((256, 4), dtype=torch.int64, device="cuda")
    for k, (p, c) in enumerate(zip(polys, coeffs)):
        view = p[1:] if p.shape[0] > 1 else p
        off, reps, period = (k * 7) % 64, 1 + k % 3, 70
        terms.append((view, dv._mont(c), off, period, reps))
        for r in range(reps):
            lo = off + r * period
            seg = want[lo: lo + view.shape[0]]
            device.fr_vec_op(seg, device.fr_vec_op(view, dv._mont(c), device.FR_MUL), device.FR_ADD, out=seg)
    got = device.fr_lincomb_terms([(256, terms)])[0]
    assert torch.equal(got, want)
