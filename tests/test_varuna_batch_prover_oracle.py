"""CPU: the restatement of the K-circuit Varuna prover (tests/varuna_batch_prover_oracle.py) against the one-circuit restatement
(oracle/varuna.py) for one circuit, and the three identities the verifier checks (ahp.rs:62, 258, 340, 384) for programs of 2–4
circuits whose constraint, variable and non-zero domains all differ, in both modes."""
import copy
import random

import pytest

from oracle import varuna as ov

import varuna_batch_prover_oracle as bpo

R = ov.R


def _challenges(rng, program):
    r = lambda: rng.randrange(2, R)          # noqa: E731
    ch = (r(), r(), r(), r(), r())
    combs = [(r(), [r() for _ in inst]) for _k, _c, inst in sorted(program, key=lambda e: e[0])]
    deltas = [[r(), r(), r()] for _ in program]
    return ch, combs, deltas


def _test_circuit(rng, mul_depth, num_constraints, num_variables, batch):
    wit = [(rng.randrange(2, R), rng.randrange(2, R)) for _ in range(batch)]
    return ov.Circuit(ov.test_circuit(*wit[0], mul_depth, num_constraints, num_variables)), \
        [ov.test_circuit(a, b, mul_depth, num_constraints, num_variables) for a, b in wit]


def _sparse(seed, n_pub, n_prv, n_con, batch=1):
    cs = bpo.satisfied_sparse_r1cs(seed, n_pub, n_prv, n_con)
    return ov.Circuit(copy.deepcopy(cs)), [copy.deepcopy(cs) for _ in range(batch)]


@pytest.mark.parametrize("shape", [(3, 7, 7), (2, 100, 70), (5, 300, 512)])
def test_one_circuit_equals_the_one_circuit_restatement(shape):
    """for one circuit the restatement equals oracle.varuna.Prover round by round, linear combinations included (short labels mapped)"""
    rng = random.Random(shape[1])
    circuit, inst = _test_circuit(rng, *shape, 2)
    ch, combs, deltas = _challenges(rng, [(0, circuit, inst)])
    alpha, eta_b, eta_c, beta, gamma = ch
    mask = ([rng.randrange(R) for _ in range(4)], [rng.randrange(R) for _ in range(6)])
    p, lcs, qs = bpo.run([(0, circuit, copy.deepcopy(inst))], ch, combs, deltas, mask)
    o = ov.Prover(circuit, copy.deepcopy(inst))
    o.set_mask_poly(*mask)
    o.first_round(); o.assignments(); o.second_round(*combs[0])
    o.third_round(alpha, eta_b, eta_c, *combs[0])
    o.fourth_round(alpha, beta)
    o.fifth_round(deltas[0])
    assert p.w_polys[0] == o.w_polys and p.z_polys[0] == o.z_polys
    assert (p.h_0, p.g_1, p.h_1, p.h_2) == (o.h_0, o.g_1, o.h_1, o.h_2)
    assert p.gs[0] == o.gs and p.lhs[0] == o.lhs and p.third_sums[0] == o.third_sums and p.fourth_sums[0] == o.fourth_sums
    want_lcs, want_qs = o.linear_combinations(alpha, eta_b, eta_c, beta, deltas[0], gamma, *combs[0])
    short = {p.label(0, "w", j): f"w_{j}" for j in range(2)}
    short.update({p.label(0, n, m): f"{n}_{'abc'[m]}" for n in ("a_poly", "b_poly") for m in range(3)})
    short.update({p.label(0, f"g_{m}"): f"g_{m}" for m in "abc"})
    rename = lambda lst: sorted((short.get(k, k), [(c, short.get(t, t)) for c, t in v]) for k, v in lst)   # noqa: E731
    assert rename(lcs) == rename(want_lcs)
    assert sorted((short.get(k, k), v) for k, v in qs) == sorted(want_qs)


def _program(n):
    """n circuits whose R, C and K all differ (TestCircuits and satisfied sparse R1CS with a hot column)"""
    rng = random.Random(n)
    shapes = [lambda: _test_circuit(rng, 2, 20, 14, 2), lambda: _sparse(3, 4, 60, 40), lambda: _test_circuit(rng, 3, 130, 100, 1),
              lambda: _sparse(4, 8, 150, 300, 2)]
    return [(k, *shapes[k]()) for k in range(n)]


def _check_identities(p, lcs, qs):
    points = dict(qs)
    for name in ("rowcheck_zerocheck", "lineval_sumcheck", "matrix_sumcheck"):
        assert p.evaluate_lc(dict(lcs)[name], points[name][1]) == 0, name


@pytest.mark.parametrize("n", [2, 3, 4])
@pytest.mark.parametrize("zk", [False, True])
def test_identities_vanish_for_several_circuits(n, zk):
    program = _program(n)
    sizes = [(c.constraint_domain.size, c.variable_domain.size, c.max_non_zero_domain.size) for _k, c, _i in program]
    for dim in range(3):
        assert len({s[dim] for s in sizes[:2]}) == 2                    # every selector has target ≠ source somewhere
    rng = random.Random(10 * n + zk)
    ch, combs, deltas = _challenges(rng, program)
    mask = ([rng.randrange(R) for _ in range(4)], [rng.randrange(R) for _ in range(6)]) if zk else None
    p, lcs, qs = bpo.run(program, ch, combs, deltas, mask)
    _check_identities(p, lcs, qs)


def test_unsatisfied_instance_breaks_the_rowcheck():
    program = _program(3)
    k, c, inst = program[1]
    bad = copy.deepcopy(inst)
    bad[0].private[0] = (bad[0].private[0] + 1) % R
    program[1] = (k, c, bad)
    rng = random.Random(99)
    ch, combs, deltas = _challenges(rng, program)
    with pytest.raises(AssertionError, match="non-zero remainder"):             # the reference's prover stops here (second.rs)
        bpo.run(copy.deepcopy(program), ch, combs, deltas)
    p, lcs, qs = bpo.run(program, ch, combs, deltas, strict=False)
    assert p.evaluate_lc(dict(lcs)["rowcheck_zerocheck"], ch[0]) != 0


def test_input_order_does_not_change_the_result():
    program = _program(3)
    rng = random.Random(7)
    ch, combs, deltas = _challenges(rng, program)
    a = bpo.run(copy.deepcopy(program), ch, combs, deltas)
    b = bpo.run(copy.deepcopy(program[::-1]), ch, combs, deltas)
    assert a[1] == b[1] and a[2] == b[2]
    assert a[0].polynomials() == b[0].polynomials()
