"""TEST INFRASTRUCTURE ONLY — CPU restatement (Python big integers) of the scalar side of VarunaSNARK::verify_batch, literal and in the
reference's order, with commitments kept symbolic (a commitment is {base label: scalar}, so a G1 sum is a dict sum):

    algorithms/src/snark/varuna/ahp/ahp.rs:172-445         construct_linear_combinations on the verifier's side (a_poly / b_poly
                                                           from the index commitments)                     → construct_linear_combinations
    algorithms/src/snark/varuna/ahp/selectors.rs           precompute_selectors                            → selector
    algorithms/src/fft/domain.rs:258-292                   evaluate_all_lagrange_coefficients              → lagrange_coefficients
    algorithms/src/polycommit/sonic_pc/mod.rs:477-544      check_combinations                              → check_combinations
    algorithms/src/polycommit/sonic_pc/mod.rs:344-411      batch_check                                     → batch_check
    algorithms/src/polycommit/sonic_pc/mod.rs:582-635      accumulate_elems                                → accumulate_elems

The output is check_elems' input: {degree bound or None: commitment}, the combined witness and the combined adjusted witness.  It
shares no code with snarkvm_b200/varuna.py.
"""
from __future__ import annotations

from oracle.bls12_377 import fr_root_of_unity

R = 8444461749428370424248824938781546531375899335154063827935233455917409239041
ONE = None                                                 # LCTerm::One


def size_of(n: int) -> int:
    return 1 if n <= 1 else 1 << (n - 1).bit_length()


def vanishing(size: int, x: int) -> int:
    return (pow(x, size, R) - 1) % R


def selector(max_size: int, size: int, x: int) -> int:
    """precompute_selectors' entry (max_domain.size, domain.size, x)"""
    return vanishing(max_size, x) * size % R * pow(vanishing(size, x) * max_size % R, -1, R) % R


def lagrange_coefficients(size: int, tau: int) -> list:
    """evaluate_all_lagrange_coefficients for τ outside the domain: L_i(τ) = v(τ)·ω^i / (n·(τ − ω^i))"""
    w = fr_root_of_unity(size)
    v = vanishing(size, tau)
    out, wi = [], 1
    for _ in range(size):
        out.append(v * wi % R * pow(size * (tau - wi) % R, -1, R) % R)
        wi = wi * w % R
    return out


class LC:
    """LinearCombination: a label and [(coefficient, term)], term a label or ONE"""

    def __init__(self, label, terms=()):
        self.label, self.terms = label, [(c % R, t) for c, t in terms]

    def add(self, c, t):
        self.terms.append((c % R, t))
        return self

    def add_scaled(self, c, other):                       # `+= (c, &other)`
        self.terms += [(c * k % R, t) for k, t in other.terms]

    def scale(self, c):                                   # `*= c`
        self.terms = [(c * k % R, t) for k, t in self.terms]

    def sub(self, other):                                 # `-= &other`
        self.terms += [((-k) % R, t) for k, t in other.terms]


def construct_linear_combinations(circuits: list, public_inputs: list, evals: dict, third_sums: list, fourth_sums: list, ch: dict,
                                  zk: bool) -> dict:
    """circuits: per circuit (id order) {'id': hex, 'info': (num_public, num_variables, num_constraints, nnz_a, nnz_b, nnz_c)};
    public_inputs: per circuit, per instance, the formatted padded input; evals: {lc label: value} of g_1 and every g_M"""
    infos = [c["info"] for c in circuits]
    R_max = max(size_of(i[2]) for i in infos)
    C_max = max(size_of(i[1]) for i in infos)
    K_max = max(size_of(n) for i in infos for n in i[3:])
    alpha, eta_b, eta_c, beta, gamma = ch["alpha"], ch["eta_b"], ch["eta_c"], ch["beta"], ch["gamma"]
    combiners = ch["batch_combiners"]
    batch_lineval_sum = sum(cc * sum(comb * (s[0] + eta_b * s[1] + eta_c * s[2]) for comb, s in zip(inst, sums))
                            for (cc, inst), sums in zip(combiners, third_sums)) % R * pow(C_max, -1, R) % R
    lcs = {}
    rowcheck = LC("rowcheck_zerocheck")
    for i, (cc, inst) in enumerate(combiners):
        circuit_term = LC("rowcheck_zerocheck term")
        for j, comb in enumerate(inst):
            s = third_sums[i][j]
            circuit_term.add_scaled(comb, LC("rowcheck term", [(s[0] * s[1] - s[2], ONE)]))
        circuit_term.scale(selector(R_max, size_of(infos[i][2]), alpha))
        rowcheck.add_scaled(cc, circuit_term)
    rowcheck.add(-vanishing(R_max, alpha), "h_0")
    lcs["rowcheck_zerocheck"] = rowcheck
    g_1 = LC("g_1", [(1, "g_1")])
    lineval = LC("lineval_sumcheck")
    if zk:
        lineval.add(1, "mask_poly")
    for i, (cc, inst) in enumerate(combiners):
        info = infos[i]
        lag = lagrange_coefficients(size_of(info[0]), beta)
        v_x = vanishing(size_of(info[0]), beta)
        circuit_term = LC("lineval_sumcheck term")
        sa, sb, sc = (fourth_sums[i][m] * size_of(info[3 + m]) % R for m in range(3))
        for j, comb in enumerate(inst):
            w_j = f"circuit_{circuits[i]['id']}_w_{j:08}"
            x_at_beta = sum(x * l for x, l in zip(public_inputs[i][j], lag)) % R
            term = LC("lineval term")
            term.add(sa * x_at_beta, ONE).add(sa * v_x, w_j)
            term.add(sb * eta_b * x_at_beta, ONE).add(sb * eta_b * v_x, w_j)
            term.add(sc * eta_c * x_at_beta, ONE).add(sc * eta_c * v_x, w_j)
            circuit_term.add_scaled(comb, term)
        circuit_term.scale(selector(C_max, size_of(info[1]), beta))
        lineval.add_scaled(cc, circuit_term)
    lineval.add(-vanishing(C_max, beta), "h_1").add(-beta * evals["g_1"], ONE).add(-batch_lineval_sum, ONE)
    lcs["g_1"] = g_1
    lcs["lineval_sumcheck"] = lineval
    matrix = LC("matrix_sumcheck")
    for i, c in enumerate(circuits):
        info = infos[i]
        v_rc = vanishing(size_of(info[2]), alpha) * vanishing(size_of(info[1]), beta) % R
        rc = size_of(info[2]) * size_of(info[1]) % R
        for m, name in enumerate("abc"):
            sel = selector(K_max, size_of(info[3 + m]), gamma)
            g_label = f"circuit_{c['id']}_g_{name}_{0:08}"
            g_m = LC(g_label, [(1, g_label)])
            a = LC("a", [(v_rc, f"circuit_{c['id']}_row_col_val_{name}")])
            b = LC("b", [(alpha * beta, ONE), (-alpha, f"circuit_{c['id']}_col_{name}"), (-beta, f"circuit_{c['id']}_row_{name}"),
                         (1, f"circuit_{c['id']}_row_col_{name}")])
            b.scale(rc)
            b.scale(gamma * evals[g_label] + fourth_sums[i][m])
            lhs = a
            lhs.sub(b)
            lhs.scale(sel)
            matrix.add_scaled(ch["deltas"][i][m], lhs)
            lcs[g_label] = g_m
    matrix.sub(LC("h_2", [(vanishing(K_max, gamma), "h_2")]))
    lcs["matrix_sumcheck"] = matrix
    return lcs


def _axpy(acc: dict, c: int, comm: dict) -> None:
    for k, v in comm.items():
        acc[k] = (acc.get(k, 0) + c * v) % R


def check_combinations(lcs: dict, commitments: dict, query_set: list, evaluations: dict, proof: list, challenges) -> tuple:
    """commitments: {label: (symbolic commitment, degree bound)}; query_set: [(lc label, (point name, point))]; evaluations: {(lc label,
    point): value}; proof: [(w label, random_v or None)] per point name in order; challenges: the sponge's short squeezes in order"""
    evaluations = dict(evaluations)
    lc_commitments = {}
    for lc in lcs.values():
        degree_bound, comm = None, {}
        for coeff, term in lc.terms:
            if term is ONE:
                for key in evaluations:
                    if key[0] == lc.label:
                        evaluations[key] = (evaluations[key] - coeff) % R
            else:
                cur, bound = commitments[term]
                if bound is not None:
                    assert len(lc.terms) == 1 and coeff == 1, "EquationHasDegreeBounds"
                    degree_bound = bound
                _axpy(comm, coeff, cur)
        lc_commitments[lc.label] = (comm, degree_bound)
    return batch_check(lc_commitments, query_set, evaluations, proof, challenges)


def batch_check(commitments: dict, query_set: list, values: dict, proof: list, challenges) -> tuple:
    query_to_labels = {}
    for label, (point_name, point) in query_set:
        query_to_labels.setdefault(point_name, (point, set()))[1].add(label)
    assert len(proof) == len(query_to_labels)
    randomizer = 1
    combined_comms, combined_witness, combined_adjusted_witness = {}, {}, {}
    for (_name, (query, labels)), p in zip(sorted(query_to_labels.items()), proof):
        comms = [commitments[label] for label in sorted(labels)]
        vals = [values[(label, query)] for label in sorted(labels)]
        accumulate_elems(combined_comms, combined_witness, combined_adjusted_witness, comms, query, vals, p, randomizer, challenges)
        randomizer = next(challenges)
    return combined_comms, combined_witness, combined_adjusted_witness


def accumulate_elems(combined_comms, combined_witness, combined_adjusted_witness, commitments, point, values, proof, randomizer,
                     challenges) -> None:
    combined_values = 0
    for (comm, degree_bound), value in zip(commitments, values):
        curr_challenge = next(challenges)
        combined_values = (combined_values + value * curr_challenge) % R
        _axpy(combined_comms.setdefault(degree_bound, {}), randomizer * curr_challenge, comm)
    w, random_v = proof
    bases, coeffs = [{"g": 1}, {w: R - 1}], [combined_values, point]
    if random_v is not None:
        bases.append({"gamma_g": 1})
        coeffs.append(random_v)
    _axpy(combined_witness, randomizer, {w: 1})
    for b, c in zip(bases, coeffs):
        _axpy(combined_adjusted_witness, c * randomizer, b)
