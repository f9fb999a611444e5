"""TEST INFRASTRUCTURE ONLY — CPU restatement (Python big integers) of the Varuna prover rounds for K circuits in one proof.

Restates /root/reference/algorithms/src/snark/varuna for several circuits, each with its own batch of instances, on top of
oracle/varuna.py's one-circuit primitives (Domain, poly_mul, divide_by_vanishing_poly, apply_randomized_selector, and its Prover for
the per-circuit init, first round and assignments):
    varuna.rs:336-620                          prove_batch: circuits ordered by id (ahp/indexer/circuit.rs:96-100)
    ahp/prover/round_functions/first.rs:102-127   one mask polynomial over the LARGEST variable domain (hiding mode)
    ahp/prover/round_functions/second.rs:76-142   h_0 = Σ apply_randomized_selector(comb_inst·rowcheck, comb_circuit, R_max, R_i, false)
    ahp/prover/round_functions/third.rs:126-218, 280-326   h_1, g_1 over C_max (remainder witness, source C_i)
    ahp/prover/round_functions/fourth.rs:79-245   per matrix, selector from K_matrix to the global K_max
    ahp/prover/round_functions/fifth.rs:43-67     h_2 = Σ δ·lhs over all 3K matrices in circuit order
    ahp/ahp.rs:173-389                         construct_linear_combinations for K circuits, with the selectors of selectors.rs
Values are canonical integers mod r; polynomials are trimmed coefficient lists.  Labels take a circuit's `label` (its id in hex on the
device; any distinct string here): circuit_{label}_{name}_{j:08} (ahp.rs:46-50), circuit_{label}_a_poly_{m} (ahp.rs:408-409).
"""
from oracle import varuna as ov

R = ov.R


def vanish(d: ov.Domain, x: int) -> int:
    return d.evaluate_vanishing_polynomial(x)


def selector(target: ov.Domain, src: ov.Domain, x: int) -> int:
    """selectors.rs: (v_target / v_src)·(|src| / |target|) at x"""
    if target.size == src.size:
        return 1
    return vanish(target, x) * src.size % R * pow(vanish(src, x) * target.size % R, -1, R) % R


def _largest(domains) -> ov.Domain:
    return max(domains, key=lambda d: d.size)


class BatchProver:
    """`program`: [(key, ov.Circuit, [ConstraintSystem, …])]; circuits are taken in key order (the device orders by circuit id)."""

    def __init__(self, program):
        program = sorted(program, key=lambda e: e[0])
        self.keys = [k for k, _c, _i in program]
        self.circuits = [c for _k, c, _i in program]
        self.provers = [ov.Prover(c, inst) for _k, c, inst in program]
        self.batch = [p.batch for p in self.provers]
        self.R = _largest(c.constraint_domain for c in self.circuits)
        self.C = _largest(c.variable_domain for c in self.circuits)
        self.K = _largest(c.max_non_zero_domain for c in self.circuits)
        self.mask_poly = None

    def label(self, i, name, j=0):
        key = self.keys[i].hex() if isinstance(self.keys[i], bytes) else str(self.keys[i])
        if name in ("a_poly", "b_poly"):
            return f"circuit_{key}_{name}_{'abc'[j]}"
        return f"circuit_{key}_{name}_{j:08}"

    def first_round(self):
        self.w_polys = [p.first_round() for p in self.provers]
        return self.w_polys

    def assignments(self):
        self.z_polys = [p.assignments() for p in self.provers]
        return self.z_polys

    def set_mask_poly(self, h_1_mask_rand, g_1_mask_rand):
        """first.rs:102-127 over the largest variable domain"""
        n = self.C.size
        mask = [0] * (n + 4)
        for i, c in enumerate(h_1_mask_rand):
            mask[n + i] = (mask[n + i] + c) % R
            mask[i] = (mask[i] - c) % R
        for i, c in enumerate(g_1_mask_rand):
            if i:
                mask[i] = (mask[i] + c) % R
        self.mask_poly = mask
        return mask

    def second_round(self, batch_combiners, strict: bool = True):
        """second.rs:76-142.  The reference stops on a non-zero remainder (an unsatisfied instance); strict=False keeps the quotient
        instead, so that a test can show the rowcheck identity then fails."""
        h_0 = []
        for c, p, (cc, inst) in zip(self.circuits, self.provers, batch_combiners):
            Rd = c.constraint_domain
            for comb, za, zb, zc in zip(inst, p.z_a, p.z_b, p.z_c):
                rowcheck = ov.poly_scale(ov.poly_sub(ov.poly_mul(Rd.ifft(za), Rd.ifft(zb)), Rd.ifft(zc)), comb)
                if strict:
                    h_i, _ = ov.apply_randomized_selector(rowcheck, cc, self.R, Rd, False)
                else:
                    h_i = ov.poly_scale(ov.divide_by_vanishing_poly(rowcheck, Rd)[0], cc * Rd.size % R * self.R.size_inv % R)
                h_0 = ov.poly_add(h_0, h_i)
        self.h_0 = h_0
        return h_0

    def third_round(self, alpha, eta_b, eta_c, batch_combiners):
        """third.rs:126-218, 280-326: target C_max, source C_i, remainder witness"""
        h_1, xg_1, self.third_sums = [], [], []
        for c, p, z_polys, (cc, inst) in zip(self.circuits, self.provers, self.z_polys, batch_combiners):
            Rd, V = c.constraint_domain, c.variable_domain
            l_at_alpha = Rd.evaluate_all_lagrange_coefficients(alpha)
            m_polys = []
            for mt in (ov.transpose(m, V, c.input_domain) for m in (c.a, c.b, c.c)):
                m_polys.append(V.ifft([sum(val * l_at_alpha[row] for val, row in col) % R for col in mt]))
            sums = []
            for comb, z_poly in zip(inst, z_polys):
                inst_sums = []
                for m_poly, eta in zip(m_polys, (1, eta_b, eta_c)):
                    z_m = ov.poly_mul(m_poly, z_poly)
                    inst_sums.append(sum(V.fft(z_m)) % R)
                    h_i, xg_i = ov.apply_randomized_selector(z_m, cc * comb % R * eta % R, self.C, V, True)
                    h_1, xg_1 = ov.poly_add(h_1, h_i), ov.poly_add(xg_1, xg_i)
                sums.append(inst_sums)
            self.third_sums.append(sums)
        if self.mask_poly is not None:
            h_mask, xg_mask = ov.divide_by_vanishing_poly(self.mask_poly, self.C)
            h_1, xg_1 = ov.poly_add(h_1, h_mask), ov.poly_add(xg_1, xg_mask)
        self.h_1, self.g_1 = h_1, ov.trim(xg_1[1:])
        return self.g_1, self.h_1

    def fourth_round(self, alpha, beta):
        """fourth.rs:79-245: each circuit's own v_{R_i}(α)·v_{C_i}(β), selector K_M → K_max"""
        self.gs, self.lhs, self.fourth_sums, self.a_polys, self.b_polys = [], [], [], [], []
        for c in self.circuits:
            Rd, V = c.constraint_domain, c.variable_domain
            v_rc = vanish(Rd, alpha) * vanish(V, beta) % R
            consts = v_rc * Rd.size_inv % R * V.size_inv % R
            gs, lhss, sums, a_polys, b_polys = [], [], [], [], []
            for arith in c.ariths:
                Kd = arith.domain
                a_poly = Kd.ifft([v_rc * v % R for v in arith.row_col_val])
                b_poly = Kd.ifft([Rd.size * V.size % R * ((alpha - r) * (beta - cc)) % R for r, cc in zip(arith.row, arith.col)])
                inv = [(alpha - r) * (beta - cc) % R for r, cc in zip(arith.row, arith.col)]
                inv = [0 if x == 0 else consts * pow(x, -1, R) % R for x in inv]
                f = Kd.ifft([i * v % R for i, v in zip(inv, arith.row_col_val)])
                lhs, _ = ov.apply_randomized_selector(ov.poly_sub(a_poly, ov.poly_mul(b_poly, f)), 1, self.K, Kd, False)
                gs.append(ov.trim(f[1:])); lhss.append(lhs); sums.append(f[0] if f else 0)
                a_polys.append(a_poly); b_polys.append(b_poly)
            self.gs.append(gs); self.lhs.append(lhss); self.fourth_sums.append(sums)
            self.a_polys.append(a_polys); self.b_polys.append(b_polys)
        return self.gs

    def fifth_round(self, deltas):
        h_2 = []
        for ds, lhss in zip(deltas, self.lhs):
            for d, lhs in zip(ds, lhss):
                h_2 = ov.poly_add(h_2, ov.poly_scale(lhs, d))
        self.h_2 = h_2
        return h_2

    def polynomials(self):
        out = {}
        for i in range(len(self.circuits)):
            for m in range(3):
                out[self.label(i, "a_poly", m)] = self.a_polys[i][m]
                out[self.label(i, "b_poly", m)] = self.b_polys[i][m]
                out[self.label(i, f"g_{'abc'[m]}")] = self.gs[i][m]
            for j, w in enumerate(self.w_polys[i]):
                out[self.label(i, "w", j)] = w
        if self.mask_poly is not None:
            out["mask_poly"] = ov.trim(self.mask_poly)
        out.update({"h_0": self.h_0, "g_1": self.g_1, "h_1": self.h_1, "h_2": self.h_2})
        return out

    def linear_combinations(self, alpha, eta_b, eta_c, beta, deltas, gamma, batch_combiners):
        """ahp.rs:173-389 for K circuits"""
        lcs = {}
        const = 0
        for c, (cc, inst), sums in zip(self.circuits, batch_combiners, self.third_sums):
            term = sum(comb * (s[0] * s[1] - s[2]) for comb, s in zip(inst, sums)) % R
            const = (const + cc * selector(self.R, c.constraint_domain, alpha) % R * term) % R
        lcs["rowcheck_zerocheck"] = [(const, None), ((-vanish(self.R, alpha)) % R, "h_0")]
        lcs["g_1"] = [(1, "g_1")]
        lineval = [(1, "mask_poly")] if self.mask_poly is not None else []
        total = 0
        for i, (c, p, (cc, inst)) in enumerate(zip(self.circuits, self.provers, batch_combiners)):
            sums4 = [s * a.domain.size % R for s, a in zip(self.fourth_sums[i], c.ariths)]
            weight = (sums4[0] + sums4[1] * eta_b + sums4[2] * eta_c) % R
            v_x, sel = vanish(c.input_domain, beta), selector(self.C, c.variable_domain, beta)
            for j, comb in enumerate(inst):
                k = cc * comb % R * sel % R
                lineval.append((k * weight % R * ov.poly_eval(p.x_polys[j], beta) % R, None))
                lineval.append((k * weight % R * v_x % R, self.label(i, "w", j)))
            total += cc * sum(comb * (s[0] + eta_b * s[1] + eta_c * s[2]) for comb, s in zip(inst, self.third_sums[i]))
        total = total % R * self.C.size_inv % R
        lineval += [((-vanish(self.C, beta)) % R, "h_1"), ((-beta * ov.poly_eval(self.g_1, beta)) % R, None), ((-total) % R, None)]
        lcs["lineval_sumcheck"] = lineval
        points = {"rowcheck_zerocheck": ("alpha", alpha), "g_1": ("beta", beta), "lineval_sumcheck": ("beta", beta),
                  "matrix_sumcheck": ("gamma", gamma)}
        matrix = []
        for i, c in enumerate(self.circuits):
            for m, (g, s, delta, a) in enumerate(zip(self.gs[i], self.fourth_sums[i], deltas[i], c.ariths)):
                g_label = self.label(i, f"g_{'abc'[m]}")
                lcs[g_label] = [(1, g_label)]
                points[g_label] = ("gamma", gamma)
                sel = selector(self.K, a.domain, gamma)
                b_term = (gamma * ov.poly_eval(g, gamma) + s) % R
                matrix.append((delta * sel % R, self.label(i, "a_poly", m)))
                matrix.append(((-delta * sel % R * b_term) % R, self.label(i, "b_poly", m)))
        matrix.append(((-vanish(self.K, gamma)) % R, "h_2"))
        lcs["matrix_sumcheck"] = matrix
        order = sorted(lcs)
        return [(k, lcs[k]) for k in order], [(k, points[k]) for k in order]

    def evaluate_lc(self, terms, point):
        polys = self.polynomials()
        return sum(coeff * (1 if label is None else ov.poly_eval(polys[label], point)) for coeff, label in terms) % R


def run(program, ch, combs, deltas, mask=None, strict=True):
    """all five rounds and the linear combinations → (prover, lcs, query_set)"""
    alpha, eta_b, eta_c, beta, gamma = ch
    p = BatchProver(program)
    if mask is not None:
        p.set_mask_poly(*mask)
    p.first_round(); p.assignments(); p.second_round(combs, strict)
    p.third_round(alpha, eta_b, eta_c, combs)
    p.fourth_round(alpha, beta)
    p.fifth_round(deltas)
    lcs, qs = p.linear_combinations(alpha, eta_b, eta_c, beta, deltas, gamma, combs)
    return p, lcs, qs


def satisfied_sparse_r1cs(seed: int, num_public: int, num_private: int, num_constraints: int, hot: bool = True) -> ov.ConstraintSystem:
    """a satisfied constraint system with general coefficients (as test_random_sparse_r1cs_vs_oracle builds one): A rows of 1–4
    entries, B rows of 1–3, and C one entry chosen so that every row holds; `hot` puts the One variable in every row of B, so B's
    transpose has one row with every constraint in it.  A, B and C then hold different numbers of entries (a different |K| each)."""
    import random
    rng = random.Random(seed)
    cs = ov.ConstraintSystem()
    for _ in range(num_public - 1):
        cs.alloc_input(rng.randrange(R))
    for _ in range(num_private):
        cs.alloc(rng.randrange(1, R))
    var = lambda: ("pub", rng.randrange(num_public)) if rng.random() < 0.2 else ("priv", rng.randrange(num_private))   # noqa: E731
    val = lambda v: cs.public[v[1]] if v[0] == "pub" else cs.private[v[1]]                                                # noqa: E731
    for _ in range(num_constraints):
        la = [(rng.randrange(1, R), var()) for _ in range(rng.randrange(1, 5))]
        lb = [(rng.randrange(1, R), var()) for _ in range(rng.randrange(1, 4))] + ([(rng.randrange(1, R), ("pub", 0))] if hot else [])
        az = sum(c * val(v) for c, v in la) % R
        bz = sum(c * val(v) for c, v in lb) % R
        j = ("priv", rng.randrange(num_private))
        cs.enforce(la, lb, [(az * bz % R * pow(val(j), -1, R) % R, j)])
    return cs
