"""Time varuna.prove_batch against the same rounds, commitments, linear combinations and openings driven by constant challenges, the
two alternated in one process: each figure is the median of --reps runs after one warm-up run, host wall clock ending in a device
synchronise.  Non-hiding, TestCircuits of one instance each, known-trapdoor SRS, circuit ids computed before timing.  Programs:
    14, 16, 18    one TestCircuit of 2^lg constraints
    small         the 8 circuits of tools/time_batch_prove.py (2^10 … 2^14 constraints)
Prints the card and its power limit, then one JSON line per program with the transcript's device calls and permutations; the
transcript's cost is the difference of the two medians.

    python tools/time_prove_batch.py [--programs 14,16,18,small] [--reps 5]
"""
import argparse
import json
import os
import random
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_circuit_setup import card, timed  # noqa: E402

R = 8444461749428370424248824938781546531375899335154063827935233455917409239041
PROGRAMS = {"14": [14], "16": [16], "18": [18], "small": [10 + i % 5 for i in range(8)]}


def constant_rounds(program, ch):
    """prove_batch's device work with the challenges given: rounds, one commit pass per round, evaluations, openings"""
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import LabeledPolynomial, Randomness, SonicKZG10
    p = dv.BatchProver([(pk.circuit, zs) for pk, zs in program])
    ck = dv._union_committer_key([program[k][0].committer_key for k in p.positions])
    combs = ch["batch_combiners"]
    rounds, rands = {}, []
    steps = [lambda: (p.first_round(), p.assignments()), lambda: p.second_round(combs),
             lambda: p.third_round(ch["alpha"], ch["eta_b"], ch["eta_c"], combs), lambda: p.fourth_round(ch["alpha"], ch["beta"]),
             lambda: p.fifth_round(ch["deltas"])]
    for r, step in enumerate(steps, 1):
        step()
        rounds[r] = p.labeled_oracles(False, rounds=(r,))[r]
        rands += SonicKZG10.commit(ck, rounds[r])[1]
    lcs, qs = p.linear_combinations(ch["alpha"], ch["eta_b"], ch["eta_c"], ch["beta"], ch["deltas"], ch["gamma"], combs)
    [dv.BatchProver._eval(p.g_1, ch["beta"])] + [dv.BatchProver._eval(g, ch["gamma"]) for gs in p.gs for g in gs]
    polys = p.polynomials()
    ab = [LabeledPolynomial(k, v, None, None) for k, v in polys.items() if "_a_poly_" in k or "_b_poly_" in k]
    return SonicKZG10.open_combinations(ck, lcs, ab + [lp for r in sorted(rounds) for lp in rounds[r]], [Randomness() for _ in ab] + rands,
                                        qs, iter(ch["opening"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--programs", default="14,16,18,small")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import synthetic_srs
    print(card(), flush=True)
    for name in args.programs.split(","):
        lgs = PROGRAMS[name]
        rng = random.Random(len(lgs))
        circuits, zs = [], []
        for k, lg in enumerate(lgs):
            c, z = dv.test_circuit_csr(rng.randrange(2, R), rng.randrange(2, R), 2, (1 << lg) - k, (1 << lg) - 3 * k - 8, "cuda")
            circuits.append(c)
            zs.append([z])
        D = max(c.info.max_degree() for c in circuits) + 8
        powers, gpowers = synthetic_srs(D, 0x1234567, 0x89ABCDEF)
        program = [(pk, z) for (pk, _vk), z in zip(dv.batch_circuit_setup(circuits, powers, gpowers, with_id=True), zs)]
        _proof, ch, tr = dv._prove_batch(program)
        times = {"prove_batch": [], "constant": []}
        for rep in range(args.reps + 1):
            for key, fn in (("prove_batch", lambda: dv.prove_batch(program)), ("constant", lambda: constant_rounds(program, ch))):
                t, _ = timed(fn)
                if rep:
                    times[key].append(t)
        med = {k: round(1e3 * statistics.median(v), 1) for k, v in times.items()}
        print(json.dumps({"program": name, "circuits": len(lgs), "lg_constraints": lgs, "reps": args.reps,
                          "transcript_calls": tr.calls, "transcript_permutations": tr.permutations,
                          **{f"{k}_ms": v for k, v in med.items()},
                          "transcript_ms": round(med["prove_batch"] - med["constant"], 1)}), flush=True)


if __name__ == "__main__":
    main()
