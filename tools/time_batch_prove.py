"""Time Varuna proving of a whole program on the device: one K-circuit varuna.BatchProver run against a loop of one-circuit
runs (the BatchProver of one that varuna.Prover is) over the same circuits.  A run is the five rounds plus one SonicKZG10.commit pass per round (non-hiding, the
reference's degree bounds); the loop commits each circuit's rounds on their own.  Two programs of TestCircuits, one instance each:
    small   8 circuits of 2^10 … 2^14 constraints
    large   3 circuits of 2^16 … 2^18 constraints
Circuit ids are computed before timing, as setup would have done.  The loop and the batch alternate in one process; each figure is
the median of --reps runs after one warm-up run, host wall clock ending in a device synchronise.  Prints the card and its power limit,
then one JSON line per program.

    python tools/time_batch_prove.py [--programs small,large] [--reps 5]
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

PROGRAMS = {"small": [10 + i % 5 for i in range(8)], "large": [16, 17, 18]}
R = 8444461749428370424248824938781546531375899335154063827935233455917409239041


def prove(program, ck, ch, combs, deltas):
    """the rounds of one BatchProver over `program` and one commit pass per round → the commitments"""
    from snarkvm_b200 import varuna
    from snarkvm_b200.sonic_pc import SonicKZG10
    alpha, eta_b, eta_c, beta = ch
    p = varuna.BatchProver(program)
    comms = []
    steps = [lambda: (p.first_round(), p.assignments()), lambda: p.second_round(combs), lambda: p.third_round(alpha, eta_b, eta_c, combs),
             lambda: p.fourth_round(alpha, beta), lambda: p.fifth_round(deltas)]
    for r, step in enumerate(steps, 1):
        step()
        comms += list(SonicKZG10.commit(ck, p.labeled_oracles(label=lambda i, name, j=0: f"{i}_{name}_{j}", rounds=(r,))[r])[0])
    return comms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--programs", default="small,large")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    from snarkvm_b200 import varuna
    from snarkvm_b200.sonic_pc import CommitterKey, synthetic_srs
    print(card(), flush=True)
    for name in args.programs.split(","):
        lgs = PROGRAMS[name]
        rng = random.Random(len(lgs))
        program = []
        for k, lg in enumerate(lgs):
            c, z = varuna.test_circuit_csr(rng.randrange(2, R), rng.randrange(2, R), 2, (1 << lg) - k, (1 << lg) - 3 * k - 8, "cuda")
            program.append((c, [z]))
        varuna.circuit_ids([c for c, _ in program])
        D = 2 * max(1 << lg for lg in lgs) + 8
        powers, gpowers = synthetic_srs(D, 0x1234567, 0x89ABCDEF)
        bounds = sorted({b for c, _ in program for b in c.info.degree_bounds()})
        ck = CommitterKey.trim(powers, gpowers, supported_degree=D, supported_hiding_bound=1, enforced_degree_bounds=bounds)
        r = lambda: rng.randrange(2, R)          # noqa: E731
        ch = (r(), r(), r(), r())
        order = sorted(range(len(program)), key=lambda k: program[k][0].id())
        combs = {k: (r(), [r()]) for k in order}
        deltas = {k: [r(), r(), r()] for k in order}
        batch = lambda: prove(program, ck, ch, [combs[k] for k in order], [deltas[k] for k in order])       # noqa: E731
        loop = lambda: [c for k, e in enumerate(program) for c in prove([e], ck, ch, [combs[k]], [deltas[k]])]   # noqa: E731
        times = {"loop": [], "batch": []}
        for rep in range(args.reps + 1):
            t_loop, _ = timed(loop)
            t_batch, _ = timed(batch)
            if rep:
                times["loop"].append(t_loop)
                times["batch"].append(t_batch)
        print(json.dumps({"program": name, "circuits": len(lgs), "lg_constraints": lgs, "reps": args.reps,
                          "loop_ms": round(1e3 * statistics.median(times["loop"]), 1),
                          "batch_ms": round(1e3 * statistics.median(times["batch"]), 1)}), flush=True)


if __name__ == "__main__":
    main()
