"""Time varuna.prove_batch_many of P jobs against a loop of P prove_batch calls, the two alternated in one process: each figure is the
median of --reps runs after one warm-up run, host wall clock ending in a device synchronise.  Before timing, every proof of the
batched call is checked byte for byte against the loop's.  Non-hiding, known-trapdoor SRS, one instance per circuit, each job with
its own seeded assignments.  Programs:
    12, 14, 16    one TestCircuit of 2^lg constraints
    small         the 8 circuits of tools/time_prove_batch.py (2^10 … 2^14 constraints)
Prints the card and its power limit, then one JSON line per (program, P): proofs/s of both, the batched call's `stats` split, the
transcript's calls and permutations per job.  Also times one polynomial of 2^22 coefficients through device.poly_evaluate and
device.poly_divide_by_linear (one-segment calls of the batched kernels).

    python tools/time_prove_batch_many.py [--programs 12,14,16,small] [--batches 1,8,32] [--reps 3]
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
PROGRAMS = {"12": [12], "14": [14], "16": [16], "small": [10 + i % 5 for i in range(8)]}


def jobs_of(lgs, P):
    """P jobs of the program's circuits (set up once), each job with its own seeded assignments"""
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import synthetic_srs
    shapes = [((1 << lg) - k, (1 << lg) - 3 * k - 8) for k, lg in enumerate(lgs)]
    rng = random.Random(len(lgs))
    circuits = [dv.test_circuit_csr(rng.randrange(2, R), rng.randrange(2, R), 2, nc, nv, "cuda")[0] for nc, nv in shapes]
    D = max(c.info.max_degree() for c in circuits) + 8
    powers, gpowers = synthetic_srs(D, 0x1234567, 0x89ABCDEF)
    pks = [pk for pk, _vk in dv.batch_circuit_setup(circuits, powers, gpowers, with_id=True)]
    jobs = []
    for _p in range(P):
        jobs.append([(pk, [dv.test_circuit_csr(rng.randrange(2, R), rng.randrange(2, R), 2, nc, nv, "cuda")[1]])
                     for pk, (nc, nv) in zip(pks, shapes)])
    return jobs


def one_long_polynomial(lg=22, reps=20):
    """median ms of poly_evaluate and poly_divide_by_linear on 2^lg coefficients"""
    import numpy as np
    import torch
    from snarkvm_b200 import device, varuna as dv
    n = 1 << lg
    p = torch.from_numpy(np.random.default_rng(1).integers(0, 2**62, size=(n, 4), dtype=np.uint64).view(np.int64)).cuda()
    z = dv._mont(123456789)
    out = {}
    for name, fn in (("poly_evaluate", lambda: device.poly_evaluate(p, z)), ("poly_divide_by_linear", lambda: device.poly_divide_by_linear(p, z))):
        fn()
        out[f"{name}_2^{lg}_ms"] = round(1e3 * statistics.median(timed(fn)[0] for _ in range(reps)), 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--programs", default="12,14,16,small")
    ap.add_argument("--batches", default="1,8,32")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    from snarkvm_b200 import varuna as dv
    print(card(), flush=True)
    print(json.dumps(one_long_polynomial()), flush=True)
    for name in args.programs.split(","):
        lgs = PROGRAMS[name]
        for P in (int(x) for x in args.batches.split(",")):
            jobs = jobs_of(lgs, P)
            many = dv._prove_batch_many(jobs)
            loop = [dv.prove_batch(job) for job in jobs]
            assert [p.to_bytes() for p, _c, _t in many] == [p.to_bytes() for p in loop], f"{name} P={P}: proofs differ"
            times, stats = {"many": [], "loop": []}, []
            for rep in range(args.reps + 1):
                st = {}
                for key, fn in (("many", lambda: dv.prove_batch_many(jobs, stats=st)), ("loop", lambda: [dv.prove_batch(j) for j in jobs])):
                    t, _ = timed(fn)
                    if rep:
                        times[key].append(t)
                if rep:
                    stats.append(st)
            med = {k: statistics.median(v) for k, v in times.items()}
            split = {k: round(1e3 * statistics.median(s[k] for s in stats), 1) for k in ("transcript", "rounds", "commitments", "openings", "host")}
            tr = many[0][2]
            print(json.dumps({"program": name, "circuits": len(lgs), "lg_constraints": lgs, "P": P, "reps": args.reps, "checked": True,
                              "many_proofs_per_s": round(P / med["many"], 2), "loop_proofs_per_s": round(P / med["loop"], 2),
                              "many_ms": round(1e3 * med["many"], 1), "loop_ms": round(1e3 * med["loop"], 1),
                              "speedup": round(med["loop"] / med["many"], 2), "many_stats_ms": split,
                              "transcript_calls": stats[0]["transcript_calls"], "commitment_passes": stats[0]["commitment_passes"],
                              "transcript_permutations_per_job": tr.permutations}), flush=True)
            del jobs, many, loop


if __name__ == "__main__":
    main()
