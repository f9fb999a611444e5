"""Time varuna.verify_batch_many: P proofs per call (the same prove_batch proof P times, so every transcript does the same work) for
one-circuit programs of 2^14, 2^16 and 2^18 constraints and the 8-circuit program of tools/time_batch_prove.py (2^10 … 2^14), one
instance per circuit, non-hiding, on a known-trapdoor setup.  Each call is broken into its stages as verify_batch_many reports them
(validation, transcript, x(β), MSM pass, pairing, host), each ending in a device synchronise.  Each figure is the median of --reps
calls after one warm-up call.  Prints the card and its power limit, then one JSON line per (program, P) with the transcripts'
permutation count.

    python tools/time_verify_batch.py [--programs 14,16,18,small] [--proofs 1,16,256] [--reps 5]
"""
import argparse
import json
import os
import random
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_circuit_setup import card  # noqa: E402

PROGRAMS = {"14": [14], "16": [16], "18": [18], "small": [10 + i % 5 for i in range(8)]}
R = 8444461749428370424248824938781546531375899335154063827935233455917409239041
BETA, GAMMA = 0x1234567, 0x89ABCDEF


def _ints(t):
    import numpy as np
    from snarkvm_b200 import device
    h = device.fr_from_mont(t).cpu().numpy().view(np.uint64)
    return [sum(int(v) << (64 * i) for i, v in enumerate(row)) for row in h]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--programs", default="14,16,18,small")
    ap.add_argument("--proofs", default="1,16,256")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    from snarkvm_b200 import varuna
    from snarkvm_b200.sonic_pc import synthetic_srs
    print(card(), flush=True)
    for name in args.programs.split(","):
        lgs = PROGRAMS[name]
        rng = random.Random(len(lgs))
        circuits, zs = [], []
        for k, lg in enumerate(lgs):
            c, z = varuna.test_circuit_csr(rng.randrange(2, R), rng.randrange(2, R), 2, (1 << lg) - k, (1 << lg) - 3 * k - 8, "cuda")
            circuits.append(c)
            zs.append(z)
        D = max(c.info.max_degree() for c in circuits) + 8
        powers, gpowers = synthetic_srs(D, BETA, GAMMA)
        keys = varuna.batch_circuit_setup(circuits, powers, gpowers, with_id=True)
        proof = varuna.prove_batch([(pk, [z]) for (pk, _vk), z in zip(keys, zs)])
        kti = [(vk, [_ints(z[: c.num_public])]) for (_pk, vk), c, z in zip(keys, circuits, zs)]
        verifier = varuna.UniversalVerifier.synthetic(BETA, max_degree=D, bounds=[(1 << k) - 2 for k in range(1, D.bit_length())])
        for P in [int(p) for p in args.proofs.split(",")]:
            batch = [(kti, proof)] * P
            runs = []
            for rep in range(args.reps + 1):
                stats = {}
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                verdicts = varuna.verify_batch_many(verifier, batch, stats=stats)
                torch.cuda.synchronize()
                stats["total"] = time.perf_counter() - t0
                assert verdicts == [True] * P
                if rep:
                    runs.append(stats)
            med = {k: round(1e3 * statistics.median(r[k] for r in runs), 2)
                   for k in ("total", "validation", "transcript", "x_at_beta", "msm", "pairing", "host")}
            print(json.dumps({"program": name, "circuits": len(lgs), "lg_constraints": lgs, "proofs": P, "reps": args.reps,
                              "permutations_per_proof": runs[0]["permutations"][0], **{f"{k}_ms": v for k, v in med.items()},
                              "per_proof_ms": round(med["total"] / P, 3)}), flush=True)


if __name__ == "__main__":
    main()
