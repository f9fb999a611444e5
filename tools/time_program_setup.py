"""Time a whole program's Varuna setup and certificates on the device: a loop of one-circuit calls against one batched call, for
    index        varuna.Circuit per circuit               against varuna.index_circuits
    setup        varuna.circuit_setup per circuit         against varuna.batch_circuit_setup (no circuit id)
    setup_id     the same with with_id=True (the ids are cleared before every run)
    prove_vk     varuna.prove_vk per proving key          against varuna.prove_vk_batch
    verify_vk    varuna.verify_vk per circuit             against varuna.verify_vk_batch (ids cleared: a verifier hashes the circuit)
Two programs of TestCircuits (nnz = constraints per matrix) on a synthetic SRS:
    small   32 circuits of 2^10 … 2^14 constraints
    large    8 circuits of 2^16 … 2^18 constraints
Every phase is host wall clock ending in a device synchronise; the loop and the batch alternate in one process, and each figure is
the median of --reps runs after one warm-up run.  Both variants' outputs are compared.  Prints the card and its power limit, then one
JSON line per program and phase.

    python tools/time_program_setup.py [--programs small,large] [--reps 5]
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

PROGRAMS = {"small": [10 + i % 5 for i in range(32)], "large": [16 + i % 3 for i in range(8)]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--programs", default="small,large")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    from snarkvm_b200 import varuna
    from snarkvm_b200.sonic_pc import synthetic_srs
    print(card(), flush=True)
    R = varuna.R_MOD
    for name in args.programs.split(","):
        lgs = PROGRAMS[name]
        base = [varuna.test_circuit_csr(3, 5, 2, 1 << lg, (1 << lg) - 10, "cuda")[0] for lg in lgs]
        specs = [(c.a, c.b, c.c, c.num_public, c.num_variables) for c in base]
        srs = synthetic_srs(max(c.info.max_degree() for c in base), 0x1234567890ABCDEF, 0xFEDCBA09)
        rng = random.Random(1)
        ch = [[rng.randrange(R) for _ in range(12)] for _ in base]
        xi = [rng.randrange(R) for _ in base]

        def clear_ids():
            for c in base:
                c._id = None

        def setup_loop(with_id):
            clear_ids()
            return [varuna.circuit_setup(c, *srs, with_id=with_id) for c in base]

        def setup_batch(with_id):
            clear_ids()
            return varuna.batch_circuit_setup(base, *srs, with_id=with_id)

        keys = setup_batch(True)
        pks, vks = [pk for pk, _ in keys], [vk for _, vk in keys]
        certs = varuna.prove_vk_batch(pks, ch, [[x, 1] for x in xi])

        def verify_loop():
            clear_ids()
            return [varuna.verify_vk(c, vk, cert, h, x) for c, vk, cert, h, x in zip(base, vks, certs, ch, xi)]

        def verify_batch():
            clear_ids()
            return varuna.verify_vk_batch(base, vks, certs, ch, xi)

        phases = {
            "index": (lambda: [varuna.Circuit(*s) for s in specs], lambda: varuna.index_circuits(specs)),
            "setup": (lambda: setup_loop(False), lambda: setup_batch(False)),
            "setup_id": (lambda: setup_loop(True), lambda: setup_batch(True)),
            "prove_vk": (lambda: [varuna.prove_vk(pk, h, [x, 1]) for pk, h, x in zip(pks, ch, xi)],
                         lambda: varuna.prove_vk_batch(pks, ch, [[x, 1] for x in xi])),
            "verify_vk": (verify_loop, verify_batch),
        }
        for phase, (loop, batch) in phases.items():
            t_loop, t_batch = [], []
            for rep in range(args.reps + 1):
                tl, out_l = timed(loop)
                tb, out_b = timed(batch)
                if rep:
                    t_loop.append(tl)
                    t_batch.append(tb)
            if phase.startswith("setup"):
                assert all((a[1].circuit_commitments == b[1].circuit_commitments).all() and a[1].id == b[1].id for a, b in zip(out_l, out_b))
            elif phase == "prove_vk":
                assert all((a.w == b.w).all() for a, b in zip(out_l, out_b))
            elif phase == "verify_vk":
                assert all(a.matches and b.matches and a.evaluation == b.evaluation and (a.lhs == b.lhs).all() for a, b in zip(out_l, out_b))
            loop_ms, batch_ms = statistics.median(t_loop) * 1e3, statistics.median(t_batch) * 1e3
            print(json.dumps({"program": name, "circuits": len(lgs), "log_constraints": f"{min(lgs)}-{max(lgs)}", "phase": phase,
                              "loop_ms": round(loop_ms, 2), "batch_ms": round(batch_ms, 2), "speedup": round(loop_ms / batch_ms, 2),
                              "reps": args.reps}), flush=True)
        del base, specs, srs, keys, pks, vks, certs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
