"""Time the Varuna verifying-key certificate on the device, for TestCircuits of 2^16, 2^18 and 2^20 constraints on a synthetic SRS:
    id_kernel    Matrix.serialize() of A, B and C (k_csr_serialize), CUDA events
    id_d2h       the three byte streams copied to the host
    id_blake2s   hashlib.blake2s over CircuitInfo and the three streams (one host core)
    prove_vk     varuna.prove_vk: twelve iFFTs over K, the one-pass combination, the division by (x − z) and one |K|-point MSM
    verify_vk    varuna.verify_vk with the circuit id already cached, split into
                   index     varuna.Circuit(A, B, C, …): the re-indexing verify_vk needs (matrix_evals and transposes)
                   lagrange  the three K's Lagrange coefficients at the point
                   dots      the three matrix_evals_dot launches
                   msm       the 14-point MSM of lhs
Each phase is host wall clock ending in a device synchronise (id_kernel: CUDA events); the median of --reps runs after one warm-up
run.  Prints the card and its power limit, then one JSON line per size.

    python tools/time_certificate.py [--logs 16,18,20] [--reps 5]
"""
import argparse
import hashlib
import json
import os
import random
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_circuit_setup import card, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--logs", default="16,18,20")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import numpy as np
    import torch
    from snarkvm_b200 import device, varuna
    from snarkvm_b200.sonic_pc import synthetic_srs
    print(card(), flush=True)
    R = varuna.R_MOD
    rng = random.Random(1)
    for lg in (int(x) for x in args.logs.split(",")):
        n = 1 << lg
        base, _z = varuna.test_circuit_csr(3, 5, 2, n, n - 10, "cuda")
        srs = synthetic_srs(base.info.max_degree(), 0x1234567890ABCDEF, 0xFEDCBA09)
        pk, vk = varuna.circuit_setup(base, srs[0], srs[1], with_id=True)
        challenges = [rng.randrange(R) for _ in range(12)]
        xi = rng.randrange(R)
        point, combiners = challenges[-1], [1] + challenges[:-1]
        mats = (base.a, base.b, base.c)
        phases = {k: [] for k in ("id_kernel", "id_d2h", "id_blake2s", "prove_vk", "verify_vk", "index", "lagrange", "dots", "msm")}
        cert = None
        for rep in range(args.reps + 1):
            start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            start.record()
            streams = [m.serialize() for m in mats]
            stop.record()
            torch.cuda.synchronize()
            phases["id_kernel"].append(start.elapsed_time(stop) / 1e3)
            t, host = timed(lambda: [s.cpu().numpy() for s in streams])
            phases["id_d2h"].append(t)

            def blake():
                h = hashlib.blake2s(digest_size=32)
                h.update(base.info.to_bytes_le())
                for b in host:
                    h.update(b.data)
                return h.digest()
            t, digest = timed(blake)
            phases["id_blake2s"].append(t)
            assert digest == vk.id
            del streams, host
            t, cert = timed(lambda: varuna.prove_vk(pk, challenges, iter([xi, 1])))
            phases["prove_vk"].append(t)
            t, _ = timed(lambda: varuna.verify_vk(base, vk, cert, challenges, xi))
            phases["verify_vk"].append(t)
            t, circuit = timed(lambda: varuna.Circuit(base.a, base.b, base.c, base.num_public, base.num_variables))
            phases["index"].append(t)
            t, lags = timed(lambda: [a.domain.evaluate_all_lagrange_coefficients(point) for a in circuit.ariths])
            phases["lagrange"].append(t)
            t, _ = timed(lambda: [device.matrix_evals_dot(a.row, a.col, a.row_col_val, l) for a, l in zip(circuit.ariths, lags)])
            phases["dots"].append(t)
            bases = torch.zeros((14, device.AFFINE_STRIDE), dtype=torch.uint8, device="cuda")
            bases[:12] = torch.from_numpy(np.stack([varuna._affine(c) for c in vk.circuit_commitments])).cuda()
            bases[12] = device.generator_mul(torch.tensor([[1, 0, 0, 0]], dtype=torch.int64, device="cuda"))[0]
            bases[13] = torch.from_numpy(varuna._affine(cert.w)).cuda()
            sc = torch.from_numpy(np.array([[(s >> (64 * i)) & (2**64 - 1) for i in range(4)]
                                            for s in [xi * c % R for c in combiners] + [xi, point]], dtype=np.uint64).view(np.int64)).cuda()
            t, _ = timed(lambda: device.msm(bases, sc))
            phases["msm"].append(t)
            del circuit, lags
        res = {"constraints": n, "nnz_per_matrix": base.a.nnz, "K": base.max_non_zero_domain.size,
               "id_stream_bytes": sum(8 + 8 * m.nrows + 40 * m.nnz for m in mats), "reps": args.reps}
        for k, v in phases.items():
            res[f"{k}_ms"] = round(statistics.median(v[1:]) * 1e3, 2)
        print(json.dumps(res), flush=True)
        del base, srs, pk, vk, cert
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
