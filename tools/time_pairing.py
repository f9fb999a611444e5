"""Time the BLS12-377 pairing on the device:
    prepare        device.g2_prepare of --prepare G2 points (per-point time reported)
    products       device.pairing_products of N two-pair checks e(s_i·G, H)·e(−s_i·G, H), N = 1, 64, 4096, 32767
    verify_vk      varuna.verify_vk_batch of the 32-circuit program of tools/time_program_setup.py (2^10 … 2^14 constraints),
                   without and with a UniversalVerifier (the difference is the pairing checks)
Every figure is host wall clock ending in a device synchronise (each call synchronises once), the median of --reps runs after one
warm-up run.  Prints the card and its power limit, then one JSON line per measurement.

    python tools/time_pairing.py [--reps 5] [--prepare 1024]
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


def median_ms(fn, reps):
    ts = []
    out = None
    for rep in range(reps + 1):
        t, out = timed(fn)
        if rep:
            ts.append(t)
    return statistics.median(ts) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--prepare", type=int, default=1024)
    args = ap.parse_args()
    import numpy as np
    import torch
    from snarkvm_b200 import device, varuna
    from snarkvm_b200.sonic_pc import synthetic_srs
    print(card(), flush=True)
    R = varuna.R_MOD

    g2 = device.generate_bases_g2(args.prepare, seed=7)
    ms, _ = median_ms(lambda: device.g2_prepare(g2), args.reps)
    print(json.dumps({"phase": "prepare", "points": args.prepare, "ms": round(ms, 3), "us_per_point": round(ms * 1e3 / args.prepare, 2),
                      "reps": args.reps}), flush=True)

    verifier = varuna.UniversalVerifier.synthetic(0x1234567890ABCDEF)
    for n in (1, 64, 4096, 32767):
        rng = random.Random(n)
        s = [rng.randrange(1, R) for _ in range(n)]
        limbs = np.array([[(v >> (64 * i)) & (2**64 - 1) for i in range(4)] for v in s], dtype=np.uint64)
        pts = device.generator_mul(torch.from_numpy(limbs.view(np.int64)).cuda()).cpu().numpy()
        g1 = np.repeat(pts, 2, axis=0)
        for k in range(n):                                            # −s·G: y ↦ q − y
            y = int.from_bytes(g1[2 * k + 1, 48:96].tobytes(), "little")
            g1[2 * k + 1, 48:96] = np.frombuffer(((varuna.Q_MOD - y) % varuna.Q_MOD).to_bytes(48, "little"), dtype=np.uint8)
        g1 = torch.from_numpy(g1).cuda()
        idx = torch.zeros(2 * n, dtype=torch.int32, device="cuda")
        starts = torch.arange(0, 2 * n + 1, 2, dtype=torch.int32, device="cuda")
        ms, (_gt, ones) = median_ms(lambda: device.pairing_products(g1, idx, verifier.prepared, starts), args.reps)
        assert bool(ones.all())
        print(json.dumps({"phase": "products", "checks": n, "pairs": 2 * n, "ms": round(ms, 3), "us_per_pairing": round(ms * 1e3 / (2 * n), 2),
                          "reps": args.reps}), flush=True)

    lgs = [10 + i % 5 for i in range(32)]
    base = [varuna.test_circuit_csr(3, 5, 2, 1 << lg, (1 << lg) - 10, "cuda")[0] for lg in lgs]
    srs = synthetic_srs(max(c.info.max_degree() for c in base), 0x1234567890ABCDEF, 0xFEDCBA09)
    rng = random.Random(1)
    ch = [[rng.randrange(R) for _ in range(12)] for _ in base]
    xi = [rng.randrange(R) for _ in base]
    keys = varuna.batch_circuit_setup(base, *srs, with_id=True)
    pks, vks = [pk for pk, _ in keys], [vk for _, vk in keys]
    certs = varuna.prove_vk_batch(pks, ch, [[x, 1] for x in xi])
    t_plain, t_verdict = [], []
    for rep in range(args.reps + 1):
        tp, plain = timed(lambda: varuna.verify_vk_batch(base, vks, certs, ch, xi))
        tv, verdict = timed(lambda: varuna.verify_vk_batch(base, vks, certs, ch, xi, verifier=verifier))
        if rep:
            t_plain.append(tp)
            t_verdict.append(tv)
    assert all(v.valid for v in verdict) and all((a.lhs == b.lhs).all() for a, b in zip(plain, verdict))
    print(json.dumps({"phase": "verify_vk_batch", "circuits": len(lgs), "log_constraints": "10-14",
                      "without_verifier_ms": round(statistics.median(t_plain) * 1e3, 2),
                      "with_verifier_ms": round(statistics.median(t_verdict) * 1e3, 2), "reps": args.reps}), flush=True)


if __name__ == "__main__":
    main()
