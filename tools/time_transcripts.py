"""Time the device Poseidon sponge and the certificates that draw their challenges from it:
    transcripts  device.poseidon_transcripts on 1, 32, 1024 and 32768 certificate-shaped transcripts (the op lists of
                 varuna.certificate_challenges for keys with random commitments: 40 absorbed Fq, 12 + 1 + 1 nonnative squeezes)
    prove_vk     varuna.prove_vk_batch for the 32-circuit "small" program of tools/time_program_setup.py, challenges given / derived
    verify_vk    varuna.verify_vk_batch(verifier=…) for the same program, challenges given / derived
Host wall clock around each call, ending in a device synchronise; the median of --reps runs after one warm-up run.  Also prints the
oracle's CPU time for one certificate transcript (oracle/poseidon.py, Python big integers) and its permutation count.  Prints the
card and its power limit first, then one JSON line per measurement.

    python tools/time_transcripts.py [--reps 5]
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

from time_circuit_setup import card, timed  # noqa: E402
from time_program_setup import PROGRAMS  # noqa: E402


def median_time(fn, reps):
    timed(fn)
    return statistics.median(timed(fn)[0] for _ in range(reps))


def random_keys(count, rng):
    import numpy as np
    from snarkvm_b200 import varuna
    Q = varuna.Q_MOD
    one = (1 << 384) % Q
    keys = []
    for _ in range(count):
        comms = np.zeros((12, 18), dtype=np.uint64)
        for i in range(12):
            for j in range(2):
                comms[i, 6 * j: 6 * j + 6] = np.frombuffer((rng.randrange(Q) * one % Q).to_bytes(48, "little"), dtype=np.uint64)
            comms[i, 12:18] = np.frombuffer(one.to_bytes(48, "little"), dtype=np.uint64)
        info = varuna.CircuitInfo(*(rng.randrange(1, 1 << 20) for _ in range(6)))
        keys.append(varuna.CircuitVerifyingKey(info, comms, bytes(rng.randrange(256) for _ in range(32))))
    return keys


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import numpy as np
    import torch
    from oracle import poseidon as op
    from snarkvm_b200 import device, poseidon, varuna
    from snarkvm_b200.sonic_pc import synthetic_srs
    print(card(), flush=True)
    rng = random.Random(1)

    # the oracle, one certificate transcript on the CPU
    key = random_keys(1, rng)[0]
    qinv = pow((1 << 384) % varuna.Q_MOD, -1, varuna.Q_MOD)
    affine = [tuple(int.from_bytes(row[6 * j: 6 * j + 6].tobytes(), "little") * qinv % varuna.Q_MOD for j in range(2))
              for row in key.circuit_commitments]
    params = poseidon.parameters(poseidon.FIELD_FQ, 2)
    t0 = time.perf_counter()
    s = op.certificate_sponge(varuna.Q_MOD, 377, params, key.circuit_info.to_bytes_le(), affine, key.id)
    op.certificate_challenges(s)
    cpu = time.perf_counter() - t0
    print(json.dumps({"what": "oracle_cpu_per_transcript", "device": "CPU (Python big integers)", "ms": round(cpu * 1e3, 3),
                      "permutations": s.permutations}), flush=True)
    assert varuna.certificate_challenges([key])[0] == op.certificate_challenges(
        op.certificate_sponge(varuna.Q_MOD, 377, params, key.circuit_info.to_bytes_le(), affine, key.id))

    for k in (1, 32, 1024, 32768):
        ops, op_start, inputs = varuna._certificate_transcripts(random_keys(k, rng) if k <= 1024 else random_keys(1024, rng) * 32)
        args_d = (torch.from_numpy(ops).cuda(), torch.from_numpy(op_start).cuda(), torch.from_numpy(inputs.view(np.int64)).cuda())
        t = median_time(lambda: device.poseidon_transcripts(poseidon.FIELD_FQ, *args_d, 0, 14 * k), args.reps)
        print(json.dumps({"what": "poseidon_transcripts", "transcripts": k, "ms": round(t * 1e3, 3),
                          "us_per_transcript": round(t * 1e6 / k, 3), "permutations_per_transcript": s.permutations}), flush=True)

    lgs = PROGRAMS["small"]
    base = [varuna.test_circuit_csr(3, 5, 2, 1 << lg, (1 << lg) - 10, "cuda")[0] for lg in lgs]
    srs = synthetic_srs(max(c.info.max_degree() for c in base), 0x1234567890ABCDEF, 0xFEDCBA09)
    verifier = varuna.UniversalVerifier.synthetic(0x1234567890ABCDEF)
    keys = varuna.batch_circuit_setup(base, *srs, with_id=True)
    pks, vks = [pk for pk, _ in keys], [vk for _, vk in keys]
    derived = varuna.certificate_challenges(vks)
    ch, opening = [d[0] for d in derived], [d[1] for d in derived]
    certs = varuna.prove_vk_batch(pks)
    assert all(a.w.tobytes() == b.w.tobytes() for a, b in zip(certs, varuna.prove_vk_batch(pks, ch, opening)))
    assert all(r.valid for r in varuna.verify_vk_batch(base, vks, certs, verifier=verifier))
    for name, fn in [("prove_vk_batch given", lambda: varuna.prove_vk_batch(pks, ch, opening)),
                     ("prove_vk_batch derived", lambda: varuna.prove_vk_batch(pks)),
                     ("verify_vk_batch given", lambda: varuna.verify_vk_batch(base, vks, certs, ch, [o[0] for o in opening], verifier)),
                     ("verify_vk_batch derived", lambda: varuna.verify_vk_batch(base, vks, certs, verifier=verifier)),
                     ("certificate_challenges", lambda: varuna.certificate_challenges(vks))]:
        t = median_time(fn, args.reps)
        print(json.dumps({"what": name, "circuits": len(base), "ms": round(t * 1e3, 3)}), flush=True)


if __name__ == "__main__":
    main()
