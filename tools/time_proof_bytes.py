"""Time varuna.proofs_from_bytes on the 8 compressed genesis proofs (tests/golden/varuna_bytes), repeated to 1, 64 and 4096 proofs
per call (12 G1 points each), validated.  Each call is split into the host walk (every blob's layout, every point's bytes gathered)
and the one k_g1_deserialize launch, timed with CUDA events alone, with validation and without (square root only); beside them
k_g1_validate alone on the decoded images, the Affine::check that validation adds.  Each figure is the median of --reps runs
after one warm-up.  Prints the card and its power limit, then one JSON line per proof count.

    python tools/time_proof_bytes.py [--proofs 1,64,4096] [--reps 5]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from time_circuit_setup import card  # noqa: E402


def _events(fn, reps):
    import torch
    fn()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return statistics.median(out)


def _clock(fn, reps):
    fn()
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        out.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--proofs", default="1,64,4096")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import numpy as np
    import torch
    from snarkvm_b200 import device
    from snarkvm_b200 import varuna as dv
    print(card())
    golden = os.path.join(ROOT, "tests", "golden", "varuna_bytes")
    proofs = []
    for k in range(8):
        with open(os.path.join(golden, f"genesis_proof_{k}.bin"), "rb") as f:
            proofs.append(f.read())
    for n in (int(v) for v in args.proofs.split(",")):
        blobs = [proofs[k % 8] for k in range(n)]

        def walk():
            points = []
            for b in blobs:
                dv._walk_proof(dv._Walk(b, 0, True, points))
            return points
        points = walk()
        raw = torch.from_numpy(np.frombuffer(b"".join(b for b, _f in points), dtype=np.uint8).copy()).cuda()
        images, status = device.g1_deserialize(raw, True, True)
        assert not status.any()
        row = {"proofs": n, "points": len(points),
               "from_bytes_ms": _clock(lambda: dv.proofs_from_bytes(blobs), args.reps),
               "host_walk_ms": _clock(walk, args.reps),
               "deserialize_validated_ms": _events(lambda: device.g1_deserialize(raw, True, True), args.reps),
               "deserialize_sqrt_only_ms": _events(lambda: device.g1_deserialize(raw, True, False), args.reps),
               "g1_validate_ms": _events(lambda: device.g1_validate(images), args.reps)}
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
