"""Time Varuna circuit setup on the device in three phases, for TestCircuits of 2^16, 2^18 and 2^20 constraints on a synthetic SRS:
    circuit      varuna.Circuit(A, B, C, …): matrix_evals and the three transposes (the CSR arrays are already resident)
    interpolate  Circuit.index_polynomials(): twelve iFFTs over K
    commit       the one SonicKZG10.commit pass over the twelve index polynomials (trim included)
Each phase is host wall clock ending in a device synchronise; the median of --reps runs after one warm-up run.  On a tree whose
Circuit has no index_polynomials (before device circuit setup existed) only the circuit phase is timed.  Prints the card and its
power limit, then one JSON line per size.

    python tools/time_circuit_setup.py [--logs 16,18,20] [--reps 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card() -> str:
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # noqa: BLE001
        q = "power limit unknown"
    return f"{name}, power limit {q}"


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--logs", default="16,18,20")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    from snarkvm_b200 import varuna
    print(card(), flush=True)
    full = hasattr(varuna.Circuit, "index_polynomials")
    for lg in (int(x) for x in args.logs.split(",")):
        n = 1 << lg
        base, _z = varuna.test_circuit_csr(3, 5, 2, n, n - 10, "cuda")       # the CSR matrices, uploaded once
        build = lambda: varuna.Circuit(base.a, base.b, base.c, base.num_public, base.num_variables)   # noqa: E731
        phases = {"circuit": [], "interpolate": [], "commit": []}
        srs = None
        if full:
            from snarkvm_b200.sonic_pc import CommitterKey, LabeledPolynomial, SonicKZG10, synthetic_srs
            d = base.info.max_degree()
            srs = synthetic_srs(d, 0x1234567890ABCDEF, 0xFEDCBA09)
        for rep in range(args.reps + 1):
            t, circuit = timed(build)
            phases["circuit"].append(t)
            if full:
                t, polys = timed(circuit.index_polynomials)
                phases["interpolate"].append(t)
                info = circuit.info

                def commit():
                    ck = CommitterKey.trim(srs[0], srs[1], info.max_degree(), (), 1, info.degree_bounds())
                    return SonicKZG10.commit(ck, [LabeledPolynomial(k, p) for k, p in polys.items()])
                t, _ = timed(commit)
                phases["commit"].append(t)
            del circuit
        res = {"constraints": n, "nnz_per_matrix": base.a.nnz, "reps": args.reps}
        for k, v in phases.items():
            if v:
                res[f"{k}_ms"] = round(statistics.median(v[1:]) * 1e3, 2)
        print(json.dumps(res), flush=True)
        del base, srs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
