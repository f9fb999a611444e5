"""Window-layout sweep of the resident G1 MSM (device.msm, CUDA events around whole calls), candidates alternated in one process.

    python tools/sweep_msm_windows.py --lg 22 23 24 --layouts 0 18*13,20 c20 --levels 4 5 6 [--rounds 3] [--reps 3]

A layout is "0" (today's uniform plan for the size), "cN" (uniform N-bit windows, SNARKVM_B200_MSM_C) or a width list for
SNARKVM_B200_MSM_WINDOWS ("18*13,20": 13 windows of 18 bits and a 20-bit top window); "-" as a level keeps the plan's own.
Every round times every (layout, levels) candidate once, in a rotated order; the table gives each candidate's median over the
rounds and its spread (max − min).  Results are checked against the first candidate's.  Prints the card and its power limit."""
import argparse
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ENV = ("SNARKVM_B200_MSM_C", "SNARKVM_B200_MSM_WINDOWS", "SNARKVM_B200_MSM_LEVELS")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as exc:  # noqa: BLE001
        return f"unknown ({exc!r})"


def set_layout(layout: str, levels: str):
    for k in ENV:
        os.environ.pop(k, None)
    if layout.startswith("c"):
        os.environ["SNARKVM_B200_MSM_C"] = layout[1:]
    else:
        os.environ["SNARKVM_B200_MSM_WINDOWS"] = layout
    if levels != "-":
        os.environ["SNARKVM_B200_MSM_LEVELS"] = levels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lg", type=int, nargs="+", default=[22, 23, 24])
    ap.add_argument("--layouts", nargs="+", default=["0", "18*13,20", "c20"])
    ap.add_argument("--levels", nargs="+", default=["4", "5", "6"])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3, help="calls per timing")
    args = ap.parse_args()

    import torch
    from snarkvm_b200 import device

    print(f"card: {card()}", flush=True)
    cands = [(lay, lev) for lay in args.layouts for lev in args.levels]
    for lg in args.lg:
        n = 1 << lg
        bases = device.generate_bases(n, 7)
        g = torch.Generator(device="cuda")
        g.manual_seed(lg)
        scal = torch.randint(-2**63, 2**63 - 1, (n, 4), dtype=torch.int64, device="cuda", generator=g)
        scal[:, 3] &= (1 << 60) - 1                                     # < r
        want = None
        times = {c: [] for c in cands}
        for c in cands:                                                 # warm-up, and the outputs must agree
            set_layout(*c)
            out = device.msm(bases, scal)
            torch.cuda.synchronize()
            if want is None:
                want = out
            assert (out == want).all(), (lg, c)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for r in range(args.rounds):
            order = cands[r % len(cands):] + cands[:r % len(cands)]
            for c in order:
                set_layout(*c)
                device.msm(bases, scal)                                 # the scratch pool settles at this plan's size
                torch.cuda.synchronize()
                e0.record()
                for _ in range(args.reps):
                    device.msm(bases, scal)
                e1.record()
                torch.cuda.synchronize()
                times[c].append(e0.elapsed_time(e1) / args.reps)
        best = min(cands, key=lambda c: statistics.median(times[c]))
        for c in cands:
            t = times[c]
            print(f"2^{lg}  layout={c[0]:<10} levels={c[1]:<2} median {statistics.median(t):8.2f} ms  spread {max(t) - min(t):5.2f} ms"
                  f"{'  <- best' if c == best else ''}", flush=True)
        del bases, scal
        torch.cuda.empty_cache()
    for k in ENV:
        os.environ.pop(k, None)


if __name__ == "__main__":
    main()
