"""Per-kernel time of one resident G1 MSM (the headline workload of bench.py at its default size), from torch.profiler.

    python tools/profile_msm_phases.py --lg 24 --out OUTDIR          (on the GPU; SNARKVM_B200_MSM_SCRATCH_GB sets the group count)

The MSM is first timed with CUDA events and the profiler off (median of --reps calls), then ONE call is traced with CUDA
activities.  Kernels are listed by name with their launch count, summed time and share of the traced call's kernel time.
OUTDIR receives the table (msm_phases_2^lg.md), the same rows as JSON and the Chrome trace.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
from torch.autograd import DeviceType  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from snarkvm_b200 import device  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # noqa: BLE001
        q = "power limit unknown"
    return f"{name}, {q}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lg", type=int, default=24)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", required=True)
    ap.add_argument("--tag", default="", help="appended to the output file names")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    os.makedirs(args.out, exist_ok=True)

    n = 1 << args.lg
    bases = device.generate_bases(n, seed=0xB200)
    g = torch.Generator(device="cuda")
    g.manual_seed(1234)
    scal = torch.randint(-2**63, 2**63 - 1, (n, 4), dtype=torch.int64, device="cuda", generator=g)
    scal[:, 3] &= (1 << 60) - 1
    for _ in range(3):
        device.msm(bases, scal)
    torch.cuda.synchronize()
    ms = []
    for _ in range(args.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        device.msm(bases, scal)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))

    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        device.msm(bases, scal)
        torch.cuda.synchronize()
    rows = {}
    for e in prof.events():
        if e.device_type != DeviceType.CUDA:
            continue
        r = rows.setdefault(e.name, [0, 0.0])
        r[0] += 1
        r[1] += e.time_range.elapsed_us() / 1e3
    total = sum(r[1] for r in rows.values())
    table = sorted(({"kernel": k, "launches": v[0], "ms": v[1], "share": v[1] / total} for k, v in rows.items()),
                   key=lambda r: -r["ms"])

    plan = device.msm_plan(n)
    head = (f"2^{args.lg}-point G1 MSM, {card()}; SNARKVM_B200_MSM_SCRATCH_GB={os.environ.get('SNARKVM_B200_MSM_SCRATCH_GB', 'unset')}; "
            f"plan {plan}; call {float(np.median(ms)):.2f} ms (median of {args.reps}, profiler off); traced kernels {total:.2f} ms")
    lines = [head, "", "| kernel | launches | ms | share |", "|---|---|---|---|"]
    lines += [f"| `{r['kernel'][:90]}` | {r['launches']} | {r['ms']:.2f} | {100 * r['share']:.1f} % |" for r in table]
    text = "\n".join(lines)
    print(text, flush=True)
    stem = os.path.join(args.out, f"msm_phases_2^{args.lg}{args.tag}")
    with open(stem + ".md", "w") as f:
        f.write(text + "\n")
    with open(stem + ".json", "w") as f:
        json.dump({"header": head, "call_ms": ms, "kernels": table}, f, indent=1)
    prof.export_chrome_trace(stem + ".trace.json")


if __name__ == "__main__":
    main()
