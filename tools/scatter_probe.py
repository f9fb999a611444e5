"""Where the level-0 record scatter of the resident G1 MSM spends its time (bench.py's headline shape).

    python tools/scatter_probe.py [--lg 24] [--plan 18*13,20] [--reps 7] [--out OUTDIR]       (on the GPU)

Builds tools/scatter_probe.cu with nvcc into a temporary directory, generates the bench inputs (2^lg bases from
device.generate_bases(seed=0xB200), scalars from bench.random_scalars(…, 1234)), and times seven variants of the scatter with
CUDA events, alternated round by round, median of --reps each:

  (a) as built: reads, digits, cursor atomics, barriers and the 96-byte records (six lanes per record)
  (b) (a) without the record stores
  (c) positions from one earlier run of (a) instead of the cursor atomics: reads and stores only
  (d) (c), every record one whole 128-byte line (x, ±y, 32 B of zeros) by eight lanes at a 128-byte stride
  (e) (c) at the 96-byte stride, two records of one slot pair written by the same instruction (synthetic pairing)
  (f) (a) with (d)'s 128-byte lines: cursor atomics and whole-line stores
  (g) (f) with evict-first stores (st.global.cs): the records stream past L2 instead of evicting the cursors

Prints the card and its power limit, then one row per variant: ms, ns per record, and the bytes the variant stores.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from snarkvm_b200 import device  # noqa: E402

VARIANTS = [("a", 0, "as built"), ("b", 1, "no record stores"), ("c", 2, "stores only (positions precomputed)"),
            ("d", 3, "stores only, 128-B lines"), ("e", 4, "stores only, 96 B, two records per instruction"),
            ("f", 6, "128-B lines with cursor atomics"), ("g", 7, "(f), evict-first stores")]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # noqa: BLE001
        q = "power limit unknown"
    return f"{name}, {q}"


def build(tmp):
    so = os.path.join(tmp, "scatter_probe.so")
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-shared", "-Xcompiler", "-fPIC",
                           "-o", so, os.path.join(ROOT, "tools", "scatter_probe.cu")])
    lib = ctypes.CDLL(so)
    lib.probe_hist.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_uint32,
                               ctypes.c_void_p, ctypes.c_void_p]
    lib.probe_scatter.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int,
                                  ctypes.c_int, ctypes.c_int, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                  ctypes.c_void_p]
    return lib


def parse_plan(s):
    low, top = s.split(",")
    c, k = (int(v) for v in low.split("*"))
    return c, k + 1, int(top)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lg", type=int, default=24)
    ap.add_argument("--plan", default="18*13,20", help="c*(windows-1),c_top as in SNARKVM_B200_MSM_WINDOWS")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    c, nwin, c_top = parse_plan(args.plan)
    nbuckets = 1 << (c - 1)
    nsets = nwin - 1 + (1 << (c_top - c))
    tb = nsets * nbuckets
    n = 1 << args.lg

    with tempfile.TemporaryDirectory() as tmp:
        lib = build(tmp)
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        bases = device.generate_bases(n, seed=0xB200)
        stride = bases.shape[1]
        scal = torch.from_numpy(bench.random_scalars(n, 1234).view(np.int64)).cuda()
        hist = torch.zeros(tb + 1, dtype=torch.int32, device="cuda")
        assert lib.probe_hist(scal.data_ptr(), n, c, c_top, nwin, nbuckets, hist.data_ptr(), stream) == 0
        start = torch.zeros(tb + 1, dtype=torch.int64, device="cuda")
        start[1:] = torch.cumsum(hist[:tb].to(torch.int64), 0)
        records = int(start[-1])
        start = start.to(torch.int32)
        cursors = torch.empty_like(start)
        pos = torch.empty(nwin * n, dtype=torch.int32, device="cuda")
        dense = torch.empty(records * 128 + 256, dtype=torch.uint8, device="cuda")

        def run(mode):
            cursors.copy_(start)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rc = lib.probe_scatter(mode, scal.data_ptr(), n, bases.data_ptr(), stride, c, c_top, nwin, nbuckets, cursors.data_ptr(),
                                   pos.data_ptr(), dense.data_ptr(), stream)
            e1.record()
            assert rc == 0, rc
            torch.cuda.synchronize()
            return e0.elapsed_time(e1)

        run(5)                                           # positions for (c)–(e), from the cursors exactly as (a) hands them out
        assert torch.equal(cursors[:tb], start[1:]), "cursors did not end at the next bucket's start"
        for _, mode, _ in VARIANTS:
            run(mode)                                    # warm-up
        ms = {k: [] for k, _, _ in VARIANTS}
        for _ in range(args.reps):
            for k, mode, _ in VARIANTS:
                ms[k].append(run(mode))

    stored = {"a": 96, "b": 0, "c": 96, "d": 128, "e": 96, "f": 128, "g": 128}
    head = (f"2^{args.lg} points, plan {args.plan} ({nwin} windows, {tb} buckets), {records} records; {card()}; "
            f"median of {args.reps}, alternated")
    lines = [head, "", "| variant | ms | ns per record | stored | GB/s stored |", "|---|---|---|---|---|"]
    rows = []
    for k, _, name in VARIANTS:
        m = float(np.median(ms[k]))
        rows.append({"variant": k, "what": name, "ms": m, "all_ms": ms[k]})
        lines.append(f"| ({k}) {name} | {m:.2f} | {m * 1e6 / records:.3f} | {records * stored[k] / 1e9:.1f} GB | "
                     f"{records * stored[k] / (m * 1e6):.0f} |")
    text = "\n".join(lines)
    print(text, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "scatter_probe.md"), "w") as f:
            f.write(text + "\n")
        with open(os.path.join(args.out, "scatter_probe.json"), "w") as f:
            json.dump({"header": head, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
