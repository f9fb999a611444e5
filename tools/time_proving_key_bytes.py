"""Time the byte form of Varuna proving keys on keys shaped like two mainnet credits.aleo keys: `transfer_public` (12 326
constraints, |K| up to 2^16) and `inclusion` (134 767 constraints, |K| up to 2^19).  Each key is built with exactly the CircuitInfo
of the mainnet key (random CSR entries, one synthetic known-trapdoor SRS), set up in the hiding mode, so its bytes are as long as
the mainnet `.prover` file minus its version byte (checked).  Per key: to_bytes and from_bytes end to end (host clock, ending in a
synchronisation), the host header walk with its three row walks, the row walks alone, the upload, the Fr record decode and the 97-byte
G1 decode with and without validation (CUDA events), and the SHA-256 and Blake2s over the bytes as read (host clock).  Each figure
is the median of --reps runs after one warm-up.  Prints the card and its power limit, then one JSON line per key.

    python tools/time_proving_key_bytes.py [--keys transfer_public,inclusion] [--reps 5]
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

# CircuitInfo of the mainnet keys (tests/golden/varuna_bytes/*.verifier) and their .prover sizes
SHAPES = {"transfer_public": ((16, 12337, 12326, 28244, 38007, 16680), 28913482),
          "inclusion": ((4, 134564, 134767, 290115, 173792, 241076), 233812212)}


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
    import torch
    fn()
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(out)


def _matrix(rng, nrows, nnz, nvars, dev):
    """a CSR matrix of nnz entries spread over nrows rows, distinct sorted columns per row, random nonzero values"""
    import numpy as np
    from snarkvm_b200.varuna import Matrix
    per = np.full(nrows, nnz // nrows, dtype=np.int64)
    per[: nnz % nrows] += 1
    row_ptr = np.concatenate([[0], np.cumsum(per)])
    row_of = np.repeat(np.arange(nrows), per)
    u = rng.integers(0, nvars - per.max() + 1, size=nnz)
    u = u[np.lexsort((u, row_of))]
    cols = u + np.arange(nnz) - row_ptr[row_of]                          # sorted draws plus their place: increasing in a row
    vals = rng.integers(1, 2**63, size=(nnz, 4), dtype=np.uint64)
    vals[:, 3] &= np.uint64((1 << 58) - 1)                             # below r: a Montgomery image of a nonzero element
    return Matrix(row_ptr, cols, vals, dev)


def key_like(name):
    import numpy as np
    from snarkvm_b200 import varuna as dv
    from snarkvm_b200.sonic_pc import synthetic_srs
    info, _size = SHAPES[name]
    npub, nvars, ncons, *nnz = info
    rng = np.random.default_rng(1)
    circuit = dv.index_circuits([tuple(_matrix(rng, ncons, n, nvars, "cuda") for n in nnz) + (npub, nvars)])[0]
    powers, gpowers = synthetic_srs(circuit.info.max_degree(True), 0x1234567890ABCDEF, 0xFEDCBA09)
    return dv.batch_circuit_setup([circuit], powers, gpowers, zk=True, with_id=True)[0][0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", default="transfer_public,inclusion")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    from snarkvm_b200 import device, sonic_pc
    from snarkvm_b200 import varuna as dv
    print(card())
    dev = torch.device("cuda")
    for name in args.keys.split(","):
        pk = key_like(name)
        blob = pk.to_bytes()
        assert 1 + len(blob) == SHAPES[name][1], (name, len(blob))
        mv = memoryview(blob)
        L = dv._walk_proving_key(sonic_pc.ByteReader(mv, 0, "blob 0"))
        d_blob = sonic_pc.upload(mv, torch.empty(len(blob), dtype=torch.uint8, device=dev))
        runs = L.ck.runs()
        raw = sonic_pc.gather_records(d_blob, runs, sonic_pc.POINT_BYTES)
        c = pk.circuit
        segments = []
        for (o, rp), m in zip(L.matrices, (c.a, c.b, c.c)):
            segments.append((o, m.nnz, 40, torch.empty_like(m.vals), torch.empty_like(m.cols), c.num_variables,
                             torch.from_numpy(rp).to(dev)))
        for e, a in zip(L.evals, c.ariths):
            for n in ("row", "col", "row_col_val"):
                segments.append((e[n], a.domain.size, 32, torch.empty_like(getattr(a, n)), None, 0, None))
        assert device.fr_records_decode(d_blob, segments) == [None] * len(segments)
        row = {"key": name, "bytes": len(blob), "points": sum(n for _o, n in runs),
               "fr_records": sum(s[1] for s in segments), "matrix_entries": sum(m.nnz for m in (c.a, c.b, c.c)),
               "to_bytes_ms": _clock(lambda: pk.to_bytes(), args.reps),
               "from_bytes_ms": _clock(lambda: dv.CircuitProvingKey.from_bytes(blob), args.reps),
               "from_bytes_unvalidated_ms": _clock(lambda: dv.CircuitProvingKey.from_bytes(blob, validate=False), args.reps),
               "header_walk_ms": _clock(lambda: dv._walk_proving_key(sonic_pc.ByteReader(mv, 0, "blob 0")), args.reps),
               "row_walks_ms": _clock(lambda: [device.matrix_row_walk(mv, o + 8, c.num_constraints, m.nnz)
                                               for (o, _rp), m in zip(L.matrices, (c.a, c.b, c.c))], args.reps),
               "upload_ms": _clock(lambda: sonic_pc.upload(mv, d_blob), args.reps),
               "gather_points_ms": _events(lambda: sonic_pc.gather_records(d_blob, runs, sonic_pc.POINT_BYTES), args.reps),
               "fr_decode_ms": _events(lambda: device.fr_records_decode(d_blob, segments), args.reps),
               "g1_decode_validated_ms": _events(lambda: device.g1_deserialize(raw, device.G1_TO_BYTES, True), args.reps),
               "g1_decode_unvalidated_ms": _events(lambda: device.g1_deserialize(raw, device.G1_TO_BYTES, False), args.reps),
               "sha256_ms": _clock(lambda: L.ck.sha256(mv), args.reps),
               "blake2s_ms": _clock(lambda: dv._blake2s(mv, L.id_span), args.reps)}
        print(json.dumps(row), flush=True)
        del pk, d_blob, raw, segments
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
