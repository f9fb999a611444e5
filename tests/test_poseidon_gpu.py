"""The device Poseidon sponge (csrc/poseidon.cu through device.poseidon_transcripts) against the reference's Fr snapshots and against
the big-integer sponge (oracle/poseidon.py), over Fq and Fr: random operation lists around every rate boundary, zero-length
operations, field-corpus absorbs, many transcripts of different lengths in one call, and malformed lists and inputs, which must be
refused with nothing written."""
import ctypes
import json
import os
import random

import numpy as np
import pytest

from oracle import poseidon as op
from snarkvm_b200 import poseidon as ps

import field_corpus as fc

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
KIND = {"absorb": ps.OP_ABSORB, "squeeze": ps.OP_SQUEEZE, "nonnative": ps.OP_SQUEEZE_NONNATIVE, "short": ps.OP_SQUEEZE_SHORT_NONNATIVE}


def _encode(field, transcripts):
    """[[(kind, ints or count), …], …] → (ops, op_start, inputs, nout, nout_fr) host arrays; outputs packed per transcript in order"""
    ops, starts, values = [], [0], []
    nout = nout_fr = 0
    for t in transcripts:
        for kind, arg in t:
            if kind == "absorb":
                ops.append((KIND[kind], len(arg), len(values)))
                values += list(arg)
            elif kind == "squeeze":
                ops.append((KIND[kind], arg, nout))
                nout += arg
            else:
                ops.append((KIND[kind], arg, nout_fr))
                nout_fr += arg
        starts.append(len(ops))
    words = ps.FIELDS[field][2]
    inputs = ps.to_mont_words(field, values) if values else np.zeros((0, words), dtype=np.uint32)
    return (np.array(ops, dtype=np.int32).reshape(-1, 3), np.array(starts, dtype=np.int32), inputs, nout, nout_fr)


def _run(field, transcripts):
    import torch
    from snarkvm_b200 import device
    ops, starts, inputs, nout, nout_fr = _encode(field, transcripts)
    out, out_fr = device.poseidon_transcripts(field, torch.from_numpy(ops).cuda(), torch.from_numpy(starts).cuda(),
                                              torch.from_numpy(np.ascontiguousarray(inputs).view(np.int64)).cuda(), nout, nout_fr)
    return (ps.from_mont_words(field, out.cpu().numpy()), ps.from_mont_words(ps.FIELD_FR, out_fr.cpu().numpy()))


def _oracle(field, transcripts):
    p, bits, _n = ps.FIELDS[field]
    native, fr = [], []
    for t in transcripts:
        s = op.Sponge(p, bits, ps.parameters(field, 2))
        for kind, arg in t:
            if kind == "absorb":
                s.absorb_native_field_elements(arg)
            elif kind == "squeeze":
                native += s.squeeze_native_field_elements(arg)
            else:
                fr += s.get_fe(arg, kind == "short")
    return native, fr


def test_reference_snapshots_word_for_word():
    """the 100 transcripts of test_poseidon_sponge_consistency in one call, Montgomery words equal to the snapshots'"""
    import torch
    from snarkvm_b200 import device
    with open(os.path.join(HERE, "golden", "poseidon_vectors.json")) as f:
        golden = json.load(f)["absorb_squeeze"]
    cases = [(a, s) for a in range(10) for s in range(10)]
    ops, starts, inputs, nout, _ = _encode(ps.FIELD_FR, [[("absorb", [1237812] * a), ("squeeze", s)] for a, s in cases])
    out, out_fr = device.poseidon_transcripts(ps.FIELD_FR, torch.from_numpy(ops).cuda(), torch.from_numpy(starts).cuda(),
                                              torch.from_numpy(inputs.view(np.int64)).cuda(), nout, 0)
    want = ps.to_mont_words(ps.FIELD_FR, [v for a, s in cases for v in golden[f"{a},{s}"]])
    assert out_fr.numel() == 0
    assert (out.cpu().numpy().view(np.uint32) == want).all()


def _random_transcript(rng, p, pool, max_ops=9):
    t = []
    for _ in range(rng.randrange(max_ops + 1)):
        kind = rng.choice(["absorb", "absorb", "squeeze", "nonnative", "short"])
        n = rng.choice([0, 1, 2, 3, 4, 5, rng.randrange(6, 14)])
        if kind == "absorb":
            t.append((kind, [rng.choice(pool) if rng.random() < 0.5 else rng.randrange(p) for _ in range(n)]))
        else:
            t.append((kind, n))
    return t


@pytest.mark.parametrize("field", [ps.FIELD_FQ, ps.FIELD_FR])
def test_random_operation_lists_against_the_oracle(field):
    """400 transcripts of different lengths in one call: every operation kind, counts 0 … 13 on both sides of each rate boundary,
    absorbs drawn half from the field corpus (0, p − 1, values next to 2^(32k), mostly-ones limbs)"""
    rng = random.Random(100 + field)
    p, _bits, n = ps.FIELDS[field]
    pool = fc.fixed_values(p, n) + fc.mostly_ones(rng, p, n, 20)
    assert 0 in pool and p - 1 in pool
    transcripts = [_random_transcript(rng, p, pool) for _ in range(400)]
    transcripts[0] = []                                                   # no operation at all
    transcripts[1] = [("absorb", []), ("squeeze", 0), ("nonnative", 0), ("short", 0)]
    transcripts[2] = [("squeeze", 3), ("absorb", [p - 1, 0]), ("short", 5), ("nonnative", 12), ("short", 1), ("short", 1)]
    assert _run(field, transcripts) == _oracle(field, transcripts)


@pytest.mark.parametrize("field", [ps.FIELD_FQ, ps.FIELD_FR])
def test_every_boundary_pair(field):
    """absorb a, then each squeeze kind of n, then absorb b, then squeeze m: a, b ∈ 0 … 4, n, m ∈ 0 … 4"""
    rng = random.Random(7 + field)
    p = ps.FIELDS[field][0]
    transcripts = []
    for a in range(5):
        for kind in ("squeeze", "nonnative", "short"):
            for nn in range(5):
                for b in range(5):
                    transcripts.append([("absorb", [rng.randrange(p) for _ in range(a)]), (kind, nn),
                                        ("absorb", [rng.randrange(p) for _ in range(b)]), ("squeeze", rng.randrange(5))])
    assert _run(field, transcripts) == _oracle(field, transcripts)


def _raw(field, ops, starts, inputs, nout, nout_fr):
    """the C entry point with sentinel-filled outputs → (return code, bad transcript, outputs unchanged)"""
    import torch
    from snarkvm_b200 import _lib, device
    words = ps.FIELDS[field][2]
    out = torch.full((max(nout, 1), words // 2), 0x5A5A5A5A5A5A5A5A, dtype=torch.int64, device="cuda")
    out_fr = torch.full((max(nout_fr, 1), 4), 0x5A5A5A5A5A5A5A5A, dtype=torch.int64, device="cuda")
    before = (out.clone(), out_fr.clone())
    ops_d = torch.from_numpy(np.ascontiguousarray(ops, dtype=np.int32)).cuda()
    starts_d = torch.from_numpy(np.ascontiguousarray(starts, dtype=np.int32)).cuda()
    in_d = torch.from_numpy(np.ascontiguousarray(inputs, dtype=np.uint32).view(np.int64)).cuda()
    bad = ctypes.c_int64(-1)
    code = _lib.lib().snarkvm_b200_poseidon_transcripts_device(
        field, ps.device_parameters(field, "cuda").data_ptr(), ops_d.data_ptr(), starts_d.data_ptr(), len(starts) - 1, len(ops),
        in_d.data_ptr(), len(inputs), out.data_ptr(), nout, out_fr.data_ptr(), nout_fr, ctypes.byref(bad), device._stream())
    torch.cuda.synchronize()
    return code, bad.value, bool((out == before[0]).all() and (out_fr == before[1]).all())


@pytest.mark.parametrize("field", [ps.FIELD_FQ, ps.FIELD_FR])
def test_malformed_lists_and_inputs_are_refused(field):
    import torch
    from snarkvm_b200 import CudaError, device
    rng = random.Random(3)
    p, _bits, n = ps.FIELDS[field]
    good = [[("absorb", [rng.randrange(p) for _ in range(3)]), ("squeeze", 2), ("nonnative", 2)] for _ in range(6)]
    ops, starts, inputs, nout, nout_fr = _encode(field, good)
    code, bad, untouched = _raw(field, ops, starts, inputs, nout, nout_fr)
    assert code == 0 and bad == -1 and not untouched
    cases = []
    big = inputs.copy()
    big[3 * 4 + 1] = np.frombuffer(p.to_bytes(4 * n, "little"), dtype=np.uint32)            # = p: no field element
    cases.append(("input = p", ops, starts, big, nout, nout_fr, 4))
    top = inputs.copy()
    top[3 * 2] = 0xFFFFFFFF
    cases.append(("input all ones", ops, starts, top, nout, nout_fr, 2))
    for row, col, value, who in [(3 * 3, 0, 7, 3),                          # unknown kind
                                 (3 * 1 + 1, 2, nout - 1, 1),               # squeeze past nout
                                 (3 * 5 + 2, 2, nout_fr - 1, 5),            # nonnative past nout_fr
                                 (3 * 2, 2, len(inputs) - 2, 2),            # absorb past nin
                                 (3 * 4, 1, 0x7FFFFFFF, 4)]:                # absorb count overflowing
        o = ops.copy()
        o[row, col] = value
        cases.append((f"op {row},{col}", o, starts, inputs, nout, nout_fr, who))
    s = starts.copy()
    s[3], s[4] = s[4], s[3]
    cases.append(("op_start out of order", ops, s, inputs, nout, nout_fr, 3))
    s = starts.copy()
    s[-1] = len(ops) + 1
    cases.append(("op_start past nops", ops, s, inputs, nout, nout_fr, 5))
    for name, o, s, i, no, nf, who in cases:
        code, bad, untouched = _raw(field, o, s, i, no, nf)
        assert code != 0 and bad == who and untouched, name
    with pytest.raises(CudaError) as ei:
        device.poseidon_transcripts(field, torch.from_numpy(ops).cuda(), torch.from_numpy(starts).cuda(),
                                    torch.from_numpy(big.view(np.int64)).cuda(), nout, nout_fr)
    assert ei.value.transcript == 4
    with pytest.raises(ValueError):
        device.poseidon_transcripts(field, torch.from_numpy(ops).cuda(), torch.from_numpy(starts).cuda(),
                                    torch.from_numpy(inputs.view(np.int64)).cuda()[:, :2], nout, nout_fr)
    out, out_fr = device.poseidon_transcripts(field, torch.from_numpy(ops[:0]).cuda(), torch.from_numpy(starts[:1]).cuda(),
                                              torch.from_numpy(inputs[:0].view(np.int64)).cuda(), 0, 0)
    assert out.numel() == 0 and out_fr.numel() == 0
