"""GPU: every field operation of ff.cuh / ec.cuh and every group operation of ec.cuh / quad.cuh, one element at a time on the operand
corpus of tests/field_corpus.py, compared limb for limb with Python big integers (oracle/bls12_377.py, oracle/g2.py).

The field operations run in test kernels compiled in three translation units: msm.cu (FF_CALL_MUL: products and squares call the
out-of-line mul_call / sqr_call that the MSM kernels call), ntt.cu (inlined into the test kernel — its own inline site, not
the machine code of the NTT butterflies) and pairing.cu (FF_CALL_MUL too, but its own out-of-line copies, which every product of
the pairing calls)."""
import numpy as np
import pytest

import field_corpus as fc

pytestmark = pytest.mark.gpu

CTX = {"msm": 0, "ntt": 1, "pairing": 2}
FIELD = {"fr": 0, "fq": 1, "fq2": 2}
OP = {"add": 0, "sub": 1, "neg": 2, "dbl": 3, "half": 4, "mul": 5, "mul_inline": 6, "mul_call": 7, "mul_karatsuba": 8,
      "sqr": 9, "sqr_inline": 10, "sqr_call": 11, "inverse": 12, "to_mont": 13, "from_mont": 14, "times5": 15,
      "coop_mul": 16, "coop_inverse": 17,
      "xyzz_add": 32, "xyzz_add_affine": 33, "xyzz_dbl": 34, "xyzz_mul_u32": 35, "xyzz_to_affine": 36,
      "quad_add": 37, "quad_dbl": 38, "quad_add_affine": 39}
INVERSE_CAP = 2000
FIELD_OPS = ["add", "sub", "neg", "dbl", "half", "mul", "mul_inline", "mul_call", "mul_karatsuba", "sqr", "sqr_inline", "sqr_call",
             "inverse", "to_mont", "from_mont", "coop_mul", "coop_inverse"]


def _expected(name, op, a, b):
    p, n = fc.FIELDS[name]
    R = fc.mont_r(p, n)
    rinv = pow(R, -1, p)
    if op == "add":
        return (a + b) % p
    if op == "sub":
        return (a - b) % p
    if op == "neg":
        return (-a) % p
    if op == "dbl":
        return 2 * a % p
    if op == "half":
        return a * pow(2, -1, p) % p
    if op in ("mul", "mul_inline", "mul_call", "mul_karatsuba", "coop_mul"):
        return a * b * rinv % p
    if op in ("sqr", "sqr_inline", "sqr_call"):
        return a * a * rinv % p
    if op in ("inverse", "coop_inverse"):
        return 0 if a == 0 else R * R * pow(a, -1, p) % p
    if op == "to_mont":
        return a * R % p
    if op == "from_mont":
        return a * rinv % p
    raise ValueError(op)


def _run_field(ctx, field, op, a_words, b_words, words):
    import torch
    from snarkvm_b200 import _lib
    n = a_words.shape[0]
    dev = torch.device("cuda:0")
    da = torch.from_numpy(np.ascontiguousarray(a_words).view(np.int32)).to(dev)
    db = torch.from_numpy(np.ascontiguousarray(b_words).view(np.int32)).to(dev)
    out = torch.full((n, words), -1, dtype=torch.int32, device=dev)
    _lib.check(_lib.lib().snarkvm_b200_test_field_op_device(CTX[ctx], FIELD[field], OP[op], out.data_ptr(), da.data_ptr(),
                                                             db.data_ptr(), n, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return out.cpu().numpy().view(np.uint32)


def _operands(name, op):
    if op == "half":
        vals = fc.half_values(name)
        return vals, vals
    pairs = fc.field_pairs(name)
    if op in ("inverse", "coop_inverse"):
        pairs = pairs[:INVERSE_CAP // 2] + pairs[-INVERSE_CAP // 2:]
    return [a for a, _ in pairs], [b for _, b in pairs]


@pytest.mark.parametrize("op", FIELD_OPS)
@pytest.mark.parametrize("name", ["fr", "fq"])
@pytest.mark.parametrize("ctx", list(CTX))
def test_field_op_matches_big_integers(ctx, name, op):
    p, n = fc.FIELDS[name]
    A, B = _operands(name, op)
    got = fc.from_limbs(_run_field(ctx, name, op, fc.to_limbs(A, n), fc.to_limbs(B, n), n))
    bad = [(hex(a), hex(b), hex(g)) for a, b, g in zip(A, B, got) if g != _expected(name, op, a, b)]
    assert not bad, f"{ctx}/{name}/{op}: {len(bad)} of {len(A)} wrong, first {bad[:3]}"


@pytest.mark.parametrize("op", ["add", "sub", "neg", "dbl", "mul", "sqr", "inverse"])
@pytest.mark.parametrize("ctx", list(CTX))
def test_fq2_op_matches_big_integers(ctx, op):
    from oracle import g2 as og2
    q, R = fc.Q, fc.QR
    pairs = fc.fq2_pairs()
    A = [a for a, _ in pairs]
    B = [b for _, b in pairs]
    flat = lambda xs: fc.to_limbs([c for x in xs for c in x], 12).reshape(len(xs), 24)   # noqa: E731
    out = _run_field(ctx, "fq2", op, flat(A), flat(B), 24)
    got = fc.from_limbs(out.reshape(-1, 12))
    got = list(zip(got[::2], got[1::2]))
    rinv = fc.QR_INV
    for a, b, g in zip(A, B, got):
        if op == "add":
            want = og2.f2_add(a, b)
        elif op == "sub":
            want = og2.f2_sub(a, b)
        elif op == "neg":
            want = og2.f2_neg(a)
        elif op == "dbl":
            want = og2.f2_add(a, a)
        elif op in ("mul", "sqr"):
            w = og2.f2_mul(a, b if op == "mul" else a)               # bilinear: image(x)·image(y)·R⁻¹ = image(x·y)
            want = (w[0] * rinv % q, w[1] * rinv % q)
        else:
            x = (a[0] * rinv % q, a[1] * rinv % q)
            want = (0, 0) if x == (0, 0) else tuple(c * R % q for c in og2.f2_inv(x))
        assert g == want, (ctx, op, a, b, g, want)


@pytest.mark.parametrize("ctx", list(CTX))
def test_times5_matches_big_integers(ctx):
    A = [a for a, _ in fc.field_pairs("fq")]
    got = fc.from_limbs(_run_field(ctx, "fq", "times5", fc.to_limbs(A, 12), fc.to_limbs(A, 12), 12))
    assert got == [5 * a % fc.Q for a in A]


def _run_curve(group, op, cases):
    import torch
    from snarkvm_b200 import _lib
    dev = torch.device("cuda:0")
    comps = 4 if group == "g1" else 8
    a = fc.to_limbs([w for c in cases for w in c[0]], 12).reshape(len(cases), 12 * comps)
    b = fc.to_limbs([w for c in cases for w in c[1]], 12).reshape(len(cases), 12 * comps)
    k = np.array([c[2] for c in cases], dtype=np.uint32)
    da, db, dk = (torch.from_numpy(x.view(np.int32)).to(dev) for x in (a, b, k))
    out = torch.full((len(cases), 12 * comps), -1, dtype=torch.int32, device=dev)
    _lib.check(_lib.lib().snarkvm_b200_test_curve_op_device(0 if group == "g1" else 1, OP[op], out.data_ptr(), da.data_ptr(),
                                                             db.data_ptr(), dk.data_ptr(), len(cases),
                                                             torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    res = out.cpu().numpy().view(np.uint32)
    return [fc.from_limbs(row.reshape(comps, 12)) for row in res]


CURVE_OPS = [("g1", "xyzz_add", "add"), ("g1", "xyzz_add_affine", "add_affine"), ("g1", "xyzz_dbl", "dbl"),
             ("g1", "xyzz_mul_u32", "mul_u32"), ("g1", "quad_add", "add"), ("g1", "quad_dbl", "dbl"),
             ("g1", "quad_add_affine", "add_affine"),
             ("g2", "xyzz_add", "add"), ("g2", "xyzz_add_affine", "add_affine"), ("g2", "xyzz_dbl", "dbl"),
             ("g2", "xyzz_mul_u32", "mul_u32")]


@pytest.mark.parametrize("group,op,kind", CURVE_OPS)
def test_curve_op_matches_big_integers(group, op, kind):
    cases = fc.group_cases(group, kind)
    got = _run_curve(group, op, cases)
    for i, (words, (a, b, k, want)) in enumerate(zip(got, cases)):
        assert fc.decode_xyzz(words, group) == want, (group, op, i, k)


@pytest.mark.parametrize("group", ["g1", "g2"])
def test_to_affine_matches_big_integers(group):
    cases = fc.group_cases(group, "to_affine")
    got = _run_curve(group, "xyzz_to_affine", cases)
    w = 1 if group == "g1" else 2
    for words, (_, _, _, want) in zip(got, cases):
        x = [v * fc.QR_INV % fc.Q for v in words[:w]]
        y = [v * fc.QR_INV % fc.Q for v in words[w:2 * w]]
        flag = words[2 * w]
        if want is None:
            assert flag == 1 and x == [0] * w and y == [1] + [0] * (w - 1)          # Affine::zero() = (0, 1, inf)
        else:
            assert flag == 0
            assert (x[0] if w == 1 else tuple(x)) == want[0] and (y[0] if w == 1 else tuple(y)) == want[1]


def test_entry_points_reject_unknown_contexts_and_ops():
    """every context in CTX (msm, ntt, pairing) accepts a valid op; the values around them are no context; an op a field does not
    take is rejected in every context"""
    import torch
    from snarkvm_b200 import _lib
    L = _lib.lib()
    buf = torch.zeros(96, dtype=torch.int32, device="cuda:0")
    p = buf.data_ptr()
    s = torch.cuda.current_stream().cuda_stream
    for ctx in CTX.values():
        assert L.snarkvm_b200_test_field_op_device(ctx, FIELD["fr"], OP["add"], p, p, p, 1, s) == 0, ctx
        assert L.snarkvm_b200_test_field_op_device(ctx, FIELD["fq2"], OP["half"], p, p, p, 1, s) != 0, ctx
    for ctx in (-1, len(CTX)):
        assert L.snarkvm_b200_test_field_op_device(ctx, FIELD["fr"], OP["add"], p, p, p, 1, s) != 0, ctx
    assert L.snarkvm_b200_test_curve_op_device(1, OP["quad_add"], p, p, p, p, 1, s) != 0
    torch.cuda.synchronize()
