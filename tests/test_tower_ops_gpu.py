"""GPU: the pairing's Fq6 / Fq12 tower, line evaluation, G2 line steps, exp_by_x and final exponentiation, one element at a time on
the operand corpus of tests/tower_corpus.py, compared word for word with the big-int restatement (tests/pairing_oracle.py).

The test kernels are compiled in pairing.cu, so they call the same functions, and the same out-of-line Fq products, as the pairing
kernels.  The oracle's Fq6 product is the schoolbook one, its Fq12 squaring a full product, and mul_by_034 / ell are checked against
the full product with the sparse element, so the comparison does not share the device's Karatsuba / CH-SQR2 / complex-squaring
schedules.  Also here: the public pairing entry points with padded strides, and one check with more pairs than one block holds."""
import random

import numpy as np
import pytest

from oracle import bls12_377 as py
from oracle import g2 as og2

import pairing_oracle as po
import tower_corpus as tc
from helpers import affine_array

pytestmark = pytest.mark.gpu
Q = tc.Q
F2_ZERO = (0, 0)
OP = {"fq6_mul": 48, "fq6_sqr": 49, "fq6_mul_by_01": 50, "fq6_mul_by_nonresidue": 51, "fq6_inverse": 52, "fq6_frobenius": 53,
      "fq12_mul": 54, "fq12_sqr": 55, "fq12_mul_by_034": 56, "fq12_cyclotomic_square": 57, "fq12_inverse": 58, "fq12_conjugate": 59,
      "fq12_frobenius": 60, "fq12_is_one": 61, "fq12_exp_by_x": 62, "fq12_final_exponentiation": 63, "fq12_ell": 64,
      "g2_doubling_step": 65, "g2_addition_step": 66}
INVALID_VALUE = 1                                                    # cudaErrorInvalidValue
F6_ZERO = po.F6_ZERO
F12_ZERO = (F6_ZERO, F6_ZERO)


def _run(op, a, b=None, c=None, k=0, out_words=None):
    """the device op on word arrays a (and b, c) → [n, out_words] uint32"""
    import torch
    from snarkvm_b200 import _lib
    dev = torch.device("cuda:0")
    n = a.shape[0]
    t = [None if x is None else torch.from_numpy(np.ascontiguousarray(x).view(np.int32)).to(dev) for x in (a, b, c)]
    out = torch.full((n, out_words or a.shape[1]), -1, dtype=torch.int32, device=dev)
    _lib.check(_lib.lib().snarkvm_b200_test_tower_op_device(OP[op], k, out.data_ptr(), *[None if x is None else x.data_ptr() for x in t],
                                                             n, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return out.cpu().numpy().view(np.uint32)


def _compare(op, got, want, inputs):
    bad = [(i, inputs[i]) for i, (g, w) in enumerate(zip(got, want)) if g != w]
    assert not bad, f"{op}: {len(bad)} of {len(want)} wrong, first at {bad[0][0]}: input {bad[0][1]}"


def _sparse6(b0, b1): return (b0, b1, F2_ZERO)
def _sparse12(c0, c3, c4): return ((c0, F2_ZERO, F2_ZERO), (c3, c4, F2_ZERO))


# ---- Fq6 ----
@pytest.mark.parametrize("op", ["fq6_sqr", "fq6_mul_by_nonresidue", "fq6_inverse"])
def test_fq6_unary_op(op):
    els = [e for _, e in tc.elements("f6")]
    got = tc.from_words(_run(op, tc.words(els)), "f6")
    if op == "fq6_sqr":
        want = [po.f6_mul(a, a) for a in els]
    elif op == "fq6_mul_by_nonresidue":
        want = [po.f6_mul(a, (F2_ZERO, (1, 0), F2_ZERO)) for a in els]                # ·v
    else:
        want = [F6_ZERO if a == F6_ZERO else po.f6_inv(a) for a in els]                # zero ↦ zero
        assert all(a == F6_ZERO or po.f6_mul(a, w) == po.F6_ONE for a, w in zip(els, want))
    _compare(op, got, want, els)


def test_fq6_mul():
    ps = tc.pairs("f6")
    got = tc.from_words(_run("fq6_mul", tc.words([a for a, _ in ps]), tc.words([b for _, b in ps])), "f6")
    _compare("fq6_mul", got, [po.f6_mul(a, b) for a, b in ps], ps)


def test_fq6_mul_by_01():
    cases = tc.mul_by_01_cases()
    got = tc.from_words(_run("fq6_mul_by_01", tc.words([a for a, _ in cases]), tc.words([b for _, b in cases])), "f6")
    _compare("fq6_mul_by_01", got, [po.f6_mul(a, _sparse6(*b)) for a, b in cases], cases)


@pytest.mark.parametrize("k", range(6))
def test_fq6_frobenius(k):
    els = [e for _, e in tc.elements("f6")]
    got = tc.from_words(_run("fq6_frobenius", tc.words(els), k=k), "f6")
    _compare(f"fq6_frobenius({k})", got, [po.f6_frob(a, k) for a in els], els)


# ---- Fq12 ----
@pytest.mark.parametrize("op", ["fq12_sqr", "fq12_inverse", "fq12_conjugate"])
def test_fq12_unary_op(op):
    els = [e for _, e in tc.elements("f12")]
    got = tc.from_words(_run(op, tc.words(els)), "f12")
    if op == "fq12_sqr":
        want = [po.f12_mul(a, a) for a in els]
    elif op == "fq12_inverse":
        want = [F12_ZERO if a == F12_ZERO else po.f12_inv(a) for a in els]             # zero ↦ zero
        assert all(a == F12_ZERO or po.f12_mul(a, w) == po.F12_ONE for a, w in zip(els, want))
    else:
        want = [po.f12_conj(a) for a in els]
    _compare(op, got, want, els)


def test_fq12_mul():
    ps = tc.pairs("f12")
    got = tc.from_words(_run("fq12_mul", tc.words([a for a, _ in ps]), tc.words([b for _, b in ps])), "f12")
    _compare("fq12_mul", got, [po.f12_mul(a, b) for a, b in ps], ps)


@pytest.mark.parametrize("k", range(12))
def test_fq12_frobenius(k):
    els = [e for _, e in tc.elements("f12")]
    got = tc.from_words(_run("fq12_frobenius", tc.words(els), k=k), "f12")
    _compare(f"fq12_frobenius({k})", got, [po.f12_frob(a, k) for a in els], els)


def test_fq12_mul_by_034():
    cases = tc.mul_by_034_cases()
    got = tc.from_words(_run("fq12_mul_by_034", tc.words([f for f, _ in cases]), tc.words([c for _, c in cases])), "f12")
    _compare("fq12_mul_by_034", got, [po.f12_mul(f, _sparse12(*c)) for f, c in cases], cases)


def test_fq12_ell():
    """ell(f, (c0, c1, c2), p) = f · ((c0·p.y, 0, 0) + (c1·p.x, c2, 0)·w)"""
    cases = tc.ell_cases()
    got = tc.from_words(_run("fq12_ell", tc.words([f for f, _, _ in cases]), tc.words([c for _, c, _ in cases]),
                             tc.words([p for _, _, p in cases]), out_words=144), "f12")
    want = [po.f12_mul(f, _sparse12(po.f2_mul_fp(c[0], p[1]), po.f2_mul_fp(c[1], p[0]), c[2])) for f, c, p in cases]
    _compare("fq12_ell", got, want, cases)


@pytest.fixture(scope="module")
def cyclotomic():
    return tc.cyclotomic_elements()


def test_fq12_cyclotomic_square(cyclotomic):
    got = tc.from_words(_run("fq12_cyclotomic_square", tc.words(cyclotomic)), "f12")
    _compare("fq12_cyclotomic_square", got, [po.f12_mul(g, g) for g in cyclotomic], cyclotomic)


def test_fq12_exp_by_x(cyclotomic):
    got = tc.from_words(_run("fq12_exp_by_x", tc.words(cyclotomic)), "f12")
    want = [po.exp_by_x(g) for g in cyclotomic]
    assert want == [po.f12_pow(g, po.X) for g in cyclotomic]
    _compare("fq12_exp_by_x", got, want, cyclotomic)


def test_fq12_is_one():
    cases = tc.is_one_cases()
    got = _run("fq12_is_one", tc.words([e for e, _, _ in cases]), out_words=1)[:, 0]
    bad = [(w, e) for (e, want, w), g in zip(cases, got) if g != (1 if want else 0)]
    assert not bad, f"is_one: {len(bad)} of {len(cases)} wrong, first with word {bad[0][0]} changed"


def _miller_values():
    """device Miller values of a few pairs of random points, and the device GT of each pair on its own"""
    from snarkvm_b200 import device
    import torch
    rng = random.Random(11)
    g2s = [og2.g2_mul(og2.G2_GEN, rng.randrange(1, py.R_MOD)) for _ in range(3)] + [og2.G2_GEN]
    g1s = [py.g1_mul(py.G1_GENERATOR, rng.randrange(1, py.R_MOD)) for _ in range(3)] + [py.G1_GENERATOR]
    prepared = device.g2_prepare(_g2(g2s))
    pairs = [(i, j) for i in range(4) for j in range(4) if (i + j) % 2 == 0]
    gt, _, miller = device.pairing_products(torch.from_numpy(affine_array([g1s[i] for i, _ in pairs])).cuda(),
                                            _i32([j for _, j in pairs]), prepared, _i32(list(range(len(pairs) + 1))), miller=True)
    return [bytes(r) for r in miller.cpu().numpy()], [bytes(r) for r in gt.cpu().numpy()]


def test_fq12_final_exponentiation():
    """structured elements (Fq6 elements go to one, zero to zero), general elements, and device Miller values, whose results must
    also be the GT values pairing_products returned for them"""
    cases = tc.final_exp_cases()
    mv, gts = _miller_values()
    cases += [("miller", po.gt_from_bytes(b)) for b in mv]
    els = [e for _, e in cases]
    out = _run("fq12_final_exponentiation", tc.words(els))
    got = tc.from_words(out, "f12")
    want = []
    for f, e in cases:
        if f == "zero":
            want.append(F12_ZERO)                        # the device's documented zero ↦ zero (the oracle's inverse raises on it)
        else:
            w = po.final_exponentiation(e)
            assert f != "in_fq6" or w == po.F12_ONE
            want.append(w)
    _compare("fq12_final_exponentiation", got, want, cases)
    assert [r.tobytes() for r in out[-len(mv):]] == gts


# ---- G2 line steps ----
def test_g2_doubling_step():
    states = tc.line_states()
    out = _run("g2_doubling_step", tc.words(states), out_words=144)
    got_r, got_c = tc.from_words(out[:, :72], "f2x3"), tc.from_words(out[:, 72:], "f2x3")
    want = [po._doubling_step(s) for s in states]
    _compare("g2_doubling_step", list(zip(got_r, got_c)), want, states)


def test_g2_addition_step():
    cases = tc.addition_cases()
    out = _run("g2_addition_step", tc.words([s for s, _ in cases]), tc.words([q for _, q in cases]), out_words=144)
    got_r, got_c = tc.from_words(out[:, :72], "f2x3"), tc.from_words(out[:, 72:], "f2x3")
    want = [po._addition_step(s, q) for s, q in cases]
    _compare("g2_addition_step", list(zip(got_r, got_c)), want, cases)


def test_entry_point_rejects_bad_ops_k_and_alignment():
    import torch
    from snarkvm_b200 import _lib
    L = _lib.lib()
    buf = torch.zeros(4 * 144, dtype=torch.int32, device="cuda:0")
    p = buf.data_ptr()
    s = torch.cuda.current_stream().cuda_stream
    call = lambda op, k, out=p, a=p, n=1: L.snarkvm_b200_test_tower_op_device(op, k, out, a, p, p, n, s)   # noqa: E731
    for op, k in [(47, 0), (67, 0), (OP["fq6_frobenius"], 6), (OP["fq6_frobenius"], -1), (OP["fq12_frobenius"], 12),
                  (OP["fq12_mul"], 1)]:
        assert call(op, k) == INVALID_VALUE, (op, k)
    assert call(OP["fq12_mul"], 0, a=p + 4) == INVALID_VALUE                       # Fq loads are 16-byte vectors
    assert L.snarkvm_b200_test_tower_op_device(OP["fq12_mul"], 0, p, p, None, None, 1, s) == INVALID_VALUE
    assert call(OP["fq12_frobenius"], 11, n=0) == 0
    assert call(OP["fq6_frobenius"], 5) == 0 and call(OP["fq12_frobenius"], 11) == 0
    torch.cuda.synchronize()


# ---- the public entry points: padded strides, many pairs in one check ----
def _g2(points):
    import torch
    return torch.from_numpy(np.frombuffer(b"".join(og2.g2_affine_bytes(p) for p in points), dtype=np.uint8).reshape(-1, 200).copy()).cuda()


def _i32(v):
    import torch
    return torch.tensor(v, dtype=torch.int32, device="cuda")


def _padded(images: np.ndarray, used: int, stride: int, rng: np.random.Generator):
    """rows of `images` at `stride` bytes, every byte after the first `used` of a row (the flag's padding and the stride's) garbage"""
    import torch
    out = rng.integers(0, 256, size=(images.shape[0], stride), dtype=np.uint8)
    out[:, :used] = images[:, :used]
    return torch.from_numpy(out).cuda()


def test_padded_strides_equal_the_default_stride():
    """G2 points at strides 208 and 256 and G1 points at 112 and 128, every padding byte garbage (the flag's own padding too):
    prepared points, GT values, verdicts and Miller values equal those of the default strides"""
    import torch
    from snarkvm_b200 import device
    rng = np.random.default_rng(12)
    g2s = [og2.G2_GEN, None] + tc.fc.g2_points(3, 5)[1:]
    g1s = tc.fc.g1_points(5, 6) + [None]
    g2img = np.frombuffer(b"".join(og2.g2_affine_bytes(p) for p in g2s), dtype=np.uint8).reshape(-1, 200)
    g1img = np.concatenate([affine_array(g1s), affine_array(g1s[::-1])])
    idx = _i32([i % len(g2s) for i in range(g1img.shape[0])])
    starts = _i32([0, 1, 3, 6, 12])                                     # check 1 holds a G2 point at infinity, check 3 a G1 one
    prep = device.g2_prepare(torch.from_numpy(g2img.copy()).cuda())
    gt, is_one, mv = device.pairing_products(torch.from_numpy(g1img).cuda(), idx, prep, starts, miller=True)
    for stride in (208, 256):
        assert (device.g2_prepare(_padded(g2img, 193, stride, rng), stride=stride) == prep).all(), stride
    for stride in (112, 128):
        gt2, is_one2, mv2 = device.pairing_products(_padded(g1img, 97, stride, rng), idx, prep, starts, g1_stride=stride, miller=True)
        assert (gt2 == gt).all() and (is_one2 == is_one).all() and (mv2 == mv).all(), stride
    assert bytes(gt[1].cpu().numpy()) == po.gt_bytes(po.product_of_pairings([(g1s[1], g2s[1]), (g1s[2], g2s[2])]))


def test_one_check_with_many_pairs():
    """260 pairs in one check (three 128-thread blocks of k_miller_pairs) against the oracle's product of pairings, G1 and G2
    points at infinity among them"""
    import torch
    from snarkvm_b200 import device
    rng = random.Random(13)
    g2s = tc.fc.g2_points(4, 7) + [None]
    preps = [po.g2_prepare(q) for q in g2s]
    g1s = tc.fc.g1_points(64, 8)
    n = 260
    pairs = [(None if i % 97 == 5 else g1s[rng.randrange(len(g1s))], rng.randrange(len(g2s))) for i in range(n)]
    gt, is_one, mv = device.pairing_products(torch.from_numpy(affine_array([p for p, _ in pairs])).cuda(), _i32([j for _, j in pairs]),
                                             device.g2_prepare(_g2(g2s)), _i32([0, n]), miller=True)
    shared = po.miller_loop([(p, preps[j]) for p, j in pairs])
    assert bytes(gt[0].cpu().numpy()) == po.gt_bytes(po.final_exponentiation(shared)) and not bool(is_one[0])
    prod = po.F12_ONE
    for r in mv.cpu().numpy():
        prod = po.f12_mul(prod, po.gt_from_bytes(bytes(r)))
    assert prod == shared
