"""GPU: the NTT above 2^24.  test_ntt_gpu.py compares every mode with the oracle up to 2^25, the smallest four-pass plan; here:

* 2^26 and 2^27, four-pass plans of 7+7+6+6 and 7+7+7+6 stages, too large for a full oracle transform in test time.  Sparse
  inputs are checked against the definition of the transform with Python integers, and dense inputs by the radix-2 split
  identity, whose halves are transforms of the size below (2^25 is checked against the oracle, 2^26 here);
* small transforms reading a twiddle table grown to 2^27 with a stride of up to 2^26;
* ntt_batch_ with more transforms of one two-pass size than one grid row of 65 535 holds.

Values are compared as canonical Montgomery limbs.  The transforms are linear, and so is the Montgomery image v ↦ v·2^256 mod r,
so the big-integer sums below are taken over the limb images directly."""
import random

import numpy as np
import pytest

from oracle import bls12_377 as py

from helpers import fr_ints_to_mont_array, put_near_r, random_fr_mont, scalars_from_ints
from test_ntt_gpu import MODES, _dev, _host

pytestmark = pytest.mark.gpu

R, G = py.R_MOD, py.FR_GENERATOR


@pytest.fixture(autouse=True)
def _release_memory():
    """Each case holds gigabytes of HBM: return them to the device before the next case."""
    yield
    import torch
    torch.cuda.empty_cache()


def _rows(t, idx):
    """rows idx of a device Fr tensor as Python integers (limb images)"""
    import torch
    return [py.from_limbs(r) for r in t[torch.tensor(idx, device=t.device)].cpu().numpy().view(np.uint64)]


def _fill(x, seed):
    """x ← seeded values below r (top limb below 2^60) with the r − 1 / r − 2 rows of put_near_r, generated on the device → x"""
    import torch
    g = torch.Generator(device=x.device).manual_seed(seed)
    torch.randint(-2**63, 2**63 - 1, tuple(x.shape), dtype=torch.int64, device=x.device, generator=g, out=x)
    x[:, 3] &= (1 << 60) - 1
    return put_near_r(x)


@pytest.mark.parametrize("lg", [26, 27])
def test_four_pass_sparse_by_definition(lg):
    """65 nonzeros — one in each 64th of the columns of the first pass's 2^7-row view, at a random row, and one at n − 1 — and 517
    outputs — random k and k = 0, 1, n/2 − 1, n/2, n − 1 — against Σ x_j·(g^t·ω^k)^j forward and n^{-1}·g^{−t·k}·Σ x_j·ω^{−jk}
    inverse, t = 1 for the coset modes.  Nothing runs on the device but the transform under test."""
    import torch
    from snarkvm_b200 import device
    from snarkvm_b200.cuda import NTTDirection, NTTType
    n = 1 << lg
    rng = random.Random(lg)
    cols = n >> 7
    pos = sorted({rng.randrange(128) * cols + i * (cols // 64) + rng.randrange(cols // 64) for i in range(64)} | {n - 1})
    vals = [rng.randrange(R) for _ in pos]
    vals[0], vals[-1] = R - 1, R - 2
    ks = sorted({rng.randrange(n) for _ in range(512)} | {0, 1, n // 2 - 1, n // 2, n - 1})
    x = torch.zeros((n, 4), dtype=torch.int64, device="cuda")
    x[torch.tensor(pos, device="cuda")] = torch.from_numpy(scalars_from_ints(vals).view(np.int64)).cuda()
    y, scratch = torch.empty_like(x), torch.empty_like(x)
    w = py.fr_root_of_unity(n)
    w_inv, n_inv, g_inv = pow(w, -1, R), pow(n, -1, R), pow(G, -1, R)
    for d, t in MODES:
        y.copy_(x)
        got = _rows(device.ntt_(y, NTTDirection(d), NTTType(t), scratch), ks)
        bad = []
        for k, v in zip(ks, got):
            if d == 0:
                base = pow(G, t, R) * pow(w, k, R) % R
                want = sum(c * pow(base, j, R) for j, c in zip(pos, vals)) % R
            else:
                base = pow(w_inv, k, R)
                want = n_inv * pow(g_inv, t * k, R) * sum(c * pow(base, j, R) for j, c in zip(pos, vals)) % R
            if v != want:
                bad.append(k)
        assert not bad, (lg, d, t, len(bad), bad[:8])


@pytest.mark.parametrize("lg", [26, 27])
def test_four_pass_split_identity(lg):
    """Dense inputs, h = n/2: Y = NTT_n(x), E = NTT_h(x[0::2]) and O = NTT_h(x[1::2]) satisfy Y[k] = E[k] + ω^k·O[k] and
    Y[k + h] = E[k] − ω^k·O[k], with coset_fft(x) = fft(x∘g^j).  For Z = iNTT_n(y), iE = iNTT_h(y[0::2]) and iO = iNTT_h(y[1::2]),
    the identity Z[k] = ½(iE[k] + ω^{−k}·iO[k]), Z[k + h] = ½(iE[k] − ω^{−k}·iO[k]) is checked in
    the equivalent form iE = Z[:h] + Z[h:], iO = ω^k·(Z[:h] − Z[h:]), with coset_ifft(y) = ifft(y)∘g^{−j}.  Then iNTT ∘ NTT is the
    identity for the standard and the coset pair.  HBM: x, its scratch, the halves, ω^k and g^k for k < h, and the twiddle table
    — 4.5·2^lg Fr, 18 GiB at 2^27."""
    import torch
    from snarkvm_b200 import device
    from snarkvm_b200.cuda import NTTDirection, NTTType
    MUL, ADD, SUB = device.FR_MUL, device.FR_ADD, device.FR_SUB
    n, h = 1 << lg, 1 << (lg - 1)
    w_k = device.domain_elements(lg)[:h].clone()
    g_k = torch.empty_like(w_k)                                           # g^k by doubling: g_k[m:2m] = g^m·g_k[:m]
    g_k[0] = torch.from_numpy(fr_ints_to_mont_array([1]).view(np.int64)).cuda()
    m = 1
    while m < h:
        device.fr_vec_op(g_k[:m], fr_ints_to_mont_array([pow(G, m, R)])[0], MUL, out=g_k[m:2 * m])
        m *= 2
    rng = random.Random(lg)
    idx = sorted({rng.randrange(h) for _ in range(1000)} | {0, 1, h - 1})
    w = py.fr_root_of_unity(n)
    assert _rows(w_k, idx) == [py.fr_to_mont(pow(w, i, R)) for i in idx]
    assert _rows(g_k, idx) == [py.fr_to_mont(pow(G, i, R)) for i in idx]

    a, b, s = (torch.empty((n, 4), dtype=torch.int64, device="cuda") for _ in range(3))
    e, o, u, v = b[:h], b[h:], s[:h], s[h:]
    for d, t in MODES:
        seed = 100 * lg + 2 * d + t
        _fill(a, seed)
        b.view(2, h, 4).copy_(a.view(h, 2, 4).transpose(0, 1))             # b = [x[0::2] | x[1::2]]
        if d == 0 and t == 1:                                             # the halves of x∘g^j: g^2m·x[2m] and g·g^2m·x[2m + 1]
            for half in (e, o):
                device.fr_vec_op(half, g_k, MUL, out=half)
                device.fr_vec_op(half, g_k, MUL, out=half)
            device.fr_vec_op(o, fr_ints_to_mont_array([G])[0], MUL, out=o)
        device.ntt_(a, NTTDirection(d), NTTType(t), s)
        device.ntt_(e, NTTDirection(d), NTTType.Standard, s)
        device.ntt_(o, NTTDirection(d), NTTType.Standard, s)
        if d == 0:
            device.fr_vec_op(o, w_k, MUL, out=u)
            assert torch.equal(device.fr_vec_op(e, u, ADD, out=v), a[:h]), (lg, d, t, "low half")
            assert torch.equal(device.fr_vec_op(e, u, SUB, out=v), a[h:]), (lg, d, t, "high half")
            device.ntt_(a, NTTDirection.Inverse, NTTType(t), s)
            assert torch.equal(a, _fill(b, seed)), (lg, t, "round trip")
        else:
            if t == 1:                                                    # ifft(y)[j] = coset_ifft(y)[j]·g^j
                device.fr_vec_op(a[:h], g_k, MUL, out=a[:h])
                device.fr_vec_op(a[h:], g_k, MUL, out=a[h:])
                device.fr_vec_op(a[h:], fr_ints_to_mont_array([pow(G, h, R)])[0], MUL, out=a[h:])
            assert torch.equal(device.fr_vec_op(a[:h], a[h:], ADD, out=u), e), (lg, d, t, "even half")
            device.fr_vec_op(a[:h], a[h:], SUB, out=u)
            assert torch.equal(device.fr_vec_op(u, w_k, MUL, out=u), o), (lg, d, t, "odd half")


def test_small_transforms_read_a_2_27_table(oracle_cpu):
    """The twiddle table is cached per device and only grows, and a transform of 2^lg reads it with a stride of 2^(lgN − lg).  Grow
    it to lgN = 27 first, so the strides are the same whatever ran before: domain_elements(27) against powers of ω, then one-pass
    (2^1, 2^2, 2^11), two-pass (2^12, 2^16) and three-pass (2^17, 2^19) transforms in all four modes against the oracle, and
    domain_elements(3) against the oracle's FFT of X."""
    from snarkvm_b200 import device
    from snarkvm_b200.cuda import NTTDirection, NTTType
    n = 1 << 27
    rng = random.Random(27)
    idx = sorted({rng.randrange(n) for _ in range(1000)} | {0, 1, n // 2 - 1, n // 2, n - 1})
    w = py.fr_root_of_unity(n)
    assert _rows(device.domain_elements(27), idx) == [py.fr_to_mont(pow(w, i, R)) for i in idx]
    for lg in (1, 2, 11, 12, 16, 17, 19):
        x = put_near_r(random_fr_mont(1 << lg, seed=2700 + lg))
        for d, t in MODES:
            got = device.ntt_(_dev(x), NTTDirection(d), NTTType(t))
            assert (_host(got) == oracle_cpu.ntt(x, d, t)).all(), (lg, d, t)
    poly_x = np.zeros((8, 4), dtype=np.uint64)
    poly_x[1] = fr_ints_to_mont_array([1])[0]
    assert (_host(device.domain_elements(3)) == oracle_cpu.ntt(poly_x, 0, 0)).all()


def test_ntt_batch_two_grid_rows_two_pass():
    """65 537 transforms of 2^12, the smallest two-pass size, in one ntt_batch_ call: the second grid row holds transforms 65 535
    and 65 536, whose pointers and scratch slices start at the row's first index.  Every transform must equal ntt_ of a fresh copy
    of its input.  The batch is views of one 8.6 GB tensor; the fresh copies are regenerated from its seed, so two copies and the
    batch's scratch are the most that is live."""
    import torch
    from snarkvm_b200 import device
    from snarkvm_b200.cuda import NTTDirection, NTTType
    count, lg = 65537, 12
    n, chunk = 1 << lg, 4096
    got = torch.empty((count * n, 4), dtype=torch.int64, device="cuda")
    scratch = torch.empty((n, 4), dtype=torch.int64, device="cuda")
    for seed, (d, t) in enumerate(((NTTDirection.Forward, NTTType.Standard), (NTTDirection.Inverse, NTTType.Coset))):
        device.ntt_batch_(list(_fill(got, seed).view(count, n, 4).unbind(0)), d, t)
        want = _fill(torch.empty_like(got), seed).view(count, n, 4)
        for i in range(count):
            device.ntt_(want[i], d, t, scratch)
        g = got.view(count, n, 4)
        bad = [i for i in range(0, count, chunk) if not torch.equal(g[i:i + chunk], want[i:i + chunk])]
        assert not bad, (d, t, "transforms from", bad)
        del want, g
