"""GPU parity: the CUDA NTT vs the oracle, bit-exact (Fr values are canonical Montgomery limbs).
Restates test_fft_correctness_cuda (algorithms/src/fft/domain.rs:1140-1218: sizes 2^2…2^19 ×
{NTT, iNTT, coset NTT, coset iNTT} vs the CPU path) and fft_composition (fft/tests.rs:287-328)."""
import numpy as np
import pytest

from helpers import put_near_r, random_fr_mont

pytestmark = pytest.mark.gpu

MODES = [(0, 0), (1, 0), (0, 1), (1, 1)]    # (direction, type)


def _dev(x):
    import torch
    return torch.from_numpy(x.view(np.int64).copy()).cuda()


def _host(t):
    return t.cpu().numpy().view(np.uint64)


@pytest.mark.parametrize("lg", list(range(0, 20)))
def test_ntt_host_ffi_vs_oracle(oracle_cpu, lg):
    """through the drop-in symbol snarkvm_ntt with HOST buffers, exactly as fft/domain.rs:375-438 calls it"""
    from snarkvm_b200 import cuda
    n = 1 << lg
    x = random_fr_mont(n, seed=100 + lg)
    for d, t in MODES:
        got = x.copy()
        cuda.NTT(n, got, cuda.NTTInputOutputOrder.NN, cuda.NTTDirection(d), cuda.NTTType(t))
        want = oracle_cpu.ntt(x, d, t)
        assert (got == want).all(), (lg, d, t)


@pytest.mark.parametrize("lg", [20, 21, 22, 25])
def test_ntt_host_ffi_pipelined_vs_oracle(oracle_cpu, lg, monkeypatch):
    """snarkvm_ntt from 2^20 elements: the host buffer is uploaded / downloaded by column ranges under the first and last pass
    (ntt_host_pipelined) — pageable numpy memory (staged through the pinned ring row by row) and pinned memory (2-D DMA straight
    from the caller's buffer), all four transforms; the plain path (switch off) must agree.  2^25 is a four-pass plan: two
    middle passes between the column ranges, and 32 ranges for the 1 GiB pageable buffer."""
    import torch
    from snarkvm_b200 import cuda
    n = 1 << lg
    x = put_near_r(random_fr_mont(n, seed=300 + lg))
    pinned = torch.empty((n, 4), dtype=torch.int64).pin_memory()
    for d, t in MODES:
        want = oracle_cpu.ntt(x, d, t)
        got = x.copy()
        cuda.NTT(n, got, cuda.NTTInputOutputOrder.NN, cuda.NTTDirection(d), cuda.NTTType(t))
        assert (got == want).all(), (lg, d, t, "pageable")
        pinned.numpy()[:] = x.view(np.int64)
        buf = pinned.numpy().view(np.uint64)
        cuda.NTT(n, buf, cuda.NTTInputOutputOrder.NN, cuda.NTTDirection(d), cuda.NTTType(t))
        assert (buf == want).all(), (lg, d, t, "pinned")
    got = x.copy()                                                        # the other orders keep the plain path
    cuda.NTT(n, got, cuda.NTTInputOutputOrder.NR, cuda.NTTDirection(0), cuda.NTTType(0))
    back = got.copy()
    cuda.NTT(n, back, cuda.NTTInputOutputOrder.RN, cuda.NTTDirection(1), cuda.NTTType(0))
    assert (back == x).all()


@pytest.mark.parametrize("lg", [1, 5, 11, 12, 13, 16, 17, 20, 21])
def test_ntt_device_api_vs_oracle(oracle_cpu, lg):
    from snarkvm_b200.algorithms import EvaluationDomain
    n = 1 << lg
    x = random_fr_mont(n, seed=7 * lg)
    dom = EvaluationDomain.new(n)
    for name, d, t in (("fft_in_place", 0, 0), ("ifft_in_place", 1, 0), ("coset_fft_in_place", 0, 1),
                       ("coset_ifft_in_place", 1, 1)):
        got = _host(getattr(dom, name)(_dev(x)))
        assert (got == oracle_cpu.ntt(x, d, t)).all(), (lg, name)


def test_ntt_resizes_short_input(oracle_cpu):
    """`coeffs.resize(self.size(), T::zero())` (domain.rs:171): 600 coefficients on the size-1024 domain"""
    from snarkvm_b200.algorithms import EvaluationDomain
    x = random_fr_mont(600, seed=5)
    dom = EvaluationDomain.new(600)
    assert dom.size == 1024
    padded = np.zeros((1024, 4), dtype=np.uint64)
    padded[:600] = x
    assert (dom.fft(x) == oracle_cpu.ntt(padded, 0, 0)).all()
    assert (_host(dom.fft(_dev(x))) == oracle_cpu.ntt(padded, 0, 0)).all()


def test_ntt_edge_vectors(oracle_cpu):
    """all-zero, all (r−1), delta and constant inputs"""
    from oracle import bls12_377 as py
    from snarkvm_b200.algorithms import EvaluationDomain
    n = 1 << 13
    dom = EvaluationDomain.new(n)
    rm1 = np.array(py.to_limbs(py.R_MOD - 1, 4), dtype=np.uint64)
    one = np.array(py.to_limbs(py.FR_MONT_R, 4), dtype=np.uint64)
    cases = [np.zeros((n, 4), dtype=np.uint64), np.tile(rm1, (n, 1)), np.tile(one, (n, 1))]
    delta = np.zeros((n, 4), dtype=np.uint64)
    delta[1] = one
    cases.append(delta)
    for x in cases:
        for name, d, t in (("fft", 0, 0), ("ifft", 1, 0), ("coset_fft", 0, 1), ("coset_ifft", 1, 1)):
            assert (getattr(dom, name)(x) == oracle_cpu.ntt(x, d, t)).all(), name


@pytest.mark.parametrize("lg", [20, 24])
def test_ntt_full_size_properties(oracle_cpu, lg):
    """BASELINE config 3 sizes: round trips (fft_composition), linearity, and a strided spot check of
    individual outputs against Horner evaluation with the oracle's field arithmetic."""
    import torch
    from oracle import bls12_377 as py
    from snarkvm_b200 import device
    from snarkvm_b200.cuda import NTTDirection, NTTType
    n = 1 << lg
    x = random_fr_mont(n, seed=lg)
    dx = _dev(x)
    y = device.ntt_(dx.clone(), NTTDirection.Forward, NTTType.Standard)
    back = device.ntt_(y.clone(), NTTDirection.Inverse, NTTType.Standard)
    assert torch.equal(back, dx)
    cy = device.ntt_(dx.clone(), NTTDirection.Forward, NTTType.Coset)
    assert not torch.equal(cy, y)
    assert torch.equal(device.ntt_(cy, NTTDirection.Inverse, NTTType.Coset), dx)
    assert (_host(y) == oracle_cpu.ntt(x, 0, 0)).all()
    # y_0 = Σ x_j and y_{n/2} = Σ (−1)^j x_j, summed with Python integers on the canonical values
    vals = oracle_cpu.fr_from_mont(x)
    def to_int(rows):
        acc = 0
        for k in range(4):
            acc += sum(int(v) for v in rows[:, k]) << (64 * k)
        return acc
    s_even, s_odd = to_int(vals[0::2]), to_int(vals[1::2])
    yh = _host(y[[0, n // 2]])
    assert py.fr_from_mont(py.from_limbs(yh[0])) == (s_even + s_odd) % py.R_MOD
    assert py.fr_from_mont(py.from_limbs(yh[1])) == (s_even - s_odd) % py.R_MOD


def test_polymul_vs_oracle(oracle_cpu):
    """snarkvm_polymul / PolyMultiplier::multiply (multiplier.rs:70-134) incl. the corner cases of snarkvm.cu:195-210"""
    from snarkvm_b200 import cuda
    from snarkvm_b200.algorithms import PolyMultiplier
    p1, p2, p3 = random_fr_mont(300, 1), random_fr_mont(500, 2), random_fr_mont(200, 3)
    got = cuda.polymul(1024, [p1, p2, p3], [])
    assert (got == oracle_cpu.polymul([p1, p2, p3], [], 10)).all()
    e = random_fr_mont(1024, 4)
    assert (cuda.polymul(1024, [p1, p2], [e]) == oracle_cpu.polymul([p1, p2], [e], 10)).all()
    assert (cuda.polymul(1024, [p1], []) == oracle_cpu.polymul([p1], [], 10)).all()           # 1 polynomial ⇒ copy
    assert (cuda.polymul(1024, [], [e]) == oracle_cpu.ntt(e, 1, 0)).all()                     # 1 evaluation ⇒ iNTT
    assert (cuda.polymul(1024, [], []) == 0).all()                                            # nothing ⇒ untouched zeros
    pm = PolyMultiplier()
    pm.add_polynomial(p1, "a"); pm.add_polynomial(p2, "b")
    assert (pm.multiply() == oracle_cpu.polymul([p1, p2], [], 10)).all()
    pm = PolyMultiplier()
    pm.add_polynomial(_dev(p1)); pm.add_polynomial(_dev(p3))
    assert (_host(pm.multiply()) == oracle_cpu.polymul([p1, p3], [], 9)).all()
    big1, big2 = random_fr_mont(1 << 15, 8), random_fr_mont(1 << 15, 9)
    assert (cuda.polymul(1 << 16, [big1, big2], []) == oracle_cpu.polymul([big1, big2], [], 16)).all()


def test_fr_mont_conversions(oracle_cpu):
    from snarkvm_b200 import device
    x = random_fr_mont(5000, seed=77)
    assert (_host(device.fr_from_mont(_dev(x))) == oracle_cpu.fr_from_mont(x)).all()
    assert (_host(device.fr_to_mont(_dev(x))) == oracle_cpu.fr_to_mont(x)).all()


def _bitrev_perm(n):
    lg = n.bit_length() - 1
    idx = np.arange(n, dtype=np.uint64)
    rev = np.zeros(n, dtype=np.uint64)
    for b in range(lg):
        rev |= ((idx >> np.uint64(b)) & np.uint64(1)) << np.uint64(lg - 1 - b)
    return rev.astype(np.int64)


@pytest.mark.parametrize("lg", [3, 10, 13])
def test_ntt_input_output_orders(oracle_cpu, lg):
    """NR / RN / RR of the FFI enum (lib.rs:22-28): R = bit-reversed index order on that side."""
    from snarkvm_b200 import cuda
    n = 1 << lg
    x = random_fr_mont(n, seed=900 + lg)
    perm = _bitrev_perm(n)
    for d, t in MODES:
        want = oracle_cpu.ntt(x, d, t)
        got = x.copy(); cuda.NTT(n, got, cuda.NTTInputOutputOrder.NR, cuda.NTTDirection(d), cuda.NTTType(t))
        assert (got == want[perm]).all()
        got = np.ascontiguousarray(x[perm]); cuda.NTT(n, got, cuda.NTTInputOutputOrder.RN, cuda.NTTDirection(d), cuda.NTTType(t))
        assert (got == want).all()
        got = np.ascontiguousarray(x[perm]); cuda.NTT(n, got, cuda.NTTInputOutputOrder.RR, cuda.NTTDirection(d), cuda.NTTType(t))
        assert (got == want[perm]).all()


@pytest.mark.parametrize("lg", [22, 23, 24, 25])
def test_ntt_large_sizes_vs_oracle(oracle_cpu, lg):
    """BASELINE config 3 (and the sizes between, whose pass splits differ: 8+7+7, 8+8+7, 8+8+8) and the smallest four-pass
    plan, 7+6+6+6: all four (direction, type) modes against the oracle's fft_in_place, element by element."""
    import torch
    from snarkvm_b200 import device
    from snarkvm_b200.cuda import NTTDirection, NTTType
    n = 1 << lg
    x = put_near_r(random_fr_mont(n, seed=2200 + lg))
    dx = _dev(x)
    scratch = torch.empty_like(dx)
    for d, t in MODES:
        y = device.ntt_(dx.clone(), NTTDirection(d), NTTType(t), scratch)
        assert (_host(y) == oracle_cpu.ntt(x, d, t)).all(), (lg, d, t)
        del y
