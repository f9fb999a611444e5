"""GPU parity: the CUDA MSM vs the oracle, bit-exact on the to_affine()-normalised projective image.
Restates test_msm / test_msm_cuda (algorithms/src/msm/variable_base/mod.rs:90-119: sizes 1…1000 and
2^2…2^16 vs the CPU algorithms) and the unequal-length test (msm/tests.rs:53-67)."""
import os
import random

import numpy as np
import pytest

from oracle import bls12_377 as py

from helpers import (affine_array, generated_base_multiplier, generated_base_multipliers, oracle_bases,
                     random_canonical_fr, scalars_from_ints)

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _dev(x):
    import torch
    if x.dtype == np.uint64:
        x = x.view(np.int64)
    return torch.from_numpy(x.copy()).cuda()


@pytest.fixture(scope="module")
def bases64k(oracle_cpu):
    return oracle_bases(oracle_cpu, 1 << 16, seed=3)


@pytest.mark.parametrize("n", [1, 2, 3, 5, 10, 14, 15, 16, 31, 32, 33, 50, 100, 500, 1000, 1024, 1025, 4096, 1 << 14, 1 << 16])
def test_msm_host_ffi_vs_oracle(oracle_cpu, bases64k, n):
    """through the drop-in symbol snarkvm_msm with HOST buffers, as variable_base/mod.rs:33-42 calls it"""
    from snarkvm_b200.algorithms import VariableBase
    scal = random_canonical_fr(n, seed=n)
    got = VariableBase.msm(bases64k[:n], scal)
    want = oracle_cpu.msm(bases64k[:n], scal, oracle_cpu.BATCHED)
    assert (got == want).all(), n
    if n <= 1000:
        assert (got == oracle_cpu.msm(bases64k[:n], scal, oracle_cpu.NAIVE)).all()


def test_msm_unequal_lengths(oracle_cpu, bases64k):
    from snarkvm_b200.algorithms import VariableBase
    scal = random_canonical_fr(700, seed=1)
    assert (VariableBase.msm(bases64k[:1000], scal) == oracle_cpu.msm(bases64k[:700], scal, 0)).all()


def test_msm_edge_scalars_and_points(oracle_cpu, bases64k):
    """zero / one / r−1 scalars, ∞ bases, duplicated bases with equal scalars (doubling inside a bucket),
    P and −P with equal scalars (cancellation inside a bucket)."""
    from snarkvm_b200.algorithms import VariableBase
    n = 2048
    bases = bases64k[:n].copy()
    scal = random_canonical_fr(n, seed=9)
    scal[0:16] = 0
    scal[16:32] = scalars_from_ints([1])[0]
    scal[32:48] = scalars_from_ints([py.R_MOD - 1])[0]
    bases[48:64, 96] = 1                                              # infinity flag set (coordinates ignored)
    bases[100:200] = bases[300]; scal[100:200] = scal[300]           # 101 copies of one (point, scalar)
    neg = affine_array([py.g1_neg(py.affine_from_bytes(bases[400].tobytes()))])[0]
    bases[401] = neg; scal[401] = scal[400]
    got = VariableBase.msm(bases, scal)
    assert (got == oracle_cpu.msm(bases, scal, 0)).all()
    assert (got == oracle_cpu.msm(bases, scal, 1)).all()


def test_msm_degenerate_results(oracle_cpu, bases64k):
    from snarkvm_b200.algorithms import VariableBase
    inf = np.frombuffer(py.projective_bytes_normalised(None), dtype=np.uint64)
    n = 512
    zeros = np.zeros((n, 4), dtype=np.uint64)
    assert (VariableBase.msm(bases64k[:n], zeros) == inf).all()                         # all-zero scalars
    allinf = bases64k[:n].copy(); allinf[:, 96] = 1
    assert (VariableBase.msm(allinf, random_canonical_fr(n, 4)) == inf).all()           # all-∞ bases
    assert (VariableBase.msm(bases64k[:n], zeros[:0]) == inf).all()                     # empty
    # Σ s·P + Σ s·(−P) = ∞
    pts = [py.affine_from_bytes(bases64k[i].tobytes()) for i in range(64)]
    both = affine_array(pts + [py.g1_neg(p) for p in pts])
    s = random_canonical_fr(64, 5)
    assert (VariableBase.msm(both, np.concatenate([s, s])) == inf).all()


def test_msm_skewed_distributions(oracle_cpu, bases64k):
    """the reference bench's shape (benches/msm/variable_base.rs:29-32): few distinct bases repeated many
    times, and ALL scalars equal — every window has one hot bucket."""
    from snarkvm_b200.algorithms import VariableBase
    n = 1 << 15
    rep = np.tile(bases64k[:32], (n // 32, 1))
    scal = random_canonical_fr(n, seed=13)
    assert (VariableBase.msm(rep, scal) == oracle_cpu.msm(rep, scal, 1)).all()
    same = np.tile(scal[:1], (n, 1))
    got = VariableBase.msm(bases64k[:n], same)
    assert (got == oracle_cpu.msm(bases64k[:n], same, 1)).all()
    assert (VariableBase.msm(rep, same) == oracle_cpu.msm(rep, same, 1)).all()


def test_msm_real_srs_points(oracle_cpu):
    with open(os.path.join(HERE, "golden", "powers_of_beta_15_first512.usrs"), "rb") as f:
        pts = py.parse_usrs_points(f.read(), 512)
    from snarkvm_b200.algorithms import VariableBase
    bases = affine_array(pts)
    scal = random_canonical_fr(512, seed=21)
    got = VariableBase.msm(bases, scal)
    assert (got == oracle_cpu.msm(bases, scal, 0)).all()
    sc_int = [py.from_limbs(r) for r in scal[:48]]
    assert VariableBase.msm(bases[:48], scal[:48]).tobytes() == py.projective_bytes_normalised(py.msm_naive(pts[:48], sc_int))


def test_generated_bases_match_scalar_multiples(oracle_cpu):
    """snarkvm_b200_generate_bases_device: P_i = h(seed, i)·G — checked against the oracle's mul_bits."""
    from snarkvm_b200 import device
    seed = 0xB200
    b = device.generate_bases(300, seed).cpu().numpy()
    g = affine_array([py.G1_GENERATOR])[0]
    for i in (0, 1, 2, 77, 299):
        k = generated_base_multiplier(seed, i)
        want = oracle_cpu.g1_mul(g, scalars_from_ints([k])[0])
        assert b[i, 96] == 0 and (b[i, 97:] == 0).all()
        assert b[i, :96].tobytes() == want.tobytes()[:96], i
        assert oracle_cpu.g1_is_on_curve(b[i])


@pytest.mark.parametrize("lg", [17, 18])
def test_msm_device_api_vs_oracle(oracle_cpu, lg):
    from snarkvm_b200 import device
    n = 1 << lg
    bases = device.generate_bases(n, seed=lg)
    scal = random_canonical_fr(n, seed=lg)
    got = device.msm(bases, _dev(scal))
    assert (got == oracle_cpu.msm(bases.cpu().numpy(), scal, 0)).all()


def test_kzg_commit_vs_oracle(oracle_cpu):
    """KZG10::commit core: Montgomery coefficients → to_bigint → MSM (kzg10/mod.rs:98-156, 455-474)"""
    from snarkvm_b200.algorithms import KZG10
    from snarkvm_b200 import device
    n = 1 << 14
    powers = device.generate_bases(n, seed=99)
    coeffs = random_canonical_fr(n, seed=31)              # Montgomery images of random field elements
    coeffs[-100:] = 0                                     # trailing zero coefficients (skip_leading_zeros…)
    got = KZG10.commit(powers, _dev(coeffs))
    plain = oracle_cpu.fr_from_mont(coeffs)
    assert (got == oracle_cpu.msm(powers.cpu().numpy(), plain, 0)).all()


def test_window_sums_and_host_finish(oracle_cpu):
    """the sharded-MSM pieces on one GPU: window sums in HBM → host fold == full MSM; and two half shards
    summed by the device rank-sum kernel == the full MSM."""
    import torch
    from snarkvm_b200 import device
    n = 1 << 13
    bases = device.generate_bases(n, seed=5)
    scal = random_canonical_fr(n, seed=6)
    dscal = _dev(scal)
    plan = device.msm_plan(n)
    sums = device.msm_window_sums(bases, dscal)
    want = oracle_cpu.msm(bases.cpu().numpy(), scal, 0)
    assert (device.msm_finish(sums.cpu().numpy(), plan["c"]) == want).all()
    h = n // 2
    planh = device.msm_plan(h)
    s0 = device.msm_window_sums(bases[:h].contiguous(), dscal[:h].contiguous())
    s1 = device.msm_window_sums(bases[h:].contiguous(), dscal[h:].contiguous())
    tot = device.xyzz_sum_ranks(torch.stack([s0, s1]).contiguous(), 2, planh["nwin"])
    assert (device.msm_finish(tot.cpu().numpy(), planh["c"]) == want).all()


# default plans (c, pair levels) of the sizes below: 2^19, 2^21 and 2^23 are the only sizes that run c = 13, and c = 16 / 17
# with 4 / 5 levels, on the plain path
DEFAULT_PLANS = {19: (13, 2), 20: (15, 3), 21: (16, 4), 22: (16, 4), 23: (17, 5), 24: (17, 5)}


@pytest.mark.parametrize("lg", [19, 20, 21, 22, 23, 24])
def test_msm_full_size_properties(oracle_cpu, lg):
    """BASELINE config 2 sizes through size-independent properties: (1) bases are known multiples k_i·G, so
    Σ s_i·P_i = (Σ s_i·k_i mod r)·G — one scalar multiplication by the oracle; (2) linearity in the scalars;
    (3) up to 2^20 also the full oracle MSM."""
    from snarkvm_b200 import device
    n = 1 << lg
    seed = 1000 + lg
    p = device.msm_plan(n)
    assert (p["c"], p["levels"]) == DEFAULT_PLANS[lg]
    bases = device.generate_bases(n, seed)
    scal = random_canonical_fr(n, seed=lg)
    got = device.msm(bases, _dev(scal))
    # (1) closed form
    ks = np.zeros((n, 4), dtype=np.uint64)
    ks[:, 0] = generated_base_multipliers(seed, n)
    dot = oracle_cpu.fr_dot_canonical(scal, ks)
    g = affine_array([py.G1_GENERATOR])[0]
    want = oracle_cpu.g1_mul(g, dot)
    assert (got == want).all()
    if lg <= 20:
        assert (got == oracle_cpu.msm(bases.cpu().numpy(), scal, 0)).all()
    # (2) msm(s) + msm(t) == msm(s + t mod r)
    t = random_canonical_fr(n, seed=lg + 50)
    st = np.empty_like(scal)
    for i0 in range(0, n, 1 << 18):
        a = scal[i0:i0 + (1 << 18)]
        b = t[i0:i0 + (1 << 18)]
        st[i0:i0 + (1 << 18)] = _add_mod_r(a, b)
    lhs = oracle_cpu.g1_add(got, device.msm(bases, _dev(t)))
    assert (lhs == device.msm(bases, _dev(st))).all()


@pytest.mark.parametrize("lg", [19, 21, 23])
def test_msm_full_size_adversarial(oracle_cpu, lg):
    """The default plans of 2^19, 2^21 and 2^23 points on a hostile input, by the closed form: a run of one repeated
    (point, scalar), points next to their negations with equal scalars, ∞ rows, and half of all scalars equal (a hot bucket in
    every window over a full background, through every pair level and the hot-bucket folds)."""
    import torch
    import msm_corpus as mc
    from snarkvm_b200 import device
    n = 1 << lg
    seed = 3000 + lg
    bases = device.generate_bases(n, seed)
    ks = np.zeros((n, 4), dtype=np.uint64)
    ks[:, 0] = generated_base_multipliers(seed, n)
    idx = np.arange(n // 3, n // 3 + 6000)                           # edited rows: a small slice, so the host copy stays small
    b = mc.Bases(bases[idx[0]:idx[-1] + 1].cpu().numpy(), ks[idx].copy())
    b.repeat(0, np.arange(1, 2000))
    b.alternate(2000, np.arange(2000, 2200))
    pairs = np.arange(2200, 4000, 2)                                   # P_i, −P_i with equal scalars
    b.rows[pairs + 1] = b.rows[pairs]
    b.ks[pairs + 1] = b.ks[pairs]
    b.negate(pairs + 1)
    b.infinity(np.arange(4000, 4100))
    bases[idx[0]:idx[-1] + 1] = torch.from_numpy(b.rows).cuda()
    ks[idx] = b.ks
    scal = random_canonical_fr(n, seed=lg + 11)
    rng = np.random.default_rng(lg)
    scal[rng.permutation(n)[: n // 2]] = scal[0]
    scal[idx[:2000]] = scal[idx[0]]
    scal[idx[2000:2200]] = scal[idx[2000]]
    scal[idx[pairs + 1]] = scal[idx[pairs]]
    b.ks = ks
    got = device.msm(bases, _dev(scal))
    assert (got == mc.closed_form(oracle_cpu, b, scal)).all()


def _add_mod_r(a, b):
    """(a + b) mod r on uint64 [n, 4] limb arrays (vectorised carry chain)."""
    r = np.array(py.to_limbs(py.R_MOD, 4), dtype=np.uint64)
    out = np.empty_like(a)
    carry = np.zeros(a.shape[0], dtype=np.uint64)
    for k in range(4):
        s = a[:, k] + b[:, k]
        c1 = s < a[:, k]
        s2 = s + carry
        c2 = s2 < s
        out[:, k] = s2
        carry = (c1 | c2).astype(np.uint64)
    # subtract r where out >= r (no carry out of 256 bits since a, b < r < 2^253)
    ge = np.ones(a.shape[0], dtype=bool); gt = np.zeros(a.shape[0], dtype=bool)
    for k in (3, 2, 1, 0):
        gt |= ge & (out[:, k] > r[k]); ge &= out[:, k] == r[k]
    sel = gt | ge
    borrow = np.zeros(a.shape[0], dtype=np.uint64)
    sub = np.empty_like(out)
    for k in range(4):
        d = out[:, k] - r[k]
        b1 = out[:, k] < r[k]
        d2 = d - borrow
        b2 = d < borrow
        sub[:, k] = d2
        borrow = (b1 | b2).astype(np.uint64)
    out[sel] = sub[sel]
    return out


@pytest.mark.parametrize("levels,c", [(1, 6), (2, 7), (4, 5), (6, 4)])
def test_msm_pair_levels_edge_cases(oracle_cpu, bases64k, monkeypatch, levels, c):
    """The batched-affine pair levels (normally enabled only from 2^21 points) forced on small inputs so that
    their special cases run: equal points (doubling through 2·y), opposite points (cancellation to ∞), ∞ inputs,
    odd bucket sizes, hot buckets (all scalars equal) and repeated bases."""
    from snarkvm_b200.algorithms import VariableBase
    monkeypatch.setenv("SNARKVM_B200_MSM_LEVELS", str(levels))
    monkeypatch.setenv("SNARKVM_B200_MSM_C", str(c))
    n = 3000
    bases = bases64k[:n].copy()
    scal = random_canonical_fr(n, seed=40 + levels)
    scal[0:16] = 0
    scal[16:32] = scalars_from_ints([1])[0]
    scal[32:48] = scalars_from_ints([py.R_MOD - 1])[0]
    bases[48:64, 96] = 1
    bases[100:301] = bases[400]; scal[100:301] = scal[400]            # 202 copies of one (point, scalar): doublings at every level
    neg = affine_array([py.g1_neg(py.affine_from_bytes(bases[500].tobytes()))])[0]
    bases[501:521:2] = neg; bases[502:522:2] = bases[500]; scal[500:522] = scal[500]   # P, −P, P, −P … in the same buckets
    want = oracle_cpu.msm(bases, scal, 1)
    assert (VariableBase.msm(bases, scal) == want).all()
    same = np.tile(scal[700:701], (n, 1))                             # every window has one hot bucket
    assert (VariableBase.msm(bases, same) == oracle_cpu.msm(bases, same, 1)).all()
    rep = np.tile(bases64k[:8], (n // 8, 1))                           # 8 distinct bases repeated
    assert (VariableBase.msm(rep, scal) == oracle_cpu.msm(rep, scal, 1)).all()
    assert (VariableBase.msm(rep, same) == oracle_cpu.msm(rep, same, 1)).all()
    inf = np.frombuffer(py.projective_bytes_normalised(None), dtype=np.uint64)
    assert (VariableBase.msm(bases, np.zeros((n, 4), dtype=np.uint64)) == inf).all()


@pytest.mark.parametrize("levels,c,mb", [(1, 9, 2), (3, 8, 9), (2, 11, 13)])
def test_msm_record_scatter_window_groups(oracle_cpu, bases64k, monkeypatch, levels, c, mb):
    """The record-scatter sort (k_scatter_records) with a scratch budget so small that the bucket sets are processed in many
    groups: every group re-derives the digits and emits only its own windows; jobs of a batch and the hiding segment (second
    base array) cross group boundaries too."""
    from snarkvm_b200 import device
    from snarkvm_b200.algorithms import KZG10, VariableBase
    monkeypatch.setenv("SNARKVM_B200_MSM_LEVELS", str(levels))
    monkeypatch.setenv("SNARKVM_B200_MSM_C", str(c))
    monkeypatch.setenv("SNARKVM_B200_MSM_SCRATCH_MB", str(mb))
    n = 20000
    bases = bases64k[:n].copy()
    scal = random_canonical_fr(n, seed=77 + levels)
    scal[:40] = 0
    bases[40:60, 96] = 1                                              # points at infinity
    scal[100:400] = scal[99]                                          # a hot bucket in every window
    assert (VariableBase.msm(bases, scal) == oracle_cpu.msm(bases, scal, 1)).all()
    # a batch whose jobs straddle group boundaries, Montgomery coefficients, with blinding terms on a second base array
    dbases = _dev(bases64k)
    gamma = device.generate_bases(8, seed=99)
    gamma_h = gamma.cpu().numpy()
    lens, blens = [9000, 0, 20000, 1, 13000], [3, 2, 0, 0, 8]
    polys = [random_canonical_fr(k, seed=300 + i) for i, k in enumerate(lens)]
    blinds = [random_canonical_fr(k, seed=400 + i) if k else None for i, k in enumerate(blens)]
    got = KZG10.batch_commit(dbases, [_dev(p) for p in polys], gamma, [None if b is None else _dev(b) for b in blinds])
    for i, (p, b) in enumerate(zip(polys, blinds)):
        want = oracle_cpu.msm(bases64k[:len(p)], oracle_cpu.fr_from_mont(p), 0)
        if b is not None:
            want = oracle_cpu.g1_add(want, oracle_cpu.msm(gamma_h[:len(b)], oracle_cpu.fr_from_mont(b), 0))
        assert (got[i] == want).all(), i


def test_registered_bases(oracle_cpu, bases64k):
    """snarkvm_b200_register_bases: snarkvm_msm recognises the registered host pointer and skips the upload"""
    from snarkvm_b200 import CudaError, cuda
    n = 5000
    pts = np.ascontiguousarray(bases64k[:n])
    scal = random_canonical_fr(n, seed=3)
    want = oracle_cpu.msm(pts, scal, 0)
    cuda.register_bases(pts)
    try:
        assert (cuda.msm(pts, scal) == want).all()
        assert (cuda.msm(pts, scal[:1234]) == oracle_cpu.msm(pts[:1234], scal[:1234], 0)).all()   # prefix of the registered slice
    finally:
        cuda.unregister_bases(pts)
    assert (cuda.msm(pts, scal) == want).all()                      # falls back to uploading
    with pytest.raises(CudaError):
        cuda.unregister_bases(pts)


def test_ffi_concurrent_callers(oracle_cpu, bases64k):
    """The reference enters the FFI from many rayon workers at once (sonic_pc/mod.rs:186-245: all commitments of a
    round in parallel; ExecutionPool of FFTs).  Eight host threads call snarkvm_msm / snarkvm_ntt concurrently
    (ctypes releases the GIL); every result must equal the oracle's."""
    import threading
    from snarkvm_b200 import cuda
    from helpers import random_fr_mont
    jobs, results, errors = [], {}, []
    for k in range(8):
        n = 3000 + 517 * k
        scal = random_canonical_fr(n, seed=200 + k)
        x = random_fr_mont(1 << (10 + k % 4), seed=300 + k)
        jobs.append((k, n, scal, x))

    def work(k, n, scal, x):
        try:
            for _ in range(3):
                m = cuda.msm(bases64k[:n], scal)
                y = x.copy()
                cuda.NTT(x.shape[0], y, cuda.NTTInputOutputOrder.NN, cuda.NTTDirection.Forward, cuda.NTTType.Coset)
            results[k] = (m, y)
        except Exception as e:      # pragma: no cover
            errors.append(e)

    threads = [threading.Thread(target=work, args=j) for j in jobs]
    [t.start() for t in threads]
    [t.join() for t in threads]
    assert not errors, errors
    for k, n, scal, x in jobs:
        assert (results[k][0] == oracle_cpu.msm(bases64k[:n], scal, 0)).all(), k
        assert (results[k][1] == oracle_cpu.ntt(x, 0, 1)).all(), k


def test_srs_decode_real_powers(oracle_cpu):
    """SRS ingest: the first 512 mainnet powers (uncompressed canonical) decoded on the device == the reference's in-memory
    Affine images; a corrupted coordinate, an out-of-range coordinate and an infinity record are detected / handled."""
    import torch
    from snarkvm_b200 import device
    with open(os.path.join(HERE, "golden", "powers_of_beta_15_first512.usrs"), "rb") as f:
        blob = f.read()
    pts = py.parse_usrs_points(blob, 512)
    payload = np.frombuffer(blob[8:8 + 512 * 96], dtype=np.uint8).copy()
    bases, invalid = device.srs_decode(torch.from_numpy(payload).cuda())
    assert invalid == 0
    assert (bases.cpu().numpy() == affine_array(pts)).all()
    bad = payload.copy()
    bad[5 * 96 + 3] ^= 1                                   # point 5: x changed → off the curve
    bad[9 * 96:9 * 96 + 48] = 0xFF; bad[9 * 96 + 47] = 0x3F   # point 9: x ≥ q
    bad[12 * 96:13 * 96] = 0; bad[12 * 96 + 95] = 0x40        # point 12: infinity
    got, invalid = device.srs_decode(torch.from_numpy(bad).cuda())
    assert invalid == 2
    g = got.cpu().numpy()
    assert g[12].tobytes() == py.affine_bytes(None)
    keep = [i for i in range(512) if i not in (5, 9, 12)]
    assert (g[keep] == affine_array(pts)[keep]).all()


@pytest.mark.parametrize("n,pre_c,pre_levels", [(3000, 5, 1), (3000, 7, 3), (1 << 14, None, None), (1 << 17, None, None)])
def test_precomputed_bases_vs_oracle(oracle_cpu, bases64k, monkeypatch, n, pre_c, pre_levels):
    """Fixed-base tables 2^{c·w}·P_i (snarkvm_b200_msm_precompute_device): same group element as the oracle MSM, for full and
    prefix lengths (kzg10/mod.rs:121-135 slices the powers), with the pair-level special cases in play (equal / opposite points,
    ∞ bases, hot buckets — now ACROSS windows, since all windows share one bucket set)."""
    from snarkvm_b200 import device
    if pre_c is not None:
        monkeypatch.setenv("SNARKVM_B200_MSM_PRE_C", str(pre_c))
        monkeypatch.setenv("SNARKVM_B200_MSM_PRE_LEVELS", str(pre_levels))
    if n <= (1 << 16):
        bases = bases64k[:n].copy()
        bases[48:64, 96] = 1
        bases[100:301] = bases[400]
        neg = affine_array([py.g1_neg(py.affine_from_bytes(bases[500].tobytes()))])[0]
        bases[501:521:2] = neg; bases[502:522:2] = bases[500]
        dbases = _dev(bases)
    else:
        dbases = device.generate_bases(n, seed=77)
        bases = dbases.cpu().numpy()
    pre = device.PrecomputedBases(dbases)
    assert pre.npoints == n and pre.table_bytes == n * pre.nwin * 128
    scal = random_canonical_fr(n, seed=60 + (pre_c or 0))
    scal[0:16] = 0
    scal[16:32] = scalars_from_ints([1])[0]
    scal[32:48] = scalars_from_ints([py.R_MOD - 1])[0]
    scal[100:301] = scal[400]
    scal[500:522] = scal[500]
    assert (pre.msm(_dev(scal)) == oracle_cpu.msm(bases, scal, 1)).all()
    for m in (1, 2, 700, n - 1):
        assert (pre.msm(_dev(scal[:m])) == oracle_cpu.msm(bases[:m], scal[:m], 1)).all(), m
    same = np.tile(scal[700:701], (n, 1))
    assert (pre.msm(_dev(same)) == oracle_cpu.msm(bases, same, 1)).all()
    inf = np.frombuffer(py.projective_bytes_normalised(None), dtype=np.uint64)
    assert (pre.msm(_dev(np.zeros((n, 4), dtype=np.uint64))) == inf).all()
    assert (pre.msm(_dev(scal)[:0]) == inf).all()
    # KZG commit over the table: Montgomery coefficients in, to_bigint on the device
    coeffs = random_canonical_fr(n, seed=61)
    assert (pre.kzg_commit(_dev(coeffs)) == oracle_cpu.msm(bases, oracle_cpu.fr_from_mont(coeffs), 1)).all()
    with pytest.raises(ValueError):
        pre.msm(_dev(random_canonical_fr(n + 1, seed=1)))
    pre.free()


def test_precomputed_bases_full_size(oracle_cpu):
    """2^22 points through the closed form Σ s_i·k_i·G (bases are known multiples of G) and against the windowed path"""
    from snarkvm_b200 import device
    lg = 22
    n = 1 << lg
    seed = 2000 + lg
    bases = device.generate_bases(n, seed)
    pre = device.PrecomputedBases(bases)
    scal = random_canonical_fr(n, seed=lg + 7)
    got = pre.msm(_dev(scal))
    ks = np.zeros((n, 4), dtype=np.uint64)
    ks[:, 0] = generated_base_multipliers(seed, n)
    g = affine_array([py.G1_GENERATOR])[0]
    assert (got == oracle_cpu.g1_mul(g, oracle_cpu.fr_dot_canonical(scal, ks))).all()
    assert (got == device.msm(bases, _dev(scal))).all()
    pre.free()


@pytest.mark.parametrize("chunks,n", [("2", 3001), ("3", 1 << 14), ("16", 20), ("5", 4), ("1:3:4", 1 << 14), ("7:1", 1000)])
def test_msm_ffi_chunked_upload(oracle_cpu, bases64k, monkeypatch, chunks, n):
    """snarkvm_msm cuts big host buffers into point ranges whose upload overlaps the previous range's kernels
    (default: 1/8, 3/8, 1/2 of the points from 2^23); forced here on small inputs, including ranges of one point."""
    from snarkvm_b200.algorithms import VariableBase
    monkeypatch.setenv("SNARKVM_B200_MSM_CHUNKS", str(chunks))
    scal = random_canonical_fr(n, seed=len(chunks) + n)
    scal[0] = 0
    bases = bases64k[:n].copy()
    bases[1, 96] = 1
    assert (VariableBase.msm(bases, scal) == oracle_cpu.msm(bases, scal, 1)).all()


def test_registered_bases_precomputed(oracle_cpu, bases64k):
    """snarkvm_b200_register_bases_precomputed: snarkvm_msm on the registered slice runs over the fixed-base tables — same group
    element, also for a prefix of the slice (fewer scalars than registered points)."""
    from snarkvm_b200 import cuda
    n = 5000
    bases = np.ascontiguousarray(bases64k[:n])
    scal = random_canonical_fr(n, seed=88)
    cuda.register_bases_precomputed(bases)
    try:
        assert (cuda.msm(bases, scal) == oracle_cpu.msm(bases, scal, 0)).all()
        assert (cuda.msm(bases, scal[:1234]) == oracle_cpu.msm(bases[:1234], scal[:1234], 0)).all()
    finally:
        cuda.unregister_bases(bases)
    assert (cuda.msm(bases, scal) == oracle_cpu.msm(bases, scal, 0)).all()      # plain path again after unregistering


@pytest.mark.parametrize("lg,levels", [(16, None), (16, 2), (17, 1), (18, None), (18, 3)])
def test_msm_half_repeated_scalars(oracle_cpu, monkeypatch, lg, levels):
    """Half of the scalars equal to ONE random value over a uniform background (e.g. commit_lagrange of an evaluation
    vector with a dominant value): every window then has one hot bucket on top of ~all other buckets being non-empty,
    which needs more fold outputs than #buckets + hot/32 (round-1 ADVICE: the fold launch was sized from the hottest
    bucket only and left partials unwritten).  With and without pair levels."""
    from snarkvm_b200 import device
    if levels is not None:
        monkeypatch.setenv("SNARKVM_B200_MSM_LEVELS", str(levels))
    n = 1 << lg
    bases = device.generate_bases(n, seed=500 + lg)
    scal = random_canonical_fr(n, seed=700 + lg)
    rng = np.random.default_rng(lg)
    hot = rng.permutation(n)[: n // 2]
    scal[hot] = scal[0]
    got = device.msm(bases, _dev(scal))
    assert (got == oracle_cpu.msm(bases.cpu().numpy(), scal, 0)).all()
    # a few dozen hot values instead of one
    scal2 = random_canonical_fr(n, seed=800 + lg)
    scal2[hot] = scal2[rng.integers(0, 48, size=hot.size)]
    assert (device.msm(bases, _dev(scal2)) == oracle_cpu.msm(bases.cpu().numpy(), scal2, 0)).all()


def test_msm_rejects_scalars_above_253_bits(oracle_cpu, bases64k):
    """Scalars are canonical integers < r < 2^253 (to_bigint output).  A BigInteger256 with bits 253..255 set is outside what the
    signed-digit windows cover: the call must return an error (the Rust caller then falls back to its CPU path,
    variable_base/mod.rs:39-43) instead of a silently wrong point."""
    from snarkvm_b200 import CudaError, cuda
    n = 2000
    scal = random_canonical_fr(n, seed=5)
    assert (cuda.msm(bases64k[:n], scal) == oracle_cpu.msm(bases64k[:n], scal, 0)).all()
    bad = scal.copy()
    bad[777, 3] |= np.uint64(1 << 63)
    with pytest.raises(CudaError):
        cuda.msm(bases64k[:n], bad)
    bad = scal.copy()
    bad[3, 3] |= np.uint64(1 << 61)
    with pytest.raises(CudaError):
        cuda.msm(bases64k[:n], bad)


def test_kzg_commit_hiding_full_size(oracle_cpu):
    """BASELINE config 4: KZG10::commit of a 2^22-coefficient polynomial with hiding_bound = Some(1)
    (kzg10/mod.rs:98-156: commitment + MSM(powers_of_beta_times_gamma_g, blinding polynomial of degree hiding_bound + 1))."""
    from snarkvm_b200 import device
    from snarkvm_b200.algorithms import KZG10
    n = 1 << 22
    powers = device.generate_bases(n, seed=4100)
    gamma = device.generate_bases(8, seed=4101)
    coeffs = random_canonical_fr(n, seed=4102)                 # Montgomery images
    blind = random_canonical_fr(3, seed=4103)                  # hiding_bound + 2 coefficients (degree hiding_bound + 1)
    got = KZG10.commit(powers, _dev(coeffs), gamma, _dev(blind))
    a = oracle_cpu.msm(powers.cpu().numpy(), oracle_cpu.fr_from_mont(coeffs), 0)
    b = oracle_cpu.msm(gamma.cpu().numpy()[:3], oracle_cpu.fr_from_mont(blind), 0)
    assert (got == oracle_cpu.g1_add(a, b)).all()


def test_msm_batch_one_pass(oracle_cpu, bases64k, monkeypatch):
    """snarkvm_b200_msm_batch_device / kzg_commit_batch: many scalar vectors over the same resident bases in ONE pass
    (sonic_pc/mod.rs:177-257) — different lengths, an empty vector, a length-1 vector, equal vectors; every sum must equal the
    oracle's MSM of that vector alone."""
    from snarkvm_b200 import device
    from snarkvm_b200.algorithms import KZG10
    dbases = _dev(bases64k)
    lens = [5000, 0, 1, 65536, 12345, 5000, 777, 40000]
    vecs = [random_canonical_fr(n, seed=900 + i) for i, n in enumerate(lens)]
    vecs[5] = vecs[0].copy()
    got = device.msm_batch(dbases, [_dev(v) for v in vecs])
    for i, v in enumerate(vecs):
        assert (got[i] == oracle_cpu.msm(bases64k[:len(v)], v, 0)).all(), i
    # Montgomery coefficients (KZG commit) + pair levels forced on
    monkeypatch.setenv("SNARKVM_B200_MSM_LEVELS", "3")
    got = KZG10.batch_commit(dbases, [_dev(v) for v in vecs])
    for i, v in enumerate(vecs):
        assert (got[i] == oracle_cpu.msm(bases64k[:len(v)], oracle_cpu.fr_from_mont(v), 0)).all(), i


def test_kzg_commit_batch_hiding_one_pass(oracle_cpu, bases64k):
    """A round of hiding commitments in one pass: polynomial i gets Σ_j blinding_i[j]·gamma_powers[j] through a second scalar
    segment of the same sum; some polynomials are not hiding (None), one is empty but hiding."""
    from snarkvm_b200 import device
    from snarkvm_b200.algorithms import KZG10
    dbases = _dev(bases64k)
    gamma = device.generate_bases(16, seed=31337)
    gamma_h = gamma.cpu().numpy()
    lens = [3000, 20000, 0, 65536, 9]
    blens = [3, 0, 2, 4, 16]
    polys = [random_canonical_fr(n, seed=50 + i) for i, n in enumerate(lens)]
    blinds = [random_canonical_fr(n, seed=70 + i) if n else None for i, n in enumerate(blens)]
    got = KZG10.batch_commit(dbases, [_dev(p) for p in polys], gamma, [None if b is None else _dev(b) for b in blinds])
    for i, (p, b) in enumerate(zip(polys, blinds)):
        want = oracle_cpu.msm(bases64k[:len(p)], oracle_cpu.fr_from_mont(p), 0)
        if b is not None:
            want = oracle_cpu.g1_add(want, oracle_cpu.msm(gamma_h[:len(b)], oracle_cpu.fr_from_mont(b), 0))
        assert (got[i] == want).all(), i
    # the single-commitment entry point takes the same route
    one = KZG10.commit(dbases, _dev(polys[0]), gamma, _dev(blinds[0]))
    assert (one == got[0]).all()


def test_msm_batch_large_round(oracle_cpu):
    """8 × 2^17-coefficient polynomials in one pass (a Varuna-sized round): the batch plan turns pair levels on although each
    polynomial alone would run without them."""
    from snarkvm_b200 import device
    n = 1 << 17
    bases = device.generate_bases(n, seed=4242)
    bh = bases.cpu().numpy()
    vecs = [random_canonical_fr(n - 1000 * i, seed=600 + i) for i in range(8)]
    got = device.msm_batch(bases, [_dev(v) for v in vecs])
    for i, v in enumerate(vecs):
        assert (got[i] == oracle_cpu.msm(bh[:len(v)], v, 0)).all(), i
    pre = device.PrecomputedBases(bases)
    got = pre.kzg_commit_batch([_dev(v) for v in vecs[:4]])
    for i, v in enumerate(vecs[:4]):
        assert (got[i] == oracle_cpu.msm(bh[:len(v)], oracle_cpu.fr_from_mont(v), 0)).all(), i
    pre.free()


def test_msm_concurrent_large_calls_share_scratch_budget(oracle_cpu):
    """Eight host threads call snarkvm_msm with 2^20 points each while the scratch budget only fits about two calls: the others
    must WAIT for their turn (no cudaErrorMemoryAllocation ⇒ silent CPU fallback on the Rust side), all results must be right, and
    the high-water mark must respect the budget."""
    import threading
    from snarkvm_b200 import cuda, device
    n = 1 << 20
    seed = 999
    bases = device.generate_bases(n, seed).cpu().numpy()
    ks = np.zeros((n, 4), dtype=np.uint64)
    ks[:, 0] = generated_base_multipliers(seed, n)
    g = affine_array([py.G1_GENERATOR])[0]
    scal = [random_canonical_fr(n, seed=10 + k) for k in range(8)]
    cuda.msm(bases, scal[0])                                    # warm up: pool + one call's scratch
    one_call = device.msm_scratch_stats()["peak"]
    old_limit = device.msm_scratch_stats()["limit"]
    device.msm_set_scratch_limit(int(one_call * 2.5))
    results, errors = {}, []

    def work(k):
        try:
            results[k] = cuda.msm(bases, scal[k])
        except Exception as e:      # pragma: no cover
            errors.append(e)

    try:
        threads = [threading.Thread(target=work, args=(k,)) for k in range(8)]
        [t.start() for t in threads]
        [t.join() for t in threads]
        st = device.msm_scratch_stats()
    finally:
        device.msm_set_scratch_limit(old_limit)
    assert not errors, errors
    assert st["peak"] <= int(one_call * 2.5) and st["in_use"] == 0
    for k in range(8):
        want = oracle_cpu.g1_mul(g, oracle_cpu.fr_dot_canonical(scal[k], ks))
        assert (results[k] == want).all(), k


def test_warp_cooperative_field_arithmetic_selftest():
    """ff.cuh coop_mul / coop_inverse (one Fq element spread over a warp, used for the CTA-shared inversions of the pair levels)
    against the per-thread multiplier, on the device: 0, 1, q − 1, a long-carry value and 20000 pseudo-random elements."""
    import ctypes
    import torch
    from snarkvm_b200 import _lib
    bad = ctypes.c_uint32(123)
    with torch.cuda.device(0):
        _lib.check(_lib.lib().snarkvm_b200_selftest_coop(20000, 0xC0FFEE, ctypes.byref(bad), torch.cuda.current_stream().cuda_stream))
    assert bad.value == 0


@pytest.mark.gpu
@pytest.mark.parametrize("n", [64, 1000, 4096, 1 << 13, 1 << 15])
def test_msm_quad_latency_path_edge_cases(oracle_cpu, bases64k, n):
    """the four-lanes-per-point tail (csrc/quad.cuh: k_bucket_accumulate_q8 up to 2^12 points, k_bucket_reduce_quad /
    k_window_combine_quad up to 1024 buckets per window) on the inputs that reach its special cases: every scalar equal (one
    bucket per window holds all points: 17 item partials per bucket, no folds), one point repeated with one scalar (doubling
    inside quad_add_affine and quad_add), P and −P with one scalar (cancellation), ∞ points and zero scalars (∞ operands)."""
    from snarkvm_b200.algorithms import VariableBase
    scal = random_canonical_fr(n, seed=100 + n)
    same = np.tile(scal[:1], (n, 1))
    assert (VariableBase.msm(bases64k[:n], same) == oracle_cpu.msm(bases64k[:n], same, 1)).all()
    rep = np.tile(bases64k[7:8], (n, 1))
    assert (VariableBase.msm(rep, same) == oracle_cpu.msm(rep, same, 1)).all()                 # n copies of (P, s)
    assert (VariableBase.msm(rep, scal) == oracle_cpu.msm(rep, scal, 1)).all()                 # one point, random scalars
    mixed = bases64k[:n].copy(); ms = scal.copy()
    half = n // 2
    neg = affine_array([py.g1_neg(py.affine_from_bytes(bases64k[i].tobytes())) for i in range(min(half, 32))])
    mixed[half:half + len(neg)] = neg; ms[half:half + len(neg)] = ms[:len(neg)]               # P_i and −P_i, equal scalars
    mixed[1::5, 96] = 1                                                                         # ∞ points
    ms[2::7] = 0
    ms[3::11] = ms[3]                                                                           # a hot bucket over a background
    got = VariableBase.msm(mixed, ms)
    assert (got == oracle_cpu.msm(mixed, ms, 0)).all()
    assert (got == oracle_cpu.msm(mixed, ms, 1)).all()
