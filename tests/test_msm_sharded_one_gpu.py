"""The sharded MSM (snarkvm_b200/sharded.py) on one GPU, every rank's work run in one process, one rank after another.

A sharded MSM runs every rank under the window plan of the LARGEST shard, so shorter and empty shards run under a plan sized
for more points than they hold; the ranks' window sums are gathered and added window by window (k_xyzz_sum_ranks), and host
buffers go through snarkvm_b200_msm_window_sums_host, which uploads point ranges on a second stream and adds the ranges' sums
on the device.  The only collective, the all-gather, is a torch.stack here.

The bases are generated (P_i = k_i·G with known 64-bit k_i), so each window sum has a closed form in the scalar field:
S_w = (Σ_i d_w(s_i)·k_i mod r)·G, d_w the signed c-bit digit of the uniform recoding.  Every window is checked on its own,
which two wrong windows cannot pass together.  The recoding model needs no GPU; the rest of the module does."""
import sys

import numpy as np
import pytest

from oracle import bls12_377 as py

import msm_corpus as mc
from helpers import generated_base_multipliers, random_canonical_fr, scalars_from_ints
from test_msm_digits_model import recode


def _have_cuda() -> bool:
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:  # noqa: BLE001
        return False


def gpu(f):
    return pytest.mark.gpu(pytest.mark.skipif(not _have_cuda(), reason="needs a CUDA device")(f))


R = py.R_MOD
INF = np.frombuffer(py.projective_bytes_normalised(None), dtype=np.uint64)
G = np.frombuffer(py.affine_bytes(py.G1_GENERATOR), dtype=np.uint8)
# the window sizes of every plan this module runs under (window_closed_forms refuses any other: the model is checked on these)
MODEL_C = (4, 6, 7, 8, 9, 11, 15, 16, 17)


# ---------------------------------------------------------------------------------------------------------------------------
# window-sum oracle
# ---------------------------------------------------------------------------------------------------------------------------
def signed_digits(scalars: np.ndarray, c: int) -> np.ndarray:
    """The uniform signed c-bit recoding of canonical scalars (uint64 [n, 4]) → int64 [nwin, n], nwin = 253 // c + 1:
    window w takes the c-bit field at bit c·w plus the carry out of window w − 1; a value above 2^(c−1) becomes
    value − 2^c and carries one into window w + 1."""
    s = np.ascontiguousarray(scalars, dtype=np.uint64).reshape(-1, 4)
    nwin = 253 // c + 1
    half = 1 << (c - 1)
    mask = np.uint64((1 << c) - 1)
    carry = np.zeros(s.shape[0], dtype=np.int64)
    out = np.empty((nwin, s.shape[0]), dtype=np.int64)
    for w in range(nwin):
        limb, sh = divmod(w * c, 64)
        field = s[:, limb] >> np.uint64(sh)
        if sh and limb < 3:
            field |= s[:, limb + 1] << np.uint64(64 - sh)
        raw = (field & mask).astype(np.int64) + carry
        neg = raw > half
        out[w] = np.where(neg, raw - (1 << c), raw)
        carry = neg.astype(np.int64)
    return out


@pytest.mark.parametrize("c", MODEL_C)
def test_signed_digits_match_the_recoding_model(c):
    """the vectorised recoding gives the device loop's digits (test_msm_digits_model.recode) on the digit-boundary corpus"""
    corpus = mc.digit_boundary_scalars(c)
    got = signed_digits(scalars_from_ints(corpus), c)
    for i, s in enumerate(corpus):
        digits, carry = recode(s, c)
        assert carry == 0
        want = [-mag if neg else mag for _raw, neg, mag in digits]
        assert got[:, i].tolist() == want, (c, s)


def _mul_g(cpu, k: int) -> np.ndarray:
    k %= R
    return INF.copy() if k == 0 else cpu.g1_mul(G, scalars_from_ints([k])[0])


def _fr_int(limbs) -> int:
    return py.from_limbs([int(v) for v in limbs])


def window_closed_forms(cpu, ks: np.ndarray, scalars: np.ndarray, plan_n: int) -> list:
    """The normalised projective image of every window sum S_w = Σ_i d_w(s_i)·P_i under the plan of plan_n points, for bases
    P_i = k_i·G (ks: canonical uint64 [n, 4])."""
    from snarkvm_b200 import device
    plan = device.msm_plan(plan_n)
    c = plan["c"]
    assert c in MODEL_C and plan["nwin"] == 253 // c + 1, plan
    n = scalars.shape[0]
    if n == 0:
        return [INF.copy() for _ in range(plan["nwin"])]
    d = signed_digits(scalars, c)
    out = []
    for w in range(plan["nwin"]):
        pos = np.zeros((n, 4), dtype=np.uint64)
        neg = np.zeros((n, 4), dtype=np.uint64)
        pos[:, 0] = np.where(d[w] > 0, d[w], 0)
        neg[:, 0] = np.where(d[w] < 0, -d[w], 0)
        k = _fr_int(cpu.fr_dot_canonical(pos, ks[:n])) - _fr_int(cpu.fr_dot_canonical(neg, ks[:n]))
        out.append(_mul_g(cpu, k))
    return out


def total_closed_form(cpu, ks: np.ndarray, scalars: np.ndarray) -> np.ndarray:
    if scalars.shape[0] == 0:
        return INF.copy()
    return _mul_g(cpu, _fr_int(cpu.fr_dot_canonical(scalars, ks[:scalars.shape[0]])))


def assert_windows(sums, want: list, what) -> None:
    """every window sum (XYZZ, [nwin, 24] int64 in HBM or on the host) equals its normalised image in `want`"""
    from snarkvm_b200 import device
    h = sums.cpu().numpy() if hasattr(sums, "cpu") else np.asarray(sums)
    assert h.shape[0] == len(want), (what, h.shape, len(want))
    bad = [w for w in range(len(want)) if not (device.msm_finish(h[w:w + 1], 0) == want[w]).all()]
    assert not bad, (what, "wrong windows", bad)


def assert_same_windows(a, b, what) -> None:
    """two sets of window sums are equal window by window as group elements"""
    from snarkvm_b200 import device
    ha, hb = a.cpu().numpy(), b.cpu().numpy()
    assert ha.shape == hb.shape, what
    bad = [w for w in range(ha.shape[0]) if not (device.msm_finish(ha[w:w + 1], 0) == device.msm_finish(hb[w:w + 1], 0)).all()]
    assert not bad, (what, "windows differ", bad)


# ---------------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------------
def _ks(seed: int, n: int) -> np.ndarray:
    ks = np.zeros((n, 4), dtype=np.uint64)
    ks[:, 0] = generated_base_multipliers(seed, n)
    return ks


def _dev(x: np.ndarray):
    import torch
    if x.dtype == np.uint64:
        x = x.view(np.int64)
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _pinned(x: np.ndarray):
    """a page-locked copy of x → (numpy view, the owning tensor)"""
    import torch
    t = torch.empty(x.shape, dtype=torch.uint8 if x.dtype == np.uint8 else torch.int64, pin_memory=True)
    a = t.numpy().view(x.dtype)
    a[...] = x
    return a, t


def _poisoned_out(nwin: int):
    """window-sum buffer filled with a pattern no result has, so a sum the call never wrote shows"""
    import torch
    return torch.full((nwin, 24), 0x5A5A5A5A5A5A5A5A, dtype=torch.int64, device="cuda")


# ---------------------------------------------------------------------------------------------------------------------------
# ranks in one process
# ---------------------------------------------------------------------------------------------------------------------------
def run_ranks(cpu, bases, scal: np.ndarray, ks: np.ndarray, shards: list, plan_n: int, want_total=None):
    """msm_window_sums of every shard (lo, hi) under the plan of plan_n, each rank's windows against their closed forms,
    the gathered ranks added by xyzz_sum_ranks window by window and folded → the normalised total"""
    import torch
    from snarkvm_b200 import device
    plan = device.msm_plan(plan_n)
    dscal = _dev(scal)
    sums = []
    for r, (lo, hi) in enumerate(shards):
        s = device.msm_window_sums(bases[lo:hi], dscal[lo:hi], plan_npoints=plan_n)
        assert tuple(s.shape) == (plan["nwin"], 24)
        assert_windows(s, window_closed_forms(cpu, ks[lo:hi], scal[lo:hi], plan_n), ("rank", r, lo, hi))
        sums.append(s)
    tot = device.xyzz_sum_ranks(torch.stack(sums).contiguous(), len(shards), plan["nwin"])
    got = device.msm_finish(tot.cpu().numpy(), plan["c"])
    if want_total is not None:
        assert (got == want_total).all()
    return tot, got


def _oracle_total(cpu, bases_host: np.ndarray, ks: np.ndarray, scal: np.ndarray) -> np.ndarray:
    """the oracle's MSM up to 2^16 points (and the closed form with it), the closed form above"""
    want = total_closed_form(cpu, ks, scal)
    if scal.shape[0] <= 1 << 16:
        assert (cpu.msm(bases_host[:scal.shape[0]], scal, 0) == want).all()
    return want


@gpu
@pytest.mark.parametrize("n, world, plan_n", [
    (3, 8, None),                   # one point in each of three ranks, five empty ranks
    (9, 8, None),                   # 2, 2, 2, 2, 1 points and three empty ranks
    (17377, 3, None),               # 5793, 5793, 5791: the last shard's own plan has another c
    (2000, 2, 1 << 20),             # 1000-point shards under c = 15 with three pair levels
    (2000, 2, 1 << 22),             # … and under c = 16 with four
    (1 << 17, 2, 1 << 20),          # 2^16-point shards under the same plans
    (1 << 17, 2, 1 << 22),
    (1 << 20, 8, None),             # eight 2^17-point ranks
])
def test_ranks_under_the_largest_shards_plan(oracle_cpu, n, world, plan_n):
    """every rank's every window against its closed form, and the rank sum against the oracle"""
    from snarkvm_b200 import device, sharded
    shards = [sharded.shard_range(n, r, world) for r in range(world)]
    sizes = [hi - lo for lo, hi in shards]
    assert sum(sizes) == n
    if plan_n is None:
        plan_n = max(sizes)
    assert plan_n >= max(sizes)
    if n in (3, 9):
        assert sizes.count(0) >= 3
    if n == 17377:
        # the precondition of the case: the smallest shard alone would run another window size than the plan it runs under
        assert sizes == [5793, 5793, 5791]
        assert device.msm_plan(min(sizes))["c"] != device.msm_plan(plan_n)["c"]
    if plan_n == 1 << 20:
        assert (device.msm_plan(plan_n)["c"], device.msm_plan(plan_n)["levels"]) == (15, 3)
    if plan_n == 1 << 22:
        assert (device.msm_plan(plan_n)["c"], device.msm_plan(plan_n)["levels"]) == (16, 4)
    seed = 0x5100 + n % 9973 + world
    bases = device.generate_bases(n, seed)
    ks = _ks(seed, n)
    scal = random_canonical_fr(n, seed=n + world)
    want = _oracle_total(oracle_cpu, bases.cpu().numpy() if n <= 1 << 16 else None, ks, scal)
    tot, _ = run_ranks(oracle_cpu, bases, scal, ks, shards, plan_n, want)
    # the rank sum window by window: the windows of the whole input under the same plan
    assert_windows(tot, window_closed_forms(oracle_cpu, ks, scal, plan_n), "rank sum")


@gpu
def test_rank_sums_equal_opposite_and_infinite(oracle_cpu):
    """k_xyzz_sum_ranks on ranks whose sums are equal (every window doubles), opposite (every window cancels to ∞), all ∞, and
    an ∞ rank between two others"""
    import torch
    from snarkvm_b200 import device
    n = 4096
    seed = 0x5200
    bases = device.generate_bases(n, seed)
    ks = _ks(seed, n)
    scal = random_canonical_fr(n, seed=77)
    b = mc.Bases(bases.cpu().numpy(), ks.copy())
    b.negate(np.arange(n))
    neg = torch.from_numpy(b.rows).cuda()
    allinf = bases.clone()
    allinf[:, 96] = 1
    nwin = device.msm_plan(n)["nwin"]
    c = device.msm_plan(n)["c"]
    dscal = _dev(scal)
    s_pos = device.msm_window_sums(bases, dscal, plan_npoints=n)
    s_neg = device.msm_window_sums(neg, dscal, plan_npoints=n)
    s_inf = device.msm_window_sums(allinf, dscal, plan_npoints=n)
    assert_windows(s_pos, window_closed_forms(oracle_cpu, ks, scal, n), "P")
    assert_windows(s_neg, window_closed_forms(oracle_cpu, b.ks, scal, n), "-P")
    assert_windows(s_inf, [INF] * nwin, "all ∞")
    single = total_closed_form(oracle_cpu, ks, scal)

    def ranks(*parts):
        return device.xyzz_sum_ranks(torch.stack(parts).contiguous(), len(parts), nwin)

    both = np.concatenate([ks, ks]), np.concatenate([scal, scal])
    doubled = ranks(s_pos, s_pos)
    assert_windows(doubled, window_closed_forms(oracle_cpu, both[0], both[1], n), "equal ranks")
    assert (device.msm_finish(doubled.cpu().numpy(), c) == total_closed_form(oracle_cpu, *both)).all()
    assert_windows(ranks(s_pos, s_neg), [INF] * nwin, "opposite ranks")
    assert_windows(ranks(s_neg, s_pos, s_pos), window_closed_forms(oracle_cpu, ks, scal, n), "−P + P + P")
    assert_windows(ranks(s_inf, s_inf, s_inf), [INF] * nwin, "all ranks ∞")
    mid = ranks(s_pos, s_inf, s_pos)
    assert_windows(mid, window_closed_forms(oracle_cpu, both[0], both[1], n), "∞ rank between two")
    assert (device.msm_finish(ranks(s_inf, s_pos).cpu().numpy(), c) == single).all()


# ---------------------------------------------------------------------------------------------------------------------------
# the host-buffer path
# ---------------------------------------------------------------------------------------------------------------------------
def _host_case(cpu, n: int, seed: int, plan_n: int, closed: bool = True):
    """generated bases on the device and the host, scalars, the device-tensor path's windows and the closed forms"""
    from snarkvm_b200 import device
    bases = device.generate_bases(max(n, 1), seed)[:n]
    ks = _ks(seed, n)
    scal = random_canonical_fr(n, seed=seed + 1)
    ref = device.msm_window_sums(bases, _dev(scal), plan_npoints=plan_n)
    want = window_closed_forms(cpu, ks, scal, plan_n) if closed else None
    return bases.cpu().numpy(), scal, ks, ref, want


def _host_call(plan_n: int, pts: np.ndarray, sc: np.ndarray, flags=None):
    from snarkvm_b200 import device
    out = _poisoned_out(device.msm_plan(plan_n)["nwin"])
    device.msm_window_sums_host(out, flags, plan_n, pts, sc)
    return out


@gpu
@pytest.mark.parametrize("n, chunks, plan_n", [
    (50000, None, None),            # one range, pageable points staged through the pinned ring
    (50000, "2", None),             # two equal ranges: the d_parts fold
    (50000, "1:3:4", None),         # three unequal ranges, the first below the staging threshold
    (20, "16", None),               # one-point ranges (sixteen of them for twenty points)
    (3000, None, 1 << 16),          # a plan for more points than the shard holds
    (3000, "3", 1 << 16),
    (0, None, 1000),                # an empty shard: all-∞ sums
])
def test_host_path_matches_device_path(oracle_cpu, monkeypatch, n, chunks, plan_n):
    """msm_window_sums_host from pinned and from pageable numpy buffers: every window equals the device-tensor path's window
    and its closed form.  Pageable buffers are overwritten as soon as the call returns (the upload has staged them by then)."""
    import torch
    if chunks is None:
        monkeypatch.delenv("SNARKVM_B200_MSM_CHUNKS", raising=False)
    else:
        monkeypatch.setenv("SNARKVM_B200_MSM_CHUNKS", chunks)
    plan_n = plan_n or n
    seed = 0x5300 + n + len(chunks or "")
    pts, scal, ks, ref, want = _host_case(oracle_cpu, n, seed, plan_n)
    assert_windows(ref, want, "device path")
    # pinned first: its device buffers come fresh from the pool, so a kernel that ran ahead of its upload would read other data
    p_pts, p_t = _pinned(pts)
    p_sc, s_t = _pinned(scal)
    got_pinned = _host_call(plan_n, p_pts, p_sc)
    torch.cuda.synchronize()
    assert_windows(got_pinned, want, "pinned")
    assert_same_windows(got_pinned, ref, "pinned vs device path")
    pg_pts, pg_sc = pts.copy(), scal.copy()
    got_pageable = _host_call(plan_n, pg_pts, pg_sc)
    pg_pts[:] = 0x3C
    pg_sc[:] = np.uint64(0x0123456789ABCDEF)
    torch.cuda.synchronize()
    assert_windows(got_pageable, want, "pageable")
    assert_same_windows(got_pageable, ref, "pageable vs device path")
    del p_t, s_t


@gpu
def test_host_path_default_ranges_at_2_23(oracle_cpu, monkeypatch):
    """2^23 points: the default four ranges (1/16, 1/8, 1/4, the rest), pinned and pageable; each window against the
    device-tensor path and the fold against the closed form"""
    import torch
    from snarkvm_b200 import device
    monkeypatch.delenv("SNARKVM_B200_MSM_CHUNKS", raising=False)
    n = 1 << 23
    seed = 0x5323
    pts, scal, ks, ref, _ = _host_case(oracle_cpu, n, seed, n, closed=False)
    c = device.msm_plan(n)["c"]
    assert c in MODEL_C
    want = total_closed_form(oracle_cpu, ks, scal)
    assert (device.msm_finish(ref.cpu().numpy(), c) == want).all()
    p_pts, p_t = _pinned(pts)
    p_sc, s_t = _pinned(scal)
    got = _host_call(n, p_pts, p_sc)
    torch.cuda.synchronize()
    assert_same_windows(got, ref, "pinned vs device path")
    assert (device.msm_finish(got.cpu().numpy(), c) == want).all()
    del p_t, s_t
    got = _host_call(n, pts, scal)
    torch.cuda.synchronize()
    assert_same_windows(got, ref, "pageable vs device path")
    assert (device.msm_finish(got.cpu().numpy(), c) == want).all()


def _calls_in_flight(cpu) -> list:
    """Three msm_sharded_async calls on numpy inputs (world 1), all issued while the stream is still busy with earlier work, so
    none of their kernels has run when the next call starts its upload.  A call's device buffers go back to the library's pool
    once it has been enqueued, and the next call of the same size is handed them again: its upload may begin only once the
    stream has passed the call before, or that call reads the next one's inputs.  The pageable inputs are overwritten as soon
    as their call returns.  → the calls whose result differs from its closed form"""
    import torch
    from snarkvm_b200 import device, sharded
    n = 1 << 18
    inputs, jobs, keep = [], [], []
    for k, pinned in enumerate((True, True, False)):
        seed = 0x5400 + k
        pts = device.generate_bases(n, seed).cpu().numpy()
        scal = random_canonical_fr(n, seed=seed)
        jobs.append(total_closed_form(cpu, _ks(seed, n), scal))
        if pinned:
            (pts, t1), (scal, t2) = _pinned(pts), _pinned(scal)
            keep += [t1, t2]
        inputs.append((pts, scal, pinned))
    # one call of the same size first, waited for: the pool then holds free blocks of exactly the sizes the calls ask for
    warm = sharded.msm_sharded_async(inputs[2][0].copy(), inputs[2][1].copy(), plan_npoints=n).result()
    assert (warm == jobs[2]).all()
    torch.cuda.synchronize()
    # a spin kernel on the library's stream (the current one) keeps it busy for a few hundred ms while the calls are issued;
    # it allocates nothing, so no buffer of the calls can be one it still uses
    torch.cuda._sleep(1 << 29)
    pend = []
    for pts, scal, pinned in inputs:
        pend.append(sharded.msm_sharded_async(pts, scal, plan_npoints=n))
        if not pinned:
            pts[:] = 0x3C
            scal[:] = np.uint64(7)
    return [k for k, (p, want) in enumerate(zip(pend, jobs)) if not (p.result() == want).all()]


@gpu
def test_sharded_async_calls_in_flight():
    """_calls_in_flight in a fresh process, whose library pool holds only the blocks of this test's own calls"""
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here]))
    r = subprocess.run([sys.executable, "-s", os.path.abspath(__file__), "calls-in-flight"], env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert r.stdout.strip().splitlines()[-1] == "wrong calls: []", r.stdout[-2000:]


# ---------------------------------------------------------------------------------------------------------------------------
# overflow flags
# ---------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("host", [False, True])
def test_overflow_flag_of_one_rank(oracle_cpu, monkeypatch, host):
    """bit 253 set in one scalar of rank 1 (in the first of its four ranges on the host path, so a flag cleared between ranges
    would lose it): only rank 1's flag is set, its PendingMsm raises CudaError, and a clean call with the same flags tensor
    clears the flag"""
    import torch
    from snarkvm_b200 import device, sharded
    from snarkvm_b200._lib import CudaError
    monkeypatch.setenv("SNARKVM_B200_MSM_CHUNKS", "4")
    n, world = 3000, 3
    seed = 0x5500 + host
    bases = device.generate_bases(n, seed)
    ks = _ks(seed, n)
    clean = random_canonical_fr(n, seed=seed)
    scal = clean.copy()
    shards = [sharded.shard_range(n, r, world) for r in range(world)]
    plan_n = max(hi - lo for lo, hi in shards)
    bad = shards[1][0] + 5
    scal[bad, 3] |= np.uint64(1 << (253 - 192))
    host_pts = bases.cpu().numpy()
    dscal = _dev(scal)
    flags = [torch.full((1,), 0x70, dtype=torch.int32, device="cuda") for _ in range(world)]

    def call(r, sc, fl):
        lo, hi = shards[r]
        if host:
            return _host_call(plan_n, host_pts[lo:hi], np.ascontiguousarray(sc[lo:hi]), fl)
        return device.msm_window_sums(bases[lo:hi], _dev(sc[lo:hi]), plan_npoints=plan_n, flags=fl)

    for r in range(world):
        call(r, scal, flags[r])
    assert [int(f.item()) for f in flags] == [0, 1, 0]
    for r, (lo, hi) in enumerate(shards):
        inputs = (host_pts[lo:hi], np.ascontiguousarray(scal[lo:hi])) if host else (bases[lo:hi], dscal[lo:hi])
        p = sharded.msm_sharded_async(*inputs, plan_npoints=plan_n)
        if r == 1:
            with pytest.raises(CudaError):
                p.result()
        else:
            assert (p.result() == total_closed_form(oracle_cpu, ks[lo:hi], clean[lo:hi])).all()
    s = call(1, clean, flags[1])
    torch.cuda.synchronize()
    assert int(flags[1].item()) == 0
    lo, hi = shards[1]
    assert_windows(s, window_closed_forms(oracle_cpu, ks[lo:hi], clean[lo:hi], plan_n), "clean rank 1")


# ---------------------------------------------------------------------------------------------------------------------------
# strides and padding
# ---------------------------------------------------------------------------------------------------------------------------
def _restride(rows, stride: int, seed: int, keep: int = 97):
    """the `keep` meaningful bytes of every row (coordinates and infinity flag: 97 for G1, 193 for G2) in rows of `stride`
    bytes, random bytes after them"""
    import torch
    g = torch.Generator(device="cpu").manual_seed(seed)
    out = torch.randint(0, 256, (rows.shape[0], stride), dtype=torch.uint8, generator=g).to(rows.device)
    out[:, :keep] = rows[:, :keep]
    return out


@gpu
@pytest.mark.parametrize("stride", [104, 112, 128, 200])
def test_g1_strides_with_garbage_padding(oracle_cpu, monkeypatch, stride):
    """every G1 entry point that takes a stride gives, on rows of `stride` bytes with random bytes after the infinity flag,
    exactly what it gives on the clean 104-byte rows; the two host-buffer calls also in three ranges, whose offsets are
    multiples of the stride"""
    import torch
    from snarkvm_b200 import _lib, cuda, device
    n = 2048
    seed = 0x5600
    clean = device.generate_bases(n, seed)
    clean[100:110, 96] = 1                                             # ∞ rows: the flag byte alone decides
    scal = random_canonical_fr(n, seed=3)
    scal2 = random_canonical_fr(n - 300, seed=4)
    dscal, dscal2 = _dev(scal), _dev(scal2)
    ks = _ks(seed, n)
    ks[100:110] = 0
    want = total_closed_form(oracle_cpu, ks, scal)
    assert (device.msm(clean, dscal) == want).all()
    assert (oracle_cpu.msm(clean.cpu().numpy(), scal, 0) == want).all()
    pad = _restride(clean, stride, seed=stride)
    assert (pad[:, 97:].cpu().numpy() != 0).any(axis=1).all()          # every row has garbage in its padding
    host_pad = pad.cpu().numpy()

    assert (device.msm(pad, dscal, stride) == want).all()
    plan_n = 5000
    ref = device.msm_window_sums(clean, dscal, plan_npoints=plan_n)
    assert_same_windows(device.msm_window_sums(pad, dscal, stride, plan_npoints=plan_n), ref, "window sums")
    for chunks in ("1", "3"):
        monkeypatch.setenv("SNARKVM_B200_MSM_CHUNKS", chunks)
        assert (cuda.msm(host_pad, scal) == want).all(), chunks
        got = _poisoned_out(device.msm_plan(plan_n)["nwin"])
        device.msm_window_sums_host(got, None, plan_n, host_pad, scal, stride)
        torch.cuda.synchronize()
        assert_same_windows(got, ref, ("host window sums", chunks))
    monkeypatch.delenv("SNARKVM_B200_MSM_CHUNKS")
    assert (device.msm_batch(pad, [dscal, dscal2], stride) == device.msm_batch(clean, [dscal, dscal2])).all()
    pre = device.PrecomputedBases(pad, stride)
    try:
        assert (pre.msm(dscal) == want).all()
    finally:
        pre.free()
    # two overlapping slices of one base array, merged in whole strides
    polys = [_dev(random_canonical_fr(1500, seed=5)), _dev(random_canonical_fr(1800, seed=6))]
    a = device.sonic_commit_batch([clean[0:1500], clean[200:2000]], polys)
    b = device.sonic_commit_batch([pad[0:1500], pad[200:2000]], polys, stride=stride)
    assert (a == b).all()
    assert (a[0] == device.kzg_commit(clean[:1500], polys[0])).all()
    # the G1 FFT; every output row's first 104 bytes (coordinates, flag word) are written, the rest of a wider row is not
    lg = 10
    fin = clean[:1 << lg].clone()
    fin[100:110] = clean[0]
    fin[100:110, 96] = 0
    fpad = _restride(fin, stride, seed=stride + 1)
    for inverse in (False, True):
        ref_ntt = device.g1_ntt(fin, inverse)
        got_ntt = device.g1_ntt(fpad, inverse, stride)
        assert torch.equal(got_ntt[:, :104], ref_ntt), (stride, inverse)
        # in-stride ≠ out-stride, through the C entry point
        for out_stride in sorted({104, 128, 200} - {stride}):
            out = torch.zeros((1 << lg, out_stride), dtype=torch.uint8, device="cuda")
            _lib.check(_lib.lib().snarkvm_b200_g1_ntt_device(out.data_ptr(), out_stride, fpad.data_ptr(), stride, lg, int(inverse),
                                                              torch.cuda.current_stream().cuda_stream))
            assert torch.equal(out[:, :104], ref_ntt), (stride, out_stride, inverse)
            assert not out[:, 104:].any()


@gpu
def test_g2_stride_with_garbage_padding():
    """msm_g2 on rows of 208 bytes, and of 200 bytes, with random bytes after the infinity flag == on the clean rows"""
    from snarkvm_b200 import device
    n = 1000
    clean = device.generate_bases_g2(n, seed=0x5700)
    clean[50:60, 192] = 1
    scal = _dev(random_canonical_fr(n, seed=8))
    want = device.msm_g2(clean, scal)
    for stride in (200, 208):
        pad = _restride(clean, stride, seed=stride, keep=193)
        assert (pad[:, 193:].cpu().numpy() != 0).any(axis=1).all()
        assert (device.msm_g2(pad, scal, stride) == want).all(), stride



def test_host_window_sums_reject_bad_layouts():
    """msm_window_sums_host passes raw host pointers to the library, so it refuses arrays whose memory is not laid out as
    [n, stride] uint8 points and [n, 4] uint64 scalars before anything is enqueued"""
    import torch
    from snarkvm_b200 import device
    out = torch.zeros((24, 24), dtype=torch.int64)
    pts = np.zeros((8, 112), dtype=np.uint8)
    sc = np.zeros((8, 4), dtype=np.uint64)
    bad_points = [
        (TypeError, pts[:, :104], 104),                                # rows not contiguous
        (TypeError, pts.view(np.uint64), 112),                         # not bytes
        (TypeError, pts.reshape(-1), 112),                             # flat
        (TypeError, np.asfortranarray(pts), 112),
        (TypeError, list(pts), 112),
        (ValueError, pts, 104),                                        # row size is not the stride
    ]
    for err, p, stride in bad_points:
        with pytest.raises(err, match="points"):
            device.msm_window_sums_host(out, None, 1000, p, sc, stride)
    wide = np.zeros((8, 8), dtype=np.uint64)
    bad_scalars = [
        wide[:, :4],                                                   # rows not contiguous
        sc[::2],                                                       # every other row
        sc.view(np.int64),
        sc.view(np.uint8),
        sc.reshape(-1),
        np.asfortranarray(sc),
        np.zeros((8, 5), dtype=np.uint64),
    ]
    for s in bad_scalars:
        with pytest.raises(TypeError, match="scalars"):
            device.msm_window_sums_host(out, None, 1000, pts, s, 112)
    with pytest.raises(ValueError, match="points"):
        device.msm_window_sums_host(out, None, 1000, pts[:4], sc, 112)


if __name__ == "__main__" and sys.argv[1:] == ["calls-in-flight"]:
    from oracle import cpu as _cpu
    _cpu.build()
    print("wrong calls:", _calls_in_flight(_cpu))
