"""The G1 MSM's dispatch matrix (csrc/msm.cu, the MsmPath that msm_path() picks for msm_core): every case pins one choice of
accumulation (MsmPath::acc, with its item_cap), hot-bucket folds (MsmPath::fold) and reduction tail (MsmPath::tail), asserts
from a torch.profiler trace of one call which kernels ran (and which did not), then runs the input
families of msm_corpus.py through it and compares every result with the closed form Σ s_i·k_i·G (+ the torsion rows' part
in big integers), and with the oracle's MSM where the input has no torsion rows and is small.

The kernel assertion is what keeps a case on its path: if a later plan change moves it elsewhere, the case fails instead of
silently testing something else.  Templates are matched exactly (k_bucket_reduce<true> is neither k_bucket_reduce<false>
nor k_bucket_reduce_quad); a name without template arguments matches that kernel only."""
from collections import Counter

import numpy as np
import pytest

from oracle import bls12_377 as py

import msm_corpus as mc
from helpers import random_canonical_fr

pytestmark = pytest.mark.gpu

ENV = ("SNARKVM_B200_MSM_C", "SNARKVM_B200_MSM_LEVELS", "SNARKVM_B200_MSM_SCRATCH_MB", "SNARKVM_B200_MSM_PRE_C",
       "SNARKVM_B200_MSM_PRE_LEVELS")


def _dev(x):
    import torch
    if x.dtype == np.uint64:
        x = x.view(np.int64)
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _norm(name: str) -> str:
    name = name.split("(")[0].strip()
    if name.startswith("void "):
        name = name[5:]
    return name.replace("b200::", "")


def traced(fn):
    """(fn(), Counter of the CUDA kernels it launched, by demangled name without namespace / parameter list).
    The profiler now and then hands back a trace that lacks the first kernels of the call, or all of them.  Every MSM opens
    with the digit histogram (k_digits<false, ·>), so a trace without it is incomplete; fn is deterministic and is traced again."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    for _ in range(4):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            torch.zeros(1, device="cuda").add_(1)                # a kernel before the traced call
            torch.cuda.synchronize()
            out = fn()
            torch.cuda.synchronize()
        kern = Counter(_norm(e.name) for e in prof.events() if e.device_type == DeviceType.CUDA)
        if any(k.startswith("k_digits<false") for k in kern):
            break
    return out, kern


def launches(kern: Counter, spec: str) -> int:
    if "<" in spec:
        return kern.get(spec, 0)
    return sum(v for k, v in kern.items() if k.split("<")[0] == spec)


def check_kernels(kern: Counter, must=(), must_not=(), counts=None):
    names = sorted(k for k in kern if k.startswith("k_"))
    for spec in must:
        assert launches(kern, spec) > 0, (spec, names)
    for spec in must_not:
        assert launches(kern, spec) == 0, (spec, names)
    for spec, want in (counts or {}).items():
        got = launches(kern, spec)
        assert (want(got) if callable(want) else got == want), (spec, got, names)


def set_env(monkeypatch, env: dict):
    for k in ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, str(v))


def adversarial_bases(n: int, seed: int, torsion: bool = True) -> mc.Bases:
    """generated bases with a run of one repeated point, alternating P / −P, ∞ rows and (optionally) torsion rows"""
    from snarkvm_b200 import device
    b = mc.Bases.generated(device.generate_bases(n, seed).cpu().numpy(), seed)
    run = np.arange(n // 8, n // 8 + max(8, n // 16))
    b.repeat(int(run[0]), run[1:])
    b.alternate(n // 4, np.arange(n // 4, n // 4 + min(64, n // 8)))
    b.infinity(np.arange(5, n, 37))
    if torsion:
        t = n // 2
        k = max(4, n // 64)
        b.torsion_points(np.arange(t, t + k), "t2")
        b.torsion_points(np.arange(t + k, t + 2 * k), "t3")
        b.torsion_points(np.arange(t + 2 * k, t + 3 * k), "t3neg")
    return b


def adversarial_scalars(kind: str, n: int, seed: int) -> np.ndarray:
    """a scalar family, with equal scalars on the repeated run and on the P / −P rows, and on every torsion block"""
    s = mc.scalar_family(kind, n, seed)
    run = np.arange(n // 8, n // 8 + max(8, n // 16))
    s[run] = s[run[0]]
    s[n // 4:n // 4 + min(64, n // 8)] = s[n // 4]
    t, k = n // 2, max(4, n // 64)
    for j in range(3):
        s[t + j * k:t + (j + 1) * k] = s[t + j * k]
    return s


def run_case(cpu, b: mc.Bases, families, seed, must=(), must_not=(), counts=None, oracle_limit=4096):
    """every family through device.msm on b; the first call is traced and its kernels checked"""
    from snarkvm_b200 import device
    n = b.rows.shape[0]
    bases = _dev(b.rows)
    for f, kind in enumerate(families):
        scal = adversarial_scalars(kind, n, seed + f)
        if f == 0:
            got, kern = traced(lambda: device.msm(bases, _dev(scal)))
            check_kernels(kern, must, must_not, counts)
        else:
            got = device.msm(bases, _dev(scal))
        assert (got == mc.closed_form(cpu, b, scal)).all(), kind
        if n <= oracle_limit and not b.torsion:
            assert (got == cpu.msm(b.rows, scal, 1)).all(), kind


QUAD_TAIL = ("k_bucket_reduce_quad", "k_window_combine_quad")
CLASSIC_TAIL = ("k_bucket_reduce<false>", "k_group_sum")
LARGE_TAIL = ("k_bucket_reduce<true>", "k_window_combine_quad")


def test_path_q8(oracle_cpu, monkeypatch):
    """200 points: one warp per work item, quad reduction, no folds"""
    set_env(monkeypatch, {})
    b = adversarial_bases(200, seed=11)
    run_case(oracle_cpu, b, mc.SCALAR_FAMILIES, 100, must=("k_bucket_accumulate_q8",) + QUAD_TAIL,
             must_not=("k_fold_hot_quad", "k_bucket_accumulate", "k_bucket_accumulate_g8", "k_partial_group_sum", "k_bucket_reduce<true>",
                       "k_bucket_reduce<false>", "k_scatter_records<false, false>"))


def test_path_g8(oracle_cpu, monkeypatch):
    """3000 points (c = 8, 96k entries): eight lanes per item, 32 points per item; all-equal scalars put 3000 entries = 94
    items into one bucket per window, so the one scheduled k_fold_hot_quad round has work"""
    from snarkvm_b200 import device
    set_env(monkeypatch, {})
    assert device.msm_plan(3000)["c"] == 8
    b = adversarial_bases(3000, seed=12)
    run_case(oracle_cpu, b, ("equal",) + mc.SCALAR_FAMILIES, 200, must=("k_bucket_accumulate_g8",) + QUAD_TAIL,
             must_not=("k_bucket_accumulate_q8", "k_bucket_accumulate", "k_partial_group_sum"), counts={"k_fold_hot_quad": 1})


def test_path_short_items(oracle_cpu, monkeypatch):
    """2^14 points (c = 11): one thread per item of 8 points, two scheduled 32:1 fold rounds, 128 quad chunks per window
    combined by one k_combine_level_quad level"""
    set_env(monkeypatch, {})
    b = adversarial_bases(1 << 14, seed=13)
    run_case(oracle_cpu, b, ("equal",) + mc.SCALAR_FAMILIES, 300,
             must=("k_bucket_accumulate", "k_combine_level_quad") + QUAD_TAIL,
             must_not=("k_bucket_accumulate_q8", "k_bucket_accumulate_g8", "k_partial_group_sum", "k_combine_level_quadseq"),
             counts={"k_fold_hot_quad": 2})


def test_path_c11(oracle_cpu, monkeypatch):
    """2^16 points (c = 11, carry-only top window with ≈ n/2 points in one bucket): items of 16, k_combine_level_quad (m = 128)"""
    from snarkvm_b200 import device
    set_env(monkeypatch, {})
    assert device.msm_plan(1 << 16)["c"] == 11
    b = adversarial_bases(1 << 16, seed=14)
    run_case(oracle_cpu, b, mc.SCALAR_FAMILIES, 400, must=("k_bucket_accumulate", "k_combine_level_quad", "k_fold_hot_quad") + QUAD_TAIL,
             must_not=("k_partial_group_sum", "k_bucket_reduce<true>", "k_bucket_reduce<false>"))


@pytest.mark.parametrize("c", [12, 13, 14])
def test_path_classic_tail(oracle_cpu, monkeypatch, c):
    """plain c = 12–14 (2048–8192 buckets per window, no pair levels): scan-driven 32:1 folds (three scheduled rounds at
    20000 points), the per-chunk reduction k_bucket_reduce<false> and the k_group_sum tree; none of the quad kernels"""
    set_env(monkeypatch, {"SNARKVM_B200_MSM_C": c, "SNARKVM_B200_MSM_LEVELS": 0})
    b = adversarial_bases(20000, seed=15 + c)
    run_case(oracle_cpu, b, mc.SCALAR_FAMILIES, 500 + c, must=("k_bucket_accumulate", "k_group_counts") + CLASSIC_TAIL,
             must_not=("k_fold_hot_quad", "k_bucket_reduce_quad", "k_bucket_reduce<true>", "k_combine_level_quad",
                       "k_combine_level_quadseq", "k_window_combine_quad", "k_pair_level2<false, 4>"),
             counts={"k_partial_group_sum": 3, "k_group_sum": 3 if c < 14 else lambda k: k >= 3})


@pytest.mark.parametrize("n", [20000, 1 << 16])
@pytest.mark.parametrize("c", [15, 16, 17, 20])
def test_path_large_tail(oracle_cpu, monkeypatch, n, c):
    """plain c ≥ 15 without pair levels: hot buckets folded to ONE partial by k_fold_hot_quad (keep = 1; three rounds are
    scheduled; equal scalars fold a bucket in 3 rounds, half-equal in 2, few-hot in 1, so k_bucket_reduce<true> reads the
    partial from both buffers of the round parity), then k_combine_level_quadseq / k_combine_level_quad levels"""
    set_env(monkeypatch, {"SNARKVM_B200_MSM_C": c, "SNARKVM_B200_MSM_LEVELS": 0})
    b = adversarial_bases(n, seed=20 + c)
    run_case(oracle_cpu, b, ("equal", "half_equal", "few_hot", "special", "uniform"), 600 + c,
             must=("k_bucket_accumulate", "k_combine_level_quadseq") + LARGE_TAIL,
             must_not=("k_partial_group_sum", "k_bucket_reduce<false>", "k_group_sum", "k_bucket_reduce_quad"),
             counts={"k_fold_hot_quad": 3})


def test_path_large_tail_small_groups(oracle_cpu, monkeypatch):
    """c = 15 with pair levels and an 8 MB scratch budget: about two windows per group, so the tail's combine levels have too few
    groups for the sequential kernel and run k_combine_level_quad only"""
    set_env(monkeypatch, {"SNARKVM_B200_MSM_C": 15, "SNARKVM_B200_MSM_LEVELS": 2, "SNARKVM_B200_MSM_SCRATCH_MB": 8})
    b = adversarial_bases(20000, seed=30)
    run_case(oracle_cpu, b, mc.SCALAR_FAMILIES, 700,
             must=("k_scatter_records<false, false>", "k_pair_level2<false, 4>", "k_bucket_accumulate_dense", "k_combine_level_quad")
             + LARGE_TAIL, must_not=("k_combine_level_quadseq", "k_bucket_accumulate"),
             counts={"k_window_combine_quad": lambda k: k >= 4})


def test_path_pair_levels_many_outputs_per_lane(oracle_cpu, monkeypatch):
    """2^16 points, c = 6, 3 pair levels: level 0 has ≈ 1.4 M outputs, about 21 per lane on 132 SMs, so the cp.async ring and
    the forward / backward walks see degenerate pairs in the middle of a lane's run: equal points, P + (−P), ∞ inputs, the
    order-2 point doubled (denominator 2y = 0: must give ∞, not a zero in the CTA's shared inversion) and points with x = 0.
    Whole inputs of degenerate pairs too: all ∞, all P / −P, all the order-2 point."""
    from snarkvm_b200 import device
    set_env(monkeypatch, {"SNARKVM_B200_MSM_C": 6, "SNARKVM_B200_MSM_LEVELS": 3})
    n = 1 << 16
    b = adversarial_bases(n, seed=31)
    t = np.arange(1000, n, 97)                                  # more torsion rows spread over the array
    b.torsion_points(t[0::3], "t2").torsion_points(t[1::3], "t3").torsion_points(t[2::3], "t3neg")
    must = ("k_scatter_records<false, false>", "k_pair_desc<false>", "k_pair_level2<false, 4>", "k_bucket_accumulate_dense")
    run_case(oracle_cpu, b, mc.SCALAR_FAMILIES, 800, must=must + QUAD_TAIL, must_not=("k_bucket_accumulate",),
             counts={"k_pair_level2<false, 4>": 3})
    inf = np.frombuffer(py.projective_bytes_normalised(None), dtype=np.uint64)
    scal = random_canonical_fr(n, seed=801)
    same = np.tile(scal[:1], (n, 1))
    allinf = b.copy().infinity(np.arange(n))
    assert (device.msm(_dev(allinf.rows), _dev(scal)) == inf).all()
    cancel = b.copy().alternate(3, np.arange(n))                 # P, −P, … with equal scalars
    assert (device.msm(_dev(cancel.rows), _dev(same)) == inf).all()
    pairs = b.copy()                                             # P_i, −P_i with equal scalars (different points, torsion rows too)
    pairs.rows[1::2] = pairs.rows[0::2]
    pairs.negate(np.arange(1, n, 2))
    ps = scal.copy(); ps[1::2] = ps[0::2]
    assert (device.msm(_dev(pairs.rows), _dev(ps)) == inf).all()
    t2 = b.copy().torsion_points(np.arange(n), "t2")
    for s in (scal, same):
        assert (device.msm(_dev(t2.rows), _dev(s)) == mc.closed_form(oracle_cpu, t2, s)).all()
    t3 = b.copy().torsion_points(np.arange(0, n, 2), "t3").torsion_points(np.arange(1, n, 2), "t3neg")
    assert (device.msm(_dev(t3.rows), _dev(scal)) == mc.closed_form(oracle_cpu, t3, scal)).all()


def test_default_plans():
    from snarkvm_b200 import device
    for lg, want in ((19, (13, 2)), (21, (16, 4)), (23, (17, 5)), (20, (15, 3)), (22, (16, 4)), (24, (17, 5))):
        p = device.msm_plan(1 << lg)
        assert (p["c"], p["levels"]) == want, lg


@pytest.mark.parametrize("levels", [0, 2])
@pytest.mark.parametrize("c", [2, 3, 5, 7, 11, 13, 16, 17, 20, 23])
def test_digit_sweep(oracle_cpu, monkeypatch, c, levels):
    """the digit-boundary corpus for this c (every window at raw = half, half + 1 and 2^c, carry chains, top windows at their
    maximum), as canonical scalars and as Montgomery coefficients (KZG commit: to_bigint on the device), with and without
    pair levels (the histogram of k_digits and the cursors of k_scatter_records must agree)"""
    from snarkvm_b200 import device
    set_env(monkeypatch, {"SNARKVM_B200_MSM_C": c, "SNARKVM_B200_MSM_LEVELS": levels})
    n = 2000
    vals = mc.digit_boundary_scalars(c, seed=levels)
    scal = random_canonical_fr(n, seed=900 + c)
    scal[:len(vals)] = mc.to_limbs(vals)
    b = adversarial_bases(n, seed=40 + c, torsion=False)
    bases = _dev(b.rows)
    want = mc.closed_form(oracle_cpu, b, scal)
    got, kern = traced(lambda: device.msm(bases, _dev(scal)))
    check_kernels(kern, must=("k_scatter_records<false, false>",) if levels else ("k_digits<true, false>",),
                  must_not=() if levels else ("k_scatter_records<false, false>",))
    assert (got == want).all()
    mont = np.zeros_like(scal)
    mont[:] = mc.mont_limbs([py.from_limbs(r) for r in scal])
    assert (device.kzg_commit(bases, _dev(mont)) == want).all()
    if c in (5, 11):
        assert (got == oracle_cpu.msm(b.rows, scal, 1)).all()


@pytest.mark.parametrize("pre_c", [13, 14, 16])
def test_path_flat_tables(oracle_cpu, monkeypatch, pre_c):
    """precomputed tables (one bucket set for all windows), window size chosen when the tables are built: all-equal scalars put
    2^16 entries per window digit into one bucket, 2048 items after one pair level, so three fold rounds; c = 13/14 end in the
    k_group_sum tree, c = 16 in k_bucket_reduce<true> after folds to one partial"""
    from snarkvm_b200 import device
    set_env(monkeypatch, {"SNARKVM_B200_MSM_PRE_C": pre_c, "SNARKVM_B200_MSM_PRE_LEVELS": 1})
    n = 1 << 16
    b = adversarial_bases(n, seed=50 + pre_c, torsion=False)
    pre = device.PrecomputedBases(_dev(b.rows))
    try:
        assert pre.c == pre_c
        for f, kind in enumerate(("equal", "half_equal", "special")):
            scal = adversarial_scalars(kind, n, 1000 + f)
            if f == 0:
                got, kern = traced(lambda: pre.msm(_dev(scal)))
                tail = CLASSIC_TAIL if pre_c < 15 else LARGE_TAIL
                folds = {"k_partial_group_sum" if pre_c < 15 else "k_fold_hot_quad": lambda k: k >= 3}
                check_kernels(kern, must=("k_scatter_records<false, true>", "k_pair_level2<false, 4>") + tail, counts=folds,
                              must_not=("k_bucket_reduce<true>",) if pre_c < 15 else ("k_group_sum", "k_bucket_reduce<false>"))
            else:
                got = pre.msm(_dev(scal))
            assert (got == mc.closed_form(oracle_cpu, b, scal)).all(), kind
        mont = mc.mont_limbs([py.from_limbs(r) for r in scal[:4096]])
        assert (pre.kzg_commit(_dev(mont)) == mc.closed_form(oracle_cpu, b, scal[:4096])).all()
    finally:
        pre.free()


@pytest.mark.parametrize("n,c,kinds", [(2000, 12, ("uniform", "equal")), (2000, 15, ("uniform", "equal")),
                                       (1 << 15, None, ("equal", "half_equal"))])
def test_path_g2(monkeypatch, n, c, kinds):
    """G2: the bucket reduction and k_g2_group_sum tree at c = 12 and 15; at 2^15 points the scheduled 32:1 folds
    (k_g2_partial_group_sum, three rounds) have work with equal and half-equal scalars.  Checked by the closed form
    (Σ s_i·h_i mod r)·G2 over generated bases."""
    from oracle import g2
    from snarkvm_b200 import device
    from helpers import generated_base_multipliers
    set_env(monkeypatch, {"SNARKVM_B200_MSM_C": c} if c else {})
    seed = 60 + n
    bases = device.generate_bases_g2(n, seed)
    ks = generated_base_multipliers(seed, n)
    for f, kind in enumerate(kinds):
        scal = mc.scalar_family(kind, n, 1100 + f)
        if f == 0:
            got, kern = traced(lambda: device.msm_g2(bases, _dev(scal)))
            check_kernels(kern, must=("k_g2_accumulate", "k_g2_bucket_reduce", "k_g2_group_sum"),
                          counts={"k_g2_partial_group_sum": lambda k: k >= 2})
        else:
            got = device.msm_g2(bases, _dev(scal))
        dot = sum(int(k) * py.from_limbs(s) for k, s in zip(ks, scal)) % py.R_MOD
        assert (got == np.frombuffer(g2.g2_projective_bytes_normalised(g2.g2_mul(g2.G2_GEN, dot)), dtype=np.uint64)).all(), kind
