"""Mixed window layouts (SNARKVM_B200_MSM_WINDOWS: nwin − 1 windows of c bits and a wider top window whose digits fill several
bucket sets) forced onto small inputs, through every reduction tail that applies a set's digit offset: the quad tail of large
bucket sets (with and without pair levels, in one and in three window groups), the classic per-chunk tail and the quad tail of
small sets.  Each case checks its kernels from a trace and every result against the closed form (and the oracle where small)."""
import pytest

import msm_corpus as mc
from test_msm_paths_gpu import (CLASSIC_TAIL, LARGE_TAIL, QUAD_TAIL, _dev, adversarial_bases, adversarial_scalars, run_case,
                                set_env)

pytestmark = pytest.mark.gpu


def mixed(monkeypatch, layout: str, env: dict):
    set_env(monkeypatch, env)
    monkeypatch.setenv("SNARKVM_B200_MSM_WINDOWS", layout)


def test_mixed_large_tail_adversarial(oracle_cpu, monkeypatch):
    """the 2^24 layout (13 × 18 bits + a 20-bit top window in four sets of 2^17 buckets) on 20000 adversarial rows: hot
    buckets, ∞, P / −P runs, torsion rows; all 17 sets in one group"""
    mixed(monkeypatch, "18*13,20", {"SNARKVM_B200_MSM_LEVELS": 0})
    b = adversarial_bases(20000, seed=40)
    run_case(oracle_cpu, b, ("equal", "half_equal", "few_hot", "special", "uniform"), 900,
             must=("k_bucket_accumulate", "k_fold_hot_quad") + LARGE_TAIL,
             must_not=("k_bucket_reduce<false>", "k_group_sum", "k_bucket_reduce_quad"),
             counts={"k_window_combine_quad": 1})


def test_mixed_pair_levels_three_groups(oracle_cpu, monkeypatch):
    """the same layout with two pair levels and an 18 MB scratch budget: 5 + 5 + 4 windows per group, the last group holding the
    top window's four sets"""
    mixed(monkeypatch, "18*13,20", {"SNARKVM_B200_MSM_LEVELS": 2, "SNARKVM_B200_MSM_SCRATCH_MB": 18})
    b = adversarial_bases(20000, seed=41)
    run_case(oracle_cpu, b, mc.SCALAR_FAMILIES, 910,
             must=("k_scatter_records<false, false>", "k_pair_level2<false, 4>", "k_bucket_accumulate_dense") + LARGE_TAIL,
             must_not=("k_bucket_accumulate",), counts={"k_window_combine_quad": 3, "k_scatter_records<false, false>": 3})


def test_mixed_classic_tail(oracle_cpu, monkeypatch):
    """20 × 12 bits + a 14-bit top window (four sets of 2048 buckets) through k_bucket_reduce<false> and the k_group_sum tree"""
    mixed(monkeypatch, "12*20,14", {"SNARKVM_B200_MSM_LEVELS": 0})
    b = adversarial_bases(20000, seed=42)
    run_case(oracle_cpu, b, mc.SCALAR_FAMILIES, 920, must=("k_bucket_accumulate",) + CLASSIC_TAIL,
             must_not=("k_bucket_reduce_quad", "k_bucket_reduce<true>", "k_window_combine_quad"))


def test_mixed_small_quad_tail(oracle_cpu, monkeypatch):
    """31 × 8 bits + a 10-bit top window (four sets of 128 buckets) on 3000 points: the quad reduction of small sets"""
    mixed(monkeypatch, "8*31,10", {})
    b = adversarial_bases(3000, seed=43)
    run_case(oracle_cpu, b, ("equal",) + mc.SCALAR_FAMILIES, 930, must=QUAD_TAIL,
             must_not=("k_bucket_reduce<true>", "k_bucket_reduce<false>"))


def test_mixed_batch_matches_single_sums(oracle_cpu, monkeypatch):
    """three sums in one pass (the set offsets repeat per job) against the closed form of each"""
    from snarkvm_b200 import device
    mixed(monkeypatch, "18*13,20", {"SNARKVM_B200_MSM_LEVELS": 1})
    n = 20000
    b = adversarial_bases(n, seed=44, torsion=False)
    bases = _dev(b.rows)
    vecs = [adversarial_scalars(kind, n, 940 + k) for k, kind in enumerate(("uniform", "special", "equal"))]
    vecs[1] = vecs[1][: n // 2]
    got = device.msm_batch(bases, [_dev(v) for v in vecs])
    for k, v in enumerate(vecs):
        assert (got[k] == mc.closed_form(oracle_cpu, b, v)).all(), k


def test_invalid_layout_falls_back_to_uniform(oracle_cpu, monkeypatch):
    """a width list the plan cannot take (the top window too narrow to absorb the carry) leaves the uniform plan in force"""
    mixed(monkeypatch, "18*13,19", {"SNARKVM_B200_MSM_LEVELS": 0})
    b = adversarial_bases(4096, seed=45)
    run_case(oracle_cpu, b, ("uniform",), 950, must=QUAD_TAIL)
