"""Single inputs of the MSM pair levels.  A bucket with an odd count leaves one input without a partner at every level; it is
copied to the bucket's last output by k_pair_desc and takes no step of k_pair_level2, whose lanes walk real pairs only and
write each pair's output at the position its descriptor names.  These cases put odd counts everywhere (counts 1, 2 and 3 side
by side, every bucket odd through all levels), one hot bucket over a full background, degenerate pairs next to single ∞
outputs, the 2^24 window layout in one and several groups, ∞ bases in the level-0 records, the precomputed tables and a KZG
batch, and check every sum against the closed form Σ s_i·k_i·G (and the oracle's MSM where the input is small)."""
import numpy as np
import pytest

from oracle import bls12_377 as py

import msm_corpus as mc
from helpers import random_canonical_fr
from test_msm_paths_gpu import _dev, adversarial_bases, adversarial_scalars, check_kernels, set_env, traced

pytestmark = pytest.mark.gpu

PAIR_KERNELS = ("k_pair_desc<false>", "k_pair_level2<false, 4>", "k_bucket_accumulate_dense")


def repeated_digit_scalars(reps) -> np.ndarray:
    """scalar j repeated reps[j] times, with digit j + 1 in every 6-bit window below bit 252 (no signed-digit carries): with
    c = 6, bucket j of every window holds exactly reps[j] entries"""
    pattern = sum(1 << (6 * w) for w in range(42))
    vals = [(j + 1) * pattern for j, r in enumerate(reps) for _ in range(r)]
    return mc.to_limbs(vals)


def plain_bases(n: int, seed: int) -> mc.Bases:
    from snarkvm_b200 import device
    return mc.Bases.generated(device.generate_bases(n, seed).cpu().numpy(), seed)


def check(cpu, b, scal, oracle=True):
    from snarkvm_b200 import device
    got = device.msm(_dev(b.rows), _dev(scal))
    assert (got == mc.closed_form(cpu, b, scal)).all()
    if oracle and not b.torsion:
        assert (got == cpu.msm(b.rows, scal, 1)).all()
    return got


@pytest.mark.parametrize("reps", [[1, 2, 3] * 10 + [1], [17] * 31, [2 ** k + 1 for k in range(1, 6)] * 6 + [3]],
                         ids=["counts_1_2_3", "all_odd", "odd_at_every_level"])
def test_odd_bucket_counts(oracle_cpu, monkeypatch, reps):
    """c = 6 (31 buckets in use per window), four pair levels: single inputs at level 0 and above, next to pairs"""
    set_env(monkeypatch, {"SNARKVM_B200_MSM_C": 6, "SNARKVM_B200_MSM_LEVELS": 4})
    scal = repeated_digit_scalars(reps)
    b = plain_bases(scal.shape[0], 70)
    _, kern = traced(lambda: check(oracle_cpu, b, scal))
    check_kernels(kern, must=PAIR_KERNELS, counts={"k_pair_level2<false, 4>": 4})


def test_hot_bucket_over_full_background(oracle_cpu, monkeypatch):
    """2^16 points, c = 10, three levels: most scalars equal (one bucket per window holds ~60 % of the entries), the rest
    uniform, so a warp's pairs sit inside one huge bucket while its neighbours' span many small ones"""
    set_env(monkeypatch, {"SNARKVM_B200_MSM_C": 10, "SNARKVM_B200_MSM_LEVELS": 3})
    n = 1 << 16
    b = adversarial_bases(n, seed=71, torsion=False)
    scal = random_canonical_fr(n, seed=1710)
    hot = np.random.default_rng(1711).random(n) < 0.6
    scal[hot] = scal[0]
    check(oracle_cpu, b, scal, oracle=False)
    scal[:] = scal[0]                                            # every entry in one bucket per window
    check(oracle_cpu, b, scal, oracle=False)


def test_degenerate_pairs_and_infinite_singles(oracle_cpu, monkeypatch):
    """P and −P, equal points and ∞ bases under equal scalars, in buckets of odd and even counts: classify_pair takes its rare
    paths on paired entries, and single outputs are ∞ or a point whose partner cancelled"""
    set_env(monkeypatch, {"SNARKVM_B200_MSM_C": 6, "SNARKVM_B200_MSM_LEVELS": 3})
    reps = [1, 2, 3, 4, 5, 7, 9, 2, 3, 1] * 3 + [5]
    scal = repeated_digit_scalars(reps)
    n = scal.shape[0]
    b = plain_bases(n, 72)
    starts = np.concatenate([[0], np.cumsum(reps)])
    for j in range(len(reps)):                                   # rows of scalar j: one bucket per window
        rows = np.arange(starts[j], starts[j + 1])
        if j % 3 == 0:
            b.infinity(rows)
        elif j % 3 == 1 and len(rows) > 1:
            b.alternate(int(rows[0]), rows)                      # P, −P, P, …
        elif len(rows) > 1:
            b.repeat(int(rows[0]), rows[1:])                     # equal points: doublings
    check(oracle_cpu, b, scal)
    inf = np.frombuffer(py.projective_bytes_normalised(None), dtype=np.uint64)
    allinf = b.copy().infinity(np.arange(n))
    from snarkvm_b200 import device
    assert (device.msm(_dev(allinf.rows), _dev(scal)) == inf).all()


@pytest.mark.parametrize("scratch_mb", [None, 1024])
def test_2p24_layout_groups(oracle_cpu, monkeypatch, scratch_mb):
    """2^21 points in the 2^24 window layout (13 × 18 bits + a 20-bit top window), five levels, in one group and in several"""
    env = {"SNARKVM_B200_MSM_LEVELS": 5}
    if scratch_mb:
        env["SNARKVM_B200_MSM_SCRATCH_MB"] = scratch_mb
    set_env(monkeypatch, env)
    monkeypatch.delenv("SNARKVM_B200_MSM_SCRATCH_GB", raising=False)
    monkeypatch.setenv("SNARKVM_B200_MSM_WINDOWS", "18*13,20")
    from snarkvm_b200 import device
    n = 1 << 21
    b = adversarial_bases(n, seed=73)
    bases = _dev(b.rows)
    for f, kind in enumerate(("uniform", "few_hot")):
        scal = adversarial_scalars(kind, n, 1730 + f)
        if f == 0:
            got, kern = traced(lambda: device.msm(bases, _dev(scal)))
            groups = kern.get("k_scatter_records<false, false>", 0)
            assert (groups > 1) if scratch_mb else groups == 1, groups
            check_kernels(kern, must=PAIR_KERNELS, counts={"k_pair_level2<false, 4>": 5 * groups})
        else:
            got = device.msm(bases, _dev(scal))
        assert (got == mc.closed_form(oracle_cpu, b, scal)).all(), kind


def test_infinite_bases_in_level0_records(oracle_cpu, monkeypatch):
    """c = 6, three levels, every 7th base ∞ under counts 1, 2 and 3: ∞ records reach level 0 as single inputs and as either
    input of a pair, and single ∞ inputs survive the copy to the bucket's last output"""
    set_env(monkeypatch, {"SNARKVM_B200_MSM_C": 6, "SNARKVM_B200_MSM_LEVELS": 3})
    reps = [1, 2, 3] * 10 + [5]
    scal = repeated_digit_scalars(reps)
    b = plain_bases(scal.shape[0], 74)
    b.infinity(np.arange(0, scal.shape[0], 7))
    _, kern = traced(lambda: check(oracle_cpu, b, scal))
    check_kernels(kern, must=PAIR_KERNELS)
    n = 20000
    b = adversarial_bases(n, seed=75)
    for f, kind in enumerate(mc.SCALAR_FAMILIES):
        check(oracle_cpu, b, adversarial_scalars(kind, n, 1750 + f), oracle=False)


def test_precomputed_tables(oracle_cpu, monkeypatch):
    """the precomputed-table path (one shared bucket set, records from the tables) with two pair levels"""
    from snarkvm_b200 import device
    set_env(monkeypatch, {"SNARKVM_B200_MSM_PRE_C": 13, "SNARKVM_B200_MSM_PRE_LEVELS": 2})
    n = 1 << 15
    b = adversarial_bases(n, seed=76, torsion=False)
    pre = device.PrecomputedBases(_dev(b.rows))
    try:
        for f, kind in enumerate(("uniform", "equal", "special")):
            scal = adversarial_scalars(kind, n, 1760 + f)
            assert (pre.msm(_dev(scal)) == mc.closed_form(oracle_cpu, b, scal)).all(), kind
    finally:
        pre.free()


def test_kzg_batch(oracle_cpu, monkeypatch):
    """several KZG commitments in one pass (Montgomery coefficients, jobs of different lengths) through three pair levels"""
    from snarkvm_b200 import device
    set_env(monkeypatch, {"SNARKVM_B200_MSM_C": 9, "SNARKVM_B200_MSM_LEVELS": 3})
    n = 20000
    b = adversarial_bases(n, seed=77, torsion=False)
    lens = [20000, 1, 777, 12345]
    polys = [random_canonical_fr(k, seed=1770 + i) for i, k in enumerate(lens)]
    polys[2][:] = polys[2][0]                                    # one hot bucket per window in one job
    got = device.kzg_commit_batch(_dev(b.rows), [_dev(p) for p in polys])
    for i, p in enumerate(polys):
        want = mc.closed_form(oracle_cpu, b, oracle_cpu.fr_from_mont(p))
        assert (got[i] == want).all(), i


@pytest.mark.parametrize("lg", [16, 20])
def test_level_count_does_not_change_results(oracle_cpu, monkeypatch, lg):
    """levels 4, 5 and 6 forced through SNARKVM_B200_MSM_LEVELS give the same sum"""
    from snarkvm_b200 import device
    n = 1 << lg
    b = adversarial_bases(n, seed=78)
    bases = _dev(b.rows)
    scal = adversarial_scalars("few_hot", n, 1780)
    want = mc.closed_form(oracle_cpu, b, scal)
    for levels in (4, 5, 6):
        set_env(monkeypatch, {"SNARKVM_B200_MSM_C": 12, "SNARKVM_B200_MSM_LEVELS": levels})
        assert (device.msm(bases, _dev(scal)) == want).all(), levels
