"""From 2^22 points the pair-level G1 MSM runs its window groups on two streams, the caller's and an auxiliary one, with a
scratch set per group in flight.  Every case is checked against the closed form (Σ s_i·h_i)·G of generated bases P_i = h_i·G: forced group
counts (an odd count leaves one stream a group behind), a call on a non-default stream read after synchronising only that
stream, and two host threads calling at once on two streams."""
import threading

import numpy as np
import pytest

from oracle import bls12_377 as py

from helpers import affine_array, generated_base_multipliers, random_canonical_fr

pytestmark = pytest.mark.gpu

ENV = ("SNARKVM_B200_MSM_C", "SNARKVM_B200_MSM_LEVELS", "SNARKVM_B200_MSM_WINDOWS", "SNARKVM_B200_MSM_SCRATCH_GB",
       "SNARKVM_B200_MSM_SCRATCH_MB")
SEED = 0x6E0


@pytest.fixture(autouse=True)
def plain_env(monkeypatch):
    for k in ENV:
        monkeypatch.delenv(k, raising=False)


@pytest.fixture(scope="module")
def bases_by_lg():
    from snarkvm_b200 import device
    cache = {}

    def get(lg):
        if lg not in cache:
            cache.clear()
            cache[lg] = device.generate_bases(1 << lg, seed=SEED)
        return cache[lg]
    return get


def closed_form(oracle_cpu, scal):
    ks = np.zeros((len(scal), 4), dtype=np.uint64)
    ks[:, 0] = generated_base_multipliers(SEED, len(scal))
    return oracle_cpu.g1_mul(affine_array([py.G1_GENERATOR])[0], oracle_cpu.fr_dot_canonical(scal, ks))


def _dev(x):
    import torch
    return torch.from_numpy(x.view(np.int64).copy()).cuda()


# Group counts from msm_core's sizing (two groups run at once, from 2^22 points): per window 212 B per point (128-byte level-0
# records), each of the two groups in flight sized for half the budget.  2^22 (c = 16, 16 windows, 848 MiB per window):
# 14000 MB → 8 + 8, 12000 MB → 6 + 6 + 4; no budget splits 16 windows into five groups, so that case takes c = 15
# (17 windows): 7000 MB → 4 + 4 + 4 + 4 + 1.  2^23 (c = 17, 15 windows, 1696 MiB per window): 28000 MB → 8 + 7, 20000 MB →
# 5 + 5 + 5, 12000 MB → 3 + 3 + 3 + 3 + 3.
@pytest.mark.parametrize("lg,scratch_mb,c,groups", [
    (22, 14000, None, 2), (22, 12000, None, 3), (22, 7000, 15, 5),
    (23, 28000, None, 2), (23, 20000, None, 3), (23, 12000, None, 5),
])
def test_forced_group_counts(oracle_cpu, bases_by_lg, monkeypatch, lg, scratch_mb, c, groups):
    from snarkvm_b200 import device
    monkeypatch.setenv("SNARKVM_B200_MSM_SCRATCH_MB", str(scratch_mb))
    if c is not None:
        monkeypatch.setenv("SNARKVM_B200_MSM_C", str(c))
    assert device.msm_plan(1 << lg)["levels"] > 0
    scal = random_canonical_fr(1 << lg, seed=100 * lg + groups)
    got = device.msm(bases_by_lg(lg), _dev(scal))
    assert (got == closed_form(oracle_cpu, scal)).all(), (lg, groups)


def test_result_in_order_on_a_side_stream(oracle_cpu, bases_by_lg):
    """window sums written on a non-default stream are complete once that stream alone is synchronised"""
    import torch
    from snarkvm_b200 import device
    n = 1 << 22
    bases = bases_by_lg(22)
    scal = random_canonical_fr(n, seed=7)
    plan = device.msm_plan(n)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        d_scal = _dev(scal)
        sums = device.msm_window_sums(bases, d_scal)
        s.synchronize()
        host = sums.cpu().numpy()
    assert (device.msm_finish(host, plan["c"]) == closed_form(oracle_cpu, scal)).all()


def test_two_threads_two_streams(oracle_cpu, bases_by_lg):
    """two host threads, each on its own stream, call the pipelined MSM at the same time"""
    import torch
    from snarkvm_b200 import device
    n = 1 << 22
    bases = bases_by_lg(22)
    scal = [random_canonical_fr(n, seed=20 + k) for k in range(2)]
    d_scal = [_dev(v) for v in scal]
    torch.cuda.synchronize()
    results, errors = {}, []
    barrier = threading.Barrier(2)

    def work(k):
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                barrier.wait()
                results[k] = [device.msm(bases, d_scal[k]) for _ in range(2)]
        except Exception as e:      # pragma: no cover
            errors.append(e)

    threads = [threading.Thread(target=work, args=(k,)) for k in range(2)]
    [t.start() for t in threads]
    [t.join() for t in threads]
    assert not errors, errors
    for k in range(2):
        want = closed_form(oracle_cpu, scal[k])
        assert all((r == want).all() for r in results[k]), k
