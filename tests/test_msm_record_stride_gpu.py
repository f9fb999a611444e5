"""The 128-byte level-0 records of the plain-bases pair levels (k_scatter_records writes each record as one whole line, level 0
reads it at that stride, level 1 writes 96-byte points over the same area) across several window groups.  A stride mistake in
the group-relative positions (*pos_base) or in the reuse of the record area by level 1 shows only when a later group writes
over an earlier group's area, so the 2^24 window layout runs here in seven groups and in one, against the closed form."""
import pytest

import msm_corpus as mc
from test_msm_paths_gpu import LARGE_TAIL, _dev, adversarial_bases, adversarial_scalars, check_kernels, set_env, traced

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("scratch_gb,groups", [(1, 7), (None, 1)])
def test_record_stride_window_groups(oracle_cpu, monkeypatch, scratch_gb, groups):
    """2^21 points, 13 × 18 bits + a 20-bit top window, four pair levels: 2^21 × 212 B per window against a 1 GiB budget
    gives two windows per group (the last group holds the top window's four sets); the default budget gives one group"""
    from snarkvm_b200 import device
    set_env(monkeypatch, {"SNARKVM_B200_MSM_LEVELS": 4})
    monkeypatch.setenv("SNARKVM_B200_MSM_WINDOWS", "18*13,20")
    if scratch_gb is None:
        monkeypatch.delenv("SNARKVM_B200_MSM_SCRATCH_GB", raising=False)
    else:
        monkeypatch.setenv("SNARKVM_B200_MSM_SCRATCH_GB", str(scratch_gb))
    n = 1 << 21
    b = adversarial_bases(n, seed=60)
    bases = _dev(b.rows)
    for f, kind in enumerate(("uniform", "special", "few_hot")):
        scal = adversarial_scalars(kind, n, 960 + f)
        if f == 0:
            got, kern = traced(lambda: device.msm(bases, _dev(scal)))
            check_kernels(kern, must=("k_pair_level2<false, 4>", "k_bucket_accumulate_dense") + LARGE_TAIL,
                          must_not=("k_bucket_accumulate",),
                          counts={"k_scatter_records<false, false>": groups})
        else:
            got = device.msm(bases, _dev(scal))
        assert (got == mc.closed_form(oracle_cpu, b, scal)).all(), kind
