"""CPU: the nonnative absorption of the Fq sponge (parameters, limbs, compression) in snarkvm_b200/poseidon.py and in its
restatement tests/varuna_transcript_oracle.py, and the order of prove_batch's transcript."""
import random

import pytest

import varuna_transcript_oracle as vto
from oracle import poseidon as op
from snarkvm_b200 import poseidon

R, Q = vto.R, vto.Q


def _params():
    return poseidon.parameters(poseidon.FIELD_FQ)


def test_find_parameters():
    assert vto.find_parameters(377, 253, vto.WEIGHT) == (5, 51)
    assert poseidon.find_parameters(377, 253, poseidon.OPT_WEIGHT) == (5, 51)
    assert (poseidon.NONNATIVE_LIMBS, poseidon.NONNATIVE_LIMB_BITS) == (5, 51)
    for base, target in ((377, 253), (253, 377), (253, 253), (377, 377), (200, 100)):
        for a, b in ((vto.WEIGHT, poseidon.OPT_WEIGHT), ("constraints", poseidon.OPT_CONSTRAINTS)):
            assert vto.find_parameters(base, target, a) == poseidon.find_parameters(base, target, b), (base, target, a)


def test_overhead_of_noise_two():
    assert vto.overhead(2) == poseidon.overhead(2) == 2
    for x in (1, 3, 4, 5, 7, 8, 255, 256, 257):
        assert vto.overhead(x) == poseidon.overhead(x), x


@pytest.mark.parametrize("v", [0, 1, R - 1, (1 << 51) - 1, 1 << 51, (1 << 252) + 12345] + [random.Random(k).randrange(R) for k in range(8)])
def test_limbs_recombine(v):
    limbs = vto.limbs(v, 5, 51)
    assert len(limbs) == 5 and all(0 <= x < 1 << 51 for x in limbs)
    assert sum(x << (51 * (4 - i)) for i, x in enumerate(limbs)) == v            # big limb first


@pytest.mark.parametrize("n", range(1, 8))
def test_compression_matches_brute_force(n):
    """stream lengths 1–7: pairs merge as first · 2^53 + second, an odd last limb stays alone"""
    rng = random.Random(n)
    src = [rng.randrange(1 << 51) for _ in range(n)]
    want = []
    for i in range(0, n, 2):
        want.append(src[i] * 2 ** (51 + 2) + src[i + 1] if i + 1 < n else src[i])
    assert vto.compress(src, 51) == want


@pytest.mark.parametrize("count", [0, 1, 2, 3, 4, 7])
def test_nonnative_encoding_matches_restatement(count):
    rng = random.Random(100 + count)
    values = [rng.choice([0, 1, R - 1, rng.randrange(R)]) for _ in range(count)]
    got = poseidon.nonnative_field_elements(values)
    assert got == vto.compress([x for v in values for x in vto.limbs(v, 5, 51)], 51)
    assert len(got) == (5 * count + 1) // 2 and all(0 <= x < Q for x in got)
    # the same elements absorbed natively give the same sponge
    a, b = vto.PoseidonSponge(Q, 377, _params()), op.Sponge(Q, 377, _params())
    a.absorb_nonnative_field_elements(values)
    b.absorb_native_field_elements(got)
    assert a.state == b.state and a.mode == b.mode
    with pytest.raises(ValueError):
        poseidon.nonnative_field_elements([R])


def _view(rng, batch_sizes, zk):
    pt = lambda: (rng.randrange(Q), rng.randrange(Q))          # noqa: E731 — the transcript does not need points on the curve
    K = len(batch_sizes)
    return {"w": [pt() for _ in range(sum(batch_sizes))], "mask": pt() if zk else None, "h_0": pt(), "g_1": pt(), "h_1": None,
            "g_a": [pt() for _ in range(K)], "g_b": [pt() for _ in range(K)], "g_c": [pt() for _ in range(K)], "h_2": pt(),
            "third_sums": [[[rng.randrange(R) for _ in range(3)] for _ in range(b)] for b in batch_sizes],
            "fourth_sums": [[rng.randrange(R) for _ in range(3)] for _ in range(K)],
            "evaluations": [rng.randrange(R) for _ in range(1 + 3 * K)]}


@pytest.mark.parametrize("batch_sizes,zk", [([1], False), ([1], True), ([1, 2, 4], False)])
def test_prove_batch_transcript_order(batch_sizes, zk):
    rng = random.Random(len(batch_sizes))
    K, n_public = len(batch_sizes), 4
    public = [[[1] + [rng.randrange(R) for _ in range(n_public - 1)] for _ in range(b)] for b in batch_sizes]
    vks = [[(rng.randrange(Q), rng.randrange(Q)) for _ in range(11)] + [None] for _ in range(K)]
    ch, log, _s = vto.prove_batch_transcript(_params(), batch_sizes, public, vks, _view(rng, batch_sizes, zk))
    want = [("absorb_bytes", 11)]
    for b in batch_sizes:
        want += [("absorb_bytes", 8)] + [("absorb_nonnative", n_public)] * b
    want += [("absorb_native", 36)] * K
    want += [("absorb_native", 3 * (sum(batch_sizes) + zk))]
    want += [("squeeze", b - 1 + (1 if i else 0)) for i, b in enumerate(batch_sizes)]
    want += [("absorb_native", 3), ("squeeze", 3), ("absorb_native", 6)]
    want += [("absorb_nonnative", 3)] * sum(batch_sizes) + [("squeeze", 1)]
    want += [("absorb_native", 9 * K)] + [("absorb_nonnative", 3)] * K + [("squeeze", 2)] + [("squeeze", 3)] * (K - 1)
    want += [("absorb_native", 3), ("squeeze", 1), ("absorb_nonnative", 1 + 3 * K)]
    want += [("squeeze_short", 1)] * (2 + 3 + 3 * K + 2)
    assert log == want
    # the first circuit gets no circuit combiner, a batch of one no instance combiner
    assert ch["batch_combiners"][0][0] == 1
    for (cc, inst), b in zip(ch["batch_combiners"], batch_sizes):
        assert len(inst) == b and inst[0] == 1
    assert ch["deltas"][0][0] == 1 and len(ch["deltas"]) == K and all(len(d) == 3 for d in ch["deltas"])
    assert len(ch["opening"]) == 3 * K + 7
