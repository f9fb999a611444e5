"""Host model of the pair levels' descriptor pass (csrc/msm.cu: k_pair_desc, warp_bucket_first, warp_bucket_walk).

A level's buckets hold cnt_b inputs; bucket b has ⌊cnt_b/2⌋ pairs and, when cnt_b is odd, one single input.  Pair j is found
by one binary search per warp of 32 · DESC_CHUNKS pairs over the pair scan, then per 32-pair chunk by a walk that loads 32
bucket boundaries per round and counts the ones at or below each lane's index with a five-step shuffle search.  The model
replays that lane by lane and must give exactly the brute-force list: (first input, output position) of every pair and the
(input, output position) of every single input."""
import numpy as np
import pytest

DESC_CHUNKS = 8


def scan(c):
    return np.concatenate([[0], np.cumsum(c, dtype=np.int64)]).astype(np.int64)


def bucket_first(off, nb, x):
    lo, hi = 0, nb
    while hi - lo > 1:
        mid = (lo + hi) >> 1
        if off[mid] <= x:
            lo = mid
        else:
            hi = mid
    return lo


def bucket_walk(off, nb, b, xs):
    """warp_bucket_walk for the 32 lanes' indices xs (nondecreasing, off[b] <= xs[0])"""
    res = [b] * 32
    done = [False] * 32
    for rnd in range(2):
        e = [int(off[b + 1 + lane]) if b + 1 + lane <= nb else 0xFFFFFFFF for lane in range(32)]
        for lane in range(32):
            c, s = 0, 16
            while s >= 1:
                if e[c + s - 1] <= xs[lane]:
                    c += s
                s >>= 1
            if not done[lane] and e[31] > xs[lane]:
                res[lane], done[lane] = b + c, True
        if all(done):
            return res
        b += 32
    for lane in range(32):
        if not done[lane]:
            lo, hi = b, nb
            while hi - lo > 1:
                mid = (lo + hi) >> 1
                if off[mid] <= xs[lane]:
                    lo = mid
                else:
                    hi = mid
            res[lane] = lo
    return res


def model(cnt):
    nb = len(cnt)
    off_in, off_out, pair_off = scan(cnt), scan((cnt + 1) // 2), scan(cnt // 2)
    total = int(pair_off[nb])
    pairs = {}
    for j0w in range(0, total, 32 * DESC_CHUNKS):
        b = bucket_first(pair_off, nb, j0w)
        for j0 in range(j0w, min(j0w + 32 * DESC_CHUNKS, total), 32):
            xs = [min(j0 + lane, total - 1) for lane in range(32)]
            bj = bucket_walk(pair_off, nb, b, xs)
            b = bj[31]
            for lane in range(32):
                j = j0 + lane
                if j < total:
                    i = j - int(pair_off[bj[lane]])
                    assert j not in pairs
                    pairs[j] = (int(off_in[bj[lane]]) + 2 * i, int(off_out[bj[lane]]) + i)
    singles = [(int(off_in[b + 1]) - 1, int(off_out[b + 1]) - 1) for b in range(nb) if cnt[b] & 1]
    return [pairs[j] for j in range(total)], singles


def brute(cnt):
    pairs, singles, base_in, base_out = [], [], 0, 0
    for c in cnt.tolist():
        for i in range(c // 2):
            pairs.append((base_in + 2 * i, base_out + i))
        if c & 1:
            singles.append((base_in + c - 1, base_out + c // 2))
        base_in += c
        base_out += (c + 1) // 2
    return pairs, singles


CASES = {
    "random_small": lambda r: r.integers(0, 8, 3000),
    "with_zeros": lambda r: np.where(r.random(4000) < 0.6, 0, r.integers(0, 5, 4000)),
    "ones_and_zeros": lambda r: r.integers(0, 2, 5000),                  # no pairs at all, long runs without any
    "one_huge": lambda r: np.concatenate([r.integers(0, 4, 700), [20001], r.integers(0, 4, 900)]),
    "huge_among_empty": lambda r: np.concatenate([np.zeros(3000, np.int64), [4097], np.zeros(2000, np.int64), [3]]),
    "counts_1_2_3": lambda r: np.tile([1, 2, 3], 700),
    "mixed_scale": lambda r: r.integers(0, 2, 3000) * r.integers(0, 200, 3000),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_descriptor_enumeration_matches_brute_force(case):
    cnt = np.asarray(CASES[case](np.random.default_rng(len(case))), dtype=np.int64)
    assert model(cnt) == brute(cnt)


def test_outputs_cover_every_position_once():
    """pairs and singles together fill the level's outputs 0 … Σ⌈cnt/2⌉ − 1 exactly once, and consecutive pairs of a bucket
    write consecutive outputs"""
    cnt = np.random.default_rng(5).integers(0, 9, 2500)
    pairs, singles = model(cnt)
    outs = sorted([o for _, o in pairs] + [o for _, o in singles])
    assert outs == list(range(int(((cnt + 1) // 2).sum())))
