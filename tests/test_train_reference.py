"""tests/train_reference.py against brute-force pure-Python restatements on tiny integer inputs, where ties are everywhere.
CPU only: nothing here needs a GPU or the library."""
import itertools

import numpy as np
import pytest

from tests import train_reference as T

F32 = np.float32


def brute_lloyd_step(x, c):
    """One assignment (ties to the smaller id) and update (empty: keep) in Python floats."""
    nc, d = len(c), len(c[0])
    sums, cnt = [[0.0] * d for _ in range(nc)], [0] * nc
    for row in x:
        best, bd = 0, None
        for k in range(nc):
            dist = sum((row[j] - c[k][j]) ** 2 for j in range(d))
            if bd is None or dist < bd:
                best, bd = k, dist
        cnt[best] += 1
        for j in range(d):
            sums[best][j] += row[j]
    return [[sums[k][j] / cnt[k] for j in range(d)] if cnt[k] else list(c[k]) for k in range(nc)], cnt


def brute_pairs(cnt):
    empties = [i for i, v in enumerate(cnt) if v == 0]
    order = sorted(range(len(cnt)), key=lambda i: (-cnt[i], i))
    out = []
    for e, dst in enumerate(empties):
        if cnt[order[e]] < 2:
            break
        out.append((dst, order[e]))
    return out


@pytest.mark.parametrize("seed", range(20))
def test_one_lloyd_step_matches_brute_force(seed):
    rng = np.random.default_rng(seed)
    n, d, nc = int(rng.integers(3, 14)), int(rng.integers(1, 4)), int(rng.integers(1, 6))
    x = rng.integers(-2, 3, (n, d)).astype(F32)   # small integers: equal distances everywhere
    t = T.kmeans(x, nc, 1)
    seeds = [int(i * n / nc) for i in range(nc)]
    assert seeds == T.strided(n, nc).tolist()
    want, cnt = brute_lloyd_step(x.tolist(), [x[i].tolist() for i in seeds])
    assert np.array_equal(t.centroids, np.array(want))
    assert np.array_equal(t.counts, np.array(cnt, float))
    # an empty cluster keeps its seed exactly; a mean carries the bound of its fp32 sum and division
    empty = np.array(cnt) == 0
    assert not t.delta[empty].any()
    S = np.abs(x.astype(np.float64)).sum(0)
    assert (t.delta[~empty] <= (n * T.U * 1.001) * S + T.U * np.abs(t.centroids[~empty])).all()


@pytest.mark.parametrize("seed", range(30))
def test_split_pairing_matches_brute_force(seed):
    rng = np.random.default_rng(seed)
    cnt = rng.integers(0, 4, int(rng.integers(2, 12)))   # many equal counts, some below 2
    pairs, tied = T.split_pairs(cnt)
    assert pairs == brute_pairs(cnt.tolist())
    srcs = [s for _, s in pairs]
    assert tied <= len(pairs) and (tied > 0) == any(sum(1 for v in cnt if v == cnt[s]) > 1 for s in srcs)


def test_split_nudges_both_copies_by_the_fp32_formula():
    # rows: two exact duplicates seed clusters 0 and 1 (cluster 1 goes empty), cluster 2 has 3 members
    x = np.array([[1, 2, 3], [1, 2, 3], [9, 9, 9], [10, 10, 10], [11, 12, 13]], F32)
    t = T.kmeans(x, 3, 2, seeds=[0, 1, 2])
    assert t.splits == 1 and t.tied_splits == 0
    # after iteration 0: cluster 0 = {0, 1} (the tie goes to the smaller id), cluster 1 empty, cluster 2 = rows 2..4
    v = np.array([10.0, 31 / 3, 35 / 3])
    eps = np.array([-1, 1, -1]) / 1024
    dst = v * (1 + eps) + eps * float(F32(1e-3))
    src = v * (1 - eps) - eps * float(F32(1e-3))
    # iteration 1 assigns with the split copies; rows 2 .. 4 sit on either side of the nudge
    c1 = np.array([[1, 2, 3], dst, src])
    want, _ = brute_lloyd_step(x.tolist(), c1.tolist())
    assert np.allclose(t.centroids, np.array(want), rtol=0, atol=1e-12)


@pytest.mark.parametrize("seed", range(20))
def test_majority_with_ties_matches_brute_force(seed):
    rng = np.random.default_rng(seed)
    n, nbytes, nc = int(rng.integers(2, 12)), int(rng.integers(1, 3)), int(rng.integers(1, 5))
    x = rng.integers(0, 4, (n, nbytes)).astype(np.uint8)   # two low bits only: duplicates and ties
    seeds = T.strided(n, nc)
    bits = [[(int(b) >> t) & 1 for b in row for t in range(8)] for row in x]
    c = [list(bits[i]) for i in seeds]
    a = [min(range(nc), key=lambda k: (sum(p != q for p, q in zip(r, c[k])), k)) for r in bits]
    for k in range(nc):
        mem = [bits[i] for i in range(n) if a[i] == k]
        for j in range(len(c[k])):
            ones = sum(m[j] for m in mem)
            if 2 * ones > len(mem):
                c[k][j] = 1
            elif 2 * ones < len(mem):
                c[k][j] = 0
    t = T.kmajority(x, nc, 1)
    want = np.packbits(np.array(c, np.uint8), axis=1, bitorder="little")
    assert np.array_equal(t.centroids[:, :nbytes], want)
    assert (t.centroids[:, nbytes:] == 0).all() and t.centroids.shape[1] == 16


def test_majority_tie_keeps_the_bit_and_the_perturbation_sets_it():
    # cluster 0 (seed row 0) = rows 0, 1: bit 0 is 1 in one of them, a tie; the seed's bit 0 is 0, so it stays 0
    x = np.array([[0b10], [0b11], [0xF0], [0xF0]], np.uint8)
    t = T.kmajority(x, 2, 1)
    assert t.centroids[0, 0] == 0b10 and t.ties >= 1
    assert T.kmajority(x, 2, 1, tie_sets=True).centroids[0, 0] == 0b11


def test_majority_middle_member_split_and_early_stop():
    # the seeds (rows 0 and 3) are equal: every row goes to cluster 0 (ties to the smaller id), whose majority is 0b111;
    # empty cluster 1 takes its middle member in row order, row 7 // 2 = 3 (= 1).  Iteration 1: the rows equal to 1 go to
    # cluster 1, the other five to cluster 0, whose majority is 0b1111
    x = np.array([[1], [3], [255], [1], [15], [254], [7]], np.uint8)
    t1 = T.kmajority(x, 2, 2)
    assert t1.splits == 1 and t1.centroids[:, 0].tolist() == [0b1111, 1]
    t = T.kmajority(x, 2, 10)
    assert t.stopped_early and t.iterations < 10 and t.empty_final == 0


def test_ambiguity_flag_fires_on_a_near_tie_and_not_on_separated_data():
    rng = np.random.default_rng(0)
    centres = np.array([[0, 0], [100, 0], [0, 100]], F32)
    x = (centres[np.arange(300) % 3] + rng.standard_normal((300, 2))).astype(F32)
    t = T.kmeans(x, 3, 5)
    assert not t.ambiguous and t.last_change == 0
    # one row exactly half-way between two centroids after the first update: decided by rounding alone
    y = np.array([[0, 0], [10, 0], [5, 0]], F32)
    t = T.kmeans(y, 2, 3, seeds=[0, 1])
    assert t.ambiguous, "a row on the bisector must be flagged"
    # a row 1e-7 (relative) off the bisector is within the fp32 tolerance too
    z = np.array([[0, 0], [10, 0], [5.000001, 0]], F32)
    assert T.kmeans(z, 2, 1, seeds=[0, 1]).ambiguous


def test_duplicate_seeds_are_exact_ties_not_ambiguity():
    x = np.array([[1, 1], [1, 1], [8, 8], [9, 9]], F32)
    t = T.kmeans(x, 3, 1, seeds=[0, 1, 2])
    assert not t.ambiguous and t.counts.tolist() == [2, 0, 2]


def test_build_decisions_and_sample_rule():
    assert [T.default_nlist(n) for n in (0, 1, 3000, 10 ** 6, 10 ** 9 * 400)] == [4, 4, 219, 4000, 65536]
    assert T.use_ivf(2000, 10, 10) and not T.use_ivf(1999, 10, 10)
    assert T.use_ivf(2400, 300, 300) and not T.use_ivf(2399, 300, 300) and not T.use_ivf(5000, 299, 300)
    assert np.array_equal(T.sample_rows(65536, 7), np.arange(65536))
    r = T.sample_rows(70001, 7)
    assert len(r) == 65536 and r[0] == 0 and r[-1] == int(65535 * 70001 / 65536) and (np.diff(r) >= 1).all()
    assert len(T.sample_rows(600000, 2048)) == 256 * 2048
    for n, ns in ((100, 100), (65536, 65536), (70000, 65536), (140000, 65536)):
        x = np.arange(n)[:, None]
        s = T.pq_sample(x)
        assert len(s) == ns and s[0, 0] == 0
        assert (np.diff(s[:, 0]) == max(1, n // ns)).all()


def test_sq_ranges_host_arithmetic():
    x = np.array([[-1.5, 2, 0.1], [3.25, 2, -0.7], [0.5, 2, 0.3]], F32)
    s = T.sq_ranges(x)
    lo, hi = x.min(0), x.max(0)
    for j in range(3):
        step = F32((hi[j] - lo[j]) / F32(255)) if hi[j] > lo[j] else F32(1)
        assert s[1, j] == step and s[2, j] == F32(F32(1) / step) and s[3, j] == F32(lo[j] + F32(F32(128) * step))
    assert s[1, 1] == 1 and s[3, 1] == 130
    assert np.array_equal(T.sq_ranges(x, fused_mid=True), s)


def test_every_small_case_agrees_with_exhaustive_pairing():
    for cnt in itertools.product(range(3), repeat=4):
        assert T.split_pairs(np.array(cnt))[0] == brute_pairs(list(cnt))
