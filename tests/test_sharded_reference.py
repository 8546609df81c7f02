"""The cross-shard merge reference (tests/sharded_reference.py) on the CPU: `merge` against a plain Python loop, the merge of
exact per-shard answers against the exact answer over all rows, and negative controls that `compare` rejects."""
import numpy as np
import pytest

from myscaledb_b200.sharding import shard_range
from tests import sharded_reference as SR

F32 = np.float32


def _loop_merge(lists, k, descending):
    """The merge as a Python loop over tuples: sort key (distance or -distance, id), k kept, tail (sentinel, -1)."""
    nq = lists[0][0].shape[0]
    out = []
    for q in range(nq):
        ent = []
        for d, i in lists:
            for j in range(d.shape[1]):
                if i[q, j] >= 0:
                    ent.append((-float(d[q, j]) if descending else float(d[q, j]), int(i[q, j]), d[q, j]))
        ent.sort(key=lambda e: (e[0], e[1]))
        ent = ent[:k]
        out.append([(e[2], e[1]) for e in ent] + [(SR.sentinel(descending), -1)] * (k - len(ent)))
    dis = np.array([[e[0] for e in row] for row in out], F32)
    ids = np.array([[e[1] for e in row] for row in out], np.int64)
    return dis, ids


@pytest.mark.parametrize("descending", [False, True])
@pytest.mark.parametrize("seed", range(4))
def test_merge_equals_a_plain_loop(seed, descending):
    rng = np.random.default_rng(seed)
    nq, k = 7, 5
    lists = []
    base = 0
    for _ in range(int(rng.integers(1, 5))):
        ki = int(rng.integers(1, 9))
        d = rng.integers(-3, 4, (nq, ki)).astype(F32)             # few values: many ties across lists
        d[rng.random((nq, ki)) < 0.1] = F32(-0.0)
        i = base + rng.integers(0, 50, (nq, ki))
        i[rng.random((nq, ki)) < 0.3] = -1                        # unused slots anywhere in a list
        d[i < 0] = -np.inf if descending else np.inf
        lists.append((d, i.astype(np.int64)))
        base += 1000
    got = SR.merge(lists, k, descending)
    want = _loop_merge(lists, k, descending)
    assert not SR.compare(want, got)
    assert (got[1] >= -1).all()


def _sharded_exact(metric, x, y, k, world, alive=None, offsets=None):
    lists = []
    for r in range(world):
        lo, hi = shard_range(len(y), world, r)
        off = lo if offsets is None else offsets[r]
        lists.append(SR.integer_topk(metric, x, y[lo:hi], k, None if alive is None else alive[lo:hi], id_offset=off))
    return lists


@pytest.mark.parametrize("metric", [SR.L2, SR.IP])
@pytest.mark.parametrize("world", [2, 3, 4])
def test_merge_of_exact_shards_is_the_exact_answer(metric, world):
    rng = np.random.default_rng(world + 10 * metric)
    n, d, nq, k = 103, 16, 9, 7
    y = rng.integers(-8, 9, (n, d)).astype(F32)
    y[60:70] = y[5:15]                                            # duplicate rows on other shards: ties
    x = rng.integers(-8, 9, (nq, d)).astype(F32)
    x[:3] = y[5:8]
    alive = rng.random(n) < 0.7
    lo, hi = shard_range(n, world, world - 1)
    alive[lo:hi] = False                                           # a filter that removes a whole shard
    for a in (None, alive):
        merged = SR.merge(_sharded_exact(metric, x, y, k, world, a), k, metric == SR.IP)
        assert not SR.compare(SR.integer_topk(metric, x, y, k, a), merged)
    # k above the rows of every shard
    big = SR.merge(_sharded_exact(metric, x, y, 60, world), 60, metric == SR.IP)
    assert not SR.compare(SR.integer_topk(metric, x, y, 60), big)


def _case():
    rng = np.random.default_rng(7)
    n, d, nq, k = 40, 8, 5, 6
    y = rng.integers(-8, 9, (n, d)).astype(F32)
    y[30] = y[3]                                                   # row 3 (shard 0) and row 30 (shard 1) tie for query 0
    x = rng.integers(-8, 9, (nq, d)).astype(F32)
    x[0] = y[3]
    return y, x, k


def test_compare_rejects_a_tie_won_by_the_larger_id():
    y, x, k = _case()
    want = SR.merge(_sharded_exact(SR.L2, x, y, k, 2), k, False)
    assert want[1][0, :2].tolist() == [3, 30] and want[0][0, 0] == want[0][0, 1] == 0
    d, i = want[0].copy(), want[1].copy()
    i[0, :2] = [30, 3]
    assert SR.compare(want, (d, i))


def test_compare_rejects_an_id_offset_off_by_one():
    y, x, k = _case()
    want = SR.merge(_sharded_exact(SR.L2, x, y, k, 2), k, False)
    lo1 = shard_range(len(y), 2, 1)[0]
    got = SR.merge(_sharded_exact(SR.L2, x, y, k, 2, offsets=[0, lo1 + 1]), k, False)
    assert SR.compare(want, got)


def test_compare_rejects_a_dropped_shard():
    y, x, k = _case()
    lists = _sharded_exact(SR.IP, x, y, k, 3)
    want = SR.merge(lists, k, True)
    for drop in range(3):
        assert SR.compare(want, SR.merge(lists[:drop] + lists[drop + 1:], k, True)), drop


def test_compare_rejects_a_stale_answer_from_before_an_append():
    y, x, k = _case()
    before = SR.merge(_sharded_exact(SR.L2, x, y, k, 2), k, False)
    y2 = np.concatenate([y, x[1:2]])                              # the appended row is query 1's exact match
    after = SR.merge(_sharded_exact(SR.L2, x, y2, k, 2), k, False)
    assert after[1][1, 0] == len(y) and after[0][1, 0] == 0
    assert SR.compare(after, before)


def test_compare_rejects_a_tail_that_is_not_filled():
    y, x, k = _case()
    for metric in (SR.L2, SR.IP):
        want = SR.merge(_sharded_exact(metric, x, y[:4], k, 2), k, metric == SR.IP)   # 4 rows < k: a tail on every query
        assert (want[1][:, 4:] == -1).all() and (want[0][:, 4:] == SR.sentinel(metric == SR.IP)).all()
        d, i = want[0].copy(), want[1].copy()
        d[:, 4:] = 0                                                                     # tail distances left unwritten
        assert SR.compare(want, (d, i))
        d, i = want[0].copy(), want[1].copy()
        d[:, 4:] = SR.sentinel(metric != SR.IP)                                          # the other direction's sentinel
        assert SR.compare(want, (d, i))
