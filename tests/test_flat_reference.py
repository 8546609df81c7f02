"""CPU checks of tests/flat_reference.py: the reference against a plain Python loop on tiny inputs, and the comparator's
negative controls (each kind of wrong answer must be rejected)."""
import math

import numpy as np
import pytest

from tests import flat_reference as fr
from tests.util import to_bf16_values

F32 = np.float32
PATH_DTYPES = [("scan", fr.F32), ("scan", fr.BF16), ("bf16", fr.BF16), ("tf32", fr.F32)]


def _loop_distances(metric, dtype, path, y, x):
    """(key, returned distance) of every pair with Python floats, one pair at a time."""
    ys = to_bf16_values(y) if dtype == fr.BF16 else y
    xo = to_bf16_values(x) if path == "bf16" else x
    key = np.zeros((len(x), len(y)))
    dis = np.zeros((len(x), len(y)))

    def unit(v):
        ss = math.fsum(float(a) * float(a) for a in v)
        f = 1.0 if ss < float(np.finfo(F32).eps) else 1.0 / math.sqrt(ss)
        return [float(a) * f for a in v]

    for q in range(len(x)):
        for r in range(len(y)):
            a, b = [float(v) for v in xo[q]], [float(v) for v in ys[r]]
            if metric == fr.IP:
                s = math.fsum(p * t for p, t in zip(a, b))
                key[q, r], dis[q, r] = -s, s
            elif metric == fr.COSINE:
                s = math.fsum(p * t for p, t in zip(unit(a), unit(b)))
                key[q, r] = dis[q, r] = 1.0 - s
            else:
                direct = math.fsum((float(p) - t) ** 2 for p, t in zip(x[q], b))
                dis[q, r] = direct
                key[q, r] = direct if path == "scan" else math.fsum(p * p for p in a) + math.fsum(t * t for t in b) - 2 * math.fsum(
                    p * t for p, t in zip(a, b))
    return key, dis


@pytest.mark.parametrize("path,dtype", PATH_DTYPES)
@pytest.mark.parametrize("metric", [fr.L2, fr.IP, fr.COSINE])
def test_reference_matches_a_python_loop(metric, path, dtype):
    rng = np.random.default_rng(metric * 10 + len(path) + dtype)
    y = rng.standard_normal((7, 5)).astype(F32)
    y[3] = 1e-4          # squared norm 5e-8 < FLT_EPSILON: the cosine factor is 1
    y[4] = 0.0
    x = rng.standard_normal((3, 5)).astype(F32)
    x[1] = 0.0
    r = fr.reference(metric, dtype, path, y, x, 4)
    key, dis = _loop_distances(metric, dtype, path, y, x)
    np.testing.assert_allclose(r.key, key, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(r.dis, dis, rtol=1e-12, atol=1e-12)
    assert (r.key_tol >= 0).all() and (r.dis_tol >= 0).all()
    if path == "bf16":
        # the bf16 query operand is not the fp32 query: the tensor-core reference must differ from the scan's
        assert not np.allclose(fr.reference(metric, dtype, "scan", y, x, 4).key, r.key, rtol=1e-9, atol=0)


def test_tolerances_follow_the_derivation():
    u = 2.0 ** -24
    m_sum = 768 / 32 + 13
    scan = {fr.IP: m_sum * u, fr.L2: (m_sum + 2) * u, fr.COSINE: (2 * m_sum + 8) * u}
    for metric in (fr.L2, fr.IP, fr.COSINE):
        assert fr.tolerances("scan", fr.F32, 768, metric) == (scan[metric], scan[metric], None)
    m, md, w = fr.tolerances("bf16", fr.BF16, 768, fr.L2)
    assert m == (m_sum + 4) * u and md == scan[fr.L2]
    assert w[0] == 34 * u * 48 and w[767] == 34 * u and w[16] == 34 * u * 47
    assert fr.tolerances("bf16", fr.BF16, 768, fr.IP)[0] == 0
    assert fr.tolerances("bf16", fr.BF16, 768, fr.COSINE)[0] == (m_sum + 8) * u
    m, _, w = fr.tolerances("tf32", fr.F32, 768, fr.IP)
    assert m == 32 * u and w[0] == 18 * u * 3 * 96 and w[767] == 18 * u * 3
    # bf16 rows pad to 64 elements, fp32 rows to 4
    assert fr.tolerances("bf16", fr.BF16, 65, fr.L2)[0] == fr.tolerances("bf16", fr.BF16, 128, fr.L2)[0]
    assert fr.tolerances("scan", fr.F32, 5, fr.L2) == fr.tolerances("scan", fr.F32, 8, fr.L2)
    # the weighted product bound: one column at the start of a 768-d tf32 row sees every later step
    r = fr.reference(fr.IP, fr.F32, "tf32", np.eye(1, 768, 0, dtype=F32), np.ones((1, 768), F32), 1)
    assert r.key_tol[0, 0] == pytest.approx(32 * u + 18 * u * 3 * 96)


def _case(metric=fr.L2, path="scan", dtype=fr.F32, n=300, nq=4, k=10, quirk=False, seed=0):
    rng = np.random.default_rng(seed)
    y = rng.standard_normal((n, 16)).astype(F32)
    x = rng.standard_normal((nq, 16)).astype(F32)
    r = fr.reference(metric, dtype, path, y, x, k, quirk=quirk)
    return r, fr.ideal_answer(r)


@pytest.mark.parametrize("path,dtype", PATH_DTYPES)
@pytest.mark.parametrize("metric", [fr.L2, fr.IP, fr.COSINE])
def test_comparator_accepts_the_ideal_answer(metric, path, dtype):
    r, (dis, ids) = _case(metric, path, dtype)
    assert fr.compare(r, dis, ids) == []
    assert fr.compare(r, dis, ids + (1 << 33), id_offset=1 << 33) == []
    assert fr.error_ratio(r, dis, ids) <= 1.0


@pytest.mark.parametrize("metric", [fr.L2, fr.IP, fr.COSINE])
def test_comparator_rejects_each_wrong_answer(metric):
    r, (dis, ids) = _case(metric)
    k = r.k

    def rejects(d, i, what):
        assert fr.compare(r, d, i), what

    # a swapped id: rank 0 takes a row that is not in the top k
    i = ids.copy()
    i[0, 0] = next(v for v in range(r.n) if v not in ids[0])
    rejects(dis, i, "swapped id")
    # a dropped row: the best row is missing, the rest move up and the k-th slot takes the (k+1)-th row
    i, d = ids.copy(), dis.copy()
    cand = np.lexsort((np.arange(r.n), r.key[0]))
    i[0] = cand[1:k + 1]
    d[0] = r.dis[0, i[0]].astype(F32)
    rejects(d, i, "dropped row")
    # a duplicate id
    i = ids.copy()
    i[1, 3] = i[1, 2]
    rejects(dis, i, "duplicate id")
    # a distance off by twice its bound
    d = dis.copy()
    j = 4
    d[2, j] = F32(r.dis[2, ids[2, j]] + 2 * r.dis_tol[2, ids[2, j]] * (1 if metric != fr.IP else -1))
    rejects(d, ids, "distance off by twice its bound")
    # an unsorted pair
    i, d = ids.copy(), dis.copy()
    i[3, [5, 6]] = i[3, [6, 5]]
    d[3, [5, 6]] = d[3, [6, 5]]
    rejects(d, i, "unsorted pair")
    # a wrong tail sentinel: more slots than rows
    r2, (d2, i2) = _case(metric, n=5, k=8)
    assert fr.compare(r2, d2, i2) == []
    d2 = d2.copy()
    d2[0, 7] = F32(-fr.FLT_MAX if metric != fr.IP else fr.FLT_MAX)
    assert fr.compare(r2, d2, i2), "wrong tail sentinel"
    # a tail slot filled although rows were left, and an unfilled slot in the middle
    i2b = i2.copy()
    i2b[1, 2] = -1
    assert fr.compare(r2, d2, i2b)


def test_comparator_equal_distances_and_the_ip_quirk():
    # exact ties (identical rows) must come in ascending id order on every metric
    y = np.repeat(np.arange(1, 4, dtype=F32)[:, None], 8, axis=1)
    y = np.concatenate([y, y, y])                     # rows 0-2, 3-5, 6-8 are copies of each other
    x = np.full((1, 8), 0.5, F32)
    for metric in (fr.L2, fr.IP, fr.COSINE):
        r = fr.reference(metric, fr.F32, "scan", y, x, 9)
        dis, ids = fr.ideal_answer(r)
        assert fr.compare(r, dis, ids) == []
        i = ids.copy()
        t = np.nonzero(dis[0, :-1] == dis[0, 1:])[0][0]
        i[0, [t, t + 1]] = i[0, [t + 1, t]]
        assert fr.compare(r, dis, i), metric
    # IP quirk: rows scoring <= FLT_MIN are never returned and the tail holds FLT_MIN
    rng = np.random.default_rng(3)
    y = rng.standard_normal((50, 8)).astype(F32)
    x = rng.standard_normal((3, 8)).astype(F32)
    r = fr.reference(fr.IP, fr.F32, "scan", y, x, 40, quirk=True)
    dis, ids = fr.ideal_answer(r)
    assert (ids == -1).any() and (dis[ids == -1] == F32(fr.FLT_MIN)).all()
    assert fr.compare(r, dis, ids) == []
    d = dis.copy()
    d[ids == -1] = -fr.FLT_MAX
    assert fr.compare(r, d, ids)
    # a NaN row is never eligible; returning it is rejected
    y[7] = np.nan
    r = fr.reference(fr.L2, fr.F32, "scan", y, x, 10)
    dis, ids = fr.ideal_answer(r)
    assert 7 not in ids and fr.compare(r, dis, ids) == []
    i = ids.copy()
    i[0, -1] = 7
    assert fr.compare(r, dis, i)


def test_alive_bitmap_limits_the_filled_slots():
    rng = np.random.default_rng(4)
    y = rng.standard_normal((40, 8)).astype(F32)
    x = rng.standard_normal((2, 8)).astype(F32)
    alive = np.zeros(40, bool)
    alive[[3, 17, 30]] = True
    r = fr.reference(fr.COSINE, fr.BF16, "bf16", y, x, 5, alive=alive)
    dis, ids = fr.ideal_answer(r)
    assert sorted(ids[0, :3].tolist()) == [3, 17, 30] and (ids[:, 3:] == -1).all()
    assert fr.compare(r, dis, ids) == []
    i = ids.copy()
    i[0, 2] = 4
    assert fr.compare(r, dis, i)
