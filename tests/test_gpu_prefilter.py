"""Pre-filtered exact search (prefilter.cu): a selective filter's rows are compacted and only they are scored.

Every case runs the same search forced to the full masked scan (prefilter 1), in auto (0) and forced to the gathered path
(2), and requires identical ids and bit-identical distances.  last_rows_scored proves which path ran: the corpus size after
a full scan, the kept rows after a gathered one."""
import threading

import numpy as np
import pytest

import myscaledb_b200 as b2
from myscaledb_b200 import search as S
from tests.util import to_bf16_values

pytestmark = pytest.mark.gpu
F32 = np.float32
FLT_MIN = np.finfo(np.float32).tiny

N = 20_037           # not a multiple of 8, 32 or 256
D = 96
BIG, BIG_D = 180_001, 768    # 553 MB of fp32 rows: above the smallest corpus auto pre-filters (512 MiB of rows)
BIN_BIG = 4_200_001          # x 128 bytes: 538 MB


def bitmap(n, rows, garbage=True):
    """LSB-first bitmap of n bits with `rows` set; with garbage=True every bit past n in the last byte is set too."""
    b = np.zeros((n + 7) // 8, np.uint8)
    rows = np.asarray(rows, np.int64)
    np.bitwise_or.at(b, rows >> 3, (1 << (rows & 7)).astype(np.uint8))
    if garbage and n % 8:
        b[-1] |= np.uint8((0xFF << (n % 8)) & 0xFF)
    return b


def budget(n, row_bytes):
    return min(n // 8, (1 << 30) // row_bytes)


def kept(n, count, seed, edges=True):
    """`count` distinct rows of n, the first and the last among them when edges is set and count >= 2"""
    rng = np.random.default_rng(seed)
    if count == 0:
        return np.zeros(0, np.int64)
    if edges and count >= 2:
        mid = rng.choice(np.arange(1, n - 1), count - 2, replace=False)
        return np.sort(np.concatenate([[0, n - 1], mid]))
    return np.sort(rng.choice(n, count, replace=False))


def identical(a, b):
    assert np.array_equal(a[1], b[1]), "ids differ"
    assert np.array_equal(np.ascontiguousarray(a[0]).view(np.uint32), np.ascontiguousarray(b[0]).view(np.uint32)), "distances differ"


def three_modes(c, q, k, bits):
    out = {}
    for mode in (1, 0, 2):
        c.set_prefilter(mode)
        d, i = c.search(q, k, alive_bits=bits)
        out[mode] = (d, i, c.last_rows_scored())
    c.set_prefilter(0)
    return out


def check(c, n, row_bytes, q, k, rows, bits=None, auto=None):
    """never / auto / always agree; never scores n rows, always scores len(rows) when they fit the budget.
    auto: True / False = the gathered / full path must have run, None = either."""
    bits = bitmap(n, rows) if bits is None else bits
    r = three_modes(c, q, k, bits)
    identical(r[1], r[0])
    identical(r[1], r[2])
    assert r[1][2] == n
    assert r[2][2] == (len(rows) if len(rows) <= budget(n, row_bytes) else n)
    if auto is not None:
        assert r[0][2] == (len(rows) if auto else n)
    ids = r[1][1]
    assert np.isin(ids[ids >= 0], rows).all()
    return r[1]


def float_rows(metric, n, seed, d=D):
    rng = np.random.default_rng(seed)
    y = rng.standard_normal((n, d), dtype=F32)
    if metric == b2.L2:
        y += 40.0                     # far from the origin: the tensor path's L2 re-score decides the distances
    if metric == b2.COSINE:
        y[::97] = 0.0                 # zero rows (no normalisation)
    return y


_CORPORA = {}


def float_corpus(dtype, metric):
    key = (dtype, metric)
    if key not in _CORPORA:
        y = float_rows(metric, N, 11 + metric)
        if dtype == S.BF16:
            y = to_bf16_values(y)
        _CORPORA[key] = (b2.Corpus(metric, D, dtype=dtype).append(y), y)
    return _CORPORA[key]


def row_bytes_of(dtype, d):
    return {S.F32: ((d + 3) // 4 * 4) * 4, S.BF16: ((d + 63) // 64 * 64) * 2, S.BIN: d // 8}[dtype]


def queries(metric, nq, seed, d=D):
    q = np.random.default_rng(seed).standard_normal((nq, d)).astype(F32)
    return q + 40.0 if metric == b2.L2 else q


@pytest.mark.parametrize("dtype", [S.F32, S.BF16])
@pytest.mark.parametrize("metric", [b2.L2, b2.IP, b2.COSINE])
@pytest.mark.parametrize("nq,k", [(1, 10), (3, 1), (8, 100), (20, 10), (129, 100), (1025, 10)])
def test_float_alive_counts(dtype, metric, nq, k):
    c, _ = float_corpus(dtype, metric)
    q = queries(metric, nq, nq)
    rb = row_bytes_of(dtype, D)
    b = budget(N, rb)
    for count in (0, 1, max(k - 3, 1), k, 300, b, b + 1, N // 2):
        check(c, N, rb, q, k, kept(N, count, seed=count))


@pytest.mark.parametrize("dtype", [S.F32, S.BF16])
@pytest.mark.parametrize("metric", [b2.L2, b2.IP, b2.COSINE])
def test_float_large_k(dtype, metric):
    c, _ = float_corpus(dtype, metric)
    rb = row_bytes_of(dtype, D)
    for nq, k in ((1, 1024), (20, 1024), (129, 1024)):
        check(c, N, rb, queries(metric, nq, 5), k, kept(N, 1500, seed=k))
    c.set_path(S.PATH_SCAN)              # k = 2048 runs on the scan path only
    try:
        check(c, N, rb, queries(metric, 3, 6), 2048, kept(N, 2400, seed=7))
    finally:
        c.set_path(S.PATH_AUTO)


@pytest.mark.parametrize("dtype", [S.F32, S.BF16])
@pytest.mark.parametrize("path", [S.PATH_SCAN, S.PATH_TENSOR])
def test_ties_duplicate_rows(dtype, path):
    """integer-valued rows, every row present three times: equal distances everywhere, the smaller row id must win"""
    rng = np.random.default_rng(3)
    base = rng.integers(-2, 3, (3000, 64)).astype(F32)
    y = np.repeat(base, 3, axis=0)
    n = len(y)
    c = b2.Corpus(b2.IP, 64, dtype=dtype).append(y).set_path(path)
    q = rng.integers(-2, 3, (24, 64)).astype(F32)
    rows = np.sort(np.concatenate([np.arange(0, n, 7), np.arange(1, n, 11)]))
    rows = np.unique(rows)[: budget(n, row_bytes_of(dtype, 64))]
    check(c, n, row_bytes_of(dtype, 64), q, 50, rows)
    c.close()


@pytest.mark.parametrize("bits", [1024, 200])     # 1024: b1 tensor-core eligible rows; 200 bits = 25-byte rows: scan only
@pytest.mark.parametrize("metric", [b2.HAMMING, b2.JACCARD])
@pytest.mark.parametrize("nq,k", [(1, 10), (3, 1), (20, 100), (129, 10), (1025, 10)])
def test_binary_alive_counts(bits, metric, nq, k):
    rng = np.random.default_rng(bits + metric)
    y = rng.integers(0, 256, (N, bits // 8), dtype=np.uint8)
    q = rng.integers(0, 256, (nq, bits // 8), dtype=np.uint8)
    c = b2.Corpus(metric, bits, dtype=S.BIN).append(y)
    rb = bits // 8
    b = budget(N, rb)
    for count in (0, 1, max(k - 3, 1), k, 300, b, b + 1, N // 2):
        check(c, N, rb, q, k, kept(N, count, seed=count + 1))
    c.close()


@pytest.mark.parametrize("dtype", [S.F32, S.BF16])
def test_auto_on_a_large_corpus(dtype):
    """auto gathers a sparse filter and scans a dense one, on both kernel families; a small corpus is never gathered"""
    n = BIG if dtype == S.F32 else 2 * BIG
    y = float_rows(b2.IP, n, 21, BIG_D)
    c = b2.Corpus(b2.IP, BIG_D, dtype=dtype).append(y)
    rb = row_bytes_of(dtype, BIG_D)
    for nq in (1, 20, 1024):
        q = queries(b2.IP, nq, 22, BIG_D)
        check(c, n, rb, q, 10, kept(n, 50, seed=1), auto=True)
        check(c, n, rb, q, 10, kept(n, n // 100, seed=2), auto=True)
        check(c, n, rb, q, 10, kept(n, n // 2, seed=3), auto=False)
        # no filter: the full scan, whatever the mode
        for mode in (0, 2):
            c.set_prefilter(mode)
            c.search(q, 10)
            assert c.last_rows_scored() == n
    c.close()
    small, _ = float_corpus(dtype, b2.IP)
    check(small, N, row_bytes_of(dtype, D), queries(b2.IP, 20, 23), 10, kept(N, 50, seed=4), auto=False)


def test_garbage_bits_past_n_are_ignored():
    c, _ = float_corpus(S.F32, b2.L2)
    rows = kept(N, 40, seed=9)
    clean, dirty = bitmap(N, rows, garbage=False), bitmap(N, rows, garbage=True)
    assert not np.array_equal(clean, dirty)
    q = queries(b2.L2, 4, 9)
    a = check(c, N, row_bytes_of(S.F32, D), q, 50, rows, bits=dirty)
    b = check(c, N, row_bytes_of(S.F32, D), q, 50, rows, bits=clean)
    identical(a, b)


def test_search_append_search():
    y = float_rows(b2.IP, 30_001, 31)
    c = b2.Corpus(b2.IP, D).append(y[:20_001])
    q = queries(b2.IP, 8, 31)
    check(c, 20_001, row_bytes_of(S.F32, D), q, 20, kept(20_001, 200, seed=1))
    c.append(y[20_001:])
    check(c, 30_001, row_bytes_of(S.F32, D), q, 20, kept(30_001, 2000, seed=2))
    check(c, 30_001, row_bytes_of(S.F32, D), q, 20, kept(30_001, 100, seed=3))
    c.close()


def test_two_threads_different_filters():
    y = float_rows(b2.L2, BIG, 41, BIG_D)
    c = b2.Corpus(b2.L2, BIG_D).append(y)
    q = queries(b2.L2, 4, 41, BIG_D)
    bits = [bitmap(BIG, kept(BIG, 64 + 500 * t, seed=t)) for t in range(2)]
    c.set_prefilter(1)
    want = [c.search(q, 10, alive_bits=b) for b in bits]
    c.set_prefilter(0)
    for t in range(2):
        identical(c.search(q, 10, alive_bits=bits[t]), want[t])
        assert c.last_rows_scored() == 64 + 500 * t
    errors = []

    def worker(t):
        try:
            for _ in range(25):
                identical(c.search(q, 10, alive_bits=bits[t]), want[t])
        except Exception as e:   # noqa: BLE001 -- reported by the main thread
            errors.append(e)

    th = [threading.Thread(target=worker, args=(t,)) for t in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors
    c.close()


def _never(metric, y, q, k, bits, dtype=S.F32, d=BIG_D):
    c = b2.Corpus(metric, d, dtype=dtype).append(y).set_prefilter(1)
    out = c.search(q, k, alive_bits=bits)
    c.close()
    return out


def gathered(call, rows):
    """run a one-shot call and require that it scored exactly `rows` rows (the pre-filtered path)"""
    out = call()
    assert S.thread_last_rows_scored() == rows
    return out


def test_one_shot_flat_and_binary_knn():
    """the one-shot calls run auto on a corpus large enough to be pre-filtered"""
    y = float_rows(b2.COSINE, BIG, 51, BIG_D)
    q = queries(b2.COSINE, 3, 51, BIG_D)
    bits = bitmap(BIG, kept(BIG, 120, seed=5))
    for metric in (b2.L2, b2.IP, b2.COSINE):
        got = gathered(lambda: b2.flat_knn(metric, q, y, 10, alive_bits=bits), 120)
        identical(got, _never(metric, y, q, 10, bits))
    rng = np.random.default_rng(52)
    yb = rng.integers(0, 256, (BIN_BIG, 128), dtype=np.uint8)
    qb = rng.integers(0, 256, (20, 128), dtype=np.uint8)      # 20 queries of 1024 bits: the b1 tensor-core path
    bb = bitmap(BIN_BIG, kept(BIN_BIG, 300, seed=6))
    for metric in (b2.HAMMING, b2.JACCARD):
        got = gathered(lambda: b2.binary_knn(metric, qb, yb, 10, alive_bits=bb), 300)
        identical(got, _never(metric, yb, qb, 10, bb, S.BIN, 1024))


def test_one_shot_metric_change_and_larger_part_on_one_thread():
    """The per-thread scratch corpus is re-dimensioned in place: after small parts of metrics with side arrays (binary and
    L2: row_bias, cosine: row_scale), an IP part that is much larger keeps those short arrays.  The gathered path must read
    only the side arrays its metric uses."""
    assert S.lib().b200_thread_release() == 0
    rng = np.random.default_rng(55)
    small = float_rows(b2.L2, 1000, 55, BIG_D)
    qs = queries(b2.L2, 2, 55, BIG_D)
    b2.binary_knn(b2.HAMMING, rng.integers(0, 256, (2, 128), dtype=np.uint8), rng.integers(0, 256, (1000, 128), dtype=np.uint8), 5)
    b2.part_scan(b2.L2, qs, small, 5)
    b2.flat_knn(b2.COSINE, qs, small, 5)
    y = float_rows(b2.IP, BIG, 56, BIG_D)
    q = queries(b2.IP, 3, 56, BIG_D)
    rows = kept(BIG, 2000, seed=56)
    bits = bitmap(BIG, rows)
    want = _never(b2.IP, y, q, 10, bits)
    identical(gathered(lambda: b2.flat_knn(b2.IP, q, y, 10, alive_bits=bits), 2000), want)   # a short row_scale left over
    b2.part_scan(b2.L2, qs, small, 5)
    identical(gathered(lambda: b2.flat_knn(b2.IP, q, y, 10, alive_bits=bits), 2000), want)   # a short row_bias left over
    assert S.lib().b200_thread_release() == 0


def test_one_shot_part_scan_row_exists_and_ip_quirk():
    y = float_rows(b2.IP, BIG, 61, BIG_D)
    q = queries(b2.IP, 2, 61, BIG_D)
    rows = kept(BIG, 150, seed=6)
    bits = bitmap(BIG, rows)
    row_exists = np.zeros(BIG, np.uint8)
    row_exists[rows] = 1
    k = 200                               # more than the kept rows: negative IP scores reach the result and are dropped
    d_ref, i_ref = _never(b2.IP, y, q, k, bits)
    keep = (i_ref >= 0) & (d_ref > FLT_MIN)
    want = (np.where(keep, d_ref, FLT_MIN).astype(F32), np.where(keep, i_ref, -1))
    assert (~keep & (i_ref >= 0)).any()
    identical(gathered(lambda: b2.part_scan(b2.IP, q, y, k, filter_bits=bits), 150), want)
    identical(gathered(lambda: b2.part_scan(b2.IP, q, y, k, row_exists=row_exists), 150), want)
    identical(gathered(lambda: b2.part_scan(b2.L2, q, y, 10, filter_bits=bits), 150), _never(b2.L2, y, q, 10, bits))
    rng = np.random.default_rng(62)
    yb = rng.integers(0, 256, (BIN_BIG, 128), dtype=np.uint8)
    qb = rng.integers(0, 256, (20, 128), dtype=np.uint8)
    bb = bitmap(BIN_BIG, kept(BIN_BIG, 300, seed=7))
    got = gathered(lambda: b2.part_scan(b2.HAMMING, qb, yb, 10, filter_bits=bb), 300)
    identical(got, _never(b2.HAMMING, yb, qb, 10, bb, S.BIN, 1024))


def _index_modes(ix, q, k, bits, n, alive, extra=""):
    """prefilter 1 / 0 / 2 on an exact index path: identical answers; 1 scores every row, 2 only the kept ones (auto scans in
    full: these parts are below the smallest corpus auto pre-filters)"""
    out, rows = [], []
    for m in (1, 0, 2):
        out.append(ix.search(q, k, params=f"{extra}prefilter={m}", alive_bits=bits))
        rows.append(S.thread_last_rows_scored())
    identical(out[0], out[1])
    identical(out[0], out[2])
    assert rows == [n, n, alive]
    return out[0]


@pytest.mark.parametrize("metric", [b2.L2, b2.COSINE])
def test_index_flat_fallback_and_exact_batch(metric):
    y = float_rows(metric, N, 71)
    q = queries(metric, 20, 71)
    bits = bitmap(N, kept(N, 90, seed=7))
    flat = b2.VectorIndex("FLAT", metric, D).build(y)
    ref = _index_modes(flat, q, 10, bits, N, 90)
    small = b2.VectorIndex("IVFFLAT", metric, D, "ncentroids=4096").build(y)   # below 8 * nlist rows: the FLAT fallback
    assert not small.info()["uses_ivf"]
    identical(_index_modes(small, q, 10, bits, N, 90), ref)
    ivf = b2.VectorIndex("IVFFLAT", metric, D, "ncentroids=16").build(y)
    assert ivf.info()["uses_ivf"]
    identical(_index_modes(ivf, q, 10, bits, N, 90, "exact_batch=1, "), ref)
    # the list scan is not affected by prefilter
    ls = [ivf.search(q, 10, params=f"nprobe=4, prefilter={m}", alive_bits=bits) for m in (1, 0, 2)]
    identical(ls[0], ls[1])
    identical(ls[0], ls[2])
    with pytest.raises(S.B200Error):
        flat.search(q, 10, params="prefilter=3", alive_bits=bits)
    for ix in (flat, small, ivf):
        ix.close()


def test_index_binaryflat():
    rng = np.random.default_rng(81)
    y = rng.integers(0, 256, (N, 128), dtype=np.uint8)
    q = rng.integers(0, 256, (20, 128), dtype=np.uint8)
    ix = b2.VectorIndex("BINARYFLAT", b2.HAMMING, 1024).build(y)
    bits = bitmap(N, kept(N, 70, seed=8))
    identical(_index_modes(ix, q, 10, bits, N, 70), _never(b2.HAMMING, y, q, 10, bits, S.BIN, 1024))
    ix.close()


def test_set_prefilter_rejects_unknown_modes():
    c, _ = float_corpus(S.F32, b2.IP)
    for bad in (-1, 3):
        with pytest.raises(S.B200Error):
            c.set_prefilter(bad)
