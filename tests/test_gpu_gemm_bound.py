"""Every per-query list of the flat tensor-core top-k (two per CTA and query for bf16 and binary rows, one for fp32 rows, 16 CTAs
per query tile at 1 024 queries) shares one bound with the query's other lists: the best k-th key any of them has reached.
The lists filter against the smaller of their own k-th key and that bound.  What the shared bound can get wrong is checked here
bit for bit against the CPU oracle on integer-valued data (every product is exact, ties are everywhere):
  * 897, 1 000 and 1 024 queries (the last query tile partly padding, whose rows must neither read nor publish a bound) at
    corpus sizes from fewer tiles than CTAs to several tiles per CTA;
  * IP / L2 on bf16 rows, IP / L2 on fp32 rows (3xTF32), Hamming / Jaccard on binary rows, with and without an alive bitmap,
    at k = 10, 32 and 100;
  * rows repeated across the corpus, so equal keys straddle CTAs, the bound equals the k-th key and the smallest ids must win;
  * NaN and inf rows at 1 024 queries: only finite keys are published."""
import numpy as np
import pytest

import myscaledb_b200 as b2
import oracle as orc
from myscaledb_b200 import search as S

pytestmark = pytest.mark.gpu
F32 = np.float32
D = 64
NBYTES = 48
NQS = (897, 1000, 1024)
KS = (10, 32, 100)
# corpus tiles of 256 rows: 16, 17, 33, a partial 34th and 41 (at 8 query tiles: 16 CTAs per query tile)
SIZES = (4096, 4352, 8448, 8449, 10317)


def assert_exact(dg, ig, do, io, what):
    assert np.array_equal(ig, io), f"{what}: {int((ig != io).sum())} ids differ"
    assert np.array_equal(np.where(io >= 0, dg, 0), np.where(io >= 0, do, 0)), what


def tensor_search(c, x, k, alive):
    c.set_path(S.PATH_TENSOR)
    c.set_prefilter(1)   # the alive bitmap goes into the kernel's side entries
    return c.search(x, k, alive_bits=alive)


@pytest.mark.parametrize("n", SIZES)
def test_float_rows_against_the_oracle(n):
    rng = np.random.default_rng(n)
    y = rng.integers(-4, 5, (n, D), dtype=np.int8).astype(F32)
    x = rng.integers(-4, 5, (max(NQS), D), dtype=np.int8).astype(F32)
    mask = orc.pack_bits(rng.random(n) < 0.6)
    for metric in (b2.IP, b2.L2):
        ref = {a is None: orc.knn_flat(metric, x, y, max(KS), a) for a in (None, mask)}
        for dtype in (S.BF16, S.F32):
            c = b2.Corpus(metric, D, dtype=dtype).append(y)
            try:
                for alive in (None, mask):
                    do, io = ref[alive is None]
                    for nq in NQS:
                        for k in KS:
                            dg, ig = tensor_search(c, x[:nq], k, alive)
                            assert_exact(dg, ig, do[:nq, :k], io[:nq, :k], f"dtype={dtype} metric={metric} nq={nq} k={k}")
            finally:
                c.close()


@pytest.mark.parametrize("n", SIZES)
def test_binary_rows_against_the_oracle(n):
    rng = np.random.default_rng(3 * n)
    y = rng.integers(0, 256, (n, NBYTES), dtype=np.uint8)
    x = rng.integers(0, 256, (max(NQS), NBYTES), dtype=np.uint8)
    mask = orc.pack_bits(rng.random(n) < 0.6)
    for metric in (b2.HAMMING, b2.JACCARD):
        c = b2.Corpus(metric, NBYTES * 8, dtype=S.BIN).append(y)
        try:
            for alive in (None, mask):
                do, io = orc.knn_binary(metric, x, y, max(KS), alive)
                for nq in NQS:
                    for k in KS:
                        dg, ig = tensor_search(c, x[:nq], k, alive)
                        assert c.last_variant()[0] == S.KERNEL_GEMM_B1
                        assert_exact(dg, ig, do[:nq, :k], io[:nq, :k], f"metric={metric} nq={nq} k={k}")
        finally:
            c.close()


@pytest.mark.parametrize("k", KS)
def test_repeated_rows_keep_the_smallest_ids(k):
    """300 distinct rows repeated over 40 tiles: every key occurs about 34 times, spread over CTAs and warpgroups."""
    rng = np.random.default_rng(k)
    base = rng.integers(-3, 4, (300, D), dtype=np.int8).astype(F32)
    n = 40 * 256 + 100
    y = base[np.arange(n) % 300]
    x = rng.integers(-3, 4, (1024, D), dtype=np.int8).astype(F32)
    for metric in (b2.IP, b2.L2):
        c = b2.Corpus(metric, D, dtype=S.BF16).append(y)
        try:
            dg, ig = tensor_search(c, x, k, None)
        finally:
            c.close()
        do, io = orc.knn_flat(metric, x, y, k)
        assert_exact(dg, ig, do, io, f"repeated rows metric={metric}")


@pytest.mark.parametrize("k", [10, 32])
@pytest.mark.parametrize("dtype", [S.BF16, S.F32], ids=["bf16", "f32"])
def test_nan_and_inf_rows_at_1024_queries(dtype, k):
    rng = np.random.default_rng(17)
    n = 33 * 256 + 9
    y = rng.integers(-4, 5, (n, D), dtype=np.int8).astype(F32)
    x = rng.integers(-4, 5, (1024, D), dtype=np.int8).astype(F32)
    bad = rng.choice(n, 300, replace=False)
    y[bad[:100]] = np.nan
    y[bad[100:200], 3] = np.inf
    y[bad[200:], 5] = -np.inf
    keep = np.setdiff1d(np.arange(n), bad)
    c = b2.Corpus(b2.L2, D, dtype=dtype).append(y)
    try:
        with np.errstate(all="ignore"):
            dg, ig = tensor_search(c, x, k, None)
    finally:
        c.close()
    do, io = orc.knn_flat(b2.L2, x, y[keep], k)
    assert_exact(dg, ig, do, keep[io], "non-finite rows")
    assert not np.isin(ig, bad).any()
