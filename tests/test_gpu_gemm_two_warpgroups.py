"""The bf16 and binary tensor-core top-k run two consumer warpgroups per CTA: warpgroup w owns rows [128 w, 128 w + 128) of
every 256-row corpus tile, with its own side entries (row norms, popcounts, alive bits) and its own per-query lists, and the
CTA publishes two partial lists per query.  What only that structure can get wrong is checked here bit for bit against the
CPU oracle on integer-valued data (every product and sum is exact, ties are everywhere):
  * corpus sizes at which the second warpgroup's half is empty, partial and full, in the only tile and in the last of many;
  * L2 and Hamming / Jaccard, whose keys need the per-row side entry of exactly the right row, with and without an alive bitmap;
  * winners that all sit in first halves, or all in second halves: a dropped partial list loses every one of them;
  * a k whose lists leave shared memory for the global scratch (one region per warpgroup)."""
import numpy as np
import pytest

import myscaledb_b200 as b2
import oracle as orc
from myscaledb_b200 import search as S

pytestmark = pytest.mark.gpu
F32 = np.float32
REMAINDERS = (1, 127, 128, 129, 255, 256, 257, 384, 385)
SIZES = REMAINDERS + tuple(4096 + r for r in REMAINDERS)
D = 192           # three bf16 k-blocks: the 3-stage ring wraps inside a tile
NBYTES = 144      # one binary k-block and a partial second
NQ = 200          # two query tiles, the second partly padding
K_SMEM, K_GMEM = 10, 100


def assert_exact(dg, ig, do, io):
    assert np.array_equal(ig, io), f"{int((ig != io).sum())} ids differ"
    assert np.array_equal(np.where(io >= 0, dg, 0), np.where(io >= 0, do, 0))


def tensor_search(c, x, k, alive, kernel):
    c.set_path(S.PATH_TENSOR)
    c.set_prefilter(1)   # the alive bitmap goes into the kernel's side entries, not into a compacted copy
    dg, ig = c.search(x, k, alive_bits=alive)
    assert c.last_variant()[:3] == (kernel, 1, 1)
    return dg, ig


@pytest.mark.parametrize("n", SIZES)
def test_bf16_rows_at_half_and_tile_boundaries(n):
    rng = np.random.default_rng(n)
    y = rng.integers(-4, 5, (n, D), dtype=np.int8).astype(F32)
    x = rng.integers(-4, 5, (NQ, D), dtype=np.int8).astype(F32)
    mask = rng.random(n) < 0.5
    for metric in (b2.IP, b2.L2):
        c = b2.Corpus(metric, D, dtype=S.BF16).append(y)
        try:
            for alive in (None, orc.pack_bits(mask)):
                for k in (K_SMEM, K_GMEM):
                    dg, ig = tensor_search(c, x, k, alive, S.KERNEL_GEMM_BF16)
                    do, io = orc.knn_flat(metric, x, y, k, alive)
                    assert_exact(dg, ig, do, io)
        finally:
            c.close()


@pytest.mark.parametrize("n", SIZES)
def test_binary_rows_at_half_and_tile_boundaries(n):
    rng = np.random.default_rng(7 * n)
    y = rng.integers(0, 256, (n, NBYTES), dtype=np.uint8)
    x = rng.integers(0, 256, (NQ, NBYTES), dtype=np.uint8)
    mask = rng.random(n) < 0.5
    for metric in (b2.HAMMING, b2.JACCARD):
        c = b2.Corpus(metric, NBYTES * 8, dtype=S.BIN).append(y)
        try:
            for alive in (None, orc.pack_bits(mask)):
                for k in (K_SMEM, K_GMEM):
                    dg, ig = tensor_search(c, x, k, alive, S.KERNEL_GEMM_B1)
                    do, io = orc.knn_binary(metric, x, y, k, alive)
                    assert_exact(dg, ig, do, io)
        finally:
            c.close()


@pytest.mark.parametrize("winners_in_half", [0, 1])
@pytest.mark.parametrize("metric", [b2.IP, b2.L2], ids=["IP", "L2"])
def test_all_winners_in_one_warpgroups_half(metric, winners_in_half):
    """Rows of one half of every tile are near the queries, the other half's are far away: the result is one warpgroup's lists."""
    n = 40 * 256 + 200
    rng = np.random.default_rng(11 + winners_in_half)
    x = rng.integers(1, 4, (NQ, D), dtype=np.int8).astype(F32)            # positive queries
    near = (np.arange(n) % 256) // 128 == winners_in_half
    y = rng.integers(1, 4, (n, D), dtype=np.int8).astype(F32)
    y[~near] *= -1                                                          # IP: negative scores; L2: far from every query
    c = b2.Corpus(metric, D, dtype=S.BF16).append(y)
    try:
        for k in (K_SMEM, K_GMEM):
            dg, ig = tensor_search(c, x, k, None, S.KERNEL_GEMM_BF16)
            do, io = orc.knn_flat(metric, x, y, k)
            assert_exact(dg, ig, do, io)
            assert near[ig].all()
    finally:
        c.close()


def test_side_entries_belong_to_the_warpgroups_own_rows():
    """L2 keys are ||y||^2 - 2 q.y with ||y||^2 from the side array.  Row r + 128 is row r scaled by 3: the dot products of the two
    halves differ by the factor alone, so a key built from the other half's norm ranks a wrong row first."""
    n = 16 * 256
    rng = np.random.default_rng(3)
    base = rng.integers(-2, 3, (n // 2, D), dtype=np.int8).astype(F32).reshape(16, 128, D)
    y = np.concatenate([base, 3 * base], axis=1).reshape(n, D)
    x = rng.integers(-2, 3, (NQ, D), dtype=np.int8).astype(F32)
    mask = rng.random(n) < 0.5
    c = b2.Corpus(b2.L2, D, dtype=S.BF16).append(y)
    try:
        for alive in (None, orc.pack_bits(mask)):
            dg, ig = tensor_search(c, x, K_SMEM, alive, S.KERNEL_GEMM_BF16)
            do, io = orc.knn_flat(b2.L2, x, y, K_SMEM, alive)
            assert_exact(dg, ig, do, io)
    finally:
        c.close()
