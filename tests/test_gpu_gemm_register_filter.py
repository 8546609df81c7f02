"""The flat tensor-core top-k filters each group of 32 corpus columns straight from the accumulator registers: a lane reduces its
wgmma fragment to the best key of each of its rows, the quad and an owner lane per query row complete the test, and only a
group that can enter some list is staged in shared memory for its owners.  Lane L of warp w owns query row 16 w + L (L < 16) or
64 + 16 w + L - 16 of the tile, so a wrong owner, a wrong fragment row or a skipped group loses exactly the winners of one
(group, half, warp position).

Every query's best rows are placed in one chosen 32-column group of one 256-row tile: query q is aligned with "channel" q % 32,
and the rows of channel c fill group c % 4 of half (c // 4) % 2 of one tile, the last (partial) tile among them.  Over the
queries of a batch every channel meets every warp position of the tile.  Integer-valued data keeps every product and sum exact,
so ids and distances must equal the CPU oracle's bit for bit (cosine, whose keys carry an fp32 norm, to the bf16 contract of
tests/util.py), for IP, L2, cosine, Hamming and Jaccard, with and without an alive bitmap, with lists in shared memory
(k = 10) and in global scratch (k = 100), for batches with padding rows, and on the bf16, 3xTF32 and binary kernels."""
import numpy as np
import pytest

import myscaledb_b200 as b2
import oracle as orc
from myscaledb_b200 import search as S

from .util import check_topk

pytestmark = pytest.mark.gpu
F32 = np.float32
CHANNELS = 32
D = 128            # two bf16 k-blocks, four 3xTF32 k-blocks
NBYTES = 144       # one binary k-block and a partial second
N_TILES = 20       # + a partial last tile
TAIL = 100         # rows of the last tile: groups 0..2 of its first half full, group 3 partial
NQS = (200, 1025)  # padding rows in the last query tile
KS = (10, 100)


def layout():
    """n and, per channel, the rows of its group (channel c: group c % 4, half (c // 4) % 2, tile spread over the corpus; the
    channels 0..3 sit in the partial last tile)."""
    n = N_TILES * 256 + TAIL
    rows = {}
    for c in range(CHANNELS):
        g, h = c % 4, (c // 4) % 2
        t = N_TILES if c < 4 else (3 * c) % N_TILES
        r0 = t * 256 + h * 128 + g * 32
        rows[c] = np.arange(r0, min(r0 + 32, n))
    return n, rows


def float_data(nq, seed):
    n, rows = layout()
    rng = np.random.default_rng(seed)
    # integers up to 120 (exact in bf16), sums below 2^24; the noise is wide enough that rows rarely tie exactly in cosine
    y = rng.integers(-9, 10, (n, D)).astype(F32)
    x = rng.integers(-9, 10, (nq, D)).astype(F32)
    x[np.arange(nq), np.arange(nq) % CHANNELS] = 120
    for c, r in rows.items():
        y[r, c] = 60 + rng.integers(0, 21, len(r))
    return x, y


def binary_data(nq, seed):
    n, rows = layout()
    rng = np.random.default_rng(seed)
    y = rng.integers(0, 256, (n, NBYTES), dtype=np.uint8)
    pat = rng.integers(0, 256, (CHANNELS, NBYTES), dtype=np.uint8)
    x = pat[np.arange(nq) % CHANNELS].copy()
    x ^= (rng.random((nq, NBYTES)) < 0.02).astype(np.uint8) << rng.integers(0, 8, (nq, NBYTES)).astype(np.uint8)
    for c, r in rows.items():
        y[r] = pat[c] ^ ((rng.random((len(r), NBYTES)) < 0.05).astype(np.uint8) << rng.integers(0, 8, (len(r), NBYTES)).astype(np.uint8))
    return x, y


def alive_bits(n, use, seed):
    if not use:
        return None
    return orc.pack_bits(np.random.default_rng(seed).random(n) < 0.7)


def tensor_search(c, x, k, alive, kernel):
    c.set_path(S.PATH_TENSOR)
    c.set_prefilter(1)   # the alive bitmap goes into the kernel's side entries, not into a compacted copy
    dg, ig = c.search(x, k, alive_bits=alive)
    assert c.last_variant()[0] == kernel
    return dg, ig


def assert_exact(dg, ig, do, io):
    assert np.array_equal(ig, io), f"{int((ig != io).sum())} ids differ"
    assert np.array_equal(np.where(io >= 0, dg, 0), np.where(io >= 0, do, 0))


def assert_channel_winners(ig, nq, alive):
    """The setup does what it claims: without a bitmap, each query's best row is one of its channel's rows."""
    if alive is not None:
        return
    _, rows = layout()
    for q in range(nq):
        assert ig[q, 0] in rows[q % CHANNELS], q


@pytest.mark.parametrize("use_alive", [False, True], ids=["all", "alive"])
@pytest.mark.parametrize("nq", NQS)
@pytest.mark.parametrize("dtype", ["bf16", "tf32"])
@pytest.mark.parametrize("metric", [b2.IP, b2.L2, b2.COSINE], ids=["IP", "L2", "COSINE"])
def test_float_winners_in_one_group(metric, dtype, nq, use_alive):
    x, y = float_data(nq, 100 + nq)
    n = len(y)
    alive = alive_bits(n, use_alive, nq)
    kernel = S.KERNEL_GEMM_BF16 if dtype == "bf16" else S.KERNEL_GEMM_TF32X3
    c = b2.Corpus(metric, D, dtype=S.BF16 if dtype == "bf16" else S.F32).append(y)
    try:
        for k in KS:
            dg, ig = tensor_search(c, x, k, alive, kernel)
            if metric == b2.COSINE:
                do, io = orc.search_without_index(metric, x, y, k, alive)
                check_topk(metric, x, y, dg, ig, do, io)
            else:
                do, io = orc.knn_flat(metric, x, y, k, alive)
                assert_exact(dg, ig, do, io)
            assert_channel_winners(ig, nq, alive)
    finally:
        c.close()


@pytest.mark.parametrize("use_alive", [False, True], ids=["all", "alive"])
@pytest.mark.parametrize("nq", NQS)
@pytest.mark.parametrize("metric", [b2.HAMMING, b2.JACCARD], ids=["HAMMING", "JACCARD"])
def test_binary_winners_in_one_group(metric, nq, use_alive):
    x, y = binary_data(nq, 200 + nq)
    n = len(y)
    alive = alive_bits(n, use_alive, nq + 1)
    c = b2.Corpus(metric, NBYTES * 8, dtype=S.BIN).append(y)
    try:
        for k in KS:
            dg, ig = tensor_search(c, x, k, alive, S.KERNEL_GEMM_B1)
            do, io = orc.knn_binary(metric, x, y, k, alive)
            assert_exact(dg, ig, do, io)
            assert_channel_winners(ig, nq, alive)
    finally:
        c.close()
