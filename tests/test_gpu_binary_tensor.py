"""Binary (Hamming / Jaccard) search on the tensor cores: gemm_topk_kernel<B1> (wgmma .b1 AND + popcount, fused top-k).

Every key is an integer expression below 2^24 (Jaccard: one IEEE division of two such integers), so the tensor-core path must
return the SAME BYTES as the popcount scan and exactly the oracle's ids and distances, tails (-1 / FLT_MAX) included."""
import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import myscaledb_b200 as b2
import oracle as orc
from myscaledb_b200 import search as S

pytestmark = pytest.mark.gpu
FLT_MAX = np.finfo(np.float32).max
ERR_UNSUPPORTED = 3


def min_nq(nbytes):
    """kBinaryTensorMinQB2 in capi.cu: auto sends binary batches of at least this many queries to the tensor cores"""
    return -(-20480 // (nbytes * nbytes))


def rows(rng, n, nbytes):
    return rng.integers(0, 256, (n, nbytes), dtype=np.uint8)


def search(c, path, x, k, alive=None):
    c.set_path(path)
    dis, ids = c.search(x, k, alive_bits=alive)
    return dis, ids, c.last_variant()[0]


def assert_same_bytes(a, b):
    assert np.array_equal(a[1], b[1])
    assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32))


def assert_oracle(metric, x, y, k, dis, ids, alive=None):
    do, io = orc.knn_binary(metric, x, y, k, alive)
    assert np.array_equal(ids, io)
    assert np.array_equal(np.where(io >= 0, dis, 0), np.where(io >= 0, do, 0))
    assert (dis[io < 0] == FLT_MAX).all()


def check_paths(metric, y, x, k, alive=None):
    """path 2 against the oracle and byte for byte against path 1"""
    c = b2.Corpus(metric, y.shape[1] * 8, dtype=S.BIN).append(y)
    dt, it, kt = search(c, 2, x, k, alive)
    ds, is_, ks = search(c, 1, x, k, alive)
    c.close()
    assert kt == S.KERNEL_GEMM_B1 and ks == S.KERNEL_SCAN
    assert_same_bytes((dt, it), (ds, is_))
    assert_oracle(metric, x, y, k, dt, it, alive)
    return dt, it


# (nq, k, metric, with an alive bitmap): cycled over the (n, width) grid so every value meets every tile size
COMBOS = [(1, 1, b2.HAMMING, False), (129, 10, b2.JACCARD, True), (1024, 100, b2.HAMMING, True), (1025, 1024, b2.JACCARD, False),
          (1, 1024, b2.JACCARD, True), (129, 100, b2.HAMMING, False)]


@pytest.mark.parametrize("n", [1, 255, 256, 257, 513, 70_000])
# < one k-block, < one, exactly one, a partial second, two; 4096 bits (4 k-blocks) and the widest rows, 65536 bits (64)
@pytest.mark.parametrize("nbytes", [16, 48, 128, 144, 256, 512, 8192])
def test_oracle_parity_at_tile_and_kblock_boundaries(n, nbytes):
    rng = np.random.default_rng(n * 1000 + nbytes)
    combos = COMBOS if n < 70_000 else COMBOS[:3]
    wide = nbytes > 256                     # the oracle's time: at most 4 MB of rows and 2^29 row bytes x queries per call
    if wide:
        n = min(n, (1 << 22) // nbytes - 1)
    y = rows(rng, n, nbytes)
    for nq, k, metric, with_alive in combos:
        if wide:
            nq = min(nq, max(1, (1 << 29) // (n * nbytes)))
        x = rows(rng, nq, nbytes)
        alive = orc.pack_bits(rng.random(n) < 0.7) if with_alive else None
        check_paths(metric, y, x, k, alive)


@pytest.mark.parametrize("metric", [b2.HAMMING, b2.JACCARD])
def test_scale_two_million_rows(metric):
    n, nbytes = 2_000_003, 128
    rng = np.random.default_rng(metric)
    y = rows(rng, n, nbytes)
    x = rows(rng, 2048, nbytes)
    c = b2.Corpus(metric, nbytes * 8, dtype=S.BIN).append(y)
    for nq in (1024, 2048):
        for k in (10, 100):
            t = search(c, 2, x[:nq], k)
            s = search(c, 1, x[:nq], k)
            assert t[2] == S.KERNEL_GEMM_B1 and s[2] == S.KERNEL_SCAN
            assert_same_bytes(t, s)
            assert_oracle(metric, x[:2], y, k, t[0][:2], t[1][:2])
    c.close()


def test_ties_and_degenerate_rows():
    rng = np.random.default_rng(5)
    y = np.repeat(rows(rng, 1, 128), 70_000, axis=0)
    x = rows(rng, 200, 128)
    for metric in (b2.HAMMING, b2.JACCARD):
        c = b2.Corpus(metric, 1024, dtype=S.BIN).append(y)
        for path in (0, 2):                       # every key ties, across CTAs and tiles: ids 0..k-1
            dis, ids, kern = search(c, path, x, 10)
            assert kern == S.KERNEL_GEMM_B1
            assert (ids == np.arange(10)[None, :]).all()
            assert (dis == dis[:, :1]).all()
        c.close()
    # all-zero rows and queries: Jaccard or == 0 -> 0 (a non-zero query against zero rows -> 1), Hamming = popc(q)
    y = np.zeros((3000, 64), np.uint8)
    x = rows(rng, 150, 64)
    x[::3] = 0
    pq = np.unpackbits(x, axis=1).sum(1).astype(np.float32)
    dis, ids = check_paths(b2.HAMMING, y, x, 20)
    assert (dis == pq[:, None]).all() and (ids == np.arange(20)[None, :]).all()
    dis, ids = check_paths(b2.JACCARD, y, x, 20)
    assert (dis == np.where(pq == 0, 0.0, 1.0)[:, None]).all() and (ids == np.arange(20)[None, :]).all()


@pytest.mark.parametrize("p_alive", [0.0, 0.001, 0.5, 1.0])
@pytest.mark.parametrize("metric", [b2.HAMMING, b2.JACCARD])
def test_filters_with_k_above_the_alive_count(p_alive, metric):
    rng = np.random.default_rng(int(p_alive * 1000) + metric)
    n, k = 1000, 1024
    y = rows(rng, n, 32)
    x = rows(rng, 200, 32)
    alive = orc.pack_bits(rng.random(n) < p_alive)
    dis, ids = check_paths(metric, y, x, k, alive)
    n_alive = int(np.unpackbits(alive, bitorder="little")[:n].sum())
    assert (ids[:, n_alive:] == -1).all() and (ids[:, :n_alive] >= 0).all()


@settings(max_examples=40, deadline=None)
@given(st.integers(1, 3000), st.integers(1, 16), st.integers(1, 300), st.integers(1, 64), st.integers(0, 2 ** 31),
       st.sampled_from([b2.HAMMING, b2.JACCARD]), st.sampled_from([0, 1, 2]), st.booleans())
def test_random_inputs_every_path_exact(n, width16, nq, k, seed, metric, path, with_alive):
    rng = np.random.default_rng(seed)
    nbytes = 16 * width16
    y = rows(rng, n, nbytes)
    x = rows(rng, nq, nbytes)
    alive = orc.pack_bits(rng.random(n) < 0.6) if with_alive else None
    c = b2.Corpus(metric, nbytes * 8, dtype=S.BIN).append(y)
    dis, ids, kern = search(c, path, x, k, alive)
    c.close()
    want = {0: S.KERNEL_GEMM_B1 if nq >= min_nq(nbytes) else S.KERNEL_SCAN, 1: S.KERNEL_SCAN, 2: S.KERNEL_GEMM_B1}[path]
    assert kern == want
    assert_oracle(metric, x, y, k, dis, ids, alive)


def test_auto_dispatch_and_unsupported_widths():
    rng = np.random.default_rng(9)
    y = rows(rng, 5000, 32)
    c = b2.Corpus(b2.HAMMING, 256, dtype=S.BIN).append(y)
    m = min_nq(32)
    assert m == 20
    for nq, want in ((1, S.KERNEL_SCAN), (m - 1, S.KERNEL_SCAN), (m, S.KERNEL_GEMM_B1), (1500, S.KERNEL_GEMM_B1)):
        x = rows(rng, nq, 32)
        dis, ids, kern = search(c, 0, x, 10)
        assert kern == want, nq
        assert_oracle(b2.HAMMING, x, y, 10, dis, ids)
    c.close()
    y = rows(rng, 5000, 128)                     # 1024 bits: one query stays on the scan, two go to the tensor cores
    c = b2.Corpus(b2.JACCARD, 1024, dtype=S.BIN).append(y)
    for nq, want in ((1, S.KERNEL_SCAN), (2, S.KERNEL_GEMM_B1)):
        x = rows(rng, nq, 128)
        dis, ids, kern = search(c, 0, x, 10)
        assert kern == want, nq
        assert_oracle(b2.JACCARD, x, y, 10, dis, ids)
    c.close()
    # 33-byte rows: not a 16-byte multiple -> auto stays on the scan, a forced tensor path is refused
    y = rows(rng, 5000, 33)
    x = rows(rng, 100, 33)
    c = b2.Corpus(b2.JACCARD, 264, dtype=S.BIN).append(y)
    dis, ids, kern = search(c, 0, x, 10)
    assert kern == S.KERNEL_SCAN
    assert_oracle(b2.JACCARD, x, y, 10, dis, ids)
    with pytest.raises(b2.B200Error) as ei:
        search(c, 2, x, 10)
    assert ei.value.code == ERR_UNSUPPORTED and "16 bytes" in str(ei.value)
    c.close()


@pytest.mark.parametrize("metric", [b2.HAMMING, b2.JACCARD])
def test_host_buffer_entry_points_use_the_tensor_cores(metric):
    """b200_binary_knn / binary b200_part_scan keep a per-thread scratch corpus: above the threshold they run the b1 kernel,
    which launches one kernel more than the scan path (the query popcounts)."""
    rng = np.random.default_rng(11 + metric)
    n = 20_000
    y = rows(rng, n, 64)
    x = rows(rng, 4 * min_nq(64), 64)
    exists = (rng.random(n) < 0.8).astype(np.uint8)
    calls = [lambda q: b2.binary_knn(metric, q, y, 15),
             lambda q: b2.part_scan(metric, q, y, 15, filter_bits=orc.pack_bits(exists != 0)),
             lambda q: b2.part_scan(metric, q, y, 15, row_exists=exists)]
    for call in calls:
        launches = []
        for q in (x[:min_nq(64) - 1], x):
            S.launch_count(reset=True)
            dis, ids = call(q)
            launches.append(S.launch_count())
            alive = None if call is calls[0] else orc.pack_bits(exists != 0)
            assert_oracle(metric, q, y, 15, dis, ids, alive)
        assert launches[1] == launches[0] + 1, launches


def test_search_device_with_id_offset_and_device_alive_bitmap():
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(13)
    n, nq, k = 30_000, 300, 25
    y = rows(rng, n, 128)
    x = rows(rng, nq, 128)
    alive = orc.pack_bits(rng.random(n) < 0.5)
    for metric in (b2.HAMMING, b2.JACCARD):
        c = b2.Corpus(metric, 1024, dtype=S.BIN).append(y)
        c.set_path(2)
        dh, ih = c.search(x, k, alive_bits=alive)
        tq = torch.from_numpy(x).cuda()
        ta = torch.from_numpy(alive).cuda()
        od = torch.empty((nq, k), device="cuda")
        oi = torch.empty((nq, k), dtype=torch.int64, device="cuda")
        s = torch.cuda.current_stream().cuda_stream
        c.search_device(tq.data_ptr(), nq, k, od.data_ptr(), oi.data_ptr(), id_offset=1000, alive_ptr=ta.data_ptr(), stream=s)
        torch.cuda.synchronize()
        assert c.last_variant()[0] == S.KERNEL_GEMM_B1
        assert np.array_equal(oi.cpu().numpy(), np.where(ih >= 0, ih + 1000, -1))
        assert np.array_equal(od.cpu().numpy().view(np.uint32), dh.view(np.uint32))
        c.close()
