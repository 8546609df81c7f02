"""Binary vector indexes (BINARYFLAT / BINARYIVF / BINARYHNSW / BINARYMSTG) on the GPU.

BINARYIVF lists hold the exact row bytes and every key is an integer expression below 2^24 (Jaccard: one IEEE division of two
such integers), so with every list probed the index must return the SAME BYTES as the exact binary corpus (ids, distances, the
smaller-id tie rule and the -1 / FLT_MAX tails), and at any nprobe every returned distance is exact."""
import os
import subprocess

import numpy as np
import pytest

import myscaledb_b200 as b2
import oracle as orc
from myscaledb_b200 import search as S

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_INVALID, ERR_UNSUPPORTED = 1, 3
NLIST = 16


def clustered(rng, n, nbytes, n_centres=24, flip=0.08, centres=None):
    """rows that flip each bit of a random centre with probability `flip`; plus exact duplicates and all-zero rows (ties)"""
    if centres is None:
        centres = rng.integers(0, 2, (n_centres, nbytes * 8), dtype=np.uint8)
    bits = centres[rng.integers(0, len(centres), n)] ^ (rng.random((n, nbytes * 8)) < flip).astype(np.uint8)
    y = np.packbits(bits, axis=1)
    y[rng.integers(0, n, n // 50)] = 0
    y[rng.integers(0, n, n // 20)] = y[rng.integers(0, n, n // 20)]
    return y, centres


def corpus_search(metric, y, x, k, alive=None):
    c = b2.Corpus(metric, y.shape[1] * 8, dtype=S.BIN).append(y)
    try:
        return c.search(x, k, alive_bits=alive)
    finally:
        c.close()


def same_bytes(a, b):
    return np.array_equal(a[1], b[1]) and np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32))


def exact_dist(metric, q, row):
    a, b = np.unpackbits(q).astype(np.int64), np.unpackbits(row).astype(np.int64)
    x_and, x_or = int((a & b).sum()), int((a | b).sum())
    if metric == b2.HAMMING:
        return np.float32(x_or - x_and)
    return np.float32(0.0) if x_or == 0 else np.float32(np.float32(x_or - x_and) / np.float32(x_or))


@pytest.mark.parametrize("metric", [b2.HAMMING, b2.JACCARD])
@pytest.mark.parametrize("nbits", [64, 200, 256, 1024, 1032, 2048])
def test_all_lists_probed_is_the_exact_corpus_answer(metric, nbits):
    rng = np.random.default_rng(nbits + metric)
    nb = nbits // 8
    n = 6000
    y, cen = clustered(rng, n, nb)
    ix = b2.VectorIndex("BINARYIVF", metric, nbits, f"ncentroids={NLIST}").build(y)
    assert ix.info()["uses_ivf"] and ix.info()["n"] == n
    xq, _ = clustered(rng, 1025, nb, centres=cen)
    xq[3] = 0
    xq[5] = y[17]
    alive = orc.pack_bits(rng.random(n) < 0.7)
    sparse = orc.pack_bits(np.arange(n) % 97 == 0)   # 62 rows alive: k = 100 and 1024 leave tails
    for nq in (1, 17, 129, 1025):
        x = xq[:nq]
        for k in (1, 10, 100, 1024):
            for a in (None, alive, sparse) if nq in (17, 1025) else (None,):
                got = ix.search(x, k, params=f"nprobe={NLIST}", alive_bits=a)
                ref = corpus_search(metric, y, x, k, a)
                assert same_bytes(got, ref), (nq, k, a is None)
                if nq == 17 and k in (10, 1024):
                    do, io = orc.knn_binary(metric, x, y, k, a)
                    assert np.array_equal(got[1], io)
                    assert np.array_equal(got[0], do)
    ix.close()


@pytest.mark.parametrize("metric", [b2.HAMMING, b2.JACCARD])
def test_every_returned_distance_is_exact_at_small_nprobe(metric):
    rng = np.random.default_rng(5)
    y, cen = clustered(rng, 8000, 40)
    x, _ = clustered(rng, 64, 40, centres=cen)
    ix = b2.VectorIndex("BINARYIVF", metric, 320, "ncentroids=32").build(y)
    dis, ids = ix.search(x, 20, params="nprobe=2")
    assert (ids >= 0).any()
    for q in range(len(x)):
        for j in range(20):
            if ids[q, j] >= 0:
                assert dis[q, j] == exact_dist(metric, x[q], y[ids[q, j]])
        keyed = [(dis[q, j], ids[q, j]) for j in range(20) if ids[q, j] >= 0]
        assert keyed == sorted(keyed)
    ix.close()


def test_recall_at_nprobe_4_on_clustered_data():
    rng = np.random.default_rng(9)
    y, cen = clustered(rng, 60000, 32, n_centres=200, flip=0.1)
    x, _ = clustered(rng, 200, 32, centres=cen)
    ix = b2.VectorIndex("BINARYIVF", b2.HAMMING, 256, "ncentroids=64").build(y)
    _, ids = ix.search(x, 10, params="nprobe=4")
    _, truth = corpus_search(b2.HAMMING, y, x, 10)
    recall = np.mean([len(set(ids[q]) & set(truth[q])) / 10 for q in range(len(x))])
    # the build is deterministic, so the value reproduces: 0.980 on an H100 (0.964 at nprobe 1, 0.9725 at 2)
    assert recall >= 0.95, recall
    ix.close()


@pytest.mark.parametrize("metric", [b2.HAMMING, b2.JACCARD])
def test_build_is_deterministic_and_streamed_build_equals_one_shot(metric):
    rng = np.random.default_rng(21)
    y, cen = clustered(rng, 7000, 16)
    x, _ = clustered(rng, 50, 16, centres=cen)
    a = b2.VectorIndex("BINARYIVF", metric, 128, f"ncentroids={NLIST}").build(y)
    b = b2.VectorIndex("BINARYIVF", metric, 128, f"ncentroids={NLIST}").build(y)
    s = b2.VectorIndex("BINARYIVF", metric, 128, f"ncentroids={NLIST}")
    s.reserve(len(y)).train(y)
    for lo in range(0, len(y), 2500):
        s.add(y[lo:lo + 2500])
    s.finalize()
    assert np.array_equal(a.list_sizes(), b.list_sizes()) and np.array_equal(a.list_sizes(), s.list_sizes())
    ra = a.search(x, 10, params="nprobe=3")
    assert same_bytes(ra, b.search(x, 10, params="nprobe=3")) and same_bytes(ra, s.search(x, 10, params="nprobe=3"))
    for i in (a, b, s):
        i.close()


@pytest.mark.parametrize("index_type", ["BINARYFLAT", "BINARYIVF"])
def test_save_load_roundtrip_and_corrupt_files(index_type, tmp_path):
    rng = np.random.default_rng(3)
    y, cen = clustered(rng, 5000, 25)
    x, _ = clustered(rng, 40, 25, centres=cen)
    ix = b2.VectorIndex(index_type, b2.JACCARD, 200, f"ncentroids={NLIST}").build(y)
    assert ix.info()["uses_ivf"] == (index_type == "BINARYIVF")
    before = ix.search(x, 10, params="nprobe=4")
    path = tmp_path / "b.idx"
    ix.save(path)
    ix.close()
    ld = b2.VectorIndex.load(path, 200, metric=b2.JACCARD)
    assert same_bytes(before, ld.search(x, 10, params="nprobe=4"))
    ld.close()
    raw = path.read_bytes()
    (tmp_path / "t.idx").write_bytes(raw[: len(raw) - 1000])
    with pytest.raises(b2.B200Error) as e:
        b2.VectorIndex.load(tmp_path / "t.idx", 200, metric=b2.JACCARD)
    assert e.value.code == ERR_INVALID
    bad = bytearray(raw)
    bad[12:16] = (1).to_bytes(4, "little")   # metric JACCARD -> IP on a binary type
    (tmp_path / "c.idx").write_bytes(bytes(bad))
    with pytest.raises(b2.B200Error) as e:
        b2.VectorIndex.load(tmp_path / "c.idx", 200, metric=b2.JACCARD)
    assert e.value.code == ERR_INVALID


def test_small_part_fallback_type_names_and_refused_requests():
    rng = np.random.default_rng(4)
    y, cen = clustered(rng, 1500, 32)
    x, _ = clustered(rng, 20, 32, centres=cen)
    small = b2.VectorIndex("BinaryIVF", b2.HAMMING, 256).build(y)
    assert not small.info()["uses_ivf"]
    assert same_bytes(small.search(x, 10), corpus_search(b2.HAMMING, y, x, 10))
    small.close()
    big, _ = clustered(rng, 6000, 32, centres=cen)
    for t in ("BINARYHNSW", "binarymstg"):
        ix = b2.VectorIndex(t, b2.JACCARD, 256, f"ncentroids={NLIST}").build(big)
        assert ix.info()["uses_ivf"]
        assert same_bytes(ix.search(x, 10, params=f"nprobe={NLIST}", first_stage_only=True), corpus_search(b2.JACCARD, big, x, 10))
        assert ix.last_num_candidates == 10
        with pytest.raises(b2.B200Error) as e:
            ix.refine(x, np.zeros((20, 5), np.int64), 3)
        assert e.value.code == ERR_UNSUPPORTED
        with pytest.raises(b2.B200Error) as e:
            ix.search(x, 10, params="exact_batch=1")
        assert e.value.code == ERR_UNSUPPORTED
        ix.close()
    for t, m, d in (("BINARYIVF", b2.L2, 256), ("IVFFLAT", b2.HAMMING, 256), ("BINARYFLAT", b2.IP, 256), ("FLAT", b2.JACCARD, 256),
                    ("BINARYIVF", b2.HAMMING, 100), ("BINARYFLAT", b2.JACCARD, 65544)):
        with pytest.raises(b2.B200Error) as e:
            b2.VectorIndex(t, m, d)
        assert e.value.code == ERR_INVALID, (t, m, d)
    many = b2.VectorIndex("BINARYIVF", b2.HAMMING, 256, "ncentroids=1100").build(np.concatenate([big, big]))
    with pytest.raises(b2.B200Error) as e:
        many.search(x, 10, params="nprobe=1050")
    assert e.value.code == ERR_UNSUPPORTED
    assert same_bytes(many.search(x, 10, params="nprobe=1100"), corpus_search(b2.HAMMING, np.concatenate([big, big]), x, 10))
    many.close()


def test_search_device_timing_memory_and_cache():
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(8)
    n, nq, k = 9000, 70, 12
    y, cen = clustered(rng, n, 48)
    x, _ = clustered(rng, nq, 48, centres=cen)
    alive = orc.pack_bits(rng.random(n) < 0.6)
    ix = b2.VectorIndex("BINARYIVF", b2.HAMMING, 384, "ncentroids=24").build(y)
    dh, ih = ix.search(x, k, params="nprobe=5", alive_bits=alive)
    tq, ta = torch.from_numpy(x).cuda(), torch.from_numpy(alive).cuda()
    od = torch.empty((nq, k), device="cuda")
    oi = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    ix.search_device(tq.data_ptr(), nq, k, od.data_ptr(), oi.data_ptr(), params="nprobe=5", id_offset=500, alive_ptr=ta.data_ptr(),
                     stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert np.array_equal(oi.cpu().numpy(), np.where(ih >= 0, ih + 500, -1))
    assert np.array_equal(od.cpu().numpy().view(np.uint32), dh.view(np.uint32))
    ix.enable_timing(True)
    ix.search(x, k, params="nprobe=5")
    scan = ix.last_scan(reset=True)
    assert scan["launches"] >= 1 and scan["kernel_ms"] > 0 and scan["rows_streamed"] > 0 and scan["payload_row_bytes"] == 48
    info = ix.info()
    pool_rows = (-(-n // 256) + info["nlist"]) * 256
    assert ix.memory_bytes() >= pool_rows * (48 + 4 + 4) + info["nlist"] * 48
    h = S.cache_put("binary-ivf/part0", ix)
    got, kind = S.cache_get("binary-ivf/part0")
    assert got == h and kind == S.CACHE_INDEX
    S.cache_release("binary-ivf/part0")
    S.cache_expire("binary-ivf/part0")


def test_binary_ivf_through_the_shim():
    exe = os.path.join(ROOT, "tests", "cpp", "binary_index_shim")
    if not os.path.exists(exe):
        pytest.skip("binary_index_shim not built (run __graft_entry__.build())")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "BINARY INDEX OK" in r.stdout, r.stdout + r.stderr
