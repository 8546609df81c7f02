"""Device memory the library holds (b200_device_bytes): every index type, a corpus, the per-thread scratch corpus and a BM25
index give all of it back when freed; a train that fails after its quantisers exist leaks nothing and a retrain builds the
same index as a fresh one; the count covers what an index reports as memory_bytes().

The count is the library's own (every device buffer it allocates), not cudaMemGetInfo, so these checks are exact on a shared
device.  Hybrid fusion keeps a per-device scratch for the whole process: the module allocates it before any baseline."""
import numpy as np
import pytest

import myscaledb_b200 as b2
import oracle as orc
from myscaledb_b200._lib import lib
from myscaledb_b200.search import B200Error, device_bytes
from tests.test_gpu_binary_index import clustered, corpus_search

pytestmark = pytest.mark.gpu
F32 = np.float32
ERR_UNSUPPORTED = 3
D = 64


@pytest.fixture(scope="module", autouse=True)
def _fusion_scratch():
    b2.hybrid_fusion_batch("rsf", [[(0, 0, 1, 0.5)]], [[(0, 0, 2, 1.0)]], 2)


def _clustered(n, d, n_centres, seed, spread=0.3, nq=64):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((n_centres, d)).astype(F32)
    y = centres[rng.integers(0, n_centres, n)] + spread * rng.standard_normal((n, d)).astype(F32)
    q = centres[rng.integers(0, n_centres, nq)] + spread * rng.standard_normal((nq, d)).astype(F32)
    return y.astype(F32), q.astype(F32)


def _recall(ids, truth):
    return np.mean([len(set(a.tolist()) & set(b.tolist())) / len(b) for a, b in zip(ids, truth)])


# every index type, with its second stage, graph, OPQ + anisotropic codebooks (IVFPQ under IP) and host rows (SCANN)
TYPES = [("FLAT", b2.L2, ""), ("IVFFLAT", b2.L2, "ncentroids=32"),
         ("IVFPQ", b2.IP, "ncentroids=32, M=16, opq=1, opq_iters=2, aq_threshold=0.2, refine_factor=4"),
         ("MSTG", b2.COSINE, "ncentroids=32, graph_degree=32"), ("IVFSQ", b2.L2, "ncentroids=32, refine_factor=4"),
         ("SCANN", b2.L2, "ncentroids=32, keep_raw=2"), ("HNSWFLAT", b2.IP, "ncentroids=32, graph_degree=32"),
         ("HNSWSQ", b2.L2, "ncentroids=32"), ("HNSWPQ", b2.L2, "ncentroids=32, M=16"),
         ("BINARYFLAT", b2.HAMMING, ""), ("BINARYIVF", b2.HAMMING, "ncentroids=32"), ("BINARYHNSW", b2.JACCARD, "ncentroids=32"),
         ("BINARYMSTG", b2.HAMMING, "ncentroids=32, graph_degree=32")]


@pytest.mark.parametrize("index_type,metric,params", TYPES, ids=[t[0] for t in TYPES])
def test_every_index_type_returns_its_memory(index_type, metric, params, tmp_path):
    if metric in (b2.HAMMING, b2.JACCARD):
        y, cen = clustered(np.random.default_rng(3), 4000, D // 8, n_centres=40)
        q, _ = clustered(np.random.default_rng(4), 16, D // 8, centres=cen)
    else:
        y, q = _clustered(4000, D, 40, 3, nq=16)
    base = device_bytes()
    ix = b2.VectorIndex(index_type, metric, D, params).build(y)
    assert device_bytes() - base >= ix.memory_bytes() > 0
    ix.search(q, 10)
    ix.save(tmp_path / "ix.bin")
    loaded = b2.VectorIndex.load(tmp_path / "ix.bin", D, metric)
    ix.close()
    loaded.search(q, 10)
    loaded.close()
    assert device_bytes() == base


def test_corpus_with_appends_and_a_prefiltered_search_returns_its_memory():
    y, q = _clustered(6000, D, 40, 5, nq=8)
    alive = np.zeros(len(y), bool)
    alive[::97] = True
    base = device_bytes()
    c = b2.Corpus(b2.L2, D).append(y[:2500]).append(y[2500:])
    c.search(q, 10)
    c.set_prefilter(2)
    c.search(q, 10, alive_bits=orc.pack_bits(alive))
    c.close()
    assert device_bytes() == base


def test_thread_release_returns_the_scratch_corpus():
    y, q = _clustered(3000, D, 40, 6, nq=8)
    assert lib().b200_thread_release() == 0
    base = device_bytes()
    b2.flat_knn(b2.L2, q, y, 10)
    assert device_bytes() > base
    assert lib().b200_thread_release() == 0
    assert device_bytes() == base


def test_bm25_returns_its_memory():
    rng = np.random.default_rng(7)
    words = [f"w{i}" for i in range(300)]
    base = device_bytes()
    ix = b2.BM25Index(1)
    for r in range(2000):
        ix.add_doc(r, [" ".join(rng.choice(words, size=12))])
    ix.commit()
    ix.search_batch(["w1 w2 w3", "w10 w200", "w7"], 10)
    ix.close()
    assert device_bytes() == base


def _ivfpq():
    y, q = _clustered(40000, 64, 300, 8)
    return "IVFPQ", y, q, b2.IP, 64, "ncentroids=64, M=32, opq=1, opq_iters=4", "nprobe=64", 0.6


def _ivfsq():
    y, q = _clustered(60000, 96, 500, 9)
    return "IVFSQ", y, q, b2.L2, 96, "ncentroids=64", "nprobe=64", 0.9


def _binaryivf():
    rng = np.random.default_rng(9)
    y, cen = clustered(rng, 60000, 32, n_centres=200, flip=0.1)
    q, _ = clustered(rng, 200, 32, centres=cen)
    return "BINARYIVF", y, q, b2.HAMMING, 256, "ncentroids=64", "nprobe=4", 0.95


@pytest.mark.parametrize("make", [_ivfpq, _ivfsq, _binaryivf], ids=["IVFPQ-opq", "IVFSQ", "BINARYIVF"])
def test_failed_train_leaks_nothing_and_a_retrain_builds_the_index(make):
    """reserve(2^32) makes the pool allocation refuse the train after the centroids, codebooks and rotation exist; the index
    stays untrained, so the caller may reserve again and retrain.  The float recall floors are those of test_gpu_index.py, the
    binary one that of test_gpu_binary_index.py (two builds need not match bit for bit: k-means sums with float atomics)."""
    kind, y, q, metric, d, params, search, floor = make()
    base = device_bytes()
    ix = b2.VectorIndex(kind, metric, d, params)
    ix.reserve(1 << 32)
    with pytest.raises(B200Error) as e:
        ix.train(y)
    assert e.value.code == ERR_UNSUPPORTED and "2^32 - 1 pool rows" in str(e.value)
    ix.reserve(len(y)).train(y).add(y).finalize()
    fresh = b2.VectorIndex(kind, metric, d, params).reserve(len(y)).train(y).add(y).finalize()
    assert ix.memory_bytes() == fresh.memory_bytes()
    fresh.close()
    _, ids = ix.search(q, 10, search)
    _, truth = corpus_search(metric, y, q, 10) if metric == b2.HAMMING else orc.search_without_index(metric, q, y, 10)
    assert _recall(ids, truth) >= floor
    ix.close()
    assert device_bytes() == base
