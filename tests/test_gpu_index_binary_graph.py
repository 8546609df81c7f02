"""BINARYMSTG with a neighbour graph (graph_degree=D): the graph is built from the index's own (exact) list search and walked over
the binary list rows in HBM.  List rows are exact, so the walk's keys are exact integers (Hamming) or one IEEE division of two
integers (Jaccard): the graph equals the numpy reference, and the search equals the reference walk (tests/binary_graph_reference.py)
id for id and distance bit for bit on any data, ties (everywhere under Hamming) included.  Filters, persistence, sizes and
refusals are as documented."""
import numpy as np
import pytest

import myscaledb_b200 as b2
import oracle as orc
from myscaledb_b200.search import B200Error
from oracle import pack_bits
from tests import binary_graph_reference as BG
from tests import graph_reference as G
from tests.test_gpu_binary_index import corpus_search

pytestmark = pytest.mark.gpu
INVALID, UNSUPPORTED = 1, 3
HEADER_VERSION, HEADER_HAS_RAW, HEADER_RESERVED0 = 4, 44, 68   # byte offsets in the B2IX header
METRIC = {b2.HAMMING: BG.HAMMING, b2.JACCARD: BG.JACCARD}


def _bits(rng, n, nbits, centres, flip):
    """rows that flip each bit of a random centre with probability flip, packed; generated in blocks of <= 2^24 bits"""
    out = []
    step = max(1, (1 << 24) // nbits)
    for r0 in range(0, n, step):
        m = min(step, n - r0)
        out.append(np.packbits(centres[rng.integers(0, len(centres), m)] ^ (rng.random((m, nbits)) < flip).astype(np.uint8), axis=1))
    return np.concatenate(out)


def _data(nbits, n, seed, nq=8, n_centres=64, flip=0.08):
    rng = np.random.default_rng(seed)
    centres = rng.integers(0, 2, (n_centres, nbits), dtype=np.uint8)
    y = _bits(rng, n, nbits, centres, flip)
    y[rng.integers(0, n, max(1, n // 100))] = 0                        # all-zero rows: Jaccard's 0 / 0
    y[rng.integers(0, n, n // 20)] = y[rng.integers(0, n, n // 20)]    # duplicates: tied keys
    q = _bits(rng, nq, nbits, centres, flip)
    q[min(1, nq - 1)] = 0
    return y, q


def _index(metric, y, D, extra=""):
    return b2.VectorIndex("BINARYMSTG", metric, y.shape[1] * 8, f"graph_degree={D}" + extra).build(y)


def _check_graph(ix, y, D):
    _, ids = ix.search(y, 2 * D + 1, "graph=0")
    want = G.build(G.candidates(ids), D)
    got = ix.graph()
    assert got is not None and got.shape == (len(y), D)
    assert np.array_equal(got, want), f"{int((got != want).any(1).sum())} of {len(y)} graph rows differ from the reference"


def _row_pad(nbits):
    rb = nbits // 8
    kb = min(128, -(-rb // 16) * 16)
    return -(-rb // kb) * kb


# ---------------------------------------------------------------------------------------------------------------------------
# 1. the graph is the reference's
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nbits", [256, 200])
@pytest.mark.parametrize("D", [16, 32])
@pytest.mark.parametrize("metric", [b2.HAMMING, b2.JACCARD])
def test_graph_is_the_reference(metric, D, nbits):
    y, _ = _data(nbits, 10000, 1 + metric)
    ix = _index(metric, y, D, ",ncentroids=32")
    assert ix.info()["uses_ivf"]
    _check_graph(ix, y, D)
    ph = ix.phase_ms()
    assert ph["coarse"] > 0 and ph["plan"] > 0 and ph["scan"] > 0   # candidates | prune | merge


def test_graph_streamed_build_is_the_reference():
    y, _ = _data(200, 10000, 2)
    ix = b2.VectorIndex("BINARYMSTG", b2.JACCARD, 200, "graph_degree=16,ncentroids=32").reserve(len(y)).train(y[::3])
    for off in range(0, len(y), 3500):
        ix.add(y[off:off + 3500])
    ix.finalize()
    _check_graph(ix, y, 16)


# ---------------------------------------------------------------------------------------------------------------------------
# 2. the search is the reference walk, id for id and bit for bit; 3. every distance is BINARYFLAT's
# ---------------------------------------------------------------------------------------------------------------------------
WIDTHS = {64: (8000, 32), 200: (8000, 32), 1024: (8000, 32), 65536: (3000, 8)}
_cache = {}


def _built(metric, nbits):
    key = (metric, nbits)
    if key not in _cache:
        n, nl = WIDTHS[nbits]
        y, q = _data(nbits, n, 3 + nbits + metric)
        ix = _index(metric, y, 16, f",ncentroids={nl}")
        _cache[key] = (ix, y, q, ix.graph())
    return _cache[key]


@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("nbits", list(WIDTHS))
@pytest.mark.parametrize("metric", [b2.HAMMING, b2.JACCARD])
def test_search_is_the_reference(metric, nbits, filtered):
    ix, y, q, g = _built(metric, nbits)
    D, k = 16, 10
    alive = np.random.default_rng(5).random(len(y)) < 0.5 if filtered else None
    bits = pack_bits(alive) if filtered else None
    for ef in (16, 64, 1024):   # at 1024 the iteration cap (510 parents) stops the walk
        for first in (False, True):   # first_stage_only and refine_factor change nothing: the keys are exact
            dis, ids = ix.search(q, k, f"ef_s={ef}" + ("" if first else ",refine_factor=8"), first_stage_only=first, alive_bits=bits)
            assert ix.last_num_candidates == k
            seeds = ix.last_seeds()
            assert seeds is not None and seeds.shape == (len(q), min(max(ef, k), G.MAX_SEEDS))
            wd, wi, scored = BG.search(g, y, q, seeds, max(ef, k), k, G.iteration_cap(D), METRIC[metric], alive)
            assert np.array_equal(ids, wi), f"ef_s={ef}: ids differ from the reference"
            assert dis.tobytes() == wd.tobytes(), f"ef_s={ef}: distances differ from the reference"
            st = ix.last_scan()
            assert st["rows_streamed"] == int(scored.sum())
            assert st["payload_row_bytes"] == _row_pad(nbits) and st["work_items"] == len(q)
        # 3. exactness: each returned distance is the binary corpus' distance of that (query, id) ...
        got = ids >= 0
        for i in range(len(q)):
            want = BG.keys(y, q[i], ids[i][got[i]], METRIC[metric])
            assert dis[i][got[i]].tobytes() == want.tobytes()
        if filtered:
            assert alive[ids[got]].all()
    # ... and the oracle's for every id both return
    do, io = orc.knn_binary(metric, q, y, 50)
    dis, ids = ix.search(q, 10, "ef_s=64")
    for i in range(len(q)):
        ref = dict(zip(io[i].tolist(), do[i].tolist()))
        for j, v in enumerate(ids[i].tolist()):
            if v in ref:
                assert np.float32(ref[v]) == dis[i, j], (i, v)


@pytest.mark.parametrize("metric", [b2.HAMMING, b2.JACCARD])
def test_search_width_is_the_reference(metric):
    ix, y, q0, g = _built(metric, 200)
    rng = np.random.default_rng(6)
    near = np.unpackbits(y[rng.integers(0, len(y), 292)], axis=1) ^ (rng.random((292, y.shape[1] * 8)) < 0.05).astype(np.uint8)
    q = np.concatenate([q0, np.packbits(near, axis=1)])
    D, k, ef = 16, 10, 64
    base = None
    for W in (1, 2, 4, 8):
        for nq in (1, 300):
            dis, ids = ix.search(q[:nq], k, f"ef_s={ef},search_width={W}")
            wd, wi, scored = BG.search(g, y, q[:nq], ix.last_seeds(), ef, k, G.iteration_cap(D, W), METRIC[metric], None, W)
            assert np.array_equal(ids, wi) and dis.tobytes() == wd.tobytes(), (W, nq)
            st = ix.last_scan()
            assert st["rows_streamed"] == int(scored.sum()) and st["work_items"] == nq * W
        if W == 1:
            base = ix.search(q, k, f"ef_s={ef}")
            assert base[0].tobytes() == dis.tobytes() and base[1].tobytes() == ids.tobytes()


# ---------------------------------------------------------------------------------------------------------------------------
# 4. recall on clustered binary data
# ---------------------------------------------------------------------------------------------------------------------------
def _recall(dis, ids, td, k):
    """tie-aware recall@k: returned rows whose distance is within the k-th exact distance (Hamming ties are common)"""
    kth = td[:, k - 1:k]
    return float(((ids >= 0) & (dis <= kth)).sum()) / (len(ids) * k)


@pytest.mark.parametrize("metric", [b2.HAMMING, b2.JACCARD])
def test_recall_and_ef(metric):
    y, q = _data(256, 200000, 8, nq=1000, n_centres=1000, flip=0.1)
    ix = _index(metric, y, 32)
    td, _ = corpus_search(metric, y, q, 10)

    def rec(ef):
        dis, ids = ix.search(q, 10, f"ef_s={ef}")
        return _recall(dis, ids, td, 10)

    r32, r128, r256 = rec(32), rec(128), rec(256)
    print(f"binary graph recall@10 metric={metric}: ef_s 32 {r32:.4f}, 128 {r128:.4f}, 256 {r256:.4f}")
    assert r128 >= 0.95, f"recall@10 at ef_s=128: {r128:.4f}"
    assert r256 >= r32, (r32, r256)


# ---------------------------------------------------------------------------------------------------------------------------
# 5. filters
# ---------------------------------------------------------------------------------------------------------------------------
def _device_search(ix, q, k, params="", alive=None):
    import torch
    tq = torch.from_numpy(q).cuda()
    ta = torch.from_numpy(pack_bits(alive)).cuda() if alive is not None else None
    od = torch.empty((len(q), k), dtype=torch.float32, device="cuda")
    oi = torch.empty((len(q), k), dtype=torch.int64, device="cuda")
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    ix.search_device(tq.data_ptr(), len(q), k, od.data_ptr(), oi.data_ptr(), params, alive_ptr=ta.data_ptr() if ta is not None else 0,
                     stream=side.cuda_stream)
    side.synchronize()
    return od.cpu().numpy(), oi.cpu().numpy()


def test_filters():
    y, q = _data(256, 50000, 9, nq=64)
    n, k = len(y), 10
    rng = np.random.default_rng(10)
    ix = _index(b2.HAMMING, y, 32)
    alive = rng.random(n) < 0.5
    dis, ids = ix.search(q, k, "ef_s=128", alive_bits=pack_bits(alive))
    assert not ix.last_probe()[1]
    assert alive[ids[ids >= 0]].all() and (ids >= 0).all()
    # 1 %: the walk answers (no exact pass: the index keeps no exact corpus), kept ids only, possibly fewer than k
    alive = rng.random(n) < 0.01
    dis, ids = ix.search(q, 100, "prefilter=2", alive_bits=pack_bits(alive))
    assert not ix.last_probe()[1]
    assert ix.last_seeds() is not None
    assert alive[ids[ids >= 0]].all() and (ids >= 0).any()
    assert (dis[ids < 0] == np.finfo(np.float32).max).all()
    # graph=0 with every list probed is the exact complete answer
    nl = ix.info()["nlist"]
    ed, ei = ix.search(q, 100, f"graph=0,nprobe={nl}", alive_bits=pack_bits(alive))
    od, oi = orc.knn_binary(b2.HAMMING, q, y, 100, pack_bits(alive))
    assert np.array_equal(ei, oi) and ed.tobytes() == od.tobytes()
    # the device entry walks the graph: kept ids only, the host entry's answer
    hd, hi = ix.search(q, k, "", alive_bits=pack_bits(alive))
    dd, di = _device_search(ix, q, k, "", alive)
    assert alive[di[di >= 0]].all()
    assert dd.tobytes() == hd.tobytes() and di.tobytes() == hi.tobytes()


# ---------------------------------------------------------------------------------------------------------------------------
# 6. persistence and sizes
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", [b2.HAMMING, b2.JACCARD])
def test_persistence_and_sizes(tmp_path, metric):
    nbits = 200
    y, q = _data(nbits, 20000, 11 + metric, nq=32)
    n, D, k = len(y), 32, 10
    ix = _index(metric, y, D)
    path = tmp_path / "g.b2ix"
    ix.save(path)
    raw = bytearray(path.read_bytes())
    assert int.from_bytes(raw[HEADER_VERSION:HEADER_VERSION + 4], "little") == 4
    assert int.from_bytes(raw[HEADER_RESERVED0:HEADER_RESERVED0 + 4], "little") == D
    v2 = bytearray(raw[:len(raw) - n * D * 4])
    v2[HEADER_VERSION:HEADER_VERSION + 4] = (2).to_bytes(4, "little")
    v2[HEADER_RESERVED0:HEADER_RESERVED0 + 4] = (0).to_bytes(4, "little")
    (tmp_path / "plain.b2ix").write_bytes(bytes(v2))
    plain = b2.VectorIndex.load(tmp_path / "plain.b2ix", nbits, metric)
    loaded = b2.VectorIndex.load(path, nbits, metric)
    assert plain.graph() is None
    assert np.array_equal(loaded.graph(), ix.graph())
    for prm in ("graph=0", "graph=0,nprobe=7"):
        a, b, c = loaded.search(q, k, prm), plain.search(q, k, prm), ix.search(q, k, prm)
        assert a[0].tobytes() == b[0].tobytes() == c[0].tobytes() and a[1].tobytes() == b[1].tobytes() == c[1].tobytes(), prm
        assert loaded.last_seeds() is None
    for prm in ("ef_s=96", "ef_s=32,search_width=4"):
        a, b = ix.search(q, k, prm), loaded.search(q, k, prm)
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes(), prm
    assert loaded.memory_bytes() - plain.memory_bytes() == n * D * 4 + n * 4
    ix.search(q, k, "ef_s=1024")
    st = ix.last_scan()
    assert st["work_items"] == len(q) and st["payload_row_bytes"] == _row_pad(nbits)
    assert 0 < st["rows_streamed"] <= len(q) * (G.MAX_SEEDS + G.iteration_cap(D) * G.WIDTH * D)
    bad = bytearray(raw)
    bad[len(bad) - 4:] = n.to_bytes(4, "little")
    (tmp_path / "bad.b2ix").write_bytes(bytes(bad))
    with pytest.raises(B200Error) as e:
        b2.VectorIndex.load(tmp_path / "bad.b2ix", nbits, metric)
    assert e.value.code == INVALID
    # a v4 BINARYMSTG file claiming rows: its lists are the only copy of its rows, so no exact pass may ever read such rows
    with_rows = bytearray(raw)
    with_rows[HEADER_HAS_RAW:HEADER_HAS_RAW + 4] = (1).to_bytes(4, "little")
    (tmp_path / "rows.b2ix").write_bytes(bytes(with_rows))
    with pytest.raises(B200Error) as e:
        b2.VectorIndex.load(tmp_path / "rows.b2ix", nbits, metric)
    assert e.value.code == INVALID


# ---------------------------------------------------------------------------------------------------------------------------
# 7. refusals and edges
# ---------------------------------------------------------------------------------------------------------------------------
def test_refusals_and_small_part(tmp_path):
    with pytest.raises(B200Error) as e:
        b2.VectorIndex("BINARYMSTG", b2.HAMMING, 256, "graph_degree=24")
    assert e.value.code == INVALID
    for t in ("BINARYHNSW", "BINARYIVF"):
        with pytest.raises(B200Error) as e:
            b2.VectorIndex(t, b2.HAMMING, 256, "graph_degree=16")
        assert e.value.code == UNSUPPORTED
    for D in (16, 32, 64):
        b2.VectorIndex("BINARYMSTG", b2.JACCARD, 256, f"graph_degree={D}").close()
    y, q = _data(256, 20000, 12, nq=4)
    ix = _index(b2.HAMMING, y, 16, ",ncentroids=64")
    for prm, code in (("ef_s=2000", INVALID), ("search_width=3", INVALID), ("exact_batch=1", UNSUPPORTED)):
        with pytest.raises(B200Error) as e:
            ix.search(q, 10, prm)
        assert e.value.code == code, prm
    with pytest.raises(B200Error) as e:
        ix.search(q, 1025)
    assert e.value.code == UNSUPPORTED
    ix.search(q, 1024, "ef_s=16")   # k = 1024 walks (ef raised to k)
    # graph=0 answers byte for byte as the same index without a graph, whose file is a v2 file
    plain = b2.VectorIndex("BINARYMSTG", b2.HAMMING, 256, "ncentroids=64").build(y)
    assert plain.graph() is None
    for prm in ("nprobe=1", "nprobe=5", "nprobe=64"):
        a, b = ix.search(q, 20, "graph=0," + prm), plain.search(q, 20, prm)
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes(), prm
    plain.save(tmp_path / "p.b2ix")
    assert int.from_bytes((tmp_path / "p.b2ix").read_bytes()[HEADER_VERSION:HEADER_VERSION + 4], "little") == 2
    # below the inverted-file threshold: BINARYFLAT, no graph
    y, q = _data(256, 1000, 13)
    small = _index(b2.HAMMING, y, 16)
    assert not small.info()["uses_ivf"] and small.graph() is None
    small.search(q, 5)
    assert small.last_seeds() is None


def test_widest_rows_build_in_chunks_sized_by_their_bytes():
    """65 536-bit rows at nprobe=1: the build's query scratch is its chunk's row bytes (about 0.5 GB), where 4 bytes per bit
    for every row (84 GB here) would not fit on the card"""
    rng = np.random.default_rng(15)
    n, nbits, D = 320_000, 65536, 16
    y = rng.integers(0, 256, (n, nbits // 8), dtype=np.uint8)
    ix = _index(b2.HAMMING, y, D, ",nprobe=1,ncentroids=512")
    g = ix.graph()
    assert g is not None and g.shape == (n, D) and (g != G.NO_ID).any(1).mean() > 0.99
    dis, ids = ix.search(y[:4], 10, "ef_s=64")
    assert (ids[:, 0] == np.arange(4)).all() and (dis[:, 0] == 0).all()   # each query row finds itself at distance 0
    ix.close()


def test_sharded_world_one_is_the_plain_search():
    import torch
    from myscaledb_b200.sharding import Comm
    y, x = _data(256, 8000, 14, nq=7)
    ix = _index(b2.JACCARD, y, 16, ",ncentroids=32")
    comm = Comm(0, 1, Comm.unique_id())
    st = torch.cuda.Stream()
    q = torch.from_numpy(x).cuda()
    try:
        for prm in ("graph=0,nprobe=8", "graph=1,ef_s=64", "ef_s=32,search_width=2"):
            for nq, k, off in ((7, 5, 0), (7, 10, (1 << 32) + 3), (1, 7, 0)):
                outs = []
                for sharded in (True, False):
                    od = torch.empty((nq, k), dtype=torch.float32, device="cuda")
                    oi = torch.empty((nq, k), dtype=torch.int64, device="cuda")
                    torch.cuda.synchronize()
                    if sharded:
                        comm.sharded_index_search(ix, b2.JACCARD, q.data_ptr(), nq, k, prm, od.data_ptr(), oi.data_ptr(), off, st.cuda_stream)
                    else:
                        ix.search_device(q.data_ptr(), nq, k, od.data_ptr(), oi.data_ptr(), params=prm, id_offset=off, stream=st.cuda_stream)
                    st.synchronize()
                    outs.append((od.cpu().numpy().tobytes(), oi.cpu().numpy().tobytes()))
                assert outs[0] == outs[1], (prm, nq, k, off)
    finally:
        torch.cuda.synchronize()
        comm.close()
