"""HNSWFLAT with a neighbour graph (graph_degree=D): the graph built at finalize equals the numpy reference built from the
index's own list search, the graph search equals the reference loop id for id and bit for bit on integer data (where ties are
everywhere, so the tie rule is pinned), distances are exact on float data, recall is high, filters keep their rows, and the
other paths, persistence, sizes and refusals are as documented."""
import numpy as np
import pytest

import myscaledb_b200 as b2
import oracle as orc
from myscaledb_b200.search import B200Error
from oracle import pack_bits
from tests import graph_reference as G
from tests.util import check_topk

pytestmark = pytest.mark.gpu
F32 = np.float32
INVALID, UNSUPPORTED = 1, 3
HEADER_VERSION, HEADER_RESERVED0 = 4, 68   # byte offsets in the B2IX header


def _clustered(n, d, seed, nq=256, n_centres=200, spread=0.3):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((n_centres, d)).astype(F32)
    y = centres[rng.integers(0, n_centres, n)] + spread * rng.standard_normal((n, d)).astype(F32)
    q = centres[rng.integers(0, n_centres, nq)] + spread * rng.standard_normal((nq, d)).astype(F32)
    return y.astype(F32), q.astype(F32)


def _integer(n, d, seed, nq=24):
    """small integers: every distance is exact in fp32 in any summation order"""
    rng = np.random.default_rng(seed)
    centres = rng.integers(-6, 7, (100, d))
    y = centres[rng.integers(0, 100, n)] + rng.integers(-1, 2, (n, d))
    q = centres[rng.integers(0, 100, nq)] + rng.integers(-1, 2, (nq, d))
    return y.astype(F32), q.astype(F32)


def _metric_name(metric):
    return {b2.L2: "l2", b2.IP: "ip", b2.COSINE: "cosine"}[metric]


def _graph_index(metric, y, D, extra=""):
    return b2.VectorIndex("HNSWFLAT", metric, y.shape[1], f"graph_degree={D}" + extra).build(y)


def _check_graph(ix, y, D):
    _, ids = ix.search(y, 2 * D + 1, "graph=0")
    want = G.build(G.candidates(ids), D)
    got = ix.graph()
    assert got is not None and got.shape == (len(y), D)
    assert np.array_equal(got, want), f"{int((got != want).any(1).sum())} of {len(y)} graph rows differ from the reference"


@pytest.mark.parametrize("metric", [b2.L2, b2.IP])
@pytest.mark.parametrize("D", [16, 32])
def test_graph_is_the_reference(metric, D):
    y, _ = _clustered(20000, 64, 1)
    _check_graph(_graph_index(metric, y, D), y, D)


def test_graph_streamed_build_is_the_reference():
    y, _ = _clustered(20000, 64, 2)
    ix = b2.VectorIndex("HNSWFLAT", b2.L2, 64, "graph_degree=16").reserve(len(y)).train(y[::3])
    for off in range(0, len(y), 7000):
        ix.add(y[off:off + 7000])
    ix.finalize()
    _check_graph(ix, y, 16)


def test_graph_structure_cosine():
    y, _ = _clustered(20000, 64, 3)
    D = 32
    g = _graph_index(b2.COSINE, y, D).graph()
    n = len(y)
    for a in range(0, n, 97):
        row = g[a]
        valid = row[row != G.NO_ID]
        assert (row[len(valid):] == G.NO_ID).all(), "padding only at the tail"
        assert (valid < n).all() and len(set(valid.tolist())) == len(valid) and a not in valid
    assert ((g != G.NO_ID).sum(1) >= D // 2).mean() > 0.99


@pytest.mark.parametrize("metric", [b2.L2, b2.IP])
@pytest.mark.parametrize("filtered", [False, True])
def test_search_is_the_reference(metric, filtered):
    y, q = _integer(20000, 32, 4)
    D, k = 16, 10
    ix = _graph_index(metric, y, D)
    g = ix.graph()
    alive = np.random.default_rng(5).random(len(y)) < 0.5 if filtered else None
    for ef in (16, 64, 1024):   # 16 is raised to k; at 1024 the iteration cap (510 parents) stops the walk
        dis, ids = ix.search(q, k, f"ef_s={ef}", alive_bits=pack_bits(alive) if filtered else None)
        seeds = ix.last_seeds()
        assert seeds is not None and seeds.shape == (len(q), min(max(ef, k), G.MAX_SEEDS))
        rd, ri, scored = G.search(g, y, q, seeds, max(ef, k), k, G.iteration_cap(D), _metric_name(metric), alive)
        assert np.array_equal(ids, ri), f"ef_s={ef}: ids differ from the reference"
        assert dis.tobytes() == rd.tobytes(), f"ef_s={ef}: distances differ from the reference"
        assert ix.last_scan()["rows_streamed"] == int(scored.sum())
        assert ix.last_num_candidates == k


@pytest.mark.parametrize("metric", [b2.L2, b2.IP, b2.COSINE])
def test_distances_exact_sorted_deterministic(metric):
    y, q = _clustered(20000, 64, 6)
    ix = _graph_index(metric, y, 32)
    k = 20
    dis, ids = ix.search(q, k, "ef_s=64")
    dis2, ids2 = ix.search(q, k, "ef_s=64")
    assert dis.tobytes() == dis2.tobytes() and ids.tobytes() == ids2.tobytes(), "two identical calls differ"
    assert (ids >= 0).all()
    for i in range(len(q)):
        assert len(set(ids[i].tolist())) == k
    yy = y[ids].astype(np.float64)
    qq = q.astype(np.float64)[:, None, :]
    if metric == b2.L2:
        ref = ((yy - qq) ** 2).sum(-1)
    elif metric == b2.IP:
        ref = (yy * qq).sum(-1)
    else:
        ref = 1 - (yy * qq).sum(-1) / (np.linalg.norm(yy, axis=-1) * np.linalg.norm(qq, axis=-1))
    np.testing.assert_allclose(dis, ref, rtol=1e-5, atol=2e-5 if metric != b2.L2 else 0)
    step = np.diff(dis, axis=1)
    assert (step <= 0).all() if metric == b2.IP else (step >= 0).all()


def test_recall_and_ef():
    y, q = _clustered(200000, 96, 7, nq=1000, n_centres=1000)
    ix = _graph_index(b2.L2, y, 32)
    _, truth = orc.search_without_index(orc.L2, q, y, 10)

    def rec(ef):
        _, ids = ix.search(q, 10, f"ef_s={ef}")
        return np.mean([len(set(ids[i]) & set(truth[i])) / 10 for i in range(len(q))])

    r32, r128, r256 = rec(32), rec(128), rec(256)
    assert r128 >= 0.95, f"recall@10 at ef_s=128: {r128:.4f}"
    assert r256 >= r32, (r32, r256)


def test_filters():
    y, q = _clustered(50000, 64, 8)
    n, k = len(y), 10
    ix = _graph_index(b2.L2, y, 32)
    rng = np.random.default_rng(9)
    # 50 %: every id kept, recall against the filtered exact answer
    alive = rng.random(n) < 0.5
    dis, ids = ix.search(q, k, "ef_s=128", alive_bits=pack_bits(alive))
    assert not ix.last_probe()[1]
    assert alive[ids[ids >= 0]].all()
    _, truth = orc.search_without_index(orc.L2, q, y, k, alive=pack_bits(alive))
    rec = np.mean([len(set(ids[i]) & set(truth[i])) / k for i in range(len(q))])
    assert rec >= 0.9, f"recall@10 under a 50 % filter: {rec:.4f}"
    # 1 % through the host entry at k = 100: kept share x rows at the cap (32 + 255 x 32) < 2k, and the gathered exact pass
    # takes the kept rows (prefilter=2: up to n / 8 of them), so it answers
    alive = rng.random(n) < 0.01
    dis, ids = ix.search(q, 100, "prefilter=2", alive_bits=pack_bits(alive))
    assert ix.last_probe()[1], "the exact rule did not answer a 1 % filter"
    do, io = orc.search_without_index(orc.L2, q, y, 100, alive=pack_bits(alive))
    check_topk(b2.L2, q, y, dis, ids, do, io)
    # the device entry always walks the graph: kept ids, exact distances, short answers allowed
    import torch
    tq = torch.from_numpy(q).cuda()
    ta = torch.from_numpy(pack_bits(alive)).cuda()
    od = torch.empty((len(q), k), dtype=torch.float32, device="cuda")
    oi = torch.empty((len(q), k), dtype=torch.int64, device="cuda")
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    ix.search_device(tq.data_ptr(), len(q), k, od.data_ptr(), oi.data_ptr(), "", alive_ptr=ta.data_ptr(), stream=side.cuda_stream)
    side.synchronize()
    dd, ii = od.cpu().numpy(), oi.cpu().numpy()
    got = ii >= 0
    assert alive[ii[got]].all()
    ref = ((y[np.where(got, ii, 0)].astype(np.float64) - q.astype(np.float64)[:, None, :]) ** 2).sum(-1)
    np.testing.assert_allclose(dd[got], ref[got], rtol=1e-5)


def test_paths_persistence_and_sizes(tmp_path):
    y, q = _clustered(20000, 64, 10)
    n, D, k = len(y), 32, 10
    ix = _graph_index(b2.L2, y, D)
    path = tmp_path / "g.b2ix"
    ix.save(path)
    raw = bytearray(path.read_bytes())
    assert int.from_bytes(raw[HEADER_VERSION:HEADER_VERSION + 4], "little") == 4
    assert int.from_bytes(raw[HEADER_RESERVED0:HEADER_RESERVED0 + 4], "little") == D
    # the same index without the key: the v2 file the index was before its graph
    v2 = bytearray(raw[:len(raw) - n * D * 4])
    v2[HEADER_VERSION:HEADER_VERSION + 4] = (2).to_bytes(4, "little")
    v2[HEADER_RESERVED0:HEADER_RESERVED0 + 4] = (0).to_bytes(4, "little")
    (tmp_path / "plain.b2ix").write_bytes(bytes(v2))
    plain = b2.VectorIndex.load(tmp_path / "plain.b2ix", 64, b2.L2)
    loaded = b2.VectorIndex.load(path, 64, b2.L2)
    assert plain.graph() is None
    assert np.array_equal(loaded.graph(), ix.graph())
    for prm in ("graph=0", "exact_batch=1"):
        a = loaded.search(q, k, prm)
        b = plain.search(q, k, prm)
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes(), prm
        assert loaded.last_seeds() is None
    a, b = ix.search(q, k, "ef_s=96"), loaded.search(q, k, "ef_s=96")
    assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
    assert loaded.memory_bytes() - plain.memory_bytes() == n * D * 4
    # rows scored per query stay within the seeds and the iteration cap
    ix.search(q, k, "ef_s=1024")
    st = ix.last_scan()
    assert st["work_items"] == len(q) and st["payload_row_bytes"] == 64 * 4
    assert 0 < st["rows_streamed"] <= len(q) * (G.MAX_SEEDS + G.iteration_cap(D) * G.WIDTH * D)
    # a graph id >= n is refused at load
    bad = bytearray(raw)
    bad[len(bad) - 4:] = n.to_bytes(4, "little")
    (tmp_path / "bad.b2ix").write_bytes(bytes(bad))
    with pytest.raises(B200Error) as e:
        b2.VectorIndex.load(tmp_path / "bad.b2ix", 64, b2.L2)
    assert e.value.code == INVALID
    # the graph needs the HBM rows
    with pytest.raises(B200Error) as e:
        ix.set_raw_placement(2)
    assert e.value.code == UNSUPPORTED
    for prm in ("ef_s=2000",):
        with pytest.raises(B200Error):
            ix.search(q, k, prm)


def test_refusals_and_small_part():
    for t, metric, d in (("IVFFLAT", b2.L2, 32), ("HNSWSQ", b2.L2, 32), ("HNSWPQ", b2.L2, 32), ("BINARYHNSW", b2.HAMMING, 64)):
        with pytest.raises(B200Error) as e:
            b2.VectorIndex(t, metric, d, "graph_degree=32")
        assert e.value.code == UNSUPPORTED, t
    for prm in ("graph_degree=32,keep_raw=0", "graph_degree=32,keep_raw=2"):
        with pytest.raises(B200Error) as e:
            b2.VectorIndex("HNSWFLAT", b2.L2, 32, prm)
        assert e.value.code == UNSUPPORTED, prm
    with pytest.raises(B200Error) as e:
        b2.VectorIndex("HNSWFLAT", b2.L2, 32, "graph_degree=24")
    assert e.value.code == INVALID
    # below the inverted-file threshold: FLAT, no graph
    y, q = _clustered(1000, 32, 11)
    ix = _graph_index(b2.L2, y, 16)
    assert not ix.info()["uses_ivf"] and ix.graph() is None
    ix.search(q, 5)
    assert ix.last_seeds() is None
