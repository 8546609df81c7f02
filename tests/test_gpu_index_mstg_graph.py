"""MSTG with a neighbour graph (graph_degree=D): the graph is built from the index's own list search's first stage and walked
over the bf16 list rows in HBM; with fp32 rows (in HBM or in host memory) the walk's best kc = min(1024, k x refine_factor)
rows are re-ranked exactly.  The graph equals the numpy reference, the search equals the reference walk plus an exact re-rank
id for id and bit for bit on integer data (bf16 holds small integers exactly, so every key is exact and ties are real),
distances are those of the bf16 / fp32 rows on float data, and placement, filters, persistence and refusals are as
documented."""
import numpy as np
import pytest

import myscaledb_b200 as b2
import oracle as orc
from myscaledb_b200.search import B200Error
from oracle import pack_bits
from tests import graph_reference as G
from tests import ivf_reference as R
from tests.util import check_topk, to_bf16_values

pytestmark = pytest.mark.gpu
F32 = np.float32
INVALID, UNSUPPORTED = 1, 3
HEADER_VERSION, HEADER_RESERVED0 = 4, 68   # byte offsets in the B2IX header
REFINE = 4                                 # MSTG's default refine_factor


def _clustered(n, d, seed, nq=64, n_centres=200, spread=0.3):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((n_centres, d)).astype(F32)
    y = centres[rng.integers(0, n_centres, n)] + spread * rng.standard_normal((n, d)).astype(F32)
    q = centres[rng.integers(0, n_centres, nq)] + spread * rng.standard_normal((nq, d)).astype(F32)
    return y.astype(F32), q.astype(F32)


def _integer(n, d, seed, nq=12):
    """small integers: bf16 holds them exactly and every distance is exact in fp32 in any summation order"""
    rng = np.random.default_rng(seed)
    centres = rng.integers(-6, 7, (100, d))
    y = centres[rng.integers(0, 100, n)] + rng.integers(-1, 2, (n, d))
    q = centres[rng.integers(0, 100, nq)] + rng.integers(-1, 2, (nq, d))
    return y.astype(F32), q.astype(F32)


def _metric_name(metric):
    return {b2.L2: "l2", b2.IP: "ip", b2.COSINE: "cosine"}[metric]


def _mstg(metric, y, D, extra=""):
    return b2.VectorIndex("MSTG", metric, y.shape[1], f"graph_degree={D}" + extra).build(y)


def _check_graph(ix, y, D):
    _, ids = ix.search(y, 2 * D + 1, "graph=0", first_stage_only=True)
    want = G.build(G.candidates(ids), D)
    got = ix.graph()
    assert got is not None and got.shape == (len(y), D)
    assert np.array_equal(got, want), f"{int((got != want).any(1).sum())} of {len(y)} graph rows differ from the reference"


@pytest.mark.parametrize("metric", [b2.L2, b2.IP])
@pytest.mark.parametrize("D", [16, 32])
def test_graph_is_the_reference(metric, D):
    y, _ = _clustered(20000, 64, 1)
    _check_graph(_mstg(metric, y, D), y, D)


def test_graph_streamed_build_is_the_reference():
    y, _ = _clustered(20000, 64, 2)
    ix = b2.VectorIndex("MSTG", b2.L2, 64, "graph_degree=16").reserve(len(y)).train(y[::3])
    for off in range(0, len(y), 7000):
        ix.add(y[off:off + 7000])
    ix.finalize()
    _check_graph(ix, y, 16)


def test_graph_with_host_rows_is_the_reference():
    y, _ = _clustered(20000, 64, 3)
    ix = _mstg(b2.L2, y, 16, ",keep_raw=2")
    assert ix.host_memory_bytes() > 0
    _check_graph(ix, y, 16)


@pytest.mark.parametrize("d", [100, 768])
@pytest.mark.parametrize("metric", [b2.L2, b2.IP])
@pytest.mark.parametrize("filtered", [False, True])
def test_search_is_the_reference(d, metric, filtered):
    y, q = _integer(8000, d, 4)
    D, k = 16, 10
    kc = k * REFINE
    ix = _mstg(metric, y, D)
    g = ix.graph()
    alive = np.random.default_rng(5).random(len(y)) < 0.5 if filtered else None
    bits = pack_bits(alive) if filtered else None
    for ef in (16, 64, 1024):   # at 1024 the iteration cap (510 parents) stops the walk
        dis, ids = ix.search(q, k, f"ef_s={ef}", alive_bits=bits)
        assert ix.last_num_candidates == kc
        seeds = ix.last_seeds()
        assert seeds is not None and seeds.shape == (len(q), min(max(ef, kc), G.MAX_SEEDS))
        _, wi, scored = G.search(g, y, q, seeds, max(ef, kc), kc, G.iteration_cap(D), _metric_name(metric), alive)
        rd, ri = R.rerank(y, q, wi, k, metric)
        assert np.array_equal(ids, ri), f"ef_s={ef}: ids differ from the reference"
        assert dis.tobytes() == rd.tobytes(), f"ef_s={ef}: distances differ from the reference"
        assert ix.last_scan()["rows_streamed"] == int(scored.sum())
        # the first stage alone: the walk's best k at ef = max(ef_s, k)
        dis, ids = ix.search(q, k, f"ef_s={ef}", first_stage_only=True, alive_bits=bits)
        assert ix.last_num_candidates == k
        fd, fi, scored = G.search(g, y, q, ix.last_seeds(), max(ef, k), k, G.iteration_cap(D), _metric_name(metric), alive)
        assert np.array_equal(ids, fi) and dis.tobytes() == fd.tobytes(), f"ef_s={ef}: first stage differs from the reference"
        assert ix.last_scan()["rows_streamed"] == int(scored.sum())


@pytest.mark.parametrize("metric", [b2.L2, b2.IP, b2.COSINE])
def test_float_distances_sorted_deterministic(metric):
    y, q = _clustered(20000, 768, 6)
    ix = _mstg(metric, y, 32)
    k = 10
    yy = y.astype(np.float64)
    qq = q.astype(np.float64)
    if metric == b2.COSINE:
        yy /= np.linalg.norm(yy, axis=1, keepdims=True)
        qq /= np.linalg.norm(qq, axis=1, keepdims=True)
    stored = to_bf16_values(yy.astype(F32)).astype(np.float64)   # the list rows (cosine: unit rows)

    def ref(rows, ids):
        r = rows[ids]
        if metric == b2.L2:
            return ((r - qq[:, None, :]) ** 2).sum(-1)
        ip = (r * qq[:, None, :]).sum(-1)
        return ip if metric == b2.IP else 1 - ip

    for first in (True, False):
        dis, ids = ix.search(q, k, "ef_s=64", first_stage_only=first)
        dis2, ids2 = ix.search(q, k, "ef_s=64", first_stage_only=first)
        assert dis.tobytes() == dis2.tobytes() and ids.tobytes() == ids2.tobytes(), "two identical calls differ"
        assert (ids >= 0).all()
        for i in range(len(q)):
            assert len(set(ids[i].tolist())) == k
        np.testing.assert_allclose(dis, ref(stored if first else yy, ids), rtol=1e-5, atol=2e-5 if metric != b2.L2 else 0)
        step = np.diff(dis, axis=1)
        assert (step <= 0).all() if metric == b2.IP else (step >= 0).all()
    assert ix.last_scan()["payload_row_bytes"] == 768 * 2


@pytest.mark.parametrize("metric", [b2.L2, b2.IP])
def test_k_1024_is_re_ranked(metric):
    """k x refine_factor capped at 1024 = k: the walk's rows are still re-ranked exactly (float data, where the bf16 keys differ
    from the fp32 ones, so a missing second stage shows in the distances).  A walk may stay inside its cluster and return
    fewer than 1024 rows: the tail is -1."""
    y, q = _clustered(20000, 64, 15, nq=8, n_centres=20)
    ix = _mstg(metric, y, 16)
    k = 1024
    qq = q.astype(np.float64)[:, None, :]

    def exact(ids):
        yy = y[np.maximum(ids, 0)].astype(np.float64)
        return ((yy - qq) ** 2).sum(-1) if metric == b2.L2 else (yy * qq).sum(-1)

    dis, ids = ix.search(q, k, "ef_s=64")
    assert ix.last_num_candidates == k
    got = ids >= 0
    assert (got.sum(1) >= 100).all() and (got[:, :-1] >= got[:, 1:]).all(), "returned rows first, then the -1 tail"
    np.testing.assert_allclose(dis[got], exact(ids)[got], rtol=1e-5, atol=0 if metric == b2.L2 else 2e-5)
    step = np.diff(dis, axis=1)
    assert (step <= 0).all() if metric == b2.IP else (step >= 0).all()
    # the walk's own (bf16) distances are not those: the check above would see a missing re-rank
    fd, fi = ix.search(q, k, "ef_s=64", first_stage_only=True)
    fg = fi >= 0
    assert not np.allclose(fd[fg], exact(fi)[fg], rtol=1e-5, atol=0)


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


def test_placement_moves_both_ways():
    y, q = _clustered(20000, 96, 7)
    n, D, k = len(y), 32, 10
    ix = _mstg(b2.L2, y, D)
    hbm = ix.memory_bytes()
    a = ix.search(q, k, "ef_s=64")
    ad = _device_search(ix, q, k, "ef_s=64")
    assert ad[0].tobytes() == a[0].tobytes() and ad[1].tobytes() == a[1].tobytes()
    ix.set_raw_placement(2)
    assert ix.host_memory_bytes() == n * 96 * 4
    assert hbm - ix.memory_bytes() >= n * 96 * 4
    for got in (ix.search(q, k, "ef_s=64"), _device_search(ix, q, k, "ef_s=64")):
        assert got[0].tobytes() == a[0].tobytes() and got[1].tobytes() == a[1].tobytes(), "host placement answers differ"
    assert ix.last_scan()["payload_row_bytes"] == 128 * 2
    ix.set_raw_placement(1)
    assert ix.host_memory_bytes() == 0
    b = ix.search(q, k, "ef_s=64")
    assert b[0].tobytes() == a[0].tobytes() and b[1].tobytes() == a[1].tobytes()
    # no fp32 rows: the build queries with the bf16 list rows, and answers carry first-stage distances, k candidates
    z = _mstg(b2.L2, y, D, ",keep_raw=0")
    _check_graph(z, to_bf16_values(y), D)
    dis, ids = z.search(q, k, "ef_s=64")
    assert z.last_num_candidates == k and (ids >= 0).all()
    ref = ((to_bf16_values(y)[ids].astype(np.float64) - q.astype(np.float64)[:, None, :]) ** 2).sum(-1)
    np.testing.assert_allclose(dis, ref, rtol=1e-5)


def test_recall_and_ef():
    y, q = _clustered(200000, 96, 8, nq=1000, n_centres=1000)
    ix = _mstg(b2.L2, y, 32, ",keep_raw=2")
    _, truth = orc.search_without_index(orc.L2, q, y, 10)

    def rec(ef):
        _, ids = ix.search(q, 10, f"ef_s={ef}")
        return np.mean([len(set(ids[i]) & set(truth[i])) / 10 for i in range(len(q))])

    r32, r128, r256 = rec(32), rec(128), rec(256)
    assert r128 >= 0.95, f"recall@10 at ef_s=128: {r128:.4f}"
    assert r256 >= r32, (r32, r256)


def test_filters():
    y, q = _clustered(50000, 64, 9)
    n, k = len(y), 10
    rng = np.random.default_rng(10)
    ix = _mstg(b2.L2, y, 32)
    alive = rng.random(n) < 0.5
    dis, ids = ix.search(q, k, "ef_s=128", alive_bits=pack_bits(alive))
    assert not ix.last_probe()[1]
    assert alive[ids[ids >= 0]].all()
    _, truth = orc.search_without_index(orc.L2, q, y, k, alive=pack_bits(alive))
    rec = np.mean([len(set(ids[i]) & set(truth[i])) / k for i in range(len(q))])
    assert rec >= 0.9, f"recall@10 under a 50 % filter: {rec:.4f}"
    # 1 % on the host entry: the exact rule answers over the HBM rows; with the rows in host memory the walk answers
    alive = rng.random(n) < 0.01
    dis, ids = ix.search(q, 100, "prefilter=2", alive_bits=pack_bits(alive))
    assert ix.last_probe()[1], "the exact rule did not answer a 1 % filter"
    do, io = orc.search_without_index(orc.L2, q, y, 100, alive=pack_bits(alive))
    check_topk(b2.L2, q, y, dis, ids, do, io)
    ix.set_raw_placement(2)
    dis, ids = ix.search(q, 100, "prefilter=2", alive_bits=pack_bits(alive))
    assert not ix.last_probe()[1]
    assert alive[ids[ids >= 0]].all() and (ids >= 0).any()
    # the device entry walks the graph: kept ids only
    dd, ii = _device_search(ix, q, k, "", alive)
    assert alive[ii[ii >= 0]].all()


@pytest.mark.parametrize("keep_raw", [1, 2])
def test_persistence_and_sizes(tmp_path, keep_raw):
    y, q = _clustered(20000, 64, 11)
    n, D, k = len(y), 32, 10
    ix = _mstg(b2.L2, y, D, f",keep_raw={keep_raw}")
    path = tmp_path / "g.b2ix"
    ix.save(path)
    raw = bytearray(path.read_bytes())
    assert int.from_bytes(raw[HEADER_VERSION:HEADER_VERSION + 4], "little") == 4
    assert int.from_bytes(raw[HEADER_RESERVED0:HEADER_RESERVED0 + 4], "little") == D
    v2 = bytearray(raw[:len(raw) - n * D * 4])
    v2[HEADER_VERSION:HEADER_VERSION + 4] = (2).to_bytes(4, "little")
    v2[HEADER_RESERVED0:HEADER_RESERVED0 + 4] = (0).to_bytes(4, "little")
    (tmp_path / "plain.b2ix").write_bytes(bytes(v2))
    plain = b2.VectorIndex.load(tmp_path / "plain.b2ix", 64, b2.L2)
    loaded = b2.VectorIndex.load(path, 64, b2.L2)
    assert plain.graph() is None
    assert np.array_equal(loaded.graph(), ix.graph())
    assert loaded.host_memory_bytes() == ix.host_memory_bytes()
    for prm in ("graph=0", "exact_batch=1") if keep_raw == 1 else ("graph=0",):
        a = loaded.search(q, k, prm)
        b = plain.search(q, k, prm)
        c = ix.search(q, k, prm)
        assert a[0].tobytes() == b[0].tobytes() == c[0].tobytes() and a[1].tobytes() == b[1].tobytes() == c[1].tobytes(), prm
        assert loaded.last_seeds() is None
    for first in (False, True):
        a, b = ix.search(q, k, "ef_s=96", first_stage_only=first), loaded.search(q, k, "ef_s=96", first_stage_only=first)
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
    assert loaded.memory_bytes() - plain.memory_bytes() == n * D * 4 + n * 4
    ix.search(q, k, "ef_s=1024")
    st = ix.last_scan()
    assert st["work_items"] == len(q) and st["payload_row_bytes"] == 64 * 2
    assert 0 < st["rows_streamed"] <= len(q) * (G.MAX_SEEDS + G.iteration_cap(D) * G.WIDTH * D)
    bad = bytearray(raw)
    bad[len(bad) - 4:] = n.to_bytes(4, "little")
    (tmp_path / "bad.b2ix").write_bytes(bytes(bad))
    with pytest.raises(B200Error) as e:
        b2.VectorIndex.load(tmp_path / "bad.b2ix", 64, b2.L2)
    assert e.value.code == INVALID


def test_refusals_and_small_part():
    with pytest.raises(B200Error) as e:
        b2.VectorIndex("MSTG", b2.L2, 32, "graph_degree=24")
    assert e.value.code == INVALID
    for prm in ("graph_degree=16,keep_raw=0", "graph_degree=16,keep_raw=1", "graph_degree=16,keep_raw=2", "graph_degree=64"):
        b2.VectorIndex("MSTG", b2.L2, 32, prm).close()
    y, q = _clustered(20000, 32, 12, nq=4)
    ix = _mstg(b2.L2, y, 16)
    with pytest.raises(B200Error) as e:
        ix.search(q, 10, "ef_s=2000")
    assert e.value.code == INVALID
    with pytest.raises(B200Error) as e:
        ix.search(q, 1025)
    assert e.value.code == UNSUPPORTED
    # below the inverted-file threshold: FLAT, no graph
    y, q = _clustered(1000, 32, 13)
    ix = _mstg(b2.L2, y, 16)
    assert not ix.info()["uses_ivf"] and ix.graph() is None
    ix.search(q, 5)
    assert ix.last_seeds() is None


def test_sharded_world_one_is_the_plain_search():
    import torch
    from myscaledb_b200.sharding import Comm
    y, x = _clustered(8000, 64, 14, nq=7)
    ix = _mstg(b2.L2, y, 16)
    comm = Comm(0, 1, Comm.unique_id())
    st = torch.cuda.Stream()
    q = torch.from_numpy(x).cuda()
    try:
        for prm in ("graph=0,nprobe=8", "graph=1,ef_s=64"):
            for nq, k, off in ((7, 5, 0), (7, 10, (1 << 32) + 3), (1, 7, 0)):
                outs = []
                for sharded in (True, False):
                    od = torch.empty((nq, k), dtype=torch.float32, device="cuda")
                    oi = torch.empty((nq, k), dtype=torch.int64, device="cuda")
                    torch.cuda.synchronize()
                    if sharded:
                        comm.sharded_index_search(ix, b2.L2, q.data_ptr(), nq, k, prm, od.data_ptr(), oi.data_ptr(), off, st.cuda_stream)
                    else:
                        ix.search_device(q.data_ptr(), nq, k, od.data_ptr(), oi.data_ptr(), params=prm, id_offset=off, stream=st.cuda_stream)
                    st.synchronize()
                    outs.append((od.cpu().numpy().tobytes(), oi.cpu().numpy().tobytes()))
                assert outs[0] == outs[1], (prm, nq, k, off)
    finally:
        torch.cuda.synchronize()
        comm.close()
