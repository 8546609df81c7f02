"""Graph search on a thread-block cluster per query (search_width=W): the W CTAs of a cluster expand the first W unexpanded
entries of the list per iteration, one parent each.  W = 1 is the default and today's walk byte for byte; at W = 2 / 4 / 8 the
HNSWFLAT and MSTG walks equal the reference loop with width=W (graph_reference.search) id for id and bit for bit on integer
data, at nq = 1 and at more clusters than are resident at once, through the host and device entries, the sharded search and
a saved index; on float data they are deterministic, exact and as good as W = 1; an unknown W is refused where the walk
runs and ignored where it does not."""
import numpy as np
import pytest

import myscaledb_b200 as b2
import oracle as orc
from myscaledb_b200.search import B200Error
from oracle import pack_bits
from tests import graph_reference as G
from tests import ivf_reference as R
from tests.util import to_bf16_values

pytestmark = pytest.mark.gpu
F32 = np.float32
INVALID, UNSUPPORTED = 1, 3
REFINE = 4                  # MSTG's default refine_factor
SMEM_OPTIN = 232448         # bytes of shared memory a block may use (227 KB)


def _clustered(n, d, seed, nq=64, n_centres=200, spread=0.3):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((n_centres, d)).astype(F32)
    y = centres[rng.integers(0, n_centres, n)] + spread * rng.standard_normal((n, d)).astype(F32)
    q = centres[rng.integers(0, n_centres, nq)] + spread * rng.standard_normal((nq, d)).astype(F32)
    return y.astype(F32), q.astype(F32)


def _integer(n, d, seed, nq=8):
    """small integers (the generator of the graph tests): bf16 holds them exactly and every distance is exact in fp32 in any
    summation order"""
    rng = np.random.default_rng(seed)
    centres = rng.integers(-6, 7, (100, d))
    y = centres[rng.integers(0, 100, n)] + rng.integers(-1, 2, (n, d))
    q = centres[rng.integers(0, 100, nq)] + rng.integers(-1, 2, (nq, d))
    return y.astype(F32), q.astype(F32)


def _metric_name(metric):
    return {b2.L2: "l2", b2.IP: "ip", b2.COSINE: "cosine"}[metric]


def _same(a, b):
    return a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()


def _smem(q_len, ef, k, filtered, w):
    """bytes of shared memory of one CTA of the walk (graph_smem_layout in csrc/graph_sm90.cu)"""
    lists = 4 * ef * 4 + 2 * ef
    step = 4 * 64 * w * 4 + 64 * 4 + (2 * 64 * 4 if w > 1 else 0)
    alive = 4 * k * 4 if filtered else 0
    return -(-(q_len * 4 + G.VISITED_SLOTS * 4 + lists + step + alive + 32 * 4) // 16) * 16


def _hnsw_check(ix, g, y, q, D, W, metric, alive, ef, k=10):
    bits = pack_bits(alive) if alive is not None else None
    dis, ids = ix.search(q, k, f"ef_s={ef}, search_width={W}", alive_bits=bits)
    seeds = ix.last_seeds()
    rd, ri, scored = G.search(g, y, q, seeds, max(ef, k), k, G.iteration_cap(D, W), _metric_name(metric), alive, width=W)
    assert np.array_equal(ids, ri), f"D={D} W={W} ef_s={ef}: ids differ from the reference"
    assert dis.tobytes() == rd.tobytes(), f"D={D} W={W} ef_s={ef}: distances differ from the reference"
    st = ix.last_scan()
    assert st["rows_streamed"] == int(scored.sum())
    assert st["work_items"] == len(q) * W
    return dis, ids


def _mstg_check(ix, y, q, D, W, metric, alive, ef, k=10):
    """the walk over the bf16 rows at kc = k x refine_factor, re-ranked exactly; then the first stage alone"""
    bits = pack_bits(alive) if alive is not None else None
    g, rows = ix.graph(), to_bf16_values(y)
    kc = k * REFINE
    dis, ids = ix.search(q, k, f"ef_s={ef}, search_width={W}", alive_bits=bits)
    assert ix.last_num_candidates == kc
    _, wi, scored = G.search(g, rows, q, ix.last_seeds(), max(ef, kc), kc, G.iteration_cap(D, W), _metric_name(metric), alive, width=W)
    rd, ri = R.rerank(y, q, wi, k, metric)
    assert np.array_equal(ids, ri), f"W={W} ef_s={ef}: ids differ from the reference"
    assert dis.tobytes() == rd.tobytes(), f"W={W} ef_s={ef}: distances differ from the reference"
    assert ix.last_scan()["rows_streamed"] == int(scored.sum())
    assert ix.last_scan()["work_items"] == len(q) * W
    dis, ids = ix.search(q, k, f"ef_s={ef}, search_width={W}", first_stage_only=True, alive_bits=bits)
    fd, fi, scored = G.search(g, rows, q, ix.last_seeds(), max(ef, k), k, G.iteration_cap(D, W), _metric_name(metric), alive, width=W)
    assert np.array_equal(ids, fi) and dis.tobytes() == fd.tobytes(), f"W={W} ef_s={ef}: first stage differs from the reference"
    assert ix.last_scan()["rows_streamed"] == int(scored.sum())


# ---------------------------------------------------------------------------------------------------------------------------
# 1. W = 1 is the default
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("typ", ["HNSWFLAT", "MSTG"])
def test_width_1_is_the_default(typ):
    y, q = _clustered(20000, 64, 20, nq=32)
    ix = b2.VectorIndex(typ, b2.L2, 64, "graph_degree=32").build(y)
    alive = np.random.default_rng(21).random(len(y)) < 0.5
    for bits in (None, pack_bits(alive)):
        for ef in (32, 256):
            a = ix.search(q, 10, f"ef_s={ef}", alive_bits=bits)
            rows = ix.last_scan()["rows_streamed"]
            b = ix.search(q, 10, f"ef_s={ef}, search_width=1", alive_bits=bits)
            assert _same(a, b), f"{typ} ef_s={ef}: search_width=1 differs from no key"
            st = ix.last_scan()
            assert st["rows_streamed"] == rows and st["work_items"] == len(q)


# ---------------------------------------------------------------------------------------------------------------------------
# 2. HNSWFLAT equals the reference
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hnsw_integer():
    y, q = _integer(20000, 32, 4)
    return y, q, {}


def _hnsw_index(data, metric, D):
    y, _, cache = data
    if (metric, D) not in cache:
        cache[(metric, D)] = b2.VectorIndex("HNSWFLAT", metric, 32, f"graph_degree={D}").build(y)
    return cache[(metric, D)]


@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("metric", [b2.L2, b2.IP])
@pytest.mark.parametrize("W", [2, 4, 8])
@pytest.mark.parametrize("D", [16, 32])
def test_hnswflat_is_the_reference(hnsw_integer, D, W, metric, filtered):
    y, q, _ = hnsw_integer
    ix = _hnsw_index(hnsw_integer, metric, D)
    g = ix.graph()
    alive = np.random.default_rng(5).random(len(y)) < 0.5 if filtered else None
    for ef in (16, 64, 1024):   # 16 is raised to k; at 1024 the iteration cap stops the walk
        _hnsw_check(ix, g, y, q, D, W, metric, alive, ef)


def test_hnswflat_degree_64_width_8_stops_at_the_cap():
    y, q = _integer(20000, 32, 22)
    D, W = 64, 8
    assert G.iteration_cap(D, W) == 15
    ix = b2.VectorIndex("HNSWFLAT", b2.L2, 32, f"graph_degree={D}").build(y)
    g = ix.graph()
    alive = np.random.default_rng(23).random(len(y)) < 0.5
    for a in (None, alive):
        _hnsw_check(ix, g, y, q, D, W, b2.L2, a, 1024)
        assert ix.last_scan()["rows_streamed"] <= len(q) * (G.MAX_SEEDS + 15 * W * D)


# ---------------------------------------------------------------------------------------------------------------------------
# 3. MSTG equals the reference
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("keep_raw", [1, 2])
@pytest.mark.parametrize("W", [2, 8])
@pytest.mark.parametrize("d", [100, 768])
def test_mstg_is_the_reference(d, W, keep_raw):
    y, q = _integer(8000, d, 24)
    D = 16
    metric = (b2.L2, b2.IP)[(d + W + keep_raw) % 2]
    ix = b2.VectorIndex("MSTG", metric, d, f"graph_degree={D}, keep_raw={keep_raw}").build(y)
    alive = np.random.default_rng(25).random(len(y)) < 0.5
    for a in (None, alive):
        for ef in (16, 64):
            _mstg_check(ix, y, q, D, W, metric, a, ef)


# ---------------------------------------------------------------------------------------------------------------------------
# 4. batch shapes: one query, and more clusters than are resident at once
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nq", [1, 300])
def test_batch_shapes(nq):
    y, q = _integer(20000, 32, 26, nq=nq)
    D = 32
    ix = b2.VectorIndex("HNSWFLAT", b2.L2, 32, f"graph_degree={D}").build(y)
    g = ix.graph()
    for W in (2, 8):
        _hnsw_check(ix, g, y, q, D, W, b2.L2, None, 32)
    y, q = _integer(8000, 100, 27, nq=nq)
    ms = b2.VectorIndex("MSTG", b2.L2, 100, "graph_degree=16").build(y)
    _mstg_check(ms, y, q, 16, 4, b2.L2, None, 32)


# ---------------------------------------------------------------------------------------------------------------------------
# 5. float data: deterministic, exact, sorted, and recall as W = 1's
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("typ", ["HNSWFLAT", "MSTG"])
@pytest.mark.parametrize("metric", [b2.L2, b2.IP, b2.COSINE])
def test_float_data(typ, metric):
    y, q = _clustered(20000, 768, 28, nq=128)
    ix = b2.VectorIndex(typ, metric, 768, "graph_degree=32").build(y)
    k = 10
    yy, qq = y.astype(np.float64), q.astype(np.float64)
    if metric == b2.COSINE:
        yy /= np.linalg.norm(yy, axis=1, keepdims=True)
        qq /= np.linalg.norm(qq, axis=1, keepdims=True)
    orc_metric = {b2.L2: orc.L2, b2.IP: orc.IP, b2.COSINE: orc.COSINE}[metric]
    _, truth = orc.search_without_index(orc_metric, q, y, k)

    def recall(ids):
        return np.mean([len(set(ids[i]) & set(truth[i])) / k for i in range(len(q))])

    r1 = recall(ix.search(q, k, "ef_s=64")[1])
    for W in (2, 8):
        dis, ids = ix.search(q, k, f"ef_s=64, search_width={W}")
        again = ix.search(q, k, f"ef_s=64, search_width={W}")
        assert _same((dis, ids), again), f"W={W}: two identical calls differ"
        assert (ids >= 0).all()
        for i in range(len(q)):
            assert len(set(ids[i].tolist())) == k
        r = yy[ids]   # HNSWFLAT and MSTG's re-rank: the fp32 rows (cosine: unit rows)
        ref = ((r - qq[:, None, :]) ** 2).sum(-1) if metric == b2.L2 else (r * qq[:, None, :]).sum(-1)
        if metric == b2.COSINE:
            ref = 1 - ref
        np.testing.assert_allclose(dis, ref, rtol=1e-5, atol=2e-5 if metric != b2.L2 else 0)
        step = np.diff(dis, axis=1)
        assert (step <= 0).all() if metric == b2.IP else (step >= 0).all()
        rw = recall(ids)
        assert rw >= r1 - 0.01, f"{typ} W={W}: recall@10 {rw:.4f} against {r1:.4f} at W = 1"


# ---------------------------------------------------------------------------------------------------------------------------
# 6. entries and persistence
# ---------------------------------------------------------------------------------------------------------------------------
def test_device_entry_sharded_and_persistence(tmp_path):
    import torch
    from myscaledb_b200.sharding import Comm
    y, q = _clustered(20000, 64, 29, nq=48)
    k, prm = 10, "ef_s=96, search_width=4"
    alive = np.random.default_rng(30).random(len(y)) < 0.5
    ix = b2.VectorIndex("HNSWFLAT", b2.L2, 64, "graph_degree=32").build(y)
    host = ix.search(q, k, prm, alive_bits=pack_bits(alive))
    tq = torch.from_numpy(q).cuda()
    ta = torch.from_numpy(pack_bits(alive)).cuda()
    od = torch.empty((len(q), k), dtype=torch.float32, device="cuda")
    oi = torch.empty((len(q), k), dtype=torch.int64, device="cuda")
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    ix.search_device(tq.data_ptr(), len(q), k, od.data_ptr(), oi.data_ptr(), prm, alive_ptr=ta.data_ptr(), stream=side.cuda_stream)
    side.synchronize()
    assert _same(host, (od.cpu().numpy(), oi.cpu().numpy())), "the device entry differs from the host entry"
    comm = Comm(0, 1, Comm.unique_id())
    try:
        od.fill_(0)
        oi.fill_(0)
        torch.cuda.synchronize()
        comm.sharded_index_search(ix, b2.L2, tq.data_ptr(), len(q), k, prm, od.data_ptr(), oi.data_ptr(), 0, side.cuda_stream, alive_ptr=ta.data_ptr())
        side.synchronize()
        assert _same(host, (od.cpu().numpy(), oi.cpu().numpy())), "the sharded search differs from the host entry"
    finally:
        comm.close()
    path = tmp_path / "g.b2ix"
    ix.save(path)
    loaded = b2.VectorIndex.load(path, 64, b2.L2)
    for bits in (None, pack_bits(alive)):
        assert _same(ix.search(q, k, prm, alive_bits=bits), loaded.search(q, k, prm, alive_bits=bits)), "the loaded index differs"


# ---------------------------------------------------------------------------------------------------------------------------
# 7. refusals
# ---------------------------------------------------------------------------------------------------------------------------
def test_unknown_widths_refused_where_the_walk_runs():
    y, q = _clustered(20000, 64, 31, nq=8)
    for typ in ("HNSWFLAT", "MSTG"):
        ix = b2.VectorIndex(typ, b2.L2, 64, "graph_degree=16").build(y)
        plain = b2.VectorIndex(typ, b2.L2, 64, "").build(y)
        for w in (0, 3, 16, -1):
            with pytest.raises(B200Error) as e:
                ix.search(q, 10, f"search_width={w}")
            assert e.value.code == INVALID, (typ, w)
            for prm in ("graph=0", "exact_batch=1"):
                assert _same(ix.search(q, 10, f"{prm}, search_width={w}"), ix.search(q, 10, prm)), (typ, w, prm)
            assert _same(plain.search(q, 10, f"search_width={w}"), plain.search(q, 10, "")), (typ, w, "no graph")


def test_widest_mstg_rows():
    """At d = B200_MAX_FLOAT_DIM the walk's shared memory at ef_s = k = 1024 under a filter fits W = 1 only: W = 8 is refused
    there (B200_ERR_UNSUPPORTED) when the layout exceeds the limit, and walks as the reference at a smaller list."""
    d = 32640
    y, q = _integer(3000, d, 32, nq=2)
    ix = b2.VectorIndex("MSTG", b2.L2, d, "graph_degree=16").build(y)
    alive = np.random.default_rng(33).random(len(y)) < 0.5
    bits = pack_bits(alive)
    assert _smem(d, 1024, 1024, True, 1) <= SMEM_OPTIN
    if _smem(d, 1024, 1024, True, 8) > SMEM_OPTIN:
        with pytest.raises(B200Error) as e:
            ix.search(q, 1024, "ef_s=1024, search_width=8", alive_bits=bits)
        assert e.value.code == UNSUPPORTED
    else:
        dis, ids = ix.search(q, 1024, "ef_s=1024, search_width=8", alive_bits=bits)
        _, wi, _ = G.search(ix.graph(), to_bf16_values(y), q, ix.last_seeds(), 1024, 1024, G.iteration_cap(16, 8), "l2", alive, width=8)
        rd, ri = R.rerank(y, q, wi, 1024, b2.L2)
        assert np.array_equal(ids, ri) and dis.tobytes() == rd.tobytes()
    _mstg_check(ix, y, q, 16, 8, b2.L2, alive, 64)
