"""Two-stage indexes with their fp32 re-rank rows in pinned host memory (keep_raw=2): the second stage gathers its candidate
rows over PCIe (gather_host_rows_kernel) and re-ranks them with the same kernel as the HBM placement, so every answer must
equal the HBM placement's byte for byte (dis, ids and num_candidates compared on their raw bytes).  One index is moved
between the placements (set_raw_placement) wherever two answers are compared: k-means is not bitwise reproducible
between builds."""
import numpy as np
import pytest

import myscaledb_b200 as b2
from myscaledb_b200.search import B200Error
from tests import ivf_reference as R

pytestmark = pytest.mark.gpu
F32 = np.float32
INVALID, UNSUPPORTED = 1, 3
HEADER_HAS_RAW = 44   # byte offset of has_raw in the B2IX header (tests/ivf_reference.py HEADER)
STAGE_BYTES = 256 << 20   # kHostStageBytes (csrc/ivf.cu)


def _clustered(n, d, seed, nq=1025, n_centres=300, spread=0.3):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((n_centres, d)).astype(F32)
    y = centres[rng.integers(0, n_centres, n)] + spread * rng.standard_normal((n, d)).astype(F32)
    q = centres[rng.integers(0, n_centres, nq)] + spread * rng.standard_normal((nq, d)).astype(F32)
    return y.astype(F32), q.astype(F32)


def _d_pad(d):
    return -(-d // 4) * 4


def _answer(ix, q, k, params="", first_stage_only=False, alive_bits=None):
    dis, ids = ix.search(q, k, params, first_stage_only=first_stage_only, alive_bits=alive_bits)
    return dis.tobytes(), ids.tobytes(), ix.last_num_candidates


def _sweep(ix, q, alive):
    """Answers of every shape of the sweep: nq x k x nprobe x bitmap, plus k x refine_factor clamped at 1024 and first_stage_only."""
    out = {}
    for nq in (1, 7, 256, 1025):
        for k in (1, 10, 100):
            for nprobe in (4, 64):
                for bits in (None, alive):
                    out[(nq, k, nprobe, bits is None)] = _answer(ix, q[:nq], k, f"nprobe={nprobe}", alive_bits=bits)
    out["clamped"] = _answer(ix, q[:256], 100, "nprobe=16, refine_factor=16")
    out["first_stage"] = _answer(ix, q[:256], 10, "nprobe=16", first_stage_only=True)
    return out


CASES = [("MSTG", 98, "ncentroids=64"),                              # d_pad 100: padding columns
         ("SCANN", 96, "ncentroids=64, M=6"),                         # d / M = 16: 8-bit table look-up scan
         ("SCANN", 96, "ncentroids=64, M=24, bit_size=4"),            # 4-bit codes
         ("IVFFLAT", 98, "ncentroids=64, refine_factor=8"),
         ("IVFSQ", 98, "ncentroids=64, refine_factor=8"),
         ("HNSWFLAT", 98, "ncentroids=64")]


@pytest.mark.parametrize("metric", [b2.L2, b2.IP, b2.COSINE], ids=["L2", "IP", "COSINE"])
@pytest.mark.parametrize("typ,d,params", CASES, ids=[f"{c[0]}-{c[2].split(', ', 1)[-1]}" for c in CASES])
def test_same_index_both_placements_byte_identical(typ, d, params, metric):
    n = 20000
    y, q = _clustered(n, d, seed=d + metric)
    alive = np.packbits(np.random.default_rng(metric).random(n) < 0.6, bitorder="little")
    ix = b2.VectorIndex(typ, metric, d, params + ", keep_raw=1").build(y)
    assert ix.info()["uses_ivf"]
    hbm_bytes = ix.memory_bytes()
    assert ix.host_memory_bytes() == 0
    a = _sweep(ix, q, alive)
    ix.set_raw_placement(2)
    assert ix.host_memory_bytes() == n * _d_pad(d) * 4
    assert ix.memory_bytes() <= hbm_bytes - n * _d_pad(d) * 4
    b = _sweep(ix, q, alive)
    ix.set_raw_placement(1)
    assert ix.host_memory_bytes() == 0 and ix.memory_bytes() == hbm_bytes
    c = _sweep(ix, q, alive)
    for key in a:
        assert a[key] == b[key], f"host placement differs from HBM at {key}"
        assert a[key] == c[key], f"HBM placement after the round trip differs at {key}"
    assert a["clamped"][2] == 1024 and a["first_stage"][2] == 10


def test_staging_chunks_byte_identical():
    """1024 candidates x 768-d = 3 MB of rows per query: 300 queries need four staging chunks of 85 queries."""
    n, d, k = 20000, 768, 100
    y, q = _clustered(n, d, seed=11, nq=300)
    per_q = 1024 * d * 4
    qchunk = STAGE_BYTES // per_q
    assert len(q) * per_q > 3 * STAGE_BYTES
    ix = b2.VectorIndex("MSTG", b2.L2, d, "ncentroids=64").build(y)
    prm = "nprobe=64, refine_factor=16"
    hbm = _answer(ix, q, k, prm)
    ix.set_raw_placement(2)
    host = _answer(ix, q, k, prm)
    assert host == hbm and host[2] == 1024
    parts = [ix.search(q[i:i + qchunk], k, prm) for i in range(0, len(q), qchunk)]
    assert np.concatenate([p[0] for p in parts]).tobytes() == host[0]
    assert np.concatenate([p[1] for p in parts]).tobytes() == host[1]


def _build_variants(y, d, metric, params):
    """The same rows through every build path with keep_raw=2."""
    import torch

    n = len(y)
    out = {"build": b2.VectorIndex("MSTG", metric, d, params).build(y)}
    ix = b2.VectorIndex("MSTG", metric, d, params).reserve(n).train(y[::3])
    for a, b in ((0, 1), (1, 4000), (4000, 11111), (11111, n)):   # uneven chunks
        ix.add(y[a:b])
    out["streamed"] = ix.finalize()
    t = torch.from_numpy(y).cuda()
    ix = b2.VectorIndex("MSTG", metric, d, params).reserve(n).train_device(t.data_ptr(), n)
    ix.add_device(t.data_ptr(), 7000).add_device(t[7000:].data_ptr(), n - 7000)
    torch.cuda.synchronize()
    out["add_device"] = ix.finalize()
    ix = b2.VectorIndex("MSTG", metric, d, params).train(y)   # no reserve: the host array grows chunk by chunk
    for a, b in ((0, 5000), (5000, 9000), (9000, n)):
        ix.add(y[a:b])
    out["grown"] = ix.finalize()
    return out


@pytest.mark.parametrize("metric", [b2.L2, b2.COSINE], ids=["L2", "COSINE"])
def test_built_on_the_host(metric, tmp_path):
    n, d, k = 20000, 98, 10
    y, q = _clustered(n, d, seed=21 + metric, nq=64)
    params = "ncentroids=64"
    no_rows = b2.VectorIndex("MSTG", metric, d, params + ", keep_raw=0").build(y).memory_bytes()
    for name, ix in _build_variants(y, d, metric, params + ", keep_raw=2").items():
        assert ix.info()["n"] == n
        assert ix.memory_bytes() == no_rows, f"{name}: HBM bytes include the host rows"
        assert ix.host_memory_bytes() == n * _d_pad(d) * 4, name
        host = _answer(ix, q, k, "nprobe=8")
        path = tmp_path / f"{name}.b2ix"
        ix.save(path)
        ix.set_raw_placement(1)
        assert _answer(ix, q, k, "nprobe=8") == host, name
        # the rows written from host memory are the prepared rows, and the refined distances are theirs
        s = R.read_index(path)
        assert s.has_raw == 2
        if metric == b2.L2:
            assert np.array_equal(s.rows, y), name
        else:   # unit rows (the device's normalisation; the reference's copy of it may round the last bit differently)
            assert np.abs(s.rows - R.prepare_queries(y, metric)).max() <= 1e-6, name
        dis, ids = np.frombuffer(host[0], F32).reshape(-1, k), np.frombuffer(host[1], np.int64).reshape(-1, k)
        Q = R.prepare_queries(q, metric).astype(np.float64)
        assert (ids >= 0).all()
        Y = s.rows[ids].astype(np.float64)
        if metric == b2.L2:
            ref, tol = ((Q[:, None, :] - Y) ** 2).sum(2), R.TOL_REL * ((Q * Q).sum(1)[:, None] + (Y * Y).sum(2) + 2 * np.abs(np.einsum("qd,qkd->qk", Q, Y)))
        else:
            ip = np.einsum("qd,qkd->qk", Q, Y)
            ref, tol = 1 - ip, R.TOL_REL * (1 + np.einsum("qd,qkd->qk", np.abs(Q), np.abs(Y)))
        assert (np.abs(dis - ref) <= tol).all(), f"{name}: refined distance off by {np.abs(dis - ref).max():.3g}"
        assert (np.diff(dis, axis=1) >= 0).all()


def test_refine_and_search_device_on_a_side_stream():
    import torch

    n, d, k = 20000, 98, 10
    y, q = _clustered(n, d, seed=31, nq=40)
    ix = b2.VectorIndex("MSTG", b2.IP, d, "ncentroids=64").build(y)
    rng = np.random.default_rng(3)
    cand = rng.integers(0, n, (40, 64)).astype(np.int64)
    cand[:, ::5] = -1
    cand[:, 1::7] = n + rng.integers(0, 1000, cand[:, 1::7].shape)
    cand[3] = -1                                                        # a query without any candidate
    off = (1 << 32) + 5
    alive = np.packbits(rng.random(n) < 0.5, bitorder="little")

    def run():
        r = ix.refine(q, cand, k)
        tq = torch.from_numpy(q).cuda()
        ta = torch.from_numpy(alive).cuda()
        od = torch.empty((len(q), k), dtype=torch.float32, device="cuda")
        oi = torch.empty((len(q), k), dtype=torch.int64, device="cuda")
        side = torch.cuda.Stream()
        torch.cuda.synchronize()
        ix.search_device(tq.data_ptr(), len(q), k, od.data_ptr(), oi.data_ptr(), params="nprobe=8", id_offset=off,
                         alive_ptr=ta.data_ptr(), stream=side.cuda_stream)
        side.synchronize()
        return r[0].tobytes(), r[1].tobytes(), od.cpu().numpy().tobytes(), oi.cpu().numpy()

    hbm = run()
    ix.set_raw_placement(2)
    host = run()
    assert hbm[:3] == host[:3] and np.array_equal(hbm[3], host[3])
    ids = host[3]
    assert ((ids == -1) | (ids >= off)).all() and (ids >= off).any()
    r_ids = np.frombuffer(host[1], np.int64).reshape(40, k)
    assert (r_ids[3] == -1).all() and (r_ids[r_ids >= 0] < n).all()


def test_persistence(tmp_path):
    n, d, k = 20000, 98, 10
    y, q = _clustered(n, d, seed=41, nq=64)
    ix = b2.VectorIndex("MSTG", b2.L2, d, "ncentroids=64").build(y)
    ix.save(tmp_path / "hbm.b2ix")
    ix.set_raw_placement(2)
    ix.save(tmp_path / "host.b2ix")
    a, b = (tmp_path / "hbm.b2ix").read_bytes(), (tmp_path / "host.b2ix").read_bytes()
    assert len(a) == len(b) and a[:HEADER_HAS_RAW] == b[:HEADER_HAS_RAW] and a[HEADER_HAS_RAW + 4:] == b[HEADER_HAS_RAW + 4:]
    assert np.frombuffer(a, np.int32, 1, HEADER_HAS_RAW)[0] == 1 and np.frombuffer(b, np.int32, 1, HEADER_HAS_RAW)[0] == 2
    want = _answer(ix, q, k, "nprobe=8")
    la = b2.VectorIndex.load(tmp_path / "hbm.b2ix", d)
    lb = b2.VectorIndex.load(tmp_path / "host.b2ix", d)
    assert lb.host_memory_bytes() == n * _d_pad(d) * 4 and la.host_memory_bytes() == 0
    assert _answer(la, q, k, "nprobe=8") == want and _answer(lb, q, k, "nprobe=8") == want
    la.set_raw_placement(2)
    assert la.memory_bytes() == lb.memory_bytes()
    lb.save(tmp_path / "again.b2ix")
    assert (tmp_path / "again.b2ix").read_bytes() == b
    # a 4-bit PQ index (B2IX v3) takes host rows too
    s4 = b2.VectorIndex("SCANN", b2.L2, 96, "ncentroids=64, M=24, bit_size=4").build(_clustered(n, 96, seed=42)[0])
    q4 = _clustered(n, 96, seed=42, nq=64)[1]
    s4.set_raw_placement(2)
    s4.save(tmp_path / "pq4.b2ix")
    l4 = b2.VectorIndex.load(tmp_path / "pq4.b2ix", 96)
    assert l4.host_memory_bytes() > 0 and _answer(l4, q4, k, "nprobe=8") == _answer(s4, q4, k, "nprobe=8")

    def refused(name, data):
        p = tmp_path / name
        p.write_bytes(data)
        with pytest.raises(B200Error) as e:
            b2.VectorIndex.load(p, d)
        assert e.value.code == INVALID, name

    def patched(data, has_raw):
        data = bytearray(data)
        data[HEADER_HAS_RAW:HEADER_HAS_RAW + 4] = np.int32(has_raw).tobytes()
        return bytes(data)

    refused("has_raw3.b2ix", patched(b, 3))
    refused("truncated.b2ix", b[:72 + (n // 2) * d * 4])
    bits = np.random.default_rng(5).integers(0, 256, (20000, 16), dtype=np.uint8)
    b2.VectorIndex("BINARYIVF", b2.HAMMING, 128, "ncentroids=64").build(bits).save(tmp_path / "bin.b2ix")
    refused("bin2.b2ix", patched((tmp_path / "bin.b2ix").read_bytes(), 2))
    b2.VectorIndex("FLAT", b2.L2, d).build(y[:3000]).save(tmp_path / "flat.b2ix")
    refused("flat2.b2ix", patched((tmp_path / "flat.b2ix").read_bytes(), 2))


def test_refusals_and_no_ops():
    n, d, k = 20000, 98, 10
    y, q = _clustered(n, d, seed=51, nq=16)

    def code(fn):
        with pytest.raises(B200Error) as e:
            fn()
        return e.value.code

    ix = b2.VectorIndex("MSTG", b2.L2, d, "ncentroids=64, keep_raw=2").build(y)
    assert code(lambda: ix.search(q, k, "exact_batch=1")) == UNSUPPORTED
    ix.search(q, k, "nprobe=8")                                             # the list search still answers
    for typ, rows, params in (("FLAT", y[:5000], ""), ("MSTG", y[:1500], "ncentroids=64")):   # 1500 rows: the small-part FLAT fallback
        host = b2.VectorIndex(typ, b2.L2, d, params + (", " if params else "") + "keep_raw=2").build(rows)
        hbm = b2.VectorIndex(typ, b2.L2, d, params).build(rows)
        assert not host.info()["uses_ivf"] and host.host_memory_bytes() == 0 and host.memory_bytes() == hbm.memory_bytes()
        assert _answer(host, q, k) == _answer(hbm, q, k)
        assert _answer(host, q, k, "exact_batch=1") == _answer(hbm, q, k, "exact_batch=1")
        assert code(lambda: host.set_raw_placement(2)) == UNSUPPORTED
    bits = np.random.default_rng(5).integers(0, 256, (20000, 16), dtype=np.uint8)
    assert code(lambda: b2.VectorIndex("BINARYIVF", b2.HAMMING, 128, "ncentroids=64").build(bits).set_raw_placement(2)) == UNSUPPORTED
    assert code(lambda: b2.VectorIndex("MSTG", b2.L2, d, "ncentroids=64, keep_raw=0").build(y).set_raw_placement(2)) == INVALID
    assert code(lambda: b2.VectorIndex("MSTG", b2.L2, d, "ncentroids=64").reserve(n).train(y).set_raw_placement(2)) == INVALID
    assert code(lambda: ix.set_raw_placement(3)) == INVALID
    ix.set_raw_placement(2)                                                 # already there: a no-op
    assert ix.host_memory_bytes() == n * _d_pad(d) * 4
