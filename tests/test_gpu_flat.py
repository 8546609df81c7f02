"""GPU parity tests (run on an H100: pytest -m gpu).  Every call goes through the C ABI
of libb200search.so (ctypes) and is checked against the CPU oracle / the reference goldens."""
import numpy as np
import pytest

import myscaledb_b200 as b2
import oracle as orc
from myscaledb_b200 import search as S
from tests.util import check_topk, exact_distance, to_bf16_values

pytestmark = pytest.mark.gpu
F32 = np.float32


def _nnn(lo, hi, d=3):
    return np.repeat(np.arange(lo, hi, dtype=np.float32)[:, None], d, axis=1)


# ------------------------------------------------------------------ reference goldens
def test_golden_00001_flat_index(goldens):
    g = goldens["00001_flat_l2"]
    c = b2.Corpus(b2.L2, 3).append(_nnn(0, 100))
    dis, ids = c.search(np.array([g["query"]], F32), g["k"])
    assert ids[0].tolist() == [e[0] for e in g["expect"]]
    np.testing.assert_allclose(dis[0], [e[1] for e in g["expect"]], rtol=1e-6)


def test_golden_00012_part_scan_with_empty_rows(goldens):
    g = goldens["00012_bruteforce_l2"]
    y = _nnn(0, 10030)
    y[10:30] = np.finfo(np.float32).max
    dis, ids = b2.part_scan(b2.L2, np.array([g["query"]], F32), y, g["k"], block_rows=128)
    assert ids[0].tolist() == [e[0] for e in g["expect"]]
    np.testing.assert_allclose(dis[0], [e[1] for e in g["expect"]], rtol=1e-5)


def _expect(dis, ids, exp, k, rtol=1e-6):
    n = len(exp)
    assert ids[0, :n].tolist() == [e[0] for e in exp]
    np.testing.assert_allclose(dis[0, :n], [e[1] for e in exp], rtol=rtol)
    assert (ids[0, n:k] == -1).all()


def test_golden_00003_prewhere_filter(goldens):
    g = goldens["00003_prewhere"]
    idv = np.arange(100)
    bits = orc.pack_bits((idv < 10) | (idv > 60))
    q = np.array([g["query"]], F32)
    dis, ids = b2.part_scan(b2.L2, q, _nnn(0, 100), g["k"], block_rows=1024, filter_bits=bits)
    _expect(dis, ids, g["expect"], g["k"])
    c = b2.Corpus(b2.L2, 3).append(_nnn(0, 100))  # FLAT index + DenseBitmap filter
    dis, ids = c.search(q, g["k"], alive_bits=bits)
    _expect(dis, ids, g["expect"], g["k"])


def test_golden_00008_empty_vectors(goldens):
    g = goldens["00008_empty_vectors"]
    y = _nnn(0, 430)
    y[10:30] = np.finfo(np.float32).max
    q = np.array([g["query"]], F32)
    dis, ids = b2.part_scan(b2.L2, q, y, g["k"], block_rows=1024)
    _expect(dis, ids, g["expect_flat"], g["k"])
    keep = np.r_[0:10, 30:430]  # an index is built from the rows that exist; labels map back through the row ids
    ix = b2.VectorIndex("IVFFLAT", b2.L2, 3, "ncentroids = 10").build(y[keep])
    dis, pos = ix.search(q, g["k"], "nprobe=10")
    assert keep[pos[0]].tolist() == [e[0] for e in g["expect_ivfflat"]]
    np.testing.assert_allclose(dis[0], [e[1] for e in g["expect_ivfflat"]], rtol=1e-6)


@pytest.mark.parametrize("name", ["00009_bruteforce_prewhere", "00011_bruteforce_prewhere_sparse"])
def test_golden_00009_00011_bruteforce_with_prewhere(goldens, name):
    g = goldens[name]
    idv = np.arange(10030)
    m = ((idv > 5000) | np.isin(idv, [9, 31, 999, 1])) if name.startswith("00009") else ((idv < 50) | np.isin(idv, [51, 55, 99, 100, 9999]))
    y = _nnn(0, 10030)
    y[10:30] = np.finfo(np.float32).max
    dis, ids = b2.part_scan(b2.L2, np.array([g["query"]], F32), y, g["k"], block_rows=128, filter_bits=orc.pack_bits(m))
    _expect(dis, ids, g["expect"], g["k"], rtol=1e-5)


def test_golden_00016_lightweight_delete(goldens):
    g = goldens["00016_lightweight_delete"]
    row_exists = np.ones(2100, np.uint8)
    row_exists[2] = 0
    dis, ids = b2.part_scan(b2.L2, np.array([g["query"]], F32), _nnn(0, 2100), g["k"], block_rows=1024, row_exists=row_exists)
    _expect(dis, ids, g["expect"], g["k"])


@pytest.mark.parametrize("name,metric", [("00002_batch_l2", b2.L2), ("00002_batch_ip", b2.IP)])
def test_golden_00002_batch(goldens, name, metric):
    g = goldens[name]
    q = np.array(g["queries"], F32)
    y = _nnn(0, 100)
    dis, ids = b2.part_scan(metric, q, y, g["k"])
    got = [[int(ids[qi, j]), qi, float(dis[qi, j])] for qi in range(3) for j in range(g["k"])]
    exp = g["expect"]
    assert [r[:2] for r in got] == [e[:2] for e in exp]
    np.testing.assert_allclose([r[2] for r in got], [e[2] for e in exp], rtol=2e-6)


def test_golden_00014_cosine(goldens):
    g = goldens["00014_cosine_bruteforce"]
    n = np.arange(1000, dtype=np.float32)
    y = np.stack([n, n + 3, n + 1], axis=1)
    dis, ids = b2.part_scan(b2.COSINE, np.array([g["query"]], F32), y, g["k"])
    assert ids[0].tolist() == [e[0] for e in g["expect"]]
    np.testing.assert_allclose(dis[0], [e[1] for e in g["expect"]], rtol=0, atol=2e-7)


@pytest.mark.parametrize("metric,prefix", [(b2.HAMMING, "hamming"), (b2.JACCARD, "jaccard")])
def test_golden_00038_binary(goldens, metric, prefix):
    g = goldens["00038_binary"]
    y = np.repeat((np.arange(1024) % 256).astype(np.uint8)[:, None], 4, axis=1)
    q = np.array([g["query"]], np.uint8)
    dis, ids = b2.part_scan(metric, q, y, 20)
    exp = g[prefix + "_brute"]
    assert ids[0].tolist() == [e[0] for e in exp]
    assert dis[0].tolist() == [float(F32(e[1])) for e in exp]
    mask = np.zeros(1024, bool); mask[101:120] = True
    dis, ids = b2.part_scan(metric, q, y, 20, filter_bits=orc.pack_bits(mask))
    exp = g[prefix + "_filter"]
    assert ids[0][:len(exp)].tolist() == [e[0] for e in exp] and (ids[0][len(exp):] == -1).all()
    bq = np.array(g["batch_queries"], np.uint8)
    dis, ids = b2.part_scan(metric, bq, y, 10)
    got = [[int(ids[qi, j]), qi, float(dis[qi, j])] for qi in range(3) for j in range(10)]
    assert got == [[e[0], e[1], float(F32(e[2]))] for e in g[prefix + "_batch"]]
    row_exists = np.ones(1024, np.uint8); row_exists[:200] = 0
    if metric == b2.HAMMING:
        dis, ids = b2.part_scan(metric, q, y, 10, row_exists=row_exists)
        assert [[int(i), float(d)] for i, d in zip(ids[0], dis[0])] == g["hamming_after_lwd_lt200"]


def test_golden_00028_768d_and_00035_ties(goldens):
    g = goldens["00028_mstg_768"]
    n = np.arange(1000, dtype=np.float64)[:, None]; x = np.arange(768, dtype=np.float64)[None, :]
    y = (0.00001 * (n * 768 + x + 1) * np.where(x % 2 == 0, -1.0, 1.0)).astype(np.float32)
    q = np.array([g["query"]], F32)
    dis, ids = b2.flat_knn(b2.L2, q, y, 5)
    assert ids[0].tolist() == [e[0] for e in g["expect_l2"]]
    np.testing.assert_allclose(dis[0], [e[1] for e in g["expect_l2"]], rtol=1e-4)
    dis, ids = b2.flat_knn(b2.COSINE, q, y, 5)
    assert ids[0].tolist() == [e[0] for e in g["expect_cosine"]]
    np.testing.assert_allclose(dis[0], [e[1] for e in g["expect_cosine"]], rtol=1e-4)
    alive = np.ones(1000, bool); alive[0] = False; alive[2] = False
    dis, ids = b2.flat_knn(b2.COSINE, q, y, 5, alive_bits=orc.pack_bits(alive))
    assert ids[0].tolist() == [e[0] for e in g["expect_cosine_after_delete_id2"]]
    t = goldens["00035_ties"]
    idv = np.array([n for n in range(1001) if n != 1])
    yy = np.repeat(idv.astype(np.float32)[:, None], 16, axis=1)
    dis, ids = b2.part_scan(b2.L2, np.array([t["query"]], F32), yy, 10)
    assert [[int(idv[i]), float(d)] for i, d in zip(ids[0], dis[0])] == t["expect_unfiltered"]
    dis, ids = b2.part_scan(b2.L2, np.array([t["query"]], F32), yy, 10, filter_bits=orc.pack_bits(idv < 11))
    assert [[int(idv[i]), float(d)] for i, d in zip(ids[0], dis[0])] == t["expect_filtered"]


# ------------------------------------------------------------------ scan kernel vs oracle
@pytest.mark.parametrize("metric", [b2.L2, b2.IP, b2.COSINE])
@pytest.mark.parametrize("n,d,nq,k", [(10000, 128, 1, 10), (5003, 17, 3, 7), (20011, 768, 8, 30), (3001, 96, 13, 100),
                                      (77, 5, 2, 100), (1, 8, 1, 3)])
def test_scan_matches_oracle(metric, n, d, nq, k):
    rng = np.random.default_rng(n + d + nq)
    y = rng.standard_normal((n, d)).astype(F32)
    x = rng.standard_normal((nq, d)).astype(F32)
    do, io = orc.search_without_index(metric, x, y, k)
    # the fp32 FMA scan kernel itself (path 1), whatever the batch size
    c = b2.Corpus(metric, d).append(y)
    c.set_path(1)
    dg, ig = c.search(x, k)
    c.close()
    check_topk(metric, x, y, dg, ig, do, io)
    # the one-shot entry point with automatic path selection: IP / cosine batches of >= 5 queries run on the 3xTF32
    # tensor-core kernel, whose ~1e-5 relative error may swap a near tie (still inside the 1e-4 contract)
    dg, ig = b2.flat_knn(metric, x, y, k)
    check_topk(metric, x, y, dg, ig, do, io, min_exact=0.999 if (nq < 5 or metric == b2.L2) else 0.99)


def test_scan_alive_bitmap_and_ip_min_quirk():
    rng = np.random.default_rng(5)
    y = rng.standard_normal((9000, 64)).astype(F32)
    x = rng.standard_normal((4, 64)).astype(F32)
    alive = rng.random(9000) < 0.3
    dg, ig = b2.flat_knn(b2.L2, x, y, 20, alive_bits=orc.pack_bits(alive))
    do, io = orc.search_without_index(orc.L2, x, y, 20, alive=orc.pack_bits(alive))
    check_topk(b2.L2, x, y, dg, ig, do, io)
    assert alive[ig].all()
    # vectorScanWithoutIndex IP quirk: scores <= FLT_MIN are never returned
    yneg = -np.abs(y); xpos = np.abs(x)
    dg, ig = b2.part_scan(b2.IP, xpos, yneg, 5)
    do, io = orc.part_scan(orc.IP, xpos, yneg, 5)
    assert (ig == -1).all() and (io == -1).all()
    row_exists = (rng.random(9000) < 0.9).astype(np.uint8)
    dg, ig = b2.part_scan(b2.IP, x, y, 10, row_exists=row_exists)
    do, io = orc.part_scan(orc.IP, x, y, 10, block_rows=1024, row_exists=row_exists)
    check_topk(b2.IP, x, y, dg, ig, do, io)


def test_scan_bf16_corpus():
    rng = np.random.default_rng(11)
    y = to_bf16_values(rng.standard_normal((30000, 768)).astype(F32))
    x = rng.standard_normal((5, 768)).astype(F32)
    for metric in (b2.L2, b2.IP, b2.COSINE):
        c = b2.Corpus(metric, 768, dtype=S.BF16).append(y)
        c.set_path(1)
        dg, ig = c.search(x, 10)
        do, io = orc.search_without_index(metric, x, y, 10)
        check_topk(metric, x, y, dg, ig, do, io)
        c.close()


# ------------------------------------------------------------------ tensor-core GEMM path vs oracle
@pytest.mark.parametrize("metric", [b2.IP, b2.L2, b2.COSINE])
@pytest.mark.parametrize("n,d,nq,k,path", [(20000, 768, 128, 10, 2), (5000, 64, 37, 30, 2), (70001, 128, 300, 10, 2),
                                           (70001, 128, 300, 10, 3), (70001, 128, 300, 10, 4), (70001, 128, 300, 10, 7), (1000, 96, 20, 50, 2),
                                           (33333, 768, 1024, 10, 2), (33333, 768, 1024, 10, 4), (33333, 768, 1024, 10, 5),
                                           (33333, 768, 1024, 10, 6), (33333, 768, 1024, 10, 7), (33333, 768, 512, 10, 2),
                                           (33333, 768, 512, 30, 7), (257, 64, 129, 5, 2), (9000, 512, 256, 10, 2), (9000, 512, 256, 10, 7),
                                           (9000, 832, 256, 10, 2)])
def test_gemm_path_matches_oracle(metric, n, d, nq, k, path):
    """b200_corpus_set_path codes 2..7 all select the tensor-core kernel (3..7 named instantiations of an earlier target
    and must keep working).  The same at >= 2 M rows: tests/test_gpu_gemm_scale.py."""
    rng = np.random.default_rng(n + d + nq + metric)
    y = to_bf16_values(rng.standard_normal((n, d)).astype(F32))
    x = to_bf16_values(rng.standard_normal((nq, d)).astype(F32))
    c = b2.Corpus(metric, d, dtype=S.BF16).append(y)
    c.set_path(path)
    dg, ig = c.search(x, k)
    c.close()
    do, io = orc.knn_flat_parts(orc.IP if metric != orc.L2 else orc.L2, *( _prep_cos(x, y) if metric == b2.COSINE else (x, y)), k, 4)
    if metric == b2.COSINE:
        do = 1 - do
    # fp32 tensor-core accumulation order differs from the CPU: near ties may swap
    check_topk(metric, x, y, dg, ig, do, io, rtol=2e-4, atol=2e-4 if metric == b2.L2 else 2e-5, min_exact=0.99)


def _prep_cos(x, y):
    x = x.copy(); y = y.copy()
    orc.lib().orc_normalize(x.ctypes.data_as(orc.C.POINTER(orc.C.c_float)), orc.C.c_int64(x.shape[0]), orc.C.c_int(x.shape[1]))
    orc.lib().orc_normalize(y.ctypes.data_as(orc.C.POINTER(orc.C.c_float)), orc.C.c_int64(y.shape[0]), orc.C.c_int(y.shape[1]))
    return x, y


@pytest.mark.parametrize("metric", [b2.IP, b2.L2, b2.COSINE])
@pytest.mark.parametrize("n,d,nq,k", [(20000, 768, 128, 10), (5000, 64, 37, 30), (70001, 128, 300, 10), (1000, 96, 20, 50),
                                      (33333, 768, 1024, 10), (257, 50, 129, 5), (9000, 100, 256, 100), (4000, 1536, 16, 10)])
def test_tf32x3_path_matches_oracle(metric, n, d, nq, k):
    """fp32 corpus, batch of queries: three TF32 tensor-core products per k-step (ip_gemm_sm90.cu) must give
    fp32-class results on arbitrary fp32 inputs (NOT pre-rounded), i.e. the same tolerance as the fp32 FMA scan."""
    rng = np.random.default_rng(7 * n + d + nq + metric)
    y = rng.standard_normal((n, d)).astype(F32)
    x = rng.standard_normal((nq, d)).astype(F32)
    c = b2.Corpus(metric, d).append(y)
    c.set_path(2)
    dg, ig = c.search(x, k)
    c.close()
    do, io = orc.knn_flat_parts(orc.IP if metric != orc.L2 else orc.L2, *(_prep_cos(x, y) if metric == b2.COSINE else (x, y)), k, 4)
    if metric == b2.COSINE:
        do = 1 - do
    check_topk(metric, x, y, dg, ig, do, io, rtol=4e-5, atol=2e-5 if metric == b2.L2 else 2e-6, min_exact=0.995)
    # against fp64 ground truth: ~1e-5 relative (measured; the tensor core's fp32 accumulator truncates), an order
    # inside the 1e-4 contract and ~100x tighter than one TF32 pass or bf16 operands
    for q in range(0, nq, max(1, nq // 8)):
        t = np.array([exact_distance(metric, x[q], y[j]) for j in ig[q]])
        assert np.abs(t - dg[q]).max() <= 4e-5 * max(1.0, np.abs(t).max())


def test_tf32x3_auto_path_filter_and_scan_agreement():
    """Auto path for an fp32 corpus and >= 16 queries is the tensor-core kernel; it must agree with the fp32 FMA
    scan (two independent GPU paths) under a DenseBitmap filter, through the one-shot b200_flat_knn as well."""
    rng = np.random.default_rng(77)
    y = rng.standard_normal((120000, 200)).astype(F32)
    x = rng.standard_normal((64, 200)).astype(F32)
    alive = rng.random(120000) < 0.3
    bits = orc.pack_bits(alive)
    c = b2.Corpus(b2.L2, 200).append(y)
    n0 = S.launch_count()
    d2, i2 = c.search(x, 10, alive_bits=bits)
    c.set_path(1); d1, i1 = c.search(x, 10, alive_bits=bits)
    c.close()
    assert alive[i2].all()
    check_topk(b2.L2, x, y, d2, i2, d1, i1, rtol=4e-5, atol=2e-5, min_exact=0.995)
    d3, i3 = b2.flat_knn(b2.L2, x, y, 10, alive_bits=bits)
    assert (i3 == i2).all() and np.allclose(d3, d2, rtol=0, atol=0)
    assert S.launch_count() > n0


def test_gemm_path_alive_bitmap():
    rng = np.random.default_rng(21)
    y = to_bf16_values(rng.standard_normal((40000, 256)).astype(F32))
    x = to_bf16_values(rng.standard_normal((64, 256)).astype(F32))
    alive = rng.random(40000) < 0.5
    c = b2.Corpus(b2.IP, 256, dtype=S.BF16).append(y)
    c.set_path(2)
    dg, ig = c.search(x, 10, alive_bits=orc.pack_bits(alive))
    c.close()
    do, io = orc.knn_flat(orc.IP, x, y, 10, alive=orc.pack_bits(alive))
    check_topk(b2.IP, x, y, dg, ig, do, io, rtol=2e-4, atol=2e-5, min_exact=0.99)
    assert alive[ig].all()


def test_gemm_equals_scan_large_property():
    """Size-independent property at a size the oracle cannot reach quickly: the two
    independent GPU paths (fp32 FMA scan vs tensor-core GEMM) must return the same ids."""
    rng = np.random.default_rng(33)
    y = to_bf16_values(rng.standard_normal((400000, 768)).astype(F32))
    x = to_bf16_values(rng.standard_normal((256, 768)).astype(F32))
    c = b2.Corpus(b2.IP, 768, dtype=S.BF16).append(y)
    c.set_path(2); d2, i2 = c.search(x, 10)
    c.set_path(1); d1, i1 = c.search(x, 10)
    c.close()
    check_topk(b2.IP, x, y, d2, i2, d1, i1, rtol=2e-4, atol=2e-5, min_exact=0.99)
    assert (np.diff(d2, axis=1) <= 0).all()  # sorted best-first


def test_topk_merge_device_matches_oracle_merge():
    """b200_topk_merge_device_ex against the oracle of getTotalTopSearchResultImpl (orc.merge_parts,
    MergeTreeBaseSearchManager.cpp:207-299) on integer scores, i.e. with ties everywhere: tie_mode 1 must reproduce the
    multimap order exactly (ascending: earlier part first; reverse walk for IP / BM25: later-inserted first) including the
    part index of every winner; tie_mode 0 is this library's (score, smaller id) contract; ids are full 64-bit values."""
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(3)
    for L, nq, k_in, k in ((8, 33, 10, 10), (3, 5, 30, 7), (16, 9, 100, 100), (2, 4, 5, 8)):
        for desc in (False, True):
            sc = rng.integers(-6, 7, (L, nq, k_in)).astype(F32)
            sc = -np.sort(-sc, axis=2) if desc else np.sort(sc, axis=2)     # each part's list is sorted best-first
            ids = (rng.permutation(L * nq * k_in).reshape(L, nq, k_in).astype(np.int64) + (1 << 33)) * 3   # beyond 2^32
            ids[L - 1, nq - 1, k_in // 2:] = -1                           # a part that returned fewer than k rows
            td, ti = torch.tensor(sc).cuda(), torch.tensor(ids).cuda()
            od = torch.empty((nq, k), dtype=torch.float32, device="cuda"); oi = torch.empty((nq, k), dtype=torch.int64, device="cuda")
            ol = torch.empty((nq, k), dtype=torch.int32, device="cuda")
            for tie_mode in (0, 1):
                S.topk_merge_device_ex(td.data_ptr(), ti.data_ptr(), L, nq * k_in, nq * k_in, nq, k_in, k, desc, tie_mode,
                                       od.data_ptr(), oi.data_ptr(), ol.data_ptr())
                torch.cuda.synchronize()
                gd, gi, gl = od.cpu().numpy(), oi.cpu().numpy(), ol.cpu().numpy()
                for q in range(nq):
                    m = ids[:, q, :].reshape(-1) >= 0
                    s1 = sc[:, q, :].reshape(-1)[m]; lab = ids[:, q, :].reshape(-1)[m]
                    part = np.repeat(np.arange(L), k_in)[m]
                    if tie_mode == 1:
                        es, ep, el = orc.merge_parts(s1, part, lab, k, desc)
                        n = len(es)
                        assert gi[q, :n].tolist() == el.tolist() and gl[q, :n].tolist() == ep.tolist(), (L, nq, k_in, k, desc, q)
                        np.testing.assert_array_equal(gd[q, :n], es)
                    else:
                        order = np.lexsort((lab, -s1 if desc else s1))[:k]
                        n = len(order)
                        assert gi[q, :n].tolist() == lab[order].tolist()
                        np.testing.assert_array_equal(gd[q, :n], s1[order])
                    assert (gi[q, n:] == -1).all()
    # the plain entry points (tie_mode 0) still work on the [L][nq][k] layout
    L, nq, k = 4, 6, 10
    dis = np.sort(rng.standard_normal((L, nq, k)).astype(F32), axis=2)
    ids = rng.permutation(L * nq * k).reshape(L, nq, k).astype(np.int64)
    td, ti = torch.tensor(dis).cuda(), torch.tensor(ids).cuda()
    od = torch.empty((nq, k), dtype=torch.float32, device="cuda"); oi = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    b2.topk_merge_device(td.data_ptr(), ti.data_ptr(), L, nq, k, False, od.data_ptr(), oi.data_ptr())
    torch.cuda.synchronize()
    for q in range(nq):
        order = np.lexsort((ids[:, q].reshape(-1), dis[:, q].reshape(-1)))[:k]
        assert oi[q].cpu().numpy().tolist() == ids[:, q].reshape(-1)[order].tolist()


def test_concurrent_searches_are_reentrant():
    """ClickHouse calls the library from one ThreadPool worker per part, concurrently."""
    import threading
    rng = np.random.default_rng(77)
    parts = [rng.standard_normal((20000, 64)).astype(F32) for _ in range(4)]
    x = rng.standard_normal((6, 64)).astype(F32)
    shared = b2.Corpus(b2.L2, 64).append(parts[0])
    expect = [orc.knn_flat(orc.L2, x, p, 10) for p in parts]
    errors = []

    def worker(i):
        try:
            for _ in range(5):
                dg, ig = b2.flat_knn(b2.L2, x, parts[i], 10)          # own temporary corpus
                check_topk(b2.L2, x, parts[i], dg, ig, *expect[i])
                dg, ig = shared.search(x, 10)                         # one index shared by all threads
                check_topk(b2.L2, x, parts[0], dg, ig, *expect[0])
        except Exception as e:  # noqa: BLE001
            errors.append(repr(e))
    ts = [threading.Thread(target=worker, args=(i,)) for i in range(4)]
    [t.start() for t in ts]; [t.join() for t in ts]
    assert not errors, errors
