"""FLAT search paths against the float64 reference of the stored corpus (tests/flat_reference.py): the staged scan, the
fused single-query scan, bf16 on the tensor cores and fp32 (3xTF32) on the tensor cores, for L2, IP and cosine, at the
shapes where such kernels break; then targeted tests of the IP quirk, the L2 re-score, tiny norms, NaN / inf rows, the
device entry points, chunked appends, schedules, the per-thread scratch corpus and the refusals.

Non-finite rows.  A row whose distance is not finite (a NaN coordinate; under L2 and cosine also an infinite one) is never
returned and never displaces a finite row, on every path.  Under IP an infinite coordinate has no single meaning across
the paths (the scan ranks an inner product of +inf first; the 3xTF32 split turns the row into NaN), so such rows are
outside the IP contract and not tested.

Run with -s to see the largest error / bound ratio of every path."""
import os

import numpy as np
import pytest

import myscaledb_b200 as b2
import oracle as orc
from myscaledb_b200 import search as S
from myscaledb_b200._lib import lib
from tests import flat_reference as fr
from tests.util import check_topk, to_bf16_values

pytestmark = pytest.mark.gpu
F32 = np.float32
METRICS = [b2.L2, b2.IP, b2.COSINE]

# the four flat paths: (reference path, corpus dtype or None = alternate, set_path code, entry)
PATHS = {
    "staged": ("scan", None, S.PATH_SCAN, "device"),
    "fused": ("scan", None, S.PATH_SCAN, "host"),
    "bf16": ("bf16", S.BF16, S.PATH_TENSOR, "host"),
    "tf32": ("tf32", S.F32, S.PATH_TENSOR, "host"),
}
KERNEL = {"bf16": S.KERNEL_GEMM_BF16, "tf32": S.KERNEL_GEMM_TF32X3}

# Edge combos: shapes cycled (not a Cartesian product), wide rows with small batches and large batches with narrow rows,
# n at the edges (1, k - 1, k, 255 - 257 rows).  k is KS[k index % len(KS)].
DS = [1, 3, 17, 63, 64, 65, 100, 129, 768, 1536, 2048, 4096]
NQS = [2049, 1025, 1024, 129, 128, 127, 65, 64, 20, 19, 9, 8, 5, 4, 2, 1]
KS_TC = [1, 16, 17, 32, 100, 257, 1024]
KS_SCAN = KS_TC + [2048]
NS = ["1", "k-1", "k", 255, 256, 257, 1000]
ALIVES = [None, "dead", "k-1", "single", "tiles", "ragged"]
EDGE = [(DS[i % 12], NQS[i % 16], i % 8, NS[i % 7], ALIVES[i % 6]) for i in range(24)]
# Full combos: n = max(4 k + 3, 1000), so every k selects among more eligible rows than it keeps (at k = 1024 the
# per-thread lists of the tensor-core kernels live in global scratch), with the bitmaps that leave rows alive
FULL = [(2048, 65, 0, "4k", "tiles"), (4096, 20, 1, "4k", "ragged"), (1536, 129, 2, "4k", None), (65, 1025, 3, "4k", "tiles"),
        (768, 64, 4, "4k", "ragged"), (129, 128, 5, "4k", "tiles"), (100, 9, 6, "4k", "ragged"), (64, 19, 7, "4k", None),
        (2048, 5, 6, "4k", None), (17, 2049, 5, "4k", "ragged")]
COMBOS = EDGE + FULL

RATIOS = {}
LAST = {"variant": None}   # (kernel, cta_group, pairs_per_cluster, grid) of the last run_path search


def _note_ratio(path, r, dis, ids, id_offset=0):
    v = fr.error_ratio(r, dis, ids, id_offset)
    RATIOS[path] = max(RATIOS.get(path, 0.0), v)
    return v


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    for p, v in sorted(RATIOS.items()):
        print(f"largest error / bound ratio, {p}: {v:.3g}")


def alive_mask(kind, n, k, rng):
    """bool[n] (None = no bitmap) and the packed bitmap, whose bits past row n - 1 are set."""
    if kind is None:
        return None, None
    a = np.zeros(n, bool)
    if kind == "k-1":
        a[rng.choice(n, min(n, max(0, k - 1)), replace=False)] = True
    elif kind == "single":
        a[rng.integers(n)] = True
    elif kind == "tiles":
        a[:] = rng.random(n) < 0.7
        for t in range(0, n, 512):
            a[t:t + 256] = False                   # every other 256-row tile entirely dead
    elif kind == "ragged":
        a[:] = rng.random(n) < 0.5
    bits = orc.pack_bits(a)
    if n % 8:
        bits[-1] |= np.uint8((0xff << (n % 8)) & 0xff)   # bits past the last row must be ignored
    return a, bits


def search(c, x, k, bits=None, entry="host", id_offset=0, stream=None):
    """Corpus search through the host entry point or through search_device (device queries, bitmap and outputs)."""
    if entry == "host":
        return c.search(x, k, alive_bits=bits)
    import torch
    nq = len(x)
    tq = torch.from_numpy(np.ascontiguousarray(x, F32)).cuda()
    ta = torch.from_numpy(bits).cuda() if bits is not None else None
    od = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    oi = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    s = stream.cuda_stream if stream is not None else 0
    c.search_device(tq.data_ptr(), nq, k, od.data_ptr(), oi.data_ptr(), id_offset=id_offset,
                    alive_ptr=ta.data_ptr() if ta is not None else 0, stream=s)
    if stream is not None:
        stream.synchronize()
    return od.cpu().numpy(), oi.cpu().numpy()


def run_path(name, metric, y, x, k, alive=None, bits=None, dtype=None, id_offset=0):
    """Search y with x on one named path; returns (reference, dis, ids) after checking the kernel that ran."""
    rpath, pd, code, entry = PATHS[name]
    dtype = pd if pd is not None else dtype
    c = b2.Corpus(metric, y.shape[1], dtype=dtype).append(y)
    c.set_path(code)
    n0 = S.launch_count()
    dis, ids = search(c, x, k, bits, "device" if id_offset else entry, id_offset=id_offset)
    launches = S.launch_count() - n0
    LAST["variant"] = c.last_variant()
    kern = LAST["variant"][0]
    c.close()
    if name in KERNEL:
        assert kern == KERNEL[name], (name, kern)
    else:
        assert kern == S.KERNEL_SCAN
    if name == "fused":
        assert launches == 1, f"the fused scan is one launch, this call made {launches}"
    r = fr.reference(metric, fr.BF16 if dtype == S.BF16 else fr.F32, rpath, y, x, k, alive=alive)
    return r, dis, ids


def check(name, r, dis, ids, what, id_offset=0):
    bad = fr.compare(r, dis, ids, id_offset)
    assert not bad, f"{name} {what}: {len(bad)} problems: {bad[:4]}"
    _note_ratio(name, r, dis, ids, id_offset)


# ------------------------------------------------------------------ the matrix
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("name", list(PATHS))
def test_paths_match_the_reference(name, metric):
    scan = PATHS[name][0] == "scan"
    ks = KS_SCAN if name == "staged" else KS_TC
    selecting = set()   # (k, alive kind, d) of the combos with more eligible rows than k
    for i, (d, nq, ki, nspec, akind) in enumerate(COMBOS):
        k = ks[ki % len(ks)]
        if name == "fused":
            nq = min(nq, 8)
        n = {"1": 1, "k-1": max(1, k - 1), "k": k, "4k": max(4 * k + 3, 1000)}.get(nspec, nspec)
        rng = np.random.default_rng(1000 * i + 10 * metric + len(name))
        y = rng.standard_normal((n, d)).astype(F32)
        x = rng.standard_normal((nq, d)).astype(F32)
        alive, bits = alive_mask(akind, n, k, rng)
        dtype = (S.F32, S.BF16)[i % 2] if scan else None
        r, dis, ids = run_path(name, metric, y, x, k, alive, bits, dtype)
        check(name, r, dis, ids, f"combo {i} d={d} nq={nq} k={k} n={n} alive={akind} dtype={dtype}")
        if (n if alive is None else int(alive.sum())) > k:
            selecting.add((k, akind if akind != "tiles" or n >= 512 else "tiles, n < 512", d))
    # every k, and every bitmap that can leave more than k rows alive, really selected a top k at least once ("dead",
    # "single" and "k-1" leave at most k rows by construction: they test the unfilled tail)
    assert {e[0] for e in selecting} == set(ks), sorted(selecting)
    assert {None, "tiles", "ragged"} <= {e[1] for e in selecting}, sorted(selecting)
    assert {1536, 2048, 4096} <= {e[2] for e in selecting}, sorted(selecting)


@pytest.fixture(scope="module")
def million_rows():
    rng = np.random.default_rng(2024)
    return rng.standard_normal((1_000_003, 64)).astype(F32), rng.standard_normal((8, 64)).astype(F32)


@pytest.mark.parametrize("name", list(PATHS))
def test_a_million_rows(million_rows, name):
    """The persistent schedule of the tensor-core kernels walks thousands of tiles; the scan splits rows over many blocks."""
    y, x = million_rows
    for metric in METRICS:
        k = 100
        r, dis, ids = run_path(name, metric, y, x, k, dtype=S.BF16 if metric == b2.IP else S.F32)
        check(name, r, dis, ids, f"1M rows metric {metric}")


# ------------------------------------------------------------------ 1. IP quirk on every path part_scan reaches
@pytest.mark.parametrize("nq,k,kernel", [(3, 10, S.KERNEL_SCAN), (9, 10, S.KERNEL_GEMM_TF32X3), (9, 300, S.KERNEL_SCAN)])
def test_ip_quirk_on_every_part_scan_path(nq, k, kernel):
    """part_scan never returns a row scoring <= FLT_MIN.  fp32 IP goes to the fused scan for 1 - 4 queries, to 3xTF32 for
    5 or more with k <= 256 and to the staged scan above; a Corpus built the same way shows which kernel ran."""
    rng = np.random.default_rng(nq + k)
    n, d = 3000, 96
    y = -np.abs(rng.standard_normal((n, d))).astype(F32)
    pos = rng.choice(n, 6, replace=False)
    y[pos] = -y[pos]                                   # only 6 rows score above zero against a positive query
    x = np.abs(rng.standard_normal((nq, d))).astype(F32)
    x[0] = -x[0]                                       # ... and the first query scores above zero everywhere but there
    c = b2.Corpus(b2.IP, d).append(y)
    c.search(x, k)
    assert c.last_variant()[0] == kernel
    c.close()
    dis, ids = b2.part_scan(b2.IP, x, y, k)
    r = fr.reference(fr.IP, fr.F32, "tf32" if kernel == S.KERNEL_GEMM_TF32X3 else "scan", y, x, k, quirk=True)
    check("quirk", r, dis, ids, f"nq={nq} k={k}")
    assert (ids[1:, 6:] == -1).all() and (dis[1:, 6:] == F32(fr.FLT_MIN)).all()
    do, io = orc.part_scan(orc.IP, x, y, k)
    check_topk(b2.IP, x, y, dis, ids, do, io, rtol=4e-5, atol=2e-6, min_exact=0.99)


# ------------------------------------------------------------------ 2. L2 re-score far from the origin
def _far_clusters(rng, n, nq, d=768):
    """768-d clusters with ||y||^2 ~ 840 and neighbour distances ~ 115 (DESIGN section 4)."""
    cent = rng.standard_normal((20, d))
    y = cent[rng.integers(20, size=n)] + 0.27 * rng.standard_normal((n, d))
    x = cent[rng.integers(20, size=nq)] + 0.27 * rng.standard_normal((nq, d))
    return y.astype(F32), x.astype(F32)


@pytest.mark.parametrize("name", ["bf16", "tf32"])
def test_l2_rescore_far_from_the_origin(name):
    rng = np.random.default_rng(84)
    y, x = _far_clusters(rng, 20000, 64)
    assert 700 < (y.astype(np.float64) ** 2).sum(1).mean() < 1000
    dtype = PATHS[name][1]
    for k in (10, 100):
        r, dis, ids = run_path(name, b2.L2, y, x, k)
        check(name, r, dis, ids, f"far clusters k={k}")
        assert (np.diff(dis, axis=1) >= 0).all()
        # search_device with an id offset past 2^32: the re-score reads row id - offset
        off = 1 << 33
        r, dis_d, ids_d = run_path(name, b2.L2, y, x, k, id_offset=off)
        check(name, r, dis_d, ids_d, f"far clusters k={k} id_offset=2^33", id_offset=off)
        assert np.array_equal(ids_d, np.where(ids >= 0, ids + off, -1))
        assert np.array_equal(dis_d.view(np.uint32), dis.view(np.uint32))
    # negative control: without the re-score the expanded form's cancellation is far outside the bound
    os.environ["B200_GEMM_RESCORE_L2"] = "0"
    try:
        c = b2.Corpus(b2.L2, y.shape[1], dtype=dtype).append(y)
    finally:
        del os.environ["B200_GEMM_RESCORE_L2"]
    c.set_path(2)
    dis, ids = c.search(x, 10)
    c.close()
    r = fr.reference(fr.L2, fr.BF16 if dtype == S.BF16 else fr.F32, PATHS[name][0], y, x, 10)
    assert fr.compare(r, dis, ids), "the comparator accepted distances of the expanded form"


# ------------------------------------------------------------------ 3. cosine near zero norm
@pytest.mark.parametrize("name", list(PATHS))
def test_cosine_zero_and_tiny_norms(name):
    rng = np.random.default_rng(7)
    n, d, k = 600, 100, 40
    eps = float(np.finfo(F32).eps)

    def scaled(m, sq):
        v = rng.standard_normal((m, d))
        return (v / np.linalg.norm(v, axis=1, keepdims=True) * np.sqrt(sq)).astype(F32)

    y = rng.standard_normal((n, d)).astype(F32)
    y[0:10] = 0.0
    y[10:40] = scaled(30, 0.97 * eps)                 # just below FLT_EPSILON: factor 1
    y[40:70] = scaled(30, 1.03 * eps)                 # just above: normalised
    y[70:75] = 0.0
    for r_ in range(70, 75):                          # exactly FLT_EPSILON (2^-24 + 2^-24, exact in fp32 and bf16): normalised
        y[r_, rng.choice(d, 2, replace=False)] = 2.0 ** -12
    x = np.concatenate([np.zeros((1, d), F32), scaled(1, 0.97 * eps), scaled(1, 1.03 * eps), y[15:16], y[45:46], y[72:73],
                        rng.standard_normal((2, d)).astype(F32)])     # 8 queries: the fused scan takes them
    dtype = S.BF16 if name in ("staged", "bf16") else S.F32
    # the stored squared norms lie on the intended side of FLT_EPSILON (the device's fp32 sums err by ~1e-6 relative)
    sq = (fr.stored_rows(y, fr.BF16 if dtype == S.BF16 else fr.F32).astype(np.float64) ** 2).sum(1)
    assert (sq[10:40] < 0.99 * eps).all() and (sq[40:70] > 1.01 * eps).all() and (sq[70:75] == eps).all()
    r, dis, ids = run_path(name, b2.COSINE, y, x, k, dtype=dtype)
    check(name, r, dis, ids, "tiny norms")
    # the zero query has distance 1 to every row: the smallest ids win
    assert ids[0].tolist() == list(range(k)) and (dis[0] == 1).all()


# ------------------------------------------------------------------ 4. NaN and inf rows
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("name", list(PATHS))
def test_nan_and_inf_rows(name, metric):
    rng = np.random.default_rng(11 + metric)
    n, d = 300, 64
    y = rng.standard_normal((n, d)).astype(F32)
    bad = rng.choice(n, 40, replace=False)
    y[bad[:10]] = np.nan                               # whole rows
    y[bad[10:20], 5] = np.nan                          # one coordinate
    if metric != b2.IP:
        y[bad[20:30], 7] = np.inf
        y[bad[30:40], 9] = -np.inf
    x = rng.standard_normal((8, d)).astype(F32)
    for k in (100, 290):                               # 290 > the finite rows: the tail must stay empty
        r, dis, ids = run_path(name, metric, y, x, k, dtype=S.F32)
        check(name, r, dis, ids, f"non-finite rows k={k}")
        assert not np.isin(ids, bad[:40 if metric != b2.IP else 20]).any()


# ------------------------------------------------------------------ 5. device entry points
@pytest.mark.parametrize("name", ["staged", "bf16", "tf32"])
def test_search_device_stream_bitmap_and_offset(name):
    import torch
    rng = np.random.default_rng(5)
    n, d, nq, k = 5000, 100, 20, 30
    y = rng.standard_normal((n, d)).astype(F32)
    x = rng.standard_normal((nq, d)).astype(F32)
    alive, bits = alive_mask("ragged", n, k, rng)
    off = (1 << 32) + 7
    st = torch.cuda.Stream()
    for metric in METRICS:
        rpath, pd, code, _ = PATHS[name]
        dtype = pd if pd is not None else S.BF16
        c = b2.Corpus(metric, d, dtype=dtype).append(y)
        c.set_path(code)
        dh, ih = c.search(x, k, alive_bits=bits)
        dd, idd = search(c, x, k, bits, "device", id_offset=off, stream=st)
        c.close()
        r = fr.reference(metric, fr.BF16 if dtype == S.BF16 else fr.F32, rpath, y, x, k, alive=alive)
        check(name, r, dd, idd, f"search_device metric {metric}", id_offset=off)
        assert np.array_equal(idd, np.where(ih >= 0, ih + off, -1))
        assert np.array_equal(dd.view(np.uint32), dh.view(np.uint32))


@pytest.mark.parametrize("dtype,d", [(S.BF16, 128), (S.F32, 100)])
def test_adopt_device_equals_append(dtype, d):
    import torch
    rng = np.random.default_rng(d)
    n = 3001
    y = rng.standard_normal((n, d)).astype(F32)
    x = rng.standard_normal((24, d)).astype(F32)
    t = torch.from_numpy(y).cuda()
    if dtype == S.BF16:
        t = t.to(torch.bfloat16)
        assert np.array_equal(t.float().cpu().numpy(), to_bf16_values(y))
    t = t.contiguous()
    torch.cuda.synchronize()
    for metric in METRICS:
        for path, k in ((S.PATH_SCAN, 10), (S.PATH_TENSOR, 64)):
            a = b2.Corpus(metric, d, dtype=dtype).append(y).set_path(path)
            b = b2.Corpus(metric, d, dtype=dtype).adopt_device(t.data_ptr(), n).set_path(path)
            assert b.size == n
            da, ia = a.search(x, k)
            db, ib = b.search(x, k)
            a.close(); b.close()
            assert np.array_equal(ia, ib) and np.array_equal(da.view(np.uint32), db.view(np.uint32)), (metric, path)
    del t


# ------------------------------------------------------------------ 6. appends in chunks
@pytest.mark.parametrize("dtype", [S.F32, S.BF16])
def test_chunked_appends_equal_one_append(dtype):
    """Each append computes its rows' norms at an offset, and a growing corpus reallocates and copies its side arrays."""
    rng = np.random.default_rng(66 + dtype)
    d = 64
    chunks = [1, 255, 257, 10000]
    y = rng.standard_normal((sum(chunks), d)).astype(F32)
    x = rng.standard_normal((32, d)).astype(F32)
    for metric in METRICS:
        one = b2.Corpus(metric, d, dtype=dtype).append(y)
        many = b2.Corpus(metric, d, dtype=dtype)
        o = 0
        for m in chunks:
            many.append(y[o:o + m])
            o += m
        assert many.size == len(y)
        for path in (S.PATH_SCAN, S.PATH_TENSOR):
            one.set_path(path); many.set_path(path)
            d1, i1 = one.search(x, 50)
            d2, i2 = many.search(x, 50)
            assert np.array_equal(i1, i2) and np.array_equal(d1.view(np.uint32), d2.view(np.uint32)), (metric, path)
        one.close(); many.close()
        name = "bf16" if dtype == S.BF16 else "tf32"
        r = fr.reference(metric, fr.BF16 if dtype == S.BF16 else fr.F32, PATHS[name][0], y, x, 50)
        check(name, r, d2, i2, f"chunked appends metric {metric}")


# ------------------------------------------------------------------ 7. byte identity across schedules
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("dtype", [S.BF16, S.F32])
def test_tensor_core_schedules_are_byte_identical(dtype, metric):
    rng = np.random.default_rng(3 * metric + dtype)
    n, d, k = 5000, 64, 17
    y = rng.standard_normal((n, d)).astype(F32)
    x = rng.standard_normal((2049, d)).astype(F32)
    c = b2.Corpus(metric, d, dtype=dtype).append(y)
    c.set_path(2)
    dis, ids = c.search(x, k)
    assert c.last_variant()[0] == (S.KERNEL_GEMM_BF16 if dtype == S.BF16 else S.KERNEL_GEMM_TF32X3)

    def same(a, b, what):
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)), what

    parts = [c.search(x[o:o + m], k) for o, m in ((0, 1024), (1024, 1024), (2048, 1))]
    same((dis, ids), (np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])), "2049 vs 1024 + 1024 + 1")
    b = x[:200]
    rd, ri = c.search(b[::-1], k)
    same((dis[:200], ids[:200]), (rd[::-1], ri[::-1]), "reversed batch")
    for q in (0, 77, 199):
        same((dis[q:q + 1], ids[q:q + 1]), c.search(x[q:q + 1], k), f"query {q} alone")
    for path in range(3, 8):
        c.set_path(path)
        same((dis[:300], ids[:300]), c.search(x[:300], k), f"path code {path}")
    c.close()


@pytest.mark.parametrize("dtype", [S.F32, S.BF16])
def test_fused_scan_equals_the_staged_scan(dtype):
    """The fused single-launch form normalises cosine queries in the kernel and merges in its last block; it must give the
    same bytes as the staged form (pad, normalise, scan, merge kernels), which B200_FUSED_SCAN=0 selects at create."""
    rng = np.random.default_rng(9 + dtype)
    n, d = 20000, 100
    y = rng.standard_normal((n, d)).astype(F32)
    alive, bits = alive_mask("ragged", n, 0, rng)
    for metric in METRICS:
        fused = b2.Corpus(metric, d, dtype=dtype).append(y).set_path(1)
        os.environ["B200_FUSED_SCAN"] = "0"
        try:
            staged = b2.Corpus(metric, d, dtype=dtype).append(y).set_path(1)
        finally:
            del os.environ["B200_FUSED_SCAN"]
        for nq, k in ((1, 1), (2, 16), (4, 17), (5, 100), (8, 1024)):    # nq <= 2: queries inline (nq * d <= 256)
            x = rng.standard_normal((nq, d)).astype(F32)
            for b in (None, bits):
                n0 = S.launch_count()
                a = fused.search(x, k, alive_bits=b)
                assert S.launch_count() - n0 == 1
                n0 = S.launch_count()
                s = staged.search(x, k, alive_bits=b)
                assert S.launch_count() - n0 > 1
                assert np.array_equal(a[1], s[1]) and np.array_equal(a[0].view(np.uint32), s[0].view(np.uint32)), (metric, nq, k)
        fused.close(); staged.close()


def _fused_survivors(r, q, grid, k):
    """Candidates of query q that pass the fused tail's bound, for d_pad = 16 fp32 rows, computed from the reference keys.
    Row schedule of flat_scan_kernel at d_pad = 16: 4 lanes per row (group), 8 rows per warp step, 4 consecutive rows per
    group and step (U), 8 warps per block; the bound is the k-th smallest of the minima of the first 256 blocks."""
    rows = np.arange(r.n)
    block = ((rows // 4) % (grid * 8 * 8)) // (8 * 8)
    key = r.key[q]
    lists = []
    for b in range(grid):
        m = rows[block == b]
        lists.append(np.sort(key[m])[:k])
    mins = np.sort([l[0] for l in lists[:256] if len(l)])
    bound = mins[k - 1]
    return sum(int((l <= bound).sum()) for l in lists)


def test_fused_scan_branches():
    """The fused tail: the bound from the block minima (staged candidates, at least k blocks) with few survivors (the rank
    branch), 256 < survivors <= 1024 (the warp lists) and more than 1024 (the plain sweep); blocks of fewer than k rows (no
    bound); the query tile shrinking at large d * k.  The grid comes from last_variant, the survivor counts from the
    reference keys and the kernel's row schedule.  The queries ride in the kernel parameters where nq * d <= 256 (d = 8,
    16) and are copied at d = 4096; which form ran is not visible from outside, both are checked against the reference."""
    torch = pytest.importorskip("torch")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng(21)
    cases = [  # n, d, nq, k, rows tied with the best distance, survivors (lo, hi]
        (200000, 16, 1, 5, 0, (0, 256)),
        (200000, 16, 1, 8, 600, (256, 1024)),
        (200000, 16, 1, 8, 3000, (1024, 1 << 30)),
        (50000, 8, 2, 300, 0, None),
        (3000, 4096, 8, 1024, 0, None),
    ]
    for n, d, nq, k, tied, surv in cases:
        y = rng.standard_normal((n, d)).astype(F32)
        x = rng.standard_normal((nq, d)).astype(F32)
        for metric in (b2.L2, b2.IP):
            yy = y.copy()
            if tied:   # copies of the query (L2: distance 0) or of 3x the query (IP: far above every random row)
                yy[rng.choice(n, tied, replace=False)] = x[0] * (1 if metric == b2.L2 else 3)
            r, dis, ids = run_path("fused", metric, yy, x, k, dtype=S.F32)
            grid = LAST["variant"][3]
            check("fused", r, dis, ids, f"branch n={n} d={d} nq={nq} k={k} tied={tied}")
            if surv is not None:
                assert grid >= k and grid * k <= 8192, (grid, k)          # staged candidates, block-minima bound
                ns = _fused_survivors(r, 0, grid, k)
                assert surv[0] < ns <= surv[1], (n, k, tied, grid, ns)
            elif d == 8:
                assert grid * k > 8192 and n / grid < k, (grid, k)       # not staged; no block holds k rows: no bound
            else:
                assert grid == (2 * sms) // 8, (grid, sms)               # one query per tile: 8 tiles share 2 * SMs blocks
            if tied:   # exact ties: the smallest ids win, in ascending order
                assert np.array_equal(ids, fr.ideal_answer(r)[1]), (n, d, k, tied)


# ------------------------------------------------------------------ 8. the per-thread scratch corpus
def _quirk(dis, ids):
    keep = dis > F32(fr.FLT_MIN)
    return np.where(keep, dis, F32(fr.FLT_MIN)), np.where(keep, ids, -1)


def test_scratch_corpus_reuse_matches_fresh_corpora():
    rng = np.random.default_rng(99)
    calls = []
    for kind, metric, n, d, nq, k in (("flat", b2.L2, 3000, 64, 3, 10), ("part", b2.IP, 2000, 768, 9, 300),
                                      ("bin", b2.HAMMING, 5000, 256, 40, 12), ("flat", b2.COSINE, 9000, 17, 30, 17),
                                      ("part", b2.L2, 700, 129, 1, 1), ("flat", b2.IP, 4000, 768, 6, 100),
                                      ("bin", b2.JACCARD, 300, 128, 2, 5), ("part", b2.COSINE, 12000, 3, 25, 5),
                                      ("flat", b2.L2, 100, 1536, 64, 32)):
        if kind == "bin":
            y = rng.integers(0, 256, (n, d // 8), dtype=np.uint8)
            x = rng.integers(0, 256, (nq, d // 8), dtype=np.uint8)
        else:
            y = rng.standard_normal((n, d)).astype(F32)
            x = rng.standard_normal((nq, d)).astype(F32)
        exists = (rng.random(n) < 0.8).astype(np.uint8)
        calls.append((kind, metric, y, x, k, d, exists))

    def via_scratch(kind, metric, y, x, k, d, exists):
        if kind == "flat":
            return b2.flat_knn(metric, x, y, k, alive_bits=orc.pack_bits(exists != 0))
        if kind == "bin":
            return b2.binary_knn(metric, x, y, k)
        return b2.part_scan(metric, x, y, k, row_exists=exists)

    def via_fresh(kind, metric, y, x, k, d, exists):
        c = b2.Corpus(metric, d, dtype=S.BIN if kind == "bin" else S.F32).append(y)
        r = c.search(x, k, alive_bits=None if kind == "bin" else orc.pack_bits(exists != 0))
        c.close()
        return _quirk(*r) if kind == "part" and metric == b2.IP else r

    expect = [via_fresh(*cl) for cl in calls]
    for rnd in range(2):
        for cl, (de, ie) in zip(calls, expect):
            dg, ig = via_scratch(*cl)
            assert np.array_equal(ig, ie) and np.array_equal(dg.view(np.uint32), de.view(np.uint32)), (rnd, cl[0], cl[1], cl[5])
        assert lib().b200_thread_release() == 0


# ------------------------------------------------------------------ 9. refusals
def test_out_of_limit_k_is_refused_before_any_launch():
    rng = np.random.default_rng(1)
    y = rng.standard_normal((500, 64)).astype(F32)
    x = rng.standard_normal((4, 64)).astype(F32)
    for dtype, path, k in ((S.BF16, 2, 1025), (S.F32, 2, 1025), (S.F32, 1, 2049), (S.BF16, 1, 2049), (S.F32, 0, 2049)):
        c = b2.Corpus(b2.COSINE, 64, dtype=dtype).append(y).set_path(path)
        for entry in ("host", "device"):
            n0 = S.launch_count()
            with pytest.raises(S.B200Error) as e:
                search(c, x, k, None, entry)
            assert e.value.code == 3, e.value            # B200_ERR_UNSUPPORTED
            assert S.launch_count() == n0, (dtype, path, k, entry)
        c.close()
