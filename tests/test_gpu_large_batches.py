"""Search at batch sizes beyond the launch-grid limit (65535 blocks on gridDim.y) against the references.

The FMA scan puts its query tiles (qt = 1, 4 or 8 queries) on gridDim.y, the binary scan one query per y-block and the coarse
score tiles of the inverted-file probe 64 queries per y-block; each launcher cuts a larger batch into slices.  Every case
checks three things:
  (a) the float64 / exact reference agrees on a sample of the batch that holds every query within 2 of each slice boundary,
      the first and the last query and ~1000 random ones;
  (b) the whole answer is byte for byte the concatenation of sub-batches that each stay under the limit and take the same
      path (forced path or parameters, so the kernel choice cannot change with the batch size);
  (c) the case ran the path it targets (last_variant, last_coarse, last_probe) and, for the scan, the qt that puts the
      batch past the limit (scan_qt below, a copy of the host's choice).
The last section guards paths that already cut batches into chunks (GEMM, list scans, graph walks, refine) with (b), (c)
and a light sample, and pins the inverted-file refusal of a batch with too many candidate slots.
A case is skipped when the device has too little free memory for it."""
import numpy as np
import pytest
import torch

import myscaledb_b200 as b2
from myscaledb_b200 import search as S
from myscaledb_b200.search import B200Error
from tests import flat_reference as fr
from tests import graph_reference as G
from tests import ivf_reference as R
from tests import pq4_reference as P4
from tests import pq_lut_reference as L
from tests.util import to_bf16_values

pytestmark = pytest.mark.gpu
F32 = np.float32
MAX_GRID_Y = 65535
COARSE_TILE = 64          # queries per y-block of coarse_scores_kernel (kCoarseTile, csrc/ivf.cu)
N = 4096                  # corpus rows: keeps the float64 reference cheap
STEP = 32768              # sub-batch size of check (b): under every limit, a multiple of the 1024-query GEMM chunks
ERR_UNSUPPORTED = 3


def scan_qt(nq, d_pad, k):
    """Queries per y-block of the FMA scan: a copy of the choice in search_core (csrc/capi.cu) with scan_smem_bytes
    (csrc/flat_scan.cu).  Keep in step with both: the cases below pick their shapes from it."""
    def smem(qt):
        return max(qt * d_pad * 4 + 8 * qt * k * 8, 9 * k * 8)
    qt = 1 if nq == 1 else 4 if nq <= 4 else 8
    while qt > 1 and smem(qt) > 100 * 1024:
        qt = 4 if qt == 8 else 1
    assert smem(qt) <= 200 * 1024
    return qt


def sample(nq, slice_q, seed, n_random=1000):
    """Query indices for check (a): +-2 around every multiple of slice_q inside the batch, the first and last query and
    n_random random ones."""
    s = {0, nq - 1}
    for b in range(slice_q, nq, slice_q):
        s.update(q for q in range(b - 2, b + 3) if 0 <= q < nq)
    s.update(np.random.default_rng(seed).integers(0, nq, n_random).tolist())
    return np.array(sorted(s))


def need_gb(gb):
    free = torch.cuda.mem_get_info()[0] / 2**30
    if free < gb:
        pytest.skip(f"needs ~{gb} GB of free device memory, {free:.1f} GB free")


def by_sub_batches(run, nq, step=STEP):
    parts = [run(a, min(nq, a + step)) for a in range(0, nq, step)]
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])


def assert_same(a, b, what):
    assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes(), f"{what}: differs from its sub-batches"


def flat_check(metric, dtype, y, x, dis, ids, k, slice_q, alive=None, quirk=False, id_offset=0, n_random=1000):
    qs = sample(len(x), slice_q, 7, n_random)
    r = fr.reference(metric, dtype, "scan", y, x[qs], k, alive=alive, quirk=quirk)
    bad = fr.compare(r, dis[qs], ids[qs], id_offset)
    assert not bad, f"{len(bad)} problems, first: {bad[:4]}"


def data(n, nq, d, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((n, d)).astype(F32), rng.standard_normal((nq, d)).astype(F32)


# ---------------------------------------------------------------------------------------------------------------------------
# A. the FMA scan
# ---------------------------------------------------------------------------------------------------------------------------
Y32, X32 = data(N, 70001, 32, 1)


@pytest.mark.parametrize("metric", [b2.L2, b2.IP, b2.COSINE])
@pytest.mark.parametrize("entry,nq", [("corpus", 65536), ("corpus", 70001), ("flat_knn", 70001), ("part_scan", 70001),
                                      ("device", 70001)])
def test_scan_qt1(entry, nq, metric):
    """fp32, k = 1000: always the scan, one query per y-block"""
    need_gb(4)
    k, x = 1000, X32[:nq]
    assert scan_qt(nq, 32, k) == 1 and nq > MAX_GRID_Y
    c = b2.Corpus(metric, 32).append(Y32)
    alive, quirk, off = None, entry == "part_scan" and metric == b2.IP, 0
    if entry == "device":
        alive = np.random.default_rng(3).random(N) < 0.7
        off = (1 << 32) + 5
        d_alive = torch.from_numpy(np.packbits(alive, bitorder="little")).cuda()

    def run(a, b):
        if entry == "corpus":
            return c.search(x[a:b], k)
        if entry == "flat_knn":
            return b2.flat_knn(metric, x[a:b], Y32, k)
        if entry == "part_scan":
            return b2.part_scan(metric, x[a:b], Y32, k)
        q = torch.from_numpy(x[a:b]).cuda()
        dis = torch.empty((b - a, k), dtype=torch.float32, device="cuda")
        ids = torch.empty((b - a, k), dtype=torch.int64, device="cuda")
        c.search_device(q.data_ptr(), b - a, k, dis.data_ptr(), ids.data_ptr(), id_offset=off, alive_ptr=d_alive.data_ptr())
        torch.cuda.synchronize()
        return dis.cpu().numpy(), ids.cpu().numpy()

    whole = run(0, nq)
    if entry == "corpus":
        assert c.last_variant()[0] == S.KERNEL_SCAN
    flat_check(metric, fr.F32, Y32, x, *whole, k, MAX_GRID_Y, alive=alive, quirk=quirk, id_offset=off)
    assert_same(whole, by_sub_batches(run, nq), entry)
    c.close()


def _index_rows(typ, n, params, x, k, search_params="", alive_bits=None):
    ix = b2.VectorIndex(typ, b2.L2, 32, params).build(Y32[:n])
    return ix, lambda a, b: ix.search(x[a:b], k, search_params, alive_bits=alive_bits)


@pytest.mark.parametrize("case", ["FLAT", "fallback", "exact_batch", "prefilter"])
def test_scan_qt1_index_exact_paths(case):
    """the exact paths of the index: a FLAT index, the small-part fallback of IVFFLAT, exact_batch=1 and the gathered
    (pre-filtered) corpus"""
    need_gb(4)
    k, nq, x = 1000, 70001, X32
    assert scan_qt(nq, 32, k) == 1 and nq > MAX_GRID_Y
    n, alive = N, None
    if case == "FLAT":
        ix, run = _index_rows("FLAT", N, "", x, k)
    elif case == "fallback":
        n = 1500                                          # below max(2000, 8 nlist) rows: answered by an exact scan
        ix, run = _index_rows("IVFFLAT", n, "ncentroids=16", x, k)
    elif case == "exact_batch":
        ix, run = _index_rows("IVFFLAT", N, "ncentroids=16", x, k, "exact_batch=1")
    else:
        alive = np.zeros(N, bool)
        alive[np.random.default_rng(5).choice(N, 200, replace=False)] = True
        bits = np.packbits(alive, bitorder="little")
        ix, run = _index_rows("FLAT", N, "", x, k, "prefilter=2", bits)
    whole = run(0, nq)
    probe, _ = ix.last_probe()
    assert (probe == 0).all(), "an exact pass answers"
    assert S.thread_last_rows_scored() == (200 if case == "prefilter" else n)
    flat_check(b2.L2, fr.F32, Y32[:n], x, *whole, k, MAX_GRID_Y, alive=alive)
    assert_same(whole, by_sub_batches(run, nq), case)
    ix.close()


@pytest.mark.parametrize("dtype,d,k,nq,path", [(S.F32, 32, 300, 262141, S.PATH_AUTO),        # qt = 4
                                               (S.F32, 32, 10, 524281, S.PATH_SCAN),        # qt = 8
                                               (S.BF16, 64, 10, 524281, S.PATH_SCAN),
                                               (S.BF16, 64, 2048, 65536, S.PATH_AUTO)])     # qt = 1, k past the GEMM limit
def test_scan_qt4_qt8_and_bf16(dtype, d, k, nq, path):
    need_gb(6)
    d_pad = fr.d_pad_of(dtype, d)
    qt = scan_qt(nq, d_pad, k)
    assert nq > MAX_GRID_Y * qt, (qt, nq)
    y, x = data(N, nq, d, 11)
    c = b2.Corpus(b2.L2, d, dtype=dtype).append(y).set_path(path)
    whole = c.search(x, k)
    assert c.last_variant()[0] == S.KERNEL_SCAN
    flat_check(b2.L2, dtype, y, x, *whole, k, MAX_GRID_Y * qt)
    assert_same(whole, by_sub_batches(lambda a, b: c.search(x[a:b], k), nq), f"qt={qt}")
    c.close()


def test_below_the_limit_one_scan_launch():
    """a batch at the limit launches what a small batch launches; one query tile more adds exactly one scan launch"""
    need_gb(4)
    k = 1000
    c = b2.Corpus(b2.L2, 32).append(Y32)
    counts = {}
    for nq in (1000, MAX_GRID_Y, MAX_GRID_Y + 1):
        assert scan_qt(nq, 32, k) == 1
        S.launch_count(reset=True)
        c.search(X32[:nq], k)
        counts[nq] = S.launch_count()
    assert counts[MAX_GRID_Y] == counts[1000]
    assert counts[MAX_GRID_Y + 1] == counts[1000] + 1
    c.close()


# ---------------------------------------------------------------------------------------------------------------------------
# B. the binary scan
# ---------------------------------------------------------------------------------------------------------------------------
POPC = np.array([bin(i).count("1") for i in range(256)], np.int32)


def binary_reference(metric, x, y, k):
    """exact Hamming / Jaccard keys (Jaccard rounded once to fp32, as the kernel divides), top k by (key, id)"""
    dis = np.empty((len(x), k), F32)
    ids = np.empty((len(x), k), np.int64)
    for a in range(0, len(x), 64):
        xa = x[a:a + 64, None, :]
        if metric == b2.HAMMING:
            key = POPC[xa ^ y[None]].sum(2).astype(F32)
        else:
            o, n = POPC[xa | y[None]].sum(2), POPC[xa & y[None]].sum(2)
            key = np.where(o == 0, F32(0), (o - n).astype(F32) / np.maximum(o, 1).astype(F32)).astype(F32)
        for i in range(len(key)):
            top = np.lexsort((np.arange(len(y)), key[i]))[:k]
            dis[a + i, :len(top)], ids[a + i, :len(top)] = key[i, top], top
    return dis, ids


def binary_check(metric, x, y, dis, ids, k, n_random=1000):
    qs = sample(len(x), MAX_GRID_Y, 9, n_random)
    rd, ri = binary_reference(metric, x[qs], y, k)
    assert np.array_equal(ids[qs], ri), "ids differ from the exact reference"
    assert dis[qs].tobytes() == rd.tobytes(), "distances differ from the exact reference"


YB25 = np.random.default_rng(21).integers(0, 256, (N, 25), dtype=np.uint8)
XB25 = np.random.default_rng(22).integers(0, 256, (70001, 25), dtype=np.uint8)


@pytest.mark.parametrize("metric", [b2.HAMMING, b2.JACCARD])
@pytest.mark.parametrize("entry,k,nq", [("binary_knn", 1024, 70001), ("binary_knn", 10, 65536), ("part_scan", 10, 70001),
                                        ("BINARYFLAT", 1024, 65536), ("BINARYIVF", 10, 70001)])
def test_binary_scan_25_byte_rows(entry, k, nq, metric):
    """200-bit rows are not a multiple of 16 bytes: always the scan, one query per y-block"""
    need_gb(4)
    x, y = XB25[:nq], YB25
    ix = None
    if entry == "binary_knn":
        def run(a, b):
            return b2.binary_knn(metric, x[a:b], y, k)
    elif entry == "part_scan":
        def run(a, b):
            return b2.part_scan(metric, x[a:b], y, k)
    else:
        if entry == "BINARYIVF":
            y = y[:1500]                                  # the small-part fallback: an exact scan
        ix = b2.VectorIndex(entry, metric, 200, "ncentroids=16" if entry == "BINARYIVF" else "").build(y)

        def run(a, b):
            return ix.search(x[a:b], k)
    whole = run(0, nq)
    if ix is not None:
        assert (ix.last_probe()[0] == 0).all(), "an exact pass answers"
    assert S.thread_last_rows_scored() == len(y)
    binary_check(metric, x, y, *whole, k)
    assert_same(whole, by_sub_batches(run, nq), entry)
    if ix is not None:
        ix.close()


@pytest.mark.parametrize("metric", [b2.HAMMING, b2.JACCARD])
def test_binary_scan_32_byte_rows_forced(metric):
    need_gb(4)
    k, nq = 100, 70001
    rng = np.random.default_rng(31)
    y, x = rng.integers(0, 256, (N, 32), dtype=np.uint8), rng.integers(0, 256, (nq, 32), dtype=np.uint8)
    c = b2.Corpus(metric, 256, dtype=S.BIN).append(y).set_path(S.PATH_SCAN)
    whole = c.search(x, k)
    assert c.last_variant()[0] == S.KERNEL_SCAN
    binary_check(metric, x, y, *whole, k)
    assert_same(whole, by_sub_batches(lambda a, b: c.search(x[a:b], k), nq), "32-byte rows")
    c.close()


# ---------------------------------------------------------------------------------------------------------------------------
# C / D. the coarse probe of the inverted-file indexes
# ---------------------------------------------------------------------------------------------------------------------------
def _clustered(n, nq, d, seed, n_centres=64):
    rng = np.random.default_rng(seed)
    centres = 3 * rng.standard_normal((n_centres, d))
    y = centres[rng.integers(0, n_centres, n)] + 0.5 * rng.standard_normal((n, d))
    q = centres[rng.integers(0, n_centres, nq)] + 0.5 * rng.standard_normal((nq, d))
    return y.astype(F32), q.astype(F32)


def ivf_check(stored, x, dis, ids, k, nprobe, slice_q, alive=None, n_random=1000):
    qs = sample(len(x), slice_q, 13, n_random)
    ref = R.reference_search(stored, x[qs], k, nprobe, alive)
    bad = R.compare(ref, dis[qs], ids[qs])
    assert not bad, f"{len(bad)} problems, first: {bad[:4]}"


def test_coarse_probe_on_the_scan_kernel(tmp_path):
    """nprobe = 400 of 512 centroids at d = 16 on the scan kernel: k = 400 puts it at qt = 1"""
    need_gb(8)
    nq, nprobe, k = 65536, 400, 10
    assert scan_qt(nq, 16, nprobe) == 1
    y, x = _clustered(8192, nq, 16, 41)
    ix = b2.VectorIndex("IVFFLAT", b2.L2, 16, "ncentroids=512, keep_raw=0").build(y)
    ix.save(tmp_path / "ix")
    stored = R.read_index(tmp_path / "ix")
    prm = f"nprobe={nprobe}, coarse_path=1"

    def run(a, b):
        return ix.search(x[a:b], k, prm, first_stage_only=True)
    whole = run(0, nq)
    assert ix.last_coarse() == 1
    ivf_check(stored, x, *whole, k, nprobe, MAX_GRID_Y, n_random=300)
    assert_same(whole, by_sub_batches(run, nq), "coarse_path=1")
    ix.close()


@pytest.fixture(scope="module")
def tiles_index(tmp_path_factory):
    """nlist = 16: a chunk of 2^26 / 16 queries would need 65536 coarse tiles"""
    y, x = _clustered(N, 4194304, 8, 51, n_centres=16)
    ix = b2.VectorIndex("IVFFLAT", b2.L2, 8, "ncentroids=16, keep_raw=0").build(y)
    path = tmp_path_factory.mktemp("tiles") / "ix"
    ix.save(path)
    yield ix, R.read_index(path), x
    ix.close()


def test_coarse_tiles(tiles_index):
    need_gb(6)
    ix, stored, x = tiles_index
    nq, nprobe, k = len(x), 9, 1
    assert nq > MAX_GRID_Y * COARSE_TILE

    def run(a, b):
        return ix.search(x[a:b], k, f"nprobe={nprobe}", first_stage_only=True)
    whole = run(0, nq)
    assert ix.last_coarse() == 3
    ivf_check(stored, x, *whole, k, nprobe, MAX_GRID_Y * COARSE_TILE)
    assert_same(whole, by_sub_batches(run, nq, step=1 << 21), "coarse tiles")


def test_coarse_tiles_filter_probe(tiles_index):
    """filter_probe=1 under a filter computes the coarse keys itself (the second copy of the chunk rule); every sampled
    query must equal a filtered search with nprobe = its own p_q, and the reference at that nprobe"""
    need_gb(8)
    ix, stored, x = tiles_index
    nq, nprobe, k = len(x), 9, 1
    alive = np.random.default_rng(61).random(N) < 0.3
    bits = np.packbits(alive, bitorder="little")

    def run(a, b):
        return ix.search(x[a:b], k, f"nprobe={nprobe}, filter_probe=1", first_stage_only=True, alive_bits=bits)
    whole = run(0, nq)
    probe, exact = ix.last_probe()
    assert not exact and (probe >= nprobe).all()
    qs = sample(nq, MAX_GRID_Y * COARSE_TILE, 17, 500)
    for p in np.unique(probe[qs]):
        sel = qs[probe[qs] == p]
        one = ix.search(x[sel], k, f"nprobe={p}, coarse_path=3", first_stage_only=True, alive_bits=bits)
        assert_same((whole[0][sel], whole[1][sel]), one, f"filter_probe p_q={p}")
        ref = R.reference_search(stored, x[sel], k, int(p), alive)
        bad = R.compare(ref, *one)
        assert not bad, f"{len(bad)} problems, first: {bad[:4]}"
    assert_same(whole, by_sub_batches(run, nq, step=1 << 21), "filter_probe")


# ---------------------------------------------------------------------------------------------------------------------------
# E. paths that already cut batches into chunks
# ---------------------------------------------------------------------------------------------------------------------------
NQ_E = 70001


@pytest.mark.parametrize("kind", ["bf16", "tf32", "b1"])
def test_gemm_paths(kind):
    need_gb(4)
    k = 10
    if kind == "b1":
        rng = np.random.default_rng(71)
        y, x = rng.integers(0, 256, (N, 32), dtype=np.uint8), rng.integers(0, 256, (NQ_E, 32), dtype=np.uint8)
        c = b2.Corpus(b2.HAMMING, 256, dtype=S.BIN).append(y)
    else:
        y, x = data(N, NQ_E, 64, 72)
        c = b2.Corpus(b2.IP if kind == "bf16" else b2.L2, 64, dtype=S.BF16 if kind == "bf16" else S.F32).append(y)
    whole = c.search(x, k)
    assert c.last_variant()[0] == {"bf16": S.KERNEL_GEMM_BF16, "tf32": S.KERNEL_GEMM_TF32X3, "b1": S.KERNEL_GEMM_B1}[kind]
    qs = sample(NQ_E, 1024, 73, 64)
    if kind == "b1":
        rd, ri = binary_reference(b2.HAMMING, x[qs], y, k)
        assert np.array_equal(whole[1][qs], ri) and whole[0][qs].tobytes() == rd.tobytes()
    else:
        r = fr.reference(c.metric, c.dtype, kind, y, x[qs], k)
        bad = fr.compare(r, whole[0][qs], whole[1][qs])
        assert not bad, f"{len(bad)} problems, first: {bad[:4]}"
    assert_same(whole, by_sub_batches(lambda a, b: c.search(x[a:b], k), NQ_E), kind)
    c.close()


# (index type, extra params, reader, reference search): IVFPQ at M = 8 decodes 4-dim sub-vectors on the tensor cores, at M = 2
# (16-dim sub-vectors) and with 4-bit codes it scans by table look-up, in sub-batches of queries
LIST_SCANS = {"IVFFLAT": ("IVFFLAT", "", R.read_index, R.reference_search),
              "IVFSQ": ("IVFSQ", "", R.read_index, R.reference_search),
              "IVFPQ-M8": ("IVFPQ", ", M=8", R.read_index, R.reference_search),
              "IVFPQ-lut": ("IVFPQ", ", M=2", R.read_index, L.reference_search),
              "IVFPQ-4bit": ("IVFPQ", ", M=8, bit_size=4", P4.read_index4, P4.reference_search)}


@pytest.mark.parametrize("name", list(LIST_SCANS))
def test_list_scans(name, tmp_path):
    need_gb(8)
    typ, params, read, ref_search = LIST_SCANS[name]
    k, nprobe = 10, 8
    y, x = _clustered(8192, NQ_E, 32, 81)
    ix = b2.VectorIndex(typ, b2.L2, 32, "ncentroids=64, keep_raw=0" + params).build(y)
    ix.save(tmp_path / "ix")
    stored = read(tmp_path / "ix")

    def run(a, b):
        return ix.search(x[a:b], k, f"nprobe={nprobe}", first_stage_only=True)
    whole = run(0, NQ_E)
    assert (ix.last_probe()[0] == nprobe).all()
    qs = sample(NQ_E, MAX_GRID_Y, 83, 100)
    bad = R.compare(ref_search(stored, x[qs], k, nprobe), whole[0][qs], whole[1][qs])
    assert not bad, f"{len(bad)} problems, first: {bad[:4]}"
    assert_same(whole, by_sub_batches(run, NQ_E), name)
    ix.close()


def _integer(n, nq, d, seed):
    """small integers: bf16 holds them exactly and every distance is exact in fp32 in any summation order"""
    rng = np.random.default_rng(seed)
    centres = rng.integers(-6, 7, (100, d))
    y = centres[rng.integers(0, 100, n)] + rng.integers(-1, 2, (n, d))
    q = centres[rng.integers(0, 100, nq)] + rng.integers(-1, 2, (nq, d))
    return y.astype(F32), q.astype(F32)


@pytest.fixture(scope="module")
def graph_indexes():
    y, x = _integer(20000, NQ_E, 32, 91)
    built = {}

    def get(typ):
        if typ not in built:
            built[typ] = b2.VectorIndex(typ, b2.L2, 32, "graph_degree=32").build(y)
        return built[typ], y, x
    yield get
    for ix in built.values():
        ix.close()


@pytest.mark.parametrize("width", [1, 8])
@pytest.mark.parametrize("typ", ["HNSWFLAT", "MSTG"])
def test_graph_walks(graph_indexes, typ, width):
    """HNSWFLAT and MSTG's first stage walk W parents per step, one cluster of W CTAs per query"""
    need_gb(4)
    k, ef, D = 10, 32, 32
    ix, y, x = graph_indexes(typ)
    prm = f"ef_s={ef}, search_width={width}"

    def run(a, b):
        return ix.search(x[a:b], k, prm, first_stage_only=True)
    whole = run(0, NQ_E)
    seeds = ix.last_seeds()
    assert seeds is not None and ix.last_scan()["work_items"] == NQ_E * width
    qs = sample(NQ_E, MAX_GRID_Y, 93, 32)
    rows = y if typ == "HNSWFLAT" else to_bf16_values(y)
    rd, ri, _ = G.search(ix.graph(), rows, x[qs], seeds[qs], max(ef, k), k, G.iteration_cap(D, width), "l2", None, width=width)
    assert np.array_equal(whole[1][qs], ri) and whole[0][qs].tobytes() == rd.tobytes(), "the walk differs from the reference"
    assert_same(whole, by_sub_batches(run, NQ_E), f"{typ} W={width}")


def test_refine():
    need_gb(4)
    k, kc = 10, 64
    y, x = _integer(N, NQ_E, 32, 95)
    ix = b2.VectorIndex("IVFFLAT", b2.L2, 32, "ncentroids=16").build(y)
    # distinct candidates per query (61 is prime to N), the last few unused (-1) on every other query
    cand = (np.random.default_rng(96).integers(0, N, (NQ_E, 1)) + 61 * np.arange(kc)) % N
    cand[::2, -5:] = -1
    whole = ix.refine(x, cand, k)
    qs = sample(NQ_E, MAX_GRID_Y, 97, 200)
    rd, ri = R.rerank(y, x[qs], cand[qs], k, R.L2)
    assert np.array_equal(whole[1][qs], ri) and whole[0][qs].tobytes() == rd.tobytes(), "refine differs from the reference"
    assert_same(whole, by_sub_batches(lambda a, b: ix.refine(x[a:b], cand[a:b], k), NQ_E), "refine")
    ix.close()


def test_candidate_slot_limit_is_refused_and_the_index_still_answers(tmp_path):
    """nq x nprobe x chunks x k1 >= 2^32 is refused (split the batch): 65536 x 64 x 1 x 1024; the next call is answered"""
    need_gb(8)
    y, x = _clustered(8192, 65536, 16, 99)
    ix = b2.VectorIndex("IVFFLAT", b2.L2, 16, "ncentroids=64").build(y)
    ix.save(tmp_path / "ix")
    stored = R.read_index(tmp_path / "ix")
    with pytest.raises(B200Error) as e:
        ix.search(x, 64, "nprobe=64, refine_factor=16")
    assert e.value.code == ERR_UNSUPPORTED and "split the batch" in str(e.value)
    dg, ig = ix.search(x[:256], 10, "nprobe=8", first_stage_only=True)
    bad = R.compare(R.reference_search(stored, x[:256], 10, 8), dg, ig)
    assert not bad, f"{len(bad)} problems after the refusal, first: {bad[:4]}"
    ix.close()
