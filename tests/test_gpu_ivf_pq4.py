"""PQ indexes with 4-bit codes (bit_size = 4) are scanned by table look-up from 16-entry tables (ivf_pq4_sm90.cu): checked
here against the float64 reference of the stored index (tests/pq4_reference.py, which reads the v3 file, unpacks the
nibbles and scores from the fp32 queries and the fp32 16-entry codebook), with the same 3e-5 x (sum of |terms|) tolerance
as the other scans.  The negative controls at the end show that the comparator rejects a mis-coded nibble, exchanged
nibbles and a bf16-rounded table."""
import numpy as np
import pytest

import myscaledb_b200 as b2
from tests import ivf_reference as R
from tests import pq4_reference as P
from tests.util import to_bf16_values

pytestmark = pytest.mark.gpu
F32 = np.float32
METRICS = (b2.L2, b2.IP, b2.COSINE)
ERR_INVALID, ERR_UNSUPPORTED = 1, 3
N, NLIST = 4000, 32
SHAPES = [(96, 24), (96, 96), (100, 50), (250, 10), (768, 96), (768, 384), (1536, 192), (2048, 1024)]
SMEM_LIMIT = 232448   # 227 KB of shared memory per block


def _data(n, d, seed, nq=64, n_centres=24, hot=0):
    """Clustered rows around a non-zero mean; `hot` of the queries sit around one centre (its lists get many queries)."""
    rng = np.random.default_rng(seed)
    mean = 1.0 + 0.5 * rng.standard_normal(d)
    centres = mean + rng.standard_normal((n_centres, d))
    y = centres[rng.integers(0, n_centres, n)] + 0.3 * rng.standard_normal((n, d))
    pick = np.concatenate([np.zeros(hot, np.int64), rng.integers(0, n_centres, nq - hot)])
    q = centres[pick] + 0.3 * rng.standard_normal((nq, d))
    return y.astype(F32), q.astype(F32)


def _params(m, extra=""):
    return f"ncentroids={NLIST}, bit_size=4" + (f", M={m}" if m else "") + (", " + extra if extra else "")


def _saved(ix, path):
    ix.save(path)
    return P.read_index4(path)


def _parity(s, ix, q, k, nprobe, params="", alive=None):
    dg, ig = ix.search(q, k, f"nprobe={nprobe}" + (", " + params if params else ""), first_stage_only=True,
                       alive_bits=None if alive is None else np.packbits(alive, bitorder="little"))
    ref = P.reference_search(s, q, k, nprobe, alive)
    bad = R.compare(ref, dg, ig)
    assert not bad, f"{len(bad)} problems, first: {bad[:6]}"
    return dg, ig, ref


class _Cache:
    def __init__(self, tmp):
        self.tmp, self.got = tmp, {}

    def get(self, d, m, metric, kind="IVFPQ"):
        key = (d, m, metric, kind)
        if key not in self.got:
            y, q = _data(N, d, seed=1000 * d + 10 * metric + m)
            ix = b2.VectorIndex(kind, metric, d, _params(m)).build(y)
            assert ix.info()["uses_ivf"]
            path = self.tmp / f"{kind}_{d}_{m}_{metric}.b2ix"
            s = _saved(ix, path)
            self.got[key] = (ix, s, y, q, path)
        return self.got[key]


@pytest.fixture(scope="module")
def cache(tmp_path_factory):
    return _Cache(tmp_path_factory.mktemp("pq4"))


def _same(a, b):
    return np.array_equal(a[1], b[1]) and np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------------------
# parity against the float64 reference
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,m", SHAPES)
@pytest.mark.parametrize("metric", METRICS)
def test_first_stage_parity(cache, d, m, metric):
    ix, s, y, q, _ = cache.get(d, m, metric)
    assert (s.m, s.dsub, s.code_bytes) == (m, d // m, P.code_bytes(m))
    _parity(s, ix, q, 10, 4)


@pytest.mark.parametrize("kind", ["SCANN", "IVFPQ", "HNSWPQ"])
def test_default_m_at_768(cache, kind):
    # twice the 8-bit default M = 48: the same 48 code bytes per row
    ix, s, _, q, _ = cache.get(768, 0, b2.L2, kind)
    assert ix.info()["m"] == 96 and s.dsub == 8 and s.code_bytes == 48
    _parity(s, ix, q, 10, 4)


@pytest.mark.parametrize("d,m", [(96, 24), (100, 50), (250, 10), (2048, 256)])
def test_default_m(d, m, tmp_path):
    y, q = _data(N, d, seed=d)
    ix = b2.VectorIndex("IVFPQ", b2.L2, d, _params(0)).build(y)
    assert ix.info()["m"] == m
    s = _saved(ix, tmp_path / "dflt.b2ix")
    _parity(s, ix, q[:16], 10, 4)


# ---------------------------------------------------------------------------------------------------------------------------
# edges
# ---------------------------------------------------------------------------------------------------------------------------
EDGE = [(96, 24, b2.L2), (250, 10, b2.COSINE), (768, 96, b2.IP)]


@pytest.mark.parametrize("case", EDGE)
def test_batch_shapes(cache, case):
    ix, s, _, _, _ = cache.get(*case)
    _, q = _data(N, s.d, seed=5 + s.d, nq=600, hot=300)
    for nq in (1, 17, 600):
        _parity(s, ix, q[:nq], 10, 6)
    per_list = np.bincount(R.coarse_probe(s, R.prepare_queries(q, s.metric), 6)[0].ravel(), minlength=s.nlist)
    assert per_list.max() > 128, per_list


@pytest.mark.parametrize("case", EDGE)
def test_k_edges(cache, case):
    ix, s, _, q, _ = cache.get(*case)
    for k in (1, 10, 100, 1024):
        _, ig, _ = _parity(s, ix, q[:24], k, 8)
    assert (ig == -1).any(), "k = 1024 over 8 lists should leave unfilled slots"
    with pytest.raises(b2.B200Error) as e:
        ix.search(q[:2], 1025, "nprobe=8", first_stage_only=True)
    assert e.value.code == ERR_UNSUPPORTED


@pytest.mark.parametrize("case", EDGE)
def test_nprobe_edges(cache, case):
    ix, s, _, q, _ = cache.get(*case)
    for nprobe in (1, NLIST - 1, NLIST, NLIST + 7):
        _parity(s, ix, q, 20, nprobe)


@pytest.mark.parametrize("case", EDGE)
def test_alive_bitmaps(cache, case):
    ix, s, _, q, _ = cache.get(*case)
    rng = np.random.default_rng(5)
    for frac in (0.01, 0.5, 0.0):
        alive = rng.random(N) < frac
        _, ig, _ = _parity(s, ix, q, 20, 8, alive=alive)
        assert alive[ig[ig >= 0]].all()
    assert (ig == -1).all()


def test_search_device_id_offset_and_device_bitmap(cache):
    import torch
    ix, s, _, q, _ = cache.get(100, 50, b2.L2)
    alive = np.random.default_rng(6).random(N) < 0.5
    bits = np.packbits(alive, bitorder="little")
    bits = np.concatenate([bits, np.zeros((-len(bits)) % 4, np.uint8)])
    nq, k = len(q), 20
    tq, ta = torch.from_numpy(q).cuda(), torch.from_numpy(bits).cuda()
    od = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    oi = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    ix.search_device(tq.data_ptr(), nq, k, od.data_ptr(), oi.data_ptr(), params="nprobe=8", first_stage_only=True, id_offset=1000,
                     alive_ptr=ta.data_ptr(), stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    dd, ii = od.cpu().numpy(), oi.cpu().numpy()
    dh, ih, _ = _parity(s, ix, q, k, 8, alive=alive)
    assert np.array_equal(np.where(ii >= 0, ii - 1000, -1), ih) and np.array_equal(dd, dh)


LENGTHS = (0, 1, 255, 256, 257, 511, 512, 513)


def test_page_boundaries(tmp_path):
    d, nl = 96, len(LENGTHS)
    rng = np.random.default_rng(11)
    centres = 1.0 + 8.0 * rng.standard_normal((nl, d))
    sample = (np.repeat(centres, 64, axis=0) + 0.1 * rng.standard_normal((64 * nl, d))).astype(F32)
    rows = np.concatenate([centres[c] + 0.1 * rng.standard_normal((ln, d)) for c, ln in enumerate(LENGTHS)]).astype(F32)
    rows = rows[rng.permutation(len(rows))]
    ix = b2.VectorIndex("IVFPQ", b2.L2, d, f"ncentroids={nl}, M=24, bit_size=4")
    ix.reserve(sum(LENGTHS)).train(sample)
    ix.add(rows[:700]).add(rows[700:]).finalize()
    s = _saved(ix, tmp_path / "pages.b2ix")
    assert sorted(s.list_len.tolist()) == sorted(LENGTHS), s.list_len
    q = (np.repeat(centres, 3, axis=0) + 0.1 * rng.standard_normal((3 * nl, d))).astype(F32)
    for ppc in (0, 1, 2, 3):
        for nprobe, k in ((1, 300), (3, 600)):
            _parity(s, ix, q, k, nprobe, params=f"pages_per_chunk={ppc}" if ppc else "")


def test_exact_ties_return_the_smallest_ids(tmp_path):
    d = 96
    y, _ = _data(N, d, seed=21)
    rng = np.random.default_rng(22)
    v = (1.0 + 6.0 * rng.standard_normal(d)).astype(F32)
    copies = np.sort(rng.choice(N, 300, replace=False))
    y[copies] = v
    ix = b2.VectorIndex("IVFPQ", b2.L2, d, _params(24)).build(y)
    s = _saved(ix, tmp_path / "ties.b2ix")
    lst = [l for l in range(s.nlist) if np.isin(copies, s.ids[l]).any()]
    assert len(lst) == 1 and s.list_len[lst[0]] > R.PAGE, "the copies should share one list of more than a page"
    dg, ig = ix.search(v[None, :], 10, "nprobe=4", first_stage_only=True)
    assert ig[0].tolist() == copies[:10].tolist()
    assert (dg[0] == dg[0, 0]).all()
    _parity(s, ix, v[None, :], 10, 4)


# ---------------------------------------------------------------------------------------------------------------------------
# query groups: the scan takes an item's queries G at a time, G = the largest of 8, 4, 2 whose G tables (64 M B each), G list
# pairs (16 k B each) and G candidate buffers (4 KB each) fit in half of the 227 KB (two CTAs per SM), else 1
# ---------------------------------------------------------------------------------------------------------------------------
def _smem(m, k, g):
    return g * (64 * m + -(-16 * k // 16) * 16 + 4096) + 912


def test_query_groups_of_eight(cache):
    # M = 24, k = 10: eight queries' tables, lists and buffers take 46 KB, so G = 8; the 600-query batch probes one list
    # with more than 128 queries (full groups) and the 17-query batch ends items with partial groups
    assert _smem(24, 10, 8) <= SMEM_LIMIT // 2
    ix, s, _, _, _ = cache.get(96, 24, b2.L2)
    _, q = _data(N, s.d, seed=101, nq=600, hot=300)
    r600 = _parity(s, ix, q, 10, 6)
    r17 = _parity(s, ix, q[:17], 10, 6)
    assert np.array_equal(r600[1][:17], r17[1]) and np.array_equal(r600[0][:17].view(np.uint32), r17[0].view(np.uint32))


def test_query_group_of_one_at_m_2048_k_1024(cache):
    # M = 2048 (128 KB tables) and k = 1024: two queries' tables, lists and buffers would need 296 KB, more than the 227 KB a
    # block can have, so the scan must run one query at a time (G = 1)
    assert _smem(2048, 1024, 2) > SMEM_LIMIT and _smem(2048, 1024, 1) <= SMEM_LIMIT
    ix, s, _, q, _ = cache.get(2048, 2048, b2.L2)
    _parity(s, ix, q[:20], 1024, 3)
    _parity(s, ix, q[:20], 10, 3)


# ---------------------------------------------------------------------------------------------------------------------------
# byte-identical results however the scan is cut
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", EDGE)
def test_schedule_invariance(cache, case):
    ix, s, _, q, _ = cache.get(*case)
    base = "nprobe=8"
    r0 = ix.search(q, 10, base, first_stage_only=True)
    for extra in ("pages_per_chunk=1", "pages_per_chunk=2", "pages_per_chunk=16", "shared_bound=0"):
        assert _same(r0, ix.search(q, 10, base + ", " + extra, first_stage_only=True)), extra
    alone = [ix.search(q[i:i + 1], 10, base, first_stage_only=True) for i in range(len(q))]
    assert _same(r0, (np.concatenate([a[0] for a in alone]), np.concatenate([a[1] for a in alone]))), "queries searched alone"
    dr, ir = ix.search(q[::-1].copy(), 10, base, first_stage_only=True)
    assert _same(r0, (dr[::-1], ir[::-1])), "reversed batch"


def test_table_sub_batches_at_m_2048(cache):
    # 2100 queries x 128 KB of tables exceed the 256 MB table scratch: the batch runs as two sub-batches (2048 + 52)
    ix, s, _, _, _ = cache.get(2048, 2048, b2.L2)
    _, q = _data(N, s.d, seed=77, nq=2100)
    full = ix.search(q, 10, "nprobe=4", first_stage_only=True)
    a, b = ix.search(q[:1050], 10, "nprobe=4", first_stage_only=True), ix.search(q[1050:], 10, "nprobe=4", first_stage_only=True)
    assert _same(full, (np.concatenate([a[0], b[0]]), np.concatenate([a[1], b[1]])))
    _parity(s, ix, q[2040:2060], 10, 4)   # across the sub-batch boundary (2048)


# ---------------------------------------------------------------------------------------------------------------------------
# build invariants
# ---------------------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d,m", [(100, 50), (250, 25)])   # even and odd M
def test_build_invariants_one_shot_and_streamed(metric, d, m, tmp_path):
    y, _ = _data(N, d, seed=7 + metric)
    a = b2.VectorIndex("IVFPQ", metric, d, _params(m)).build(y)
    sa = _saved(a, tmp_path / "a.b2ix")
    P.check_build(sa, a, y)
    b = b2.VectorIndex("IVFPQ", metric, d, _params(m)).reserve(N).train(y)
    off, sizes, i = 0, [1, 255, 257, 1000], 0
    while off < N:
        b.add(y[off:off + sizes[i % 4]])
        off += sizes[i % 4]
        i += 1
    b.finalize()
    # k-means training is not bitwise reproducible from run to run (8-bit indexes neither), so the two builds are held to the
    # same invariants and the same stored shape rather than compared byte for byte
    sb = _saved(b, tmp_path / "b.b2ix")
    P.check_build(sb, b, y)
    assert (sa.version, sa.m, sa.dsub, sa.code_bytes, sa.n) == (sb.version, sb.m, sb.dsub, sb.code_bytes, sb.n)


def test_last_scan_reports_the_4bit_stride(cache):
    for d, m, stride in ((768, 96, 48), (250, 10, 16), (2048, 1024, 512)):
        ix, s, _, q, _ = cache.get(d, m, b2.L2)
        ix.search(q[:4], 10, "nprobe=4", first_stage_only=True)
        ls = ix.last_scan()
        assert ls["payload_row_bytes"] == stride == s.code_bytes and ls["rows_streamed"] > 0


def test_memory_bytes_counts_the_16_entry_codebook(tmp_path):
    # A loaded index holds exactly its pages (pool = pages used).  The same rows at 4 bits (M = 24) and at 8 bits (M = 32,
    # table look-up, no bf16 copy) share the raw rows and the coarse table; what is left must be each index's lists:
    # centroids + pages x 256 x (code row + id + L2 bias) + 12 B per page + the fp32 codebook (16 or 256 entries)
    d = 96
    y, _ = _data(N, d, seed=12)
    left = []
    for bits, m, ncw in ((4, 24, 16), (8, 32, 256)):
        b2.VectorIndex("IVFPQ", b2.L2, d, f"ncentroids={NLIST}, M={m}, bit_size={bits}").build(y).save(tmp_path / f"{bits}.b2ix")
        s = (P.read_index4 if bits == 4 else R.read_index)(tmp_path / f"{bits}.b2ix")
        ix = b2.VectorIndex.load(tmp_path / f"{bits}.b2ix", d, b2.L2)
        lists = NLIST * d * 4 + s.pages_used * R.PAGE * (s.code_bytes + 8) + s.pages_used * 12 + m * ncw * (d // m) * 4
        left.append(ix.memory_bytes() - lists)
    assert left[0] == left[1] > 0, left


# ---------------------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [5, 6, 16])
@pytest.mark.parametrize("kind", ["IVFPQ", "SCANN", "HNSWPQ"])
def test_other_code_widths_are_refused(kind, bits):
    with pytest.raises(b2.B200Error) as e:
        b2.VectorIndex(kind, b2.L2, 96, f"ncentroids={NLIST}, bit_size={bits}")
    assert e.value.code == ERR_UNSUPPORTED


def test_other_types_ignore_bit_size():
    y, q = _data(N, 96, seed=3)
    ix = b2.VectorIndex("IVFFLAT", b2.L2, 96, f"ncentroids={NLIST}, bit_size=5").build(y)
    assert ix.search(q[:2], 10, "nprobe=4")[1].shape == (2, 10)


def test_m_beyond_the_limit_is_refused():
    d = 4098                                         # M = 2049 divides d; the limit is 2048
    y, _ = _data(N, d, seed=41)
    with pytest.raises(b2.B200Error) as e:
        b2.VectorIndex("IVFPQ", b2.L2, d, _params(2049)).build(y)
    assert e.value.code == ERR_UNSUPPORTED and "M <= 2048" in str(e.value), str(e.value)


# ---------------------------------------------------------------------------------------------------------------------------
# persistence
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [(96, 24, b2.L2), (250, 10, b2.COSINE), (768, 96, b2.IP)])
def test_save_load_roundtrip(cache, case, tmp_path):
    ix, s, _, q, path = cache.get(*case)
    assert s.version == 3 and s.reserved0 == 4
    d0 = ix.search(q, 10, "nprobe=8")
    re = b2.VectorIndex.load(path, s.d, case[2])
    assert re.info()["m"] == s.m
    assert _same(d0, re.search(q, 10, "nprobe=8"))
    _parity(s, re, q, 10, 8)
    re.save(tmp_path / "again.b2ix")
    assert open(path, "rb").read() == open(tmp_path / "again.b2ix", "rb").read()


def test_an_8_bit_index_still_saves_as_v2(tmp_path):
    y, _ = _data(N, 96, seed=8)
    for params in (f"ncentroids={NLIST}, M=32", f"ncentroids={NLIST}, M=32, bit_size=8"):
        b2.VectorIndex("IVFPQ", b2.L2, 96, params).build(y).save(tmp_path / "v2.b2ix")
        s = R.read_index(tmp_path / "v2.b2ix")
        assert s.version == 2 and s.reserved0 == 0 and s.codebook.shape == (32, 256, 3)


def test_truncated_and_corrupt_v3_files_are_refused(cache, tmp_path):
    _, s, _, _, path = cache.get(96, 24, b2.L2)
    raw = open(path, "rb").read()
    hdr = R.HEADER.itemsize
    codebook_at = hdr + s.n * s.d * 4 + NLIST * s.d * 4 + NLIST * 4     # rows, centroids, list lengths, then the codebook
    bad = {
        "truncated_header": raw[:hdr - 8],
        "truncated_codebook": raw[:codebook_at + 100],
        "truncated_pages": raw[:-1000],
    }

    def patch(**fields):
        h = np.frombuffer(raw[:hdr], R.HEADER, count=1).copy()
        for f, v in fields.items():
            h[f] = v
        return h.tobytes() + raw[hdr:]

    bad["width_8_in_v3"] = patch(reserved0=8)
    bad["width_0_in_v3"] = patch(reserved0=0)
    bad["code_bytes_too_small"] = patch(code_bytes=0)
    bad["code_bytes_not_16_aligned"] = patch(code_bytes=24)
    bad["m_times_dsub_not_d"] = patch(m=23)
    bad["m_above_the_limit"] = patch(d=3000, m=3000, dsub=1, code_bytes=1504)
    bad["version_4"] = patch(version=4)
    for name, blob in bad.items():
        p = tmp_path / f"{name}.b2ix"
        p.write_bytes(blob)
        with pytest.raises(b2.B200Error) as e:
            b2.VectorIndex.load(p, s.d, b2.L2)
        assert e.value.code == ERR_INVALID, name


# ---------------------------------------------------------------------------------------------------------------------------
# second stage and recall
# ---------------------------------------------------------------------------------------------------------------------------
def test_scann_refine_returns_exact_distances_of_first_stage_candidates(cache):
    ix, s, _, q, _ = cache.get(768, 0, b2.L2, "SCANN")
    dg, ig = ix.search(q, 10, "nprobe=8")
    assert ix.last_num_candidates == 160          # SCANN's default refine_factor 16
    ref = P.reference_search(s, q, 160, 8)
    Q = R.prepare_queries(q, s.metric).astype(np.float64)
    rows = s.rows.astype(np.float64)
    for qi in range(len(q)):
        if ref.flagged[qi]:
            continue
        cand = ref.cand[qi]
        edge = ref.key[qi, cand[min(160, len(cand)) - 1]]
        for j, i in enumerate(ig[qi][ig[qi] >= 0]):
            p = ref.pos_of[int(i)]
            assert ref.key[qi, p] <= edge + ref.tol[qi, p], f"q{qi}: refined id {i} was not a first-stage candidate"
            exact = ((Q[qi] - rows[i]) ** 2).sum()
            assert abs(dg[qi, j] - exact) <= 1e-5 * max(exact, 1e-30), (qi, j, dg[qi, j], exact)


def test_scann_4bit_recall_floor_at_768_clustered():
    n, d, k = 60_000, 768, 10
    rng = np.random.default_rng(3)     # the data of test_scann_recall_floor_at_768_clustered (8-bit codes)
    centres = rng.standard_normal((600, d)).astype(F32)
    y = (centres[rng.integers(0, 600, n)] + 0.3 * rng.standard_normal((n, d))).astype(F32)
    q = (centres[rng.integers(0, 600, 200)] + 0.3 * rng.standard_normal((200, d))).astype(F32)
    ix = b2.VectorIndex("SCANN", b2.L2, d, "ncentroids=256, bit_size=4").build(y)
    assert ix.info()["m"] == 96
    _, ids = ix.search(q, k, "nprobe=16")
    flat = b2.Corpus(b2.L2, d).append(y)
    _, truth = flat.search(q, k)
    flat.close()
    rec = float(np.mean([len(set(a.tolist()) & set(b.tolist())) / k for a, b in zip(ids, truth)]))
    # measured 1.000 on an H100 80GB HBM3 (700 W power limit); the floor leaves room for k-means and codebook variation
    assert rec >= 0.9, rec


# ---------------------------------------------------------------------------------------------------------------------------
# negative controls
# ---------------------------------------------------------------------------------------------------------------------------
def _top_row(s, ig):
    l = next(l for l in range(s.nlist) if (s.ids[l] == ig[0, 0]).any())
    return l, int(np.nonzero(s.ids[l] == ig[0, 0])[0][0])


def test_negative_control_swapped_nibble(cache):
    ix, s, _, q, _ = cache.get(768, 96, b2.IP)
    dg, ig, _ = _parity(s, ix, q, 10, 4)
    # one code of a returned row swapped for its second-nearest fp32 codeword (where that moves the key most)
    l, r = _top_row(s, ig)
    codes = P.unpack(s.codes[l][r:r + 1], s.m)[0]
    res = s.rows[ig[0, 0]].astype(np.float64) - s.centroids[l].astype(np.float64)
    qv = R.prepare_queries(q[:1], s.metric)[0].astype(np.float64)
    cb = s.codebook.astype(np.float64)
    best = None
    for j in range(s.m):
        dd = ((res[j * s.dsub:(j + 1) * s.dsub][None, :] - cb[j]) ** 2).sum(1)
        second = int(np.argsort(dd, kind="stable")[1])
        delta = abs(qv[j * s.dsub:(j + 1) * s.dsub] @ (cb[j, second] - cb[j, codes[j]]))
        if best is None or delta > best[0]:
            best = (delta, j, second)
    bad = s.copy()
    codes[best[1]] = best[2]
    bad.codes[l][r] = P.pack(codes[None, :], s.code_bytes)[0]
    assert R.compare(P.reference_search(bad, q, 10, 4), dg, ig), "a mis-coded sub-quantiser went unnoticed"


def test_negative_control_exchanged_nibbles(cache):
    # every byte's low and high nibbles exchanged: the reference of a packing-order bug
    ix, s, _, q, _ = cache.get(768, 96, b2.IP)
    dg, ig, _ = _parity(s, ix, q, 10, 4)
    bad = s.copy()
    bad.codes = [((c & 15) << 4 | (c >> 4)).astype(np.uint8) for c in s.codes]
    assert R.compare(P.reference_search(bad, q, 10, 4), dg, ig), "exchanged nibbles went unnoticed"


def test_negative_control_bf16_table(tmp_path):
    # Zero-mean rows, so that the residual term, not the centroid term, dominates the tolerance (with clustered data around a
    # far mean the centroid term's share of the tolerance would hide a bf16 table).
    d, m = 768, 96
    rng = np.random.default_rng(51)
    y, q = rng.standard_normal((N, d)).astype(F32), rng.standard_normal((64, d)).astype(F32)
    ix = b2.VectorIndex("IVFPQ", b2.IP, d, _params(m)).build(y)
    s = _saved(ix, tmp_path / "zero_mean.b2ix")
    dg, ig, _ = _parity(s, ix, q, 10, 4)
    assert not R.compare(P.reference_search(s, q, 10, 4, table_round=lambda t: t), dg, ig), "the table form of the reference disagrees"
    assert R.compare(P.reference_search(s, q, 10, 4, table_round=to_bf16_values), dg, ig), "a bf16 table went unnoticed"
