"""PQ indexes whose sub-vectors the tensor-core decoder cannot take (d / M outside {1, 2, 4, 8}) are scanned by table
look-up (ivf_pq_lut_sm90.cu): checked here against the float64 reference of the stored index (tests/pq_lut_reference.py, on
the reader and comparator of tests/ivf_reference.py), which scores them from the fp32 queries and the fp32 codebook, with the
same 3e-5 x (sum of |terms|) tolerance as the other scans.  The negative controls at the end show that the comparator rejects
a mis-coded row and a bf16-rounded table."""
import numpy as np
import pytest

import myscaledb_b200 as b2
from tests import ivf_reference as R
from tests import pq_lut_reference as L
from tests.util import to_bf16_values

pytestmark = pytest.mark.gpu
F32 = np.float32
METRICS = (b2.L2, b2.IP, b2.COSINE)
ERR_UNSUPPORTED = 3
N, NLIST = 4000, 32
SHAPES = [(96, 32), (100, 10), (250, 25), (768, 48), (768, 24), (1536, 96), (2048, 128)]


def _data(n, d, seed, nq=64, n_centres=24, hot=0):
    """Clustered rows around a non-zero mean; `hot` of the queries sit around one centre (its lists get many queries)."""
    rng = np.random.default_rng(seed)
    mean = 1.0 + 0.5 * rng.standard_normal(d)
    centres = mean + rng.standard_normal((n_centres, d))
    y = centres[rng.integers(0, n_centres, n)] + 0.3 * rng.standard_normal((n, d))
    pick = np.concatenate([np.zeros(hot, np.int64), rng.integers(0, n_centres, nq - hot)])
    q = centres[pick] + 0.3 * rng.standard_normal((nq, d))
    return y.astype(F32), q.astype(F32)


def _saved(ix, path):
    ix.save(path)
    return R.read_index(path)


def _parity(s, ix, q, k, nprobe, params="", alive=None):
    dg, ig = ix.search(q, k, f"nprobe={nprobe}" + (", " + params if params else ""), first_stage_only=True,
                       alive_bits=None if alive is None else np.packbits(alive, bitorder="little"))
    ref = L.reference_search(s, q, k, nprobe, alive)
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
            ix = b2.VectorIndex(kind, metric, d, f"ncentroids={NLIST}" + (f", M={m}" if m else "")).build(y)
            assert ix.info()["uses_ivf"]
            path = self.tmp / f"{kind}_{d}_{m}_{metric}.b2ix"
            s = _saved(ix, path)
            assert L.is_lut(s), (s.m, s.dsub)
            self.got[key] = (ix, s, y, q, path)
        return self.got[key]


@pytest.fixture(scope="module")
def cache(tmp_path_factory):
    return _Cache(tmp_path_factory.mktemp("pq_lut"))


# ---------------------------------------------------------------------------------------------------------------------------
# parity against the float64 reference
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,m", SHAPES)
@pytest.mark.parametrize("metric", METRICS)
def test_first_stage_parity(cache, d, m, metric):
    ix, s, y, q, _ = cache.get(d, m, metric)
    _parity(s, ix, q, 10, 4)


# ---------------------------------------------------------------------------------------------------------------------------
# edges
# ---------------------------------------------------------------------------------------------------------------------------
EDGE = [(96, 32, b2.L2), (100, 10, b2.COSINE), (768, 48, b2.IP)]


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
    ix, s, _, q, _ = cache.get(100, 10, b2.L2)
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
    ix = b2.VectorIndex("IVFPQ", b2.L2, d, f"ncentroids={nl}, M=32")
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
    ix = b2.VectorIndex("IVFPQ", b2.L2, d, f"ncentroids={NLIST}, M=32").build(y)
    s = _saved(ix, tmp_path / "ties.b2ix")
    lst = [l for l in range(s.nlist) if np.isin(copies, s.ids[l]).any()]
    assert len(lst) == 1 and s.list_len[lst[0]] > R.PAGE, "the copies should share one list of more than a page"
    dg, ig = ix.search(v[None, :], 10, "nprobe=4", first_stage_only=True)
    assert ig[0].tolist() == copies[:10].tolist()
    assert (dg[0] == dg[0, 0]).all()
    _parity(s, ix, v[None, :], 10, 4)


# ---------------------------------------------------------------------------------------------------------------------------
# byte-identical results however the scan is cut
# ---------------------------------------------------------------------------------------------------------------------------
def _same(a, b):
    return np.array_equal(a[1], b[1]) and np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32))


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


def test_query_sub_batches_at_m_128(cache):
    # 2100 queries x 128 KB of tables exceed the 256 MB table scratch: the batch runs as two sub-batches
    ix, s, _, _, _ = cache.get(2048, 128, b2.L2)
    _, q = _data(N, s.d, seed=77, nq=2100)
    full = ix.search(q, 10, "nprobe=4", first_stage_only=True)
    a, b = ix.search(q[:1050], 10, "nprobe=4", first_stage_only=True), ix.search(q[1050:], 10, "nprobe=4", first_stage_only=True)
    assert _same(full, (np.concatenate([a[0], b[0]]), np.concatenate([a[1], b[1]])))
    _parity(s, ix, q[2040:2060], 10, 4)   # across the sub-batch boundary (2048)


# ---------------------------------------------------------------------------------------------------------------------------
# build invariants
# ---------------------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("metric", METRICS)
def test_build_invariants_one_shot_and_streamed(metric, tmp_path):
    d, m = 100, 10
    y, _ = _data(N, d, seed=7 + metric)
    a = b2.VectorIndex("IVFPQ", metric, d, f"ncentroids={NLIST}, M={m}").build(y)
    sa = _saved(a, tmp_path / "a.b2ix")
    L.check_build(sa, a, y)
    b = b2.VectorIndex("IVFPQ", metric, d, f"ncentroids={NLIST}, M={m}").reserve(N).train(y)
    off, sizes, i = 0, [1, 255, 257, 1000], 0
    while off < N:
        b.add(y[off:off + sizes[i % 4]])
        off += sizes[i % 4]
        i += 1
    b.finalize()
    L.check_build(_saved(b, tmp_path / "b.b2ix"), b, y)


# ---------------------------------------------------------------------------------------------------------------------------
# defaults and refusals
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["SCANN", "IVFPQ", "HNSWPQ"])
def test_default_m_at_768(cache, kind):
    ix, s, _, q, _ = cache.get(768, 0, b2.L2, kind)
    assert ix.info()["m"] == 48 and s.dsub == 16
    _parity(s, ix, q, 10, 4)


def test_m_beyond_the_table_limit_is_refused():
    y, _ = _data(N, 1548, seed=41)
    with pytest.raises(b2.B200Error) as e:
        b2.VectorIndex("IVFPQ", b2.L2, 1548, f"ncentroids={NLIST}, M=129").build(y)
    assert e.value.code == ERR_UNSUPPORTED and "M <= 128" in str(e.value), str(e.value)


# ---------------------------------------------------------------------------------------------------------------------------
# second stage and persistence
# ---------------------------------------------------------------------------------------------------------------------------
def test_scann_refine_returns_exact_distances_of_first_stage_candidates(cache):
    ix, s, _, q, _ = cache.get(768, 0, b2.L2, "SCANN")
    dg, ig = ix.search(q, 10, "nprobe=8")
    assert ix.last_num_candidates == 160          # SCANN's default refine_factor 16
    ref = L.reference_search(s, q, 160, 8)
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


@pytest.mark.parametrize("case", [(96, 32, b2.L2), (250, 25, b2.COSINE), (768, 48, b2.IP)])
def test_save_load_roundtrip(cache, case):
    ix, s, _, q, path = cache.get(*case)
    d0 = ix.search(q, 10, "nprobe=8")
    re = b2.VectorIndex.load(path, s.d, case[2])
    assert re.info()["m"] == s.m
    assert _same(d0, re.search(q, 10, "nprobe=8"))
    _parity(s, re, q, 10, 8)


def test_scann_recall_floor_at_768_clustered():
    n, d, k = 60_000, 768, 10
    rng = np.random.default_rng(3)     # the clustered() shape of tools/bench_aux.py: unit-normal centres, spread 0.3
    centres = rng.standard_normal((600, d)).astype(F32)
    y = (centres[rng.integers(0, 600, n)] + 0.3 * rng.standard_normal((n, d))).astype(F32)
    q = (centres[rng.integers(0, 600, 200)] + 0.3 * rng.standard_normal((200, d))).astype(F32)
    ix = b2.VectorIndex("SCANN", b2.L2, d, "ncentroids=256").build(y)
    assert ix.info()["m"] == 48
    _, ids = ix.search(q, k, "nprobe=16")
    flat = b2.Corpus(b2.L2, d).append(y)
    _, truth = flat.search(q, k)
    flat.close()
    rec = float(np.mean([len(set(a.tolist()) & set(b.tolist())) / k for a, b in zip(ids, truth)]))
    # measured 1.000 on an H100 80GB HBM3 (400 W power limit); the floor leaves room for k-means and codebook variation
    assert rec >= 0.9, rec


# ---------------------------------------------------------------------------------------------------------------------------
# negative controls
# ---------------------------------------------------------------------------------------------------------------------------
def test_negative_control_swapped_code(cache):
    ix, s, _, q, _ = cache.get(768, 48, b2.IP)
    dg, ig, _ = _parity(s, ix, q, 10, 4)
    # one code of a returned row swapped for its second-nearest fp32 codeword (where that moves the key most)
    l = next(l for l in range(s.nlist) if (s.ids[l] == ig[0, 0]).any())
    r = int(np.nonzero(s.ids[l] == ig[0, 0])[0][0])
    res = s.rows[ig[0, 0]].astype(np.float64) - s.centroids[l].astype(np.float64)
    qv = R.prepare_queries(q[:1], s.metric)[0].astype(np.float64)
    cb = s.codebook.astype(np.float64)
    best = None
    for j in range(s.m):
        dd = ((res[j * s.dsub:(j + 1) * s.dsub][None, :] - cb[j]) ** 2).sum(1)
        second = int(np.argsort(dd, kind="stable")[1])
        delta = abs(qv[j * s.dsub:(j + 1) * s.dsub] @ (cb[j, second] - cb[j, s.codes[l][r, j]]))
        if best is None or delta > best[0]:
            best = (delta, j, second)
    bad = s.copy()
    bad.codes[l][r, best[1]] = best[2]
    assert R.compare(L.reference_search(bad, q, 10, 4), dg, ig), "a mis-coded sub-quantiser went unnoticed"



def test_negative_control_bf16_table(tmp_path):
    # An index scored with a bf16-rounded table: the scan's fp32 table is what the comparator holds it to.  Zero-mean rows, so
    # that the residual term, not the centroid term, dominates the tolerance (with clustered data around a far mean the
    # centroid term's share of the tolerance would hide a bf16 table).
    d, m = 768, 48
    rng = np.random.default_rng(51)
    y, q = rng.standard_normal((N, d)).astype(F32), rng.standard_normal((64, d)).astype(F32)
    ix = b2.VectorIndex("IVFPQ", b2.IP, d, f"ncentroids={NLIST}, M={m}").build(y)
    s = _saved(ix, tmp_path / "zero_mean.b2ix")
    dg, ig, _ = _parity(s, ix, q, 10, 4)
    assert not R.compare(L.reference_search(s, q, 10, 4, table_round=lambda t: t), dg, ig), "the table form of the reference disagrees"
    assert R.compare(L.reference_search(s, q, 10, 4, table_round=to_bf16_values), dg, ig), "a bf16 table went unnoticed"
