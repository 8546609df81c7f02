"""The float inverted-file scans (IVFFLAT / MSTG / HNSWFLAT bf16 lists, IVFSQ / HNSWSQ 8-bit codes, IVFPQ / SCANN / HNSWPQ PQ
codes) against a float64 reference of the stored index (tests/ivf_reference.py).

Every index is built here, saved, and decoded from its file by the reference's own reader; the reference ranks every row of
the probed lists by the first-stage key of its payload.  The comparator holds each returned distance to
3e-5 x (sum of the absolute values of the key's terms): far below the effect of one wrong term, one decoded sub-quantiser or
one wrong SQ step, so a scan that skips a page, mis-decodes a code or prunes a true neighbour fails here.  The negative
controls at the end show that the comparator does reject those faults."""
import numpy as np
import pytest

import myscaledb_b200 as b2
from tests import ivf_reference as R
from tests.util import to_bf16_values

pytestmark = pytest.mark.gpu
F32 = np.float32
METRICS = (b2.L2, b2.IP, b2.COSINE)
ERR_UNSUPPORTED = 3
N, NLIST = 4000, 32

# payload -> (index type, sub-vector length for PQ)
PAYLOADS = {"bf16": ("IVFFLAT", 0), "sq8": ("IVFSQ", 0), "pq1": ("IVFPQ", 1), "pq2": ("IVFPQ", 2), "pq4": ("IVFPQ", 4),
            "pq8": ("IVFPQ", 8)}
DIMS = {"bf16": (64, 100, 192, 768), "sq8": (64, 100, 192, 768), "pq1": (64, 100, 192, 216), "pq2": (64, 100, 192, 216),
        "pq4": (64, 100, 192, 216), "pq8": (64, 192, 216)}
# every (payload, metric) pair, and every width of a payload, with the metric rotating over the widths
CASES = [(p, METRICS[(i + pi) % 3], d) for pi, p in enumerate(PAYLOADS) for i, d in enumerate(DIMS[p])]


def _data(n, d, seed, nq=64, n_centres=24, hot=0):
    """Clustered rows around a non-zero mean (so SQ's mid and the IP constants are not zero); `hot` of the queries sit
    around one centre, so that its lists are probed by many queries."""
    rng = np.random.default_rng(seed)
    mean = 1.0 + 0.5 * rng.standard_normal(d)
    centres = mean + rng.standard_normal((n_centres, d))
    y = centres[rng.integers(0, n_centres, n)] + 0.3 * rng.standard_normal((n, d))
    pick = np.concatenate([np.zeros(hot, np.int64), rng.integers(0, n_centres, nq - hot)])
    q = centres[pick] + 0.3 * rng.standard_normal((nq, d))
    return y.astype(F32), q.astype(F32)


def _params(payload, d, extra=""):
    dsub = PAYLOADS[payload][1]
    p = f"ncentroids={NLIST}" + (f", M={d // dsub}" if dsub else "")
    return p + (", " + extra if extra else "")


def _saved(ix, path):
    ix.save(path)
    return R.read_index(path)


def _assert_parity(stored, ix, q, k, nprobe, params="", alive=None, first_stage_only=True):
    dg, ig = ix.search(q, k, f"nprobe={nprobe}" + (", " + params if params else ""), first_stage_only=first_stage_only,
                       alive_bits=None if alive is None else np.packbits(alive, bitorder="little"))
    ref = R.reference_search(stored, q, k, nprobe, alive)
    bad = R.compare(ref, dg, ig)
    assert not bad, f"{len(bad)} problems, first: {bad[:6]}"
    return dg, ig, ref


class _Cache:
    def __init__(self, tmp):
        self.tmp, self.got = tmp, {}

    def get(self, payload, metric, d):
        key = (payload, metric, d)
        if key not in self.got:
            y, q = _data(N, d, seed=1000 * d + 10 * metric + len(self.got))
            ix = b2.VectorIndex(PAYLOADS[payload][0], metric, d, _params(payload, d)).build(y)
            assert ix.info()["uses_ivf"]
            path = self.tmp / f"{payload}_{metric}_{d}.b2ix"
            self.got[key] = (ix, _saved(ix, path), y, q, path)
        return self.got[key]


@pytest.fixture(scope="module")
def cache(tmp_path_factory):
    return _Cache(tmp_path_factory.mktemp("ivf_ref"))


# ---------------------------------------------------------------------------------------------------------------------------
# a. build invariants
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("payload", ["bf16", "sq8", "pq2"])
@pytest.mark.parametrize("metric", METRICS)
def test_build_invariants_one_shot_and_streamed(payload, metric, tmp_path):
    d = 100
    y, _ = _data(N, d, seed=7 + metric)
    a = b2.VectorIndex(PAYLOADS[payload][0], metric, d, _params(payload, d)).build(y)
    R.check_build(_saved(a, tmp_path / "a.b2ix"), a, y)
    # streamed: chunks of 1, 255, 257 and 1000 rows split list tails across add() calls
    b = b2.VectorIndex(PAYLOADS[payload][0], metric, d, _params(payload, d)).reserve(N).train(y)
    off, sizes = 0, [1, 255, 257, 1000]
    for i in range(N):
        if off >= N:
            break
        b.add(y[off:off + sizes[i % 4]])
        off += sizes[i % 4]
    b.finalize()
    R.check_build(_saved(b, tmp_path / "b.b2ix"), b, y)


# ---------------------------------------------------------------------------------------------------------------------------
# b. first-stage parity matrix
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("payload,metric,d", CASES)
def test_first_stage_parity(cache, payload, metric, d):
    ix, s, y, q, _ = cache.get(payload, metric, d)
    _assert_parity(s, ix, q, 10, 4)


# ---------------------------------------------------------------------------------------------------------------------------
# c. plan and epilogue edges
# ---------------------------------------------------------------------------------------------------------------------------
EDGE_INDEXES = [("bf16", b2.L2, 64), ("sq8", b2.IP, 64), ("pq1", b2.COSINE, 64)]


@pytest.mark.parametrize("case", EDGE_INDEXES)
def test_batch_shapes_split_lists_and_mix_item_kinds(cache, case):
    ix, s, y, _, _ = cache.get(*case)
    _, q = _data(N, s.d, seed=1000 * s.d + 10 * s.metric, nq=600, hot=300)   # the hot centre's lists: > 128 queries each
    for nq in (1, 16, 17, 128, 129, 600):
        _assert_parity(s, ix, q[:nq] if nq < 600 else q, 10, 6)
    per_list = np.bincount(R.coarse_probe(s, R.prepare_queries(q, s.metric), 6)[0].ravel(), minlength=s.nlist)
    assert per_list.max() > 128 and per_list[per_list > 0].min() <= 16, per_list


@pytest.mark.parametrize("case", EDGE_INDEXES)
def test_k_edges(cache, case):
    ix, s, y, q, _ = cache.get(*case)
    for k in (1, 10, 100, 256, 257, 1024):
        dg, ig, ref = _assert_parity(s, ix, q[:24], k, 8)
    assert (ig == -1).any(), "k = 1024 over 8 lists should leave unfilled slots"
    with pytest.raises(b2.B200Error) as e:
        ix.search(q[:2], 1025, "nprobe=8", first_stage_only=True)
    assert e.value.code == ERR_UNSUPPORTED


@pytest.mark.parametrize("case", EDGE_INDEXES)
def test_nprobe_edges(cache, case):
    ix, s, y, q, _ = cache.get(*case)
    for nprobe in (1, 2, NLIST - 1, NLIST, NLIST + 7):
        _assert_parity(s, ix, q, 20, nprobe)


@pytest.mark.parametrize("case", EDGE_INDEXES)
def test_alive_bitmaps(cache, case):
    ix, s, y, q, _ = cache.get(*case)
    rng = np.random.default_rng(5)
    for frac in (0.01, 0.5, 0.0):
        alive = rng.random(N) < frac
        dg, ig, _ = _assert_parity(s, ix, q, 20, 8, alive=alive)
        assert alive[ig[ig >= 0]].all()
    assert (ig == -1).all()


def test_search_device_id_offset_and_device_bitmap(cache):
    import torch
    ix, s, y, q, _ = cache.get("sq8", b2.IP, 64)
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
    dh, ih, _ = _assert_parity(s, ix, q, k, 8, alive=alive)
    assert np.array_equal(np.where(ii >= 0, ii - 1000, -1), ih) and np.array_equal(dd, dh)


# ---------------------------------------------------------------------------------------------------------------------------
# d. page geometry: lists of designed lengths
# ---------------------------------------------------------------------------------------------------------------------------
LENGTHS = (0, 1, 255, 256, 257, 511, 512, 513)


@pytest.mark.parametrize("payload", ["bf16", "sq8", "pq4"])
def test_page_boundaries(payload, tmp_path):
    d, nl = 64, len(LENGTHS)
    rng = np.random.default_rng(11)
    centres = 1.0 + 8.0 * rng.standard_normal((nl, d))
    # train on a sample ordered cluster by cluster with equal counts: the k-means seeds (rows i * n / nlist) are one per cluster
    sample = (np.repeat(centres, 64, axis=0) + 0.1 * rng.standard_normal((64 * nl, d))).astype(F32)
    rows = np.concatenate([centres[c] + 0.1 * rng.standard_normal((ln, d)) for c, ln in enumerate(LENGTHS)]).astype(F32)
    rows = rows[rng.permutation(len(rows))]
    total = sum(LENGTHS)
    assert total >= max(2000, 8 * nl)
    ix = b2.VectorIndex(PAYLOADS[payload][0], b2.L2, d, f"ncentroids={nl}" + (", M=16" if payload == "pq4" else ""))
    ix.reserve(total).train(sample)
    ix.add(rows[:700]).add(rows[700:]).finalize()
    s = _saved(ix, tmp_path / "pages.b2ix")
    assert sorted(s.list_len.tolist()) == sorted(LENGTHS), s.list_len
    q = (np.repeat(centres, 3, axis=0) + 0.1 * rng.standard_normal((3 * nl, d))).astype(F32)
    for ppc in (0, 1, 2, 3):
        for nprobe, k in ((1, 300), (3, 600)):
            _assert_parity(s, ix, q, k, nprobe, params=f"pages_per_chunk={ppc}" if ppc else "")


# ---------------------------------------------------------------------------------------------------------------------------
# e. schedule invariance: the answer does not depend on how the scan is cut into work items
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", EDGE_INDEXES)
def test_schedule_invariance(cache, case, monkeypatch):
    ix, s, y, q, _ = cache.get(*case)
    k, base = 10, "nprobe=8"
    d0, i0 = ix.search(q, k, base, first_stage_only=True)
    same = lambda d1, i1: np.array_equal(i0, i1) and np.array_equal(d0.view(np.uint32), d1.view(np.uint32))
    for extra in ("pages_per_chunk=1", "pages_per_chunk=2", "pages_per_chunk=16", "pages_per_chunk=64", "shared_bound=0"):
        assert same(*ix.search(q, k, base + ", " + extra, first_stage_only=True)), extra
    monkeypatch.setenv("B200_IVF_COOP", "0")            # read at every launch: every item on per-lane lists
    assert same(*ix.search(q, k, base, first_stage_only=True)), "B200_IVF_COOP=0"
    monkeypatch.delenv("B200_IVF_COOP")
    alone = [ix.search(q[i:i + 1], k, base, first_stage_only=True) for i in range(len(q))]
    assert same(np.concatenate([a[0] for a in alone]), np.concatenate([a[1] for a in alone])), "queries searched alone"
    dr, ir = ix.search(q[::-1].copy(), k, base, first_stage_only=True)
    assert same(dr[::-1], ir[::-1]), "reversed batch"
    flagged = R.coarse_probe(s, R.prepare_queries(q, s.metric), 8)[2]
    for cp in (1, 2, 3):
        d1, i1 = ix.search(q, k, base + f", coarse_path={cp}", first_stage_only=True)
        diff = ~((i1 == i0).all(1) & (d1 == d0).all(1))
        assert not (diff & ~flagged).any(), f"coarse_path={cp} differs on a query without a probe tie"


# ---------------------------------------------------------------------------------------------------------------------------
# f. exact ties across a page boundary
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("payload", ["bf16", "sq8", "pq4"])
def test_exact_ties_return_the_smallest_ids(payload, tmp_path):
    d = 64
    y, _ = _data(N, d, seed=21)
    rng = np.random.default_rng(22)
    v = (1.0 + 6.0 * rng.standard_normal(d)).astype(F32)       # far from the clusters: its copies form a list of their own
    copies = np.sort(rng.choice(N, 300, replace=False))
    y[copies] = v
    ix = b2.VectorIndex(PAYLOADS[payload][0], b2.L2, d, _params(payload, d)).build(y)
    s = _saved(ix, tmp_path / "ties.b2ix")
    lst = [l for l in range(s.nlist) if np.isin(copies, s.ids[l]).any()]
    assert len(lst) == 1 and s.list_len[lst[0]] > R.PAGE, "the copies should share one list of more than a page"
    dg, ig = ix.search(v[None, :], 10, "nprobe=4", first_stage_only=True)
    assert ig[0].tolist() == copies[:10].tolist()
    assert (dg[0] == dg[0, 0]).all()
    _assert_parity(s, ix, v[None, :], 10, 4)


# ---------------------------------------------------------------------------------------------------------------------------
# g. many lists: the coarse probe beyond the select kernel
# ---------------------------------------------------------------------------------------------------------------------------
def test_large_nlist_coarse_probe(tmp_path):
    d, nl = 32, 2100
    y, q = _data(20000, d, seed=31, nq=8, n_centres=400)
    ix = b2.VectorIndex("IVFFLAT", b2.L2, d, f"ncentroids={nl}").build(y)
    assert ix.info()["uses_ivf"]
    s = _saved(ix, tmp_path / "wide.b2ix")
    for nprobe in (1024, 1025, 2048):
        _assert_parity(s, ix, q, 50, nprobe)
    # 2048 < nprobe < nlist: beyond the exact centroid ranking's k limit, a clean refusal (never a CUDA error)
    with pytest.raises(b2.B200Error) as e:
        ix.search(q, 50, "nprobe=2049", first_stage_only=True)
    assert e.value.code == ERR_UNSUPPORTED and "2048" in str(e.value)


# ---------------------------------------------------------------------------------------------------------------------------
# h. two stages and persistence
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [("bf16", b2.L2, 64), ("sq8", b2.COSINE, 100), ("pq2", b2.IP, 100)])
def test_refine_takes_first_stage_candidates_and_returns_exact_distances(cache, case):
    ix, s, y, q, _ = cache.get(*case)
    dg, ig = ix.search(q, 100, "nprobe=8, refine_factor=16")
    assert ix.last_num_candidates == 1024
    ref = R.reference_search(s, q, 1024, 8)
    Q = R.prepare_queries(q, s.metric).astype(np.float64)
    rows = s.rows.astype(np.float64)
    for qi in range(len(q)):
        if ref.flagged[qi]:
            continue
        cand = ref.cand[qi]
        edge = ref.key[qi, cand[min(1024, len(cand)) - 1]]
        for j, i in enumerate(ig[qi][ig[qi] >= 0]):
            p = ref.pos_of[int(i)]
            assert ref.key[qi, p] <= edge + ref.tol[qi, p], f"q{qi}: refined id {i} was not a first-stage candidate"
            x, yv = Q[qi], rows[i]
            if s.metric == R.L2:
                exact, terms = ((x - yv) ** 2).sum(), ((x - yv) ** 2).sum()
            else:
                ip, terms = (x * yv).sum(), np.abs(x * yv).sum()
                exact = ip if s.metric == R.IP else 1 - ip
                terms += s.metric == R.COSINE
            assert abs(dg[qi, j] - exact) <= 1e-5 * max(terms, 1e-30), (qi, j, dg[qi, j], exact)


@pytest.mark.parametrize("case", [("sq8", b2.IP, 64), ("sq8", b2.COSINE, 100), ("pq2", b2.IP, 100), ("pq2", b2.COSINE, 192)])
def test_save_load_roundtrip_ip_and_cosine_code_payloads(cache, case):
    ix, s, y, q, path = cache.get(*case)
    assert not any(b is not None for b in s.bias)      # IP / cosine pages carry no row_bias
    d0, i0 = ix.search(q, 10, "nprobe=8")
    re = b2.VectorIndex.load(path, s.d, case[1])
    d1, i1 = re.search(q, 10, "nprobe=8")
    assert np.array_equal(i0, i1) and np.array_equal(d0.view(np.uint32), d1.view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------------------
# PQ widths: the scan keeps the codebook in shared memory beside a 2-stage ring, which fits up to d = 220
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("payload", ["pq1", "pq8"])
def test_pq_216_dims_search_at_k_1_and_1024(cache, payload):
    ix, s, y, q, _ = cache.get(payload, [m for p, m, d in CASES if p == payload and d == 216][0], 216)
    for k in (1, 1024):
        _assert_parity(s, ix, q[:16], k, 8)


@pytest.mark.parametrize("d", [224, 320])
def test_pq_wider_than_the_scan_is_refused_at_build(d):
    y, _ = _data(N, d, seed=41)
    with pytest.raises(b2.B200Error) as e:
        b2.VectorIndex("IVFPQ", b2.L2, d, f"ncentroids={NLIST}, M={d // 8}").build(y)
    assert e.value.code == ERR_UNSUPPORTED and "d <= 220" in str(e.value)


# ---------------------------------------------------------------------------------------------------------------------------
# i. negative controls: the comparator rejects the faults it is meant to catch
# ---------------------------------------------------------------------------------------------------------------------------
def test_negative_controls(cache):
    # one SQ code of a returned row off by one, on the dimension that weighs most in its key
    ix, s, y, q, _ = cache.get("sq8", b2.IP, 64)
    dg, ig, _ = _assert_parity(s, ix, q, 10, 4)
    bad = s.copy()
    qs = np.abs(to_bf16_values(R.prepare_queries(q[:1], s.metric) * s.sq[1]))[0]
    l, r = next((l, int(np.nonzero(bad.ids[l] == ig[0, 0])[0][0])) for l in range(s.nlist) if (bad.ids[l] == ig[0, 0]).any())
    j = int(np.argmax(qs))
    bad.codes[l][r, j] = bad.codes[l][r, j] + 1 if bad.codes[l][r, j] < 255 else 254
    assert R.compare(R.reference_search(bad, q, 10, 4), dg, ig), "a wrong SQ code went unnoticed"

    # one PQ code of a returned row swapped for its second-nearest codeword (the sub-quantiser where that matters most)
    ix, s, y, q, _ = cache.get("pq2", b2.IP, 100)
    dg, ig, _ = _assert_parity(s, ix, q, 10, 4)
    l = next(l for l in range(s.nlist) if (s.ids[l] == ig[0, 0]).any())
    r = int(np.nonzero(s.ids[l] == ig[0, 0])[0][0])
    res = s.rows[ig[0, 0]].astype(np.float64) - s.centroids[l].astype(np.float64)
    qb = to_bf16_values(R.prepare_queries(q[:1], s.metric))[0].astype(np.float64)
    cbh = to_bf16_values(s.codebook).astype(np.float64)
    best = None
    for j in range(s.m):
        dd = ((res[j * s.dsub:(j + 1) * s.dsub][None, :] - s.codebook[j].astype(np.float64)) ** 2).sum(1)
        second = int(np.argsort(dd, kind="stable")[1])
        delta = abs(qb[j * s.dsub:(j + 1) * s.dsub] @ (cbh[j, second] - cbh[j, s.codes[l][r, j]]))
        if best is None or delta > best[0]:
            best = (delta, j, second)
    bad = s.copy()
    bad.codes[l][r, best[1]] = best[2]
    assert R.compare(R.reference_search(bad, q, 10, 4), dg, ig), "a mis-decoded sub-quantiser went unnoticed"

    # the last page of one probed list dropped: a list holding one of the returned rows in its last page
    ix, s, y, q, _ = cache.get("bf16", b2.L2, 64)
    dg, ig, _ = _assert_parity(s, ix, q, 10, 4)
    for l in range(s.nlist):
        last = (len(s.ids[l]) - 1) // R.PAGE * R.PAGE
        if len(s.ids[l]) and np.isin(s.ids[l][last:], ig[0]).any():
            break
    else:
        pytest.fail("no returned row of query 0 sits in the last page of its list")
    bad = s.copy()
    bad.truncate_list(l, last)
    assert R.compare(R.reference_search(bad, q, 10, 4), dg, ig), "a skipped tail page went unnoticed"
