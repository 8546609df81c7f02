"""Unusable rows and queries on the float indexes (include/b200_search.h, "Unusable rows").

A row or query is unusable when the fp32 sum of the squares of its coordinates is not finite: a NaN or infinite coordinate,
or one whose square overflows.  A ClickHouse Float32 column can hold such values, and nothing before the index removes them.
Checked here, against tests/ivf_reference.py, tests/train_reference.py and tests/graph_reference.py:
  * the stored index: every usable row in its nearest list exactly once, every unusable one in none (its row id and fp32 row
    kept), for every build style (one-shot build, reserve / train on a clean sample / add dirty chunks, train on a dirty
    sample, train_device / add_device from torch);
  * training: centroids, SQ ranges and PQ codebooks equal the reference trained on the usable rows of the sample alone, and
    are finite (one -inf in an SQ sample made every query constant NaN);
  * search: no unusable id ever, min(k, usable rows) filled slots when every list is probed, the first stage against the
    float64 reference, filter_probe's promise and depths under a filter that keeps mostly unusable rows;
  * graphs: rows in no list have empty adjacency rows, no edge reaches them, the graph is the reference's;
  * queries: NaN queries (and infinite ones under L2 / cosine) return nothing, and change no other query's answer, byte for
    byte, at the positions that split the 128-query work items of a 1025-query batch;
  * cosine rows and queries of zero or tiny norm (below FLT_EPSILON) are usable and kept as given;
  * persistence: save / load answer byte-identically (v2, v3, v4 files), and load refuses list lengths above n and an MSTG
    graph edge to a row in no list;
  * the exact paths (exact_batch=1, the small-part fallback) keep FLAT's rule;
  * the default look-up scan at d = 768, build()'s strided training sample, and the HNSWFLAT walk against its reference."""
import numpy as np
import pytest

import myscaledb_b200 as b2
from myscaledb_b200.search import B200Error
from tests import graph_reference as G
from tests import ivf_reference as R
from tests import pq4_reference as P4
from tests import pq_lut_reference as L
from tests import train_reference as T
from tests.test_gpu_index_filtered import _fp64_depth
from tests.test_gpu_index_widths import _check_refined

pytestmark = pytest.mark.gpu
F32 = np.float32
N, D, NLIST, NPROBE, NC = 50000, 64, 256, 16, 32
RUN = (10100, 10400)   # 300 consecutive unusable ids across the 256-row boundary at 10240
NAN, INF = np.float32(np.nan), np.float32(np.inf)

# name -> (type, metric, params, how the stored file is checked: "build" ivf_reference's check_build and reference_search,
# "lut" / "pq4" those of pq_lut_reference / pq4_reference (the look-up scans of ivf_pq_lut_sm90.cu / ivf_pq4_sm90.cu, the
# latter from a v3 file), "ref" ivf_reference's reference_search and check_lists only (anisotropic codes are not the nearest
# codewords; keep_raw=0 stores no fp32 rows), None: a v4 graph file, checked through the graph instead)
INDEXES = {
    "ivfflat": ("IVFFLAT", b2.L2, "", "build"),
    "ivfsq": ("IVFSQ", b2.IP, "", "build"),
    "hnswsq": ("HNSWSQ", b2.COSINE, "", "build"),
    "ivfpq_d8": ("IVFPQ", b2.COSINE, "M=8", "build"),
    "scann_lut": ("SCANN", b2.L2, "M=4", "lut"),
    "scann_4bit": ("SCANN", b2.IP, "M=16, bit_size=4", "pq4"),
    "ivfpq_aq": ("IVFPQ", b2.IP, "M=8, aq_threshold=0.2", "ref"),
    "mstg_raw0": ("MSTG", b2.L2, "keep_raw=0", "ref"),
    "mstg_raw1": ("MSTG", b2.IP, "keep_raw=1", "build"),
    "mstg_raw2": ("MSTG", b2.COSINE, "keep_raw=2", "build"),
    "hnswflat_g16": ("HNSWFLAT", b2.L2, "graph_degree=16", None),
    "mstg_g16": ("MSTG", b2.IP, "graph_degree=16", None),
}
GRAPHS = ("hnswflat_g16", "mstg_g16")


def _spoil(y, rows, rng):
    """Makes rows unusable, cycling through the kinds: whole-row NaN, one NaN, +inf, -inf, mixed +-inf, one 1e20 (its square
    overflows)."""
    d = y.shape[1]
    for t, r in enumerate(rows):
        j = int(rng.integers(0, d))
        kind = t % 6
        if kind == 0:
            y[r] = NAN
        elif kind == 1:
            y[r, j] = NAN
        elif kind == 2:
            y[r, j] = INF
        elif kind == 3:
            y[r, j] = -INF
        elif kind == 4:
            y[r, j], y[r, (j + 1) % d] = INF, -INF
        else:
            y[r, j] = 1e20


def _data(seed, n=N, d=D, nl=NLIST, nq=1025):
    """Clustered rows with unusable ones on the k-means seed rows floor(i n / nlist) (build() trains on every row here), in
    the id run RUN and at several hundred random places, and zero / tiny-norm rows; clustered queries."""
    rng = np.random.default_rng(seed)
    mean = 1.0 + 0.5 * rng.standard_normal(d)
    centres = mean + 2.0 * rng.standard_normal((NC, d))
    y = (centres[rng.integers(0, NC, n)] + 0.5 * rng.standard_normal((n, d))).astype(F32)
    q = (centres[rng.integers(0, NC, nq)] + 0.5 * rng.standard_normal((nq, d))).astype(F32)
    bad = np.unique(np.concatenate([T.strided(n, nl), np.arange(*RUN), rng.choice(n, 400, replace=False)]))
    _spoil(y, bad, rng)
    free = np.setdiff1d(np.arange(n), bad)
    small = rng.choice(free, 40, replace=False)
    y[small[:20]] = 0.0
    y[small[20:]] = (1e-6 * rng.standard_normal((20, d))).astype(F32)   # sum of squares ~6e-11 < FLT_EPSILON
    assert (R.usable(y) == ~np.isin(np.arange(n), bad)).all()
    return y, q


def _bad_queries(q, rng):
    """q with unusable queries at 0, 127, 128 (the edges of the 128-query work items) and the last position: NaN, one NaN,
    +inf, -inf; returns (queries, positions, which are NaN)."""
    q = q.copy()
    pos = np.array([0, 127, 128, len(q) - 1])
    q[0] = NAN
    q[127, 5] = NAN
    q[128, 9] = INF
    q[-1, 3] = -INF
    return q, pos, np.array([True, True, False, False])


class _Cache:
    def __init__(self, tmp):
        self.tmp, self.got = tmp, {}
        self.y, self.q = _data(3)
        self.ok = R.usable(self.y)

    def get(self, name):
        if name not in self.got:
            ty, metric, params, how = INDEXES[name]
            ix = b2.VectorIndex(ty, metric, D, f"ncentroids={NLIST}, " + params).build(self.y)
            assert ix.info()["uses_ivf"] and ix.info()["n"] == N
            s = None
            if how:
                path = self.tmp / f"{name}.b2ix"
                ix.save(path)
                s = _reader(how)(path)
            self.got[name] = (ix, s)
        return self.got[name]


@pytest.fixture(scope="module")
def cache(tmp_path_factory):
    return _Cache(tmp_path_factory.mktemp("nonfinite"))


def _no_bad_ids(ids, ok):
    got = ids[ids >= 0]
    assert ok[got].all(), f"unusable rows returned: {sorted(set(got[~ok[got]].tolist()))[:8]}"


def _full(ids, want):
    filled = (ids >= 0).sum(1)
    assert (filled == want).all(), f"{int((filled != want).sum())} of {len(ids)} queries fill {filled.min()}..{filled.max()} slots, want {want}"


def _reader(how):
    return P4.read_index4 if how == "pq4" else R.read_index


def _ref(how):
    """The reference module of a stored index's first stage."""
    return {"lut": L, "pq4": P4}.get(how, R)


def _check_stored(how, s, ix, y):
    if how == "ref":
        if s.has_raw:
            R.check_lists(s, ix, y)
    else:
        _ref(how).check_build(s, ix, y)


def _assert_first_stage(how, s, q, k, nprobe, dg, ig, alive=None):
    bad = R.compare(_ref(how).reference_search(s, q, k, nprobe, alive), dg, ig)
    assert not bad, f"nprobe={nprobe}: {len(bad)} problems, first: {bad[:4]}"


def _assert_depths(how, s, q, k, p, alive, dg, ig):
    """filter_probe=1: the depths against the float64 recomputation from the stored lists (a difference only at a near-tie of
    the coarse keys), and each group of queries with one depth against the reference probing that many lists."""
    Q = R.prepare_queries(q, s.metric)
    want = _fp64_depth(s, Q, alive, k, NPROBE, NLIST)
    for i in np.nonzero(want != p)[0]:
        flagged = [R.coarse_probe(s, Q[i:i + 1], int(v))[2][0] for v in (want[i], p[i])]
        assert any(flagged), f"query {i}: depth {p[i]}, fp64 {want[i]} without a near-tie at the cut"
    for pv in np.unique(p):
        g = np.nonzero(p == pv)[0]
        _assert_first_stage(how, s, q[g], k, int(pv), dg[g], ig[g], alive)


def _two_stage(name):
    return INDEXES[name][0] not in ("IVFFLAT", "HNSWFLAT") and "keep_raw=0" not in INDEXES[name][2]


# ---------------------------------------------------------------------------------------------------------------------------
# the stored index and the searches of a one-shot build
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(INDEXES))
def test_stored_index(cache, name):
    ix, s = cache.get(name)
    sizes = ix.list_sizes()
    assert int(sizes.sum()) == int(cache.ok.sum()), "list sizes must add up to the usable rows"
    if s is None:
        return
    ids, _, _ = s.flat()
    assert np.array_equal(np.sort(ids), np.nonzero(cache.ok)[0])
    _check_stored(INDEXES[name][3], s, ix, cache.y)


@pytest.mark.parametrize("name", list(INDEXES))
def test_search_never_returns_an_unusable_row(cache, name):
    ix, s = cache.get(name)
    q, k = cache.q[:64], 100
    usable_rows = int(cache.ok.sum())
    lists = f"nprobe={NLIST}" + (", graph=0" if name in GRAPHS else "")   # every list, also on the graph types
    runs = [(lists, False)]
    if _two_stage(name):
        runs.append((lists, True))
    if name in GRAPHS:
        runs.append(("", False))   # the graph walk
    for params, fso in runs:
        dg, ig = ix.search(q, k, params, first_stage_only=fso)
        _no_bad_ids(ig, cache.ok)
        _full(ig, min(k, usable_rows))
        assert np.isfinite(dg[ig >= 0]).all()
    if s is None:
        return
    how = INDEXES[name][3]
    for nprobe in (NPROBE, NLIST):
        dg, ig = ix.search(q, k, f"nprobe={nprobe}", first_stage_only=True)
        _assert_first_stage(how, s, q, k, nprobe, dg, ig)
    if _two_stage(name):   # the exact second stage of the first stage's k x refine_factor candidates
        k, rf = 10, 8
        _, cand = ix.search(q, k * rf, f"nprobe={NPROBE}", first_stage_only=True)
        dg, ig = ix.search(q, k, f"nprobe={NPROBE}, refine_factor={rf}")
        assert ix.last_num_candidates == k * rf
        _no_bad_ids(ig, cache.ok)
        _check_refined(s, q, cand, dg, ig, k)


@pytest.mark.parametrize("name", [n for n in INDEXES if n not in GRAPHS])
def test_filter_probe_counts_only_rows_in_a_list(cache, name):
    ix, s = cache.get(name)
    rng = np.random.default_rng(len(name))
    alive = ~cache.ok
    alive[rng.choice(np.nonzero(cache.ok)[0], 5, replace=False)] = True
    bits = np.packbits(alive, bitorder="little")
    q, k = cache.q[:64], 10
    want = min(k, int((alive & cache.ok).sum()))
    for fso in (False, True):
        dg, ig = ix.search(q, k, f"nprobe={NPROBE}, filter_probe=1", first_stage_only=fso, alive_bits=bits)
        _no_bad_ids(ig, cache.ok)
        _full(ig, want)
        assert alive[ig[ig >= 0]].all()
    p, exact = ix.last_probe()
    assert not exact
    if s is None:
        return
    _assert_depths(INDEXES[name][3], s, q, k, p, alive, dg, ig)
    if _two_stage(name):
        # the whole answer: the exact second stage of the first stage's k1 = k x refine_factor candidates, whose depths are
        # those of a first-stage search for k1
        rf = 8
        _, cand = ix.search(q, k * rf, f"nprobe={NPROBE}, filter_probe=1", first_stage_only=True, alive_bits=bits)
        dg, ig = ix.search(q, k, f"nprobe={NPROBE}, filter_probe=1, refine_factor={rf}", alive_bits=bits)
        _full(ig, want)
        _check_refined(s, q, cand, dg, ig, k)


# ---------------------------------------------------------------------------------------------------------------------------
# build styles
# ---------------------------------------------------------------------------------------------------------------------------
STYLES = ("train_clean_add_dirty", "train_dirty", "device")


@pytest.mark.parametrize("name", ["ivfsq", "ivfpq_d8", "mstg_raw1", "scann_lut"])
@pytest.mark.parametrize("style", STYLES)
def test_build_styles(cache, name, style, tmp_path):
    ty, metric, params, how = INDEXES[name]
    y, ok = cache.y, cache.ok
    ix = b2.VectorIndex(ty, metric, D, f"ncentroids={NLIST}, " + params).reserve(N)
    if style == "device":
        torch = pytest.importorskip("torch")
        t = torch.from_numpy(y).cuda()
        ix.train_device(t.data_ptr(), N)
        for a in range(0, N, 12345):
            ix.add_device(t[a:a + 12345].data_ptr(), min(12345, N - a))
        torch.cuda.synchronize()
    else:
        ix.train(y[ok][::3] if style == "train_clean_add_dirty" else y[::2])
        for a in range(0, N, 12345):
            ix.add(y[a:a + 12345])
    ix.finalize()
    assert ix.info()["uses_ivf"] and ix.info()["n"] == N
    assert int(ix.list_sizes().sum()) == int(ok.sum())
    q, k = cache.q[:64], 50
    dg, ig = ix.search(q, k, f"nprobe={NLIST}")
    _no_bad_ids(ig, ok)
    _full(ig, k)
    ix.save(tmp_path / "ix.b2ix")
    s = _reader(how)(tmp_path / "ix.b2ix")
    _check_stored(how, s, ix, y)
    dg, ig = ix.search(q, k, f"nprobe={NPROBE}", first_stage_only=True)
    _assert_first_stage(how, s, q, k, NPROBE, dg, ig)


# ---------------------------------------------------------------------------------------------------------------------------
# training on the usable rows of the sample
# ---------------------------------------------------------------------------------------------------------------------------
def _dirty_sample(seed, n_good, d, nl, nbad):
    """A separated-cluster sample whose usable rows are the reference's input; the unusable ones sit on the seed rows
    floor(i n / nl) of the whole sample and at random places, so training on every row would seed on them."""
    from tests.test_gpu_index_train import separated

    rng = np.random.default_rng(seed)
    good, _ = separated(rng, n_good, d, nl)
    n = n_good + nbad
    bad = np.zeros(n, bool)
    bad[T.strided(n, nl)[:nbad]] = True
    rest = nbad - int(bad.sum())
    if rest:
        bad[rng.choice(np.nonzero(~bad)[0], rest, replace=False)] = True
    y = np.zeros((n, d), F32)
    y[~bad] = good
    _spoil(y, np.nonzero(bad)[0], rng)
    return y, good


@pytest.mark.parametrize("metric", [b2.L2, b2.IP, b2.COSINE])
def test_coarse_kmeans_trains_on_usable_rows(metric, tmp_path):
    nl, d = 64, 17
    y, good = _dirty_sample(21 + metric, 3001, d, nl, 100)
    ix = b2.VectorIndex("IVFFLAT", metric, d, f"ncentroids={nl}").reserve(len(y)).train(y).add(y).finalize()
    ix.save(tmp_path / "ix.b2ix")
    s = R.read_index(tmp_path / "ix.b2ix")
    assert np.isfinite(s.centroids).all()
    t = T.kmeans(T.train_rows(good, metric), nl, 10)
    assert not t.ambiguous, t.why
    bad = T.centroid_problems(s.centroids, t)
    assert not bad, bad
    R.check_build(s, ix, y)


@pytest.mark.parametrize("metric", [b2.L2, b2.IP])
def test_sq_ranges_ignore_an_infinite_coordinate(metric, tmp_path):
    """One -inf in a column of the sample made step = inf and mid = NaN, so every query's constant was NaN."""
    nl, d = 16, 32
    rng = np.random.default_rng(31)
    good = (rng.standard_normal((4000, d)) + 3.0 * rng.standard_normal((nl, d))[rng.integers(0, nl, 4000)]).astype(F32)
    y = good.copy()
    y[1234, 7] = -INF
    ok = R.usable(y)
    ix = b2.VectorIndex("IVFSQ", metric, d, f"ncentroids={nl}").build(y)
    ix.save(tmp_path / "ix.b2ix")
    s = R.read_index(tmp_path / "ix.b2ix")
    assert np.isfinite(s.sq).all()
    bad = T.sq_problems(s.sq, y[ok])
    assert not bad, bad
    R.check_build(s, ix, y)
    q = good[:50] + 0.1
    dg, ig = ix.search(q, 10, f"nprobe={nl}")
    _full(ig, 10)
    assert ok[ig].all() and np.isfinite(dg).all()


@pytest.mark.parametrize("d,m,bits", [(16, 8, 8), (16, 8, 4)])
def test_pq_codebooks_train_on_usable_rows(d, m, bits, tmp_path):
    from tests import pq4_reference as P4
    from tests.test_gpu_index_train import pq_data

    rng = np.random.default_rng(d * m + bits)
    ncw = 16 if bits == 4 else 256
    good = pq_data(rng, 4096, d, d // m, ncw)
    n = len(good) + 60
    bad = np.zeros(n, bool)
    bad[T.strided(n, 2)] = True
    bad[rng.choice(np.nonzero(~bad)[0], 58, replace=False)] = True
    y = np.zeros((n, d), F32)
    y[~bad] = good
    _spoil(y, np.nonzero(bad)[0], rng)
    ix = b2.VectorIndex("IVFPQ", b2.L2, d, f"ncentroids=2, M={m}, bit_size={bits}")
    ix.reserve(n).train(y).add(y).finalize()
    assert int(ix.list_sizes().sum()) == len(good)
    path = tmp_path / "ix.b2ix"
    ix.save(path)
    s = (P4.read_index4 if bits == 4 else R.read_index)(path)
    assert np.isfinite(s.centroids).all() and np.isfinite(s.codebook).all()
    t = T.kmeans(good, 2, 10)
    assert not t.ambiguous, t.why
    assert not T.centroid_problems(s.centroids, t)
    p = T.pq_codebooks(good, s.centroids, m, bits)
    assert not p.ambiguous
    bad = T.codebook_problems(s.codebook, p)
    assert not bad, bad[:4]


def test_too_few_usable_rows_fall_back_to_flat(cache):
    y = cache.y[:4000].copy()
    y[200:] = NAN   # at most 200 usable rows: below max(2000, 8 nlist)
    ix = b2.VectorIndex("IVFFLAT", b2.L2, D, "ncentroids=64").reserve(0).train(y).add(y).finalize()
    assert not ix.info()["uses_ivf"]
    dg, ig = ix.search(y[:5] + 0.0, 10)
    _no_bad_ids(ig, R.usable(y))


# ---------------------------------------------------------------------------------------------------------------------------
# graphs
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", GRAPHS)
def test_graph_leaves_out_rows_in_no_list(cache, name):
    ix, _ = cache.get(name)
    g = ix.graph()
    Dg = g.shape[1]
    bad = ~cache.ok
    assert (g[bad] == G.NO_ID).all(), "a row in no list has edges"
    e = g[g != G.NO_ID].astype(np.int64)
    assert not bad[e].any(), "an edge reaches a row in no list"
    mstg = INDEXES[name][0] == "MSTG"
    _, ids = ix.search(cache.y, 2 * Dg + 1, "graph=0", first_stage_only=mstg)
    ids[bad] = -1
    want = G.build(G.candidates(ids), Dg)
    assert np.array_equal(g, want), f"{int((g != want).any(1).sum())} graph rows differ from the reference"


# ---------------------------------------------------------------------------------------------------------------------------
# queries
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(INDEXES))
def test_unusable_queries(cache, name):
    ix, _ = cache.get(name)
    metric = INDEXES[name][1]
    rng = np.random.default_rng(9)
    qb, pos, is_nan = _bad_queries(cache.q, rng)
    others = np.setdiff1d(np.arange(len(qb)), pos)
    lists = ", graph=0" if name in GRAPHS else ""
    runs = [(f"nprobe={NPROBE}" + lists, False), (f"nprobe={NLIST}" + lists, False)]
    if _two_stage(name):
        runs.append((f"nprobe={NPROBE}" + lists, True))
    if name in GRAPHS:
        runs.append(("", False))   # the graph walk
    for params, fso in runs:
        for k in (10, 100):
            clean = ix.search(cache.q, k, params, first_stage_only=fso)
            dg, ig = ix.search(qb, k, params, first_stage_only=fso)
            assert dg[others].tobytes() == clean[0][others].tobytes(), f"{params}, k={k}: a bad query changed another's distances"
            assert ig[others].tobytes() == clean[1][others].tobytes(), f"{params}, k={k}: a bad query changed another's ids"
            empty = pos[is_nan] if metric == b2.IP else pos
            assert (ig[empty] == -1).all(), f"{params}, k={k}: an unusable query returned rows"
            _no_bad_ids(ig, cache.ok)


@pytest.mark.parametrize("name", ["ivfflat", "ivfsq", "ivfpq_d8", "hnswsq", "mstg_raw2", "mstg_g16"])
def test_cosine_tiny_queries(cache, name):
    """Zero and tiny-norm queries are usable: they stay as given (no normalisation), their key is 1 - <q, x>."""
    ix, s = cache.get(name)
    if INDEXES[name][1] != b2.COSINE:
        ix = b2.VectorIndex(INDEXES[name][0], b2.COSINE, D, f"ncentroids={NLIST}, " + INDEXES[name][2]).build(cache.y)
        s = None
    rng = np.random.default_rng(13)
    q = np.concatenate([np.zeros((2, D), F32), (1e-6 * rng.standard_normal((6, D))).astype(F32), cache.q[:8]])
    dg, ig = ix.search(q, 10, f"nprobe={NLIST}")
    _full(ig, 10)
    _no_bad_ids(ig, cache.ok)
    assert np.isfinite(dg).all()
    assert (np.abs(dg[:2] - 1.0) <= 1e-6).all(), "a zero query's cosine distance is 1"
    if s is not None:
        dg, ig = ix.search(q, 10, f"nprobe={NPROBE}", first_stage_only=True)
        bad = R.compare(R.reference_search(s, q, 10, NPROBE), dg, ig)
        assert not bad, bad[:4]


# ---------------------------------------------------------------------------------------------------------------------------
# persistence
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(INDEXES))
def test_save_load_answers_identically(cache, name, tmp_path):
    ix, _ = cache.get(name)
    metric = INDEXES[name][1]
    path = tmp_path / "ix.b2ix"
    ix.save(path)
    lx = b2.VectorIndex.load(path, D, metric)
    assert lx.info()["n"] == N
    assert np.array_equal(lx.list_sizes(), ix.list_sizes())
    q = _bad_queries(cache.q[:300], None)[0]
    for params in (f"nprobe={NPROBE}", f"nprobe={NLIST}"):
        a, b = ix.search(q, 20, params), lx.search(q, 20, params)
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes(), params
    if name in GRAPHS:
        assert np.array_equal(lx.graph(), ix.graph())


def test_load_refuses_more_list_rows_than_n(cache, tmp_path):
    ix, _ = cache.get("mstg_raw0")   # no fp32 rows: n sizes nothing else in the file
    path = tmp_path / "ix.b2ix"
    ix.save(path)
    raw = bytearray(open(path, "rb").read())
    h = np.frombuffer(bytes(raw), R.HEADER, count=1)[0].copy()
    total = int(ix.list_sizes().sum())
    assert total < N
    b2.VectorIndex.load(path, D, b2.L2).close()   # fewer list rows than n: the unusable rows are in no list
    h["n"] = total - 1
    raw[:R.HEADER.itemsize] = h.tobytes()
    open(path, "wb").write(bytes(raw))
    with pytest.raises(B200Error, match="list lengths"):
        b2.VectorIndex.load(path, D, b2.L2)


def test_load_refuses_an_mstg_edge_to_a_row_in_no_list(cache, tmp_path):
    ix, _ = cache.get("mstg_g16")
    path = tmp_path / "ix.b2ix"
    ix.save(path)
    raw = bytearray(open(path, "rb").read())
    Dg = 16
    gbytes = N * Dg * 4
    g = np.frombuffer(bytes(raw[-gbytes:]), "<u4").reshape(N, Dg)
    assert np.array_equal(g, ix.graph())
    u = int(np.nonzero(~cache.ok)[0][0])
    g = g.copy()
    g[int(np.nonzero(cache.ok)[0][0]), 0] = u
    raw[-gbytes:] = g.tobytes()
    open(path, "wb").write(bytes(raw))
    with pytest.raises(B200Error, match="no list"):
        b2.VectorIndex.load(path, D, b2.IP)


# ---------------------------------------------------------------------------------------------------------------------------
# exact paths keep FLAT's rule
# ---------------------------------------------------------------------------------------------------------------------------
def _assert_flat_rule(y, q, k, metric, dg, ig):
    """FLAT's rule against a float64 reference of every row: the rows whose fp32 distance is finite compete, every returned
    id is one of them with its distance within tolerance, min(k, such rows) slots fill, and every row clearly inside the top
    k is returned.  Rows in no list take part like any other: after the cosine normalisation a row whose square overflows
    is a zero row (distance 1), and under IP its inner product is finite."""
    rows = R.prepare_queries(y, metric).astype(np.float64)
    Q = R.prepare_queries(q, metric).astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        for i in range(len(q)):
            if metric == R.L2:
                dist = ((rows - Q[i]) ** 2).sum(1)
                terms = (rows * rows).sum(1) + (Q[i] * Q[i]).sum() + 2 * np.abs(rows * Q[i]).sum(1)   # the expanded form
            else:
                ip = rows @ Q[i]
                dist = ip if metric == R.IP else 1 - ip
                terms = np.abs(rows * Q[i]).sum(1) + 1
            fin = np.isfinite(dist.astype(np.float32))
            key = -dist if metric == R.IP else dist
            tol = 1e-4 * terms + 1e-6
            got = ig[i][ig[i] >= 0]
            assert len(got) == min(k, int(fin.sum())), f"q{i}: {len(got)} slots filled"
            assert fin[got].all(), f"q{i}: a row with a non-finite distance is returned"
            assert (np.abs(dg[i, :len(got)] - dist[got]) <= tol[got]).all(), f"q{i}: a distance is not its row's"
            kth = np.sort(key[fin])[len(got) - 1]
            must = np.nonzero(fin & (key < kth - tol - tol[got].max()))[0]
            assert set(must.tolist()) <= set(got.tolist()), f"q{i}: rows clearly inside the top {k} are missing"


@pytest.mark.parametrize("metric", [b2.L2, b2.IP, b2.COSINE])
def test_exact_paths_keep_the_flat_rule(cache, metric):
    q, k = cache.q[:16], 20
    y = cache.y.copy()
    if metric == b2.IP:   # an infinite coordinate is outside FLAT's rule under IP
        y[np.isinf(y).any(1)] = NAN
    else:   # exact_batch=1 of a two-stage index with its fp32 rows in HBM
        ix, _ = cache.get("ivfflat" if metric == b2.L2 else "hnswsq")
        dg, ig = ix.search(q, k, "exact_batch=1")
        _assert_flat_rule(cache.y, q, k, metric, dg, ig)
    small = y[:1500]   # below max(2000, 8 nlist): the FLAT fallback
    fx = b2.VectorIndex("IVFFLAT", metric, D, f"ncentroids={NLIST}").build(small)
    assert not fx.info()["uses_ivf"]
    dg, ig = fx.search(q, k)
    _assert_flat_rule(small, q, k, metric, dg, ig)


# ---------------------------------------------------------------------------------------------------------------------------
# the default look-up scan at d = 768, build()'s strided sample, the graph walk against its reference
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ty,metric", [("IVFPQ", b2.L2), ("SCANN", b2.COSINE)])
def test_wide_rows_take_the_default_lookup_scan(ty, metric, tmp_path):
    n, d, nl = 20000, 768, 64
    y, q = _data(17, n=n, d=d, nl=nl)
    ok = R.usable(y)
    ix = b2.VectorIndex(ty, metric, d, f"ncentroids={nl}").build(y)
    assert ix.info()["n"] == n and int(ix.list_sizes().sum()) == int(ok.sum())
    ix.save(tmp_path / "ix.b2ix")
    s = R.read_index(tmp_path / "ix.b2ix")
    assert L.is_lut(s) and s.dsub == 16
    R.check_lists(s, ix, y)
    assert np.isfinite(s.codebook).all()
    qs, k = q[:32], 20
    for nprobe in (8, nl):
        dg, ig = ix.search(qs, k, f"nprobe={nprobe}", first_stage_only=True)
        _assert_first_stage("lut", s, qs, k, nprobe, dg, ig)
    _, ig = ix.search(q, k, f"nprobe={nl}")
    _no_bad_ids(ig, ok)
    _full(ig, k)
    qb, pos, _ = _bad_queries(q, None)
    others = np.setdiff1d(np.arange(len(q)), pos)
    clean, dirty = ix.search(q, k, "nprobe=8"), ix.search(qb, k, "nprobe=8")
    assert dirty[0][others].tobytes() == clean[0][others].tobytes() and dirty[1][others].tobytes() == clean[1][others].tobytes()
    assert (dirty[1][pos] == -1).all()
    alive = ~ok
    alive[np.nonzero(ok)[0][::4000]] = True
    bits = np.packbits(alive, bitorder="little")
    dg, ig = ix.search(qs, 10, "nprobe=8, filter_probe=1", first_stage_only=True, alive_bits=bits)
    _full(ig, min(10, int((alive & ok).sum())))
    _no_bad_ids(ig, ok)
    p, _ = ix.last_probe()
    for pv in np.unique(p):
        g = np.nonzero(p == pv)[0]
        _assert_first_stage("lut", s, qs[g], 10, int(pv), dg[g], ig[g], alive)


def test_build_trains_on_the_usable_rows_of_its_strided_sample(tmp_path):
    """n > max(256 nlist, 65536): build() trains on rows floor(i n / 65536); unusable rows sit on the k-means seeds of that
    sample and elsewhere in and outside it.  Well-separated clusters with one seed of the usable sample in each, so the
    reference trajectory is unambiguous."""
    rng = np.random.default_rng(23)
    n, d, nl = 70001, 17, 7
    rows = T.sample_rows(n, nl)
    assert len(rows) == 65536 < n
    bad = np.zeros(n, bool)
    bad[rows[T.strided(65536, nl)]] = True
    bad[rng.choice(rows, 40, replace=False)] = True
    bad[rng.choice(np.setdiff1d(np.arange(n), rows), 40, replace=False)] = True
    kept = rows[~bad[rows]]
    lab = rng.integers(0, nl, n)
    lab[kept[T.strided(len(kept), nl)]] = np.arange(nl)   # the seeds of the k-means over the usable sample
    y = (10 * rng.standard_normal((nl, d)))[lab] + 0.3 * rng.standard_normal((n, d))
    y = y.astype(F32)
    _spoil(y, np.nonzero(bad)[0], rng)
    ix = b2.VectorIndex("IVFFLAT", b2.L2, d, f"ncentroids={nl}").build(y)
    ix.save(tmp_path / "ix.b2ix")
    s = R.read_index(tmp_path / "ix.b2ix")
    R.check_build(s, ix, y)
    samp = y[rows][~bad[rows]]
    t = T.kmeans(samp, nl, 10)
    assert not t.ambiguous, t.why
    problems = T.centroid_problems(s.centroids, t)
    assert not problems, problems


@pytest.mark.parametrize("metric", [b2.L2, b2.IP])
def test_graph_walk_is_the_reference(metric):
    """HNSWFLAT on small integers (every distance exact in fp32): the walk equals the reference walk id for id and byte for
    byte, and never meets a row in no list."""
    from tests.test_gpu_index_graph import _integer, _metric_name

    y, q = _integer(20000, 32, 4)
    rng = np.random.default_rng(29)
    _spoil(y, np.unique(np.concatenate([T.strided(len(y), 141), rng.choice(len(y), 300, replace=False)])), rng)
    ok = R.usable(y)
    Dg, k = 16, 10
    ix = b2.VectorIndex("HNSWFLAT", metric, 32, f"graph_degree={Dg}").build(y)
    g = ix.graph()
    assert (g[~ok] == G.NO_ID).all() and ok[g[g != G.NO_ID].astype(np.int64)].all()
    for ef in (16, 64):
        dis, ids = ix.search(q, k, f"ef_s={ef}")
        rd, ri, _ = G.search(g, y, q, ix.last_seeds(), max(ef, k), k, G.iteration_cap(Dg), _metric_name(metric))
        assert np.array_equal(ids, ri), f"ef_s={ef}: ids differ from the reference"
        assert dis.tobytes() == rd.tobytes(), f"ef_s={ef}: distances differ from the reference"
        _no_bad_ids(ids, ok)
