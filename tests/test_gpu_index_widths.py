"""The inverted-file and graph indexes at production embedding widths (1024 .. 8192) and at odd widths (d % 4 in {1, 3}, the
64 / 65 and 128 / 129 k-block edges), against the references of the narrower checks: the float64 first-stage reference and
its comparator (tests/ivf_reference.py, tests/pq_lut_reference.py, tests/pq4_reference.py), the exact re-rank, the graph walk
(tests/graph_reference.py) and the training reference (tests/train_reference.py).  The comparator's tolerance is the fixed
3e-5 x (sum of the absolute values of the key's terms) plus, for rows wider than 768, the truncation bound of the
tensor-core product (ivf_reference.tc_weights, the model of tests/flat_reference.py).  The negative controls at the end show
that at 4096-d it still rejects one wrong SQ code, one bf16 ulp and a dropped page, on data built for it: one dimension
carries about half of every key, so that a one-step fault there is large against the sum of all terms (on evenly spread
data one bf16 ulp of one of 4096 dimensions is below the tolerance).  The width limit B200_MAX_FLOAT_DIM of the
inverted-file types is served at the limit and refused one step past it."""
import numpy as np
import pytest

import myscaledb_b200 as b2
from oracle import pack_bits
from tests import graph_reference as G
from tests import ivf_reference as R
from tests import pq4_reference as P4
from tests import pq_lut_reference as L
from tests import train_reference as T
from tests.test_gpu_index_train import separated, sq_rows
from tests.util import check_topk, to_bf16_values

pytestmark = pytest.mark.gpu
F32 = np.float32
METRICS = (b2.L2, b2.IP, b2.COSINE)
ERR_UNSUPPORTED = 3
N, NLIST = 4000, 32
WIDE = (1024, 1536, 3072, 4096, 8192)
ODD = (1, 3, 17, 63, 65, 127, 129, 257)
GATHER = (1021, 1025, 2049)          # either side of the host-row gather's 1024-float pass
MAX_D = 32640                        # B200_MAX_FLOAT_DIM (include/b200_search.h)


def _data(n, d, seed, nq=32, n_centres=24):
    """Clustered rows around a non-zero mean (as in test_gpu_ivf_reference.py)."""
    rng = np.random.default_rng(seed)
    mean = 1.0 + 0.5 * rng.standard_normal(d)
    centres = mean + rng.standard_normal((n_centres, d))
    y = centres[rng.integers(0, n_centres, n)] + 0.3 * rng.standard_normal((n, d))
    q = centres[rng.integers(0, n_centres, nq)] + 0.3 * rng.standard_normal((nq, d))
    return y.astype(F32), q.astype(F32)


def _integer(n, d, seed, nq=8):
    """small integers (as in the graph tests): bf16 holds them exactly and every key is exact in fp32 in any summation order
    up to d = 2^24 / 14^2 = 85598"""
    rng = np.random.default_rng(seed)
    centres = rng.integers(-6, 7, (100, d))
    y = centres[rng.integers(0, 100, n)] + rng.integers(-1, 2, (n, d))
    q = centres[rng.integers(0, 100, nq)] + rng.integers(-1, 2, (nq, d))
    return y.astype(F32), q.astype(F32)


def _saved(ix, path, reader=R.read_index):
    ix.save(path)
    return reader(path)


def _parity(s, ix, q, k, nprobe, params="", ref=R.reference_search):
    dg, ig = ix.search(q, k, f"nprobe={nprobe}" + (", " + params if params else ""), first_stage_only=True)
    bad = R.compare(ref(s, q, k, nprobe), dg, ig)
    assert not bad, f"{len(bad)} problems, first: {bad[:6]}"
    return dg, ig


def _d_pad(d):
    return -(-d // 4) * 4


def _d_pad64(d):
    return -(-d // 64) * 64


# ---------------------------------------------------------------------------------------------------------------------------
# 1. list scans, first stage: bf16 lists (IVFFLAT / MSTG) and SQ8 codes, every width, the metric rotating
# ---------------------------------------------------------------------------------------------------------------------------
LIST_TYPES = {"bf16": ("IVFFLAT", "MSTG"), "sq8": ("IVFSQ",)}
LIST_CASES = [(p, LIST_TYPES[p][i % len(LIST_TYPES[p])], METRICS[(i + pi) % 3], d)
              for pi, p in enumerate(LIST_TYPES) for i, d in enumerate(WIDE + ODD)]


@pytest.mark.parametrize("payload,typ,metric,d", LIST_CASES)
def test_list_scan_first_stage(payload, typ, metric, d, tmp_path):
    y, q = _data(N, d, seed=d + 10 * metric)
    ix = b2.VectorIndex(typ, metric, d, f"ncentroids={NLIST}").build(y)
    assert ix.info()["uses_ivf"]
    s = _saved(ix, tmp_path / "ix.b2ix")
    R.check_build(s, ix, y)
    _parity(s, ix, q, 10, 4)
    assert ix.last_scan()["payload_row_bytes"] == (_d_pad64(d) * 2 if payload == "bf16" else -(-d // 16) * 16)


@pytest.mark.parametrize("payload", ["bf16", "sq8"])
def test_list_scan_batch_k_nprobe_at_3072(payload, tmp_path):
    d = 3072
    y, q = _data(N, d, seed=77, nq=129)
    ix = b2.VectorIndex(LIST_TYPES[payload][0], b2.L2, d, f"ncentroids={NLIST}").build(y)
    s = _saved(ix, tmp_path / "ix.b2ix")
    for nq in (1, 129):
        for k in (1, 100, 1024):
            for nprobe in (1, 9, NLIST):
                _parity(s, ix, q[:nq], k, nprobe)


# ---------------------------------------------------------------------------------------------------------------------------
# 2. PQ at odd widths: the tensor-core decoder at dsub = 1, the look-up scans at odd sub-vector lengths
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [d for d in ODD if d <= 220] + [220])
def test_pq_decoder_dsub_1(d, tmp_path):
    metric = METRICS[d % 3]
    y, q = _data(N, d, seed=300 + d)
    ix = b2.VectorIndex("IVFPQ", metric, d, f"ncentroids={NLIST}, M={d}").build(y)
    s = _saved(ix, tmp_path / "pq.b2ix")
    assert s.dsub == 1 and not L.is_lut(s)
    _parity(s, ix, q, 10, 4)


@pytest.mark.parametrize("d,m", [(129, 43), (255, 17), (1023, 31)])
@pytest.mark.parametrize("bits", [8, 4])
def test_pq_lookup_odd_subvectors(d, m, bits, tmp_path):
    metric = METRICS[(d + bits) % 3]
    y, q = _data(N, d, seed=400 + d + bits)
    ix = b2.VectorIndex("IVFPQ", metric, d, f"ncentroids={NLIST}, M={m}, bit_size={bits}").build(y)
    if bits == 8:
        s = _saved(ix, tmp_path / "pq.b2ix")
        assert L.is_lut(s) and s.dsub == d // m
        _parity(s, ix, q, 10, 4, ref=L.reference_search)
    else:
        s = _saved(ix, tmp_path / "pq.b2ix", reader=P4.read_index4)
        assert s.dsub == d // m
        _parity(s, ix, q, 10, 4, ref=P4.reference_search)


# ---------------------------------------------------------------------------------------------------------------------------
# 3. the coarse probe at production widths, every path forced
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", WIDE)
def test_coarse_paths(d, tmp_path):
    nl = 128
    metric = METRICS[d % 3]
    y, q = _data(N, d, seed=500 + d, nq=16, n_centres=160)
    ix = b2.VectorIndex("IVFFLAT", metric, d, f"ncentroids={nl}").build(y)
    s = _saved(ix, tmp_path / "ix.b2ix")
    Q = R.prepare_queries(q, metric)
    for nprobe in (1, 8, 9, 64):
        flagged = R.coarse_probe(s, Q, nprobe)[2]
        ref = R.reference_search(s, q, 10, nprobe)
        base = ix.search(q, 10, f"nprobe={nprobe}", first_stage_only=True)
        for cp in (1, 2, 3):
            dg, ig = ix.search(q, 10, f"nprobe={nprobe}, coarse_path={cp}", first_stage_only=True)
            assert ix.last_coarse() == cp, f"nprobe={nprobe}: coarse_path={cp} ran path {ix.last_coarse()}"
            bad = R.compare(ref, dg, ig)
            assert not bad, f"nprobe={nprobe} coarse_path={cp}: {bad[:6]}"
            diff = ~((ig == base[1]).all(1) & (dg == base[0]).all(1))
            assert not (diff & ~flagged).any(), f"nprobe={nprobe}: coarse_path={cp} differs on a query without a probe tie"


# ---------------------------------------------------------------------------------------------------------------------------
# 4. the exact second stage, fp32 rows in HBM and in host memory
# ---------------------------------------------------------------------------------------------------------------------------
def _refine_bound(d_pad, terms):
    """fp32 error of the library's exact key (refine_kernel): each of 32 lanes reads ceil(d_pad / 128) float4 and sums their
    4 ceil(d_pad / 128) terms in a chain of fmaf, five shuffle adds follow, an L2 term adds one rounding of x - y and the cosine
    distance 1 + key one more: |error| <= (4 ceil(d_pad / 128) + 7) x 2^-24 x (sum of |terms|)."""
    return (4 * -(-d_pad // 128) + 7) * 2.0 ** -24 * terms


def _check_refined(s, q, cand, dg, ig, k):
    """dg / ig: the library's top k of the candidate ids cand [nq][k1] by its exact fp32 key.  Every returned id is a
    candidate; its distance is its exact key within the bound; the list is sorted best first, equal distances by id; the
    answer is the reference top k by (key, id) except where two keys lie within the bound of each other."""
    metric = s.metric
    Qp = R.prepare_queries(q, metric).astype(np.float64)
    rows = s.rows.astype(np.float64)
    rd, ri = R.rerank(s.rows, R.prepare_queries(q, metric), cand, k, metric)
    for i in range(len(q)):
        got = dg[i][ig[i] >= 0].astype(np.float64) * (-1 if metric == R.IP else 1)
        gid = ig[i][ig[i] >= 0]
        assert ((got[1:] > got[:-1]) | ((got[1:] == got[:-1]) & (gid[1:] > gid[:-1]))).all(), f"q{i}: not sorted best first"
        c = cand[i][cand[i] >= 0]
        assert set(ig[i][ig[i] >= 0].tolist()) <= set(c.tolist()), f"q{i}: a refined id is not a first-stage candidate"
        assert (ig[i] >= 0).sum() == min(k, len(c))
        y = rows[c]
        if metric == R.L2:
            exact = ((y - Qp[i]) ** 2).sum(1)
            terms = exact
        else:
            exact = y @ Qp[i]
            terms = np.abs(y * Qp[i]).sum(1) + (metric == R.COSINE)
            exact = exact if metric == R.IP else 1 - exact
        tol = _refine_bound(_d_pad(s.d), terms)
        pos = {int(v): j for j, v in enumerate(c.tolist())}
        for j, v in enumerate(ig[i][ig[i] >= 0].tolist()):
            p = pos[v]
            assert abs(dg[i, j] - exact[p]) <= tol[p] + 1e-30, f"q{i} rank {j}: {dg[i, j]!r} vs exact {exact[p]!r}"
        if np.array_equal(ig[i], ri[i]):
            continue
        # ids differ from the reference only inside a near-tie: every reference row clearly better than the k-th is present
        key = exact if metric != R.IP else -exact
        kth = np.sort(key)[min(k, len(c)) - 1]
        must = c[key < kth - tol - tol.max()]
        missing = set(must.tolist()) - set(ig[i].tolist())
        assert not missing, f"q{i}: rows {sorted(missing)[:5]} clearly inside the top {k} are missing"


REFINE_CASES = [(("MSTG", "IVFSQ")[i % 2], METRICS[i % 3], d) for i, d in enumerate(WIDE + ODD + GATHER)]


@pytest.mark.parametrize("typ,metric,d", REFINE_CASES)
def test_refine_both_placements(typ, metric, d, tmp_path):
    y, q = _data(N, d, seed=600 + d, nq=16)
    k, rf, nprobe = 10, 16, 6
    k1 = k * rf
    ix = b2.VectorIndex(typ, metric, d, f"ncentroids={NLIST}, keep_raw=1").build(y)
    s = _saved(ix, tmp_path / "ix.b2ix")
    _, cand = ix.search(q, k1, f"nprobe={nprobe}", first_stage_only=True)
    prm = f"nprobe={nprobe}, refine_factor={rf}"
    dg, ig = ix.search(q, k, prm)
    assert ix.last_num_candidates == k1
    _check_refined(s, q, cand, dg, ig, k)
    ix.set_raw_placement(2)
    assert ix.host_memory_bytes() == N * _d_pad(d) * 4   # host rows of d_pad floats: above 1024 the gather makes several passes
    dh, ih = ix.search(q, k, prm)
    assert dh.tobytes() == dg.tobytes() and ih.tobytes() == ig.tobytes(), "host placement differs from HBM"


# ---------------------------------------------------------------------------------------------------------------------------
# 5. graph walks on integer data: id for id and byte for byte against the reference walk (+ the exact re-rank)
# ---------------------------------------------------------------------------------------------------------------------------
GRAPH_DIMS = (1, 3, 17, 65, 129, 257, 1024, 1536, 3072, 4096)
GRAPH_KINDS = (("HNSWFLAT", 1), ("MSTG", 0), ("MSTG", 1), ("MSTG", 2))
GRAPH_CASES = [(t, kr, (b2.L2, b2.IP)[(i + j) % 2], d) for i, d in enumerate(GRAPH_DIMS) for j, (t, kr) in enumerate(GRAPH_KINDS)]
REFINE = 4   # MSTG's default refine_factor


def _graph_check(ix, typ, keep_raw, metric, y, q, k, ef, alive):
    mname = "l2" if metric == b2.L2 else "ip"
    dis, ids = ix.search(q, k, f"ef_s={ef}", alive_bits=None if alive is None else pack_bits(alive))
    two_stage = typ == "MSTG" and keep_raw != 0
    kc = min(1024, k * REFINE) if two_stage else k
    assert ix.last_num_candidates == kc
    seeds = ix.last_seeds()
    walk_rows = to_bf16_values(y) if typ == "MSTG" else y
    wd, wi, scored = G.search(ix.graph(), walk_rows, q, seeds, max(ef, kc), kc, G.iteration_cap(16), mname, alive)
    rd, ri = R.rerank(y, q, wi, k, metric) if two_stage else (wd, wi)
    assert np.array_equal(ids, ri), f"ef_s={ef}: ids differ from the reference"
    assert dis.tobytes() == rd.tobytes(), f"ef_s={ef}: distances differ from the reference"
    assert ix.last_scan()["rows_streamed"] == int(scored.sum())


@pytest.mark.parametrize("typ,keep_raw,metric,d", GRAPH_CASES)
def test_graph_walk(typ, keep_raw, metric, d):
    y, q = _integer(3000, d, seed=700 + d)
    ix = b2.VectorIndex(typ, metric, d, f"graph_degree=16, keep_raw={keep_raw}").build(y)
    alive = np.random.default_rng(d).random(len(y)) < 0.5
    for filt in (None, alive):
        _graph_check(ix, typ, keep_raw, metric, y, q, 10, 64, filt)
    if typ == "MSTG":   # the bf16 walk read rows of d_pad64 / 64 k-blocks: 1, 2, 3, 5, 16, 24, 48 and 64 over GRAPH_DIMS
        assert ix.last_scan()["payload_row_bytes"] // 128 == _d_pad64(d) // 64


@pytest.mark.parametrize("typ", ["MSTG", "HNSWFLAT"])
def test_graph_walk_8192_largest_lists(typ):
    d = 8192
    y, q = _integer(3000, d, seed=800, nq=2)
    ix = b2.VectorIndex(typ, b2.L2, d, "graph_degree=16").build(y)
    alive = np.random.default_rng(801).random(len(y)) < 0.5
    _graph_check(ix, typ, 1, b2.L2, y, q, 1024, 1024, alive)


# ---------------------------------------------------------------------------------------------------------------------------
# 6. training at width
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [1536, 3072])
def test_coarse_kmeans_wide(d, tmp_path):
    nl = 24
    metric = METRICS[d % 3]
    y, _ = separated(np.random.default_rng(900 + d), 2003, d, nl)
    ix = b2.VectorIndex("IVFFLAT", metric, d, f"ncentroids={nl}")
    ix.reserve(len(y)).train(y).add(y).finalize()
    s = _saved(ix, tmp_path / "ix.b2ix")
    t = T.kmeans(T.train_rows(y, metric), nl, 10)
    assert not t.ambiguous, f"test data design error: the reference trajectory is ambiguous: {t.why}"
    assert t.empty_final == 0 and t.counts.min() >= 1
    bad = T.centroid_problems(s.centroids, t)
    assert not bad, bad


def test_sq_ranges_wide(tmp_path):
    n, d, nl = 3001, 4096, 7
    y = sq_rows(np.random.default_rng(950), n, d, nl)
    ix = b2.VectorIndex("IVFSQ", b2.L2, d, f"ncentroids={nl}")
    ix.reserve(n).train(y).add(y).finalize()
    s = _saved(ix, tmp_path / "ix.b2ix")
    x = T.train_rows(y, b2.L2)
    assert not T.sq_problems(s.sq, x), T.sq_problems(s.sq, x)
    t = T.kmeans(x, nl, 10)
    assert not t.ambiguous, f"test data design error: the reference trajectory is ambiguous: {t.why}"
    assert not T.centroid_problems(s.centroids, t)


# ---------------------------------------------------------------------------------------------------------------------------
# 7. the float width limit: served at B200_MAX_FLOAT_DIM, refused one step past it
# ---------------------------------------------------------------------------------------------------------------------------
LIST_FLOAT_TYPES = ("IVFFLAT", "IVFSQ", "IVFPQ", "SCANN", "MSTG", "HNSWFLAT", "HNSWSQ", "HNSWPQ")


@pytest.mark.parametrize("typ", LIST_FLOAT_TYPES)
def test_width_limit_refused_one_step_past(typ):
    with pytest.raises(b2.B200Error) as e:
        b2.VectorIndex(typ, b2.L2, MAX_D + 1, "")
    assert e.value.code == ERR_UNSUPPORTED and str(MAX_D) in str(e.value)
    b2.VectorIndex(typ, b2.L2, MAX_D, "").close()


def test_width_limit_leaves_flat_and_binary_alone():
    b2.VectorIndex("FLAT", b2.L2, 65536, "").close()
    b2.VectorIndex("BINARYFLAT", b2.HAMMING, 65536, "").close()


@pytest.mark.parametrize("metric", [b2.L2, b2.IP])
def test_width_limit_served(metric, tmp_path):
    """At d = B200_MAX_FLOAT_DIM every search configuration fits: the exact second stage at k = 1024, the graph walks at
    ef_s = k = 1024 under a filter (the widest shared-memory layout), the list scans, a FLAT scan, and save / load."""
    d, n = MAX_D, 2100     # above the 2000 rows below which a part is served by a FLAT scan
    y, q = _integer(n, d, seed=1000 + metric, nq=2)
    alive = np.random.default_rng(1001).random(n) < 0.5
    ivf = "ncentroids=8"
    flat = b2.VectorIndex("FLAT", metric, d, "").build(y)
    dis, ids = flat.search(q, 10)
    do, io = R.rerank(y, q, np.tile(np.arange(n), (len(q), 1)), 10, metric)
    check_topk(metric, q, y, dis, ids, do, io)
    flat.close()
    # bf16 lists and SQ codes: first stage, then the second stage at k = 1024 over every row
    for typ in ("IVFFLAT", "IVFSQ"):
        ix = b2.VectorIndex(typ, metric, d, ivf + ", keep_raw=1").build(y)
        s = _saved(ix, tmp_path / f"{typ}.b2ix")
        _parity(s, ix, q, 10, 8)
        _, cand = ix.search(q, 1024, "nprobe=8", first_stage_only=True)
        dg, ig = ix.search(q, 1024, "nprobe=8, refine_factor=2")
        rd, ri = R.rerank(y, q, cand, 1024, metric)
        assert np.array_equal(ig, ri) and dg.tobytes() == rd.tobytes(), f"{typ}: refine at k = 1024"
        re = b2.VectorIndex.load(tmp_path / f"{typ}.b2ix", d, metric)
        d2, i2 = re.search(q, 1024, "nprobe=8, refine_factor=2")
        assert np.array_equal(i2, ig) and d2.tobytes() == dg.tobytes(), f"{typ}: loaded index answers differently"
        re.close()
        ix.close()
    for typ, kr in (("MSTG", 1), ("HNSWFLAT", 1)):
        ix = b2.VectorIndex(typ, metric, d, f"{ivf}, graph_degree=16, keep_raw={kr}").build(y)
        _graph_check(ix, typ, kr, metric, y, q, 1024, 1024, alive)
        ix.save(tmp_path / f"{typ}.b2ix")
        re = b2.VectorIndex.load(tmp_path / f"{typ}.b2ix", d, metric)
        _graph_check(re, typ, kr, metric, y, q, 1024, 1024, alive)
        re.close()
        ix.close()


def test_loader_refuses_wider_files(tmp_path):
    y, _ = _data(2100, 64, seed=1100)
    ix = b2.VectorIndex("IVFFLAT", b2.L2, 64, "ncentroids=4").build(y)
    path = tmp_path / "ix.b2ix"
    ix.save(path)
    raw = bytearray(open(path, "rb").read())
    raw[16:20] = np.int32(MAX_D + 1).tobytes()          # header field d
    bad = tmp_path / "wide.b2ix"
    open(bad, "wb").write(bytes(raw))
    with pytest.raises(b2.B200Error) as e:
        b2.VectorIndex.load(bad, MAX_D + 1, b2.L2)
    assert e.value.code == ERR_UNSUPPORTED and str(MAX_D) in str(e.value)


# ---------------------------------------------------------------------------------------------------------------------------
# 8. negative controls at 4096-d: the width-scaled tolerance still sees one wrong code, one bf16 ulp and a dropped page
# ---------------------------------------------------------------------------------------------------------------------------
def _heavy(d, seed):
    """Rows and queries whose dimension 0 carries about half of every key: the dimension a one-step fault weighs most."""
    y, q = _data(N, d, seed)
    y[:, 0] *= 48
    q[:, 0] *= 48
    return y, q


def _locate(s, i):
    l = next(l for l in range(s.nlist) if (s.ids[l] == i).any())
    return l, int(np.nonzero(s.ids[l] == i)[0][0])


def test_negative_controls_4096(tmp_path):
    d = 4096
    y, q = _heavy(d, 1200)
    ix = b2.VectorIndex("IVFSQ", b2.IP, d, f"ncentroids={NLIST}").build(y)
    s = _saved(ix, tmp_path / "sq.b2ix")
    dg, ig = _parity(s, ix, q, 10, 4)
    qs = np.abs(to_bf16_values(R.prepare_queries(q[:1], s.metric) * s.sq[1]))[0]
    j = int(np.argmax(qs))
    bad = s.copy()
    l, r = _locate(bad, ig[0, 0])
    bad.codes[l][r, j] = bad.codes[l][r, j] + 1 if bad.codes[l][r, j] < 255 else 254
    assert R.compare(R.reference_search(bad, q, 10, 4), dg, ig), "a wrong SQ code went unnoticed at 4096-d"

    ix = b2.VectorIndex("IVFFLAT", b2.IP, d, f"ncentroids={NLIST}").build(y)   # IP: no y - q cancellation on dim 0
    s = _saved(ix, tmp_path / "bf16.b2ix")
    dg, ig = _parity(s, ix, q, 10, 4)
    j = int(np.argmax(np.abs(q[0])))
    bad = s.copy()
    l, r = _locate(bad, ig[0, 0])
    v = bad.vals[l][r, j]
    bits = (np.array([v], F32).view(np.uint32) >> 16).astype(np.uint16) + np.uint16(1)   # one bf16 ulp away from zero
    bad.vals[l][r, j] = R.bf16_bits_to_f32(bits)[0]
    assert R.compare(R.reference_search(bad, q, 10, 4), dg, ig), "one bf16 ulp went unnoticed at 4096-d"

    for l in range(s.nlist):
        last = (len(s.ids[l]) - 1) // R.PAGE * R.PAGE
        if len(s.ids[l]) and np.isin(s.ids[l][last:], ig).any():
            break
    else:
        pytest.fail("no returned row sits in the last page of its list")
    bad = s.copy()
    bad.truncate_list(l, last)
    assert R.compare(R.reference_search(bad, q, 10, 4), dg, ig), "a skipped tail page went unnoticed at 4096-d"
