"""Filter-aware list probing (`filter_probe=1`) on the float inverted-file indexes.

Under a selective or correlated filter a plain search probes `nprobe` lists and may find fewer than k kept rows there.  With
the key every query probes, in (coarse key, list id) order, as many lists as its first k1 kept rows need (at least nprobe, at
most max_nprobe), and the scan streams only the pages that hold a kept row.  Checked here:
  * complete answers: min(k, kept rows) filled slots, every one kept, no duplicates (a plain search fails this);
  * each group of queries with the same depth p against the float64 reference of the stored index probing p lists, and the
    depth itself against one recomputed in float64 from the stored lists and the bitmap;
  * byte identity with a plain filtered search of the group at nprobe=p, coarse_path=3 (so the page skipping changes nothing),
    with the default search where every query reaches k1 within nprobe lists, and without a filter;
  * the exact rule (a host bitmap within both 16 x nprobe x n / nlist rows and the gathered exact path's limit, fp32 rows in
    HBM) on both sides of its limit, query sub-ranges of a batch above the scratch budget, and the keys' edges."""
import os
import re

import numpy as np
import pytest

import myscaledb_b200 as b2
from myscaledb_b200.search import B200Error
from tests import ivf_reference as R

pytestmark = pytest.mark.gpu
F32 = np.float32
ERR_UNSUPPORTED = 3
N, D, NLIST, NPROBE, NC = 50000, 64, 256, 16, 32
# the exact rule's limit with prefilter=2: kFilterProbeExactFactor x nprobe x n / nlist (csrc/ivf.cu), capped by the gathered
# path's n / 8 (csrc/capi.cu prefilter_limit); with prefilter=0 (auto) a corpus this small is never gathered, so never the rule
EXACT_LIMIT = min(16 * NPROBE * N // NLIST, N // 8)

# name -> (type, metric, build params, first stage modelled by tests/ivf_reference.py)
INDEXES = {
    "ivfflat": ("IVFFLAT", b2.L2, "", True),
    "ivfsq": ("IVFSQ", b2.IP, "", True),
    "ivfpq_d8": ("IVFPQ", b2.L2, "M=8", True),
    "scann_lut": ("SCANN", b2.IP, "M=4", False),          # d / M = 16: the table look-up scan
    "scann_4bit": ("SCANN", b2.L2, "M=16, bit_size=4", False),
    "mstg_raw0": ("MSTG", b2.L2, "keep_raw=0", True),
    "mstg_raw1": ("MSTG", b2.COSINE, "keep_raw=1", True),
    "mstg_raw2": ("MSTG", b2.IP, "keep_raw=2", True),
    "hnswflat": ("HNSWFLAT", b2.L2, "", True),
}
FILTERS = ("r0.5", "r0.05", "r0.005", "r0.0005", "far", "runs")
NQS = (1, 7, 256, 1025)
KS = (1, 10, 100)


def _data(seed, n=N, d=D, nq=2048):
    """Clustered rows; the queries sit around the first half of the centres, so the rows of the other half are far."""
    rng = np.random.default_rng(seed)
    mean = 1.0 + 0.5 * rng.standard_normal(d)
    centres = mean + 2.0 * rng.standard_normal((NC, d))
    lab = rng.integers(0, NC, n)
    y = centres[lab] + 0.5 * rng.standard_normal((n, d))
    q = centres[rng.integers(0, NC // 2, nq)] + 0.5 * rng.standard_normal((nq, d))
    return y.astype(F32), q.astype(F32), lab, centres


def _filter(kind, lab, centres, seed, n=N):
    rng = np.random.default_rng(seed)
    if kind.startswith("r0"):
        a = rng.random(n) < float(kind[1:])
        a[rng.integers(0, n)] = True
        return a
    if kind == "far":   # the rows of the three centres farthest from the queries' centres
        far = NC // 2 + np.argsort(-np.linalg.norm(centres[NC // 2:] - centres[:NC // 2].mean(0), axis=1))[:3]
        return np.isin(lab, far)
    a = np.zeros(n, bool)   # id runs
    for s in rng.integers(0, n - 100, 5):
        a[s:s + 100] = True
    return a


class _Cache:
    def __init__(self, tmp):
        self.tmp, self.got = tmp, {}
        self.y, self.q, self.lab, self.centres = _data(7)

    def get(self, name):
        if name not in self.got:
            ty, metric, extra = INDEXES[name][:3]
            ix = b2.VectorIndex(ty, metric, D, f"ncentroids={NLIST}" + (", " + extra if extra else "")).build(self.y)
            assert ix.info()["uses_ivf"]
            s = None
            if INDEXES[name][3]:
                path = self.tmp / f"{name}.b2ix"
                ix.save(path)
                s = R.read_index(path)
            self.got[name] = (ix, s)
        return self.got[name]


@pytest.fixture(scope="module")
def cache(tmp_path_factory):
    return _Cache(tmp_path_factory.mktemp("filtered"))


def _bits(alive):
    return np.packbits(alive, bitorder="little")


def _assert_complete(ids, k, alive):
    want = min(k, int(alive.sum()))
    filled = (ids >= 0).sum(1)
    assert (filled == want).all(), f"{int((filled < want).sum())} of {len(ids)} queries are short (want {want})"
    assert (ids[:, want:] == -1).all()
    got = ids[:, :want]
    assert alive[got].all(), "a returned row is not kept"
    srt = np.sort(got, axis=1)
    assert (srt[:, 1:] != srt[:, :-1]).all(), "duplicate ids"


def _same(a, b):
    return a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()


def _assert_groups_identical(ix, q, k, p, bits, out, fso, nc):
    """Each group of queries with depth p equals a plain filtered search of the group with nprobe=p, coarse_path=3."""
    for pv in np.unique(p):
        if pv > 1024:
            continue
        g = np.nonzero(p == pv)[0]
        ref = ix.search(q[g], k, f"nprobe={pv}, coarse_path=3", first_stage_only=fso, alive_bits=bits)
        assert _same((out[0][g], out[1][g]), ref), f"group p={pv} ({len(g)} queries) differs from the plain search"
        assert ix.last_num_candidates == nc


def _fp64_depth(s, Q, alive, k1, nprobe, max_nprobe):
    """p_q from the stored lists: lists by fp64 L2 centroid distance (ties to the smaller id), kept rows per list."""
    C = s.centroids.astype(np.float64)
    Q64 = Q.astype(np.float64)
    dist = ((Q64[:, None, :] - C[None, :, :]) ** 2).sum(2)
    order = np.argsort(dist, axis=1, kind="stable")
    per_list = np.array([int(alive[s.ids[l].astype(np.int64)].sum()) for l in range(s.nlist)])
    W = np.cumsum(per_list[order], axis=1)
    reach = np.where(W[:, -1] >= k1, (W >= k1).argmax(1) + 1, s.nlist)
    return np.minimum(max_nprobe, np.maximum(nprobe, reach))


def _assert_reference(s, q, k, p, alive, dg, ig):
    Q = R.prepare_queries(q, s.metric)
    want = _fp64_depth(s, Q, alive, k, NPROBE, NLIST)
    for i in np.nonzero(want != p)[0]:
        flagged = [R.coarse_probe(s, Q[i:i + 1], int(v))[2][0] for v in (want[i], p[i])]
        assert any(flagged), f"query {i}: depth {p[i]}, fp64 {want[i]} without a near-tie at the cut"
    for pv in np.unique(p):
        g = np.nonzero(p == pv)[0]
        bad = R.compare(R.reference_search(s, q[g], k, int(pv), alive), dg[g], ig[g])
        assert not bad, f"p={pv}: {len(bad)} problems, first: {bad[:4]}"


CASES = [(name, f, NQS[(i + j) % 4], KS[(i + 2 * j) % 3]) for i, name in enumerate(INDEXES) for j, f in enumerate(FILTERS)]


@pytest.mark.parametrize("name,flt,nq,k", CASES)
def test_filter_probe_matrix(cache, name, flt, nq, k):
    ix, s = cache.get(name)
    q = cache.q[:nq]
    alive = _filter(flt, cache.lab, cache.centres, seed=len(name) + nq)
    bits = _bits(alive)
    key = f"nprobe={NPROBE}, filter_probe=1"
    out = ix.search(q, k, key, alive_bits=bits)
    nc = ix.last_num_candidates
    _assert_complete(out[1], k, alive)
    p, exact = ix.last_probe()
    assert len(p) == nq and not exact   # prefilter=0 never gathers a corpus this small: the lists answer
    assert (p >= NPROBE).all() and (p <= NLIST).all()
    _assert_groups_identical(ix, q, k, p, bits, out, False, nc)
    # the first stage alone: its depths against the fp64 reference
    fs = ix.search(q, k, key, first_stage_only=True, alive_bits=bits)
    _assert_complete(fs[1], k, alive)
    p, exact = ix.last_probe()
    assert not exact
    if nq <= 256:
        _assert_groups_identical(ix, q, k, p, bits, fs, True, k)
        if s is not None:
            m = min(nq, 64)
            _assert_reference(s, q[:m], k, p[:m], alive, fs[0][:m], fs[1][:m])


def test_plain_search_is_short_under_a_far_filter(cache):
    """What the key fixes: without it the far filter leaves queries short."""
    ix, _ = cache.get("mstg_raw0")
    alive = _filter("far", cache.lab, cache.centres, 0)
    _, ids = ix.search(cache.q[:256], 10, f"nprobe={NPROBE}", alive_bits=_bits(alive))
    assert ((ids >= 0).sum(1) < 10).any()
    p, exact = ix.last_probe()
    assert (p == NPROBE).all() and not exact


@pytest.mark.parametrize("name,fso", [("ivfflat", True), ("mstg_raw0", False), ("mstg_raw1", False), ("mstg_raw2", False), ("scann_lut", True)])
def test_reaching_k1_within_nprobe_equals_the_default_search(cache, name, fso):
    ix, _ = cache.get(name)
    q = cache.q[:300]
    alive = _filter("r0.5", cache.lab, cache.centres, 3)
    bits = _bits(alive)
    got = ix.search(q, 10, f"nprobe={NPROBE}, filter_probe=1", first_stage_only=fso, alive_bits=bits)
    p, exact = ix.last_probe()
    assert (p == NPROBE).all() and not exact
    assert _same(got, ix.search(q, 10, f"nprobe={NPROBE}", first_stage_only=fso, alive_bits=bits))
    # without a filter the key changes nothing
    got = ix.search(q, 10, f"nprobe={NPROBE}, filter_probe=1", first_stage_only=fso)
    assert _same(got, ix.search(q, 10, f"nprobe={NPROBE}", first_stage_only=fso))
    assert (ix.last_probe()[0] == NPROBE).all()


def test_exact_rule_and_device_entry(cache):
    import torch

    alive = _filter("r0.0005", cache.lab, cache.centres, 5)
    assert alive.sum() <= EXACT_LIMIT
    bits = _bits(alive)
    q, k = cache.q[:100], 10
    ix, _ = cache.get("mstg_raw1")
    got = ix.search(q, k, f"nprobe={NPROBE}, prefilter=2, filter_probe=1", alive_bits=bits)
    assert ix.last_probe()[1]
    assert _same(got, ix.search(q, k, f"nprobe={NPROBE}, prefilter=2, exact_batch=1", alive_bits=bits))
    # the same bitmap where the exact pass would not gather the kept rows (prefilter auto below its corpus size, never):
    # the lists answer
    for pf in (0, 1):
        got = ix.search(q, k, f"nprobe={NPROBE}, prefilter={pf}, filter_probe=1", alive_bits=bits)
        assert not ix.last_probe()[1]
        _assert_complete(got[1], k, alive)
    # a bitmap above the gathered path's limit (n / 8) but within 16 x nprobe x n / nlist: the lists answer
    wide = _filter("r0.5", cache.lab, cache.centres, 6)
    assert EXACT_LIMIT < wide.sum() <= 16 * NPROBE * N // NLIST
    got = ix.search(q, k, f"nprobe={NPROBE}, prefilter=2, filter_probe=1", alive_bits=_bits(wide))
    p, exact = ix.last_probe()
    assert not exact and (p >= NPROBE).all()
    _assert_complete(got[1], k, wide)
    _assert_groups_identical(ix, q, k, p, _bits(wide), got, False, ix.last_num_candidates)
    # the device entry has no host count: the list path, complete, on a side stream
    tq = torch.from_numpy(q).cuda()
    ta = torch.from_numpy(bits).cuda()
    od = torch.empty((len(q), k), dtype=torch.float32, device="cuda")
    oi = torch.empty((len(q), k), dtype=torch.int64, device="cuda")
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    ix.search_device(tq.data_ptr(), len(q), k, od.data_ptr(), oi.data_ptr(), params=f"nprobe={NPROBE}, filter_probe=1",
                     alive_ptr=ta.data_ptr(), stream=side.cuda_stream)
    side.synchronize()
    p, exact = ix.last_probe()
    assert not exact and (p >= NPROBE).all()
    _assert_complete(oi.cpu().numpy(), k, alive)
    # no fp32 rows in HBM: never the exact rule
    for name in ("mstg_raw0", "mstg_raw2"):
        ix, _ = cache.get(name)
        ix.search(q, k, f"nprobe={NPROBE}, prefilter=2, filter_probe=1", alive_bits=bits)
        assert not ix.last_probe()[1]


def test_max_nprobe_and_binary_refusal(cache):
    ix, _ = cache.get("mstg_raw0")
    alive = _filter("far", cache.lab, cache.centres, 0)
    bits = _bits(alive)
    q = cache.q[:200]
    ix.search(q, 10, f"nprobe={NPROBE}, filter_probe=1", alive_bits=bits)
    deep = ix.last_probe()[0]
    assert deep.max() > 24
    ix.search(q, 10, f"nprobe={NPROBE}, max_nprobe=24, filter_probe=1", alive_bits=bits)
    p = ix.last_probe()[0]
    assert (p == np.minimum(deep, 24)).all()
    # a cap below nprobe does not lower nprobe: every query probes nprobe lists, as the plain search
    got = ix.search(q, 10, f"nprobe={NPROBE}, max_nprobe=3, filter_probe=1", alive_bits=bits)
    assert (ix.last_probe()[0] == NPROBE).all()
    assert _same(got, ix.search(q, 10, f"nprobe={NPROBE}, coarse_path=3", alive_bits=bits))
    # binary indexes refuse the key
    rng = np.random.default_rng(1)
    yb = rng.integers(0, 256, (5000, 16), dtype=np.uint8)
    bx = b2.VectorIndex("BINARYIVF", b2.HAMMING, 128, "ncentroids=16").build(yb)
    with pytest.raises(B200Error) as e:
        bx.search(yb[:4], 5, "nprobe=4, filter_probe=1", alive_bits=np.full(5000 // 8, 0xff, np.uint8))
    assert e.value.code == ERR_UNSUPPORTED


def _budget():
    src = open(os.path.join(os.path.dirname(__file__), "..", "myscaledb_b200", "csrc", "ivf.cu")).read()
    m = re.search(r"kFilterProbeScratchBytes = 1ll << (\d+);", src)
    s = re.search(r"kFilterProbeSlotBytes = (\d+);", src)
    return 1 << int(m.group(1)), int(s.group(1))


def test_batch_above_the_budget_runs_in_sub_ranges(tmp_path):
    n, d, nl, nq, k = 200000, 64, 4096, 8192, 400
    y, q, lab, centres = _data(11, n=n, d=d, nq=nq)
    ix = b2.VectorIndex("IVFFLAT", b2.L2, d, f"ncentroids={nl}, keep_raw=0").build(y)   # no exact rule: the lists answer
    # a sparse random filter: a few kept rows in most lists, so every query probes hundreds of lists that hold one
    alive = np.random.default_rng(12).random(n) < 0.02
    bits = _bits(alive)
    key = f"nprobe={NPROBE}, filter_probe=1"
    dg, ig = ix.search(q, k, key, alive_bits=bits)
    p, exact = ix.last_probe()
    assert not exact and (p < nl).all()
    ix.save(tmp_path / "ix.b2ix")
    s = R.read_index(tmp_path / "ix.b2ix")
    most = max(int(alive[s.ids[l].astype(np.int64)].sum()) for l in range(nl))
    budget, _ = _budget()
    k1 = k   # one stage
    # the least the batch needs: each query reaches k1 kept rows, so it probes at least k1 / (most kept rows in a list) lists
    # that hold one, and each such slot needs a partial list of k1 entries (8 B each + its worst key)
    assert nq * -(-k1 // most) * (k1 * 8 + 4) > budget
    _assert_complete(ig, k, alive)
    parts = [ix.search(q[a:a + 512], k, key, alive_bits=bits) for a in range(0, nq, 512)]
    assert dg.tobytes() == np.concatenate([x[0] for x in parts]).tobytes()
    assert ig.tobytes() == np.concatenate([x[1] for x in parts]).tobytes()
