"""The binary inverted-file search (BINARYIVF, and the BINARYHNSW / BINARYMSTG names it serves) at partial probes, against the
exact reference of the stored index (tests/binary_ivf_reference.py).

Every index is built here, saved, and decoded from its file by the reference's own reader.  The reference probes the lists
nearest the query under Hamming distance to the stored centroid bytes (ties to the smaller list id) and keys every kept row
of those lists exactly, so the library must return the same ids and the same distance BITS in every slot: a scan that skips a
page, a probe that picks the wrong list, a merge that drops a partial list or a bound that prunes a true neighbour fails
here.  The negative controls at the end show that the comparator rejects those faults on a GPU-built index."""
import numpy as np
import pytest

import myscaledb_b200 as b2
from tests import binary_ivf_reference as B
from tests.test_gpu_binary_index import clustered

pytestmark = pytest.mark.gpu
METRICS = (b2.HAMMING, b2.JACCARD)
# width in bits -> (rows, nlist): lists of several pages at every width, fewer rows at the widest
WIDTHS = {64: (200_000, 64), 200: (100_000, 64), 1032: (40_000, 32), 4096: (12_000, 16), 65536: (3_000, 8)}


def rows(rng, n, nb, centres, flip=0.08):
    """clustered() rows around the given centres, generated in blocks of at most 2^22 bits (its bit matrix is fp64)"""
    step = max(1, (1 << 22) // (8 * nb))
    return np.concatenate([clustered(rng, min(step, n - r0), nb, centres=centres, flip=flip)[0] for r0 in range(0, n, step)])


def data(nbits, n, seed, nq=64):
    rng = np.random.default_rng(seed)
    nb = nbits // 8
    centres = rng.integers(0, 2, (24, nbits), dtype=np.uint8)
    y = rows(rng, n, nb, centres)
    q = rows(rng, nq, nb, centres)
    q[3] = 0                    # Jaccard's 0 / 0 against the all-zero rows
    q[5] = y[17]
    return y, q, centres


def saved(ix, path):
    ix.save(path)
    return B.read_binary_index(path)


def same_bytes(a, b):
    return np.array_equal(a[1], b[1]) and np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32))


def assert_parity(s, ix, q, k, nprobe, params="", alive=None, ref=None):
    dg, ig = ix.search(q, k, f"nprobe={nprobe}" + (", " + params if params else ""), alive_bits=alive)
    ref = B.reference_search(s, q, k, nprobe, alive) if ref is None else ref
    bad = B.compare(ref, dg, ig)
    assert not bad, bad
    return dg, ig, ref


class _Cache:
    def __init__(self, tmp):
        self.tmp, self.got = tmp, {}

    def get(self, metric, nbits):
        key = (metric, nbits)
        if key not in self.got:
            n, nl = WIDTHS[nbits]
            y, q, cen = data(nbits, n, seed=nbits + metric)
            ix = b2.VectorIndex("BINARYIVF", metric, nbits, f"ncentroids={nl}").build(y)
            assert ix.info()["uses_ivf"]
            s = saved(ix, self.tmp / f"b{metric}_{nbits}.b2ix")
            assert s.list_len.max() > B.PAGE
            self.got[key] = (ix, s, y, q, cen)
        return self.got[key]


@pytest.fixture(scope="module")
def cache(tmp_path_factory):
    return _Cache(tmp_path_factory.mktemp("bin_ivf_ref"))


# ---------------------------------------------------------------------------------------------------------------------------
# a. build invariants
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", METRICS)
def test_build_invariants_one_shot_streamed_and_device(metric, tmp_path):
    torch = pytest.importorskip("torch")
    nbits, n, nl = 200, 20_000, 32
    y, _, _ = data(nbits, n, seed=7 + metric)
    params = f"ncentroids={nl}"
    a = b2.VectorIndex("BINARYIVF", metric, nbits, params).build(y)
    sa = saved(a, tmp_path / "a.b2ix")
    B.check_binary_build(sa, y)
    # streamed: chunks of 1, 255, 257 and 5000 rows split list tails across add() calls
    b = b2.VectorIndex("BINARYIVF", metric, nbits, params).reserve(n).train(y)
    off, sizes = 0, (1, 255, 257, 5000)
    for i in range(n):
        if off >= n:
            break
        b.add(y[off:off + sizes[i % 4]])
        off += sizes[i % 4]
    b.finalize()
    sb = saved(b, tmp_path / "b.b2ix")
    B.check_binary_build(sb, y)
    t = torch.from_numpy(y).cuda()
    c = b2.VectorIndex("BINARYIVF", metric, nbits, params).reserve(n).train_device(t.data_ptr(), n)
    c.add_device(t.data_ptr(), 7001).add_device(t[7001:].data_ptr(), n - 7001).finalize()
    sc = saved(c, tmp_path / "c.b2ix")
    B.check_binary_build(sc, y)
    assert np.array_equal(sa.centroids, sb.centroids) and np.array_equal(sa.centroids, sc.centroids)
    for i in (a, b, c):
        i.close()


# ---------------------------------------------------------------------------------------------------------------------------
# b. partial-probe parity: every metric, width and nprobe edge
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nprobe", ["1", "2", "7", "nlist-1", "nlist", "nlist+5"])
@pytest.mark.parametrize("nbits", list(WIDTHS))
@pytest.mark.parametrize("metric", METRICS)
def test_partial_probe_parity(cache, metric, nbits, nprobe):
    ix, s, y, q, _ = cache.get(metric, nbits)
    npr = {"nlist-1": s.nlist - 1, "nlist": s.nlist, "nlist+5": s.nlist + 5}.get(nprobe) or int(nprobe)
    ref = B.reference_search(s, q, 20, npr)
    for k in (1, 20):
        assert_parity(s, ix, q, k, npr, ref=ref.head(len(q), k))


# ---------------------------------------------------------------------------------------------------------------------------
# c. the coarse probe on both of its kernels, and its tie rule
# ---------------------------------------------------------------------------------------------------------------------------
def test_coarse_probe_on_the_scan_and_the_tensor_path(cache):
    ix, s, y, _, cen = cache.get(b2.HAMMING, 64)
    # the centroid table is a 16-byte binary corpus: its auto path scans below ceil(20480 / 16^2) = 80 queries
    assert s.cent_pad == 16 and -(-20480 // (s.cent_pad * s.cent_pad)) == 80
    q = rows(np.random.default_rng(3), 1025, 8, cen)
    for nq in (1, 79, 80, 1025):
        for nprobe in (1, 7, 40):
            assert_parity(s, ix, q[:nq], 10, nprobe)


def tied_queries(s, rng, nq):
    """Queries halfway between two stored centroids whose bits differ in an even count: equal Hamming distance to both."""
    rb = s.row_bytes
    cb = np.unpackbits(s.centroids[:, :rb], axis=1)
    out = []
    while len(out) < nq:
        a, b = rng.choice(s.nlist, 2, replace=False)
        diff = np.nonzero(cb[a] != cb[b])[0]
        if len(diff) % 2 or not len(diff):
            continue
        x = cb[a].copy()
        x[rng.choice(diff, len(diff) // 2, replace=False)] ^= 1
        out.append(np.packbits(x))
    return np.stack(out)


@pytest.mark.parametrize("metric", METRICS)
def test_coarse_ties_probe_the_smaller_list(cache, metric):
    ix, s, y, _, _ = cache.get(metric, 64)
    q = tied_queries(s, np.random.default_rng(4 + metric), 256)
    for nprobe in (1, 2, 7):
        tied = B.coarse_ties(s, q, nprobe)
        assert tied.sum() >= 8, f"nprobe={nprobe}: {int(tied.sum())} queries with a tie at the probe's edge"
        for nq in (40, 256):   # both coarse kernels
            assert_parity(s, ix, q[:nq], 10, nprobe)


# ---------------------------------------------------------------------------------------------------------------------------
# d. cooperative and per-lane items in one launch; k and chunking edges; schedule invariance
# ---------------------------------------------------------------------------------------------------------------------------
def hot_queries(cen, nq, seed):
    """Queries on the centres with weights 1, 1/2, 1/4, ...: the lists of the first centres are probed by hundreds of queries,
    those of the last by a few or none (the order is shuffled, so every prefix batch mixes them)."""
    rng = np.random.default_rng(seed)
    w = 0.5 ** np.arange(len(cen))
    pick = rng.choice(len(cen), nq, p=w / w.sum())
    q = np.concatenate([rows(rng, int((pick == c).sum()), 8, cen[c:c + 1]) for c in np.unique(pick)])
    return q[rng.permutation(nq)]


MIX_NQ, MIX_K, MIX_NPROBE = (1, 16, 17, 129, 1025, 5000), (1, 10, 17, 100, 256, 257, 1024), 4


@pytest.fixture(scope="module")
def mixed(cache):
    out = {}
    for metric in METRICS:
        ix, s, y, _, cen = cache.get(metric, 64)
        q = hot_queries(cen, MIX_NQ[-1], 11 + metric)
        out[metric] = (ix, s, q, B.reference_search(s, q, max(MIX_K), MIX_NPROBE))
    return out


@pytest.mark.parametrize("metric", METRICS)
def test_mixed_item_kinds_k_and_chunk_edges(mixed, metric):
    ix, s, q, ref = mixed[metric]
    for nq in (1025, 5000):
        per_list = np.bincount(ref.probed[:nq].ravel(), minlength=s.nlist)
        assert per_list.max() > 128 and 0 < per_list[per_list > 0].min() <= 16, per_list
    for nq in MIX_NQ:
        for k in MIX_K:
            for ppc in (0, 1, 2, 16, 64):
                dg, ig = ix.search(q[:nq], k, f"nprobe={MIX_NPROBE}" + (f", pages_per_chunk={ppc}" if ppc else ""))
                bad = B.compare(ref.head(nq, k), dg, ig)
                assert not bad, (nq, k, ppc, bad)


@pytest.mark.parametrize("metric", METRICS)
def test_schedule_invariance(mixed, metric, monkeypatch):
    ix, s, q, ref = mixed[metric]
    for k in (10, 256, 1024):
        base = ix.search(q, k, f"nprobe={MIX_NPROBE}")
        assert not B.compare(ref.head(len(q), k), *base)
        assert same_bytes(base, ix.search(q, k, f"nprobe={MIX_NPROBE}, shared_bound=0")), ("shared_bound=0", k)
        monkeypatch.setenv("B200_IVF_COOP", "0")            # read at every launch: every item on per-lane lists
        assert same_bytes(base, ix.search(q, k, f"nprobe={MIX_NPROBE}")), ("B200_IVF_COOP=0", k)
        monkeypatch.delenv("B200_IVF_COOP")


# ---------------------------------------------------------------------------------------------------------------------------
# e. filters
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", METRICS)
def test_alive_bitmaps(cache, metric):
    ix, s, y, q, _ = cache.get(metric, 64)
    n, k, nprobe = len(y), 20, 7
    rng = np.random.default_rng(5 + metric)
    probed = B.coarse_probe(s, q, nprobe)
    ids, lst, _ = s.flat()
    dead_lists = np.ones(n, bool)
    dead_lists[ids[np.isin(lst, probed[0][:3])]] = False       # query 0's three nearest lists entirely filtered
    for name, keep in (("dense", rng.random(n) < 0.5), ("sparse", rng.random(n) < 0.0004), ("empty", np.zeros(n, bool)),
                       ("dead lists", dead_lists)):
        alive = np.packbits(keep, bitorder="little")
        dg, ig, _ = assert_parity(s, ix, q, k, nprobe, alive=alive)
        assert keep[ig[ig >= 0]].all(), name
        if name == "sparse":
            assert (ig == -1).any() and (ig >= 0).any(), "fewer than k kept rows in the probed lists"
        if name == "empty":
            assert (ig == -1).all()
        if name == "dead lists":
            assert not np.isin(ig[0], ids[np.isin(lst, probed[0][:3])]).any() and (ig[0] >= 0).all()


def test_search_device_id_offset_and_device_bitmap(cache):
    torch = pytest.importorskip("torch")
    ix, s, y, q, _ = cache.get(b2.JACCARD, 200)
    alive = np.packbits(np.random.default_rng(6).random(len(y)) < 0.5, bitorder="little")
    nq, k = len(q), 20
    dh, ih, _ = assert_parity(s, ix, q, k, 7, alive=alive)
    tq, ta = torch.from_numpy(q).cuda(), torch.from_numpy(alive).cuda()
    od = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    oi = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    ix.search_device(tq.data_ptr(), nq, k, od.data_ptr(), oi.data_ptr(), params="nprobe=7", id_offset=1000,
                     alive_ptr=ta.data_ptr(), stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert np.array_equal(oi.cpu().numpy(), np.where(ih >= 0, ih + 1000, -1))
    assert np.array_equal(od.cpu().numpy().view(np.uint32), dh.view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------------------
# f. type names, ignored keys, persistence
# ---------------------------------------------------------------------------------------------------------------------------
def same_content(a, b):
    return (np.array_equal(a.centroids, b.centroids) and np.array_equal(a.list_len, b.list_len) and
            all(np.array_equal(x, z) for x, z in zip(a.ids, b.ids)) and all(np.array_equal(x, z) for x, z in zip(a.pool, b.pool)) and
            all(np.array_equal(x.view(np.uint32), z.view(np.uint32)) for x, z in zip(a.popc, b.popc)))


@pytest.mark.parametrize("metric", METRICS)
def test_type_names_and_ignored_keys(metric, tmp_path):
    y, q, _ = data(256, 20_000, seed=13 + metric)
    got = {}
    for t, code in (("BINARYIVF", 10), ("BINARYHNSW", 11), ("BINARYMSTG", 12)):
        ix = b2.VectorIndex(t, metric, 256, "ncentroids=32").build(y)
        s = saved(ix, tmp_path / f"{t}.b2ix")
        assert s.type == code
        got[t] = (ix, s)
    ix0, s0 = got["BINARYIVF"]
    ans = assert_parity(s0, ix0, q, 20, 5)[:2]
    for t, (ix, s) in got.items():
        assert same_content(s0, s), t
        assert same_bytes(ans, ix.search(q, 20, "nprobe=5")), t
        assert same_bytes(ans, ix.search(q, 20, "nprobe=5, refine_factor=8")), t
        assert same_bytes(ans, ix.search(q, 20, "nprobe=5", first_stage_only=True)), t
        ix.close()


@pytest.mark.parametrize("metric,nbits", [(b2.HAMMING, 1032), (b2.JACCARD, 65536)])
def test_save_load_roundtrip(cache, metric, nbits, tmp_path):
    ix, s, y, q, _ = cache.get(metric, nbits)
    ix.save(tmp_path / "a.b2ix")
    ld = b2.VectorIndex.load(tmp_path / "a.b2ix", nbits, metric=metric)
    assert same_content(s, saved(ld, tmp_path / "b.b2ix"))
    for nprobe in (2, s.nlist - 1):
        assert same_bytes(ix.search(q, 20, f"nprobe={nprobe}"), assert_parity(s, ld, q, 20, nprobe)[:2])
    ld.close()


# ---------------------------------------------------------------------------------------------------------------------------
# g. one case at scale
# ---------------------------------------------------------------------------------------------------------------------------
def test_one_million_rows_2048_lists(tmp_path):
    y, q, _ = data(256, 1_000_000, seed=17, nq=4096)
    ix = b2.VectorIndex("BINARYIVF", b2.HAMMING, 256, "ncentroids=2048").build(y)
    s = saved(ix, tmp_path / "big.b2ix")
    assert s.nlist == 2048 and s.list_len.max() > 2 * B.PAGE
    sample = np.arange(0, 4096, 64)          # the reference's CPU time is bounded by a fixed sample of the batch
    for nprobe in (32, 1024):                # 1024: the coarse probe's k limit below nlist
        ref = B.reference_search(s, q[sample], 100, nprobe)
        for k in (10, 100):
            dg, ig = ix.search(q, k, f"nprobe={nprobe}")
            bad = B.compare(ref.head(len(sample), k), dg[sample], ig[sample])
            assert not bad, (nprobe, k, bad)
    ix.close()


# ---------------------------------------------------------------------------------------------------------------------------
# h. negative controls: the comparator rejects the faults it is meant to catch, on a GPU-built index
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", METRICS)
def test_negative_controls(cache, metric):
    ix, s, y, q, _ = cache.get(metric, 64)
    k, nprobe = 10, 2
    dg, ig, ref = assert_parity(s, ix, q, k, nprobe)
    # probing nprobe - 1 lists
    assert B.compare(B.reference_search(s, q, k, nprobe - 1), dg, ig), "a probe of nprobe - 1 lists went unnoticed"
    # the last page of a probed list that holds a winner dropped
    hit = None
    for qi in range(len(q)):
        for l in ref.probed[qi]:
            last = (len(s.ids[l]) - 1) // B.PAGE * B.PAGE
            if np.isin(s.ids[l][last:], ig[qi]).any():
                hit = l, last
                break
        if hit:
            break
    assert hit, "no winner sits in the last page of its list"
    bad = s.copy()
    bad.truncate_list(*hit)
    assert B.compare(B.reference_search(bad, q, k, nprobe), dg, ig), "a skipped tail page went unnoticed"
    # one flipped bit in a winning row
    bad = s.copy()
    l, r = bad.locate(ig[0, 0])
    bad.pool[l][r, 0] ^= 1
    assert B.compare(B.reference_search(bad, q, k, nprobe), dg, ig), "a flipped bit went unnoticed"
    # final ties toward the larger row id (clustered() duplicates rows: equal keys among the winners)
    assert (dg[:, 1:] == dg[:, :-1]).any()
    assert B.compare(B.reference_search(s, q, k, nprobe, ties="larger"), dg, ig), "ties to the larger row id went unnoticed"
    # coarse ties toward the larger list id
    tq = tied_queries(s, np.random.default_rng(4 + metric), 256)
    dt, it, _ = assert_parity(s, ix, tq, k, 1)
    assert B.compare(B.reference_search(s, tq, k, 1, coarse="larger"), dt, it), "coarse ties to the larger list went unnoticed"
