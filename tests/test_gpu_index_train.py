"""Index training against tests/train_reference.py: the coarse k-means (tiled fp32 and tensor-core assignment, empty
clusters and splits), the SQ8 ranges, the PQ codebooks and the binary k-majority, through build(), reserve/train/add and
train_device.

Every case saves the index and compares the file with the reference.  A float case first asserts that the reference
trajectory of its data is unambiguous (no assignment decided by rounding) -- a data change that breaks this is a design
error of the test, not a pass -- and that the events it exists for happened.  Seeds are rows floor(i n / nlist), so the row
order places them.  The negative controls perturb the reference's inputs only and show each comparator rejects them."""
import numpy as np
import pytest

import myscaledb_b200 as b2
from tests import ivf_reference as R
from tests import pq4_reference as P4
from tests import train_reference as T
from tests.test_gpu_binary_index import clustered

pytestmark = pytest.mark.gpu
F32 = np.float32
METRICS = (b2.L2, b2.IP, b2.COSINE)
assert (b2.L2, b2.IP, b2.COSINE) == (R.L2, R.IP, R.COSINE)


def _unambiguous(t, what):
    assert not t.ambiguous, f"test data design error: the reference trajectory of {what} is ambiguous: {t.why}"


def _match(got, t, what):
    _unambiguous(t, what)
    bad = T.centroid_problems(got, t)
    assert not bad, f"{what}: {bad}"


def _rejects(got, t, what):
    assert T.centroid_problems(got, t), f"negative control: the comparator accepts {what}"


def _labels(rng, counts, seed_labels, nc):
    """Labels of sum(counts) rows in random order, with the k-means seed rows floor(i n / nc) labelled seed_labels[i]."""
    n = int(sum(counts))
    seeds = T.strided(n, nc)
    pool = list(np.repeat(np.arange(len(counts)), counts))
    for s in seed_labels:
        pool.remove(s)
    pool = np.array(pool)
    rng.shuffle(pool)
    lab = np.empty(n, np.int64)
    free = np.ones(n, bool)
    free[seeds] = False
    lab[free] = pool
    lab[seeds] = seed_labels
    return lab


def separated(rng, n, d, nl, scale=10.0, noise=0.3):
    """n rows of nl well-separated clusters in random order, one seed row in each; cluster sizes differ."""
    counts = rng.multinomial(n - nl, np.ones(nl) / nl) + 1
    lab = _labels(rng, counts, np.arange(nl), nl)
    centres = scale * rng.standard_normal((nl, d))
    return (centres[lab] + noise * rng.standard_normal((n, d))).astype(F32), lab


def _ivf(metric, d, params, rows, train=None, total=None):
    """reserve / train / add / finalize; train defaults to the rows themselves."""
    ix = b2.VectorIndex("IVFFLAT", metric, d, params)
    ix.reserve(total or len(rows)).train(rows if train is None else train).add(rows).finalize()
    return ix


def _stored(ix, path, reader=R.read_index):
    ix.save(path)
    s = reader(path)
    ix.close()
    return s


# ---------------------------------------------------------------------------------------------------------------------------
# coarse k-means, tiled fp32 assignment
# ---------------------------------------------------------------------------------------------------------------------------
TILED = [(METRICS[i % 3], d, nl) for i, (d, nl) in enumerate((d, nl) for d in (17, 100, 768) for nl in (1, 7, 64, 100, 130))]


@pytest.mark.parametrize("metric,d,nl", TILED)
def test_coarse_kmeans_tiled(metric, d, nl, tmp_path):
    rng = np.random.default_rng(7 * d + nl + metric)
    n = 3001 if d < 768 else 2003   # not a multiple of the 64-row tile
    y, _ = separated(rng, n, d, nl)
    s = _stored(_ivf(metric, d, f"ncentroids={nl}", y), tmp_path / "ix.b2ix")
    t = T.kmeans(T.train_rows(y, metric), nl, 10)
    assert t.empty_final == 0 and t.counts.min() >= 1
    _match(s.centroids, t, f"centroids ({metric}, d={d}, nlist={nl})")


@pytest.mark.parametrize("metric", [b2.L2, b2.COSINE])
def test_coarse_kmeans_build_trains_on_the_strided_sample(metric, tmp_path):
    # n > max(256 nlist, 65536): build() trains on rows floor(i n / 65536); the rows it leaves out are shifted, so the
    # centroids of any other sample (all rows) differ
    rng = np.random.default_rng(11 + metric)
    n, d, nl = 70001, 17, 7
    rows = T.sample_rows(n, nl)
    assert len(rows) == 65536 < n
    lab = np.empty(n, np.int64)
    out = np.ones(n, bool)
    out[rows] = False
    lab[rows] = _labels(rng, np.bincount(np.concatenate([np.arange(nl), rng.integers(0, nl, 65536 - nl)]), minlength=nl),
                        np.arange(nl), nl)
    lab[out] = rng.integers(0, nl, int(out.sum()))
    centres = 10 * rng.standard_normal((nl, d))
    y = (centres[lab] + 0.3 * rng.standard_normal((n, d)) + 1.5 * out[:, None]).astype(F32)
    ix = b2.VectorIndex("IVFFLAT", metric, d, f"ncentroids={nl}").build(y)
    s = _stored(ix, tmp_path / "ix.b2ix")
    x = T.train_rows(y, metric)
    _match(s.centroids, T.kmeans(T.build_sample(x, nl), nl, 10), "centroids of build()'s sample")
    _rejects(s.centroids, T.kmeans(x, nl, 10, seeds=rows[T.strided(65536, nl)]), "centroids of every row")


def test_coarse_kmeans_train_device_from_a_torch_tensor(tmp_path):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(5)
    n, d, nl = 3001, 100, 64
    y, _ = separated(rng, n, d, nl)
    t_rows = torch.from_numpy(y).cuda()
    ix = b2.VectorIndex("IVFFLAT", b2.COSINE, d, f"ncentroids={nl}")
    ix.reserve(n).train_device(t_rows.data_ptr(), n).add(y).finalize()
    torch.cuda.synchronize()
    s = _stored(ix, tmp_path / "ix.b2ix")
    _match(s.centroids, T.kmeans(T.train_rows(y, b2.COSINE), nl, 10), "centroids trained from device rows")


# ---------------------------------------------------------------------------------------------------------------------------
# empty clusters and splits
# ---------------------------------------------------------------------------------------------------------------------------
def merge_split_data(rng, d, tied):
    """Clusters: X holds two seeds that are the same row (an exact tie: the second goes empty in iteration 0); A and B share
    one seed and merge into the largest cluster, which the empty one splits.  A - B points along the split's nudge (the
    signs of eps_j), so the split copies separate A from B.  tied: a second merged pair C + D with A + B's count, so equal
    counts decide which one is split (the smaller id).  Singles fill the other seeds; every count is distinct otherwise."""
    p = np.where(np.arange(d) & 1, 1.0, -1.0)
    base = 4.0 * np.ones(d)
    far = lambda: base + 15.0 * rng.standard_normal(d)   # noqa: E731
    cent = [far(), base + 2 * p, base - 2 * p]           # X, A, B
    counts = [400, 300, 250]
    seed_lab = [0, 0, 1]
    if tied:
        cd = far()
        cent += [cd + 2 * p, cd - 2 * p]
        counts += [310, 240]
        seed_lab += [3]
    for c in (100, 150, 200, 260, 350):
        seed_lab.append(len(cent))
        cent.append(far())
        counts.append(c)
    nc = len(seed_lab)
    lab = _labels(rng, counts, seed_lab, nc)
    y = (np.array(cent)[lab] + 0.05 * rng.standard_normal((len(lab), d))).astype(F32)
    seeds = T.strided(len(y), nc)
    y[seeds[1]] = y[seeds[0]]
    return y, nc


@pytest.mark.parametrize("d,tied", [(16, False), (33, True), (100, False)])
def test_empty_clusters_split_the_largest(d, tied, tmp_path):
    rng = np.random.default_rng(d)
    y, nc = merge_split_data(rng, d, tied)
    s = _stored(_ivf(b2.L2, d, f"ncentroids={nc}", y), tmp_path / "ix.b2ix")
    t = T.kmeans(y, nc, 10)
    assert t.splits >= 1 and t.empties >= 1 and t.empty_final == 0, (t.splits, t.empties, t.empty_final)
    assert (t.tied_splits >= 1) == tied
    _match(s.centroids, t, f"centroids after splits (d={d}, tied={tied})")


# ---------------------------------------------------------------------------------------------------------------------------
# tensor-core assignment (n nlist d > 2e11)
# ---------------------------------------------------------------------------------------------------------------------------
def test_coarse_kmeans_tensor_core_assignment(tmp_path):
    n, d, nl = 786432, 128, 2048
    assert n * nl * d > 2e11   # kmeans_device assigns by a top-1 search of the centroid table on the tensor cores
    rng = np.random.default_rng(3)
    per = n // nl
    centres = rng.standard_normal((nl, d))
    distinct = np.empty((2 * nl, d))
    distinct[0::2] = centres + 0.1 * rng.standard_normal((nl, d))
    distinct[1::2] = centres + 0.1 * rng.standard_normal((nl, d))
    distinct = distinct.astype(F32)
    ka = rng.integers(100, per - 100, nl)
    w = np.empty(2 * nl)
    w[0::2], w[1::2] = ka, per - ka
    # cluster i fills rows [i per, (i + 1) per), its first row (the seed) is its vector a
    idx = np.empty(n, np.int64)
    for i in range(nl):
        blk = np.concatenate([np.full(ka[i] - 1, 2 * i), np.full(per - ka[i], 2 * i + 1)])
        rng.shuffle(blk)
        idx[i * per] = 2 * i
        idx[i * per + 1:(i + 1) * per] = blk
    assert np.array_equal(T.strided(n, nl), np.arange(nl) * per)
    y = distinct[idx]
    ix = b2.VectorIndex("IVFFLAT", b2.L2, d, f"ncentroids={nl}")
    ix.reserve(n).train(y).add(y[:8192]).finalize()
    del y
    s = _stored(ix, tmp_path / "ix.b2ix")
    t = T.kmeans(distinct, nl, 10, w=w, seeds=2 * np.arange(nl))
    assert t.empty_final == 0
    _match(s.centroids, t, "centroids of the tensor-core assignment")


# ---------------------------------------------------------------------------------------------------------------------------
# SQ8 ranges, bit for bit
# ---------------------------------------------------------------------------------------------------------------------------
def sq_rows(rng, n, d, nl):
    y, _ = separated(rng, n, d, nl)
    y[:, 3] = -2.5            # a constant column: step 1
    y[:, 5] = 0.75
    y[:, 6] -= 40.0           # all negative
    return y


@pytest.mark.parametrize("metric", METRICS)
def test_sq_ranges_bit_for_bit(metric, tmp_path):
    rng = np.random.default_rng(20 + metric)
    n, d, nl = 3001, 24, 7
    y = sq_rows(rng, n, d, nl)
    ix = b2.VectorIndex("IVFSQ", metric, d, f"ncentroids={nl}")
    ix.reserve(n).train(y).add(y).finalize()
    s = _stored(ix, tmp_path / "ix.b2ix")
    x = T.train_rows(y, metric)
    assert not T.sq_problems(s.sq, x), T.sq_problems(s.sq, x)
    if metric != b2.COSINE:
        assert s.sq[1][3] == 1 and s.sq[1][5] == 1 and (s.sq[0][6] < 0) and (s.sq[3][6] < 0)
    _match(s.centroids, T.kmeans(x, nl, 10), "IVFSQ centroids")
    # negative control: one ulp off in one step
    got = s.sq.copy()
    got[1][0] = np.nextafter(got[1][0], F32(np.inf))
    assert T.sq_problems(got, x), "negative control: a step one ulp off is accepted"


def test_sq_ranges_of_build_sample(tmp_path):
    rng = np.random.default_rng(31)
    n, d, nl = 70001, 24, 7
    y = sq_rows(rng, n, d, nl)
    out = np.setdiff1d(np.arange(n), T.sample_rows(n, nl))
    y[out[:5], 0] = 1e3       # extremes build() does not train on
    y[out[5:9], 1] = -1e3
    s = _stored(b2.VectorIndex("IVFSQ", b2.L2, d, f"ncentroids={nl}").build(y), tmp_path / "ix.b2ix")
    assert not T.sq_problems(s.sq, T.build_sample(y, nl)), T.sq_problems(s.sq, T.build_sample(y, nl))
    assert T.sq_problems(s.sq, y), "negative control: the ranges of every row are accepted"


# ---------------------------------------------------------------------------------------------------------------------------
# PQ codebooks
# ---------------------------------------------------------------------------------------------------------------------------
def grid(rng, ncw, dsub):
    """ncw distinct points of spacing 1 in dsub dimensions, in random order: an L^dsub grid, else hypercube corners."""
    L = round(ncw ** (1.0 / dsub))
    if L ** dsub == ncw:
        pts = np.stack(np.meshgrid(*[np.arange(L)] * dsub, indexing="ij"), -1).reshape(-1, dsub) - (L - 1) / 2
    else:
        code = rng.choice(2 ** dsub, ncw, replace=False)
        pts = ((code[:, None] >> np.arange(dsub)) & 1) - 0.5
    return pts[rng.permutation(ncw)].astype(np.float64)


def pq_data(rng, n, d, dsub, ncw, n_sample=None):
    """Rows = one of 2 far-apart coarse centres + a residual group g_k (one grid point per sub-quantiser) + noise.  Group k
    fills the rows from the k-th sub-quantiser seed of the sample on, and every group is split evenly between the two lists,
    so both lists' residuals sit on the same grid.  Rows past n_sample (outside the PQ sample) get random groups, shifted."""
    ns = n if n_sample is None else n_sample
    m = d // dsub
    g = np.concatenate([grid(rng, ncw, dsub) for _ in range(m)], axis=1)   # [ncw][d]: sub-quantiser j in columns j dsub ..
    group = np.searchsorted(T.strided(ns, ncw), np.arange(ns), side="right") - 1
    half = T.strided(n, 2)[1]
    lst = (np.arange(n) + (np.arange(n) >= half)) % 2
    v = rng.choice([-1.0, 1.0], d) * 10 * (np.abs(g).max() + 1)   # the lists lie much farther apart than the groups
    coarse = np.stack([v, -v])
    y = coarse[lst] + 0.02 * rng.standard_normal((n, d))
    y[:ns] += g[group]
    if ns < n:
        y[ns:] += g[rng.integers(0, ncw, n - ns)] + 0.25
    return y.astype(F32)


PQ_CASES = [  # (d, M, bits, n)
    (16, 16, 8, 4096), (16, 8, 8, 4096), (16, 4, 8, 4096), (16, 2, 8, 4096),   # dsub 1, 2, 4, 8 (tensor-core decoder)
    (32, 2, 8, 4096),                                                          # dsub 16 (look-up scan)
    (16, 8, 4, 4096),                                                          # 4-bit codes, dsub 2 (v3 file)
]


@pytest.mark.parametrize("d,m,bits,n", PQ_CASES)
def test_pq_codebooks(d, m, bits, n, tmp_path):
    rng = np.random.default_rng(d * m + bits)
    dsub, ncw = d // m, 16 if bits == 4 else 256
    y = pq_data(rng, n, d, dsub, ncw)
    ix = b2.VectorIndex("IVFPQ", b2.L2, d, f"ncentroids=2, M={m}, bit_size={bits}")
    ix.reserve(n).train(y).add(y).finalize()
    s = _stored(ix, tmp_path / "ix.b2ix", P4.read_index4 if bits == 4 else R.read_index)
    _match(s.centroids, T.kmeans(y, 2, 10), "coarse centroids")
    p = T.pq_codebooks(y, s.centroids, m, bits)
    assert not p.ambiguous, f"test data design error: {p.coarse_ambiguous} sample rows, {[t.why for t in p.subs if t.ambiguous][:2]}"
    assert all(t.empty_final == 0 for t in p.subs)
    bad = T.codebook_problems(s.codebook, p)
    assert not bad, bad


def test_pq_codebooks_sample_is_the_first_65536_rows(tmp_path):
    # 65536 < n < 131072: the stride is 1, the sample the first 65536 rows; the rows after them are shifted, so the even
    # stride floor(i n / 65536) trains other codebooks
    rng = np.random.default_rng(41)
    n, d, m = 70000, 8, 2
    y = pq_data(rng, n, d, d // m, 256, n_sample=65536)
    ix = b2.VectorIndex("IVFPQ", b2.L2, d, f"ncentroids=2, M={m}")
    ix.reserve(n).train(y).add(y[:4096]).finalize()
    s = _stored(ix, tmp_path / "ix.b2ix")
    p = T.pq_codebooks(y, s.centroids, m, 8)
    assert not p.ambiguous, f"test data design error: {p.coarse_ambiguous}, {[t.why for t in p.subs if t.ambiguous][:2]}"
    bad = T.codebook_problems(s.codebook, p)
    assert not bad, bad
    assert T.codebook_problems(s.codebook, T.pq_codebooks(y, s.centroids, m, 8, stride_rule="even")), \
        "negative control: codebooks of the even-strided sample are accepted"


def test_pq_codebooks_with_fewer_rows_than_codewords(tmp_path):
    # 200 training rows, 256 codewords: seeds floor(i 200 / 256) repeat rows, their clusters stay empty to the end
    rng = np.random.default_rng(43)
    n, d, m = 200, 8, 4
    y = (rng.standard_normal((n, d)) + 40.0 * (np.arange(n) >= 100)[:, None]).astype(F32)
    ix = b2.VectorIndex("IVFPQ", b2.L2, d, f"ncentroids=2, M={m}")
    ix.reserve(4000).train(y).add(np.tile(y, (20, 1))).finalize()
    s = _stored(ix, tmp_path / "ix.b2ix")
    _match(s.centroids, T.kmeans(y, 2, 10), "coarse centroids")
    p = T.pq_codebooks(y, s.centroids, m, 8)
    assert not p.ambiguous and all(t.empty_final == 56 for t in p.subs), [t.empty_final for t in p.subs]
    bad = T.codebook_problems(s.codebook, p)
    assert not bad, bad


# ---------------------------------------------------------------------------------------------------------------------------
# binary k-majority, byte for byte
# ---------------------------------------------------------------------------------------------------------------------------
BIN_CASES = [  # (metric, bits, n, path, early)
    (b2.HAMMING, 64, 70000, "build", False),    # n > 65536: build() trains on the strided sample
    (b2.JACCARD, 200, 6001, "train", False),    # 25 bytes: cent_pad 32
    (b2.HAMMING, 1024, 6001, "train", True),
    (b2.JACCARD, 2048, 4001, "build", False),
]


@pytest.mark.parametrize("metric,nbits,n,path,early", BIN_CASES)
def test_binary_kmajority(metric, nbits, n, path, early, tmp_path):
    rng = np.random.default_rng(nbits + metric)
    nb, nl = nbits // 8, 16
    if early:   # well-separated, one centre per list: converges before the 10th iteration
        y, _ = clustered(rng, n, nb, n_centres=nl, flip=0.02)
    else:
        y, _ = clustered(rng, n, nb)
    train = T.sample_rows(n, nl) if path == "build" else np.arange(n)
    seeds = train[T.strided(len(train), nl)]
    if not early:   # duplicate and all-zero seed rows: empty clusters, middle-member splits
        y[seeds[1]] = y[seeds[0]]
        y[seeds[3]] = 0
        y[seeds[4]] = 0
    ix = b2.VectorIndex("BINARYIVF", metric, nbits, f"ncentroids={nl}")
    if path == "build":
        ix.build(y)
    else:
        ix.reserve(n).train(y).add(y).finalize()
    ix.save(tmp_path / "ix.b2ix")
    ix.close()
    h, cent, lens = T.read_binary_coarse(tmp_path / "ix.b2ix")
    t = T.kmajority(y[train], nl, 10)
    if early:
        assert t.stopped_early
    else:
        assert t.splits >= 1
    assert cent.shape == t.centroids.shape and np.array_equal(cent, t.centroids), \
        f"{int((cent != t.centroids).any(1).sum())} centroids differ"
    assert np.array_equal(lens, T.bin_list_lengths(y, t))


def test_binary_kmajority_ties(tmp_path):
    # ~8 random rows per list: every cluster has bits with exact ties, which keep the centroid's bit
    rng = np.random.default_rng(51)
    n, nb, nl = 2000, 8, 250
    y = rng.integers(0, 256, (n, nb), dtype=np.uint8)
    ix = b2.VectorIndex("BINARYIVF", b2.HAMMING, nb * 8, f"ncentroids={nl}")
    ix.reserve(n).train(y).add(y).finalize()
    ix.save(tmp_path / "ix.b2ix")
    ix.close()
    _, cent, _ = T.read_binary_coarse(tmp_path / "ix.b2ix")
    t = T.kmajority(y, nl, 10)
    assert t.ties > 0
    assert np.array_equal(cent, t.centroids)
    assert not np.array_equal(cent, T.kmajority(y, nl, 10, tie_sets=True).centroids), \
        "negative control: a tie that sets the bit is accepted"


# ---------------------------------------------------------------------------------------------------------------------------
# build decisions
# ---------------------------------------------------------------------------------------------------------------------------
def test_default_nlist_and_the_inverted_file_threshold():
    rng = np.random.default_rng(61)
    y = rng.standard_normal((3000, 8)).astype(F32)
    ix = b2.VectorIndex("IVFFLAT", b2.L2, 8).build(y)
    assert ix.info()["nlist"] == T.default_nlist(3000) == 219 and ix.info()["uses_ivf"]
    ix.close()
    for nl, n in ((10, 1999), (10, 2000), (300, 2399), (300, 2400)):   # total >= max(2000, 8 nlist)
        ix = b2.VectorIndex("IVFFLAT", b2.L2, 8, f"ncentroids={nl}").build(y[:n])
        assert ix.info()["uses_ivf"] == T.use_ivf(n, n, nl) == (n in (2000, 2400)), (nl, n)
        ix.close()
    for n_train in (299, 300):                                          # n >= nlist
        ix = b2.VectorIndex("IVFFLAT", b2.L2, 8, "ncentroids=300").reserve(3000).train(y[:n_train])
        assert ix.info()["uses_ivf"] == T.use_ivf(3000, n_train, 300) == (n_train == 300)
        ix.close()


# ---------------------------------------------------------------------------------------------------------------------------
# negative controls of the k-means comparator
# ---------------------------------------------------------------------------------------------------------------------------
def test_negative_control_nine_iterations(tmp_path):
    # 2-d uniform rows: Lloyd still moves rows at iteration 10 (index 9)
    x = (np.random.default_rng(14).random((2001, 2)) - 0.5).astype(F32)
    s = _stored(_ivf(b2.L2, 2, "ncentroids=12", x), tmp_path / "ix.b2ix")
    t = T.kmeans(x, 12, 10)
    assert t.last_change == 9
    _match(s.centroids, t, "centroids of moving data")
    _rejects(s.centroids, T.kmeans(x, 12, 9), "a 9-iteration trajectory")


def test_negative_control_one_row_dropped(tmp_path):
    rng = np.random.default_rng(71)
    n, d, nl = 3001, 17, 7
    y, lab = separated(rng, n, d, nl)
    s = _stored(_ivf(b2.L2, d, f"ncentroids={nl}", y), tmp_path / "ix.b2ix")
    seeds = T.strided(n, nl)
    _match(s.centroids, T.kmeans(y, nl, 10), "centroids")
    drop = int(np.setdiff1d(np.nonzero(lab == 2)[0], seeds)[0])
    keep = np.delete(np.arange(n), drop)
    assert np.bincount(lab, minlength=nl).max() <= 1000
    _rejects(s.centroids, T.kmeans(y[keep], nl, 10, seeds=np.searchsorted(keep, seeds)), "a trajectory without one row")
