"""Anisotropic PQ (`aq_threshold=T`) on IVFPQ / SCANN / HNSWPQ under IP and cosine, against tests/aq_reference.py.

Every index is saved and decoded by the existing readers (tests/ivf_reference.py, tests/pq4_reference.py): an AQ index is an
ordinary B2IX v2 / v3 PQ file.  The cases cover 8-bit codes on the tensor-core decoder (d / M in {1, 2, 4, 8}), 8-bit codes
on the look-up scan (768-d, M = 48) and 4-bit codes (M = 96 at 768-d; d / M = 2).

* codes: every stored code row equals the reference encoder run on that row with the stored centroids and codebooks, except
  rows with a decision within fp32 rounding of its runner-up (the reference flags them; the test asserts they are few);
* training: train_loss() never increases, ends below the loss of the nearest-codeword codes, and follows the reference
  trajectory started from the k-means codebooks of the same build without the key (the k-means step is the same code; the
  test asserts that both builds' centroids agree);
* search: the first stage of every scan agrees with the float64 reference of the stored index (the scans are unchanged);
* build invariants: streamed and one-shot builds, duplicate rows, save / load, keep_raw=2 against keep_raw=1;
* refusals, and negative controls of both comparators.

The k-means that AQ starts from sums cluster members with fp32 atomics, so it is not bitwise reproducible from run to run
(tests/test_gpu_ivf_pq4.py says the same of plain PQ): two builds are held to the same invariants rather than compared byte
for byte.  What AQ adds on top is deterministic: identical rows added to one index get identical codes."""
import numpy as np
import pytest

import myscaledb_b200 as b2
from tests import aq_reference as A
from tests import ivf_reference as R
from tests import pq4_reference as P
from tests import pq_lut_reference as L

pytestmark = pytest.mark.gpu
F32 = np.float32
ERR_INVALID, ERR_UNSUPPORTED = 1, 3
N, NLIST, T = 4000, 16, 0.2
AMBIGUOUS_MAX = 0.2    # data design bound: at most this share of rows may have a decision within fp32 rounding

# (type, metric, d, M, bits): tensor-core decoder at d / M = 1, 2, 4, 8; look-up scan at 768 / 48; 4-bit at M = 96 and d / M = 2
CASES = [("IVFPQ", b2.COSINE, 64, 64, 8), ("IVFPQ", b2.IP, 100, 50, 8), ("HNSWPQ", b2.COSINE, 192, 48, 8), ("SCANN", b2.IP, 128, 16, 8),
         ("SCANN", b2.COSINE, 768, 48, 8), ("IVFPQ", b2.IP, 768, 48, 8), ("SCANN", b2.COSINE, 768, 96, 4), ("IVFPQ", b2.IP, 192, 96, 4)]
IDS = [f"{t}-{'cos' if mt == b2.COSINE else 'ip'}-d{d}-M{m}-{b}bit" for t, mt, d, m, b in CASES]


def _data(n, d, seed, nq=32, n_centres=NLIST):
    """Well-separated clusters around a common direction (so inner products are not all near 0), with per-row norms
    varying under IP."""
    rng = np.random.default_rng(seed)
    mean = 2.0 * rng.standard_normal(d) / np.sqrt(d)
    centres = mean + 4.0 * rng.standard_normal((n_centres, d)) / np.sqrt(d)
    lab = rng.integers(0, n_centres, n)
    y = centres[lab] + 0.6 * rng.standard_normal((n, d)) / np.sqrt(d)
    y *= rng.uniform(0.5, 1.5, (n, 1))
    q = centres[rng.integers(0, n_centres, nq)] + 0.6 * rng.standard_normal((nq, d)) / np.sqrt(d)
    return y.astype(F32), q.astype(F32)


def _params(m, bits, extra=f"aq_threshold={T}"):
    p = f"ncentroids={NLIST}, M={m}" + (", bit_size=4" if bits == 4 else "")
    return p + (", " + extra if extra else "")


def _read(path, bits):
    return P.read_index4(path) if bits == 4 else R.read_index(path)


def _saved(ix, path, bits):
    ix.save(path)
    return _read(path, bits)


def _stored_codes(s, bits):
    ids, lst, pay = s.flat()
    return ids, lst, (P.unpack(pay, s.m) if bits == 4 else pay[:, :s.m]).astype(np.int64)


def code_problems(s, bits, eta, codes=None):
    """Rows whose stored codes differ from the reference encoder, ignoring rows it flags ambiguous.  Returns (mismatching
    unambiguous rows, ambiguous rows)."""
    ids, lst, got = _stored_codes(s, bits)
    if codes is not None:
        got = codes
    X = s.rows.astype(np.float64)[ids]
    want, amb, _ = A.encode(X, s.centroids, lst, s.codebook, eta)
    bad = np.nonzero((want != got).any(1) & ~amb)[0]
    return bad, amb


def _assert_codes(s, bits, eta, what):
    bad, amb = code_problems(s, bits, eta)
    n_amb = int(amb.sum())
    assert n_amb <= AMBIGUOUS_MAX * s.n, f"test data design error: {n_amb} of {s.n} rows have an fp32-ambiguous decision"
    assert len(bad) == 0, f"{what}: {len(bad)} rows differ from the reference encoder (first {bad[:5]}); {n_amb} ambiguous"


def _search_parity(s, ix, q, bits, nprobe=4, k=10):
    dg, ig = ix.search(q, k, f"nprobe={nprobe}", first_stage_only=True)
    if bits == 4:
        ref = P.reference_search(s, q, k, nprobe)
    elif L.is_lut(s):
        ref = L.reference_search(s, q, k, nprobe)
    else:
        ref = R.reference_search(s, q, k, nprobe)
    bad = R.compare(ref, dg, ig)
    assert not bad, f"{len(bad)} problems, first: {bad[:6]}"


class _Cache:
    def __init__(self, tmp):
        self.tmp, self.got = tmp, {}

    def get(self, case):
        if case not in self.got:
            typ, metric, d, m, bits = case
            y, q = _data(N, d, seed=d + 7 * m + metric)
            ix = b2.VectorIndex(typ, metric, d, _params(m, bits)).build(y)
            assert ix.info()["uses_ivf"]
            s = _saved(ix, self.tmp / f"{typ}_{metric}_{d}_{m}_{bits}.b2ix", bits)
            self.got[case] = (ix, s, y, q)
        return self.got[case]


@pytest.fixture(scope="module")
def cache(tmp_path_factory):
    return _Cache(tmp_path_factory.mktemp("aq"))


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_codes_match_the_reference_encoder(cache, case):
    ix, s, y, q = cache.get(case)
    assert (s.m, s.dsub) == (case[3], case[2] // case[3])
    _assert_codes(s, case[4], A.eta_of(case[2], T), "one-shot build")


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_first_stage_matches_the_stored_index(cache, case):
    ix, s, y, q = cache.get(case)
    for nprobe in (1, 4, NLIST):
        _search_parity(s, ix, q, case[4], nprobe)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_train_loss_never_increases_and_ends_below_nearest_codes(cache, case):
    ix, s, y, q = cache.get(case)
    eta, traj = ix.train_loss()
    assert eta == pytest.approx(A.eta_of(case[2], T), rel=1e-12)
    assert len(traj) == 1 + A.ITERS
    assert (np.diff(traj) <= 1e-9 * traj[0]).all(), traj
    # the stored rows are the training sample (N < 65 536 rows); the loss of their nearest codes under the final codebooks is
    # at least the loss of the anisotropic codes, and the trajectory ends at or below it
    ids, lst, _ = _stored_codes(s, case[4])
    X = s.rows.astype(np.float64)[ids]
    near, _ = A.nearest(X, s.centroids, lst, s.codebook)
    assert traj[-1] < A.mean_loss(X, s.centroids, lst, s.codebook, near, eta)


def trajectory_problems(got_traj, got_cb, want_traj, want_cb, rtol=2e-3, cb_rtol=2e-2):
    """The stated tolerance of the trajectory comparator: every mean loss within rtol, the codebooks within cb_rtol in
    Frobenius norm (a few sample rows may take another code where the k-means codebooks differ in the last bits)."""
    bad = []
    if len(got_traj) != len(want_traj):
        return [f"{len(got_traj)} losses, want {len(want_traj)}"]
    for i, (g, w) in enumerate(zip(got_traj, want_traj)):
        if abs(g - w) > rtol * abs(w):
            bad.append(f"loss {i}: {g} vs reference {w}")
    diff = np.linalg.norm(got_cb.astype(np.float64) - want_cb) / np.linalg.norm(want_cb)
    if diff > cb_rtol:
        bad.append(f"codebooks differ by {diff:.3g} (relative Frobenius)")
    return bad


@pytest.mark.parametrize("case", [CASES[3], CASES[7]], ids=[IDS[3], IDS[7]])
def test_training_follows_the_reference_trajectory(cache, case, tmp_path):
    ix, s, y, q = cache.get(case)
    typ, metric, d, m, bits = case
    plain = b2.VectorIndex(typ, metric, d, _params(m, bits, extra="")).build(y)
    sp = _saved(plain, tmp_path / "plain.b2ix", bits)
    # same k-means on the same rows: the centroids agree up to the order of fp32 sums
    assert np.allclose(sp.centroids, s.centroids, rtol=1e-4, atol=1e-6), "test data design error: k-means diverged"
    ids, lst, _ = _stored_codes(s, bits)
    order = np.argsort(ids)                       # the sample is the rows in id order
    X, lists = s.rows.astype(np.float64)[ids][order], lst[order]
    eta, traj = ix.train_loss()
    cb, want, n_amb = A.train(X, s.centroids, lists, sp.codebook, eta)
    assert n_amb <= AMBIGUOUS_MAX * len(X) * A.ITERS, f"test data design error: {n_amb} ambiguous encodings"
    bad = trajectory_problems(traj, s.codebook, want, cb)
    assert not bad, bad
    # negative control: one codebook entry moved by more than the tolerance is rejected
    moved = s.codebook.copy()
    moved[0, 0, 0] += 0.05 * np.linalg.norm(cb)
    assert trajectory_problems(traj, moved, want, cb), "negative control: the trajectory comparator accepts a moved codeword"
    plain.close()


def test_negative_control_swapped_code_is_rejected(cache):
    case = CASES[1]
    ix, s, y, q = cache.get(case)
    ids, lst, codes = _stored_codes(s, case[4])
    _, amb = code_problems(s, case[4], A.eta_of(case[2], T))
    row = int(np.nonzero(~amb)[0][5])
    codes = codes.copy()
    codes[row, 3] = (codes[row, 3] + 1) % 256
    bad, _ = code_problems(s, case[4], A.eta_of(case[2], T), codes)
    assert row in bad, "negative control: the code comparator accepts a swapped code"


@pytest.mark.parametrize("case", [CASES[1], CASES[6]], ids=[IDS[1], IDS[6]])
def test_streamed_build_and_duplicate_rows(case, tmp_path):
    typ, metric, d, m, bits = case
    y, q = _data(N, d, seed=11 + d)
    ix = b2.VectorIndex(typ, metric, d, _params(m, bits)).reserve(2 * N).train(y)
    off, sizes, i = 0, [1, 255, 257, 1000], 0
    while off < N:
        ix.add(y[off:off + sizes[i % 4]])
        off += sizes[i % 4]
        i += 1
    ix.add(y)   # the same rows again, as ids N .. 2N - 1
    ix.finalize()
    s = _saved(ix, tmp_path / "s.b2ix", bits)
    _assert_codes(s, bits, A.eta_of(d, T), "streamed build")
    ids, _, codes = _stored_codes(s, bits)
    by_id = np.empty_like(codes)
    by_id[ids] = codes
    assert (by_id[:N] == by_id[N:]).all(), "identical rows must get identical codes"
    _search_parity(s, ix, q, bits)


@pytest.mark.parametrize("case", [CASES[3], CASES[6]], ids=[IDS[3], IDS[6]])
def test_device_build_save_load_and_host_rows(case, tmp_path):
    torch = pytest.importorskip("torch")
    typ, metric, d, m, bits = case
    y, q = _data(N, d, seed=5 + d)
    ty = torch.from_numpy(y).cuda()
    ix = b2.VectorIndex(typ, metric, d, _params(m, bits, f"aq_threshold={T}, keep_raw=2, refine_factor=4"))
    ix.reserve(N).train_device(ty.data_ptr(), N).add_device(ty.data_ptr(), N).finalize()
    torch.cuda.synchronize()
    s = _saved(ix, tmp_path / "a.b2ix", bits)
    _assert_codes(s, bits, A.eta_of(d, T), "device build, rows in host memory")
    two = ix.search(q, 10, "nprobe=4")
    ix.set_raw_placement(1)
    one = ix.search(q, 10, "nprobe=4")
    assert np.array_equal(two[0], one[0]) and np.array_equal(two[1], one[1]), "keep_raw=2 must answer as keep_raw=1"
    ix.save(tmp_path / "b.b2ix")
    back = b2.VectorIndex.load(tmp_path / "b.b2ix", d, metric)
    got = back.search(q, 10, "nprobe=4")
    assert np.array_equal(got[0], one[0]) and np.array_equal(got[1], one[1])
    back.save(tmp_path / "c.b2ix")
    assert (tmp_path / "b.b2ix").read_bytes() == (tmp_path / "c.b2ix").read_bytes()
    with pytest.raises(b2.search.B200Error) as e:
        back.train_loss()
    assert e.value.code == ERR_INVALID
    # filter-aware probing composes with the AQ codes
    alive = np.zeros(N, bool)
    alive[::7] = True
    dg, ig = ix.search(q, 10, "nprobe=2, filter_probe=1", alive_bits=np.packbits(alive, bitorder="little"))
    assert alive[ig[ig >= 0]].all()
    back.close()
    ix.close()


@pytest.mark.parametrize("value", ["-0.2", "1", "1.5", "abc", "nan"])
def test_bad_thresholds_are_refused_at_create(value):
    with pytest.raises(b2.search.B200Error) as e:
        b2.VectorIndex("SCANN", b2.IP, 64, f"aq_threshold={value}")
    assert e.value.code == ERR_INVALID


@pytest.mark.parametrize("typ", ["IVFPQ", "SCANN", "HNSWPQ"])
def test_l2_is_refused_at_create(typ):
    with pytest.raises(b2.search.B200Error) as e:
        b2.VectorIndex(typ, b2.L2, 64, "aq_threshold=0.2")
    assert e.value.code == ERR_UNSUPPORTED
    b2.VectorIndex(typ, b2.L2, 64, "aq_threshold=0").close()


def test_long_sub_vectors_are_refused_at_train():
    y, _ = _data(N, 256, seed=3)
    ix = b2.VectorIndex("IVFPQ", b2.IP, 256, f"ncentroids={NLIST}, M=2, aq_threshold=0.2")
    with pytest.raises(b2.search.B200Error) as e:
        ix.build(y)
    assert e.value.code == ERR_UNSUPPORTED and "64" in str(e.value)


def test_other_types_ignore_the_key_and_zero_is_plain(tmp_path):
    for typ in ("IVFFLAT", "IVFSQ", "FLAT", "MSTG"):
        b2.VectorIndex(typ, b2.L2, 64, "aq_threshold=abc").close()
    y, q = _data(N, 64, seed=9)
    zero = b2.VectorIndex("IVFPQ", b2.IP, 64, "ncentroids=16, M=16, aq_threshold=0").build(y)
    absent = b2.VectorIndex("IVFPQ", b2.IP, 64, "ncentroids=16, M=16").build(y)
    for ix in (zero, absent):
        with pytest.raises(b2.search.B200Error) as e:
            ix.train_loss()
        assert e.value.code == ERR_INVALID
    a, b = _saved(zero, tmp_path / "z.b2ix", 8), _saved(absent, tmp_path / "a.b2ix", 8)
    assert (tmp_path / "z.b2ix").stat().st_size == (tmp_path / "a.b2ix").stat().st_size
    # both are plain PQ: every code is its nearest codeword (eta = 1 makes the anisotropic encoder the nearest search)
    for s in (a, b):
        bad, _ = code_problems(s, 8, 1.0)
        assert len(bad) == 0
