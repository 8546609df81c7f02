"""Optimised product quantisation (`opq=1`) on IVFPQ / SCANN / HNSWPQ, against tests/opq_reference.py.

An opq=1 index learns an orthonormal rotation R and keeps its inverted-file side (centroids, codebooks, codes, norm terms) in
the rotated space; the fp32 rows and every exact path stay unrotated.  Checked here:

* R: orthonormal within 1e-5 in float64 (also on rank-deficient data: constant columns, a training sample smaller than d),
  exactly I at opq_iters=0, the same in the file and through b200_index_opq; more lists than PQ sample rows;
* the stored index, through the existing list, code and norm-term checks run on the rotated rows;
* the first stage against the float64 reference of the stored index on prepared-then-rotated queries, the second stage
  against ivf_reference.rerank of the first stage's candidates (integer data: the exact keys are exact);
* quality on low-rank data (loss trajectory, recall against plain PQ) and an isotropic control;
* streamed builds, save / load, keep_raw=2, the device entry, sharded search, filters (with and without filter_probe=1),
  aq_threshold, a 1 025-query batch against single queries, and the refusals.

The k-means under the codebooks sums with fp32 atomics, so two builds are held to invariants, not compared byte for byte."""
import numpy as np
import pytest

import myscaledb_b200 as b2
from myscaledb_b200.search import B200Error
from tests import aq_reference as A
from tests import ivf_reference as R
from tests import opq_reference as O
from tests import pq4_reference as P

pytestmark = pytest.mark.gpu
F32 = np.float32
ERR_INVALID, ERR_UNSUPPORTED = 1, 3
N, NLIST, ITERS = 4000, 16, 4

# (type, metric, d, M, bits): the tensor-core decoder at d / M = 1, 2, 4, 8, the look-up scan at 768 / 48, 4-bit codes at M = 96
CASES = [("IVFPQ", b2.L2, 64, 64, 8), ("SCANN", b2.IP, 64, 32, 8), ("HNSWPQ", b2.COSINE, 64, 16, 8), ("IVFPQ", b2.L2, 128, 16, 8),
         ("SCANN", b2.COSINE, 768, 48, 8), ("IVFPQ", b2.IP, 768, 96, 4)]
IDS = [f"{t}-{ {b2.L2: 'l2', b2.IP: 'ip', b2.COSINE: 'cos'}[mt]}-d{d}-M{m}-{b}bit" for t, mt, d, m, b in CASES]


def _data(n, d, seed, nq=32):
    """Clusters in a low-rank subspace plus noise (what OPQ is for), with a common offset so inner products are not all 0."""
    rng = np.random.default_rng(seed)
    rank = max(4, d // 4)
    basis = rng.standard_normal((rank, d)) / np.sqrt(rank)
    centres = 3.0 * rng.standard_normal((NLIST, rank))
    mean = rng.standard_normal(d) / np.sqrt(d)
    lab = rng.integers(0, NLIST, n)
    y = (centres[lab] + rng.standard_normal((n, rank))) @ basis + mean + 0.05 * rng.standard_normal((n, d))
    q = (centres[rng.integers(0, NLIST, nq)] + rng.standard_normal((nq, rank))) @ basis + mean + 0.05 * rng.standard_normal((nq, d))
    return y.astype(F32), q.astype(F32)


def _params(m, bits, extra=""):
    p = f"ncentroids={NLIST}, M={m}, opq=1, opq_iters={ITERS}" + (", bit_size=4" if bits == 4 else "")
    return p + (", " + extra if extra else "")


def _check_search(s, rot, bits, ix, q, nprobe, k=10, alive=None, params=""):
    dg, ig = ix.search(q, k, f"nprobe={nprobe}" + params, first_stage_only=True, alive_bits=None if alive is None else _bits(alive))
    bad = R.compare(O.reference_search(s, rot, bits, q, k, nprobe, alive=alive), dg, ig)
    assert not bad, f"{len(bad)} problems, first: {bad[:6]}"
    return dg, ig


def _bits(alive):
    b = np.packbits(np.asarray(alive, bool), bitorder="little")
    return np.concatenate([b, np.zeros((-len(b)) % 4, np.uint8)])


def _check_rotation(ix, rot_file, iters=ITERS):
    rot, loss = ix.opq()
    assert rot.tobytes() == rot_file.tobytes(), "b200_index_opq and the file disagree on R"
    assert O.orthonormal_error(rot) <= 1e-5, O.orthonormal_error(rot)
    assert len(loss) == 1 + iters and np.isfinite(loss).all() and (loss >= 0).all()
    return rot, loss


class _Cache:
    def __init__(self, tmp):
        self.tmp, self.got = tmp, {}

    def get(self, case):
        if case not in self.got:
            typ, metric, d, m, bits = case
            y, q = _data(N, d, seed=d + 7 * m + metric)
            ix = b2.VectorIndex(typ, metric, d, _params(m, bits)).build(y)
            assert ix.info()["uses_ivf"]
            path = self.tmp / f"{typ}_{metric}_{d}_{m}_{bits}.b2ix"
            ix.save(path)
            s, rot, got_bits = O.read_index(path)
            assert got_bits == bits
            self.got[case] = (ix, s, rot, y, q, path)
        return self.got[case]


@pytest.fixture(scope="module")
def cache(tmp_path_factory):
    return _Cache(tmp_path_factory.mktemp("opq"))


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_rotation_and_stored_index(cache, case):
    ix, s, rot, y, q, _ = cache.get(case)
    assert (s.m, s.dsub) == (case[3], case[2] // case[3])
    _check_rotation(ix, rot)
    O.check_build(s, rot, case[4], ix, y)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_first_stage_matches_the_stored_index(cache, case):
    ix, s, rot, y, q, _ = cache.get(case)
    for nprobe in (1, 4, NLIST):
        _check_search(s, rot, case[4], ix, q, nprobe)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_batch_of_1025_and_single_queries_match_the_reference(cache, case):
    ix, s, rot, y, q, _ = cache.get(case)
    rng = np.random.default_rng(5)
    qq = (y[rng.integers(0, N, 1025)] + 0.05 * rng.standard_normal((1025, case[2]))).astype(F32)
    _check_search(s, rot, case[4], ix, qq, 4)
    ref = O.reference_search(s, rot, case[4], qq[:6], 10, 4)
    got = [ix.search(qq[i:i + 1], 10, "nprobe=4", first_stage_only=True) for i in range(6)]
    bad = R.compare(ref, np.concatenate([g[0] for g in got]), np.concatenate([g[1] for g in got]))
    assert not bad, bad[:6]


@pytest.mark.parametrize("case", [CASES[0], CASES[3], CASES[5]], ids=[IDS[0], IDS[3], IDS[5]])
def test_second_stage_reranks_the_first_stage_unrotated(tmp_path, case):
    """Integer rows and queries: the exact fp32 keys are exact, so the answer equals ivf_reference.rerank byte for byte."""
    typ, metric, d, m, bits = case
    rng = np.random.default_rng(11)
    centres = rng.integers(-8, 9, (NLIST, d))
    y = (centres[rng.integers(0, NLIST, N)] + rng.integers(-2, 3, (N, d))).astype(F32)
    q = (centres[rng.integers(0, NLIST, 16)] + rng.integers(-2, 3, (16, d))).astype(F32)
    ix = b2.VectorIndex(typ, metric, d, _params(m, bits, "keep_raw=1")).build(y)
    k, rf = 10, 4
    ix.save(tmp_path / "ix.b2ix")
    s, rot, _ = O.read_index(tmp_path / "ix.b2ix")
    _, cand = ix.search(q, k * rf, "nprobe=4", first_stage_only=True)
    dg, ig = ix.search(q, k, f"nprobe=4, refine_factor={rf}")
    dr, ir = R.rerank(s.rows, R.prepare_queries(q, metric), cand, k, metric)
    assert np.array_equal(ig, ir) and dg.tobytes() == dr.tobytes()
    dh, ih = ix.refine(q, cand, k)
    assert np.array_equal(ih, ir) and dh.tobytes() == dr.tobytes()
    ix.close()


def _low_rank(n, d, rank, seed, noise=0.05):
    rng = np.random.default_rng(seed)
    basis = rng.standard_normal((rank, d))
    y = rng.standard_normal((n, rank)) @ basis + noise * rng.standard_normal((n, d))
    q = rng.standard_normal((200, rank)) @ basis + noise * rng.standard_normal((200, d))
    return y.astype(F32), q.astype(F32)


def _clustered(n, d, seed):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((64, d))
    y = centres[rng.integers(0, 64, n)] + 0.5 * rng.standard_normal((n, d))
    q = centres[rng.integers(0, 64, 200)] + 0.5 * rng.standard_normal((200, d))
    return y.astype(F32), q.astype(F32)


def _recall(ix, y, q, nlist):
    _, ig = ix.search(q, 10, f"nprobe={nlist}", first_stage_only=True)
    d2 = (q.astype(np.float64) ** 2).sum(1)[:, None] + (y.astype(np.float64) ** 2).sum(1)[None, :] - 2 * q.astype(np.float64) @ y.astype(np.float64).T
    truth = np.argsort(d2, axis=1)[:, :10]
    return np.mean([len(set(a) & set(b)) / 10 for a, b in zip(ig, truth)])


def test_quality_on_low_rank_data_and_isotropic_control():
    n, d, nl = 20000, 64, 16
    base = f"ncentroids={nl}, M=8"
    y, q = _low_rank(n, d, 16, seed=3)
    plain = b2.VectorIndex("IVFPQ", b2.L2, d, base).build(y)
    opq = b2.VectorIndex("IVFPQ", b2.L2, d, base + ", opq=1").build(y)
    rot, loss = opq.opq()
    assert len(loss) == 21
    assert (loss[1:] <= loss[:-1] * 1.01).all(), loss
    assert loss[-1] <= 0.5 * loss[0], loss
    r_plain, r_opq = _recall(plain, y, q, nl), _recall(opq, y, q, nl)
    assert r_opq >= r_plain + 0.10, (r_plain, r_opq, loss)
    y, q = _clustered(n, d, seed=4)
    plain2 = b2.VectorIndex("IVFPQ", b2.L2, d, base).build(y)
    opq2 = b2.VectorIndex("IVFPQ", b2.L2, d, base + ", opq=1").build(y)
    c_plain, c_opq = _recall(plain2, y, q, nl), _recall(opq2, y, q, nl)
    assert c_opq >= c_plain - 0.02, (c_plain, c_opq)
    print(f"low-rank recall@10 plain {r_plain:.3f} opq {r_opq:.3f}; loss {loss[0]:.4g} -> {loss[-1]:.4g}; "
          f"clustered plain {c_plain:.3f} opq {c_opq:.3f}")
    for ix in (plain, opq, plain2, opq2):
        ix.close()


def test_rank_deficient_data_and_identity_control(tmp_path):
    d = 64
    y, q = _data(N, d, seed=21)
    y[:, 16:32] = 1.25                    # 16 constant columns: M = Res^T Res^ is rank-deficient
    ix = b2.VectorIndex("IVFPQ", b2.L2, d, f"ncentroids={NLIST}, M=16, opq=1").build(y)
    ix.save(tmp_path / "a.b2ix")
    s, rot, bits = O.read_index(tmp_path / "a.b2ix")
    _check_rotation(ix, rot, iters=20)
    O.check_build(s, rot, bits, ix, y)
    _check_search(s, rot, bits, ix, q, 4)
    eye = b2.VectorIndex("SCANN", b2.IP, d, f"ncentroids={NLIST}, M=16, opq=1, opq_iters=0").build(y)
    r0, l0 = eye.opq()
    assert np.array_equal(r0, np.eye(d, dtype=F32)) and len(l0) == 1
    # memory: the same shape without the key holds the same pool, lists and codebooks; R adds d x d fp32
    plain = b2.VectorIndex("SCANN", b2.IP, d, f"ncentroids={NLIST}, M=16").build(y)
    assert eye.memory_bytes() - plain.memory_bytes() == d * d * 4
    for i in (ix, eye, plain):
        i.close()


@pytest.mark.parametrize("case", [("IVFPQ", b2.L2, 64, 16), ("SCANN", b2.IP, 128, 16)], ids=["IVFPQ-l2-d64", "SCANN-ip-d128"])
def test_sample_smaller_than_d_keeps_r_orthonormal(tmp_path, case):
    """48 training rows at d = 64 / 128: M = Res^T Res^ has rank < 48, and its null space has no preferred axes, so every
    null column of U must be completed in a general direction."""
    typ, metric, d, m = case
    y, q = _data(N, d, seed=81 + d)
    ix = b2.VectorIndex(typ, metric, d, f"ncentroids={NLIST}, M={m}, opq=1")
    ix.reserve(N)
    ix.train(y[:48])
    ix.add(y)
    ix.finalize()
    assert ix.info()["uses_ivf"]
    ix.save(tmp_path / "few.b2ix")
    s, rot, bits = O.read_index(tmp_path / "few.b2ix")
    _check_rotation(ix, rot, iters=20)
    O.check_build(s, rot, bits, ix, y)
    _check_search(s, rot, bits, ix, q, 4)
    ld = b2.VectorIndex.load(tmp_path / "few.b2ix", d, metric)
    assert ld.opq()[0].tobytes() == rot.tobytes()
    a, b = ld.search(q, 10, "nprobe=4"), ix.search(q, 10, "nprobe=4")
    assert a[0].tobytes() == b[0].tobytes() and np.array_equal(a[1], b[1])
    ld.close()
    ix.close()


def test_more_lists_than_the_pq_sample(tmp_path):
    """nlist = 70 000 > the 65 536-row PQ sample: the rotated centroids outnumber the sample rows."""
    d, nl, n = 8, 70000, 70000
    rng = np.random.default_rng(91)
    y = rng.standard_normal((n, d)).astype(F32)
    ix = b2.VectorIndex("IVFPQ", b2.L2, d, f"ncentroids={nl}, M=4, opq=1, opq_iters=2")
    ix.reserve(8 * nl)
    ix.train(y)
    ix.add(y)
    ix.finalize()
    assert ix.info()["uses_ivf"] and ix.info()["nlist"] == nl
    ix.save(tmp_path / "wide.b2ix")
    s, rot, bits = O.read_index(tmp_path / "wide.b2ix")
    _check_rotation(ix, rot, iters=2)
    # a sample of rows: each in the list of its nearest stored (rotated) centroid
    ids, lst, _ = s.flat()
    pick = rng.choice(len(ids), 300, replace=False)
    X = s.rows.astype(np.float64)[ids[pick]] @ rot.astype(np.float64)
    C = s.centroids.astype(np.float64)
    dist = (X * X).sum(1)[:, None] + (C * C).sum(1)[None, :] - 2 * X @ C.T
    tol = 1e-5 * ((X * X).sum(1)[:, None] + (C * C).sum(1)[None, :] + 2 * np.abs(X) @ np.abs(C).T)
    own = dist[np.arange(len(pick)), lst[pick]]
    assert (own <= dist.min(1) + tol[np.arange(len(pick)), lst[pick]]).all(), "a row is not in its nearest rotated list"
    q = (y[rng.integers(0, n, 8)] + 0.01 * rng.standard_normal((8, d))).astype(F32)
    _check_search(s, rot, bits, ix, q, 4)
    ix.close()


def test_streamed_build_save_load_keep_raw_2_and_device_entry(tmp_path):
    import torch
    typ, metric, d, m, bits = CASES[3]
    y, q = _data(N, d, seed=31)
    ix = b2.VectorIndex(typ, metric, d, _params(m, bits))
    ix.reserve(N)
    ix.train(y[::2])
    for off in range(0, N, 900):
        ix.add(y[off:off + 900])
    ix.finalize()
    ix.save(tmp_path / "s.b2ix")
    s, rot, _ = O.read_index(tmp_path / "s.b2ix")
    _check_rotation(ix, rot)
    O.check_build(s, rot, bits, ix, y)
    _check_search(s, rot, bits, ix, q, 4)
    params = "nprobe=4, refine_factor=4"
    want = ix.search(q, 10, params)
    # device entry = host entry
    tq = torch.from_numpy(q).cuda()
    od = torch.empty((len(q), 10), dtype=torch.float32, device="cuda")
    oi = torch.empty((len(q), 10), dtype=torch.int64, device="cuda")
    ix.search_device(tq.data_ptr(), len(q), 10, od.data_ptr(), oi.data_ptr(), params=params)
    torch.cuda.synchronize()
    assert od.cpu().numpy().tobytes() == want[0].tobytes() and np.array_equal(oi.cpu().numpy(), want[1])
    # save / load: the same R, no trajectory, the same answers
    ld = b2.VectorIndex.load(tmp_path / "s.b2ix", d, metric)
    r2, l2 = ld.opq()
    assert r2.tobytes() == rot.tobytes() and len(l2) == 0
    got = ld.search(q, 10, params)
    assert got[0].tobytes() == want[0].tobytes() and np.array_equal(got[1], want[1])
    # keep_raw=2: the re-rank rows in host memory answer byte for byte as in HBM
    ix.set_raw_placement(2)
    got = ix.search(q, 10, params)
    assert got[0].tobytes() == want[0].tobytes() and np.array_equal(got[1], want[1])
    ix.close()
    ld.close()


def test_sharded_search_at_world_size_1_equals_the_index_search():
    import torch
    from myscaledb_b200.sharding import Comm
    typ, metric, d, m, bits = CASES[1]
    y, q = _data(N, d, seed=41)
    ix = b2.VectorIndex(typ, metric, d, _params(m, bits)).build(y)
    comm = Comm(0, 1, Comm.unique_id())
    st = torch.cuda.Stream()
    tq = torch.from_numpy(q).cuda()
    outs = []
    for sharded in (False, True):
        od = torch.empty((len(q), 10), dtype=torch.float32, device="cuda")
        oi = torch.empty((len(q), 10), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        if sharded:
            comm.sharded_index_search(ix, metric, tq.data_ptr(), len(q), 10, "nprobe=4", od.data_ptr(), oi.data_ptr(), 0, st.cuda_stream)
        else:
            ix.search_device(tq.data_ptr(), len(q), 10, od.data_ptr(), oi.data_ptr(), params="nprobe=4", stream=st.cuda_stream)
        st.synchronize()
        outs.append((od.cpu().numpy(), oi.cpu().numpy()))
    assert outs[0][0].tobytes() == outs[1][0].tobytes() and np.array_equal(outs[0][1], outs[1][1])
    torch.cuda.synchronize()
    comm.close()
    ix.close()


@pytest.mark.parametrize("case", [CASES[0], CASES[4]], ids=[IDS[0], IDS[4]])
def test_filtered_search_with_and_without_filter_probe(cache, case):
    ix, s, rot, y, q, _ = cache.get(case)
    bits = case[4]
    alive = np.random.default_rng(9).random(N) < 0.05
    for nprobe in (4, NLIST):
        _check_search(s, rot, bits, ix, q, nprobe, alive=alive)
    # filter_probe=1 at nlist: the page skipping alone, the same answers as the plain probe
    _check_search(s, rot, bits, ix, q, NLIST, alive=alive, params=", filter_probe=1")
    # below nlist: every query probes p_q lists (b200_index_last_probe), its first k kept rows; the answer is the reference's
    # probing p_q lists, and complete
    dg, ig = ix.search(q, 10, "nprobe=2, filter_probe=1", first_stage_only=True, alive_bits=_bits(alive))
    depth = ix.last_probe()[0]
    for p in sorted(set(depth.tolist())):
        sel = np.nonzero(depth == p)[0]
        bad = R.compare(O.reference_search(s, rot, bits, q[sel], 10, int(p), alive=alive), dg[sel], ig[sel])
        assert not bad, (p, bad[:6])
    assert ((ig >= 0).sum(1) == min(10, int(alive.sum()))).all()


def test_aq_threshold_with_opq_encodes_the_rotated_rows(tmp_path):
    d, m, t = 64, 16, 0.2
    y, q = _data(N, d, seed=51)
    ix = b2.VectorIndex("SCANN", b2.IP, d, f"ncentroids={NLIST}, M={m}, opq=1, opq_iters={ITERS}, aq_threshold={t}").build(y)
    ix.save(tmp_path / "aq.b2ix")
    s, rot, bits = O.read_index(tmp_path / "aq.b2ix")
    _check_rotation(ix, rot)
    ids, lst, pay = s.flat()
    X = O.rotated(s, rot).rows.astype(np.float64)[ids]
    want, amb, _ = A.encode(X, s.centroids, lst, s.codebook, A.eta_of(d, t))
    bad = np.nonzero((want != pay[:, :m].astype(np.int64)).any(1) & ~amb)[0]
    assert int(amb.sum()) <= 0.2 * len(ids), "test data design error: too many fp32-ambiguous rows"
    assert len(bad) == 0, f"{len(bad)} rows differ from the reference encoder on the rotated rows"
    _check_search(s, rot, bits, ix, q, 4)
    ix.close()


def test_small_part_is_flat_without_a_rotation():
    y, q = _data(500, 64, seed=61)
    ix = b2.VectorIndex("IVFPQ", b2.L2, 64, "M=16, opq=1").build(y)
    assert not ix.info()["uses_ivf"]
    with pytest.raises(B200Error) as e:
        ix.opq()
    assert e.value.code == ERR_INVALID
    dg, ig = ix.search(q, 5)
    d2 = ((q[:, None, :].astype(np.float64) - y[None, :, :]) ** 2).sum(2)
    assert np.array_equal(ig[:, 0], d2.argmin(1))
    ix.close()


def test_refusals_ignores_and_corrupt_rotation(cache, tmp_path):
    for params, code in (("opq=2", ERR_INVALID), ("opq=1, opq_iters=-1", ERR_INVALID), ("opq=-1", ERR_INVALID)):
        with pytest.raises(B200Error) as e:
            b2.VectorIndex("IVFPQ", b2.L2, 64, params)
        assert e.value.code == code, params
    with pytest.raises(B200Error) as e:
        b2.VectorIndex("SCANN", b2.L2, 4104, "opq=1")
    assert e.value.code == ERR_UNSUPPORTED
    # the other types ignore the key: a v2 file of the same size as without it
    y, _ = _data(N, 64, seed=71)
    for typ in ("IVFSQ", "IVFFLAT", "MSTG"):
        sizes = []
        for extra in ("", ", opq=1"):
            ix = b2.VectorIndex(typ, b2.L2, 64, f"ncentroids={NLIST}" + extra).build(y)
            path = tmp_path / f"{typ}{len(extra)}.b2ix"
            ix.save(path)
            raw = open(path, "rb").read()
            assert np.frombuffer(raw, R.HEADER, count=1)[0]["version"] == 2
            sizes.append(len(raw))
            with pytest.raises(B200Error) as e:
                ix.opq()
            assert e.value.code == ERR_INVALID
            ix.close()
        assert sizes[0] == sizes[1], typ
    plain = b2.VectorIndex("IVFPQ", b2.L2, 64, f"ncentroids={NLIST}, M=16").build(y)
    with pytest.raises(B200Error) as e:
        plain.opq()
    assert e.value.code == ERR_INVALID
    plain.close()
    # a v5 file whose R is no longer orthonormal, or not finite, is refused at load
    ix, s, rot, y, q, path = cache.get(CASES[0])
    raw = bytearray(open(path, "rb").read())
    d = s.d
    at = len(raw) - d * d * 4
    for bad in (rot[0, 0] * 1.01 + 1e-3, np.nan):
        b = bytearray(raw)
        b[at:at + 4] = np.array([bad], "<f4").tobytes()
        p = tmp_path / "bad.b2ix"
        open(p, "wb").write(bytes(b))
        with pytest.raises(B200Error) as e:
            b2.VectorIndex.load(p, d, CASES[0][1])
        assert e.value.code == ERR_INVALID
    # negative control of the reader: the unmodified file loads and answers as the built index
    ld = b2.VectorIndex.load(path, d, CASES[0][1])
    a, b = ld.search(q, 10, "nprobe=4"), ix.search(q, 10, "nprobe=4")
    assert a[0].tobytes() == b[0].tobytes() and np.array_equal(a[1], b[1])
    ld.close()
