"""The binary inverted-file reference (tests/binary_ivf_reference.py) on a tiny hand-built index file, without a GPU: its reader
decodes the B2IX layout, its search equals a plain Python loop over the same lists, and its comparator rejects each fault it
is meant to catch."""
import numpy as np
import pytest

from tests import binary_ivf_reference as B
from tests import ivf_reference as R

FLT_MAX = np.float32(np.finfo(np.float32).max)


def encode(metric, nbits, centroids, lists, y, index_type=10):
    """B2IX v2 bytes of a binary inverted-file index: `lists` are the row ids of each list, y the rows u8 [n][nbits / 8]."""
    rb = nbits // 8
    kb_w, row_pad, cent_pad = B.geometry(rb)
    h = np.zeros(1, R.HEADER)
    h["magic"], h["version"], h["type"], h["metric"], h["d"] = b"B2IX", 2, index_type, metric, nbits
    h["nlist"], h["default_nprobe"], h["refine_factor"], h["payload"], h["use_ivf"] = len(lists), 1, 1, 3, 1
    h["n"], h["pages_used"] = len(y), sum(-(-len(a) // B.PAGE) for a in lists)
    cent = np.zeros((len(lists), cent_pad), np.uint8)
    cent[:, :rb] = centroids
    out = [h.tobytes(), cent.tobytes(), np.array([len(a) for a in lists], "<u4").tobytes()]
    for ids in lists:
        for p0 in range(0, len(ids), B.PAGE):
            pid = np.asarray(ids[p0:p0 + B.PAGE], np.int64)
            page = np.zeros((B.PAGE, row_pad), np.uint8)
            page[:len(pid), :rb] = y[pid]
            out.append(page.reshape(B.PAGE, row_pad // kb_w, kb_w).transpose(1, 0, 2).tobytes())
            out.append(np.pad(pid, (0, B.PAGE - len(pid))).astype("<u4").tobytes())
            out.append(np.pad(B.popcount_rows(page[:len(pid)]), (0, B.PAGE - len(pid))).astype("<f4").tobytes())
    return b"".join(out)


def popc(v):
    return bin(v).count("1")


def loop_search(metric, y, centroids, lists, q, k, nprobe, alive=None):
    """The search restated with Python integers, one row at a time."""
    ints = lambda b: [int.from_bytes(bytes(r), "little") for r in b]
    Y, C, Q = ints(y), ints(centroids), ints(q)
    ids = np.full((len(Q), k), -1, np.int64)
    dis = np.full((len(Q), k), FLT_MAX, np.float32)
    for i, x in enumerate(Q):
        order = sorted(range(len(C)), key=lambda l: (popc(x ^ C[l]), l))
        probed = order if nprobe >= len(C) else order[:nprobe]
        cand = []
        for l in probed:
            for r in lists[l]:
                if alive is not None and not (alive[r // 8] >> (r % 8)) & 1:
                    continue
                a, o = popc(x & Y[r]), popc(x | Y[r])
                key = np.float32(o - a) if metric == B.HAMMING else (np.float32(0) if o == 0 else np.float32(o - a) / np.float32(o))
                cand.append((key, r))
        cand.sort()
        for j, (key, r) in enumerate(cand[:k]):
            ids[i, j], dis[i, j] = r, key
    return dis, ids


def tiny(nbits, rng):
    """Three lists around three centres (one of them spanning two pages), with duplicate rows, an all-zero row and rows equal
    to a centre; queries include an all-zero one, a copy of a row and ones equidistant from two centres."""
    rb = nbits // 8
    cen = rng.integers(0, 256, (3, rb), dtype=np.uint8)
    cen[2] = 0
    bits = np.unpackbits(cen, axis=1)
    n = 400
    lab = rng.integers(0, 3, n)
    lab[:300] = 0
    yb = bits[lab] ^ (rng.random((n, nbits)) < 0.1).astype(np.uint8)
    y = np.packbits(yb, axis=1)
    y[5] = y[6] = y[300]
    y[7] = 0
    y[8] = cen[1]
    cb = np.unpackbits(cen, axis=1)
    own = np.argmin(np.stack([(np.unpackbits(y, axis=1) != cb[l]).sum(1) for l in range(3)], 1), axis=1)
    lists = [np.nonzero(own == l)[0][::-1].copy() for l in range(3)]   # not in id order: ties must be resolved by id
    mid = cen[0].copy()
    mid[: rb // 2] = cen[1][: rb // 2]
    q = np.concatenate([y[[0, 5, 300, 399]], np.zeros((1, rb), np.uint8), mid[None, :], cen[[0, 1]]])
    return y, cen, lists, q


@pytest.fixture(params=[(B.HAMMING, 64), (B.JACCARD, 64), (B.HAMMING, 200), (B.JACCARD, 1032)])
def stored(request, tmp_path):
    metric, nbits = request.param
    rng = np.random.default_rng(nbits + metric)
    y, cen, lists, q = tiny(nbits, rng)
    path = tmp_path / "tiny.b2ix"
    path.write_bytes(encode(metric, nbits, cen, lists, y))
    return B.read_binary_index(path), metric, y, cen, lists, q


def test_reader_decodes_the_layout(stored):
    s, metric, y, cen, lists, q = stored
    assert (s.kb_w, s.row_pad) == B.geometry(y.shape[1])[:2]
    assert np.array_equal(s.centroids[:, :y.shape[1]], cen)
    for l, ids in enumerate(lists):
        assert np.array_equal(s.ids[l], ids) and np.array_equal(s.pool[l][:, :y.shape[1]], y[ids])
    assert s.list_len.max() > B.PAGE, "one list should span two pages"
    B.check_binary_build(s, y)


def test_reader_refuses_trailing_bytes(stored, tmp_path):
    s, metric, y, cen, lists, q = stored
    path = tmp_path / "long.b2ix"
    path.write_bytes(encode(metric, s.d, cen, lists, y) + b"\0")
    with pytest.raises(AssertionError, match="left after the last page"):
        B.read_binary_index(path)


def test_build_check_rejects_a_row_in_the_wrong_list(stored):
    s, metric, y, cen, lists, q = stored
    bad = s.copy()
    bad.ids[0][[0, -1]] = bad.ids[0][[-1, 0]]
    with pytest.raises(AssertionError):
        B.check_binary_build(bad, y)
    bad = s.copy()
    l, r = bad.locate(8)   # a row equal to centre 1, moved to list 2
    bad.ids[2] = np.append(bad.ids[2], bad.ids[l][r])
    bad.pool[2] = np.concatenate([bad.pool[2], bad.pool[l][r:r + 1]])
    bad.popc[2] = np.append(bad.popc[2], bad.popc[l][r])
    bad.ids[l], bad.pool[l], bad.popc[l] = (np.delete(a, r, axis=0) for a in (bad.ids[l], bad.pool[l], bad.popc[l]))
    with pytest.raises(AssertionError, match="nearest list"):
        B.check_binary_build(bad, y)


@pytest.mark.parametrize("k", [1, 5, 50, 500])
@pytest.mark.parametrize("nprobe", [1, 2, 3, 9])
def test_reference_equals_a_plain_loop(stored, k, nprobe):
    s, metric, y, cen, lists, q = stored
    alive = np.packbits(np.random.default_rng(k).random(len(y)) < 0.6, bitorder="little")
    for a in (None, alive):
        want = loop_search(metric, y, cen, lists, q, k, nprobe, a)
        ref = B.reference_search(s, q, k, nprobe, a)
        assert not B.compare(ref, *want), B.compare(ref, *want)
        assert (ref.ids[:, :min(k, 5)] >= 0).all()


def test_comparator_rejects_each_fault(stored):
    s, metric, y, cen, lists, q = stored
    k, nprobe = 10, 2
    ref = B.reference_search(s, q, k, nprobe)
    dis, ids = ref.dis.copy(), ref.ids.copy()
    assert not B.compare(ref, dis, ids)
    # a wrong tie winner: query 1 is a copy of rows 5, 6 and 300, which tie at distance 0
    assert ids[1, :3].tolist() == [5, 6, 300] and (dis[1, :3] == 0).all()
    assert B.compare(B.reference_search(s, q, k, nprobe, ties="larger"), dis, ids), "final ties toward the larger id"
    bad = ids.copy()
    bad[1, [0, 1]] = bad[1, [1, 0]]
    assert B.compare(ref, dis, bad)
    # a missing row: the first winner of query 0 removed from the stored index
    miss = s.copy()
    l, r = miss.locate(ids[0, 0])
    miss.ids[l], miss.pool[l], miss.popc[l] = (np.delete(a, r, axis=0) for a in (miss.ids[l], miss.pool[l], miss.popc[l]))
    assert B.compare(B.reference_search(miss, q, k, nprobe), dis, ids)
    # one flipped bit of a winning row
    flip = s.copy()
    l, r = flip.locate(ids[0, 0])
    flip.pool[l][r, 0] ^= 1
    assert B.compare(B.reference_search(flip, q, k, nprobe), dis, ids)
    # a probe of nprobe - 1 lists: at k = 100 the queries on centre 1 need rows of their second list
    wide = B.reference_search(s, q, 100, nprobe)
    assert (wide.ids[-1] >= 0).sum() > s.list_len[B.coarse_probe(s, q, 1)[-1, 0]]
    assert B.compare(B.reference_search(s, q, 100, nprobe - 1), wide.dis, wide.ids)
    # a tail that is not filled: k above the kept rows of one list
    few = B.reference_search(s, q, 500, 1)
    assert (few.ids == -1).any()
    d2, i2 = few.dis.copy(), few.ids.copy()
    i2[i2 == -1] = 0
    assert B.compare(few, d2, i2)
    d2, i2 = few.dis.copy(), few.ids.copy()
    d2[i2 == -1] = 0
    assert B.compare(few, d2, i2)


def test_coarse_ties_go_to_the_smaller_list(stored):
    s, metric, y, cen, lists, q = stored
    two = s.copy()
    two.centroids[1] = two.centroids[0]    # lists 0 and 1 now tie for every query
    p = B.coarse_probe(two, q, 1)
    assert (p[:, 0] != 1).all()
    assert B.coarse_ties(two, q, 1)[p[:, 0] == 0].all()
    assert (B.coarse_probe(two, q, 1, ties="larger")[p[:, 0] == 0, 0] == 1).all()
