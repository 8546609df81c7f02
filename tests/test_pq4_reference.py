"""The 4-bit PQ reference (tests/pq4_reference.py) on a B2IX v3 file written here with numpy: nibble packing, the v3 reader
and the keys against a brute-force float64 computation that decodes every code by hand.  No GPU needed."""
import numpy as np
import pytest

from tests import ivf_reference as R
from tests import pq4_reference as P


def _write_v3(path, rng, n=700, d=30, m=15, nlist=3, metric=R.L2, has_raw=True):
    dsub = d // m
    cb_bytes = P.code_bytes(m)
    rows = rng.standard_normal((n, d)).astype(np.float32)
    cent = rng.standard_normal((nlist, d)).astype(np.float32)
    book = rng.standard_normal((m, 16, dsub)).astype(np.float32)
    lst = rng.integers(0, nlist, n)
    codes = rng.integers(0, 16, (n, m)).astype(np.uint8)
    lens = np.bincount(lst, minlength=nlist)
    pages = int(sum(-(-int(x) // R.PAGE) for x in lens))
    h = np.zeros(1, R.HEADER)
    h["magic"], h["version"], h["reserved0"] = b"B2IX", 3, 4
    h["type"], h["metric"], h["d"], h["nlist"], h["m"], h["dsub"] = 2, metric, d, nlist, m, dsub
    h["payload"], h["has_raw"], h["use_ivf"], h["code_bytes"], h["n"], h["pages_used"] = R.PAYLOAD_PQ, int(has_raw), 1, cb_bytes, n, pages
    parts = [h.tobytes()]
    if has_raw:
        parts.append(rows.tobytes())
    parts += [cent.tobytes(), lens.astype("<u4").tobytes(), book.tobytes()]
    per_list = []
    for l in range(nlist):
        ids = np.nonzero(lst == l)[0]
        per_list.append(ids)
        for p0 in range(0, len(ids), R.PAGE):
            chunk = ids[p0:p0 + R.PAGE]
            page = np.zeros((R.PAGE, cb_bytes), np.uint8)
            page[:len(chunk)] = P.pack(codes[chunk], cb_bytes)
            pid = np.zeros(R.PAGE, "<u4")
            pid[:len(chunk)] = chunk
            parts += [page.tobytes(), pid.tobytes()]
            if metric == R.L2:
                parts.append(np.zeros(R.PAGE, "<f4").tobytes())
    with open(path, "wb") as f:
        f.write(b"".join(parts))
    return rows, cent, book, lst, codes, per_list


def test_pack_unpack_order():
    codes = np.array([[1, 2, 3], [15, 0, 7]], np.uint8)
    packed = P.pack(codes, 16)
    assert packed.shape == (2, 16)
    assert packed[0, 0] == 0x21 and packed[0, 1] == 0x03 and packed[1, 0] == 0x0F and packed[1, 1] == 0x07
    assert not packed[:, 2:].any()
    assert np.array_equal(P.unpack(packed, 3), codes)
    assert P.code_bytes(1) == 16 and P.code_bytes(32) == 16 and P.code_bytes(33) == 32 and P.code_bytes(96) == 48


@pytest.mark.parametrize("metric", [R.L2, R.IP, R.COSINE])
def test_reader_and_keys_against_brute_force(tmp_path, metric):
    rng = np.random.default_rng(3 + metric)
    path = tmp_path / "v3.b2ix"
    rows, cent, book, lst, codes, per_list = _write_v3(path, rng, metric=metric)
    s = P.read_index4(path)
    assert (s.version, s.reserved0, s.m, s.dsub, s.code_bytes) == (3, 4, 15, 2, 16)
    assert np.array_equal(s.codebook, book) and np.array_equal(s.centroids, cent) and np.array_equal(s.rows, rows)
    for l in range(s.nlist):
        assert np.array_equal(s.ids[l], per_list[l])
        assert np.array_equal(P.unpack(s.codes[l], s.m), codes[per_list[l]])
    q = rng.standard_normal((5, s.d)).astype(np.float32)
    Q = R.prepare_queries(q, metric).astype(np.float64)
    key, dis, tol = P.row_keys(s, R.prepare_queries(q, metric))
    ids, flat_lst, _ = s.flat()
    for qi in range(len(q)):
        for p in range(0, len(ids), 37):
            i, l = int(ids[p]), int(flat_lst[p])
            r = np.concatenate([book[j, codes[i, j]] for j in range(s.m)]).astype(np.float64)
            c = cent[l].astype(np.float64)
            if metric == R.L2:
                want = ((Q[qi] - c - r) ** 2).sum()
            elif metric == R.IP:
                want = -(Q[qi] @ (c + r))
            else:
                want = 1 - Q[qi] @ (c + r)
            assert abs(key[qi, p] - want) <= 1e-9 * (1 + abs(want)), (qi, p, key[qi, p], want)
            assert tol[qi, p] > 0
    # the table form of the keys agrees with the direct form
    t_key, _, _ = P.row_keys(s, R.prepare_queries(q, metric), table_round=lambda t: t)
    assert np.allclose(t_key, key, rtol=0, atol=1e-4)
    # top-k over all lists is the brute-force order (ties to the smaller id)
    r = P.reference_search(s, q, 10, s.nlist)
    for qi in range(len(q)):
        order = np.lexsort((ids, key[qi]))[:10]
        assert np.array_equal(r.ids[qi], ids[order])
        assert not R.compare(r, r.out_dis.astype(np.float32), r.ids)


def test_reader_refuses_a_v2_file(tmp_path):
    rng = np.random.default_rng(9)
    path = tmp_path / "v3.b2ix"
    _write_v3(path, rng)
    raw = bytearray(open(path, "rb").read())
    raw[4] = 2
    open(path, "wb").write(bytes(raw))
    with pytest.raises(AssertionError):
        P.read_index4(path)
