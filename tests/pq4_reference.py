"""Float64 reference of PQ indexes with 4-bit codes (bit_size = 4), on top of tests/ivf_reference.py.

`read_index4` decodes a B2IX v3 file: the v2 layout (tests/ivf_reference.py) with reserved0 = 4, a [m][16][dsub] fp32
codebook and code rows of round_up(ceil(M / 2), 16) bytes, code j in byte j / 2 (even j in the low nibble).  The scan
tabulates T[q][j][e] = <q_j, cb_j[e]> in fp32 from the fp32 (prepared) query and the fp32 codebook, so the key of
(query, row) is, in float64,
  L2:     ||q - c_l||^2 + 2 <c_l, r^> + ||r^||^2 - 2 <q, r^>
  IP:     -(<q, c_l> + <q, r^>)          cosine: 1 - (<q, c_l> + <q, r^>)
with r^ the fp32 codewords of the row's unpacked codes and c_l its list centroid.  The coarse probe, the query preparation
and the comparator are those of tests/ivf_reference.py.  numpy only: nothing here imports the library."""
import numpy as np

from tests import ivf_reference as R

VERSION, CODE_BITS, CODEWORDS = 3, 4, 16


def code_bytes(m):
    return -(-((m + 1) // 2) // 16) * 16


def unpack(packed, m):
    """[rows][code_bytes] u8 -> [rows][m] codes: code j is the low nibble of byte j / 2 for even j, the high one for odd j."""
    packed = np.asarray(packed, np.uint8)
    lo, hi = packed & 15, packed >> 4
    out = np.empty((len(packed), 2 * packed.shape[1]), np.uint8)
    out[:, 0::2], out[:, 1::2] = lo, hi
    return out[:, :m]


def pack(codes, nbytes):
    """[rows][m] codes < 16 -> [rows][nbytes] u8 (the inverse of unpack; padding nibbles and bytes 0)."""
    codes = np.asarray(codes, np.uint8)
    rows, m = codes.shape
    c = np.zeros((rows, 2 * nbytes), np.uint8)
    c[:, :m] = codes
    return (c[:, 0::2] | (c[:, 1::2] << 4)).astype(np.uint8)


def read_index4(path):
    """The stored 4-bit PQ index: a tests.ivf_reference.StoredIndex with codebook [m][16][dsub] fp32 and codes[l] the packed
    rows [len][code_bytes] u8 as stored (see unpack)."""
    raw = open(path, "rb").read()
    h = np.frombuffer(raw, R.HEADER, count=1)[0]
    assert h["magic"] == b"B2IX" and h["version"] == VERSION and h["reserved0"] == CODE_BITS, "not a B2IX v3 (4-bit PQ) file"
    s = R.StoredIndex()
    for f in R.HEADER.names:
        setattr(s, f, h[f].item() if f != "magic" else h[f])
    assert s.payload == R.PAYLOAD_PQ and s.use_ivf, "inverted-file PQ index expected"
    d, nl, n = s.d, s.nlist, s.n
    off = R.HEADER.itemsize

    def take(dtype, count):
        nonlocal off
        a = np.frombuffer(raw, dtype, count=count, offset=off)
        off += a.nbytes
        return a

    s.rows = take("<f4", n * d).reshape(n, d) if s.has_raw else None
    s.centroids = take("<f4", nl * d).reshape(nl, d)
    s.list_len = take("<u4", nl).astype(np.int64)
    s.codebook = take("<f4", s.m * CODEWORDS * s.dsub).reshape(s.m, CODEWORDS, s.dsub)
    s.sq = None
    cb = s.code_bytes
    for l in range(nl):
        np_ = -(-int(s.list_len[l]) // R.PAGE)
        pay, ids, bias = [], [], []
        for _ in range(np_):
            pay.append(take("u1", R.PAGE * cb).reshape(R.PAGE, cb))
            ids.append(take("<u4", R.PAGE))
            if s.metric == R.L2:
                bias.append(take("<f4", R.PAGE))
        ln = int(s.list_len[l])
        s.ids.append((np.concatenate(ids)[:ln] if ids else np.zeros(0)).astype(np.uint32))
        s.bias.append((np.concatenate(bias)[:ln] if bias else np.zeros(0)).astype(np.float32) if s.metric == R.L2 else None)
        s.codes.append((np.concatenate(pay)[:ln] if pay else np.zeros((0, cb))).astype(np.uint8))
    assert off == len(raw), f"{len(raw) - off} bytes left after the last page"
    return s


def decode(s, packed):
    """Packed code rows -> the fp32 codewords the table is built from, [rows][d] fp32."""
    codes = unpack(packed, s.m).astype(np.int64)
    return s.codebook[np.arange(s.m)[None, :], codes].reshape(len(packed), s.d)


def table_products(s, Q, packed, table_round):
    """sum_j T[q][j][code_j] with the table T[q][j][e] = <q_j, cb_j[e]> (fp32) passed through table_round (a perturbation for
    negative controls, e.g. a bf16-rounded table), [nq][rows] float64."""
    cb = s.codebook.astype(np.float64)
    codes = unpack(packed, s.m).astype(np.int64)
    Qs = np.asarray(Q, np.float64).reshape(len(Q), s.m, s.dsub)
    t = np.zeros((len(Q), len(packed)))
    for j in range(s.m):
        T = np.asarray(table_round((Qs[:, j, :] @ cb[j].T).astype(np.float32)), np.float64)   # [nq][16]
        t += T[:, codes[:, j]]
    return t


def row_keys(s, Q, table_round=None):
    """First-stage keys of every (prepared query, stored row of s.flat()): (key [nq][rows] smaller is better, distance as
    returned, tol), tol = TOL_REL x the sum of the absolute values of the key's terms, as in tests/ivf_reference.py."""
    _, lst, pay = s.flat()
    Q64 = np.asarray(Q, np.float64)
    Rv = decode(s, pay).astype(np.float64)
    C = s.centroids.astype(np.float64)
    Cr = C[lst]
    t, at = Q64 @ Rv.T, np.abs(Q64) @ np.abs(Rv).T
    if table_round is not None:
        t = table_products(s, Q, pay, table_round)
    if s.metric == R.L2:
        pc = ((Q64[:, None, :] - C[None, :, :]) ** 2).sum(2)[:, lst]     # ||q - c_l||^2
        cr = (Cr * Rv).sum(1)[None, :]
        acr = np.abs(Cr * Rv).sum(1)[None, :]
        rr = (Rv * Rv).sum(1)[None, :]
        key = pc + 2 * cr + rr - 2 * t
        return key, np.maximum(key, 0.0), R.TOL_REL * (pc + 2 * acr + rr + 2 * at)
    qc, aqc = (Q64 @ C.T)[:, lst], (np.abs(Q64) @ np.abs(C).T)[:, lst]
    sc = qc + t
    if s.metric == R.IP:
        return -sc, sc, R.TOL_REL * (aqc + at)
    return 1 - sc, 1 - sc, R.TOL_REL * (1 + aqc + at)


def reference_search(s, queries, k, nprobe, alive=None, table_round=None):
    """tests/ivf_reference.reference_search for a 4-bit PQ index.  alive: bool [n] or None; table_round: see
    table_products.  The result is checked with ivf_reference.compare."""
    Q = R.prepare_queries(queries, s.metric)
    ids, lst, _ = s.flat()
    key, dis, tol = row_keys(s, Q, table_round)
    probed, allowed, flagged = R.coarse_probe(s, Q, nprobe)
    r = R.Reference()
    r.metric, r.k, r.nq = s.metric, k, len(Q)
    r.ids_all, r.lst_all, r.key, r.dis, r.tol = ids, lst, key, dis, tol
    r.allowed, r.flagged = allowed, flagged
    r.pos_of = {int(i): p for p, i in enumerate(ids.tolist())}
    r.ids = np.full((r.nq, k), -1, np.int64)
    r.out_dis = np.full((r.nq, k), -R.FLT_MAX if s.metric == R.IP else R.FLT_MAX)
    r.cand = []
    alive_row = np.ones(len(ids), bool) if alive is None else np.asarray(alive, bool)[ids]
    for q in range(r.nq):
        cand = np.nonzero(np.isin(lst, probed[q]) & alive_row)[0]
        cand = cand[np.lexsort((ids[cand], key[q, cand]))]
        r.cand.append(cand)
        top = cand[:k]
        r.ids[q, :len(top)] = ids[top]
        r.out_dis[q, :len(top)] = dis[q, top]
    r.alive_row = alive_row
    return r


def check_build(s, ix, y):
    """Build invariants of a stored 4-bit PQ index s (read_index4) of ix built from the rows y: ivf_reference.check_lists, a
    finite codebook, zero padding nibbles and bytes, every code the nearest fp32 codeword of the row's residual and row_bias
    from the fp32 codewords."""
    ids, lst, pay, x = R.check_lists(s, ix, y)
    assert np.isfinite(s.codebook).all(), "a codeword is not finite"
    n = len(ids)
    codes = unpack(pay, s.m)
    assert (pack(codes, s.code_bytes) == pay).all(), "padding nibbles and bytes must be 0"
    X, C = x[ids].astype(np.float64), s.centroids.astype(np.float64)
    res = X - C[lst]
    cb = s.codebook.astype(np.float64)
    for j in range(s.m):
        r = res[:, j * s.dsub:(j + 1) * s.dsub]
        dd = ((r[:, None, :] - cb[j][None, :, :]) ** 2).sum(2)
        got = dd[np.arange(n), codes[:, j]]
        assert (got <= dd.min(1) + 1e-5 * ((r * r).sum(1) + (cb[j] ** 2).sum(1).max()) + 1e-12).all(), f"code {j} is not the nearest fp32 codeword"
    if s.metric == R.L2:
        Rf = decode(s, pay).astype(np.float64)
        bias = (Rf * (Rf + 2 * C[lst])).sum(1)
        S = (np.abs(Rf) * np.abs(Rf + 2 * C[lst])).sum(1)
        b = np.concatenate(s.bias).astype(np.float64)
        assert (np.abs(b - bias) <= R.TOL_REL * S + 1e-30).all(), "row_bias differs from its fp32 formula"
    else:
        assert all(a is None for a in s.bias)
