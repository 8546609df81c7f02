"""Float64 reference of a stored float inverted-file index and of its first-stage search.

`read_index` decodes a B2IX v2 file written by `VectorIndex.save` (layout: `index_save_io` in csrc/ivf.cu).
`check_build` asserts the build invariants of a stored index.
`reference_search` ranks every row of the probed lists by the key the list scan defines for its payload, computed in
float64 from the stored payload, with the device's roundings reproduced where they change a value (bf16 queries, bf16
codebooks, the SQ8 query scaling, the cosine normalisation).  `compare` checks a library answer against it.
numpy only: nothing here imports the library, so the reference cannot share a bug with it.
"""
import numpy as np

from tests.util import to_bf16_values

L2, IP, COSINE = 0, 1, 2
PAYLOAD_BF16, PAYLOAD_PQ, PAYLOAD_SQ8 = 0, 1, 2
PAGE = 256
FLT_MAX = float(np.finfo(np.float32).max)
# tolerance of a key: TOL_REL x the sum of the absolute values of its terms (fp32 accumulation over d); bf16 / SQ8 rows
# wider than TC_WIDE add the tensor-core truncation bound (tc_weights).  PQ decodes at most 220 dims, so never does.
TOL_REL = 3e-5


U = 2.0 ** -24
TC_WIDE = 768     # widest bf16 row (d_pad64) of the narrower checks, held to TOL_REL alone


def tc_weights(d):
    """Per-column weights w_i of the tensor-core truncation bound (tests/flat_reference.py): a wgmma K-step adds K = 16
    products to the fp32 accumulator after aligning them to the largest exponent and truncating, so each of the K + 1 addends
    can lose 2 u of the step's largest magnitude, at most the sum of |t_i| over the columns added so far.  Summed over the
    steps, the product part of a key is off by at most 2 (K + 1) u sum_i w_i |t_i|, with w_i = d_pad64 / 16 - i // 16 the
    K-steps from the one that adds column i to the last.  The scan adds k-blocks in column order."""
    d_pad64 = -(-d // 64) * 64
    return (d_pad64 // 16 - np.arange(d) // 16).astype(np.float64)


HEADER = np.dtype([("magic", "S4"), ("version", "<u4"), ("type", "<i4"), ("metric", "<i4"), ("d", "<i4"), ("nlist", "<i4"),
                   ("m", "<i4"), ("dsub", "<i4"), ("default_nprobe", "<i4"), ("refine_factor", "<i4"), ("payload", "<i4"),
                   ("has_raw", "<i4"), ("use_ivf", "<i4"), ("code_bytes", "<i4"), ("n", "<i8"), ("pages_used", "<u4"),
                   ("reserved0", "<u4")])
assert HEADER.itemsize == 72


def bf16_bits_to_f32(u16):
    return (np.asarray(u16, np.uint16).astype(np.uint32) << 16).view(np.float32)


class StoredIndex:
    """The decoded file.  Per list l: ids[l] (u32 row ids), bias[l] (fp32 row_bias, L2 only, else None) and the payload:
    vals[l] fp32 [len][d_pad64] (bf16 values, k-block-major pages unpacked) or codes[l] u8 [len][code_bytes]."""

    def __init__(self):
        self.ids, self.bias, self.vals, self.codes = [], [], [], []

    @property
    def d_pad64(self):
        return -(-self.d // 64) * 64

    def copy(self):
        c = StoredIndex()
        c.__dict__.update(self.__dict__)
        c.ids = [a.copy() for a in self.ids]
        c.bias = [None if a is None else a.copy() for a in self.bias]
        c.vals = [a.copy() for a in self.vals]
        c.codes = [a.copy() for a in self.codes]
        return c

    def truncate_list(self, l, rows):
        """Keep the first `rows` rows of list l (a perturbation for negative controls)."""
        self.ids[l] = self.ids[l][:rows]
        if self.bias[l] is not None:
            self.bias[l] = self.bias[l][:rows]
        if self.payload == PAYLOAD_BF16:
            self.vals[l] = self.vals[l][:rows]
        else:
            self.codes[l] = self.codes[l][:rows]
        self.list_len[l] = rows

    def flat(self):
        """All stored rows, list after list: (ids int64, list of each row, payload rows)."""
        lens = [len(a) for a in self.ids]
        ids = np.concatenate(self.ids).astype(np.int64) if lens else np.zeros(0, np.int64)
        lst = np.repeat(np.arange(self.nlist), lens)
        pay = np.concatenate(self.vals if self.payload == PAYLOAD_BF16 else self.codes)
        return ids, lst, pay


def read_index(path):
    raw = open(path, "rb").read()
    h = np.frombuffer(raw, HEADER, count=1)[0]
    assert h["magic"] == b"B2IX" and h["version"] == 2, "not a B2IX v2 file"
    s = StoredIndex()
    for f in HEADER.names:
        setattr(s, f, h[f].item() if f != "magic" else h[f])
    assert s.payload in (PAYLOAD_BF16, PAYLOAD_PQ, PAYLOAD_SQ8) and s.use_ivf, "float inverted-file index expected"
    d, nl, n = s.d, s.nlist, s.n
    off = HEADER.itemsize

    def take(dtype, count):
        nonlocal off
        a = np.frombuffer(raw, dtype, count=count, offset=off)
        off += a.nbytes
        return a

    s.rows = take("<f4", n * d).reshape(n, d) if s.has_raw else None
    s.centroids = take("<f4", nl * d).reshape(nl, d)
    s.list_len = take("<u4", nl).astype(np.int64)
    s.codebook = take("<f4", s.m * 256 * s.dsub).reshape(s.m, 256, s.dsub) if s.payload == PAYLOAD_PQ else None
    s.sq = take("<f4", 4 * d).reshape(4, d) if s.payload == PAYLOAD_SQ8 else None   # lo, step, 1 / step, mid
    row_bytes = s.d_pad64 * 2 if s.payload == PAYLOAD_BF16 else s.code_bytes
    for l in range(nl):
        np_ = -(-int(s.list_len[l]) // PAGE)
        pay, ids, bias = [], [], []
        for _ in range(np_):
            if s.payload == PAYLOAD_BF16:
                u = take("<u2", PAGE * s.d_pad64).reshape(s.d_pad64 // 64, PAGE, 64)
                pay.append(bf16_bits_to_f32(u.transpose(1, 0, 2).reshape(PAGE, s.d_pad64)))
            else:
                pay.append(take("u1", PAGE * row_bytes).reshape(PAGE, row_bytes))
            ids.append(take("<u4", PAGE))
            if s.metric == L2:
                bias.append(take("<f4", PAGE))
        ln = int(s.list_len[l])
        cat = (lambda a, w: np.concatenate(a)[:ln] if a else np.zeros((0,) + w, np.float32))
        s.ids.append(cat(ids, ()).astype(np.uint32))
        s.bias.append(cat(bias, ()).astype(np.float32) if s.metric == L2 else None)
        if s.payload == PAYLOAD_BF16:
            s.vals.append(cat(pay, (s.d_pad64,)).astype(np.float32))
        else:
            s.codes.append(cat(pay, (row_bytes,)).astype(np.uint8))
    assert off == len(raw), f"{len(raw) - off} bytes left after the last page"
    return s


def normalize_rows_f32(x):
    """The device's cosine normalisation (normalize_rows_f32_kernel): 32 lane sums of fmaf(x, x, s) over strided columns, an
    xor-butterfly of fp32 adds, x / sqrtf(s); rows with s < FLT_EPSILON stay as they are."""
    x = np.ascontiguousarray(x, np.float32)
    nq, d = x.shape
    w = -(-d // 32) * 32
    p = np.zeros((nq, w), np.float32)
    p[:, :d] = x
    p = p.reshape(nq, w // 32, 32)
    s = np.zeros((nq, 32), np.float32)
    for t in range(w // 32):
        v = p[:, t, :].astype(np.float64)
        s = (s.astype(np.float64) + v * v).astype(np.float32)   # fmaf: exact product, one rounding
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        s = s + s[:, lane ^ o]
    s = s[:, 0]
    nrm = np.sqrt(s).astype(np.float32)
    ok = s >= np.finfo(np.float32).eps
    out = x.copy()
    out[ok] = x[ok] / nrm[ok, None]
    return out


def prepare_queries(q, metric):
    q = np.ascontiguousarray(q, np.float32)
    return normalize_rows_f32(q) if metric == COSINE else q.copy()


def pq_decode(s, codes):
    """codes [rows][code_bytes] -> the bf16 codebook values the scan multiplies, [rows][d] fp32."""
    cbh = to_bf16_values(s.codebook)
    j = np.arange(s.m)
    return cbh[j[None, :], codes[:, :s.m].astype(np.int64)].reshape(len(codes), s.d)


def row_keys(s, Q, rows=None):
    """First-stage keys of every (prepared query, stored row): (key [nq][rows] smaller is better, distance as returned,
    tol).  Rows are those of s.flat() (or the given subset of their positions)."""
    ids, lst, pay = s.flat()
    if rows is not None:
        lst, pay = lst[rows], pay[rows]
    Q = np.asarray(Q, np.float32)
    Q64 = Q.astype(np.float64)
    d = s.d
    # rows wider than the narrower checks: + the truncation bound of the tensor-core product (tc_weights), over its terms
    trunc = (lambda a, b: 2 * 17 * U * ((np.abs(a) * tc_weights(d)) @ np.abs(b).T)) if s.d_pad64 > TC_WIDE else (lambda a, b: 0.0)
    if s.payload == PAYLOAD_BF16:
        qt = to_bf16_values(Q).astype(np.float64)
        Y = pay[:, :d].astype(np.float64)
        ip, aip, w = qt @ Y.T, np.abs(qt) @ np.abs(Y).T, trunc(qt, Y)
        if s.metric == L2:
            qq, yy = (qt * qt).sum(1)[:, None], (Y * Y).sum(1)[None, :]
            key = qq + yy - 2 * ip
            return key, np.maximum(key, 0.0), TOL_REL * (qq + yy + 2 * aip) + 2 * w
        if s.metric == IP:
            return -ip, ip, TOL_REL * aip + w
        return 1 - ip, 1 - ip, TOL_REL * (1 + aip) + w
    if s.payload == PAYLOAD_SQ8:
        lo, step, _, mid = (s.sq[i].astype(np.float64) for i in range(4))
        cm = pay[:, :d].astype(np.float64) - 128.0
        qs = to_bf16_values(Q * s.sq[1][None, :]).astype(np.float64)     # fp32 product, bf16 RNE (pair_fill_kernel)
        t, at, w = qs @ cm.T, np.abs(qs) @ np.abs(cm).T, trunc(qs, cm)
        qm, aqm = (Q64 @ mid)[:, None], (np.abs(Q64) @ np.abs(mid))[:, None]
        if s.metric == L2:
            v = lo[None, :] + pay[:, :d].astype(np.float64) * step[None, :]
            vv = (v * v).sum(1)[None, :]
            qq = (Q64 * Q64).sum(1)[:, None]
            key = qq - 2 * qm + vv - 2 * t
            return key, np.maximum(key, 0.0), TOL_REL * (qq + 2 * aqm + vv + 2 * at) + 2 * w
        sc = qm + t
        if s.metric == IP:
            return -sc, sc, TOL_REL * (aqm + at) + w
        return 1 - sc, 1 - sc, TOL_REL * (1 + aqm + at) + w
    # PQ on the residual: r^ = bf16 codebook entries, c = the row's list centroid
    R = pq_decode(s, pay).astype(np.float64)
    C = s.centroids.astype(np.float64)
    Cr = C[lst]
    qb = to_bf16_values(Q).astype(np.float64)
    t, at = qb @ R.T, np.abs(qb) @ np.abs(R).T
    if s.metric == L2:
        pc = ((Q64[:, None, :] - C[None, :, :]) ** 2).sum(2)[:, lst]     # ||q - c_l||^2
        cr = (Cr * R).sum(1)[None, :]
        acr = np.abs(Cr * R).sum(1)[None, :]
        rr = (R * R).sum(1)[None, :]
        key = pc + 2 * cr + rr - 2 * t
        return key, np.maximum(key, 0.0), TOL_REL * (pc + 2 * acr + rr + 2 * at)
    qc, aqc = (Q64 @ C.T)[:, lst], (np.abs(Q64) @ np.abs(C).T)[:, lst]
    sc = qc + t
    if s.metric == IP:
        return -sc, sc, TOL_REL * (aqc + at)
    return 1 - sc, 1 - sc, TOL_REL * (1 + aqc + at)


def coarse_probe(s, Q, nprobe):
    """nprobe nearest centroids by L2 (every metric), fp64, ties to the smaller list id.  Returns (probed [nq][nprobe],
    allowed: per query the set of lists a correct probe may use, flagged [nq]: the nprobe-th and (nprobe+1)-th centroid
    distances are within tolerance, so the probe set itself is ambiguous)."""
    Q64 = np.asarray(Q, np.float64)
    C = s.centroids.astype(np.float64)
    qq, cc = (Q64 * Q64).sum(1)[:, None], (C * C).sum(1)[None, :]
    dist = qq + cc - 2 * Q64 @ C.T        # expanded: no nq x nlist x d temporary; fp64 rounding << ptol
    ptol = 1e-5 * (qq + cc + 2 * np.abs(Q64) @ np.abs(C).T)
    order = np.argsort(dist, axis=1, kind="stable")
    npr = max(1, min(nprobe, s.nlist))
    probed = order[:, :npr]
    flagged = np.zeros(len(Q64), bool)
    allowed = []
    for q in range(len(Q64)):
        al = set(probed[q].tolist())
        if npr < s.nlist:
            b_in, b_out = order[q, npr - 1], order[q, npr]
            if dist[q, b_out] - dist[q, b_in] <= ptol[q, b_in] + ptol[q, b_out]:
                flagged[q] = True
                edge = dist[q, b_in]
                al |= set(np.nonzero(np.abs(dist[q] - edge) <= 2 * ptol[q])[0].tolist())
        allowed.append(al)
    return probed, allowed, flagged


class Reference:
    """Reference answer of one batch, with what the comparator needs per query."""


def reference_search(s, queries, k, nprobe, alive=None):
    """alive: bool [n] (True = may be returned) or None."""
    Q = prepare_queries(queries, s.metric)
    ids, lst, _ = s.flat()
    key, dis, tol = row_keys(s, Q)
    probed, allowed, flagged = coarse_probe(s, Q, nprobe)
    r = Reference()
    r.metric, r.k, r.nq = s.metric, k, len(Q)
    r.ids_all, r.lst_all, r.key, r.dis, r.tol = ids, lst, key, dis, tol
    r.allowed, r.flagged = allowed, flagged
    r.pos_of = {int(i): p for p, i in enumerate(ids.tolist())}
    r.ids = np.full((r.nq, k), -1, np.int64)
    r.out_dis = np.full((r.nq, k), -FLT_MAX if s.metric == IP else FLT_MAX)
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


def compare(r, dis_g, ids_g):
    """Problems of a library answer against the reference (empty list: it passes).  Per query: (1) every returned id lies in
    a list the reference probes (or a tied list of a flagged query) and is alive; (2) its distance is the reference key of
    that id within tol; (3) the distance at rank j is within tol of the reference's rank-j distance; (4) every row whose key
    is below the k-th key minus tol is present; (5) no duplicate ids; (6) the filled and unfilled slots are the reference's.
    (3), (4) and (6) are skipped for flagged queries, whose probe set is ambiguous."""
    bad = []
    empty = -FLT_MAX if r.metric == IP else FLT_MAX
    for q in range(r.nq):
        ig, dg = ids_g[q], dis_g[q].astype(np.float64)
        filled = ig >= 0
        nf = int(filled.sum())
        if not filled[:nf].all():
            bad.append(f"q{q}: unfilled slot before a filled one")
        if (dg[~filled] != empty).any():
            bad.append(f"q{q}: unfilled slot with distance other than {empty}")
        got = ig[filled].tolist()
        if len(set(got)) != len(got):
            bad.append(f"q{q}: duplicate ids")                                               # (5)
        for j, i in enumerate(got):
            p = r.pos_of.get(int(i))
            if p is None or int(r.lst_all[p]) not in r.allowed[q] or not r.alive_row[p]:
                bad.append(f"q{q} rank {j}: id {i} is not in a probed list / not alive")   # (1)
                continue
            if abs(dg[j] - r.dis[q, p]) > r.tol[q, p]:                                      # (2)
                bad.append(f"q{q} rank {j}: id {i} distance {dg[j]!r} vs reference {r.dis[q, p]!r} (tol {r.tol[q, p]:.3g})")
        if r.flagged[q]:
            continue
        cand = r.cand[q]
        nref = min(r.k, len(cand))
        if nf != nref:
            bad.append(f"q{q}: {nf} filled slots, reference {nref}")                        # (6)
            continue
        for j in range(nf):                                                                   # (3)
            p_ref = cand[j]
            p_g = r.pos_of.get(int(ig[j]))
            t = r.tol[q, p_ref] + (r.tol[q, p_g] if p_g is not None else 0.0)
            if abs(dg[j] - r.dis[q, p_ref]) > t:
                bad.append(f"q{q} rank {j}: distance {dg[j]!r} vs reference rank-{j} {r.dis[q, p_ref]!r}")
        if nref:
            kth = r.key[q, cand[nref - 1]]
            must = cand[r.key[q, cand] < kth - r.tol[q, cand]]                             # (4)
            missing = set(r.ids_all[must].tolist()) - set(got)
            if missing:
                bad.append(f"q{q}: rows {sorted(missing)[:5]} below the k-th key are missing")
    return bad


def usable(y):
    """Rows the library may index: the fp32 sum of the squares of the coordinates is finite (no NaN or infinite coordinate,
    no square that overflows), include/b200_search.h "Unusable rows"."""
    y = np.asarray(y, np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        return np.isfinite(np.square(y).sum(1, dtype=np.float32))


def check_lists(s, ix, y):
    """List invariants of a stored float inverted-file index s of ix built from the rows y, for every payload: every usable
    row in its nearest list exactly once and every unusable one in none, the list sizes, the stored fp32 rows (NaN bits
    included) and finite centroids.  Returns (ids, lists, payload rows) of s.flat() and the stored rows x."""
    y = np.asarray(y, np.float32)
    ids, lst, pay = s.flat()
    ok = usable(y)
    assert np.isfinite(s.centroids).all(), "a centroid is not finite"
    assert np.array_equal(np.sort(ids), np.nonzero(ok)[0]), "the lists do not hold every usable row, and no other, exactly once"
    assert np.array_equal(s.list_len, ix.list_sizes().astype(np.int64))
    assert int(s.list_len.sum()) == int(ok.sum())
    assert s.has_raw
    x = s.rows.astype(np.float32)
    if s.metric == COSINE:   # rows are stored unit length (those below FLT_EPSILON as given); the payload is encoded from them
        np.testing.assert_allclose(x[ok], normalize_rows_f32(y[ok]), rtol=0, atol=1e-6)
    else:
        assert x.tobytes() == y.tobytes(), "the stored fp32 rows differ from the input"
    X = x[ids].astype(np.float64)
    C = s.centroids.astype(np.float64)
    # ||x - c||^2 expanded (no n x nlist x d temporary at wide d): fp64 rounding stays far below the 1e-5 tolerance
    xx, cc = (X * X).sum(1)[:, None], (C * C).sum(1)[None, :]
    dist = xx + cc - 2 * X @ C.T
    tol = 1e-5 * (xx + cc + 2 * np.abs(X) @ np.abs(C).T)
    at = np.arange(len(ids))
    own = dist[at, lst]
    assert (own <= dist.min(1) + tol[at, lst]).all(), "a row is not in its nearest list"
    return ids, lst, pay, x


def check_build(s, ix, y):
    """Build invariants of a stored float inverted-file index s (read_index) of ix built from the rows y: check_lists, then
    the payload (bf16 RNE, SQ codes and padding, nearest bf16-decoded PQ codewords) and row_bias."""
    d = s.d
    ids, lst, pay, x = check_lists(s, ix, y)
    X = x[ids].astype(np.float64)
    C = s.centroids.astype(np.float64)
    n = len(ids)
    if s.payload == PAYLOAD_BF16:
        assert np.array_equal(pay[:, :d], to_bf16_values(x[ids])), "bf16 payload is not RNE of the row"
        assert (pay[:, d:] == 0).all()
        Y = pay[:, :d].astype(np.float64)
        bias, S = (Y * Y).sum(1), (Y * Y).sum(1)
    elif s.payload == PAYLOAD_SQ8:
        lo, step, inv = s.sq[0], s.sq[1], s.sq[2]
        want = np.clip(np.rint((x[ids] - lo) * inv), 0, 255)                     # the device's fp32 arithmetic
        got = pay[:, :d].astype(np.float64)
        t = (X - lo.astype(np.float64)) * inv.astype(np.float64)
        near_half = np.abs(t - np.floor(t) - 0.5) < 1e-5 * np.maximum(1.0, np.abs(t))
        assert ((got == want) | ((np.abs(got - want) == 1) & near_half)).all(), "SQ codes differ from rint((x - lo) / step)"
        assert (pay[:, d:] == 128).all(), "SQ padding bytes must decode to 0"
        v = lo.astype(np.float64) + got * step.astype(np.float64)
        bias, S = (v * v).sum(1), (v * v).sum(1)
    else:
        res = X - C[lst]
        cb = s.codebook.astype(np.float64)
        for j in range(s.m):
            r = res[:, j * s.dsub:(j + 1) * s.dsub]
            dd = ((r[:, None, :] - cb[j][None, :, :]) ** 2).sum(2)
            got = dd[np.arange(n), pay[:, j]]
            assert (got <= dd.min(1) + 1e-5 * ((r * r).sum(1) + (cb[j] ** 2).sum(1).max()) + 1e-12).all(), f"PQ code {j} is not the nearest codeword"
        assert (pay[:, s.m:] == 0).all(), "PQ padding bytes must be 0"
        Rh = pq_decode(s, pay).astype(np.float64)
        bias = (Rh * (Rh + 2 * C[lst])).sum(1)
        S = (np.abs(Rh) * np.abs(Rh + 2 * C[lst])).sum(1)
    if s.metric == L2:
        b = np.concatenate(s.bias).astype(np.float64)
        assert (np.abs(b - bias) <= TOL_REL * S + 1e-30).all(), "row_bias differs from its formula"
    else:
        assert all(a is None for a in s.bias)


def rerank(rows, q, cand, k, metric):
    """Exact second stage: candidates [nq][kc] (-1 = none) of the prepared queries q against the stored fp32 rows -> the top k
    by (fp32 key, id), (dis float32 [nq][k], ids int64 [nq][k]).  The key is the float64 value rounded once to fp32: the
    library's key wherever its fp32 sum is exact (small integers), else within its rounding (see the callers' bounds)."""
    nq = len(q)
    empty = -FLT_MAX if metric == IP else FLT_MAX
    dis = np.full((nq, k), empty, np.float32)
    ids = np.full((nq, k), -1, np.int64)
    for i in range(nq):
        c = cand[i][cand[i] >= 0]
        yy, qq = rows[c].astype(np.float64), np.asarray(q[i], np.float64)
        key = (((yy - qq) ** 2).sum(1) if metric == L2 else -(yy @ qq)).astype(np.float32)
        order = np.lexsort((c, key))[:k]
        ids[i, :len(order)] = c[order]
        dis[i, :len(order)] = key[order] if metric == L2 else (-key[order] if metric == IP else 1 - (-key[order]))
    return dis, ids
