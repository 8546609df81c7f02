"""Float64 reference of what a FLAT corpus stores and of the distances each flat search path returns.

`reference(...)` takes the caller's fp32 rows and queries, reproduces the roundings the device applies before any
arithmetic (bf16 rows, bf16 query operands on the bf16 tensor-core path, the cosine normalisation with its FLT_EPSILON
rule), and computes every (query, row) distance in float64.  `compare` checks a library answer against it.
numpy only: nothing here imports the library, so the reference cannot share a bug with it.

Paths (what `path` names):
  "scan"  flat_scan_kernel, staged or fused: fp32 queries (cosine: normalised), rows as stored (fp32 or bf16), fp32 FMA
          sums; the returned distance is the key (L2), -key (IP) or 1 + key (cosine).
  "bf16"  the bf16 tensor-core kernel: the query operand is bf16(q); the cosine query factor is 1 / ||bf16(q)||, the row
          factor 1 / ||stored row||.  L2 ranks by ||q'||^2 + ||y||^2 - 2 q'.y and returns the re-score: the direct sum of
          squared differences between the fp32 query and the stored row (rescore_l2_kernel), re-sorted by (distance, id).
  "tf32"  the 3xTF32 tensor-core kernel on fp32 rows: the fp32 values, no extra rounding; L2 as for "bf16".

Tolerances.  A returned distance D = sum of terms t_i is held to tol * A, A = sum |t_i| (plus 1 for the constant of the
cosine distance).  tol = m * u, u = 2^-24 (fp32 unit roundoff), m = the number of fp32 roundings a term can see on its way
into the sum (the classical gamma_m bound of a recursive sum; a rounding toward zero counts as 2).  With d_pad the stored
row length (a multiple of 4 for fp32 rows, of 64 for bf16 rows):
  m_sum  = d_pad / 32 + 13: a warp sums a row, each lane at most ceil(chunks / 32) 16-byte chunks of 4 or 8 elements in a
           chain of FMAs (<= d_pad / 32 + 8), then 5 butterfly adds.  The row norms of the side arrays (row_norms_kernel),
           the cosine query normalisation and the re-score sum have this depth as well.
  scan (per metric):
         IP      m_sum: the key is the sum times -1, returned negated (both exact).
         L2      m_sum + 2: the rounded difference q - y, squared, adds 2.
         cosine  2 m_sum + 8: the normalised query and the row factor each carry half the relative error of their squared
                 norm (m_sum / 2) plus a square root and a division (2); key = sum * factor and 1 + key add 2.
  Tensor cores.  A wgmma K-step adds K products to the fp32 accumulator after aligning them to the largest exponent and
  truncating (measured on the H100: coherent-sign 3xTF32 sums lose ~130 u, four times what one rounding per step
  allows).  Each of the K + 1 addends can lose 2 u of the step's largest magnitude, which is at most S_s, the sum of
  |t_i| over the columns added so far.  Summed over the steps: 2 (K + 1) u sum_s S_s = 2 (K + 1) u sum_i w_i |t_i|, with
  w_i the number of K-steps from the one that adds column i to the last.  So the product part of a tensor-core key is
  held to 2 (K + 1) u W, W = sum_i w_i |t_i|, on top of m u A:
  bf16:  K = 16, one step per 16 columns (w_i = d_pad / 16 - i // 16); bf16 x bf16 products are exact in fp32.
  tf32:  K = 8, three steps (lo*hi, hi*lo, hi*hi) per 8 columns (w_i = 3 (d_pad / 8 - i // 8)), plus 32 u A: the split
         x = hi + lo truncates hi to TF32 (|lo| < 2^-10 |x|) and rounds lo to TF32 (error <= 2^-21 |x|); the three
         products drop lo*lo (<= 2^-20 |x y|): <= 2^-19 = 32 u per term.
  and m per metric, for what the epilogue adds to the accumulator:
         IP      0: the key is the accumulator negated, returned negated again.
         L2      m_sum + 4: ||y||^2 and ||q'||^2 are fp32 sums of depth m_sum (row_norms_kernel); the row factor, the
                 bias and ||q'||^2 are added with up to 4 roundings.
         cosine  m_sum + 8: the factors 1 / ||y|| and 1 / ||q'|| each carry m_sum / 2 + 2; key = acc * row factor and
                 1 - key * query factor add 3, rounded up to 4.
  The L2 re-score of the tensor-core paths returns a scan-form sum: it is held to the L2 scan tolerance, m_sum + 2.
The ranking key of every path (the expanded L2 form on the tensor cores) has the same tolerance over its own terms
(||q'||^2 + ||y||^2 + 2 sum |q'_i y_i|; W over the product 2 q'.y).

Contract checked by `compare`, per query:
  1. every returned id is in range, eligible (alive, finite distance, and under the IP quirk possibly > FLT_MIN), unique;
  2. every returned distance is within its bound of the float64 distance of that id;
  3. the list is sorted best first, and equal returned distances come in ascending id order.  Where the returned
     distance is a rounded function of the key (cosine: 1 + key, 1 - key / ||q||), two different keys can round to the
     same distance in key order; such a pair is accepted unless the two reference keys are exactly equal;
  4. nothing is missed: no eligible row outside the list has a key better than the worst returned key by more than the
     two bounds;
  5. exactly min(k, eligible rows) slots are filled, as a prefix; the rest hold id -1 and the sentinel: FLT_MAX, -FLT_MAX
     for IP, FLT_MIN under the IP quirk (part_scan: scores <= FLT_MIN are never returned, so the filled count lies
     between the rows surely above FLT_MIN and those possibly above it).
NaN rows: never eligible, so never returned, and they cannot displace a finite row (check 4).
"""
import numpy as np

from tests.util import to_bf16_values

L2, IP, COSINE = 0, 1, 2
F32, BF16 = 0, 1
U = 2.0 ** -24
FLT_EPS = float(np.finfo(np.float32).eps)
FLT_MAX = float(np.finfo(np.float32).max)
FLT_MIN = float(np.finfo(np.float32).tiny)
PATHS = ("scan", "bf16", "tf32")


def d_pad_of(dtype, d):
    return -(-d // 64) * 64 if dtype == BF16 else -(-d // 4) * 4


def tolerances(path, dtype, d, metric):
    """(m u of the ranking key, m u of the returned distance, per-column weights 2 (K + 1) u w_i of the tensor-core product
    or None), as derived in the module docstring."""
    dp = d_pad_of(dtype, d)
    m_sum = dp / 32 + 13
    scan = {IP: m_sum, L2: m_sum + 2, COSINE: 2 * m_sum + 8}[metric] * U
    if path == "scan":
        return scan, scan, None
    col = np.arange(d)
    m = {IP: 0, L2: m_sum + 4, COSINE: m_sum + 8}[metric] * U
    if path == "bf16":
        return m, scan, 2 * 17 * U * (dp // 16 - col // 16)
    if path == "tf32":
        return 32 * U + m, scan, 2 * 9 * U * 3 * (dp // 8 - col // 8)
    raise ValueError(path)


def stored_rows(y, dtype):
    """The values a corpus holds for fp32 rows y: fp32 as given, or bf16 round-to-nearest-even."""
    y = np.ascontiguousarray(y, np.float32)
    return to_bf16_values(y) if dtype == BF16 else y.copy()


def _unit(a):
    """Rows scaled to unit norm in float64; rows whose squared norm is below FLT_EPSILON keep a factor of 1
    (VectorDataset::normalize, row_norms_kernel)."""
    ss = (a * a).sum(1)
    f = np.where(ss < FLT_EPS, 1.0, 1.0 / np.sqrt(np.where(ss > 0, ss, 1.0)))
    return a * f[:, None]


def _direct_l2(X, Y):
    """sum_i (x_i - y_i)^2 in float64 for every (query, row), in blocks, without the cancellation of the expanded form."""
    out = np.empty((len(X), len(Y)))
    rb = max(1, (1 << 22) // max(1, Y.shape[1]))
    for r0 in range(0, len(Y), rb):
        Yb = Y[r0:r0 + rb]
        qb = max(1, (1 << 22) // (len(Yb) * max(1, Y.shape[1])))
        for q0 in range(0, len(X), qb):
            out[q0:q0 + qb, r0:r0 + rb] = ((X[q0:q0 + qb, None, :] - Yb[None, :, :]) ** 2).sum(2)
    return out


class Reference:
    """Per query and row: key (smaller is better), key_tol, dis (as returned), dis_tol, eligible."""


def reference(metric, dtype, path, y, x, k, alive=None, quirk=False):
    """y: the caller's fp32 rows [n][d]; x: fp32 queries [nq][d]; alive: bool [n] or None; quirk: the IP FLT_MIN rule of
    part_scan."""
    assert path in PATHS and not (path == "bf16" and dtype != BF16) and not (path == "tf32" and dtype != F32)
    n, d = y.shape
    Y = stored_rows(y, dtype).astype(np.float64)
    X = np.ascontiguousarray(x, np.float32)
    Xop = to_bf16_values(X) if path == "bf16" else X          # the query operand of the path
    Q = Xop.astype(np.float64)
    tol_key, tol_dis, w = tolerances(path, dtype, d, metric)
    w = np.zeros(d) if w is None else w
    with np.errstate(all="ignore"):
        if metric == COSINE:
            Qn, Yn = _unit(Q), _unit(Y)
            ip, aip, wip = Qn @ Yn.T, np.abs(Qn) @ np.abs(Yn).T, (np.abs(Qn) * w) @ np.abs(Yn).T
            key = 1.0 - ip
            dis, key_a = key, 1.0 + aip
            dis_a, key_w = key_a, wip
        elif metric == IP:
            ip, aip, wip = Q @ Y.T, np.abs(Q) @ np.abs(Y).T, (np.abs(Q) * w) @ np.abs(Y).T
            key, dis, key_a, dis_a, key_w = -ip, ip, aip, aip, wip
        else:
            Xf = X.astype(np.float64)
            qq, yy = (Q * Q).sum(1)[:, None], (Y * Y).sum(1)[None, :]
            ip, aip, wip = Q @ Y.T, np.abs(Q) @ np.abs(Y).T, (np.abs(Q) * w) @ np.abs(Y).T
            expanded = qq + yy - 2 * ip
            direct = _direct_l2(Xf, Y)   # the scan sum / the re-score, from the fp32 query
            dis, dis_a = direct, direct
            if path == "scan":
                key, key_a, key_w = direct, direct, 0.0
            else:
                key, key_a, key_w = expanded, qq + yy + 2 * aip, 2 * wip
        r = Reference()
        r.metric, r.path, r.k, r.n, r.nq, r.quirk = metric, path, k, n, len(X), quirk
        r.key, r.dis = key, dis
        r.key_tol = tol_key * key_a + key_w
        # IP and cosine return the key itself (negated / shifted); L2 returns the scan sum or the re-score
        r.dis_tol = r.key_tol if metric != L2 else tol_dis * dis_a
        ok = np.isfinite(key) & np.isfinite(dis)
    if alive is not None:
        ok &= np.asarray(alive, bool)[None, :n]
    r.possible = ok.copy()
    r.sure = ok.copy()
    if quirk:
        r.possible &= dis + r.dis_tol > FLT_MIN
        r.sure &= dis - r.dis_tol > FLT_MIN
    r.lossy = metric == COSINE
    return r


def sentinel(metric, quirk=False):
    return np.float32(FLT_MIN if quirk else (-FLT_MAX if metric == IP else FLT_MAX))


def compare(r, dis_g, ids_g, id_offset=0):
    """Problems of a library answer against the reference (empty list: it passes); see the module docstring."""
    bad = []
    dis_g = np.asarray(dis_g, np.float32)
    ids_g = np.asarray(ids_g, np.int64)
    assert dis_g.shape == ids_g.shape == (r.nq, r.k), (dis_g.shape, ids_g.shape)
    empty = sentinel(r.metric, r.quirk)
    desc = r.metric == IP
    for q in range(r.nq):
        ig, dg = ids_g[q], dis_g[q]
        filled = ig != -1
        nf = int(filled.sum())
        if not filled[:nf].all():
            bad.append(f"q{q}: unfilled slot before a filled one")
        tail = ~filled
        if (dg[tail].view(np.uint32) != empty.view(np.uint32)).any():
            bad.append(f"q{q}: unfilled slot with distance {dg[tail][dg[tail] != empty][:3]} instead of {empty}")
        rows = ig[filled] - id_offset
        if ((rows < 0) | (rows >= r.n)).any():                                                 # 1
            bad.append(f"q{q}: ids out of range {ig[filled][(rows < 0) | (rows >= r.n)][:5]}")
            continue
        if len(set(rows.tolist())) != len(rows):
            bad.append(f"q{q}: duplicate ids")
        if not r.possible[q, rows].all():
            bad.append(f"q{q}: ineligible rows returned {rows[~r.possible[q, rows]][:5]}")
        d64 = dg[filled].astype(np.float64)
        err = np.abs(d64 - r.dis[q, rows])
        off = ~(err <= r.dis_tol[q, rows])                                                      # 2 (NaN fails)
        if off.any():
            j = int(np.argmax(off))
            bad.append(f"q{q} rank {j}: id {rows[j]} distance {d64[j]!r} vs reference {r.dis[q, rows[j]]!r} "
                       f"(bound {r.dis_tol[q, rows[j]]:.3g}); {int(off.sum())} such")
        for j in range(nf - 1):                                                                 # 3
            a, b = d64[j], d64[j + 1]
            worse = a < b if desc else a > b
            if worse or (a == b and rows[j] > rows[j + 1]
                         and (not r.lossy or r.key[q, rows[j]] == r.key[q, rows[j + 1]])):
                bad.append(f"q{q} ranks {j},{j + 1}: ({a!r}, {rows[j]}) before ({b!r}, {rows[j + 1]})")
                break
        n_sure, n_poss = min(r.k, int(r.sure[q].sum())), min(r.k, int(r.possible[q].sum()))
        if not n_sure <= nf <= n_poss:                                                          # 5
            bad.append(f"q{q}: {nf} filled slots, expected {n_sure}" + (f"..{n_poss}" if n_poss != n_sure else ""))
        if nf:                                                                                  # 4
            w = rows[int(np.argmax(r.key[q, rows]))]
            out = np.ones(r.n, bool)
            out[rows] = False
            must = out & r.sure[q] & (r.key[q] + r.key_tol[q] < r.key[q, w] - r.key_tol[q, w])
            if must.any():
                bad.append(f"q{q}: rows {np.nonzero(must)[0][:5].tolist()} better than the worst returned key are missing")
    return bad


def error_ratio(r, dis_g, ids_g, id_offset=0):
    """Largest |returned - reference| / bound over the filled slots (how much of the tolerance an answer uses)."""
    ids_g = np.asarray(ids_g, np.int64)
    q, j = np.nonzero(ids_g != -1)
    if not len(q):
        return 0.0
    rows = ids_g[q, j] - id_offset
    err = np.abs(np.asarray(dis_g, np.float32)[q, j].astype(np.float64) - r.dis[q, rows])
    return float((err / np.maximum(r.dis_tol[q, rows], 1e-300)).max())


def ideal_answer(r):
    """The answer the contract describes, from the reference itself: the k best eligible rows by (key, id), distances
    rounded to fp32.  Used by the comparator's own tests."""
    dis = np.full((r.nq, r.k), sentinel(r.metric, r.quirk), np.float32)
    ids = np.full((r.nq, r.k), -1, np.int64)
    for q in range(r.nq):
        cand = np.nonzero(r.sure[q])[0]
        top = cand[np.lexsort((cand, r.key[q, cand]))][:r.k]
        fd = r.dis[q, top].astype(np.float32)      # ordered by the fp32 distance as returned, then id
        top = top[np.lexsort((top, -fd if r.metric == IP else fd))]
        dis[q, :len(top)] = r.dis[q, top].astype(np.float32)
        ids[q, :len(top)] = top
    return dis, ids
