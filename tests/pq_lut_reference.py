"""Float64 reference of the PQ table look-up scan (d / M outside {1, 2, 4, 8}), on top of tests/ivf_reference.py.

The look-up scan tabulates T[q][j][e] = <q_j, cb_j[e]> in fp32 from the fp32 (prepared) query and the fp32 codebook, so unlike
the tensor-core decoder there is no bf16 rounding to reproduce: the key of (query, row) is, in float64,
  L2:     ||q - c_l||^2 + 2 <c_l, r^> + ||r^||^2 - 2 <q, r^>
  IP:     -(<q, c_l> + <q, r^>)          cosine: 1 - (<q, c_l> + <q, r^>)
with r^ the fp32 codewords of the row's codes and c_l its list centroid.  The file reader, the coarse probe, the query
preparation and the comparator are those of tests/ivf_reference.py.  numpy only: nothing here imports the library."""
import numpy as np

from tests import ivf_reference as R


def is_lut(s):
    """PQ scanned by table look-up rather than decoded to bf16 tensor-core tiles."""
    return s.payload == R.PAYLOAD_PQ and s.dsub not in (1, 2, 4, 8)


def pq_decode(s, codes):
    """codes [rows][code_bytes] -> the fp32 codewords the look-up table is built from, [rows][d] fp32."""
    j = np.arange(s.m)
    return s.codebook[j[None, :], codes[:, :s.m].astype(np.int64)].reshape(len(codes), s.d)


def lut_products(s, Q, codes, table_round):
    """sum_j T[q][j][code_j] with the table T[q][j][e] = <q_j, cb_j[e]> passed through table_round (a perturbation for
    negative controls: e.g. a bf16-rounded table), [nq][rows] float64."""
    cb = s.codebook.astype(np.float64)
    Qs = np.asarray(Q, np.float64).reshape(len(Q), s.m, s.dsub)
    t = np.zeros((len(Q), len(codes)))
    for j in range(s.m):
        T = np.asarray(table_round((Qs[:, j, :] @ cb[j].T).astype(np.float32)), np.float64)   # [nq][256]
        t += T[:, codes[:, j].astype(np.int64)]
    return t


def row_keys(s, Q, table_round=None):
    """First-stage keys of every (prepared query, stored row of s.flat()): (key [nq][rows] smaller is better, distance as
    returned, tol), tol = TOL_REL x the sum of the absolute values of the key's terms, as in tests/ivf_reference.py."""
    assert is_lut(s), "a table look-up PQ index expected"
    _, lst, pay = s.flat()
    Q64 = np.asarray(Q, np.float64)
    Rv = pq_decode(s, pay).astype(np.float64)
    C = s.centroids.astype(np.float64)
    Cr = C[lst]
    t, at = Q64 @ Rv.T, np.abs(Q64) @ np.abs(Rv).T
    if table_round is not None:
        t = lut_products(s, Q, pay, table_round)
    tol_rel = R.TOL_REL
    if s.metric == R.L2:
        pc = ((Q64[:, None, :] - C[None, :, :]) ** 2).sum(2)[:, lst]     # ||q - c_l||^2
        cr = (Cr * Rv).sum(1)[None, :]
        acr = np.abs(Cr * Rv).sum(1)[None, :]
        rr = (Rv * Rv).sum(1)[None, :]
        key = pc + 2 * cr + rr - 2 * t
        return key, np.maximum(key, 0.0), tol_rel * (pc + 2 * acr + rr + 2 * at)
    qc, aqc = (Q64 @ C.T)[:, lst], (np.abs(Q64) @ np.abs(C).T)[:, lst]
    sc = qc + t
    if s.metric == R.IP:
        return -sc, sc, tol_rel * (aqc + at)
    return 1 - sc, 1 - sc, tol_rel * (1 + aqc + at)


def reference_search(s, queries, k, nprobe, alive=None, table_round=None):
    """tests/ivf_reference.reference_search for a table look-up PQ index.  alive: bool [n] or None; table_round: see
    lut_products.  The result is checked with ivf_reference.compare."""
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
    """Build invariants of a stored table look-up PQ index s (ivf_reference.read_index) of ix built from the rows y:
    ivf_reference.check_lists, a finite codebook, every code the nearest fp32 codeword of the row's residual, zero padding
    bytes and row_bias from the fp32 codewords."""
    ids, lst, pay, x = R.check_lists(s, ix, y)
    assert np.isfinite(s.codebook).all(), "a codeword is not finite"
    n = len(ids)
    X, C = x[ids].astype(np.float64), s.centroids.astype(np.float64)
    res = X - C[lst]
    cb = s.codebook.astype(np.float64)
    for j in range(s.m):
        r = res[:, j * s.dsub:(j + 1) * s.dsub]
        dd = ((r[:, None, :] - cb[j][None, :, :]) ** 2).sum(2)
        got = dd[np.arange(n), pay[:, j]]
        assert (got <= dd.min(1) + 1e-5 * ((r * r).sum(1) + (cb[j] ** 2).sum(1).max()) + 1e-12).all(), f"PQ code {j} is not the nearest fp32 codeword"
    assert (pay[:, s.m:] == 0).all(), "PQ padding bytes must be 0"
    if s.metric == R.L2:
        Rf = pq_decode(s, pay).astype(np.float64)
        np.testing.assert_array_equal(Rf, cb[np.arange(s.m)[None, :], pay[:, :s.m].astype(np.int64)].reshape(n, s.d))
        bias = (Rf * (Rf + 2 * C[lst])).sum(1)
        S = (np.abs(Rf) * np.abs(Rf + 2 * C[lst])).sum(1)
        b = np.concatenate(s.bias).astype(np.float64)
        assert (np.abs(b - bias) <= R.TOL_REL * S + 1e-30).all(), "row_bias differs from its fp32 formula"
    else:
        assert all(a is None for a in s.bias)
