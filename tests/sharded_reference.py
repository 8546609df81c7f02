"""Reference of the cross-shard merge of sharded search, and an exact integer reference for integer-valued data.

A sharded search has every rank search its own rows (ids shifted by the shard's first global row id) and merges the
per-rank [nq][k] lists into the global top k.  `merge` is that merge written plainly: per query it keeps the entries with
an id >= 0, orders them by (distance, id) -- the distance negated when larger is better (IP) -- takes k, and fills the rest
with id -1 and the sentinel of `flat_reference.sentinel` (FLT_MAX, -FLT_MAX when descending).  The distances are copied,
never recomputed, so the merged answer must equal the library's byte for byte; `compare` checks exactly that.

`integer_topk` is the exact answer for rows and queries of small integers (|v| <= 8, d <= 768): every product, sum and
norm is an integer below 2^24, so fp32 and bf16 hold every value, every partial sum and every distance exactly on every
search path, and ties between equal rows are real ties that must go to the smaller id.
numpy only: nothing here imports the library, so the reference cannot share a bug with it.
"""
import numpy as np

L2, IP = 0, 1
FLT_MAX = np.float32(np.finfo(np.float32).max)


def sentinel(descending):
    return np.float32(-FLT_MAX if descending else FLT_MAX)


def merge(lists, k, descending):
    """lists: sequence of (dis [nq][k_i], ids [nq][k_i]) holding global ids (-1 = unused slot).  -> (dis [nq][k] fp32,
    ids [nq][k] int64)."""
    dis_all = np.concatenate([np.asarray(d, np.float32) for d, _ in lists], axis=1)
    ids_all = np.concatenate([np.asarray(i, np.int64) for _, i in lists], axis=1)
    nq = dis_all.shape[0]
    out_d = np.full((nq, k), sentinel(descending), np.float32)
    out_i = np.full((nq, k), -1, np.int64)
    for q in range(nq):
        keep = np.nonzero(ids_all[q] >= 0)[0]
        d, i = dis_all[q, keep], ids_all[q, keep]
        order = np.lexsort((i, -d.astype(np.float64) if descending else d))[:k]
        out_d[q, :len(order)] = d[order]
        out_i[q, :len(order)] = i[order]
    return out_d, out_i


def compare(expected, got):
    """Problems of an answer (dis, ids) against the expected one (empty list: it passes): ids equal, distance bits equal."""
    (de, ie), (dg, ig) = expected, got
    de, dg = np.asarray(de, np.float32), np.asarray(dg, np.float32)
    ie, ig = np.asarray(ie, np.int64), np.asarray(ig, np.int64)
    if de.shape != dg.shape or ie.shape != ig.shape:
        return [f"shape {dg.shape} / {ig.shape}, expected {de.shape} / {ie.shape}"]
    bad = []
    for q in np.nonzero((ie != ig).any(1) | (de.view(np.uint32) != dg.view(np.uint32)).any(1))[0][:8]:
        j = int(np.argmax((ie[q] != ig[q]) | (de[q].view(np.uint32) != dg[q].view(np.uint32))))
        bad.append(f"q{q} rank {j}: ({dg[q, j]!r}, {ig[q, j]}) expected ({de[q, j]!r}, {ie[q, j]})")
    return bad


def integer_topk(metric, x, y, k, alive=None, id_offset=0):
    """Exact top k of integer-valued fp32 queries x [nq][d] over rows y [n][d] in int64: L2 = sum (x - y)^2 ascending, IP =
    x . y descending; ties to the smaller id; alive: bool [n] or None.  -> (dis fp32, ids int64) with the unfilled tail."""
    X = np.asarray(x).astype(np.int64)
    Y = np.asarray(y).astype(np.int64)
    assert np.array_equal(X, x) and np.array_equal(Y, y), "integer_topk needs integer-valued data"
    if metric == L2:
        key = (X * X).sum(1)[:, None] + (Y * Y).sum(1)[None, :] - 2 * X @ Y.T
    elif metric == IP:
        key = -(X @ Y.T)
    else:
        raise ValueError(metric)
    assert np.abs(key).max(initial=0) < 1 << 24
    desc = metric == IP
    nq, n = key.shape
    out_d = np.full((nq, k), sentinel(desc), np.float32)
    out_i = np.full((nq, k), -1, np.int64)
    cand = np.arange(n) if alive is None else np.nonzero(np.asarray(alive, bool)[:n])[0]
    for q in range(nq):
        top = cand[np.lexsort((cand, key[q, cand]))][:k]
        out_d[q, :len(top)] = (-key[q, top] if desc else key[q, top]).astype(np.float32)
        out_i[q, :len(top)] = top + id_offset
    return out_d, out_i
