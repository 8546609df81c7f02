"""numpy reference of the BINARYMSTG graph walk (graph_degree=D): the build is graph_reference's (candidates, rank-based pruning,
reverse-edge merge); the search is graph_reference.search's loop itself, with the binary keys of the kernel, computed exactly:
Hamming popc(q) + popc(y) - 2 popc(q & y), Jaccard (or - and) / or in float32 with or = popc(q) + popc(y) - and (0 when
or = 0).  Rows and queries are packed bytes uint8 [n][d / 8]."""
from unittest import mock

import numpy as np

from tests import graph_reference as G
from tests.graph_reference import MAX_SEEDS, NO_ID, WIDTH, build, candidates, iteration_cap  # noqa: F401

HAMMING, JACCARD = "hamming", "jaccard"


def popcount(rows):
    """uint8 [n][b] -> int64 [n]: set bits per row"""
    return np.unpackbits(np.asarray(rows, np.uint8), axis=1).sum(1, dtype=np.int64)


def keys(rows, q, ids, metric, row_popc=None):
    """float32 keys of rows[ids] against one query q (uint8 [b]): the distance BINARYFLAT returns for each (q, row)"""
    rows = np.asarray(rows, np.uint8)
    q = np.asarray(q, np.uint8)
    y = rows[ids]
    a = popcount(y & q[None, :])
    py = popcount(y) if row_popc is None else row_popc[ids]
    pq = int(popcount(q[None, :])[0])
    if metric == HAMMING:
        return (pq + py - 2 * a).astype(np.float32)
    x_or = pq + py - a
    den = np.where(x_or == 0, 1, x_or).astype(np.float32)
    return np.where(x_or == 0, np.float32(0), (x_or - a).astype(np.float32) / den).astype(np.float32)


def search(graph, rows, queries, seeds, ef, k, max_iters, metric=HAMMING, alive=None, width=WIDTH):
    """graph_reference.search's own loop over binary rows: its key function is swapped for the binary keys for the call, and it
    runs with metric "l2", under which the key is the returned distance and short answers are padded with id -1 and FLT_MAX.
    seeds [nq][S] (negative = none); alive: bool [n] or None.  Returns (dis float32 [nq][k], ids int64 [nq][k], rows scored
    per query)."""
    rows = np.asarray(rows, np.uint8)
    queries = np.asarray(queries, np.uint8)
    row_popc = popcount(rows)
    n = np.asarray(graph).shape[0]

    def binary_keys(_rows, q, ids, _metric):   # q: the loop's float32 copy of the query bytes, exact
        return keys(rows, q.astype(np.uint8), ids, metric, row_popc)

    with mock.patch.object(G, "_keys", binary_keys):
        # the loop reads rows only through the key function: a placeholder of n rows stands in for them
        return G.search(graph, np.zeros((n, 1), np.float32), queries, seeds, ef, k, max_iters, "l2", alive, width)
