"""numpy reference of the HNSWFLAT neighbour graph (graph_degree=D): candidate lists, rank-based pruning, the reverse-edge merge
and the graph search loop with the kernel's exact tie rule (smaller key, then smaller id)."""
import numpy as np

NO_ID = 0xFFFFFFFF
VISITED_SLOTS = 1 << 14
MAX_SEEDS = 32
WIDTH = 1


def iteration_cap(degree, width=WIDTH):
    """Iterations one query may run: the visited table (VISITED_SLOTS ids) stays at most half full."""
    return (VISITED_SLOTS // 2 - MAX_SEEDS) // (width * degree)


def candidates(ids, row0=0):
    """ids: int64 [m][K + 1] of the list search of rows row0 .. row0 + m - 1 -> uint32 [m][K]: the row's own id dropped (or,
    when absent, the last entry), negative ids as NO_ID."""
    ids = np.asarray(ids, np.int64)
    m, k1 = ids.shape
    out = np.empty((m, k1 - 1), np.uint32)
    for i in range(m):
        row = ids[i]
        hit = np.nonzero(row == row0 + i)[0]
        self_pos = int(hit[0]) if len(hit) else k1 - 1
        keep = np.delete(row, self_pos)
        out[i] = np.where(keep >= 0, keep, NO_ID).astype(np.uint32)
    return out


def prune(cand, D, chunk=2048):
    """cand: uint32 [n][K] (NO_ID = none, at the tail) -> uint32 [n][D].  detour(A, j) = #{i < j : rank of c[j] in
    cand(c[i]) < j}; keeps the D valid candidates with the smallest (detour, j), in that order."""
    cand = np.asarray(cand, np.uint32)
    n, K = cand.shape
    c64 = cand.astype(np.int64)
    valid = cand != NO_ID
    # rank of v in cand(u) by key u * n + v
    u = np.repeat(np.arange(n, dtype=np.int64), K)
    v = c64.ravel()
    p = np.tile(np.arange(K, dtype=np.int64), n)
    m = v != NO_ID
    keys = u[m] * n + v[m]
    order = np.argsort(keys, kind="stable")
    keys, pos = keys[order], p[m][order]
    ii, jj = np.triu_indices(K, 1)
    onehot = np.zeros((len(jj), K), np.int64)
    onehot[np.arange(len(jj)), jj] = 1
    out = np.full((n, D), NO_ID, np.uint32)
    for a0 in range(0, n, chunk):
        ci, cj = c64[a0:a0 + chunk, ii], c64[a0:a0 + chunk, jj]
        ok = (ci != NO_ID) & (cj != NO_ID)
        q = np.where(ok, ci * n + cj, -1)
        idx = np.clip(np.searchsorted(keys, q), 0, max(len(keys) - 1, 0))
        found = ok & (keys[idx] == q) if len(keys) else np.zeros_like(ok)
        hit = found & (pos[idx] < jj[None, :])
        det = hit.astype(np.int64) @ onehot
        key = det * K + np.arange(K)[None, :]
        vb = valid[a0:a0 + chunk]
        key = np.where(vb, key, np.iinfo(np.int64).max)
        sel = np.argsort(key, axis=1, kind="stable")[:, :D]
        got = np.take_along_axis(cand[a0:a0 + chunk], sel, 1)
        got[~np.take_along_axis(vb, sel, 1)] = NO_ID
        out[a0:a0 + chunk] = got
    return out


def merge(pruned, D):
    """graph(B): the first D/2 pruned forward edges of B; then B's reverse sources sorted by (rank, source), at most D/2 of them
    added; then the remaining forward edges.  Duplicates skipped, at most D entries, NO_ID padding."""
    pruned = np.asarray(pruned, np.uint32)
    n = pruned.shape[0]
    A = np.repeat(np.arange(n, dtype=np.int64), D)
    r = np.tile(np.arange(D, dtype=np.int64), n)
    B = pruned.ravel().astype(np.int64)
    m = B != NO_ID
    order = np.lexsort((A[m], r[m], B[m]))
    Bs, As = B[m][order], A[m][order]
    starts = np.searchsorted(Bs, np.arange(n), "left")
    ends = np.searchsorted(Bs, np.arange(n), "right")
    graph = np.full((n, D), NO_ID, np.uint32)
    for b in range(n):
        row = []
        seen = set()

        def add(x):
            if x != NO_ID and x not in seen and len(row) < D:
                row.append(x)
                seen.add(x)
                return True
            return False

        for x in pruned[b, :D // 2]:
            add(int(x))
        added = 0
        for x in As[starts[b]:ends[b]]:
            if added >= D // 2 or len(row) >= D:
                break
            added += add(int(x))
        for x in pruned[b, D // 2:]:
            add(int(x))
        graph[b, :len(row)] = row
    return graph


def build(cand, D):
    return merge(prune(cand, D), D)


def _keys(rows, q, ids, metric):
    y = rows[ids].astype(np.float64)
    qq = q.astype(np.float64)
    if metric == "l2":
        return (((y - qq) ** 2).sum(1)).astype(np.float32)
    return (-(y @ qq)).astype(np.float32)


def search(graph, rows, queries, seeds, ef, k, max_iters, metric="l2", alive=None, width=WIDTH):
    """The kernel's loop.  rows: the stored fp32 rows [n][d] (cosine: unit rows, with metric "cosine" and unit queries);
    seeds [nq][S] (negative = none); alive: bool [n] or None.  Returns (dis float32 [nq][k], ids int64 [nq][k], rows scored
    per query): L2 the squared distance, IP the inner product, cosine 1 - cos; short answers padded with id -1."""
    graph = np.asarray(graph, np.uint32)
    n, D = graph.shape
    rows = np.asarray(rows, np.float32)
    queries = np.asarray(queries, np.float32)
    nq = queries.shape[0]
    key_metric = "l2" if metric == "l2" else "ip"
    out_d = np.empty((nq, k), np.float32)
    out_i = np.full((nq, k), -1, np.int64)
    scored_per_q = np.zeros(nq, np.int64)
    for qi in range(nq):
        q = queries[qi]
        visited = set()
        lst = []        # [key, id, expanded]
        alst = []       # (key, id)
        scored = 0

        def step(raw):
            nonlocal lst, alst, scored
            new = []
            for v in raw:
                v = int(v)
                if v < 0 or v >= n or v in visited:
                    continue
                visited.add(v)
                new.append(v)
            if not new:
                return
            keys = _keys(rows, q, np.array(new, np.int64), key_metric)
            scored += len(new)
            cands = [[float(kk), v, False] for kk, v in zip(keys, new)]
            lst = sorted(lst + cands, key=lambda e: (np.float32(e[0]), e[1]))[:ef]
            if alive is not None:
                alst = sorted(alst + [(c[0], c[1]) for c in cands if alive[c[1]]], key=lambda e: (np.float32(e[0]), e[1]))[:k]

        step(seeds[qi])
        for _ in range(max_iters):
            parents = [e for e in lst if not e[2]][:width]
            if not parents:
                break
            for e in parents:
                e[2] = True
            step(np.concatenate([graph[e[1]] for e in parents]).astype(np.int64))
        res = alst if alive is not None else [(e[0], e[1]) for e in lst[:k]]
        for j in range(k):
            if j < len(res):
                kk = np.float32(res[j][0])
                out_i[qi, j] = res[j][1]
                out_d[qi, j] = kk if metric == "l2" else (np.float32(1) - (-kk) if metric == "cosine" else -kk)
            else:
                out_d[qi, j] = -np.finfo(np.float32).max if metric == "ip" else np.finfo(np.float32).max
        scored_per_q[qi] = scored
    return out_d, out_i, scored_per_q
