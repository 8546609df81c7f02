"""CPU checks of the numpy graph reference (tests/graph_reference.py) that the GPU graph tests compare against: candidate
lists, rank-based pruning, the reverse-edge merge and the search loop, on hand-made cases."""
import numpy as np

from tests import graph_reference as G

NO = G.NO_ID


def prune_direct(cand, D):
    """The definition, one node and one pair at a time."""
    n, K = cand.shape
    out = np.full((n, D), NO, np.uint32)
    for a in range(n):
        c = [int(x) for x in cand[a]]
        det = []
        for j in range(K):
            if c[j] == NO:
                continue
            cnt = 0
            for i in range(j):
                if c[i] == NO:
                    continue
                lst = [int(x) for x in cand[c[i]]]
                if c[j] in lst and lst.index(c[j]) < j:
                    cnt += 1
            det.append((cnt, j))
        keep = sorted(det)[:D]
        for r, (_, j) in enumerate(keep):
            out[a, r] = c[j]
    return out


def test_candidates_drop_self_or_last():
    ids = np.array([[0, 5, 6, 7, 8],        # self first
                    [2, 1, 3, -1, -1],      # self inside, short list
                    [0, 1, 3, 4, 9]])       # duplicate rows: self (2) absent -> drop the last
    c = G.candidates(ids)
    assert c.tolist() == [[5, 6, 7, 8], [2, 3, NO, NO], [0, 1, 3, 4]]
    # a chunk starting at row 10
    c = G.candidates(np.array([[3, 10, 4]]), row0=10)
    assert c.tolist() == [[3, 4]]


def test_prune_hand_case():
    # node 0: candidates 1, 2, 3 (K = 4, one padding).  cand(1) ranks 2 at 0 < its position 1 in cand(0): a detour to 2.
    # cand(1) ranks 3 at 1 < 2 and cand(2) ranks 3 at 0 < 2: two detours to 3.  D = 2 keeps (0, 1) = 1, then (1, 2) = 2.
    cand = np.array([[1, 2, 3, NO],
                     [2, 3, 0, NO],
                     [3, 0, 1, NO],
                     [0, 1, 2, NO]], np.uint32)
    p = G.prune(cand, 2)
    assert p[0].tolist() == [1, 2]
    assert (p == prune_direct(cand, 2)).all()


def test_prune_matches_definition_with_padding():
    rng = np.random.default_rng(1)
    n, D = 60, 4
    K = 2 * D
    cand = np.full((n, K), NO, np.uint32)
    for a in range(n):
        others = np.delete(np.arange(n), a)
        m = int(rng.integers(2, K + 1))      # short lists: -1 candidates become padding at the tail
        cand[a, :m] = rng.choice(others, m, replace=False)
    p = G.prune(cand, D)
    assert (p == prune_direct(cand, D)).all()
    # fewer valid candidates than D: padded
    short = np.nonzero((cand != NO).sum(1) < D)[0]
    for a in short:
        assert (p[a, (cand[a] != NO).sum():] == NO).all()


def test_merge_reverse_overflow_and_order():
    D = 4
    n = 7
    pruned = np.full((n, D), NO, np.uint32)
    pruned[0] = [1, 2, 3, 4]
    for a in range(1, n):   # every other node points to 0: at rank 1 for a = 1..3, rank 0 for a = 4..6
        pruned[a] = [0, 1, NO, NO] if a >= 4 else [6, 0, NO, NO]
    g = G.merge(pruned, D)
    # forward 1, 2; reverse sources in (rank, source) order are 4, 5, 6 (rank 0), 1, 2, 3 (rank 1): only D / 2 = 2 added
    assert g[0].tolist() == [1, 2, 4, 5]
    # node 1: forward 6, 0; reverse 0 (rank 0, a duplicate: skipped, not counted), then 4, 5 (rank 1); 6 would overflow D / 2
    assert g[1].tolist() == [6, 0, 4, 5]
    # node 6: forward 0, 1; reverse 1 (duplicate), 2, 3
    assert g[6].tolist() == [0, 1, 2, 3]
    # node 5: no reverse edges, two forward edges, padding
    assert g[5].tolist() == [0, 1, NO, NO]


def test_search_complete_graph_is_exact():
    rng = np.random.default_rng(2)
    n, d, D = 40, 8, 64
    rows = rng.integers(-3, 4, (n, d)).astype(np.float32)
    q = rng.integers(-3, 4, (3, d)).astype(np.float32)
    graph = np.full((n, D), NO, np.uint32)
    for a in range(n):
        graph[a, :n - 1] = np.delete(np.arange(n), a)
    seeds = np.array([[0], [5], [-1]], np.int64)
    seeds[2, 0] = 7
    dis, ids, scored = G.search(graph, rows, q, seeds, ef=16, k=5, max_iters=10)
    for i in range(3):
        d2 = ((rows - q[i]) ** 2).sum(1)
        order = np.lexsort((np.arange(n), d2))[:5]
        assert ids[i].tolist() == order.tolist()
        assert np.array_equal(dis[i], d2[order].astype(np.float32))
    assert (scored == n).all()   # every row once
    # inner product: distance = <q, y>, best first
    dis, ids, _ = G.search(graph, rows, q, seeds, ef=16, k=5, max_iters=10, metric="ip")
    ip = rows @ q[0]
    order = np.lexsort((np.arange(n), -ip))[:5]
    assert ids[0].tolist() == order.tolist() and np.array_equal(dis[0], ip[order])


def test_search_cap_stops():
    n, d, D = 50, 2, 2
    rows = np.stack([np.arange(n), np.zeros(n)], 1).astype(np.float32)   # a path 0 - 1 - 2 - ...
    graph = np.full((n, D), NO, np.uint32)
    for a in range(n):
        nb = [x for x in (a - 1, a + 1) if 0 <= x < n]
        graph[a, :len(nb)] = nb
    q = np.array([[n - 1, 0]], np.float32)
    seeds = np.array([[0]])
    _, ids, scored = G.search(graph, rows, q, seeds, ef=4, k=1, max_iters=5)
    assert scored[0] <= 1 + 5 * D
    assert ids[0, 0] == 5        # walked 5 steps along the path
    _, ids, _ = G.search(graph, rows, q, seeds, ef=4, k=1, max_iters=1000)
    assert ids[0, 0] == n - 1


def test_search_filter_short_answer():
    n, d, D = 30, 4, 32
    rng = np.random.default_rng(3)
    rows = rng.integers(0, 5, (n, d)).astype(np.float32)
    graph = np.full((n, D), NO, np.uint32)
    for a in range(n):
        graph[a, :n - 1] = np.delete(np.arange(n), a)
    alive = np.zeros(n, bool)
    alive[[3, 17]] = True
    q = rows[:1] + 0.5
    dis, ids, _ = G.search(graph, rows, q, np.array([[0]]), ef=8, k=5, max_iters=20, alive=alive)
    d2 = ((rows[[3, 17]] - q[0]) ** 2).sum(1)
    o = np.lexsort(([3, 17], d2))
    assert ids[0, :2].tolist() == [[3, 17][i] for i in o]
    assert (ids[0, 2:] == -1).all() and (dis[0, 2:] == np.finfo(np.float32).max).all()


def test_iteration_cap_values():
    assert [G.iteration_cap(D) for D in (16, 32, 64)] == [510, 255, 127]
