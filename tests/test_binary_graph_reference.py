"""The binary graph-walk reference (tests/binary_graph_reference.py) against graph_reference on the same walk: over rows unpacked
to 0/1 floats the squared L2 distance is the Hamming distance, exactly in float32, so both references must visit, score and
return the same rows with the same distance bits.  Jaccard keys are checked against their definition, 0 / 0 included."""
import numpy as np
import pytest

from tests import binary_graph_reference as BG
from tests import graph_reference as G


def _data(n, nbits, seed, nq=6):
    rng = np.random.default_rng(seed)
    centres = rng.integers(0, 2, (8, nbits), dtype=np.uint8)
    bits = centres[rng.integers(0, 8, n)] ^ (rng.random((n, nbits)) < 0.1).astype(np.uint8)
    y = np.packbits(bits, axis=1)
    y[rng.integers(0, n, n // 20)] = y[rng.integers(0, n, n // 20)]   # duplicate rows: tied keys
    qb = centres[rng.integers(0, 8, nq)] ^ (rng.random((nq, nbits)) < 0.1).astype(np.uint8)
    return y, np.packbits(qb, axis=1)


def _graph(y, D, metric):
    """the graph of the exact 2D + 1 nearest of every row (ties to the smaller id)"""
    n = len(y)
    K1 = 2 * D + 1
    ids = np.empty((n, K1), np.int64)
    for i in range(n):
        kk = BG.keys(y, y[i], np.arange(n), metric)
        ids[i] = np.lexsort((np.arange(n), kk))[:K1]
    return G.build(G.candidates(ids), D)


@pytest.mark.parametrize("width", [1, 2, 8])
@pytest.mark.parametrize("filtered", [False, True])
def test_hamming_walk_is_the_float_walk_over_unpacked_rows(width, filtered):
    y, q = _data(400, 64, 1)
    D = 16
    g = _graph(y, D, BG.HAMMING)
    seeds = np.random.default_rng(2).integers(-1, len(y), (len(q), 8))
    alive = np.random.default_rng(3).random(len(y)) < 0.5 if filtered else None
    yf = np.unpackbits(y, axis=1).astype(np.float32)
    qf = np.unpackbits(q, axis=1).astype(np.float32)
    for ef, k in ((16, 10), (64, 10), (1024, 50)):
        cap = G.iteration_cap(D, width)
        bd, bi, bs = BG.search(g, y, q, seeds, ef, k, cap, BG.HAMMING, alive, width)
        fd, fi, fs = G.search(g, yf, qf, seeds, ef, k, cap, "l2", alive, width)
        assert np.array_equal(bi, fi) and bd.tobytes() == fd.tobytes() and np.array_equal(bs, fs), (ef, k)
        if filtered:
            assert alive[bi[bi >= 0]].all()


def test_keys_are_the_definitions():
    rng = np.random.default_rng(4)
    y = rng.integers(0, 256, (200, 25), dtype=np.uint8)
    y[:3] = 0
    for q in (rng.integers(0, 256, 25, dtype=np.uint8), np.zeros(25, np.uint8)):
        yb = np.unpackbits(y, axis=1).astype(bool)
        qb = np.unpackbits(q).astype(bool)
        a = (yb & qb).sum(1)
        o = (yb | qb).sum(1)
        ham = BG.keys(y, q, np.arange(len(y)), BG.HAMMING)
        assert np.array_equal(ham, (yb ^ qb).sum(1).astype(np.float32))
        jac = BG.keys(y, q, np.arange(len(y)), BG.JACCARD)
        want = np.array([0.0 if oo == 0 else np.float32(oo - aa) / np.float32(oo) for aa, oo in zip(a, o)], np.float32)
        assert jac.tobytes() == want.tobytes()
        if not q.any():
            assert (jac[:3] == 0).all()
