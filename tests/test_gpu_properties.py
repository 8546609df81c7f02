"""Randomised GPU-vs-oracle properties (hypothesis) on small integer-valued inputs, where fp32 / bf16 / tf32 sums are
exact and ties are everywhere, so every path of the library must return EXACTLY the oracle's ids and distances.

Part of the `gpu` suite."""

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import oracle as orc

pytestmark = pytest.mark.gpu
F32 = np.float32


def _b2():
    import myscaledb_b200 as b2
    from myscaledb_b200 import search as S
    return b2, S


@settings(max_examples=40, deadline=None)
@given(st.integers(1, 3000), st.integers(1, 40), st.integers(1, 40), st.integers(1, 20), st.integers(0, 2 ** 31),
       st.sampled_from([0, 1]), st.sampled_from([0, 1, 2]))
def test_every_path_is_exact_on_integer_data(n, d, nq, k, seed, metric, path):
    """path 0 auto, 1 FMA scan, 2 tensor cores (3xTF32 on fp32 rows): integer data in [-4, 4] -> exact arithmetic."""
    b2, S = _b2()
    rng = np.random.default_rng(seed)
    y = rng.integers(-4, 5, (n, d)).astype(F32)
    x = rng.integers(-4, 5, (nq, d)).astype(F32)
    do, io = orc.knn_flat(metric, x, y, k)
    c = b2.Corpus(metric, d).append(y)
    c.set_path(path)
    dg, ig = c.search(x, k)
    c.close()
    assert (ig == io).all()
    assert np.array_equal(np.where(io >= 0, dg, 0), np.where(io >= 0, do, 0))


@settings(max_examples=25, deadline=None)
@given(st.integers(1, 3000), st.sampled_from([64, 128, 192]), st.integers(1, 300), st.integers(1, 12), st.integers(0, 2 ** 31),
       st.sampled_from([0, 1]))
def test_bf16_corpus_paths_are_exact_on_integer_data(n, d, nq, k, seed, metric):
    b2, S = _b2()
    rng = np.random.default_rng(seed)
    y = rng.integers(-4, 5, (n, d)).astype(F32)   # exactly representable in bf16
    x = rng.integers(-4, 5, (nq, d)).astype(F32)
    do, io = orc.knn_flat(metric, x, y, k)
    for path in (1, 2, 3, 4, 7):
        c = b2.Corpus(metric, d, dtype=S.BF16).append(y)
        c.set_path(path)
        dg, ig = c.search(x, k)
        c.close()
        assert (ig == io).all(), path
        assert np.array_equal(np.where(io >= 0, dg, 0), np.where(io >= 0, do, 0)), path


@settings(max_examples=40, deadline=None)
@given(st.integers(1, 2000), st.integers(1, 8), st.integers(1, 12), st.integers(1, 64), st.integers(0, 2 ** 31),
       st.sampled_from([0, 1]), st.floats(0.0, 1.0))
def test_part_scan_blocks_filters_and_lightweight_deletes(n, d, k, block_rows, seed, metric, p_alive):
    b2, S = _b2()
    rng = np.random.default_rng(seed)
    y = rng.integers(-3, 4, (n, d)).astype(F32)
    x = rng.integers(-3, 4, (2, d)).astype(F32)
    alive = rng.random(n) < p_alive
    for kw in ({}, {"filter_bits": orc.pack_bits(alive)}, {"row_exists": alive.astype(np.uint8)}):
        do, io = orc.part_scan(metric, x, y, k, block_rows=block_rows, **kw)
        dg, ig = b2.part_scan(metric, x, y, k, block_rows=block_rows, **kw)
        assert (ig == io).all(), kw.keys()
        assert np.array_equal(np.where(io >= 0, dg, 0), np.where(io >= 0, do, 0)), kw.keys()


@settings(max_examples=40, deadline=None)
@given(st.integers(1, 3000), st.integers(1, 16), st.integers(1, 20), st.integers(1, 5), st.integers(0, 2 ** 31), st.sampled_from([3, 4]))
def test_binary_metrics(n, nbytes, k, nq, seed, metric):
    b2, S = _b2()
    rng = np.random.default_rng(seed)
    y = rng.integers(0, 256, (n, nbytes), dtype=np.uint8)
    x = rng.integers(0, 256, (nq, nbytes), dtype=np.uint8)
    do, io = orc.knn_binary(metric, x, y, k)
    dg, ig = b2.binary_knn(metric, x, y, k)
    assert (ig == io).all()
    assert np.array_equal(np.where(io >= 0, dg, 0), np.where(io >= 0, do, 0))


@settings(max_examples=30, deadline=None)
@given(st.integers(2, 200), st.integers(0, 2 ** 31), st.integers(1, 10), st.booleans())
def test_bm25_random_corpora_bit_exact(n_docs, seed, topk, operator_or):
    b2, S = _b2()
    rng = np.random.default_rng(seed)
    vocab = [f"w{i}" for i in range(30)]
    g, o = b2.BM25Index(1), orc.BM25Index(1)
    for i in range(n_docs):
        t = " ".join(rng.choice(vocab, size=int(rng.integers(1, 40))))
        g.add_doc(i, [t]); o.add_doc(i, [t])
    g.commit()
    queries = [" ".join(rng.choice(vocab, size=int(rng.integers(1, 4)), replace=False)) for _ in range(5)]
    res = g.search_batch(queries, topk, operator_or=operator_or)
    for qs, (rows, sc) in zip(queries, res):
        er, es = o.search(qs, topk, operator_or=operator_or)
        assert [int(r) for r in rows] == [int(r) for r in er], qs
        assert [float(s) for s in sc] == [float(s) for s in es], qs
