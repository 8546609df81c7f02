"""Parity of the tensor-core top-k at a scale where the persistent schedule really runs: >= 2 M rows (not a multiple of
the 256-row tile), every CTA walks hundreds of corpus tiles with pacing on, every path code that selects the tensor cores,
batches of one to eight query tiles (1024 is what bench.py times) and k = 10 / 30 / 100.

Two data sets:
  * integer-valued rows and queries in [-4, 4]: every product and partial sum is an exact integer below 2^24 in bf16
    operands / fp32 accumulators, on the GPU and in the CPU oracle alike, so ids AND distances must be bit-identical --
    and ties are everywhere, which exercises the (score, smaller id) rule of BruteForceSearch.h:77-88 / faiss heaps;
  * Gaussian bf16-valued rows (the bench's distribution) under the 1e-4 contract with the near-tie rule of tests/util.py.
The checker is the oracle's threaded CPU brute force (oracle/cpu_baseline.c, itself pinned against vs_oracle.c)."""
import numpy as np
import pytest

import myscaledb_b200 as b2
import oracle as orc
from myscaledb_b200 import search as S
from tests.util import check_topk, to_bf16_values

pytestmark = pytest.mark.gpu
F32 = np.float32
N_BIG = 2_000_003
D = 768
NQ_MAX = 2048
K_MAX = 100
NQS = (129, 512, 640, 1024, 1025, 2048)
KS = (10, 30, 100)
PATHS = (S.PATH_TENSOR, S.PATH_CG1, S.PATH_CG2, S.PATH_CG2_MC2, S.PATH_CG2_MC4, S.PATH_TS)


def _cpu_topk(metric, x, y, k):
    import os
    threads = min(64, len(os.sched_getaffinity(0)))
    r = orc.knn_flat_parts_blas(metric, x, y, k, threads)
    return r if r is not None else orc.knn_flat_parts(metric, x, y, k, threads)


@pytest.fixture(scope="module")
def int_data():
    rng = np.random.default_rng(2024)
    y = rng.integers(-4, 5, (N_BIG, D), dtype=np.int8).astype(F32)
    x = rng.integers(-4, 5, (NQ_MAX, D), dtype=np.int8).astype(F32)
    alive = rng.random(N_BIG) < 0.3
    return x, y, alive


@pytest.fixture(scope="module")
def int_corpora(int_data):
    x, y, alive = int_data
    cs = {m: b2.Corpus(m, D, dtype=S.BF16).append(y) for m in (b2.IP, b2.L2)}
    yield cs
    for c in cs.values():
        c.close()


@pytest.mark.parametrize("filtered", [False, True], ids=["all_rows", "alive_bitmap"])
@pytest.mark.parametrize("metric", [b2.IP, b2.L2], ids=["IP", "L2"])
def test_every_gemm_variant_is_bit_exact_at_2m_rows(int_data, int_corpora, metric, filtered):
    x, y, alive = int_data
    if filtered:
        keep = np.flatnonzero(alive)
        do, io = _cpu_topk(metric, x, np.ascontiguousarray(y[keep]), K_MAX)
        io = np.where(io >= 0, keep[np.maximum(io, 0)], -1)
        bits = orc.pack_bits(alive)
    else:
        do, io = _cpu_topk(metric, x, y, K_MAX)
        bits = None
    c = int_corpora[metric]
    seen, failures = set(), []
    for path in PATHS:
        c.set_path(path)
        for nq in NQS:
            for k in KS:
                dg, ig = c.search(x[:nq], k, alive_bits=bits)
                kern, cg, mc, grid = c.last_variant()
                seen.add((kern, cg, mc))
                if not (np.array_equal(ig, io[:nq, :k]) and np.array_equal(dg, do[:nq, :k])):
                    bad = int((ig != io[:nq, :k]).sum())
                    failures.append((path, nq, k, (kern, cg, mc, grid), bad))
    c.set_path(S.PATH_AUTO)
    assert not failures, f"variants differing from the oracle (path, nq, k, kernel, wrong ids): {failures[:10]}"
    # the matrix above must really have launched the bf16 tensor-core kernel (the one the benchmark times), and only it
    assert seen == {(S.KERNEL_GEMM_BF16, 1, 1)}, f"unexpected kernel variants {sorted(seen)}"


def test_auto_path_picks_the_benchmarked_instantiation(int_corpora, int_data):
    """The default path for 128 .. 2048 queries on a bf16 corpus is the bf16 tensor-core kernel (exactly what bench.py
    times at 1024); one query goes to the scan."""
    x, _, _ = int_data
    c = int_corpora[b2.IP]
    c.set_path(S.PATH_AUTO)
    for nq, want in ((1024, (S.KERNEL_GEMM_BF16, 1, 1)), (2048, (S.KERNEL_GEMM_BF16, 1, 1)), (512, (S.KERNEL_GEMM_BF16, 1, 1)),
                     (256, (S.KERNEL_GEMM_BF16, 1, 1)), (128, (S.KERNEL_GEMM_BF16, 1, 1)), (1, (S.KERNEL_SCAN, 0, 0))):
        c.search(x[:nq], 10)
        assert c.last_variant()[:3] == want, (nq, c.last_variant())


@pytest.fixture(scope="module")
def gauss_data():
    import torch
    g = torch.Generator().manual_seed(77)
    n = 1_000_003
    y = torch.randn((n, D), generator=g, dtype=torch.float32).to(torch.bfloat16).to(torch.float32).numpy()
    x = torch.randn((1024, D), generator=g, dtype=torch.float32).to(torch.bfloat16).to(torch.float32).numpy()
    return x, y


@pytest.mark.parametrize("metric", [b2.IP, b2.L2, b2.COSINE], ids=["IP", "L2", "COSINE"])
def test_gaussian_rows_within_contract_at_1m_rows(gauss_data, metric):
    x, y = gauss_data
    if metric == b2.COSINE:
        xn, yn = x.copy(), y.copy()
        for a in (xn, yn):
            orc.lib().orc_normalize(a.ctypes.data_as(orc.C.POINTER(orc.C.c_float)), orc.C.c_int64(a.shape[0]), orc.C.c_int(a.shape[1]))
        do, io = _cpu_topk(orc.IP, xn, yn, K_MAX)
        do = 1 - do
    else:
        do, io = _cpu_topk(metric, x, y, K_MAX)
    c = b2.Corpus(metric, D, dtype=S.BF16).append(y)
    try:
        for path, nq in ((S.PATH_AUTO, 1024), (S.PATH_CG2_MC2, 1024), (S.PATH_CG2, 640), (S.PATH_CG1, 129), (S.PATH_TS, 512)):
            for k in (10, 100):
                c.set_path(path)
                dg, ig = c.search(x[:nq], k)
                check_topk(metric, x[:nq], y, dg, ig, do[:nq, :k], io[:nq, :k], rtol=2e-4, atol=2e-4 if metric == b2.L2 else 2e-5,
                           min_exact=0.99)
    finally:
        c.close()
