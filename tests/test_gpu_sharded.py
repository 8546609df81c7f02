"""Sharded search (csrc/comm.cu) against the per-shard answers and a float64 reference.

One GPU: a world = 1 communicator.  Every sharded call must return the same bytes as the plain search of the same corpus /
index with the same id_offset, bitmap and path, and where a reference applies it must pass it: flat_reference.compare for
float corpora, the CPU oracle for binary corpora, ivf_reference for an inverted-file index.  Then the CUDA-graph replays:
a replay must answer as an eager call would after anything that changes what the captured nodes point at (appends,
set_path, workspaces that grew for another search, a new corpus at a freed one's address), and the capture / replay
counters show which one ran.

Two or more GPUs: one process per GPU; every rank's answer must equal sharded_reference.merge of the per-rank plain
answers (carried over gloo, not through the library), and pass the float64 / exact integer reference of all rows."""
import copy
import ctypes as C
import os
import socket
import sys
import traceback

import numpy as np
import pytest

import myscaledb_b200 as b2
import oracle as orc
from myscaledb_b200 import search as S
from myscaledb_b200._lib import lib
from myscaledb_b200.sharding import Comm, shard_range
from tests import flat_reference as fr
from tests import ivf_reference as R
from tests import sharded_reference as SR
from tests.util import to_bf16_values

pytestmark = pytest.mark.gpu
F32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_INVALID = 1
BIG_OFFSET = (1 << 32) + 3
NOTES = {}


@pytest.fixture(scope="module")
def env():
    import torch
    torch.cuda.init()
    comm = Comm(0, 1, Comm.unique_id())
    stream = torch.cuda.Stream()
    yield comm, stream
    torch.cuda.synchronize()
    comm.close()
    for k, v in NOTES.items():
        print(f"{k}: {v}")


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


class Call:
    """Device queries, bitmap and outputs of one search shape, kept so that repeated calls pass the same pointers."""

    def __init__(self, x, k, bits=None, nq=None, cap_k=None):
        import torch
        rows, cap_k = len(x), cap_k or k
        self.q = _dev(x)
        self.a = _dev(bits) if bits is not None else None
        self.od = torch.empty(rows * cap_k, dtype=torch.float32, device="cuda")
        self.oi = torch.empty(rows * cap_k, dtype=torch.int64, device="cuda")
        self.pd = torch.empty(rows * cap_k, dtype=torch.float32, device="cuda")
        self.pi = torch.empty(rows * cap_k, dtype=torch.int64, device="cuda")
        self.nq, self.k = nq or rows, k

    def _out(self, d, i):
        n = self.nq * self.k
        return d[:n].cpu().numpy().reshape(self.nq, self.k), i[:n].cpu().numpy().reshape(self.nq, self.k)

    def sharded(self, comm, c, stream, id_offset=0, use_graph=False, nq=None, k=None):
        import torch
        self.nq, self.k = nq or self.nq, k or self.k
        torch.cuda.synchronize()
        comm.sharded_corpus_search(c, self.q.data_ptr(), self.nq, self.k, self.od.data_ptr(), self.oi.data_ptr(), id_offset,
                                   stream.cuda_stream, use_graph=use_graph, alive_ptr=self.a.data_ptr() if self.a is not None else 0)
        stream.synchronize()
        return self._out(self.od, self.oi)

    def plain(self, c, stream, id_offset=0):
        import torch
        torch.cuda.synchronize()
        c.search_device(self.q.data_ptr(), self.nq, self.k, self.pd.data_ptr(), self.pi.data_ptr(), id_offset=id_offset,
                        alive_ptr=self.a.data_ptr() if self.a is not None else 0, stream=stream.cuda_stream)
        stream.synchronize()
        return self._out(self.pd, self.pi)


def same(a, b, what):
    bad = SR.compare(a, b)
    assert not bad, f"{what}: {bad[:4]}"


def flat_ok(r, ans, id_offset, what):
    bad = fr.compare(r, ans[0], ans[1], id_offset)
    assert not bad, f"{what}: {len(bad)} problems: {bad[:4]}"


def bitmap(alive):
    bits = orc.pack_bits(alive)
    if len(alive) % 8:
        bits[-1] |= np.uint8((0xff << (len(alive) % 8)) & 0xff)   # bits past the last row must be ignored
    return bits


def rpath(path, dtype):
    return "scan" if path == S.PATH_SCAN else ("bf16" if dtype == S.BF16 else "tf32")


NQS = (1, 3, 7, 64, 1025)
KS = (1, 5, 7, 10, 64, "max")


# ------------------------------------------------------------------------------------------------------------------ world 1
@pytest.mark.parametrize("dtype", [S.F32, S.BF16])
@pytest.mark.parametrize("metric", [b2.L2, b2.IP, b2.COSINE])
def test_float_corpus_every_shape_equals_plain_search_and_the_reference(env, metric, dtype):
    comm, st = env
    rng = np.random.default_rng(10 * metric + dtype)
    n, d = 2100, 65
    y = rng.standard_normal((n, d)).astype(F32)
    xs = rng.standard_normal((max(NQS), d)).astype(F32)
    c = b2.Corpus(metric, d, dtype=dtype).append(y)
    refs = {}
    for a, nq in enumerate(NQS):
        for b, kk in enumerate(KS):
            path = (S.PATH_SCAN, S.PATH_TENSOR)[(a + b) % 2]
            k = kk if kk != "max" else (2048 if path == S.PATH_SCAN else 1024)
            off = BIG_OFFSET if (a + b) % 3 == 0 else 0
            c.set_path(path)
            call = Call(xs[:nq], k)
            got = call.sharded(comm, c, st, off)
            what = f"nq={nq} k={k} path={path} offset={off}"
            same(call.plain(c, st, off), got, what)
            key = (rpath(path, dtype), nq)
            if key not in refs:
                refs[key] = fr.reference(metric, fr.BF16 if dtype == S.BF16 else fr.F32, key[0], y, xs[:nq], 1)
            r = copy.copy(refs[key])
            r.k = k
            flat_ok(r, got, off, what)
    c.close()


@pytest.mark.parametrize("metric", [b2.HAMMING, b2.JACCARD])
def test_binary_corpus_every_shape_equals_plain_search_and_the_oracle(env, metric):
    comm, st = env
    rng = np.random.default_rng(metric)
    n, nbytes = 2100, 32
    y = rng.integers(0, 256, (n, nbytes), dtype=np.uint8)
    y[1500:1600] = y[100:200]                                   # equal rows: ties to the smaller id
    xs = rng.integers(0, 256, (max(NQS), nbytes), dtype=np.uint8)
    c = b2.Corpus(metric, nbytes * 8, dtype=S.BIN).append(y)
    for a, nq in enumerate(NQS):
        for b, kk in enumerate(KS):
            path = (S.PATH_SCAN, S.PATH_TENSOR)[(a + b) % 2]
            k = kk if kk != "max" else 1024
            off = BIG_OFFSET if (a + b) % 3 == 0 else 0
            c.set_path(path)
            call = Call(xs[:nq], k)
            got = call.sharded(comm, c, st, off)
            what = f"nq={nq} k={k} path={path} offset={off}"
            same(call.plain(c, st, off), got, what)
            do, io = orc.knn_binary(metric, xs[:nq], y, k)
            same((do, np.where(io >= 0, io + off, -1)), got, what + " vs the oracle")
    c.close()


@pytest.mark.parametrize("metric,dtype", [(b2.L2, S.F32), (b2.IP, S.BF16), (b2.COSINE, S.F32)])
def test_bitmaps_offsets_and_a_shard_shorter_than_k(env, metric, dtype):
    comm, st = env
    rng = np.random.default_rng(3 + metric)
    d = 40
    for n, k in ((2101, 64), (5, 10), (1, 7)):
        y = rng.standard_normal((n, d)).astype(F32)
        x = rng.standard_normal((7, d)).astype(F32)
        c = b2.Corpus(metric, d, dtype=dtype).append(y)
        for kind in (None, "dense", "sparse", "none"):
            alive = None if kind is None else {"dense": rng.random(n) < 0.9, "sparse": rng.random(n) < 0.01,
                                               "none": np.zeros(n, bool)}[kind]
            for path in (S.PATH_SCAN, S.PATH_TENSOR):
                c.set_path(path)
                r = fr.reference(metric, fr.BF16 if dtype == S.BF16 else fr.F32, rpath(path, dtype), y, x, k, alive=alive)
                for off in (0, BIG_OFFSET):
                    call = Call(x, k, bits=None if alive is None else bitmap(alive))
                    got = call.sharded(comm, c, st, off)
                    what = f"n={n} k={k} bitmap={kind} path={path} offset={off}"
                    same(call.plain(c, st, off), got, what)
                    flat_ok(r, got, off, what)
                    if kind == "none":
                        assert (got[1] == -1).all()
        c.close()


@pytest.mark.parametrize("dtype", [S.F32, S.BF16])
def test_graph_replays_equal_eager_calls(env, dtype):
    comm, st = env
    rng = np.random.default_rng(17)
    n, d = 3000, 64
    y = rng.standard_normal((n, d)).astype(F32)
    x = rng.standard_normal((7, d)).astype(F32)
    c = b2.Corpus(b2.L2, d, dtype=dtype).append(y)
    for path in (S.PATH_SCAN, S.PATH_TENSOR):
        c.set_path(path)
        call = Call(x, 5)                                        # nq * k = 35: odd
        eager = call.sharded(comm, c, st, BIG_OFFSET, use_graph=False)
        same(call.plain(c, st, BIG_OFFSET), eager, f"eager path={path}")
        cap0, rep0 = comm.graph_stats()
        same(eager, call.sharded(comm, c, st, BIG_OFFSET, use_graph=True), "first graph call")
        assert comm.graph_stats() == (cap0 + 1, rep0 + 1), "the first call captures and launches the graph"
        for i in range(3):
            same(eager, call.sharded(comm, c, st, BIG_OFFSET, use_graph=True), f"replay {i}")
        assert comm.graph_stats() == (cap0 + 1, rep0 + 4), "later calls replay"
        same(eager, call.sharded(comm, c, st, BIG_OFFSET, use_graph=False), "eager after replays")
        assert comm.graph_stats() == (cap0 + 1, rep0 + 4), "use_graph=0 neither captures nor replays"
        other = call.sharded(comm, c, st, 0, use_graph=True)    # another id_offset is another graph
        assert comm.graph_stats() == (cap0 + 2, rep0 + 5)
        same(call.plain(c, st, 0), other, "offset 0 graph")
        flat_ok(fr.reference(fr.L2, fr.BF16 if dtype == S.BF16 else fr.F32, rpath(path, dtype), y, x, 5), other, 0, "graph")
    c.close()


def _graph_call(comm, c, call, st, off=0, **kw):
    """A graph call checked against the eager plain search that follows it; returns (answer, captures it made)."""
    cap0, _ = comm.graph_stats()
    got = call.sharded(comm, c, st, off, use_graph=True, **kw)
    same(call.plain(c, st, off), got, f"graph call nq={call.nq} k={call.k}")
    return got, comm.graph_stats()[0] - cap0


@pytest.mark.parametrize("capacity", ["within", "past"])
@pytest.mark.parametrize("dtype", [S.F32, S.BF16])
def test_replay_after_an_append_sees_the_new_rows(env, dtype, capacity):
    comm, st = env
    rng = np.random.default_rng(23)
    n, d, nq = 4000, 64, 9
    y = to_bf16_values(rng.standard_normal((n, d)).astype(F32))
    x = to_bf16_values(rng.standard_normal((nq, d)).astype(F32))  # bf16 values: a bf16 copy of a query is the query
    c = b2.Corpus(b2.L2, d, dtype=dtype, capacity=n + nq if capacity == "within" else 0).append(y)
    for path in (S.PATH_SCAN, S.PATH_TENSOR):
        c.set_path(path)
        call = Call(x, 10)
        _graph_call(comm, c, call, st, BIG_OFFSET)
        _, caps = _graph_call(comm, c, call, st, BIG_OFFSET)
        assert caps == 0
        c.append(x)                                              # row n + j is query j's exact match
        got, caps = _graph_call(comm, c, call, st, BIG_OFFSET)
        assert caps == 1, "an append must invalidate the captured graph"
        assert (got[1][:, 0] == BIG_OFFSET + n + np.arange(nq)).all() and (got[0][:, 0] == 0).all(), got[1][:, :3]
        yy = np.concatenate([y, x])
        flat_ok(fr.reference(fr.L2, fr.BF16 if dtype == S.BF16 else fr.F32, rpath(path, dtype), yy, x, 10), got, BIG_OFFSET,
                "after append")
        c.close()
        c = b2.Corpus(b2.L2, d, dtype=dtype, capacity=n + nq if capacity == "within" else 0).append(y)
    c.close()


def test_replay_after_workspaces_grow(env):
    """Batch and k alternating on the same pointers; a large plain search between replays.  The communicator's all-gather
    buffers are sized by a larger call on another corpus first, so only the corpus' workspaces move."""
    comm, st = env
    rng = np.random.default_rng(31)
    n, d = 5000, 96
    y = rng.standard_normal((n, d)).astype(F32)
    x = rng.standard_normal((1025, d)).astype(F32)
    warm = b2.Corpus(b2.IP, d).append(y[:100])
    Call(x, 100).sharded(comm, warm, st, 0)
    warm.close()
    for dtype in (S.F32, S.BF16):
        c = b2.Corpus(b2.IP, d, dtype=dtype).append(y)
        call = Call(x, 10, nq=64, cap_k=100)
        r = {nq: fr.reference(fr.IP, fr.BF16 if dtype == S.BF16 else fr.F32, rpath(S.PATH_TENSOR, dtype), y, x[:nq], 1)
             for nq in (64, 1025)}
        c.set_path(S.PATH_TENSOR)
        caps = []
        for nq, k in ((64, 10), (64, 10), (1025, 10), (64, 10), (64, 100), (64, 10)):
            got, cp = _graph_call(comm, c, call, st, nq=nq, k=k)
            caps.append(cp)
            rr = copy.copy(r[nq])
            rr.k = k
            flat_ok(rr, got, 0, f"nq={nq} k={k}")
        assert caps[:4] == [1, 0, 1, 1], ("64 x 10 again after 1025 x 10 grew the query staging: a new capture", caps)
        _, caps = _graph_call(comm, c, call, st, nq=64, k=10)
        assert caps == 0
        c.search(x, 200)                                          # a large plain search grows the staging and the lists
        _, caps = _graph_call(comm, c, call, st, nq=64, k=10)
        assert caps == 1, "workspaces reallocated by a plain search: a new capture"
        c.close()


def test_replay_after_set_path(env):
    comm, st = env
    rng = np.random.default_rng(37)
    y = rng.standard_normal((3000, 64)).astype(F32)
    x = rng.standard_normal((9, 64)).astype(F32)
    c = b2.Corpus(b2.COSINE, 64, dtype=S.BF16).append(y).set_path(S.PATH_SCAN)
    call = Call(x, 10)
    _graph_call(comm, c, call, st)
    _graph_call(comm, c, call, st)
    c.set_path(S.PATH_TENSOR)
    cap0, _ = comm.graph_stats()
    got = call.sharded(comm, c, st, 0, use_graph=True)
    assert comm.graph_stats()[0] == cap0 + 1 and c.last_variant()[0] == S.KERNEL_GEMM_BF16, "the replay kept the old path"
    same(call.plain(c, st), got, "after set_path")
    flat_ok(fr.reference(fr.COSINE, fr.BF16, "bf16", y, x, 10), got, 0, "after set_path")
    c.close()


def test_replay_on_a_new_corpus_at_a_freed_address(env):
    comm, st = env
    rng = np.random.default_rng(41)
    d = 32
    x = rng.standard_normal((5, d)).astype(F32)
    call = Call(x, 7)
    recurred, last = 0, None
    for i in range(4):
        y = rng.standard_normal((1000, d)).astype(F32)
        c = b2.Corpus(b2.L2, d).append(y).set_path(S.PATH_SCAN)
        h = c._h.value
        got, caps = _graph_call(comm, c, call, st)
        assert caps == 1, "a new corpus is never replayed from another one's graph"
        flat_ok(fr.reference(fr.L2, fr.F32, "scan", y, x, 7), got, 0, "new corpus")
        c.close()
        recurred += h == last
        last = h
    NOTES["corpus handle address recurred after close"] = f"{recurred} of 3 times"


@pytest.mark.parametrize("use_graph", [False, True])
def test_host_entry_equals_the_device_entry(env, use_graph):
    comm, st = env
    rng = np.random.default_rng(43)
    for metric, dtype, d in ((b2.L2, S.F32, 100), (b2.IP, S.BF16, 64), (b2.HAMMING, S.BIN, 256), (b2.JACCARD, S.BIN, 128)):
        if dtype == S.BIN:
            y = rng.integers(0, 256, (3000, d // 8), dtype=np.uint8)
            x = rng.integers(0, 256, (7, d // 8), dtype=np.uint8)
        else:
            y = rng.standard_normal((3000, d)).astype(F32)
            x = rng.standard_normal((7, d)).astype(F32)
        c = b2.Corpus(metric, d, dtype=dtype).append(y)
        for k in (5, 64):
            dev = Call(x, k).sharded(comm, c, st, BIG_OFFSET)
            for _ in range(2):
                host = comm.sharded_corpus_search_host(c, x, k, BIG_OFFSET, st.cuda_stream, use_graph=use_graph)
                same(dev, host, f"metric={metric} dtype={dtype} k={k}")
        wrong = np.concatenate([x, x[:, :1]], axis=1)            # a row wider than the corpus: d + 1 (binary: d + 8)
        with pytest.raises(S.B200Error) as e:
            comm.sharded_corpus_search_host(c, wrong, 5, 0, st.cuda_stream, use_graph=use_graph)
        assert e.value.code == ERR_INVALID
        c.close()


@pytest.mark.parametrize("kind", ["IVFFLAT", "IVFPQ", "HNSWFLAT"])
def test_sharded_index_search_equals_the_index_search(env, kind, tmp_path):
    import torch
    comm, st = env
    rng = np.random.default_rng(47)
    n, d = 4000, 64
    y = (rng.standard_normal((24, d))[rng.integers(0, 24, n)] + 0.3 * rng.standard_normal((n, d))).astype(F32)
    x = (y[rng.integers(0, n, 7)] + 0.1 * rng.standard_normal((7, d))).astype(F32)
    params = {"IVFFLAT": "ncentroids=32, keep_raw=0", "IVFPQ": "ncentroids=32, M=8", "HNSWFLAT": "graph_degree=16"}[kind]
    sp = "ef_s=64" if kind == "HNSWFLAT" else "nprobe=8"
    ix = b2.VectorIndex(kind, b2.L2, d, params).build(y)
    q = _dev(x)
    for nq, k, off in ((7, 5, 0), (7, 5, BIG_OFFSET), (1, 7, BIG_OFFSET), (3, 64, 0)):
        outs = []
        for sharded in (True, False):
            od = torch.empty((nq, k), dtype=torch.float32, device="cuda")
            oi = torch.empty((nq, k), dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            if sharded:
                comm.sharded_index_search(ix, b2.L2, q.data_ptr(), nq, k, sp, od.data_ptr(), oi.data_ptr(), off, st.cuda_stream)
            else:
                ix.search_device(q.data_ptr(), nq, k, od.data_ptr(), oi.data_ptr(), params=sp, id_offset=off, stream=st.cuda_stream)
            st.synchronize()
            outs.append((od.cpu().numpy(), oi.cpu().numpy()))
        same(outs[1], outs[0], f"{kind} nq={nq} k={k} offset={off}")
        if kind == "IVFFLAT":                                     # keep_raw=0: the answer is the list scan's
            ix.save(tmp_path / "ix.b2ix")
            ref = R.reference_search(R.read_index(tmp_path / "ix.b2ix"), x[:nq], k, 8)
            dg, ig = outs[0]
            bad = R.compare(ref, dg, np.where(ig >= 0, ig - off, -1))
            assert not bad, bad[:4]
    od = torch.empty(35, dtype=torch.float32, device="cuda")
    oi = torch.empty(35, dtype=torch.int64, device="cuda")
    for wrong in (b2.IP, b2.COSINE):
        with pytest.raises(S.B200Error) as e:
            comm.sharded_index_search(ix, wrong, q.data_ptr(), 7, 5, "", od.data_ptr(), oi.data_ptr(), 0, st.cuda_stream)
        assert e.value.code == ERR_INVALID
    ix.close()


def test_gather_merge_host_and_allreduce_return_their_input(env):
    comm, _ = env
    rng = np.random.default_rng(53)
    for nq, k in ((1, 5), (7, 3), (64, 10)):
        dis = np.sort(rng.random((nq, k)).astype(F32), axis=1)[:, ::-1].copy()
        ids = rng.integers(0, 1 << 40, (nq, k))
        dis[:, k - 1:] = -np.inf
        ids[:, k - 1:] = -1
        od, oi = comm.gather_merge_host(dis, ids, True)
        same((dis, ids), (od, oi), f"nq={nq} k={k}")
    c = np.array([(1 << 40) + 1, 3, 0, (1 << 63) + 5], np.uint64)
    assert np.array_equal(comm.allreduce_sum_u64(c), c)


def test_local_buffers_are_aligned_for_odd_nq_k(env):
    """Runs no kernel: the ids block of the packed record must be 8-byte aligned whatever nq * k is."""
    comm, _ = env
    for nq, k in ((1, 5), (7, 3), (3, 7), (1025, 1), (64, 10)):
        pd, pi = C.c_void_p(), C.c_void_p()
        assert lib().b200_comm_local_buffers(comm._h, C.c_int64(nq), C.c_int(k), C.byref(pd), C.byref(pi)) == 0
        assert pi.value % 8 == 0, (nq, k, pd.value, pi.value)
        assert pi.value - pd.value >= nq * k * 4


def test_local_buffers_then_gather_merge(env):
    """The building blocks at odd nq * k: a plain search writes into the local buffers, gather_merge returns its answer."""
    import torch
    comm, st = env
    rng = np.random.default_rng(59)
    y = rng.standard_normal((2000, 48)).astype(F32)
    x = rng.standard_normal((3, 48)).astype(F32)
    c = b2.Corpus(b2.IP, 48).append(y)
    q = _dev(x)
    for nq, k in ((1, 5), (3, 7), (3, 64)):
        pd, pi = C.c_void_p(), C.c_void_p()
        assert lib().b200_comm_local_buffers(comm._h, C.c_int64(nq), C.c_int(k), C.byref(pd), C.byref(pi)) == 0
        torch.cuda.synchronize()
        c.search_device(q.data_ptr(), nq, k, pd.value, pi.value, id_offset=BIG_OFFSET, stream=st.cuda_stream)
        od = torch.empty((nq, k), dtype=torch.float32, device="cuda")
        oi = torch.empty((nq, k), dtype=torch.int64, device="cuda")
        assert lib().b200_comm_gather_merge(comm._h, C.c_int64(nq), C.c_int(k), C.c_int(1), C.c_void_p(od.data_ptr()),
                                            C.c_void_p(oi.data_ptr()), C.c_void_p(st.cuda_stream)) == 0
        st.synchronize()
        got = (od.cpu().numpy(), oi.cpu().numpy())
        same(Call(x[:nq], k).plain(c, st, BIG_OFFSET), got, f"nq={nq} k={k}")
        flat_ok(fr.reference(fr.IP, fr.F32, "scan" if nq < 5 else "tf32", y, x[:nq], k), got, BIG_OFFSET, f"nq={nq} k={k}")
    c.close()


# ------------------------------------------------------------------------------------------------------------------ world > 1
def _ranges(n, world, short_last=None):
    """Row ranges of the ranks: shard_range (remainder to the last ranks), or the last rank holding only `short_last` rows."""
    if short_last is None:
        return [shard_range(n, world, r) for r in range(world)]
    head = [shard_range(n - short_last, world - 1, r) for r in range(world - 1)]
    return head + [(n - short_last, n)]


def _multi_worker(rank, world, port, results):
    try:
        sys.path.insert(0, ROOT)
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(rank)
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        uid = [Comm.unique_id() if rank == 0 else None]
        dist.broadcast_object_list(uid, 0)
        comm = Comm(rank, world, uid[0])
        st = torch.cuda.Stream()
        problems = []

        def check(what, local, got, desc, ref=None):
            """local: this rank's plain shard answer (global ids); got: its sharded answer; ref: optional (r, offset) or
            (dis, ids) exact answer over all rows (checked on rank 0)."""
            allv = [None] * world
            dist.all_gather_object(allv, (local, got))
            if rank == 0:
                want = SR.merge([a[0] for a in allv], got[0].shape[1], desc)
                for r_, (_, g) in enumerate(allv):
                    bad = SR.compare(want, g)
                    if bad:
                        problems.append(f"{what} rank {r_}: {bad[:3]}")
                if ref is not None:
                    bad = fr.compare(ref[0], got[0], got[1], ref[1]) if isinstance(ref[0], fr.Reference) else SR.compare(ref, got)
                    if bad:
                        problems.append(f"{what} vs the reference of all rows: {bad[:3]}")

        rng = np.random.default_rng(0)
        # float data, unequal shards, odd nq * k, bitmaps, a shard shorter than k, graph replays
        n, d = 5003, 65
        y = rng.standard_normal((n, d)).astype(F32)
        x = rng.standard_normal((64, d)).astype(F32)
        for metric, dtype in ((b2.L2, S.F32), (b2.IP, S.BF16), (b2.COSINE, S.F32)):
            name = {b2.L2: "L2", b2.IP: "IP", b2.COSINE: "COS"}[metric]
            for short in (None, 3):
                lo, hi = _ranges(n, world, short)[rank]
                c = b2.Corpus(metric, d, dtype=dtype).append(y[lo:hi])
                for path in (S.PATH_SCAN, S.PATH_TENSOR):
                    c.set_path(path)
                    for nq, k, filt in ((7, 5, None), (64, 10, None), (3, 7, "drop last shard"), (1, 64, "ragged")):
                        alive = None
                        if filt == "drop last shard":
                            alive = np.ones(n, bool)
                            alive[_ranges(n, world, short)[-1][0]:] = False
                        elif filt == "ragged":
                            alive = np.random.default_rng(5).random(n) < 0.5
                        call = Call(x[:nq], k, bits=None if alive is None else bitmap(alive[lo:hi]))
                        for use_graph in (False, True, True):
                            got = call.sharded(comm, c, st, lo, use_graph=use_graph)
                            local = call.plain(c, st, lo)
                            r = fr.reference(metric, fr.BF16 if dtype == S.BF16 else fr.F32, rpath(path, dtype), y, x[:nq], k, alive=alive)
                            check(f"{name} short={short} path={path} nq={nq} k={k} filter={filt} graph={use_graph}", local, got,
                                  metric == b2.IP, (r, 0))
                c.close()
        # integer-valued data, rows duplicated across shards: ties to the smaller global id, exact distances
        n, d = 1001, 96
        y = rng.integers(-8, 9, (n, d)).astype(F32)
        lo0, hi0 = shard_range(n, world, 0)
        lo1, hi1 = shard_range(n, world, world - 1)
        y[lo1:lo1 + 50] = y[lo0:lo0 + 50]
        x = np.concatenate([y[lo0:lo0 + 5], rng.integers(-8, 9, (4, d))]).astype(F32)
        lo, hi = shard_range(n, world, rank)
        for metric, name in ((b2.L2, "L2"), (b2.IP, "IP")):
            for dtype in (S.F32, S.BF16):
                c = b2.Corpus(metric, d, dtype=dtype).append(y[lo:hi])
                for path in (S.PATH_SCAN, S.PATH_TENSOR):
                    c.set_path(path)
                    for k in (5, 64):
                        call = Call(x, k)
                        got = call.sharded(comm, c, st, lo, use_graph=True)
                        check(f"{name} integer dtype={dtype} path={path} k={k}", call.plain(c, st, lo), got, metric == b2.IP,
                              SR.integer_topk(metric, x, y, k))
                c.close()
        # a row-sharded index: each rank's own index over its rows
        n, d = 8000, 64
        y = rng.standard_normal((n, d)).astype(F32)
        x = rng.standard_normal((7, d)).astype(F32)
        lo, hi = shard_range(n, world, rank)
        ix = b2.VectorIndex("IVFFLAT", b2.L2, d, "ncentroids=16").build(y[lo:hi])
        q = _dev(x)
        outs = []
        for sharded in (True, False):
            od = torch.empty((7, 5), dtype=torch.float32, device="cuda")
            oi = torch.empty((7, 5), dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            if sharded:
                comm.sharded_index_search(ix, b2.L2, q.data_ptr(), 7, 5, "nprobe=4", od.data_ptr(), oi.data_ptr(), lo, st.cuda_stream)
            else:
                ix.search_device(q.data_ptr(), 7, 5, od.data_ptr(), oi.data_ptr(), params="nprobe=4", id_offset=lo, stream=st.cuda_stream)
            st.synchronize()
            outs.append((od.cpu().numpy(), oi.cpu().numpy()))
        check("L2 index", outs[1], outs[0], False)
        ix.close()
        # BM25-style host lists: scores descending, -inf / -1 unused slots, odd nq * k
        nq, k = 3, 7
        dis = np.sort(np.random.default_rng(100 + rank).random((nq, k)).astype(F32), axis=1)[:, ::-1].copy()
        ids = np.random.default_rng(200 + rank).integers(0, 1000, (nq, k)) + rank * 1000
        dis[:, k - 2 - rank % 2:] = -np.inf
        ids[:, k - 2 - rank % 2:] = -1
        check("bm25 host lists", (dis, ids), comm.gather_merge_host(dis, ids, True), True)
        # counters above 2^32
        got = comm.allreduce_sum_u64([(1 << 33) + rank, rank, 1 << 40])
        want = np.array([(1 << 33) * world + sum(range(world)), sum(range(world)), (1 << 40) * world], np.uint64)
        if not np.array_equal(got, want):
            problems.append(f"allreduce rank {rank}: {got} != {want}")
        dist.barrier()
        comm.close()
        dist.destroy_process_group()
        results.put((rank, problems))
    except BaseException:
        results.put((rank, [traceback.format_exc()[-3000:]]))


def _gpus():
    import torch
    return torch.cuda.device_count()


@pytest.mark.parametrize("world", [2, 4])
def test_multi_gpu_sharded_search_equals_the_merge_of_the_shards(world):
    if _gpus() < world:
        pytest.skip(f"needs {world} GPUs, {_gpus()} visible")
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    results = ctx.Queue()
    ps = [ctx.Process(target=_multi_worker, args=(r, world, port, results)) for r in range(world)]
    for p in ps:
        p.start()
    got = {}
    try:
        for _ in range(world):
            rank, problems = results.get(timeout=600)
            got[rank] = problems
    finally:
        for p in ps:
            p.join(60)
        for p in ps:
            if p.is_alive():
                p.terminate()
                p.join(30)
    assert sorted(got) == list(range(world)), got
    bad = [e for r in range(world) for e in got[r]]
    assert not bad, bad[:5]
    assert all(p.exitcode == 0 for p in ps), [p.exitcode for p in ps]
