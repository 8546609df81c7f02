"""Host-side partitioning of a table's parts across the GPUs of one box.

The reference treats every MergeTree part as an independent search unit and merges per-part
top-k lists by score (src/VectorIndex/Storages/MergeTreeSelectWithHybridSearchProcessor.cpp:1149-1241
-> MergeTreeBaseSearchManager.cpp:207-299).  Here a part (or an equal row range of a big part)
is pinned to one GPU; queries are broadcast; the only exchange is one all-gather of
[nq][k] (distance fp32, global row id int64) followed by one merge kernel.
"""
from __future__ import annotations

import ctypes as C


def shard_range(total_rows: int, world: int, rank: int, align: int = 1):
    """Row range [start, stop) of `rank`: equal shares rounded to `align`, remainder to the last ranks."""
    if world <= 0 or not (0 <= rank < world):
        raise ValueError("bad world / rank")
    units = total_rows // align
    base, extra = divmod(units, world)
    start_u = rank * base + min(rank, extra)
    stop_u = start_u + base + (1 if rank < extra else 0)
    start, stop = start_u * align, stop_u * align
    if rank == world - 1:
        stop = total_rows
    return start, stop


def gather_layout(world: int, nq: int, k: int):
    """Shapes of the all-gather buffers consumed by b200_topk_merge_device."""
    return (world, nq, k)


def assign_parts(part_rows, world: int):
    """Greedy size-balanced assignment of parts to GPUs (largest first). Returns list of lists of part indices."""
    order = sorted(range(len(part_rows)), key=lambda i: -part_rows[i])
    load = [0] * world
    out = [[] for _ in range(world)]
    for i in order:
        g = min(range(world), key=lambda j: load[j])
        out[g].append(i)
        load[g] += part_rows[i]
    return out


# ----------------------------------------------------------------------------------------------
# Text side: BM25 scores must not depend on how documents are spread over GPUs.  The reference sums
# total_num_docs / total_num_tokens / doc_freq over parts before scoring
# (ReadWithHybridSearch::getStatisticForTextSearch, src/VectorIndex/Processors/ReadWithHybridSearch.cpp:89-209,
# BM25InfoInDataParts.cpp:40-94); across GPUs that is ONE all-reduce(sum) of a small int64 vector per batch.
# ----------------------------------------------------------------------------------------------
def bm25_stats_layout(n_fields: int, query_terms, fields):
    """Order of the counters in the exchanged vector: [total_docs, tokens(field 0..n_fields-1), df(field, term) ...]."""
    keys = [("docs",)] + [("tokens", f) for f in range(n_fields)]
    keys += [("df", f, t) for f in fields for t in query_terms]
    return keys


def bm25_local_stats(index, n_fields: int, query_terms, fields):
    """int64 counters of ONE shard's BM25 index (anything with total_docs / total_tokens(f) / doc_freq(t, f))."""
    total_docs = index.total_docs() if callable(index.total_docs) else index.total_docs
    out = [int(total_docs)] + [int(index.total_tokens(f)) for f in range(n_fields)]
    out += [int(index.doc_freq(t, f)) for f in fields for t in query_terms]
    return out


def bm25_global_stats(summed, n_fields: int, query_terms, fields):
    """Summed counter vector -> the `stats` dict BM25Index.search(..., stats=) takes (table-wide N, tokens, df)."""
    summed = [int(v) for v in summed]
    stats = {"total_docs": summed[0], "total_tokens": {f: summed[1 + f] for f in range(n_fields)}, "doc_freq": {}}
    pos = 1 + n_fields
    for f in fields:
        for t in query_terms:
            stats["doc_freq"][(f, t)] = summed[pos]
            pos += 1
    return stats


# ----------------------------------------------------------------------------------------------
# The communicator below the C ABI (csrc/comm.cu): NCCL all-gather of per-shard top-k + merge kernel, BM25 counter
# all-reduce, whole sharded steps (optionally one CUDA graph per step).  Python only moves the 128-byte NCCL id around.
# ----------------------------------------------------------------------------------------------
class Comm:
    def __init__(self, rank: int, world: int, unique_id: bytes, nccl_lib_path: str | None = None):
        from ._lib import lib
        from .search import _check
        self._h = C.c_void_p()
        self.rank, self.world = rank, world
        _check(lib().b200_comm_create(nccl_lib_path.encode() if nccl_lib_path else None, unique_id, C.c_int(rank), C.c_int(world),
                                      C.byref(self._h)))

    @staticmethod
    def unique_id(nccl_lib_path: str | None = None) -> bytes:
        from ._lib import lib
        from .search import _check
        buf = C.create_string_buffer(128)
        _check(lib().b200_comm_unique_id(nccl_lib_path.encode() if nccl_lib_path else None, buf))
        return buf.raw

    @classmethod
    def from_torch_distributed(cls, device):
        """One communicator rank per torch.distributed rank: rank 0 makes the id, a broadcast carries it."""
        import torch
        import torch.distributed as dist
        rank, world = dist.get_rank(), dist.get_world_size()
        t = torch.zeros(128, dtype=torch.uint8, device=device)
        if rank == 0:
            t.copy_(torch.frombuffer(bytearray(cls.unique_id()), dtype=torch.uint8))
        dist.broadcast(t, 0)
        return cls(rank, world, bytes(t.cpu().numpy().tobytes()))

    def sharded_corpus_search(self, corpus, q_ptr: int, nq: int, k: int, out_dis_ptr: int, out_ids_ptr: int, id_offset: int, stream: int,
                              use_graph: bool = True, alive_ptr: int = 0):
        from ._lib import lib
        from .search import _check
        _check(lib().b200_sharded_corpus_search(self._h, corpus._h, C.c_void_p(q_ptr), C.c_int64(nq), C.c_int(k), C.c_void_p(alive_ptr or None),
                                                C.c_int64(id_offset), C.c_void_p(out_dis_ptr), C.c_void_p(out_ids_ptr), C.c_void_p(stream),
                                                C.c_int(1 if use_graph else 0)))

    def sharded_corpus_search_host(self, corpus, queries, k: int, id_offset: int, stream: int, use_graph: bool = True, out=None):
        import numpy as np
        from ._lib import lib
        from .search import BIN, _check
        binary = corpus.dtype == BIN   # query rows are bytes [nq][d / 8]
        q = np.ascontiguousarray(queries, np.uint8 if binary else np.float32)
        nq, d = q.shape[0], q.shape[1] * (8 if binary else 1)
        dis, ids = out if out is not None else (np.empty((nq, k), np.float32), np.empty((nq, k), np.int64))
        _check(lib().b200_sharded_corpus_search_host(self._h, corpus._h, q.ctypes.data_as(C.c_void_p), C.c_int64(nq), C.c_int(d), C.c_int(k),
                                                     C.c_int64(id_offset), dis.ctypes.data_as(C.c_void_p), ids.ctypes.data_as(C.c_void_p),
                                                     C.c_void_p(stream), C.c_int(1 if use_graph else 0)))
        return dis, ids

    def sharded_index_search(self, index, metric: int, q_ptr: int, nq: int, k: int, params: str, out_dis_ptr: int, out_ids_ptr: int,
                             id_offset: int, stream: int, alive_ptr: int = 0):
        from ._lib import lib
        from .search import _check
        _check(lib().b200_sharded_index_search(self._h, index._h, C.c_int(metric), C.c_void_p(q_ptr), C.c_int64(nq), C.c_int(k), params.encode(),
                                               C.c_void_p(alive_ptr or None), C.c_int64(id_offset), C.c_void_p(out_dis_ptr),
                                               C.c_void_p(out_ids_ptr), C.c_void_p(stream)))

    def graph_stats(self):
        """(captures, replays) of the sharded corpus search's CUDA graphs on this communicator."""
        from ._lib import lib
        from .search import _check
        cap, rep = C.c_int64(), C.c_int64()
        _check(lib().b200_comm_graph_stats(self._h, C.byref(cap), C.byref(rep)))
        return cap.value, rep.value

    def gather_merge_host(self, dis, ids, descending: bool):
        """Per-shard [nq][k] lists held on the host (BM25 top-k) -> the table-wide top-k on every rank."""
        import numpy as np
        from ._lib import lib
        from .search import _check
        dis = np.ascontiguousarray(dis, np.float32)
        ids = np.ascontiguousarray(ids, np.int64)
        nq, k = dis.shape
        od, oi = np.empty_like(dis), np.empty_like(ids)
        _check(lib().b200_comm_gather_merge_host(self._h, dis.ctypes.data_as(C.c_void_p), ids.ctypes.data_as(C.c_void_p), C.c_int64(nq),
                                                 C.c_int(k), C.c_int(1 if descending else 0), od.ctypes.data_as(C.c_void_p),
                                                 oi.ctypes.data_as(C.c_void_p)))
        return od, oi

    def allreduce_sum_u64(self, counters):
        """In-place sum over the ranks (BM25 table-wide statistics); counters: list / array of non-negative ints."""
        import numpy as np
        from ._lib import lib
        from .search import _check
        a = np.ascontiguousarray(counters, np.uint64).copy()
        _check(lib().b200_comm_allreduce_sum_u64(self._h, a.ctypes.data_as(C.c_void_p), C.c_int64(a.size)))
        return a

    def close(self):
        if self._h:
            from ._lib import lib
            lib().b200_comm_free(self._h)
            self._h = C.c_void_p()
