"""Host-side mirror of the reference's operator surface for the hot path, over the C ABI.

Names follow the reference:
  flat_knn      <-> VectorIndex::tryBruteForceSearch / VIWithColumnInPart::searchWithoutIndex
                    (src/VectorIndex/Common/BruteForceSearch.h:63, VIWithDataPart.h:342)
  part_scan     <-> MergeTreeVSManager::vectorScanWithoutIndex + searchWrapper
                    (src/VectorIndex/Storages/MergeTreeVSManager.cpp:960-1679)
  Corpus.search <-> Search::VectorIndex(FLAT)::search via VIWithColumnInPart::search
                    (src/VectorIndex/Common/VIWithDataPart.cpp:858-957)
  topk_merge_device <-> MergeTreeBaseSearchManager::getTotalTopSearchResultImpl
                    (src/VectorIndex/Storages/MergeTreeBaseSearchManager.cpp:207-299)
All arithmetic happens in libb200search.so on the GPU; numpy is used for buffers only.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import lib

L2, IP, COSINE, HAMMING, JACCARD = 0, 1, 2, 3, 4
METRIC_NAMES = {"L2": L2, "IP": IP, "COSINE": COSINE, "HAMMING": HAMMING, "JACCARD": JACCARD}
F32, BF16, BIN = 0, 1, 2
# b200_corpus_set_path codes and b200_corpus_last_variant kernel ids
PATH_AUTO, PATH_SCAN, PATH_TENSOR, PATH_CG1, PATH_CG2, PATH_CG2_MC2, PATH_CG2_MC4, PATH_TS = range(8)
KERNEL_SCAN, KERNEL_GEMM_BF16, KERNEL_GEMM_TS, KERNEL_GEMM_TF32X3, KERNEL_GEMM_B1 = 1, 2, 3, 4, 5


class B200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"b200 error {code}: {msg}")
        self.code = code


def _check(rc):
    if rc != 0:
        raise B200Error(rc, lib().b200_last_error().decode(errors="replace"))


def _p(a, t):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


def _bits(a):
    return None if a is None else np.ascontiguousarray(a, np.uint8)


def flat_knn(metric, x, y, k, alive_bits=None):
    x = np.ascontiguousarray(x, np.float32)
    y = np.ascontiguousarray(y, np.float32)
    nx, d = x.shape
    ny = y.shape[0]
    dis = np.empty((nx, k), np.float32)
    ids = np.empty((nx, k), np.int64)
    ab = _bits(alive_bits)
    _check(lib().b200_flat_knn(C.c_int(metric), _p(x, C.c_float), C.c_int64(nx), _p(y, C.c_float), C.c_int64(ny),
                               C.c_int(d), C.c_int(k), _p(ab, C.c_uint8), _p(dis, C.c_float), _p(ids, C.c_int64)))
    return dis, ids


def binary_knn(metric, x, y, k, alive_bits=None):
    x = np.ascontiguousarray(x, np.uint8)
    y = np.ascontiguousarray(y, np.uint8)
    nx, nb = x.shape
    ny = y.shape[0]
    dis = np.empty((nx, k), np.float32)
    ids = np.empty((nx, k), np.int64)
    ab = _bits(alive_bits)
    _check(lib().b200_binary_knn(C.c_int(metric), _p(x, C.c_uint8), C.c_int64(nx), _p(y, C.c_uint8), C.c_int64(ny),
                                 C.c_int(nb), C.c_int(k), _p(ab, C.c_uint8), _p(dis, C.c_float), _p(ids, C.c_int64)))
    return dis, ids


def part_scan(metric, x, y, k, block_rows=8192, row_exists=None, filter_bits=None):
    binary = metric in (HAMMING, JACCARD)
    if binary:
        x = np.ascontiguousarray(x, np.uint8)
        y = np.ascontiguousarray(y, np.uint8)
        d = x.shape[1] * 8
    else:
        x = np.ascontiguousarray(x, np.float32)
        y = np.ascontiguousarray(y, np.float32)
        d = x.shape[1]
    nx, ny = x.shape[0], y.shape[0]
    dis = np.empty((nx, k), np.float32)
    ids = np.empty((nx, k), np.int64)
    re_ = None if row_exists is None else np.ascontiguousarray(row_exists, np.uint8)
    fb = _bits(filter_bits)
    _check(lib().b200_part_scan(C.c_int(metric), x.ctypes.data_as(C.c_void_p), C.c_int64(nx),
                                y.ctypes.data_as(C.c_void_p), C.c_int64(ny), C.c_int(d), C.c_int(k),
                                C.c_int64(block_rows), _p(re_, C.c_uint8), _p(fb, C.c_uint8), _p(dis, C.c_float),
                                _p(ids, C.c_int64)))
    return dis, ids


class Corpus:
    """Device-resident FLAT index / cached part column."""

    def __init__(self, metric, d, dtype=F32, capacity=0):
        self._h = C.c_void_p()
        self.metric, self.d, self.dtype = metric, d, dtype
        _check(lib().b200_corpus_create(C.c_int(metric), C.c_int(dtype), C.c_int(d), C.c_int64(capacity), C.byref(self._h)))

    @classmethod
    def borrowed(cls, handle: int, metric, d, dtype=F32):
        """Non-owning view of a corpus held by the residency cache (cache_get): never freed by this wrapper."""
        self = cls.__new__(cls)
        self._h = C.c_void_p(handle)
        self.metric, self.d, self.dtype = metric, d, dtype
        self.close = lambda: None
        return self

    def append(self, rows):
        rows = np.ascontiguousarray(rows, np.uint8 if self.dtype == BIN else np.float32)
        _check(lib().b200_corpus_append(self._h, rows.ctypes.data_as(C.c_void_p), C.c_int64(rows.shape[0])))
        return self

    def adopt_device(self, data_ptr: int, n: int):
        _check(lib().b200_corpus_adopt_device(self._h, C.c_void_p(data_ptr), C.c_int64(n)))
        return self

    def set_path(self, path: int):
        _check(lib().b200_corpus_set_path(self._h, C.c_int(path)))
        return self

    def set_prefilter(self, mode: int):
        """Pre-filtered exact search: 0 auto, 1 never (full masked scan), 2 whenever the compact copy fits the budget."""
        _check(lib().b200_corpus_set_prefilter(self._h, C.c_int(mode)))
        return self

    def last_rows_scored(self):
        """Rows the last search scored: the corpus size after a full scan, the kept rows after a pre-filtered one."""
        n = C.c_int64()
        _check(lib().b200_corpus_last_rows_scored(self._h, C.byref(n)))
        return n.value

    def last_variant(self):
        """(kernel, cta_group, pairs_per_cluster, grid) of the last search: KERNEL_SCAN / _GEMM_BF16 / _GEMM_TS / _GEMM_TF32X3 /
        _GEMM_B1 (binary rows on the tensor cores)."""
        kern, cg, mc, grid = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        _check(lib().b200_corpus_last_variant(self._h, C.byref(kern), C.byref(cg), C.byref(mc), C.byref(grid)))
        return kern.value, cg.value, mc.value, grid.value

    @property
    def size(self):
        n = C.c_int64()
        _check(lib().b200_corpus_size(self._h, C.byref(n)))
        return n.value

    def search(self, queries, k, alive_bits=None):
        q = np.ascontiguousarray(queries, np.uint8 if self.dtype == BIN else np.float32)
        nq = q.shape[0]
        dis = np.empty((nq, k), np.float32)
        ids = np.empty((nq, k), np.int64)
        ab = _bits(alive_bits)
        _check(lib().b200_corpus_search(self._h, q.ctypes.data_as(C.POINTER(C.c_float)), C.c_int64(nq), C.c_int(k),
                                        _p(ab, C.c_uint8), _p(dis, C.c_float), _p(ids, C.c_int64)))
        return dis, ids

    def search_device(self, q_ptr: int, nq: int, k: int, out_dis_ptr: int, out_ids_ptr: int, id_offset=0,
                      alive_ptr: int = 0, stream: int = 0):
        _check(lib().b200_corpus_search_device(self._h, C.c_void_p(q_ptr), C.c_int64(nq), C.c_int(k),
                                               C.c_void_p(alive_ptr or None), C.c_int64(id_offset),
                                               C.c_void_p(out_dis_ptr), C.c_void_p(out_ids_ptr),
                                               C.c_void_p(stream or None)))

    def enable_timing(self, on=True):
        _check(lib().b200_corpus_enable_timing(self._h, C.c_int(1 if on else 0)))

    def kernel_time(self, reset=False):
        """(total ms, launches) of the dominant kernel since the last reset (CUDA events)."""
        ms, n = C.c_double(), C.c_int64()
        _check(lib().b200_corpus_kernel_time(self._h, C.c_int(1 if reset else 0), C.byref(ms), C.byref(n)))
        return ms.value, n.value

    def close(self):
        if self._h:
            lib().b200_corpus_free(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def topk_merge_device(dis_ptr, ids_ptr, n_lists, nq, k, descending, out_dis_ptr, out_ids_ptr, stream=0):
    _check(lib().b200_topk_merge_device(C.c_void_p(dis_ptr), C.c_void_p(ids_ptr), C.c_int(n_lists), C.c_int64(nq),
                                        C.c_int(k), C.c_int(1 if descending else 0), C.c_void_p(out_dis_ptr),
                                        C.c_void_p(out_ids_ptr), C.c_void_p(stream or None)))


def topk_merge_device_strided(dis_ptr, ids_ptr, n_lists, dis_stride, ids_stride, nq, k, descending, out_dis_ptr,
                              out_ids_ptr, stream=0):
    _check(lib().b200_topk_merge_device_strided(C.c_void_p(dis_ptr), C.c_void_p(ids_ptr), C.c_int(n_lists),
                                                C.c_int64(dis_stride), C.c_int64(ids_stride), C.c_int64(nq), C.c_int(k),
                                                C.c_int(1 if descending else 0), C.c_void_p(out_dis_ptr),
                                                C.c_void_p(out_ids_ptr), C.c_void_p(stream or None)))


def topk_merge_device_ex(dis_ptr, ids_ptr, n_lists, dis_stride, ids_stride, nq, k_in, k, descending, tie_mode, out_dis_ptr,
                         out_ids_ptr, out_list_ptr=0, stream=0):
    """getTotalTopSearchResultImpl on device; tie_mode 1 reproduces the reference's multimap order (and reports the
    source list / part of every winner in out_list)."""
    _check(lib().b200_topk_merge_device_ex(C.c_void_p(dis_ptr), C.c_void_p(ids_ptr), C.c_int(n_lists), C.c_int64(dis_stride),
                                           C.c_int64(ids_stride), C.c_int64(nq), C.c_int(k_in), C.c_int(k),
                                           C.c_int(1 if descending else 0), C.c_int(tie_mode), C.c_void_p(out_dis_ptr),
                                           C.c_void_p(out_ids_ptr), C.c_void_p(out_list_ptr or None), C.c_void_p(stream or None)))


def thread_last_rows_scored() -> int:
    """Rows the last corpus search on this thread scored (one-shot calls, exact index paths): the corpus size after a full
    scan, the kept rows after a pre-filtered one."""
    n = C.c_int64()
    _check(lib().b200_thread_last_rows_scored(C.byref(n)))
    return n.value


def launch_count(reset=False) -> int:
    return int(lib().b200_launch_count(C.c_int(1 if reset else 0)))


def device_bytes() -> int:
    """Bytes of device memory the library holds (every index, corpus, workspace and per-thread scratch)."""
    f = lib().b200_device_bytes
    f.restype = C.c_int64
    return int(f())


class BM25Index:
    """Per-part BM25 index resident in HBM (mirror of the TantivyIndexStore calls,
    src/Storages/MergeTree/TantivyIndexStore.cpp:742-998)."""

    def __init__(self, n_fields: int = 1):
        self._h = C.c_void_p()
        self.n_fields = n_fields
        _check(lib().b200_bm25_create(C.c_uint32(n_fields), C.byref(self._h)))

    def add_doc(self, row_id: int, texts):
        """texts: per field a str or a list[str] (Array(String) column)."""
        _check(lib().b200_bm25_add_doc(self._h, C.c_uint64(row_id)))
        if isinstance(texts, str):
            texts = [texts]
        for f, t in enumerate(texts):
            for piece in ([t] if isinstance(t, str) else t):
                _check(lib().b200_bm25_add_text(self._h, C.c_uint32(f), piece.encode()))

    def commit(self):
        _check(lib().b200_bm25_commit(self._h))
        return self

    def save(self, path):
        _check(lib().b200_bm25_save(self._h, str(path).encode()))

    @classmethod
    def load(cls, path, n_fields=1):
        self = cls.__new__(cls)
        self._h = C.c_void_p()
        self.n_fields = n_fields
        _check(lib().b200_bm25_load(str(path).encode(), C.byref(self._h)))
        return self

    @property
    def total_docs(self):
        v = C.c_uint64()
        _check(lib().b200_bm25_total_docs(self._h, C.byref(v)))
        return v.value

    def total_tokens(self, field=0):
        v = C.c_uint64()
        _check(lib().b200_bm25_total_tokens(self._h, C.c_uint32(field), C.byref(v)))
        return v.value

    def doc_freq(self, term, field=0):
        v = C.c_uint64()
        _check(lib().b200_bm25_doc_freq(self._h, C.c_uint32(field), term.encode(), C.byref(v)))
        return v.value

    _qt_tls = __import__("threading").local()   # per-thread scratch of query_terms (ctypes drops the GIL during the call)

    @staticmethod
    def query_terms(sentence):
        tls = BM25Index._qt_tls
        raw = sentence.encode()
        # every distinct term is written, NUL-terminated; a term is at most 3x the bytes it came from (an invalid byte
        # decodes to U+FFFD), so 4 bytes per input byte always suffice
        need = max(4096, 4 * len(raw) + 16)
        if getattr(tls, "cap", 0) < need:
            tls.buf, tls.cap = (C.create_string_buffer(need), C.c_uint32()), need
        buf, n = tls.buf
        _check(lib().b200_bm25_query_terms(raw, buf, C.c_size_t(tls.cap), C.byref(n)))
        out, off = [], 0
        base = C.addressof(buf)
        for _ in range(n.value):
            t = C.string_at(base + off)
            out.append(t.decode())
            off += len(t) + 1
        return out

    def search_batch(self, sentences, topk, fields=(0,), alive_bits=None, operator_or=True, stats=None):
        nq = len(sentences)
        arr = (C.c_char_p * nq)(*[s.encode() for s in sentences])
        f = np.array(fields, np.uint32)
        rows = np.empty((nq, topk), np.uint64)
        scores = np.empty((nq, topk), np.float32)
        counts = np.zeros(nq, np.uint32)
        st_docs, st_tok, st_df = 0, None, None
        if stats is not None:
            st_docs = int(stats["total_docs"])
            st_tok = np.zeros(self.n_fields, np.uint64)
            for fi, v in stats["total_tokens"].items():
                st_tok[fi] = v
            st_df = np.zeros((nq, len(fields), 64), np.uint64)
            for qi, sent in enumerate(sentences):
                for ti, t in enumerate(self.query_terms(sent)[:64]):
                    for fi, fld in enumerate(fields):
                        st_df[qi, fi, ti] = stats["doc_freq"].get((fld, t), 0)
        ab = _bits(alive_bits)
        _check(lib().b200_bm25_search_batch(self._h, arr, C.c_int64(nq), _p(f, C.c_uint32), C.c_uint32(len(fields)),
                                            C.c_uint32(topk), _p(ab, C.c_uint8), C.c_int(0 if ab is None else 1),
                                            C.c_int(1 if operator_or else 0), C.c_uint64(st_docs), _p(st_tok, C.c_uint64),
                                            _p(st_df, C.c_uint64), _p(rows, C.c_uint64), _p(scores, C.c_float),
                                            _p(counts, C.c_uint32)))
        return [(rows[q, :counts[q]].copy(), scores[q, :counts[q]].copy()) for q in range(nq)]

    def last_timing(self):
        km, cm, po = C.c_double(), C.c_double(), C.c_uint64()
        _check(lib().b200_bm25_last_timing(self._h, C.byref(km), C.byref(cm), C.byref(po)))
        return dict(kernel_ms=km.value, call_ms=cm.value, postings=po.value)

    def search(self, sentence, topk, **kw):
        return self.search_batch([sentence], topk, **kw)[0]

    def close(self):
        if self._h:
            lib().b200_bm25_free(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def hybrid_fusion_batch(fusion_type, vec_lists, txt_lists, top_k, fusion_weight=0.5, fusion_k=60, vector_scan_direction=1):
    """vec_lists / txt_lists: per query a list of (shard, part, label, score), globally ordered.
    Returns per query a list of (shard, part, label, fused_score)."""
    nq = len(vec_lists)
    assert len(txt_lists) == nq
    vs = max([len(v) for v in vec_lists] + [1])
    ts = max([len(t) for t in txt_lists] + [1])

    def pack(lists, stride):
        sh = np.zeros((nq, stride), np.uint32); pa = np.zeros((nq, stride), np.uint64)
        la = np.zeros((nq, stride), np.uint64); sc = np.zeros((nq, stride), np.float32)
        cnt = np.zeros(nq, np.uint32)
        for q, lst in enumerate(lists):
            cnt[q] = len(lst)
            for i, (a, b, c, d) in enumerate(lst):
                sh[q, i], pa[q, i], la[q, i], sc[q, i] = a, b, c, d
        return sh, pa, la, sc, cnt
    v = pack(vec_lists, vs)
    t = pack(txt_lists, ts)
    o_sh = np.zeros((nq, top_k), np.uint32); o_pa = np.zeros((nq, top_k), np.uint64)
    o_la = np.zeros((nq, top_k), np.uint64); o_sc = np.zeros((nq, top_k), np.float32); o_cnt = np.zeros(nq, np.uint32)
    ft = {"rsf": 0, "rrf": 1}[fusion_type.lower()]
    _check(lib().b200_hybrid_fusion_batch(
        C.c_int(ft), C.c_int64(nq), _p(v[0], C.c_uint32), _p(v[1], C.c_uint64), _p(v[2], C.c_uint64), _p(v[3], C.c_float),
        _p(v[4], C.c_uint32), C.c_int64(vs), _p(t[0], C.c_uint32), _p(t[1], C.c_uint64), _p(t[2], C.c_uint64),
        _p(t[3], C.c_float), _p(t[4], C.c_uint32), C.c_int64(ts), C.c_float(fusion_weight), C.c_uint64(fusion_k),
        C.c_int(vector_scan_direction), C.c_uint32(top_k), _p(o_sh, C.c_uint32), _p(o_pa, C.c_uint64), _p(o_la, C.c_uint64),
        _p(o_sc, C.c_float), _p(o_cnt, C.c_uint32)))
    return [[(int(o_sh[q, i]), int(o_pa[q, i]), int(o_la[q, i]), float(o_sc[q, i])) for i in range(o_cnt[q])]
            for q in range(nq)]


def hybrid_fusion_arrays(fusion_type, vec_ids, vec_scores, txt_ids, txt_scores, top_k, fusion_weight=0.5, fusion_k=60,
                         vector_scan_direction=1):
    """Array form of hybrid_fusion_batch for one shard / part space: [nq][kv] vector ids (int64, -1 = unused slot) + distances and
    [nq][kt] text ids + bm25 scores, both globally ordered.  Returns ([nq][top_k] ids (-1 padded), [nq][top_k] fused scores, counts)."""
    vec_ids = np.ascontiguousarray(vec_ids, np.int64); txt_ids = np.ascontiguousarray(txt_ids, np.int64)
    nq, kv = vec_ids.shape
    kt = txt_ids.shape[1]
    v_cnt = (vec_ids >= 0).sum(1).astype(np.uint32); t_cnt = (txt_ids >= 0).sum(1).astype(np.uint32)
    v_la = np.where(vec_ids >= 0, vec_ids, 0).astype(np.uint64); t_la = np.where(txt_ids >= 0, txt_ids, 0).astype(np.uint64)
    v_sc = np.ascontiguousarray(vec_scores, np.float32); t_sc = np.ascontiguousarray(np.where(txt_ids >= 0, txt_scores, 0), np.float32)
    v_sh = np.zeros((nq, kv), np.uint32); v_pa = np.zeros((nq, kv), np.uint64)
    t_sh = np.zeros((nq, kt), np.uint32); t_pa = np.zeros((nq, kt), np.uint64)
    o_sh = np.zeros((nq, top_k), np.uint32); o_pa = np.zeros((nq, top_k), np.uint64)
    o_la = np.zeros((nq, top_k), np.uint64); o_sc = np.zeros((nq, top_k), np.float32); o_cnt = np.zeros(nq, np.uint32)
    ft = {"rsf": 0, "rrf": 1}[fusion_type.lower()]
    _check(lib().b200_hybrid_fusion_batch(
        C.c_int(ft), C.c_int64(nq), _p(v_sh, C.c_uint32), _p(v_pa, C.c_uint64), _p(v_la, C.c_uint64), _p(v_sc, C.c_float),
        _p(v_cnt, C.c_uint32), C.c_int64(kv), _p(t_sh, C.c_uint32), _p(t_pa, C.c_uint64), _p(t_la, C.c_uint64),
        _p(t_sc, C.c_float), _p(t_cnt, C.c_uint32), C.c_int64(kt), C.c_float(fusion_weight), C.c_uint64(fusion_k),
        C.c_int(vector_scan_direction), C.c_uint32(top_k), _p(o_sh, C.c_uint32), _p(o_pa, C.c_uint64), _p(o_la, C.c_uint64),
        _p(o_sc, C.c_float), _p(o_cnt, C.c_uint32)))
    ids = np.where(np.arange(top_k)[None, :] < o_cnt[:, None], o_la.astype(np.int64), -1)
    return ids, o_sc, o_cnt


class VectorIndex:
    """Mirror of Search::VectorIndex as driven by VIWithColumnInPart (build / search / computeTopDistanceSubset,
    src/VectorIndex/Common/VIWithDataPart.cpp:131, :926, :838-856).  type: FLAT, IVFFLAT, IVFSQ, IVFPQ, MSTG, SCANN, HNSW*, and
    for HAMMING / JACCARD the binary types BINARYFLAT, BINARYIVF, BINARYHNSW, BINARYMSTG, whose rows and queries are uint8
    [n][d / 8] (d in bits)."""

    def __init__(self, index_type, metric, d, params=""):
        self._h = C.c_void_p()
        self.d = d
        self._binary = metric in (HAMMING, JACCARD)
        _check(lib().b200_index_create(index_type.encode(), C.c_int(metric), C.c_int(d), params.encode(), C.byref(self._h)))
        self._last_nq = 0

    def _rows(self, a):
        return np.ascontiguousarray(a, np.uint8 if self._binary else np.float32)

    def build(self, rows):
        rows = self._rows(rows)
        _check(lib().b200_index_build(self._h, _p(rows, C.c_float), C.c_int64(rows.shape[0])))
        return self

    # streamed build (VIPartReader: train block, then add blocks)
    def reserve(self, total_rows):
        _check(lib().b200_index_reserve(self._h, C.c_int64(total_rows)))
        return self

    def train(self, rows):
        rows = self._rows(rows)
        _check(lib().b200_index_train(self._h, _p(rows, C.c_float), C.c_int64(rows.shape[0])))
        return self

    def add(self, rows):
        rows = self._rows(rows)
        _check(lib().b200_index_add(self._h, _p(rows, C.c_float), C.c_int64(rows.shape[0])))
        return self

    def train_device(self, ptr: int, n: int):
        _check(lib().b200_index_train_device(self._h, C.c_void_p(ptr), C.c_int64(n)))
        return self

    def add_device(self, ptr: int, n: int):
        _check(lib().b200_index_add_device(self._h, C.c_void_p(ptr), C.c_int64(n)))
        return self

    def finalize(self):
        _check(lib().b200_index_finalize(self._h))
        return self

    def search_device(self, q_ptr: int, nq: int, k: int, out_dis_ptr: int, out_ids_ptr: int, params="", first_stage_only=False,
                      id_offset=0, alive_ptr: int = 0, stream: int = 0):
        _check(lib().b200_index_search_device(self._h, C.c_void_p(q_ptr), C.c_int64(nq), C.c_int(k), params.encode(),
                                              C.c_int(1 if first_stage_only else 0), C.c_void_p(alive_ptr or None),
                                              C.c_int64(id_offset), C.c_void_p(out_dis_ptr), C.c_void_p(out_ids_ptr),
                                              C.c_void_p(stream or None)))
        self._last_nq = nq

    def enable_timing(self, on=True):
        _check(lib().b200_index_enable_timing(self._h, C.c_int(1 if on else 0)))

    def last_scan(self, reset=False):
        rows, rb, items, ms, nl = C.c_int64(), C.c_int64(), C.c_int64(), C.c_double(), C.c_int64()
        _check(lib().b200_index_last_scan(self._h, C.byref(rows), C.byref(rb), C.byref(items), C.byref(ms), C.byref(nl),
                                          C.c_int(1 if reset else 0)))
        return dict(rows_streamed=rows.value, payload_row_bytes=rb.value, work_items=items.value, kernel_ms=ms.value, launches=nl.value)

    def last_probe(self):
        """(lists each query of the last search probed, int32 [nq]; whether the filter_probe exact rule answered it).
        filter_probe=1: p_q per query; other list searches: nprobe; exact passes: 0."""
        n = self._last_nq
        out = np.zeros(n, np.int32)
        ex = C.c_int()
        _check(lib().b200_index_last_probe(self._h, _p(out, C.c_int32), C.c_int64(n), C.byref(ex)))
        return out, bool(ex.value)

    def last_coarse(self):
        """Coarse-probe path of the last search: 1 FMA scan, 2 tensor cores (3xTF32), 3 keys + select, 0 none ran."""
        p = C.c_int()
        _check(lib().b200_index_last_coarse(self._h, C.byref(p)))
        return p.value

    def graph(self):
        """graph_degree indexes: the neighbour graph, uint32 [n][D] (0xFFFFFFFF = empty slot); None without a graph."""
        deg = C.c_int()
        _check(lib().b200_index_graph(self._h, None, C.c_int64(0), C.byref(deg)))
        if deg.value == 0:
            return None
        n = self.info()["n"]
        out = np.zeros((n, deg.value), np.uint32)
        _check(lib().b200_index_graph(self._h, _p(out, C.c_uint32), C.c_int64(n), C.byref(deg)))
        return out

    def last_seeds(self):
        """Seed ids of the last search when it walked the graph, int64 [nq][S] (negative = none); None otherwise."""
        s = C.c_int()
        _check(lib().b200_index_last_seeds(self._h, None, C.c_int64(0), C.byref(s)))
        if s.value == 0:
            return None
        out = np.zeros((self._last_nq, s.value), np.int64)
        _check(lib().b200_index_last_seeds(self._h, _p(out, C.c_int64), C.c_int64(out.size), C.byref(s)))
        return out

    def train_loss(self):
        """aq_threshold indexes: (eta, float64 [1 + iterations] mean anisotropic loss of the training sample after the k-means
        codebooks, then after each iteration).  B200Error for an index not trained with the key."""
        eta, n = C.c_double(), C.c_int()
        _check(lib().b200_index_train_loss(self._h, C.byref(eta), None, C.c_int(0), C.byref(n)))
        out = np.zeros(n.value, np.float64)
        _check(lib().b200_index_train_loss(self._h, C.byref(eta), _p(out, C.c_double), C.c_int(n.value), C.byref(n)))
        return eta.value, out

    def opq(self):
        """opq=1 indexes: (R float32 [d][d], y = x.R; float64 [1 + opq_iters] mean PQ loss of the training sample at R = I,
        then after each alternation; empty for a loaded index).  B200Error for an index without the key or without a rotation."""
        n = C.c_int()
        _check(lib().b200_index_opq(self._h, None, None, C.c_int(0), C.byref(n)))
        r = np.zeros((self.d, self.d), np.float32)
        loss = np.zeros(n.value, np.float64)
        _check(lib().b200_index_opq(self._h, _p(r, C.c_float), _p(loss, C.c_double), C.c_int(n.value), C.byref(n)))
        return r, loss

    def phase_ms(self):
        a = (C.c_double * 5)()
        _check(lib().b200_index_phase_ms(self._h, a))
        return dict(zip(("coarse", "plan", "scan", "merge", "refine"), [round(v, 4) for v in a]))

    def list_sizes(self):
        nl = self.info()["nlist"]
        out = np.zeros(nl, np.uint32)
        _check(lib().b200_index_list_sizes(self._h, _p(out, C.c_uint32), C.c_int(nl)))
        return out

    def memory_bytes(self):
        b = C.c_uint64()
        _check(lib().b200_index_memory_bytes(self._h, C.byref(b)))
        return b.value

    def host_memory_bytes(self):
        """Pinned host bytes of the fp32 re-rank rows in host placement (keep_raw=2), else 0; memory_bytes() counts HBM only."""
        b = C.c_uint64()
        _check(lib().b200_index_host_memory_bytes(self._h, C.byref(b)))
        return b.value

    def set_raw_placement(self, placement: int):
        """Move a finalized index's fp32 re-rank rows to HBM (1) or pinned host memory (2)."""
        _check(lib().b200_index_set_raw_placement(self._h, C.c_int(placement)))
        return self

    def info(self):
        n, nl, m, ivf = C.c_int64(), C.c_int(), C.c_int(), C.c_int()
        _check(lib().b200_index_info(self._h, C.byref(n), C.byref(nl), C.byref(m), C.byref(ivf)))
        return dict(n=n.value, nlist=nl.value, m=m.value, uses_ivf=bool(ivf.value))

    def search(self, queries, k, params="", first_stage_only=False, alive_bits=None):
        q = self._rows(queries)
        nq = q.shape[0]
        dis = np.empty((nq, k), np.float32)
        ids = np.empty((nq, k), np.int64)
        nc = C.c_int64()
        ab = _bits(alive_bits)
        _check(lib().b200_index_search(self._h, _p(q, C.c_float), C.c_int64(nq), C.c_int(k), params.encode(),
                                       C.c_int(1 if first_stage_only else 0), _p(ab, C.c_uint8), _p(dis, C.c_float),
                                       _p(ids, C.c_int64), C.byref(nc)))
        self.last_num_candidates = nc.value
        self._last_nq = nq
        return dis, ids

    def save(self, path):
        _check(lib().b200_index_save(self._h, str(path).encode()))

    @classmethod
    def load(cls, path, d, metric=L2):
        self = cls.__new__(cls)
        self._h = C.c_void_p()
        self.d = d
        self._binary = metric in (HAMMING, JACCARD)
        self._last_nq = 0
        _check(lib().b200_index_load(str(path).encode(), C.byref(self._h)))
        return self

    def refine(self, queries, cand_ids, k):
        q = self._rows(queries)
        c = np.ascontiguousarray(cand_ids, np.int64)
        nq = q.shape[0]
        dis = np.empty((nq, k), np.float32)
        ids = np.empty((nq, k), np.int64)
        _check(lib().b200_index_refine(self._h, _p(q, C.c_float), C.c_int64(nq), _p(c, C.c_int64), C.c_int64(c.shape[1]),
                                       C.c_int(k), _p(dis, C.c_float), _p(ids, C.c_int64)))
        return dis, ids

    def close(self):
        if self._h:
            lib().b200_index_free(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def bitmap_and(a, b, nbits):
    a, b = np.ascontiguousarray(a, np.uint8), np.ascontiguousarray(b, np.uint8)
    out = np.zeros((nbits + 7) // 8, np.uint8)
    _check(lib().b200_bitmap_and(_p(a, C.c_uint8), _p(b, C.c_uint8), C.c_int64(nbits), _p(out, C.c_uint8)))
    return out


def real_bitmap(filter_bits, n_new_rows, inverted_row_ids_map, inverted_row_sources_map, own_id, total_vec):
    f = np.ascontiguousarray(filter_bits, np.uint8)
    ids = np.ascontiguousarray(inverted_row_ids_map, np.uint64)
    src = np.ascontiguousarray(inverted_row_sources_map, np.uint8)
    out = np.zeros((total_vec + 7) // 8, np.uint8)
    _check(lib().b200_real_bitmap(_p(f, C.c_uint8), C.c_int64(n_new_rows), _p(ids, C.c_uint64), _p(src, C.c_uint8),
                                  C.c_uint32(own_id), C.c_int64(total_vec), _p(out, C.c_uint8)))
    return out


def remap_labels(row_ids_map, labels):
    m = np.ascontiguousarray(row_ids_map, np.uint64)
    l = np.ascontiguousarray(labels, np.int64).copy()
    _check(lib().b200_remap_labels(_p(m, C.c_uint64), C.c_int64(m.size), _p(l, C.c_int64), C.c_int64(l.size)))
    return l


def transfer_to_old_row_ids(new_ids, new_dis, inverted_row_ids_map, inverted_row_sources_map, own_id):
    ids = np.ascontiguousarray(new_ids, np.int64); dis = np.ascontiguousarray(new_dis, np.float32)
    m = np.ascontiguousarray(inverted_row_ids_map, np.uint64); src = np.ascontiguousarray(inverted_row_sources_map, np.uint8)
    o_i = np.empty(ids.size, np.int64); o_d = np.empty(ids.size, np.float32); n = C.c_int64()
    _check(lib().b200_transfer_to_old_row_ids(_p(ids, C.c_int64), _p(dis, C.c_float), C.c_int64(ids.size), _p(m, C.c_uint64),
                                              _p(src, C.c_uint8), C.c_int64(m.size), C.c_uint32(own_id), _p(o_i, C.c_int64),
                                              _p(o_d, C.c_float), C.byref(n)))
    return o_i[:n.value], o_d[:n.value]


# --------------------------------------------------------------------------------------------------
# HBM residency cache (the device-side VICacheManager): keys are CacheKey strings; see include/b200_search.h
# --------------------------------------------------------------------------------------------------
CACHE_CORPUS, CACHE_INDEX, CACHE_BM25, CACHE_OPAQUE = 0, 1, 2, 3
_DELETER = C.CFUNCTYPE(None, C.c_void_p)


class CacheMiss(KeyError):
    pass


def cache_set_capacity(nbytes: int):
    _check(lib().b200_cache_set_capacity(C.c_uint64(nbytes)))


def cache_get(key: str):
    """-> (handle address, kind); raises CacheMiss.  The entry stays pinned until cache_release(key)."""
    h, kind = C.c_void_p(), C.c_int()
    rc = lib().b200_cache_get(key.encode(), C.byref(h), C.byref(kind))
    if rc == 6:
        raise CacheMiss(key)
    _check(rc)
    return h.value, kind.value


def cache_put(key: str, obj, nbytes: int = None):
    """Hands a Corpus / VectorIndex / BM25Index to the cache (which then owns the device object) and pins it.
    Returns the resident handle address (the existing one when the key was already cached; obj then stays the caller's)."""
    kind = CACHE_CORPUS if isinstance(obj, Corpus) else CACHE_INDEX if isinstance(obj, VectorIndex) else CACHE_BM25
    if nbytes is None:
        b = C.c_uint64()
        if kind == CACHE_CORPUS:
            _check(lib().b200_corpus_memory_bytes(obj._h, C.byref(b)))
        elif kind == CACHE_INDEX:
            _check(lib().b200_index_memory_bytes(obj._h, C.byref(b)))
        nbytes = b.value
    res = C.c_void_p()
    _check(lib().b200_cache_put(key.encode(), C.c_int(kind), obj._h, C.c_uint64(nbytes), C.byref(res)))
    if res.value == (obj._h.value if isinstance(obj._h, C.c_void_p) else obj._h):
        obj._h = C.c_void_p()  # ownership moved to the cache: the wrapper must not free it
    return res.value


def cache_put_opaque(key: str, handle: int, nbytes: int, deleter):
    """deleter: a _DELETER(ctypes callback) kept alive by the caller."""
    res = C.c_void_p()
    _check(lib().b200_cache_put_opaque(key.encode(), C.c_void_p(handle), C.c_uint64(nbytes), deleter, C.byref(res)))
    return res.value


def cache_release(key: str, handle: int | None = None):
    """Drop one pin.  Pass the handle address get / put returned when a key may have been expired and put again."""
    if handle is None:
        _check(lib().b200_cache_release(key.encode()))
    else:
        _check(lib().b200_cache_release_handle(key.encode(), C.c_void_p(handle)))


def cache_expire(key: str):
    rc = lib().b200_cache_expire(key.encode())
    if rc == 6:
        raise CacheMiss(key)
    _check(rc)


def cache_expire_prefix(prefix: str) -> int:
    n = C.c_int64()
    _check(lib().b200_cache_expire_prefix(prefix.encode(), C.byref(n)))
    return n.value


def cache_stats() -> dict:
    v = [C.c_uint64() for _ in range(6)]
    _check(lib().b200_cache_stats(*[C.byref(x) for x in v]))
    return dict(zip(("capacity", "used", "items", "hits", "misses", "evictions"), (x.value for x in v)))
