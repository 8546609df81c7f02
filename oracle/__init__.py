"""CPU oracle for the MyScaleDB ANN / BM25 hot path -- TEST INFRASTRUCTURE ONLY.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import this package.  The product
(``myscaledb_b200``) never does; ``tests/test_boundary.py`` greps for that.

Thin ctypes wrappers over ``oracle/liboracle.so`` (``vs_oracle.c``,
``bm25_oracle.c``, ``cpu_baseline.c``).  Each C function cites the reference
file:line it restates.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle.so")

L2, IP, COSINE, HAMMING, JACCARD = 0, 1, 2, 3, 4
METRICS = {"L2": L2, "IP": IP, "COSINE": COSINE, "HAMMING": HAMMING, "JACCARD": JACCARD}


def build(force: bool = False) -> str:
    srcs = [os.path.join(_HERE, f) for f in ("vs_oracle.c", "bm25_oracle.c", "cpu_baseline.c")]
    stale = force or not os.path.exists(_LIB_PATH) or any(
        os.path.getmtime(s) > os.path.getmtime(_LIB_PATH) for s in srcs
    )
    if stale:
        subprocess.check_call(["make", "-C", _HERE, "-B", "liboracle.so"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.orc_bm25_create.restype = C.c_void_p
        _lib.orc_bm25_total_docs.restype = C.c_uint64
        _lib.orc_bm25_total_tokens.restype = C.c_uint64
        _lib.orc_bm25_doc_freq.restype = C.c_uint64
        _lib.orc_bm25_search.restype = C.c_uint32
        _lib.orc_bm25_new_doc.restype = C.c_uint32
        _lib.orc_bm25_postings.restype = C.c_uint32
        _lib.orc_bm25_doc_len.restype = C.c_uint32
        _lib.orc_bm25_id_to_fieldnorm.restype = C.c_uint32
        _lib.orc_merge_parts.restype = C.c_int64
        _lib.orc_hybrid_fusion.restype = C.c_int64
    return _lib


def _p(a, t):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def pack_bits(mask) -> np.ndarray:
    """bool[n] -> LSB-first u8 bitmap (DenseBitmap::get_bitmap layout)."""
    return np.packbits(np.asarray(mask, dtype=bool), bitorder="little")


def knn_flat(metric, x, y, k, alive=None):
    """tryBruteForceSearch<FloatVector> (L2 / IP).  Returns (dis[nx,k], ids[nx,k])."""
    x, y = _f32(x), _f32(y)
    nx, d = x.shape
    ny = y.shape[0]
    dis = np.empty((nx, k), np.float32)
    ids = np.empty((nx, k), np.int64)
    lib().orc_knn_flat(C.c_int(metric), _p(x, C.c_float), C.c_int64(nx), _p(y, C.c_float), C.c_int64(ny), C.c_int(d),
                       C.c_int(k), _p(alive, C.c_uint8), _p(dis, C.c_float), _p(ids, C.c_int64))
    return dis, ids


def search_without_index(metric, x, y, k, alive=None):
    """VIWithColumnInPart::searchWithoutIndex<FloatVector> (adds cosine)."""
    x, y = _f32(x).copy(), _f32(y).copy()
    nx, d = x.shape
    ny = y.shape[0]
    dis = np.empty((nx, k), np.float32)
    ids = np.empty((nx, k), np.int64)
    lib().orc_search_without_index(C.c_int(metric), _p(x, C.c_float), C.c_int64(nx), _p(y, C.c_float), C.c_int64(ny),
                                   C.c_int(d), C.c_int(k), _p(alive, C.c_uint8), _p(dis, C.c_float),
                                   _p(ids, C.c_int64))
    return dis, ids


def knn_binary(metric, x, y, k, alive=None):
    """tryBruteForceSearch<BinaryVector>.  x,y: u8[n, nbytes].  Hamming distances are
    returned as float *values* (the reference's int32-in-float bits decoded)."""
    x = np.ascontiguousarray(x, np.uint8)
    y = np.ascontiguousarray(y, np.uint8)
    nx, nb = x.shape
    ny = y.shape[0]
    dis = np.empty((nx, k), np.float32)
    ids = np.empty((nx, k), np.int64)
    lib().orc_knn_binary(C.c_int(metric), _p(x, C.c_uint8), C.c_int64(nx), _p(y, C.c_uint8), C.c_int64(ny), C.c_int(nb),
                         C.c_int(k), _p(alive, C.c_uint8), _p(dis, C.c_float), _p(ids, C.c_int64))
    if metric == HAMMING:
        raw = dis.view(np.int32)
        dis = np.where(ids >= 0, raw.astype(np.float32), np.float32(np.finfo(np.float32).max))
    return dis, ids


def part_scan(metric, x, y, k, block_rows=8192, row_exists=None, filter_bits=None):
    """MergeTreeVSManager::vectorScanWithoutIndex + searchWrapper over one part."""
    binary = metric in (HAMMING, JACCARD)
    if binary:
        x = np.ascontiguousarray(x, np.uint8)
        y = np.ascontiguousarray(y, np.uint8)
        d = x.shape[1] * 8
    else:
        x, y = _f32(x), _f32(y)
        d = x.shape[1]
    nx, ny = x.shape[0], y.shape[0]
    dis = np.empty((nx, k), np.float32)
    ids = np.empty((nx, k), np.int64)
    re = None if row_exists is None else np.ascontiguousarray(row_exists, np.uint8)
    lib().orc_part_scan(C.c_int(metric), x.ctypes.data_as(C.c_void_p), C.c_int64(nx), y.ctypes.data_as(C.c_void_p),
                        C.c_int64(ny), C.c_int(d), C.c_int(k), C.c_int64(block_rows), _p(re, C.c_uint8),
                        _p(filter_bits, C.c_uint8), _p(dis, C.c_float), _p(ids, C.c_int64))
    return dis, ids


def merge_parts(score, part, label, top_k, desc):
    """MergeTreeBaseSearchManager::getTotalTopSearchResultImpl."""
    score = _f32(score)
    part = np.ascontiguousarray(part, np.int64)
    label = np.ascontiguousarray(label, np.int64)
    n = score.shape[0]
    os_, op, ol = np.empty(top_k, np.float32), np.empty(top_k, np.int64), np.empty(top_k, np.int64)
    c = lib().orc_merge_parts(_p(score, C.c_float), _p(part, C.c_int64), _p(label, C.c_int64), C.c_int64(n),
                              C.c_int64(top_k), C.c_int(1 if desc else 0), _p(os_, C.c_float), _p(op, C.c_int64),
                              _p(ol, C.c_int64))
    return os_[:c], op[:c], ol[:c]


def hybrid_fusion(fusion_type, vec, txt, top_k, fusion_weight=0.5, fusion_k=60, vector_scan_direction=1):
    """RankFusion / RelativeScoreFusion + hybridSearch ordering.
    vec / txt: lists of (shard, part, label, score) already globally ordered."""
    def cols(lst):
        # one exact column per field: labels go up to 2^64 - 1, beyond what a float64 holds exactly
        return (np.array([int(r[0]) for r in lst], np.uint32), np.array([int(r[1]) for r in lst], np.uint64),
                np.array([int(r[2]) for r in lst], np.uint64), np.array([r[3] for r in lst], np.float32))
    vs, vp, vl, vsc = cols(vec)
    ts, tp, tl, tsc = cols(txt)
    o_s, o_p, o_l, o_sc = (np.empty(top_k, np.uint32), np.empty(top_k, np.uint64), np.empty(top_k, np.uint64),
                           np.empty(top_k, np.float32))
    ft = {"rsf": 0, "rrf": 1}[fusion_type.lower()]
    c = lib().orc_hybrid_fusion(C.c_int(ft), _p(vs, C.c_uint32), _p(vp, C.c_uint64), _p(vl, C.c_uint64),
                                _p(vsc, C.c_float), C.c_int64(len(vec)), _p(ts, C.c_uint32), _p(tp, C.c_uint64),
                                _p(tl, C.c_uint64), _p(tsc, C.c_float), C.c_int64(len(txt)), C.c_float(fusion_weight),
                                C.c_uint64(fusion_k), C.c_int(vector_scan_direction), C.c_int64(top_k),
                                _p(o_s, C.c_uint32), _p(o_p, C.c_uint64), _p(o_l, C.c_uint64), _p(o_sc, C.c_float))
    return [(int(o_s[i]), int(o_p[i]), int(o_l[i]), float(o_sc[i])) for i in range(c)]


def knn_flat_parts(metric, x, y, k, n_parts):
    """Timed CPU baseline: one thread per part, blocked SIMD kernel inside (cpu_baseline.c)."""
    x, y = _f32(x), _f32(y)
    nx, d = x.shape
    ny = y.shape[0]
    dis = np.empty((nx, k), np.float32)
    ids = np.empty((nx, k), np.int64)
    lib().orc_knn_flat_parts(C.c_int(metric), _p(x, C.c_float), C.c_int64(nx), _p(y, C.c_float), C.c_int64(ny),
                             C.c_int(d), C.c_int(k), C.c_int(n_parts), _p(dis, C.c_float), _p(ids, C.c_int64))
    return dis, ids


def knn_flat_simd(metric, x, y, k):
    """Small-batch CPU arm: faiss' nx < 20 form (exact differences, SIMD, one thread), cpu_baseline.c."""
    x, y = _f32(x), _f32(y)
    nx, d = x.shape
    ny = y.shape[0]
    dis = np.empty((nx, k), np.float32)
    ids = np.empty((nx, k), np.int64)
    lib().orc_knn_flat_simd(C.c_int(metric), _p(x, C.c_float), C.c_int64(nx), _p(y, C.c_float), C.c_int64(ny), C.c_int(d), C.c_int(k),
                            _p(dis, C.c_float), _p(ids, C.c_int64))
    return dis, ids


def blas_path():
    """OpenBLAS shipped inside numpy's wheel (numpy.libs/libscipy_openblas64_*.so), or None."""
    import glob
    hits = glob.glob(os.path.join(os.path.dirname(np.__file__), "..", "numpy.libs", "libscipy_openblas64_*.so"))
    return hits[0] if hits else None


def knn_flat_parts_blas(metric, x, y, k, n_parts):
    """Timed CPU baseline, Faiss BLAS form: one single-threaded sgemm stream per part (cpu_baseline.c).
    Returns None when no OpenBLAS could be loaded."""
    p = blas_path()
    if p is None or lib().orc_blas_load(p.encode()) != 0:
        return None
    x, y = _f32(x), _f32(y)
    nx, d = x.shape
    ny = y.shape[0]
    dis = np.empty((nx, k), np.float32)
    ids = np.empty((nx, k), np.int64)
    rc = lib().orc_knn_flat_parts_blas(C.c_int(metric), _p(x, C.c_float), C.c_int64(nx), _p(y, C.c_float), C.c_int64(ny),
                                       C.c_int(d), C.c_int(k), C.c_int(n_parts), _p(dis, C.c_float), _p(ids, C.c_int64))
    return (dis, ids) if rc == 0 else None


class BM25Index:
    """In-memory per-part inverted index with tantivy-0.21 BM25 semantics (bm25_oracle.c)."""

    def __init__(self, n_fields: int = 1):
        self._l = lib()
        self.n_fields = n_fields
        self._h = C.c_void_p(self._l.orc_bm25_create(C.c_uint32(n_fields)))

    def __del__(self):
        try:
            self._l.orc_bm25_free(self._h)
        except Exception:
            pass

    def add_doc(self, row_id: int, texts):
        """texts: per field either a str or a list[str] (Array(String) column)."""
        self._l.orc_bm25_new_doc(self._h, C.c_uint64(row_id))
        if isinstance(texts, str):
            texts = [texts]
        for f, t in enumerate(texts):
            for piece in ([t] if isinstance(t, str) else t):
                self._l.orc_bm25_add_text(self._h, C.c_uint32(f), piece.encode())

    @property
    def total_docs(self):
        return int(self._l.orc_bm25_total_docs(self._h))

    def total_tokens(self, field=0):
        return int(self._l.orc_bm25_total_tokens(self._h, C.c_uint32(field)))

    def doc_freq(self, term: str, field=0):
        return int(self._l.orc_bm25_doc_freq(self._h, C.c_uint32(field), term.encode()))

    def doc_len(self, doc: int, field=0):
        return int(self._l.orc_bm25_doc_len(self._h, C.c_uint32(field), C.c_uint32(doc)))

    def postings(self, term: str, field=0):
        df = self.doc_freq(term, field)
        docs = np.empty(max(df, 1), np.uint32)
        tfs = np.empty(max(df, 1), np.uint32)
        self._l.orc_bm25_postings(self._h, C.c_uint32(field), term.encode(), _p(docs, C.c_uint32), _p(tfs, C.c_uint32),
                                  C.c_uint32(df))
        return docs[:df], tfs[:df]

    @staticmethod
    def query_terms(sentence: str):
        buf = C.create_string_buffer(64 * 48)
        n = lib().orc_bm25_query_terms(sentence.encode(), buf)
        return [buf.raw[i * 48:(i + 1) * 48].split(b"\0", 1)[0].decode() for i in range(n)]

    def search(self, sentence, topk, fields=(0,), alive=None, operator_or=True, stats=None):
        """stats: None or dict(total_docs=int, total_tokens={field:int}, doc_freq={(field,term):int})."""
        fields_a = np.array(fields, np.uint32)
        out_row = np.empty(topk, np.uint64)
        out_score = np.empty(topk, np.float32)
        st_docs, st_tok, st_df = 0, None, None
        if stats is not None:
            st_docs = int(stats["total_docs"])
            st_tok = np.zeros(self.n_fields, np.uint64)
            for f, v in stats["total_tokens"].items():
                st_tok[f] = v
            terms = self.query_terms(sentence)
            st_df = np.zeros(len(fields) * 64, np.uint64)
            for fi, f in enumerate(fields):
                for ti, t in enumerate(terms):
                    st_df[fi * 64 + ti] = stats["doc_freq"].get((f, t), 0)
        n = self._l.orc_bm25_search(self._h, sentence.encode(), _p(fields_a, C.c_uint32), C.c_uint32(len(fields)),
                                    C.c_uint32(topk), _p(alive, C.c_uint8), C.c_int(0 if alive is None else 1),
                                    C.c_int(1 if operator_or else 0), C.c_uint64(st_docs), _p(st_tok, C.c_uint64),
                                    _p(st_df, C.c_uint64), _p(out_row, C.c_uint64), _p(out_score, C.c_float))
        return out_row[:n].copy(), out_score[:n].copy()


def fieldnorm_to_id(n: int) -> int:
    return int(lib().orc_bm25_fieldnorm_to_id(C.c_uint32(n)))


def id_to_fieldnorm(i: int) -> int:
    return int(lib().orc_bm25_id_to_fieldnorm(C.c_int(i)))
