"""myscaledb_b200 -- H100-native (sm_90a) engine for MyScaleDB's ANN / BM25 hot path.

The product is ``libb200search.so`` (hand-written CUDA behind the C ABI of
``include/b200_search.h``).  This package is the thin host-side mirror used by the
tests and the benchmark: ctypes bindings (``_lib``) and Python classes named after the
reference's operator surface (``search``).  There is no CPU fallback: importing works
anywhere, computing needs an sm_90 GPU and the built library.
"""
from . import _lib  # noqa: F401
from .search import (  # noqa: F401
    COSINE, HAMMING, IP, JACCARD, L2, METRIC_NAMES, B200Error, BM25Index, Corpus, VectorIndex, binary_knn, flat_knn, hybrid_fusion_batch, part_scan,
    topk_merge_device,
)

__all__ = ["Corpus", "VectorIndex", "BM25Index", "hybrid_fusion_batch", "flat_knn", "binary_knn", "part_scan", "topk_merge_device", "B200Error", "L2", "IP", "COSINE",
           "HAMMING", "JACCARD", "METRIC_NAMES"]
