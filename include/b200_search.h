/*
 * b200_search.h -- C ABI of libb200search.so, the H100-native (sm_90a) engine for
 * MyScaleDB's ANN / BM25 hot path.
 *
 * This is the drop-in boundary: plain pointers and sizes only, no C++/torch types.
 * Each entry point names the reference interface it replaces (paths relative to
 * /root/reference/src).  INTEGRATION.md shows the C++ shim a MyScaleDB maintainer
 * adds on the ClickHouse side (namespace Search:: / TANTIVY::ffi_* forwarding here).
 *
 * Conventions
 *   - every function returns B200_OK (0) or an error code; b200_last_error() gives the
 *     thread-local message (the reference's libraries throw SearchIndexException /
 *     return {result, error{is_error,message}}; the C++ shim re-throws, VICommon.h:75-104);
 *   - all entry points are re-entrant: ClickHouse calls them from one ThreadPool worker
 *     per part (MergeTreeSelectWithHybridSearchProcessor.cpp:1212-1241);
 *   - float vectors are row-major fp32 [n][d]; binary vectors row-major bytes [n][d/8];
 *   - alive / filter bitmaps are LSB-first bytes, bit=1 => row may be returned
 *     (Search::DenseBitmap::get_bitmap(), MergeTreeTextSearchManager.cpp:191-194);
 *   - results: out_dis[nq*k], out_ids[nq*k], best first; unfilled slots id = -1
 *     (faiss heap convention the callers test with `ids > -1`, MergeTreeVSManager.cpp:469-488);
 *   - tie rule: better score, then smaller row id (SURVEY.md 8a);
 *   - there is NO CPU fallback: without a CUDA device every compute call fails with
 *     B200_ERR_NO_DEVICE.
 */
#ifndef B200_SEARCH_H
#define B200_SEARCH_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_OK 0
#define B200_ERR_INVALID 1     /* bad argument */
#define B200_ERR_CUDA 2        /* CUDA runtime / driver failure */
#define B200_ERR_UNSUPPORTED 3 /* valid request this build does not implement */
#define B200_ERR_NO_DEVICE 4   /* no sm_90 device visible */
#define B200_ERR_NOMEM 5
#define B200_ERR_NOT_FOUND 6   /* cache miss */

/* Search::Metric (MergeTreeVSManager.cpp:1560-1578) */
#define B200_METRIC_L2 0
#define B200_METRIC_IP 1
#define B200_METRIC_COSINE 2
#define B200_METRIC_HAMMING 3
#define B200_METRIC_JACCARD 4

/* device storage type of a resident corpus */
#define B200_DTYPE_F32 0
#define B200_DTYPE_BF16 1
#define B200_DTYPE_BIN 2

const char *b200_last_error(void);
const char *b200_version(void);
int b200_device_count(int *out_n);
int b200_set_device(int device);

/* ------------------------------------------------------------------------------------
 * Brute force from host buffers.
 * Replaces VectorIndex::tryBruteForceSearch<T> (VectorIndex/Common/BruteForceSearch.h:63-111)
 * as called by VIWithColumnInPart::searchWithoutIndex<T> (VectorIndex/Common/VIWithDataPart.h:342-382):
 * L2 = squared L2 ascending, IP descending, COSINE = normalise both (skip rows with
 * sum(x^2) < FLT_EPSILON) -> IP -> 1 - ip.  x, y are NOT modified.
 * ---------------------------------------------------------------------------------- */
int b200_flat_knn(int metric, const float *x, int64_t nx, const float *y, int64_t ny, int d, int k,
                  const uint8_t *alive_bits /*nullable*/, float *out_dis, int64_t *out_ids);

/* Binary vectors: HAMMING (faiss::hammings_knn_mc) / JACCARD (jaccard_knn),
 * BruteForceSearch.h:94-110.  Distances are returned as float VALUES (the reference
 * writes int32 Hamming distances into the float buffer, :99; the shim re-encodes).
 * Binary corpora (these calls, binary b200_part_scan and B200_DTYPE_BIN corpora) have two kernels that return the same
 * bytes: a popcount scan, and for rows of a multiple of 16 bytes (d % 128 == 0 bits) a tensor-core kernel (wgmma .b1 AND +
 * popcount) that auto-selection uses from a few queries per batch up (see b200_corpus_set_path).  Both return the same
 * ids and distances. */
int b200_binary_knn(int metric, const uint8_t *x, int64_t nx, const uint8_t *y, int64_t ny, int nbytes, int k,
                    const uint8_t *alive_bits /*nullable*/, float *out_dis, int64_t *out_ids);

/* Whole-part brute force with the semantics of MergeTreeVSManager::vectorScanWithoutIndex<T>
 * + searchWrapper<T> (VectorIndex/Storages/MergeTreeVSManager.cpp:960-1679): per-mark
 * blocks merged with "earlier block wins ties", lightweight-delete mask row_exists
 * (1 byte per row, 0 = deleted, :1435-1460), PREWHERE filter bitmap (:1042-1330), and the
 * IP initial value numeric_limits<float>::min() (:1030-1037: IP scores <= FLT_MIN are never
 * returned).  The part column is DMA'd to HBM once and scanned in one pass; block_rows only
 * documents the mark size (results are independent of it under the tie rule).
 * y is fp32 [ny][d] for float metrics or bytes [ny][d/8] for binary metrics (d in bits). */
int b200_part_scan(int metric, const void *x, int64_t nx, const void *y, int64_t ny, int d, int k,
                   int64_t block_rows, const uint8_t *row_exists /*nullable*/, const uint8_t *filter_bits /*nullable*/,
                   float *out_dis, int64_t *out_ids);

/* ------------------------------------------------------------------------------------
 * Device-resident corpus = a FLAT vector index / cached part column in HBM.
 * Replaces Search::VectorIndex<...>(IndexType::FLAT)::{build, search} as reached through
 * VIWithColumnInPart::search (VectorIndex/Common/VIWithDataPart.cpp:858-957) and the
 * VICacheManager residency model (VectorIndex/Cache/VICacheManager.cpp:65-157).
 * ---------------------------------------------------------------------------------- */
typedef struct b200_corpus b200_corpus;

int b200_corpus_create(int metric, int dtype, int d, int64_t capacity_rows, b200_corpus **out);
/* append fp32 (or binary bytes for B200_DTYPE_BIN) rows from host memory; converted to the
 * corpus dtype on device; row norms are computed on device. */
int b200_corpus_append(b200_corpus *c, const void *rows, int64_t n);
/* adopt rows that already live in HBM in the corpus dtype (the rows must be COMPLETE when this is called: the row norms
 * are computed on the corpus' own stream, which is not ordered after the caller's streams), row-major [n][d] with
 * d % 64 == 0 for bf16 (d % 4 == 0 for f32); the memory stays owned by the caller. */
int b200_corpus_adopt_device(b200_corpus *c, const void *device_rows, int64_t n);
int b200_corpus_size(const b200_corpus *c, int64_t *out_rows);
int b200_corpus_free(b200_corpus *c);

/* search with host queries/results (H2D of queries and D2H of results inside the call).
 * Pre-filtered exact search: with alive_bits given, this call (and b200_flat_knn, b200_binary_knn, b200_part_scan, and
 * b200_index_search on FLAT / BINARYFLAT / small-part fallback / exact_batch=1) counts the bitmap's set bits on the host.
 * When the filter keeps few enough rows (see b200_corpus_set_prefilter) only those rows are copied into a compact scratch
 * corpus and scored; the result is byte for byte the full scan's, and the cost follows the rows kept, not the corpus size.
 * Batch size: this call, b200_corpus_search_device, b200_flat_knn, b200_binary_knn and b200_part_scan take any nq whose
 * queries, results and per-query scratch fit in device memory; the scan and tensor-core kernels split a large batch into
 * as many launches as the grid limits need. */
int b200_corpus_search(b200_corpus *c, const float *queries, int64_t nq, int k, const uint8_t *alive_bits /*nullable*/,
                       float *out_dis, int64_t *out_ids);
/* same, queries and results in device memory, asynchronous on `stream` (a cudaStream_t
 * passed as void*; NULL = the corpus' own stream followed by a synchronise).
 * id_offset is added to every returned id (shard base for multi-GPU merges).
 * This call, b200_index_search_device and the b200_sharded_* calls always scan the whole corpus under a filter: choosing
 * the pre-filtered path needs the count of kept rows on the host, which would cost the synchronise they promise not to do. */
int b200_corpus_search_device(b200_corpus *c, const float *d_queries, int64_t nq, int k,
                              const uint8_t *d_alive_bits /*nullable*/, int64_t id_offset, float *d_out_dis,
                              int64_t *d_out_ids, void *stream);
/* Force a search path (tests, A/B measurements; production leaves 0):
 *   0 auto | 1 memory-bound scan kernel | 2 tensor cores (bf16 corpora: the bf16 wgmma kernel; fp32 corpora: the
 *   3xTF32 kernel; binary corpora: the b1 kernel, B200_ERR_UNSUPPORTED unless the rows are a multiple of 16 bytes) |
 *   3 .. 7 the same as 2 (they named tensor-core variants of an earlier target and stay accepted).
 * Auto on a binary corpus: the b1 kernel when the rows are a multiple of 16 bytes (d < 2^24 bits) and the batch has at
 * least ceil(20480 / row_bytes^2) queries (2 at 1024 bits, 20 at 256 bits), else the scan. */
int b200_corpus_set_path(b200_corpus *c, int path);
/* Pre-filtered exact search (tests, A/B measurements; production leaves 0):
 *   0 auto: the gathered path when the filter keeps at most a measured share of the rows of a large enough corpus;
 *   1 never: always the full scan that masks the filtered rows;
 *   2 whenever a filter is given and the compact copy fits the budget.
 * Every mode keeps the compact copy within 1/8 of the corpus' row bytes and 1 GiB; beyond that the full scan runs. */
int b200_corpus_set_prefilter(b200_corpus *c, int mode);
/* rows the last search on this corpus scored: its size after a full scan, the kept rows after a pre-filtered one */
int b200_corpus_last_rows_scored(b200_corpus *c, int64_t *rows);
/* the same for the last corpus search the CALLING THREAD ran, whatever corpus it was: the per-thread scratch corpus of
 * b200_flat_knn / b200_binary_knn / b200_part_scan, or the rows of an index behind the exact paths of b200_index_search */
int b200_thread_last_rows_scored(int64_t *rows);
/* which kernel the last search on this corpus launched (so a test can prove it exercised the variant it meant to) */
#define B200_KERNEL_SCAN 1 /* flat_scan_kernel, or binary_scan_kernel on binary corpora */
#define B200_KERNEL_GEMM_BF16 2   /* gemm_topk_kernel<BF16> (cta_group and pairs_per_cluster report 1) */
#define B200_KERNEL_GEMM_TS 3     /* no longer launched; the value stays reserved */
#define B200_KERNEL_GEMM_TF32X3 4 /* gemm_topk_kernel<TF32X3> */
#define B200_KERNEL_GEMM_B1 5     /* gemm_topk_kernel<B1>: binary rows, wgmma .b1 AND + popcount */
int b200_corpus_last_variant(b200_corpus *c, int *kernel, int *cta_group, int *pairs_per_cluster, int *grid);
/* CUDA-event timing of the dominant kernel (scan or GEMM, float or binary) of every search on this corpus,
 * recorded on the launching stream; used by bench.py for the roofline report. */
int b200_corpus_enable_timing(b200_corpus *c, int on);
int b200_corpus_kernel_time(b200_corpus *c, int reset, double *out_total_ms, int64_t *out_launches);
/* number of kernels this library launched on the calling thread since the last reset */
int64_t b200_launch_count(int reset);
/* bytes of device memory the library holds, over every device and thread (a diagnostic: what the library allocated
 * itself, unlike cudaMemGetInfo, which also moves with every other user of the device) */
int64_t b200_device_bytes(void);
/* b200_flat_knn / b200_binary_knn / b200_part_scan keep one grow-only scratch corpus per calling thread (device rows,
 * workspaces, stream), sized for the largest part that thread has scanned; this frees it (it is also freed at thread
 * exit).  A ClickHouse worker calls it when it goes idle. */
int b200_thread_release(void);

/* K-way merge of per-part / per-GPU top-k lists on device.
 * Replaces MergeTreeBaseSearchManager::getTotalTopSearchResultImpl
 * (VectorIndex/Storages/MergeTreeBaseSearchManager.cpp:207-299) for the sharded path:
 * d_dis/d_ids are [n_lists][nq][k] (e.g. the NCCL all-gather buffer); output [nq][k].
 * descending = 1 for IP / BM25. */
int b200_topk_merge_device(const float *d_dis, const int64_t *d_ids, int n_lists, int64_t nq, int k, int descending,
                           float *d_out_dis, int64_t *d_out_ids, void *stream);

/* Same, for a packed all-gather buffer: list l starts at d_dis + l * dis_list_stride (floats) and
 * d_ids + l * ids_list_stride (int64s), so that one NCCL all-gather of
 * {float dis[nq*k]; int64 ids[nq*k]} per rank feeds the merge directly. */
int b200_topk_merge_device_strided(const float *d_dis, const int64_t *d_ids, int n_lists, int64_t dis_list_stride,
                                   int64_t ids_list_stride, int64_t nq, int k, int descending, float *d_out_dis,
                                   int64_t *d_out_ids, void *stream);
/* General form.  Input lists hold k_in entries per query (list l, query q at d_dis + l * dis_list_stride + q * k_in),
 * sorted best first, ids < 0 = unused slot; ids are full 64-bit values (shard base + row, any magnitude).
 * tie_mode 0: equal scores -> smaller id first (this library's contract everywhere else).
 * tie_mode 1: the reference's own order -- std::multimap insertion order of getTotalTopSearchResultImpl
 *   (list 0's entries first, each list in its own order): ascending walks return the earlier-inserted of two equal
 *   scores, the reverse walk used for IP / BM25 returns the later-inserted one (MergeTreeBaseSearchManager.cpp:271).
 *   d_out_list (nullable) receives the list (part) index of every output entry, -1 for unused slots. */
int b200_topk_merge_device_ex(const float *d_dis, const int64_t *d_ids, int n_lists, int64_t dis_list_stride,
                              int64_t ids_list_stride, int64_t nq, int k_in, int k, int descending, int tie_mode,
                              float *d_out_dis, int64_t *d_out_ids, int32_t *d_out_list /*nullable*/, void *stream);

/* ------------------------------------------------------------------------------------
 * Vector indexes.  Replaces Search::createVectorIndex / VectorIndex::{build, search,
 * computeTopDistanceSubset} (VectorIndex/Common/VIWithDataPart.cpp:416-430, :131, :926, :838-856).
 * type (the reference's index type names, VectorIndex/Common/VICommon.h:178-180 and the 2_vector_search tests):
 *   "FLAT"                      exact scan of the resident rows;
 *   "IVFFLAT"                   inverted lists holding bf16 rows, candidates re-ranked exactly against the fp32 rows;
 *   "IVFSQ"                     lists of 8-bit scalar-quantised rows (one byte per dimension);
 *   "IVFPQ"                     lists of m-byte product-quantiser codes of the residual (8-bit codes, 256 codewords per
 *                               sub-quantiser; M must divide d).  Two list scans, chosen by d / M alone (no option, nothing
 *                               stored): d / M in {1, 2, 4, 8} decodes codes into tensor-core tiles and keeps the 512 B x d bf16
 *                               codebook in shared memory, so d <= 220 (wider ones, SCANN and HNSWPQ included, are refused at
 *                               train with B200_ERR_UNSUPPORTED); any other d / M is scanned by table look-up (a per-query
 *                               M x 256 fp32 table of <q_j, codeword>, at any width), which needs M <= 128 (larger M is refused
 *                               at train).  Default M: d / 8 (or d / 4, d / 2, d) up to d = 220; above, d / dsub with dsub the
 *                               smallest divisor of d that is >= 16 and keeps M <= 128 (M = 48 at d = 768, 96 at d = 1536).
 *                               "bit_size=4" (IVFPQ, SCANN and HNSWPQ; other types ignore the key) selects 4-bit codes: 16
 *                               codewords per sub-quantiser, two codes per byte (code j in byte j / 2, even j in the low
 *                               nibble), always scanned by table look-up from a per-query M x 16 fp32 table at any d / M
 *                               (1, 2, 4 and 8 included), which needs M <= 2048 (larger M is refused at train with
 *                               B200_ERR_UNSUPPORTED).  Default M at 4 bits keeps the code bytes of the 8-bit default: twice
 *                               the 8-bit default M when that default's sub-vector length is even (M = 96 at d = 768, 24 at
 *                               d = 96), else the 8-bit default (M = 10 at d = 250).  bit_size=8, or no bit_size, is the
 *                               8-bit index; any other value is refused at create with B200_ERR_UNSUPPORTED.  4-bit indexes
 *                               are saved as B2IX v3 (below).
 *                               "aq_threshold=T" (IVFPQ, SCANN and HNSWPQ; other types ignore the key; 0 < T < 1, ScaNN
 *                               recommends 0.2 for normalised data) trains and encodes with ScaNN's anisotropic loss
 *                               ||r||^2 + w <r, x>^2 (r = x - x^ the row's reconstruction error, w = (eta - 1) / ||x||^2,
 *                               eta = (d - 1) T^2 / (1 - T^2)), which weights the error along the row, the part that moves
 *                               inner products, above the error across it: the codebooks take kAqIters coordinate-descent /
 *                               least-squares iterations after k-means, and every added row takes the codes that lower its
 *                               loss from the nearest-codeword ones (csrc/ivf_aq.cu).  Codes, scans and file are those of
 *                               plain PQ (8 or 4 bits; an AQ index is an ordinary B2IX v2 / v3 file), and it composes with
 *                               keep_raw, refine_factor, filter_probe and both build styles.  Absent or 0: plain PQ, file byte
 *                               for byte.  A negative, >= 1 or non-numeric value is refused at create with B200_ERR_INVALID,
 *                               a non-zero one under L2 with B200_ERR_UNSUPPORTED (the loss is defined for inner-product
 *                               ranking), and d / M > 64 at train with B200_ERR_UNSUPPORTED;
 *                               "opq=1" (IVFPQ, SCANN and HNSWPQ; other types ignore the key) learns an orthonormal rotation
 *                               R [d][d] fp32 (y = x.R; Ge et al., optimised PQ) at train, in "opq_iters=N" alternations
 *                               (default 20, not tuned) of the PQ codebooks of the rotated residuals with an orthogonal
 *                               Procrustes step, and quantises x.R instead of x: the centroids, codebooks, codes and norm
 *                               terms live in the rotated space, and the coarse probe and the list scan take the prepared
 *                               query rotated.  The fp32 rows and every exact path (the second stage, exact_batch=1, the
 *                               pre-filter, filter_probe's exact rule, small parts) stay unrotated.  R does not change L2,
 *                               IP or cosine; each query batch pays one d x d product.  It composes with bit_size=4,
 *                               aq_threshold, keep_raw, refine_factor, filter_probe and both build styles.  opq_iters=0 keeps
 *                               R = I (still stored and applied).  A part below the inverted-file threshold stays FLAT with
 *                               no R.  Absent or 0: plain PQ, file byte for byte.  Another value of opq, or opq_iters < 0, is
 *                               refused at create with B200_ERR_INVALID, opq=1 with d > 4096 (R <= 64 MB) with
 *                               B200_ERR_UNSUPPORTED.  Saved as B2IX v5 (below);
 *   "MSTG"                      closed source upstream; here the two-stage index of SURVEY 2.5 K6: bf16 lists + exact
 *                               fp32 second stage (supportTwoStageSearch, first_stage_only, computeTopDistanceSubset).
 *                               With "graph_degree=D" it also builds a neighbour graph (as HNSWFLAT below, from each row's
 *                               2D + 1 nearest by its own list search's FIRST stage) and walks it over its bf16 list rows in
 *                               HBM; with fp32 rows (keep_raw=1, or 2: in host memory) and refine_factor > 1 the walk's best
 *                               min(1024, k x refine_factor) rows (out_num_candidates) are re-ranked exactly, otherwise
 *                               it returns first-stage distances.  Every keep_raw is accepted with it;
 *   "SCANN", "HNSWFLAT", "HNSWSQ", "HNSWPQ"   accepted and SERVED BY THE INVERTED-FILE ENGINE with the payload their
 *                               name implies (PQ + re-rank, bf16, 8-bit, PQ): they traverse no graph unless HNSWFLAT
 *                               has graph_degree below (MSTG's graph is above; ScaNN's anisotropic PQ loss is the opt-in aq_threshold above); the contract for every ANN type is recall against
 *                               FLAT, not traversal order (SURVEY 8c: parity unpinned for ANN at large N).
 *                               HNSWFLAT with "graph_degree=D" (D = 16, 32 or 64; absent or 0: the lists only) also builds a
 *                               neighbour graph [n][D] at finalize (each row's 2D nearest by its own list search, pruned by
 *                               rank, merged with reverse edges) and searches it by default: one CTA per query walks the graph
 *                               from the best min(ef_s, 32) ids of an nprobe=1 first stage, scoring each row once, exactly in
 *                               fp32.  Search keys: "ef_s=N" (list width, default 64, raised to k, at most 1024), "graph=0" (the
 *                               list search instead), "search_width=W" (W = 1, 2, 4 or 8, default 1: W parents expanded
 *                               per iteration by a cluster of W CTAs per query, for single queries and small batches; the
 *                               same scores, so the answer of W = 1 is the default's byte for byte; another W on a search
 *                               that would walk the graph: B200_ERR_INVALID, checked before the filtered exact rule as
 *                               ef_s is; ignored with graph=0, exact_batch=1 or no graph; it applies to MSTG's and
 *                               BINARYMSTG's walks too).  Any type but HNSWFLAT / MSTG / BINARYMSTG with graph_degree > 0, or HNSWFLAT
 *                               with keep_raw=0 / 2 and it: B200_ERR_UNSUPPORTED; another D: B200_ERR_INVALID.  A part
 *                               below the threshold has no graph;
 *   "BINARYFLAT"                binary rows (metric HAMMING or JACCARD, d in bits: a multiple of 8, at most 65536), exact
 *                               resident binary corpus (scan or b1 tensor-core kernel, chosen as for a binary corpus);
 *   "BINARYIVF"                 inverted lists of the row bytes, coarse quantiser trained by k-majority (Hamming, for
 *                               Jaccard too), scanned on the tensor cores (wgmma .b1 AND + popcount); list rows are exact,
 *                               so every returned distance is exact and nprobe >= nlist returns the BINARYFLAT answer
 *                               byte for byte.  nprobe must be <= 1024 unless it is >= nlist (B200_ERR_UNSUPPORTED);
 *   "BINARYHNSW", "BINARYMSTG"  accepted and served by the BINARYIVF engine (same recall contract as HNSW*).  BINARYHNSW has
 *                               no graph.  BINARYMSTG with "graph_degree=D" (16, 32 or 64; another D: B200_ERR_INVALID)
 *                               also builds a neighbour graph as MSTG does, from each row's 2D + 1 nearest by its own list
 *                               search (exact, "graph=0" at the default nprobe, queried with the row bytes read back from
 *                               the pages), and walks it by default over its binary list rows in HBM with ef_s,
 *                               search_width, graph=0 and the k <= 1024 limit as HNSWFLAT.  Every key of the walk is the
 *                               exact Hamming / Jaccard distance BINARYFLAT returns for that (query, row), so there is no
 *                               second stage (out_num_candidates = k).  Under a filter the walk always answers (a binary
 *                               inverted-file index keeps no exact corpus) and may return fewer than k rows;
 *                               "graph=0,nprobe=<nlist>" is the exact complete answer.
 * Binary types take only HAMMING / JACCARD and float types only L2 / IP / COSINE (else B200_ERR_INVALID).  For a binary
 * index every `rows` / `queries` pointer below (build, train, add, search and their _device forms) carries bytes
 * [n][d / 8] behind the `const float *` type, the convention of the binary corpora.  Binary indexes have no second stage:
 * b200_index_refine and "exact_batch=1" return B200_ERR_UNSUPPORTED; refine_factor / keep_raw are ignored and
 * first_stage_only returns the normal (already exact) answer.
 * params: the reference's key=value / JSON parameter string: "ncentroids=1024" (or nlist), "M=32", "nprobe=64" (float
 * indexes: nprobe >= nlist probes every list; below nlist, nprobe <= 2048, the k limit of the exact scan that ranks the
 * centroids above 1024 probes, else B200_ERR_UNSUPPORTED),
 * "refine_factor=8" (candidates per returned row handed to the exact second stage; 1 = first-stage distances),
 * "keep_raw=0" (do not keep the fp32 rows: no second stage, half the memory), "keep_raw=2" (keep them, in pinned, mapped
 * host memory instead of HBM: [n][d_pad] fp32 in row-id order, the values the HBM rows would hold; the second stage gathers
 * its nq x k x refine_factor candidate rows over PCIe, with keys and outputs byte-identical to the HBM placement.  It applies
 * to the float types with inverted lists; FLAT, parts below the threshold below and binary types keep their rows in HBM;
 * "exact_batch=1" is then refused with B200_ERR_UNSUPPORTED).  Parts smaller than
 * max(2000, 8 * nlist) rows are served by an exact FLAT scan (the reference's fallback_to_flat, test 00029).
 *
 * Build = the reference's reader-driven build (VIPartReader train block / add blocks, VIWithDataPart.cpp:131):
 *   b200_index_reserve(total rows)  -- createVectorIndex's total_vec: sizes the page pool
 *   b200_index_train(sample)        -- coarse k-means (+ PQ codebooks / SQ ranges) on a sample
 *   b200_index_add(chunk) ...       -- any number of chunks, row ids continue from the rows already added
 *   b200_index_finalize()
 * b200_index_build(rows, n) does all four from one host array.  *_device variants take fp32 rows already in HBM.
 *
 * Unusable rows and queries (float indexes; a ClickHouse Float32 column can hold NaN and inf).  A row or query is unusable
 * when the fp32 sum of the squares of its coordinates is not finite: a NaN or infinite coordinate, or one whose square
 * overflows (about 1e19 and up).  One device helper (warp_row_usable) decides it for training and add alike.
 *   Training: the coarse k-means, the SQ ranges, the PQ codebooks and the anisotropic iterations use only the usable rows of
 *     the sample, in their order, judged as given (before the cosine normalisation); the FLAT fallback below counts only
 *     those rows.  This holds for train, train_device and build's strided sample.
 *   Add: an unusable row keeps its row id (info's n counts it) and its fp32 row under keep_raw 1 and 2, but goes to no list,
 *     nor does a row for which the centroid search finds no list: the list sizes add up to the rows that are in a list.
 *   Search: the list scans, the exact second stage and both graph walks never return a row that is in no list;
 *     filter_probe's promise is min(k, kept rows that are in a list).  The exact paths (FLAT, the small-part fallback,
 *     exact_batch=1, the filter_probe exact rule) keep the FLAT rule instead: a row whose distance is not finite is never
 *     returned and never displaces a finite one (under IP, a row with an infinite coordinate is outside that rule).  They
 *     judge the distance, not the row, so they CAN return an unusable row whose distance is finite: one whose square
 *     overflows is a zero row after the cosine normalisation (distance 1), and under IP its inner product is finite (and
 *     may rank first).  Where the filter_probe exact rule answers, its promise is FLAT's: min(k, kept rows with a finite
 *     distance).
 *   Queries: one with a NaN coordinate returns no rows on every path and metric; one with an infinite coordinate returns no
 *     rows under L2 and cosine (under IP it is outside the contract, as for FLAT).  A non-finite query never changes the
 *     answer of another query of the batch.
 *   Cosine: rows and queries whose sum of squares is below FLT_EPSILON are usable and stay as given (no normalisation); their
 *     key is 1 - <q, x>.
 *   Files: the format is unchanged; the list lengths may add up to less than n (load refuses more than n).  A row in no list
 *     has an empty adjacency row in a v4 graph, and load refuses an MSTG or BINARYMSTG graph edge to such a row.
 * ---------------------------------------------------------------------------------- */
/* Widest float index with inverted lists (every float type but FLAT, which keeps no limit below the loader's 65536;
 * binary types take up to 65536 bits): create refuses a wider d with B200_ERR_UNSUPPORTED, and so does load for a wider
 * file.  The bound is the largest block of shared memory a search of these types needs: the graph walk over MSTG's bf16 list
 * rows at ef_s = k = 1024 under a filter holds the query (d_pad64 floats) and 101760 bytes of lists and visited table in the
 * 227 KB a block may use, so d_pad64 <= 32640.  Every other configuration fits wider: the fp32 graph walk (HNSWFLAT) up to
 * d_pad 32672, the exact second stage at k = 1024 (d_pad x 4 + 73728 bytes) up to d_pad 39680; the bf16 and SQ8 list scans
 * stream k-blocks and need no more shared memory at any width.  The graph walks at search_width=W > 1 hold (W - 1) KB + 512
 * bytes more: at ef_s = k = 1024 under a filter they are refused with B200_ERR_UNSUPPORTED above d_pad64 32256 / 31744 /
 * 30720 (MSTG) and d_pad 32288 / 31776 / 30752 (HNSWFLAT) for W = 2 / 4 / 8; create and load accept the same widths. */
#define B200_MAX_FLOAT_DIM 32640

typedef struct b200_index b200_index;
int b200_index_create(const char *type, int metric, int d, const char *params, b200_index **out);
int b200_index_build(b200_index *ix, const float *rows, int64_t n);
int b200_index_reserve(b200_index *ix, int64_t total_rows);
int b200_index_train(b200_index *ix, const float *rows, int64_t n);
int b200_index_train_device(b200_index *ix, const float *d_rows, int64_t n);
int b200_index_add(b200_index *ix, const float *rows, int64_t n);
int b200_index_add_device(b200_index *ix, const float *d_rows, int64_t n);
int b200_index_finalize(b200_index *ix);
int b200_index_info(const b200_index *ix, int64_t *n, int *nlist, int *m, int *uses_ivf);
/* first_stage_only (two-stage types): return the first-stage candidates with first-stage distances;
 * out_num_candidates receives the width the first stage ran with (SearchResult::getNumCandidates).
 * "exact_batch=1" in `params` answers by an exact pass over the fp32 rows instead (recall 1).
 * Batch size: the exact paths (FLAT, BINARYFLAT, the small-part fallback, exact_batch=1) take any batch that fits in device
 * memory, as b200_corpus_search does.  The list scans of the inverted-file types refuse, with B200_ERR_UNSUPPORTED, a batch with nq x nprobe >= 2^31 probe pairs or with nq x nprobe x chunks x k1 >= 2^32 candidate slots
 * (chunks: the pieces a long list is cut into, k1 = min(1024, k x refine_factor) on two-stage searches, else k); split such
 * a batch.  The index stays usable after a refusal.
 * Tuning / A-B switches, also in `params` (defaults are chosen from the batch shape): "pages_per_chunk=N" (pages of a list one work
 * item streams), "shared_bound=0" (do not share a per-query bound between the work items of a launch), "coarse_path=1|2|3" (centroid
 * probe by the scan kernel / the tensor-core top-k / score tiles + warp select; default 3 for nprobe > 8), "prefilter=0|1|2" (exact
 * paths of b200_index_search only -- FLAT, BINARYFLAT, the small-part fallback, exact_batch=1: as b200_corpus_set_prefilter;
 * the list scans of the IVF types are not affected).
 * Filter-aware probing, float inverted-file types only (opt-in, because it changes answers): "filter_probe=1" with a filter
 * given makes every query probe, in (coarse key, list id) order, the first
 *   p_q = min(max_nprobe, max(nprobe, the fewest lists whose kept rows reach k1))
 * lists (nlist when all of them do not reach it), k1 = min(1024, k x refine_factor) on two-stage searches, else k; of those
 * it scans the lists that hold a kept row, and of each only the pages that hold one (leaving out the others changes no
 * answer).  "max_nprobe=N" caps p_q (default nlist, clamped to [nprobe, nlist]; nprobe itself is unchanged).  With the
 * default cap every query returns min(k, kept rows) rows.  Where p_q <= 1024, a query's answer is byte-identical to a
 * filtered search of that query with "nprobe=p_q,coarse_path=3".
 * The selection costs one device -> host read-back and ONE stream synchronise in mid-search per call, however large the
 * batch (look-up-scan indexes included), in b200_index_search_device (and so b200_sharded_index_search) too.  When
 * b200_index_search gets a host bitmap, the fp32 rows are in HBM and first_stage_only is 0, the exact pass over the kept
 * rows answers instead (as "exact_batch=1") if the bitmap keeps at most 16 x nprobe x n / nlist rows AND that pass would
 * score only the kept rows for this batch, i.e. within b200_corpus_set_prefilter's limit for the "prefilter" mode given (auto
 * by default: a corpus of at least 512 MB and a share of at most 5 % / 12.5 %; 1 never; 2 up to n / 8 rows and 1 GiB of them).  nprobe >= nlist:
 * only the page skipping.  Binary types: B200_ERR_UNSUPPORTED.
 * Without a filter the key changes nothing. */
int b200_index_search(b200_index *ix, const float *queries, int64_t nq, int k, const char *params, int first_stage_only,
                      const uint8_t *alive_bits /*nullable*/, float *out_dis, int64_t *out_ids, int64_t *out_num_candidates);
/* same with device buffers, asynchronous on `stream` (NULL = the index's own stream, synchronised); id_offset is added to
 * every returned id (shard base for multi-GPU merges) */
int b200_index_search_device(b200_index *ix, const float *d_queries, int64_t nq, int k, const char *params, int first_stage_only,
                             const uint8_t *d_alive_bits /*nullable*/, int64_t id_offset, float *d_out_dis, int64_t *d_out_ids,
                             void *stream);
/* roofline inputs of the list scan: CUDA-event time of the grouped scan kernel since the last reset, bytes per list row,
 * and an upper bound of the work items of the last search.  After a graph search: the rows it scored, the bytes of one
 * row it read (HNSWFLAT: d_pad x 4, MSTG: the bf16 list row, d_pad64 x 2) and nq.
 * After the finalize of a graph_degree index, b200_index_phase_ms holds the graph build's candidates | prune | merge. */
int b200_index_phase_ms(b200_index *ix, double out_ms[5]);   /* last search: coarse | pairs+plan+gather | scan | merge | refine */
int b200_index_list_sizes(const b200_index *ix, uint32_t *out_sizes /*[nlist]*/, int capacity);
int b200_index_enable_timing(b200_index *ix, int on);
int b200_index_last_scan(b200_index *ix, int64_t *rows_streamed, int64_t *payload_row_bytes, int64_t *work_items,
                         double *kernel_ms_total, int64_t *kernel_launches, int reset);
/* lists each query of the last search probed, out_lists[nq] (capacity >= nq, else B200_ERR_INVALID; null: skipped): p_q
 * under filter_probe=1, nprobe on every other list search, 0 where an exact pass answered (FLAT, the small-part fallback,
 * exact_batch=1, the filter_probe exact rule).  out_exact (nullable) = 1 when the filter_probe exact rule answered. */
int b200_index_last_probe(b200_index *ix, int32_t *out_lists, int64_t capacity, int *out_exact);
/* coarse-probe path of the last search of a float inverted-file index (tests): 1 the FMA scan of the centroid table, 2 the
 * tensor-core (3xTF32) path, 3 the ranking keys + select kernels, 0 none ran (every list probed, an exact pass, binary). */
int b200_index_last_coarse(b200_index *ix, int *path);
/* aq_threshold indexes (tests, benchmarks): eta and the training sample's mean anisotropic loss after the k-means codebooks,
 * then after each anisotropic iteration, out_loss[*out_n] (capacity >= *out_n, else B200_ERR_INVALID; null: skipped).
 * B200_ERR_INVALID for an index not trained with the key here (plain PQ, other types, an index loaded from a file). */
int b200_index_train_loss(const b200_index *ix, double *out_eta, double *out_loss, int capacity, int *out_n);
/* opq=1 indexes (tests, benchmarks): the rotation R, out_r[d][d] fp32 row-major with y = x.R (null: skipped), and the
 * training sample's mean PQ loss (mean ||r - r^||^2 of its residuals) at R = I, then after each alternation,
 * out_loss[*out_n] (capacity >= *out_n, else B200_ERR_INVALID; null: skipped).  An index loaded from a file returns its R
 * with *out_n = 0.  B200_ERR_INVALID for an index without the key, or one that holds no rotation (not trained, or a part
 * below the inverted-file threshold, which is FLAT). */
int b200_index_opq(const b200_index *ix, float *out_r, double *out_loss, int capacity, int *out_n);
/* computeTopDistanceSubset: exact distances of candidate ids [nq][ncand] (negative = unused) -> top-k */
int b200_index_refine(b200_index *ix, const float *queries, int64_t nq, const int64_t *cand_ids, int64_t ncand, int k,
                      float *out_dis, int64_t *out_ids);
/* moves the fp32 rows of a finalized index between HBM (placement 1) and pinned host memory (2), the keep_raw values, under
 * the index mutex (waits for the device first); the move to host frees the HBM rows and their side arrays.  An index loaded
 * from an older file can so be demoted without a rebuild.  B200_ERR_INVALID for an index without rows (keep_raw=0) or not
 * finalized; B200_ERR_UNSUPPORTED where the rows are the index (FLAT, small parts, binary types) and for an HNSWFLAT graph
 * (its walk reads them; an MSTG graph walks its bf16 list rows and moves in both directions). */
int b200_index_set_raw_placement(b200_index *ix, int placement);
/* graph_degree indexes: the neighbour graph, out[n][D] u32 (0xFFFFFFFF = empty slot; capacity_rows >= n, else
 * B200_ERR_INVALID; null: skipped), *out_degree = D, or 0 when the index has no graph (then nothing is copied) */
int b200_index_graph(const b200_index *ix, uint32_t *out, int64_t capacity_rows, int *out_degree);
/* the seed ids of the last search when it walked a graph, out[nq][S] (negative = none; capacity >= nq x S, else
 * B200_ERR_INVALID; null: skipped), *out_per_query = S, or 0 when the last search did not walk a graph.  Waits for the device. */
int b200_index_last_seeds(b200_index *ix, int64_t *out, int64_t capacity, int *out_per_query);
/* VIWithColumnInPart::serialize / load (VIWithDataPart.cpp:451-525, :578-764): one self-describing file
 * ("B2IX" v2; the closed library's .vidx3 payload cannot be reproduced).  PQ indexes with 4-bit codes are written as
 * v3: the v2 layout with the header's reserved word holding the code width (4) and a [M][16][d / M] codebook; every other
 * index is written as v2.  load accepts both and validates every size it derives.  An index with its fp32 rows in host
 * memory writes the header's has_raw as 2 (every other byte as in HBM placement) and loads them straight into pinned host
 * memory again.  An index with a graph (graph_degree) is written as v4: the v2 layout with the reserved word holding D,
 * followed by the graph [n][D] u32 (HNSWFLAT with has_raw 1, MSTG with has_raw 0, 1 or 2, BINARYMSTG); load checks every
 * graph id (< n or 0xFFFFFFFF; MSTG, BINARYMSTG: a row that is in a list) before any kernel reads it.  An opq=1 index is written as v5: the v2
 * layout (reserved word 0) or the v3 one (4-bit codes, reserved word 4), followed by R [d][d] fp32; load accepts it for an
 * inverted-file IVFPQ / SCANN / HNSWPQ index with d <= 4096 and a finite R orthonormal within 1e-4 (max |R^T R - I|). */
int b200_index_save(b200_index *ix, const char *path);
int b200_index_load(const char *path, b200_index **out);
/* the same through the host's own streams (Search::IndexDataFileWriter / Reader over ClickHouse disks,
 * VectorIndex/Common/VectorIndexIO.h:33-164): the callbacks return 0 when every byte was written / read */
int b200_index_save_cb(b200_index *ix, int (*write)(void *ctx, const void *data, size_t bytes), void *ctx);
int b200_index_load_cb(int (*read)(void *ctx, void *data, size_t bytes), void *ctx, b200_index **out);
int b200_index_free(b200_index *ix);

/* ------------------------------------------------------------------------------------
 * Multi-GPU: parts / row ranges shard over the GPUs of one box, one communicator rank per GPU (one process per GPU, or
 * one host thread per device).  The reference merges per-part top-k lists on the host
 * (MergeTreeBaseSearchManager::getTotalTopSearchResultImpl, VectorIndex/Storages/MergeTreeBaseSearchManager.cpp:207-299)
 * and sums BM25 statistics over parts (ReadWithHybridSearch::getStatisticForTextSearch,
 * VectorIndex/Processors/ReadWithHybridSearch.cpp:89-209); across GPUs these are ONE ncclAllGather of the packed
 * per-shard top-k + the merge kernel, and ONE ncclAllReduce(sum) of a few counters.  NCCL is resolved with dlopen
 * (nccl_lib_path, $B200_NCCL_LIB, or the libnccl.so.2 already in the process); rank 0 creates the 128-byte unique id and
 * the host distributes it (any side channel: MPI, a file, torch.distributed.broadcast).
 * ---------------------------------------------------------------------------------- */
typedef struct b200_comm b200_comm;
int b200_comm_unique_id(const char *nccl_lib_path /*nullable*/, void *out_id_128_bytes);
int b200_comm_create(const char *nccl_lib_path /*nullable*/, const void *unique_id_128_bytes, int rank, int world, b200_comm **out);
int b200_comm_info(const b200_comm *c, int *rank, int *world);
int b200_comm_free(b200_comm *c);
/* building blocks: device buffers a shard search writes its [nq][k] result to, then all-gather + merge on `stream`.
 * The two are one packed record: dis [nq * k] fp32, padded to a multiple of 8 bytes, then ids [nq * k] int64, so *d_ids is
 * 8-byte aligned for every nq * k.  gather_merge refuses k > 2048 before it issues the all-gather. */
int b200_comm_local_buffers(b200_comm *c, int64_t nq, int k, float **d_dis, int64_t **d_ids);
int b200_comm_gather_merge(b200_comm *c, int64_t nq, int k, int descending, float *d_out_dis, int64_t *d_out_ids, void *stream);
/* the same for lists produced on the host (per-shard BM25 top-k: scores descending, unused slots score -inf / id -1);
 * uploads, all-gathers, merges and returns the table-wide top-k to the host; synchronous */
int b200_comm_gather_merge_host(b200_comm *c, const float *h_dis, const int64_t *h_ids, int64_t nq, int k, int descending,
                                float *h_out_dis, int64_t *h_out_ids);
/* in-place sum over the ranks of n host-resident uint64 counters (total_docs, total_tokens[field], doc_freq[...]) */
int b200_comm_allreduce_sum_u64(b200_comm *c, uint64_t *host_counters, int64_t n);
/* whole steps.  Every rank passes its own shard and the same queries; every rank receives the global top-k.
 * id_offset = first global row id of this rank's shard.  `stream` must be a real stream.  use_graph != 0 replays the step
 * (query conversion, tensor-core scan, all-gather, merge) as ONE CUDA graph from the second call with the same arguments.
 * A replay answers as an eager call would: the graph is captured again when the corpus changed since the capture (an
 * append, set_path, a workspace that grew for another search) or is another corpus at a reused address. */
int b200_sharded_corpus_search(b200_comm *cm, b200_corpus *corpus, const float *d_queries, int64_t nq, int k,
                               const uint8_t *d_alive_bits /*nullable*/, int64_t id_offset, float *d_out_dis, int64_t *d_out_ids,
                               void *stream, int use_graph);
/* graphs the sharded corpus search captured and replays it launched, over the communicator's life */
int b200_comm_graph_stats(b200_comm *c, int64_t *captures, int64_t *replays);
/* host queries in, host results out (H2D, scan, all-gather, merge, D2H, synchronise inside).  d must equal the corpus'
 * dimension (B200_ERR_INVALID otherwise).  Query rows are what the device entry reads: fp32 [nq][d], or for a binary corpus
 * bytes [nq][d / 8] passed through `queries`. */
int b200_sharded_corpus_search_host(b200_comm *cm, b200_corpus *corpus, const float *queries, int64_t nq, int d, int k,
                                    int64_t id_offset, float *out_dis, int64_t *out_ids, void *stream, int use_graph);
/* metric must be the index' own (B200_ERR_INVALID otherwise): it sets the merge direction */
int b200_sharded_index_search(b200_comm *cm, b200_index *ix, int metric, const float *d_queries, int64_t nq, int k, const char *params,
                              const uint8_t *d_alive_bits /*nullable*/, int64_t id_offset, float *d_out_dis, int64_t *d_out_ids,
                              void *stream);

/* ------------------------------------------------------------------------------------
 * HBM residency cache: the device-side VICacheManager (VectorIndex/Cache/VICacheManager.cpp:65-157, an
 * LRUResourceCache keyed by CacheKey = table path / part / index / column, VICacheObject.h:119-137, weighted by
 * getResourceUsage().memory_usage_bytes).  One process-wide cache; keys are the caller's CacheKey::toString().
 * Entries are pinned while a caller holds them (get / put return pinned); only unpinned entries are evicted,
 * least recently used first; an expired entry that is still pinned is freed at its last release.
 * ---------------------------------------------------------------------------------- */
#define B200_CACHE_CORPUS 0   /* b200_corpus *, freed with b200_corpus_free */
#define B200_CACHE_INDEX 1    /* b200_index *,  freed with b200_index_free */
#define B200_CACHE_BM25 2     /* b200_bm25 *,   freed with b200_bm25_free */
#define B200_CACHE_OPAQUE 3   /* caller-defined object, freed with the deleter passed to b200_cache_put_opaque */
/* VICacheManager::setCacheSize -> updateMaxWeight: shrinking evicts unpinned entries at once */
int b200_cache_set_capacity(uint64_t bytes);
/* VICacheManager::get: B200_OK (pinned handle in *handle, its kind in *kind) or B200_ERR_NOT_FOUND */
int b200_cache_get(const char *key, void **handle, int *kind);
/* VICacheManager::put / load (getOrSet): inserts `handle` weighing `bytes` and pins it; if the key is already
 * resident, *resident is the EXISTING pinned handle and `handle` stays the caller's (free it).  B200_ERR_NOMEM when
 * it does not fit even after evicting every unpinned entry (ownership stays with the caller). */
int b200_cache_put(const char *key, int kind, void *handle, uint64_t bytes, void **resident);
int b200_cache_put_opaque(const char *key, void *handle, uint64_t bytes, void (*deleter)(void *), void **resident);
/* drop one pin taken by get / put.  Pass the handle that get / put returned: if the key was expired while pinned and put
 * again (index rebuilt under the same CacheKey), two generations exist, and only the handle tells whose pin this is.
 * b200_cache_release(key) without a handle releases the live entry first and is only safe without such re-puts. */
int b200_cache_release_handle(const char *key, const void *handle);
int b200_cache_release(const char *key);
/* VICacheManager::forceExpire -> tryRemove: freed now, or at the last release if pinned */
int b200_cache_expire(const char *key);
/* removes every entry whose key starts with `prefix` (a dropped table or part: removeOldParts); returns how many */
int b200_cache_expire_prefix(const char *prefix, int64_t *out_removed);
/* VICacheManager::countItem and the CurrentMetrics counters */
int b200_cache_stats(uint64_t *capacity, uint64_t *used, uint64_t *items, uint64_t *hits, uint64_t *misses,
                     uint64_t *evictions);
/* getResourceUsage().memory_usage_bytes of a resident object (rows + side arrays / lists + codes), for `bytes` above.
 * A binary corpus counts 4 bytes per row for its per-row popcounts (used by the tensor-core path). */
int b200_corpus_memory_bytes(const b200_corpus *c, uint64_t *out_bytes);
int b200_index_memory_bytes(const b200_index *ix, uint64_t *out_bytes);
/* pinned host bytes of an index's fp32 rows in host placement (keep_raw=2), 0 otherwise; b200_index_memory_bytes counts HBM
 * only, so it does not include them */
int b200_index_host_memory_bytes(const b200_index *ix, uint64_t *out_bytes);

/* ------------------------------------------------------------------------------------
 * Filter bitmaps and decoupled-part row-id maps (VIWithMeta::{row_ids_map, inverted_row_ids_map,
 * inverted_row_sources_map}, VectorIndex/Cache/VICacheObject.h:40-117).
 * ---------------------------------------------------------------------------------- */
/* Device-resident filters (the filtered-search fast path): build the DenseBitmap in HBM from the surviving _part_offset values
 * of the PREWHERE pipeline (getFilterFromPipeline, ...SelectWithHybridSearchProcessor.cpp:906-934) or from the _row_exists
 * bytes of a lightweight delete (MergeTreeVSManager.cpp:1435-1460), intersect there, and pass the result as d_alive_bits to the
 * *_search_device / b200_sharded_* calls.  Buffers: (nbits + 7) / 8 bytes rounded up to a multiple of 4, 4-byte aligned. */
int b200_bitmap_from_offsets_device(const uint64_t *d_offsets, int64_t n, int64_t nbits, uint8_t *d_out_bits, void *stream);
int b200_bitmap_from_row_exists_device(const uint8_t *d_row_exists, int64_t n, uint8_t *d_out_bits, void *stream);
int b200_bitmap_and_device(const uint8_t *d_a, const uint8_t *d_b, int64_t nbits, uint8_t *d_out, void *stream);
/* Search::intersectDenseBitmaps (VIWithDataPart.cpp:908): out = a & b */
int b200_bitmap_and(const uint8_t *a, const uint8_t *b, int64_t nbits, uint8_t *out);
/* getRealBitmap (VectorIndex/Utils/VIUtils.cpp:479-497): filter over the merged part -> bitmap over this old part */
int b200_real_bitmap(const uint8_t *filter_bits, int64_t n_new_rows, const uint64_t *inverted_row_ids_map,
                     const uint8_t *inverted_row_sources_map, uint32_t own_id, int64_t total_vec, uint8_t *out_bits);
/* VIWithColumnInPart::transferToNewRowIds (VIWithDataPart.cpp:56-68), in place */
int b200_remap_labels(const uint64_t *row_ids_map, int64_t map_len, int64_t *labels, int64_t n);
/* VIWithColumnInPart::TransferToOldRowIds (VIWithDataPart.cpp:69-126): order-preserving filter + map */
int b200_transfer_to_old_row_ids(const int64_t *new_ids, const float *new_dis, int64_t num_candidates,
                                 const uint64_t *inverted_row_ids_map, const uint8_t *inverted_row_sources_map, int64_t map_len,
                                 uint32_t own_id, int64_t *out_ids, float *out_dis, int64_t *out_n);

/* ------------------------------------------------------------------------------------
 * BM25 full-text search (Boundary B).  Replaces the TANTIVY::ffi_* calls of TantivyIndexStore
 * (Storages/MergeTree/TantivyIndexStore.cpp): ffi_index_multi_column_docs :742,
 * ffi_index_writer_commit :824, ffi_bm25_search :908/:939, ffi_get_doc_freq :962,
 * ffi_get_total_num_docs :974, ffi_get_total_num_tokens :986.  One index per part, resident
 * in HBM; tantivy-0.21 BM25 and "default" tokenizer semantics; results are score-descending,
 * ties to the smaller doc (tantivy TopDocs).
 * ---------------------------------------------------------------------------------- */
typedef struct b200_bm25 b200_bm25;
int b200_bm25_create(uint32_t n_fields, b200_bm25 **out);
int b200_bm25_free(b200_bm25 *ix);
/* one row: add_doc(row_id) then add_text(field, text) per value (several per field for Array(String)) */
int b200_bm25_add_doc(b200_bm25 *ix, uint64_t row_id);
int b200_bm25_add_text(b200_bm25 *ix, uint32_t field, const char *text);
int b200_bm25_commit(b200_bm25 *ix);
/* ffi_load_index_reader / the index files of a part (TantivyIndexStore.cpp:646-686): one self-describing file ("B2TX" v1;
 * tantivy's segment files cannot be reproduced without the crate); load validates, uploads to HBM and returns a committed index */
int b200_bm25_save(b200_bm25 *ix, const char *path);
int b200_bm25_load(const char *path, b200_bm25 **out);
int b200_bm25_total_docs(const b200_bm25 *ix, uint64_t *out);
int b200_bm25_total_tokens(const b200_bm25 *ix, uint32_t field, uint64_t *out);
int b200_bm25_doc_freq(const b200_bm25 *ix, uint32_t field, const char *term, uint64_t *out);
/* distinct lowercase terms of a sentence, NUL-separated, in tokenisation order */
int b200_bm25_query_terms(const char *sentence, char *buf, size_t buf_len, uint32_t *out_n);
/* stat_*: table-wide statistics (ReadWithHybridSearch::getStatisticForTextSearch,
 * VectorIndex/Processors/ReadWithHybridSearch.cpp:89-209), used iff stat_total_docs > 0:
 * stat_total_tokens[n_fields of the index], stat_doc_freq[q][fq * 64 + term_index]. */
int b200_bm25_search(b200_bm25 *ix, const char *sentence, const uint32_t *fields, uint32_t n_fields_q, uint32_t topk,
                     const uint8_t *alive_bits /*over row ids*/, int use_filter, int operator_or, uint64_t stat_total_docs,
                     const uint64_t *stat_total_tokens, const uint64_t *stat_doc_freq, uint64_t *out_rows,
                     float *out_scores, uint32_t *out_n);
/* roofline inputs of the last batch on this index: scoring-kernel ms (CUDA events), wall ms inside the C call, postings walked */
int b200_bm25_last_timing(b200_bm25 *ix, double *kernel_ms, double *call_ms, uint64_t *postings);
int b200_bm25_search_batch(b200_bm25 *ix, const char *const *sentences, int64_t nq, const uint32_t *fields,
                           uint32_t n_fields_q, uint32_t topk, const uint8_t *alive_bits, int use_filter, int operator_or,
                           uint64_t stat_total_docs, const uint64_t *stat_total_tokens, const uint64_t *stat_doc_freq,
                           uint64_t *out_rows /*[nq][topk]*/, float *out_scores, uint32_t *out_counts /*[nq]*/);

/* ------------------------------------------------------------------------------------
 * Hybrid-search fusion, batched.  Replaces RankFusion / RelativeScoreFusion
 * (VectorIndex/Utils/HybridSearchUtils.cpp:164-274) + the final ordering of
 * MergeTreeHybridSearchManager::hybridSearch (VectorIndex/Storages/MergeTreeHybridSearchManager.cpp:108-171).
 * fusion_type 0 = RSF (fusion_weight, vector_scan_direction 1 asc / -1 desc), 1 = RRF (fusion_k).
 * Candidate lists are [nq][stride] arrays (already globally ordered) with per-query counts;
 * outputs [nq][top_k], fused score descending, ties in ascending (shard, part, label) order.
 * ---------------------------------------------------------------------------------- */
int b200_hybrid_fusion_batch(int fusion_type, int64_t nq, const uint32_t *vec_shard, const uint64_t *vec_part,
                             const uint64_t *vec_label, const float *vec_score, const uint32_t *vec_count, int64_t vec_stride,
                             const uint32_t *txt_shard, const uint64_t *txt_part, const uint64_t *txt_label,
                             const float *txt_score, const uint32_t *txt_count, int64_t txt_stride, float fusion_weight,
                             uint64_t fusion_k, int vector_scan_direction, uint32_t top_k, uint32_t *out_shard,
                             uint64_t *out_part, uint64_t *out_label, float *out_score, uint32_t *out_count);

#ifdef __cplusplus
}
#endif
#endif /* B200_SEARCH_H */
