// kernels.h -- parameter blocks and host launchers shared between the .cu files.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200 {

struct ScanParams {
    const void *corpus;      // [n][row_bytes]
    const float *queries;    // device fp32 [nq][d_pad] (cosine: pre-normalised)
    const float *row_scale;  // cosine: -1/||row|| (-1 for rows with sum sq < FLT_EPSILON), else null (= -1)
    const uint8_t *alive;    // LSB-first bitmap or null
    float *part_keys;        // [nq][gridDim.x][k]
    uint32_t *part_ids;
    int64_t n, nq;
    int64_t row_bytes;
    int d_pad, k, group;
    int l2, bf16;
    // fused single-launch form (small batches on a resident corpus: the call is latency-bound): raw queries [nq][q_dim]
    // are padded (and for cosine normalised) while they are staged, the LAST block of a query tile to finish merges every
    // block's partial list and writes the final result (mapped pinned host memory) -- one launch, no pad / merge kernels
    int fused;               // 0 = plain scan (queries pre-padded, partial lists only)
    int q_dim;               // fused: row length of `queries`
    int cosine;              // fused: normalise the staged queries (skip sum sq < FLT_EPSILON), output 1 + key
    int out_mode, ip_min_quirk;
    int64_t id_offset;
    unsigned int *tickets;   // fused: [gridDim.y] zeroed counters (the last block resets its own)
    float *out_dis;          // fused: [nq][k]
    int64_t *out_ids;
    volatile unsigned int *done_flag;  // fused, nullable: set to done_value once every query tile has been written
    unsigned int done_value;
    unsigned int *tiles_done;          // fused: one zeroed counter (reset by the last tile)
    int q_inline;                      // fused: the queries travel in the kernel parameters (nq * q_dim <= 256 floats)
    int stage_cap;                     // fused: candidates (gridDim.x * k) the last block may stage in shared memory, 0 = none (set by the launcher)
    float qinline[256];
};

struct BinaryScanParams {
    const uint8_t *corpus;   // [n][nbytes]
    const uint8_t *queries;  // [nq][nbytes]
    const uint8_t *alive;
    float *part_keys;
    uint32_t *part_ids;
    int64_t n, nq;
    int nbytes, k, jaccard;
};

enum { kOutKey = 0, kOutNeg = 1, kOutOnePlus = 2, kOutAddQ = 3, kOutCosQ = 4 };

struct MergeParams {
    const void *in_keys;     // float
    const void *in_ids;      // uint32 (internal partials) or int64 (external lists)
    int64_t list_stride, q_stride;
    int64_t id_list_stride;  // 0 = same as list_stride (element units of the id type)
    int n_lists, k_in, k;
    int64_t nq;
    int descending;          // external only
    int tie_mode;            // external only: 0 = smaller 64-bit id first, 1 = the reference's multimap insertion order
    int32_t *out_list;       // external, tie_mode 1: source list of every output entry (nullable)
    int out_mode;            // kOut*
    int ip_min_quirk;        // part-scan IP: drop scores <= FLT_MIN
    const float *q_add;      // kOutAddQ: ||q||^2 per query; kOutCosQ: -(1/||q||) per query
    int64_t id_offset;
    float *out_dis;
    int64_t *out_ids;
};

size_t scan_smem_bytes(int qt, int d_pad, int k);
cudaError_t launch_flat_scan(const ScanParams &p, int qt, int blocks_x, cudaStream_t s);
cudaError_t launch_binary_scan(const BinaryScanParams &p, int blocks_x, cudaStream_t s);
cudaError_t launch_topk_merge(const MergeParams &p, bool external, cudaStream_t s);
// exact squared-L2 of the k winners of every query (direct differences, fp32) + re-order by (distance, id); k <= 1024
cudaError_t launch_rescore_l2(const void *corpus, int bf16, int64_t row_bytes, int d_pad, const float *queries, int64_t nq, int64_t id_offset,
                              int k, float *dis, int64_t *ids, cudaStream_t s);

// ---- wgmma GEMM + fused top-k (ip_gemm_sm90.cu): bf16 rows, fp32 rows as 3xTF32, or binary rows ------
struct GemmTopkParams {
    const void *corpus_bf16;   // [n][d_pad] bf16, d_pad % 64 == 0 (binary kernel: [n][d_pad] bytes, d_pad % 16 == 0)
    const void *queries_bf16;  // [nq_pad][d_pad] bf16, nq_pad % 128 == 0 (3xTF32 kernel: fp32 hi plane; corpus_bf16 = fp32 rows;
                               // binary kernel: zero-padded query bytes)
    const void *queries_lo;    // 3xTF32 kernel only: fp32 lo plane [nq_pad][d_pad]
    const float *row_scale;    // per corpus row multiplier a[j] or null (= scale_const)
    float scale_const;         // -1 for IP, -2 for L2
    const float *row_bias;     // per corpus row addend b[j] or null (=0); binary kernel: popcount of row j (both metrics)
    const uint8_t *alive;      // LSB-first bitmap or null
    const float *q_popc;       // binary Jaccard: popcount of each query of the batch [nq_valid]
    int jaccard;               // binary kernel: Jaccard keys (else Hamming: scale_const = -2, row_bias = popcounts)
    float *part_keys;          // [W = gemm_consumer_warpgroups * gridDim.x / q_tiles partial lists][nq_pad][k]: consumer warpgroup w of
                               // the CTA (worker, query tile) writes list  worker * warpgroups + w
    uint32_t *part_ids;
    float *list_keys_gmem;     // scratch for lists that do not fit in shared memory: [W * q_tiles][list_cap_for(k)][128]
    uint32_t *list_ids_gmem;
    uint32_t *query_bound;     // [nq_pad] 0xffffffff-filled: the best k-th key any list of the query has reached (bound_encode)
    int64_t n;
    int nq_pad, d_pad, k;
    int nq_valid;              // queries actually in the batch (rows past it are padding)
    int q_tiles;               // nq_pad / 128
    int *progress;             // [grid / q_tiles][q_tiles] zeroed pacing counters, or null
    int stages;                // smem ring depth (filled in by the launcher)
    int lists_in_smem;         // per-thread top-k lists in shared memory (else global scratch); set by the launcher
    int sync_slack;            // tiles a CTA may run ahead of the slowest sharer of its corpus tiles
};
// per-thread top-k lists of the IVF scan may live in shared memory up to twice this k (the launcher checks the fit)
constexpr int kGemmSmemK = 128;
// Per-thread top-k lists (gemm_common.cuh, ThreadTopK) take one of two forms, chosen by k alone:
//  * rescan (k < list_tourn_min_k): k slots; an insert rescans all k entries for the new worst;
//  * tournament (k >= list_tourn_min_k): k entries + one (key, id) slot per group of 8 (k <= 64) or 16 entries holding the
//    group's worst; an insert rescans one group and the group worsts instead of all k entries.  16 keeps k = 100 at 107 slots.
// The crossover k = 17 was chosen on an earlier GPU and is not re-measured on the H100.
constexpr int list_tourn_min_k = 17;
__host__ __device__ inline int list_tourn_group(int k) { return k <= 64 ? 8 : 16; }
__host__ __device__ inline int list_cap_tourn(int k) { return k + (k + list_tourn_group(k) - 1) / list_tourn_group(k); }
// slots of a per-thread list of this k
__host__ __device__ inline int list_cap_for(int k) { return k < list_tourn_min_k ? k : list_cap_tourn(k); }
int gemm_topk_grid(int q_tiles, int64_t n, int num_sms);
// Consumer warpgroups per CTA of gemm_topk_kernel.  bf16 and binary rows: two, each owning one 128-row half of every 256-row
// corpus tile and its own per-query lists, so a CTA publishes two partial lists per query.  fp32 rows (3xTF32): one, which
// walks both halves (its hi / lo operand planes leave no room for a stage that holds both).
constexpr int gemm_consumer_warpgroups(bool f32x3) { return f32x3 ? 1 : 2; }
// returns cudaSuccess or an error; tensor maps are encoded inside
cudaError_t launch_gemm_topk(const GemmTopkParams &p, int grid, cudaStream_t s, const char **err_detail);
// fp32 rows on the tensor cores with fp32-level accuracy (3xTF32, queries pre-split into hi / lo planes)
cudaError_t launch_split_tf32(const float *src, int64_t n_src, int d_pad, float *hi, float *lo, int64_t n_pad, cudaStream_t s);
cudaError_t launch_gemm3_topk(const GemmTopkParams &p, int grid, cudaStream_t s, const char **err_detail);
// binary rows on the tensor cores (wgmma .b1 AND + popcount): Hamming or Jaccard keys, exact
cudaError_t launch_gemm_b1_topk(const GemmTopkParams &p, int grid, cudaStream_t s, const char **err_detail);

// ---- pre-filtered exact search (prefilter.cu) -----------------------------------------
// scratch the compaction of an n-bit bitmap needs (per-word counts, their exclusive scan, CUB storage)
size_t prefilter_compact_temp_bytes(int64_t n);
// d_alive: LSB-first bitmap, 4-byte aligned, readable up to the end of its last 32-bit word (bits >= n are ignored) ->
// d_ids: the ascending row ids of its set bits (as many as it has; the caller counted them)
cudaError_t launch_prefilter_compact(const uint8_t *d_alive, int64_t n, uint32_t *d_ids, void *temp, cudaStream_t s);
// out_rows[i] = rows[ids[i]] (row_bytes each), and the same for the side arrays that are not null
cudaError_t launch_prefilter_gather(const void *rows, int64_t row_bytes, const float *scale, const float *bias, const uint32_t *ids,
                                    int64_t m, void *out_rows, float *out_scale, float *out_bias, cudaStream_t s);
// ids[i] = ids[i] >= 0 ? alive_ids[ids[i]] + id_offset : -1
cudaError_t launch_prefilter_map_ids(const uint32_t *alive_ids, int64_t id_offset, int64_t *ids, int64_t count, cudaStream_t s);

// ---- host ingest (ingest.cu): pageable host memory -> device through a multi-threaded pinned ring; returns a B200_* code
int staged_h2d(void *dst, const void *src, size_t bytes, int device, cudaStream_t s);

// ---- elementwise prep kernels (prep.cu) --------------------------------------------
cudaError_t launch_f32_to_bf16_rows(const float *src, int d, void *dst, int d_pad, int64_t n, cudaStream_t s);
cudaError_t launch_pad_rows_f32(const float *src, int d, float *dst, int d_pad, int64_t n, cudaStream_t s);
// per-row sum of squares (fp32 accumulate) of a [n][d_pad] corpus; mode 0: out = ss, mode 1: out = -(ss<eps ? 1 : 1/sqrt(ss))
cudaError_t launch_row_norms(const void *rows, int bf16, int d_pad, int64_t n, int mode, float *out, cudaStream_t s);
// normalise fp32 query rows in place (cosine), skipping rows with ss < FLT_EPSILON
cudaError_t launch_normalize_rows_f32(float *rows, int d_pad, int64_t n, cudaStream_t s);
// number of set bits of each binary row [n][row_bytes], as an exact float
cudaError_t launch_popc_rows(const uint8_t *rows, int64_t row_bytes, int64_t n, float *out, cudaStream_t s);

}  // namespace b200
