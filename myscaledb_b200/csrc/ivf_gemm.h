// ivf_gemm.h -- work items and parameters of the grouped tensor-core IVF scan (ivf_gemm_sm90.cu), built by ivf.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200 {

// TMA: bf16 rows as stored | PQ / SQ8: codes decoded by extra warps | B1: binary rows (bytes), wgmma .b1 AND + popcount
enum { IVF_PRODUCER_TMA = 0, IVF_PRODUCER_PQ = 1, IVF_PRODUCER_SQ8 = 2, IVF_PRODUCER_B1 = 3 };

// queries [q_begin, q_begin + q_count) of the list-sorted pair array x pages [page_begin, page_begin + page_count) of one list
struct IvfGemmItem {
    uint32_t q_begin;     // first row of the gathered query buffer = first pair of this item
    uint32_t q_count;     // 1..128
    uint32_t page_begin;  // absolute index into list_pages
    uint32_t page_count;  // >= 1
    uint32_t row_limit;   // rows of the list from the item's first page on: rows valid in tile j = min(256, row_limit - 256 j)
    uint32_t chunk;       // which row chunk of its list this item is (selects the partial list of every pair)
};

struct IvfGemmParams {
    const IvfGemmItem *items;
    const int *n_items_ptr;           // device scalar written by the planning kernel
    const uint32_t *list_pages;       // page ids, list after list
    const float *row_bias;            // [pool rows] L2: ||y||^2 (PQ: 2<c, r^> + ||r^||^2); binary: popc(y); null for IP / cosine
    const uint32_t *row_ids;          // [pool rows] row id inside the part
    const uint8_t *alive;             // LSB-first bitmap over row ids, or null
    const uint32_t *pair_part_base;   // [pairs] first partial list of pair i; chunk c of its list writes base + c
    float *part_keys;                 // [parts][k] unsorted
    uint32_t *part_ids;
    float *part_worst;                // [parts] worst kept key when the list is full, else FLT_MAX
    float scale_const;                // -1 IP / cosine, -2 L2 and Hamming, 1 Jaccard (only marks a row live)
    float *list_keys_gmem;            // scratch when the per-thread lists do not fit in shared memory: [grid][list_cap_for(k)][128]
    uint32_t *list_ids_gmem;
    int d_pad, k;                     // d_pad: elements per query / pool row (binary: bytes, row_pad)
    int producer;                     // IVF_PRODUCER_*
    // binary payload: pages are [page][d_pad / kb_w][256 rows][kb_w bytes], kb_w = min(128, row bytes rounded up to 16)
    int kb_w, jaccard;
    const float *pair_popc;           // Jaccard: popc(q) of every sorted pair
    // code payloads
    const uint8_t *codes;             // [pool rows][code_bytes]
    const void *codebook_bf16;        // PQ: [m][256][dsub] bf16
    int code_bytes, m, dsub, codebook_bytes;
    const float *lut;                 // PQ table look-up scan: [nq][m][256] fp32, <q_j, codebook_j[e]> (needs sorted_pair, nprobe)
    // filled in by the launcher
    // Per-query bound shared by all the work items of a launch (nprobe > 1): query_bound[q] is the smallest k-th key
    // (order-preserving u32 encoding, 0xffffffff = none yet) any FULL partial list of query q has published, in absolute key space
    // (item key + pair_const).  Items read it once per page and filter with it: far lists stop inserting once a near list is done.
    uint32_t *query_bound;            // [nq] or null
    const uint32_t *sorted_pair;      // [n_pairs] sorted position -> original pair index (query = pair / nprobe)
    const float *pair_const;          // [n_pairs]
    int nprobe;
    int stages, lists_in_smem, codebook_smem_off, coop_smem_off, coop_enabled;
};

// queries_bf16: gathered query rows [n_query_rows][d_pad] (bf16; binary: bytes); pool_bf16: page pool [pool_rows][d_pad] (bf16 and
// binary payloads only)
cudaError_t launch_ivf_gemm_topk(const IvfGemmParams &p, const void *queries_bf16, int64_t n_query_rows, const void *pool_bf16,
                                 int64_t pool_rows, int grid, cudaStream_t s, const char **err_detail);

// whether a PQ codebook of codebook_bytes (m * 256 * dsub bf16) fits in shared memory beside the smallest (2-stage) operand
// ring of the decoding scan, by the launcher's own arithmetic: the scan of a wider codebook cannot be launched
bool ivf_pq_codebook_fits(int64_t codebook_bytes);

// PQ with d / M outside {1, 2, 4, 8} (ivf_pq_lut_sm90.cu): the same work items and partial lists, scanned by table look-up.
// launch_pq_lut fills lut_out [nq][m][256] = <q_j, codebook_j[e]> (fp32) from prepared queries [nq][d_pad] and the fp32 codebook
// [m][256][dsub]; launch_ivf_pq_lut_topk scans with p.lut = that table (p.stages is set by the launcher: table buffers)
cudaError_t launch_pq_lut(const float *queries, int64_t nq, int d_pad, const float *codebook, int m, int dsub, float *lut_out, cudaStream_t s);
cudaError_t launch_ivf_pq_lut_topk(const IvfGemmParams &p, int grid, cudaStream_t s, const char **err_detail);

// whether the look-up scan takes m sub-quantisers: M <= 128, and one M x 1 KB table beside the k = 1024 lists and the candidate
// buffer in shared memory, by the launcher's own arithmetic
bool ivf_pq_lut_fits(int m);

// PQ with 4-bit codes (ivf_pq4_sm90.cu): codes nibble-packed (code j in byte j / 2, even j low), codebook [m][16][dsub] fp32.
// launch_pq4_lut fills lut_out [nq][m][16] = <q_j, codebook_j[e]> (fp32); launch_ivf_pq4_topk scans the same work items into
// the same partial lists with p.lut = that table
cudaError_t launch_pq4_lut(const float *queries, int64_t nq, int d_pad, const float *codebook, int m, int dsub, float *lut_out, cudaStream_t s);
cudaError_t launch_ivf_pq4_topk(const IvfGemmParams &p, int grid, cudaStream_t s, const char **err_detail);

// the 4-bit scan's limit on M, and whether it takes m: one query's M x 64 B table beside a k = 1024 list pair and the
// candidate buffer in shared memory, by the launcher's own arithmetic
int ivf_pq4_max_m();
bool ivf_pq4_fits(int m);

}  // namespace b200
