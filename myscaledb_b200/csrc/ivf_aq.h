// ivf_aq.h -- what ivf.cu and ivf_aq.cu share: the parameters of the per-row scatter into the page pool (the AQ encoder of
// an added chunk walks the same list-sorted rows to the same slots) and the anisotropic PQ training / encoding entry points.
#pragma once
#include <vector>

#include "common.cuh"

namespace b200 {

constexpr int kPageRows = 256;

// One warp per row of the list-sorted chunk: convert / encode the row into its pool slot, record its id and norm term.
struct ScatterParams {
    const float *rows;          // chunk rows fp32 [n][stride] (cosine: already unit length)
    int64_t stride;
    const uint32_t *sorted_list;  // [n] list of sorted element i
    const uint32_t *sorted_row;   // [n] chunk row of sorted element i
    const uint32_t *seg_start, *new_base, *first_new_seq, *list_len, *tail_page;
    uint32_t id_base;
    int64_t n;
    int d, d_pad64;
    int l2;
    // bf16 payload
    __nv_bfloat16 *pool;
    // SQ8 payload
    const float *sq_lo, *sq_inv_step, *sq_step;   // per dimension
    // PQ payload
    const float *centroids;     // [nlist][d]
    const float *pq;            // [m][256][dsub] fp32 (nearest-centroid search)
    const __nv_bfloat16 *pq_bf16;  // values the scan kernel will see (null: the fp32 ones, table look-up scan)
    int m, dsub, pq_bits;          // pq_bits 4: pq is [m][16][dsub], codes two per byte (code j in byte j / 2, even j low)
    uint8_t *codes;
    int code_bytes;
    float *row_bias;
    uint32_t *row_ids;
    int payload;
    // binary payload: rows [n][stride] bytes -> pool bytes [page][row_pad / kb_w][256][kb_w]
    const uint8_t *brows;
    uint8_t *bpool;
    int row_bytes, row_pad, kb_w;
};

__device__ __forceinline__ uint32_t pool_row_of(const ScatterParams &p, uint32_t l, uint32_t pos) {
    const uint32_t seq = pos / kPageRows;
    const uint32_t page = seq < p.first_new_seq[l] ? p.tail_page[l] : p.new_base[l] + (seq - p.first_new_seq[l]);
    return page * kPageRows + (pos % kPageRows);
}

// Anisotropic PQ (ivf_aq.cu).  The longest sub-vector the codebook update solves for.
constexpr int kAqMaxDsub = 64;

// Training sample of the codebook iterations: rows x [n][d] as indexed (unit length under cosine), their lists, the
// coarse centroids [nlist][d] and the k-means codebooks pq [m][ncw][dsub], updated in place.
struct AqTrain {
    const float *x;
    int64_t n;
    int d, m, dsub, ncw;
    const uint32_t *list;
    const float *centroids;
    float *pq;
    double eta;
};
// eta and the mean sample loss after the k-means codebooks, then after each iteration, appended to *loss
int aq_train_codebooks(const AqTrain &t, std::vector<double> *loss, cudaStream_t s);
// re-encodes the rows scatter_rows_kernel just placed (its nearest-codeword codes are the start) with the anisotropic loss
int aq_encode_chunk(const ScatterParams &p, double eta, cudaStream_t s);
// dynamic shared memory of the per-row encoder: 0 when one row of d dims does not fit
size_t aq_encoder_smem(int d, int m);

}  // namespace b200
