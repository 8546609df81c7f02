// ivf.cu -- K5/K6: the inverted-file index family, its streamed GPU build, and the exact second stage.
//
// Replaces Search::createVectorIndex / Search::VectorIndex<...>::{build, search, computeTopDistanceSubset, serialize, load}
// for the index types the reference reaches through VIWithColumnInPart (reference:
// src/VectorIndex/Common/VIWithDataPart.cpp:416-430 create, :131 build, :858-957 search, :838-856 second stage,
// :451-525 / :578-764 serialize / load) and MergeTreeVSManager::executeSecondStageVectorScan
// (src/VectorIndex/Storages/MergeTreeVSManager.cpp:510-630).  The reference's implementations live in the un-vendored
// search-index library (Faiss IVF*, hnswlib, ScaNN) and the closed-source MSTG; the algorithms here are the published
// IVF ones, the layout and the execution model are ours:
//   * coarse quantiser: nlist fp32 centroids, k-means on device (assignment = exact top-1 search of the centroid table
//     on the tensor cores, 3xTF32);
//   * PAGED inverted lists: a page = 256 consecutive rows of one list in a pre-reserved pool (exactly one tensor-core tile);
//     `add` appends chunk after chunk (assign -> sort by list -> allocate pages by prefix sums -> scatter), nothing is
//     ever compacted or moved, so 100 M x 768 rows stream through a few GB of scratch (VIPartReader's chunked build);
//   * payload of a row: bf16 vector (IVFFLAT / MSTG-class first stage), one byte per dimension (IVFSQ) or m PQ codes of
//     the residual (IVFPQ / SCANN-class); + its row id and, for L2, the norm term of the expanded distance;
//   * search: coarse top-nprobe, then ALL (query, list) pairs of the batch are radix-sorted by list and cut into work
//     items (<= 128 queries x a run of pages) for the grouped tensor-core scan of ivf_gemm_sm90.cu, so a list is read
//     from HBM once per batch however many queries probe it; per-pair partial lists are merged per query;
//   * optional fp32 rows in id order (`keep_raw`) for the exact second stage (refine_kernel, warp per candidate).
// Binary indexes (BINARYIVF and the BINARYHNSW / BINARYMSTG it serves) use the same pool, pages, plan and merge: the coarse
// quantiser is trained by k-majority (Hamming assignment, per-bit majority; integer work, so deterministic), a page holds the
// row bytes k-block-major, and the list rows are exact, so there is no second stage.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include <cub/cub.cuh>

#include "common.cuh"
#include "graph.h"
#include "ivf_aq.h"
#include "ivf_gemm.h"
#include "ivf_opq.h"
#include "kernels.h"

namespace b200 {

// ------------------------------------------------------------------------------------
// k-means assignment: for every point the nearest centroid under L2 (argmin ||c||^2 - 2 x.c).
// 64 points x 64 centroids per tile, K chunks of 16, 4x4 register micro-tiles.
// ------------------------------------------------------------------------------------
constexpr int KA_T = 64, KA_K = 16;

__global__ void __launch_bounds__(256) kmeans_assign_kernel(const float *__restrict__ x, int64_t n, int64_t x_stride, int d,
                                                            const float *__restrict__ c, int nc, const float *__restrict__ cnorm,
                                                            uint32_t *__restrict__ out_idx, float *__restrict__ out_dist) {
    __shared__ float xs[KA_K][KA_T + 4];
    __shared__ float cs[KA_K][KA_T + 4];
    __shared__ float best_d[KA_T][17];
    __shared__ uint32_t best_i[KA_T][17];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;  // 16 x 16 threads, each 4 points x 4 centroids
    const int64_t p0 = (int64_t)blockIdx.x * KA_T;
    float run_d[4];
    uint32_t run_i[4];
#pragma unroll
    for (int a = 0; a < 4; a++) {
        run_d[a] = FLT_MAX;
        run_i[a] = 0;
    }
    for (int c0 = 0; c0 < nc; c0 += KA_T) {
        float acc[4][4];
#pragma unroll
        for (int a = 0; a < 4; a++)
#pragma unroll
            for (int b = 0; b < 4; b++) acc[a][b] = 0.f;
        for (int k0 = 0; k0 < d; k0 += KA_K) {
            for (int i = threadIdx.x; i < KA_T * KA_K; i += 256) {
                const int r = i / KA_K, kk = i % KA_K;
                const int64_t pr = p0 + r;
                xs[kk][r] = (pr < n && k0 + kk < d) ? x[pr * x_stride + k0 + kk] : 0.f;
                const int cr = c0 + r;
                cs[kk][r] = (cr < nc && k0 + kk < d) ? c[(int64_t)cr * d + k0 + kk] : 0.f;
            }
            __syncthreads();
#pragma unroll
            for (int kk = 0; kk < KA_K; kk++) {
                float xv[4], cv[4];
#pragma unroll
                for (int a = 0; a < 4; a++) xv[a] = xs[kk][ty * 4 + a];
#pragma unroll
                for (int b = 0; b < 4; b++) cv[b] = cs[kk][tx * 4 + b];
#pragma unroll
                for (int a = 0; a < 4; a++)
#pragma unroll
                    for (int b = 0; b < 4; b++) acc[a][b] = fmaf(xv[a], cv[b], acc[a][b]);
            }
            __syncthreads();
        }
#pragma unroll
        for (int a = 0; a < 4; a++)
#pragma unroll
            for (int b = 0; b < 4; b++) {
                const int cr = c0 + tx * 4 + b;
                if (cr < nc) {
                    const float dist = cnorm[cr] - 2.f * acc[a][b];
                    if (dist < run_d[a]) {  // ascending centroid order inside a thread: ties keep the smaller id
                        run_d[a] = dist;
                        run_i[a] = (uint32_t)cr;
                    }
                }
            }
    }
#pragma unroll
    for (int a = 0; a < 4; a++) {
        best_d[ty * 4 + a][tx] = run_d[a];
        best_i[ty * 4 + a][tx] = run_i[a];
    }
    __syncthreads();
    if (threadIdx.x < KA_T) {
        const int r = threadIdx.x;
        float bd = FLT_MAX;
        uint32_t bi = 0;
        for (int t = 0; t < 16; t++) {
            const float dv = best_d[r][t];
            const uint32_t iv = best_i[r][t];
            if (dv < bd || (dv == bd && iv < bi)) {
                bd = dv;
                bi = iv;
            }
        }
        if (p0 + r < n) {
            out_idx[p0 + r] = bi;
            if (out_dist) out_dist[p0 + r] = bd;
        }
    }
}

__global__ void kmeans_accumulate_kernel(const float *x, int64_t n, int64_t x_stride, int d, const uint32_t *idx, float *sums,
                                         uint32_t *counts) {
    const int64_t total = n * d;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / d;
        const int j = (int)(i - r * d);
        atomicAdd(&sums[(int64_t)idx[r] * d + j], x[r * x_stride + j]);
        if (j == 0) atomicAdd(&counts[idx[r]], 1u);
    }
}

__global__ void kmeans_update_kernel(float *c, const float *sums, const uint32_t *counts, int nc, int d) {
    const int64_t total = (int64_t)nc * d;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t cnt = counts[i / d];
        if (cnt) c[i] = sums[i] / (float)cnt;  // empty cluster: keep the previous centroid
    }
}

__global__ void rows_sqnorm_kernel(const float *c, int nc, int d, float *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nc) return;
    float s = 0.f;
    for (int j = 0; j < d; j++) s = fmaf(c[(int64_t)i * d + j], c[(int64_t)i * d + j], s);
    out[i] = s;
}

__global__ void gather_rows_kernel(const float *x, int64_t x_stride, const int64_t *pick, int64_t np, int d, float *out) {
    const int64_t total = np * d;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / d;
        out[i] = x[pick[r] * x_stride + (i - r * d)];
    }
}

// residual sub-vectors of one sub-quantiser: out[r][t] = x[r][j*dsub + t] - centroid[list[r]][j*dsub + t]
__global__ void residual_sub_kernel(const float *x, int64_t n, int64_t x_stride, const float *cent, const uint32_t *list, int d,
                                    int j, int dsub, float *out) {
    const int64_t total = n * dsub;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / dsub;
        const int t = (int)(i - r * dsub);
        out[i] = x[r * x_stride + j * dsub + t] - cent[(int64_t)list[r] * d + j * dsub + t];
    }
}

// pairs[2 i] = an empty cluster, pairs[2 i + 1] = a large one: the empty one becomes a nudged copy of the large one
__global__ void kmeans_split_kernel(float *c, const int *pairs, int d) {
    const int dst = pairs[2 * blockIdx.x], src = pairs[2 * blockIdx.x + 1];
    for (int j = threadIdx.x; j < d; j += blockDim.x) {
        const float v = c[(size_t)src * d + j];
        const float eps = (j & 1) ? 1.f / 1024.f : -1.f / 1024.f;
        c[(size_t)dst * d + j] = v * (1.f + eps) + eps * 1e-3f;
        c[(size_t)src * d + j] = v * (1.f - eps) - eps * 1e-3f;
    }
}

__global__ void iota_kernel(uint32_t *v, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] = (uint32_t)i;
}

static inline int gridsz(int64_t work, int threads = 256) {
    int64_t b = ceil_div(work, threads);
    return (int)std::max<int64_t>(1, std::min<int64_t>(b, 132 * 32));
}

// ------------------------------------------------------------------------------------
// build: chunk -> paged lists
// ------------------------------------------------------------------------------------
// nearest centroid ids -> u32 lists and per-list counts.  A row without one (id -1: no finite distance to any centroid) or
// flagged unusable gets `none`: 0 for the k-means of usable training rows, nlist for added rows (in no list; counted in
// cnt[nlist]).
__global__ void assign_to_u32_kernel(const int64_t *ids, int64_t n, const uint8_t *usable, uint32_t none, uint32_t *out, uint32_t *cnt) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t l = ids[i] < 0 || (usable && !usable[i]) ? none : (uint32_t)ids[i];
    out[i] = l;
    atomicAdd(&cnt[l], 1u);
}

// usable[r] = 1 when row r of x [n][d] is usable (warp_row_usable), else 0; one warp per row
__global__ void __launch_bounds__(256) row_usable_kernel(const float *x, int64_t n, int d, uint8_t *usable) {
    const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp_global; r < n; r += nwarps) {
        const bool ok = warp_row_usable(x + r * d, d);
        if (lane_id() == 0) usable[r] = ok ? 1 : 0;
    }
}

// Exclusive scan of per-thread partial sums across one 1024-thread CTA.
__device__ __forceinline__ uint32_t block_exclusive_scan_1024(uint32_t v, uint32_t *total) {
    typedef cub::BlockScan<uint32_t, 1024> Scan;
    __shared__ typename Scan::TempStorage tmp;
    uint32_t excl, tot;
    Scan(tmp).ExclusiveSum(v, excl, tot);
    __syncthreads();
    if (total) *total = tot;
    return excl;
}

// One CTA plans a chunk's page allocation: per list the rows arriving (cnt), where its segment starts in the sorted
// chunk, how many NEW pages it needs and their ids (prefix sum on top of *pages_used), and stamps the new pages.
struct AddPlan {
    const uint32_t *cnt;        // [nlist] rows of this chunk per list
    uint32_t *seg_start;        // [nlist] out: first index of the list's segment in the list-sorted chunk
    uint32_t *new_base;         // [nlist] out: first new page id of the list
    uint32_t *first_new_seq;    // [nlist] out: sequence number (page index inside the list) of its first new page
    const uint32_t *list_len;   // [nlist] rows already in the list
    uint32_t *page_owner, *page_seq;
    uint32_t *pages_used;       // in/out (device scalar)
    uint32_t pool_pages;
    int nlist;
    int *overflow;              // out: set when the pool is exhausted
};

__global__ void __launch_bounds__(1024) add_plan_kernel(const AddPlan p) {
    const int per = (p.nlist + 1023) / 1024;
    const int l0 = threadIdx.x * per, l1 = min(p.nlist, l0 + per);
    uint32_t rows = 0, pages = 0;
    for (int l = l0; l < l1; l++) {
        const uint32_t len = p.list_len[l], c = p.cnt[l];
        rows += c;
        pages += (len + c + kPageRows - 1) / kPageRows - (len + kPageRows - 1) / kPageRows;
    }
    uint32_t tot_pages = 0;
    uint32_t row_off = block_exclusive_scan_1024(rows, nullptr);
    uint32_t page_off = block_exclusive_scan_1024(pages, &tot_pages);
    const uint32_t used = *p.pages_used;
    __syncthreads();
    const bool fits = used + tot_pages <= p.pool_pages;
    for (int l = l0; l < l1; l++) {
        const uint32_t len = p.list_len[l], c = p.cnt[l];
        const uint32_t first = (len + kPageRows - 1) / kPageRows;
        const uint32_t need = (len + c + kPageRows - 1) / kPageRows - first;
        p.seg_start[l] = row_off;
        p.new_base[l] = used + page_off;
        p.first_new_seq[l] = first;
        if (fits)
            for (uint32_t t = 0; t < need; t++) {
                p.page_owner[used + page_off + t] = (uint32_t)l;
                p.page_seq[used + page_off + t] = first + t;
            }
        row_off += c;
        page_off += need;
    }
    if (threadIdx.x == 0) {
        if (fits) *p.pages_used = used + tot_pages;
        else *p.overflow = 1;
    }
}

__global__ void __launch_bounds__(256) scatter_rows_kernel(const ScatterParams p) {
    const int lane = threadIdx.x & 31;
    const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = warp_global; i < p.n; i += nwarps) {
        const uint32_t l = p.sorted_list[i], r = p.sorted_row[i];
        const uint32_t pos = p.list_len[l] + ((uint32_t)i - p.seg_start[l]);
        const uint32_t slot = pool_row_of(p, l, pos);
        const float *x = p.rows + (int64_t)r * p.stride;
        float acc = 0.f;
        if (p.payload == IVF_PRODUCER_TMA) {
            // k-block-major pages: element (row r of the page, dim j) at ((page * KB + j / 64) * 256 + r) * 64 + j % 64, so
            // that the 256 x 64 tile of one k-block is 32 KB contiguous in HBM (one DRAM-friendly TMA box per tile)
            const uint32_t page = slot / kPageRows, r_in = slot % kPageRows;
            const int kbc = p.d_pad64 / 64;
            __nv_bfloat16 *pbase = p.pool + (size_t)page * kPageRows * p.d_pad64;
            for (int j = lane; j < p.d_pad64; j += 32) {
                const __nv_bfloat16 b = __float2bfloat16_rn(j < p.d ? x[j] : 0.f);
                (void)kbc;
                pbase[((size_t)(j >> 6) * kPageRows + r_in) * 64 + (j & 63)] = b;
                const float v = __bfloat162float(b);
                acc = fmaf(v, v, acc);
            }
        } else if (p.payload == IVF_PRODUCER_SQ8) {
            uint8_t *dst = p.codes + (size_t)slot * p.code_bytes;
            for (int j = lane; j < p.code_bytes; j += 32) {
                uint32_t code = 128;  // padding decodes to 0
                if (j < p.d) {
                    const float t = rintf((x[j] - p.sq_lo[j]) * p.sq_inv_step[j]);
                    code = (uint32_t)fminf(fmaxf(t, 0.f), 255.f);
                    const float v = p.sq_lo[j] + (float)code * p.sq_step[j];   // the value this code stands for
                    acc = fmaf(v, v, acc);
                }
                dst[j] = (uint8_t)code;
            }
        } else if (p.pq_bits == 4) {
            // 4-bit PQ on the residual: lane handles code bytes lane, lane + 32, ..., each holding codes 2b (low nibble) and
            // 2b + 1 (high nibble); codes past M and the padding bytes stay 0
            uint8_t *dst = p.codes + (size_t)slot * p.code_bytes;
            const float *c = p.centroids + (size_t)l * p.d;
            for (int b = lane; b < p.code_bytes; b += 32) {
                uint32_t byte = 0;
                for (int h = 0; h < 2; h++) {
                    const int j = 2 * b + h;
                    if (j >= p.m) break;
                    const float *cb = p.pq + (size_t)j * 16 * p.dsub;
                    float bd = FLT_MAX;
                    uint32_t best = 0;
                    for (int e = 0; e < 16; e++) {
                        float s = 0.f;
                        for (int t = 0; t < p.dsub; t++) {
                            const float u = (x[j * p.dsub + t] - c[j * p.dsub + t]) - cb[e * p.dsub + t];
                            s = fmaf(u, u, s);
                        }
                        if (s < bd) {
                            bd = s;
                            best = (uint32_t)e;
                        }
                    }
                    // norm term of the expanded L2 with the fp32 codewords the look-up table is built from: 2 <c, r^> + ||r^||^2
                    const float *rv = cb + (size_t)best * p.dsub;
                    for (int t = 0; t < p.dsub; t++) acc = fmaf(rv[t], rv[t] + 2.f * c[j * p.dsub + t], acc);
                    byte |= best << (4 * h);
                }
                dst[b] = (uint8_t)byte;
            }
        } else {
            // PQ on the residual x - centroid[l]: lane handles sub-quantisers lane, lane + 32, ...
            uint8_t *dst = p.codes + (size_t)slot * p.code_bytes;
            const float *c = p.centroids + (size_t)l * p.d;
            for (int j = lane; j < p.code_bytes; j += 32) {
                uint32_t best = 0;
                if (j < p.m) {
                    const float *cb = p.pq + (size_t)j * 256 * p.dsub;
                    float bd = FLT_MAX;
                    for (int e = 0; e < 256; e++) {
                        float s = 0.f;
                        for (int t = 0; t < p.dsub; t++) {
                            const float u = (x[j * p.dsub + t] - c[j * p.dsub + t]) - cb[e * p.dsub + t];
                            s = fmaf(u, u, s);
                        }
                        if (s < bd) {
                            bd = s;
                            best = (uint32_t)e;
                        }
                    }
                    // norm term of the expanded L2 with the codebook values the scan sees: 2 <c, r^> + ||r^||^2 (bf16 for the
                    // tensor-core decoder, fp32 for the table look-up scan, which has no bf16 codebook)
                    const size_t cw = ((size_t)j * 256 + best) * p.dsub;
                    for (int t = 0; t < p.dsub; t++) {
                        const float rv = p.pq_bf16 ? __bfloat162float(p.pq_bf16[cw + t]) : p.pq[cw + t];
                        acc = fmaf(rv, rv + 2.f * c[j * p.dsub + t], acc);
                    }
                }
                dst[j] = (uint8_t)best;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) {
            p.row_ids[slot] = p.id_base + r;
            if (p.row_bias) p.row_bias[slot] = acc;
        }
    }
}

// Binary payload: one warp per row of the list-sorted chunk; the row bytes go to their k-block-major slot ([page][kb][256][kb_w],
// zero-padded to row_pad), the row's popcount to row_bias as an exact float.
__global__ void __launch_bounds__(256) scatter_bin_rows_kernel(const ScatterParams p) {
    const int lane = threadIdx.x & 31;
    const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = warp_global; i < p.n; i += nwarps) {
        const uint32_t l = p.sorted_list[i], r = p.sorted_row[i];
        const uint32_t pos = p.list_len[l] + ((uint32_t)i - p.seg_start[l]);
        const uint32_t slot = pool_row_of(p, l, pos);
        const uint8_t *x = p.brows + (int64_t)r * p.stride;
        const uint32_t page = slot / kPageRows, r_in = slot % kPageRows;
        uint8_t *pbase = p.bpool + (size_t)page * kPageRows * p.row_pad;
        int c = 0;
        for (int j = lane; j < p.row_pad; j += 32) {
            const uint32_t b = j < p.row_bytes ? x[j] : 0u;
            pbase[((size_t)(j / p.kb_w) * kPageRows + r_in) * p.kb_w + j % p.kb_w] = (uint8_t)b;
            c += __popc(b);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        if (lane == 0) {
            p.row_ids[slot] = p.id_base + r;
            p.row_bias[slot] = (float)c;
        }
    }
}

// k-majority: per-(cluster, bit) counts of the members' set bits for clusters [c0, c1); bits[(l - c0) * rb * 8 + j * 8 + t] counts
// bit t of byte j.  Integer atomics: the counts do not depend on the order of the adds.
__global__ void bin_bit_count_kernel(const uint8_t *x, int64_t n, int stride, int rb, const uint32_t *idx, uint32_t c0, uint32_t c1, uint32_t *bits) {
    const int64_t total = n * rb;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / rb;
        const int j = (int)(i - r * rb);
        const uint32_t l = idx[r];
        if (l < c0 || l >= c1) continue;
        uint32_t b = x[r * stride + j];
        uint32_t *dst = bits + ((size_t)(l - c0) * rb + j) * 8;
        while (b) {
            atomicAdd(dst + (__ffs(b) - 1), 1u);
            b &= b - 1;
        }
    }
}

// every bit of centroid c in [c0, c1) = the majority of its members' bits; an exact tie, or no member, keeps the bit
__global__ void bin_majority_kernel(uint8_t *cent, int stride, int rb, const uint32_t *bits, const uint32_t *cnt, uint32_t c0, uint32_t c1) {
    const int64_t total = (int64_t)(c1 - c0) * rb;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t cl = i / rb;
        const int j = (int)(i - cl * rb);
        const uint32_t m = cnt[c0 + cl];
        if (!m) continue;
        uint8_t *dst = cent + (size_t)(c0 + cl) * stride + j;
        uint32_t v = *dst;
        const uint32_t *b = bits + ((size_t)cl * rb + j) * 8;
        for (int t = 0; t < 8; t++) {
            const uint32_t twice = 2 * b[t];
            if (twice > m) v |= 1u << t;
            else if (twice < m) v &= ~(1u << t);
        }
        *dst = (uint8_t)v;
    }
}

// assignments that differ from the previous iteration's (prev is updated)
__global__ void count_changes_kernel(const uint32_t *idx, uint32_t *prev, int64_t n, uint32_t *changed) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || idx[i] == prev[i]) return;
    prev[i] = idx[i];
    atomicAdd(changed, 1u);
}

__global__ void gather_bytes_kernel(const uint8_t *x, int stride, const int64_t *pick, int64_t np, uint8_t *out) {
    const int64_t total = np * stride;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / stride;
        out[i] = x[pick[r] * stride + (i - r * stride)];
    }
}

__global__ void add_commit_kernel(const uint32_t *cnt, const uint32_t *new_base, const uint32_t *first_new_seq, uint32_t *list_len,
                                  uint32_t *tail_page, int nlist) {
    const int l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= nlist || cnt[l] == 0) return;
    const uint32_t len = list_len[l] + cnt[l];
    const uint32_t last_seq = (len - 1) / kPageRows;
    if (last_seq >= first_new_seq[l]) tail_page[l] = new_base[l] + (last_seq - first_new_seq[l]);
    list_len[l] = len;
}

__global__ void page_keys_kernel(const uint32_t *owner, const uint32_t *seq, uint32_t n, uint64_t *keys, uint32_t *vals) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    keys[i] = ((uint64_t)owner[i] << 32) | seq[i];
    vals[i] = i;
}

__global__ void list_pages_scan_kernel(const uint32_t *list_len, int nlist, uint32_t *list_page_off, uint32_t *neg_len) {
    // single CTA: list_page_off = exclusive scan of ceil(len / 256); neg_len = ~len (sort key for "longest list first")
    const int per = (nlist + 1023) / 1024;
    const int l0 = threadIdx.x * per, l1 = min(nlist, l0 + per);
    uint32_t pages = 0;
    for (int l = l0; l < l1; l++) pages += (list_len[l] + kPageRows - 1) / kPageRows;
    uint32_t tot = 0;
    uint32_t off = block_exclusive_scan_1024(pages, &tot);
    for (int l = l0; l < l1; l++) {
        list_page_off[l] = off;
        off += (list_len[l] + kPageRows - 1) / kPageRows;
        neg_len[l] = ~list_len[l];
    }
    if (threadIdx.x == 0) list_page_off[nlist] = tot;
}

// per-dimension min / max of the training sample (SQ8)
__global__ void dim_minmax_kernel(const float *x, int64_t n, int64_t stride, int d, float *lo, float *hi) {
    const int j = blockIdx.x;
    float mn = FLT_MAX, mx = -FLT_MAX;
    for (int64_t r = threadIdx.x; r < n; r += blockDim.x) {
        const float v = x[r * stride + j];
        mn = fminf(mn, v);
        mx = fmaxf(mx, v);
    }
    __shared__ float smn[256], smx[256];
    smn[threadIdx.x] = mn;
    smx[threadIdx.x] = mx;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) {
            smn[threadIdx.x] = fminf(smn[threadIdx.x], smn[threadIdx.x + o]);
            smx[threadIdx.x] = fmaxf(smx[threadIdx.x], smx[threadIdx.x + o]);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        lo[j] = smn[0];
        hi[j] = smx[0];
    }
}

// ------------------------------------------------------------------------------------
// search: (query, list) pairs -> work items
// ------------------------------------------------------------------------------------
__global__ void pairs_make_kernel(const int64_t *probe, int64_t n_pairs, int nlist, uint32_t *keys, uint32_t *vals, uint32_t *cnt) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_pairs) return;
    const int64_t l = probe[i];
    const uint32_t key = (l < 0 || l >= nlist) ? (uint32_t)nlist : (uint32_t)l;   // invalid probes sort behind every list
    keys[i] = key;
    vals[i] = (uint32_t)i;
    if (key < (uint32_t)nlist) atomicAdd(&cnt[key], 1u);
}

struct SearchPlan {
    const uint32_t *cnt;          // [nlist] pairs per list
    const uint32_t *list_len, *list_page_off, *list_order;   // list_order: lists by decreasing length
    uint32_t *pair_start;         // [nlist] out: first sorted pair of the list
    uint32_t *part_off;           // [nlist] out: first partial list of the list's first pair
    uint32_t *n_chunks;           // [nlist] out
    IvfGemmItem *items;           // out
    int *n_items, *n_parts;       // out (device scalars)
    unsigned long long *scan_rows;  // out: list rows the scan kernel will stream (every query tile of a list reads the whole list)
    int nlist, max_items;
    uint32_t pages_per_chunk;
};

__global__ void __launch_bounds__(1024) search_plan_kernel(const SearchPlan p) {
    const int per = (p.nlist + 1023) / 1024;
    const int l0 = threadIdx.x * per, l1 = min(p.nlist, l0 + per);
    // pass 1 in list-id order: pair_start (the sort order of the pairs)
    uint32_t pairs = 0;
    for (int l = l0; l < l1; l++) pairs += p.cnt[l];
    uint32_t poff = block_exclusive_scan_1024(pairs, nullptr);
    for (int l = l0; l < l1; l++) {
        p.pair_start[l] = poff;
        poff += p.cnt[l];
    }
    // pass 2 in decreasing-length order: items and partial lists (big lists first = LPT-like static schedule)
    uint32_t items = 0, parts = 0;
    unsigned long long rows_local = 0;
    for (int o = l0; o < l1; o++) {
        const uint32_t l = p.list_order[o];
        const uint32_t c = p.cnt[l], len = p.list_len[l];
        const uint32_t pages = (len + kPageRows - 1) / kPageRows;
        const uint32_t nch = (c && pages) ? (pages + p.pages_per_chunk - 1) / p.pages_per_chunk : 0;
        p.n_chunks[l] = nch;
        items += ((c + 127) / 128) * nch;
        parts += c * nch;
        if (nch) rows_local += (unsigned long long)((c + 127) / 128) * len;
    }
    if (threadIdx.x == 0) *p.scan_rows = 0;
    __syncthreads();
    if (rows_local) atomicAdd(p.scan_rows, rows_local);
    uint32_t tot_items = 0, tot_parts = 0;
    uint32_t ioff = block_exclusive_scan_1024(items, &tot_items);
    uint32_t paoff = block_exclusive_scan_1024(parts, &tot_parts);
    __syncthreads();
    for (int o = l0; o < l1; o++) {
        const uint32_t l = p.list_order[o];
        const uint32_t c = p.cnt[l], len = p.list_len[l], nch = p.n_chunks[l];
        p.part_off[l] = paoff;
        paoff += c * nch;
        if (!nch) continue;
        const uint32_t pages = (len + kPageRows - 1) / kPageRows;
        const uint32_t q0 = p.pair_start[l];
        for (uint32_t qt = 0; qt * 128 < c; qt++)
            for (uint32_t ch = 0; ch < nch; ch++) {
                if (ioff < (uint32_t)p.max_items) {
                    IvfGemmItem it;
                    it.q_begin = q0 + qt * 128;
                    it.q_count = min(128u, c - qt * 128);
                    it.page_begin = p.list_page_off[l] + ch * p.pages_per_chunk;
                    it.page_count = min(p.pages_per_chunk, pages - ch * p.pages_per_chunk);
                    it.row_limit = len - ch * p.pages_per_chunk * kPageRows;
                    it.chunk = ch;
                    p.items[ioff] = it;
                }
                ioff++;
            }
    }
    if (threadIdx.x == 0) {
        *p.n_items = (int)min(tot_items, (uint32_t)p.max_items);
        *p.n_parts = (int)tot_parts;
    }
}

// ------------------------------------------------------------------------------------
// Coarse probe for nprobe > 8: the centroid table is small (nlist x d fp32, L2-resident) and nprobe is a large k for it --
// the fused top-k kernels keep one k-entry list per query and, with only nlist / workers rows per list, almost every row is
// an insert.  Here the ranking keys
// ||c||^2 - 2 <x, c> of a chunk of queries are written out by a plain fp32 tile kernel (64 x 64 tiles, 4 x 4 per thread) and
// one warp per query selects its nprobe smallest with a sorted warp list: scores are read once, coalesced, and an insert is
// O(nprobe / 32).
// ------------------------------------------------------------------------------------
constexpr int kCoarseTile = 64, kCoarseTK = 16;

// Queries per coarse_scores_kernel launch: <= 256 MB of keys, and at most 65535 query tiles (gridDim.y).
static int64_t coarse_chunk(int64_t nq, int nl) {
    const int64_t by_bytes = std::max<int64_t>(64, std::min<int64_t>(nq, ((int64_t)64 << 20) / std::max(1, nl)));
    return std::min<int64_t>(by_bytes, (int64_t)65535 * kCoarseTile);
}

__global__ void __launch_bounds__(256) coarse_scores_kernel(const float *x, int64_t ldx, const float *cent, const float *cnorm, int64_t nq,
                                                            int nl, int d, float *out /*[nq][nl]*/) {
    __shared__ float sx[kCoarseTK][kCoarseTile + 4], sc[kCoarseTK][kCoarseTile + 4];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int64_t q0 = (int64_t)blockIdx.y * kCoarseTile;
    const int c0 = blockIdx.x * kCoarseTile;
    float acc[4][4] = {};
    // loads: thread t fetches element (row t / 16 + 16 r, column t % 16) of each 64 x 16 operand tile, r = 0..3
    const int lr = threadIdx.x >> 4, lc = threadIdx.x & 15;
    for (int k0 = 0; k0 < d; k0 += kCoarseTK) {
#pragma unroll
        for (int r = 0; r < 4; r++) {
            const int row = lr + 16 * r;
            const int64_t q = q0 + row;
            const int c = c0 + row;
            const int kk = k0 + lc;
            sx[lc][row] = (q < nq && kk < d) ? x[q * ldx + kk] : 0.f;
            sc[lc][row] = (c < nl && kk < d) ? cent[(size_t)c * d + kk] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < kCoarseTK; kk++) {
            const float4 a = *reinterpret_cast<const float4 *>(&sx[kk][ty * 4]);
            const float4 b = *reinterpret_cast<const float4 *>(&sc[kk][tx * 4]);
            const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int64_t q = q0 + ty * 4 + i;
        if (q >= nq) continue;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int c = c0 + tx * 4 + j;
            if (c < nl) out[q * nl + c] = fmaf(-2.f, acc[i][j], cnorm[c]);
        }
    }
}

__global__ void __launch_bounds__(256) coarse_select_kernel(const float *scores, int64_t nq, int nl, int k, float *out_key, int64_t *out_ids) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float *lk = reinterpret_cast<float *>(smem_raw) + (size_t)warp * k;
    uint32_t *li = reinterpret_cast<uint32_t *>(reinterpret_cast<float *>(smem_raw) + (size_t)8 * k) + (size_t)warp * k;
    const int64_t q = (int64_t)blockIdx.x * 8 + warp;
    if (q >= nq) return;
    WarpTopK list;
    list.init(lk, li, k);
    const float *row = scores + q * nl;
    for (int c0 = 0; c0 < nl; c0 += 32) {
        const int c = c0 + lane;
        const float key = c < nl ? row[c] : FLT_MAX;
        unsigned m = __ballot_sync(0xffffffffu, c < nl && list.passes(key, (uint32_t)c));
        while (m) {
            const int src = __ffs(m) - 1;
            m &= m - 1;
            list.insert(__shfl_sync(0xffffffffu, key, src), (uint32_t)(c0 + src));
        }
    }
    __syncwarp();
    for (int j = lane; j < k; j += 32) {
        out_key[q * k + j] = j < list.n ? lk[j] : FLT_MAX;
        out_ids[q * k + j] = j < list.n ? (int64_t)li[j] : -1;
    }
}

// One warp per sorted pair: gather (and for SQ8 scale) the query into the bf16 A-operand buffer, record where the pair's
// partial lists start, the inverse permutation, and the pair's additive constant (PQ: ||q - c||^2 or -<q, c>).
struct PairFill {
    const uint32_t *sorted_list, *sorted_pair;   // [n_pairs]
    const uint32_t *pair_start, *part_off, *n_chunks;
    const float *queries;        // [nq][d_pad] fp32, prepared (cosine: unit length)
    const float *sq_step;        // SQ8: per-dimension step (null otherwise)
    const float *centroids;      // PQ: [nlist][d] (null otherwise)
    __nv_bfloat16 *qbuf;         // [n_pairs][d_pad64] (null: no gathered rows, the table look-up scan reads its own table)
    uint32_t *inv;               // [n_pairs] original pair -> sorted position
    uint32_t *pair_part_base;    // [n_pairs]
    float *pair_const;           // [n_pairs]
    int64_t n_pairs;
    int nprobe, nlist, d, d_pad, d_pad64, l2;
    // binary payload: queries [nq][row_bytes] -> qbuf bytes [n_pairs][row_pad]; pair_const = popc(q) (Hamming) or 0 (Jaccard)
    const uint8_t *bqueries;
    uint8_t *bqbuf;
    float *pair_popc;            // [n_pairs] popc(q)
    int row_bytes, row_pad, jaccard;
};

__global__ void __launch_bounds__(256) pair_fill_kernel(const PairFill p) {
    const int lane = threadIdx.x & 31;
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= p.n_pairs) return;
    const uint32_t l = p.sorted_list[i], pr = p.sorted_pair[i];
    if (lane == 0) p.inv[pr] = (uint32_t)i;
    if (l >= (uint32_t)p.nlist) {   // invalid probe: no work item reads this row
        if (lane == 0) {
            p.pair_part_base[i] = 0;
            p.pair_const[i] = 0.f;
        }
        return;
    }
    const uint32_t q = pr / (uint32_t)p.nprobe;
    const float *x = p.queries + (size_t)q * p.d_pad;
    __nv_bfloat16 *dst = p.qbuf ? p.qbuf + (size_t)i * p.d_pad64 : nullptr;
    const float *c = p.centroids ? p.centroids + (size_t)l * p.d : nullptr;
    float acc = 0.f;
    for (int j = lane; j < p.d_pad64; j += 32) {
        float v = j < p.d ? x[j] : 0.f;
        if (c && j < p.d) {
            const float cv = c[j];
            acc = p.l2 ? fmaf(v - cv, v - cv, acc) : fmaf(-v, cv, acc);
        }
        if (p.sq_step && j < p.d) v *= p.sq_step[j];
        if (dst) dst[j] = __float2bfloat16_rn(v);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) {
        p.pair_part_base[i] = p.part_off[l] + ((uint32_t)i - p.pair_start[l]) * p.n_chunks[l];
        p.pair_const[i] = acc;
    }
}

// Binary payload: one warp per sorted pair gathers the query bytes (zero-padded to row_pad) and its popcount.
__global__ void __launch_bounds__(256) pair_fill_bin_kernel(const PairFill p) {
    const int lane = threadIdx.x & 31;
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= p.n_pairs) return;
    const uint32_t l = p.sorted_list[i], pr = p.sorted_pair[i];
    if (lane == 0) p.inv[pr] = (uint32_t)i;
    if (l >= (uint32_t)p.nlist) {
        if (lane == 0) {
            p.pair_part_base[i] = 0;
            p.pair_const[i] = 0.f;
            p.pair_popc[i] = 0.f;
        }
        return;
    }
    const uint8_t *x = p.bqueries + (size_t)(pr / (uint32_t)p.nprobe) * p.row_bytes;
    uint8_t *dst = p.bqbuf + (size_t)i * p.row_pad;
    int c = 0;
    for (int j = lane; j < p.row_pad; j += 32) {
        const uint32_t b = j < p.row_bytes ? x[j] : 0u;
        dst[j] = (uint8_t)b;
        c += __popc(b);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) {
        p.pair_part_base[i] = p.part_off[l] + ((uint32_t)i - p.pair_start[l]) * p.n_chunks[l];
        p.pair_const[i] = p.jaccard ? 0.f : (float)c;
        p.pair_popc[i] = (float)c;
    }
}

// nprobe >= nlist: every query probes every list
__global__ void probe_all_kernel(int64_t *probe, int64_t nq, int nl) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nq * nl) probe[i] = i % nl;
}

// per-query constants of the expanded distances (bf16 and SQ8 payloads; PQ has its query term in the pair constant):
// qc[q] = L2 ? ||q||^2 (- 2 <q, mid> for SQ8) : (- <q, mid> for SQ8, else 0)
__global__ void query_const_kernel(const float *queries, int64_t nq, int d, int d_pad, const float *sq_mid, int l2, int round_bf16, float *qc) {
    const int lane = threadIdx.x & 31;
    const int64_t q = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (q >= nq) return;
    const float *x = queries + (size_t)q * d_pad;
    float nn = 0.f, qm = 0.f;
    for (int j = lane; j < d; j += 32) {
        // bf16 payload: the scan multiplies bf16-rounded queries, so ||q||^2 is taken of the same values
        const float v = round_bf16 ? __bfloat162float(__float2bfloat16_rn(x[j])) : x[j];
        nn = fmaf(v, v, nn);
        if (sq_mid) qm = fmaf(x[j], sq_mid[j], qm);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        nn += __shfl_xor_sync(0xffffffffu, nn, o);
        qm += __shfl_xor_sync(0xffffffffu, qm, o);
    }
    if (lane == 0) qc[q] = l2 ? nn - 2.f * qm : -qm;
}

// One CTA per query: the partial lists of its nprobe pairs (x chunks) -> top-k, real distances.
struct IvfMerge {
    const uint32_t *inv, *pair_part_base, *sorted_list, *n_chunks;
    const float *pair_const, *query_const;
    const float *part_keys, *part_worst;
    const uint32_t *part_ids;
    float *out_dis;
    int64_t *out_ids;
    int64_t id_offset;
    int nprobe, nlist, k_part, k, metric;   // metric: B200_METRIC_*
};

__global__ void __launch_bounds__(256) ivf_merge_kernel(const IvfMerge p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float *lk = reinterpret_cast<float *>(smem_raw);                      // [8][k] + merged [k]
    uint32_t *li = reinterpret_cast<uint32_t *>(lk + (size_t)9 * p.k);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t q = blockIdx.x;
    WarpTopK list;
    list.init(lk + (size_t)warp * p.k, li + (size_t)warp * p.k, p.k);
    for (int j = lane; j < p.k; j += 32) list.keys[j] = FLT_MAX;
    __syncwarp();
    // bound: a FULL partial list's worst key (+ its pair constant) bounds the query's k_part-th key from above
    if (p.k_part >= p.k) {
        __shared__ float bound_s[8];
        float b = FLT_MAX;
        for (int pr = 0; pr < p.nprobe; pr++) {
            const uint32_t i = p.inv[q * p.nprobe + pr];
            const uint32_t l = p.sorted_list[i];
            if (l >= (uint32_t)p.nlist) continue;
            const uint32_t nch = p.n_chunks[l];
            for (uint32_t ch = threadIdx.x; ch < nch; ch += blockDim.x) {
                const float w = p.part_worst[p.pair_part_base[i] + ch];
                if (w < FLT_MAX) b = fminf(b, w + p.pair_const[i]);
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) b = fminf(b, __shfl_xor_sync(0xffffffffu, b, o));
        if (lane == 0) bound_s[warp] = b;
        __syncthreads();
        b = bound_s[0];
#pragma unroll
        for (int w = 1; w < 8; w++) b = fminf(b, bound_s[w]);
        if (b < FLT_MAX) {
            list.thr_key = b;
            list.thr_id = kNoId;
        }
    }
    for (int pr = 0; pr < p.nprobe; pr++) {
        const uint32_t i = p.inv[q * p.nprobe + pr];
        const uint32_t l = p.sorted_list[i];
        if (l >= (uint32_t)p.nlist) continue;
        const int64_t ncand = (int64_t)p.n_chunks[l] * p.k_part;
        const size_t base = (size_t)p.pair_part_base[i] * p.k_part;
        const float pc = p.pair_const[i];
        for (int64_t c0 = (int64_t)warp * 32; c0 < ncand; c0 += 256) {
            const int64_t c = c0 + lane;
            float key = FLT_MAX;
            uint32_t id = kNoId;
            bool cand = false;
            if (c < ncand) {
                id = p.part_ids[base + c];
                key = p.part_keys[base + c] + pc;
                cand = id != kNoId && list.passes(key, id);
            }
            unsigned m = __ballot_sync(0xffffffffu, cand);
            while (m) {
                const int src = __ffs(m) - 1;
                m &= m - 1;
                list.insert(__shfl_sync(0xffffffffu, key, src), __shfl_sync(0xffffffffu, id, src));
            }
        }
    }
    __syncthreads();
    float *fk = lk + (size_t)8 * p.k;
    uint32_t *fi = li + (size_t)8 * p.k;
    block_rank_merge(lk, li, 8, p.k, p.k, fk, fi);
    __syncthreads();
    const float qc = p.query_const ? p.query_const[q] : 0.f;
    for (int j = threadIdx.x; j < p.k; j += blockDim.x) {
        float dis;
        int64_t id = -1;
        if (fi[j] != kNoId) {
            const float key = fk[j] + qc;
            id = (int64_t)fi[j] + p.id_offset;
            // binary metrics: the key is the distance (Hamming: popc(y) - 2 and + popc(q); Jaccard keyed in the scan)
            dis = p.metric == B200_METRIC_L2 ? fmaxf(key, 0.f) : p.metric == B200_METRIC_IP ? -key : p.metric == B200_METRIC_COSINE ? 1.f + key : key;
        } else {
            dis = p.metric == B200_METRIC_IP ? -FLT_MAX : FLT_MAX;
        }
        p.out_dis[q * p.k + j] = dis;
        p.out_ids[q * p.k + j] = id;
    }
}

// ------------------------------------------------------------------------------------
// exact second stage: one CTA per query, one warp per candidate row (random 4*d-byte gathers)
// ------------------------------------------------------------------------------------
struct RefineParams {
    const float *queries;  // [nq][d_pad]
    const float *rows;     // [n][d_pad]; staged: the candidates' rows [nq][ncand][d_pad] (gather_host_rows_kernel)
    const int64_t *cand;   // [nq][ncand], negative = empty
    float *out_dis;        // [nq][k]
    int64_t *out_ids;
    int64_t n;
    int d_pad, ncand, k;
    int l2;                // else inner product
    int cosine;            // output 1 - ip
    int64_t id_offset;     // added to every returned id (shard base)
};

// kStaged: candidate (q, c) is read from its staging slot q * ncand + c instead of row id; nothing else differs, so the keys
// are those of the HBM rows bit for bit
template <bool kStaged>
__global__ void __launch_bounds__(256) refine_kernel(const RefineParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float *qs = reinterpret_cast<float *>(smem_raw);
    float *lk = qs + p.d_pad;
    uint32_t *li = reinterpret_cast<uint32_t *>(lk + 8 * p.k);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t q = blockIdx.x;
    for (int i = threadIdx.x; i < p.d_pad; i += 256) qs[i] = p.queries[q * p.d_pad + i];
    WarpTopK list;
    list.init(lk + (size_t)warp * p.k, li + (size_t)warp * p.k, p.k);
    for (int j = lane; j < p.k; j += 32) list.keys[j] = FLT_MAX;
    __syncthreads();
    for (int c = warp; c < p.ncand; c += 8) {
        const int64_t id = p.cand[q * p.ncand + c];
        if (id < 0 || id >= p.n) continue;  // warp-uniform
        // duplicates in the candidate set would be returned twice; the first stage never produces them
        const float4 *row = reinterpret_cast<const float4 *>(p.rows + (kStaged ? (size_t)q * p.ncand + c : (size_t)id) * p.d_pad);
        float acc = 0.f;
        for (int cc = lane; cc < p.d_pad / 4; cc += 32) {
            const float4 y = row[cc];
            const float4 x = reinterpret_cast<const float4 *>(qs)[cc];
            if (p.l2) {
                float t = x.x - y.x; acc = fmaf(t, t, acc);
                t = x.y - y.y; acc = fmaf(t, t, acc);
                t = x.z - y.z; acc = fmaf(t, t, acc);
                t = x.w - y.w; acc = fmaf(t, t, acc);
            } else {
                acc = fmaf(x.x, y.x, acc); acc = fmaf(x.y, y.y, acc);
                acc = fmaf(x.z, y.z, acc); acc = fmaf(x.w, y.w, acc);
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        list.insert(p.l2 ? acc : -acc, (uint32_t)id);
    }
    __syncthreads();
    float *fk = lk + (size_t)8 * p.k * 2;  // merged list, behind the 8 warp lists (keys + ids)
    uint32_t *fi = reinterpret_cast<uint32_t *>(fk + p.k);
    block_rank_merge(lk, li, 8, p.k, p.k, fk, fi);
    __syncthreads();
    for (int j = threadIdx.x; j < p.k; j += blockDim.x) {
        const bool have = fi[j] != kNoId;
        const float key = have ? fk[j] : 0.f;
        p.out_ids[q * p.k + j] = have ? (int64_t)fi[j] + p.id_offset : -1;
        p.out_dis[q * p.k + j] = !have ? (p.l2 || p.cosine ? FLT_MAX : -FLT_MAX) : p.l2 ? key : p.cosine ? 1.f + key : -key;
    }
}

// Rows in host memory (keep_raw=2): one warp per candidate slot of a chunk of queries copies the slot's row through the mapped
// pointer over PCIe into stage[slot][d_pad].  A lane issues every 16-byte load of kGatherRows rows before its first store, so
// that a warp keeps kGatherRows rows in flight against the link's latency.  Slots with id < 0 or id >= n are skipped, as
// refine_kernel skips them.
constexpr int kGatherVec = 8;    // float4 per lane and row in one pass: one pass covers d_pad <= 1024
constexpr int kGatherRows = 2;

__global__ void __launch_bounds__(256) gather_host_rows_kernel(const float *__restrict__ rows, int64_t n, int d_pad, const int64_t *__restrict__ cand,
                                                               int64_t nslots, float *__restrict__ stage) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int nv = d_pad / 4;
    for (int64_t s0 = warp * kGatherRows; s0 < nslots; s0 += nwarps * kGatherRows) {
        const float4 *src[kGatherRows];
        float4 *dst[kGatherRows];
        bool ok[kGatherRows];
#pragma unroll
        for (int r = 0; r < kGatherRows; r++) {
            const int64_t id = s0 + r < nslots ? cand[s0 + r] : -1;
            ok[r] = id >= 0 && id < n;
            src[r] = reinterpret_cast<const float4 *>(rows + (size_t)(ok[r] ? id : 0) * d_pad);
            dst[r] = reinterpret_cast<float4 *>(stage + (size_t)(s0 + r) * d_pad);
        }
        for (int v0 = 0; v0 < nv; v0 += 32 * kGatherVec) {
            float4 buf[kGatherRows][kGatherVec];
#pragma unroll
            for (int r = 0; r < kGatherRows; r++)
#pragma unroll
                for (int j = 0; j < kGatherVec; j++) {
                    const int v = v0 + j * 32 + lane;
                    if (ok[r] && v < nv) buf[r][j] = src[r][v];
                }
            // a store waits for its load: keep every store behind the last load, or the first one stalls the loads after it
            asm volatile("" ::: "memory");
#pragma unroll
            for (int r = 0; r < kGatherRows; r++)
#pragma unroll
                for (int j = 0; j < kGatherVec; j++) {
                    const int v = v0 + j * 32 + lane;
                    if (ok[r] && v < nv) dst[r][v] = buf[r][j];
                }
        }
    }
}

// ------------------------------------------------------------------------------------
// filter_probe=1: per-search list state under the filter, and a probe depth per query that reaches k1 kept rows
// ------------------------------------------------------------------------------------
// One CTA per list walks its page chain, thread t on row t of every page: list_alive[l] = the list's rows the bitmap keeps;
// f_pages[list_page_off[l] + j] = its pages with at least one kept row, in chain order; f_len[l] = the rows the plan and the
// scan see through them (256 per kept page, and the original tail count if the list's last page is kept: only that page is
// partial).  A dropped page holds no candidate, so the scan's answer does not change.
__global__ void __launch_bounds__(256) list_alive_kernel(const uint32_t *list_len, const uint32_t *list_page_off, const uint32_t *list_pages,
                                                         const uint32_t *row_ids, const uint8_t *alive, uint32_t *list_alive, uint32_t *f_len,
                                                         uint32_t *f_pages) {
    const int l = blockIdx.x;
    const uint32_t len = list_len[l], pages = (len + kPageRows - 1) / kPageRows, off = list_page_off[l];
    uint32_t kept_pages = 0, kept_rows = 0, flen = 0;
    for (uint32_t j = 0; j < pages; j++) {
        const uint32_t page = list_pages[off + j];
        bool keep = false;
        if (j * kPageRows + threadIdx.x < len) {
            const uint32_t id = row_ids[(size_t)page * kPageRows + threadIdx.x];
            keep = (alive[id >> 3] >> (id & 7)) & 1;
        }
        const uint32_t c = (uint32_t)__syncthreads_count(keep);
        if (c) {
            if (threadIdx.x == 0) f_pages[off + kept_pages] = page;
            kept_pages++;
            kept_rows += c;
            flen = (kept_pages - 1) * kPageRows + min((uint32_t)kPageRows, len - j * kPageRows);
        }
    }
    if (threadIdx.x == 0) {
        list_alive[l] = kept_rows;
        f_len[l] = flen;
    }
}

// coarse keys as order-preserving u32 (-0 as +0, so that equal floats stay equal)
__device__ __forceinline__ uint32_t coarse_key_u32(float f) {
    const uint32_t u = __float_as_uint(f == 0.f ? 0.f : f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

constexpr int kProbeThreads = 256;

// The first `count` lists in (key, list id) order: every list with key < `key`, then the first `ties` lists with key == `key`
// in list-id order.
struct ProbeCut {
    uint32_t key, ties, count;
};

// Shortest prefix of a query's lists in (key, id) order whose weight reaches `target`; weights min(w[l], target) (the test
// W >= target is unchanged by the clamp, and the sums stay below 2^32), or 1 with w null.  count = nl when the whole row
// does not reach it.  A radix select over the u32 keys (4 x 8 bits, histograms weighted), then the ties at the cut key in
// list-id order (thread t owns a contiguous range of ids).  Called by every thread of the CTA.
__device__ ProbeCut prefix_cut(const float *row, int nl, const uint32_t *w, uint32_t target) {
    typedef cub::BlockScan<uint32_t, kProbeThreads> Scan;
    typedef cub::BlockReduce<uint32_t, kProbeThreads> Reduce;
    __shared__ union {
        typename Scan::TempStorage scan;
        typename Reduce::TempStorage red;
    } tmp;
    __shared__ uint32_t hist[256];
    __shared__ uint32_t s_prefix, s_need, s_total, s_less, s_ties;
    const int t = threadIdx.x;
    uint32_t prefix = 0, mask = 0, need = target;
    __syncthreads();   // a previous call's readers of the shared state are done
    for (int shift = 24; shift >= 0; shift -= 8) {
        for (int i = t; i < 256; i += kProbeThreads) hist[i] = 0;
        __syncthreads();
        for (int l = t; l < nl; l += kProbeThreads) {
            const uint32_t u = coarse_key_u32(row[l]);
            if ((u & mask) != prefix) continue;
            const uint32_t wt = w ? min(w[l], target) : 1u;
            if (wt) atomicAdd(&hist[(u >> shift) & 255], wt);
        }
        __syncthreads();
        if (t == 0) {
            if (shift == 24) {
                uint32_t tot = 0;
                for (int i = 0; i < 256; i++) tot += hist[i];
                s_total = tot;
            }
            uint32_t acc = 0, b = 0;
            for (; b < 255 && acc + hist[b] < need; b++) acc += hist[b];
            s_prefix = prefix | (b << shift);
            s_need = need - acc;
        }
        __syncthreads();
        if (s_total < target) return {0xffffffffu, (uint32_t)nl, (uint32_t)nl};   // block-uniform
        prefix = s_prefix;
        need = s_need;
        mask |= 255u << shift;
    }
    const int per = (nl + kProbeThreads - 1) / kProbeThreads;
    const int l0 = min(nl, t * per), l1 = min(nl, l0 + per);
    uint32_t less = 0, eq = 0, eq_w = 0;
    for (int l = l0; l < l1; l++) {
        const uint32_t u = coarse_key_u32(row[l]);
        if (u < prefix) less++;
        else if (u == prefix) {
            eq++;
            eq_w += w ? min(w[l], target) : 1u;
        }
    }
    uint32_t eq_before, w_before;
    Scan(tmp.scan).ExclusiveSum(eq, eq_before);
    __syncthreads();
    Scan(tmp.scan).ExclusiveSum(eq_w, w_before);
    __syncthreads();
    const uint32_t n_less = Reduce(tmp.red).Sum(less);
    if (w_before < need && w_before + eq_w >= need) {   // the one thread whose range holds the cut
        uint32_t acc = w_before, c = eq_before;
        for (int l = l0; l < l1 && acc < need; l++) {
            const uint32_t u = coarse_key_u32(row[l]);
            if (u != prefix) continue;
            c++;
            acc += w ? min(w[l], target) : 1u;
        }
        s_ties = c;
    }
    if (t == 0) s_less = n_less;
    __syncthreads();
    return {prefix, s_ties, s_less + s_ties};
}

// The lists of a cut that hold a kept row, in list-id order: their count (every thread), and with out given, written to
// out[0 ..).  A list without a kept row has a filtered length of 0: probing it adds no candidate, only a slot.  Called by
// every thread of the CTA; thread t owns a contiguous range of list ids.
__device__ uint32_t cut_live_lists(const float *row, int nl, const uint32_t *list_alive, uint32_t key, uint32_t ties, int64_t *out) {
    typedef cub::BlockScan<uint32_t, kProbeThreads> Scan;
    __shared__ typename Scan::TempStorage tmp;
    const int t = threadIdx.x, per = (nl + kProbeThreads - 1) / kProbeThreads;
    const int l0 = min(nl, t * per), l1 = min(nl, l0 + per);
    uint32_t eq = 0;
    for (int l = l0; l < l1; l++) eq += coarse_key_u32(row[l]) == key;
    uint32_t eq_before, pos, total;
    __syncthreads();   // a previous call's scan storage is free
    Scan(tmp).ExclusiveSum(eq, eq_before);
    uint32_t live = 0;
    for (int l = l0, e = eq_before; l < l1; l++) {
        const uint32_t u = coarse_key_u32(row[l]);
        const bool in_cut = u < key || (u == key && (uint32_t)e++ < ties);
        live += in_cut && list_alive[l] > 0;
    }
    __syncthreads();
    Scan(tmp).ExclusiveSum(live, pos, total);
    if (out)
        for (int l = l0, e = eq_before; l < l1; l++) {
            const uint32_t u = coarse_key_u32(row[l]);
            const bool in_cut = u < key || (u == key && (uint32_t)e++ < ties);
            if (in_cut && list_alive[l] > 0) out[pos++] = l;
        }
    return total;
}

// One CTA per query of a key chunk: p_q = min(max_nprobe, max(nprobe, the lists until W >= k1)), the cut of its first p_q
// lists and live_out = how many of them hold a kept row (the lists it will probe).  totals[0] += live, totals[1] = max live.
__global__ void __launch_bounds__(kProbeThreads) probe_select_kernel(const float *keys, int nl, const uint32_t *list_alive, uint32_t k1, int nprobe,
                                                                     int max_nprobe, int *p_out, int *live_out, uint32_t *cut_key, uint32_t *cut_ties,
                                                                     unsigned long long *totals) {
    const int64_t q = blockIdx.x;
    const float *row = keys + q * nl;
    const ProbeCut wc = prefix_cut(row, nl, list_alive, k1);
    const int p = min(max_nprobe, max(nprobe, (int)wc.count));
    const ProbeCut c = p == (int)wc.count ? wc : prefix_cut(row, nl, nullptr, (uint32_t)p);
    const uint32_t live = cut_live_lists(row, nl, list_alive, c.key, c.ties, nullptr);
    if (threadIdx.x == 0) {
        p_out[q] = p;
        live_out[q] = (int)live;
        cut_key[q] = c.key;
        cut_ties[q] = c.ties;
        atomicAdd(totals, (unsigned long long)live);
        atomicMax(totals + 1, (unsigned long long)live);
    }
}

// One CTA per query: its probe row [P] = the lists of its cut that hold a kept row, in list-id order, then -1 (an invalid
// probe slot, which every later stage skips).
__global__ void __launch_bounds__(kProbeThreads) probe_emit_kernel(const float *keys, int nl, const uint32_t *list_alive, const int *live_in,
                                                                   const uint32_t *cut_key, const uint32_t *cut_ties, int P, int64_t *probe) {
    const int64_t q = blockIdx.x;
    int64_t *out = probe + q * P;
    cut_live_lists(keys + q * nl, nl, list_alive, cut_key[q], cut_ties[q], out);
    for (int j = live_in[q] + threadIdx.x; j < P; j += kProbeThreads) out[j] = -1;
}

__global__ void add_u64_kernel(const unsigned long long *src, unsigned long long *acc) { *acc += *src; }

}  // namespace b200

using namespace b200;

// ------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------
enum { IDX_FLAT = 0, IDX_IVFFLAT = 1, IDX_IVFPQ = 2, IDX_MSTG = 3, IDX_IVFSQ = 4, IDX_SCANN = 5, IDX_HNSWFLAT = 6, IDX_HNSWSQ = 7, IDX_HNSWPQ = 8,
       IDX_BINFLAT = 9, IDX_BINIVF = 10, IDX_BINHNSW = 11, IDX_BINMSTG = 12, IDX_NUM_TYPES = 13 };
static const char *kTypeNames[] = {"FLAT", "IVFFLAT", "IVFPQ", "MSTG", "IVFSQ", "SCANN", "HNSWFLAT", "HNSWSQ", "HNSWPQ",
                                   "BINARYFLAT", "BINARYIVF", "BINARYHNSW", "BINARYMSTG"};
static bool is_flat_type(int t) { return t == IDX_FLAT || t == IDX_BINFLAT; }

struct b200_index {
    int type = IDX_FLAT, metric = B200_METRIC_L2, d = 0, d_pad = 0, d_pad64 = 0;
    int nlist = 0, m = 0, dsub = 0;
    int pq_bits = 8;                // PQ code width: 8 (256 codewords, one byte per code) or 4 (16 codewords, two codes per byte)
    // aq_threshold=T (PQ types, IP / cosine): anisotropic codebooks and codes (ivf_aq.cu) with eta = (d - 1) T^2 / (1 - T^2);
    // 0: plain PQ.  aq_loss: the training sample's mean loss after the k-means codebooks, then after each iteration.
    double aq_threshold = 0, aq_eta = 0;
    std::vector<double> aq_loss;
    // opq=1 (PQ types): the rotation R [d][d] fp32, y = x.R (ivf_opq.h).  The centroids, codebooks, codes and norm terms live
    // in the rotated space, the fp32 rows do not.  opq_loss: the sample's mean PQ loss at R = I, then after each of the
    // opq_iters alternations (empty on a loaded index).  A part below the inverted-file threshold keeps no R.
    int opq = 0, opq_iters = 20;
    DevMem d_opq;                   // float [d][d]
    std::vector<double> opq_loss;
    int default_nprobe = 32, refine_factor = 4;
    int payload = IVF_PRODUCER_TMA;
    int keep_raw = -1;              // -1 auto (yes), 0 no fp32 rows (first-stage distances only), 1 yes, 2 yes, in host memory
    int code_bytes = 0;
    int64_t n = 0, reserved = 0;
    bool trained = false, built = false, use_ivf = false;
    CorpusPtr raw;                  // fp32 rows in id order (cosine: unit vectors), metric L2 or IP
    // keep_raw=2 on an inverted-file float index: raw's rows [h_rows_cap][d_pad] (same values, zero padding) in pinned,
    // mapped host memory instead; the second stage gathers its candidates over PCIe
    float *h_rows = nullptr;
    const float *h_rows_dev = nullptr;   // the device's address of h_rows
    int64_t h_rows_cap = 0;
    CorpusPtr coarse;               // centroid table as a FLAT corpus (L2)
    DevMem d_centroids;             // float [nlist][d]
    DevMem d_cnorm;                 // float [nlist] ||c||^2 (coarse probe)
    DevMem d_pq;                    // float [m][256][dsub]
    DevMem d_pq_bf16;               // bf16 [m][256][dsub]
    DevMem d_sq;                    // float [4][d]: lo, step, 1/step, mid
    // paged lists
    uint32_t pool_pages = 0, pages_used = 0;
    DevMem d_pool;                  // bf16 [pool_pages * 256][d_pad64]  |  codes [pool_pages * 256][code_bytes]
    DevMem d_row_bias;              // float [pool rows]
    DevMem d_row_ids;               // uint32 [pool rows]; the uint32 arrays below: [nlist], [nlist], [pages], [pages], [1]
    DevMem d_list_len, d_tail_page, d_page_owner, d_page_seq, d_pages_used;
    DevMem d_flag;                  // int [8]
    DevMem d_list_page_off, d_list_pages, d_list_order;   // uint32, after finalize
    std::vector<uint32_t> list_len;  // host copy after finalize
    // binary indexes: rows are bytes [n][row_bytes]; pages [page][row_pad / kb_w][256 rows][kb_w bytes]; the coarse table is
    // d_bcent zero-padded to cent_pad (16-byte) rows, searched as a Hamming corpus (zero bits change no distance)
    bool binary = false;
    int row_bytes = 0, kb_w = 0, row_pad = 0, cent_pad = 0;
    DevMem d_bcent;                 // uint8 [nlist][cent_pad]
    uint32_t max_list_pages = 0;
    int device = 0, sms = 132;
    cudaStream_t stream = nullptr;
    std::mutex mu;
    // workspaces (grow-only)
    DevMem w_rows, w_assign_i, w_assign_d, w_u32a, w_u32b, w_u32c, w_u32d, w_cnt, w_plan, w_sort, w_q, w_qraw, w_probe, w_pd, w_items,
        w_qbuf, w_inv, w_ppb, w_pconst, w_qconst, w_qb, w_cs, w_pk, w_pi, w_pw, w_lk, w_li, w_alive, w_od, w_oi, w_cand, w_host_q, w_ppopc, w_lut,
        w_stage, w_qrot;
    // build: one flag per row of the chunk or training sample, 1 = usable (row_usable_kernel)
    DevMem w_usable;
    // filter_probe=1 (per search): list_alive and the filtered lengths [2][nlist], the filtered page table [pages_used], the
    // per-query selection (p_q, cut key, cut ties, then the Σ / max totals); pinned host copy of the totals and of every p_q
    DevMem w_flist, w_fpages, w_fsel;
    void *h_fsel = nullptr;
    size_t h_fsel_cap = 0;
    // lists each query of the last search probed (b200_index_last_probe), and whether the filter_probe exact rule answered it
    std::vector<int32_t> last_probe;
    bool last_probe_exact = false;
    int last_coarse = 0;   // coarse-probe path of the last float list search (b200_index_last_coarse), 0 = none
    // statistics of the last search (tests, bench roofline): rows x payload bytes the scan kernel was asked to stream
    int64_t last_scan_rows = 0, last_items = 0;
    // graph_degree=D (HNSWFLAT, MSTG, BINARYMSTG): neighbour graph [n][D] u32 built at finalize, 0xFFFFFFFF = empty slot
    // (graph_sm90.cu); MSTG and BINARYMSTG walk their bf16 / binary list rows in place: d_row_slot[n] = row id -> pool slot,
    // derived from the page chains at finalize and at load (never saved: a load may place the pages elsewhere)
    int graph_degree = 0;
    DevMem d_graph, d_row_slot;     // uint32
    // seed ids [last_seed_nq][last_seed_s] of the last graph search (b200_index_last_seeds), and their first-stage distances
    DevMem w_seeds, w_seedd;
    int64_t last_seed_nq = 0;
    int last_seed_s = 0;
    bool last_graph = false;        // the last search walked the graph: last_scan reports the rows it scored
    bool timing = false, timed_pending = false;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    cudaEvent_t ev_ph[6] = {};      // phase boundaries of the last search: start | coarse | pairs+plan+gather | scan | merge | refine
    double phase_ms[5] = {0, 0, 0, 0, 0};
    double timed_ms = 0;
    int64_t timed_launches = 0;
};

static void timing_collect(b200_index *ix);

// internal hooks into capi.cu
extern "C" int b200_corpus_search_device(b200_corpus *c, const float *d_queries, int64_t nq, int k, const uint8_t *d_alive_bits,
                                         int64_t id_offset, float *d_out_dis, int64_t *d_out_ids, void *stream);
extern "C" int b200_corpus_set_path(b200_corpus *c, int path);
namespace b200 {
const void *corpus_device_rows(const b200_corpus *c);
int corpus_normalize_rows(b200_corpus *c);
int corpus_append_device(b200_corpus *c, const float *d_rows, int64_t n, cudaStream_t s);
int corpus_search_exact(b200_corpus *c, const void *d_queries, int64_t nq, int k, const uint8_t *d_alive, const uint8_t *h_alive,
                        int prefilter_mode, int64_t id_offset, float *d_out_dis, int64_t *d_out_ids, cudaStream_t s);
int64_t host_count_alive(const uint8_t *bits, int64_t n, int64_t limit);
int64_t corpus_prefilter_limit(const b200_corpus *c, int mode, int64_t nq, int k);
// hook for comm.cu: b200_sharded_index_search refuses a metric other than the index's
int index_metric(const b200_index *ix) { return ix->metric; }
}

// signed: a value with a leading '-' is read too (else such a key reads as absent)
static int parse_int_param(const char *json, const char *key, int defv, bool signed_value = false) {
    if (!json) return defv;
    const size_t kl = strlen(key);
    for (const char *p = strstr(json, key); p; p = strstr(p + 1, key)) {
        // whole-word match: "m" must not hit "nprobe_m..." or the tail of "num"
        const bool left_ok = p == json || !(isalnum((unsigned char)p[-1]) || p[-1] == '_');
        const char *e = p + kl;
        const bool right_ok = !(isalnum((unsigned char)*e) || *e == '_');
        if (!left_ok || !right_ok) continue;
        while (*e && (*e == '"' || *e == ':' || *e == '=' || *e == ' ' || *e == '\'')) e++;
        if (signed_value && *e == '-' && e[1] >= '0' && e[1] <= '9') return atoi(e);
        if (!(*e >= '0' && *e <= '9')) continue;
        return atoi(e);
    }
    return defv;
}

// float value of a key, whole-word matched as parse_int_param: 0 with *out = defv when the key is absent, -1 when its value is
// not a number (the value runs to the next ',', '"', '\'', '}', ' ' or the end)
static int parse_float_param(const char *json, const char *key, double defv, double *out) {
    *out = defv;
    if (!json) return 0;
    const size_t kl = strlen(key);
    for (const char *p = strstr(json, key); p; p = strstr(p + 1, key)) {
        const bool left_ok = p == json || !(isalnum((unsigned char)p[-1]) || p[-1] == '_');
        const char *e = p + kl;
        const bool right_ok = !(isalnum((unsigned char)*e) || *e == '_');
        if (!left_ok || !right_ok) continue;
        while (*e && (*e == '"' || *e == ':' || *e == '=' || *e == ' ' || *e == '\'')) e++;
        char *end = nullptr;
        const double v = (*e >= '0' && *e <= '9') || *e == '.' || *e == '-' || *e == '+' ? strtod(e, &end) : 0.0;
        if (!end || end == e || !(*end == 0 || strchr(",\"'} ", *end)) || !std::isfinite(v)) return -1;
        *out = v;
        return 0;
    }
    return 0;
}

// The search keys of a params string (include/b200_search.h), read once per search by search_opts, their only reader; params
// null: the index's defaults.  Only search_width is read signed: a negative value of another key reads as absent.  Reading
// validates nothing: each key is checked where the path that uses it runs, so a key of a path not taken is accepted as given.
struct SearchOpts {
    int exact_batch, prefilter, filter_probe;
    int nprobe;          // clamped to [1, nlist]
    int max_nprobe;      // clamped to [nprobe, nlist]
    int refine_factor;   // at least 1
    int graph, ef_s, search_width;
    int coarse_path, pages_per_chunk, shared_bound;   // A/B switches
};

static SearchOpts search_opts(const b200_index *ix, const char *params) {
    SearchOpts o;
    o.exact_batch = parse_int_param(params, "exact_batch", 0);
    o.prefilter = parse_int_param(params, "prefilter", 0);
    o.filter_probe = parse_int_param(params, "filter_probe", 0);
    o.nprobe = std::max(1, std::min(parse_int_param(params, "nprobe", ix->default_nprobe), ix->nlist));
    o.max_nprobe = std::max(o.nprobe, std::min(ix->nlist, parse_int_param(params, "max_nprobe", ix->nlist)));
    o.refine_factor = std::max(1, parse_int_param(params, "refine_factor", parse_int_param(params, "reorder_k_factor", ix->refine_factor)));
    o.graph = parse_int_param(params, "graph", 1);
    o.ef_s = parse_int_param(params, "ef_s", 64);
    o.search_width = parse_int_param(params, "search_width", 1, true);
    o.coarse_path = parse_int_param(params, "coarse_path", 0);
    o.pages_per_chunk = parse_int_param(params, "pages_per_chunk", 0);
    o.shared_bound = parse_int_param(params, "shared_bound", 1);
    return o;
}

extern "C" int b200_index_create(const char *type, int metric, int d, const char *params, b200_index **out) {
    if (!type || !out || d <= 0) return fail(B200_ERR_INVALID, "bad arguments");
    *out = nullptr;
    const bool float_metric = metric == B200_METRIC_L2 || metric == B200_METRIC_IP || metric == B200_METRIC_COSINE;
    const bool bin_metric = metric == B200_METRIC_HAMMING || metric == B200_METRIC_JACCARD;
    if (!float_metric && !bin_metric) return fail(B200_ERR_INVALID, "unknown metric");
    std::string t(type);
    for (auto &ch : t) ch = (char)toupper((unsigned char)ch);
    int ty = -1;
    for (int i = 0; i < IDX_NUM_TYPES; i++)
        if (t == kTypeNames[i]) ty = i;
    if (ty < 0)
        return fail(B200_ERR_UNSUPPORTED, "index type " + t + " is not implemented (FLAT, IVFFLAT, IVFSQ, IVFPQ, SCANN, MSTG, HNSWFLAT, HNSWSQ, HNSWPQ, "
                                          "BINARYFLAT, BINARYIVF, BINARYHNSW, BINARYMSTG)");
    const bool bin = ty >= IDX_BINFLAT;
    if (bin && !bin_metric) return fail(B200_ERR_INVALID, "binary indexes take HAMMING or JACCARD");
    if (!bin && !float_metric) return fail(B200_ERR_INVALID, "float indexes take L2, IP or COSINE");
    if (bin && (d % 8 != 0 || d > (1 << 16))) return fail(B200_ERR_INVALID, "binary dimension must be a multiple of 8 bits, at most 65536");
    if (!bin && ty != IDX_FLAT && d > B200_MAX_FLOAT_DIM)
        return fail(B200_ERR_UNSUPPORTED, "index type " + t + ": d must be at most B200_MAX_FLOAT_DIM = " + std::to_string(B200_MAX_FLOAT_DIM) + ", got " +
                                              std::to_string(d));
    // PQ code width (IVFPQ, SCANN, HNSWPQ only; the other types ignore the key)
    const bool pq_type = ty == IDX_IVFPQ || ty == IDX_SCANN || ty == IDX_HNSWPQ;
    const int pq_bits = pq_type ? parse_int_param(params, "bit_size", 8) : 8;
    if (pq_bits != 8 && pq_bits != 4) return fail(B200_ERR_UNSUPPORTED, "PQ bit_size must be 8 or 4, got " + std::to_string(pq_bits));
    // anisotropic PQ (the PQ types only; the others ignore the key): 0 < T < 1, or 0 / absent for plain PQ
    double aq_t = 0;
    if (pq_type) {
        if (parse_float_param(params, "aq_threshold", 0.0, &aq_t) != 0 || aq_t < 0 || aq_t >= 1)
            return fail(B200_ERR_INVALID, "aq_threshold must be a number with 0 < T < 1 (or 0: plain PQ)");
        if (aq_t > 0 && metric == B200_METRIC_L2)
            return fail(B200_ERR_UNSUPPORTED, "aq_threshold: the anisotropic loss is defined for inner-product ranking (IP, COSINE), not L2");
    }
    // optimised PQ (the PQ types only; the others ignore the keys): opq=1 learns a rotation in opq_iters alternations
    const int opq = pq_type ? parse_int_param(params, "opq", 0, true) : 0;
    const int opq_iters = pq_type ? parse_int_param(params, "opq_iters", 20, true) : 20;
    if (opq != 0 && opq != 1) return fail(B200_ERR_INVALID, "opq must be 0 (plain PQ) or 1 (optimised PQ), got " + std::to_string(opq));
    if (opq_iters < 0) return fail(B200_ERR_INVALID, "opq_iters must be >= 0, got " + std::to_string(opq_iters));
    if (opq && d > kOpqMaxDim)
        return fail(B200_ERR_UNSUPPORTED, "opq=1: the rotation is d x d fp32, d must be at most " + std::to_string(kOpqMaxDim) + ", got " + std::to_string(d));
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return fail(B200_ERR_NO_DEVICE, "no CUDA device visible; libb200search has no CPU fallback");
    }
    b200_index *ix = new b200_index();
    ix->type = ty;
    ix->metric = metric;
    ix->d = d;
    ix->d_pad = (int)round_up(d, 4);
    ix->d_pad64 = (int)round_up(d, 64);
    ix->nlist = parse_int_param(params, "ncentroids", parse_int_param(params, "nlist", 0));
    ix->m = parse_int_param(params, "M", parse_int_param(params, "m", 0));
    ix->pq_bits = pq_bits;
    ix->aq_threshold = aq_t;
    ix->aq_eta = (d - 1) * aq_t * aq_t / (1 - aq_t * aq_t);
    ix->opq = opq;
    ix->opq_iters = opq_iters;
    ix->default_nprobe = parse_int_param(params, "nprobe", 32);
    // payload of a list row.  The graph types of the reference (hnswlib) and ScaNN have no graph here (ScaNN's anisotropic
    // loss is the opt-in aq_threshold): they are SERVED by the inverted-file engine with the payload their suffix names
    // (recall contract, SURVEY 8c).
    switch (ty) {
        case IDX_IVFPQ: case IDX_SCANN: case IDX_HNSWPQ: ix->payload = IVF_PRODUCER_PQ; break;
        case IDX_IVFSQ: case IDX_HNSWSQ: ix->payload = IVF_PRODUCER_SQ8; break;
        case IDX_BINFLAT: case IDX_BINIVF: case IDX_BINHNSW: case IDX_BINMSTG: ix->payload = IVF_PRODUCER_B1; break;
        default: ix->payload = IVF_PRODUCER_TMA;
    }
    if (bin) {
        // Binary types: BINARYHNSW / BINARYMSTG are served by the binary inverted-file engine (BINARYMSTG walks a graph over its
        // list rows with graph_degree); list rows are exact, so there is no second stage.  k-block width kb_w = the row rounded
        // up to 16 bytes, at most 128 (one 1024-bit wgmma k-block); TMA zero-fills the rest of the 128-byte box.
        ix->binary = true;
        ix->row_bytes = d / 8;
        ix->kb_w = (int)std::min<int64_t>(128, round_up(ix->row_bytes, 16));
        ix->row_pad = (int)round_up(ix->row_bytes, ix->kb_w);
        ix->cent_pad = (int)round_up(ix->row_bytes, 16);
    }
    // candidates re-ranked exactly per returned row when fp32 rows are kept; plain IVFPQ / IVFSQ return first-stage
    // (ADC) distances like Faiss unless asked (refine_factor > 1)
    const int dflt_refine = (ty == IDX_IVFPQ || ty == IDX_IVFSQ || bin) ? 1 : (ix->payload == IVF_PRODUCER_PQ ? 16 : 4);
    ix->refine_factor = parse_int_param(params, "refine_factor", parse_int_param(params, "reorder_k_factor", dflt_refine));
    ix->keep_raw = parse_int_param(params, "keep_raw", -1);
    // graph_degree=D: HNSWFLAT, walked over its fp32 rows in HBM, MSTG, walked over its bf16 list rows with any keep_raw, or
    // BINARYMSTG, walked over its binary list rows (the reference's m is PQ M here and keeps that meaning)
    ix->graph_degree = parse_int_param(params, "graph_degree", 0);
    if (ix->graph_degree > 0) {
        if (ty != IDX_HNSWFLAT && ty != IDX_MSTG && ty != IDX_BINMSTG) {
            delete ix;
            return fail(B200_ERR_UNSUPPORTED,
                        "graph_degree: a neighbour graph is built on HNSWFLAT, MSTG and BINARYMSTG only (the other types keep quantised rows, or are BINARYHNSW / BINARYIVF)");
        }
        if (!graph_degree_ok(ix->graph_degree)) {
            const int gd = ix->graph_degree;
            delete ix;
            return fail(B200_ERR_INVALID, "graph_degree must be 16, 32 or 64 (or 0: no graph), got " + std::to_string(gd));
        }
        if (ty == IDX_HNSWFLAT && (ix->keep_raw == 0 || ix->keep_raw == 2)) {
            delete ix;
            return fail(B200_ERR_UNSUPPORTED, "graph_degree: the graph search reads the fp32 rows in HBM (keep_raw=1)");
        }
    }
    cudaGetDevice(&ix->device);
    cudaDeviceGetAttribute(&ix->sms, cudaDevAttrMultiProcessorCount, ix->device);
    if (cudaStreamCreateWithFlags(&ix->stream, cudaStreamNonBlocking) != cudaSuccess) {
        delete ix;
        return fail(B200_ERR_CUDA, "cudaStreamCreate failed");
    }
    *out = ix;
    return B200_OK;
}

extern "C" int b200_index_free(b200_index *ix) {
    if (!ix) return B200_OK;
    cudaSetDevice(ix->device);
    if (ix->stream) cudaStreamSynchronize(ix->stream);
    if (ix->h_rows) cudaFreeHost(ix->h_rows);
    if (ix->h_fsel) cudaFreeHost(ix->h_fsel);
    if (ix->ev0) cudaEventDestroy(ix->ev0);
    if (ix->ev1) cudaEventDestroy(ix->ev1);
    for (auto &e : ix->ev_ph)
        if (e) cudaEventDestroy(e);
    if (ix->stream) cudaStreamDestroy(ix->stream);
    delete ix;
    return B200_OK;
}

// PQ sub-vectors the tensor-core decoder takes (d / M = 1, 2, 4, 8); any other d / M is scanned by table look-up
static bool pq_dsub_decodable(int dsub) { return dsub == 1 || dsub == 2 || dsub == 4 || dsub == 8; }
// 4-bit codes are always scanned by table look-up (ivf_pq4_sm90.cu), whatever d / M
static bool pq_uses_lut(const b200_index *ix) {
    return ix->payload == IVF_PRODUCER_PQ && ix->use_ivf && (ix->pq_bits == 4 || !pq_dsub_decodable(ix->dsub));
}
// codewords per sub-quantiser, and the bytes of one code row: one byte per 8-bit code, two 4-bit codes per byte
static int pq_codewords(int bits) { return bits == 4 ? 16 : 256; }
static int pq_code_bytes(int m, int bits) { return (int)round_up(bits == 4 ? (m + 1) / 2 : m, 16); }

// the per-query tables of the look-up scan take at most this much scratch; larger batches run in query sub-batches
constexpr int64_t kPqLutScratchBytes = (int64_t)256 << 20;
static int64_t pq_lut_max_queries(const b200_index *ix) { return std::max<int64_t>(1, kPqLutScratchBytes / ((int64_t)ix->m * pq_codewords(ix->pq_bits) * 4)); }

static size_t payload_row_bytes(const b200_index *ix) {
    if (ix->payload == IVF_PRODUCER_B1) return (size_t)ix->row_pad;
    return ix->payload == IVF_PRODUCER_TMA ? (size_t)ix->d_pad64 * 2 : (size_t)ix->code_bytes;
}

// bytes of one caller row: fp32 [d], or binary [d / 8]
static size_t in_row_bytes(const b200_index *ix) { return ix->binary ? (size_t)ix->row_bytes : (size_t)ix->d * 4; }

// fp32 rows for the exact paths, in HBM (raw) or in host memory (h_rows)
static bool has_rows(const b200_index *ix) { return ix->raw || ix->h_rows; }

// the candidates' rows gathered from host memory take at most this much staging; larger batches re-rank in query chunks
constexpr int64_t kHostStageBytes = (int64_t)256 << 20;

// keep_raw=2: room for `rows` host rows in pinned, mapped memory; grows by allocate, copy the ix->n rows held, free
static int host_rows_reserve(b200_index *ix, int64_t rows) {
    if (ix->h_rows && ix->h_rows_cap >= rows) return B200_OK;
    const size_t row_b = (size_t)ix->d_pad * 4, bytes = (size_t)rows * row_b, keep = (size_t)ix->n * row_b;
    void *p = nullptr, *dp = nullptr;
    if (cudaHostAlloc(&p, std::max<size_t>(bytes, 16), cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) {
        cudaGetLastError();
        return fail(B200_ERR_NOMEM, "cudaHostAlloc of the host rows failed (" + std::to_string(bytes) + " bytes)");
    }
    if (cudaHostGetDevicePointer(&dp, p, 0) != cudaSuccess) {
        cudaGetLastError();
        cudaFreeHost(p);
        return fail(B200_ERR_CUDA, "cudaHostGetDevicePointer of the host rows failed");
    }
    if (ix->h_rows) {
        memcpy(p, ix->h_rows, keep);
        cudaFreeHost(ix->h_rows);
    }
    if (ix->d != ix->d_pad) memset(reinterpret_cast<char *>(p) + keep, 0, bytes - keep);   // the padding columns stay 0
    ix->h_rows = reinterpret_cast<float *>(p);
    ix->h_rows_dev = reinterpret_cast<const float *>(dp);
    ix->h_rows_cap = rows;
    return B200_OK;
}

// a new empty corpus in `out`, whose old one is freed first
static int corpus_create(int metric, int dtype, int d, int64_t capacity_rows, CorpusPtr &out) {
    out.reset();
    b200_corpus *c = nullptr;
    B200_TRY(b200_corpus_create(metric, dtype, d, capacity_rows, &c));
    out.reset(c);
    return B200_OK;
}

// k-means on device rows x [n][stride]; centroids written to d_c [nc][d].  Assignment: exact top-1 search of the centroid
// table with the FLAT engine (tensor cores from 20 rows up) when the table is large, the tiled fp32 kernel otherwise.
// warm: start from the centroids already in d_c (OPQ's alternations) instead of nc evenly strided rows.
static int kmeans_device(const float *x, int64_t n, int64_t stride, int d, int nc, int iters, float *d_c, cudaStream_t s, bool warm = false) {
    std::vector<int64_t> pick(nc);
    for (int i = 0; i < nc; i++) pick[i] = (int64_t)((double)i * (double)n / (double)nc);
    DevMem pick_b, sums_b, cn_b, cnt_b, idx_b, idx64_b, dis_b;
    B200_TRY(pick_b.alloc((size_t)nc * 8));
    B200_TRY(sums_b.alloc((size_t)nc * d * 4));
    B200_TRY(cn_b.alloc((size_t)nc * 4));
    B200_TRY(cnt_b.alloc((size_t)nc * 4));
    B200_TRY(idx_b.alloc((size_t)n * 4));
    int64_t *d_pick = pick_b.as<int64_t>();
    float *d_sums = sums_b.as<float>(), *d_cn = cn_b.as<float>();
    uint32_t *d_cnt = cnt_b.as<uint32_t>(), *d_idx = idx_b.as<uint32_t>();
    if (!warm) {
        B200_CUDA_OK(cudaMemcpyAsync(d_pick, pick.data(), (size_t)nc * 8, cudaMemcpyHostToDevice, s));
        gather_rows_kernel<<<gridsz((int64_t)nc * d), 256, 0, s>>>(x, stride, d_pick, nc, d, d_c);
        g_launches++;
    }
    const bool big = (double)n * nc * d > 2e11 && stride == d;   // tensor-core assignment pays from ~0.2 TFLOP per iteration
    if (big) {
        B200_TRY(idx64_b.alloc((size_t)n * 8));
        B200_TRY(dis_b.alloc((size_t)n * 4));
    }
    int64_t *d_idx64 = idx64_b.as<int64_t>();
    float *d_dis = dis_b.as<float>();
    CorpusPtr table;
    for (int it = 0; it < iters; it++) {
        if (big) {
            B200_TRY(corpus_create(B200_METRIC_L2, B200_DTYPE_F32, d, nc, table));
            B200_TRY(corpus_append_device(table.get(), d_c, nc, s));
            B200_TRY(b200_corpus_search_device(table.get(), x, n, 1, nullptr, 0, d_dis, d_idx64, s));
            B200_CUDA_OK(cudaMemsetAsync(d_cnt, 0, (size_t)nc * 4, s));
            assign_to_u32_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, s>>>(d_idx64, n, nullptr, 0u, d_idx, d_cnt);
            g_launches++;
        } else {
            rows_sqnorm_kernel<<<(unsigned)ceil_div(nc, 256), 256, 0, s>>>(d_c, nc, d, d_cn);
            kmeans_assign_kernel<<<(unsigned)ceil_div(n, KA_T), 256, 0, s>>>(x, n, stride, d, d_c, nc, d_cn, d_idx, nullptr);
            g_launches += 2;
        }
        B200_CUDA_OK(cudaMemsetAsync(d_sums, 0, (size_t)nc * d * 4, s));
        B200_CUDA_OK(cudaMemsetAsync(d_cnt, 0, (size_t)nc * 4, s));
        kmeans_accumulate_kernel<<<gridsz(n * d), 256, 0, s>>>(x, n, stride, d, d_idx, d_sums, d_cnt);
        kmeans_update_kernel<<<gridsz((int64_t)nc * d), 256, 0, s>>>(d_c, d_sums, d_cnt, nc, d);
        g_launches += 2;
        // empty clusters take half of the currently largest ones (both copies nudged apart; the next assignment splits the
        // members) -- without this a strided initialisation leaves a third of well-separated clusters without a centroid
        if (it + 1 < iters && nc >= 2) {
            std::vector<uint32_t> h_cnt(nc);
            B200_CUDA_OK(cudaMemcpyAsync(h_cnt.data(), d_cnt, (size_t)nc * 4, cudaMemcpyDeviceToHost, s));
            B200_CUDA_OK(cudaStreamSynchronize(s));
            std::vector<int> empties, order(nc);
            for (int i = 0; i < nc; i++) {
                order[i] = i;
                if (h_cnt[i] == 0) empties.push_back(i);
            }
            if (!empties.empty()) {
                // largest first, equal counts by the smaller cluster id: the pairing is a function of the counts alone
                std::partial_sort(order.begin(), order.begin() + std::min<size_t>(nc, empties.size()), order.end(),
                                  [&](int a, int b) { return h_cnt[a] != h_cnt[b] ? h_cnt[a] > h_cnt[b] : a < b; });
                std::vector<int> pairs;
                for (size_t e = 0; e < empties.size() && e < (size_t)nc; e++) {
                    const int src = order[e];
                    if (h_cnt[src] < 2) break;
                    pairs.push_back(empties[e]);
                    pairs.push_back(src);
                }
                if (!pairs.empty()) {
                    DevMem d_pairs;
                    B200_TRY(d_pairs.alloc(pairs.size() * 4));
                    B200_CUDA_OK(cudaMemcpyAsync(d_pairs.p, pairs.data(), pairs.size() * 4, cudaMemcpyHostToDevice, s));
                    kmeans_split_kernel<<<(unsigned)(pairs.size() / 2), 128, 0, s>>>(d_c, d_pairs.as<int>(), d);
                    g_launches++;
                    B200_CUDA_OK(cudaStreamSynchronize(s));
                }
            }
        }
    }
    B200_CUDA_OK(cudaGetLastError());
    B200_CUDA_OK(cudaStreamSynchronize(s));
    return B200_OK;
}

// total rows the index will hold (Search::createVectorIndex's total_vec, VIWithDataPart.cpp:416-430): sizes the page pool
extern "C" int b200_index_reserve(b200_index *ix, int64_t total_rows) {
    if (!ix || total_rows < 0) return fail(B200_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(ix->mu);
    if (ix->trained || ix->n) return fail(B200_ERR_INVALID, "reserve comes before train / add");
    ix->reserved = total_rows;
    return B200_OK;
}

static int upload_coarse(b200_index *ix, cudaStream_t s) {
    // L2 for every metric (unit vectors under cosine; IP indexes probe by L2 too, like Faiss's default quantiser)
    B200_TRY(corpus_create(B200_METRIC_L2, B200_DTYPE_F32, ix->d, ix->nlist, ix->coarse));
    B200_TRY(ix->d_cnorm.alloc((size_t)ix->nlist * 4));
    B200_CUDA_OK(launch_row_norms(ix->d_centroids.as<float>(), 0, ix->d, ix->nlist, 0, ix->d_cnorm.as<float>(), s));
    return corpus_append_device(ix->coarse.get(), ix->d_centroids.as<float>(), ix->nlist, s);
}

// binary centroid table as a Hamming corpus of cent_pad-byte rows (a multiple of 16 bytes: always on the b1 tensor path)
static int upload_coarse_bin(b200_index *ix, cudaStream_t s) {
    B200_TRY(corpus_create(B200_METRIC_HAMMING, B200_DTYPE_BIN, ix->cent_pad * 8, ix->nlist, ix->coarse));
    return corpus_append_device(ix->coarse.get(), reinterpret_cast<const float *>(ix->d_bcent.as<uint8_t>()), ix->nlist, s);
}

// binary rows [n][row_bytes] (device) -> dst [n][cent_pad], zero-padded: the form the coarse table is searched with
static int pad_bin_rows(const b200_index *ix, const void *d_rows, int64_t n, DevMem &dst, cudaStream_t s) {
    B200_TRY(dst.reserve((size_t)std::max<int64_t>(n, 1) * ix->cent_pad));
    if (n == 0) return B200_OK;
    B200_CUDA_OK(cudaMemsetAsync(dst.p, 0, (size_t)n * ix->cent_pad, s));
    B200_CUDA_OK(cudaMemcpy2DAsync(dst.p, ix->cent_pad, d_rows, ix->row_bytes, ix->row_bytes, n, cudaMemcpyDeviceToDevice, s));
    return B200_OK;
}

// k-majority (binary k-means) on device rows x [n][stride] bytes (zero-padded, stride % 16 == 0, rb bytes of data); centroids
// d_c [nc][stride].  Assignment: exact top-1 Hamming search of the centroid table (ties to the smaller centroid id); update: every
// centroid bit is the majority of its members' bits (a tie keeps the bit); empty clusters take the middle member (in row order)
// of the largest clusters.  Stops early when no assignment changes.  Integer work only: the result is deterministic.
static int kmajority_device(const uint8_t *x, int64_t n, int stride, int rb, int nc, int iters, uint8_t *d_c, cudaStream_t s) {
    std::vector<int64_t> pick(nc);
    for (int i = 0; i < nc; i++) pick[i] = (int64_t)((double)i * (double)n / (double)nc);
    // per-(cluster, bit) counts for <= 64 M counters (256 MB) at a time
    const int chunk = (int)std::max<int64_t>(1, std::min<int64_t>(nc, ((int64_t)64 << 20) / ((int64_t)rb * 8)));
    DevMem pick_b, idx64_b, dis_b, idx_b, prev_b, cnt_b, changed_b, bits_b;
    B200_TRY(pick_b.alloc((size_t)nc * 8));
    B200_TRY(idx64_b.alloc((size_t)n * 8));
    B200_TRY(dis_b.alloc((size_t)n * 4));
    B200_TRY(idx_b.alloc((size_t)n * 4));
    B200_TRY(prev_b.alloc((size_t)n * 4));
    B200_TRY(cnt_b.alloc((size_t)nc * 4));
    B200_TRY(changed_b.alloc(4));
    B200_TRY(bits_b.alloc((size_t)chunk * rb * 8 * 4));
    int64_t *d_pick = pick_b.as<int64_t>(), *d_idx64 = idx64_b.as<int64_t>();
    float *d_dis = dis_b.as<float>();
    uint32_t *d_idx = idx_b.as<uint32_t>(), *d_prev = prev_b.as<uint32_t>(), *d_cnt = cnt_b.as<uint32_t>(), *d_changed = changed_b.as<uint32_t>(),
             *d_bits = bits_b.as<uint32_t>();
    B200_CUDA_OK(cudaMemcpyAsync(d_pick, pick.data(), (size_t)nc * 8, cudaMemcpyHostToDevice, s));
    gather_bytes_kernel<<<gridsz((int64_t)nc * stride), 256, 0, s>>>(x, stride, d_pick, nc, d_c);
    B200_CUDA_OK(cudaMemsetAsync(d_prev, 0xff, (size_t)n * 4, s));
    g_launches++;
    std::vector<uint32_t> h_cnt(nc), h_idx;
    CorpusPtr table;
    for (int it = 0; it < iters; it++) {
        B200_TRY(corpus_create(B200_METRIC_HAMMING, B200_DTYPE_BIN, stride * 8, nc, table));
        B200_TRY(corpus_append_device(table.get(), reinterpret_cast<const float *>(d_c), nc, s));
        B200_TRY(b200_corpus_search_device(table.get(), reinterpret_cast<const float *>(x), n, 1, nullptr, 0, d_dis, d_idx64, s));
        B200_CUDA_OK(cudaMemsetAsync(d_cnt, 0, (size_t)nc * 4, s));
        B200_CUDA_OK(cudaMemsetAsync(d_changed, 0, 4, s));
        assign_to_u32_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, s>>>(d_idx64, n, nullptr, 0u, d_idx, d_cnt);
        count_changes_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, s>>>(d_idx, d_prev, n, d_changed);
        g_launches += 2;
        uint32_t changed = 0;
        B200_CUDA_OK(cudaMemcpyAsync(&changed, d_changed, 4, cudaMemcpyDeviceToHost, s));
        B200_CUDA_OK(cudaMemcpyAsync(h_cnt.data(), d_cnt, (size_t)nc * 4, cudaMemcpyDeviceToHost, s));
        B200_CUDA_OK(cudaStreamSynchronize(s));
        if (it > 0 && changed == 0) break;   // the centroids already are the majorities of this assignment
        for (int c0 = 0; c0 < nc; c0 += chunk) {
            const int c1 = std::min(nc, c0 + chunk);
            B200_CUDA_OK(cudaMemsetAsync(d_bits, 0, (size_t)(c1 - c0) * rb * 8 * 4, s));
            bin_bit_count_kernel<<<gridsz(n * rb), 256, 0, s>>>(x, n, stride, rb, d_idx, (uint32_t)c0, (uint32_t)c1, d_bits);
            bin_majority_kernel<<<gridsz((int64_t)(c1 - c0) * rb), 256, 0, s>>>(d_c, stride, rb, d_bits, d_cnt, (uint32_t)c0, (uint32_t)c1);
            g_launches += 2;
        }
        if (it + 1 < iters && nc >= 2) {
            std::vector<int> empties, order(nc);
            for (int i = 0; i < nc; i++) {
                order[i] = i;
                if (h_cnt[i] == 0) empties.push_back(i);
            }
            if (empties.empty()) continue;
            std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return h_cnt[a] > h_cnt[b]; });
            h_idx.resize(n);
            B200_CUDA_OK(cudaMemcpyAsync(h_idx.data(), d_idx, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
            B200_CUDA_OK(cudaStreamSynchronize(s));
            std::vector<int> dst_of(nc, -1);   // large cluster -> the empty one that takes its middle member
            for (size_t e = 0; e < empties.size(); e++) {
                const int src = order[e];
                if (h_cnt[src] < 2) break;
                dst_of[src] = empties[e];
            }
            std::vector<uint32_t> seen(nc, 0);
            for (int64_t r = 0; r < n; r++) {
                const uint32_t l = h_idx[r];
                if (dst_of[l] >= 0 && seen[l]++ == h_cnt[l] / 2)
                    B200_CUDA_OK(cudaMemcpyAsync(d_c + (size_t)dst_of[l] * stride, x + r * stride, stride, cudaMemcpyDeviceToDevice, s));
            }
        }
    }
    B200_CUDA_OK(cudaGetLastError());
    B200_CUDA_OK(cudaStreamSynchronize(s));
    return B200_OK;
}

// FLAT fallback for small parts (the reference's fallback_to_flat, test 00029) and the default nlist
static void decide_ivf(b200_index *ix, int64_t total, int64_t n) {
    const bool want_ivf = !is_flat_type(ix->type);
    if (want_ivf && ix->nlist <= 0)
        ix->nlist = (int)std::max<int64_t>(1, std::min<int64_t>(65536, (int64_t)(4.0 * sqrt((double)std::max<int64_t>(total, 1)))));
    ix->use_ivf = want_ivf && total >= std::max<int64_t>(2000, 8ll * ix->nlist) && n >= ix->nlist;
}

// page pool for `total` rows: every list wastes less than one page
static int alloc_pool(b200_index *ix, int64_t total, cudaStream_t s) {
    const int nl = ix->nlist;
    const int64_t pages = ceil_div(total, kPageRows) + nl;
    if (pages * kPageRows >= (int64_t)0xffffffffll) return fail(B200_ERR_UNSUPPORTED, "an index shard is limited to 2^32 - 1 pool rows");
    ix->pool_pages = (uint32_t)pages;
    const size_t rows = (size_t)pages * kPageRows;
    if (ix->d_pool.alloc(rows * payload_row_bytes(ix) + 256) != B200_OK)
        return fail(B200_ERR_NOMEM, "cudaMalloc of the page pool failed (" + std::to_string(rows * payload_row_bytes(ix)) + " bytes)");
    B200_CUDA_OK(cudaMemsetAsync(ix->d_pool.p, 0, rows * payload_row_bytes(ix), s));
    B200_TRY(ix->d_row_ids.alloc(rows * 4));
    if (ix->metric == B200_METRIC_L2 || ix->binary) B200_TRY(ix->d_row_bias.alloc(rows * 4));
    B200_TRY(ix->d_list_len.alloc((size_t)nl * 4));
    B200_TRY(ix->d_tail_page.alloc((size_t)nl * 4));
    B200_TRY(ix->d_page_owner.alloc((size_t)pages * 4));
    B200_TRY(ix->d_page_seq.alloc((size_t)pages * 4));
    B200_TRY(ix->d_pages_used.alloc(4));
    B200_TRY(ix->d_flag.alloc(32));
    B200_CUDA_OK(cudaMemsetAsync(ix->d_list_len.as<uint32_t>(), 0, (size_t)nl * 4, s));
    B200_CUDA_OK(cudaMemsetAsync(ix->d_tail_page.as<uint32_t>(), 0, (size_t)nl * 4, s));
    B200_CUDA_OK(cudaMemsetAsync(ix->d_pages_used.as<uint32_t>(), 0, 4, s));
    B200_CUDA_OK(cudaMemsetAsync(ix->d_flag.as<int>(), 0, 32, s));
    return B200_OK;
}

// binary train: k-majority coarse quantiser on a device sample [n][row_bytes] (no codebooks)
static int train_binary_locked(b200_index *ix, const void *d_rows, int64_t n) {
    cudaStream_t s = ix->stream;
    const int64_t total = ix->reserved > 0 ? ix->reserved : n;
    decide_ivf(ix, total, n);
    if (!ix->use_ivf) {
        ix->keep_raw = 1;
        ix->trained = true;
        return B200_OK;
    }
    ix->keep_raw = 0;   // list rows are exact: nothing to re-rank
    B200_TRY(pad_bin_rows(ix, d_rows, n, ix->w_rows, s));
    B200_TRY(ix->d_bcent.alloc((size_t)ix->nlist * ix->cent_pad));
    B200_TRY(kmajority_device(ix->w_rows.as<uint8_t>(), n, ix->cent_pad, ix->row_bytes, ix->nlist, 10, ix->d_bcent.as<uint8_t>(), s));
    B200_TRY(upload_coarse_bin(ix, s));
    B200_TRY(alloc_pool(ix, total, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    ix->trained = true;
    return B200_OK;
}

// opq=1: from the PQ training sample samp [ns][d] (as indexed) and its lists, the OPQ alternations (Ge et al. 2014, the
// non-parametric solution).  Res = samp - c.  Start: R = I, codebooks by k-means on Res.R (8 iterations, as plain PQ).  Then
// opq_iters times: R = polar(Res^T Res^) for the decoded codes Res^ of Res.R (the Procrustes step), and a warm-started k-means
// of 4 iterations per sub-quantiser on the new Res.R (Faiss's count).  ix->opq_loss: the mean ||Res.R - Res^||^2 of the
// sample at R = I, then after each alternation.  The codebooks of the last alternation are the index's.  Finally the
// centroids (and the coarse table) and samp are rotated in place: the AQ iterations and the lists work in the rotated space.
static int opq_train_locked(b200_index *ix, float *samp, int64_t ns, const uint32_t *d_l) {
    cudaStream_t s = ix->stream;
    const int d = ix->d, m = ix->m, dsub = ix->dsub, ncw = pq_codewords(ix->pq_bits), nl = ix->nlist;
    const size_t rows_b = (size_t)ns * d * 4;
    // resr also takes the rotated centroids at the end: nlist may exceed the sample (ncentroids > 65 536)
    DevMem res_b, resr_b, xhat_b, err_b;
    B200_TRY(ix->d_opq.alloc((size_t)d * d * 4));
    B200_TRY(res_b.alloc(rows_b));
    B200_TRY(resr_b.alloc((size_t)std::max<int64_t>(ns, nl) * d * 4));
    B200_TRY(xhat_b.alloc(rows_b));
    B200_TRY(err_b.alloc((size_t)std::max<int64_t>(ns, 1) * 8));
    float *R = ix->d_opq.as<float>(), *centroids = ix->d_centroids.as<float>(), *pq = ix->d_pq.as<float>();
    float *res = res_b.as<float>(), *resr = resr_b.as<float>(), *xhat = xhat_b.as<float>();
    double *err = err_b.as<double>();
    std::vector<double> h_err(ns);
    auto loss = [&]() {   // encode Res.R with the current codebooks (-> xhat) and append the sample's mean loss
        B200_CUDA_OK(launch_opq_encode(resr, ns, d, m, dsub, ncw, pq, xhat, err, s));
        B200_CUDA_OK(cudaMemcpyAsync(h_err.data(), err, (size_t)ns * 8, cudaMemcpyDeviceToHost, s));
        B200_CUDA_OK(cudaStreamSynchronize(s));
        double t = 0;
        for (int64_t r = 0; r < ns; r++) t += h_err[r];
        ix->opq_loss.push_back(t / (double)std::max<int64_t>(ns, 1));
        return B200_OK;
    };
    auto codebooks = [&](int iters, bool warm) {   // Res.R (-> resr), then its k-means per sub-quantiser
        B200_CUDA_OK(launch_opq_rotate(res, d, ns, d, R, resr, d, s));
        for (int j = 0; j < m; j++) B200_TRY(kmeans_device(resr + (size_t)j * dsub, ns, d, dsub, ncw, iters, pq + (size_t)j * ncw * dsub, s, warm));
        return B200_OK;
    };
    ix->opq_loss.clear();
    std::vector<float> eye((size_t)d * d, 0.f);
    for (int i = 0; i < d; i++) eye[(size_t)i * d + i] = 1.f;
    B200_CUDA_OK(cudaMemcpyAsync(R, eye.data(), (size_t)d * d * 4, cudaMemcpyHostToDevice, s));
    residual_sub_kernel<<<gridsz(ns * d), 256, 0, s>>>(samp, ns, d, centroids, d_l, d, 0, d, res);
    g_launches++;
    B200_TRY(codebooks(8, false));
    B200_TRY(loss());
    for (int it = 0; it < ix->opq_iters; it++) {
        B200_TRY(opq_procrustes(res, xhat, ns, d, R, s));
        B200_TRY(codebooks(4, true));
        B200_TRY(loss());
    }
    // the centroids and the sample into the rotated space (resr and res are free now)
    B200_CUDA_OK(launch_opq_rotate(centroids, d, nl, d, R, resr, d, s));
    B200_CUDA_OK(cudaMemcpyAsync(centroids, resr, (size_t)nl * d * 4, cudaMemcpyDeviceToDevice, s));
    B200_CUDA_OK(launch_opq_rotate(samp, d, ns, d, R, res, d, s));
    B200_CUDA_OK(cudaMemcpyAsync(samp, res, rows_b, cudaMemcpyDeviceToDevice, s));
    B200_TRY(upload_coarse(ix, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    return B200_OK;
}

// Search::VectorIndex::train: coarse quantiser (+ PQ codebooks / SQ ranges) from a sample already on the device,
// rows fp32 [n][d] contiguous.  Decides FLAT fallback for small parts (the reference's fallback_to_flat, test 00029).
static int train_device_locked(b200_index *ix, const float *d_rows, int64_t n) {
    if (ix->trained) return fail(B200_ERR_INVALID, "index already trained");
    if (ix->built) return fail(B200_ERR_INVALID, "index already built");
    if (ix->binary) return train_binary_locked(ix, d_rows, n);
    cudaStream_t s = ix->stream;
    const int d = ix->d;
    // only the usable rows of the sample train, in their order and as given (before the cosine normalisation, which would
    // turn a row whose square overflows into a zero row); a sample without an unusable row is used in place
    const float *x = d_rows;
    if (n > 0) {
        B200_TRY(ix->w_usable.reserve((size_t)n));
        B200_TRY(ix->w_assign_i.reserve((size_t)(n + 1) * 8));
        uint8_t *usable = ix->w_usable.as<uint8_t>();
        int64_t *pick = ix->w_assign_i.as<int64_t>(), *d_kept = pick + n;
        row_usable_kernel<<<gridsz(n * 32), 256, 0, s>>>(d_rows, n, d, usable);
        g_launches++;
        size_t tb = 0;
        const cub::CountingInputIterator<int64_t> iota(0);
        B200_CUDA_OK(cub::DeviceSelect::Flagged(nullptr, tb, iota, usable, pick, d_kept, n, s));
        B200_TRY(ix->w_sort.reserve(tb + 256));
        B200_CUDA_OK(cub::DeviceSelect::Flagged(ix->w_sort.p, tb, iota, usable, pick, d_kept, n, s));
        int64_t kept = 0;
        B200_CUDA_OK(cudaMemcpyAsync(&kept, d_kept, 8, cudaMemcpyDeviceToHost, s));
        B200_CUDA_OK(cudaStreamSynchronize(s));
        if (kept < n) {
            B200_TRY(ix->w_rows.reserve((size_t)std::max<int64_t>(kept, 1) * d * 4));
            if (kept) gather_rows_kernel<<<gridsz(kept * d), 256, 0, s>>>(d_rows, d, pick, kept, d, ix->w_rows.as<float>());
            g_launches++;
            x = ix->w_rows.as<float>();
            n = kept;
        }
    }
    const int64_t total = ix->reserved > 0 ? ix->reserved : n;
    decide_ivf(ix, total, n);
    if (!ix->use_ivf) {
        ix->keep_raw = 1;
        ix->trained = true;
        return B200_OK;
    }
    if (ix->payload == IVF_PRODUCER_PQ) {
        if (ix->m <= 0) {
            if (d <= 220) {   // sub-vectors of <= 8 dims, decoded on the tensor cores
                ix->m = d;
                for (int cand : {8, 4, 2, 1})
                    if (d % cand == 0) { ix->m = d / cand; break; }
            } else {          // table look-up: the smallest sub-vector of >= 16 dims that divides d and keeps M <= 128
                int dsub = 16;
                while (d % dsub || d / dsub > 128) dsub++;
                ix->m = d / dsub;
            }
            // 4-bit codes: the code bytes of the 8-bit default (twice the sub-quantisers) when its sub-vector splits in two
            if (ix->pq_bits == 4 && (d / ix->m) % 2 == 0) ix->m *= 2;
        }
        if (d % ix->m) return fail(B200_ERR_INVALID, "PQ M must divide the dimension");
        const int dsub = d / ix->m;
        if (ix->aq_threshold > 0 && dsub > kAqMaxDsub)
            return fail(B200_ERR_UNSUPPORTED, "aq_threshold: the codebook update solves for sub-vectors of at most " + std::to_string(kAqMaxDsub) +
                                                  " dims (d / M <= " + std::to_string(kAqMaxDsub) + "), got d / M = " + std::to_string(dsub));
        if (ix->aq_threshold > 0 && !aq_encoder_smem(d, ix->m))
            return fail(B200_ERR_UNSUPPORTED, "aq_threshold: a row of d = " + std::to_string(d) + " does not fit the encoder's shared memory");
        if (ix->pq_bits == 4) {
            // the 4-bit look-up scan keeps one query's M x 64 B table in shared memory, at any d / M
            if (!ivf_pq4_fits(ix->m))
                return fail(B200_ERR_UNSUPPORTED, "4-bit PQ is scanned by table look-up, whose per-query table (M x 64 B) must fit in shared memory: M <= " +
                                                      std::to_string(ivf_pq4_max_m()) + ", got M = " + std::to_string(ix->m));
        } else if (pq_dsub_decodable(dsub)) {
            // the tensor-core scan keeps the bf16 codebook (512 B x d) in shared memory beside at least a 2-stage operand ring
            if (!ivf_pq_codebook_fits((int64_t)512 * d)) {
                int dmax = d;
                while (dmax > 1 && !ivf_pq_codebook_fits((int64_t)512 * dmax)) dmax--;
                return fail(B200_ERR_UNSUPPORTED, "PQ codebook (512 B x d) must fit in shared memory next to the operand ring: d <= " + std::to_string(dmax) +
                                                      " (or choose M with d / M >= 16, scanned by table look-up)");
            }
        } else if (!ivf_pq_lut_fits(ix->m)) {
            // the table look-up scan keeps one query's M x 256 fp32 table in shared memory
            int mmax = ix->m;
            while (mmax > 1 && !ivf_pq_lut_fits(mmax)) mmax--;
            return fail(B200_ERR_UNSUPPORTED, "PQ with d / M outside {1, 2, 4, 8} is scanned by table look-up, whose per-query table (M x 1 KB) "
                                              "must fit in shared memory: M <= " + std::to_string(mmax) + ", got M = " + std::to_string(ix->m));
        }
    }
    if (ix->keep_raw < 0) ix->keep_raw = 1;
    const int nl = ix->nlist;
    // training rows: unit length under cosine
    if (ix->metric == B200_METRIC_COSINE) {
        if (x != ix->w_rows.p) {
            B200_TRY(ix->w_rows.reserve((size_t)n * d * 4));
            B200_CUDA_OK(cudaMemcpyAsync(ix->w_rows.p, x, (size_t)n * d * 4, cudaMemcpyDeviceToDevice, s));
        }
        B200_CUDA_OK(launch_normalize_rows_f32(ix->w_rows.as<float>(), d, n, s));
        x = ix->w_rows.as<float>();
    }
    B200_TRY(ix->d_centroids.alloc((size_t)nl * d * 4));
    B200_TRY(kmeans_device(x, n, d, d, nl, 10, ix->d_centroids.as<float>(), s));
    B200_TRY(upload_coarse(ix, s));
    if (ix->payload == IVF_PRODUCER_SQ8) {
        ix->code_bytes = (int)round_up(d, 16);
        B200_TRY(ix->d_sq.alloc((size_t)4 * d * 4));
        float *lo = ix->d_sq.as<float>(), *hi = ix->d_sq.as<float>() + d;
        dim_minmax_kernel<<<d, 256, 0, s>>>(x, n, d, d, lo, hi);
        g_launches++;
        std::vector<float> h((size_t)4 * d);
        B200_CUDA_OK(cudaMemcpyAsync(h.data(), ix->d_sq.as<float>(), (size_t)2 * d * 4, cudaMemcpyDeviceToHost, s));
        B200_CUDA_OK(cudaStreamSynchronize(s));
        for (int j = 0; j < d; j++) {
            const float l = h[j], u = h[d + j];
            const float step = u > l ? (u - l) / 255.f : 1.f;
            h[d + j] = step;
            h[2 * d + j] = 1.f / step;
            h[3 * d + j] = l + 128.f * step;   // value of code 128 = the zero of the offset-binary code the scan decodes
        }
        B200_CUDA_OK(cudaMemcpyAsync(ix->d_sq.as<float>(), h.data(), (size_t)4 * d * 4, cudaMemcpyHostToDevice, s));
    }
    if (ix->payload == IVF_PRODUCER_PQ) {
        const int m = ix->m, dsub = d / m;   // validated above
        const int ncw = pq_codewords(ix->pq_bits);
        ix->dsub = dsub;
        ix->code_bytes = pq_code_bytes(m, ix->pq_bits);
        B200_TRY(ix->d_pq.alloc((size_t)m * ncw * dsub * 4));
        if (!pq_uses_lut(ix)) B200_TRY(ix->d_pq_bf16.alloc((size_t)m * 256 * dsub * 2));   // the decoder's copy
        // residuals of (a sample of) the training rows, one sub-quantiser at a time
        const int64_t ns = std::min<int64_t>(n, 65536);
        DevMem a_b, ad_b, l_b, c32_b, res_b, samp_b;
        B200_TRY(a_b.alloc((size_t)ns * 8));
        B200_TRY(ad_b.alloc((size_t)ns * 4));
        B200_TRY(l_b.alloc((size_t)ns * 4));
        B200_TRY(c32_b.alloc((size_t)nl * 4));
        B200_TRY(res_b.alloc((size_t)ns * dsub * 4));
        // the first ns rows of a strided view.  Below 2 ns rows the stride is 1, so the codebooks are trained on the first 65536
        // rows as given (tests/test_gpu_index_train.py pins this): one-shot build() already passes an even-strided sample, and
        // a streamed train() of more rows than that should pass them in no particular order (not sorted by cluster)
        const int64_t step = std::max<int64_t>(1, n / ns);
        B200_TRY(samp_b.alloc((size_t)ns * d * 4));
        float *d_samp = samp_b.as<float>(), *d_res = res_b.as<float>();
        uint32_t *d_l = l_b.as<uint32_t>();
        B200_CUDA_OK(cudaMemcpy2DAsync(d_samp, (size_t)d * 4, x, (size_t)step * d * 4, (size_t)d * 4, ns, cudaMemcpyDeviceToDevice, s));
        B200_TRY(b200_corpus_search_device(ix->coarse.get(), d_samp, ns, 1, nullptr, 0, ad_b.as<float>(), a_b.as<int64_t>(), s));
        cudaMemsetAsync(c32_b.p, 0, (size_t)nl * 4, s);
        assign_to_u32_kernel<<<(unsigned)ceil_div(ns, 256), 256, 0, s>>>(a_b.as<int64_t>(), ns, nullptr, 0u, d_l, c32_b.as<uint32_t>());
        g_launches++;
        if (ix->opq) {
            B200_TRY(opq_train_locked(ix, d_samp, ns, d_l));   // R, the rotated centroids and sample, the codebooks
        } else {
            for (int j = 0; j < m; j++) {
                residual_sub_kernel<<<gridsz(ns * dsub), 256, 0, s>>>(d_samp, ns, d, ix->d_centroids.as<float>(), d_l, d, j, dsub, d_res);
                g_launches++;
                B200_TRY(kmeans_device(d_res, ns, dsub, dsub, ncw, 8, ix->d_pq.as<float>() + (size_t)j * ncw * dsub, s));
            }
        }
        if (ix->aq_threshold > 0) {
            // anisotropic iterations on the same sample, from the k-means codebooks (ivf_aq.cu); with opq=1 the sample and the
            // centroids are the rotated ones (the loss does not change under a rotation)
            const AqTrain at{d_samp, ns, d, m, dsub, ncw, d_l, ix->d_centroids.as<float>(), ix->d_pq.as<float>(), ix->aq_eta};
            ix->aq_loss.clear();
            B200_TRY(aq_train_codebooks(at, &ix->aq_loss, s));
        }
        if (ix->d_pq_bf16) B200_CUDA_OK(launch_f32_to_bf16_rows(ix->d_pq.as<float>(), dsub, ix->d_pq_bf16.as<__nv_bfloat16>(), dsub, (int64_t)m * 256, s));
        B200_CUDA_OK(cudaStreamSynchronize(s));
    }
    B200_TRY(alloc_pool(ix, total, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    ix->trained = true;
    return B200_OK;
}

extern "C" int b200_index_train_device(b200_index *ix, const float *d_rows, int64_t n) {
    if (!ix || (!d_rows && n > 0) || n < 0) return fail(B200_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(ix->mu);
    B200_CUDA_OK(cudaSetDevice(ix->device));
    return train_device_locked(ix, d_rows, n);
}

extern "C" int b200_index_train(b200_index *ix, const float *rows, int64_t n) {
    if (!ix || (!rows && n > 0) || n < 0) return fail(B200_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(ix->mu);
    B200_CUDA_OK(cudaSetDevice(ix->device));
    B200_TRY(ix->w_host_q.reserve((size_t)std::max<int64_t>(n, 1) * in_row_bytes(ix)));
    B200_TRY(staged_h2d(ix->w_host_q.p, rows, (size_t)n * in_row_bytes(ix), ix->device, ix->stream));
    B200_CUDA_OK(cudaStreamSynchronize(ix->stream));
    int rc = train_device_locked(ix, ix->w_host_q.as<float>(), n);
    ix->w_host_q.reset();
    return rc;
}

// Search::VectorIndex::add of one chunk already on the device (fp32 [n][d] contiguous, binary bytes [n][d / 8]); row ids
// continue from ix->n
static int add_device_locked(b200_index *ix, const void *d_rows_v, int64_t n) {
    const float *d_rows = reinterpret_cast<const float *>(d_rows_v);
    if (!ix->trained) return fail(B200_ERR_INVALID, "train the index before adding rows");
    if (ix->built) return fail(B200_ERR_INVALID, "index already finalized");
    if (n == 0) return B200_OK;
    cudaStream_t s = ix->stream;
    const int d = ix->d, nl = ix->nlist;
    if (ix->n + n >= (int64_t)0xffffffffll) return fail(B200_ERR_UNSUPPORTED, "an index shard is limited to 2^32 - 1 rows");
    const float *x = d_rows;
    if (ix->binary && !ix->use_ivf) {   // BINARYFLAT / small part: an exact binary corpus
        if (!ix->raw) B200_TRY(corpus_create(ix->metric, B200_DTYPE_BIN, d, std::max<int64_t>(ix->reserved, n), ix->raw));
        B200_TRY(corpus_append_device(ix->raw.get(), d_rows, n, s));
        ix->n += n;
        return B200_OK;
    }
    if (ix->metric == B200_METRIC_COSINE) {
        B200_TRY(ix->w_rows.reserve((size_t)n * d * 4));
        B200_CUDA_OK(cudaMemcpyAsync(ix->w_rows.p, d_rows, (size_t)n * d * 4, cudaMemcpyDeviceToDevice, s));
        B200_CUDA_OK(launch_normalize_rows_f32(ix->w_rows.as<float>(), d, n, s));
        x = ix->w_rows.as<float>();
    }
    if (ix->keep_raw == 1 && !ix->binary) {
        if (!ix->raw) {
            const int raw_metric = ix->metric == B200_METRIC_L2 ? B200_METRIC_L2 : B200_METRIC_IP;
            B200_TRY(corpus_create(raw_metric, B200_DTYPE_F32, d, std::max<int64_t>(ix->reserved, n), ix->raw));
        }
        B200_TRY(corpus_append_device(ix->raw.get(), x, n, s));
    } else if (ix->keep_raw == 2 && !ix->binary) {   // train resolved keep_raw=2 to 1 where the rows are the index
        B200_TRY(host_rows_reserve(ix, std::max(ix->n + n, ix->reserved)));
        B200_CUDA_OK(cudaMemcpy2DAsync(ix->h_rows + ix->n * ix->d_pad, (size_t)ix->d_pad * 4, x, (size_t)d * 4, (size_t)d * 4, n,
                                       cudaMemcpyDeviceToHost, s));
    }
    if (!ix->use_ivf) {
        ix->n += n;
        return B200_OK;
    }
    if (ix->d_opq) {   // opq=1: the assignment, the codes and the norm terms come from x.R; the fp32 rows above stay as given
        B200_TRY(ix->w_qrot.reserve((size_t)n * d * 4));
        B200_CUDA_OK(launch_opq_rotate(x, d, n, d, ix->d_opq.as<float>(), ix->w_qrot.as<float>(), d, s));
        x = ix->w_qrot.as<float>();
    }
    // ---- assign -> (list, row) sorted by list
    B200_TRY(ix->w_assign_i.reserve((size_t)n * 8));
    B200_TRY(ix->w_assign_d.reserve((size_t)n * 4));
    B200_TRY(ix->w_u32a.reserve((size_t)n * 4));
    B200_TRY(ix->w_u32b.reserve((size_t)n * 4));
    B200_TRY(ix->w_u32c.reserve((size_t)n * 4));
    B200_TRY(ix->w_u32d.reserve((size_t)n * 4));
    B200_TRY(ix->w_cnt.reserve((size_t)(nl + 1) * 4));
    B200_TRY(ix->w_plan.reserve((size_t)nl * 4 * 3));
    if (ix->binary) {
        B200_TRY(pad_bin_rows(ix, d_rows, n, ix->w_rows, s));
        x = ix->w_rows.as<float>();
    }
    B200_TRY(b200_corpus_search_device(ix->coarse.get(), x, n, 1, nullptr, 0, ix->w_assign_d.as<float>(), ix->w_assign_i.as<int64_t>(), s));
    // unusable rows (judged as given, before the cosine normalisation) and rows without a nearest centroid get the key nlist:
    // they sort behind every list, are counted in w_cnt[nl] and go to no list
    const uint8_t *usable = nullptr;
    if (!ix->binary) {
        B200_TRY(ix->w_usable.reserve((size_t)n));
        row_usable_kernel<<<gridsz(n * 32), 256, 0, s>>>(d_rows, n, d, ix->w_usable.as<uint8_t>());
        g_launches++;
        usable = ix->w_usable.as<uint8_t>();
    }
    B200_CUDA_OK(cudaMemsetAsync(ix->w_cnt.p, 0, (size_t)(nl + 1) * 4, s));
    assign_to_u32_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, s>>>(ix->w_assign_i.as<int64_t>(), n, usable, (uint32_t)nl, ix->w_u32a.as<uint32_t>(),
                                                                     ix->w_cnt.as<uint32_t>());
    iota_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, s>>>(ix->w_u32b.as<uint32_t>(), n);
    g_launches += 2;
    {
        int bits = 1;
        while ((1 << bits) <= nl) bits++;   // keys 0 .. nlist
        size_t tmp_bytes = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, ix->w_u32a.as<uint32_t>(), ix->w_u32c.as<uint32_t>(), ix->w_u32b.as<uint32_t>(),
                                        ix->w_u32d.as<uint32_t>(), (int)n, 0, bits, s);
        B200_TRY(ix->w_sort.reserve(tmp_bytes + 256));
        cub::DeviceRadixSort::SortPairs(ix->w_sort.p, tmp_bytes, ix->w_u32a.as<uint32_t>(), ix->w_u32c.as<uint32_t>(), ix->w_u32b.as<uint32_t>(),
                                        ix->w_u32d.as<uint32_t>(), (int)n, 0, bits, s);
        g_launches++;
    }
    uint32_t *seg_start = ix->w_plan.as<uint32_t>(), *new_base = seg_start + nl, *first_new = new_base + nl;
    AddPlan ap{};
    ap.cnt = ix->w_cnt.as<uint32_t>();
    ap.seg_start = seg_start;
    ap.new_base = new_base;
    ap.first_new_seq = first_new;
    ap.list_len = ix->d_list_len.as<uint32_t>();
    ap.page_owner = ix->d_page_owner.as<uint32_t>();
    ap.page_seq = ix->d_page_seq.as<uint32_t>();
    ap.pages_used = ix->d_pages_used.as<uint32_t>();
    ap.pool_pages = ix->pool_pages;
    ap.nlist = nl;
    ap.overflow = ix->d_flag.as<int>();
    add_plan_kernel<<<1, 1024, 0, s>>>(ap);
    g_launches++;
    ScatterParams sp{};
    sp.rows = x;
    sp.stride = d;
    sp.sorted_list = ix->w_u32c.as<uint32_t>();
    sp.sorted_row = ix->w_u32d.as<uint32_t>();
    sp.seg_start = seg_start;
    sp.new_base = new_base;
    sp.first_new_seq = first_new;
    sp.list_len = ix->d_list_len.as<uint32_t>();
    sp.tail_page = ix->d_tail_page.as<uint32_t>();
    sp.id_base = (uint32_t)ix->n;
    sp.d = d;
    sp.d_pad64 = ix->d_pad64;
    sp.l2 = ix->metric == B200_METRIC_L2;
    sp.pool = reinterpret_cast<__nv_bfloat16 *>(ix->d_pool.p);
    if (ix->d_sq) {
        sp.sq_lo = ix->d_sq.as<float>();
        sp.sq_step = ix->d_sq.as<float>() + d;
        sp.sq_inv_step = ix->d_sq.as<float>() + 2 * d;
    }
    sp.centroids = ix->d_centroids.as<float>();
    sp.pq = ix->d_pq.as<float>();
    sp.pq_bf16 = ix->d_pq_bf16.as<__nv_bfloat16>();
    sp.m = ix->m;
    sp.dsub = ix->dsub;
    sp.pq_bits = ix->pq_bits;
    sp.codes = reinterpret_cast<uint8_t *>(ix->d_pool.p);
    sp.code_bytes = ix->code_bytes;
    sp.row_bias = ix->d_row_bias.as<float>();
    sp.row_ids = ix->d_row_ids.as<uint32_t>();
    sp.payload = ix->payload;
    if (ix->binary) {
        sp.brows = reinterpret_cast<const uint8_t *>(d_rows);
        sp.stride = ix->row_bytes;
        sp.bpool = reinterpret_cast<uint8_t *>(ix->d_pool.p);
        sp.row_bytes = ix->row_bytes;
        sp.row_pad = ix->row_pad;
        sp.kb_w = ix->kb_w;
    }
    int over = 0;
    uint32_t in_no_list = 0;
    B200_CUDA_OK(cudaMemcpyAsync(&over, ix->d_flag.as<int>(), 4, cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaMemcpyAsync(&in_no_list, ix->w_cnt.as<uint32_t>() + nl, 4, cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    if (over) return fail(B200_ERR_NOMEM, "page pool exhausted: more rows added than b200_index_reserve() announced");
    sp.n = n - in_no_list;   // the list-sorted rows that go to a list; the rest sort behind them
    if (ix->binary) scatter_bin_rows_kernel<<<gridsz(sp.n * 32), 256, 0, s>>>(sp);
    else scatter_rows_kernel<<<gridsz(sp.n * 32), 256, 0, s>>>(sp);
    if (ix->payload == IVF_PRODUCER_PQ && ix->aq_threshold > 0) B200_TRY(aq_encode_chunk(sp, ix->aq_eta, s));   // from the nearest codes
    add_commit_kernel<<<(unsigned)ceil_div(nl, 256), 256, 0, s>>>(ix->w_cnt.as<uint32_t>(), new_base, first_new, ix->d_list_len.as<uint32_t>(), ix->d_tail_page.as<uint32_t>(), nl);
    g_launches += 2;
    B200_CUDA_OK(cudaGetLastError());
    B200_CUDA_OK(cudaStreamSynchronize(s));
    ix->n += n;
    return B200_OK;
}

extern "C" int b200_index_add_device(b200_index *ix, const float *d_rows, int64_t n) {
    if (!ix || (!d_rows && n > 0) || n < 0) return fail(B200_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(ix->mu);
    B200_CUDA_OK(cudaSetDevice(ix->device));
    // bounded scratch: sub-chunks of <= 1 M rows
    for (int64_t off = 0; off < n; off += (1 << 20))
        B200_TRY(add_device_locked(ix, reinterpret_cast<const char *>(d_rows) + off * in_row_bytes(ix), std::min<int64_t>(1 << 20, n - off)));
    return B200_OK;
}

extern "C" int b200_index_add(b200_index *ix, const float *rows, int64_t n) {
    if (!ix || (!rows && n > 0) || n < 0) return fail(B200_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(ix->mu);
    B200_CUDA_OK(cudaSetDevice(ix->device));
    const size_t rb = in_row_bytes(ix);
    const int64_t chunk = std::max<int64_t>(1024, std::min<int64_t>(1 << 20, (int64_t)(1ll << 30) / (int64_t)rb));
    for (int64_t off = 0; off < n; off += chunk) {
        const int64_t mrows = std::min(chunk, n - off);
        B200_TRY(ix->w_host_q.reserve((size_t)mrows * rb));
        B200_TRY(staged_h2d(ix->w_host_q.p, reinterpret_cast<const char *>(rows) + off * rb, (size_t)mrows * rb, ix->device, ix->stream));
        B200_CUDA_OK(cudaStreamSynchronize(ix->stream));
        B200_TRY(add_device_locked(ix, ix->w_host_q.p, mrows));
    }
    return B200_OK;
}

static int search_device_locked(b200_index *ix, const float *d_queries, int64_t nq, int k, const SearchOpts &o, int first_stage_only,
                                const uint8_t *d_alive, const uint8_t *h_alive, int64_t id_offset, float *d_out_dis, int64_t *d_out_ids,
                                int64_t *out_num_candidates, cudaStream_t s);

// scratch of one chunk of the graph build's list searches (their pairs, partial lists and candidates); sizes the chunk
constexpr int64_t kGraphBuildSearchBytes = (int64_t)512 << 20;

// row_slot[n] from the page chains of the finalized (or loaded) lists; 0xFFFFFFFF for a row in no list (an unusable row, or
// an id a loaded file repeats in place of it).  No kernel reads a pool slot through it without that check: the graph build
// gives such rows no edges, and a load refuses an MSTG graph edge to one.
static int fill_row_slot(const b200_index *ix, uint32_t *d_row_slot) {
    B200_CUDA_OK(cudaMemsetAsync(d_row_slot, 0xff, (size_t)ix->n * 4, ix->stream));
    return graph_row_slots(ix->d_list_len.as<uint32_t>(), ix->d_list_page_off.as<uint32_t>(), ix->d_list_pages.as<uint32_t>(), ix->d_row_ids.as<uint32_t>(), ix->nlist, d_row_slot, ix->stream);
}

// MSTG / BINARYMSTG graph: the walk reads its bf16 / binary list rows through d_row_slot
static int build_row_slot(b200_index *ix) {
    if (!ix->d_row_slot) B200_TRY(ix->d_row_slot.alloc(std::max<size_t>((size_t)ix->n * 4, 16)));
    return fill_row_slot(ix, ix->d_row_slot.as<uint32_t>());
}

// graph_degree=D: every row searches the index's own lists (graph=0) with its defaults for k = 2D + 1.  HNSWFLAT: nprobe and the
// exact re-rank with refine_factor, exactly ix.search(rows, 2D + 1) with graph=0.  MSTG: the first stage only, exactly
// ix.search(rows, 2D + 1, first_stage_only=True) with graph=0: the graph is built in the metric its walk scores, the same way for
// either placement of the fp32 rows, and never reads a row over PCIe.  The queries are the fp32 rows (HBM or host memory), or,
// in an index without them (MSTG keep_raw=0), the bf16 list rows.  BINARYMSTG: its lists are exact, so the search is exactly
// ix.search(rows, 2D + 1) with graph=0, its queries the row bytes read back from the binary pages (it keeps no other copy).  Its
// own id dropped, a row's 2D candidates are pruned by rank (CAGRA) and merged with the reverse edges (graph_sm90.cu).  phase_ms
// then holds candidates | prune | merge in milliseconds.
static int build_graph_locked(b200_index *ix) {
    using clk = std::chrono::steady_clock;
    const auto ms_since = [](clk::time_point t) { return std::chrono::duration<double, std::milli>(clk::now() - t).count(); };
    cudaStream_t s = ix->stream;
    const int D = ix->graph_degree, K = 2 * D, d = ix->d;
    const int64_t n = ix->n;
    const bool mstg = ix->type == IDX_MSTG;
    const int np = std::max(1, std::min(ix->default_nprobe, ix->nlist));
    const int k1 = mstg || ix->binary ? K + 1 : std::min(1024, (K + 1) * std::max(1, ix->refine_factor));
    // BINARYMSTG: the chunk's query rows (up to 8 KB each, about a row's list-search scratch) count against the budget too.  The
    // float builds keep their chunk: its size picks the list search's coarse path, so a new one could move their graphs.
    const int64_t q_row_bytes = ix->binary ? ix->row_bytes : (int64_t)d * 4;
    const int64_t chunk = std::max<int64_t>(256, std::min<int64_t>(n, kGraphBuildSearchBytes / ((int64_t)np * k1 * 8 + (ix->binary ? q_row_bytes : 0))));
    DevMem cand, pruned, q, dis, ids, slots;
    // which rows are in a list: the slot map of MSTG / BINARYMSTG, a scratch one for HNSWFLAT
    const uint32_t *row_slot = ix->d_row_slot.as<uint32_t>();
    if (!row_slot) {
        B200_TRY(slots.alloc(std::max<size_t>((size_t)n * 4, 16)));
        B200_TRY(fill_row_slot(ix, static_cast<uint32_t *>(slots.p)));
        row_slot = static_cast<const uint32_t *>(slots.p);
    }
    B200_TRY(cand.alloc(std::max<size_t>((size_t)n * K * 4, 16)));
    B200_TRY(q.alloc(std::max<size_t>((size_t)chunk * q_row_bytes, 16)));   // fp32 rows, or binary rows of d / 8 bytes
    B200_TRY(dis.alloc(std::max<size_t>((size_t)chunk * (K + 1) * 4, 16)));
    B200_TRY(ids.alloc(std::max<size_t>((size_t)chunk * (K + 1) * 8, 16)));
    auto t = clk::now();
    const float *rows = ix->raw ? reinterpret_cast<const float *>(corpus_device_rows(ix->raw.get())) : ix->h_rows;
    for (int64_t off = 0; off < n; off += chunk) {
        const int64_t m = std::min(chunk, n - off);
        if (ix->binary)
            B200_TRY(graph_bin_page_rows(ix->d_pool.p, ix->d_row_slot.as<uint32_t>(), off, m, ix->row_bytes, ix->row_pad, ix->kb_w, static_cast<uint8_t *>(q.p), s));
        else if (rows)
            B200_CUDA_OK(cudaMemcpy2DAsync(q.p, (size_t)d * 4, rows + off * ix->d_pad, (size_t)ix->d_pad * 4, (size_t)d * 4, m,
                                           ix->raw ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, s));
        else
            B200_TRY(graph_page_rows(ix->d_pool.p, ix->d_row_slot.as<uint32_t>(), off, m, d, ix->d_pad64, static_cast<float *>(q.p), s));
        B200_TRY(search_device_locked(ix, static_cast<float *>(q.p), m, K + 1, search_opts(ix, nullptr), mstg ? 1 : 0, nullptr, nullptr, 0, static_cast<float *>(dis.p),
                                      static_cast<int64_t *>(ids.p), nullptr, s));
        B200_TRY(graph_candidates(static_cast<int64_t *>(ids.p), row_slot, m, off, K, static_cast<uint32_t *>(cand.p) + off * K, s));
    }
    B200_CUDA_OK(cudaStreamSynchronize(s));
    for (DevMem *b : {&q, &dis, &ids, &slots}) b->reset();
    const double t_cand = ms_since(t);
    t = clk::now();
    B200_TRY(pruned.alloc(std::max<size_t>((size_t)n * D * 4, 16)));
    B200_TRY(graph_prune(static_cast<uint32_t *>(cand.p), n, D, static_cast<uint32_t *>(pruned.p), s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    cand.reset();
    const double t_prune = ms_since(t);
    t = clk::now();
    DevMem graph;
    B200_TRY(graph.alloc(std::max<size_t>((size_t)n * D * 4, 16)));
    B200_TRY(graph_merge(pruned.as<uint32_t>(), n, D, graph.as<uint32_t>(), s));
    ix->d_graph = std::move(graph);
    const double ph[5] = {t_cand, t_prune, ms_since(t), 0, 0};
    std::copy(ph, ph + 5, ix->phase_ms);
    return B200_OK;
}

static int finalize_locked(b200_index *ix) {
    if (ix->built) return B200_OK;
    if (!ix->trained) return fail(B200_ERR_INVALID, "index not trained");
    cudaStream_t s = ix->stream;
    if (ix->use_ivf) {
        const int nl = ix->nlist;
        B200_CUDA_OK(cudaMemcpy(&ix->pages_used, ix->d_pages_used.as<uint32_t>(), 4, cudaMemcpyDeviceToHost));
        const uint32_t np = ix->pages_used;
        B200_TRY(ix->d_list_page_off.alloc((size_t)(nl + 1) * 4));
        B200_TRY(ix->d_list_pages.alloc((size_t)std::max<uint32_t>(np, 1) * 4));
        B200_TRY(ix->d_list_order.alloc((size_t)nl * 4));
        DevMem keys_b, keys_out_b, vals_b, neg_b, neg_out_b, iota_b;
        B200_TRY(keys_b.alloc((size_t)std::max<uint32_t>(np, 1) * 8));
        B200_TRY(keys_out_b.alloc((size_t)std::max<uint32_t>(np, 1) * 8));
        B200_TRY(vals_b.alloc((size_t)std::max<uint32_t>(np, 1) * 4));
        B200_TRY(neg_b.alloc((size_t)nl * 4));
        B200_TRY(neg_out_b.alloc((size_t)nl * 4));
        B200_TRY(iota_b.alloc((size_t)nl * 4));
        uint64_t *keys = keys_b.as<uint64_t>(), *keys_out = keys_out_b.as<uint64_t>();
        uint32_t *vals = vals_b.as<uint32_t>(), *neg = neg_b.as<uint32_t>(), *neg_out = neg_out_b.as<uint32_t>(), *iota = iota_b.as<uint32_t>();
        if (np) {
            page_keys_kernel<<<(unsigned)ceil_div(np, 256), 256, 0, s>>>(ix->d_page_owner.as<uint32_t>(), ix->d_page_seq.as<uint32_t>(), np, keys, vals);
            size_t tb = 0;
            cub::DeviceRadixSort::SortPairs(nullptr, tb, keys, keys_out, vals, ix->d_list_pages.as<uint32_t>(), (int)np, 0, 64, s);
            B200_TRY(ix->w_sort.reserve(tb + 256));
            cub::DeviceRadixSort::SortPairs(ix->w_sort.p, tb, keys, keys_out, vals, ix->d_list_pages.as<uint32_t>(), (int)np, 0, 64, s);
            g_launches += 2;
        }
        list_pages_scan_kernel<<<1, 1024, 0, s>>>(ix->d_list_len.as<uint32_t>(), nl, ix->d_list_page_off.as<uint32_t>(), neg);
        iota_kernel<<<(unsigned)ceil_div(nl, 256), 256, 0, s>>>(iota, nl);
        {
            size_t tb = 0;
            cub::DeviceRadixSort::SortPairs(nullptr, tb, neg, neg_out, iota, ix->d_list_order.as<uint32_t>(), nl, 0, 32, s);
            B200_TRY(ix->w_sort.reserve(tb + 256));
            cub::DeviceRadixSort::SortPairs(ix->w_sort.p, tb, neg, neg_out, iota, ix->d_list_order.as<uint32_t>(), nl, 0, 32, s);
        }
        g_launches += 3;
        ix->list_len.resize(nl);
        B200_CUDA_OK(cudaMemcpyAsync(ix->list_len.data(), ix->d_list_len.as<uint32_t>(), (size_t)nl * 4, cudaMemcpyDeviceToHost, s));
        B200_CUDA_OK(cudaStreamSynchronize(s));
        ix->max_list_pages = 0;
        for (int l = 0; l < nl; l++) ix->max_list_pages = std::max<uint32_t>(ix->max_list_pages, (ix->list_len[l] + kPageRows - 1) / kPageRows);
    }
    // build scratch is not needed any more
    for (DevMem *a : {&ix->w_rows, &ix->w_assign_i, &ix->w_assign_d, &ix->w_u32a, &ix->w_u32b, &ix->w_u32c, &ix->w_u32d, &ix->w_plan, &ix->w_host_q, &ix->w_usable, &ix->w_qrot})
        a->reset();
    if (!ix->raw) {  // an index without a single row still answers (empty results)
        const int raw_metric = ix->metric == B200_METRIC_L2 ? B200_METRIC_L2 : B200_METRIC_IP;
        if (!ix->use_ivf) B200_TRY(corpus_create(ix->binary ? ix->metric : raw_metric, ix->binary ? B200_DTYPE_BIN : B200_DTYPE_F32, ix->d, 0, ix->raw));
    }
    // a part below the inverted-file threshold is FLAT and gets no graph
    if (ix->graph_degree > 0 && ix->use_ivf && ix->n > 0 && !ix->d_graph) {
        if (ix->type == IDX_MSTG || ix->type == IDX_BINMSTG) B200_TRY(build_row_slot(ix));
        B200_TRY(build_graph_locked(ix));
    }
    ix->built = true;
    return B200_OK;
}

extern "C" int b200_index_finalize(b200_index *ix) {
    if (!ix) return fail(B200_ERR_INVALID, "null index");
    std::lock_guard<std::mutex> lk(ix->mu);
    B200_CUDA_OK(cudaSetDevice(ix->device));
    return finalize_locked(ix);
}

// VIWithColumnInPart::buildIndex -> Search::VectorIndex::build (VIWithDataPart.cpp:131): one-shot build from host rows =
// reserve + train on a strided sample (<= 256 rows per list, the reference's train block) + add in chunks + finalize
extern "C" int b200_index_build(b200_index *ix, const float *rows, int64_t n) {
    if (!ix || (!rows && n > 0) || n < 0) return fail(B200_ERR_INVALID, "bad arguments");
    {
        std::lock_guard<std::mutex> lk(ix->mu);
        if (ix->built || ix->trained) return fail(B200_ERR_INVALID, "index already built");
        ix->reserved = n;
    }
    int nl = ix->nlist;
    const bool flat = is_flat_type(ix->type);
    if (!flat && nl <= 0) nl = (int)std::max<int64_t>(1, std::min<int64_t>(65536, (int64_t)(4.0 * sqrt((double)std::max<int64_t>(n, 1)))));
    const int64_t ns = std::min<int64_t>(n, std::max<int64_t>(256ll * std::max(nl, 1), 65536));
    if (ns == n || flat) {
        B200_TRY(b200_index_train(ix, rows, flat ? 0 : n));
    } else {
        const size_t rb = in_row_bytes(ix);
        std::vector<char> sample((size_t)ns * rb);
        for (int64_t i = 0; i < ns; i++) {
            const int64_t r = (int64_t)((double)i * (double)n / (double)ns);
            memcpy(sample.data() + i * rb, reinterpret_cast<const char *>(rows) + r * rb, rb);
        }
        B200_TRY(b200_index_train(ix, reinterpret_cast<const float *>(sample.data()), ns));
    }
    B200_TRY(b200_index_add(ix, rows, n));
    return b200_index_finalize(ix);
}

extern "C" int b200_index_memory_bytes(const b200_index *ix, uint64_t *out_bytes) {
    if (!ix || !out_bytes) return fail(B200_ERR_INVALID, "bad arguments");
    uint64_t b = 0, t = 0;
    if (ix->raw && b200_corpus_memory_bytes(ix->raw.get(), &t) == B200_OK) b += t;
    if (ix->coarse && b200_corpus_memory_bytes(ix->coarse.get(), &t) == B200_OK) b += t;
    if (ix->use_ivf) {
        const uint64_t rows = (uint64_t)ix->pool_pages * kPageRows;
        b += (uint64_t)ix->nlist * (ix->binary ? (uint64_t)ix->cent_pad : (uint64_t)ix->d * 4) + rows * (payload_row_bytes(ix) + 4 + (ix->d_row_bias ? 4 : 0)) +
             (uint64_t)ix->pool_pages * 12;
        if (ix->d_pq) b += (uint64_t)ix->m * pq_codewords(ix->pq_bits) * ix->dsub * (ix->d_pq_bf16 ? 6 : 4);   // fp32 codebook (+ the decoder's bf16 copy)
    }
    if (ix->d_opq) b += (uint64_t)ix->d * ix->d * 4;
    if (ix->d_graph) b += (uint64_t)ix->n * ix->graph_degree * 4;
    if (ix->d_row_slot) b += (uint64_t)ix->n * 4;
    *out_bytes = b;
    return B200_OK;
}

extern "C" int b200_index_host_memory_bytes(const b200_index *ix, uint64_t *out_bytes) {
    if (!ix || !out_bytes) return fail(B200_ERR_INVALID, "bad arguments");
    *out_bytes = ix->h_rows ? (uint64_t)ix->h_rows_cap * ix->d_pad * 4 : 0;
    return B200_OK;
}

// moves a finalized inverted-file float index's fp32 rows between HBM (1) and pinned host memory (2)
extern "C" int b200_index_set_raw_placement(b200_index *ix, int placement) {
    if (!ix) return fail(B200_ERR_INVALID, "null index");
    if (placement != 1 && placement != 2) return fail(B200_ERR_INVALID, "placement must be 1 (HBM) or 2 (pinned host memory)");
    std::lock_guard<std::mutex> lk(ix->mu);
    if (!ix->built) return fail(B200_ERR_INVALID, "index not finalized");
    if (ix->binary || !ix->use_ivf)
        return fail(B200_ERR_UNSUPPORTED, "the rows are the index here (FLAT, a part below the inverted-file threshold or a binary index): they stay in HBM");
    if (ix->keep_raw != 1 && ix->keep_raw != 2) return fail(B200_ERR_INVALID, "this index keeps no fp32 rows (keep_raw=0)");
    if (placement == 2 && ix->d_graph && ix->type == IDX_HNSWFLAT)
        return fail(B200_ERR_UNSUPPORTED, "graph_degree: the HNSWFLAT graph search reads the fp32 rows in HBM");
    if (placement == ix->keep_raw) return B200_OK;
    B200_CUDA_OK(cudaSetDevice(ix->device));
    // searches enqueued on the callers' streams may still read the rows that are about to be freed
    B200_CUDA_OK(cudaDeviceSynchronize());
    const size_t row_b = (size_t)ix->d_pad * 4;
    if (placement == 2 && ix->raw) {
        B200_TRY(host_rows_reserve(ix, ix->n));
        B200_CUDA_OK(cudaMemcpy(ix->h_rows, corpus_device_rows(ix->raw.get()), (size_t)ix->n * row_b, cudaMemcpyDeviceToHost));
        ix->raw.reset();
    } else if (placement == 1 && ix->h_rows) {
        const int raw_metric = ix->metric == B200_METRIC_L2 ? B200_METRIC_L2 : B200_METRIC_IP;
        CorpusPtr c;
        B200_TRY(corpus_create(raw_metric, B200_DTYPE_F32, ix->d, ix->n, c));
        const int64_t chunk = std::max<int64_t>(1, kHostStageBytes / ((int64_t)ix->d * 4));
        int rc = ix->w_rows.reserve((size_t)std::min(chunk, std::max<int64_t>(ix->n, 1)) * ix->d * 4);
        for (int64_t off = 0; rc == B200_OK && off < ix->n; off += chunk) {   // unpadded [m][d] for the corpus append
            const int64_t m = std::min(chunk, ix->n - off);
            if (cudaMemcpy2DAsync(ix->w_rows.p, (size_t)ix->d * 4, ix->h_rows + off * ix->d_pad, row_b, (size_t)ix->d * 4, m, cudaMemcpyHostToDevice,
                                  ix->stream) != cudaSuccess)
                rc = fail(B200_ERR_CUDA, "host rows -> HBM copy failed");
            else
                rc = corpus_append_device(c.get(), ix->w_rows.as<float>(), m, ix->stream);
        }
        ix->w_rows.reset();
        B200_TRY(rc);
        ix->raw = std::move(c);
        cudaFreeHost(ix->h_rows);
        ix->h_rows = nullptr;
        ix->h_rows_dev = nullptr;
        ix->h_rows_cap = 0;
        ix->w_stage.reset();
    }
    ix->keep_raw = placement;
    return B200_OK;
}

extern "C" int b200_index_info(const b200_index *ix, int64_t *n, int *nlist, int *m, int *uses_ivf) {
    if (!ix) return fail(B200_ERR_INVALID, "null index");
    if (n) *n = ix->n;
    if (nlist) *nlist = ix->nlist;
    if (m) *m = ix->m;
    if (uses_ivf) *uses_ivf = ix->use_ivf ? 1 : 0;
    return B200_OK;
}

extern "C" int b200_index_last_scan(b200_index *ix, int64_t *rows_streamed, int64_t *payload_row_bytes_out, int64_t *work_items,
                                    double *kernel_ms_total, int64_t *kernel_launches, int reset) {
    if (!ix) return fail(B200_ERR_INVALID, "null index");
    std::lock_guard<std::mutex> lk(ix->mu);
    cudaSetDevice(ix->device);
    timing_collect(ix);
    if (ix->d_flag && ix->use_ivf) {
        unsigned long long r = 0;
        if (cudaMemcpy(&r, ix->d_flag.as<int>() + 4, 8, cudaMemcpyDeviceToHost) == cudaSuccess) ix->last_scan_rows = (int64_t)r;
    }
    if (rows_streamed) *rows_streamed = ix->last_scan_rows;
    // the graph walk reads fp32 rows (HNSWFLAT), the bf16 list rows (MSTG) or the binary list rows (BINARYMSTG)
    if (payload_row_bytes_out) *payload_row_bytes_out = ix->last_graph && !ix->d_row_slot ? (int64_t)ix->d_pad * 4 : (int64_t)payload_row_bytes(ix);
    if (work_items) *work_items = ix->last_items;
    if (kernel_ms_total) *kernel_ms_total = ix->timed_ms;
    if (kernel_launches) *kernel_launches = ix->timed_launches;
    if (reset) {
        ix->timed_ms = 0;
        ix->timed_launches = 0;
    }
    return B200_OK;
}

// milliseconds of the phases of the LAST list search (timing enabled): coarse probe | pair sort + plan + query gather |
// grouped scan | per-query merge | exact second stage
extern "C" int b200_index_phase_ms(b200_index *ix, double out_ms[5]) {
    if (!ix || !out_ms) return fail(B200_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(ix->mu);
    cudaSetDevice(ix->device);
    timing_collect(ix);
    for (int i = 0; i < 5; i++) out_ms[i] = ix->phase_ms[i];
    return B200_OK;
}

// rows per inverted list (diagnostics: balance of the coarse quantiser); out_sizes[nlist]
extern "C" int b200_index_list_sizes(const b200_index *ix, uint32_t *out_sizes, int capacity) {
    if (!ix || !out_sizes) return fail(B200_ERR_INVALID, "bad arguments");
    if (!ix->built || !ix->use_ivf) return fail(B200_ERR_INVALID, "no inverted lists (FLAT index or not finalized)");
    if (capacity < ix->nlist) return fail(B200_ERR_INVALID, "buffer too small");
    memcpy(out_sizes, ix->list_len.data(), (size_t)ix->nlist * 4);
    return B200_OK;
}

extern "C" int b200_index_enable_timing(b200_index *ix, int on) {
    if (!ix) return fail(B200_ERR_INVALID, "null index");
    std::lock_guard<std::mutex> lk(ix->mu);
    ix->timing = on != 0;
    if (on && !ix->ev0) {
        cudaEventCreate(&ix->ev0);
        cudaEventCreate(&ix->ev1);
        for (auto &e : ix->ev_ph) cudaEventCreate(&e);
    }
    return B200_OK;
}

// computeTopDistanceSubset (VIWithDataPart.cpp:838-856): exact distances of a candidate id set -> top-k
static int refine_device(b200_index *ix, const float *d_q /*[nq][d_pad] prepared*/, int64_t nq, const int64_t *d_cand, int ncand,
                         int k, int64_t id_offset, float *d_out_dis, int64_t *d_out_ids, cudaStream_t s) {
    RefineParams rp{};
    rp.queries = d_q;
    rp.cand = d_cand;
    rp.out_dis = d_out_dis;
    rp.out_ids = d_out_ids;
    rp.n = ix->n;
    rp.d_pad = ix->d_pad;
    rp.ncand = ncand;
    rp.k = k;
    rp.l2 = ix->metric == B200_METRIC_L2;
    rp.cosine = ix->metric == B200_METRIC_COSINE;
    rp.id_offset = id_offset;
    const size_t smem = (size_t)ix->d_pad * 4 + (size_t)9 * k * 8;
    if (smem > (size_t)kSmemOptinBytes)   // d <= B200_MAX_FLOAT_DIM keeps this far below the limit at k = 1024
        return fail(B200_ERR_UNSUPPORTED, "exact second stage: d_pad " + std::to_string(ix->d_pad) + " at k " + std::to_string(k) + " needs " +
                                              std::to_string(smem) + " bytes of shared memory, more than " + std::to_string(kSmemOptinBytes));
    if (!ix->h_rows) {
        rp.rows = reinterpret_cast<const float *>(corpus_device_rows(ix->raw.get()));
        B200_CUDA_OK(cudaFuncSetAttribute(refine_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        refine_kernel<false><<<(unsigned)nq, 256, smem, s>>>(rp);
        g_launches++;
        B200_CUDA_OK(cudaGetLastError());
        return B200_OK;
    }
    // rows in host memory: per chunk of queries, gather the candidates' rows over PCIe into the staging buffer (the grid is
    // sized by candidate slots, so even one query's candidates spread over every SM), then re-rank from there
    const int64_t per_q = (int64_t)ncand * ix->d_pad * 4;
    const int64_t qchunk = std::max<int64_t>(1, std::min<int64_t>(nq, kHostStageBytes / per_q));
    B200_TRY(ix->w_stage.reserve((size_t)qchunk * per_q));
    B200_CUDA_OK(cudaFuncSetAttribute(refine_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    for (int64_t q0 = 0; q0 < nq; q0 += qchunk) {
        const int64_t nqc = std::min(qchunk, nq - q0), slots = nqc * ncand;
        const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(slots, 8 * kGatherRows), (int64_t)ix->sms * 8));
        gather_host_rows_kernel<<<grid, 256, 0, s>>>(ix->h_rows_dev, ix->n, ix->d_pad, d_cand + q0 * ncand, slots, ix->w_stage.as<float>());
        RefineParams cp = rp;
        cp.queries = d_q + q0 * ix->d_pad;
        cp.rows = ix->w_stage.as<float>();
        cp.cand = d_cand + q0 * ncand;
        cp.out_dis = d_out_dis + q0 * k;
        cp.out_ids = d_out_ids + q0 * k;
        refine_kernel<true><<<(unsigned)nqc, 256, smem, s>>>(cp);
        g_launches += 2;
    }
    B200_CUDA_OK(cudaGetLastError());
    return B200_OK;
}

// d_queries_raw: device fp32 [nq][d] -> ix->w_q [nq][d_pad] (cosine: unit length)
// an unusable query (warp_row_usable) becomes all NaN: a distance to it is never finite, on any path; one warp per query
__global__ void __launch_bounds__(256) nan_unusable_queries_kernel(float *q, int64_t nq, int d_pad) {
    const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp_global; r < nq; r += nwarps)
        if (!warp_row_usable(q + r * d_pad, d_pad))
            for (int j = lane_id(); j < d_pad; j += 32) q[r * d_pad + j] = __int_as_float(0x7fffffff);
}

static int prepare_queries_device(b200_index *ix, const float *d_queries_raw, int64_t nq, cudaStream_t s) {
    B200_TRY(ix->w_q.reserve((size_t)nq * ix->d_pad * 4));
    B200_CUDA_OK(launch_pad_rows_f32(d_queries_raw, ix->d, ix->w_q.as<float>(), ix->d_pad, nq, s));
    // L2 and cosine: a query with an infinite coordinate (or one whose square overflows) returns no rows, as a NaN one does.
    // Under IP such a query is outside the contract (include/b200_search.h) and is scored as given.
    if (ix->metric != B200_METRIC_IP && nq) {
        nan_unusable_queries_kernel<<<gridsz(nq * 32), 256, 0, s>>>(ix->w_q.as<float>(), nq, ix->d_pad);
        g_launches++;
    }
    if (ix->metric == B200_METRIC_COSINE) B200_CUDA_OK(launch_normalize_rows_f32(ix->w_q.as<float>(), ix->d_pad, nq, s));
    return B200_OK;
}

__global__ void cosine_finish_kernel(const float *q, int64_t nq, int d, int d_pad, int k, float *dis, const int64_t *ids) {
    // raw rows are unit vectors searched under IP with the prepared (unit) queries: distance = 1 - ip
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq * k) return;
    dis[i] = ids[i] >= 0 ? 1.f - dis[i] : FLT_MAX;
}

// cosine: the IP keys of a search over the raw (unit) rows become distances; the other metrics' keys are already
static void cosine_finish(const b200_index *ix, const float *d_q, int64_t nq, int k, float *d_out_dis, const int64_t *d_out_ids, cudaStream_t s) {
    if (ix->metric != B200_METRIC_COSINE) return;
    cosine_finish_kernel<<<(unsigned)ceil_div(nq * k, 256), 256, 0, s>>>(d_q, nq, ix->d, ix->d_pad, k, d_out_dis, d_out_ids);
    g_launches++;
}

// the prepared queries [nq][d_pad] back to [nq][d] rows in ix->w_qraw, the row form of a corpus search
static int unpad_queries(b200_index *ix, const float *d_q, int64_t nq, cudaStream_t s) {
    B200_TRY(ix->w_qraw.reserve((size_t)nq * ix->d * 4));
    if (ix->d == ix->d_pad) B200_CUDA_OK(cudaMemcpyAsync(ix->w_qraw.p, d_q, (size_t)nq * ix->d * 4, cudaMemcpyDeviceToDevice, s));
    else B200_CUDA_OK(cudaMemcpy2DAsync(ix->w_qraw.p, (size_t)ix->d * 4, d_q, (size_t)ix->d_pad * 4, (size_t)ix->d * 4, nq, cudaMemcpyDeviceToDevice, s));
    return B200_OK;
}

// Pages of a list one work item streams for a scan of n_valid (query, list) pairs (see scan_probes); forced: the
// "pages_per_chunk" A/B key, 0 = none.
static uint32_t pages_per_chunk(const b200_index *ix, int64_t n_valid, int forced) {
    const double avg_pages = std::max(1.0, (double)ix->pages_used / std::max(1, ix->nlist));
    const double est_lists = std::min<double>((double)n_valid, (double)ix->nlist);
    const double est_pages = est_lists * std::min<double>(ix->max_list_pages ? ix->max_list_pages : 1, 1.5 * avg_pages);
    const double want_items = 4.0 * ix->sms;
    // Lists probed by more than 16 queries run on per-lane top-k lists, whose cold start is paid per item: longer items pay;
    // cooperative items (<= 16 queries) keep the 16-page cap.
    const double q_per_list = (double)n_valid / std::max(1.0, est_lists);
    const double cap = q_per_list > 16.0 ? 48.0 : 16.0;
    uint32_t ppc = (uint32_t)std::min(cap, std::max(8.0, std::ceil(est_pages / want_items)));
    if (est_lists * 2 < want_items) ppc = (uint32_t)std::max(2.0, std::min<double>(ppc, std::ceil(1.5 * avg_pages * est_lists / want_items)));   // a handful of queries
    ppc = std::max<uint32_t>(ppc, (ix->max_list_pages + 63) / 64);   // at most 64 chunks per list
    ppc = std::max<uint32_t>(ppc, 1);
    if (forced) ppc = (uint32_t)forced;
    return ppc;
}

// The steps of a list search after the coarse probe, asynchronous on s: pairs sorted by list, plan, query gather, grouped
// scan, per-query merge, exact second stage.  d_q: the first stage's queries [nq][d_pad] (opq=1: rotated), d_qx: the
// prepared queries of the exact second stage.  probe: [nq][nprobe] list ids (negative = an invalid slot, skipped by every
// step).  n_valid: the count of valid slots, sizing the gathered query rows, the work items and the partial lists.  list_len / list_pages: the index's own, or the filtered ones of filter_probe=1.
static int scan_probes(b200_index *ix, const float *d_q, const float *d_qx, const float *d_queries, int64_t nq, int k, int k1, bool two_stage, const SearchOpts &o,
                       const int64_t *probe, int nprobe, int64_t n_valid, const uint32_t *list_len, const uint32_t *list_pages,
                       const uint8_t *d_alive, int64_t id_offset, float *d_out_dis, int64_t *d_out_ids, cudaStream_t s) {
    const int nl = ix->nlist;
    const int64_t n_pairs = nq * nprobe;
    if (n_pairs >= (int64_t)1 << 31) return fail(B200_ERR_UNSUPPORTED, "nq * nprobe must stay below 2^31");
    // ---- pairs sorted by list
    B200_TRY(ix->w_u32a.reserve((size_t)n_pairs * 4));
    B200_TRY(ix->w_u32b.reserve((size_t)n_pairs * 4));
    B200_TRY(ix->w_u32c.reserve((size_t)n_pairs * 4));
    B200_TRY(ix->w_u32d.reserve((size_t)n_pairs * 4));
    B200_TRY(ix->w_cnt.reserve((size_t)nl * 4));
    B200_CUDA_OK(cudaMemsetAsync(ix->w_cnt.p, 0, (size_t)nl * 4, s));
    pairs_make_kernel<<<(unsigned)ceil_div(n_pairs, 256), 256, 0, s>>>(probe, n_pairs, nl, ix->w_u32a.as<uint32_t>(),
                                                                       ix->w_u32b.as<uint32_t>(), ix->w_cnt.as<uint32_t>());
    g_launches++;
    {
        int bits = 1;
        while ((1 << bits) < nl + 1) bits++;
        size_t tb = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, tb, ix->w_u32a.as<uint32_t>(), ix->w_u32c.as<uint32_t>(), ix->w_u32b.as<uint32_t>(),
                                        ix->w_u32d.as<uint32_t>(), (int)n_pairs, 0, bits, s);
        B200_TRY(ix->w_sort.reserve(tb + 256));
        cub::DeviceRadixSort::SortPairs(ix->w_sort.p, tb, ix->w_u32a.as<uint32_t>(), ix->w_u32c.as<uint32_t>(), ix->w_u32b.as<uint32_t>(),
                                        ix->w_u32d.as<uint32_t>(), (int)n_pairs, 0, bits, s);
        g_launches++;
    }
    // ---- work items.  Long lists are cut into chunks of pages so that even a single query fills the SMs; the cut is
    //      chosen from host-side knowledge only (no device -> host round trip on the query path).
    // Lists are cut into chunks of `ppc` pages: an item never streams more than 16 pages (bounds the tail of the static
    // round-robin schedule), and small batches are split further so that every SM gets ~4 items.  Finer is NOT better: every item
    // pays one cold start of its top-k lists.  The page counts (8 to 16, 48 below) were chosen on an earlier GPU and are
    // not re-measured on the H100.  The estimate uses host-side knowledge only (no device -> host round trip on the query path): probed
    // lists <= min(pairs, nlist), their length size-biased.
    const uint32_t ppc = pages_per_chunk(ix, n_valid, o.pages_per_chunk);
    const uint32_t max_chunks = (ix->max_list_pages + ppc - 1) / ppc;
    const int64_t max_items = std::min<int64_t>(n_valid * max_chunks, (int64_t)(ceil_div(n_valid, 128) + nl) * max_chunks);
    const int64_t max_parts = n_valid * max_chunks;
    if (max_parts * k1 >= (int64_t)1 << 32) return fail(B200_ERR_UNSUPPORTED, "nq * nprobe * chunks * k too large for one batch; split the batch");
    B200_TRY(ix->w_items.reserve((size_t)max_items * sizeof(IvfGemmItem) + 64));
    B200_TRY(ix->w_plan.reserve((size_t)nl * 4 * 3));
    uint32_t *pair_start = ix->w_plan.as<uint32_t>(), *part_off = pair_start + nl, *n_chunks = part_off + nl;
    int *d_counts = ix->d_flag.as<int>() + 1;   // n_items, n_parts
    SearchPlan pl{};
    pl.cnt = ix->w_cnt.as<uint32_t>();
    pl.list_len = list_len;
    pl.list_page_off = ix->d_list_page_off.as<uint32_t>();
    pl.list_order = ix->d_list_order.as<uint32_t>();
    pl.pair_start = pair_start;
    pl.part_off = part_off;
    pl.n_chunks = n_chunks;
    pl.items = ix->w_items.as<IvfGemmItem>();
    pl.n_items = d_counts;
    pl.n_parts = d_counts + 1;
    pl.scan_rows = reinterpret_cast<unsigned long long *>(ix->d_flag.as<int>() + 4);
    pl.nlist = nl;
    pl.max_items = (int)std::min<int64_t>(max_items, INT32_MAX);
    pl.pages_per_chunk = ppc;
    search_plan_kernel<<<1, 1024, 0, s>>>(pl);
    g_launches++;
    // ---- gather queries, per-pair bookkeeping
    const bool lut = pq_uses_lut(ix), pq4 = lut && ix->pq_bits == 4;
    const size_t qrow_bytes = ix->binary ? (size_t)ix->row_pad : (size_t)ix->d_pad64 * 2;
    if (!lut) {   // the table look-up scan reads no gathered query rows
        B200_TRY(ix->w_qbuf.reserve(((size_t)n_valid + 128) * qrow_bytes));
        // the 128 rows behind the last pair are read by the last items' A tiles (query slots without a query): keep them finite
        B200_CUDA_OK(cudaMemsetAsync(ix->w_qbuf.as<char>() + (size_t)n_valid * qrow_bytes, 0, (size_t)128 * qrow_bytes, s));
    }
    B200_TRY(ix->w_inv.reserve((size_t)n_pairs * 4));
    B200_TRY(ix->w_ppb.reserve((size_t)n_pairs * 4));
    B200_TRY(ix->w_pconst.reserve((size_t)n_pairs * 4));
    B200_TRY(ix->w_qconst.reserve((size_t)nq * 4));
    PairFill pf{};
    pf.sorted_list = ix->w_u32c.as<uint32_t>();
    pf.sorted_pair = ix->w_u32d.as<uint32_t>();
    pf.pair_start = pair_start;
    pf.part_off = part_off;
    pf.n_chunks = n_chunks;
    pf.queries = d_q;
    pf.sq_step = ix->payload == IVF_PRODUCER_SQ8 ? ix->d_sq.as<float>() + ix->d : nullptr;
    pf.centroids = ix->payload == IVF_PRODUCER_PQ ? ix->d_centroids.as<float>() : nullptr;
    pf.qbuf = lut ? nullptr : ix->w_qbuf.as<__nv_bfloat16>();
    pf.inv = ix->w_inv.as<uint32_t>();
    pf.pair_part_base = ix->w_ppb.as<uint32_t>();
    pf.pair_const = ix->w_pconst.as<float>();
    pf.n_pairs = n_pairs;
    pf.nprobe = nprobe;
    pf.nlist = nl;
    pf.d = ix->d;
    pf.d_pad = ix->d_pad;
    pf.d_pad64 = ix->d_pad64;
    pf.l2 = ix->metric == B200_METRIC_L2;
    if (ix->binary) {
        B200_TRY(ix->w_ppopc.reserve((size_t)n_pairs * 4));
        pf.bqueries = reinterpret_cast<const uint8_t *>(d_queries);
        pf.bqbuf = ix->w_qbuf.as<uint8_t>();
        pf.pair_popc = ix->w_ppopc.as<float>();
        pf.row_bytes = ix->row_bytes;
        pf.row_pad = ix->row_pad;
        pf.jaccard = ix->metric == B200_METRIC_JACCARD;
        pair_fill_bin_kernel<<<(unsigned)ceil_div(n_pairs * 32, 256), 256, 0, s>>>(pf);
        g_launches++;
    } else {
        pair_fill_kernel<<<(unsigned)ceil_div(n_pairs * 32, 256), 256, 0, s>>>(pf);
        g_launches++;
        if (lut) {   // the per-query tables T[q][j][e] = <q_j, codebook_j[e]> (fp32)
            B200_TRY(ix->w_lut.reserve((size_t)nq * ix->m * pq_codewords(ix->pq_bits) * 4));
            B200_CUDA_OK(pq4 ? launch_pq4_lut(d_q, nq, ix->d_pad, ix->d_pq.as<float>(), ix->m, ix->dsub, ix->w_lut.as<float>(), s)
                             : launch_pq_lut(d_q, nq, ix->d_pad, ix->d_pq.as<float>(), ix->m, ix->dsub, ix->w_lut.as<float>(), s));
        }
        if (ix->payload != IVF_PRODUCER_PQ) {   // PQ: the pair constant (||q - c||^2 or -<q, c>) is the whole query term
            query_const_kernel<<<(unsigned)ceil_div(nq * 32, 256), 256, 0, s>>>(d_q, nq, ix->d, ix->d_pad, ix->payload == IVF_PRODUCER_SQ8 ? ix->d_sq.as<float>() + 3 * ix->d : nullptr,
                                                                                ix->metric == B200_METRIC_L2, ix->payload == IVF_PRODUCER_TMA, ix->w_qconst.as<float>());
            g_launches++;
        }
    }
    // ---- the grouped tensor-core scan
    B200_TRY(ix->w_pk.reserve((size_t)max_parts * k1 * 4));
    B200_TRY(ix->w_pi.reserve((size_t)max_parts * k1 * 4));
    B200_TRY(ix->w_pw.reserve((size_t)max_parts * 4));
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(ix->sms, max_items));
    IvfGemmParams gp{};
    gp.items = ix->w_items.as<IvfGemmItem>();
    gp.n_items_ptr = d_counts;
    gp.list_pages = list_pages;
    gp.row_bias = ix->d_row_bias.as<float>();
    gp.row_ids = ix->d_row_ids.as<uint32_t>();
    gp.alive = d_alive;
    gp.pair_part_base = ix->w_ppb.as<uint32_t>();
    gp.part_keys = ix->w_pk.as<float>();
    gp.part_ids = ix->w_pi.as<uint32_t>();
    gp.part_worst = ix->w_pw.as<float>();
    {   // shared per-query bound across the items of this launch (ivf_gemm.h); nothing to share with one list per query
        if (nprobe > 1 && o.shared_bound != 0) {
            B200_TRY(ix->w_qb.reserve((size_t)nq * 4));
            B200_CUDA_OK(cudaMemsetAsync(ix->w_qb.p, 0xff, (size_t)nq * 4, s));
            gp.query_bound = ix->w_qb.as<uint32_t>();
            gp.sorted_pair = ix->w_u32d.as<uint32_t>();
            gp.pair_const = ix->w_pconst.as<float>();
            gp.nprobe = nprobe;
        }
    }
    gp.scale_const = ix->metric == B200_METRIC_L2 ? -2.f : -1.f;
    gp.d_pad = ix->d_pad64;
    if (ix->binary) {   // Hamming ranks popc(y) - 2 and (+ popc(q) as the pair constant); Jaccard: scale 1 only marks live rows
        gp.jaccard = ix->metric == B200_METRIC_JACCARD;
        gp.scale_const = gp.jaccard ? 1.f : -2.f;
        gp.d_pad = ix->row_pad;
        gp.kb_w = ix->kb_w;
        gp.pair_popc = ix->w_ppopc.as<float>();
    }
    gp.k = k1;
    gp.producer = ix->payload;
    gp.codes = reinterpret_cast<const uint8_t *>(ix->d_pool.p);
    gp.codebook_bf16 = ix->d_pq_bf16.as<__nv_bfloat16>();
    gp.code_bytes = ix->code_bytes;
    gp.m = ix->m;
    gp.dsub = ix->dsub;
    gp.codebook_bytes = ix->payload == IVF_PRODUCER_PQ ? ix->m * 256 * ix->dsub * 2 : 0;
    if (lut) {   // the look-up scan finds its table through the pair's query
        gp.lut = ix->w_lut.as<float>();
        gp.sorted_pair = ix->w_u32d.as<uint32_t>();
        gp.nprobe = nprobe;
    } else {  // global scratch for lists that do not fit in shared memory (the launcher decides)
        B200_TRY(ix->w_lk.reserve((size_t)grid * 128 * list_cap_for(k1) * 4));
        B200_TRY(ix->w_li.reserve((size_t)grid * 128 * list_cap_for(k1) * 4));
        gp.list_keys_gmem = ix->w_lk.as<float>();
        gp.list_ids_gmem = ix->w_li.as<uint32_t>();
    }
    const char *detail = nullptr;
    if (ix->timing) {
        cudaEventRecord(ix->ev_ph[2], s);
        cudaEventRecord(ix->ev0, s);
    }
    cudaError_t e = pq4   ? launch_ivf_pq4_topk(gp, grid, s, &detail)
                    : lut ? launch_ivf_pq_lut_topk(gp, grid, s, &detail)
                          : launch_ivf_gemm_topk(gp, ix->w_qbuf.p, n_valid + 128, ix->d_pool.p, (int64_t)ix->pool_pages * kPageRows, grid, s, &detail);
    if (ix->timing) {
        cudaEventRecord(ix->ev1, s);
        cudaEventRecord(ix->ev_ph[3], s);
        ix->timed_pending = true;
    }
    if (e != cudaSuccess)
        return fail(B200_ERR_CUDA, std::string(pq4 ? "ivf_pq4_topk launch: " : lut ? "ivf_pq_lut_topk launch: " : "ivf_gemm_topk launch: ") +
                                       (detail ? detail : cudaGetErrorString(e)));
    ix->last_items = max_items;
    // ---- per-query merge of the partial lists
    float *m_dis = d_out_dis;
    int64_t *m_ids = d_out_ids;
    if (two_stage) {
        B200_TRY(ix->w_od.reserve((size_t)nq * k1 * 4));
        B200_TRY(ix->w_oi.reserve((size_t)nq * k1 * 8));
        m_dis = ix->w_od.as<float>();
        m_ids = ix->w_oi.as<int64_t>();
    }
    IvfMerge mg{};
    mg.inv = ix->w_inv.as<uint32_t>();
    mg.pair_part_base = ix->w_ppb.as<uint32_t>();
    mg.sorted_list = ix->w_u32c.as<uint32_t>();
    mg.n_chunks = n_chunks;
    mg.pair_const = ix->w_pconst.as<float>();
    mg.query_const = ix->binary || ix->payload == IVF_PRODUCER_PQ ? nullptr : ix->w_qconst.as<float>();
    mg.part_keys = gp.part_keys;
    mg.part_worst = gp.part_worst;
    mg.part_ids = gp.part_ids;
    mg.out_dis = m_dis;
    mg.out_ids = m_ids;
    mg.id_offset = two_stage ? 0 : id_offset;
    mg.nprobe = nprobe;
    mg.nlist = nl;
    mg.k_part = k1;
    mg.k = k1;
    mg.metric = ix->metric;
    {
        const size_t smem = (size_t)9 * k1 * 8;
        B200_CUDA_OK(cudaFuncSetAttribute(ivf_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ivf_merge_kernel<<<(unsigned)nq, 256, smem, s>>>(mg);
        g_launches++;
        B200_CUDA_OK(cudaGetLastError());
    }
    if (ix->timing) cudaEventRecord(ix->ev_ph[4], s);
    if (two_stage) B200_TRY(refine_device(ix, d_qx, nq, m_ids, k1, k, id_offset, d_out_dis, d_out_ids, s));
    if (ix->timing) cudaEventRecord(ix->ev_ph[5], s);
    return B200_OK;
}

// Scratch budget of a filter_probe=1 batch after its selection: about kFilterProbeSlotBytes per probe slot [query][P] (the
// probe row, the pair keys and their sort, the per-pair bookkeeping) plus, per valid slot, a gathered query row, work items
// and partial lists.  A batch above it runs those steps on query sub-ranges: every query's answer depends on that query alone.
constexpr int64_t kFilterProbeScratchBytes = 1ll << 30;
constexpr int64_t kFilterProbeSlotBytes = 40;
// The exact rule's limit in units of nprobe x n / nlist kept rows.  On 2 M x 768 rows (nprobe 16, nlist 4096, k 10, nq 1 -
// 1024; H100 SXM at 700 W, DESIGN §7) the exact pass was faster than the lists at 1 % and 3 % of the rows (2.6 x and 7.7 x
// nprobe x n / nlist) and slower at 10 % (25.6 x) for 3 of 4 batch sizes, so 1 (and 4) missed the faster path and 16 picks it.
constexpr double kFilterProbeExactFactor = 16.0;

// filter_probe=1 below nlist, after list_alive_kernel filtered the page table: the coarse keys of the batch (chunks of at most
// 256 MB), one probe depth p_q per query and the number of its first p_q lists that hold a kept row, its live lists
// (probe_select_kernel); ONE device -> host read-back (the 16-byte Σ / max of the live lists, with the nq values of p_q and of
// the live lists) and a stream synchronise; then the probe rows [nq][P] of the live lists, P = max live lists, and the rest of
// the search with nprobe := P, its buffers sized by the live lists.  Leaving out a list without a kept row changes no answer:
// it holds no candidate and the merge does not depend on the order of its inputs.
static int filter_probe_search(b200_index *ix, const float *d_q, const float *d_qx, int64_t nq, int k, int k1, bool two_stage, const SearchOpts &o,
                               const uint32_t *list_len, const uint32_t *list_pages, const uint8_t *d_alive, int64_t id_offset, float *d_out_dis,
                               int64_t *d_out_ids, cudaStream_t s) {
    const int nl = ix->nlist;
    const int64_t chunk = coarse_chunk(nq, nl);
    const bool one_chunk = nq <= chunk;
    B200_TRY(ix->w_cs.reserve((size_t)chunk * nl * 4));
    const size_t tot_off = round_up((size_t)nq * 16, 16);
    B200_TRY(ix->w_fsel.reserve(tot_off + 24));
    int *d_p = ix->w_fsel.as<int>(), *d_live = d_p + nq;
    uint32_t *d_key = reinterpret_cast<uint32_t *>(d_live + nq), *d_ties = d_key + nq;
    unsigned long long *d_tot = reinterpret_cast<unsigned long long *>(ix->w_fsel.as<char>() + tot_off);   // Σ live, max live, scan rows
    B200_CUDA_OK(cudaMemsetAsync(d_tot, 0, 24, s));
    auto coarse_keys = [&](int64_t q0, int64_t nqc) {
        coarse_scores_kernel<<<dim3((unsigned)ceil_div(nl, kCoarseTile), (unsigned)ceil_div(nqc, kCoarseTile)), 256, 0, s>>>(
            d_q + q0 * ix->d_pad, ix->d_pad, ix->d_centroids.as<float>(), ix->d_cnorm.as<float>(), nqc, nl, ix->d, ix->w_cs.as<float>());
        g_launches++;
    };
    for (int64_t q0 = 0; q0 < nq; q0 += chunk) {
        const int64_t nqc = std::min(chunk, nq - q0);
        coarse_keys(q0, nqc);
        probe_select_kernel<<<(unsigned)nqc, kProbeThreads, 0, s>>>(ix->w_cs.as<float>(), nl, ix->w_flist.as<uint32_t>(), (uint32_t)k1, o.nprobe,
                                                                   o.max_nprobe, d_p + q0, d_live + q0, d_key + q0, d_ties + q0, d_tot);
        g_launches++;
    }
    B200_CUDA_OK(cudaGetLastError());
    const size_t hb = 16 + (size_t)nq * 8;
    if (ix->h_fsel_cap < hb) {
        if (ix->h_fsel) cudaFreeHost(ix->h_fsel);
        ix->h_fsel = nullptr;
        ix->h_fsel_cap = 0;
        B200_CUDA_OK(cudaMallocHost(&ix->h_fsel, hb + hb / 4));
        ix->h_fsel_cap = hb + hb / 4;
    }
    unsigned long long *h_tot = static_cast<unsigned long long *>(ix->h_fsel);
    int32_t *h_p = reinterpret_cast<int32_t *>(h_tot + 2), *h_live = h_p + nq;
    B200_CUDA_OK(cudaMemcpyAsync(h_tot, d_tot, 16, cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaMemcpyAsync(h_p, d_p, (size_t)nq * 8, cudaMemcpyDeviceToHost, s));   // p_q and live lists
    B200_CUDA_OK(cudaStreamSynchronize(s));
    const int64_t sum_live = (int64_t)h_tot[0];
    const int P = std::max(1, (int)h_tot[1]);
    ix->last_probe.insert(ix->last_probe.end(), h_p, h_p + nq);
    if (ix->timing) cudaEventRecord(ix->ev_ph[1], s);

    // Query ranges for the steps after the selection: the whole batch when its scratch, sized as scan_probes sizes it from
    // its live lists, fits the budget; else consecutive ranges that each fit it (at least one query), each sized by its own.  On
    // the look-up-scan indexes a range also keeps its per-query tables within kPqLutScratchBytes.
    const int64_t qrow_bytes = pq_uses_lut(ix) ? 0 : (int64_t)ix->d_pad64 * 2;
    auto scratch = [&](int64_t nqr, int64_t n_valid) {
        const int64_t ppc = pages_per_chunk(ix, n_valid, o.pages_per_chunk);
        const int64_t chunks = (ix->max_list_pages + ppc - 1) / ppc;
        return nqr * P * kFilterProbeSlotBytes + n_valid * (qrow_bytes + chunks * ((int64_t)k1 * 8 + 4 + (int64_t)sizeof(IvfGemmItem)));
    };
    const int64_t qmax = pq_uses_lut(ix) ? pq_lut_max_queries(ix) : nq;
    std::vector<std::pair<int64_t, int64_t>> ranges;   // (end query, live lists of the range)
    if (nq <= qmax && scratch(nq, sum_live) <= kFilterProbeScratchBytes) {
        ranges.emplace_back(nq, sum_live);
    } else {
        for (int64_t a = 0; a < nq;) {
            int64_t b = a + 1, v = h_live[a];
            while (b < nq && b - a < qmax && scratch(b + 1 - a, v + h_live[b]) <= kFilterProbeScratchBytes) v += h_live[b++];
            ranges.emplace_back(b, v);
            a = b;
        }
    }
    int64_t longest = 0;
    for (size_t r = 0; r < ranges.size(); r++) longest = std::max(longest, ranges[r].first - (r ? ranges[r - 1].first : 0));
    B200_TRY(ix->w_probe.reserve((size_t)longest * P * 8));
    const bool split = ranges.size() > 1;
    int64_t items = 0;
    for (size_t r = 0; r < ranges.size(); r++) {
        const int64_t a = r ? ranges[r - 1].first : 0, b = ranges[r].first;
        // probe rows of queries [a, b): a one-chunk batch still has its keys, a larger one recomputes them (same kernel, same values)
        for (int64_t q0 = a; q0 < b;) {
            const int64_t q1 = one_chunk ? b : std::min(b, q0 + chunk);
            if (!one_chunk) coarse_keys(q0, q1 - q0);
            probe_emit_kernel<<<(unsigned)(q1 - q0), kProbeThreads, 0, s>>>(ix->w_cs.as<float>() + (one_chunk ? q0 * nl : 0), nl, ix->w_flist.as<uint32_t>(),
                                                                           d_live + q0, d_key + q0, d_ties + q0, P, ix->w_probe.as<int64_t>() + (q0 - a) * P);
            g_launches++;
            q0 = q1;
        }
        B200_TRY(scan_probes(ix, d_q + a * ix->d_pad, d_qx + a * ix->d_pad, nullptr, b - a, k, k1, two_stage, o, ix->w_probe.as<int64_t>(), P, ranges[r].second,
                             list_len, list_pages, d_alive, id_offset, d_out_dis + a * k, d_out_ids + a * k, s));
        items += ix->last_items;
        if (split) {   // b200_index_last_scan reports the rows of the whole batch
            add_u64_kernel<<<1, 1, 0, s>>>(reinterpret_cast<const unsigned long long *>(ix->d_flag.as<int>() + 4), d_tot + 2);
            g_launches++;
        }
    }
    if (split) B200_CUDA_OK(cudaMemcpyAsync(ix->d_flag.as<int>() + 4, d_tot + 2, 8, cudaMemcpyDeviceToDevice, s));
    ix->last_items = items;
    return B200_OK;
}

// Graph search under a filter on the host entry: a filter that keeps fewer than kGraphExactFactor x k of the rows one query
// scores at the iteration cap (kept share x rows scored < 2k) would leave the alive list short, so the gathered exact pass over
// the kept rows answers instead.  Not measured: 2 only asks for room to fill k from the kept rows met on the walk.
constexpr double kGraphExactFactor = 2.0;

// rows one graph query scores at most: its seeds, then D per expanded parent, W parents per iteration up to the iteration cap
static int64_t graph_rows_at_cap(const b200_index *ix, int nseeds, int width) {
    return nseeds + (int64_t)graph_iteration_cap(ix->graph_degree, width) * width * ix->graph_degree;
}

// The graph search, asynchronous on s (d_q: the prepared queries [nq][d_pad]): seeds from the list path's first stage at
// nprobe 1 (the best min(ef_s, 32) ids per query), then one CTA per query (search_width=W > 1: one cluster of W CTAs, W
// parents per iteration) walks the graph: graph_search_kernel over the fp32 rows in HBM (HNSWFLAT, kc = k),
// graph_search_bf16_kernel over the bf16 list rows (MSTG), or graph_search_b1_kernel over the binary list rows (BINARYMSTG, kc =
// k: its keys are the exact distances; d_queries are its query bytes).  With a second stage
// (two_stage, MSTG only; kc may equal k, at k = 1024) the walk's best kc rows are re-ranked exactly by refine_device, from HBM
// or from host memory.
static int graph_search_locked(b200_index *ix, const float *d_queries, const float *d_q, int64_t nq, int k, int kc, bool two_stage, const SearchOpts &o,
                               const uint8_t *d_alive, int64_t id_offset, float *d_out_dis, int64_t *d_out_ids, cudaStream_t s) {
    const int ef = std::max(kc, o.ef_s);
    const int width = o.search_width;   // validated by search_device_locked
    const int S = std::min(ef, kGraphMaxSeeds);
    B200_TRY(ix->w_seeds.reserve((size_t)nq * S * 8));
    B200_TRY(ix->w_seedd.reserve((size_t)nq * S * 4));
    SearchOpts seed = search_opts(ix, nullptr);   // the index's defaults at nprobe 1, whatever keys the caller passed
    seed.graph = 0;
    seed.nprobe = 1;
    B200_TRY(search_device_locked(ix, d_queries, nq, S, seed, 1, nullptr, nullptr, 0, ix->w_seedd.as<float>(), ix->w_seeds.as<int64_t>(), nullptr, s));
    ix->last_seed_nq = nq;
    ix->last_seed_s = S;
    unsigned long long *scored = reinterpret_cast<unsigned long long *>(ix->d_flag.as<int>() + 4);
    B200_CUDA_OK(cudaMemsetAsync(scored, 0, 8, s));
    if (two_stage) {
        B200_TRY(ix->w_od.reserve((size_t)nq * kc * 4));
        B200_TRY(ix->w_oi.reserve((size_t)nq * kc * 8));
    }
    GraphB1Params bp{};
    GraphSearchParams &gp = bp.g;
    gp.queries = ix->binary ? nullptr : d_q;
    if (ix->d_row_slot) {
        gp.pages = ix->d_pool.p;
        gp.row_slot = ix->d_row_slot.as<uint32_t>();
    } else {
        gp.rows = reinterpret_cast<const float *>(corpus_device_rows(ix->raw.get()));
    }
    gp.graph = ix->d_graph.as<uint32_t>();
    gp.seeds = ix->w_seeds.as<int64_t>();
    gp.alive = d_alive;
    gp.out_dis = two_stage ? ix->w_od.as<float>() : d_out_dis;
    gp.out_ids = two_stage ? ix->w_oi.as<int64_t>() : d_out_ids;
    gp.rows_scored = scored;
    gp.n = ix->n;
    gp.id_offset = two_stage ? 0 : id_offset;
    gp.d_pad = ix->d_pad;
    gp.d_pad64 = ix->d_pad64;
    gp.degree = ix->graph_degree;
    gp.nseeds = S;
    gp.ef = ef;
    gp.k = kc;
    gp.max_iters = graph_iteration_cap(ix->graph_degree, width);
    gp.l2 = ix->metric == B200_METRIC_L2 || ix->binary;
    if (ix->binary) {
        bp.queries = reinterpret_cast<const uint8_t *>(d_queries);
        bp.row_popc = ix->d_row_bias.as<float>();
        bp.row_bytes = ix->row_bytes;
        bp.row_pad = ix->row_pad;
        bp.kb_w = ix->kb_w;
        bp.jaccard = ix->metric == B200_METRIC_JACCARD;
        B200_TRY(graph_search_b1(bp, nq, width, s));
    } else {
        B200_TRY(graph_search(gp, nq, width, s));
    }
    if (two_stage) B200_TRY(refine_device(ix, d_q, nq, ix->w_oi.as<int64_t>(), kc, k, id_offset, d_out_dis, d_out_ids, s));
    else cosine_finish(ix, d_q, nq, k, d_out_dis, d_out_ids, s);
    ix->last_items = nq * width;   // CTAs launched
    ix->last_graph = true;
    return B200_OK;
}

// The whole search on the device, asynchronous on s.  d_queries: fp32 [nq][d]; outputs [nq][k].  h_alive: the host copy of
// d_alive when the caller has one (the exact paths may then score only the rows it keeps), else null.
static int search_device_locked(b200_index *ix, const float *d_queries, int64_t nq, int k, const SearchOpts &o, int first_stage_only,
                                const uint8_t *d_alive, const uint8_t *h_alive, int64_t id_offset, float *d_out_dis, int64_t *d_out_ids,
                                int64_t *out_num_candidates, cudaStream_t s) {
    if (out_num_candidates) *out_num_candidates = k;
    if (nq == 0) return B200_OK;
    if (o.prefilter < 0 || o.prefilter > 2) return fail(B200_ERR_INVALID, "prefilter must be 0 (auto), 1 (never) or 2 (always)");
    // filter_probe=1 below nlist keeps its look-up tables within the budget itself, under its one synchronise
    const bool fselect_bounds_lut = o.filter_probe && d_alive && ix->use_ivf && o.nprobe < ix->nlist;
    if (pq_uses_lut(ix) && o.exact_batch != 1 && k <= 1024 && !fselect_bounds_lut) {
        // the look-up scan's tables are nq x M KB (4-bit codes: nq x M x 64 B): a larger batch runs as consecutive query
        // sub-batches through the whole search (every query's answer depends on that query alone, so the results are those of
        // one batch)
        const int64_t qmax = pq_lut_max_queries(ix);
        if (nq > qmax) {
            for (int64_t q0 = 0; q0 < nq; q0 += qmax)
                B200_TRY(search_device_locked(ix, d_queries + q0 * ix->d, std::min(qmax, nq - q0), k, o, first_stage_only, d_alive, h_alive, id_offset,
                                              d_out_dis + q0 * k, d_out_ids + q0 * k, out_num_candidates, s));
            return B200_OK;
        }
    }
    if (ix->binary) {
        // binary queries are bytes [nq][d / 8]; list rows are exact, so refine_factor / keep_raw / first_stage_only change nothing
        if (o.exact_batch == 1) return fail(B200_ERR_UNSUPPORTED, "exact_batch=1 is not available on binary indexes (their lists are exact)");
        if (o.filter_probe) return fail(B200_ERR_UNSUPPORTED, "filter_probe is not available on binary indexes (their coarse probe ranks at most 1024 lists)");
        if (!ix->use_ivf) {
            ix->last_probe.insert(ix->last_probe.end(), nq, 0);
            return corpus_search_exact(ix->raw.get(), d_queries, nq, k, d_alive, h_alive, o.prefilter, id_offset, d_out_dis, d_out_ids, s);
        }
    } else {
        B200_TRY(prepare_queries_device(ix, d_queries, nq, s));
    }
    const float *d_q = ix->w_q.as<float>();
    bool exact = !ix->use_ivf || o.exact_batch == 1;
    // graph_degree indexes walk their graph unless asked for the lists (graph=0) or the exact pass (exact_batch=1)
    const bool graph = ix->d_graph && !exact && o.graph != 0;
    // the walk returns kc rows per query: HNSWFLAT's are exact (kc = k); MSTG's are re-ranked from the fp32 rows when it has a
    // second stage (graph_two_stage, the list path's two_stage; kc = min(1024, k x refine_factor), its k1)
    int kc = k;
    bool graph_two_stage = false;
    if (graph) {
        if (k > kGraphMaxEf) return fail(B200_ERR_UNSUPPORTED, "k > 1024 on the graph search");
        if (o.ef_s > kGraphMaxEf) return fail(B200_ERR_INVALID, "ef_s must be at most 1024, got " + std::to_string(o.ef_s));
        if (!graph_width_ok(o.search_width)) return fail(B200_ERR_INVALID, "search_width must be 1, 2, 4 or 8, got " + std::to_string(o.search_width));
        if (ix->d_row_slot && !ix->binary) {   // BINARYMSTG: the walk's keys are the exact distances
            graph_two_stage = has_rows(ix) && o.refine_factor > 1 && !first_stage_only;
            if (graph_two_stage) kc = std::min(kGraphMaxEf, k * o.refine_factor);
        }
        if (out_num_candidates) *out_num_candidates = kc;
        // the exact rule scans the fp32 rows in HBM: without them (MSTG keep_raw=0 | 2) the walk always answers, and so does
        // BINARYMSTG's (its lists are the only copy of its rows; a load refuses a v4 binary file with rows)
        if (d_alive && h_alive && ix->raw && !ix->binary) {
            const int64_t rows_cap = graph_rows_at_cap(ix, std::min(std::max(kc, o.ef_s), kGraphMaxSeeds), o.search_width);
            const int64_t limit = std::min<int64_t>((int64_t)std::ceil(kGraphExactFactor * kc * (double)ix->n / (double)rows_cap) - 1,
                                                    corpus_prefilter_limit(ix->raw.get(), o.prefilter, nq, k));
            exact = limit >= 0 && host_count_alive(h_alive, ix->n, limit) <= limit;
            ix->last_probe_exact = exact;
        }
    } else if (!exact && o.filter_probe && d_alive && h_alive && ix->raw && !first_stage_only) {
        // filter_probe exact rule: a filter that keeps at most kFilterProbeExactFactor x the rows one query's plain probe scans
        // on average is answered by the exact pass over the kept rows (complete and exact) -- only when that pass takes its
        // gathered path for this batch (prefilter mode, nq, k): past the gathered path's limit it would scan every row
        const int64_t limit = std::min<int64_t>((int64_t)(kFilterProbeExactFactor * o.nprobe * (double)ix->n / (double)ix->nlist),
                                                corpus_prefilter_limit(ix->raw.get(), o.prefilter, nq, k));
        exact = limit >= 0 && host_count_alive(h_alive, ix->n, limit) <= limit;
        ix->last_probe_exact = exact;
    }
    if (exact) {
        if (out_num_candidates) *out_num_candidates = k;
        ix->last_probe.insert(ix->last_probe.end(), nq, 0);
        if (ix->keep_raw == 2)
            return fail(B200_ERR_UNSUPPORTED, "exact_batch=1 is not available with the fp32 rows in host memory (keep_raw=2 placement): "
                                              "the exact pass would stream every row over PCIe");
        if (!ix->raw) return fail(B200_ERR_INVALID, "exact search needs the fp32 rows (keep_raw=0 index)");
        // FLAT / fallback-to-flat: exact scan of the raw rows.  The raw corpus wants [nq][d] rows: strip the padding again.
        B200_TRY(unpad_queries(ix, d_q, nq, s));
        B200_TRY(corpus_search_exact(ix->raw.get(), ix->w_qraw.as<float>(), nq, k, d_alive, h_alive, o.prefilter, id_offset, d_out_dis, d_out_ids, s));
        cosine_finish(ix, d_q, nq, k, d_out_dis, d_out_ids, s);
        return B200_OK;
    }
    if (graph) return graph_search_locked(ix, d_queries, d_q, nq, k, kc, graph_two_stage, o, d_alive, id_offset, d_out_dis, d_out_ids, s);
    if (k > 1024) return fail(B200_ERR_UNSUPPORTED, "k > 1024 on IVF indexes");
    const int nl = ix->nlist;
    const int nprobe = o.nprobe;
    if (ix->binary && nprobe < nl && nprobe > 1024)
        return fail(B200_ERR_UNSUPPORTED, "binary indexes probe at most 1024 lists (the binary corpus k limit), or all of them (nprobe >= nlist)");
    const bool two_stage = has_rows(ix) && o.refine_factor > 1 && !first_stage_only && !ix->binary;
    const int k1 = two_stage ? std::min(1024, k * o.refine_factor) : k;
    if (out_num_candidates) *out_num_candidates = k1;
    // filter_probe=1 under a filter: the scan sees only the pages with kept rows, and below nlist every query probes as deep
    // as its first k1 kept rows need
    const bool fprobe = o.filter_probe && d_alive;
    const bool fselect = fprobe && nprobe < nl;
    const int64_t n_pairs = nq * nprobe;
    if (!fselect && n_pairs >= (int64_t)1 << 31) return fail(B200_ERR_UNSUPPORTED, "nq * nprobe must stay below 2^31");
    if (!fselect) ix->last_probe.insert(ix->last_probe.end(), nq, nprobe);

    if (ix->timing) cudaEventRecord(ix->ev_ph[0], s);
    // opq=1: the coarse probe and the list scan take the rotated queries; the exact second stage keeps the prepared ones
    const float *d_qx = d_q;
    if (ix->d_opq) {
        B200_TRY(ix->w_qrot.reserve((size_t)nq * ix->d_pad * 4));
        B200_CUDA_OK(launch_opq_rotate(d_qx, ix->d_pad, nq, ix->d, ix->d_opq.as<float>(), ix->w_qrot.as<float>(), ix->d_pad, s));
        d_q = ix->w_qrot.as<float>();
    }
    const uint32_t *list_len = ix->d_list_len.as<uint32_t>(), *list_pages = ix->d_list_pages.as<uint32_t>();
    if (fprobe) {
        B200_TRY(ix->w_flist.reserve((size_t)nl * 8));
        B200_TRY(ix->w_fpages.reserve((size_t)std::max<uint32_t>(ix->pages_used, 1) * 4));
        list_alive_kernel<<<(unsigned)nl, 256, 0, s>>>(ix->d_list_len.as<uint32_t>(), ix->d_list_page_off.as<uint32_t>(), ix->d_list_pages.as<uint32_t>(), ix->d_row_ids.as<uint32_t>(), d_alive,
                                                       ix->w_flist.as<uint32_t>(), ix->w_flist.as<uint32_t>() + nl, ix->w_fpages.as<uint32_t>());
        g_launches++;
        list_len = ix->w_flist.as<uint32_t>() + nl;
        list_pages = ix->w_fpages.as<uint32_t>();
        if (fselect)
            return filter_probe_search(ix, d_q, d_qx, nq, k, k1, two_stage, o, list_len, list_pages, d_alive, id_offset, d_out_dis, d_out_ids, s);
    }
    // ---- coarse probe: nprobe nearest centroids per query (exact FLAT search of the centroid table)
    B200_TRY(ix->w_probe.reserve((size_t)n_pairs * 8));
    B200_TRY(ix->w_pd.reserve((size_t)n_pairs * 4));
    if (ix->binary) {
        if (nprobe >= nl) {
            probe_all_kernel<<<(unsigned)ceil_div(n_pairs, 256), 256, 0, s>>>(ix->w_probe.as<int64_t>(), nq, nl);
            g_launches++;
        } else {
            B200_TRY(pad_bin_rows(ix, d_queries, nq, ix->w_qraw, s));
            B200_TRY(b200_corpus_search_device(ix->coarse.get(), ix->w_qraw.as<float>(), nq, nprobe, nullptr, 0, ix->w_pd.as<float>(), ix->w_probe.as<int64_t>(), s));
        }
    } else {
        B200_TRY(unpad_queries(ix, d_q, nq, s));
        // The centroid table is small and nprobe is a large k for it: the tensor-core path keeps one k-list per query lane
        // and never gets a selective threshold when k / nlist is a few percent.  The scan kernel's warp lists cost O(k / 32) per
        // insert: use it when its estimated time (FMA-bound, ~1.4 TB/s of table bytes per 8-query pass) undercuts ~1 us per
        // (query, 32 probes) of the tensor-core path.  Both rates of this model were taken on an earlier GPU and are
        // not re-measured on the H100; they only pick between two exact paths.
        const double t_scan = (double)ceil_div(nq, 8) * nl * ix->d_pad * 4.0 / 1.4e12;
        const double t_gemm = 1e-6 * (double)nq * std::max(1.0, nprobe / 32.0) + 30e-6;
        bool use_scan = nprobe > 8 && t_scan < t_gemm;
        // nprobe > 8: full ranking keys + warp select (coarse_scores_kernel / coarse_select_kernel above)
        int coarse_path = nprobe > 8 && nprobe <= 1024 ? 3 : use_scan ? 1 : 2;
        if (o.coarse_path) coarse_path = o.coarse_path;
        if (coarse_path == 3) {
            const int64_t chunk = coarse_chunk(nq, nl);
            B200_TRY(ix->w_cs.reserve((size_t)chunk * nl * 4));
            const size_t sel_smem = (size_t)8 * nprobe * 8;
            if (sel_smem > 48 * 1024) B200_CUDA_OK(cudaFuncSetAttribute(coarse_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sel_smem));
            for (int64_t q0 = 0; q0 < nq; q0 += chunk) {
                const int64_t nqc = std::min(chunk, nq - q0);
                coarse_scores_kernel<<<dim3((unsigned)ceil_div(nl, kCoarseTile), (unsigned)ceil_div(nqc, kCoarseTile)), 256, 0, s>>>(
                    d_q + q0 * ix->d_pad, ix->d_pad, ix->d_centroids.as<float>(), ix->d_cnorm.as<float>(), nqc, nl, ix->d, ix->w_cs.as<float>());
                coarse_select_kernel<<<(unsigned)ceil_div(nqc, 8), 256, sel_smem, s>>>(ix->w_cs.as<float>(), nqc, nl, nprobe, ix->w_pd.as<float>() + q0 * nprobe,
                                                                                       ix->w_probe.as<int64_t>() + q0 * nprobe);
                g_launches += 2;
            }
            B200_CUDA_OK(cudaGetLastError());
            ix->last_coarse = 3;
        } else {
            // chosen 2: the corpus' own choice by batch size; forced 2: the tensor-core path whatever the batch
            b200_corpus_set_path(ix->coarse.get(), coarse_path == 1 ? 1 : o.coarse_path == 2 ? 2 : 0);
            const int rc = b200_corpus_search_device(ix->coarse.get(), ix->w_qraw.as<float>(), nq, nprobe, nullptr, 0, ix->w_pd.as<float>(), ix->w_probe.as<int64_t>(), s);
            b200_corpus_set_path(ix->coarse.get(), 0);
            B200_TRY(rc);
            int kernel = 0;
            B200_TRY(b200_corpus_last_variant(ix->coarse.get(), &kernel, nullptr, nullptr, nullptr));
            ix->last_coarse = kernel == B200_KERNEL_SCAN ? 1 : 2;
        }
    }

    if (ix->timing) cudaEventRecord(ix->ev_ph[1], s);
    return scan_probes(ix, d_q, d_qx, d_queries, nq, k, k1, two_stage, o, ix->w_probe.as<int64_t>(), nprobe, n_pairs, list_len, list_pages, d_alive,
                       id_offset, d_out_dis, d_out_ids, s);
}

static void timing_collect(b200_index *ix) {
    if (!ix->timing || !ix->timed_pending) return;
    float ms = 0;
    if (cudaEventSynchronize(ix->ev1) == cudaSuccess && cudaEventElapsedTime(&ms, ix->ev0, ix->ev1) == cudaSuccess) {
        ix->timed_ms += ms;
        ix->timed_launches++;
    }
    if (cudaEventSynchronize(ix->ev_ph[5]) == cudaSuccess)
        for (int i = 0; i < 5; i++) {
            float pm = 0;
            if (cudaEventElapsedTime(&pm, ix->ev_ph[i], ix->ev_ph[i + 1]) == cudaSuccess) ix->phase_ms[i] = pm;
        }
    ix->timed_pending = false;
}

// the start of a search under ix->mu: the index's device, the previous search's timing collected, the last_* diagnostics cleared
static int begin_search_locked(b200_index *ix) {
    B200_CUDA_OK(cudaSetDevice(ix->device));
    timing_collect(ix);
    ix->last_probe.clear();
    ix->last_probe_exact = false;
    ix->last_coarse = 0;
    ix->last_graph = false;
    return B200_OK;
}

// Search::VectorIndex::search with device buffers, asynchronous on `stream` (NULL: the index's stream, synchronised)
extern "C" int b200_index_search_device(b200_index *ix, const float *d_queries, int64_t nq, int k, const char *params, int first_stage_only,
                                        const uint8_t *d_alive_bits, int64_t id_offset, float *d_out_dis, int64_t *d_out_ids, void *stream) {
    if (!ix || (!d_queries && nq > 0) || !d_out_dis || !d_out_ids || nq < 0 || k <= 0) return fail(B200_ERR_INVALID, "bad arguments");
    if (!ix->built) return fail(B200_ERR_INVALID, "index not built");
    std::lock_guard<std::mutex> lk(ix->mu);
    B200_TRY(begin_search_locked(ix));
    cudaStream_t s = stream ? reinterpret_cast<cudaStream_t>(stream) : ix->stream;
    B200_TRY(search_device_locked(ix, d_queries, nq, k, search_opts(ix, params), first_stage_only, d_alive_bits, nullptr, id_offset, d_out_dis, d_out_ids, nullptr, s));
    if (!stream) B200_CUDA_OK(cudaStreamSynchronize(s));
    return B200_OK;
}

// Search::VectorIndex::search(queries, k, params, first_stage_only, filter) (VIWithDataPart.cpp:926), host buffers
extern "C" int b200_index_search(b200_index *ix, const float *queries, int64_t nq, int k, const char *params, int first_stage_only,
                                 const uint8_t *alive_bits, float *out_dis, int64_t *out_ids, int64_t *out_num_candidates) {
    if (!ix || (!queries && nq > 0) || !out_dis || !out_ids || nq < 0 || k <= 0) return fail(B200_ERR_INVALID, "bad arguments");
    if (!ix->built) return fail(B200_ERR_INVALID, "index not built");
    if (out_num_candidates) *out_num_candidates = k;
    if (nq == 0) return B200_OK;
    std::lock_guard<std::mutex> lk(ix->mu);
    B200_TRY(begin_search_locked(ix));
    cudaStream_t s = ix->stream;
    B200_TRY(ix->w_host_q.reserve((size_t)nq * in_row_bytes(ix)));
    B200_TRY(ix->w_cand.reserve((size_t)nq * k * 12 + 16));
    B200_CUDA_OK(cudaMemcpyAsync(ix->w_host_q.p, queries, (size_t)nq * in_row_bytes(ix), cudaMemcpyHostToDevice, s));
    const uint8_t *d_alive = nullptr;
    if (alive_bits) {
        const size_t ab = (size_t)ceil_div(ix->n, 8);
        B200_TRY(ix->w_alive.reserve(ab + 16));
        B200_CUDA_OK(cudaMemcpyAsync(ix->w_alive.p, alive_bits, ab, cudaMemcpyHostToDevice, s));
        d_alive = ix->w_alive.as<uint8_t>();
    }
    float *r_d = ix->w_cand.as<float>();
    int64_t *r_i = reinterpret_cast<int64_t *>(reinterpret_cast<char *>(ix->w_cand.p) + (size_t)round_up(nq * k * 4, 8));
    B200_TRY(search_device_locked(ix, ix->w_host_q.as<float>(), nq, k, search_opts(ix, params), first_stage_only, d_alive, alive_bits, 0, r_d, r_i, out_num_candidates, s));
    B200_CUDA_OK(cudaMemcpyAsync(out_dis, r_d, (size_t)nq * k * 4, cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaMemcpyAsync(out_ids, r_i, (size_t)nq * k * 8, cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    timing_collect(ix);
    return B200_OK;
}

extern "C" int b200_index_train_loss(const b200_index *ix, double *out_eta, double *out_loss, int capacity, int *out_n) {
    if (!ix) return fail(B200_ERR_INVALID, "bad arguments");
    if (ix->aq_loss.empty()) return fail(B200_ERR_INVALID, "this index was not trained with aq_threshold (or is a loaded one)");
    const int n = (int)ix->aq_loss.size();
    if (out_loss && capacity < n) return fail(B200_ERR_INVALID, "train_loss: capacity " + std::to_string(capacity) + " < " + std::to_string(n));
    if (out_eta) *out_eta = ix->aq_eta;
    if (out_loss) std::copy(ix->aq_loss.begin(), ix->aq_loss.end(), out_loss);
    if (out_n) *out_n = n;
    return B200_OK;
}

extern "C" int b200_index_opq(const b200_index *ix, float *out_r, double *out_loss, int capacity, int *out_n) {
    if (!ix) return fail(B200_ERR_INVALID, "bad arguments");
    if (!ix->opq) return fail(B200_ERR_INVALID, "this index was not created with opq=1");
    if (!ix->d_opq) return fail(B200_ERR_INVALID, "this index holds no rotation (not trained yet, or a part below the inverted-file threshold: FLAT)");
    const int n = (int)ix->opq_loss.size();
    if (out_loss && capacity < n) return fail(B200_ERR_INVALID, "opq: capacity " + std::to_string(capacity) + " < " + std::to_string(n));
    if (out_r) {
        B200_CUDA_OK(cudaSetDevice(ix->device));
        B200_CUDA_OK(cudaMemcpy(out_r, ix->d_opq.as<float>(), (size_t)ix->d * ix->d * 4, cudaMemcpyDeviceToHost));
    }
    if (out_loss) std::copy(ix->opq_loss.begin(), ix->opq_loss.end(), out_loss);
    if (out_n) *out_n = n;
    return B200_OK;
}

extern "C" int b200_index_last_probe(b200_index *ix, int32_t *out_lists, int64_t capacity, int *out_exact) {
    if (!ix) return fail(B200_ERR_INVALID, "null index");
    std::lock_guard<std::mutex> lk(ix->mu);
    if (out_lists) {
        if (capacity < (int64_t)ix->last_probe.size()) return fail(B200_ERR_INVALID, "buffer smaller than the last search's nq");
        std::copy(ix->last_probe.begin(), ix->last_probe.end(), out_lists);
    }
    if (out_exact) *out_exact = ix->last_probe_exact ? 1 : 0;
    return B200_OK;
}

extern "C" int b200_index_last_coarse(b200_index *ix, int *path) {
    if (!ix || !path) return fail(B200_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> lk(ix->mu);
    *path = ix->last_coarse;
    return B200_OK;
}

extern "C" int b200_index_graph(const b200_index *ix, uint32_t *out, int64_t capacity_rows, int *out_degree) {
    if (!ix) return fail(B200_ERR_INVALID, "null index");
    const int D = ix->d_graph ? ix->graph_degree : 0;
    if (out_degree) *out_degree = D;
    if (out && D) {
        if (capacity_rows < ix->n) return fail(B200_ERR_INVALID, "buffer smaller than the index's rows");
        B200_CUDA_OK(cudaSetDevice(ix->device));
        B200_CUDA_OK(cudaMemcpy(out, ix->d_graph.as<uint32_t>(), (size_t)ix->n * D * 4, cudaMemcpyDeviceToHost));
    }
    return B200_OK;
}

extern "C" int b200_index_last_seeds(b200_index *ix, int64_t *out, int64_t capacity, int *out_per_query) {
    if (!ix) return fail(B200_ERR_INVALID, "null index");
    std::lock_guard<std::mutex> lk(ix->mu);
    const int S = ix->last_graph ? ix->last_seed_s : 0;
    if (out_per_query) *out_per_query = S;
    if (out && S) {
        if (capacity < ix->last_seed_nq * S) return fail(B200_ERR_INVALID, "buffer smaller than the last search's nq x seeds");
        B200_CUDA_OK(cudaSetDevice(ix->device));
        B200_CUDA_OK(cudaDeviceSynchronize());   // the search may still run on the caller's stream
        B200_CUDA_OK(cudaMemcpy(out, ix->w_seeds.p, (size_t)ix->last_seed_nq * S * 8, cudaMemcpyDeviceToHost));
    }
    return B200_OK;
}

// computeTopDistanceSubset: queries [nq][d], candidates [nq][ncand] (negative = unused) -> exact top-k
extern "C" int b200_index_refine(b200_index *ix, const float *queries, int64_t nq, const int64_t *cand_ids, int64_t ncand, int k,
                                 float *out_dis, int64_t *out_ids) {
    if (!ix || !queries || !cand_ids || !out_dis || !out_ids || nq < 0 || ncand <= 0 || k <= 0)
        return fail(B200_ERR_INVALID, "bad arguments");
    if (!ix->built) return fail(B200_ERR_INVALID, "index not built");
    if (ix->binary) return fail(B200_ERR_UNSUPPORTED, "binary indexes have no second stage (their lists are exact)");
    if (!has_rows(ix)) return fail(B200_ERR_INVALID, "this index keeps no fp32 rows (keep_raw=0): no second stage");
    if (k > 1024) return fail(B200_ERR_UNSUPPORTED, "k > 1024 in refine");
    if (nq == 0) return B200_OK;
    std::lock_guard<std::mutex> lk(ix->mu);
    B200_CUDA_OK(cudaSetDevice(ix->device));
    cudaStream_t s = ix->stream;
    B200_TRY(ix->w_host_q.reserve((size_t)nq * ix->d * 4));
    B200_CUDA_OK(cudaMemcpyAsync(ix->w_host_q.p, queries, (size_t)nq * ix->d * 4, cudaMemcpyHostToDevice, s));
    B200_TRY(prepare_queries_device(ix, ix->w_host_q.as<float>(), nq, s));
    B200_TRY(ix->w_probe.reserve((size_t)nq * ncand * 8));
    B200_TRY(ix->w_od.reserve((size_t)nq * k * 4));
    B200_TRY(ix->w_oi.reserve((size_t)nq * k * 8));
    B200_CUDA_OK(cudaMemcpyAsync(ix->w_probe.p, cand_ids, (size_t)nq * ncand * 8, cudaMemcpyHostToDevice, s));
    B200_TRY(refine_device(ix, ix->w_q.as<float>(), nq, ix->w_probe.as<int64_t>(), (int)ncand, k, 0, ix->w_od.as<float>(), ix->w_oi.as<int64_t>(), s));
    B200_CUDA_OK(cudaMemcpyAsync(out_dis, ix->w_od.p, (size_t)nq * k * 4, cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaMemcpyAsync(out_ids, ix->w_oi.p, (size_t)nq * k * 8, cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    return B200_OK;
}

// ------------------------------------------------------------------------------------
// persistence: VIWithColumnInPart::serialize / load (reference: src/VectorIndex/Common/VIWithDataPart.cpp:451-525,
// :578-764) write `<idx>-*.vidx3` through Search::IndexDataFileWriter; the on-disk format of the closed library
// is not reproducible, so this is our own single-file layout ("B2IX" v2): header, fp32 rows (when kept), then the
// quantisers and the pages in list order.  Loading re-uploads to HBM (pages become consecutive) and validates the header.
// Binary types (9..12, metrics HAMMING / JACCARD, payload 3): BINARYFLAT stores its row bytes [n][d / 8] in place of the fp32
// rows; the inverted types store the centroid bytes [nlist][cent_pad] in place of the fp32 centroids, then the list lengths
// and the pages (pool bytes, row ids, popcounts) like the float lists.
// ------------------------------------------------------------------------------------
namespace {
struct IxHeader {
    char magic[4];
    uint32_t version;
    int32_t type, metric, d, nlist, m, dsub, default_nprobe, refine_factor, payload, has_raw, use_ivf, code_bytes;
    int64_t n;
    uint32_t pages_used, reserved0;
};
// the byte stream is the caller's: a FILE (b200_index_save / _load) or the host's own stream objects
// (b200_index_save_cb / _load_cb: Search::IndexDataFileWriter / Reader over ClickHouse disks, VectorIndexIO.h:33-164)
struct Io {
    int (*write)(void *, const void *, size_t) = nullptr;
    int (*read)(void *, void *, size_t) = nullptr;
    void *ctx = nullptr;
};
bool wr(Io *f, const void *p, size_t bytes) { return bytes == 0 || (f->write && f->write(f->ctx, p, bytes) == 0); }
bool rd(Io *f, void *p, size_t bytes) { return bytes == 0 || (f->read && f->read(f->ctx, p, bytes) == 0); }
int file_write(void *ctx, const void *p, size_t bytes) { return fwrite(p, 1, bytes, reinterpret_cast<FILE *>(ctx)) == bytes ? 0 : 1; }
int file_read(void *ctx, void *p, size_t bytes) { return fread(p, 1, bytes, reinterpret_cast<FILE *>(ctx)) == bytes ? 0 : 1; }
}  // namespace

static int index_save_io(b200_index *ix, Io *f) {
    if (!ix->built) return fail(B200_ERR_INVALID, "index not built");
    std::lock_guard<std::mutex> lk(ix->mu);
    B200_CUDA_OK(cudaSetDevice(ix->device));
    IxHeader h{};
    memcpy(h.magic, "B2IX", 4);
    // v3: the v2 layout with reserved0 = the PQ code width (4) and a [m][16][dsub] codebook; every other index stays v2
    // v4: the v2 layout with reserved0 = the graph degree D, followed by the graph [n][D] u32 (graph_degree indexes)
    // v5: an opq=1 index: the v2 layout (reserved0 = 0) or the v3 one (reserved0 = 4), followed by R [d][d] fp32
    const bool pq4 = pq_uses_lut(ix) && ix->pq_bits == 4;
    h.version = ix->d_opq ? 5 : pq4 ? 3 : ix->d_graph ? 4 : 2;
    h.reserved0 = pq4 ? 4 : ix->d_graph ? (uint32_t)ix->graph_degree : 0;
    h.type = ix->type; h.metric = ix->metric; h.d = ix->d; h.nlist = ix->nlist; h.m = ix->m; h.dsub = ix->dsub;
    // has_raw 2: the same rows, to be loaded into host memory (keep_raw=2 placement)
    h.default_nprobe = ix->default_nprobe; h.refine_factor = ix->refine_factor; h.payload = ix->payload; h.has_raw = ix->h_rows ? 2 : ix->raw ? 1 : 0;
    h.use_ivf = ix->use_ivf ? 1 : 0; h.code_bytes = ix->code_bytes; h.n = ix->n; h.pages_used = ix->pages_used;
    bool ok = wr(f, &h, sizeof(h));
    try {
        if (ok && ix->raw && ix->binary) {   // binary rows as stored: [n][d / 8] bytes
            const size_t rb = (size_t)ix->row_bytes;
            const int64_t chunk = std::max<int64_t>(1, (64ll << 20) / (int64_t)rb);
            std::vector<char> buf((size_t)chunk * rb);
            const char *rows = reinterpret_cast<const char *>(corpus_device_rows(ix->raw.get()));
            for (int64_t off = 0; ok && off < ix->n; off += chunk) {
                const int64_t mrows = std::min(chunk, ix->n - off);
                ok = cudaMemcpy(buf.data(), rows + off * rb, (size_t)mrows * rb, cudaMemcpyDeviceToHost) == cudaSuccess && wr(f, buf.data(), (size_t)mrows * rb);
            }
        } else if (ok && ix->raw) {  // fp32 rows, unpadded (cosine indexes hold unit vectors; they are written as stored)
            const int64_t chunk = std::max<int64_t>(1, (64ll << 20) / ((int64_t)ix->d_pad * 4));
            std::vector<float> buf((size_t)chunk * ix->d_pad);
            const float *rows = reinterpret_cast<const float *>(corpus_device_rows(ix->raw.get()));
            for (int64_t off = 0; ok && off < ix->n; off += chunk) {
                const int64_t mrows = std::min(chunk, ix->n - off);
                if (cudaMemcpy(buf.data(), rows + off * ix->d_pad, (size_t)mrows * ix->d_pad * 4, cudaMemcpyDeviceToHost) != cudaSuccess) ok = false;
                for (int64_t r = 0; ok && r < mrows; r++) ok = wr(f, buf.data() + r * ix->d_pad, (size_t)ix->d * 4);
            }
        } else if (ok && ix->h_rows) {   // the same bytes, straight from host memory
            for (int64_t r = 0; ok && r < ix->n; r++) ok = wr(f, ix->h_rows + r * ix->d_pad, (size_t)ix->d * 4);
        }
        if (ok && ix->use_ivf) {
            std::vector<char> tmp;
            auto dump = [&](const void *dptr, size_t bytes) {
                tmp.resize(bytes);
                if (bytes && cudaMemcpy(tmp.data(), dptr, bytes, cudaMemcpyDeviceToHost) != cudaSuccess) return false;
                return wr(f, tmp.data(), bytes);
            };
            ok = (ix->binary ? dump(ix->d_bcent.as<uint8_t>(), (size_t)ix->nlist * ix->cent_pad) : dump(ix->d_centroids.as<float>(), (size_t)ix->nlist * ix->d * 4)) &&
                 wr(f, ix->list_len.data(), (size_t)ix->nlist * 4);
            if (ok && ix->d_pq) ok = dump(ix->d_pq.as<float>(), (size_t)ix->m * pq_codewords(ix->pq_bits) * ix->dsub * 4);
            if (ok && ix->d_sq) ok = dump(ix->d_sq.as<float>(), (size_t)4 * ix->d * 4);
            std::vector<uint32_t> pages(ix->pages_used);
            if (ok && ix->pages_used)
                ok = cudaMemcpy(pages.data(), ix->d_list_pages.as<uint32_t>(), (size_t)ix->pages_used * 4, cudaMemcpyDeviceToHost) == cudaSuccess;
            const size_t pb = (size_t)kPageRows * payload_row_bytes(ix);
            for (uint32_t i = 0; ok && i < ix->pages_used; i++) {
                const size_t row0 = (size_t)pages[i] * kPageRows;
                ok = dump(reinterpret_cast<const char *>(ix->d_pool.p) + (size_t)pages[i] * pb, pb) && dump(ix->d_row_ids.as<uint32_t>() + row0, kPageRows * 4);
                if (ok && ix->d_row_bias) ok = dump(ix->d_row_bias.as<float>() + row0, kPageRows * 4);
            }
        }
        if (ok && ix->d_opq) {
            std::vector<float> r((size_t)ix->d * ix->d);
            ok = cudaMemcpy(r.data(), ix->d_opq.as<float>(), r.size() * 4, cudaMemcpyDeviceToHost) == cudaSuccess && wr(f, r.data(), r.size() * 4);
        }
        if (ok && ix->d_graph) {
            const size_t rb = (size_t)ix->graph_degree * 4;
            const int64_t chunk = std::max<int64_t>(1, (64ll << 20) / (int64_t)rb);
            std::vector<char> buf((size_t)chunk * rb);
            for (int64_t off = 0; ok && off < ix->n; off += chunk) {
                const int64_t mrows = std::min(chunk, ix->n - off);
                ok = cudaMemcpy(buf.data(), ix->d_graph.as<uint32_t>() + off * ix->graph_degree, (size_t)mrows * rb, cudaMemcpyDeviceToHost) == cudaSuccess &&
                     wr(f, buf.data(), (size_t)mrows * rb);
            }
        }
    } catch (const std::bad_alloc &) {
        ok = false;
    }
    return ok ? B200_OK : fail(B200_ERR_INVALID, "index serialisation: write failed");
}

extern "C" int b200_index_save(b200_index *ix, const char *path) {
    if (!ix || !path) return fail(B200_ERR_INVALID, "bad arguments");
    FILE *fp = fopen(path, "wb");
    if (!fp) return fail(B200_ERR_INVALID, std::string("cannot open ") + path);
    Io io;
    io.write = file_write;
    io.ctx = fp;
    int rc = index_save_io(ix, &io);
    if (fclose(fp) != 0 && rc == B200_OK) rc = fail(B200_ERR_INVALID, std::string("write failed: ") + path);
    return rc;
}

extern "C" int b200_index_save_cb(b200_index *ix, int (*write)(void *ctx, const void *data, size_t bytes), void *ctx) {
    if (!ix || !write) return fail(B200_ERR_INVALID, "bad arguments");
    Io io;
    io.write = write;
    io.ctx = ctx;
    return index_save_io(ix, &io);
}

static int index_load_io(Io *f, b200_index **out) {
    *out = nullptr;
    IxHeader h{};
    if (!rd(f, &h, sizeof(h)) || memcmp(h.magic, "B2IX", 4) != 0 || h.version < 2 || h.version > 5)
        return fail(B200_ERR_INVALID, "not a B2IX v2 / v3 / v4 / v5 index file");
    // a truncated or corrupt file must fail here, not in a kernel: every size below is derived from these fields
    const bool bin = h.type >= IDX_BINFLAT;
    // v3: an inverted-file PQ index with 4-bit codes (reserved0 = 4), nibble-packed code rows and a [m][16][dsub] codebook
    // v5: an opq=1 PQ index (IVFPQ, SCANN, HNSWPQ; d <= kOpqMaxDim) with v3's reserved0 (4: 4-bit codes, 0: 8-bit)
    if (h.version == 5 && !(h.payload == IVF_PRODUCER_PQ && h.use_ivf && (h.type == IDX_IVFPQ || h.type == IDX_SCANN || h.type == IDX_HNSWPQ) &&
                            h.d > 0 && h.d <= kOpqMaxDim && (h.reserved0 == 0 || h.reserved0 == 4)))
        return fail(B200_ERR_INVALID, "corrupt index header (v5: an inverted-file IVFPQ / SCANN / HNSWPQ index with d <= " + std::to_string(kOpqMaxDim) +
                                          " and reserved0 0 or 4 expected)");
    const int pq_bits = h.version == 3 || (h.version == 5 && h.reserved0 == 4) ? 4 : 8;
    if (pq_bits == 4 &&
        !(h.reserved0 == 4 && h.payload == IVF_PRODUCER_PQ && h.use_ivf && h.m > 0 && h.dsub > 0 && (int64_t)h.m * h.dsub == h.d &&
          h.code_bytes >= pq_code_bytes(h.m, 4) && h.code_bytes % 16 == 0 && ivf_pq4_fits(h.m)))
        return fail(B200_ERR_INVALID, "corrupt index header (4-bit PQ with M <= " + std::to_string(ivf_pq4_max_m()) + " expected)");
    // v4: an inverted-file index with a graph of degree reserved0: HNSWFLAT with its fp32 rows in HBM, MSTG with any rows, or
    // BINARYMSTG without rows (its inverted lists hold the only copy)
    const bool walks_pages = h.type == IDX_MSTG || h.type == IDX_BINMSTG;   // the graph walk reads the list rows through the slot map
    if (h.version == 4 && !(graph_degree_ok((int)h.reserved0) && h.use_ivf &&
                            ((h.type == IDX_HNSWFLAT && h.has_raw == 1) || (h.type == IDX_MSTG && h.payload == IVF_PRODUCER_TMA) ||
                             (h.type == IDX_BINMSTG && h.payload == IVF_PRODUCER_B1 && h.has_raw == 0))))
        return fail(B200_ERR_INVALID, "corrupt index header (v4: an HNSWFLAT graph of degree 16, 32 or 64 over HBM rows, an MSTG graph, or a "
                                      "BINARYMSTG graph without rows, expected)");
    const bool sane = h.type >= 0 && h.type < IDX_NUM_TYPES && h.metric >= 0 && h.metric <= 4 && (h.metric >= B200_METRIC_HAMMING) == bin &&
                      h.d > 0 && h.d <= (1 << 16) && (!bin || h.d % 8 == 0) && h.n >= 0 &&
                      h.n < (int64_t)0xffffffffll && h.payload >= 0 && h.payload <= 3 && (h.payload == IVF_PRODUCER_B1) == bin &&
                      (!h.use_ivf || (h.nlist > 0 && h.nlist <= (1 << 24) && (uint64_t)h.pages_used <= (uint64_t)h.n / kPageRows + (uint64_t)h.nlist + 1)) &&
                      (h.payload != IVF_PRODUCER_PQ || !h.use_ivf || (h.m > 0 && h.dsub > 0 && h.m * h.dsub == h.d && h.code_bytes >= (pq_bits == 4 ? (h.m + 1) / 2 : h.m) && h.code_bytes % 16 == 0)) &&
                      (h.payload != IVF_PRODUCER_SQ8 || !h.use_ivf || (h.code_bytes >= h.d && h.code_bytes % 16 == 0)) && (h.has_raw || h.use_ivf) &&
                      h.has_raw >= 0 && h.has_raw <= 2 && (h.has_raw != 2 || (!bin && h.use_ivf));   // 2: host rows, float lists only
    if (!sane) return fail(B200_ERR_INVALID, "corrupt index header");
    b200_index *ix = nullptr;
    int rc = b200_index_create(kTypeNames[h.type], h.metric, h.d, "", &ix);
    if (rc != B200_OK) return rc;
    auto bail = [&](const std::string &msg) {
        b200_index_free(ix);
        return fail(B200_ERR_INVALID, msg);
    };
    try {
        ix->nlist = h.nlist; ix->m = h.m; ix->dsub = h.dsub; ix->pq_bits = pq_bits; ix->default_nprobe = h.default_nprobe; ix->refine_factor = h.refine_factor;
        ix->payload = h.payload; ix->use_ivf = h.use_ivf != 0; ix->code_bytes = h.code_bytes; ix->keep_raw = h.has_raw;
        const int raw_metric = h.metric == B200_METRIC_L2 ? B200_METRIC_L2 : B200_METRIC_IP;
        if (h.has_raw && bin) {
            if (corpus_create(h.metric, B200_DTYPE_BIN, h.d, h.n, ix->raw) != B200_OK) return bail(b200_last_error());
            const size_t rb = (size_t)ix->row_bytes;
            const int64_t chunk = std::max<int64_t>(1, (64ll << 20) / (int64_t)rb);
            std::vector<char> buf((size_t)chunk * rb);
            for (int64_t off = 0; off < h.n; off += chunk) {
                const int64_t mrows = std::min(chunk, h.n - off);
                if (!rd(f, buf.data(), (size_t)mrows * rb)) return bail("truncated index file (rows)");
                if (b200_corpus_append(ix->raw.get(), buf.data(), mrows) != B200_OK) return bail(b200_last_error());
            }
        } else if (h.has_raw == 2) {   // straight into pinned host memory, never through HBM
            if (host_rows_reserve(ix, h.n) != B200_OK) return bail(b200_last_error());
            const int64_t chunk = std::max<int64_t>(1, (64ll << 20) / ((int64_t)h.d * 4));
            std::vector<float> buf((size_t)chunk * h.d);
            for (int64_t off = 0; off < h.n; off += chunk) {
                const int64_t mrows = std::min(chunk, h.n - off);
                if (!rd(f, buf.data(), (size_t)mrows * h.d * 4)) return bail("truncated index file (rows)");
                for (int64_t r = 0; r < mrows; r++) memcpy(ix->h_rows + (off + r) * ix->d_pad, buf.data() + r * h.d, (size_t)h.d * 4);
            }
        } else if (h.has_raw) {
            if (corpus_create(raw_metric, B200_DTYPE_F32, h.d, h.n, ix->raw) != B200_OK) return bail(b200_last_error());
            const int64_t chunk = std::max<int64_t>(1, (64ll << 20) / ((int64_t)h.d * 4));
            std::vector<float> buf((size_t)chunk * h.d);
            for (int64_t off = 0; off < h.n; off += chunk) {
                const int64_t mrows = std::min(chunk, h.n - off);
                if (!rd(f, buf.data(), (size_t)mrows * h.d * 4)) return bail("truncated index file (rows)");
                if (b200_corpus_append(ix->raw.get(), buf.data(), mrows) != B200_OK) return bail(b200_last_error());
            }
        }
        ix->n = h.n;
        std::vector<uint8_t> in_list;   // row id -> it is in a list
        if (ix->use_ivf) {
            std::vector<char> tmp;
            auto slurp = [&](DevMem &dst, size_t bytes) {
                tmp.resize(bytes);
                if (!rd(f, tmp.data(), bytes)) return false;
                return dst.alloc(bytes + 256) == B200_OK && cudaMemcpy(dst.p, tmp.data(), bytes, cudaMemcpyHostToDevice) == cudaSuccess;
            };
            const int nl = h.nlist;
            ix->list_len.resize(nl);
            if (!(bin ? slurp(ix->d_bcent, (size_t)nl * ix->cent_pad) : slurp(ix->d_centroids, (size_t)nl * h.d * 4)) ||
                !rd(f, ix->list_len.data(), (size_t)nl * 4))
                return bail("truncated index file (quantiser)");
            uint64_t total = 0, pages = 0;
            std::vector<uint32_t> page_off(nl + 1, 0);
            for (int l = 0; l < nl; l++) {
                total += ix->list_len[l];
                page_off[l] = (uint32_t)pages;
                pages += (ix->list_len[l] + kPageRows - 1) / kPageRows;
                ix->max_list_pages = std::max<uint32_t>(ix->max_list_pages, (ix->list_len[l] + kPageRows - 1) / kPageRows);
            }
            page_off[nl] = (uint32_t)pages;
            // unusable rows are in no list: the lists hold at most n rows
            if (total > (uint64_t)h.n || pages != h.pages_used) return bail("corrupt index file (list lengths do not add up)");
            if (h.payload == IVF_PRODUCER_PQ) {
                if (!slurp(ix->d_pq, (size_t)h.m * pq_codewords(pq_bits) * h.dsub * 4)) return bail("truncated index file (codebook)");
                if (pq_bits == 4) {
                    // validated with the header: the 4-bit look-up scan reads the fp32 codebook
                } else if (pq_dsub_decodable(h.dsub)) {   // the tensor-core decoder's bf16 copy; the table look-up scan reads the fp32 codebook
                    if (ix->d_pq_bf16.alloc((size_t)h.m * 256 * h.dsub * 2) != B200_OK) return bail("cudaMalloc failed");
                    if (launch_f32_to_bf16_rows(ix->d_pq.as<float>(), h.dsub, ix->d_pq_bf16.as<__nv_bfloat16>(), h.dsub, (int64_t)h.m * 256, ix->stream) != cudaSuccess)
                        return bail("codebook conversion failed");
                } else if (!ivf_pq_lut_fits(h.m)) {
                    return bail("corrupt index header (PQ M too large for the table look-up scan)");
                }
            }
            if (h.payload == IVF_PRODUCER_SQ8 && !slurp(ix->d_sq, (size_t)4 * h.d * 4)) return bail("truncated index file (SQ ranges)");
            ix->pool_pages = ix->pages_used = h.pages_used;
            const size_t pb = (size_t)kPageRows * payload_row_bytes(ix), rows = (size_t)std::max<uint32_t>(h.pages_used, 1) * kPageRows;
            if (ix->d_pool.alloc(rows * payload_row_bytes(ix) + 256) != B200_OK || ix->d_row_ids.alloc(rows * 4) != B200_OK ||
                ((h.metric == B200_METRIC_L2 || bin) && ix->d_row_bias.alloc(rows * 4) != B200_OK))
                return bail("cudaMalloc of the page pool failed");
            std::vector<char> page(pb);
            std::vector<uint32_t> ids(kPageRows);
            std::vector<float> bias(kPageRows);
            in_list.assign((size_t)h.n, 0);
            uint32_t pg = 0;
            for (int l = 0; l < nl; l++) {
                const uint32_t np = (ix->list_len[l] + kPageRows - 1) / kPageRows;
                for (uint32_t t = 0; t < np; t++, pg++) {
                    if (!rd(f, page.data(), pb) || !rd(f, ids.data(), kPageRows * 4) || (ix->d_row_bias && !rd(f, bias.data(), kPageRows * 4)))
                        return bail("truncated index file (pages)");
                    const uint32_t valid = std::min<uint32_t>(kPageRows, ix->list_len[l] - t * kPageRows);
                    for (uint32_t r = 0; r < valid; r++) {
                        if (ids[r] >= (uint64_t)h.n) return bail("corrupt index file (row id out of range)");
                        in_list[ids[r]] = 1;
                    }
                    const size_t row0 = (size_t)pg * kPageRows;
                    if (cudaMemcpy(reinterpret_cast<char *>(ix->d_pool.p) + (size_t)pg * pb, page.data(), pb, cudaMemcpyHostToDevice) != cudaSuccess ||
                        cudaMemcpy(ix->d_row_ids.as<uint32_t>() + row0, ids.data(), kPageRows * 4, cudaMemcpyHostToDevice) != cudaSuccess ||
                        (ix->d_row_bias && cudaMemcpy(ix->d_row_bias.as<float>() + row0, bias.data(), kPageRows * 4, cudaMemcpyHostToDevice) != cudaSuccess))
                        return bail("H2D failed");
                }
            }
            std::vector<uint32_t> iota_pages(std::max<uint32_t>(h.pages_used, 1)), order(nl);
            for (uint32_t i = 0; i < h.pages_used; i++) iota_pages[i] = i;
            for (int l = 0; l < nl; l++) order[l] = (uint32_t)l;
            std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return ix->list_len[a] > ix->list_len[b]; });
            auto up = [&](DevMem &dst, const std::vector<uint32_t> &v, size_t count) {
                return dst.alloc(std::max<size_t>(count, 1) * 4) == B200_OK && cudaMemcpy(dst.p, v.data(), count * 4, cudaMemcpyHostToDevice) == cudaSuccess;
            };
            if (!up(ix->d_list_pages, iota_pages, h.pages_used) || !up(ix->d_list_page_off, page_off, (size_t)nl + 1) || !up(ix->d_list_order, order, nl) ||
                !up(ix->d_list_len, ix->list_len, nl) || ix->d_flag.alloc(32) != B200_OK)
                return bail("cudaMalloc failed");
            cudaMemset(ix->d_flag.as<int>(), 0, 32);
            if ((bin ? upload_coarse_bin(ix, ix->stream) : upload_coarse(ix, ix->stream)) != B200_OK) return bail(b200_last_error());
            if (cudaStreamSynchronize(ix->stream) != cudaSuccess) return bail("upload failed");
        }
        if (h.version == 5) {   // R: finite and orthonormal before any row or query is rotated by it
            std::vector<float> r((size_t)h.d * h.d);
            if (!rd(f, r.data(), r.size() * 4)) return bail("truncated index file (OPQ rotation)");
            for (float v : r)
                if (!std::isfinite(v)) return bail("corrupt index file (OPQ rotation not finite)");
            double err = 0;
            if (ix->d_opq.alloc(r.size() * 4) != B200_OK ||
                cudaMemcpy(ix->d_opq.as<float>(), r.data(), r.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess ||
                opq_orthonormal_error(ix->d_opq.as<float>(), h.d, &err, ix->stream) != B200_OK)
                return bail(std::string("OPQ rotation upload: ") + b200_last_error());
            if (!(err <= kOpqLoadTol)) return bail("corrupt index file (OPQ rotation not orthonormal: max |R^T R - I| = " + std::to_string(err) + ")");
            ix->opq = 1;
        }
        if (h.version == 4) {   // every id < n or 0xFFFFFFFF before a kernel walks the graph; (BINARY)MSTG: every id in a list (it has a pool slot)
            const int D = (int)h.reserved0;
            const size_t rb = (size_t)D * 4;
            const int64_t chunk = std::max<int64_t>(1, (64ll << 20) / (int64_t)rb);
            std::vector<uint32_t> buf((size_t)chunk * D);
            if (ix->d_graph.alloc(std::max<size_t>((size_t)h.n * rb, 16)) != B200_OK) return bail("cudaMalloc of the graph failed");
            ix->graph_degree = D;
            for (int64_t off = 0; off < h.n; off += chunk) {
                const int64_t mrows = std::min(chunk, h.n - off);
                if (!rd(f, buf.data(), (size_t)mrows * rb)) return bail("truncated index file (graph)");
                for (int64_t e = 0; e < mrows * D; e++) {
                    if (buf[e] == kNoId) continue;
                    if (buf[e] >= (uint64_t)h.n) return bail("corrupt index file (graph id out of range)");
                    if (walks_pages && !in_list[buf[e]]) return bail("corrupt index file (graph edge to a row in no list)");
                }
                if (cudaMemcpy(ix->d_graph.as<uint32_t>() + off * D, buf.data(), (size_t)mrows * rb, cudaMemcpyHostToDevice) != cudaSuccess) return bail("H2D failed");
            }
            // MSTG / BINARYMSTG: the slot map of the pages as loaded here
            if (walks_pages && (build_row_slot(ix) != B200_OK || cudaStreamSynchronize(ix->stream) != cudaSuccess))
                return bail(std::string("graph row slot map: ") + b200_last_error());
        }
    } catch (const std::bad_alloc &) {
        return bail("out of host memory while loading the index");
    }
    ix->trained = true;
    ix->built = true;
    *out = ix;
    return B200_OK;
}

extern "C" int b200_index_load(const char *path, b200_index **out) {
    if (!path || !out) return fail(B200_ERR_INVALID, "bad arguments");
    *out = nullptr;
    FILE *fp = fopen(path, "rb");
    if (!fp) return fail(B200_ERR_INVALID, std::string("cannot open ") + path);
    Io io;
    io.read = file_read;
    io.ctx = fp;
    const int rc = index_load_io(&io, out);
    fclose(fp);
    return rc;
}

extern "C" int b200_index_load_cb(int (*read)(void *ctx, void *data, size_t bytes), void *ctx, b200_index **out) {
    if (!read || !out) return fail(B200_ERR_INVALID, "bad arguments");
    Io io;
    io.read = read;
    io.ctx = ctx;
    return index_load_io(&io, out);
}
