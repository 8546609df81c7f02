// ivf_pq_lut_sm90.cu -- K5b: the PQ list scan by table look-up (asymmetric distance computation), for the PQ indexes whose
// sub-vectors the tensor-core decoder of ivf_gemm_sm90.cu cannot take: d / M outside {1, 2, 4, 8}, at any width.
//
// The pair constant (||q - c||^2 or -<q, c>, pair_fill_kernel) and the row bias (L2: 2 <c, r^> + ||r^||^2) leave one
// query-by-row term, <q, r^> = sum_j <q_j, cb_j[code_j]>, and it does not depend on the list.  pq_lut_kernel tabulates
// T[q][j][e] = <q_j, cb_j[e]> once per query of the batch (fp32, from the fp32 query and the fp32 codebook); the scan sums
// M table entries per row:
//   key = scale * sum_j T[q][j][code_j] + bias,  scale = -2 (L2) or -1 (IP / cosine)
// and consumes the same work items, writes the same [pair][chunk][k] partial lists and part_worst, and shares the same
// per-query bound as the tensor-core scan, so the plan, the merge and the second stage do not change.
//
// One CTA of 256 threads walks items blockIdx.x, blockIdx.x + grid, ...; inside an item the queries are the outer loop:
//   * the query's table (M KB) is copied into shared memory by one cp.async.bulk completing on an mbarrier; when two tables
//     fit, the next query's table lands while this one scans;
//   * thread t owns row t of every page: 16-byte code loads (an item's pages are read again for each of its queries, from
//     L2), M fp32 look-ups summed in fp32, the key, the alive bit, and a threshold filter into a shared candidate buffer;
//   * the buffer is sorted (bitonic, by (key, pool row)) and rank-merged into the query's sorted k-list when the next page
//     could overflow it, when it can fill a list that is not full yet, and at the end of the item.
// Pool rows of one list increase with the row ids, so (key, pool row) order is (key, row id) order: ties keep the smaller id.
#include <algorithm>

#include "gemm_common.cuh"
#include "ivf_gemm.h"

namespace b200 {
namespace lut {
using gemm::mbar_init;
using gemm::mbar_arrive_expect_tx;
using gemm::mbar_wait;
using gemm::bound_encode;
using gemm::bound_decode;

constexpr int THREADS = 256;    // one thread per page row
constexpr int PAGE = 256;       // rows per page (kPageRows of ivf.cu)
constexpr int CAND = 2048;      // candidate buffer entries, a power of two
constexpr int MAX_M = 128;      // sub-quantisers: the table of one query is at most 128 KB
constexpr int MISC_BYTES = 96;  // two mbarriers + per-warp candidate counts of two pages

// dynamic shared memory: nbuf tables [m][256] fp32 | list keys [2][k] | list ids [2][k] | candidates keys [CAND], ids [CAND] | misc
__host__ __device__ inline int smem_bytes(int m, int k, int nbuf) {
    return nbuf * m * 1024 + (int)round_up((int64_t)k * 16, 16) + CAND * 8 + MISC_BYTES;
}

__device__ __forceinline__ void bulk_load(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src),
                 "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// T[q][j][e] = <q_j, cb_j[e]>: block (8 queries, sub-quantiser j), thread e; fp32 fmaf over the sub-vector in order
constexpr int LUT_QB = 8;
__global__ void __launch_bounds__(256) pq_lut_kernel(const float *__restrict__ queries, int64_t nq, int d_pad, const float *__restrict__ cb, int m,
                                                     int dsub, float *__restrict__ out) {
    const int j = blockIdx.y, e = threadIdx.x;
    const int64_t q0 = (int64_t)blockIdx.x * LUT_QB;
    const float *c = cb + ((size_t)j * 256 + e) * dsub;
    const float *x[LUT_QB];
#pragma unroll
    for (int i = 0; i < LUT_QB; i++) x[i] = queries + (size_t)std::min<int64_t>(q0 + i, nq - 1) * d_pad + (size_t)j * dsub;
    float acc[LUT_QB];
#pragma unroll
    for (int i = 0; i < LUT_QB; i++) acc[i] = 0.f;
    for (int t = 0; t < dsub; t++) {
        const float cv = c[t];
#pragma unroll
        for (int i = 0; i < LUT_QB; i++) acc[i] = fmaf(x[i][t], cv, acc[i]);
    }
#pragma unroll
    for (int i = 0; i < LUT_QB; i++)
        if (q0 + i < nq) out[((size_t)(q0 + i) * m + j) * 256 + e] = acc[i];
}

__global__ void __launch_bounds__(THREADS, 2) ivf_pq_lut_topk_kernel(const IvfGemmParams p) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int m = p.m, k = p.k, nbuf = p.stages;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const size_t tbl_words = (size_t)m * 256;
    float *tables = reinterpret_cast<float *>(smem);
    float *lkeys = reinterpret_cast<float *>(smem + (size_t)nbuf * m * 1024);   // [2][k]
    uint32_t *lids = reinterpret_cast<uint32_t *>(lkeys + 2 * k);              // [2][k]
    float *ck = reinterpret_cast<float *>(smem + (size_t)nbuf * m * 1024 + round_up((int64_t)k * 16, 16));
    uint32_t *ci = reinterpret_cast<uint32_t *>(ck + CAND);
    uint64_t *bar = reinterpret_cast<uint64_t *>(ci + CAND);
    int *wcnt = reinterpret_cast<int *>(bar + 2);                              // [2 pages][8 warps]

    const int n_items = *p.n_items_ptr;
    int it = blockIdx.x;
    if (it >= n_items) return;
    if (tid == 0) {
        mbar_init(&bar[0], 1);
        mbar_init(&bar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const uint32_t tbytes = (uint32_t)m * 1024u;
    // thread 0: the table of the query of sorted pair `pair` into buffer b (every thread is done with b's previous table)
    auto issue = [&](int b, uint32_t pair) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        mbar_arrive_expect_tx(&bar[b], tbytes);
        bulk_load(tables + b * tbl_words, p.lut + (size_t)(p.sorted_pair[pair] / (uint32_t)p.nprobe) * tbl_words, tbytes, &bar[b]);
    };
    // the task after (item it, slot sl) of this CTA's walk: its sorted pair, or 0xffffffff
    auto next_pair = [&](const IvfGemmItem &item, uint32_t sl) -> uint32_t {
        if (sl + 1 < item.q_count) return item.q_begin + sl + 1;
        if (it + (int)gridDim.x < n_items) return p.items[it + gridDim.x].q_begin;
        return 0xffffffffu;
    };
    if (tid == 0) issue(0, p.items[it].q_begin);
    uint32_t seq = 0;
    for (; it < n_items; it += gridDim.x) {
        const IvfGemmItem item = p.items[it];
        for (uint32_t sl = 0; sl < item.q_count; sl++, seq++) {
            const int b = nbuf == 2 ? (int)(seq & 1) : 0;
            const uint32_t parity = nbuf == 2 ? (seq >> 1) & 1 : seq & 1;
            if (nbuf == 2 && tid == 0) {
                const uint32_t np_ = next_pair(item, sl);
                if (np_ != 0xffffffffu) issue(b ^ 1, np_);
            }
            const uint32_t pair = item.q_begin + sl;
            uint32_t *bound_slot = p.query_bound ? p.query_bound + p.sorted_pair[pair] / (uint32_t)p.nprobe : nullptr;
            const float pc = bound_slot ? p.pair_const[pair] : 0.f;
            float last_pub = FLT_MAX;
            // the query's sorted list (lkeys / lids buffer `cur`): block-uniform state
            int n = 0, cur = 0, cnt = 0;
            float thr_key = FLT_MAX;
            uint32_t thr_id = 0;
            mbar_wait(&bar[b], parity);
            const float *T = tables + b * tbl_words;
            for (uint32_t j = 0; j < item.page_count; j++) {
                const uint32_t row0 = p.list_pages[item.page_begin + j] * (uint32_t)PAGE;
                const uint32_t valid = min((uint32_t)PAGE, item.row_limit - j * (uint32_t)PAGE);
                const uint32_t row = row0 + tid;
                float key = FLT_MAX;
                bool cand = false;
                if ((uint32_t)tid < valid) {
                    bool ok = true;
                    if (p.alive) {
                        const uint32_t id = p.row_ids[row];
                        ok = (p.alive[id >> 3] >> (id & 7)) & 1;
                    }
                    if (ok) {
                        // the bound in this pair's key space, a few ulps loose (the merge adds pair_const back in fp32)
                        float ext = FLT_MAX;
                        if (bound_slot) {
                            const uint32_t u = __ldcg(bound_slot);
                            if (u != 0xffffffffu) {
                                const float g = bound_decode(u);
                                ext = g - pc;
                                ext += (fabsf(ext) + fabsf(pc) + fabsf(g)) * 4e-7f;
                            }
                        }
                        const uint4 *cr = reinterpret_cast<const uint4 *>(p.codes + (size_t)row * p.code_bytes);
                        float acc = 0.f;
                        for (int j0 = 0; j0 < m; j0 += 16) {
                            const uint4 w = cr[j0 >> 4];
                            const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
                            const float *Tj = T + (size_t)j0 * 256;
                            float s = 0.f;
#pragma unroll
                            for (int t = 0; t < 16; t++)
                                if (j0 + t < m) s += Tj[t * 256 + ((ww[t >> 2] >> ((t & 3) * 8)) & 255u)];
                            acc += s;
                        }
                        key = fmaf(p.scale_const, acc, p.row_bias ? p.row_bias[row] : 0.f);
                        cand = key <= ext && better(key, row, thr_key, thr_id);
                    }
                }
                // candidate slots by a block-wide prefix count (per-warp counts double-buffered by page parity)
                const unsigned bal = __ballot_sync(0xffffffffu, cand);
                int *wc = wcnt + (j & 1) * 8;
                if (lane == 0) wc[warp] = __popc(bal);
                __syncthreads();
                int before = cnt, total = cnt;
#pragma unroll
                for (int w = 0; w < THREADS / 32; w++) {
                    const int c = wc[w];
                    before += w < warp ? c : 0;
                    total += c;
                }
                if (cand) {
                    const int pos = before + __popc(bal & ((1u << lane) - 1u));
                    ck[pos] = key;
                    ci[pos] = row;
                }
                cnt = total;
                if (cnt > 0 && (cnt > CAND - PAGE || (n < k && n + cnt >= k) || j + 1 == item.page_count)) {
                    __syncthreads();   // the candidates are written
                    int n2 = 2;
                    while (n2 < cnt) n2 <<= 1;
                    for (int i = cnt + tid; i < n2; i += THREADS) {
                        ck[i] = FLT_MAX;
                        ci[i] = kNoId;
                    }
                    __syncthreads();
                    for (int size = 2; size <= n2; size <<= 1)
                        for (int stride = size >> 1; stride > 0; stride >>= 1) {
                            for (int t = tid; t < (n2 >> 1); t += THREADS) {
                                const int i = ((t / stride) * 2 * stride) + (t % stride), i2 = i + stride;
                                const float ka = ck[i], kb = ck[i2];
                                const uint32_t ia = ci[i], ib = ci[i2];
                                if (better(kb, ib, ka, ia) == ((i & size) == 0)) {
                                    ck[i] = kb; ci[i] = ib;
                                    ck[i2] = ka; ci[i2] = ia;
                                }
                            }
                            __syncthreads();
                        }
                    // rank merge of list[0, n) and cand[0, mc): an entry's position in the union (the two sets are disjoint)
                    const int mc = min(cnt, k);
                    const float *ak = lkeys + cur * k;
                    const uint32_t *ai = lids + cur * k;
                    float *ok = lkeys + (cur ^ 1) * k;
                    uint32_t *oi = lids + (cur ^ 1) * k;
                    for (int a = tid; a < n; a += THREADS) {
                        const float kk = ak[a];
                        const uint32_t id = ai[a];
                        int lo = 0, hi = mc;
                        while (lo < hi) {
                            const int mid = (lo + hi) >> 1;
                            if (better(ck[mid], ci[mid], kk, id)) lo = mid + 1; else hi = mid;
                        }
                        if (a + lo < k) { ok[a + lo] = kk; oi[a + lo] = id; }
                    }
                    for (int c = tid; c < mc; c += THREADS) {
                        const float kk = ck[c];
                        const uint32_t id = ci[c];
                        int lo = 0, hi = n;
                        while (lo < hi) {
                            const int mid = (lo + hi) >> 1;
                            if (better(ak[mid], ai[mid], kk, id)) lo = mid + 1; else hi = mid;
                        }
                        if (c + lo < k) { ok[c + lo] = kk; oi[c + lo] = id; }
                    }
                    __syncthreads();
                    n = min(n + mc, k);
                    cur ^= 1;
                    cnt = 0;
                    if (n == k) {
                        thr_key = ok[k - 1];
                        thr_id = oi[k - 1];
                        // publish: a full list's k-th key bounds the query's k-th key over all its lists
                        if (bound_slot && thr_key < last_pub) {
                            last_pub = thr_key;
                            if (tid == 0) atomicMin(bound_slot, bound_encode(thr_key + pc));
                        }
                    }
                }
            }
            // this (pair, chunk)'s partial list: pool rows mapped to row ids, worst kept key aside
            const size_t part = (size_t)p.pair_part_base[pair] + item.chunk;
            const float *fk = lkeys + cur * k;
            const uint32_t *fi = lids + cur * k;
            for (int e = tid; e < k; e += THREADS) {
                const bool have = e < n;
                p.part_keys[part * k + e] = have ? fk[e] : FLT_MAX;
                p.part_ids[part * k + e] = have ? p.row_ids[fi[e]] : kNoId;
            }
            if (tid == 0) p.part_worst[part] = n == k ? thr_key : FLT_MAX;
            __syncthreads();   // the table, the lists and the candidates are free again
            if (nbuf == 1 && tid == 0) {
                const uint32_t np_ = next_pair(item, sl);
                if (np_ != 0xffffffffu) issue(0, np_);
            }
        }
    }
}

}  // namespace lut

bool ivf_pq_lut_fits(int m) { return m >= 1 && m <= lut::MAX_M && lut::smem_bytes(m, 1024, 1) <= gemm::SMEM_LIMIT; }

cudaError_t launch_pq_lut(const float *queries, int64_t nq, int d_pad, const float *codebook, int m, int dsub, float *lut_out, cudaStream_t s) {
    if (nq <= 0) return cudaSuccess;
    lut::pq_lut_kernel<<<dim3((unsigned)ceil_div(nq, lut::LUT_QB), (unsigned)m), 256, 0, s>>>(queries, nq, d_pad, codebook, m, dsub, lut_out);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t launch_ivf_pq_lut_topk(const IvfGemmParams &p_in, int grid, cudaStream_t s, const char **err_detail) {
    *err_detail = nullptr;
    IvfGemmParams p = p_in;
    if (!p.lut || !p.sorted_pair || p.nprobe < 1 || p.code_bytes % 16 || p.code_bytes < p.m || p.k < 1 || p.k > 1024 || !ivf_pq_lut_fits(p.m)) {
        *err_detail = "PQ table look-up scan: table, sorted pairs, 16-byte code rows, 1 <= k <= 1024 and M <= 128 needed";
        return cudaErrorInvalidValue;
    }
    // two table buffers (the next query's table lands during this one's scan) when they fit
    p.stages = lut::smem_bytes(p.m, p.k, 2) <= gemm::SMEM_LIMIT ? 2 : 1;
    const int smem = lut::smem_bytes(p.m, p.k, p.stages);
    cudaError_t e = cudaFuncSetAttribute(lut::ivf_pq_lut_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    int per_sm = 1;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lut::ivf_pq_lut_topk_kernel, lut::THREADS, smem);
    if (e != cudaSuccess) return e;
    lut::ivf_pq_lut_topk_kernel<<<grid * std::max(1, per_sm), lut::THREADS, smem, s>>>(p);
    g_launches++;
    return cudaGetLastError();
}

}  // namespace b200
