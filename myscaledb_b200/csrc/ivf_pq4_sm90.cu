// ivf_pq4_sm90.cu -- K5c: the PQ list scan by table look-up for 4-bit codes (bit_size = 4): 16 codewords per sub-quantiser,
// two codes per byte (code j in byte j / 2, even j in the low nibble).
//
// The key splits as for the 8-bit look-up scan (ivf_pq_lut_sm90.cu): the pair constant, the row bias and
//   key = scale * sum_j T[q][j][code_j] + bias,  scale = -2 (L2) or -1 (IP / cosine)
// with T[q][j][e] = <q_j, cb_j[e]> for e < 16, tabulated in fp32 by pq4_lut_kernel.  The scan consumes the same work items,
// writes the same [pair][chunk][k] partial lists and part_worst and shares the same per-query bound, so the plan, the merge
// and the second stage do not change.
//
// What 4 bits change: a sub-quantiser's table row is 16 consecutive fp32 words, so the 32 look-ups of a warp at the same j hit
// 16 distinct banks or broadcast one word (no bank conflicts), and one query's table is only 64 M bytes.  So a CTA holds the
// tables of a group of G queries and reads each row's codes once per group rather than once per query:
//   * one CTA of 256 threads walks items blockIdx.x, blockIdx.x + grid, ...; an item's queries are taken G at a time, their
//     tables copied into shared memory by cp.async.bulk completing on one mbarrier;
//   * thread t owns row t of every page: 16-byte code loads (32 codes each), G fp32 sums from the G tables, the alive bit,
//     and per query the shared bound and a threshold filter into that query's candidate buffer;
//   * a query's buffer is sorted (bitonic, by (key, pool row)) and rank-merged into its sorted k-list when the next page could
//     overflow it, when it can fill a list that is not full yet, and at the end of the item.
// G is chosen at launch (largest of 8, 4, 2 whose G tables, G list pairs and G candidate buffers leave room for two CTAs per
// SM, else 1).  A query's sums, filter and merges do not depend on G or on the other queries of its group, so results are
// byte-identical however the batch is grouped.  Ties keep the smaller row id: pool rows of one list increase with the ids.
#include <algorithm>

#include "gemm_common.cuh"
#include "ivf_gemm.h"

namespace b200 {
namespace pq4 {
using gemm::mbar_init;
using gemm::mbar_arrive_expect_tx;
using gemm::mbar_wait;
using gemm::bound_encode;
using gemm::bound_decode;

constexpr int THREADS = 256;   // one thread per page row
constexpr int PAGE = 256;      // rows per page (kPageRows of ivf.cu)
constexpr int CAND = 512;      // candidate buffer entries per query, a power of two >= PAGE
constexpr int MAX_M = 2048;    // sub-quantisers: one query's table is at most 128 KB
constexpr int MAX_G = 8;       // queries per group
constexpr uint32_t NO_QUERY = 0xffffffffu;

// block-uniform state of one query of the group (written by thread 0 behind a barrier, read by all)
struct QState {
    int n, cur, cnt, ncnt;     // kept list entries, its buffer, candidates held, candidates after this page
    float thr_key, last_pub, pc;
    uint32_t thr_id, q;        // q: query of the shared bound, or NO_QUERY
    uint32_t pad[3];
};
constexpr int MISC_BYTES = 16 + 2 * MAX_G * 8 * 4 + MAX_G * (int)sizeof(QState);   // mbarrier | per-warp counts [2][G][8] | states

__host__ __device__ inline int list_bytes(int k) { return (int)round_up((int64_t)k * 16, 16); }
// dynamic shared memory: G tables [m][16] fp32 | G list pairs keys [2][k], ids [2][k] | G candidate buffers keys, ids [CAND] | misc
__host__ __device__ inline int smem_bytes(int m, int k, int g) { return g * (m * 64 + list_bytes(k) + CAND * 8) + MISC_BYTES; }

// queries per group: the largest of 8, 4, 2 that leaves room for two CTAs per SM, else 1
inline int group_size(int m, int k) {
    for (int g = MAX_G; g > 1; g >>= 1)
        if (smem_bytes(m, k, g) <= gemm::SMEM_LIMIT / 2) return g;
    return 1;
}

__device__ __forceinline__ void bulk_load(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src),
                 "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// T[q][j][e] = <q_j, cb_j[e]>, e < 16: block (8 queries, 16 sub-quantisers), thread (j % 16, e); fp32 fmaf over the sub-vector
// in order, as pq_lut_kernel does for 256 codewords
constexpr int LUT_QB = 8;
__global__ void __launch_bounds__(256) pq4_lut_kernel(const float *__restrict__ queries, int64_t nq, int d_pad, const float *__restrict__ cb, int m,
                                                      int dsub, float *__restrict__ out) {
    const int j = blockIdx.y * 16 + (threadIdx.x >> 4), e = threadIdx.x & 15;
    if (j >= m) return;
    const int64_t q0 = (int64_t)blockIdx.x * LUT_QB;
    const float *c = cb + ((size_t)j * 16 + e) * dsub;
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
        if (q0 + i < nq) out[((size_t)(q0 + i) * m + j) * 16 + e] = acc[i];
}

template <int G>
__global__ void __launch_bounds__(THREADS, 2) ivf_pq4_topk_kernel(const IvfGemmParams p) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int m = p.m, k = p.k;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int tbl_words = m * 16, lb = list_bytes(k);
    float *tables = reinterpret_cast<float *>(smem);
    unsigned char *lists = smem + (size_t)G * m * 64;
    unsigned char *cands = lists + (size_t)G * lb;
    uint64_t *bar = reinterpret_cast<uint64_t *>(cands + (size_t)G * CAND * 8);
    int *wcnt = reinterpret_cast<int *>(bar + 2);                                   // [2 pages][G][8 warps]
    QState *qs = reinterpret_cast<QState *>(wcnt + 2 * MAX_G * 8);
    auto lkeys = [&](int g) { return reinterpret_cast<float *>(lists + (size_t)g * lb); };          // [2][k]
    auto lids = [&](int g) { return reinterpret_cast<uint32_t *>(lists + (size_t)g * lb) + 2 * k; };  // [2][k]
    auto ckeys = [&](int g) { return reinterpret_cast<float *>(cands + (size_t)g * CAND * 8); };
    auto cids = [&](int g) { return reinterpret_cast<uint32_t *>(cands + (size_t)g * CAND * 8) + CAND; };

    const int n_items = *p.n_items_ptr;
    int it = blockIdx.x;
    if (it >= n_items) return;
    if (tid == 0) {
        mbar_init(&bar[0], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const uint32_t tbytes = (uint32_t)m * 64u;
    // thread 0: the tables of the group of item `item` starting at slot g0 (every thread is done with the previous group's)
    auto issue = [&](const IvfGemmItem &item, uint32_t g0) {
        const uint32_t gn = min((uint32_t)G, item.q_count - g0);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        mbar_arrive_expect_tx(&bar[0], gn * tbytes);
        for (uint32_t g = 0; g < gn; g++)
            bulk_load(tables + (size_t)g * tbl_words, p.lut + (size_t)(p.sorted_pair[item.q_begin + g0 + g] / (uint32_t)p.nprobe) * tbl_words, tbytes,
                      &bar[0]);
    };
    if (tid == 0) issue(p.items[it], 0);
    uint32_t parity = 0;
    for (; it < n_items; it += gridDim.x) {
        const IvfGemmItem item = p.items[it];
        for (uint32_t g0 = 0; g0 < item.q_count; g0 += G, parity ^= 1) {
            const int gn = (int)min((uint32_t)G, item.q_count - g0);
            if (tid < gn) {
                const uint32_t pair = item.q_begin + g0 + tid;
                QState st{};
                st.thr_key = FLT_MAX;
                st.last_pub = FLT_MAX;
                st.q = p.query_bound ? p.sorted_pair[pair] / (uint32_t)p.nprobe : NO_QUERY;
                st.pc = p.query_bound ? p.pair_const[pair] : 0.f;
                qs[tid] = st;
            }
            __syncthreads();
            mbar_wait(&bar[0], parity);
            for (uint32_t j = 0; j < item.page_count; j++) {
                const uint32_t row0 = p.list_pages[item.page_begin + j] * (uint32_t)PAGE;
                const uint32_t valid = min((uint32_t)PAGE, item.row_limit - j * (uint32_t)PAGE);
                const uint32_t row = row0 + tid;
                bool live = false;
                float key[G];
#pragma unroll
                for (int g = 0; g < G; g++) key[g] = FLT_MAX;
                if ((uint32_t)tid < valid) {
                    live = true;
                    if (p.alive) {
                        const uint32_t id = p.row_ids[row];
                        live = (p.alive[id >> 3] >> (id & 7)) & 1;
                    }
                }
                if (live) {
                    // G sums from one pass over the row's codes; each sum keeps two partial sums (low / high nibbles)
                    float acc[G];
#pragma unroll
                    for (int g = 0; g < G; g++) acc[g] = 0.f;
                    const uint4 *cr = reinterpret_cast<const uint4 *>(p.codes + (size_t)row * p.code_bytes);
                    for (int j0 = 0; j0 < m; j0 += 32) {
                        const uint4 w = cr[j0 >> 5];
                        const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
                        const float *Tj = tables + (size_t)j0 * 16;
#pragma unroll
                        for (int g = 0; g < G; g++) {
                            const float *T = Tj + (size_t)g * tbl_words;
                            float s0 = 0.f, s1 = 0.f;
#pragma unroll
                            for (int t = 0; t < 32; t += 2) {
                                const uint32_t b = ww[t >> 3] >> ((t & 7) * 4);
                                if (j0 + t < m) s0 += T[t * 16 + (b & 15u)];
                                if (j0 + t + 1 < m) s1 += T[(t + 1) * 16 + ((b >> 4) & 15u)];
                            }
                            acc[g] += s0 + s1;
                        }
                    }
                    const float bias = p.row_bias ? p.row_bias[row] : 0.f;
#pragma unroll
                    for (int g = 0; g < G; g++) key[g] = fmaf(p.scale_const, acc[g], bias);
                }
                // per query: the bound in this pair's key space (a few ulps loose), the threshold filter, the warp counts
                unsigned bal[G];
                int *wc = wcnt + (j & 1) * MAX_G * 8;
#pragma unroll
                for (int g = 0; g < G; g++) {
                    bool cand = false;
                    if (live && g < gn) {
                        float ext = FLT_MAX;
                        if (qs[g].q != NO_QUERY) {
                            const uint32_t u = __ldcg(p.query_bound + qs[g].q);
                            if (u != 0xffffffffu) {
                                const float gb = bound_decode(u), pc = qs[g].pc;
                                ext = gb - pc;
                                ext += (fabsf(ext) + fabsf(pc) + fabsf(gb)) * 4e-7f;
                            }
                        }
                        cand = key[g] <= ext && better(key[g], row, qs[g].thr_key, qs[g].thr_id);
                    }
                    bal[g] = __ballot_sync(0xffffffffu, cand);
                    if (lane == 0) wc[g * 8 + warp] = __popc(bal[g]);
                }
                __syncthreads();
                // candidate slots by a block-wide prefix count
#pragma unroll
                for (int g = 0; g < G; g++) {
                    if (g < gn) {
                        int before = qs[g].cnt, total = before;
#pragma unroll
                        for (int w = 0; w < THREADS / 32; w++) {
                            const int c = wc[g * 8 + w];
                            before += w < warp ? c : 0;
                            total += c;
                        }
                        if ((bal[g] >> lane) & 1u) {
                            const int pos = before + __popc(bal[g] & ((1u << lane) - 1u));
                            ckeys(g)[pos] = key[g];
                            cids(g)[pos] = row;
                        }
                        if (tid == 0) qs[g].ncnt = total;
                    }
                }
                __syncthreads();   // the candidates and the counts are written
                bool merged = false;
#pragma unroll 1
                for (int g = 0; g < gn; g++) {
                    const int cnt = qs[g].ncnt, n = qs[g].n;
                    if (!(cnt > 0 && (cnt > CAND - PAGE || (n < k && n + cnt >= k) || j + 1 == item.page_count))) {
                        if (tid == 0) qs[g].cnt = cnt;   // next read behind the next page's first barrier
                        continue;
                    }
                    merged = true;
                    const int cur = qs[g].cur;
                    float *ck = ckeys(g);
                    uint32_t *ci = cids(g);
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
                    const float *ak = lkeys(g) + cur * k;
                    const uint32_t *ai = lids(g) + cur * k;
                    float *ok = lkeys(g) + (cur ^ 1) * k;
                    uint32_t *oi = lids(g) + (cur ^ 1) * k;
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
                    const int nn = min(n + mc, k);
                    QState st = qs[g];
                    st.n = nn;
                    st.cur = cur ^ 1;
                    st.cnt = 0;
                    if (nn == k) {
                        st.thr_key = ok[k - 1];
                        st.thr_id = oi[k - 1];
                        // publish: a full list's k-th key bounds the query's k-th key over all its lists
                        if (st.q != NO_QUERY && st.thr_key < st.last_pub) {
                            st.last_pub = st.thr_key;
                            if (tid == 0) atomicMin(p.query_bound + st.q, bound_encode(st.thr_key + st.pc));
                        }
                    }
                    __syncthreads();   // every thread has read this query's state
                    if (tid == 0) qs[g] = st;
                }
                if (merged) __syncthreads();   // the new states are visible before the next page reads them
            }
            __syncthreads();   // the last page's counts are written
            // the (pair, chunk) partial lists of the group: pool rows mapped to row ids, worst kept key aside
            for (int g = 0; g < gn; g++) {
                const QState st = qs[g];
                const uint32_t pair = item.q_begin + g0 + g;
                const size_t part = (size_t)p.pair_part_base[pair] + item.chunk;
                const float *fk = lkeys(g) + st.cur * k;
                const uint32_t *fi = lids(g) + st.cur * k;
                for (int e = tid; e < k; e += THREADS) {
                    const bool have = e < st.n;
                    p.part_keys[part * k + e] = have ? fk[e] : FLT_MAX;
                    p.part_ids[part * k + e] = have ? p.row_ids[fi[e]] : kNoId;
                }
                if (tid == 0) p.part_worst[part] = st.n == k ? st.thr_key : FLT_MAX;
            }
            __syncthreads();   // the tables, the lists, the candidates and the states are free again
            if (tid == 0) {
                if (g0 + G < item.q_count) issue(item, g0 + G);
                else if (it + (int)gridDim.x < n_items) issue(p.items[it + gridDim.x], 0);
            }
        }
    }
}

template <int G>
cudaError_t launch_group(const IvfGemmParams &p, int grid, cudaStream_t s) {
    const int smem = smem_bytes(p.m, p.k, G);
    cudaError_t e = cudaFuncSetAttribute(ivf_pq4_topk_kernel<G>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    int per_sm = 1;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ivf_pq4_topk_kernel<G>, THREADS, smem);
    if (e != cudaSuccess) return e;
    ivf_pq4_topk_kernel<G><<<grid * std::max(1, per_sm), THREADS, smem, s>>>(p);
    g_launches++;
    return cudaGetLastError();
}

}  // namespace pq4

int ivf_pq4_max_m() { return pq4::MAX_M; }

bool ivf_pq4_fits(int m) { return m >= 1 && m <= pq4::MAX_M && pq4::smem_bytes(m, 1024, 1) <= gemm::SMEM_LIMIT; }

cudaError_t launch_pq4_lut(const float *queries, int64_t nq, int d_pad, const float *codebook, int m, int dsub, float *lut_out, cudaStream_t s) {
    if (nq <= 0) return cudaSuccess;
    pq4::pq4_lut_kernel<<<dim3((unsigned)ceil_div(nq, pq4::LUT_QB), (unsigned)ceil_div(m, 16)), 256, 0, s>>>(queries, nq, d_pad, codebook, m, dsub,
                                                                                                            lut_out);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t launch_ivf_pq4_topk(const IvfGemmParams &p, int grid, cudaStream_t s, const char **err_detail) {
    *err_detail = nullptr;
    if (!p.lut || !p.sorted_pair || p.nprobe < 1 || p.code_bytes % 16 || p.code_bytes < (p.m + 1) / 2 || p.k < 1 || p.k > 1024 || !ivf_pq4_fits(p.m)) {
        *err_detail = "4-bit PQ table look-up scan: table, sorted pairs, 16-byte code rows, 1 <= k <= 1024 and M <= 2048 needed";
        return cudaErrorInvalidValue;
    }
    switch (pq4::group_size(p.m, p.k)) {
        case 8: return pq4::launch_group<8>(p, grid, s);
        case 4: return pq4::launch_group<4>(p, grid, s);
        case 2: return pq4::launch_group<2>(p, grid, s);
        default: return pq4::launch_group<1>(p, grid, s);
    }
}

}  // namespace b200
