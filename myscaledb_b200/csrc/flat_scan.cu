// flat_scan.cu -- memory-bound FLAT scan kernels (K1/K3/K4) and the k-way merge (K7).
//
// K1/K3  flat_scan_kernel : squared-L2 / inner-product / cosine of <= 8 queries per pass
//        against a row-major corpus (fp32 or bf16) with 128-bit streaming loads,
//        sub-warp groups per row, warp-shuffle reduction and a fused per-warp top-k.
//        Replaces faiss::knn_L2sqr / knn_inner_product as called from
//        tryBruteForceSearch (reference: VectorIndex/Common/BruteForceSearch.h:77-88).
//        HBM-bound: algorithmic bytes = n * d * sizeof(elem) per pass.
// K4     binary_scan_kernel : Hamming / Jaccard via __popc (BruteForceSearch.h:96-105).
// K7     topk_merge_kernel : merges P sorted lists per query; replaces the running merge
//        in searchWrapper (MergeTreeVSManager.cpp:1652-1678) and the multimap merge in
//        getTotalTopSearchResultImpl (MergeTreeBaseSearchManager.cpp:207-299).
#include <algorithm>

#include "common.cuh"
#include "kernels.h"

namespace b200 {

constexpr int kScanThreads = 256;
constexpr int kScanWarps = kScanThreads / 32;

// ------------------------------------------------------------------------------------
template <bool BF16>
struct ChunkTraits;
template <>
struct ChunkTraits<false> {
    static constexpr int kElems = 4;
    __device__ static __forceinline__ void unpack(const uint4 &r, float (&f)[4]) {
        f[0] = __uint_as_float(r.x);
        f[1] = __uint_as_float(r.y);
        f[2] = __uint_as_float(r.z);
        f[3] = __uint_as_float(r.w);
    }
};
template <>
struct ChunkTraits<true> {
    static constexpr int kElems = 8;
    __device__ static __forceinline__ void unpack(const uint4 &r, float (&f)[8]) {
        f[0] = __uint_as_float(r.x << 16);
        f[1] = __uint_as_float(r.x & 0xffff0000u);
        f[2] = __uint_as_float(r.y << 16);
        f[3] = __uint_as_float(r.y & 0xffff0000u);
        f[4] = __uint_as_float(r.z << 16);
        f[5] = __uint_as_float(r.z & 0xffff0000u);
        f[6] = __uint_as_float(r.w << 16);
        f[7] = __uint_as_float(r.w & 0xffff0000u);
    }
};

// QT queries per pass; U rows x CU 16-byte chunks per lane are loaded BEFORE any arithmetic, so
// every lane keeps U * CU independent 128-bit loads in flight (issuing only U left the scan well short of the HBM peak at
// the low occupancy this kernel runs at).
// L2 = squared-L2 vs inner product (cosine = inner product scaled by the stored inverse row norm).
// candidate read of the fused tail: partial lists in global memory written by other blocks (L2, .cg) or staged in shared memory
template <typename T>
__device__ __forceinline__ T ld_cand(const T *p, bool staged) { return staged ? *p : __ldcg(p); }

template <int QT, int U, int CU, bool L2, bool BF16>
__global__ void __launch_bounds__(kScanThreads, 2) flat_scan_kernel(const ScanParams p) {
    using CT = ChunkTraits<BF16>;
    constexpr int E = CT::kElems;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float *qs = reinterpret_cast<float *>(smem_raw);                        // [QT][d_pad]
    float *lk = qs + (size_t)QT * p.d_pad;                                   // [warps][QT][k]
    uint32_t *li = reinterpret_cast<uint32_t *>(lk + (size_t)kScanWarps * QT * p.k);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t q0 = (int64_t)blockIdx.y * QT;
    const int nq_here = (int)min((int64_t)QT, p.nq - q0);

    // stage queries (zero-padded) in shared memory.  bf16 rows consume 8 query floats per 16-byte chunk: they are
    // stored as two float4 planes ([chunk][0..3] and [chunk][4..7]) so that consecutive lanes read consecutive
    // 16-byte words (a single 32-byte-strided array costs a 2-way bank conflict on every LDS.128).
    for (int i = threadIdx.x; i < QT * p.d_pad; i += kScanThreads) {
        const int q = i / p.d_pad, j = i - q * p.d_pad;
        const float v = (q < nq_here) ? (p.fused ? (j < p.q_dim ? (p.q_inline ? p.qinline[(q0 + q) * p.q_dim + j] : p.queries[(q0 + q) * p.q_dim + j]) : 0.f)
                                                  : p.queries[(q0 + q) * p.d_pad + j])
                                      : 0.f;
        if (E == 8) {
            const int c = j >> 3, e = j & 7;
            qs[q * p.d_pad + (e >> 2) * (p.d_pad >> 1) + c * 4 + (e & 3)] = v;
        } else {
            qs[i] = v;
        }
    }
    WarpTopK lists[QT];
#pragma unroll
    for (int q = 0; q < QT; q++)
    {
        lists[q].init(lk + ((size_t)warp * QT + q) * p.k, li + ((size_t)warp * QT + q) * p.k, p.k);
        for (int j = lane; j < p.k; j += 32) lists[q].keys[j] = FLT_MAX;  // sentinel for the block merge
    }
    __syncthreads();
    if (p.fused && p.cosine) {
        // VectorDataset::normalize on the staged queries (VectorDataset.h:99-117): one warp per query.  The sum visits the
        // elements in their natural order (not the two-plane order of bf16 rows), as normalize_rows_f32_kernel does, so that
        // the fused and the staged form give the same bits.
        for (int q = warp; q < nq_here; q += kScanWarps) {
            float ss = 0.f;
            for (int j = lane; j < p.d_pad; j += 32) {
                const float v = qs[q * p.d_pad + (E == 8 ? ((j & 7) >> 2) * (p.d_pad >> 1) + (j >> 3) * 4 + (j & 3) : j)];
                ss = fmaf(v, v, ss);
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
            if (!(ss < FLT_EPSILON)) {
                const float nrm = sqrtf(ss);
                for (int j = lane; j < p.d_pad; j += 32) qs[q * p.d_pad + j] = qs[q * p.d_pad + j] / nrm;
            }
        }
        __syncthreads();
    }

    const int G = p.group;           // lanes per row (power of two)
    const int R = 32 / G;            // rows per warp step
    const int sub = lane / G, gl = lane - sub * G;
    const int64_t total_groups = (int64_t)gridDim.x * kScanWarps * R;
    const int64_t gidx = ((int64_t)blockIdx.x * kScanWarps + warp) * R + sub;
    const int chunks = p.d_pad / E;
    const unsigned char *base = reinterpret_cast<const unsigned char *>(p.corpus);

    for (int64_t it = 0;; it++) {
        // a group owns U CONSECUTIVE rows per step (one contiguous U * row_bytes span: DRAM-page friendly)
        const int64_t row0 = (gidx + it * total_groups) * U;
        // warp-uniform exit: the smallest row of this step over the warp is for sub == 0
        if (row0 - (int64_t)sub * U >= p.n) break;
        float acc[U][QT];
        bool valid[U];
        const uint4 *rp[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const int64_t row = row0 + u;
            valid[u] = row < p.n;
            if (valid[u] && p.alive) valid[u] = (p.alive[row >> 3] >> (row & 7)) & 1;
            rp[u] = reinterpret_cast<const uint4 *>(base + (size_t)(valid[u] ? row : 0) * p.row_bytes);
#pragma unroll
            for (int q = 0; q < QT; q++) acc[u][q] = 0.f;
        }
        for (int c0 = gl; c0 < chunks; c0 += G * CU) {
            uint4 raw[U][CU];
#pragma unroll
            for (int j = 0; j < CU; j++)
#pragma unroll
                for (int u = 0; u < U; u++)
                    raw[u][j] = (valid[u] && c0 + j * G < chunks) ? ldg_stream(rp[u] + c0 + j * G) : make_uint4(0, 0, 0, 0);
#pragma unroll
            for (int j = 0; j < CU; j++) {
                const int c = c0 + j * G;
                if (c < chunks) {
                    float y[U][E];
#pragma unroll
                    for (int u = 0; u < U; u++) CT::unpack(raw[u][j], y[u]);
#pragma unroll
                    for (int q = 0; q < QT; q++) {
                        float x[E];
#pragma unroll
                        for (int e4 = 0; e4 < E / 4; e4++) {
                            const float4 t = *reinterpret_cast<const float4 *>(
                                qs + (size_t)q * p.d_pad + (E == 8 ? (size_t)e4 * (p.d_pad >> 1) + (size_t)c * 4 : (size_t)c * 4));
                            x[e4 * 4 + 0] = t.x;
                            x[e4 * 4 + 1] = t.y;
                            x[e4 * 4 + 2] = t.z;
                            x[e4 * 4 + 3] = t.w;
                        }
#pragma unroll
                        for (int u = 0; u < U; u++) {
#pragma unroll
                            for (int e = 0; e < E; e++) {
                                if (L2) {
                                    const float t = x[e] - y[u][e];
                                    acc[u][q] = fmaf(t, t, acc[u][q]);
                                } else {
                                    acc[u][q] = fmaf(x[e], y[u][e], acc[u][q]);
                                }
                            }
                        }
                    }
                }
            }
        }
        // reduce over the G lanes of each group
        for (int o = G >> 1; o > 0; o >>= 1) {
#pragma unroll
            for (int u = 0; u < U; u++)
#pragma unroll
                for (int q = 0; q < QT; q++) acc[u][q] += __shfl_xor_sync(0xffffffffu, acc[u][q], o);
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
            const int64_t row = row0 + u;
            float scale = 1.f;
            if (!L2) scale = (p.row_scale && valid[u]) ? p.row_scale[row] : -1.f;
#pragma unroll
            for (int q = 0; q < QT; q++) {
                const float key = L2 ? acc[u][q] : acc[u][q] * scale;
                const bool cand = valid[u] && gl == 0 && q < nq_here && lists[q].passes(key, (uint32_t)row);
                unsigned m = __ballot_sync(0xffffffffu, cand);
                while (m) {
                    const int src = __ffs(m) - 1;
                    m &= m - 1;
                    const float ck = __shfl_sync(0xffffffffu, key, src);
                    const uint32_t ci = __shfl_sync(0xffffffffu, (uint32_t)row, src);
                    lists[q].insert(ck, ci);
                }
            }
        }
    }
    __syncthreads();
    // block merge: the 8 warp lists of every query -> this block's partial list (slots beyond a warp's n hold FLT_MAX)
    for (int q = 0; q < nq_here; q++)
        block_rank_merge(lk + (size_t)q * p.k, li + (size_t)q * p.k, kScanWarps, QT * p.k, p.k,
                         p.part_keys + ((q0 + q) * (int64_t)gridDim.x + blockIdx.x) * p.k,
                         p.part_ids + ((q0 + q) * (int64_t)gridDim.x + blockIdx.x) * p.k);
    if (!p.fused) return;
    // ---- fused form: the last block of this query tile merges the gridDim.x partial lists of each of its queries
    __shared__ unsigned int s_ticket;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_ticket = atomicAdd(&p.tickets[blockIdx.y], 1u);
    __syncthreads();
    if (s_ticket != gridDim.x - 1) return;
    __threadfence();
    // the staging area is free now: [warps][k] keys + ids, merged list behind it (launch reserves (warps + 1) * k * 8 bytes)
    float *mk = reinterpret_cast<float *>(smem_raw);
    uint32_t *mi = reinterpret_cast<uint32_t *>(mk + (size_t)kScanWarps * p.k);
    float *fk = reinterpret_cast<float *>(mi + (size_t)kScanWarps * p.k);
    uint32_t *fi = reinterpret_cast<uint32_t *>(fk + p.k);
    for (int q = 0; q < nq_here; q++) {
        __syncthreads();
        WarpTopK list;
        list.init(mk + (size_t)warp * p.k, mi + (size_t)warp * p.k, p.k);
        for (int j = lane; j < p.k; j += 32) list.keys[j] = FLT_MAX;
        __syncwarp();
        const float *pkeys = p.part_keys + (q0 + q) * (int64_t)gridDim.x * p.k;
        const uint32_t *pids = p.part_ids + (q0 + q) * (int64_t)gridDim.x * p.k;
        const int64_t ncand = (int64_t)gridDim.x * p.k;
        const bool staged = p.stage_cap >= ncand;
        if (staged) {
            // Staged form.  The tail is ONE block and latency-bound (the SMs are idle for most of it): every
            // L2 round trip on its critical path counts.  All candidates come in with independent loads, 4 per thread in flight;
            // the bound, the survivor compaction and the warp lists then work from shared memory.
            float *sk = reinterpret_cast<float *>(fi + p.k);
            uint32_t *si = reinterpret_cast<uint32_t *>(sk + p.stage_cap);
            for (int64_t c0 = threadIdx.x; c0 < ncand; c0 += kScanThreads * 4) {
                float kk[4];
                uint32_t ii[4];
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const int64_t c = c0 + (int64_t)u * kScanThreads;
                    kk[u] = c < ncand ? __ldcg(pkeys + c) : FLT_MAX;
                    ii[u] = c < ncand ? __ldcg(pids + c) : kNoId;
                }
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const int64_t c = c0 + (int64_t)u * kScanThreads;
                    if (c < ncand) {
                        sk[c] = kk[u];
                        si[c] = ii[u];
                    }
                }
            }
            __syncthreads();
            pkeys = sk;
            pids = si;
        }
        __shared__ __align__(16) float cand_k[1024];
        __shared__ uint32_t cand_i[1024];
        __shared__ int cand_n;
        {
            __shared__ float bound_s[kScanWarps];
            __shared__ float bound2_s;
            float b = FLT_MAX;
            if (staged && (int)gridDim.x >= p.k) {
                // Bound = the k-th smallest of the blocks' BEST keys: at least k candidates (those minima) are <= it, so it bounds
                // the global k-th key -- and it is tight even when every block saw only a few rows (cfg 1: 34 rows per block; a
                // block's own k-th key would let ~30 % of all candidates through).  The minima are gathered into a compact array
                // (reusing the survivor buffer) so that the rank count is one LDS.128 per four comparisons.
                float *mins = cand_k;   // gridDim.x <= 8192 / k <= 1024 when k >= 8; guarded below
                // any k candidates bound the k-th key: the minima of the first 256 blocks are enough (one round of the rank count)
                const int nb = min((int)gridDim.x, kScanThreads);
                const bool fits = true;
                if (fits) {
                    for (int l = threadIdx.x; l < ((nb + 3) & ~3); l += kScanThreads)
                        mins[l] = (l < nb && pids[(int64_t)l * p.k] != kNoId) ? pkeys[(int64_t)l * p.k] : FLT_MAX;
                    if (threadIdx.x == 0) bound2_s = FLT_MAX;
                    __syncthreads();
                    for (int l = threadIdx.x; l < nb; l += kScanThreads) {
                        const float m = mins[l];
                        int rank = 0;
#pragma unroll 8
                        for (int o = 0; o < nb; o += 4) {
                            const float4 v = *reinterpret_cast<const float4 *>(mins + o);
                            rank += (v.x < m || (v.x == m && o < l)) ? 1 : 0;
                            rank += (v.y < m || (v.y == m && o + 1 < l)) ? 1 : 0;
                            rank += (v.z < m || (v.z == m && o + 2 < l)) ? 1 : 0;
                            rank += (v.w < m || (v.w == m && o + 3 < l)) ? 1 : 0;
                        }
                        if (rank == p.k - 1) bound2_s = m;
                    }
                    __syncthreads();
                    b = bound2_s;
                }
            }
            if (!(b < FLT_MAX)) {
                // every block's list is sorted and complete: the smallest k-th key over the blocks also bounds the global k-th key
                for (int l = threadIdx.x; l < (int)gridDim.x; l += kScanThreads)
                    if (ld_cand(pids + (int64_t)l * p.k + (p.k - 1), staged) != kNoId) b = fminf(b, ld_cand(pkeys + (int64_t)l * p.k + (p.k - 1), staged));
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) b = fminf(b, __shfl_xor_sync(0xffffffffu, b, o));
                if (lane == 0) bound_s[warp] = b;
                __syncthreads();
                b = bound_s[0];
#pragma unroll
                for (int w = 1; w < kScanWarps; w++) b = fminf(b, bound_s[w]);
            }
            if (b < FLT_MAX) {
                list.thr_key = b;
                list.thr_id = kNoId;
            }
            __syncthreads();
        }
        // Survivors of the bound are few (~k): every thread first sweeps its share of the candidates with independent loads
        // (no vote between them, so the L2 latencies overlap) and appends survivors to a compact shared array; only those go
        // through the warp lists.  (Voting after every load would put 12 dependent L2 round trips on the critical path.)
        if (threadIdx.x == 0) cand_n = 0;
        __syncthreads();
        const float bound_key = list.thr_key;
        for (int64_t c = threadIdx.x; c < ncand; c += kScanThreads) {
            const uint32_t id = ld_cand(pids + c, staged);
            const float key = ld_cand(pkeys + c, staged);
            if (id != kNoId && key <= bound_key) {
                const int pos = atomicAdd(&cand_n, 1);
                if (pos < 1024) {
                    cand_k[pos] = key;
                    cand_i[pos] = id;
                }
            }
        }
        __syncthreads();
        const int n_surv = cand_n;
        bool ranked = false;
        if (n_surv <= kScanThreads) {
            // few survivors (the usual case, ~k): rank each among the others and write the result in order -- no warp lists, no merge
            for (int j = threadIdx.x; j < p.k; j += kScanThreads) {
                fk[j] = FLT_MAX;
                fi[j] = kNoId;
            }
            __syncthreads();
            if ((int)threadIdx.x < n_surv) {
                const float key = cand_k[threadIdx.x];
                const uint32_t id = cand_i[threadIdx.x];
                int rank = 0;
                for (int o = 0; o < n_surv; o++) rank += better(cand_k[o], cand_i[o], key, id) ? 1 : 0;
                if (rank < p.k) {
                    fk[rank] = key;
                    fi[rank] = id;
                }
            }
            ranked = true;
        } else if (n_surv <= 1024) {
            for (int c0 = warp * 32; c0 < n_surv; c0 += kScanThreads) {
                const int c = c0 + lane;
                const float key = c < n_surv ? cand_k[c] : FLT_MAX;
                const uint32_t id = c < n_surv ? cand_i[c] : kNoId;
                unsigned m = __ballot_sync(0xffffffffu, c < n_surv && list.passes(key, id));
                while (m) {
                    const int src = __ffs(m) - 1;
                    m &= m - 1;
                    list.insert(__shfl_sync(0xffffffffu, key, src), __shfl_sync(0xffffffffu, id, src));
                }
            }
        } else {
            // more survivors than the compact array holds (huge k or many ties): the plain sweep
            for (int64_t c0 = (int64_t)warp * 32; c0 < ncand; c0 += kScanThreads) {
                const int64_t c = c0 + lane;
                float key = FLT_MAX;
                uint32_t id = kNoId;
                bool cand = false;
                if (c < ncand) {
                    key = ld_cand(pkeys + c, staged);
                    id = ld_cand(pids + c, staged);
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
        if (!ranked) block_rank_merge(mk, mi, kScanWarps, p.k, p.k, fk, fi);
        __syncthreads();
        for (int j = threadIdx.x; j < p.k; j += kScanThreads) {
            float dis;
            int64_t id;
            if (fi[j] != kNoId) {
                const float key = fk[j];
                id = (int64_t)fi[j] + p.id_offset;
                dis = p.out_mode == kOutKey ? key : p.out_mode == kOutNeg ? -key : 1.f + key;
                if (p.ip_min_quirk && !(dis > FLT_MIN)) {
                    id = -1;
                    dis = FLT_MIN;
                }
            } else {
                id = -1;
                dis = (p.out_mode == kOutNeg) ? -FLT_MAX : FLT_MAX;
                if (p.ip_min_quirk) dis = FLT_MIN;
            }
            p.out_dis[(q0 + q) * p.k + j] = dis;
            p.out_ids[(q0 + q) * p.k + j] = id;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        p.tickets[blockIdx.y] = 0;            // ready for the next call
        __threadfence_system();               // results (mapped host memory) before the flag
        const unsigned int t = atomicAdd(p.tiles_done, 1u);
        if (t == gridDim.y - 1) {
            *p.tiles_done = 0;
            if (p.done_flag) {
                __threadfence_system();
                *p.done_flag = p.done_value;
            }
        }
    }
}

// ------------------------------------------------------------------------------------
// K4: binary vectors.  One thread per row, grid.y = query.
// ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kScanThreads) binary_scan_kernel(const BinaryScanParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint8_t *qb = smem_raw;                                                         // [nbytes] (padded to 16)
    float *lk = reinterpret_cast<float *>(smem_raw + round_up(p.nbytes, 16));       // [warps][k]
    uint32_t *li = reinterpret_cast<uint32_t *>(lk + (size_t)kScanWarps * p.k);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t q = blockIdx.y;
    for (int i = threadIdx.x; i < p.nbytes; i += kScanThreads) qb[i] = p.queries[q * p.nbytes + i];
    WarpTopK list;
    list.init(lk + (size_t)warp * p.k, li + (size_t)warp * p.k, p.k);
    for (int j = lane; j < p.k; j += 32) list.keys[j] = FLT_MAX;
    __syncthreads();
    const int64_t stride = (int64_t)gridDim.x * kScanThreads;
    for (int64_t row0 = (int64_t)blockIdx.x * kScanThreads + warp * 32; row0 < p.n; row0 += stride) {
        const int64_t row = row0 + lane;
        bool valid = row < p.n;
        if (valid && p.alive) valid = (p.alive[row >> 3] >> (row & 7)) & 1;
        float key = FLT_MAX;
        if (valid) {
            const uint8_t *y = p.corpus + (size_t)row * p.nbytes;
            int x_or = 0, x_and = 0, x_xor = 0;
            if ((p.nbytes & 3) == 0) {
                const uint32_t *yw = reinterpret_cast<const uint32_t *>(y);
                const uint32_t *qw = reinterpret_cast<const uint32_t *>(qb);
                for (int j = 0; j < p.nbytes / 4; j++) {
                    const uint32_t a = qw[j], b = yw[j];
                    x_xor += __popc(a ^ b);
                    x_and += __popc(a & b);
                    x_or += __popc(a | b);
                }
            } else {
                for (int j = 0; j < p.nbytes; j++) {
                    const uint32_t a = qb[j], b = y[j];
                    x_xor += __popc(a ^ b);
                    x_and += __popc(a & b);
                    x_or += __popc(a | b);
                }
            }
            key = p.jaccard ? (x_or == 0 ? 0.f : (float)(x_or - x_and) / (float)x_or) : (float)x_xor;
        }
        const bool cand = valid && list.passes(key, (uint32_t)row);
        unsigned m = __ballot_sync(0xffffffffu, cand);
        while (m) {
            const int src = __ffs(m) - 1;
            m &= m - 1;
            list.insert(__shfl_sync(0xffffffffu, key, src), __shfl_sync(0xffffffffu, (uint32_t)row, src));
        }
    }
    __syncthreads();
    block_rank_merge(lk, li, kScanWarps, p.k, p.k, p.part_keys + (q * (int64_t)gridDim.x + blockIdx.x) * p.k,
                     p.part_ids + (q * (int64_t)gridDim.x + blockIdx.x) * p.k);
}

// ------------------------------------------------------------------------------------
// K7: merge.  One block per query; 8 warps filter slices of the candidate set into warp
// lists, warp 0 merges them and writes the final, converted result.
// ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kScanThreads) topk_merge_kernel(const MergeParams p) {
    using IdT = uint32_t;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float *lk = reinterpret_cast<float *>(smem_raw);
    uint32_t *li = reinterpret_cast<uint32_t *>(lk + (size_t)kScanWarps * p.k);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t q = blockIdx.x;
    WarpTopK list;
    list.init(lk + (size_t)warp * p.k, li + (size_t)warp * p.k, p.k);
    for (int j = lane; j < p.k; j += 32) list.keys[j] = FLT_MAX;
    __syncwarp();
    const float *keys = reinterpret_cast<const float *>(p.in_keys);
    const IdT *ids = reinterpret_cast<const IdT *>(p.in_ids);
    const int64_t ncand = (int64_t)p.n_lists * p.k_in;
    // Pre-filter.  Every input list is sorted best-first and holds its partition's full top-k_in, so with k_in >= k
    // the k-th entry of ANY list bounds the global k-th key from above: candidates beyond the smallest such bound
    // cannot be in the result.  Typically ~2k of the n_lists * k candidates survive, which keeps the warp-list
    // inserts (O(k / 32) each) off the critical path for k in the hundreds (IVF: 32 lists x 160).
    if (p.k_in >= p.k) {
        __shared__ float bound_s[kScanWarps];
        float b = FLT_MAX;
        for (int l = threadIdx.x; l < p.n_lists; l += kScanThreads) {
            const int64_t off = (int64_t)l * p.list_stride + q * p.q_stride + (p.k - 1);
            const int64_t ioff = (int64_t)l * (p.id_list_stride ? p.id_list_stride : p.list_stride) + q * p.q_stride + (p.k - 1);
            float v = keys[off];
            if ((uint32_t)ids[ioff] == kNoId) v = FLT_MAX;
            b = fminf(b, v);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) b = fminf(b, __shfl_xor_sync(0xffffffffu, b, o));
        if (lane == 0) bound_s[warp] = b;
        __syncthreads();
        b = bound_s[0];
#pragma unroll
        for (int w = 1; w < kScanWarps; w++) b = fminf(b, bound_s[w]);
        if (b < FLT_MAX) {
            list.thr_key = b;       // keys equal to the bound still pass (largest id as the tie-break)
            list.thr_id = kNoId;
        }
    }
    for (int64_t c0 = (int64_t)warp * 32; c0 < ncand; c0 += kScanThreads) {
        const int64_t c = c0 + lane;
        float key = FLT_MAX;
        uint32_t id = kNoId;
        bool cand = false;
        if (c < ncand) {
            const int64_t l = c / p.k_in, j = c - l * p.k_in;
            const int64_t off = l * p.list_stride + q * p.q_stride + j;
            const int64_t ioff = l * (p.id_list_stride ? p.id_list_stride : p.list_stride) + q * p.q_stride + j;
            id = (uint32_t)ids[ioff];
            key = keys[off];
            cand = id != kNoId && list.passes(key, id);
        }
        unsigned m = __ballot_sync(0xffffffffu, cand);
        while (m) {
            const int src = __ffs(m) - 1;
            m &= m - 1;
            list.insert(__shfl_sync(0xffffffffu, key, src), __shfl_sync(0xffffffffu, id, src));
        }
    }
    __syncthreads();
    float *fk = lk + (size_t)kScanWarps * p.k * 2;  // merged list, behind the warp lists (keys + ids)
    uint32_t *fi = reinterpret_cast<uint32_t *>(fk + p.k);
    block_rank_merge(lk, li, kScanWarps, p.k, p.k, fk, fi);
    __syncthreads();
    {
        for (int j = threadIdx.x; j < p.k; j += kScanThreads) {
            float dis;
            int64_t id;
            if (fi[j] != kNoId) {
                const float key = fk[j];
                id = (int64_t)fi[j] + p.id_offset;
                switch (p.out_mode) {
                    case kOutKey: dis = key; break;
                    case kOutNeg: dis = -key; break;
                    case kOutOnePlus: dis = 1.f + key; break;
                    case kOutCosQ: dis = 1.f - key * p.q_add[q]; break;  // key = -ip/||y||, q_add = -1/||q||
                    default: dis = fmaxf(key + p.q_add[q], 0.f); break;  // kOutAddQ
                }
                if (p.ip_min_quirk && !(dis > FLT_MIN)) {
                    // vectorScanWithoutIndex IP init = numeric_limits<float>::min() (smallest positive)
                    id = -1;
                    dis = FLT_MIN;
                }
            } else {
                id = -1;
                dis = (p.out_mode == kOutNeg) ? -FLT_MAX : FLT_MAX;
                if (p.ip_min_quirk) dis = FLT_MIN;
            }
            p.out_dis[q * p.k + j] = dis;
            p.out_ids[q * p.k + j] = id;
        }
    }
}


// ------------------------------------------------------------------------------------
// K7 (external form): merge of per-part / per-GPU lists that carry 64-bit ids.  Entries are ordered by
// (key, order word): tie_mode 0 -> the 64-bit id itself (contract: better score, then smaller id);
// tie_mode 1 -> the insertion sequence l * k_in + j of std::multimap::emplace in
// getTotalTopSearchResultImpl (MergeTreeBaseSearchManager.cpp:207-299): ascending walks give the
// earlier-inserted equal key first, the reverse walk (IP / BM25) the later-inserted one (:271).
// ------------------------------------------------------------------------------------
constexpr uint64_t kSeqFlip = 0x7fffffffffffffffull;

__global__ void __launch_bounds__(kScanThreads) topk_merge_ext_kernel(const MergeParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint64_t *li = reinterpret_cast<uint64_t *>(smem_raw);                       // [warps + 1][k] order words
    float *lk = reinterpret_cast<float *>(li + (size_t)(kScanWarps + 1) * p.k);  // [warps + 1][k] keys
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t q = blockIdx.x;
    WarpTopKT<uint64_t> list;
    list.init(lk + (size_t)warp * p.k, li + (size_t)warp * p.k, p.k);
    for (int j = lane; j < p.k; j += 32) list.keys[j] = FLT_MAX;
    __syncwarp();
    const float *keys = reinterpret_cast<const float *>(p.in_keys);
    const int64_t *ids = reinterpret_cast<const int64_t *>(p.in_ids);
    const int64_t id_stride = p.id_list_stride ? p.id_list_stride : p.list_stride;
    const int64_t ncand = (int64_t)p.n_lists * p.k_in;
    if (p.k_in >= p.k) {  // same bound as the internal merge: the k-th entry of any full sorted list
        __shared__ float bound_s[kScanWarps];
        float b = FLT_MAX;
        for (int l = threadIdx.x; l < p.n_lists; l += kScanThreads) {
            const float v = keys[(int64_t)l * p.list_stride + q * p.q_stride + (p.k - 1)];
            const bool have = ids[(int64_t)l * id_stride + q * p.q_stride + (p.k - 1)] >= 0;
            b = fminf(b, have ? (p.descending ? -v : v) : FLT_MAX);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) b = fminf(b, __shfl_xor_sync(0xffffffffu, b, o));
        if (lane == 0) bound_s[warp] = b;
        __syncthreads();
        b = bound_s[0];
#pragma unroll
        for (int w = 1; w < kScanWarps; w++) b = fminf(b, bound_s[w]);
        if (b < FLT_MAX) {
            list.thr_key = b;
            list.thr_id = kNoId64;
        }
    }
    for (int64_t c0 = (int64_t)warp * 32; c0 < ncand; c0 += kScanThreads) {
        const int64_t c = c0 + lane;
        float key = FLT_MAX;
        uint64_t ord = kNoId64;
        bool cand = false;
        if (c < ncand) {
            const int64_t l = c / p.k_in, j = c - l * p.k_in;
            const int64_t full = ids[l * id_stride + q * p.q_stride + j];
            if (full >= 0) {
                const float v = keys[l * p.list_stride + q * p.q_stride + j];
                key = p.descending ? -v : v;
                ord = p.tie_mode == 0 ? (uint64_t)full : (p.descending ? kSeqFlip - (uint64_t)c : (uint64_t)c);
                cand = list.passes(key, ord);
            }
        }
        unsigned m = __ballot_sync(0xffffffffu, cand);
        while (m) {
            const int src = __ffs(m) - 1;
            m &= m - 1;
            list.insert(__shfl_sync(0xffffffffu, key, src), __shfl_sync(0xffffffffu, ord, src));
        }
    }
    __syncthreads();
    float *fk = lk + (size_t)kScanWarps * p.k;
    uint64_t *fi = li + (size_t)kScanWarps * p.k;
    block_rank_merge(lk, li, kScanWarps, p.k, p.k, fk, fi);
    __syncthreads();
    for (int j = threadIdx.x; j < p.k; j += kScanThreads) {
        float dis = p.descending ? -FLT_MAX : FLT_MAX;
        int64_t id = -1;
        int32_t src_list = -1;
        if (fi[j] != kNoId64) {
            dis = p.descending ? -fk[j] : fk[j];
            if (p.tie_mode == 0) {
                id = (int64_t)fi[j];
            } else {
                const int64_t c = (int64_t)(p.descending ? kSeqFlip - fi[j] : fi[j]);
                const int64_t l = c / p.k_in, jj = c - l * p.k_in;
                id = ids[l * id_stride + q * p.q_stride + jj];
                src_list = (int32_t)l;
            }
        }
        p.out_dis[q * p.k + j] = dis;
        p.out_ids[q * p.k + j] = id;
        if (p.out_list) p.out_list[q * p.k + j] = src_list;
    }
}

// ------------------------------------------------------------------------------------
// Exact L2 of the winners.  The tensor-core paths rank by ||y||^2 - 2 x.y (+ ||x||^2), faiss' BLAS form
// (BruteForceSearch.h:77-88 for nx >= 20); for data far from the origin the expansion cancels and the ~1e-5 relative
// error of the product (3xTF32, bf16 operands) grows to ~2e-4 of the distance (for example 768-d clusters at |y|^2 = 840,
// d^2 = 115).  The k winners of every query are therefore re-scored with the direct sum of squared differences in fp32
// (one warp per winner, the same arithmetic as the scan kernel) and re-ordered by (distance, id).  One CTA per query.
// ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) rescore_l2_kernel(const void *corpus, int bf16, int64_t row_bytes, int d_pad, const float *queries,
                                                         int64_t id_offset, int k, float *dis, int64_t *ids) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float *sd = reinterpret_cast<float *>(smem_raw);               // [k]
    int64_t *si = reinterpret_cast<int64_t *>(sd + ((k + 1) & ~1));  // [k]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t q = blockIdx.x;
    const float *x = queries + q * d_pad;
    for (int j = warp; j < k; j += 8) {
        const int64_t id = ids[q * k + j];
        float acc = 0.f;
        if (id >= 0) {
            const unsigned char *row = reinterpret_cast<const unsigned char *>(corpus) + (size_t)(id - id_offset) * row_bytes;
            if (bf16) {
                const uint4 *rp = reinterpret_cast<const uint4 *>(row);
                for (int c = lane; c < d_pad / 8; c += 32) {
                    float y[8];
                    ChunkTraits<true>::unpack(rp[c], y);
#pragma unroll
                    for (int e = 0; e < 8; e++) {
                        const float t = x[c * 8 + e] - y[e];
                        acc = fmaf(t, t, acc);
                    }
                }
            } else {
                const float4 *rp = reinterpret_cast<const float4 *>(row);
                for (int c = lane; c < d_pad / 4; c += 32) {
                    const float4 y = rp[c];
                    float t = x[c * 4] - y.x; acc = fmaf(t, t, acc);
                    t = x[c * 4 + 1] - y.y; acc = fmaf(t, t, acc);
                    t = x[c * 4 + 2] - y.z; acc = fmaf(t, t, acc);
                    t = x[c * 4 + 3] - y.w; acc = fmaf(t, t, acc);
                }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        }
        if (lane == 0) {
            sd[j] = id >= 0 ? acc : FLT_MAX;
            si[j] = id >= 0 ? id : INT64_MAX;
        }
    }
    __syncthreads();
    // rank sort by (distance, id); unused slots (id = -1) keep the tail
    for (int j = threadIdx.x; j < k; j += blockDim.x) {
        const float dj = sd[j];
        const int64_t ij = si[j];
        int rank = 0;
        for (int e = 0; e < k; e++) rank += (sd[e] < dj || (sd[e] == dj && (si[e] < ij || (si[e] == ij && e < j)))) ? 1 : 0;
        dis[q * k + rank] = ij == INT64_MAX ? FLT_MAX : dj;
        ids[q * k + rank] = ij == INT64_MAX ? -1 : ij;
    }
}

cudaError_t launch_rescore_l2(const void *corpus, int bf16, int64_t row_bytes, int d_pad, const float *queries, int64_t nq, int64_t id_offset,
                              int k, float *dis, int64_t *ids, cudaStream_t s) {
    if (nq == 0) return cudaSuccess;
    const size_t smem = (size_t)((k + 1) & ~1) * 4 + (size_t)k * 8;
    rescore_l2_kernel<<<(unsigned)nq, 256, smem, s>>>(corpus, bf16, row_bytes, d_pad, queries, id_offset, k, dis, ids);
    g_launches++;
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------
// host launchers
// ------------------------------------------------------------------------------------
// Query tiles ride on gridDim.y, at most 65535 of them per launch: a larger batch launches slice after slice, each with its
// queries and partial lists offset to the slice's first query.  The fused form (<= 8 queries) is always one slice.
constexpr int64_t kMaxGridY = 65535;

template <int QT, int U, int CU>
static cudaError_t launch_scan_qt(const ScanParams &p, int blocks_x, size_t smem, cudaStream_t s) {
    auto go = [&](auto kern) -> cudaError_t {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        const int64_t slice = p.fused ? p.nq : kMaxGridY * QT;
        for (int64_t q0 = 0; q0 < p.nq; q0 += slice) {
            ScanParams ps = p;
            ps.nq = std::min(slice, p.nq - q0);
            ps.queries += q0 * p.d_pad;
            ps.part_keys += q0 * blocks_x * p.k;
            ps.part_ids += q0 * blocks_x * p.k;
            kern<<<dim3(blocks_x, (unsigned)ceil_div(ps.nq, QT)), kScanThreads, smem, s>>>(ps);
            g_launches++;
            if ((e = cudaGetLastError()) != cudaSuccess) return e;
        }
        return cudaSuccess;
    };
    if (p.l2) return p.bf16 ? go(flat_scan_kernel<QT, U, CU, true, true>) : go(flat_scan_kernel<QT, U, CU, true, false>);
    return p.bf16 ? go(flat_scan_kernel<QT, U, CU, false, true>) : go(flat_scan_kernel<QT, U, CU, false, false>);
}

size_t scan_smem_bytes(int qt, int d_pad, int k) {
    // + one merged list for the fused form's last-block merge (which reuses the front of the buffer)
    return std::max((size_t)qt * d_pad * 4 + (size_t)kScanWarps * qt * k * 8, (size_t)(kScanWarps + 1) * k * 8);
}

cudaError_t launch_flat_scan(const ScanParams &p_in, int qt, int blocks_x, cudaStream_t s) {
    ScanParams p = p_in;
    size_t smem = scan_smem_bytes(qt, p.d_pad, p.k);
    p.stage_cap = 0;
    if (p.fused && (size_t)blocks_x * p.k <= 8192) {
        // the last block stages every partial list in shared memory with independent loads (one L2 round trip instead of one per
        // 256 candidates): [warps + 1][k] lists, then blocks_x * k keys and ids
        p.stage_cap = blocks_x * p.k;
        smem = std::max(smem, (size_t)(kScanWarps + 1) * p.k * 8 + (size_t)p.stage_cap * 8);
    }
    const int elems = p.bf16 ? 8 : 4;
    const int cpl = (int)ceil_div(p.d_pad / elems, p.group);  // 16-byte chunks per lane and row
    // loads in flight per lane: short rows -> 4 rows x 1 chunk; long rows -> 4 chunks x (4 | 2) rows
    if (cpl <= 2) {
        switch (qt) {
            case 1: return launch_scan_qt<1, 4, 1>(p, blocks_x, smem, s);
            case 4: return launch_scan_qt<4, 4, 1>(p, blocks_x, smem, s);
            default: return launch_scan_qt<8, 4, 1>(p, blocks_x, smem, s);
        }
    }
    switch (qt) {
        case 1: return launch_scan_qt<1, 4, 4>(p, blocks_x, smem, s);
        case 4: return launch_scan_qt<4, 2, 4>(p, blocks_x, smem, s);
        default: return launch_scan_qt<8, 2, 4>(p, blocks_x, smem, s);
    }
}

cudaError_t launch_binary_scan(const BinaryScanParams &p, int blocks_x, cudaStream_t s) {
    const size_t smem = round_up(p.nbytes, 16) + (size_t)kScanWarps * p.k * 8;
    cudaError_t e = cudaFuncSetAttribute(binary_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    // one query per y-block: slices of at most kMaxGridY queries, as in launch_scan_qt
    for (int64_t q0 = 0; q0 < p.nq; q0 += kMaxGridY) {
        BinaryScanParams ps = p;
        ps.nq = std::min(kMaxGridY, p.nq - q0);
        ps.queries += q0 * p.nbytes;
        ps.part_keys += q0 * blocks_x * p.k;
        ps.part_ids += q0 * blocks_x * p.k;
        binary_scan_kernel<<<dim3(blocks_x, (unsigned)ps.nq), kScanThreads, smem, s>>>(ps);
        g_launches++;
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    return cudaSuccess;
}

cudaError_t launch_topk_merge(const MergeParams &p, bool external, cudaStream_t s) {
    const size_t smem = (size_t)(kScanWarps + 1) * p.k * (external ? 12 : 8);
    auto go = [&](auto kern) -> cudaError_t {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        kern<<<(unsigned)p.nq, kScanThreads, smem, s>>>(p);
        g_launches++;
        return cudaGetLastError();
    };
    return external ? go(topk_merge_ext_kernel) : go(topk_merge_kernel);
}

}  // namespace b200
