// graph_sm90.cu -- the neighbour graph of an HNSWFLAT, MSTG or BINARYMSTG index (graph_degree=D): candidate lists -> rank-based
// pruning -> reverse edges and merge at build, and the graph search over fp32 rows (HNSWFLAT), the bf16 list pages (MSTG) or the
// binary list pages (BINARYMSTG), one CTA per query or, at search_width=W > 1, one cluster of W CTAs per query that expands W
// parents per iteration (DESIGN §3).
#include <cooperative_groups.h>
#include <cub/cub.cuh>

#include <map>
#include <mutex>
#include <tuple>

#include "common.cuh"
#include "graph.h"
#include "ivf_aq.h"

namespace b200 {

// ------------------------------------------------------------------------------------
// build
// ------------------------------------------------------------------------------------
__global__ void graph_candidates_kernel(const int64_t *__restrict__ ids, const uint32_t *__restrict__ row_slot, int64_t m, int64_t row0, int K,
                                        uint32_t *__restrict__ cand) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const int64_t *row = ids + i * (K + 1);
    uint32_t *out = cand + i * K;
    if (row_slot[row0 + i] == kNoId) {
        for (int j = 0; j < K; j++) out[j] = kNoId;
        return;
    }
    int self = K;   // absent (duplicate rows): drop the last entry
    for (int j = 0; j < K + 1; j++)
        if (row[j] == row0 + i) {
            self = j;
            break;
        }
    for (int j = 0, o = 0; j < K + 1; j++) {
        if (j == self) continue;
        out[o++] = row[j] >= 0 ? (uint32_t)row[j] : kNoId;
    }
}

int graph_candidates(const int64_t *d_ids, const uint32_t *d_row_slot, int64_t m, int64_t row0, int K, uint32_t *d_cand, cudaStream_t s) {
    if (m == 0) return B200_OK;
    graph_candidates_kernel<<<(unsigned)ceil_div(m, 256), 256, 0, s>>>(d_ids, d_row_slot, m, row0, K, d_cand);
    g_launches++;
    B200_CUDA_OK(cudaGetLastError());
    return B200_OK;
}

// One block per node A, cand(A) = c[0..K) in shared memory, also sorted by id for membership.  Thread pair (i, p) looks up
// v = cand(c[i])[p]: when v = c[j] with i < j and p < j, c[i] is a detour to c[j] (c[j] ranks ahead of position j in the list of
// a closer candidate).  The detour counts are integer sums, so the result does not depend on the order of the additions.
__global__ void __launch_bounds__(256) graph_prune_kernel(const uint32_t *__restrict__ cand, int64_t n, int K, int D, uint32_t *__restrict__ pruned) {
    __shared__ uint32_t c[2 * kGraphMaxDegree], sid[2 * kGraphMaxDegree];
    __shared__ int spos[2 * kGraphMaxDegree], det[2 * kGraphMaxDegree];
    const int64_t a = blockIdx.x;
    const int tid = threadIdx.x;
    if (tid < K) {
        const uint32_t v = cand[a * K + tid];
        c[tid] = v < (uint64_t)n ? v : kNoId;
        det[tid] = 0;
    }
    __syncthreads();
    if (tid < K) {   // rank by (id, position): ids are distinct, the position only orders the padding
        const uint32_t v = c[tid];
        int r = 0;
        for (int j = 0; j < K; j++) r += c[j] < v || (c[j] == v && j < tid);
        sid[r] = v;
        spos[r] = tid;
    }
    __syncthreads();
    for (int e = tid; e < K * K; e += blockDim.x) {
        const int i = e / K, pp = e - i * K;
        const uint32_t u = c[i];
        if (u == kNoId) continue;
        const uint32_t v = cand[(int64_t)u * K + pp];
        if (v == kNoId) continue;
        int lo = 0, hi = K;   // first sorted entry >= v
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (sid[mid] < v) lo = mid + 1;
            else hi = mid;
        }
        if (lo < K && sid[lo] == v) {
            const int j = spos[lo];
            if (j > i && pp < j) atomicAdd(&det[j], 1);
        }
    }
    __syncthreads();
    __shared__ int nvalid;
    if (tid == 0) {
        int nv = 0;
        for (int j = 0; j < K; j++) nv += c[j] != kNoId;
        nvalid = nv;
    }
    if (tid < K && c[tid] != kNoId) {
        const int key = det[tid] * K + tid;
        int r = 0;
        for (int j = 0; j < K; j++) r += c[j] != kNoId && det[j] * K + j < key;
        if (r < D) pruned[a * D + r] = c[tid];
    }
    __syncthreads();
    for (int r = nvalid + tid; r < D; r += blockDim.x) pruned[a * D + r] = kNoId;
}

int graph_prune(const uint32_t *d_cand, int64_t n, int D, uint32_t *d_pruned, cudaStream_t s) {
    if (n == 0) return B200_OK;
    graph_prune_kernel<<<(unsigned)n, 256, 0, s>>>(d_cand, n, 2 * D, D, d_pruned);
    g_launches++;
    B200_CUDA_OK(cudaGetLastError());
    return B200_OK;
}

// triple (B, r, A) of edge A -> B at rank r as key B * D + r, value A, in A-major order; empty slots get the key n * D
__global__ void graph_triples_kernel(const uint32_t *__restrict__ pruned, int64_t n, int D, uint64_t *__restrict__ keys, uint32_t *__restrict__ vals) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n * D) return;
    const uint32_t b = pruned[e];
    const int64_t a = e / D, r = e - a * D;
    keys[e] = b != kNoId ? (uint64_t)b * D + r : (uint64_t)n * D;
    vals[e] = (uint32_t)a;
}

__device__ __forceinline__ bool graph_row_has(const uint32_t *row, int cnt, uint32_t v) {
    for (int t = 0; t < cnt; t++)
        if (row[t] == v) return true;
    return false;
}

// graph(B): the first D / 2 pruned forward edges, then at most D / 2 reverse sources in (rank, source) order, then the rest of
// the forward edges; duplicates skipped, at most D entries, empty slots 0xFFFFFFFF
__global__ void graph_merge_kernel(const uint32_t *__restrict__ pruned, const uint64_t *__restrict__ keys, const uint32_t *__restrict__ vals,
                                   int64_t n, int D, uint32_t *__restrict__ graph) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n) return;
    const uint32_t *fwd = pruned + b * D;
    uint32_t *row = graph + b * D;
    int cnt = 0;
    for (int r = 0; r < D / 2; r++) {
        const uint32_t v = fwd[r];
        if (v != kNoId && !graph_row_has(row, cnt, v)) row[cnt++] = v;
    }
    const int64_t total = n * D;
    int64_t lo = 0, hi = total;   // first key >= b * D
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (keys[mid] < (uint64_t)b * D) lo = mid + 1;
        else hi = mid;
    }
    for (int added = 0; lo < total && keys[lo] < (uint64_t)(b + 1) * D && added < D / 2 && cnt < D; lo++) {
        const uint32_t v = vals[lo];
        if (!graph_row_has(row, cnt, v)) {
            row[cnt++] = v;
            added++;
        }
    }
    for (int r = D / 2; r < D && cnt < D; r++) {
        const uint32_t v = fwd[r];
        if (v != kNoId && !graph_row_has(row, cnt, v)) row[cnt++] = v;
    }
    for (; cnt < D; cnt++) row[cnt] = kNoId;
}

int graph_merge(const uint32_t *d_pruned, int64_t n, int D, uint32_t *d_graph, cudaStream_t s) {
    if (n == 0) return B200_OK;
    const int64_t e = n * D;
    if (e >= (int64_t)1 << 31) return fail(B200_ERR_UNSUPPORTED, "graph build: n x graph_degree must stay below 2^31");
    DevMem keys, keys_out, vals, vals_out, tmp;
    size_t tb = 0;
    int end_bit = 1;
    while (end_bit < 64 && ((uint64_t)e >> end_bit) != 0) end_bit++;
    cub::DeviceRadixSort::SortPairs(nullptr, tb, keys.as<uint64_t>(), keys_out.as<uint64_t>(), vals.as<uint32_t>(), vals_out.as<uint32_t>(), (int)e, 0,
                                    end_bit, s);
    if (keys.alloc((size_t)e * 8) != B200_OK || keys_out.alloc((size_t)e * 8) != B200_OK || vals.alloc((size_t)e * 4) != B200_OK ||
        vals_out.alloc((size_t)e * 4) != B200_OK || tmp.alloc(tb + 256) != B200_OK)
        return fail(B200_ERR_NOMEM, "graph build: cudaMalloc of the reverse-edge scratch failed (" + std::to_string(e * 24) + " bytes)");
    graph_triples_kernel<<<(unsigned)ceil_div(e, 256), 256, 0, s>>>(d_pruned, n, D, keys.as<uint64_t>(), vals.as<uint32_t>());
    // stable: equal (B, r) keys keep the A-ascending order of the triples
    cub::DeviceRadixSort::SortPairs(tmp.p, tb, keys.as<uint64_t>(), keys_out.as<uint64_t>(), vals.as<uint32_t>(), vals_out.as<uint32_t>(), (int)e, 0, end_bit,
                                    s);
    graph_merge_kernel<<<(unsigned)ceil_div(n, 128), 128, 0, s>>>(d_pruned, keys_out.as<uint64_t>(), vals_out.as<uint32_t>(), n, D, d_graph);
    g_launches += 3;
    const cudaError_t err = cudaStreamSynchronize(s);
    if (err != cudaSuccess) return fail(B200_ERR_CUDA, std::string("graph merge: ") + cudaGetErrorString(err));
    return B200_OK;
}

// One CTA per list walks its page chain, thread t on row t of every page (as list_alive_kernel in ivf.cu): the list's valid
// rows record their pool slot under their id.  Slots past the list's length are never read; a row in no list keeps the
// caller's 0xFFFFFFFF.
__global__ void __launch_bounds__(kPageRows) row_slot_kernel(const uint32_t *__restrict__ list_len, const uint32_t *__restrict__ list_page_off,
                                                             const uint32_t *__restrict__ list_pages, const uint32_t *__restrict__ row_ids,
                                                             uint32_t *__restrict__ row_slot) {
    const int l = blockIdx.x;
    const uint32_t len = list_len[l], off = list_page_off[l];
    for (uint32_t j = 0; j * kPageRows < len; j++) {
        if (j * kPageRows + threadIdx.x >= len) break;
        const uint32_t slot = list_pages[off + j] * kPageRows + threadIdx.x;
        row_slot[row_ids[slot]] = slot;
    }
}

int graph_row_slots(const uint32_t *d_list_len, const uint32_t *d_list_page_off, const uint32_t *d_list_pages, const uint32_t *d_row_ids, int nlist,
                    uint32_t *d_row_slot, cudaStream_t s) {
    if (nlist == 0) return B200_OK;
    row_slot_kernel<<<(unsigned)nlist, kPageRows, 0, s>>>(d_list_len, d_list_page_off, d_list_pages, d_row_ids, d_row_slot);
    g_launches++;
    B200_CUDA_OK(cudaGetLastError());
    return B200_OK;
}

// rows [m][d] fp32 = the bf16 page rows of ids row0 .. row0 + m - 1 (the graph build's queries of an index without fp32 rows)
__global__ void page_rows_kernel(const __nv_bfloat16 *__restrict__ pool, const uint32_t *__restrict__ row_slot, int64_t row0, int64_t m, int d, int d_pad64,
                                 float *__restrict__ out) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m * d) return;
    const int64_t i = e / d;
    const int j = (int)(e - i * d);
    const uint32_t slot = row_slot[row0 + i];
    out[e] = slot == kNoId ? 0.f : __bfloat162float(pool[(((size_t)(slot / kPageRows) * (d_pad64 / 64) + j / 64) * kPageRows + slot % kPageRows) * 64 + j % 64]);
}

int graph_page_rows(const void *d_pool, const uint32_t *d_row_slot, int64_t row0, int64_t m, int d, int d_pad64, float *d_out, cudaStream_t s) {
    if (m == 0) return B200_OK;
    page_rows_kernel<<<(unsigned)ceil_div(m * d, 256), 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16 *>(d_pool), d_row_slot, row0, m, d, d_pad64, d_out);
    g_launches++;
    B200_CUDA_OK(cudaGetLastError());
    return B200_OK;
}

// rows [m][row_bytes] = the binary page rows of ids row0 .. row0 + m - 1 (the graph build's queries of a BINARYMSTG index)
__global__ void bin_page_rows_kernel(const uint8_t *__restrict__ pool, const uint32_t *__restrict__ row_slot, int64_t row0, int64_t m, int row_bytes,
                                     int row_pad, int kb_w, uint8_t *__restrict__ out) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m * row_bytes) return;
    const int64_t i = e / row_bytes;
    const int j = (int)(e - i * row_bytes);
    const uint32_t slot = row_slot[row0 + i];
    out[e] = slot == kNoId ? 0 : pool[(((size_t)(slot / kPageRows) * (row_pad / kb_w) + j / kb_w) * kPageRows + slot % kPageRows) * kb_w + j % kb_w];
}

int graph_bin_page_rows(const void *d_pool, const uint32_t *d_row_slot, int64_t row0, int64_t m, int row_bytes, int row_pad, int kb_w, uint8_t *d_out,
                        cudaStream_t s) {
    if (m == 0) return B200_OK;
    bin_page_rows_kernel<<<(unsigned)ceil_div(m * row_bytes, 256), 256, 0, s>>>(static_cast<const uint8_t *>(d_pool), d_row_slot, row0, m, row_bytes,
                                                                                 row_pad, kb_w, d_out);
    g_launches++;
    B200_CUDA_OK(cudaGetLastError());
    return B200_OK;
}

// ------------------------------------------------------------------------------------
// search: one CTA per query (W = 1), or one cluster of W CTAs per query (search_width=W)
// ------------------------------------------------------------------------------------
namespace {
namespace cg = cooperative_groups;
static_assert(kGraphMaxDegree >= kGraphMaxSeeds, "a step takes the seeds");
static_assert(kGraphMaxWidth <= 8, "sh[16 ..) and sh[24 ..) hold one int per rank of a cluster");

struct GraphSmem {
    int64_t qs, vis, ek0, ei0, ek1, ei1, ck, ci, sk, si, nb, pk, pi, ak0, ai0, ak1, ai1, sh, ef0, ef1, total;
};

// ck / ci / sk / si: the candidates of a step (W rows of at most kGraphMaxDegree); nb: this CTA's neighbour row; pk / pi
// (W > 1 only): this CTA's sorted candidates, which the other CTAs of its cluster read
__host__ __device__ inline GraphSmem graph_smem_layout(int d_pad, int ef, int k, bool filtered, int width) {
    GraphSmem L{};
    const int ka = filtered ? k : 0;
    const int64_t batch = (int64_t)kGraphMaxDegree * width, pub = width > 1 ? kGraphMaxDegree : 0;
    int64_t o = 0;
    L.qs = o; o += (int64_t)d_pad * 4;
    L.vis = o; o += (int64_t)kGraphVisitedSlots * 4;
    L.ek0 = o; o += (int64_t)ef * 4;
    L.ei0 = o; o += (int64_t)ef * 4;
    L.ek1 = o; o += (int64_t)ef * 4;
    L.ei1 = o; o += (int64_t)ef * 4;
    L.ck = o; o += batch * 4;
    L.ci = o; o += batch * 4;
    L.sk = o; o += batch * 4;
    L.si = o; o += batch * 4;
    L.nb = o; o += kGraphMaxDegree * 4;
    L.pk = o; o += pub * 4;
    L.pi = o; o += pub * 4;
    L.ak0 = o; o += (int64_t)ka * 4;
    L.ai0 = o; o += (int64_t)ka * 4;
    L.ak1 = o; o += (int64_t)ka * 4;
    L.ai1 = o; o += (int64_t)ka * 4;
    L.sh = o; o += 32 * 4;
    L.ef0 = o; o += ef;
    L.ef1 = o; o += ef;
    L.total = (o + 15) / 16 * 16;
    return L;
}

__device__ __forceinline__ uint32_t vis_slot(uint32_t id) { return (id * 0x9E3779B1u) >> (32 - kGraphVisitedLog2); }

__device__ __forceinline__ bool vis_contains(const uint32_t *vis, uint32_t id) {
    for (uint32_t s = vis_slot(id);; s = (s + 1) & (kGraphVisitedSlots - 1)) {
        const uint32_t v = vis[s];
        if (v == id) return true;
        if (v == kNoId) return false;
    }
}

// distinct ids only; the slot an id lands in depends on the order of the inserts, membership does not
__device__ __forceinline__ void vis_insert(uint32_t *vis, uint32_t id) {
    for (uint32_t s = vis_slot(id);; s = (s + 1) & (kGraphVisitedSlots - 1)) {
        const uint32_t old = atomicCAS(&vis[s], kNoId, id);
        if (old == kNoId || old == id) return;
    }
}

// entries of the sorted a[0..len) better than (key, id)
__device__ __forceinline__ int count_better(const float *ak, const uint32_t *ai, int len, float key, uint32_t id) {
    int lo = 0, hi = len;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (better(ak[mid], ai[mid], key, id)) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// out[0..min(cap, cnt + nc)) = the best of the sorted list (cnt entries) and the sorted candidates (nc, disjoint ids); new
// candidates unexpanded.  Every thread of the CTA calls it.
__device__ __forceinline__ void merge_lists(const float *lk, const uint32_t *li, const uint8_t *lf, int cnt, const float *ck, const uint32_t *ci,
                                            int nc, int cap, float *ok, uint32_t *oi, uint8_t *of) {
    for (int p = threadIdx.x; p < cnt; p += blockDim.x) {
        const int np = p + count_better(ck, ci, nc, lk[p], li[p]);
        if (np < cap) {
            ok[np] = lk[p];
            oi[np] = li[p];
            if (of) of[np] = lf[p];
        }
    }
    for (int r = threadIdx.x; r < nc; r += blockDim.x) {
        const int np = r + count_better(lk, li, cnt, ck[r], ci[r]);
        if (np < cap) {
            ok[np] = ck[r];
            oi[np] = ci[r];
            if (of) of[np] = 0;
        }
    }
}

// Every thread of the CTA calls it with a flag: *below = the set flags of the threads below it; returns the set flags of the
// CTA.  scratch: one int per warp, free again when it returns.
__device__ __forceinline__ int cta_count_flags(bool flag, int *scratch, int *below) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const unsigned bal = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) scratch[warp] = __popc(bal);
    __syncthreads();
    int b = __popc(bal & ((1u << lane) - 1)), all = 0;
    for (int w = 0; w < kGraphThreads / 32; w++) {
        const int c = scratch[w];
        b += w < warp ? c : 0;
        all += c;
    }
    *below = b;
    __syncthreads();
    return all;
}

// Shared memory: the query, the visited table, two ef-entry lists (keys, ids, expanded flags) used in turn, the step's
// candidates (adjacency order, then sorted), the neighbour row, two k-entry lists of alive rows (filtered searches only).
// A step: warp 0 drops empty slots, repeats within the row and visited ids, compacts the rest in row order and inserts them
// into the visited table; a warp per row scores them (`score`: 128-bit loads, fp32, fixed lane order); they are sorted by
// (key, id) and rank-merged into the ef list (and, those the bitmap keeps, into the alive list).  Every answer-bearing step is
// a sort or a merge by (key, id): the result does not depend on thread timing.  q_len: the query's floats in shared memory
// (>= d_pad, zero beyond it) as stage(qs, q, i) writes them, one 4-byte word i per call; score(id, qs, lane) returns, on every
// lane, the warp's L2 distance or inner product of row id (binary rows: their distance).
//
// W > 1 (search_width=W): the W CTAs of a cluster walk one query, each holding the same copy of the lists and the visited
// table.  An iteration takes the first W unexpanded entries; CTA r loads the row of parent r into its nb (phase A), cluster
// barrier 1.  Phase B: CTA r puts the valid ids of the rows of ranks below r (read from their nb) into its visited table, so
// the step above keeps the ids of its own row that are valid, unvisited, and not earlier in the concatenation of the W rows;
// it scores and sorts them into pk / pi, their count in sh[0]; cluster barrier 2.  Phase C: every CTA copies the W sorted
// runs in rank order, puts the ids of higher ranks into its visited table and rank-merges the runs: each CTA then applies the
// same candidates, and every copy of the state stays the same (the visited tables hold the same ids).  A CTA writes nb only
// in phase A (read by others in phase B, before barrier 2) and pk / pi / sh[0] only in phase B (read in phase C, before the
// next barrier 1).  Every barrier sits on control flow that depends on the shared state alone, so all CTAs reach it; a last
// one keeps every CTA's shared memory until no other reads it.  CTA 0 writes the answer.
template <int W, class Stage, class Score>
__device__ __forceinline__ void graph_walk(const GraphSearchParams &p, int q_len, Stage stage, Score score) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const bool filtered = p.alive != nullptr;
    const GraphSmem L = graph_smem_layout(q_len, p.ef, p.k, filtered, W);
    float *qs = reinterpret_cast<float *>(smem_raw + L.qs);
    uint32_t *vis = reinterpret_cast<uint32_t *>(smem_raw + L.vis);
    // the two lists of each kind are at a fixed byte distance: list `b` of a kind is its list 0 plus b x that distance
    float *ek0 = reinterpret_cast<float *>(smem_raw + L.ek0);
    uint32_t *ei0 = reinterpret_cast<uint32_t *>(smem_raw + L.ei0);
    uint8_t *ef0 = smem_raw + L.ef0;
    const int64_t dek = L.ek1 - L.ek0, dei = L.ei1 - L.ei0, def = L.ef1 - L.ef0, dak = L.ak1 - L.ak0, dai = L.ai1 - L.ai0;
    float *ck = reinterpret_cast<float *>(smem_raw + L.ck), *sk = reinterpret_cast<float *>(smem_raw + L.sk);
    uint32_t *ci = reinterpret_cast<uint32_t *>(smem_raw + L.ci), *si = reinterpret_cast<uint32_t *>(smem_raw + L.si);
    uint32_t *nb = reinterpret_cast<uint32_t *>(smem_raw + L.nb);
    // where a step sorts this CTA's candidates: the step's sorted candidates (W = 1), or the run the cluster reads (W > 1)
    float *rk = W == 1 ? sk : reinterpret_cast<float *>(smem_raw + L.pk);
    uint32_t *ri = W == 1 ? si : reinterpret_cast<uint32_t *>(smem_raw + L.pi);
    float *ak0 = reinterpret_cast<float *>(smem_raw + L.ak0);
    uint32_t *ai0 = reinterpret_cast<uint32_t *>(smem_raw + L.ai0);
    auto ek = [&](int b) { return reinterpret_cast<float *>(reinterpret_cast<unsigned char *>(ek0) + b * dek); };
    auto ei = [&](int b) { return reinterpret_cast<uint32_t *>(reinterpret_cast<unsigned char *>(ei0) + b * dei); };
    auto ef = [&](int b) { return ef0 + b * def; };
    auto ak = [&](int b) { return reinterpret_cast<float *>(reinterpret_cast<unsigned char *>(ak0) + b * dak); };
    auto ai = [&](int b) { return reinterpret_cast<uint32_t *>(reinterpret_cast<unsigned char *>(ai0) + b * dai); };
    int *sh = reinterpret_cast<int *>(smem_raw + L.sh);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t q = blockIdx.x / W;
    int rank = 0;
    if constexpr (W > 1) rank = (int)cg::this_cluster().block_rank();
    const int nwarps = kGraphThreads / 32;
    for (int i = tid; i < q_len; i += kGraphThreads) stage(qs, q, i);
    for (int i = tid; i < kGraphVisitedSlots; i += kGraphThreads) vis[i] = kNoId;
    if (rank == 0)   // the seeds are the row of rank 0 in the first step
        for (int j = tid; j < p.nseeds; j += kGraphThreads) {
            const int64_t v = p.seeds[q * p.nseeds + j];
            nb[j] = v >= 0 && v < p.n ? (uint32_t)v : kNoId;
        }
    __syncthreads();
    int cur = 0, cnt = 0, acur = 0, acnt = 0;
    unsigned long long scored = 0;

    // one step over the rows of ranks 0 .. np - 1, m ids each (W = 1: over nb[0..m))
    auto step = [&](int m, int np) {
        if constexpr (W > 1) {
            cg::cluster_group cluster = cg::this_cluster();
            cluster.sync();   // barrier 1: the rows are in the nb of ranks 0 .. np - 1
            const int pre = min(rank, np) * m;
            for (int e = tid; e < pre; e += kGraphThreads) {
                const uint32_t v = cluster.map_shared_rank(nb, e / m)[e % m];
                if (v < (uint64_t)p.n) vis_insert(vis, v);
            }
            __syncthreads();
            if (rank >= np) m = 0;
        }
        if (warp == 0) {
            int nc = 0;
            for (int b = 0; b < m; b += 32) {
                const int j = b + lane;
                const uint32_t v = j < m ? nb[j] : kNoId;
                bool fresh = v < (uint64_t)p.n;
                for (int t = 0; fresh && t < j; t++) fresh = nb[t] != v;
                if (fresh) fresh = !vis_contains(vis, v);
                const unsigned bal = __ballot_sync(0xffffffffu, fresh);
                if (fresh) ci[nc + __popc(bal & ((1u << lane) - 1))] = v;
                nc += __popc(bal);
            }
            __syncwarp();
            for (int c = lane; c < nc; c += 32) vis_insert(vis, ci[c]);
            if (lane == 0) sh[0] = nc;
        }
        __syncthreads();
        const int nc = sh[0];
        for (int c = warp; c < nc; c += nwarps) {
            const float acc = score(ci[c], qs, lane);
            if (lane == 0) ck[c] = p.l2 ? acc : -acc;
        }
        if constexpr (W == 1) scored += (unsigned long long)nc;
        __syncthreads();
        if (tid < nc) {   // sort by (key, id); nc <= kGraphMaxDegree < kGraphThreads
            const float key = ck[tid];
            const uint32_t id = ci[tid];
            int r = 0;
            for (int c = 0; c < nc; c++) r += better(ck[c], ci[c], key, id);
            rk[r] = key;
            ri[r] = id;
        }
        __syncthreads();
        int total = nc;   // the step's candidates, sorted in sk / si
        if constexpr (W > 1) {
            cg::cluster_group cluster = cg::this_cluster();
            cluster.sync();   // barrier 2: every rank's sorted run is in its pk / pi, its length in its sh[0]
            int *runs = sh + 24;
            if (tid < W) runs[tid] = *cluster.map_shared_rank(sh, tid);
            __syncthreads();
            total = 0;
            for (int r = 0; r < W; r++) total += runs[r];
            // run r at ck / ci [off, off + runs[r]), in rank order
            for (int e = tid; e < W * kGraphMaxDegree; e += kGraphThreads) {
                const int r = e / kGraphMaxDegree, j = e % kGraphMaxDegree;
                if (j >= runs[r]) continue;
                int off = 0;
                for (int t = 0; t < r; t++) off += runs[t];
                const uint32_t id = cluster.map_shared_rank(ri, r)[j];
                ck[off + j] = cluster.map_shared_rank(rk, r)[j];
                ci[off + j] = id;
                if (r > rank) vis_insert(vis, id);
            }
            __syncthreads();
            // rank-merge: an entry's place is its place in its run plus the entries of the other runs better than it
            for (int e = tid; e < W * kGraphMaxDegree; e += kGraphThreads) {
                const int r = e / kGraphMaxDegree, j = e % kGraphMaxDegree;
                if (j >= runs[r]) continue;
                int off = 0;
                for (int t = 0; t < r; t++) off += runs[t];
                const float key = ck[off + j];
                const uint32_t id = ci[off + j];
                int pos = j;
                for (int t = 0, o = 0; t < W; o += runs[t], t++)
                    if (t != r) pos += count_better(ck + o, ci + o, runs[t], key, id);
                sk[pos] = key;
                si[pos] = id;
            }
            scored += (unsigned long long)total;
            __syncthreads();
        }
        merge_lists(ek(cur), ei(cur), ef(cur), cnt, sk, si, total, p.ef, ek(cur ^ 1), ei(cur ^ 1), ef(cur ^ 1));
        cur ^= 1;
        cnt = min(p.ef, cnt + total);
        if (filtered) {   // the kept ones, still sorted, into ck / ci (free after the sort)
            int na = 0;
            if constexpr (W == 1) {
                if (tid < nc) {
                    const uint32_t id = si[tid];
                    if ((p.alive[id >> 3] >> (id & 7)) & 1) {
                        int r = 0;
                        for (int c = 0; c < tid; c++) r += (p.alive[si[c] >> 3] >> (si[c] & 7)) & 1;
                        ck[r] = sk[tid];
                        ci[r] = id;
                    }
                }
                if (tid == 0) {
                    int kept = 0;
                    for (int c = 0; c < nc; c++) kept += (p.alive[si[c] >> 3] >> (si[c] & 7)) & 1;
                    sh[1] = kept;
                }
                __syncthreads();
                na = sh[1];
            } else {   // up to W x kGraphMaxDegree candidates: compacted a CTA-width at a time
                for (int b = 0; b < total; b += kGraphThreads) {
                    const int t = b + tid;
                    const uint32_t id = t < total ? si[t] : 0;
                    const bool keep = t < total && ((p.alive[id >> 3] >> (id & 7)) & 1);
                    int below;
                    const int all = cta_count_flags(keep, sh + 8, &below);
                    if (keep) {
                        ck[na + below] = sk[t];
                        ci[na + below] = id;
                    }
                    na += all;
                }
                __syncthreads();
            }
            merge_lists(ak(acur), ai(acur), nullptr, acnt, ck, ci, na, p.k, ak(acur ^ 1), ai(acur ^ 1), nullptr);
            acur ^= 1;
            acnt = min(p.k, acnt + na);
        }
        __syncthreads();
    };

    step(p.nseeds, 1);
    for (int it = 0; it < p.max_iters; it++) {
        if constexpr (W == 1) {
            // parent: the first unexpanded entry of the list
            int first = INT_MAX;
            for (int e = tid; e < cnt; e += kGraphThreads)
                if (!ef(cur)[e]) {
                    first = e;
                    break;
                }
            first = __reduce_min_sync(0xffffffffu, first);
            if (lane == 0) sh[8 + warp] = first;
            __syncthreads();
            if (tid == 0) {
                int f = INT_MAX;
                for (int w = 0; w < nwarps; w++) f = min(f, sh[8 + w]);
                sh[2] = f;
                if (f != INT_MAX) {
                    ef(cur)[f] = 1;
                    sh[3] = (int)ei(cur)[f];
                }
            }
            __syncthreads();
            if (sh[2] == INT_MAX) break;
            const uint32_t parent = (uint32_t)sh[3];
            for (int j = tid; j < p.degree; j += kGraphThreads) nb[j] = p.graph[(size_t)parent * p.degree + j];
            __syncthreads();
            step(p.degree, 1);
        } else {
            // parents: the first W unexpanded entries of the list (fewer when fewer remain) into sh[16 ..), a CTA-width at a time.
            // np and the list are the same in every CTA of the cluster, so all of them break together.
            int np = 0;
            for (int b = 0; b < cnt && np < W; b += kGraphThreads) {
                const int e = b + tid;
                const bool un = e < cnt && !ef(cur)[e];
                int below;
                const int all = cta_count_flags(un, sh + 8, &below);
                if (un && np + below < W) {
                    sh[16 + np + below] = (int)ei(cur)[e];
                    ef(cur)[e] = 1;
                }
                np = min(W, np + all);
            }
            __syncthreads();
            if (np == 0) break;
            if (rank < np) {
                const uint32_t parent = (uint32_t)sh[16 + rank];
                for (int j = tid; j < p.degree; j += kGraphThreads) nb[j] = p.graph[(size_t)parent * p.degree + j];
            }
            __syncthreads();
            step(p.degree, np);
        }
    }
    if constexpr (W > 1) cg::this_cluster().sync();   // no CTA leaves while another may still read its shared memory

    if (rank == 0) {
        const float *fk = filtered ? ak(acur) : ek(cur);
        const uint32_t *fi = filtered ? ai(acur) : ei(cur);
        const int have_n = filtered ? acnt : min(cnt, p.k);
        for (int j = tid; j < p.k; j += kGraphThreads) {
            const bool have = j < have_n;
            p.out_ids[q * p.k + j] = have ? (int64_t)fi[j] + p.id_offset : -1;
            p.out_dis[q * p.k + j] = have ? (p.l2 ? fk[j] : -fk[j]) : (p.l2 ? FLT_MAX : -FLT_MAX);
        }
        if (tid == 0) atomicAdd(p.rows_scored, scored);
    }
}

// HNSWFLAT: rows scored from the fp32 rows in HBM
template <int W>
__device__ __forceinline__ void graph_walk_fp32(const GraphSearchParams &p) {
    const auto stage = [&](float *qs, int64_t q, int i) { qs[i] = i < p.d_pad ? p.queries[q * p.d_pad + i] : 0.f; };
    graph_walk<W>(p, p.d_pad, stage, [&](uint32_t v, const float *qs, int lane) {
        const float4 *row = reinterpret_cast<const float4 *>(p.rows + (size_t)v * p.d_pad);
        const float4 *x4 = reinterpret_cast<const float4 *>(qs);
        float acc = 0.f;
        for (int cc = lane; cc < p.d_pad / 4; cc += 32) {
            const float4 y = __ldg(row + cc);
            const float4 x = x4[cc];
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
        return acc;
    });
}

// MSTG: rows scored in place from the bf16 list pages, row v at pool slot row_slot[v] ([page][d_pad64 / 64][256][64] bf16).
// Lane l reads 16 bytes (8 dims) of the 128-byte segment of k-block l / 8 + 4j, widens them to fp32 and accumulates against
// the query in its fixed order; the lane tree below is fixed, so a key depends on the row and the query alone.  The query's
// dims of a k-block sit in shared memory as [half][part][4]: dim 8 part + 4 half + e at 32 half + 4 part + e, so that the 8
// lanes of a quarter-warp read its two float4 of each k-block from 128 contiguous bytes each (no bank conflict).
// acc plus the terms of the two dims of a bf16 pair (low half first) against the query's x0, x1
__device__ __forceinline__ float bf16x2_term(int l2, uint32_t u, float x0, float x1, float acc) {
    const float y0 = __uint_as_float(u << 16), y1 = __uint_as_float(u & 0xffff0000u);
    if (l2) {
        float t = x0 - y0; acc = fmaf(t, t, acc);
        t = x1 - y1; return fmaf(t, t, acc);
    }
    acc = fmaf(x0, y0, acc);
    return fmaf(x1, y1, acc);
}

template <int W>
__device__ __forceinline__ void graph_walk_bf16(const GraphSearchParams &p) {
    const auto qpos = [](int i) { return (i & ~63) | ((i >> 2) & 1) << 5 | ((i >> 3) & 7) << 2 | (i & 3); };
    const auto stage = [&](float *qs, int64_t q, int i) { qs[qpos(i)] = i < p.d_pad ? p.queries[q * p.d_pad + i] : 0.f; };
    graph_walk<W>(p, p.d_pad64, stage, [&](uint32_t v, const float *qs, int lane) {
        const uint32_t slot = p.row_slot[v];
        const int kbs = p.d_pad64 / 64, seg = lane >> 3, part = lane & 7;
        const __nv_bfloat16 *pool = static_cast<const __nv_bfloat16 *>(p.pages);
        const uint4 *row = reinterpret_cast<const uint4 *>(pool + ((size_t)(slot / kPageRows) * kbs * kPageRows + slot % kPageRows) * 64) + part;
        const float4 *x4 = reinterpret_cast<const float4 *>(qs) + part;
        float acc = 0.f;
        for (int kb = seg; kb < kbs; kb += 4) {
            const uint4 u = __ldg(row + (size_t)kb * kPageRows * 8);
            const float4 xa = x4[kb * 16], xb = x4[kb * 16 + 8];
            acc = bf16x2_term(p.l2, u.x, xa.x, xa.y, acc);
            acc = bf16x2_term(p.l2, u.y, xa.z, xa.w, acc);
            acc = bf16x2_term(p.l2, u.z, xb.x, xb.y, acc);
            acc = bf16x2_term(p.l2, u.w, xb.z, xb.w, acc);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        return acc;
    });
}

// BINARYMSTG: rows scored in place from the binary list pages ([page][row_pad / kb_w][256][kb_w] bytes), row v at pool slot
// row_slot[v].  The query's bytes sit in shared memory as row_pad / 4 words, zero beyond row_bytes.  Lane l ANDs the 16-byte
// chunks l, l + 32, ... of the row with the query and counts the set bits; the shuffle tree sums the lanes' counts.  With
// popc(q) (summed once by every warp) and the stored popc(y), the key is BINARYFLAT's distance: Hamming popc(q) + popc(y) - 2
// and; Jaccard (or - and) / or with or = popc(q) + popc(y) - and (0 when or = 0), one IEEE division.  Every count is an exact
// integer, so a key equals the exact scan's distance of that (query, row) to the bit.
template <int W>
__device__ __forceinline__ void graph_walk_b1(const GraphB1Params &b) {
    const GraphSearchParams &p = b.g;
    const uint8_t *qb = b.queries + (int64_t)(blockIdx.x / W) * b.row_bytes;
    int qpop = 0;
    for (int j = threadIdx.x & 31; j < b.row_bytes; j += 32) qpop += __popc((uint32_t)qb[j]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) qpop += __shfl_xor_sync(0xffffffffu, qpop, o);
    const auto stage = [&](float *qs, int64_t, int i) {
        uint32_t w = 0;
        for (int e = 0; e < 4; e++)
            if (4 * i + e < b.row_bytes) w |= (uint32_t)qb[4 * i + e] << (8 * e);
        reinterpret_cast<uint32_t *>(qs)[i] = w;
    };
    graph_walk<W>(p, b.row_pad / 4, stage, [&](uint32_t v, const float *qs, int lane) {
        const uint32_t slot = p.row_slot[v];
        const int cpk = b.kb_w / 16;   // 16-byte chunks per k-block
        const uint8_t *row = static_cast<const uint8_t *>(p.pages) + (size_t)(slot / kPageRows) * kPageRows * b.row_pad + (size_t)(slot % kPageRows) * b.kb_w;
        const uint4 *x4 = reinterpret_cast<const uint4 *>(qs);
        int a = 0;
        for (int c = lane; c < b.row_pad / 16; c += 32) {
            const int kb = c / cpk;
            const uint4 y = __ldg(reinterpret_cast<const uint4 *>(row + (size_t)kb * kPageRows * b.kb_w) + (c - kb * cpk));
            const uint4 x = x4[c];
            a += __popc(x.x & y.x) + __popc(x.y & y.y) + __popc(x.z & y.z) + __popc(x.w & y.w);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
        const int yp = (int)b.row_popc[slot];
        if (!b.jaccard) return (float)(qpop + yp - 2 * a);
        const int x_or = qpop + yp - a;
        return x_or == 0 ? 0.f : (float)(x_or - a) / (float)x_or;
    });
}
}  // namespace

__global__ void __launch_bounds__(kGraphThreads) graph_search_kernel(const GraphSearchParams p) { graph_walk_fp32<1>(p); }

// (kGraphThreads, 2): without the occupancy hint ptxas keeps this walk to 32 registers and spills; two CTAs per SM is what its
// shared memory allows at the largest lists anyway
__global__ void __launch_bounds__(kGraphThreads, 2) graph_search_bf16_kernel(const GraphSearchParams p) { graph_walk_bf16<1>(p); }

// the walks at search_width = W > 1: one cluster of W CTAs per query (grid nq x W, cluster (W, 1, 1)).  (kGraphThreads, 2) on
// both: without it ptxas keeps the fp32 walk to 40 registers and spills
template <int W>
__global__ void __launch_bounds__(kGraphThreads, 2) graph_search_cluster_kernel(const GraphSearchParams p) { graph_walk_fp32<W>(p); }
template <int W>
__global__ void __launch_bounds__(kGraphThreads, 2) graph_search_bf16_cluster_kernel(const GraphSearchParams p) { graph_walk_bf16<W>(p); }

// BINARYMSTG's walk over the binary list pages, and its cluster forms; (kGraphThreads, 2) as the bf16 walk
__global__ void __launch_bounds__(kGraphThreads, 2) graph_search_b1_kernel(const GraphB1Params p) { graph_walk_b1<1>(p); }
template <int W>
__global__ void __launch_bounds__(kGraphThreads, 2) graph_search_b1_cluster_kernel(const GraphB1Params p) { graph_walk_b1<W>(p); }

size_t graph_search_smem(int q_len, int ef, int k, bool filtered, int width) {
    return (size_t)graph_smem_layout(q_len, ef, k, filtered, width).total;
}

namespace {
template <int W>
const void *graph_cluster_kernel(bool bf16) {
    return bf16 ? (const void *)graph_search_bf16_cluster_kernel<W> : (const void *)graph_search_cluster_kernel<W>;
}

// cudaOccupancyMaxActiveClusters of (device, kernel, dynamic shared memory), asked once per key
int graph_max_active_clusters(const void *fn, const cudaLaunchConfig_t &cfg, int *clusters) {
    static std::mutex mu;
    static std::map<std::tuple<int, const void *, size_t>, int> known;
    int dev = 0;
    B200_CUDA_OK(cudaGetDevice(&dev));
    const auto key = std::make_tuple(dev, fn, cfg.dynamicSmemBytes);
    std::lock_guard<std::mutex> lock(mu);
    const auto it = known.find(key);
    if (it != known.end()) {
        *clusters = it->second;
        return B200_OK;
    }
    B200_CUDA_OK(cudaOccupancyMaxActiveClusters(clusters, fn, &cfg));
    known[key] = *clusters;
    return B200_OK;
}

// nq clusters of W CTAs (W > 1) of the walk fn, its one parameter at arg
int graph_launch_clusters(const void *fn, void *arg, size_t smem, int64_t nq, int W, cudaStream_t s) {
    if (nq > INT32_MAX / W) return fail(B200_ERR_UNSUPPORTED, "graph search: nq x search_width must stay below 2^31");
    cudaLaunchConfig_t cfg{};
    cudaLaunchAttribute attr{};
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = (unsigned)W;
    attr.val.clusterDim.y = 1;
    attr.val.clusterDim.z = 1;
    cfg.gridDim = dim3((unsigned)(nq * W));
    cfg.blockDim = dim3(kGraphThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    int clusters = 0;
    B200_TRY(graph_max_active_clusters(fn, cfg, &clusters));
    if (clusters < 1)
        return fail(B200_ERR_UNSUPPORTED, "graph search: a cluster of " + std::to_string(W) + " CTAs with " + std::to_string(smem) +
                                              " bytes of shared memory each cannot be resident on this device");
    void *args[] = {arg};
    B200_CUDA_OK(cudaLaunchKernelExC(&cfg, fn, args));
    return B200_OK;
}
}  // namespace

int graph_search(const GraphSearchParams &p, int64_t nq, int width, cudaStream_t s) {
    if (nq == 0) return B200_OK;
    const int W = width;
    if (!graph_width_ok(W)) return fail(B200_ERR_INVALID, "search_width must be 1, 2, 4 or 8, got " + std::to_string(W));
    const bool bf16 = p.pages != nullptr;
    const size_t smem = graph_search_smem(bf16 ? p.d_pad64 : p.d_pad, p.ef, p.k, p.alive != nullptr, W);
    const void *fn = W == 1   ? (bf16 ? (const void *)graph_search_bf16_kernel : (const void *)graph_search_kernel)
                     : W == 2 ? graph_cluster_kernel<2>(bf16)
                     : W == 4 ? graph_cluster_kernel<4>(bf16)
                              : graph_cluster_kernel<8>(bf16);
    // d <= B200_MAX_FLOAT_DIM keeps this below the limit at W = 1; W > 1 adds (W - 1) KB for the step's candidates and 512 B
    // for the published run, refused at the widest d_pad at ef = k = 1024 with a filter (include/b200_search.h)
    if (smem > (size_t)kSmemOptinBytes)
        return fail(B200_ERR_UNSUPPORTED, "graph search: d_pad " + std::to_string(bf16 ? p.d_pad64 : p.d_pad) + " at ef " + std::to_string(p.ef) +
                                              (W > 1 ? " and search_width " + std::to_string(W) : std::string()) + " needs " + std::to_string(smem) +
                                              " bytes of shared memory, more than " + std::to_string(kSmemOptinBytes));
    B200_CUDA_OK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (W == 1) {
        if (bf16) graph_search_bf16_kernel<<<(unsigned)nq, kGraphThreads, smem, s>>>(p);
        else graph_search_kernel<<<(unsigned)nq, kGraphThreads, smem, s>>>(p);
    } else {
        B200_TRY(graph_launch_clusters(fn, const_cast<GraphSearchParams *>(&p), smem, nq, W, s));
    }
    g_launches++;
    B200_CUDA_OK(cudaGetLastError());
    return B200_OK;
}

int graph_search_b1(const GraphB1Params &p, int64_t nq, int width, cudaStream_t s) {
    if (nq == 0) return B200_OK;
    const int W = width;
    if (!graph_width_ok(W)) return fail(B200_ERR_INVALID, "search_width must be 1, 2, 4 or 8, got " + std::to_string(W));
    // the query is at most 8 KB (65536 bits): every ef, k and W fits
    const size_t smem = graph_search_smem(p.row_pad / 4, p.g.ef, p.g.k, p.g.alive != nullptr, W);
    if (smem > (size_t)kSmemOptinBytes)
        return fail(B200_ERR_UNSUPPORTED, "graph search: a " + std::to_string(p.row_pad) + "-byte binary query at ef " + std::to_string(p.g.ef) +
                                              " needs " + std::to_string(smem) + " bytes of shared memory, more than " + std::to_string(kSmemOptinBytes));
    const void *fn = W == 1   ? (const void *)graph_search_b1_kernel
                     : W == 2 ? (const void *)graph_search_b1_cluster_kernel<2>
                     : W == 4 ? (const void *)graph_search_b1_cluster_kernel<4>
                              : (const void *)graph_search_b1_cluster_kernel<8>;
    B200_CUDA_OK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (W == 1) graph_search_b1_kernel<<<(unsigned)nq, kGraphThreads, smem, s>>>(p);
    else B200_TRY(graph_launch_clusters(fn, const_cast<GraphB1Params *>(&p), smem, nq, W, s));
    g_launches++;
    B200_CUDA_OK(cudaGetLastError());
    return B200_OK;
}

}  // namespace b200
