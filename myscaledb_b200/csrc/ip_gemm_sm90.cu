// ip_gemm_sm90.cu -- K2: batched multi-query x corpus inner product as a dense GEMM on the Hopper tensor cores
// (wgmma, operands staged by TMA), with the top-k selection FUSED into the epilogue: the [nq x N] score matrix is
// never written to memory.  Three operand types share the kernel:
//   * bf16 queries x bf16 corpus (K2);
//   * fp32 queries x fp32 corpus with fp32-level accuracy ("3xTF32", K2b): every fp32 value is split into two TF32
//     numbers  x = hi + lo  (hi = x with the low 13 mantissa bits cleared, lo = tf32(x - hi)) and
//     q.y = q_lo.y_hi + q_hi.y_lo + q_hi.y_hi  (+ q_lo.y_lo ~ 2^-22, dropped) is accumulated in fp32 by three wgmma per
//     k-step: error ~2^-21 relative per product, the same class as an fp32 FMA chain in another summation order
//     (tests/test_gpu_flat.py bounds it).  The queries are split once per batch (split_tf32_kernel); the corpus k-block
//     is split in shared memory by the consumer warpgroup itself while the previous k-block's MMAs run.
//   * binary queries x binary corpus (K2c): wgmma m64n128k256 .b1 AND + popcount counts the common set bits of a query and a
//     row in s32.  Hamming = popc(q) + popc(y) - 2 and, Jaccard = (or - and) / or with or = popc(q) + popc(y) - and; every
//     term is an integer below 2^24, so the keys are exactly those of binary_scan_kernel (flat_scan.cu).
//
// Replaces faiss::knn_inner_product / knn_L2sqr for nx >= 20 (the BLAS sgemm path) reached from tryBruteForceSearch
// (reference: VectorIndex/Common/BruteForceSearch.h:77-88) and the FLAT Search::VectorIndex::search scan
// (VectorIndex/Common/VIWithDataPart.cpp:926).
//
// One CTA = 128 queries (one query tile for its whole life) x corpus tiles of 256 rows (worker, worker + W, ...).  A tile is
// computed as two N = 128 halves; per half, two wgmma m64n128 (query rows 0..63 / 64..127) per k-step accumulate in the
// registers of one warpgroup.  Each warp of it holds 32 query rows of the fragment, and each lane of the warp owns the top-k
// list of one of them; the warp tests every group of 32 columns from the registers and stages only a group that can enter a
// list (see "hand-off" below).
//   bf16 and binary rows: warps 0..3 and 4..7 are two consumer warpgroups, warpgroup w owns half w of every tile.  A stage of
//               the ring holds the query k-block and the corpus k-block of all 256 rows, so the query k-block is fetched once
//               per tile, not once per half.  The warpgroups share nothing but the ring: each has its own per-warp staging
//               and per-query lists, and a CTA publishes two partial lists per query.
//   fp32 rows:  warps 0..3 are the one consumer warpgroup; it walks both halves, a stage holds one half's corpus k-block
//               (with the hi / lo planes a stage of both halves would leave no room for a ring).
//   next warp   TMA producer (one lane), ring of full / empty mbarriers.
// The key that is ranked is  acc * row_scale[j] + row_bias[j]  (smaller = better):
//   IP: -acc | L2: ||y||^2 - 2 acc (+||q||^2 added at merge) | cosine: -acc / ||y|| | Hamming: popc(y) - 2 and (+popc(q) added
//   at merge);  filtered / out-of-range rows: scale 0, bias +inf.
//   Jaccard is not affine in the count: every group is staged, and the owner maps its counts to keys (jaccard_negkey).
#include <cstdlib>
#include <type_traits>

#include "gemm_common.cuh"

namespace b200 {
namespace gemm {

// Shared-memory layout of gemm_topk_kernel per operand type, ring depth and list placement.
//   [stage 0] .. [stage st - 1]   stage = [A hi][A lo][B (hi after the split) of WG halves][B lo]; lo planes: fp32 rows only
//   per consumer warp: the staging buffer of the hand-off's slow path, [32 columns][32 query rows] floats, swizzled
//   full / empty mbarriers
//   per consumer warpgroup: the 128 per-lane lists, when they are kept in shared memory
template <Operand OP>
struct Op {
    using L = Layout<OP>;   // operand geometry (k-block, planes); the offsets below are this kernel's own
    using Acc = typename std::conditional<OP == Operand::B1, int32_t, float>::type;   // wgmma accumulator type
    static constexpr bool F32X3 = L::F32X3;
    static constexpr int KB = L::KB, MMA_K = L::MMA_K, A_PLANE = L::A_PLANE, B_PLANE = L::B_PLANE, PLANES = L::PLANES;
    static constexpr int WG = gemm_consumer_warpgroups(F32X3);
    // + the TMA producer warp.  With two consumer warpgroups the block is three whole warpgroups: registers are budgeted per
    // warpgroup (65536 / 384 = 168 each), and setmaxnreg then moves the idle share of the producer's to the consumers, which need
    // their 128 accumulators and the epilogue's working set (40 + 2 x 232 = 3 x 168).
    static constexpr int THREADS = WG == 1 ? EPI_THREADS + 32 : 3 * EPI_THREADS;
    static constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;
    static constexpr int B_ROWS = WG * HN;                   // corpus rows per stage (one TMA box)
    static constexpr int PASSES = BN / B_ROWS;               // halves a warpgroup walks per tile
    static constexpr int STAGE_BYTES = PLANES * (A_PLANE + WG * B_PLANE);
    static constexpr int TX_BYTES = PLANES * A_PLANE + WG * B_PLANE;   // what TMA writes (the B lo plane is computed)
    static constexpr int STAGING_BYTES = 32 * 32 * 4;        // per consumer warp
    static constexpr int MAX_ST = F32X3 ? 2 : 3;
    static_assert(MAX_ST <= MAX_STAGES, "barrier arrays");
    __host__ __device__ static constexpr int off_staging(int st) { return st * STAGE_BYTES; }
    __host__ __device__ static constexpr int off_bar(int st) { return off_staging(st) + WG * 4 * STAGING_BYTES; }
    __host__ __device__ static constexpr int off_list(int st) { return off_bar(st) + 256; }
    static constexpr int list_bytes(int k_smem) { return k_smem * EPI_THREADS * 8; }   // one warpgroup's lists
    static size_t smem_bytes(int st, int k_smem) { return (size_t)off_list(st) + (size_t)WG * list_bytes(k_smem) + SMEM_ALIGN_SLACK; }
    static bool lists_fit(int k_smem) { return smem_bytes(2, k_smem) <= (size_t)SMEM_LIMIT; }
    static int stages_for(int k_smem) {
        int st = MAX_ST;
        while (st > 2 && smem_bytes(st, k_smem) > (size_t)SMEM_LIMIT) st--;
        return st;
    }
};

template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

// named barrier of the consumer warpgroup (id 1; 0 is __syncthreads): the fp32 corpus split before the MMAs read it
__device__ __forceinline__ void wg_bar(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(wg + 1) : "memory"); }

// ---- hand-off from the accumulator registers to the per-lane lists ----
// Fragment layout of wgmma m64nN (acc_store): warp w of the warpgroup, lane l holds rows r = 16 w + l / 4 and r + 8 of the
// M = 64 half in d0 (rows 0..63 of the query tile) and the same rows + 64 in d1, columns 8 i + 2 (l % 4) (+ 1).  So warp w
// holds 32 query rows of the tile, and lane L of that warp owns the list of one of them ("slot" L):
//   slot s < 16: row 16 w + s,   slot s >= 16: row 64 + 16 w + (s - 16).
// A lane's four fragment rows r, r + 8, 64 + r, 72 + r ("rho" 0..3) are slots l / 4 + 8 rho.
__device__ __forceinline__ int slot_row(int warp, int slot) { return (slot < 16 ? 0 : 48) + 16 * warp + slot; }

// Group G of 32 columns of the half as negated keys (larger = better, the max-tree form of epilogue_chunk):
// u[8 rho + 2 i + e] = column 8 i + 2 (l % 4) + e of the group, fragment row rho.
//   plain IP (and the AND counts of Jaccard): the score;  side keys: -(acc * scale + bias).
// sc / bi: the side entries of column 32 G + lane of the half (fetched by SHFL).  s32 accumulators (AND counts) hold the bits of
// their fp32 value by now (acc_to_f32).
__device__ __forceinline__ float acc_f32(float x) { return x; }
__device__ __forceinline__ float acc_f32(int32_t x) { return __int_as_float(x); }
template <int G, typename T>
__device__ __forceinline__ void group_keys(float (&u)[32], const T (&d0)[64], const T (&d1)[64], bool side, float sc, float bi, int lane) {
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int x = 4 * (4 * G + i);
        u[2 * i] = acc_f32(d0[x]);
        u[2 * i + 1] = acc_f32(d0[x + 1]);
        u[8 + 2 * i] = acc_f32(d0[x + 2]);
        u[8 + 2 * i + 1] = acc_f32(d0[x + 3]);
        u[16 + 2 * i] = acc_f32(d1[x]);
        u[16 + 2 * i + 1] = acc_f32(d1[x + 1]);
        u[24 + 2 * i] = acc_f32(d1[x + 2]);
        u[24 + 2 * i + 1] = acc_f32(d1[x + 3]);
    }
    if (!side) return;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const int col = 8 * (j >> 1) + 2 * (lane & 3) + (j & 1);
        const float s = __shfl_sync(0xffffffffu, sc, col), b = __shfl_sync(0xffffffffu, bi, col);
#pragma unroll
        for (int rho = 0; rho < 4; rho++) {
            float &x = u[8 * rho + j];
            x = -fmaf(x, s, b);
        }
    }
}

// group_keys for the g of a loop that is not unrolled (the accumulator registers want compile-time indices)
template <int G = 0, typename T>
__device__ __forceinline__ void group_keys_at(int g, float (&u)[32], const T (&d0)[64], const T (&d1)[64], bool side, const float (&sc)[4],
                                              const float (&bi)[4], int lane) {
    if (g == G) group_keys<G>(u, d0, d1, side, sc[G], bi[G], lane);
    else if constexpr (G + 1 < HN / 32) group_keys_at<G + 1>(g, u, d0, d1, side, sc, bi, lane);
}

// Max over the quad of the lane's four fragment-row maxima m[rho], one row per lane (a reduce-scatter in three SHFL): lane l
// ends with the row rho = 2 (l & 1) + (l & 2) / 2, i.e. owner slot l / 4 + 8 rho.
__device__ __forceinline__ float quad_rows_max(const float (&m)[4], int lane) {
    const bool b0 = lane & 1, b1 = lane & 2;
    const float s0 = __shfl_xor_sync(0xffffffffu, b0 ? m[0] : m[2], 1);
    const float s1 = __shfl_xor_sync(0xffffffffu, b0 ? m[1] : m[3], 1);
    const float k0 = fmaxf(b0 ? m[2] : m[0], s0), k1 = fmaxf(b0 ? m[3] : m[1], s1);
    const float s = __shfl_xor_sync(0xffffffffu, b1 ? k0 : k1, 2);
    return fmaxf(b1 ? k1 : k0, s);
}

// x = hi + lo with both parts exactly representable in TF32 (so the result does not depend on how the tensor core
// would round a raw fp32 operand).  hi by truncation: FLT_MAX (the reference's padding value for empty rows,
// MergeTreeVSManager.cpp:1380) stays finite.
__device__ __forceinline__ void split_tf32(uint32_t x, uint32_t &hi, uint32_t &lo) {
    hi = x & 0xffffe000u;
    const float r = __uint_as_float(x) - __uint_as_float(hi);
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lo) : "f"(r));
}

__global__ void split_tf32_kernel(const float *__restrict__ src, int64_t n_src, int d_pad, float *__restrict__ hi,
                                  float *__restrict__ lo, int64_t n_pad) {
    const int64_t total = n_pad * d_pad;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / d_pad;
        uint32_t h = 0, l = 0;
        if (r < n_src) split_tf32(__float_as_uint(src[i]), h, l);
        hi[i] = __uint_as_float(h);
        lo[i] = __uint_as_float(l);
    }
}

template <Operand OP>
__global__ void __launch_bounds__(Op<OP>::THREADS, 1)
gemm_topk_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_qlo,
                 const __grid_constant__ CUtensorMap map_c, const GemmTopkParams p) {
    using O = Op<OP>;
    const int STAGES = p.stages;
    extern __shared__ unsigned char smem_dyn[];
    // 1024-byte aligned, derived from smem_dyn by an offset so that the compiler keeps the shared address space
    unsigned char *smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
    uint64_t *full_bar = reinterpret_cast<uint64_t *>(smem + O::off_bar(STAGES));
    uint64_t *empty_bar = full_bar + MAX_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qt = blockIdx.x % p.q_tiles;
    const int worker = blockIdx.x / p.q_tiles;
    const int W = gridDim.x / p.q_tiles;  // the host launches a multiple of q_tiles CTAs
    const int64_t n_tiles = (p.n + BN - 1) / BN;
    const int kb_count = (p.d_pad + O::KB - 1) / O::KB;

    if (warp == O::WG * 4 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_q)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_c)) : "memory");
        for (int i = 0; i < STAGES; i++) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], O::WG * 4);  // one arrival per consumer warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp >= O::WG * 4) {
        if constexpr (O::WG == 2) setmaxnreg_dec<O::PRODUCER_REGS>();
        if (warp != O::WG * 4) return;   // the rest of the producer's warpgroup only hands over its registers
        // ===================== TMA producer =====================
        int stage = 0;
        uint32_t phase = 0;
        int ordinal = 0;
        bool pacing = p.progress != nullptr;
        for (int64_t t = worker; t < n_tiles; t += W, ordinal++) {
            // Pacing: the CTAs that stream the SAME corpus tiles for different query tiles stay within `sync_slack`
            // tiles of each other, so a tile is fetched from HBM once and served to the others from L2.  Only pacing, no
            // data dependency: plain volatile counters.  Bounded wait (~50 us): if the sharers are not co-resident
            // (another kernel holds SMs) pacing is dropped instead of risking a co-residency deadlock.  Lane g reads sharer g's
            // counter, so a check is one L2 round trip rather than one per sharer: a tile's check has to end within the few
            // k-blocks the ring holds ahead of the consumers.
            if (pacing) {
                volatile int *prog = p.progress + (size_t)worker * p.q_tiles;
                if (lane == 0) prog[qt] = ordinal + 1;
                __syncwarp();
                int spins = 0;
                while (spins < 256) {
                    bool behind = false;
                    for (int g = lane; g < p.q_tiles; g += 32) behind |= prog[g] < ordinal + 1 - p.sync_slack;
                    if (!__any_sync(0xffffffffu, behind)) break;
                    __nanosleep(200);
                    spins++;
                }
                if (spins >= 256) {
                    if (lane == 0) prog[qt] = 0x7fffffff;  // never hold anybody back again
                    pacing = false;
                }
            }
            __syncwarp();
            for (int h = 0; h < O::PASSES; h++) {
                for (int kb = 0; kb < kb_count; kb++) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    if (elect_one()) {
                        unsigned char *st = smem + stage * O::STAGE_BYTES;
                        mbar_arrive_expect_tx(&full_bar[stage], O::TX_BYTES);
                        tma_load_2d(&map_q, &full_bar[stage], st, kb * O::KB, qt * BM);
                        if constexpr (O::F32X3) tma_load_2d(&map_qlo, &full_bar[stage], st + O::A_PLANE, kb * O::KB, qt * BM);
                        tma_load_2d(&map_c, &full_bar[stage], st + O::PLANES * O::A_PLANE, kb * O::KB, (int)(t * BN + h * O::B_ROWS));
                    }
                    __syncwarp();
                    if (++stage == STAGES) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            }
        }
    } else {
        // ===================== consumer warpgroup: MMAs, then the fused top-k =====================
        if constexpr (O::WG == 2) setmaxnreg_inc<O::CONSUMER_REGS>();
        const int wg = threadIdx.x / EPI_THREADS;   // with two warpgroups: the half of every tile this one owns
        const int tid = threadIdx.x % EPI_THREADS;  // thread of the warpgroup = slot of its list in the interleaved lists
        const int wwarp = tid >> 5;                 // warp of the warpgroup
        const int qrow = slot_row(wwarp, lane);     // query row (inside the tile) of this lane's list
        const bool use_side = p.row_scale || p.row_bias || p.alive || p.scale_const != -1.f;
        const bool jaccard = OP == Operand::B1 && p.jaccard;
        // everything the epilogue writes is private to the warp: the two warpgroups drift apart by up to the ring's depth
        float *staging = reinterpret_cast<float *>(smem + O::off_staging(STAGES) + (wg * 4 + wwarp) * O::STAGING_BYTES);
        const uint32_t staging_s = smem_u32(staging);
        // partial list  worker * WG + wg  of query tile qt (the merge reads [list][nq_pad][k])
        const size_t producer = ((size_t)worker * O::WG + wg) * p.q_tiles + qt;
        ThreadTopK list;
        list.n = 0;
        list.worst = 0;
        // rows past the batch (zero padding up to the tile size) must never pay for the slow path: nothing beats -FLT_MAX
        list.thr_key = (qt * BM + qrow < p.nq_valid) ? FLT_MAX : -FLT_MAX;
        list.thr_id = 0;
        const int list_cap = list_cap_for(p.k);
        if (p.lists_in_smem) {
            unsigned char *lists = smem + O::off_list(STAGES) + wg * O::list_bytes(list_cap);
            list_bind(list, reinterpret_cast<float *>(lists), reinterpret_cast<uint32_t *>(lists + O::list_bytes(list_cap) / 2), tid, p.k);
        } else {
            list_bind(list, p.list_keys_gmem + producer * list_cap * EPI_THREADS, p.list_ids_gmem + producer * list_cap * EPI_THREADS,
                      tid, p.k);
        }
        const int q = qt * BM + qrow;   // this lane's query in the batch
        const bool live = q < p.nq_valid;
        // binary Jaccard: popc(q) of this lane's query row (0 for padding rows)
        const int pq = (jaccard && live) ? (int)p.q_popc[q] : 0;
        const uint32_t smem0 = smem_u32(smem);
        int stage = 0;
        uint32_t phase = 0;
        typename O::Acc d0[64], d1[64];
        for (int64_t t = worker; t < n_tiles; t += W) {
            const int64_t n0 = t * BN;
            const bool tail = n0 + BN > p.n;
            for (int pass = 0; pass < O::PASSES; pass++) {
                const int h = O::WG == 1 ? pass : wg;   // the half of the tile
                // the query's shared bound: the best k-th key any of its lists has published (in flight during the MMAs)
                const uint32_t bound_u = live ? __ldcg(p.query_bound + q) : 0xffffffffu;
                // side entries of columns 32 g + lane of the half (in flight during the MMAs)
                float sc[HN / 32] = {}, bi[HN / 32] = {};
                if (use_side) {
#pragma unroll
                    for (int g = 0; g < HN / 32; g++) {
                        const int64_t r = n0 + h * HN + 32 * g + lane;
                        bool ok = r < p.n;
                        if (ok && p.alive) ok = (p.alive[r >> 3] >> (r & 7)) & 1;
                        sc[g] = ok ? (p.row_scale ? p.row_scale[r] : p.scale_const) : 0.f;
                        bi[g] = ok ? (p.row_bias ? p.row_bias[r] : 0.f) : __int_as_float(0x7f800000);
                    }
                }
                int prev = -1;
                for (int kb = 0; kb < kb_count; kb++) {
                    mbar_wait(&full_bar[stage], phase);
                    const uint32_t st = smem0 + stage * O::STAGE_BYTES;
                    if constexpr (O::F32X3) {
                        // corpus k-block -> (y_hi in place, y_lo in the 4th plane); same swizzled offsets
                        uint4 *b = reinterpret_cast<uint4 *>(smem + stage * O::STAGE_BYTES + 2 * O::A_PLANE);
                        uint4 *bl = b + O::B_PLANE / 16;
#pragma unroll
                        for (int i = 0; i < O::B_PLANE / 16 / EPI_THREADS; i++) {
                            const uint4 raw = b[tid + i * EPI_THREADS];
                            uint4 hi, lo;
                            split_tf32(raw.x, hi.x, lo.x);
                            split_tf32(raw.y, hi.y, lo.y);
                            split_tf32(raw.z, hi.z, lo.z);
                            split_tf32(raw.w, hi.w, lo.w);
                            b[tid + i * EPI_THREADS] = hi;
                            bl[tid + i * EPI_THREADS] = lo;
                        }
                        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic stores -> wgmma operand reads
                        wg_bar(wg);
                    }
                    wgmma_fence();
                    if constexpr (O::F32X3) {
                        const uint64_t ahi = make_smem_desc(st), alo = make_smem_desc(st + O::A_PLANE);
                        const uint64_t b = make_smem_desc(st + 2 * O::A_PLANE), blo = make_smem_desc(st + 2 * O::A_PLANE + O::B_PLANE);
                        constexpr uint64_t M1 = (64 * 128) >> 4;  // second M half: 64 rows further
#pragma unroll
                        for (int k = 0; k < O::KB / O::MMA_K; k++) {
                            const uint64_t off = (uint64_t)(k * (O::MMA_K * 4 >> 4));
                            const uint32_t acc0 = (kb | k) != 0 ? 1u : 0u;  // small terms first
                            wgmma_tf32_n128(d0, alo + off, b + off, acc0);
                            wgmma_tf32_n128(d1, alo + M1 + off, b + off, acc0);
                            wgmma_tf32_n128(d0, ahi + off, blo + off, 1u);
                            wgmma_tf32_n128(d1, ahi + M1 + off, blo + off, 1u);
                            wgmma_tf32_n128(d0, ahi + off, b + off, 1u);
                            wgmma_tf32_n128(d1, ahi + M1 + off, b + off, 1u);
                        }
                    } else if constexpr (OP == Operand::B1) {
                        const uint64_t a = make_smem_desc(st), b = make_smem_desc(st + O::A_PLANE + wg * O::B_PLANE);
                        constexpr uint64_t M1 = (64 * 128) >> 4;
#pragma unroll
                        for (int k = 0; k < O::KB / O::MMA_K; k++) {
                            const uint64_t off = (uint64_t)(k * (O::MMA_K >> 4));   // 32 bytes per k-step
                            const uint32_t acc0 = (kb | k) != 0 ? 1u : 0u;
                            wgmma_b1_n128(d0, a + off, b + off, acc0);
                            wgmma_b1_n128(d1, a + M1 + off, b + off, acc0);
                        }
                    } else {
                        const uint64_t a = make_smem_desc(st), b = make_smem_desc(st + O::A_PLANE + wg * O::B_PLANE);
                        constexpr uint64_t M1 = (64 * 128) >> 4;
#pragma unroll
                        for (int k = 0; k < O::KB / O::MMA_K; k++) {
                            const uint64_t off = (uint64_t)(k * (O::MMA_K * 2 >> 4));
                            const uint32_t acc0 = (kb | k) != 0 ? 1u : 0u;
                            wgmma_bf16_n128(d0, a + off, b + off, acc0);
                            wgmma_bf16_n128(d1, a + M1 + off, b + off, acc0);
                        }
                    }
                    wgmma_commit();
                    // the previous k-block's MMAs have retired: its stage goes back to the producer
                    wgmma_wait<1>();
                    if (prev >= 0) {
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&empty_bar[prev]);
                    }
                    prev = stage;
                    if (++stage == STAGES) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
                wgmma_wait<0>();
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty_bar[prev]);
                if constexpr (OP == Operand::B1) {
                    // AND counts -> fp32 (exact: below 2^24), once, in place: the hand-off reads them as floats
#pragma unroll
                    for (int i = 0; i < 64; i++) {
                        d0[i] = __float_as_int((float)d0[i]);
                        d1[i] = __float_as_int((float)d1[i]);
                    }
                }
                // Fast path, from the registers: per group of 32 columns each lane reduces its fragment to the best negated
                // key of each of its four rows (28 FMNMX), the quad to one row per lane (3 SHFL), which is tested against the
                // owner's threshold with the non-strict test of epilogue_chunk, and one vote.  Thresholds only tighten, so the
                // ones read before the four tests admit at least what epilogue_chunk will.  The threshold is the smaller of the
                // list's own k-th key and the query's shared bound.  Keys here are absolute per query (the per-query constant is
                // added at the merge), so the bound is exact; a key equal to it is still admitted, so ties keep their
                // smallest-id winner.
                const float bound = bound_u == 0xffffffffu ? FLT_MAX : bound_decode(bound_u);
                const float thr = __shfl_sync(0xffffffffu, fminf(list.thr_key, bound), (lane >> 2) + 8 * (2 * (lane & 1) + ((lane >> 1) & 1)));
                // Jaccard keys are not affine in the count: every group takes the slow path, where the owners key it.
                uint32_t slow = jaccard ? (1u << HN / 32) - 1 : 0;   // groups where some owner of the warp may insert
                if (!jaccard) {
#pragma unroll
                    for (int g = 0; g < HN / 32; g++) {
                        float u[32], m[4];
                        group_keys_at(g, u, d0, d1, use_side, sc, bi, lane);   // g is a constant here
#pragma unroll
                        for (int rho = 0; rho < 4; rho++) {
                            const float *x = u + 8 * rho;
                            m[rho] = fmaxf(fmaxf(fmaxf(x[0], x[1]), fmaxf(x[2], x[3])), fmaxf(fmaxf(x[4], x[5]), fmaxf(x[6], x[7])));
                        }
                        if (__any_sync(0xffffffffu, quad_rows_max(m, lane) >= -thr)) slow |= 1u << g;
                    }
                }
                // Slow path: the warp stages such a group in its buffer, [column j][slot s] at j * 32 + (s ^ 8 ((j / 2) % 4))
                // (conflict-free both for the fragment stores and for the owners' column reads), and each owner runs
                // epilogue_chunk on its 32 columns, parking its keys over the buffer.
#pragma unroll 1
                while (slow) {
                    const int g = __ffs(slow) - 1;
                    slow &= slow - 1;
                    float u[32];
                    group_keys_at(g, u, d0, d1, use_side && !jaccard, sc, bi, lane);
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        const int col = 8 * (j >> 1) + 2 * (lane & 3) + (j & 1);
#pragma unroll
                        for (int rho = 0; rho < 4; rho++) {
                            const uint32_t a = staging_s + 4 * (col * 32 + (((lane >> 2) + 8 * rho) ^ (8 * (lane & 3))));
                            asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(u[8 * rho + j]) : "memory");
                        }
                    }
                    __syncwarp();
                    float v[32];
#pragma unroll
                    for (int j = 0; j < 32; j++) {
                        const uint32_t a = staging_s + 4 * (j * 32 + (lane ^ (8 * ((j >> 1) & 3))));
                        asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v[j]) : "r"(a) : "memory");
                    }
                    __syncwarp();   // every owner holds its row before any parks keys over the buffer
                    if (jaccard) {   // AND counts -> negated keys; column j's side entries are lane j's
                        const float s = g == 0 ? sc[0] : g == 1 ? sc[1] : g == 2 ? sc[2] : sc[3];
                        const float b = g == 0 ? bi[0] : g == 1 ? bi[1] : g == 2 ? bi[2] : bi[3];
#pragma unroll
                        for (int j = 0; j < 32; j++) v[j] = jaccard_negkey(v[j], pq, __shfl_sync(0xffffffffu, s, j), __shfl_sync(0xffffffffu, b, j));
                    }
                    epilogue_chunk<32>(list, v, false, nullptr, nullptr, (uint32_t)(n0 + h * HN + 32 * g), tail, p.n, staging + lane,
                                       bound);
                    __syncwarp();   // ... and the parked keys are read before the next group is staged
                }
                // a full list's k-th key bounds the query's k-th key over all its lists; only finite keys (NaN / inf rows)
                if (live && list.n == list.k && list.thr_key < bound && fabsf(list.thr_key) <= FLT_MAX)
                    atomicMin(p.query_bound + q, bound_encode(list.thr_key));
            }
        }
        // publish this lane's per-query partial list
        float *ok = p.part_keys + (producer * BM + qrow) * p.k;
        uint32_t *oi = p.part_ids + (producer * BM + qrow) * p.k;
        list_publish(list, ok, oi);
    }
}

// 2-D tensor map over row-major [rows][d_pad] (bf16, fp32 or bytes of binary rows), box = [box_rows][one 128-byte row],
// 128-byte swizzle.  fp32: the last k-block may hang over d_pad (TMA zero-fills), so fp32 corpora keep their 16-byte row
// padding.  Binary: rows shorter than 128 bytes and a partial last k-block are zero-filled as well (zero bits add nothing to
// an AND count); the row stride must be a multiple of 16 bytes.
static bool encode_map(CUtensorMap *map, const void *base, int64_t rows, int d_pad, int box_rows, Operand op) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return false;
    const int es = op == Operand::TF32X3 ? 4 : op == Operand::BF16 ? 2 : 1;
    const CUtensorMapDataType type = op == Operand::TF32X3 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                     : op == Operand::BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                                           : CU_TENSOR_MAP_DATA_TYPE_UINT8;
    const cuuint64_t dims[2] = {(cuuint64_t)d_pad, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)d_pad * es};
    const cuuint32_t box[2] = {(cuuint32_t)(128 / es), (cuuint32_t)box_rows};
    const cuuint32_t estr[2] = {1, 1};
    return fn(map, type, 2, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <Operand OP>
static cudaError_t launch(const CUtensorMap &map_q, const CUtensorMap &map_qlo, const CUtensorMap &map_c, const GemmTopkParams &p_in,
                          int grid, cudaStream_t s) {
    using O = Op<OP>;
    GemmTopkParams p = p_in;
    // Per-thread lists sit in shared memory whenever they fit, even when that squeezes the operand ring: every insert rescans
    // the list, and from global scratch that is k L2 round trips.
    const int list_cap = list_cap_for(p.k);
    p.lists_in_smem = O::lists_fit(list_cap) ? 1 : 0;
    const int k_smem = p.lists_in_smem ? list_cap : 0;
    p.stages = O::stages_for(k_smem);
    const size_t smem = O::smem_bytes(p.stages, k_smem);
    auto kern = gemm_topk_kernel<OP>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    kern<<<grid, O::THREADS, smem, s>>>(map_q, map_qlo, map_c, p);
    g_launches++;
    return cudaGetLastError();
}

}  // namespace gemm

int gemm_topk_grid(int q_tiles, int64_t n, int num_sms) {
    const int64_t n_tiles = ceil_div(n, gemm::BN);
    int64_t g = (int64_t)q_tiles * (n_tiles < 1 ? 1 : n_tiles);
    if (g > num_sms) g = num_sms;
    if (g < q_tiles) g = q_tiles;
    return (int)g;
}

cudaError_t launch_split_tf32(const float *src, int64_t n_src, int d_pad, float *hi, float *lo, int64_t n_pad, cudaStream_t s) {
    if (n_pad == 0) return cudaSuccess;
    int64_t b = ceil_div(n_pad * d_pad, 256);
    if (b > 132 * 8) b = 132 * 8;
    gemm::split_tf32_kernel<<<(int)b, 256, 0, s>>>(src, n_src, d_pad, hi, lo, n_pad);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t launch_gemm_topk(const GemmTopkParams &p, int grid, cudaStream_t s, const char **err_detail) {
    *err_detail = nullptr;
    if (grid % p.q_tiles != 0) {
        *err_detail = "grid must be a multiple of q_tiles";
        return cudaErrorInvalidValue;
    }
    CUtensorMap map_q, map_c;
    if (!gemm::encode_map(&map_q, p.queries_bf16, p.nq_pad, p.d_pad, gemm::BM, gemm::Operand::BF16) ||
        !gemm::encode_map(&map_c, p.corpus_bf16, p.n, p.d_pad, gemm::Op<gemm::Operand::BF16>::B_ROWS, gemm::Operand::BF16)) {
        *err_detail = "cuTensorMapEncodeTiled failed";
        return cudaErrorInvalidValue;
    }
    return gemm::launch<gemm::Operand::BF16>(map_q, map_q, map_c, p, grid, s);
}

cudaError_t launch_gemm3_topk(const GemmTopkParams &p, int grid, cudaStream_t s, const char **err_detail) {
    *err_detail = nullptr;
    if (grid % p.q_tiles != 0 || !p.queries_lo) {
        *err_detail = "gemm3: grid must be a multiple of q_tiles, queries_lo set";
        return cudaErrorInvalidValue;
    }
    CUtensorMap map_qhi, map_qlo, map_c;
    if (!gemm::encode_map(&map_qhi, p.queries_bf16, p.nq_pad, p.d_pad, gemm::BM, gemm::Operand::TF32X3) ||
        !gemm::encode_map(&map_qlo, p.queries_lo, p.nq_pad, p.d_pad, gemm::BM, gemm::Operand::TF32X3) ||
        !gemm::encode_map(&map_c, p.corpus_bf16, p.n, p.d_pad, gemm::Op<gemm::Operand::TF32X3>::B_ROWS, gemm::Operand::TF32X3)) {
        *err_detail = "cuTensorMapEncodeTiled failed";
        return cudaErrorInvalidValue;
    }
    return gemm::launch<gemm::Operand::TF32X3>(map_qhi, map_qlo, map_c, p, grid, s);
}

cudaError_t launch_gemm_b1_topk(const GemmTopkParams &p, int grid, cudaStream_t s, const char **err_detail) {
    *err_detail = nullptr;
    if (grid % p.q_tiles != 0 || p.d_pad % 16 != 0 || !p.row_bias || (p.jaccard && !p.q_popc)) {
        *err_detail = "gemm b1: grid must be a multiple of q_tiles, rows a multiple of 16 bytes, popcounts set";
        return cudaErrorInvalidValue;
    }
    CUtensorMap map_q, map_c;
    if (!gemm::encode_map(&map_q, p.queries_bf16, p.nq_pad, p.d_pad, gemm::BM, gemm::Operand::B1) ||
        !gemm::encode_map(&map_c, p.corpus_bf16, p.n, p.d_pad, gemm::Op<gemm::Operand::B1>::B_ROWS, gemm::Operand::B1)) {
        *err_detail = "cuTensorMapEncodeTiled failed";
        return cudaErrorInvalidValue;
    }
    return gemm::launch<gemm::Operand::B1>(map_q, map_q, map_c, p, grid, s);
}

}  // namespace b200
