// ivf_gemm_sm90.cu -- K5: the inverted-file scan as a GROUPED tensor-core top-k.
//
// Replaces the list scan inside Search::VectorIndex<...>::search for the IVF family (IVFFLAT / IVFSQ / IVFPQ / the
// two-stage "MSTG"-class index), reached from VIWithColumnInPart::search (reference:
// src/VectorIndex/Common/VIWithDataPart.cpp:926).  The reference's Faiss scans one (query, list) pair at a time on one
// core.  Here the (query, probed list) pairs of a whole batch are first sorted BY LIST (ivf.cu), so that a list's rows
// are streamed from HBM once for ALL queries that probe it, and the distances of <= 128 such queries x 256 rows are one
// wgmma tile (M = 128 queries, N = 256 rows as two N = 128 halves, K = d): the same fused top-k epilogue as
// ip_gemm_sm90.cu keeps one private k-list per query and the [queries x rows] scores never reach memory.
//
// Work item = (queries [q_begin, q_begin + q_count) of the list-sorted pair array) x (pages [page_begin, +page_count) of
// one list).  Inverted lists are PAGED: a page is 256 consecutive pool rows = exactly one tile, lists grow by
// appending pages (streamed build, no compaction), long lists are split over several items / SMs.
// Persistent CTAs walk items blockIdx.x, blockIdx.x + grid, ... (items are ordered by decreasing work on the host):
//   warps 0..3  consumer warpgroup: wgmma into registers, accumulators staged in shared memory, then the epilogue:
//               thread t = query slot t; key = acc * scale + bias (L2: ||y||^2 - 2 q.y; IP / cosine: -q.y);
//               rows beyond the page fill, filtered rows -> +inf
//   warp 4      TMA producer: A = 128 gathered bf16 query rows (k-block of 64), B = one half page's k-block
//               (PRODUCER_TMA: bf16 rows as stored)
//   warps 5..8  (PRODUCER_PQ / PRODUCER_SQ8) decoder warps: read the half page's codes, look the sub-vectors up in the
//               shared-memory codebook (PQ) or widen int8 (SQ8) and write the 128-byte-swizzled bf16 B tile themselves
// PRODUCER_B1 (binary indexes): A = gathered query bytes, B = a half page's k-block of kb_w <= 128 bytes per row, zero-filled
// by TMA to the 128-byte box; four wgmma m64n128k256 .b1 AND + popcount per k-block and M half (SASS BGMMA), s32 counts
// staged as exact fp32.  Hamming key = popc(y) - 2 and (scale / bias path, popc(q) is the pair constant); Jaccard keys come
// from jaccard_keys32 with popc(q) of the lane's pair, exactly as gemm_topk_kernel<B1> keys them.
// HBM-bound by design: algorithmic bytes = (rows of the probed pages) x payload bytes per row, once per item.
#include <algorithm>
#include <cstdlib>
#include <type_traits>

#include "gemm_common.cuh"
#include "ivf_coop.cuh"
#include "ivf_gemm.h"

namespace b200 {
namespace gemm {

constexpr int IVF_THREADS_TMA = NUM_THREADS;   // consumer warpgroup + producer warp
constexpr int IVF_DEC_WARPS = 4;               // extra decoder warps of the code payloads
constexpr int IVF_THREADS_DEC = IVF_THREADS_TMA + IVF_DEC_WARPS * 32;

// smem: the Layout<Operand::BF16> of gemm_common.cuh.  Code payloads add a codebook region behind the lists.

template <int PRODUCER, int DSUB>
__global__ void __launch_bounds__(PRODUCER == IVF_PRODUCER_PQ || PRODUCER == IVF_PRODUCER_SQ8 ? IVF_THREADS_DEC : IVF_THREADS_TMA, 1)
ivf_gemm_topk_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_c, const IvfGemmParams p) {
    using C = Layout<Operand::BF16>;   // Layout<Operand::B1> has the same bytes
    constexpr bool B1 = PRODUCER == IVF_PRODUCER_B1;
    const int STAGES = p.stages;
    extern __shared__ unsigned char smem_dyn[];
    unsigned char *smem = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    unsigned char *sA = smem;                  // stage s: A at sA + s * STAGE_BYTES, B A_PLANE bytes further
    unsigned char *sB = smem + C::A_PLANE;
    float *acc = reinterpret_cast<float *>(smem + C::off_acc(STAGES));
    float *side_scale = reinterpret_cast<float *>(smem + C::off_side(STAGES));
    float *side_bias = side_scale + BN;
    uint64_t *full_bar = reinterpret_cast<uint64_t *>(smem + C::off_bar(STAGES));
    uint64_t *empty_bar = full_bar + MAX_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int kb_count = B1 ? p.d_pad / p.kb_w : p.d_pad / BK;
    constexpr bool DEC = PRODUCER == IVF_PRODUCER_PQ || PRODUCER == IVF_PRODUCER_SQ8;
    const int n_items = *p.n_items_ptr;

    if (warp == 4 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_q)) : "memory");
        if (!DEC) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_c)) : "memory");
        for (int i = 0; i < STAGES; i++) {
            // full: the TMA transaction (+ one arrival per decoder warp that wrote its quarter of the B tile)
            mbar_init(&full_bar[i], DEC ? 1 + IVF_DEC_WARPS : 1);
            mbar_init(&empty_bar[i], 4);   // one arrival per consumer warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (DEC) {
        // codebook -> shared memory (behind the per-thread lists): PQ [m][256][dsub] bf16; SQ8 has none
        if (PRODUCER == IVF_PRODUCER_PQ) {
            uint4 *dst = reinterpret_cast<uint4 *>(smem + p.codebook_smem_off);
            const uint4 *src = reinterpret_cast<const uint4 *>(p.codebook_bf16);
            for (int i = threadIdx.x; i < p.codebook_bytes / 16; i += blockDim.x) dst[i] = src[i];
        }
    }
    __syncthreads();

    if (warp == 4) {
        // ===================== TMA producer =====================
        int stage = 0;
        uint32_t phase = 0;
        for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
            const IvfGemmItem item = p.items[it];
            for (uint32_t j = 0; j < item.page_count; j++) {
                const uint32_t page = p.list_pages[item.page_begin + j];
                for (int h = 0; h < BN / HN; h++) {
                    for (int kb = 0; kb < kb_count; kb++) {
                        mbar_wait(&empty_bar[stage], phase ^ 1);
                        if (elect_one()) {
                            mbar_arrive_expect_tx(&full_bar[stage], DEC ? C::A_PLANE : C::TX_BYTES);
                            tma_load_2d(&map_q, &full_bar[stage], sA + stage * C::STAGE_BYTES, kb * (B1 ? Layout<Operand::B1>::KB : BK), (int)item.q_begin);
                            // bf16 pages are stored k-block-major ([page][k-block][256 rows][64]): one B tile = 32 KB CONTIGUOUS in HBM
                            // (binary pages: [page][k-block][256 rows][kb_w bytes], the same tile coordinates)
                            if (!DEC)
                                tma_load_2d(&map_c, &full_bar[stage], sB + stage * C::STAGE_BYTES, 0,
                                            (int)((page * (uint32_t)kb_count + kb) * (uint32_t)BN + h * HN));
                        }
                        __syncwarp();
                        if (++stage == STAGES) {
                            stage = 0;
                            phase ^= 1;
                        }
                    }
                }
            }
        }
    } else if (warp < 4) {
        // ===================== consumer warpgroup: MMAs, then the fused top-k, one list per (item, query slot) =====================
        const int quarter = warp;
        const int row = threadIdx.x;                  // query slot inside the item
        float *scratch = reinterpret_cast<float *>(smem + C::off_scratch(STAGES)) + row;
        ThreadTopK list;
        const int list_cap = list_cap_for(p.k);
        if (p.lists_in_smem)
            list_bind(list, reinterpret_cast<float *>(smem + C::off_list(STAGES)),
                      reinterpret_cast<uint32_t *>(smem + C::off_list(STAGES) + (size_t)list_cap * EPI_THREADS * 4), row, p.k);
        else
            list_bind(list, p.list_keys_gmem + (size_t)blockIdx.x * list_cap * EPI_THREADS,
                      p.list_ids_gmem + (size_t)blockIdx.x * list_cap * EPI_THREADS, row, p.k);
        // cooperative lists (items with <= kCoopMax queries), owned by warp 0 (query slots 0..31)
        const CoopSmem cs = coop_smem_carve(smem + p.coop_smem_off, smem + C::off_scratch(STAGES), p.k);
        float *tile_row = cs.tilebuf + (size_t)(lane < kCoopMax ? lane : 0) * kTileBufStride;
        const uint32_t sa0 = smem_u32(sA), sb0 = smem_u32(sB);
        int stage = 0;
        uint32_t phase = 0;
        typename std::conditional<B1, int32_t, float>::type d0[64], d1[64];
        for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
            const IvfGemmItem item = p.items[it];
            const bool coop = item.q_count <= (uint32_t)p.coop_enabled;   // 0 = off, else the largest cooperative item (<= kCoopMax)
            // binary Jaccard: popc(q) of this lane's pair (0 for slots without a query)
            const int pq = (B1 && p.jaccard && (uint32_t)row < item.q_count) ? (int)p.pair_popc[item.q_begin + row] : 0;
            list.n = 0;
            list.worst = 0;
            list.thr_key = ((uint32_t)row < item.q_count) ? FLT_MAX : -FLT_MAX;   // padding slots never enter the slow path
            list.thr_id = 0;
            float coop_thr = list.thr_key;
            // shared per-query bound (nprobe > 1): this lane's query and the constant that makes its keys absolute
            uint32_t *bound_slot = nullptr;
            float pc = 0.f, last_pub = FLT_MAX;
            if (p.query_bound && (uint32_t)row < item.q_count) {
                bound_slot = p.query_bound + p.sorted_pair[item.q_begin + row] / (uint32_t)p.nprobe;
                pc = p.pair_const ? p.pair_const[item.q_begin + row] : 0.f;
            }
            if (coop && quarter == 0) {
                if (lane < kCoopMax) {
                    CoopState st;
                    st.n = 0; st.thr_key = FLT_MAX; st.thr_id = 0; st.buf = 0;
                    cs.state[lane] = st;
                }
                __syncwarp();
            }
            // Only slots 0 .. q_count - 1 carry queries.  Every other slot multiplies whatever rows follow in the gathered
            // query buffer (other pairs' queries, or never-written slack): their keys may be anything, -inf included, so they are
            // kept away from the tile buffer by a NaN threshold (no comparison with NaN is true) -- -FLT_MAX is not enough.
            if (coop && !(quarter == 0 && (uint32_t)lane < item.q_count)) coop_thr = __int_as_float(0x7fc00000);
            for (uint32_t j = 0; j < item.page_count; j++) {
                const uint32_t page = p.list_pages[item.page_begin + j];
                const uint32_t row0 = page * (uint32_t)BN;
                const uint32_t valid = item.row_limit - j * (uint32_t)BN;   // rows of the list left from this page on (>= 1)
                uint32_t bound_u = 0xffffffffu;
                if (bound_slot) bound_u = __ldcg(bound_slot);   // in flight during the MMAs
                // this page's side entries (in flight during the MMAs; written after the first barrier below)
                float sc[BN / EPI_THREADS], bi[BN / EPI_THREADS];
#pragma unroll
                for (int i = 0; i < BN / EPI_THREADS; i++) {
                    const int c = row + i * EPI_THREADS;
                    bool ok = (uint32_t)c < valid;
                    if (ok && p.alive) {
                        const uint32_t id = p.row_ids[row0 + c];
                        ok = (p.alive[id >> 3] >> (id & 7)) & 1;
                    }
                    sc[i] = ok ? p.scale_const : 0.f;
                    bi[i] = ok ? (p.row_bias ? p.row_bias[row0 + c] : 0.f) : __int_as_float(0x7f800000);
                }
                uint32_t chunk_mask = 0;
                for (int h = 0; h < BN / HN; h++) {
                    int prev = -1;
                    for (int kb = 0; kb < kb_count; kb++) {
                        mbar_wait(&full_bar[stage], phase);
                        wgmma_fence();
                        const uint64_t a = make_smem_desc(sa0 + stage * C::STAGE_BYTES), b = make_smem_desc(sb0 + stage * C::STAGE_BYTES);
                        constexpr uint64_t M1 = (64 * 128) >> 4;   // second M half: 64 rows further
                        if constexpr (B1) {
                            using L = Layout<Operand::B1>;
#pragma unroll
                            for (int k = 0; k < L::KB / L::MMA_K; k++) {
                                const uint64_t off = (uint64_t)(k * (L::MMA_K >> 4));   // 32 bytes per k-step
                                wgmma_b1_n128(d0, a + off, b + off, (kb | k) != 0 ? 1u : 0u);
                                wgmma_b1_n128(d1, a + M1 + off, b + off, (kb | k) != 0 ? 1u : 0u);
                            }
                        } else {
#pragma unroll
                            for (int k = 0; k < BK / UMMA_K; k++) {
                                const uint64_t off = (uint64_t)(k * (UMMA_K * 2 >> 4));
                                wgmma_bf16_n128(d0, a + off, b + off, (kb | k) != 0 ? 1u : 0u);
                                wgmma_bf16_n128(d1, a + M1 + off, b + off, (kb | k) != 0 ? 1u : 0u);
                            }
                        }
                        wgmma_commit();
                        wgmma_wait<1>();   // the previous k-block's MMAs have retired: its stage goes back to the producer
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
                    // the bound in this item's key space, a few ulps loose (the merge adds pair_const back in fp32); superset-safe
                    float ext = FLT_MAX;
                    if (bound_u != 0xffffffffu) {
                        const float g = bound_decode(bound_u);
                        ext = g - pc;
                        ext += (fabsf(ext) + fabsf(pc) + fabsf(g)) * 4e-7f;
                    }
                    const float coop_flt = (coop_thr != coop_thr) ? coop_thr : fminf(coop_thr, ext);   // NaN (no query on this lane) stays NaN
#pragma unroll
                    for (int q = 0; q < HN / ACC_COLS; q++) {
                        wg_bar();   // every slot's reads of the previous staging (accumulators, side arrays, tile buffer) are done
                        if (h == 0 && q == 0) {
#pragma unroll
                            for (int i = 0; i < BN / EPI_THREADS; i++) {
                                side_scale[row + i * EPI_THREADS] = sc[i];
                                side_bias[row + i * EPI_THREADS] = bi[i];
                            }
                        }
                        if (q == 0) acc_store<0>(acc, d0, d1);
                        else acc_store<1>(acc, d0, d1);
                        wg_bar();
#pragma unroll 1
                        for (int cc = 0; cc < ACC_COLS / 32; cc++) {
                            float v[32];
                            acc_load32(acc, row, cc * 32, v);
                            const int chunk = (h * HN + q * ACC_COLS) / 32 + cc;
                            if (B1 && p.jaccard) {
                                // negated keys (max-tree form of epilogue_chunk); the cooperative form takes the keys themselves
                                jaccard_keys32(v, pq, side_scale + chunk * 32, side_bias + chunk * 32);
                                if (coop) {
#pragma unroll
                                    for (int j = 0; j < 32; j++) v[j] = -v[j];
                                    coop_stage_chunk<false>(coop_flt, v, nullptr, nullptr, tile_row, chunk, chunk_mask, lane);
                                } else {
                                    epilogue_chunk(list, v, false, nullptr, nullptr, row0 + chunk * 32, false, 0, scratch, ext);
                                }
                            } else if (coop) {
                                coop_stage_chunk(coop_flt, v, side_scale + chunk * 32, side_bias + chunk * 32, tile_row, chunk, chunk_mask, lane);
                            } else {
                                epilogue_chunk(list, v, true, side_scale + chunk * 32, side_bias + chunk * 32, row0 + chunk * 32, false, 0, scratch, ext);
                            }
                        }
                    }
                }
                if (coop && quarter == 0) coop_merge_tile(cs, p.k, (int)item.q_count, chunk_mask, row0, lane, coop_thr);
                // publish: a full list's k-th key bounds the query's k-th key over all its lists
                if (bound_slot) {
                    const float mine_thr = coop ? coop_thr : (list.n == list.k ? list.thr_key : FLT_MAX);
                    if (mine_thr < last_pub) {
                        last_pub = mine_thr;
                        atomicMin(bound_slot, bound_encode(mine_thr + pc));
                    }
                }
            }
            // publish this (item, query slot)'s partial list: pool rows mapped to row ids, worst kept key aside
            if (coop) {
                if (quarter == 0) {
                    __syncwarp();
                    for (uint32_t sl = 0; sl < item.q_count; sl++) {
                        const size_t part = (size_t)p.pair_part_base[item.q_begin + sl] + item.chunk;
                        const CoopState st = cs.state[sl];
                        const float *lkeys = cs.keys[st.buf] + (size_t)sl * p.k;
                        const uint32_t *lids = cs.ids[st.buf] + (size_t)sl * p.k;
                        for (int e = lane; e < p.k; e += 32) {
                            const bool have = e < st.n;
                            p.part_keys[part * p.k + e] = have ? lkeys[e] : FLT_MAX;
                            p.part_ids[part * p.k + e] = have ? p.row_ids[lids[e]] : kNoId;
                        }
                        if (lane == 0) p.part_worst[part] = st.n == p.k ? st.thr_key : FLT_MAX;
                    }
                    __syncwarp();
                }
            } else if ((uint32_t)row < item.q_count) {
                const size_t part = (size_t)p.pair_part_base[item.q_begin + row] + item.chunk;
                float *ok = p.part_keys + part * p.k;
                uint32_t *oi = p.part_ids + part * p.k;
                for (int e = 0; e < p.k; e++) {
                    const bool have = e < list.n;
                    ok[e] = have ? list.keys[e * EPI_THREADS] : FLT_MAX;
                    oi[e] = have ? p.row_ids[list.ids[e * EPI_THREADS]] : kNoId;
                }
                p.part_worst[part] = list.n == p.k ? list.thr_key : FLT_MAX;
            }
        }
    } else if (DEC) {
        // ===================== decoder warps: codes -> bf16 B tile (128-byte swizzled, K-major) =====================
        // warp w decodes rows [w * 32, w * 32 + 32) of the half page; a lane owns one row and writes its 8 16-byte
        // chunks of the k-block: chunk c of row r lives at r * 128 + ((c ^ (r & 7)) << 4) inside the 8-row / 1024-byte atoms
        const int dw = warp - 5;
        int stage = 0;
        uint32_t phase = 0;
        const unsigned char *cb = smem + p.codebook_smem_off;
        for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
            const IvfGemmItem item = p.items[it];
            for (uint32_t j = 0; j < item.page_count; j++) {
                const uint32_t page = p.list_pages[item.page_begin + j];
                const uint8_t *codes = p.codes + (size_t)page * BN * p.code_bytes;
                {
                    // The code loads below are consumed right away: without help every (k-block, row pass) waits one HBM
                    // latency.  Pull the NEXT page of this CTA's walk (codes and row biases) into L2 while this one is decoded.
                    uint32_t next_page = 0xffffffffu;
                    if (j + 1 < item.page_count) next_page = p.list_pages[item.page_begin + j + 1];
                    else if (it + (int)gridDim.x < n_items) next_page = p.list_pages[p.items[it + gridDim.x].page_begin];
                    if (next_page != 0xffffffffu) {
                        const unsigned char *nc = p.codes + (size_t)next_page * BN * p.code_bytes;
                        const int lines = (BN * p.code_bytes + 127) >> 7;
                        for (int l = dw * 32 + lane; l < lines; l += 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(nc + (size_t)l * 128));
                        if (p.row_bias && dw == 0 && lane < (BN * 4) / 128)
                            asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const unsigned char *>(p.row_bias + (size_t)next_page * BN) + lane * 128));
                    }
                }
                for (int h = 0; h < BN / HN; h++) {
                    for (int kb = 0; kb < kb_count; kb++) {
                        mbar_wait(&empty_bar[stage], phase ^ 1);
                        unsigned char *bt = sB + stage * C::STAGE_BYTES;
                        // this lane's row of the half tile (page row h * HN + r; the same swizzle phase)
                        const int r = dw * 32 + lane;
                        uint4 raw[4];
                        {
                            constexpr int LD_BYTES = PRODUCER == IVF_PRODUCER_SQ8 ? BK : BK / (DSUB > 0 ? DSUB : 1);   // code bytes per row and k-block
                            const int boff = kb * LD_BYTES;
                            const uint8_t *cr = codes + (size_t)(h * HN + r) * p.code_bytes + boff;
                            if (LD_BYTES >= 16) {
#pragma unroll
                                for (int t = 0; t < LD_BYTES / 16; t++)
                                    raw[t] = (boff + t * 16 < p.code_bytes) ? *reinterpret_cast<const uint4 *>(cr + t * 16)
                                                                            : (PRODUCER == IVF_PRODUCER_SQ8 ? make_uint4(0x80808080u, 0x80808080u, 0x80808080u, 0x80808080u)
                                                                                                            : make_uint4(0, 0, 0, 0));
                            } else {
                                const uint2 v = (boff < p.code_bytes) ? *reinterpret_cast<const uint2 *>(cr) : make_uint2(0, 0);
                                raw[0] = make_uint4(v.x, v.y, 0, 0);
                            }
                        }
                        {
                            unsigned char *rowp = bt + (r >> 3) * 1024 + (r & 7) * 128;
                            if (PRODUCER == IVF_PRODUCER_SQ8) {
                                // 64 int8 codes of this k-block -> 64 bf16 (exact: |code| <= 127); query side carries the scales
#pragma unroll
                                for (int c4 = 0; c4 < 4; c4++) {
                                    const uint4 w = raw[c4];
                                    const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
                                    uint32_t o[8];
#pragma unroll
                                    for (int b = 0; b < 4; b++) {
                                        // bytes are offset-binary (value + 128).  No I2F (quarter-rate pipe: 196 k conversions per
                                        // page would take longer than the page's HBM time): a byte dropped into the mantissa of 2^23
                                        // is the float 8388608 + byte, one FADD removes the offset exactly, and the upper halves of
                                        // two floats are the two bf16 (|value| <= 128 is exact in bf16).  PRMT + FADD + 1/2 PRMT each.
                                        const float f0 = __uint_as_float(__byte_perm(ww[b], 0x4B000000u, 0x7440)) - 8388736.f;
                                        const float f1 = __uint_as_float(__byte_perm(ww[b], 0x4B000000u, 0x7441)) - 8388736.f;
                                        const float f2 = __uint_as_float(__byte_perm(ww[b], 0x4B000000u, 0x7442)) - 8388736.f;
                                        const float f3 = __uint_as_float(__byte_perm(ww[b], 0x4B000000u, 0x7443)) - 8388736.f;
                                        o[b * 2] = __byte_perm(__float_as_uint(f0), __float_as_uint(f1), 0x7632);
                                        o[b * 2 + 1] = __byte_perm(__float_as_uint(f2), __float_as_uint(f3), 0x7632);
                                    }
                                    const int c0 = c4 * 2;
                                    *reinterpret_cast<uint4 *>(rowp + (((c0) ^ (r & 7)) << 4)) = make_uint4(o[0], o[1], o[2], o[3]);
                                    *reinterpret_cast<uint4 *>(rowp + (((c0 + 1) ^ (r & 7)) << 4)) = make_uint4(o[4], o[5], o[6], o[7]);
                                }
                            } else {
                                // PQ: dims [kb * 64, kb * 64 + 64) = sub-quantisers [kb * 64 / DSUB, ...), each code byte selects
                                // DSUB bf16 values of the shared-memory codebook [m][256][DSUB]; the codes of one k-block are
                                // NSUB consecutive bytes of the row (row stride and offsets are multiples of 16 / NSUB)
                                constexpr int NSUB = BK / (DSUB > 0 ? DSUB : 1);   // 64, 32, 16, 8 codes per k-block
                                constexpr int BYTES_PER = (DSUB > 0 ? DSUB : 1) * 2;
                                const int j0 = kb * NSUB;
                                uint32_t cw[NSUB / 4];
                                if (NSUB >= 16) {
#pragma unroll
                                    for (int t = 0; t < NSUB / 16; t++) {
                                        const uint4 v = raw[t];
                                        cw[t * 4] = v.x; cw[t * 4 + 1] = v.y; cw[t * 4 + 2] = v.z; cw[t * 4 + 3] = v.w;
                                    }
                                } else {
                                    cw[0] = raw[0].x; cw[1] = raw[0].y;
                                }
                                constexpr int PER_CHUNK_F = 16 / BYTES_PER;
                                const int valid = min(NSUB, p.m - j0);          // sub-quantisers of this k-block that exist
                                if (valid % PER_CHUNK_F == 0) {
                                    // Fast form (whole 16-byte chunks valid or absent): 32-bit shared addresses and ld.shared, one
                                    // predicate per chunk (64-bit generic addresses and a predicate per code would dominate the
                                    // decoder's issue slots at dsub = 1).
                                    const int valid_chunks = valid > 0 ? valid / PER_CHUNK_F : 0;
                                    const uint32_t cb_s = smem_u32(cb) + (uint32_t)j0 * 256u * BYTES_PER;
#pragma unroll
                                    for (int chunk = 0; chunk < NSUB / PER_CHUNK_F; chunk++) {
                                        uint32_t w0 = 0, w1 = 0, w2 = 0, w3 = 0;
                                        if (chunk < valid_chunks) {
#pragma unroll
                                            for (int t = 0; t < PER_CHUNK_F; t++) {
                                                const int s = chunk * PER_CHUNK_F + t;
                                                const uint32_t byte = __byte_perm(cw[s >> 2], 0, 0x4440 | (s & 3));
                                                const uint32_t addr = cb_s + byte * BYTES_PER + (uint32_t)s * 256u * BYTES_PER;
                                                if (DSUB == 8) {
                                                    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(w0), "=r"(w1), "=r"(w2), "=r"(w3) : "r"(addr));
                                                } else if (DSUB == 4) {
                                                    uint32_t a0, a1;
                                                    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(a0), "=r"(a1) : "r"(addr));
                                                    if (t == 0) { w0 = a0; w1 = a1; } else { w2 = a0; w3 = a1; }
                                                } else if (DSUB == 2) {
                                                    uint32_t a0;
                                                    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(a0) : "r"(addr));
                                                    if (t == 0) w0 = a0; else if (t == 1) w1 = a0; else if (t == 2) w2 = a0; else w3 = a0;
                                                } else {
                                                    uint32_t a0;
                                                    asm volatile("ld.shared.u16 %0, [%1];" : "=r"(a0) : "r"(addr));
                                                    uint32_t &dst = t < 2 ? w0 : t < 4 ? w1 : t < 6 ? w2 : w3;
                                                    dst = (t & 1) ? __byte_perm(dst, a0, 0x5410) : a0;
                                                }
                                            }
                                        }
                                        *reinterpret_cast<uint4 *>(rowp + ((chunk ^ (r & 7)) << 4)) = make_uint4(w0, w1, w2, w3);
                                    }
                                } else {
                                    uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
                                    for (int s = 0; s < NSUB; s++) {
                                        const int jj = j0 + s;
                                        const uint32_t code = (cw[s >> 2] >> ((s & 3) * 8)) & 255u;
                                        constexpr int PER_CHUNK = 16 / BYTES_PER;      // look-ups per 16-byte chunk
                                        const int slot = s % PER_CHUNK;
                                        if (jj < p.m) {
                                            const unsigned char *e = cb + ((size_t)jj * 256 + code) * BYTES_PER;
                                            if (DSUB == 8) {
                                                const uint4 v = *reinterpret_cast<const uint4 *>(e);
                                                w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w;
                                            } else if (DSUB == 4) {
                                                const uint2 v = *reinterpret_cast<const uint2 *>(e);
                                                w[slot * 2] = v.x; w[slot * 2 + 1] = v.y;
                                            } else if (DSUB == 2) {
                                                w[slot] = *reinterpret_cast<const uint32_t *>(e);
                                            } else {
                                                const uint32_t v = *reinterpret_cast<const uint16_t *>(e);
                                                if (slot & 1) w[slot >> 1] |= v << 16; else w[slot >> 1] = v;
                                            }
                                        }
                                        if (slot == PER_CHUNK - 1) {
                                            const int chunk = s / PER_CHUNK;
                                            *reinterpret_cast<uint4 *>(rowp + ((chunk ^ (r & 7)) << 4)) = make_uint4(w[0], w[1], w[2], w[3]);
                                            w[0] = w[1] = w[2] = w[3] = 0;
                                        }
                                    }
                                }
                            }
                        }
                        // generic-proxy writes -> visible to the async proxy (wgmma reads smem through it)
                        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&full_bar[stage]);
                        if (++stage == STAGES) {
                            stage = 0;
                            phase ^= 1;
                        }
                    }
                }
            }
        }
    }
}

// Dynamic shared memory of the scan with `st` ring stages, k_smem per-thread list slots in shared memory and a PQ codebook
// of codebook_bytes (0 for the other payloads), cooperative lists not counted: ring, accumulator staging, side arrays,
// barriers, epilogue scratch, lists, codebook, the 1 KB alignment slack and 48 bytes of kernel-side slack.
static int ivf_smem_need(int st, int k_smem, int codebook_bytes) {
    return Layout<Operand::BF16>::off_list(st) + k_smem * EPI_THREADS * 8 + (int)round_up(codebook_bytes, 1024) + SMEM_ALIGN_SLACK + 48;
}

template <int PRODUCER, int DSUB>
static cudaError_t launch_ivf(const CUtensorMap &map_q, const CUtensorMap &map_c, IvfGemmParams p, int grid, cudaStream_t s) {
    constexpr bool DEC = PRODUCER == IVF_PRODUCER_PQ || PRODUCER == IVF_PRODUCER_SQ8;
    // ring depth: as deep as the per-thread lists (and the PQ codebook) leave room for
    const int codebook = PRODUCER == IVF_PRODUCER_PQ ? p.codebook_bytes : 0;
    // Shared-memory budget: operand ring (32 KB per stage) + accumulator staging + cooperative lists + per-thread lists.  Items with many queries
    // insert into per-thread lists ~k ln(rows / k) times per lane, and every insert rescans the list: k L2 round trips from
    // global scratch against k shared-memory loads -- so the per-thread lists get shared memory even at the price of
    // a 3-stage ring; only when they do not fit beside 3 stages do they move to global scratch (and the ring gets 4 stages).
    auto need = [&](int st, int k_smem) { return ivf_smem_need(st, k_smem, codebook); };
    const int coop_bytes = p.k <= 256 ? (int)round_up(coop_smem_bytes(p.k), 16) : 0;
    p.coop_enabled = coop_bytes > 0 && need(2, 0) + coop_bytes <= SMEM_LIMIT ? kCoopMax : 0;
    if (const char *ev = getenv("B200_IVF_COOP")) p.coop_enabled = std::min(p.coop_enabled, atoi(ev));   // A/B and debugging
    const int coop_used = p.coop_enabled ? coop_bytes : 0;
    int stages = 4;
    p.lists_in_smem = 0;
    const int list_cap = list_cap_for(p.k);
    if (list_cap <= 2 * kGemmSmemK)
        for (int st = 4; st >= 3; st--)
            if (need(st, list_cap) + coop_used <= SMEM_LIMIT) {
                stages = st;
                p.lists_in_smem = 1;
                break;
            }
    if (!p.lists_in_smem) {
        while (stages > 2 && need(stages, 0) + coop_used > SMEM_LIMIT) stages--;
        if (need(stages, 0) + coop_used > SMEM_LIMIT) return cudaErrorInvalidValue;
    }
    p.stages = stages;
    const int k_smem = p.lists_in_smem ? list_cap : 0;
    p.coop_smem_off = (int)round_up(Layout<Operand::BF16>::off_list(stages) + k_smem * EPI_THREADS * 8, 16);
    p.codebook_smem_off = (int)round_up(p.coop_smem_off + coop_used, 16);
    const size_t smem = (size_t)need(stages, k_smem) + coop_used;
    auto kern = ivf_gemm_topk_kernel<PRODUCER, DSUB>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    kern<<<grid, DEC ? IVF_THREADS_DEC : IVF_THREADS_TMA, smem, s>>>(map_q, map_c, p);
    g_launches++;
    return cudaGetLastError();
}

}  // namespace gemm

bool ivf_pq_codebook_fits(int64_t codebook_bytes) {
    return codebook_bytes <= gemm::SMEM_LIMIT && gemm::ivf_smem_need(2, 0, (int)codebook_bytes) <= gemm::SMEM_LIMIT;
}

cudaError_t launch_ivf_gemm_topk(const IvfGemmParams &p, const void *queries_bf16, int64_t n_query_rows, const void *pool_bf16,
                                 int64_t pool_rows, int grid, cudaStream_t s, const char **err_detail) {
    *err_detail = nullptr;
    CUtensorMap map_q, map_c;
    if (!gemm::encode_rows_map(&map_q, queries_bf16, n_query_rows, p.d_pad, gemm::BM)) {
        *err_detail = "cuTensorMapEncodeTiled failed (queries)";
        return cudaErrorInvalidValue;
    }
    if (p.producer == IVF_PRODUCER_TMA) {
        // the pool as a [pool_rows * k-blocks][64] matrix: tile (page, kb) = rows [(page * kb_count + kb) * 256, +256)
        if (!gemm::encode_rows_map(&map_c, pool_bf16, pool_rows * (p.d_pad / gemm::BK), gemm::BK, gemm::HN)) {
            *err_detail = "cuTensorMapEncodeTiled failed (pool)";
            return cudaErrorInvalidValue;
        }
        return gemm::launch_ivf<IVF_PRODUCER_TMA, 0>(map_q, map_c, p, grid, s);
    }
    if (p.producer == IVF_PRODUCER_B1) {
        // bytes: the gathered queries [n_query_rows][row_pad] and the pool as a [pool_rows * k-blocks][kb_w] matrix, both read in
        // 128-byte boxes (columns past a row, or past a kb_w < 128 k-block, arrive as zeros)
        if (p.kb_w % 16 || p.d_pad % p.kb_w || !p.row_bias || (p.jaccard && !p.pair_popc)) {
            *err_detail = "binary IVF scan: kb_w a multiple of 16 dividing the row, popcounts set";
            return cudaErrorInvalidValue;
        }
        if (!gemm::encode_bytes_map(&map_q, queries_bf16, n_query_rows, p.d_pad, gemm::BM) ||
            !gemm::encode_bytes_map(&map_c, pool_bf16, pool_rows * (p.d_pad / p.kb_w), p.kb_w, gemm::HN)) {
            *err_detail = "cuTensorMapEncodeTiled failed (binary queries / pool)";
            return cudaErrorInvalidValue;
        }
        return gemm::launch_ivf<IVF_PRODUCER_B1, 0>(map_q, map_c, p, grid, s);
    }
    map_c = map_q;  // unused by the decoding producers
    if (p.producer == IVF_PRODUCER_SQ8) return gemm::launch_ivf<IVF_PRODUCER_SQ8, 0>(map_q, map_c, p, grid, s);
    switch (p.dsub) {
        case 1: return gemm::launch_ivf<IVF_PRODUCER_PQ, 1>(map_q, map_c, p, grid, s);
        case 2: return gemm::launch_ivf<IVF_PRODUCER_PQ, 2>(map_q, map_c, p, grid, s);
        case 4: return gemm::launch_ivf<IVF_PRODUCER_PQ, 4>(map_q, map_c, p, grid, s);
        case 8: return gemm::launch_ivf<IVF_PRODUCER_PQ, 8>(map_q, map_c, p, grid, s);
    }
    *err_detail = "PQ decode producer needs dsub in {1, 2, 4, 8}";
    return cudaErrorInvalidValue;
}

}  // namespace b200
