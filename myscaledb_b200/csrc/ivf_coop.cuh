// ivf_coop.cuh -- tile-wise cooperative top-k of the grouped IVF scan (ivf_gemm_sm90.cu), kept in a header so that
// tests/cuda/coop_merge_test.cu can drive exactly this code with synthetic tiles and compare it with a CPU sort.
#pragma once
#include "gemm_common.cuh"

namespace b200 {
namespace gemm {

// Items with only a few queries (the usual case for small batches: every probed list is visited by one or two queries)
// would leave all the top-k work to one or two lanes of the per-thread scheme, and every item starts with an empty list:
// ~k ln(rows / k) + k inserts per item, each a latency-bound dependent chain, while the other warps wait on the epilogue
// barrier behind the one busy warp.  For q_count <= kCoopMax the warp of query
// slots 0..31 therefore works TILE-wise and in bulk: lanes whose chunk minimum beats their threshold park the chunk's keys
// in a per-slot tile buffer; after the tile the warp compacts each slot's
// candidates, sorts them with a bitonic network in shared memory and rank-merges them with the slot's sorted k-list
// (binary searches, all lanes busy) instead of up to 256 dependent inserts per tile.
constexpr int kCoopMax = 16;
constexpr int kTileBufStride = BN;       // [16][256] floats = exactly the 16 KB slow-path scratch of the per-thread mode, which
                                         // it aliases (an item is either cooperative or per-thread); columns are XOR-swizzled
                                         // with the slot so that lanes parking the same column hit different banks

struct CoopState {   // one per query slot, in shared memory
    float thr_key;
    uint32_t thr_id;
    int n;
    int buf;         // which of the slot's two list buffers is current
};

struct CoopSmem {
    float *keys[2];          // [kCoopMax][k] x 2 (double buffer for the rank merge)
    uint32_t *ids[2];
    CoopState *state;        // [kCoopMax]
    float *tilebuf;          // [kCoopMax][kTileBufStride]
    float *cand_keys;        // [BN]
    uint32_t *cand_ids;      // [BN]
};
__host__ __device__ inline size_t coop_smem_bytes(int k) {
    return (size_t)kCoopMax * k * 8 * 2 + kCoopMax * sizeof(CoopState) + (size_t)BN * 8 + 64;
}
static_assert(kCoopMax * kTileBufStride * 4 <= SCRATCH_BYTES, "the tile buffer aliases the epilogue scratch");
__device__ __forceinline__ CoopSmem coop_smem_carve(unsigned char *base, unsigned char *scratch_base, int k) {
    CoopSmem c;
    c.keys[0] = reinterpret_cast<float *>(base);
    c.keys[1] = c.keys[0] + (size_t)kCoopMax * k;
    c.ids[0] = reinterpret_cast<uint32_t *>(c.keys[1] + (size_t)kCoopMax * k);
    c.ids[1] = c.ids[0] + (size_t)kCoopMax * k;
    c.state = reinterpret_cast<CoopState *>(c.ids[1] + (size_t)kCoopMax * k);
    c.tilebuf = reinterpret_cast<float *>(scratch_base);
    c.cand_keys = reinterpret_cast<float *>(c.state + kCoopMax);
    c.cand_ids = reinterpret_cast<uint32_t *>(c.cand_keys + BN);
    return c;
}

// One 32-column chunk in cooperative mode: transform (AFFINE: v * scale + bias; else v already holds the keys), and park the
// keys if this lane's slot can use any of them.
template <bool AFFINE = true>
__device__ __forceinline__ void coop_stage_chunk(float thr, float (&v)[32], const float *scale, const float *bias, float *tile_row /* this lane's slot */,
                                                 int chunk, uint32_t &chunk_mask, int swz /* slot & 31 */) {
    if (AFFINE) side_fma32(v, scale, bias);
    float m0 = fminf(v[0], v[1]), m1 = fminf(v[2], v[3]), m2 = fminf(v[4], v[5]), m3 = fminf(v[6], v[7]);
#pragma unroll
    for (int j = 8; j < 32; j += 8) {
        m0 = fminf(m0, fminf(v[j], v[j + 1]));
        m1 = fminf(m1, fminf(v[j + 2], v[j + 3]));
        m2 = fminf(m2, fminf(v[j + 4], v[j + 5]));
        m3 = fminf(m3, fminf(v[j + 6], v[j + 7]));
    }
    if (fminf(fminf(m0, m1), fminf(m2, m3)) <= thr) {
#pragma unroll
        for (int j = 0; j < 32; j++) tile_row[chunk * 32 + (j ^ swz)] = v[j];
        chunk_mask |= 1u << chunk;
    }
}

// After a tile: the warp folds the parked keys of every slot into that slot's sorted list.  Returns (to lane s) the new
// threshold of slot s through `thr`.
__device__ __forceinline__ void coop_merge_tile(const CoopSmem &cs, int k, int q_count, uint32_t chunk_mask, uint32_t row0, int lane, float &thr) {
    for (int s = 0; s < q_count; s++) {
        const uint32_t cm = __shfl_sync(0xffffffffu, chunk_mask, s);
        if (!cm) continue;
        CoopState st = cs.state[s];
        const float *tb = cs.tilebuf + (size_t)s * kTileBufStride;
        // ---- compaction of the candidates that beat the current threshold
        int c = 0;
        for (uint32_t m = cm; m; m &= m - 1) {
            const int ch = __ffs(m) - 1;
            const float key = tb[ch * 32 + (lane ^ s)];
            const uint32_t id = row0 + (uint32_t)(ch * 32 + lane);
            const bool pass = better(key, id, st.thr_key, st.thr_id);
            const unsigned bal = __ballot_sync(0xffffffffu, pass);
            if (pass) {
                const int pos = c + __popc(bal & ((1u << lane) - 1u));
                cs.cand_keys[pos] = key;
                cs.cand_ids[pos] = id;
            }
            c += __popc(bal);
        }
        if (c == 0) continue;
        int n2 = 32;
        while (n2 < c) n2 <<= 1;
        for (int i = c + lane; i < n2; i += 32) {
            cs.cand_keys[i] = FLT_MAX;
            cs.cand_ids[i] = kNoId;
        }
        __syncwarp();
        // ---- bitonic sort of cand[0, n2) by (key, id)
        for (int size = 2; size <= n2; size <<= 1)
            for (int stride = size >> 1; stride > 0; stride >>= 1) {
                for (int t = lane; t < (n2 >> 1); t += 32) {
                    const int i = ((t / stride) * 2 * stride) + (t % stride), j = i + stride;
                    const float ki = cs.cand_keys[i], kj = cs.cand_keys[j];
                    const uint32_t ii = cs.cand_ids[i], ij = cs.cand_ids[j];
                    const bool up = (i & size) == 0;
                    if (better(kj, ij, ki, ii) == up) {
                        cs.cand_keys[i] = kj; cs.cand_ids[i] = ij;
                        cs.cand_keys[j] = ki; cs.cand_ids[j] = ii;
                    }
                }
                __syncwarp();
            }
        // ---- rank merge of list[0, n) and cand[0, m): element -> its position in the union, kept if < k
        const int m_c = c < k ? c : k;
        const float *lk = cs.keys[st.buf] + (size_t)s * k;
        const uint32_t *li = cs.ids[st.buf] + (size_t)s * k;
        float *ok = cs.keys[st.buf ^ 1] + (size_t)s * k;
        uint32_t *oi = cs.ids[st.buf ^ 1] + (size_t)s * k;
        for (int a = lane; a < st.n; a += 32) {
            const float key = lk[a];
            const uint32_t id = li[a];
            int lo = 0, hi = m_c;   // candidates strictly better than this list element
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (better(cs.cand_keys[mid], cs.cand_ids[mid], key, id)) lo = mid + 1; else hi = mid;
            }
            const int rank = a + lo;
            if (rank < k) { ok[rank] = key; oi[rank] = id; }
        }
        for (int b = lane; b < m_c; b += 32) {
            const float key = cs.cand_keys[b];
            const uint32_t id = cs.cand_ids[b];
            int lo = 0, hi = st.n;  // list elements better than this candidate (ids are unique: no ties between the two sets)
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (better(lk[mid], li[mid], key, id)) lo = mid + 1; else hi = mid;
            }
            const int rank = b + lo;
            if (rank < k) { ok[rank] = key; oi[rank] = id; }
        }
        __syncwarp();
        st.n = st.n + m_c < k ? st.n + m_c : k;
        st.buf ^= 1;
        if (st.n == k) {
            st.thr_key = ok[k - 1];
            st.thr_id = oi[k - 1];
        }
        if (lane == 0) cs.state[s] = st;
        if (lane == s) thr = st.thr_key;
        __syncwarp();
    }
}

}  // namespace gemm
}  // namespace b200
