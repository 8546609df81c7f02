// fusion.cu -- K9: hybrid-search fusion, batched over queries.
//
// Replaces RankFusion / RelativeScoreFusion / computeNormalizedScore
// (reference: src/VectorIndex/Utils/HybridSearchUtils.cpp:164-209, :212-274, :276-314) and the
// ordering step of MergeTreeHybridSearchManager::hybridSearch
// (src/VectorIndex/Storages/MergeTreeHybridSearchManager.cpp:108-171): results keyed by
// (shard_num, part_index, label), fused score descending, equal scores in ascending key order
// (std::map iteration order fed into std::multimap<Float32, ..., std::greater>).
// One CTA per query; the candidate lists (<= 2 x num_candidates entries) live in shared memory.
// Latency-bound by construction (tens of entries per query); batched so that nq = 512 is one launch.
#include <mutex>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "kernels.h"

namespace b200 {

struct FusionParams {
    const uint32_t *v_shard, *t_shard;
    const uint64_t *v_part, *v_label, *t_part, *t_label;
    const float *v_score, *t_score;
    const uint32_t *v_count, *t_count;
    int64_t v_stride, t_stride;
    int fusion_type;  // 0 RSF, 1 RRF
    float weight;
    uint64_t fusion_k;
    int direction;    // 1 ascending vector metric, -1 descending
    uint32_t top_k;
    uint32_t *o_shard;
    uint64_t *o_part, *o_label;
    float *o_score;
    uint32_t *o_count;
};

struct FEntry {
    uint32_t shard;
    uint64_t part, label;
    float score;
};

__device__ __forceinline__ bool key_eq(const FEntry &a, uint32_t s, uint64_t p, uint64_t l) {
    return a.shard == s && a.part == p && a.label == l;
}
__device__ __forceinline__ bool key_lt(const FEntry &a, const FEntry &b) {
    if (a.shard != b.shard) return a.shard < b.shard;
    if (a.part != b.part) return a.part < b.part;
    return a.label < b.label;
}

// computeNormalizedScore: min/max from the last/first element, swapped if ascending
__device__ __forceinline__ float norm_score(float s, float first, float last) {
    float mn = last, mx = first;
    if (mn == mx) return 1.0f;
    if (mn > mx) {
        const float t = mn;
        mn = mx;
        mx = t;
    }
    return __fdiv_rn(__fsub_rn(s, mn), __fsub_rn(mx, mn));
}

__global__ void __launch_bounds__(128) hybrid_fusion_kernel(const FusionParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    FEntry *e = reinterpret_cast<FEntry *>(smem_raw);
    __shared__ uint32_t n_entries;
    const int64_t q = blockIdx.x;
    const uint32_t nv = p.v_count[q], nt = p.t_count[q];
    const uint32_t *vs = p.v_shard + q * p.v_stride, *ts = p.t_shard + q * p.t_stride;
    const uint64_t *vp = p.v_part + q * p.v_stride, *vl = p.v_label + q * p.v_stride;
    const uint64_t *tp = p.t_part + q * p.t_stride, *tl = p.t_label + q * p.t_stride;
    const float *vsc = p.v_score + q * p.v_stride, *tsc = p.t_score + q * p.t_stride;

    // The entries are built in the reference's map order, so duplicate keys inside one list sum exactly as it does:
    // RankFusion adds the vector ranks, then the text ranks; RelativeScoreFusion ASSIGNS the text parts (a text key listed
    // twice keeps its last part), then ADDS the vector parts one by one.
    if (threadIdx.x == 0) {
        uint32_t n = 0;
        auto at = [&](uint32_t s, uint64_t pa, uint64_t l) -> FEntry & {   // map[key]: new keys start at 0
            uint32_t j = 0;
            for (; j < n; j++)
                if (key_eq(e[j], s, pa, l)) return e[j];
            e[n].shard = s;
            e[n].part = pa;
            e[n].label = l;
            e[n].score = 0.f;
            return e[n++];
        };
        if (p.fusion_type == 1) {
            for (uint32_t i = 0; i < nv; i++) {
                FEntry &x = at(vs[i], vp[i], vl[i]);
                x.score = __fadd_rn(x.score, __fdiv_rn(1.0f, (float)(p.fusion_k + i + 1)));
            }
            for (uint32_t i = 0; i < nt; i++) {
                FEntry &x = at(ts[i], tp[i], tl[i]);
                x.score = __fadd_rn(x.score, __fdiv_rn(1.0f, (float)(p.fusion_k + i + 1)));
            }
        } else {
            for (uint32_t i = 0; i < nt; i++)
                at(ts[i], tp[i], tl[i]).score = __fmul_rn(norm_score(tsc[i], tsc[0], tsc[nt - 1]), p.weight);
            const float w1 = __fsub_rn(1.0f, p.weight);
            for (uint32_t i = 0; i < nv; i++) {
                const float ns = norm_score(vsc[i], vsc[0], vsc[nv - 1]);
                FEntry &x = at(vs[i], vp[i], vl[i]);
                x.score = __fadd_rn(x.score, p.direction == -1 ? __fmul_rn(ns, w1) : __fmul_rn(__fsub_rn(1.0f, ns), w1));
            }
        }
        n_entries = n;
    }
    __syncthreads();
    const uint32_t n = n_entries;
    // rank by (score desc, key asc); keys are unique so ranks are too
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        uint32_t rank = 0;
        for (uint32_t j = 0; j < n; j++)
            if (e[j].score > e[i].score || (e[j].score == e[i].score && key_lt(e[j], e[i]))) rank++;
        if (rank < p.top_k) {
            const int64_t o = q * p.top_k + rank;
            p.o_shard[o] = e[i].shard;
            p.o_part[o] = e[i].part;
            p.o_label[o] = e[i].label;
            p.o_score[o] = e[i].score;
        }
    }
    if (threadIdx.x == 0) p.o_count[q] = n < p.top_k ? n : p.top_k;
}

}  // namespace b200

using namespace b200;

extern "C" int b200_hybrid_fusion_batch(int fusion_type, int64_t nq, const uint32_t *vec_shard, const uint64_t *vec_part,
                                        const uint64_t *vec_label, const float *vec_score, const uint32_t *vec_count,
                                        int64_t vec_stride, const uint32_t *txt_shard, const uint64_t *txt_part,
                                        const uint64_t *txt_label, const float *txt_score, const uint32_t *txt_count,
                                        int64_t txt_stride, float fusion_weight, uint64_t fusion_k, int vector_scan_direction,
                                        uint32_t top_k, uint32_t *out_shard, uint64_t *out_part, uint64_t *out_label,
                                        float *out_score, uint32_t *out_count) {
    if (nq < 0 || vec_stride < 0 || txt_stride < 0 || top_k == 0 || !vec_count || !txt_count || !out_shard || !out_part ||
        !out_label || !out_score || !out_count || (fusion_type != 0 && fusion_type != 1))
        return fail(B200_ERR_INVALID, "bad arguments");
    if (vec_stride + txt_stride > 2048) return fail(B200_ERR_UNSUPPORTED, "more than 2048 candidates per query");
    if (nq == 0) return B200_OK;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return fail(B200_ERR_NO_DEVICE, "no CUDA device visible; libb200search has no CPU fallback");
    }
    // one staging buffer, carved
    const size_t nv = (size_t)nq * vec_stride, nt = (size_t)nq * txt_stride, no = (size_t)nq * top_k;
    size_t off = 0;
    auto carve = [&](size_t bytes) {
        const size_t o = off;
        off += (bytes + 255) & ~(size_t)255;
        return o;
    };
    const size_t o_vs = carve(nv * 4), o_vp = carve(nv * 8), o_vl = carve(nv * 8), o_vsc = carve(nv * 4), o_vc = carve(nq * 4);
    const size_t o_ts = carve(nt * 4), o_tp = carve(nt * 8), o_tl = carve(nt * 8), o_tsc = carve(nt * 4), o_tc = carve(nq * 4);
    const size_t o_os = carve(no * 4), o_op = carve(no * 8), o_ol = carve(no * 8), o_osc = carve(no * 4), o_oc = carve(nq * 4);
    // Per-device scratch, grown on demand and kept: a device buffer, a pinned host mirror and a stream of its own.  (cudaMalloc /
    // cudaFree and pageable copies per call would synchronise the device and walk the allocator, which is slow next to a large
    // resident index.)
    int dev = 0;
    B200_CUDA_OK(cudaGetDevice(&dev));
    static std::mutex g_mu;
    struct PerDevice {
        DevMem d;
        char *h = nullptr;
        cudaStream_t s = nullptr;
    };
    static PerDevice g_scratch[64];
    if (dev < 0 || dev >= 64) return fail(B200_ERR_UNSUPPORTED, "device ordinal above 63");
    std::lock_guard<std::mutex> lk(g_mu);
    PerDevice &sc = g_scratch[dev];
    if (!sc.s) B200_CUDA_OK(cudaStreamCreateWithFlags(&sc.s, cudaStreamNonBlocking));
    if (off + 256 > sc.d.size()) {
        if (sc.h) cudaFreeHost(sc.h);
        sc.h = nullptr;
        const size_t want = (off + 256) * 2;
        B200_TRY(sc.d.alloc(want));
        if (cudaMallocHost(&sc.h, want) != cudaSuccess) {
            sc.d.reset();
            return fail(B200_ERR_NOMEM, "cudaMallocHost failed in fusion");
        }
    }
    char *d = sc.d.as<char>();
    cudaStream_t s = sc.s;
    int rc = B200_OK;
    // inputs: packed into the pinned mirror at their carved offsets, then ONE copy (o_vs .. end of o_tc is contiguous)
    auto up = [&](size_t o, const void *src, size_t bytes) {
        if (bytes) memcpy(sc.h + o, src, bytes);
    };
    up(o_vs, vec_shard, nv * 4); up(o_vp, vec_part, nv * 8); up(o_vl, vec_label, nv * 8); up(o_vsc, vec_score, nv * 4);
    up(o_vc, vec_count, nq * 4);
    up(o_ts, txt_shard, nt * 4); up(o_tp, txt_part, nt * 8); up(o_tl, txt_label, nt * 8); up(o_tsc, txt_score, nt * 4);
    up(o_tc, txt_count, nq * 4);
    if (cudaMemcpyAsync(d, sc.h, o_os, cudaMemcpyHostToDevice, s) != cudaSuccess) rc = fail(B200_ERR_CUDA, "H2D copy failed in fusion");
    if (rc == B200_OK) {
        FusionParams p{};
        p.v_shard = (const uint32_t *)(d + o_vs); p.v_part = (const uint64_t *)(d + o_vp); p.v_label = (const uint64_t *)(d + o_vl);
        p.v_score = (const float *)(d + o_vsc); p.v_count = (const uint32_t *)(d + o_vc); p.v_stride = vec_stride;
        p.t_shard = (const uint32_t *)(d + o_ts); p.t_part = (const uint64_t *)(d + o_tp); p.t_label = (const uint64_t *)(d + o_tl);
        p.t_score = (const float *)(d + o_tsc); p.t_count = (const uint32_t *)(d + o_tc); p.t_stride = txt_stride;
        p.fusion_type = fusion_type; p.weight = fusion_weight; p.fusion_k = fusion_k; p.direction = vector_scan_direction;
        p.top_k = top_k;
        p.o_shard = (uint32_t *)(d + o_os); p.o_part = (uint64_t *)(d + o_op); p.o_label = (uint64_t *)(d + o_ol);
        p.o_score = (float *)(d + o_osc); p.o_count = (uint32_t *)(d + o_oc);
        const size_t smem = (size_t)(vec_stride + txt_stride + 1) * sizeof(FEntry);
        // 2048 candidates take 64 KB, above the 48 KB a kernel gets without opting in
        if (cudaFuncSetAttribute(hybrid_fusion_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
            cudaGetLastError();
            rc = fail(B200_ERR_CUDA, "cannot grant the fusion kernel its shared memory");
        } else {
            hybrid_fusion_kernel<<<(unsigned)nq, 128, smem, s>>>(p);
            g_launches++;
            if (cudaGetLastError() != cudaSuccess) rc = fail(B200_ERR_CUDA, "fusion kernel launch failed");
        }
    }
    // outputs: one copy back into the mirror, then scattered to the caller's arrays
    if (rc == B200_OK && cudaMemcpyAsync(sc.h + o_os, d + o_os, off - o_os, cudaMemcpyDeviceToHost, s) != cudaSuccess)
        rc = fail(B200_ERR_CUDA, "D2H copy failed in fusion");
    if (cudaStreamSynchronize(s) != cudaSuccess && rc == B200_OK) rc = fail(B200_ERR_CUDA, "fusion kernel failed");
    if (rc == B200_OK) {
        memcpy(out_shard, sc.h + o_os, no * 4);
        memcpy(out_part, sc.h + o_op, no * 8);
        memcpy(out_label, sc.h + o_ol, no * 8);
        memcpy(out_score, sc.h + o_osc, no * 4);
        memcpy(out_count, sc.h + o_oc, (size_t)nq * 4);
    }
    return rc;
}
