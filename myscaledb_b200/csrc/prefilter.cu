// prefilter.cu -- pre-filtered exact search: the rows a selective filter keeps are copied into a compact corpus, the
// unchanged scan / tensor-core kernels score only those, and the winners' compact ids are mapped back to row ids.
//
// An exact top-k over the kept rows equals the top-k of a full scan that masks the other rows: the kernels run the same
// per-row arithmetic either way, and the compact rows keep their row order, so the tie rule (smaller id wins) holds too.
//   compaction: per-word popcount of the alive bitmap -> one exclusive scan (cub::DeviceScan) -> per-word scatter of the
//               set bits' row ids (u32, ascending).  Bits at positions >= n are ignored.
//   gather:     a warp copies one kept row (padded row layout, corpus dtype) and its side-array entries.
//   map-back:   out_id = id >= 0 ? alive_ids[id] + id_offset : -1 over the final [nq][k] ids.
#include <algorithm>

#include <cub/cub.cuh>

#include "common.cuh"
#include "kernels.h"

namespace b200 {

namespace {

constexpr int kThreads = 256;

int blocks_for(int64_t work, int64_t per_block) {
    return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(work, per_block), 132 * 16));
}

// 32-bit word w of the bitmap with the bits at positions >= n cleared (the last byte may carry garbage past n)
__device__ __forceinline__ uint32_t alive_word(const uint32_t *words, int64_t w, int64_t n) {
    uint32_t v = words[w];
    const int64_t rem = n - w * 32;
    if (rem < 32) v &= (1u << rem) - 1u;
    return v;
}

__global__ void alive_word_popc_kernel(const uint32_t *words, int64_t n, int64_t nwords, uint32_t *cnt) {
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < nwords; w += (int64_t)gridDim.x * blockDim.x)
        cnt[w] = __popc(alive_word(words, w, n));
}

__global__ void alive_scatter_kernel(const uint32_t *words, int64_t n, int64_t nwords, const uint32_t *off, uint32_t *ids) {
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < nwords; w += (int64_t)gridDim.x * blockDim.x) {
        uint32_t v = alive_word(words, w, n);
        uint32_t pos = off[w];
        while (v) {
            ids[pos++] = (uint32_t)(w * 32) + (uint32_t)(__ffs(v) - 1);
            v &= v - 1u;
        }
    }
}

// one warp per kept row: 16-byte copies when the row length allows (every float / bf16 layout), bytes otherwise
__global__ void gather_rows_kernel(const char *rows, int64_t row_bytes, const float *scale, const float *bias, const uint32_t *ids,
                                   int64_t m, char *out_rows, float *out_scale, float *out_bias) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); i < m; i += warps) {
        const uint32_t r = ids[i];
        const char *src = rows + (int64_t)r * row_bytes;
        char *dst = out_rows + i * row_bytes;
        if (row_bytes % 16 == 0) {
            for (int64_t b = (int64_t)lane * 16; b < row_bytes; b += 32 * 16)
                *reinterpret_cast<uint4 *>(dst + b) = __ldg(reinterpret_cast<const uint4 *>(src + b));
        } else {
            for (int64_t b = lane; b < row_bytes; b += 32) dst[b] = src[b];
        }
        if (lane == 0) {
            if (scale) out_scale[i] = scale[r];
            if (bias) out_bias[i] = bias[r];
        }
    }
}

__global__ void map_ids_kernel(const uint32_t *alive_ids, int64_t id_offset, int64_t *ids, int64_t count) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t id = ids[i];
        ids[i] = id >= 0 ? (int64_t)alive_ids[id] + id_offset : -1;
    }
}

// the one CUB instantiation of the compaction: its size query (tmp = null) and its launch
cudaError_t exclusive_sum(void *tmp, size_t &tmp_bytes, uint32_t *in, uint32_t *out, int64_t nwords, cudaStream_t s) {
    return cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, in, out, (int)nwords, s);
}

size_t scan_temp_bytes(int64_t nwords) {
    size_t tb = 0;
    exclusive_sum(nullptr, tb, nullptr, nullptr, nwords, nullptr);
    return tb;
}

}  // namespace

// temp layout: [counts nwords u32 | offsets nwords u32 | cub scan storage], each part 256-byte aligned
size_t prefilter_compact_temp_bytes(int64_t n) {
    const int64_t nwords = std::max<int64_t>(1, ceil_div(n, 32));
    return 2 * (size_t)round_up(nwords * 4, 256) + round_up((int64_t)scan_temp_bytes(nwords), 256);
}

cudaError_t launch_prefilter_compact(const uint8_t *d_alive, int64_t n, uint32_t *d_ids, void *temp, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    const int64_t nwords = ceil_div(n, 32);
    const uint32_t *words = reinterpret_cast<const uint32_t *>(d_alive);
    uint32_t *cnt = reinterpret_cast<uint32_t *>(temp);
    uint32_t *off = reinterpret_cast<uint32_t *>(reinterpret_cast<char *>(temp) + round_up(nwords * 4, 256));
    void *scan_tmp = reinterpret_cast<char *>(temp) + 2 * round_up(nwords * 4, 256);
    size_t tb = scan_temp_bytes(nwords);
    alive_word_popc_kernel<<<blocks_for(nwords, kThreads), kThreads, 0, s>>>(words, n, nwords, cnt);
    g_launches++;
    cudaError_t e = exclusive_sum(scan_tmp, tb, cnt, off, nwords, s);
    if (e != cudaSuccess) return e;
    g_launches += 2;   // CUB's single-pass scan: an init kernel and the scan kernel
    alive_scatter_kernel<<<blocks_for(nwords, kThreads), kThreads, 0, s>>>(words, n, nwords, off, d_ids);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t launch_prefilter_gather(const void *rows, int64_t row_bytes, const float *scale, const float *bias, const uint32_t *ids,
                                    int64_t m, void *out_rows, float *out_scale, float *out_bias, cudaStream_t s) {
    if (m <= 0) return cudaSuccess;
    gather_rows_kernel<<<blocks_for(m, kThreads / 32), kThreads, 0, s>>>(reinterpret_cast<const char *>(rows), row_bytes, scale, bias, ids, m,
                                                                        reinterpret_cast<char *>(out_rows), out_scale, out_bias);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t launch_prefilter_map_ids(const uint32_t *alive_ids, int64_t id_offset, int64_t *ids, int64_t count, cudaStream_t s) {
    if (count <= 0) return cudaSuccess;
    map_ids_kernel<<<blocks_for(count, kThreads), kThreads, 0, s>>>(alive_ids, id_offset, ids, count);
    g_launches++;
    return cudaGetLastError();
}

}  // namespace b200
