// rowmap.cu -- K10 / a11: filter-bitmap algebra and the row-id remaps of decoupled (merged) parts.
//
// Replaces Search::intersectDenseBitmaps (reference: src/VectorIndex/Common/VIWithDataPart.cpp:908, :560),
// getRealBitmap (src/VectorIndex/Utils/VIUtils.cpp:479-497), VIWithColumnInPart::transferToNewRowIds
// (src/VectorIndex/Common/VIWithDataPart.cpp:56-68) and TransferToOldRowIds (:69-126).
// All are byte/integer gathers over at most N bits or k labels; bit-exact by construction.
// HBM-bound: n/8 bytes per bitmap, 8-9 bytes per mapped row.
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "kernels.h"

namespace b200 {

__global__ void bitmap_and_kernel(const uint32_t *a, const uint32_t *b, int64_t nwords, uint32_t *out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nwords; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = a[i] & b[i];
}

// real_filter.set(inverted_row_ids_map[new_row]) for every set bit new_row with sources[new_row] == own_id
__global__ void real_bitmap_kernel(const uint8_t *filter, int64_t n_new, const uint64_t *inv_ids, const uint8_t *inv_src, uint32_t own_id,
                                   int64_t total_vec, uint32_t *out_words) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_new; r += (int64_t)gridDim.x * blockDim.x) {
        if (!((filter[r >> 3] >> (r & 7)) & 1)) continue;
        if (inv_src[r] != own_id) continue;
        const uint64_t old_row = inv_ids[r];
        if ((int64_t)old_row < total_vec) atomicOr(&out_words[old_row >> 5], 1u << (old_row & 31));
    }
}

__global__ void remap_labels_kernel(const uint64_t *map, int64_t map_len, int64_t *labels, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t l = labels[i];
        if (l != -1 && l < map_len) labels[i] = (int64_t)map[l];
    }
}

// filter->set(offset) for every surviving _part_offset of the PREWHERE pipeline (getFilterFromPipeline,
// src/VectorIndex/Storages/MergeTreeSelectWithHybridSearchProcessor.cpp:906-934), built where the searches consume it
__global__ void bitmap_from_offsets_kernel(const uint64_t *offsets, int64_t n, int64_t nbits, uint32_t *out_words) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t o = offsets[i];
        if ((int64_t)o < nbits) atomicOr(&out_words[o >> 5], 1u << (o & 31));
    }
}
// lightweight delete: bit = _row_exists[i] != 0 (MergeTreeVSManager.cpp:1435-1460)
__global__ void bitmap_from_bytes_kernel(const uint8_t *row_exists, int64_t n, uint8_t *out_bits) {
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < (n + 7) / 8; b += (int64_t)gridDim.x * blockDim.x) {
        uint32_t v = 0;
        for (int j = 0; j < 8; j++)
            if (b * 8 + j < n && row_exists[b * 8 + j]) v |= 1u << j;
        out_bits[b] = (uint8_t)v;
    }
}

}  // namespace b200

using namespace b200;

// Device-resident filter bitmaps (SURVEY 8 f2): the bitmap is BUILT in HBM from what the PREWHERE pipeline produces and handed
// to b200_corpus_search_device / b200_index_search_device / b200_sharded_*_search as d_alive_bits -- no n/8-byte upload per call.
// d_out_bits: device buffer of (nbits + 7) / 8 bytes rounded up to a multiple of 4, zeroed by the call.  Asynchronous on `stream`.
extern "C" int b200_bitmap_from_offsets_device(const uint64_t *d_offsets, int64_t n, int64_t nbits, uint8_t *d_out_bits, void *stream) {
    if ((!d_offsets && n > 0) || !d_out_bits || n < 0 || nbits < 0) return fail(B200_ERR_INVALID, "bad arguments");
    if ((reinterpret_cast<uintptr_t>(d_out_bits) & 3) != 0) return fail(B200_ERR_INVALID, "the bitmap buffer must be 4-byte aligned");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    B200_CUDA_OK(cudaMemsetAsync(d_out_bits, 0, (size_t)round_up(ceil_div(nbits, 8), 4), s));
    if (n) {
        bitmap_from_offsets_kernel<<<(int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, 256), 132 * 16)), 256, 0, s>>>(
            d_offsets, n, nbits, reinterpret_cast<uint32_t *>(d_out_bits));
        g_launches++;
        B200_CUDA_OK(cudaGetLastError());
    }
    return B200_OK;
}
extern "C" int b200_bitmap_from_row_exists_device(const uint8_t *d_row_exists, int64_t n, uint8_t *d_out_bits, void *stream) {
    if ((!d_row_exists && n > 0) || !d_out_bits || n < 0) return fail(B200_ERR_INVALID, "bad arguments");
    if (n == 0) return B200_OK;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    bitmap_from_bytes_kernel<<<(int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(ceil_div(n, 8), 256), 132 * 16)), 256, 0, s>>>(d_row_exists, n, d_out_bits);
    g_launches++;
    B200_CUDA_OK(cudaGetLastError());
    return B200_OK;
}
// out = a & b, all three device resident ((nbits + 7) / 8 bytes rounded up to a multiple of 4)
extern "C" int b200_bitmap_and_device(const uint8_t *d_a, const uint8_t *d_b, int64_t nbits, uint8_t *d_out, void *stream) {
    if (!d_a || !d_b || !d_out || nbits < 0) return fail(B200_ERR_INVALID, "bad arguments");
    if (nbits == 0) return B200_OK;
    const int64_t nwords = ceil_div(nbits, 32);
    bitmap_and_kernel<<<(int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(nwords, 256), 132 * 16)), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const uint32_t *>(d_a), reinterpret_cast<const uint32_t *>(d_b), nwords, reinterpret_cast<uint32_t *>(d_out));
    g_launches++;
    B200_CUDA_OK(cudaGetLastError());
    return B200_OK;
}

namespace {
int device_ok() {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
        cudaGetLastError();
        return fail(B200_ERR_NO_DEVICE, "no CUDA device visible; libb200search has no CPU fallback");
    }
    return B200_OK;
}
int blocks_for(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, 256), 132 * 16)); }
}  // namespace

// intersectDenseBitmaps: out = a & b over nbits bits (LSB-first bytes)
extern "C" int b200_bitmap_and(const uint8_t *a, const uint8_t *b, int64_t nbits, uint8_t *out) {
    if (!a || !b || !out || nbits < 0) return fail(B200_ERR_INVALID, "bad arguments");
    B200_TRY(device_ok());
    if (nbits == 0) return B200_OK;
    const int64_t nbytes = ceil_div(nbits, 8), nwords = ceil_div(nbytes, 4);
    DevMem s;
    B200_TRY(s.alloc((size_t)nwords * 4 * 3));
    char *d = s.as<char>();
    B200_CUDA_OK(cudaMemset(d, 0, (size_t)nwords * 4 * 3));
    B200_CUDA_OK(cudaMemcpy(d, a, nbytes, cudaMemcpyHostToDevice));
    B200_CUDA_OK(cudaMemcpy(d + nwords * 4, b, nbytes, cudaMemcpyHostToDevice));
    bitmap_and_kernel<<<blocks_for(nwords), 256>>>((const uint32_t *)d, (const uint32_t *)(d + nwords * 4), nwords,
                                                   (uint32_t *)(d + nwords * 8));
    g_launches++;
    B200_CUDA_OK(cudaGetLastError());
    B200_CUDA_OK(cudaMemcpy(out, d + nwords * 8, nbytes, cudaMemcpyDeviceToHost));
    return B200_OK;
}

// getRealBitmap: filter over the NEW (merged) part's offsets -> bitmap over this OLD part's rows (total_vec bits)
extern "C" int b200_real_bitmap(const uint8_t *filter_bits, int64_t n_new_rows, const uint64_t *inverted_row_ids_map,
                                const uint8_t *inverted_row_sources_map, uint32_t own_id, int64_t total_vec, uint8_t *out_bits) {
    if (!filter_bits || !inverted_row_ids_map || !inverted_row_sources_map || !out_bits || n_new_rows < 0 || total_vec < 0)
        return fail(B200_ERR_INVALID, "bad arguments");
    B200_TRY(device_ok());
    const int64_t fbytes = ceil_div(n_new_rows, 8), owords = ceil_div(ceil_div(total_vec, 8), 4);
    if (total_vec == 0) return B200_OK;
    DevMem s;
    const size_t o_f = 0, o_ids = round_up(fbytes, 256), o_src = o_ids + (size_t)n_new_rows * 8, o_out = round_up(o_src + n_new_rows, 256);
    B200_TRY(s.alloc(o_out + (size_t)owords * 4 + 256));
    char *d = s.as<char>();
    B200_CUDA_OK(cudaMemset(d + o_out, 0, (size_t)owords * 4));
    if (n_new_rows) {
        B200_CUDA_OK(cudaMemcpy(d + o_f, filter_bits, fbytes, cudaMemcpyHostToDevice));
        B200_CUDA_OK(cudaMemcpy(d + o_ids, inverted_row_ids_map, (size_t)n_new_rows * 8, cudaMemcpyHostToDevice));
        B200_CUDA_OK(cudaMemcpy(d + o_src, inverted_row_sources_map, n_new_rows, cudaMemcpyHostToDevice));
        real_bitmap_kernel<<<blocks_for(n_new_rows), 256>>>((const uint8_t *)(d + o_f), n_new_rows, (const uint64_t *)(d + o_ids),
                                                            (const uint8_t *)(d + o_src), own_id, total_vec, (uint32_t *)(d + o_out));
        g_launches++;
        B200_CUDA_OK(cudaGetLastError());
    }
    B200_CUDA_OK(cudaMemcpy(out_bits, d + o_out, ceil_div(total_vec, 8), cudaMemcpyDeviceToHost));
    return B200_OK;
}

// transferToNewRowIds: labels[i] = row_ids_map[labels[i]] unless -1 (in place)
extern "C" int b200_remap_labels(const uint64_t *row_ids_map, int64_t map_len, int64_t *labels, int64_t n) {
    if (!row_ids_map || !labels || map_len < 0 || n < 0) return fail(B200_ERR_INVALID, "bad arguments");
    B200_TRY(device_ok());
    if (n == 0 || map_len == 0) return B200_OK;
    DevMem s;
    const size_t o_l = round_up(map_len * 8, 256);
    B200_TRY(s.alloc(o_l + (size_t)n * 8 + 256));
    char *d = s.as<char>();
    B200_CUDA_OK(cudaMemcpy(d, row_ids_map, (size_t)map_len * 8, cudaMemcpyHostToDevice));
    B200_CUDA_OK(cudaMemcpy(d + o_l, labels, (size_t)n * 8, cudaMemcpyHostToDevice));
    remap_labels_kernel<<<blocks_for(n), 256>>>((const uint64_t *)d, map_len, (int64_t *)(d + o_l), n);
    g_launches++;
    B200_CUDA_OK(cudaGetLastError());
    B200_CUDA_OK(cudaMemcpy(labels, d + o_l, (size_t)n * 8, cudaMemcpyDeviceToHost));
    return B200_OK;
}

// TransferToOldRowIds: keep candidate i iff id != -1, id < map size and sources[id] == own_id; id -> inverted_row_ids_map[id].
// Compaction preserves order; <= num_candidates entries, done on the host side of the call (k-sized).
extern "C" int b200_transfer_to_old_row_ids(const int64_t *new_ids, const float *new_dis, int64_t num_candidates,
                                            const uint64_t *inverted_row_ids_map, const uint8_t *inverted_row_sources_map,
                                            int64_t map_len, uint32_t own_id, int64_t *out_ids, float *out_dis, int64_t *out_n) {
    if (!new_ids || !new_dis || !inverted_row_ids_map || !inverted_row_sources_map || !out_ids || !out_dis || !out_n)
        return fail(B200_ERR_INVALID, "bad arguments");
    // k-sized gather: the reference does this on <= num_reorder entries (:96-111); the map lookups are the device
    // kernel above when the maps are resident; for host-resident maps a k-entry loop is the whole job.
    int64_t m = 0;
    for (int64_t i = 0; i < num_candidates; i++) {
        const int64_t id = new_ids[i];
        if (id == -1 || id >= map_len) continue;
        if (inverted_row_sources_map[id] != own_id) continue;
        out_ids[m] = (int64_t)inverted_row_ids_map[id];
        out_dis[m] = new_dis[i];
        m++;
    }
    *out_n = m;
    return B200_OK;
}
