// prep.cu -- small elementwise kernels that put host-format columns into the HBM layout
// the scan / GEMM kernels want: zero-padded rows (16-byte multiples; 64-element multiples
// for the tensor-core path), optional bf16 conversion, per-row norms, per-row popcounts of binary rows.
//
// Reference counterparts: VectorDataset<T>::normalize (VectorIndex/Common/VectorDataset.h:99-117)
// and the ColumnArray -> contiguous float[n*d] copy in
// MergeTreeVSManager::vectorScanWithoutIndex (VectorIndex/Storages/MergeTreeVSManager.cpp:1380-1392).
#include "common.cuh"
#include "kernels.h"

namespace b200 {

__global__ void f32_to_bf16_rows_kernel(const float *__restrict__ src, int d, __nv_bfloat16 *__restrict__ dst, int d_pad,
                                        int64_t n) {
    const int64_t total = n * d_pad;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / d_pad;
        const int j = (int)(i - r * d_pad);
        dst[i] = __float2bfloat16_rn(j < d ? src[r * d + j] : 0.f);
    }
}

__global__ void pad_rows_f32_kernel(const float *__restrict__ src, int d, float *__restrict__ dst, int d_pad, int64_t n) {
    const int64_t total = n * d_pad;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / d_pad;
        const int j = (int)(i - r * d_pad);
        dst[i] = j < d ? src[r * d + j] : 0.f;
    }
}

// one warp per row, fp32 accumulation
__global__ void row_norms_kernel(const void *__restrict__ rows, int bf16, int d_pad, int64_t n, int mode,
                                 float *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp_global; r < n; r += nwarps) {
        float s = 0.f;
        if (bf16) {
            const __nv_bfloat16 *p = reinterpret_cast<const __nv_bfloat16 *>(rows) + r * d_pad;
            for (int j = lane; j < d_pad; j += 32) {
                const float v = __bfloat162float(p[j]);
                s = fmaf(v, v, s);
            }
        } else {
            const float *p = reinterpret_cast<const float *>(rows) + r * d_pad;
            for (int j = lane; j < d_pad; j += 32) s = fmaf(p[j], p[j], s);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) out[r] = mode == 0 ? s : -(s < FLT_EPSILON ? 1.f : 1.f / sqrtf(s));
    }
}

__global__ void normalize_rows_f32_kernel(float *rows, int d_pad, int64_t n) {
    const int lane = threadIdx.x & 31;
    const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp_global; r < n; r += nwarps) {
        float *p = rows + r * d_pad;
        float s = 0.f;
        for (int j = lane; j < d_pad; j += 32) s = fmaf(p[j], p[j], s);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (s < FLT_EPSILON) continue;  // VectorDataset.h:110
        const float nrm = sqrtf(s);
        for (int j = lane; j < d_pad; j += 32) p[j] = p[j] / nrm;
    }
}

// one warp per binary row; byte loads, so any row length and alignment
__global__ void popc_rows_kernel(const uint8_t *__restrict__ rows, int64_t row_bytes, int64_t n, float *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp_global; r < n; r += nwarps) {
        const uint8_t *p = rows + r * row_bytes;
        int c = 0;
        for (int64_t j = lane; j < row_bytes; j += 32) c += __popc((uint32_t)p[j]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        if (lane == 0) out[r] = (float)c;
    }
}

static int grid_for(int64_t work, int threads) {
    int64_t b = ceil_div(work, threads);
    if (b > 132 * 16) b = 132 * 16;
    if (b < 1) b = 1;
    return (int)b;
}

cudaError_t launch_f32_to_bf16_rows(const float *src, int d, void *dst, int d_pad, int64_t n, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    f32_to_bf16_rows_kernel<<<grid_for(n * d_pad, 256), 256, 0, s>>>(src, d, reinterpret_cast<__nv_bfloat16 *>(dst), d_pad, n);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t launch_pad_rows_f32(const float *src, int d, float *dst, int d_pad, int64_t n, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    pad_rows_f32_kernel<<<grid_for(n * d_pad, 256), 256, 0, s>>>(src, d, dst, d_pad, n);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t launch_row_norms(const void *rows, int bf16, int d_pad, int64_t n, int mode, float *out, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    row_norms_kernel<<<grid_for(n * 32, 256), 256, 0, s>>>(rows, bf16, d_pad, n, mode, out);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t launch_normalize_rows_f32(float *rows, int d_pad, int64_t n, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    normalize_rows_f32_kernel<<<grid_for(n * 32, 256), 256, 0, s>>>(rows, d_pad, n);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t launch_popc_rows(const uint8_t *rows, int64_t row_bytes, int64_t n, float *out, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    popc_rows_kernel<<<grid_for(n * 32, 256), 256, 0, s>>>(rows, row_bytes, n, out);
    g_launches++;
    return cudaGetLastError();
}

}  // namespace b200
