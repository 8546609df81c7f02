// Micro-benchmark of the per-thread top-k list (gemm_common.cuh) on a synthetic stream shaped like one epilogue warp-group of the
// flat tensor-core kernel: 128 lists, `chunks` 32-wide chunks of pseudo-random keys each.  Prints time and event counters for
// rescan / append lists in shared or global memory.  Not part of the test suite; build with the line below and run it by hand.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O2 -std=c++17 -DB200_LIST_STATS -I myscaledb_b200/csrc tests/cuda/list_perf.cu -o tests/cuda/list_perf
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "gemm_common.cuh"

using namespace b200;
using namespace b200::gemm;

__device__ __forceinline__ float rnd(uint32_t a, uint32_t b) {   // ~N(0,1)-ish: sum of 4 uniforms
    uint32_t x = a * 0x9E3779B1u ^ b * 0x85EBCA6Bu;
    float s = 0.f;
    for (int i = 0; i < 4; i++) {
        x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
        s += (float)(x >> 8) * (1.f / 16777216.f);
    }
    return s - 2.f;
}

__global__ void __launch_bounds__(128) perf_kernel(int chunks, int k, int cap, int in_smem, int pad, float *g_keys, uint32_t *g_ids, float *out_keys, uint32_t *out_ids) {
    extern __shared__ unsigned char smem[];
    float *scratch_all = reinterpret_cast<float *>(smem);
    const int t = threadIdx.x;
    ThreadTopK list;
    list.n = 0; list.worst = 0; list.thr_key = FLT_MAX; list.thr_id = 0;
    if (pad < 0) scratch_all[t] = 0.f;   // keeps the padding argument alive
    float *kb = in_smem ? reinterpret_cast<float *>(smem + SCRATCH_BYTES) : g_keys + (size_t)blockIdx.x * cap * EPI_THREADS;
    uint32_t *ib = in_smem ? reinterpret_cast<uint32_t *>(smem + SCRATCH_BYTES + (size_t)cap * EPI_THREADS * 4) : g_ids + (size_t)blockIdx.x * cap * EPI_THREADS;
    list_bind(list, kb, ib, t, k, cap);
    if (pad == 1) {   // the one-lane rescan form whatever k
        list.coop = 0; list.stride = EPI_THREADS; list.keys = kb + t; list.ids = ib + t;
    }
    __shared__ __align__(16) float one[32], zero[32];
    if (t < 32) { one[t] = 1.f; zero[t] = 0.f; }
    __syncthreads();
    for (int c = 0; c < chunks; c++) {
        float v[32];
#pragma unroll
        for (int j = 0; j < 32; j++) v[j] = rnd((uint32_t)(c * 32 + j), (uint32_t)(blockIdx.x * 128 + t));
        __syncwarp();
        epilogue_chunk(list, v, true, one, zero, (uint32_t)c * 32u, false, 0, scratch_all + t);
    }
    list_publish(list, out_keys + ((size_t)blockIdx.x * 128 + t) * k, out_ids + ((size_t)blockIdx.x * 128 + t) * k);
}

int main(int argc, char **argv) {
    const int chunks = argc > 1 ? atoi(argv[1]) : 17000;   // 10 M rows / 18 clusters / 32
    const int grid = 132;
    const int big_smem = argc > 2 ? atoi(argv[2]) : 1;
    for (int k : {10, 30, 64, 100}) {
        for (int mode = -1; mode < 4; mode++) {          // 3: tournament (group worsts)          // -1 one-lane rescan, 0 default (cooperative from k = 17), 1 append (2k / k+32), 2 append with 4k slots
            for (int in_smem = 1; in_smem >= 0; in_smem--) {
                const int cap = mode <= 0 ? k : mode == 3 ? list_cap_tourn(k) : mode == 1 ? (2 * k > k + 32 ? 2 * k : k + 32) : 4 * k > k + 64 ? 4 * k : k + 64;
                size_t smem = SCRATCH_BYTES + (in_smem ? (size_t)cap * EPI_THREADS * 8 : 0);
                if (smem > 220 * 1024) continue;
                if (big_smem) smem = 220 * 1024;   // like the tensor-core kernels: the operand ring leaves ~28 KB of L1
                float *g_keys, *ok; uint32_t *g_ids, *oi;
                cudaMalloc(&g_keys, (size_t)grid * cap * EPI_THREADS * 4); cudaMalloc(&g_ids, (size_t)grid * cap * EPI_THREADS * 4);
                cudaMalloc(&ok, (size_t)grid * 128 * k * 4); cudaMalloc(&oi, (size_t)grid * 128 * k * 4);
                cudaFuncSetAttribute(perf_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
                unsigned long long zero4[4] = {0, 0, 0, 0}, st[4] = {0, 0, 0, 0};
                (void)zero4;
                cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
                perf_kernel<<<grid, 128, smem>>>(chunks, k, cap, in_smem, mode == -1 ? 1 : 0, g_keys, g_ids, ok, oi);   // warm-up
#ifdef B200_LIST_STATS
                cudaMemcpyToSymbol(g_list_stats, zero4, sizeof(zero4));
#endif
                cudaEventRecord(e0);
                perf_kernel<<<grid, 128, smem>>>(chunks, k, cap, in_smem, mode == -1 ? 1 : 0, g_keys, g_ids, ok, oi);
                cudaEventRecord(e1);
                if (cudaDeviceSynchronize() != cudaSuccess) { printf("failed: %s\n", cudaGetErrorString(cudaGetLastError())); return 2; }
                float ms; cudaEventElapsedTime(&ms, e0, e1);
#ifdef B200_LIST_STATS
                cudaMemcpyFromSymbol(st, g_list_stats, sizeof(st));
#endif
                const double warps = grid * 4.0;
                printf("k %3d cap %3d %-6s %-6s  %8.3f ms   per warp: slow-path events %8.0f  compactions %7.1f  select rounds/compaction %5.1f  appends/lane %7.1f\n", k, cap,
                       mode == -1 ? "1-lane" : mode == 0 ? "deflt" : mode == 3 ? "tourn" : "append", in_smem ? "smem" : "global", ms, st[0] / warps, st[1] / warps,
                       st[1] ? (double)st[2] / 32.0 / st[1] : 0.0, st[3] / (warps * 32));
                cudaFree(g_keys); cudaFree(g_ids); cudaFree(ok); cudaFree(oi);
            }
        }
    }
    return 0;
}
