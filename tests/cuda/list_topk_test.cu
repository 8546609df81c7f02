// Unit test of the per-thread top-k list (csrc/gemm_common.cuh: list_insert / epilogue_chunk / list_publish) outside the
// tensor-core kernels: 128 threads = 128 independent "queries", each shown the same number of 32-wide chunks of synthetic keys
// (heavy ties included); the published list of every thread must equal the k smallest (key, id) of what it was shown -- in the
// rescan and in the tournament form at every k (list_bind picks one of them by k; the test overrides `tourn` to run both).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O2 -std=c++17 -I myscaledb_b200/csrc tests/cuda/list_topk_test.cu -o tests/cuda/list_topk_test
#include <algorithm>
#include <cstdio>
#include <random>
#include <vector>

#include "gemm_common.cuh"

using namespace b200;
using namespace b200::gemm;

__global__ void list_test_kernel(const float *keys /*[chunks][128][32]*/, int chunks, int k, int tourn, float *list_keys, uint32_t *list_ids,
                                 float *out_keys, uint32_t *out_ids) {
    __shared__ float scratch_all[32 * EPI_THREADS];
    const int t = threadIdx.x;
    ThreadTopK list;
    list.n = 0;
    list.worst = 0;
    list.thr_key = FLT_MAX;
    list.thr_id = 0;
    list_bind(list, list_keys, list_ids, t, k);
    list.tourn = tourn;
    __shared__ __align__(16) float one[32], zero[32];   // side arrays live in shared memory (ld.shared in side_fma32)
    for (int j = 0; j < 32; j++) {
        if (t == 0) {
            one[j] = 1.f;
            zero[j] = 0.f;
        }
    }
    __syncthreads();
    for (int c = 0; c < chunks; c++) {
        float v[32];
        for (int j = 0; j < 32; j++) v[j] = keys[((size_t)c * EPI_THREADS + t) * 32 + j];
        __syncwarp();
        epilogue_chunk(list, v, true, one, zero, (uint32_t)c * 32u, false, 0, scratch_all + t);
    }
    list_publish(list, out_keys + (size_t)t * k, out_ids + (size_t)t * k);
}

int main() {
    std::mt19937 rng(1234);
    int cases = 0, bad = 0;
    for (int k : {1, 10, 16, 17, 30, 64, 100, 256}) {
        for (int tourn = 0; tourn < 2; tourn++) {
            const int cap = tourn ? list_cap_tourn(k) : k;
            for (int dist = 0; dist < 4; dist++) {
                const int chunks = dist == 3 ? 3 : 200;
                std::vector<float> h((size_t)chunks * EPI_THREADS * 32);
                for (size_t i = 0; i < h.size(); i++) {
                    const int c = (int)(i / (EPI_THREADS * 32)), j = (int)(i % 32);
                    switch (dist) {
                        case 0: h[i] = std::uniform_real_distribution<float>(-1.f, 1.f)(rng); break;
                        case 1: h[i] = (float)(int)(rng() % 7);                       break;   // ties everywhere
                        case 2: h[i] = -(float)(c * 32 + j);                          break;   // every key beats all before it
                        default: h[i] = (float)(rng() % 1000);                        break;   // fewer rows than cap
                    }
                }
                float *d_keys, *d_lk, *d_ok;
                uint32_t *d_li, *d_oi;
                cudaMalloc(&d_keys, h.size() * 4);
                cudaMalloc(&d_lk, (size_t)cap * EPI_THREADS * 4);
                cudaMalloc(&d_li, (size_t)cap * EPI_THREADS * 4);
                cudaMalloc(&d_ok, (size_t)k * EPI_THREADS * 4);
                cudaMalloc(&d_oi, (size_t)k * EPI_THREADS * 4);
                cudaMemcpy(d_keys, h.data(), h.size() * 4, cudaMemcpyHostToDevice);
                list_test_kernel<<<1, EPI_THREADS>>>(d_keys, chunks, k, tourn, d_lk, d_li, d_ok, d_oi);
                if (cudaDeviceSynchronize() != cudaSuccess) {
                    printf("kernel failed: %s\n", cudaGetErrorString(cudaGetLastError()));
                    return 2;
                }
                std::vector<float> ok((size_t)k * EPI_THREADS);
                std::vector<uint32_t> oi((size_t)k * EPI_THREADS);
                cudaMemcpy(ok.data(), d_ok, ok.size() * 4, cudaMemcpyDeviceToHost);
                cudaMemcpy(oi.data(), d_oi, oi.size() * 4, cudaMemcpyDeviceToHost);
                for (int t = 0; t < EPI_THREADS; t++) {
                    std::vector<std::pair<float, uint32_t>> all;
                    for (int c = 0; c < chunks; c++)
                        for (int j = 0; j < 32; j++) all.push_back({h[((size_t)c * EPI_THREADS + t) * 32 + j], (uint32_t)(c * 32 + j)});
                    std::sort(all.begin(), all.end());
                    for (int e = 0; e < k; e++) {
                        const bool have = e < (int)all.size();
                        const float wk = have ? all[e].first : FLT_MAX;
                        const uint32_t wi = have ? all[e].second : kNoId;
                        if (ok[(size_t)t * k + e] != wk || oi[(size_t)t * k + e] != wi) {
                            if (bad < 10)
                                printf("MISMATCH tourn %d k %d cap %d dist %d thread %d slot %d: got (%g, %u) want (%g, %u)\n", tourn, k, cap, dist, t, e,
                                       ok[(size_t)t * k + e], oi[(size_t)t * k + e], wk, wi);
                            bad++;
                            break;
                        }
                    }
                }
                cases++;
                cudaFree(d_keys); cudaFree(d_lk); cudaFree(d_li); cudaFree(d_ok); cudaFree(d_oi);
            }
        }
    }
    printf("%d cases, %d mismatching lists\n", cases, bad);
    return bad ? 1 : 0;
}
