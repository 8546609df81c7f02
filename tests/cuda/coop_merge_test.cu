// Unit test of the cooperative tile merge (csrc/ivf_coop.cuh) outside the tensor-core kernel: one warp, synthetic tiles.
// For every slot the final sorted list must equal the k smallest (key, id) of everything the slot was shown.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O2 -std=c++17 -I myscaledb_b200/csrc tests/cuda/coop_merge_test.cu -o tests/cuda/coop_merge_test
#include <algorithm>
#include <cstdio>
#include <random>
#include <vector>

#include "ivf_coop.cuh"

using namespace b200;
using namespace b200::gemm;

__global__ void coop_test_kernel(const float *keys /*[tiles][slots][256]*/, int tiles, int slots, int k, float *out_keys, uint32_t *out_ids, int *out_n) {
    extern __shared__ unsigned char smem[];
    const int lane = threadIdx.x;
    unsigned char *scratch = smem;                       // 16 KB tile buffer
    const CoopSmem cs = coop_smem_carve(smem + SCRATCH_BYTES, scratch, k);
    if (lane < kCoopMax) {
        CoopState st;
        st.n = 0; st.thr_key = FLT_MAX; st.thr_id = 0; st.buf = 0;
        cs.state[lane] = st;
    }
    __syncwarp();
    float thr = lane < slots ? FLT_MAX : -FLT_MAX;
    float *tile_row = cs.tilebuf + (size_t)(lane < kCoopMax ? lane : 0) * kTileBufStride;
    for (int t = 0; t < tiles; t++) {
        uint32_t chunk_mask = 0;
        for (int chunk = 0; chunk < 8; chunk++) {
            float v[32];
            __shared__ __align__(16) float one[32], zero[32];   // the side arrays live in shared memory (ld.shared in side_fma32)
            for (int j = 0; j < 32; j++) {
                v[j] = lane < slots ? keys[((size_t)t * slots + lane) * 256 + chunk * 32 + j] : 0.f;
                if (lane == 0) {
                    one[j] = 1.f;
                    zero[j] = 0.f;
                }
            }
            __syncwarp();
            coop_stage_chunk(thr, v, one, zero, tile_row, chunk, chunk_mask, lane);
        }
        __syncwarp();
        coop_merge_tile(cs, k, slots, chunk_mask, (uint32_t)t * 256u, lane, thr);
    }
    __syncwarp();
    for (int s = 0; s < slots; s++) {
        const CoopState st = cs.state[s];
        if (lane == 0) out_n[s] = st.n;
        for (int e = lane; e < st.n; e += 32) {
            out_keys[s * k + e] = cs.keys[st.buf][(size_t)s * k + e];
            out_ids[s * k + e] = cs.ids[st.buf][(size_t)s * k + e];
        }
    }
}

int main() {
    std::mt19937 rng(7);
    int failures = 0, cases = 0;
    for (int k : {1, 10, 40, 100, 256})
        for (int slots : {1, 2, 7, 16})
            for (int tiles : {1, 2, 3, 9})
                for (int mode = 0; mode < 3; mode++) {   // 0: gaussian, 1: integer keys (ties), 2: descending (every tile improves everything)
                    std::vector<float> h((size_t)tiles * slots * 256);
                    std::normal_distribution<float> nd(0.f, 1.f);
                    for (size_t i = 0; i < h.size(); i++) h[i] = mode == 0 ? nd(rng) : mode == 1 ? (float)(rng() % 17) : (float)(h.size() - i);
                    float *d_keys, *d_ok; uint32_t *d_oi; int *d_n;
                    cudaMalloc(&d_keys, h.size() * 4); cudaMalloc(&d_ok, (size_t)slots * k * 4); cudaMalloc(&d_oi, (size_t)slots * k * 4); cudaMalloc(&d_n, slots * 4);
                    cudaMemcpy(d_keys, h.data(), h.size() * 4, cudaMemcpyHostToDevice);
                    const size_t smem = SCRATCH_BYTES + coop_smem_bytes(k) + 64;
                    cudaFuncSetAttribute(coop_test_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
                    coop_test_kernel<<<1, 32, smem>>>(d_keys, tiles, slots, k, d_ok, d_oi, d_n);
                    if (cudaDeviceSynchronize() != cudaSuccess) { std::printf("CUDA error: %s\n", cudaGetErrorString(cudaGetLastError())); return 2; }
                    std::vector<float> ok((size_t)slots * k); std::vector<uint32_t> oi((size_t)slots * k); std::vector<int> on(slots);
                    cudaMemcpy(ok.data(), d_ok, ok.size() * 4, cudaMemcpyDeviceToHost); cudaMemcpy(oi.data(), d_oi, oi.size() * 4, cudaMemcpyDeviceToHost);
                    cudaMemcpy(on.data(), d_n, slots * 4, cudaMemcpyDeviceToHost);
                    cases++;
                    for (int s = 0; s < slots; s++) {
                        std::vector<std::pair<float, uint32_t>> all;
                        for (int t = 0; t < tiles; t++) for (int c = 0; c < 256; c++) all.push_back({h[((size_t)t * slots + s) * 256 + c], (uint32_t)(t * 256 + c)});
                        std::sort(all.begin(), all.end());
                        const int want = std::min<int>(k, (int)all.size());
                        bool bad = on[s] != want;
                        for (int e = 0; !bad && e < want; e++) bad = ok[s * k + e] != all[e].first || oi[s * k + e] != all[e].second;
                        if (bad) {
                            failures++;
                            if (failures < 8) std::printf("MISMATCH k=%d slots=%d tiles=%d mode=%d slot=%d n=%d (want %d) first got (%g,%u) want (%g,%u)\n", k, slots, tiles, mode, s,
                                                          on[s], want, ok[s * k], oi[s * k], all[0].first, all[0].second);
                        }
                    }
                    cudaFree(d_keys); cudaFree(d_ok); cudaFree(d_oi); cudaFree(d_n);
                }
    std::printf("%s: %d cases, %d slot mismatches\n", failures ? "COOP MERGE FAILED" : "COOP MERGE OK", cases, failures);
    return failures ? 1 : 0;
}
