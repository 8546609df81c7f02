// ingest.cu -- host ingest path: pageable host memory -> HBM at PCIe speed.
//
// The reference hands brute-force search a part column that lives in ordinary (pageable) heap memory
// (MergeTreeVSManager::vectorScanWithoutIndex copies ColumnArray data into a std::vector<float>,
// VectorIndex/Storages/MergeTreeVSManager.cpp:1335-1392), and VIPartReader hands index build chunks the same way
// (VectorIndex/Common/VIPartReader.h:170-304).  cudaMemcpy from pageable memory is staged by the driver through one
// bounce buffer on the calling thread (one core's memcpy rate); here several threads fill a ring of pinned chunks and
// every filled chunk is queued as its own async H2D copy, so the bus, not a core, is the limit.  SURVEY section 8(f)3.
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <thread>
#include <vector>

#include "common.cuh"
#include "kernels.h"

namespace b200 {
namespace {

constexpr size_t kChunk = 8u << 20;   // 8 MiB per pinned slot
constexpr int kSlots = 8;             // 64 MiB of pinned memory per process
constexpr size_t kMinStaged = 32u << 20;

struct Stager {
    std::mutex mu;
    char *pinned = nullptr;
    cudaEvent_t ev[kSlots] = {};
    bool tried = false;
    // events belong to the device that is current when they are created: one stager per device, created with that
    // device current (one process-wide event set fails on the second GPU of a multi-device process)
    bool init(int device) {
        if (tried) return pinned != nullptr;
        tried = true;
        if (cudaSetDevice(device) != cudaSuccess) return false;
        if (cudaHostAlloc(reinterpret_cast<void **>(&pinned), kChunk * kSlots, cudaHostAllocDefault) != cudaSuccess) {
            cudaGetLastError();
            pinned = nullptr;
            return false;
        }
        for (auto &e : ev) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
        return true;
    }
};
constexpr int kMaxDevices = 64;
Stager g_stagers[kMaxDevices];

int stager_threads() {
    if (const char *ev = getenv("B200_INGEST_THREADS")) return std::max(0, atoi(ev));
    const unsigned hw = std::thread::hardware_concurrency();
    return (int)std::min<unsigned>(8, std::max<unsigned>(1, hw / 2));
}

}  // namespace

// Copies `bytes` from host `src` to device `dst` on stream `s` and returns once every byte is QUEUED and the pinned
// ring is no longer needed (i.e. after a stream synchronise for the staged form).  Small copies, B200_INGEST_THREADS=0
// or a failed pinned allocation use plain cudaMemcpyAsync.
int staged_h2d(void *dst, const void *src, size_t bytes, int device, cudaStream_t s) {
    const int threads = bytes >= kMinStaged ? stager_threads() : 0;
    if (threads <= 0) {
        B200_CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s));
        return B200_OK;
    }
    if (device < 0 || device >= kMaxDevices) {
        B200_CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s));
        return B200_OK;
    }
    Stager &g_stager = g_stagers[device];
    std::lock_guard<std::mutex> lk(g_stager.mu);
    if (!g_stager.init(device)) {
        B200_CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s));
        return B200_OK;
    }
    const int64_t n_chunks = (int64_t)((bytes + kChunk - 1) / kChunk);
    std::atomic<int64_t> next{0};
    std::atomic<int64_t> queued[kSlots];
    for (auto &q : queued) q.store(-1);
    std::atomic<int> first_error{(int)cudaSuccess};
    auto work = [&]() {
        if (cudaSetDevice(device) != cudaSuccess) {
            first_error.store((int)cudaErrorInvalidDevice);
            return;
        }
        for (;;) {
            const int64_t i = next.fetch_add(1);
            if (i >= n_chunks) break;
            const int slot = (int)(i % kSlots);
            if (i >= kSlots) {  // the previous user of this slot must have been queued, then drained
                while (queued[slot].load(std::memory_order_acquire) != i - kSlots) {
                    if (first_error.load() != (int)cudaSuccess) return;
                    std::this_thread::yield();
                }
                cudaEventSynchronize(g_stager.ev[slot]);
            }
            const size_t off = (size_t)i * kChunk, len = std::min(kChunk, bytes - off);
            char *stage = g_stager.pinned + (size_t)slot * kChunk;
            memcpy(stage, reinterpret_cast<const char *>(src) + off, len);
            cudaError_t e = cudaMemcpyAsync(reinterpret_cast<char *>(dst) + off, stage, len, cudaMemcpyHostToDevice, s);
            if (e == cudaSuccess) e = cudaEventRecord(g_stager.ev[slot], s);
            if (e != cudaSuccess) first_error.store((int)e);
            queued[slot].store(i, std::memory_order_release);  // also on error: nobody may wait forever
        }
    };
    std::vector<std::thread> pool;
    const int t = (int)std::min<int64_t>(threads, n_chunks);
    for (int j = 1; j < t; j++) pool.emplace_back(work);
    work();
    for (auto &th : pool) th.join();
    const cudaError_t e = (cudaError_t)first_error.load();
    if (e != cudaSuccess) return fail(B200_ERR_CUDA, std::string("staged host->device copy: ") + cudaGetErrorString(e));
    B200_CUDA_OK(cudaStreamSynchronize(s));  // the ring is free for the next caller
    return B200_OK;
}

}  // namespace b200
