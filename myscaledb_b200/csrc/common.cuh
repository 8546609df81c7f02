// common.cuh -- shared device/host helpers for libb200search (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <atomic>
#include <memory>
#include <float.h>
#include <string>

#include "../../include/b200_search.h"

namespace b200 {

// ----------------------------------------------------------------------------------
// error plumbing (thread-local message, C-ABI returns a code)
// ----------------------------------------------------------------------------------
void set_error(const std::string &msg);
int fail(int code, const std::string &msg);
extern thread_local int64_t g_launches;

#define B200_CUDA_OK(expr)                                                                         \
    do {                                                                                           \
        cudaError_t _e = (expr);                                                                   \
        if (_e != cudaSuccess)                                                                     \
            return ::b200::fail(B200_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
    } while (0)

#define B200_TRY(expr)             \
    do {                           \
        int _rc = (expr);          \
        if (_rc != B200_OK) return _rc; \
    } while (0)

// bytes the DevMem buffers of the process hold (b200_device_bytes)
inline std::atomic<int64_t> g_device_bytes{0};

// The one owner of device memory: every cudaMalloc and cudaFree of the library is here.  Move-only; the destructor frees.
// cudaFree waits for the device, so a buffer dropped on an error path is never freed under a kernel still reading it.
struct DevMem {
    void *p = nullptr;
    size_t cap = 0;
    uint64_t reallocs = 0;   // times p changed: a CUDA graph that baked p in is stale once this moves (corpus_state_epoch)

    DevMem() = default;
    DevMem(const DevMem &) = delete;
    DevMem &operator=(const DevMem &) = delete;
    DevMem(DevMem &&o) noexcept : p(o.p), cap(o.cap) {
        o.p = nullptr;
        o.cap = 0;
    }
    DevMem &operator=(DevMem &&o) noexcept {
        if (this != &o) {
            reset();
            p = o.p;
            cap = o.cap;
            o.p = nullptr;
            o.cap = 0;
        }
        return *this;
    }
    ~DevMem() { reset(); }

    // exactly `bytes`, in place of what the buffer held
    int alloc(size_t bytes) {
        reset();
        cudaError_t e = cudaMalloc(&p, bytes);
        if (e != cudaSuccess) {
            cudaGetLastError();
            p = nullptr;
            return fail(B200_ERR_NOMEM, "cudaMalloc(" + std::to_string(bytes) + ") failed: " + cudaGetErrorString(e));
        }
        cap = bytes;
        g_device_bytes += (int64_t)bytes;
        return B200_OK;
    }
    // grow-only workspace: at least `bytes`, with a quarter of slack so that slowly growing batches rarely reallocate
    int reserve(size_t bytes) { return bytes <= cap ? B200_OK : alloc(bytes + bytes / 4 + 256); }
    void reset() {
        reallocs++;
        if (!p) return;
        cudaFree(p);
        g_device_bytes -= (int64_t)cap;
        p = nullptr;
        cap = 0;
    }
    template <typename T>
    T *as() const { return reinterpret_cast<T *>(p); }
    size_t size() const { return cap; }
    explicit operator bool() const { return p != nullptr; }
};

// a corpus the library created for itself, freed with b200_corpus_free
struct CorpusFree {
    void operator()(b200_corpus *c) const { b200_corpus_free(c); }
};
using CorpusPtr = std::unique_ptr<b200_corpus, CorpusFree>;

__host__ __device__ static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
__host__ __device__ static inline int64_t round_up(int64_t a, int64_t b) { return ceil_div(a, b) * b; }

// opt-in dynamic shared memory of one block on sm_90 (227 KB)
constexpr int kSmemOptinBytes = 232448;

constexpr uint32_t kNoId = 0xffffffffu;
constexpr uint64_t kNoId64 = ~0ull;
template <typename IdT> struct NoId;
template <> struct NoId<uint32_t> { static constexpr uint32_t value = kNoId; };
template <> struct NoId<uint64_t> { static constexpr uint64_t value = kNoId64; };

// ----------------------------------------------------------------------------------
// ordering: smaller key is better, ties -> smaller id.  All metrics are mapped to
// such a key (IP: -score, cosine: -cos) so one top-k serves every metric.
// ----------------------------------------------------------------------------------
__host__ __device__ __forceinline__ bool better(float ka, uint32_t ia, float kb, uint32_t ib) {
    return ka < kb || (ka == kb && ia < ib);
}
__host__ __device__ __forceinline__ bool better(float ka, uint64_t ia, float kb, uint64_t ib) {
    return ka < kb || (ka == kb && ia < ib);
}

#ifdef __CUDACC__
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// The one rule for an unusable row or query (include/b200_search.h, "Unusable rows"): the fp32 sum of the squares of its d
// coordinates is not finite (a NaN or infinite coordinate, or one whose square overflows).  Every lane of the warp calls it
// and gets the answer.
__device__ __forceinline__ bool warp_row_usable(const float *x, int d) {
    float s = 0.f;
    for (int j = lane_id(); j < d; j += 32) s = fmaf(x[j], x[j], s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    return isfinite(s);
}

// Warp-cooperative sorted top-k list living in shared (or global) memory.
// keys/ids: k slots, sorted best-first, `n` valid.  All 32 lanes call with the same
// (key,id); n/thr are warp-uniform registers.
template <typename IdT>
struct WarpTopKT {
    float *keys;
    IdT *ids;
    int k;
    int n;
    float thr_key;      // key of the current k-th (FLT_MAX while n < k)
    IdT thr_id;

    __device__ __forceinline__ void init(float *keys_, IdT *ids_, int k_) {
        keys = keys_;
        ids = ids_;
        k = k_;
        n = 0;
        // faiss heap neutral value: only keys strictly below FLT_MAX ever enter
        // (so +inf distances of FLT_MAX-padded empty rows never do; NaN never does)
        thr_key = FLT_MAX;
        thr_id = 0;
    }

    // cheap pre-test usable per lane on its own candidate
    __device__ __forceinline__ bool passes(float key, IdT id) const {
        return better(key, id, thr_key, thr_id);
    }

    __device__ __forceinline__ void insert(float key, IdT id) {
        if (!passes(key, id)) return;
        const int lane = lane_id();
        int cnt = 0;
        for (int j = lane; j < n; j += 32) cnt += better(keys[j], ids[j], key, id) ? 1 : 0;
        const int pos = warp_sum(cnt);
        if (pos >= k) return;
        const int new_n = n < k ? n + 1 : k;
        // shift [pos, new_n-1) one slot to the right, highest chunk first
        const int last = new_n - 2;  // last index that moves
        if (last >= pos) {
            for (int base = pos + ((last - pos) / 32) * 32; base >= pos; base -= 32) {
                const int j = base + lane;
                float kv = 0.f;
                IdT iv = 0;
                const bool mv = j <= last;
                if (mv) {
                    kv = keys[j];
                    iv = ids[j];
                }
                __syncwarp();
                if (mv) {
                    keys[j + 1] = kv;
                    ids[j + 1] = iv;
                }
                __syncwarp();
            }
        }
        if (lane == 0) {
            keys[pos] = key;
            ids[pos] = id;
        }
        __syncwarp();
        n = new_n;
        if (n == k) {
            thr_key = keys[k - 1];
            thr_id = ids[k - 1];
        }
    }
};
using WarpTopK = WarpTopKT<uint32_t>;

// Rank-merge of L sorted lists (best-first, unused tail slots hold FLT_MAX keys) of k entries each, list l at
// keys + l * list_stride, into out[0..k): the rank of an element in the union is its own index plus, for every other
// list, the number of entries ahead of it (lower bound by binary search; ties -> smaller id, then smaller list index).
// Every thread of the CTA calls it after a __syncthreads() that completes the lists; out may be shared or global
// (distinct from the inputs).  Replaces "warp 0 inserts the other warps' lists one element at a time", which is
// O(L k^2 / 32) and dominated IVF probes with k in the hundreds.
template <typename IdT>
__device__ __forceinline__ void block_rank_merge(const float *keys, const IdT *ids, int L, int list_stride, int k,
                                                 float *out_keys, IdT *out_ids) {
    for (int j = threadIdx.x; j < k; j += blockDim.x) {
        out_keys[j] = FLT_MAX;
        out_ids[j] = NoId<IdT>::value;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < L * k; e += blockDim.x) {
        const int l = e / k, j = e - l * k;
        const float key = keys[(size_t)l * list_stride + j];
        if (!(key < FLT_MAX)) continue;
        const IdT id = ids[(size_t)l * list_stride + j];
        int rank = j;
        for (int l2 = 0; l2 < L && rank < k; l2++) {
            if (l2 == l) continue;
            const float *k2 = keys + (size_t)l2 * list_stride;
            const IdT *i2 = ids + (size_t)l2 * list_stride;
            int lo = 0, hi = k;  // first index whose entry is NOT better than (key, id)
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (better(k2[mid], i2[mid], key, id)) lo = mid + 1;
                else hi = mid;
            }
            if (l2 < l && lo < k && k2[lo] == key && i2[lo] == id) lo++;
            rank += lo;
        }
        if (rank < k) {
            out_keys[rank] = key;
            out_ids[rank] = id;
        }
    }
}

// ---- small PTX wrappers -----------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint4 ldg_stream(const uint4 *p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}
#endif  // __CUDACC__

}  // namespace b200
