// gemm_common.cuh -- PTX wrappers (mbarrier, TMA, wgmma), the accumulator hand-off, the per-thread top-k list and the
// chunk filter shared by the tensor-core kernels (ip_gemm_sm90.cu, ivf_gemm_sm90.cu).
#pragma once
#include <cuda.h>

#include "common.cuh"
#include "kernels.h"

namespace b200 {
namespace gemm {


constexpr int BM = 128;            // queries per CTA tile (two wgmma M = 64 halves)
constexpr int BN = 256;            // corpus rows per tile (side arrays, pacing, IVF pages)
constexpr int HN = 128;            // corpus rows per MMA pass: the tile is computed as two N = 128 halves
constexpr int BK = 64;             // bf16 per k-block = one 128-byte swizzle row
constexpr int UMMA_K = 16;         // bf16 wgmma K
constexpr int EPI_THREADS = 128;   // the consumer warpgroup: MMAs, then the top-k epilogue (thread t = query row t)
constexpr int NUM_THREADS = EPI_THREADS + 32;  // IVF kernel: + one TMA producer warp (warp 4)
constexpr int SMEM_ALIGN_SLACK = 1024;
constexpr int MAX_STAGES = 4;
constexpr int SMEM_LIMIT = kSmemOptinBytes;

constexpr int SCRATCH_BYTES = 32 * EPI_THREADS * 4;  // IVF kernel: epilogue slow-path scratch [32][128] floats
// Accumulator hand-off of the IVF kernel (the flat kernel filters from the registers and stages only the groups of 32 columns that
// can enter a list, ip_gemm_sm90.cu): the warpgroup's registers are written column-major into shared memory, 64 columns at a time
// ([ACC_COLS][ACC_LD] floats; the padding of 4 makes both the fragment stores and the per-row reads of the epilogue
// conflict-free).  It takes the place of tensor memory: the epilogue reads its query row in chunks of 32 columns.  Staging a
// quarter of the tile rather than a half keeps 33 KB of shared memory for the operand ring, the lists and the PQ codebook.
constexpr int ACC_COLS = 64;
constexpr int ACC_LD = BM + 4;
constexpr int ACC_BYTES = ACC_COLS * ACC_LD * 4;     // 33 KB

// Operand type of a tensor-core kernel: bf16 rows, fp32 rows as 3xTF32, or binary rows (1-bit AND + popcount, s32 sums)
enum class Operand { BF16, TF32X3, B1 };

// Operand geometry of the tensor-core kernels, and the shared-memory layout of the IVF kernel for a ring of `st` stages (the flat
// kernel's is Op in ip_gemm_sm90.cu).  Every k-block row is one 128-byte swizzle row (64 bf16, 32 fp32 or 1024 bits); for binary
// rows an "element" is a byte.  A plane is the k-block of 128 rows; fp32 rows (TF32X3, flat kernel only) have hi and lo planes.
// IVF stage s: the query k-block and the half tile's corpus k-block.
template <Operand OP>
struct Layout {
    static constexpr bool F32X3 = OP == Operand::TF32X3;
    static constexpr int KB = F32X3 ? 32 : OP == Operand::B1 ? 128 : 64;     // elements per k-block
    static constexpr int MMA_K = F32X3 ? 8 : OP == Operand::B1 ? 32 : 16;    // elements per wgmma (b1: 256 bits)
    static constexpr int A_PLANE = BM * 128;                // 16 KB
    static constexpr int B_PLANE = HN * 128;                // 16 KB
    static constexpr int PLANES = F32X3 ? 2 : 1;            // hi / lo
    static constexpr int STAGE_BYTES = PLANES * (A_PLANE + B_PLANE);
    static constexpr int TX_BYTES = STAGE_BYTES - (PLANES - 1) * B_PLANE;   // what TMA writes (the B lo plane is computed)
    __host__ __device__ static constexpr int off_acc(int st) { return st * STAGE_BYTES; }
    __host__ __device__ static constexpr int off_side(int st) { return off_acc(st) + ACC_BYTES; }  // scale[256], bias[256]
    __host__ __device__ static constexpr int off_bar(int st) { return off_side(st) + 2 * BN * 4; }
    __host__ __device__ static constexpr int off_scratch(int st) { return off_bar(st) + 256; }
    __host__ __device__ static constexpr int off_list(int st) { return off_scratch(st) + SCRATCH_BYTES; }
};

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t addr, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(addr), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    while (!mbar_try_wait(addr, parity)) {
    }
}

__device__ __forceinline__ void tma_load_2d(const CUtensorMap *map, uint64_t *bar, void *dst, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
            smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}

// one lane of a converged warp (keeps the surrounding control flow warp-uniform)
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile(
        "{\n\t"
        ".reg .pred P;\n\t"
        "elect.sync _|P, 0xffffffff;\n\t"
        "selp.b32 %0, 1, 0, P;\n\t"
        "}\n"
        : "=r"(pred));
    return pred != 0;
}

// order-preserving float <-> u32 (atomicMin on the encoding = min of the floats): the shared per-query bound of the IVF scans
__device__ __forceinline__ uint32_t bound_encode(float f) {
    const uint32_t b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float bound_decode(uint32_t u) { return (u & 0x80000000u) ? __uint_as_float(u & 0x7fffffffu) : __uint_as_float(~u); }

// named barrier of the consumer warpgroup (id 1; 0 is __syncthreads)
__device__ __forceinline__ void wg_bar() { asm volatile("bar.sync 1, 128;" ::: "memory"); }

// wgmma shared-memory descriptor of a K-major, 128-byte swizzled operand tile: rows of 128 B, 8-row atoms of 1024 B.
// Other stages / k-steps / row offsets are plain adds on the 14-bit (address >> 4) field (shared addresses < 2^18).
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);  // start address
    d |= (uint64_t)1 << 16;                      // leading byte offset (unused for swizzled K-major)
    d |= (uint64_t)(1024 >> 4) << 32;            // stride byte offset: 8 rows * 128 B
    d |= (uint64_t)1 << 62;                      // SWIZZLE_128B
    return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// the 64 accumulator operands of one wgmma m64n128, constraint C: "+f" (fp32) or "+r" (s32)
#define B200_ACC64_AS(C, v)                                                                                                     \
    C(v[0]), C(v[1]), C(v[2]), C(v[3]), C(v[4]), C(v[5]), C(v[6]), C(v[7]), C(v[8]), C(v[9]), C(v[10]), C(v[11]), C(v[12]),     \
        C(v[13]), C(v[14]), C(v[15]), C(v[16]), C(v[17]), C(v[18]), C(v[19]), C(v[20]), C(v[21]), C(v[22]), C(v[23]), C(v[24]), \
        C(v[25]), C(v[26]), C(v[27]), C(v[28]), C(v[29]), C(v[30]), C(v[31]), C(v[32]), C(v[33]), C(v[34]), C(v[35]), C(v[36]), \
        C(v[37]), C(v[38]), C(v[39]), C(v[40]), C(v[41]), C(v[42]), C(v[43]), C(v[44]), C(v[45]), C(v[46]), C(v[47]), C(v[48]), \
        C(v[49]), C(v[50]), C(v[51]), C(v[52]), C(v[53]), C(v[54]), C(v[55]), C(v[56]), C(v[57]), C(v[58]), C(v[59]), C(v[60]), \
        C(v[61]), C(v[62]), C(v[63])
#define B200_ACC64(v) B200_ACC64_AS("+f", v)
#define B200_ACC64_REGS                                                                                                         \
    "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, " \
    "%26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, "   \
    "%50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"

// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, bf16 operands (both K-major in shared memory), fp32 accumulators
__device__ __forceinline__ void wgmma_bf16_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " B200_ACC64_REGS ", %64, %65, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : B200_ACC64(d)
        : "l"(adesc), "l"(bdesc), "r"(accum));
}
// D[64 x 128] (+)= A[64 x 8] * B[128 x 8]^T, tf32 operands (K-major), fp32 accumulators
__device__ __forceinline__ void wgmma_tf32_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 " B200_ACC64_REGS ", %64, %65, p, 1, 1;\n\t"
        "}\n"
        : B200_ACC64(d)
        : "l"(adesc), "l"(bdesc), "r"(accum));
}
// D[64 x 128] (+)= popc(A[64 x 256 bits] AND B[128 x 256 bits]), binary operands (K-major, 32 bytes per row and k-step), s32
// accumulators.  Both operands share one byte layout, so which bit of a byte pairs with which does not matter.
__device__ __forceinline__ void wgmma_b1_n128(int32_t (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k256.s32.b1.b1.and.popc " B200_ACC64_REGS ", %64, %65, p;\n\t"
        "}\n"
        : B200_ACC64_AS("+r", d)
        : "l"(adesc), "l"(bdesc), "r"(accum));
}

// Store columns [64 Q, 64 Q + 64) of the warpgroup's two 64 x 128 accumulator fragments column-major into acc
// ([ACC_COLS][ACC_LD]) as fp32 (s32 AND counts convert exactly: they are below 2^24).  Fragment layout of wgmma m64nN: warp w
// of the warpgroup, lane l holds rows 16 w + l / 4 (+ 8) and columns 8 i + 2 (l % 4) (+ 1), in d[4 i] (row, column),
// d[4 i + 1] (row, column + 1), d[4 i + 2] (row + 8, column), d[4 i + 3] (row + 8, column + 1).
template <int Q, typename T>
__device__ __forceinline__ void acc_store(float *acc, const T (&d0)[64], const T (&d1)[64]) {
    const int warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    const int r = warp * 16 + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < ACC_COLS / 8; j++) {
        const int i = Q * (ACC_COLS / 8) + j;
        float *col = acc + (8 * j + c) * ACC_LD + r;
        col[0] = (float)d0[4 * i];
        col[ACC_LD] = (float)d0[4 * i + 1];
        col[8] = (float)d0[4 * i + 2];
        col[ACC_LD + 8] = (float)d0[4 * i + 3];
        col[64] = (float)d1[4 * i];
        col[ACC_LD + 64] = (float)d1[4 * i + 1];
        col[72] = (float)d1[4 * i + 2];
        col[ACC_LD + 72] = (float)d1[4 * i + 3];
    }
}
// this thread's query row, 32 columns from column c0 of the staged accumulator
__device__ __forceinline__ void acc_load32(const float *acc, int row, int c0, float (&v)[32]) {
    const float *p = acc + c0 * ACC_LD + row;
#pragma unroll
    for (int j = 0; j < 32; j++) v[j] = p[j * ACC_LD];
}

// Per-thread top-k as an UNSORTED buffer (element j at [j * EPI_THREADS]: bank-conflict free in smem,
// coalesced in global scratch) plus the position of its current worst element.  An insert overwrites
// the worst slot and rescans the k slots with independent loads; a sorted list would pay a dependent
// load-compare-store chain per shifted element, which makes the start-up "insert storm" of a launch expensive.
// The buffer is sorted once, when the CTA publishes its partial list.  From k = list_tourn_min_k it is the tournament form
// (kernels.h, list_insert).
struct ThreadTopK {
    float *keys;       // entry j of this thread's list: keys[j * EPI_THREADS]
    uint32_t *ids;
    int k, n, worst;
    int tourn;         // k >= list_tourn_min_k: slots [k, list_cap_for(k)) hold the worst (key, id) of every group of 8 / 16 entries; `worst` = a group
    float thr_key;     // key of the current worst kept element (FLT_MAX while n < k)
    uint32_t thr_id;
};

// keys_base / ids_base: the lists of the CTA's 128 threads, interleaved (entry j of all 128 lists side by side), with
// list_cap_for(k) slots each.  The stride is the compile-time constant EPI_THREADS, so the rescans address their entries with
// immediate offsets.
__device__ __forceinline__ void list_bind(ThreadTopK &t, float *keys_base, uint32_t *ids_base, int row, int k) {
    t.k = k;
    t.tourn = k >= list_tourn_min_k ? 1 : 0;
    t.keys = keys_base + row;
    t.ids = ids_base + row;
}

__device__ __forceinline__ void list_insert(ThreadTopK &t, float key, uint32_t id) {
    if (!better(key, id, t.thr_key, t.thr_id)) return;
    if (t.tourn) {
        // Two-level form: the worst entry of each group of G = 8 / 16 is cached behind the list, so an insert rescans ONE group (to
        // find the slot of the entry it evicts and that group's new worst) and the group worsts: 2 (G + k / G) loads instead of 2 k.
        const int G = list_tourn_group(t.k);
        const int ng = (t.k + G - 1) / G;
        if (t.n < t.k) {
            t.keys[t.n * EPI_THREADS] = key;
            t.ids[t.n * EPI_THREADS] = id;
            t.n++;
            if (t.n < t.k) return;
            for (int g = 0; g < ng; g++) {   // the list just became full: every group's worst, once
                const int base = g * G, end = base + G < t.k ? base + G : t.k;
                float wk = t.keys[base * EPI_THREADS];
                uint32_t wi = t.ids[base * EPI_THREADS];
                for (int j = base + 1; j < end; j++) {
                    const float kj = t.keys[j * EPI_THREADS];
                    const uint32_t ij = t.ids[j * EPI_THREADS];
                    if (better(wk, wi, kj, ij)) {
                        wk = kj;
                        wi = ij;
                    }
                }
                t.keys[(t.k + g) * EPI_THREADS] = wk;
                t.ids[(t.k + g) * EPI_THREADS] = wi;
            }
        } else {
            const int g = t.worst;   // the group that holds the evicted entry (= the current threshold)
            const int base = g * G, end = base + G < t.k ? base + G : t.k;
            float wk = 0.f;
            uint32_t wi = 0;
            int slot = -1;
            bool have = false;
            for (int j = base; j < end; j++) {
                float kj = t.keys[j * EPI_THREADS];
                uint32_t ij = t.ids[j * EPI_THREADS];
                if (slot < 0 && kj == t.thr_key && ij == t.thr_id) {
                    slot = j;
                    kj = key;
                    ij = id;
                }
                if (!have || better(wk, wi, kj, ij)) {
                    wk = kj;
                    wi = ij;
                    have = true;
                }
            }
            if (slot < 0) slot = base;   // cannot happen (ids are unique and the threshold is an entry of this group); never write out of range
            t.keys[slot * EPI_THREADS] = key;
            t.ids[slot * EPI_THREADS] = id;
            t.keys[(t.k + g) * EPI_THREADS] = wk;
            t.ids[(t.k + g) * EPI_THREADS] = wi;
        }
        float wk = t.keys[t.k * EPI_THREADS];
        uint32_t wi = t.ids[t.k * EPI_THREADS];
        int wg = 0;
        for (int g = 1; g < ng; g++) {
            const float kg = t.keys[(t.k + g) * EPI_THREADS];
            const uint32_t ig = t.ids[(t.k + g) * EPI_THREADS];
            if (better(wk, wi, kg, ig)) {
                wk = kg;
                wi = ig;
                wg = g;
            }
        }
        t.worst = wg;
        t.thr_key = wk;
        t.thr_id = wi;
        return;
    }
    if (t.n < t.k) {
        t.keys[t.n * EPI_THREADS] = key;
        t.ids[t.n * EPI_THREADS] = id;
        t.n++;
        if (t.n < t.k) return;
    } else {
        t.keys[t.worst * EPI_THREADS] = key;
        t.ids[t.worst * EPI_THREADS] = id;
    }
    // rescan for the worst (largest key, ties -> larger id)
    float wk = t.keys[0];
    uint32_t wi = t.ids[0];
    int wp = 0;
    for (int j = 1; j < t.k; j++) {
        const float kj = t.keys[j * EPI_THREADS];
        const uint32_t ij = t.ids[j * EPI_THREADS];
        if (better(wk, wi, kj, ij)) {
            wk = kj;
            wi = ij;
            wp = j;
        }
    }
    t.worst = wp;
    t.thr_key = wk;
    t.thr_id = wi;
}

// sort the n kept entries best-first (insertion sort, once per kernel) and publish them
static __device__ __noinline__ void list_publish(ThreadTopK &t, float *out_keys, uint32_t *out_ids) {
    for (int i = 1; i < t.n; i++) {
        const float ki = t.keys[i * EPI_THREADS];
        const uint32_t ii = t.ids[i * EPI_THREADS];
        int j = i;
        while (j > 0 && better(ki, ii, t.keys[(j - 1) * EPI_THREADS], t.ids[(j - 1) * EPI_THREADS])) {
            t.keys[j * EPI_THREADS] = t.keys[(j - 1) * EPI_THREADS];
            t.ids[j * EPI_THREADS] = t.ids[(j - 1) * EPI_THREADS];
            j--;
        }
        t.keys[j * EPI_THREADS] = ki;
        t.ids[j * EPI_THREADS] = ii;
    }
    for (int j = 0; j < t.k; j++) {
        out_keys[j] = j < t.n ? t.keys[j * EPI_THREADS] : FLT_MAX;
        out_ids[j] = j < t.n ? t.ids[j * EPI_THREADS] : kNoId;
    }
}

// v[j] = v[j] * scale[j] + bias[j] for the 32 columns of a chunk; scale / bias are the per-tile side arrays in SHARED memory.
// Explicit ld.shared: through generic pointers the compiler emitted LD.E.128 (generic path, scoreboarded like a global load).
__device__ __forceinline__ void side_fma32(float (&v)[32], const float *scale, const float *bias) {
    const uint32_t sa = smem_u32(scale), ba = smem_u32(bias);
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
        float s0, s1, s2, s3, b0, b1, b2, b3;
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(s0), "=f"(s1), "=f"(s2), "=f"(s3) : "r"(sa + j * 4));
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(b0), "=f"(b1), "=f"(b2), "=f"(b3) : "r"(ba + j * 4));
        v[j] = fmaf(v[j], s0, b0);
        v[j + 1] = fmaf(v[j + 1], s1, b1);
        v[j + 2] = fmaf(v[j + 2], s2, b2);
        v[j + 3] = fmaf(v[j + 3], s3, b3);
    }
}

// Jaccard key of one AND count (as fp32), with the integer expression and the IEEE division of binary_scan_kernel, returned
// negated for the max-tree form of epilogue_chunk.  A row with side scale 0 (filtered, out of range) gives -inf, i.e. key +inf,
// which never enters a list.
__device__ __forceinline__ float jaccard_negkey(float v, int pq, float scale, float popc_y) {
    const bool live = scale != 0.f;
    const int x_and = (int)v, x_or = pq + (live ? (int)popc_y : 0) - x_and;
    const float key = x_or == 0 ? 0.f : (float)(x_or - x_and) / (float)x_or;
    return live ? -key : __int_as_float(0xff800000);
}

// jaccard_negkey of one chunk of 32 staged AND counts; scale / popc_y are the tile's side arrays in SHARED memory.
__device__ __forceinline__ void jaccard_keys32(float (&v)[32], int pq, const float *scale, const float *popc_y) {
    const uint32_t sa = smem_u32(scale), ba = smem_u32(popc_y);
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
        float s[4], b[4];
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(s[0]), "=f"(s[1]), "=f"(s[2]), "=f"(s[3]) : "r"(sa + j * 4));
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(b[0]), "=f"(b[1]), "=f"(b[2]), "=f"(b[3]) : "r"(ba + j * 4));
#pragma unroll
        for (int i = 0; i < 4; i++) v[j + i] = jaccard_negkey(v[j + i], pq, s[i], b[i]);
    }
}

// Filter one chunk of 32 accumulator columns of this thread's query row.
// Fast path (steady state): reduce the chunk to its best key with FMNMX3 trees, one warp vote,
// done.  Slow path (some lane of the warp can improve its list; frequent only during the first
// tiles of a launch): every lane parks its 32 keys in a shared-memory scratch column and the WARP
// loops while any lane still has a candidate bit, each lane popping its own lowest bit and doing
// an inlined insert (per-element calls under divergence serialise the lanes during the start-up
// "insert storm" of a launch).
// scratch: this thread's column of a [32][LD] float array.  It may be the 32 staged accumulator columns the chunk was loaded
// from: only this thread reads its row of them, and it holds them in v by now.
template <int LD = EPI_THREADS>
__device__ __forceinline__ void epilogue_chunk(ThreadTopK &list, float (&v)[32], bool use_side, const float *scale,
                                               const float *bias, uint32_t id0, bool tail, int64_t n, float *scratch,
                                               float ext_bound = FLT_MAX /* a valid upper bound of the k-th key known from elsewhere */) {
    const float thr = fminf(list.thr_key, ext_bound);
    bool mine;
    if (use_side) {
        side_fma32(v, scale, bias);  // 16 broadcast LDS.128
        float m0 = fminf(v[0], v[1]), m1 = fminf(v[2], v[3]), m2 = fminf(v[4], v[5]), m3 = fminf(v[6], v[7]);
#pragma unroll
        for (int j = 8; j < 32; j += 8) {
            m0 = fminf(m0, fminf(v[j], v[j + 1]));
            m1 = fminf(m1, fminf(v[j + 2], v[j + 3]));
            m2 = fminf(m2, fminf(v[j + 4], v[j + 5]));
            m3 = fminf(m3, fminf(v[j + 6], v[j + 7]));
        }
        mine = fminf(fminf(m0, m1), fminf(m2, m3)) <= thr;
    } else {
        // plain IP: rank on the raw score with max trees; the key (-score) is formed only when needed
        float m0 = fmaxf(v[0], v[1]), m1 = fmaxf(v[2], v[3]), m2 = fmaxf(v[4], v[5]), m3 = fmaxf(v[6], v[7]);
#pragma unroll
        for (int j = 8; j < 32; j += 8) {
            m0 = fmaxf(m0, fmaxf(v[j], v[j + 1]));
            m1 = fmaxf(m1, fmaxf(v[j + 2], v[j + 3]));
            m2 = fmaxf(m2, fmaxf(v[j + 4], v[j + 5]));
            m3 = fmaxf(m3, fmaxf(v[j + 6], v[j + 7]));
        }
        mine = fmaxf(fmaxf(m0, m1), fmaxf(m2, m3)) >= -thr;
    }
    if (__any_sync(0xffffffffu, mine)) {
        uint32_t mask = 0;
#pragma unroll
        for (int j = 0; j < 32; j++) {
            const float key = use_side ? v[j] : -v[j];
            scratch[j * LD] = key;
            if (key <= thr) mask |= 1u << j;
        }
        if (tail && !use_side) {  // rows past the end of the corpus (zero-filled by TMA) are not candidates
            const int64_t left = n - (int64_t)id0;
            mask = left >= 32 ? mask : left <= 0 ? 0u : (mask & ((1u << left) - 1u));
        }
        while (__any_sync(0xffffffffu, mask != 0)) {
            if (mask) {
                const int j = __ffs(mask) - 1;
                mask &= mask - 1;
                list_insert(list, scratch[j * LD], id0 + (uint32_t)j);
            }
        }
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(ptr);
    }
    return fn;
}

// 2-D bf16 tensor map over row-major [rows][d_pad], box = [box_rows][64 elements], 128-byte swizzle
inline bool encode_rows_map(CUtensorMap *map, const void *base, int64_t rows, int d_pad, int box_rows) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return false;
    const cuuint64_t dims[2] = {(cuuint64_t)d_pad, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)d_pad * 2};
    const cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
    const cuuint32_t estr[2] = {1, 1};
    return fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(base), dims, strides, box, estr,
              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// 2-D byte tensor map over row-major [rows][row_bytes] (binary rows), box = [box_rows][128 bytes], 128-byte swizzle.  Columns
// past row_bytes are zero-filled by TMA (zero bits add nothing to an AND count); row_bytes must be a multiple of 16.
inline bool encode_bytes_map(CUtensorMap *map, const void *base, int64_t rows, int row_bytes, int box_rows) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return false;
    const cuuint64_t dims[2] = {(cuuint64_t)row_bytes, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)row_bytes};
    const cuuint32_t box[2] = {128, (cuuint32_t)box_rows};
    const cuuint32_t estr[2] = {1, 1};
    return fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void *>(base), dims, strides, box, estr,
              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace gemm
}  // namespace b200
