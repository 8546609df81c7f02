// ivf_aq.cu -- anisotropic (score-aware) product quantisation for IVFPQ / SCANN / HNSWPQ under IP and cosine
// (`aq_threshold=T`, Guo et al., "Accelerating Large-Scale Inference with Anisotropic Vector Quantization", ICML 2020).
//
// The codes and the file format are those of plain PQ; only the choice of codebooks and codes differs.
//   * x is the row as indexed (unit length under cosine).  Its reconstruction is x^ = c_l + sum_j e_j (c_l its list centroid,
//     e_j its codeword in sub-space j), the residual r = x - x^.
//   * loss l(x, x^) = ||r||^2 + w <r, x>^2, w = (eta - 1) / ||x||^2 (w = 0 when ||x|| = 0), eta = (d - 1) T^2 / (1 - T^2):
//     ScaNN's parallel-cost multiplier for a row of unit norm.  Dividing by ||x||^2 weights the error along x against the
//     error across it the same way for every row, whatever its norm.  eta = 1 (T^2 = 1 / d) is plain squared error.
//   * encoder (every sample row of every iteration, every added row): start from the nearest-codeword codes, then up to
//     kAqSweeps sweeps over j = 0 .. M - 1, stopping after a sweep that changed no code.  With s = <r, x> - <r_j, x_j> (the
//     other sub-spaces' part), candidate e of sub-space j costs ||a_j - e||^2 + w (s + <a_j - e, x_j>)^2 (a_j = x_j - c_l,j)
//     up to a constant; the code moves to the cheapest candidate (smallest index among equals) only when that is strictly
//     cheaper than the current one, so l never increases and the result is deterministic.  One warp per row, the candidates
//     of a sub-space split across lanes, fp32, a warp arg-min.
//   * codebook update (kAqIters iterations after the k-means codebooks on the 65 536-row sample): encode the sample, then for
//     j = 0 .. M - 1 solve, for every codeword e of sub-space j with members S (codes fixed),
//         (|S| I + sum_S w_i x_ij x_ij^T) e = sum_S [a_ij + w_i (<a_ij, x_ij> + s_ij) x_ij],   s_ij = p_i - <r_ij, x_ij>,
//     the exact minimiser of the members' loss over that block (positive definite for eta > 0), then refresh every
//     p_i = <r_i, x_i>.  A codeword without members keeps its value.  The normal equations are accumulated in fp64 in row order
//     (members found by a stable sort on the code, no floating-point atomics) and solved by Cholesky in fp64; the codebook
//     stays fp32, so two builds of the same rows give the same bytes.
#include <algorithm>
#include <cmath>
#include <vector>

#include <cub/cub.cuh>

#include "common.cuh"
#include "ivf_aq.h"

namespace b200 {

// Neither constant is tuned: the benchmark (tools/bench_aux.py aq) reports the sample loss after every iteration.
constexpr int kAqSweeps = 4;   // coordinate-descent sweeps of the encoder at most
constexpr int kAqIters = 5;    // encode + codebook-update iterations after the k-means codebooks
constexpr int kAqWarps = 4;    // rows (warps) per encoder block
constexpr int kAqBatch = 8;    // members staged at a time by the codebook update

// per-warp shared memory of the encoder: x and a = x - c_l (fp32 [d] each), <r_k, x_k> per sub-space (fp32 [m]), codes [m]
__host__ __device__ static inline size_t aq_warp_smem(int d, int m) { return (size_t)8 * d + 4 * (size_t)m + round_up(m, 16); }

size_t aq_encoder_smem(int d, int m) {
    const size_t b = kAqWarps * aq_warp_smem(d, m);
    return b <= (size_t)200 * 1024 ? b : 0;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// lexicographic (value, index) arg-min across the warp: every lane ends with the winner
__device__ __forceinline__ void warp_argmin(float &v, uint32_t &i, float &aux) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, o);
        const uint32_t oi = __shfl_xor_sync(0xffffffffu, i, o);
        const float oa = __shfl_xor_sync(0xffffffffu, aux, o);
        if (ov < v || (ov == v && oi < i)) {
            v = ov;
            i = oi;
            aux = oa;
        }
    }
}

// Coordinate descent of one row (the calling warp).  xs = x, as = x - c_l, code = the start codes; on return code holds the
// row's anisotropic codes.  pd is scratch [m].
__device__ void aq_encode_row(const float *xs, const float *as, float *pd, uint8_t *code, const float *__restrict__ pq, int d, int m,
                              int dsub, int ncw, float eta) {
    const int lane = threadIdx.x & 31;
    float nx = 0.f;
    for (int t = lane; t < d; t += 32) nx = fmaf(xs[t], xs[t], nx);
    nx = warp_sum(nx);
    const float w = nx > 0.f ? (eta - 1.f) / nx : 0.f;
    for (int k = lane; k < m; k += 32) {   // <r_k, x_k> of the start codes
        const float *e = pq + ((size_t)k * ncw + code[k]) * dsub;
        float dd = 0.f;
        for (int t = 0; t < dsub; t++) dd = fmaf(as[k * dsub + t] - e[t], xs[k * dsub + t], dd);
        pd[k] = dd;
    }
    __syncwarp();
    for (int sweep = 0; sweep < kAqSweeps; sweep++) {
        bool changed = false;
        for (int j = 0; j < m; j++) {
            float s = 0.f;
            for (int k = lane; k < m; k += 32)
                if (k != j) s += pd[k];
            s = warp_sum(s);
            const float *cb = pq + (size_t)j * ncw * dsub;
            const float *aj = as + j * dsub, *xj = xs + j * dsub;
            const uint32_t cur = code[j];
            float best = FLT_MAX, best_dd = 0.f, cur_l = 0.f;
            uint32_t bi = 0xffffffffu;
            for (int e = lane; e < ncw; e += 32) {
                const float *ce = cb + (size_t)e * dsub;
                float q = 0.f, dd = 0.f;
                for (int t = 0; t < dsub; t++) {
                    const float u = aj[t] - ce[t];
                    q = fmaf(u, u, q);
                    dd = fmaf(u, xj[t], dd);
                }
                const float pe = s + dd;
                const float l = fmaf(w, pe * pe, q);
                if (l < best) {   // ascending e inside a lane: ties keep the smaller index
                    best = l;
                    bi = (uint32_t)e;
                    best_dd = dd;
                }
                if ((uint32_t)e == cur) cur_l = l;
            }
            cur_l = __shfl_sync(0xffffffffu, cur_l, cur & 31);
            warp_argmin(best, bi, best_dd);
            if (best < cur_l && bi != cur) {
                changed = true;
                __syncwarp();
                if (lane == 0) {
                    code[j] = (uint8_t)bi;
                    pd[j] = best_dd;
                }
                __syncwarp();
            }
        }
        if (!changed) break;
    }
}

// one row into the warp's shared memory: xs = x, as = x - c_l (the residual the nearest-codeword search of scatter_rows_kernel sees)
__device__ __forceinline__ void aq_load_row(const float *x, const float *c, int d, float *xs, float *as) {
    for (int t = threadIdx.x & 31; t < d; t += 32) {
        xs[t] = x[t];
        as[t] = x[t] - c[t];
    }
}

struct AqSmem {
    float *xs, *as, *pd;
    uint8_t *code;
};
__device__ __forceinline__ AqSmem aq_smem(int d, int m) {
    extern __shared__ __align__(16) unsigned char aq_sm[];
    unsigned char *base = aq_sm + (size_t)(threadIdx.x >> 5) * aq_warp_smem(d, m);
    AqSmem r;
    r.xs = reinterpret_cast<float *>(base);
    r.as = r.xs + d;
    r.pd = r.as + d;
    r.code = reinterpret_cast<uint8_t *>(r.pd + m);
    return r;
}

// Added rows: one warp per row of the list-sorted chunk, after scatter_rows_kernel wrote its nearest-codeword codes into the
// row's pool slot; the anisotropic codes replace them (8-bit: a byte per code; 4-bit: code j in byte j / 2, even j low).
__global__ void __launch_bounds__(kAqWarps * 32) aq_encode_slots_kernel(const ScatterParams p, float eta) {
    const int lane = threadIdx.x & 31;
    const AqSmem sm = aq_smem(p.d, p.m);
    const int ncw = p.pq_bits == 4 ? 16 : 256;
    const int64_t nwarps = (int64_t)gridDim.x * kAqWarps;
    for (int64_t i = (int64_t)blockIdx.x * kAqWarps + (threadIdx.x >> 5); i < p.n; i += nwarps) {
        const uint32_t l = p.sorted_list[i], r = p.sorted_row[i];
        const uint32_t pos = p.list_len[l] + ((uint32_t)i - p.seg_start[l]);
        uint8_t *dst = p.codes + (size_t)pool_row_of(p, l, pos) * p.code_bytes;
        aq_load_row(p.rows + (int64_t)r * p.stride, p.centroids + (size_t)l * p.d, p.d, sm.xs, sm.as);
        for (int j = lane; j < p.m; j += 32) sm.code[j] = p.pq_bits == 4 ? (dst[j >> 1] >> (4 * (j & 1))) & 15 : dst[j];
        __syncwarp();
        aq_encode_row(sm.xs, sm.as, sm.pd, sm.code, p.pq, p.d, p.m, p.dsub, ncw, eta);
        __syncwarp();
        if (p.pq_bits == 4) {
            for (int b = lane; 2 * b < p.m; b += 32)
                dst[b] = (uint8_t)(sm.code[2 * b] | (2 * b + 1 < p.m ? sm.code[2 * b + 1] << 4 : 0));
        } else {
            for (int j = lane; j < p.m; j += 32) dst[j] = sm.code[j];
        }
        __syncwarp();
    }
}

// Training sample: one warp per row; the start codes are the nearest codewords (the arithmetic of scatter_rows_kernel), the
// result goes to codes [n][m], one byte per code.
__global__ void __launch_bounds__(kAqWarps * 32) aq_encode_sample_kernel(const AqTrain t, float eta, uint8_t *codes) {
    const int lane = threadIdx.x & 31;
    const AqSmem sm = aq_smem(t.d, t.m);
    const int64_t nwarps = (int64_t)gridDim.x * kAqWarps;
    for (int64_t i = (int64_t)blockIdx.x * kAqWarps + (threadIdx.x >> 5); i < t.n; i += nwarps) {
        aq_load_row(t.x + i * t.d, t.centroids + (size_t)t.list[i] * t.d, t.d, sm.xs, sm.as);
        __syncwarp();
        for (int j = 0; j < t.m; j++) {
            const float *cb = t.pq + (size_t)j * t.ncw * t.dsub;
            float bd = FLT_MAX, unused = 0.f;
            uint32_t best = 0xffffffffu;
            for (int e = lane; e < t.ncw; e += 32) {
                float s = 0.f;
                for (int q = 0; q < t.dsub; q++) {
                    const float u = sm.as[j * t.dsub + q] - cb[e * t.dsub + q];
                    s = fmaf(u, u, s);
                }
                if (s < bd) {
                    bd = s;
                    best = (uint32_t)e;
                }
            }
            warp_argmin(bd, best, unused);
            if (lane == 0) sm.code[j] = (uint8_t)best;
        }
        __syncwarp();
        aq_encode_row(sm.xs, sm.as, sm.pd, sm.code, t.pq, t.d, t.m, t.dsub, t.ncw, eta);
        __syncwarp();
        for (int j = lane; j < t.m; j += 32) codes[i * t.m + j] = sm.code[j];
        __syncwarp();
    }
}

// fp64 state of every sample row from scratch: p_i = <r_i, x_i>, w_i and the loss ||r_i||^2 + w_i p_i^2 (one warp per row,
// lane-strided sums reduced in a fixed tree)
__global__ void __launch_bounds__(256) aq_state_kernel(const AqTrain t, double eta, const uint8_t *codes, double *p, double *w, double *loss) {
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < t.n; i += nwarps) {
        const float *x = t.x + i * t.d, *c = t.centroids + (size_t)t.list[i] * t.d;
        double rx = 0, rr = 0, xx = 0;
        for (int q = lane; q < t.d; q += 32) {
            const int j = q / t.dsub;
            const double xv = x[q];
            const double r = xv - (double)c[q] - (double)t.pq[((size_t)j * t.ncw + codes[i * t.m + j]) * t.dsub + (q - j * t.dsub)];
            rx += r * xv;
            rr += r * r;
            xx += xv * xv;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            rx += __shfl_xor_sync(0xffffffffu, rx, o);
            rr += __shfl_xor_sync(0xffffffffu, rr, o);
            xx += __shfl_xor_sync(0xffffffffu, xx, o);
        }
        if (lane == 0) {
            const double wi = xx > 0 ? (eta - 1.0) / xx : 0.0;
            p[i] = rx;
            w[i] = wi;
            loss[i] = rr + wi * rx * rx;
        }
    }
}

// sort keys of sub-space j: the code of every row, and the members per codeword
__global__ void aq_column_kernel(const uint8_t *codes, int64_t n, int m, int j, uint8_t *key, uint32_t *row, uint32_t *cnt) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t k = codes[i * m + j];
    key[i] = k;
    row[i] = (uint32_t)i;
    atomicAdd(&cnt[k], 1u);
}

// One block per codeword e of sub-space j: accumulate its normal equations over its members in row order (fp64; every matrix
// and right-hand-side entry owned by one thread), solve by Cholesky and store e in fp32.  old_cb keeps sub-space j's codebook
// before the update (the members' current residuals).
__global__ void __launch_bounds__(256) aq_update_kernel(const AqTrain t, int j, const uint32_t *member, const uint32_t *cnt,
                                                        const double *p, const double *w, const float *old_cb) {
    __shared__ double A[kAqMaxDsub][kAqMaxDsub + 1];
    __shared__ double rhs[kAqMaxDsub];
    __shared__ double X[kAqBatch][kAqMaxDsub], Aa[kAqBatch][kAqMaxDsub];
    __shared__ double W[kAqBatch], Beta[kAqBatch];
    const int e = blockIdx.x, ds = t.dsub;
    const uint32_t count = cnt[e];
    if (count == 0) return;   // no members: the codeword keeps its value
    uint32_t start = 0;
    for (int k = 0; k < e; k++) start += cnt[k];
    const int nent = ds * ds + ds;   // entries: A row-major, then rhs
    for (int q = threadIdx.x; q < nent; q += blockDim.x) {
        if (q < ds * ds) A[q / ds][q % ds] = 0.0;
        else rhs[q - ds * ds] = 0.0;
    }
    const float *eo = old_cb + (size_t)e * ds;
    for (uint32_t b0 = 0; b0 < count; b0 += kAqBatch) {
        const int nb = count - b0 < (uint32_t)kAqBatch ? (int)(count - b0) : kAqBatch;
        __syncthreads();
        for (int q = threadIdx.x; q < nb * ds; q += blockDim.x) {
            const int mb = q / ds, tt = q % ds;
            const uint32_t i = member[start + b0 + mb];
            const int col = j * ds + tt;
            const double xv = t.x[(size_t)i * t.d + col];
            X[mb][tt] = xv;
            Aa[mb][tt] = xv - (double)t.centroids[(size_t)t.list[i] * t.d + col];
        }
        __syncthreads();
        if (threadIdx.x < nb) {
            const int mb = threadIdx.x;
            const uint32_t i = member[start + b0 + mb];
            double ax = 0, rx = 0;
            for (int tt = 0; tt < ds; tt++) {
                ax += Aa[mb][tt] * X[mb][tt];
                rx += (Aa[mb][tt] - (double)eo[tt]) * X[mb][tt];
            }
            W[mb] = w[i];
            Beta[mb] = w[i] * (ax + (p[i] - rx));
        }
        __syncthreads();
        for (int q = threadIdx.x; q < nent; q += blockDim.x) {
            if (q < ds * ds) {
                const int a = q / ds, b = q % ds;
                double acc = A[a][b];
                for (int mb = 0; mb < nb; mb++) acc += W[mb] * (X[mb][a] * X[mb][b]);
                A[a][b] = acc;
            } else {
                const int a = q - ds * ds;
                double acc = rhs[a];
                for (int mb = 0; mb < nb; mb++) acc += Aa[mb][a] + Beta[mb] * X[mb][a];
                rhs[a] = acc;
            }
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        // Cholesky A = L L^T in the lower triangle, then L y = rhs and L^T e = y
        for (int a = 0; a < ds; a++) A[a][a] += (double)count;
        for (int a = 0; a < ds; a++) {
            for (int b = 0; b <= a; b++) {
                double v = A[a][b];
                for (int k = 0; k < b; k++) v -= A[a][k] * A[b][k];
                A[a][b] = a == b ? sqrt(v) : v / A[b][b];
            }
        }
        for (int a = 0; a < ds; a++) {
            double v = rhs[a];
            for (int k = 0; k < a; k++) v -= A[a][k] * rhs[k];
            rhs[a] = v / A[a][a];
        }
        for (int a = ds - 1; a >= 0; a--) {
            double v = rhs[a];
            for (int k = a + 1; k < ds; k++) v -= A[k][a] * rhs[k];
            rhs[a] = v / A[a][a];
        }
        float *dst = t.pq + ((size_t)j * t.ncw + e) * ds;
        for (int a = 0; a < ds; a++) dst[a] = (float)rhs[a];
    }
}

// p_i after sub-space j's update: the residual block moves from a_j - e_old to a_j - e_new, so p_i gains <e_old - e_new, x_ij>
__global__ void aq_refresh_kernel(const AqTrain t, int j, const uint8_t *codes, const float *old_cb, double *p) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= t.n) return;
    const int c = codes[i * t.m + j];
    const float *eo = old_cb + (size_t)c * t.dsub, *en = t.pq + ((size_t)j * t.ncw + c) * t.dsub;
    const float *x = t.x + i * t.d + j * t.dsub;
    double dp = 0;
    for (int q = 0; q < t.dsub; q++) dp += ((double)eo[q] - (double)en[q]) * (double)x[q];
    p[i] += dp;
}

static int aq_grid(int64_t rows) { return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(rows, kAqWarps), 132 * 16)); }

int aq_encode_chunk(const ScatterParams &p, double eta, cudaStream_t s) {
    const size_t smem = aq_encoder_smem(p.d, p.m);
    if (!smem) return fail(B200_ERR_UNSUPPORTED, "aq_threshold: a row of d = " + std::to_string(p.d) + " does not fit the encoder's shared memory");
    B200_CUDA_OK(cudaFuncSetAttribute(aq_encode_slots_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    aq_encode_slots_kernel<<<aq_grid(p.n), kAqWarps * 32, smem, s>>>(p, (float)eta);
    g_launches++;
    B200_CUDA_OK(cudaGetLastError());
    return B200_OK;
}

// mean of the per-row losses, summed on the host in row order
static int aq_mean_loss(const double *d_loss, int64_t n, std::vector<double> &h, double *out, cudaStream_t s) {
    h.resize(n);
    B200_CUDA_OK(cudaMemcpyAsync(h.data(), d_loss, (size_t)n * 8, cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    double sum = 0;
    for (int64_t i = 0; i < n; i++) sum += h[i];
    *out = n ? sum / (double)n : 0.0;
    return B200_OK;
}

int aq_train_codebooks(const AqTrain &t, std::vector<double> *loss, cudaStream_t s) {
    const size_t smem = aq_encoder_smem(t.d, t.m);
    if (!smem) return fail(B200_ERR_UNSUPPORTED, "aq_threshold: a row of d = " + std::to_string(t.d) + " does not fit the encoder's shared memory");
    B200_CUDA_OK(cudaFuncSetAttribute(aq_encode_sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t n = t.n;
    const int bits = t.ncw == 16 ? 4 : 8;
    DevMem codes_b, key_b, key_s_b, row_b, member_b, cnt_b, p_b, w_b, dl_b, old_cb_b, tmp;
    size_t tmp_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, key_b.as<uint8_t>(), key_s_b.as<uint8_t>(), row_b.as<uint32_t>(), member_b.as<uint32_t>(), (int)n, 0,
                                    bits, s);
    B200_TRY(codes_b.alloc((size_t)n * t.m));
    B200_TRY(key_b.alloc((size_t)n));
    B200_TRY(key_s_b.alloc((size_t)n));
    B200_TRY(row_b.alloc((size_t)n * 4));
    B200_TRY(member_b.alloc((size_t)n * 4));
    B200_TRY(cnt_b.alloc((size_t)t.ncw * 4));
    B200_TRY(p_b.alloc((size_t)n * 8));
    B200_TRY(w_b.alloc((size_t)n * 8));
    B200_TRY(dl_b.alloc((size_t)n * 8));
    B200_TRY(old_cb_b.alloc((size_t)t.ncw * t.dsub * 4));
    B200_TRY(tmp.alloc(tmp_bytes + 256));
    uint8_t *codes = codes_b.as<uint8_t>(), *key = key_b.as<uint8_t>(), *key_s = key_s_b.as<uint8_t>();
    uint32_t *row = row_b.as<uint32_t>(), *member = member_b.as<uint32_t>(), *cnt = cnt_b.as<uint32_t>();
    double *p = p_b.as<double>(), *w = w_b.as<double>(), *dl = dl_b.as<double>();
    float *old_cb = old_cb_b.as<float>();
    std::vector<double> h;
    const int rows_grid = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n * 32, 256), 132 * 32));
    for (int it = 0; it < kAqIters; it++) {
        aq_encode_sample_kernel<<<aq_grid(n), kAqWarps * 32, smem, s>>>(t, (float)t.eta, codes);
        aq_state_kernel<<<rows_grid, 256, 0, s>>>(t, t.eta, codes, p, w, dl);
        g_launches += 2;
        double mean = 0;
        if (it == 0) {
            B200_CUDA_OK(cudaGetLastError());
            B200_TRY(aq_mean_loss(dl, n, h, &mean, s));
            loss->push_back(mean);
        }
        for (int j = 0; j < t.m; j++) {
            float *cbj = t.pq + (size_t)j * t.ncw * t.dsub;
            B200_CUDA_OK(cudaMemcpyAsync(old_cb, cbj, (size_t)t.ncw * t.dsub * 4, cudaMemcpyDeviceToDevice, s));
            B200_CUDA_OK(cudaMemsetAsync(cnt, 0, (size_t)t.ncw * 4, s));
            aq_column_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, s>>>(codes, n, t.m, j, key, row, cnt);
            B200_CUDA_OK(cub::DeviceRadixSort::SortPairs(tmp.p, tmp_bytes, key, key_s, row, member, (int)n, 0, bits, s));
            aq_update_kernel<<<t.ncw, 256, 0, s>>>(t, j, member, cnt, p, w, old_cb);
            aq_refresh_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, s>>>(t, j, codes, old_cb, p);
            g_launches += 4;
            B200_CUDA_OK(cudaGetLastError());
        }
        aq_state_kernel<<<rows_grid, 256, 0, s>>>(t, t.eta, codes, p, w, dl);
        g_launches++;
        B200_CUDA_OK(cudaGetLastError());
        B200_TRY(aq_mean_loss(dl, n, h, &mean, s));
        loss->push_back(mean);
    }
    B200_CUDA_OK(cudaStreamSynchronize(s));
    return B200_OK;
}

}  // namespace b200
