// ivf_opq.cu -- optimised product quantisation (OPQ; Ge et al., TPAMI 2014; Faiss OPQMatrix) for the PQ index types.
//
// An opq=1 index quantises x.R instead of x, for an orthonormal R [d][d] learned at train time by alternating the PQ
// codebooks of the rotated residuals with an orthogonal Procrustes step (ivf.cu, train_device_locked).  This file holds
// the kernels of both halves:
//   * the row rotation y = x.R (fp32 SIMT; one fmaf chain per element in column order, so a row's rotation does not depend
//     on the batch it comes in), used for the training sample, every added chunk and every query batch;
//   * the PQ encode / decode of the rotated sample and its per-row loss;
//   * the Procrustes step R = polar(Res^T Res^) in float64: M accumulated by a tiled float64 GEMM, a one-sided (Hestenes)
//     Jacobi SVD with round-robin pair ordering (one CTA per disjoint column pair, d / 2 pairs per round), U completed on
//     the null space of a rank-deficient M by Gram-Schmidt, R = U V^T.  No floating-point atomics anywhere: R is a function
//     of the codebooks and the sample.
#include <algorithm>
#include <cmath>
#include <vector>

#include "ivf_opq.h"

namespace b200 {

// ------------------------------------------------------------------------------------
// row rotation
// ------------------------------------------------------------------------------------
constexpr int kRotTile = 64, kRotK = 16;
// batches up to this many rows take the one-thread-per-output kernel (a handful of queries); larger ones the tiled one
constexpr int64_t kRotRowsKernelMax = 16;

// 64 rows x 64 columns per CTA, K chunks of 16, 4 x 4 outputs per thread; the chunks and the columns inside a chunk are
// added in order, each output by one fmaf chain (columns past d load 0: fmaf(0, 0, acc) = acc, as acc is never -0)
__global__ void __launch_bounds__(256) opq_rotate_kernel(const float *__restrict__ x, int64_t ldx, int64_t n, int d, const float *__restrict__ R,
                                                         float *__restrict__ y, int64_t ldy) {
    __shared__ __align__(16) float xs[kRotK][kRotTile + 4];
    __shared__ __align__(16) float rs[kRotK][kRotTile + 4];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int c0 = blockIdx.x * kRotTile;
    for (int64_t r0 = (int64_t)blockIdx.y * kRotTile; r0 < n; r0 += (int64_t)gridDim.y * kRotTile) {
        float acc[4][4];
#pragma unroll
        for (int a = 0; a < 4; a++)
#pragma unroll
            for (int b = 0; b < 4; b++) acc[a][b] = 0.f;
        for (int k0 = 0; k0 < d; k0 += kRotK) {
            for (int i = threadIdx.x; i < kRotTile * kRotK; i += 256) {
                const int r = i / kRotK, kk = i % kRotK;
                xs[kk][r] = (r0 + r < n && k0 + kk < d) ? x[(r0 + r) * ldx + k0 + kk] : 0.f;
                const int kr = i / kRotTile, c = i % kRotTile;
                rs[kr][c] = (k0 + kr < d && c0 + c < d) ? R[(int64_t)(k0 + kr) * d + c0 + c] : 0.f;
            }
            __syncthreads();
#pragma unroll
            for (int kk = 0; kk < kRotK; kk++) {
                const float4 xv = *reinterpret_cast<const float4 *>(&xs[kk][ty * 4]);
                const float4 rv = *reinterpret_cast<const float4 *>(&rs[kk][tx * 4]);
                const float xa[4] = {xv.x, xv.y, xv.z, xv.w}, rb[4] = {rv.x, rv.y, rv.z, rv.w};
#pragma unroll
                for (int a = 0; a < 4; a++)
#pragma unroll
                    for (int b = 0; b < 4; b++) acc[a][b] = fmaf(xa[a], rb[b], acc[a][b]);
            }
            __syncthreads();
        }
#pragma unroll
        for (int a = 0; a < 4; a++) {
            const int64_t r = r0 + ty * 4 + a;
#pragma unroll
            for (int b = 0; b < 4; b++) {
                const int c = c0 + tx * 4 + b;
                if (r < n && c < ldy) y[r * ldy + c] = acc[a][b];
            }
        }
    }
}

// small batches: one thread per output element, the same fmaf chain over i = 0 .. d - 1
__global__ void __launch_bounds__(128) opq_rotate_rows_kernel(const float *__restrict__ x, int64_t ldx, int d, const float *__restrict__ R,
                                                              float *__restrict__ y, int64_t ldy) {
    const int64_t r = blockIdx.y;
    const int j = blockIdx.x * 128 + threadIdx.x;
    if (j >= ldy) return;
    float acc = 0.f;
    if (j < d) {
        const float *xr = x + r * ldx;
#pragma unroll 8
        for (int i = 0; i < d; i++) acc = fmaf(__ldg(xr + i), __ldg(R + (int64_t)i * d + j), acc);
    }
    y[r * ldy + j] = acc;
}

cudaError_t launch_opq_rotate(const float *x, int64_t ldx, int64_t n, int d, const float *R, float *y, int64_t ldy, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    if (n <= kRotRowsKernelMax) {
        opq_rotate_rows_kernel<<<dim3((unsigned)ceil_div(ldy, 128), (unsigned)n), 128, 0, s>>>(x, ldx, d, R, y, ldy);
    } else {
        const int64_t row_tiles = std::min<int64_t>(ceil_div(n, kRotTile), 65535);
        opq_rotate_kernel<<<dim3((unsigned)ceil_div(ldy, kRotTile), (unsigned)row_tiles), 256, 0, s>>>(x, ldx, n, d, R, y, ldy);
    }
    g_launches++;
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------
// PQ encode / decode of the training sample and its loss
// ------------------------------------------------------------------------------------
// one thread per (sub-quantiser, row), sub-quantiser-major: the 32 lanes of a warp read the same codebook
__global__ void __launch_bounds__(256) opq_encode_kernel(const float *__restrict__ x, int64_t n, int d, int m, int dsub, int ncw,
                                                         const float *__restrict__ pq, float *__restrict__ xhat) {
    const int64_t total = n * m;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int j = (int)(i / n);
        const int64_t r = i - (int64_t)j * n;
        const float *xs = x + r * d + (int64_t)j * dsub;
        const float *cb = pq + (int64_t)j * ncw * dsub;
        float best = FLT_MAX;
        int bi = 0;
        for (int e = 0; e < ncw; e++) {
            float s = 0.f;
            for (int t = 0; t < dsub; t++) {
                const float df = xs[t] - cb[(int64_t)e * dsub + t];
                s = fmaf(df, df, s);
            }
            if (s < best) {   // ascending codes: ties keep the smaller one
                best = s;
                bi = e;
            }
        }
        for (int t = 0; t < dsub; t++) xhat[r * d + (int64_t)j * dsub + t] = cb[(int64_t)bi * dsub + t];
    }
}

// err[r] = ||x[r] - xhat[r]||^2 in float64: lane-strided sums, then a fixed xor butterfly; one warp per row
__global__ void __launch_bounds__(256) opq_row_err_kernel(const float *__restrict__ x, const float *__restrict__ xhat, int64_t n, int d,
                                                          double *__restrict__ err) {
    const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int lane = threadIdx.x & 31;
    for (int64_t r = warp_global; r < n; r += nwarps) {
        double s = 0;
        for (int i = lane; i < d; i += 32) {
            const double df = (double)x[r * d + i] - (double)xhat[r * d + i];
            s = fma(df, df, s);
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) err[r] = s;
    }
}

static int grid_of(int64_t work, int threads = 256) { return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(work, threads), 132 * 32)); }

cudaError_t launch_opq_encode(const float *x, int64_t n, int d, int m, int dsub, int ncw, const float *pq, float *xhat, double *err, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    opq_encode_kernel<<<grid_of(n * m), 256, 0, s>>>(x, n, d, m, dsub, ncw, pq, xhat);
    opq_row_err_kernel<<<grid_of(n * 32), 256, 0, s>>>(x, xhat, n, d, err);
    g_launches += 2;
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------
// Procrustes step
// ------------------------------------------------------------------------------------
// C[i][j] = sum_k A[k][i] B[k][j] (i < n1, j < n2) in float64, k in order: 64 x 64 outputs per CTA, 4 x 4 per thread
template <typename T>
__global__ void __launch_bounds__(256) atb_f64_kernel(const T *__restrict__ A, int64_t lda, const T *__restrict__ B, int64_t ldb, int64_t K, int n1, int n2,
                                                      double *__restrict__ C) {
    __shared__ double as[16][64], bs[16][64];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int i0 = blockIdx.y * 64, j0 = blockIdx.x * 64;
    double acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; a++)
#pragma unroll
        for (int b = 0; b < 4; b++) acc[a][b] = 0.0;
    for (int64_t k0 = 0; k0 < K; k0 += 16) {
        for (int t = threadIdx.x; t < 16 * 64; t += 256) {
            const int kk = t / 64, c = t % 64;
            const int64_t k = k0 + kk;
            as[kk][c] = (k < K && i0 + c < n1) ? (double)A[k * lda + i0 + c] : 0.0;
            bs[kk][c] = (k < K && j0 + c < n2) ? (double)B[k * ldb + j0 + c] : 0.0;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < 16; kk++) {
            double av[4], bv[4];
#pragma unroll
            for (int a = 0; a < 4; a++) av[a] = as[kk][ty * 4 + a];
#pragma unroll
            for (int b = 0; b < 4; b++) bv[b] = bs[kk][tx * 4 + b];
#pragma unroll
            for (int a = 0; a < 4; a++)
#pragma unroll
                for (int b = 0; b < 4; b++) acc[a][b] = fma(av[a], bv[b], acc[a][b]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int a = 0; a < 4; a++)
#pragma unroll
        for (int b = 0; b < 4; b++) {
            const int i = i0 + ty * 4 + a, j = j0 + tx * 4 + b;
            if (i < n1 && j < n2) C[(int64_t)i * n2 + j] = acc[a][b];
        }
}

// sum of v over the CTA (blockDim.x a multiple of 32, at most 1024): warp butterflies, then the warp sums in warp order;
// every thread gets the total
__device__ __forceinline__ double block_sum_f64(double v, double *red /*[32]*/) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[w] = v;
    __syncthreads();
    double t = 0;
    for (int i = 0; i < nw; i++) t += red[i];
    return t;
}

// relative orthogonality |a_p . a_q| <= kJacobiTol ||a_p|| ||a_q|| at which a pair is left alone; sweeps are capped
constexpr double kJacobiTol = 1e-12;
constexpr int kJacobiMaxSweeps = 40;

// One round of the round-robin ordering over np (even) players, player np - 1 fixed: pair 0 = (np - 1, round), pair i =
// ((round + i) mod (np - 1), (round - i) mod (np - 1)).  Each CTA orthogonalises its column pair of A (column-major [d][d])
// and applies the same rotation to V.  A player >= d (odd d) sits the round out.
__global__ void __launch_bounds__(256) jacobi_round_kernel(double *__restrict__ A, double *__restrict__ V, int d, int np, int round, int *__restrict__ rotated) {
    __shared__ double red[32];
    const int i = blockIdx.x;
    int p = i == 0 ? np - 1 : (round + i) % (np - 1);
    int q = i == 0 ? round : (round - i + (np - 1)) % (np - 1);
    if (p > q) {
        const int t = p;
        p = q;
        q = t;
    }
    if (q >= d) return;
    double *ap = A + (int64_t)p * d, *aq = A + (int64_t)q * d;
    double sa = 0, sb = 0, sg = 0;
    for (int t = threadIdx.x; t < d; t += blockDim.x) {
        const double x = ap[t], y = aq[t];
        sa = fma(x, x, sa);
        sb = fma(y, y, sb);
        sg = fma(x, y, sg);
    }
    const double alpha = block_sum_f64(sa, red);
    const double beta = block_sum_f64(sb, red);
    const double gamma = block_sum_f64(sg, red);
    if (!(alpha > 0 && beta > 0) || !(fabs(gamma) > kJacobiTol * sqrt(alpha) * sqrt(beta))) return;
    const double zeta = (beta - alpha) / (2 * gamma);
    const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + hypot(1.0, zeta));
    const double c = 1 / sqrt(1 + t * t), s = c * t;
    double *vp = V + (int64_t)p * d, *vq = V + (int64_t)q * d;
    for (int e = threadIdx.x; e < d; e += blockDim.x) {
        const double x = ap[e], y = aq[e];
        ap[e] = c * x - s * y;
        aq[e] = s * x + c * y;
        const double u = vp[e], w = vq[e];
        vp[e] = c * u - s * w;
        vq[e] = s * u + c * w;
    }
    if (threadIdx.x == 0) *rotated = 1;
}

__global__ void identity_f64_kernel(double *V, int d) {
    const int64_t total = (int64_t)d * d;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
        V[i] = (i / d == i % d) ? 1.0 : 0.0;
}

// columns whose norm is at most this share of the largest are the null space of M: Gram-Schmidt replaces them
constexpr double kNullRel = 1e-10;

// the smallest v over the CTA and its index (ties: the smaller index); every thread gets both.  Order-free, so deterministic.
__device__ __forceinline__ void block_argmin_f64(double v, int i, double *rv /*[32]*/, int *ri /*[32]*/, double *out_v, int *out_i) {
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, i, o);
        if (ov < v || (ov == v && oi < i)) {
            v = ov;
            i = oi;
        }
    }
    const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) {
        rv[w] = v;
        ri[w] = i;
    }
    __syncthreads();
    double bv = rv[0];
    int bi = ri[0];
    for (int t = 1; t < nw; t++)
        if (rv[t] < bv || (rv[t] == bv && ri[t] < bi)) {
            bv = rv[t];
            bi = ri[t];
        }
    *out_v = bv;
    *out_i = bi;
}

// A (column-major, the converged A V = U S) -> U: columns normalised; a column of a (numerically) zero singular value is
// replaced by the unit vector e_c with the largest component outside the columns accepted so far, orthogonalised against
// them by two classical Gram-Schmidt passes.  With the accepted columns orthonormal, that component's square is
// 1 - w[c], w[c] = sum over accepted t of U[c][t]^2, and its largest value is at least (null columns left) / d > 0, so
// every null column gets a direction and U stays orthonormal whatever the orientation of the null space.  One CTA of 1024
// threads; w, v, coef: [d] float64 scratch.
__global__ void __launch_bounds__(1024) polar_complete_kernel(double *__restrict__ A, int d, double *__restrict__ w, double *__restrict__ v,
                                                              double *__restrict__ coef) {
    __shared__ int ok[kOpqMaxDim];
    __shared__ double red[32];
    __shared__ int redi[32];
    __shared__ double smax;
    for (int j = threadIdx.x; j < d; j += blockDim.x) {
        double s = 0;
        for (int i = 0; i < d; i++) s = fma(A[(int64_t)j * d + i], A[(int64_t)j * d + i], s);
        w[j] = sqrt(s);   // the column norms first
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double mx = 0;
        for (int j = 0; j < d; j++) mx = fmax(mx, w[j]);
        smax = mx;
    }
    __syncthreads();
    const double tol = smax * kNullRel;
    for (int j = threadIdx.x; j < d; j += blockDim.x) ok[j] = w[j] > tol && w[j] > 0;
    __syncthreads();
    for (int64_t e = threadIdx.x; e < (int64_t)d * d; e += blockDim.x)
        if (ok[e / d]) A[e] /= w[e / d];
    __syncthreads();
    for (int c = threadIdx.x; c < d; c += blockDim.x) {   // w[c]: the accepted columns' weight on axis c
        double s = 0;
        for (int t = 0; t < d; t++)
            if (ok[t]) s = fma(A[(int64_t)t * d + c], A[(int64_t)t * d + c], s);
        w[c] = s;
    }
    __syncthreads();
    for (int k = 0; k < d; k++) {
        if (ok[k]) continue;
        double bv = 0;
        int cand = 0;
        {
            double mv = DBL_MAX;
            int mi = d;
            for (int c = threadIdx.x; c < d; c += blockDim.x)
                if (w[c] < mv) {   // ascending c per thread: ties keep the smaller one
                    mv = w[c];
                    mi = c;
                }
            block_argmin_f64(mv, mi, red, redi, &bv, &cand);
        }
        for (int i = threadIdx.x; i < d; i += blockDim.x) v[i] = i == cand ? 1.0 : 0.0;
        __syncthreads();
        for (int pass = 0; pass < 2; pass++) {
            for (int t = threadIdx.x; t < d; t += blockDim.x) {
                double s = 0;
                if (ok[t])
                    for (int i = 0; i < d; i++) s = fma(A[(int64_t)t * d + i], v[i], s);
                coef[t] = s;
            }
            __syncthreads();
            for (int i = threadIdx.x; i < d; i += blockDim.x) {
                double s = v[i];
                for (int t = 0; t < d; t++)
                    if (ok[t]) s = fma(-coef[t], A[(int64_t)t * d + i], s);
                v[i] = s;
            }
            __syncthreads();
        }
        double part = 0;
        for (int i = threadIdx.x; i < d; i += blockDim.x) part = fma(v[i], v[i], part);
        const double inv = 1 / sqrt(block_sum_f64(part, red));
        for (int i = threadIdx.x; i < d; i += blockDim.x) {
            const double u = v[i] * inv;
            A[(int64_t)k * d + i] = u;
            w[i] = fma(u, u, w[i]);
        }
        __syncthreads();
        if (threadIdx.x == 0) ok[k] = 1;
        __syncthreads();
    }
}

__global__ void f64_to_f32_kernel(const double *a, int64_t n, float *out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = (float)a[i];
}

int opq_procrustes(const float *res, const float *xhat, int64_t n, int d, float *R, cudaStream_t s) {
    const size_t dd = (size_t)d * d;
    DevMem A_b, V_b, P_b, scratch_b, flag_b;
    B200_TRY(A_b.alloc(dd * 8));
    B200_TRY(V_b.alloc(dd * 8));
    B200_TRY(P_b.alloc(dd * 8));
    B200_TRY(scratch_b.alloc((size_t)3 * d * 8));
    B200_TRY(flag_b.alloc(4));
    double *A = A_b.as<double>(), *V = V_b.as<double>(), *P = P_b.as<double>(), *scratch = scratch_b.as<double>();
    int *flag = flag_b.as<int>();
    const dim3 tiles((unsigned)ceil_div(d, 64), (unsigned)ceil_div(d, 64));
    // A column-major = M^T row-major: A[j][i] = M[i][j] = sum_r res[r][i] xhat[r][j]
    atb_f64_kernel<float><<<tiles, 256, 0, s>>>(xhat, d, res, d, n, d, d, A);
    identity_f64_kernel<<<grid_of((int64_t)dd), 256, 0, s>>>(V, d);
    g_launches += 2;
    const int np = d + (d & 1);
    for (int sweep = 0; sweep < kJacobiMaxSweeps; sweep++) {
        int any = 0;
        B200_CUDA_OK(cudaMemsetAsync(flag, 0, 4, s));
        for (int r = 0; r < np - 1; r++) jacobi_round_kernel<<<(unsigned)(np / 2), 256, 0, s>>>(A, V, d, np, r, flag);
        g_launches += np - 1;
        B200_CUDA_OK(cudaGetLastError());
        B200_CUDA_OK(cudaMemcpyAsync(&any, flag, 4, cudaMemcpyDeviceToHost, s));
        B200_CUDA_OK(cudaStreamSynchronize(s));
        if (!any) break;
    }
    polar_complete_kernel<<<1, 1024, 0, s>>>(A, d, scratch, scratch + d, scratch + 2 * d);
    // R[i][j] = sum_k U[i][k] V[j][k]: U and V are column-major, so this is A^T B over k
    atb_f64_kernel<double><<<tiles, 256, 0, s>>>(A, d, V, d, d, d, d, P);
    f64_to_f32_kernel<<<grid_of((int64_t)dd), 256, 0, s>>>(P, (int64_t)dd, R);
    g_launches += 3;
    B200_CUDA_OK(cudaGetLastError());
    B200_CUDA_OK(cudaStreamSynchronize(s));
    return B200_OK;
}

// out[i] = max_j |P[i][j] - (i == j)|, one thread per row
__global__ void eye_row_err_kernel(const double *P, int d, double *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= d) return;
    double e = 0;
    for (int j = 0; j < d; j++) e = fmax(e, fabs(P[(int64_t)i * d + j] - (i == j ? 1.0 : 0.0)));
    out[i] = e;
}

int opq_orthonormal_error(const float *R, int d, double *max_err, cudaStream_t s) {
    DevMem P_b;
    B200_TRY(P_b.alloc(((size_t)d * d + d) * 8));
    double *P = P_b.as<double>();
    atb_f64_kernel<float><<<dim3((unsigned)ceil_div(d, 64), (unsigned)ceil_div(d, 64)), 256, 0, s>>>(R, d, R, d, d, d, d, P);
    eye_row_err_kernel<<<(unsigned)ceil_div(d, 128), 128, 0, s>>>(P, d, P + (size_t)d * d);
    g_launches += 2;
    std::vector<double> h(d);
    const cudaError_t e = cudaMemcpyAsync(h.data(), P + (size_t)d * d, (size_t)d * 8, cudaMemcpyDeviceToHost, s);
    const cudaError_t e2 = cudaStreamSynchronize(s);
    if (e != cudaSuccess || e2 != cudaSuccess) return fail(B200_ERR_CUDA, std::string("OPQ rotation check: ") + cudaGetErrorString(e != cudaSuccess ? e : e2));
    double m = 0;
    for (double v : h) m = std::max(m, v);   // NaN rows (none: R is checked finite first) would not raise it
    *max_err = m;
    return B200_OK;
}

}  // namespace b200
