// ivf_opq.h -- optimised product quantisation (opq=1 on IVFPQ / SCANN / HNSWPQ): the rotation R [d][d] fp32, row-major,
// y = x.R, that the inverted-file side of such an index lives in (ivf_opq.cu).
#pragma once
#include <vector>

#include "common.cuh"

namespace b200 {

// widest rows an OPQ index takes: R is d x d fp32, at most 64 MB
constexpr int kOpqMaxDim = 4096;

// y[r][j] = sum_i x[r][i] R[i][j] for r < n, j < d, and y[r][j] = 0 for d <= j < ldy.  Every element is one fmaf chain over
// i = 0 .. d - 1 in order, whatever n, the tile or the grid: a row's rotation depends on that row and d alone.
cudaError_t launch_opq_rotate(const float *x, int64_t ldx, int64_t n, int d, const float *R, float *y, int64_t ldy, cudaStream_t s);

// PQ encode + decode of rows x [n][d] with codebooks pq [m][ncw][dsub]: xhat[r] = the nearest codeword of every sub-vector
// (ties: the smaller code), err[r] = ||x[r] - xhat[r]||^2 (float64, fixed order)
cudaError_t launch_opq_encode(const float *x, int64_t n, int d, int m, int dsub, int ncw, const float *pq, float *xhat, double *err, cudaStream_t s);

// Orthogonal Procrustes step: R = polar(res^T xhat) = U V^T (float64 one-sided Jacobi SVD, U completed on the null space by
// Gram-Schmidt), written as fp32 [d][d].  res, xhat: [n][d] fp32.  No floating-point atomics: R depends on the inputs alone.
int opq_procrustes(const float *res, const float *xhat, int64_t n, int d, float *R, cudaStream_t s);

// max |R^T R - I| of a device R [d][d] fp32, in float64 (load validates a stored rotation against kOpqLoadTol)
int opq_orthonormal_error(const float *R, int d, double *max_err, cudaStream_t s);
constexpr double kOpqLoadTol = 1e-4;

}  // namespace b200
