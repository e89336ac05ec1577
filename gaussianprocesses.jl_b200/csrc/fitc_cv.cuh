// fitc_cv.cuh -- row kernels of the sparse engine's cross-validation schedule (gpb200_fitc_get_inverse_diag,
// gpb200_fitc_cv_param, gpb200_fitc_cv_block; see fitc_cv.cu and the schedule in fitc_engine.cu).  Every reduction runs in a
// fixed order (one warp per row, lane-strided partial sums, xor butterfly), so repeated calls are bitwise equal.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "kprog.cuh"

// kind 0 (FITC kernel parameter): delta[i] = dk(x_i, x_i)/dtheta_j - 2 G[i,:].C[i,:]; kind 1 (SoR / DTC kernel parameter):
// delta = 0; kind 2 (noise variance): delta = 1.  Rows i < nrows; da[i] = delta[i] alpha[i] for i < nrows, 0 for
// nrows <= i < rows_pad.  G, C and x are read for kind 0 only.
cudaError_t fitc_cv_delta_launch(int kind, const KProg& P, const double* x, int64_t ldx, int j, const double* G, const double* C,
                                 int64_t ld, int64_t ncols, int64_t nrows, int64_t rows_pad, const double* alpha, double* delta,
                                 double* da, cudaStream_t st, int64_t* launches);
// fused output rows of one parameter (G may be NULL = 0):
//   zja[i] = delta_i alpha_i / lam_i + G_i.beta / lam_i + Ch_i.w
//   dg[i]  = delta_i / lam_i^2 + 2 G_i.Ch_i / lam_i - 2 delta_i K_i.Ch_i / lam_i^2 + P_i.Ch_i
cudaError_t fitc_cv_rows_launch(const double* G, const double* Ch, const double* K, const double* P, int64_t ld, int64_t nrows,
                                int64_t ncols, const double* lam, const double* delta, const double* alpha, const double* beta,
                                const double* w, double* zja, double* dg, cudaStream_t st, int64_t* launches);
// out[i] = 1/lam_i - q_i / lam_i^2
cudaError_t fitc_cv_invdiag_launch(int64_t n, const double* lam, const double* q, double* out, cudaStream_t st, int64_t* launches);
// E[i,m] += G[i,m] / lam_i - delta_i K[i,m] / lam_i^2   (G may be NULL = 0)
cudaError_t fitc_cv_eblock_launch(double* E, const double* G, const double* K, int64_t ld, int64_t nrows, int64_t ncols,
                                  const double* lam, const double* delta, cudaStream_t st, int64_t* launches);
// Q = H - R - R'   (n x n)
cudaError_t fitc_cv_qs_launch(double* Q, const double* H, const double* R, int64_t ld, int64_t n, cudaStream_t st, int64_t* launches);
// w = a - b - c
cudaError_t fitc_cv_wvec_launch(int64_t n, double* w, const double* a, const double* b, const double* c, cudaStream_t st,
                                int64_t* launches);
// rows r < nv: xout[r, :d] = x[idx[r], :d], lamout[r] = lam[idx[r]], delout[r] = delta[idx[r]] (delta may be NULL)
cudaError_t fitc_cv_gather_launch(int64_t nv, const long long* idx, const double* x, int64_t ldx, int d, double* xout,
                                  const double* lam, double* lamout, const double* delta, double* delout, cudaStream_t st,
                                  int64_t* launches);
// out[r, r] += 1/lam_r (which 0) or delta_r / lam_r^2 (which 1), r < nv
cudaError_t fitc_cv_diag_launch(double* out, int64_t ld, int64_t nv, int which, const double* lam, const double* delta,
                                cudaStream_t st, int64_t* launches);
