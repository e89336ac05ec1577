// vec.cuh -- O(N^2) / O(N) kernels: blocked triangular solves with one right-hand side,
// deterministic reductions, predictive mean / variance epilogues (see vec.cu)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
// y = L^-1 r (r is destroyed, y receives the result; length Npad), L lower in F (row-major), Dinv = inverted diagonal tiles
cudaError_t trsv_lower_fwd(const double* F, int64_t ldf, const double* Dinv, double* r, double* y, int64_t Npad, cudaStream_t st, int64_t* launches);
// a = L^-T z (z is destroyed, a receives the result)
cudaError_t trsv_lower_bwd(const double* F, int64_t ldf, const double* DinvT, double* z, double* a, int64_t Npad, cudaStream_t st, int64_t* launches);
// out[0] = sum_i a[i]*b[i] (b may equal a); fixed-order tree, one CTA
cudaError_t dot_launch(const double* a, const double* b, int64_t n, double* out, cudaStream_t st, int64_t* launches);
cudaError_t sum_launch(const double* a, int64_t n, double* out, cudaStream_t st, int64_t* launches);
// mu[m] = sum_n Kst[m,n] alpha[n]
cudaError_t rowdot_launch(const double* Kst, int64_t ldk, const double* alpha, int64_t M, int64_t N, double* mu, cudaStream_t st, int64_t* launches);
// var[m] = kdiag[m] - sum_n Vt[m,n]^2
cudaError_t rowvar_launch(const double* Vt, int64_t ldk, const double* kdiag, int64_t M, int64_t N, double* var, cudaStream_t st, int64_t* launches);
// FP64 issue-rate microbenchmark: tflops[0] = DMMA.16x8x16, tflops[1] = DFMA (register operands)
cudaError_t fp64_peak_measure(cudaStream_t st, int64_t* launches, double* tflops);
// elementwise: op 0 out=a+s | 1 out=a/b | 2 out+=a | 3 out=(a-b)/c | 4 out=log(a) | 5 out=1/a | 6 out=a-b
cudaError_t ew_launch(int op, int64_t n, double* out, const double* a, const double* b, const double* c, double s, cudaStream_t st, int64_t* launches);
// mode 0: A[:, j] *= 1/sqrt(v[j]) (j < ncols) ; mode 1: A[r, :] *= 1/v[r] (r < nrows)
cudaError_t scale_launch(int mode, double* A, int64_t ld, int64_t nrows, int64_t ncols, const double* v, cudaStream_t st, int64_t* launches);
// FITC gradient helpers (see gpb200_fitc_grad_kernel)
cudaError_t rowdot2_launch(const double* A, const double* B, int64_t ld, int64_t nrows, int64_t ncols, double* q, cudaStream_t st, int64_t* launches);
cudaError_t fitc_g_launch(int64_t n, const double* alpha, const double* lam, const double* q, double* g, cudaStream_t st, int64_t* launches);
cudaError_t fitc_wfu_launch(double* P2, const double* P1, int64_t ld, int64_t nrows, int64_t ncols, const double* alpha,
                            const double* lam, const double* g, const double* beta, cudaStream_t st, int64_t* launches);
cudaError_t colscale_launch(double* A, int64_t ld, int64_t nrows, int64_t ncols, const double* v, cudaStream_t st, int64_t* launches);
cudaError_t symmetrize_launch(double* A, int64_t ld, int64_t n, cudaStream_t st, int64_t* launches);
cudaError_t fitc_wuu_launch(double* Wuu, const double* T, const double* Kinv, const double* Sinv, int64_t ld, int64_t n,
                            const double* beta, cudaStream_t st, int64_t* launches);
// single-launch variants (flag-synchronised CTAs); flags: int[Npad/128 + 1], flags[Npad/128] != 0 after the run = watchdog fired
cudaError_t trsv_lower_fwd_fused(const double* F, int64_t ldf, const double* Dinv, const double* r, double* y, int64_t Npad,
                                 int* flags, cudaStream_t st, int64_t* launches);
cudaError_t trsv_lower_bwd_fused(const double* F, int64_t ldf, const double* DinvT, const double* z, double* a, int64_t Npad,
                                 int* flags, cudaStream_t st, int64_t* launches);
// posterior sampling (gpb200_rand): SPD matrix with nugget + identity padding in the lower tiles; A[i, :] += v (any nrows)
cudaError_t spd_from_cov_launch(double* dst, int64_t ldd, const double* src, int64_t lds, int64_t n, int64_t npad, double nugget, cudaStream_t st, int64_t* launches);
cudaError_t add_rowvec_launch(double* A, int64_t ld, const double* v, int64_t nrows, int64_t ncols, cudaStream_t st, int64_t* launches);
// out[a * nv + b] = src[idx[a] * ld + idx[b]]   (principal sub-matrix on an index set; cross-validation folds)
cudaError_t gather_block_launch(double* out, const double* src, int64_t ld, const long long* idx, int64_t nv, cudaStream_t st, int64_t* launches);
