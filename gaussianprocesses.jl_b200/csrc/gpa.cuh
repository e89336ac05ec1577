// gpa.cuh -- O(N^2) kernels of the GPA path (non-Gaussian likelihoods, src/GPA.jl): triangular matrix-vector products
// over the lower triangle of the factor and the prefix / suffix scans that build Z' for the reverse-mode Cholesky (see gpa.cu)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
// f = L v   (L: lower triangle of F incl. the diagonal tiles; F's strict-upper tiles are never read)
cudaError_t gpa_trmv_launch(const double* F, int64_t ldf, const double* v, double* f, int64_t Npad, cudaStream_t st, int64_t* launches);
// u = L' g
cudaError_t gpa_trmv_t_launch(const double* F, int64_t ldf, const double* g, double* u, int64_t Npad, cudaStream_t st, int64_t* launches);
// row b of Z' (Z = lower part of M_s W, M_s[i,j] = u[max(i,j)] v[min(i,j)], W = L^-1) from row b of W': the strict-upper tiles of
// W' are read from G, the diagonal tile from DinvT; the strict-upper tiles of Z' go to F, the diagonal tiles (clean upper) to ZdT
cudaError_t gpa_scan_launch(const double* G, int64_t ld, const double* DinvT, const double* u, const double* v, double* F,
                            double* ZdT, int64_t Npad, cudaStream_t st, int64_t* launches);
