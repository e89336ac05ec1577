// gram_fast.cuh -- TMA-staged SEIso Gram build and fused gradient trace (see gram_fast.cu)
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

// host-prepared constants of k = s2 exp(-r / (2 l2)) = 2^(r c) * s2,  c = c_hi + c_lo = -log2(e) / (2 l2)
struct SeIsoFast {
    double c_hi, c_lo;
    double il2, s2;
    double tab[64];                 // s2 * 2^(j/64), correctly rounded
};
// false if (l2, s2) lie outside the range in which the exponent arithmetic of the fast exp is safe
bool seiso_fast_prepare(double l2, double s2, SeIsoFast* out);
// mapX: plain TMA descriptor of the inputs stored [N x dx] (dx even, <= 8, zero padded), box 128 x dx;
// mapXT: descriptor of the transposed copy [dx x N] (row pitch Npad), box dx x 128
cudaError_t gram_seiso_tma_launch(const CUtensorMap* mapX, const CUtensorMap* mapXT, int dx, const SeIsoFast& sf, int64_t N, int64_t Npad,
                                  const double* noise_var, int64_t n_noise, double nugget, double* G, int64_t ldg,
                                  cudaStream_t st, int64_t* launches, int own_tiles, int nranks, int rank, int own_axis);
// part: [tiles][3] scratch; out[0..2] = {dmll/dll, dmll/dlsigma, tr(A)} (same contract as trace_launch's fast path)
cudaError_t trace_seiso_tma_launch(const CUtensorMap* mapX, const CUtensorMap* mapXT, int dx, const SeIsoFast& sf, int64_t N, int64_t Npad,
                                   const double* alpha, const double* Kinv, int64_t ldg, double* part, double* out,
                                   cudaStream_t st, int64_t* launches, int bm_mod, int bm_rem, int bm_div);
