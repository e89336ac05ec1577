// gram.cuh -- launchers of the Gram / cross-Gram / gradient-trace kernels (see gram.cu)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "kprog.cuh"

// lower tiles of K_y (+ noise on the diagonal, identity in the padding) into G (row-major, ld = ldg)
cudaError_t gram_lower_launch(const KProg& P, const double* x, int64_t ldx, int d, int64_t N, int64_t Npad,
                              const double* noise_var, int64_t n_noise, double nugget, double* G, int64_t ldg,
                              cudaStream_t st, int64_t* launches, int own_tiles = 0, int nranks = 1, int rank = 0, int own_axis = 0, int bm_min = 0);
// Kst[m, n] = k(xs_m, x_n), M_pad x N_pad, zero padding
cudaError_t crossgram_launch(const KProg& P, const double* xs, int64_t ldxs, int64_t M, int64_t Mpad, const double* x,
                             int64_t ldx, int64_t N, int64_t Npad, int d, double* Kst, int64_t ldk, cudaStream_t st, int64_t* launches);
// Kss[m, m'] = k(xs_m, xs_m'), full M_pad x M_pad
cudaError_t gram_full_launch(const KProg& P, const double* xs, int64_t ldxs, int64_t M, int64_t Mpad, int d,
                             double* Kss, int64_t ldk, cudaStream_t st, int64_t* launches);
cudaError_t kdiag_launch(const KProg& P, const double* xs, int64_t ldxs, int64_t M, double* out, cudaStream_t st, int64_t* launches);
// number of accumulators per tile: n_theta + 1 (last = tr(A)); 3 for the specialised SEIso program (kprog_fast)
int trace_num_acc(const KProg& P, int d);
// part: [tiles][nacc] scratch; out: [nacc] = {dmll_kernel[0..n_theta), tr(A)}
cudaError_t trace_launch(const KProg& P, const double* x, int64_t ldx, int d, int64_t N, int64_t Npad,
                         const double* alpha, const double* Kinv, int64_t ldg, double* part, double* out,
                         cudaStream_t st, int64_t* launches, int bm_mod = 1, int bm_rem = 0, int bm_div = 1);
// FITC gradient pieces: rectangular weighted trace (tmp_out[p] = sum W .* dK/dθ_p over the rectangle; part must hold
// ceil(N1/128)*ceil(N2/128)*n_theta doubles) and g_i * dk(x_i,x_i)/dθ_p written as out[p*N + i]
cudaError_t trace_rect_launch(const KProg& P, const double* x1, int64_t ldx1, int64_t N1, const double* x2, int64_t ldx2,
                              int64_t N2, int d, const double* W, int64_t ldw, double* part, double* tmp_out,
                              cudaStream_t st, int64_t* launches);
cudaError_t kdiag_grad_launch(const KProg& P, const double* x, int64_t ldx, int64_t N, const double* gvec, double* out,
                              cudaStream_t st, int64_t* launches);
// D[i, k] = dk(x_i, x_k)/dtheta_j, full N_pad x N_pad (zero padding)  -- grad_slice! (src/kernels/kernels.jl:96-131).
// Rows row0 .. row0 + rows only (multiples of 128; rows < 0: to Npad), row row0 + r stored at D[r * ldd].
cudaError_t gram_grad_full_launch(const KProg& P, const double* x, int64_t ldx, int d, int64_t N, int64_t Npad, int j,
                                  double* D, int64_t ldd, cudaStream_t st, int64_t* launches, int64_t row0 = 0, int64_t rows = -1);
// D[m, n] = dk(x1_m, x2_n)/dtheta_j, N1_pad x N2_pad (multiples of 128), zero padding: the rectangular form for the sparse
// engine's cross-validation (dK_fu of a chunk of training rows against the inducing points)
cudaError_t crossgram_grad_launch(const KProg& P, const double* x1, int64_t ldx1, int64_t N1, int64_t N1pad, const double* x2,
                                  int64_t ldx2, int64_t N2, int64_t N2pad, int d, int j, double* D, int64_t ldd, cudaStream_t st,
                                  int64_t* launches);
// predictive gradients (M x d outputs, point-major):  dmu[m, :] = sum_i dk(xs_m, z_i)/dxs_m a_i ;  with W = W1 - W2 (either may
// be null; row m at W + m * ldw, n columns read): dvar[m, :] = 2c dk(xs_m, xs_m)/dxs_m - 2 sum_i dk(xs_m, z_i)/dxs_m W[m, i].
// Both null: dmu only.  Fixed-order sums.
cudaError_t crossgram_dx_launch(const KProg& P, const double* xs, int64_t ldxs, int64_t M, const double* z, int64_t ldz, int64_t n,
                                int d, const double* a, const double* W1, const double* W2, int64_t ldw, double c, double* dmu,
                                double* dvar, cudaStream_t st, int64_t* launches);
// inducing-point gradient (M x d output, point-major): out[j, :] = [out[j, :] if accumulate] + sum_i W(i, j) dk(u_j, z_i)/du_j
// over the n rows z_i with mask[i] != 0 (mask may be null), W(i, j) = W[i * ldw + j] (+ W[j * ldw + i] if sym).  Fixed-order sums.
cudaError_t inducing_dx_launch(const KProg& P, const double* u, int64_t ldu, int64_t M, const double* z, int64_t ldz, int64_t n,
                               int d, const double* W, int64_t ldw, int sym, const double* mask, double* out, int accumulate,
                               cudaStream_t st, int64_t* launches);
// training-input gradient (N x d output, point-major), over the lower triangle of A = a a' - G (a = alpha, 0 when null):
//   out[i, :] = sum_{j <= i} A_ij dk(x_i, x_j)/dx_i + sum_{l > i} A_li dk(x_i, x_l)/dx_i
// reading only the tile rows t with ((t / bm_div) % bm_mod) == bm_rem (all when bm_mod <= 1; the others count 0) and no row
// or column >= N.  fast: the single-SEIso specialisation (needs kprog_fast(P, d) and d <= 8).  Fixed-order sums.
cudaError_t inputs_dx_launch(const KProg& P, bool fast, const double* x, int64_t ldx, int d, int64_t N, const double* alpha,
                             const double* G, int64_t ldg, double* out, cudaStream_t st, int64_t* launches, int bm_mod,
                             int bm_rem, int bm_div);
// training-input gradient of the sparse mll over n rows x_i (output rows point-major, d wide):
//   out[row(i), :] (=, or += when accumulate) sum_{j < M} W[i * ldw + j] d1k(x_i, u_j) + 2 c_i d1k(x_i, x_i)
// (d1k: derivative in the first argument; c may be null: 0), over the rows with mask[i] != 0 (mask may be null; the others
// are neither read nor written), row(i) = map[i] (map may be null: i).  One warp per row; the single SEIso leaf with d <= 8
// takes a register specialisation.  Fixed-order sums.
cudaError_t rows_dx_launch(const KProg& P, const double* x, int64_t ldx, int64_t n, const double* u, int64_t ldu, int64_t M, int d,
                           const double* W, int64_t ldw, const double* c, const double* mask, const long long* map, double* out,
                           int accumulate, cudaStream_t st, int64_t* launches);
// F[j, i] = F[i, j] for every element of the strict-lower 128-tiles of the Npad x Npad matrix F (diagonal tiles untouched)
cudaError_t mirror_lower_tiles_launch(double* F, int64_t ld, int64_t Npad, cudaStream_t st, int64_t* launches);
