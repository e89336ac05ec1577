// fsa.cuh -- kernels of the Full Scale Approximation (src/sparse/full_scale_approximation.jl): the block-diagonal
// Lambda = blockdiag(Lambda_i) of thousands of dense blocks of different sizes, stored packed (block i padded to
// B_i = ceil(b_i/128)*128 rows, row-major, leading dimension B_i) and processed as lists of aligned 128 x 128 tiles, so
// that every block-diagonal operation is one launch over all blocks of a staging chunk (see fsa.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "kprog.cuh"

// One work item of the grouped tile GEMM: C = beta*C + alpha * A B' on one 128 x 128 tile,
// A: 128 x K and B: 128 x K row-major (lda, ldb, ldc even, pointers 16-byte aligned), K a multiple of 16.
// lower != 0 writes only the elements i >= j of the tile (diagonal tiles of a symmetric block).
struct FsaGemmItem {
    double* C;
    const double* A;
    const double* B;
    long long ldc, lda, ldb;
    int K;
    int lower;
    double alpha, beta;
};
cudaError_t fsa_gemm_launch(const FsaGemmItem* items, int n, cudaStream_t st, int64_t* launches);

// One tile of a block's Gram matrix: dst[i][j] = k(x_{row_i+i}, x_{row_j+j}) over padded rows, + diag_add on the real
// diagonal, identity on padding rows (mask 0); diag != 0: only i >= j is written.
struct FsaGramItem {
    double* dst;
    long long ld;
    long long row_i, row_j;
    int diag;
    int pad_;
};
cudaError_t fsa_gram_launch(const KProg& P, const double* xb, int d, const FsaGramItem* items, int n, const double* mask,
                            double diag_add, cudaStream_t st, int64_t* launches);

// Block-diagonal row products over the Np padded rows (row r lies in block rblk[r], which starts at padded row bstart[b],
// has B_b = bsize[b] rows and its packed matrix at offset boff[b]); r_l = r - bstart:
//   mode 0: y[r] = sum_{k <= r_l} M[r_l][k] v[bstart + k]      (lower triangle, y = M v)
//   mode 1: y[r] = sum_{k >= r_l} M[r_l][k] v[bstart + k]      (upper triangle)
//   mode 2: y[r] = sum_{k <= r_l} M[r_l][k]^2                  (squared row norms of the lower triangle)
// one warp per row, fixed summation order.
cudaError_t fsa_bdmv_launch(int mode, const double* packed, const int* rblk, const long long* bstart, const int* bsize,
                            const long long* boff, const double* v, double* y, long long Np, cudaStream_t st, int64_t* launches);
// A[i][j] = 0 where rowmask[i] == 0 (rowmask may be NULL) or colmask[j] == 0 (colmask may be NULL), i < nrows, j < ncols
cudaError_t fsa_mask_launch(double* A, long long ld, long long nrows, long long ncols, const double* rowmask,
                            const double* colmask, cudaStream_t st, int64_t* launches);
// dst[pos[i]] = src[i] (scatter 1) or dst[i] = src[pos[i]] (scatter 0), i < n
cudaError_t fsa_permute_launch(int scatter, const double* src, const long long* pos, long long n, double* dst, cudaStream_t st, int64_t* launches);
// out[i] = mask[i] * (a[i] - b[i])
cudaError_t fsa_resid_launch(double* out, const double* a, const double* b, const double* mask, long long n, cudaStream_t st, int64_t* launches);
// dst[i][j] += a[row_i + i] * a[row_j + j] on every item tile (the alpha_i alpha_i' part of the FSA gradient weights)
cudaError_t fsa_outer_launch(const FsaGramItem* items, int n, const double* a, cudaStream_t st, int64_t* launches);
// Block-diagonal weighted gradient trace: out[p] = sum over the item tiles of sum_ij dst[i][j] dk(x_{row_i+i}, x_{row_j+j})/dθ_p
// over real rows (mask != 0), for all P = P.n_theta parameters in one pass; the kernel derivatives are recomputed from x.
// part: n * n_theta scratch; per-tile partials are summed in a fixed order (two runs agree bit for bit).
cudaError_t fsa_trace_launch(const KProg& P, const double* xb, int d, const FsaGramItem* items, int n, const double* mask,
                             double* part, double* out, cudaStream_t st, int64_t* launches);
// C[i][j] += alpha * A[j][i], i < nrows, j < ncols
cudaError_t fsa_axpy_t_launch(double* C, long long ldc, const double* A, long long lda, long long nrows, long long ncols,
                              double alpha, cudaStream_t st, int64_t* launches);
// Prediction pieces.  One tile of a test-block x training-block cross-Gram: dst[i][j] = k(xs_{row_i+i}, xb_{row_j+j}) with
// xs / xb the staged test / padded training inputs, 0 on training padding rows (mask 0).
cudaError_t fsa_crossgram_launch(const KProg& P, const double* xs, const double* xb, int d, const FsaGramItem* items, int n,
                                 const double* mask, cudaStream_t st, int64_t* launches);
// Row products of 128-row tiles: out[i] = sum_{k < K} A[i][k] v[k] (sq = 0) or sum_{k < K} A[i][k]^2 (sq = 1), i < 128
struct FsaRowItem {
    const double* A;
    const double* v;
    double* out;
    long long lda;
    int K;
    int sq;
};
cudaError_t fsa_rowdot_launch(const FsaRowItem* items, int n, cudaStream_t st, int64_t* launches);
// out[i] = q[i] - g2[i] - r2neg[i]: k** - |V*|^2 - |G|^2 + |R|^2 from q = k** - |V*|^2 and r2neg = -|R|^2
cudaError_t fsa_var_launch(double* out, const double* q, const double* g2, const double* r2neg, long long n, cudaStream_t st, int64_t* launches);
// Predictive gradients of block-paired predictions, one CTA per item (one real test point):
//   dmu[out, :]  = sum_{j < M} dk(x*, z_j)/dx* (u_j - Wb[row, j]) + sum_i dk(x*, xb_i)/dx* alpha_i
//   dvar[out, :] = dk(x*, x*)/dx* + sum_{j < M} dk(x*, z_j)/dx* 2 (S1[row, j] - S2[row, j]) + sum_i dk(x*, xb_i)/dx* E[row, i - b0]
// with x* = xs[row], i over the real rows (mask != 0) of the paired block [b0, b0 + nb) of the padded training inputs xb.
// Wb may be null (0); dvar null: dmu only (S1, S2, E unread).  xs, z and xb have leading dimension d, the coefficient rows
// ldw, E lde.  Every coordinate is summed by one fixed tree, so a row's result does not depend on the launch it is in.
struct FsaDxItem {
    long long row;          // row of xs and of the coefficient rows Wb / S1 / S2 / E
    long long out;          // row of dmu / dvar
    long long b0;           // first padded training row of the paired block
    long long nb;           // padded rows of the paired block (0: unpaired)
};
cudaError_t fsa_crossgram_dx_launch(const KProg& P, const double* xs, const double* z, const double* xb, int d, long long M,
                                    const double* u, const double* Wb, const double* S1, const double* S2, long long ldw,
                                    const double* mask, const double* alpha, const double* E, long long lde,
                                    const FsaDxItem* items, int n, double* dmu, double* dvar, cudaStream_t st, int64_t* launches);
// Training-input gradient of the block-diagonal part: for every real row i (< n) of the item's 128-row tile row of a block
// with B x B weights G (row-major, ld B; rows 0 .. n-1 real, the rest padding), whose row 0 is padded row row0 of xb,
//   out[row(i), :] (=, or += when accumulate) sum_{l < n} (G[i][l] + G[l][i]) d1k(x_i, x_l)
// (d1k: derivative in the first argument; the l = i term is G[i][i] times the derivative of k(x_i, x_i)), row(i) =
// map[row0 + i] (map may be null: row0 + i).  One CTA per item, one thread per row, no atomics: fixed-order sums.
struct FsaBlockDxItem {
    const double* G;
    long long row0;
    int B;                  // padded block size, the leading dimension of G
    int n;                  // real rows of the block
    int tile;               // tile row: rows 128 tile .. 128 tile + 127
    int pad_;
};
cudaError_t fsa_block_dx_launch(const KProg& P, const double* xb, int d, const FsaBlockDxItem* items, int n, const long long* map,
                                double* out, int accumulate, cudaStream_t st, int64_t* launches);
