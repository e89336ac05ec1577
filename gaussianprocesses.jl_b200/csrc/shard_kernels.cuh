// shard_kernels.cuh -- data-movement kernels of the row-sharded multi-GPU schedules (shard_impl.cuh):
// panel scatter / all-gather unpack, generic transposes, diagonal-block packing.  All bandwidth-bound, O(N * NB) per panel.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

// block-cyclic ownership of 128-row tiles: tile t belongs to rank (t / rb) % R
struct ShardOwn {
    int R, me, rb;
};
// number of tiles t' < t owned by rank q
__host__ __device__ inline long long shard_own_before(long long t, int q, int rb, int R) {
    const long long cyc = (long long)rb * R;
    const long long c = t / cyc, rem = t % cyc;
    long long extra = rem - (long long)q * rb;
    if (extra < 0) extra = 0;
    if (extra > rb) extra = rb;
    return c * rb + extra;
}

// dst (n x n, ld ldd) = lower triangle of src (ld lds), zeros above the diagonal
cudaError_t shard_copy_lower(double* dst, int64_t ldd, const double* src, int64_t lds, int n, cudaStream_t st, int64_t* launches);
// own tile rows t >= t1 (rows r >= 128*t1): F[r, c0..c0+nb) = G[r, c0..c0+nb);  S_me[(li(r)), 0..nb) = same (ld nbp),
// li = local index of the row among this rank's rows >= 128*t1
cudaError_t shard_scatter_rows(const double* G, double* F, int64_t ld, int64_t Npad, int c0, int nb, int t1, double* S_me,
                               int nbp, ShardOwn own, cudaStream_t st, int64_t* launches);
// all rows r >= 128*t1: P[r, 0..nb) = S[owner(r)][li(r)][0..nb) ; S regions of `per_rank` doubles each
cudaError_t shard_unpack_panel(double* P, int nbp, int64_t Npad, int nb, int t1, const double* S, int64_t per_rank,
                               ShardOwn own, cudaStream_t st, int64_t* launches);
// dst[j * ldd + i] = src[i * lds + j], i < rows, j < cols
cudaError_t shard_transpose(double* dst, int64_t ldd, const double* src, int64_t lds, int64_t rows, int64_t cols, cudaStream_t st, int64_t* launches);
// P[(j0 + c), i] (ld nbp) = W_JJ[c, i] for c >= i (strictly-lower tiles from G, diagonal tiles from Dinv), 0 for c < i
cudaError_t shard_pack_wblock(double* P, int nbp, const double* G, int64_t ld, const double* Dinv, int j0, int nb, cudaStream_t st, int64_t* launches);
// out[i] = sum_q in[q * stride + i]  (fixed rank order), i < n
cudaError_t shard_sum_ranks(double* out, const double* in, int64_t stride, int nranks, int64_t n, cudaStream_t st, int64_t* launches);
// out[0] = min_q in[q]
cudaError_t shard_min_ranks(int* out, const int* in, int nranks, cudaStream_t st, int64_t* launches);

// ---- cross-validation on row-sharded storage.  "Compact" vectors hold one entry per own row, own tiles in ascending order:
// own row r of tile t sits at li = shard_own_before(t, me) * 128 + r % 128.
// dst[j * ldd + i] = src[i * lds + j] for i < rows, j < cols, only where destination row j lies in an own tile
cudaError_t shard_transpose_own(double* dst, int64_t ldd, const double* src, int64_t lds, int64_t rows, int64_t cols, ShardOwn own,
                                cudaStream_t st, int64_t* launches);
// own rows in the tiles covering rows 0 .. n (length of the compact vectors)
int64_t shard_own_rows(int64_t n, ShardOwn own);
// own rows r < N: out[2 li] = <Y_r, alpha>, out[2 li + 1] = <G_r, Y_r> over ncols columns (0 for padding rows)
cudaError_t shard_rowdot_own(const double* Y, const double* G, int64_t ld, int64_t ncols, const double* alpha, int64_t N, ShardOwn own,
                             double* out, cudaStream_t st, int64_t* launches);
// out[li] = G[r, r] for the own rows r of the tiles covering 0 .. N
cudaError_t shard_diag_own(const double* G, int64_t ld, int64_t N, ShardOwn own, double* out, cudaStream_t st, int64_t* launches);
// out[a * nv + b] = src[max(ia, ib) * ld + min(ia, ib)] where that row is own, else 0 (i* = idx[*]): summed over the ranks, the
// exactly symmetric principal sub-block of a matrix whose lower triangle is stored
cudaError_t shard_gather_block_own(double* out, const double* src, int64_t ld, const long long* idx, int64_t nv, ShardOwn own,
                                   cudaStream_t st, int64_t* launches);

// ---- replicated storage (gpb200.cu).  inverse_dist splits a level s of the triangular inverse when (s / 128) % nranks == 0:
// rank q computes the 128-wide tile columns t % nranks == q of every W21 block, its "slice" (wr = s / nranks columns; local
// column jl <-> block column ((jl / 128) * nranks + q) * 128 + jl % 128).  Problem z of the level starts at p = 2 s z and has
// n2_z = min(s, Np - p - s) rows (<= 0: none).
// out[z s wr + i wr + jl] = G[(p + s + i) ld + p + gj(jl, self)], i < n2_z  (this rank's slice of every W21 block)
cudaError_t shard_pack_slices(const double* G, int64_t ld, double* out, int s, int nranks, int self, int Np, cudaStream_t st,
                              int64_t* launches);
// for every rank q != self: its slice from in + q per_rank (laid out as pack_slices writes it) into W21 (rows p + s + i,
// columns p + gj(jl, q)) and, transposed, into G's strict-upper block (rows p + gj, columns p + s + i).  The rank's own slice
// is left alone: its lower half was written by the GEMM, its transpose by the GEMM's Ct epilogue.
cudaError_t shard_unpack_slices(double* G, int64_t ld, const double* in, int64_t per_rank, int s, int nranks, int self, int Np,
                                cudaStream_t st, int64_t* launches);
// cholesky_dist_p2p: after a system-wide fence, *peer_sig_words[q] = value (release, system scope) for q < n_peer (<= 32)
cudaError_t shard_signal_peers(int* const* peer_sig_words, int n_peer, int value, cudaStream_t st, int64_t* launches);
// one thread spins (acquire, system scope) until *word >= target; after about 2^27 polls it sets *err = 1 and returns
cudaError_t shard_wait_signal(const int* word, int target, int* err, cudaStream_t st, int64_t* launches);
