// potrf_base.cu -- the latency-critical leaf of the blocked Cholesky: one CTA factors a 128 x 128
// diagonal tile and inverts its factor.
//
// Replaces, at tile granularity, LAPACK dpotrf('U') behind cholesky!(Symmetric(F,:U))
// (/root/reference/src/GP.jl:110).  Outputs per tile at diagonal offset p:
//   F[p.., p..]      lower triangle  <- L_dd            (K_y = L L', L = U')
//   Dinv [p.., 0..128)               <- W = L_dd^-1     (clean lower-triangular tile)
//   DinvT[p.., 0..128)               <- W'              (clean upper-triangular tile)
//   logd[p + j]                      <- log(d_j) = 2 log L_jj      (logdet = sum, GPE.jl:210)
//   info                             <- p + j + 1 of the first non-positive pivot (atomicMin)
//
// Design: the tile lives in shared memory (row stride 129 doubles), factored in 16-wide panels.
//   phase 1, per 16-column panel:  (a) warp 0 factors the 16 x 16 diagonal block in registers (rows across lanes, pivots and
//            columns exchanged by shuffles);  (b) every row below solves its 16 unknowns against that block (one thread per
//            row, forward substitution with broadcast reads);  (c) rank-16 update of the trailing lower triangle, 8 x 8
//            register tiles per thread, 16 shared-memory loads per 64 FMAs.
//   phase 2: the 16 x 16 diagonal blocks are inverted (one warp per block, one column per lane), then W = L^-1 is built block
//            row by block row:  W[i, j] = -W_ii * sum_{j <= k < i} L[i, k] W[k, j]  (two small products per block row).
// ~40 barriers per tile and N^3/6-class FMA counts.  Written with plain unrolled loops the 16 x 16 block stays in local memory
// and phase 2 becomes a chain of dependent shared-memory dot products; the template recursion and the register-tiled
// right-looking phase 2 avoid both.
#include "potrf_base.cuh"
#include <math.h>

namespace {

constexpr int T = 128;
constexpr int LDS = 129;
constexpr int NTB = 256;
constexpr int PB = 16;                                     // panel width

__device__ __forceinline__ double& WT(double* S, int m, int j) { return S[j * LDS + m + 1]; }      // W[m][j], m >= j, in the upper part

// 16 x 16 Cholesky in registers, rows across lanes (lane i = lane & 15 holds a[0..15] of row i).  Template recursion keeps every
// array index a compile-time constant: with plain unrolled loops the compiler kept a[] in local memory (LDL/STL), which made
// the serial 16 x 16 blocks a large share of the tile.
template <int J, int K>
struct Chol16Upd {
    static __device__ __forceinline__ void run(double (&a)[PB], double lij, int i) {
        const double lkj = __shfl_sync(0xffffffffu, lij, K);
        if (i >= K) a[K] = fma(-lij, lkj, a[K]);
        Chol16Upd<J, K + 1>::run(a, lij, i);
    }
};
template <int J>
struct Chol16Upd<J, PB> {
    static __device__ __forceinline__ void run(double (&)[PB], double, int) {}
};
template <int J>
struct Chol16Step {
    static __device__ __forceinline__ void run(double (&a)[PB], int i, int lane, double* invd, int* info, int pj) {
        double d = __shfl_sync(0xffffffffu, a[J], J);
        const bool bad = !(d > 0.0);                          // not positive definite (or NaN): record, keep going
        if (bad && lane == 0) atomicMin(info, pj + J + 1);
        d = bad ? 1.0 : d;
        const double rs = rsqrt(d);
        const double lij = (i == J) ? d * rs : a[J] * rs;     // L[i][J] for i >= J (0 above the diagonal: a[J] is 0 there)
        if (i >= J) a[J] = lij;
        if (lane == J) invd[J] = rs;                          // 1 / L[J][J]
        Chol16Upd<J, J + 1>::run(a, lij, i);
        Chol16Step<J + 1>::run(a, i, lane, invd, info, pj);
    }
};
template <>
struct Chol16Step<PB> {
    static __device__ __forceinline__ void run(double (&)[PB], int, int, double*, int*, int) {}
};
// column c of the inverse of a 16 x 16 lower-triangular block L (rows broadcast from shared memory): x[i], i = 0..15
template <int I, int M>
struct Inv16Dot {
    static __device__ __forceinline__ double run(const double* lrow, const double (&x)[PB], double s) {
        return Inv16Dot<I, M + 1>::run(lrow, x, fma(-lrow[M], x[M], s));
    }
};
template <int I>
struct Inv16Dot<I, I> {
    static __device__ __forceinline__ double run(const double*, const double (&)[PB], double s) { return s; }
};
template <int I>
struct Inv16Row {
    static __device__ __forceinline__ void run(const double* Lblk, const double* invd, int c, double (&x)[PB]) {
        const double s = Inv16Dot<I, 0>::run(Lblk + I * LDS, x, (I == c) ? 1.0 : 0.0);
        x[I] = (I >= c) ? s * invd[I] : 0.0;
        Inv16Row<I + 1>::run(Lblk, invd, c, x);
    }
};
template <>
struct Inv16Row<PB> {
    static __device__ __forceinline__ void run(const double*, const double*, int, double (&)[PB]) {}
};
// phase 2, step BK: Acc[r][j] += sum_k L[r][16 BK + k] W[16 BK + k][j] for the row blocks a > BK and column blocks b <= BK
// (W[m][j] and Acc[m][j] are kept at S[j][m+1]); in the diagonal column block W[16 BK + k][j] = 0 for k < j - 16 BK
template <int BK>
__device__ __forceinline__ void inverse_update(double* S, int ty, int tx) {
    double acc[8][8];
#pragma unroll
    for (int a_ = BK + 1; a_ < 8; ++a_)
#pragma unroll
        for (int b_ = 0; b_ <= BK; ++b_) acc[a_][b_] = 0.0;
#pragma unroll 4
    for (int k = 0; k < PB; ++k) {
        double av[8], bv[8];
#pragma unroll
        for (int a_ = BK + 1; a_ < 8; ++a_) av[a_] = S[(ty + PB * a_) * LDS + PB * BK + k];
#pragma unroll
        for (int b_ = 0; b_ <= BK; ++b_) bv[b_] = (b_ == BK && k < tx) ? 0.0 : S[(tx + PB * b_) * LDS + PB * BK + k + 1];
#pragma unroll
        for (int a_ = BK + 1; a_ < 8; ++a_)
#pragma unroll
            for (int b_ = 0; b_ <= BK; ++b_) acc[a_][b_] = fma(av[a_], bv[b_], acc[a_][b_]);
    }
#pragma unroll
    for (int a_ = BK + 1; a_ < 8; ++a_)
#pragma unroll
        for (int b_ = 0; b_ <= BK; ++b_) S[(tx + PB * b_) * LDS + ty + PB * a_ + 1] += acc[a_][b_];
}
// rank-16 trailing update for the 16-blocks >= T0 (compile-time: the 8 x 8 register tile only carries the live blocks)
template <int T0>
__device__ __forceinline__ void trailing_update(double* S, int c0, int ty, int tx) {
    double acc[8][8];
#pragma unroll
    for (int a_ = T0; a_ < 8; ++a_)
#pragma unroll
        for (int b_ = T0; b_ < 8; ++b_) acc[a_][b_] = 0.0;
#pragma unroll 4
    for (int k = 0; k < PB; ++k) {
        double av[8], bv[8];
#pragma unroll
        for (int a_ = T0; a_ < 8; ++a_) av[a_] = S[(ty + PB * a_) * LDS + c0 + k];
#pragma unroll
        for (int b_ = T0; b_ < 8; ++b_) bv[b_] = S[(tx + PB * b_) * LDS + c0 + k];
#pragma unroll
        for (int a_ = T0; a_ < 8; ++a_)
#pragma unroll
            for (int b_ = T0; b_ < 8; ++b_)
                if (a_ >= b_) acc[a_][b_] = fma(av[a_], bv[b_], acc[a_][b_]);      // blocks above the diagonal are never stored
    }
#pragma unroll
    for (int a_ = T0; a_ < 8; ++a_)
#pragma unroll
        for (int b_ = T0; b_ < 8; ++b_) {
            const int r = ty + PB * a_, c = tx + PB * b_;
            if (a_ >= b_ && r >= c) S[r * LDS + c] -= acc[a_][b_];
        }
}

// One tile.  G / Dinv / DinvT / logd point at the tile's origin (Dinv and DinvT share the leading dimension ldd); `p` is the
// tile's diagonal offset in the peers' buffers and info_base + j + 1 is recorded for a non-positive pivot j.  kWriteF = false
// skips the L output (the batched block-diagonal factorisation of fsa.cu needs only the two inverse tiles).
template <bool kWriteF>
__device__ __forceinline__ void potrf128_blk_tile(const double* __restrict__ G, long long ldg, double* __restrict__ F, long long ldf,
                                                  double* __restrict__ Dinv, double* __restrict__ DinvT, long long ldd,
                                                  double* __restrict__ logd, int* __restrict__ info, int info_base, int p,
                                                  const PotrfPeers& peers) {
    extern __shared__ double S[];                  // [128][129] tile | W16[8][16][17] | T[16][129] | invd[128]
    double* W16 = S + T * LDS;
    double* Tb = W16 + 8 * PB * 17;
    double* invd = Tb + PB * LDS;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

    for (int idx = tid; idx < T * T; idx += NTB) {
        const int m = idx >> 7, n = idx & 127;
        S[m * LDS + n] = (n <= m) ? G[(long long)m * ldg + n] : 0.0;
    }
    if (tid < T) S[tid * LDS + T] = 0.0;                  // column 128 holds W[127][.]: the phase-2 accumulators start from zero
    __syncthreads();

    // ------------------------------- phase 1: Cholesky, 16-column panels -------------------------------
#pragma unroll 1
    for (int pb = 0; pb < T / PB; ++pb) {
        const int c0 = pb * PB;
        if (warp == 0) {
            // (a) 16 x 16 diagonal block in registers: lane i (< 16) holds row i
            const int i = lane & 15;
            double a[PB];
#pragma unroll
            for (int k = 0; k < PB; ++k) a[k] = (k <= i) ? S[(c0 + i) * LDS + c0 + k] : 0.0;
            Chol16Step<0>::run(a, i, lane, invd + c0, info, info_base + c0);
            if (lane < PB) {
#pragma unroll
                for (int k = 0; k < PB; ++k) if (k <= i) S[(c0 + i) * LDS + c0 + k] = a[k];
            }
        }
        __syncthreads();
        // (b) rows below the block: x_j = (a_j - sum_{k<j} x_k L[j][k]) / L[j][j], one thread per row
        {
            const int r = c0 + PB + tid;
            if (r < T) {
                double x[PB];
#pragma unroll
                for (int j = 0; j < PB; ++j) x[j] = S[r * LDS + c0 + j];
#pragma unroll
                for (int j = 0; j < PB; ++j) {
                    double s = x[j];
#pragma unroll
                    for (int k = 0; k < j; ++k) s = fma(-x[k], S[(c0 + j) * LDS + c0 + k], s);
                    x[j] = s * invd[c0 + j];
                }
#pragma unroll
                for (int j = 0; j < PB; ++j) S[r * LDS + c0 + j] = x[j];
            }
        }
        __syncthreads();
        // (c) trailing update S[r][c] -= sum_k L[r][c0+k] L[c][c0+k], r >= c >= c0 + 16: thread (ty, tx) owns rows ty + 16 a, cols tx + 16 b
        {
            const int ty = tid >> 4, tx = tid & 15;
            switch (pb + 1) {                                 // first trailing 16-block
            case 1: trailing_update<1>(S, c0, ty, tx); break;
            case 2: trailing_update<2>(S, c0, ty, tx); break;
            case 3: trailing_update<3>(S, c0, ty, tx); break;
            case 4: trailing_update<4>(S, c0, ty, tx); break;
            case 5: trailing_update<5>(S, c0, ty, tx); break;
            case 6: trailing_update<6>(S, c0, ty, tx); break;
            case 7: trailing_update<7>(S, c0, ty, tx); break;
            default: break;
            }
        }
        __syncthreads();
    }

    // pivots: logd = log(d_j) = 2 log L_jj
    if (tid < T) {
        const double lg = 2.0 * log(S[tid * LDS + tid]);
        logd[tid] = lg;
        for (int q = 0; q < peers.n; ++q) peers.logd[q][p + tid] = lg;
    }
    // L (lower triangle) to global memory
    for (int idx = tid; kWriteF && idx < T * T; idx += NTB) {
        const int m = idx >> 7, j = idx & 127;
        if (j <= m) {
            const double v = S[m * LDS + j];
            F[(long long)m * ldf + j] = v;
            for (int q = 0; q < peers.n; ++q) peers.F[q][(long long)(p + m) * ldf + p + j] = v;
        }
    }

    // ------------------------------- phase 2: W = L^-1 -------------------------------
    // 16 x 16 diagonal-block inverses: warp w handles block w, lane c (< 16) computes column c by forward substitution
    {
        const int c0 = warp * PB, c = lane & 15;
        double x[PB];
        Inv16Row<0>::run(S + c0 * LDS + c0, invd + c0, c, x);
        if (lane < PB) {
#pragma unroll
            for (int i = 0; i < PB; ++i) W16[(warp * PB + i) * 17 + c] = x[i];
        }
    }
    __syncthreads();
    // diagonal blocks of W into the upper part of S: W[m][j] -> S[j][m+1]
    for (int idx = tid; idx < 8 * PB * PB; idx += NTB) {
        const int b = idx >> 8, i = (idx >> 4) & 15, j = idx & 15;
        if (i >= j) WT(S, b * PB + i, b * PB + j) = W16[(b * PB + i) * 17 + j];
    }
    __syncthreads();
    // right-looking over row blocks: the accumulators Acc[i][j] = sum_k L[i][k] W[k][j] of the off-diagonal blocks live where
    // W[i][j] will be (upper part of S, zero so far).  Step bk: finalise row block bk (W = -W16[bk] Acc), then every row block
    // below receives the rank-16 contribution L[., bk] W[bk, .] with an 8 x 8 register tile per thread.
#pragma unroll 1
    for (int bk = 0; bk < T / PB; ++bk) {
        const int r0 = bk * PB;
        if (bk > 0) {
            for (int j = tid; j < r0; j += NTB) {                 // one thread per column j < 16 bk
                double x[PB], w[PB];
#pragma unroll
                for (int i = 0; i < PB; ++i) x[i] = WT(S, r0 + i, j);
#pragma unroll
                for (int i = 0; i < PB; ++i) {
                    double acc_ = 0.0;
#pragma unroll
                    for (int k = 0; k <= i; ++k) acc_ = fma(W16[(r0 + i) * 17 + k], x[k], acc_);
                    w[i] = -acc_;
                }
#pragma unroll
                for (int i = 0; i < PB; ++i) WT(S, r0 + i, j) = w[i];
            }
            __syncthreads();
        }
        const int ty = tid >> 4, tx = tid & 15;
        switch (bk) {
        case 0: inverse_update<0>(S, ty, tx); break;
        case 1: inverse_update<1>(S, ty, tx); break;
        case 2: inverse_update<2>(S, ty, tx); break;
        case 3: inverse_update<3>(S, ty, tx); break;
        case 4: inverse_update<4>(S, ty, tx); break;
        case 5: inverse_update<5>(S, ty, tx); break;
        case 6: inverse_update<6>(S, ty, tx); break;
        default: break;
        }
        __syncthreads();
    }

    // ---- write W (clean lower) and W' (clean upper) ----
    for (int idx = tid; idx < T * T; idx += NTB) {
        const int r = idx >> 7, c = idx & 127;
        const double wl = (c <= r) ? S[c * LDS + r + 1] : 0.0;
        const double wu = (c >= r) ? S[r * LDS + c + 1] : 0.0;
        Dinv[(long long)r * ldd + c] = wl;
        DinvT[(long long)r * ldd + c] = wu;
        for (int q = 0; q < peers.n; ++q) {
            peers.Dinv[q][(long long)(p + r) * T + c] = wl;
            peers.DinvT[q][(long long)(p + r) * T + c] = wu;
        }
    }
}

__global__ void __launch_bounds__(NTB, 1)
potrf128_blk_kernel(const double* __restrict__ G, long long ldg, double* __restrict__ F, long long ldf,
                    double* __restrict__ Dinv, double* __restrict__ DinvT, double* __restrict__ logd,
                    int* __restrict__ info, int p0, int tile_stride, const PotrfPeers peers) {
    const int p = p0 + blockIdx.x * tile_stride;
    potrf128_blk_tile<true>(G + (long long)p * ldg + p, ldg, F + (long long)p * ldf + p, ldf, Dinv + (long long)p * T,
                            DinvT + (long long)p * T, T, logd + p, info, p, p, peers);
}

// pointer-table entry point: CTA b factors the tile of items[b]
__global__ void __launch_bounds__(NTB, 1) potrf128_ptr_kernel(const Potrf128Item* __restrict__ items, int* __restrict__ info) {
    const Potrf128Item it = items[blockIdx.x];
    const PotrfPeers none{};
    potrf128_blk_tile<false>(it.G, it.ld, nullptr, 0, it.Dinv, it.DinvT, it.ld, it.logd, info, it.info_base, 0, none);
}

// dynamic shared memory of both entry points (layout: potrf128_blk_tile)
constexpr size_t SMEM_BLK = (size_t)(T * LDS + 8 * PB * 17 + PB * LDS + T) * sizeof(double);
bool g_attr_set_blk = false, g_attr_set_ptr = false;

}  // namespace

cudaError_t potrf128_launch(const double* G, int64_t ldg, double* F, int64_t ldf, double* Dinv, double* DinvT,
                            double* logd, int* info, int p0, int ntiles, int tile_stride, cudaStream_t st, int64_t* launches,
                            const PotrfPeers* peers) {
    PotrfPeers pp{};
    if (peers) pp = *peers;
    if (!g_attr_set_blk) {
        cudaError_t e = cudaFuncSetAttribute(potrf128_blk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BLK);
        if (e != cudaSuccess) return e;
        g_attr_set_blk = true;
    }
    potrf128_blk_kernel<<<ntiles, NTB, SMEM_BLK, st>>>(G, ldg, F, ldf, Dinv, DinvT, logd, info, p0, tile_stride, pp);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t potrf128_ptr_launch(const Potrf128Item* items, int n, int* info, cudaStream_t st, int64_t* launches) {
    if (n <= 0) return cudaSuccess;
    if (!g_attr_set_ptr) {
        cudaError_t e = cudaFuncSetAttribute(potrf128_ptr_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BLK);
        if (e != cudaSuccess) return e;
        g_attr_set_ptr = true;
    }
    potrf128_ptr_kernel<<<n, NTB, SMEM_BLK, st>>>(items, info);
    if (launches) ++*launches;
    return cudaGetLastError();
}
