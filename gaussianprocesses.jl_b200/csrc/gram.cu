// gram.cu -- Gram-matrix build, cross-Gram and the fused gradient-trace kernel.
//
// Replaces the reference's scalar loops
//   cov!(cK, k, X, data)            src/kernels/kernels.jl:39-50   (symmetric, j>=i + mirror)
//   cov!(cK, k, X1, X2, data)       src/kernels/kernels.jl:56-71   (rectangular, predict)
//   dmll_kern!(dmll, k, X, data, A) src/GPE.jl:219-241             (1/2 sum_ij A_ij dK_ij/dθ)
// and removes the N x N distance cache (IsotropicData.R, src/kernels/stationary.jl:34-40):
// distances are recomputed from the 128 x d input tiles staged in shared memory.  When two staged tiles (and a kernel's
// reduction scratch) exceed the device's opt-in shared memory per block (d >= 110 on an H100), the tile kernels read the
// points in place from global memory instead: the same values enter the same arithmetic, so the results are bitwise
// those of the staged kernels (and of fsa_gram, which always reads global memory).  Padding rows are never read.
//
// Tile-per-CTA (128 x 128 outputs, 256 threads): the two input tiles are staged in shared memory
// (row stride padded to an odd number of doubles -> conflict-free column reads), each warp owns 16
// rows, each lane 2 x 2 adjacent columns, so a warp stores 512 contiguous bytes per row (16-byte
// vector stores).  Only lower-triangle tiles (bm >= bn) are built: the factorisation reads the
// lower triangle only, halving HBM writes versus the reference's mirrored full matrix.
#include "gram.cuh"
#include <math.h>

namespace {

constexpr int TB = 128;        // tile edge
constexpr int NT = 256;        // threads

__device__ __forceinline__ void load_xtile(double* s, const double* __restrict__ x, long long ldx, int d, int ds,
                                           long long row0, long long nrows_valid) {
    // s[r*ds + k] = x[(row0+r)*ldx + k] for r < 128 (zero beyond the valid rows)
    for (int idx = threadIdx.x; idx < TB * d; idx += NT) {
        const int r = idx / d, k = idx - r * d;
        const long long gr = row0 + r;
        s[r * ds + k] = (gr < nrows_valid) ? x[gr * ldx + k] : 0.0;
    }
}

// The tile of points row0 .. row0+127 as (base, row stride): staged into s when `staged`, else x itself in global memory
// (rows past the valid count are then not addressable, and every kernel guards them before it evaluates the program).
struct XTile {
    const double* p;
    long long ld;
    __device__ __forceinline__ const double* row(int r) const { return p + r * ld; }
};
__device__ __forceinline__ XTile xtile(bool staged, double* s, const double* x, long long ldx, int d, long long row0,
                                       long long nrows_valid) {
    if (!staged) return XTile{x + row0 * ldx, ldx};
    load_xtile(s, x, ldx, d, d | 1, row0, nrows_valid);
    return XTile{s, d | 1};
}

// ------------------------------------------------------------------------------------------
// symmetric Gram, lower tiles:  G[i,j] = k(x_i,x_j) + [i==j] noise_i ; padding = identity
// ------------------------------------------------------------------------------------------
template <bool FAST>
__global__ void __launch_bounds__(NT) gram_lower_kernel(const __grid_constant__ KProg P, const double* __restrict__ x,
                                                        long long ldx, int d, long long N, long long Npad,
                                                        const double* __restrict__ noise_var, long long n_noise,
                                                        double nugget, double* __restrict__ G, long long ldg,
                                                        int own_tiles, int nranks, int rank, int own_axis, int bm_min,
                                                        int staged) {
    const int bm = blockIdx.y, bn = blockIdx.x;
    if (bn > bm || bm < bm_min) return;
    // multi-GPU ownership: block columns (replicated storage, own_axis 0) or block rows (row-sharded storage, own_axis 1)
    if (own_tiles > 0 && (((own_axis ? bm : bn) / own_tiles) % nranks) != rank) return;
    extern __shared__ double sm[];
    const int ds = d | 1;
    double* sXi = sm;
    double* sXj = sm + TB * ds;
    const XTile ti = xtile(staged, sXi, x, ldx, d, (long long)bm * TB, N);
    const XTile tj = xtile(staged, sXj, x, ldx, d, (long long)bn * TB, N);
    __syncthreads();

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double mh = 0.0, s2 = 0.0;
    if (FAST) { mh = -0.5 / P.par[0]; s2 = P.par[1]; }
    if (FAST && d <= 8 && staged) {
        // register-cached variant: the lane's 4 column points live in registers, a row point is read
        // once per row (8 broadcast LDS) -> 2 LDS per output instead of 16: FP64-ALU bound, not LSU bound
        double xjr[4][8];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int c = (q >> 1) * 64 + lane * 2 + (q & 1);
#pragma unroll
            for (int k = 0; k < 8; ++k) xjr[q][k] = (k < d) ? sXj[c * ds + k] : 0.0;
        }
#pragma unroll 1
        for (int rr = 0; rr < 16; ++rr) {
            const int r = warp * 16 + rr;
            const long long gi = (long long)bm * TB + r;
            double xir[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) xir[k] = (k < d) ? sXi[r * ds + k] : 0.0;
            double v[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const long long gj = (long long)bn * TB + (q >> 1) * 64 + lane * 2 + (q & 1);
                double r2 = 0.0;
#pragma unroll
                for (int k = 0; k < 8; ++k) { const double df = xir[k] - xjr[q][k]; r2 += df * df; }
                double kv = s2 * exp(mh * r2);
                if (gi >= N || gj >= N) kv = (gi == gj) ? 1.0 : 0.0;
                else if (gi == gj) kv += ((n_noise == 1) ? noise_var[0] : noise_var[gi]) + nugget;
                v[q] = kv;
            }
            double* row = G + gi * ldg + (long long)bn * TB + lane * 2;
            *reinterpret_cast<double2*>(row) = make_double2(v[0], v[1]);
            *reinterpret_cast<double2*>(row + 64) = make_double2(v[2], v[3]);
        }
        return;
    }
#pragma unroll 1
    for (int rr = 0; rr < 16; ++rr) {
        const int r = warp * 16 + rr;
        const long long gi = (long long)bm * TB + r;
        const double* xi = ti.row(r);
#pragma unroll
        for (int b = 0; b < 2; ++b) {
            const int c0 = b * 64 + lane * 2;
            double v[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int c = c0 + e;
                const long long gj = (long long)bn * TB + c;
                const double* xj = tj.row(c);
                double kv = 0.0;
                if (gi < N && gj < N) {                    // a padding row is never read
                    if (FAST) {
                        double r2 = 0.0;
                        for (int k = 0; k < d; ++k) { const double df = xi[k] - xj[k]; r2 += df * df; }
                        kv = s2 * exp(mh * r2);
                    } else {
                        kv = kprog_eval<false>(P, xi, xj, nullptr);
                    }
                }
                if (gi >= N || gj >= N) kv = (gi == gj) ? 1.0 : 0.0;
                else if (gi == gj) kv += ((n_noise == 1) ? noise_var[0] : noise_var[gi]) + nugget;
                v[e] = kv;
            }
            *reinterpret_cast<double2*>(G + gi * ldg + (long long)bn * TB + c0) = make_double2(v[0], v[1]);
        }
    }
}

// ------------------------------------------------------------------------------------------
// cross-Gram: Kst[m,n] = k(xs_m, x_n)   (M_pad x N_pad, zero padding)
// ------------------------------------------------------------------------------------------
template <bool FAST>
__global__ void __launch_bounds__(NT) crossgram_kernel(const __grid_constant__ KProg P, const double* __restrict__ xs,
                                                       long long ldxs, long long M, const double* __restrict__ x,
                                                       long long ldx, long long N, int d, double* __restrict__ Kst,
                                                       long long ldk, int staged) {
    const int bm = blockIdx.y, bn = blockIdx.x;
    extern __shared__ double sm[];
    const int ds = d | 1;
    const XTile ti = xtile(staged, sm, xs, ldxs, d, (long long)bm * TB, M);
    const XTile tj = xtile(staged, sm + TB * ds, x, ldx, d, (long long)bn * TB, N);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double mh = 0.0, s2 = 0.0;
    if (FAST) { mh = -0.5 / P.par[0]; s2 = P.par[1]; }
#pragma unroll 1
    for (int rr = 0; rr < 16; ++rr) {
        const int r = warp * 16 + rr;
        const long long gi = (long long)bm * TB + r;
        const double* xi = ti.row(r);
#pragma unroll
        for (int b = 0; b < 2; ++b) {
            const int c0 = b * 64 + lane * 2;
            double v[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int c = c0 + e;
                const long long gj = (long long)bn * TB + c;
                const double* xj = tj.row(c);
                double kv = 0.0;
                if (gi < M && gj < N) {                    // a padding row is never read
                    if (FAST) {
                        double r2 = 0.0;
                        for (int k = 0; k < d; ++k) { const double df = xi[k] - xj[k]; r2 += df * df; }
                        kv = s2 * exp(mh * r2);
                    } else {
                        kv = kprog_eval<false>(P, xi, xj, nullptr);
                    }
                }
                v[e] = kv;
            }
            *reinterpret_cast<double2*>(Kst + gi * ldk + (long long)bn * TB + c0) = make_double2(v[0], v[1]);
        }
    }
}

// prior variances k(xs_m, xs_m)
__global__ void kdiag_kernel(const __grid_constant__ KProg P, const double* __restrict__ xs, long long ldxs,
                             long long M, double* __restrict__ out) {
    const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    const double* xi = xs + m * ldxs;
    out[m] = kprog_eval<false>(P, xi, xi, nullptr);
}

// prior covariance K** (M_pad x M_pad, full, zero padding) -- used by full_cov prediction
template <bool FAST>
__global__ void __launch_bounds__(NT) gram_full_kernel(const __grid_constant__ KProg P, const double* __restrict__ xs,
                                                       long long ldxs, long long M, int d, double* __restrict__ Kss,
                                                       long long ldk, int staged) {
    const int bm = blockIdx.y, bn = blockIdx.x;
    extern __shared__ double sm[];
    const int ds = d | 1;
    const XTile ti = xtile(staged, sm, xs, ldxs, d, (long long)bm * TB, M);
    const XTile tj = xtile(staged, sm + TB * ds, xs, ldxs, d, (long long)bn * TB, M);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double mh = 0.0, s2 = 0.0;
    if (FAST) { mh = -0.5 / P.par[0]; s2 = P.par[1]; }
#pragma unroll 1
    for (int rr = 0; rr < 16; ++rr) {
        const int r = warp * 16 + rr;
        const long long gi = (long long)bm * TB + r;
        const double* xi = ti.row(r);
#pragma unroll
        for (int b = 0; b < 2; ++b) {
            const int c0 = b * 64 + lane * 2;
            double v[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int c = c0 + e;
                const long long gj = (long long)bn * TB + c;
                const double* xj = tj.row(c);
                double kv = 0.0;
                if (gi < M && gj < M) {                    // a padding row is never read
                    if (FAST) {
                        double r2 = 0.0;
                        for (int k = 0; k < d; ++k) { const double df = xi[k] - xj[k]; r2 += df * df; }
                        kv = s2 * exp(mh * r2);
                    } else {
                        kv = kprog_eval<false>(P, xi, xj, nullptr);
                    }
                }
                v[e] = kv;
            }
            *reinterpret_cast<double2*>(Kss + gi * ldk + (long long)bn * TB + c0) = make_double2(v[0], v[1]);
        }
    }
}

// dK/dtheta_j as a full symmetric matrix (N_pad x N_pad, zero padding): grad_slice! of the reference
// (/root/reference/src/kernels/kernels.jl:96-131), needed by the cross-validation gradients (src/crossvalidation.jl:67-170, 253-341).
// Tile row blockIdx.y holds global tile row bm0 + blockIdx.y: a row-sharded handle generates D in row batches (D points at row bm0 * 128).
__global__ void __launch_bounds__(NT) gram_grad_full_kernel(const __grid_constant__ KProg P, const double* __restrict__ x, long long ldx,
                                                            long long N, int d, int j, double* __restrict__ D, long long ldd, int bm0,
                                                            int staged) {
    const int bm = bm0 + blockIdx.y, bn = blockIdx.x;
    D += (long long)blockIdx.y * TB * ldd;
    extern __shared__ double sm[];
    const int ds = d | 1;
    const XTile ti = xtile(staged, sm, x, ldx, d, (long long)bm * TB, N);
    const XTile tj = xtile(staged, sm + TB * ds, x, ldx, d, (long long)bn * TB, N);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double gbuf[GPB200_MAX_THETA];
#pragma unroll 1
    for (int rr = 0; rr < 16; ++rr) {
        const int r = warp * 16 + rr;
        const long long gi = (long long)bm * TB + r;
        const double* xi = ti.row(r);
#pragma unroll 1
        for (int b = 0; b < 4; ++b) {
            const int c = (b >> 1) * 64 + lane * 2 + (b & 1);
            const long long gj = (long long)bn * TB + c;
            double v = 0.0;
            if (gi < N && gj < N) { kprog_eval<true>(P, xi, tj.row(c), gbuf); v = gbuf[j]; }
            D[r * ldd + gj] = v;
        }
    }
}

// dK(x1, x2)/dtheta_j as a rectangular matrix (N1_pad x N2_pad, zero padding): the cross-validation schedule of the sparse
// engine regenerates dK_fu / dK_Vu per chunk from it (gpb200_fitc_cv_param, gpb200_fitc_cv_block).
__global__ void __launch_bounds__(NT) crossgram_grad_kernel(const __grid_constant__ KProg P, const double* __restrict__ x1,
                                                            long long ldx1, long long N1, const double* __restrict__ x2,
                                                            long long ldx2, long long N2, int d, int j, double* __restrict__ D,
                                                            long long ldd, int staged) {
    const int bm = blockIdx.y, bn = blockIdx.x;
    extern __shared__ double sm[];
    const int ds = d | 1;
    const XTile ti = xtile(staged, sm, x1, ldx1, d, (long long)bm * TB, N1);
    const XTile tj = xtile(staged, sm + TB * ds, x2, ldx2, d, (long long)bn * TB, N2);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double gbuf[GPB200_MAX_THETA];
#pragma unroll 1
    for (int rr = 0; rr < 16; ++rr) {
        const int r = warp * 16 + rr;
        const long long gi = (long long)bm * TB + r;
        const double* xi = ti.row(r);
#pragma unroll 1
        for (int b = 0; b < 4; ++b) {
            const int c = (b >> 1) * 64 + lane * 2 + (b & 1);
            const long long gj = (long long)bn * TB + c;
            double v = 0.0;
            if (gi < N1 && gj < N2) { kprog_eval<true>(P, xi, tj.row(c), gbuf); v = gbuf[j]; }
            D[gi * ldd + gj] = v;
        }
    }
}

// ------------------------------------------------------------------------------------------
// fused gradient trace over the lower triangle of Kinv (tile-per-CTA):
//   part[tile][p]        = sum_{i>j in tile} A_ij dK_ij/dθ_p + 1/2 sum_{i==j} A_ii dK_ii/dθ_p
//   part[tile][n_theta]  = sum_{i==j} A_ii                      (-> tr(A), dmll_noise GPE.jl:274)
// A_ij = α_i α_j − Kinv_ij  (GPE.jl:151-164).  Kernel derivatives are recomputed from x.
// Reduction order is fixed (lane tree -> warp order -> tile order): bitwise reproducible.
// ------------------------------------------------------------------------------------------
template <bool FAST>
__global__ void __launch_bounds__(NT) trace_kernel(const __grid_constant__ KProg P, const double* __restrict__ x,
                                                   long long ldx, int d, long long N, const double* __restrict__ alpha,
                                                   const double* __restrict__ Kinv, long long ldg,
                                                   double* __restrict__ part, int tiles, int bm_mod, int bm_rem, int bm_div,
                                                   int staged) {
    // triangular tile index
    const int lin = blockIdx.x;
    int bm = (int)((sqrt(8.0 * (double)lin + 1.0) - 1.0) * 0.5);
    while (bm * (bm + 1) / 2 > lin) --bm;
    while ((bm + 1) * (bm + 2) / 2 <= lin) ++bm;
    const int bn = lin - bm * (bm + 1) / 2;
    const int np = P.n_theta;
    if (bm_mod > 1 && ((bm / bm_div) % bm_mod) != bm_rem) {  // tile row owned by another rank
        const int na = FAST ? 3 : np + 1;
        for (int p = threadIdx.x; p < na; p += NT) part[(long long)lin * na + p] = 0.0;
        return;
    }

    extern __shared__ double sm[];
    const int ds = d | 1;
    double* sAi = sm + (staged ? 2 * TB * ds : 0);
    double* sAj = sAi + TB;
    double* sRed = sAj + TB;             // [8 warps][np+1]
    const XTile ti = xtile(staged, sm, x, ldx, d, (long long)bm * TB, N);
    const XTile tj = xtile(staged, sm + TB * ds, x, ldx, d, (long long)bn * TB, N);
    for (int i = threadIdx.x; i < TB; i += NT) {
        const long long gi = (long long)bm * TB + i, gj = (long long)bn * TB + i;
        sAi[i] = gi < N ? alpha[gi] : 0.0;
        sAj[i] = gj < N ? alpha[gj] : 0.0;
    }
    __syncthreads();

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double acc[FAST ? 3 : GPB200_MAX_THETA + 1];
    const int nacc = FAST ? 3 : np + 1;
    for (int p = 0; p < nacc; ++p) acc[p] = 0.0;
    double gbuf[FAST ? 1 : GPB200_MAX_THETA];
    double il2 = 0.0, mh = 0.0, s2 = 0.0;
    if (FAST) { il2 = 1.0 / P.par[0]; mh = -0.5 / P.par[0]; s2 = P.par[1]; }

#pragma unroll 1
    for (int rr = 0; rr < 16; ++rr) {
        const int r = warp * 16 + rr;
        const long long gi = (long long)bm * TB + r;
        if (gi >= N) continue;
        const double* xi = ti.row(r);
        const double ai = sAi[r];
#pragma unroll
        for (int b = 0; b < 2; ++b) {
            const int c0 = b * 64 + lane * 2;
            const long long gj0 = (long long)bn * TB + c0;
            if (gj0 > gi) continue;                       // strictly upper part of a diagonal tile
            const double2 kin = *reinterpret_cast<const double2*>(Kinv + gi * ldg + gj0);
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int c = c0 + e;
                const long long gj = gj0 + e;
                if (gj > gi || gj >= N) continue;
                const double kinv = e ? kin.y : kin.x;
                const double A = ai * sAj[c] - kinv;
                const double w = (gi == gj) ? 0.5 * A : A;
                const double* xj = tj.row(c);
                if (FAST) {
                    double r2 = 0.0;
                    for (int k = 0; k < d; ++k) { const double df = xi[k] - xj[k]; r2 += df * df; }
                    const double kv = s2 * exp(mh * r2);
                    acc[0] += w * (r2 * il2 * kv);        // se_iso.jl:41  dk/dll = r/ℓ² k
                    acc[1] += w * (2.0 * kv);             // stationary.jl:28 dk/dlσ = 2k
                    if (gi == gj) acc[2] += A;
                } else {
                    kprog_eval<true>(P, xi, xj, gbuf);
                    for (int p = 0; p < np; ++p) acc[p] += w * gbuf[p];
                    if (gi == gj) acc[np] += A;
                }
            }
        }
    }
    // lane tree, then fixed warp order
    for (int p = 0; p < nacc; ++p) {
        double v = acc[p];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
        if (lane == 0) sRed[warp * nacc + p] = v;
    }
    __syncthreads();
    for (int p = threadIdx.x; p < nacc; p += NT) {
        double v = 0.0;
        for (int w8 = 0; w8 < NT / 32; ++w8) v += sRed[w8 * nacc + p];
        part[(long long)lin * nacc + p] = v;
    }
}

// out[p] = sum over tiles (fixed-order pairwise tree inside one CTA per p)
__global__ void reduce_partials_kernel(const double* __restrict__ part, int tiles, int nacc, double* __restrict__ out) {
    const int p = blockIdx.x;
    __shared__ double s[256];
    double v = 0.0;
    for (int t = threadIdx.x; t < tiles; t += 256) v += part[(long long)t * nacc + p];
    s[threadIdx.x] = v;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[p] = s[0];
}

// ------------------------------------------------------------------------------------------
// rectangular weighted trace (FITC gradient): part[tile][p] = sum_{i,m in tile} W[i,m] dk(x1_i, x2_m)/dθ_p
// ------------------------------------------------------------------------------------------
template <bool FAST>
__global__ void __launch_bounds__(NT) trace_rect_kernel(const __grid_constant__ KProg P, const double* __restrict__ x1,
                                                        long long ldx1, long long N1, const double* __restrict__ x2,
                                                        long long ldx2, long long N2, int d,
                                                        const double* __restrict__ W, long long ldw,
                                                        double* __restrict__ part, int staged) {
    const int bm = blockIdx.y, bn = blockIdx.x;
    const int np = P.n_theta;
    extern __shared__ double sm[];
    const int ds = d | 1;
    double* sRed = sm + (staged ? 2 * TB * ds : 0);
    const XTile ti = xtile(staged, sm, x1, ldx1, d, (long long)bm * TB, N1);
    const XTile tj = xtile(staged, sm + TB * ds, x2, ldx2, d, (long long)bn * TB, N2);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double acc[FAST ? 2 : GPB200_MAX_THETA];
    const int nacc = FAST ? 2 : np;
    for (int p = 0; p < nacc; ++p) acc[p] = 0.0;
    double gbuf[FAST ? 1 : GPB200_MAX_THETA];
    double il2 = 0.0, mh = 0.0, s2 = 0.0;
    if (FAST) { il2 = 1.0 / P.par[0]; mh = -0.5 / P.par[0]; s2 = P.par[1]; }
#pragma unroll 1
    for (int rr = 0; rr < 16; ++rr) {
        const int r = warp * 16 + rr;
        const long long gi = (long long)bm * TB + r;
        if (gi >= N1) continue;
        const double* xi = ti.row(r);
#pragma unroll
        for (int b = 0; b < 2; ++b) {
            const int c0 = b * 64 + lane * 2;
            const long long gj0 = (long long)bn * TB + c0;
            if (gj0 >= N2) continue;
            const double2 wv = *reinterpret_cast<const double2*>(W + gi * ldw + gj0);
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const long long gj = gj0 + e;
                if (gj >= N2) continue;
                const double w = e ? wv.y : wv.x;
                const double* xj = tj.row(c0 + e);
                if (FAST) {
                    double r2 = 0.0;
                    for (int k = 0; k < d; ++k) { const double df = xi[k] - xj[k]; r2 += df * df; }
                    const double kv = s2 * exp(mh * r2);
                    acc[0] += w * (r2 * il2 * kv);
                    acc[1] += w * (2.0 * kv);
                } else {
                    kprog_eval<true>(P, xi, xj, gbuf);
                    for (int p = 0; p < np; ++p) acc[p] += w * gbuf[p];
                }
            }
        }
    }
    for (int p = 0; p < nacc; ++p) {
        double v = acc[p];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
        if (lane == 0) sRed[warp * nacc + p] = v;
    }
    __syncthreads();
    const long long lin = (long long)blockIdx.y * gridDim.x + blockIdx.x;
    for (int p = threadIdx.x; p < nacc; p += NT) {
        double v = 0.0;
        for (int w8 = 0; w8 < NT / 32; ++w8) v += sRed[w8 * nacc + p];
        part[lin * nacc + p] = v;
    }
}

// out[i*np + p] = g[i] * dk(x_i, x_i)/dθ_p     (diagonal term of the FITC gradient)
__global__ void kdiag_grad_kernel(const __grid_constant__ KProg P, const double* __restrict__ x, long long ldx,
                                  long long N, const double* __restrict__ gvec, double* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    double gbuf[GPB200_MAX_THETA];
    const double* xi = x + i * ldx;
    kprog_eval<true>(P, xi, xi, gbuf);
    const double gi = gvec[i];
    for (int p = 0; p < P.n_theta; ++p) out[(long long)p * N + i] = gi * gbuf[p];
}

// predictive gradients, one CTA per test point m (x* staged in shared memory):
//   dmu[m, :]  = sum_i dk(xs_m, z_i)/dxs_m a_i
//   dvar[m, :] = 2c dk(xs_m, xs_m)/dxs_m - 2 sum_i dk(xs_m, z_i)/dxs_m W[m, i],  W = W1 - W2 (either may be null; both
//   null: dmu only -- the sparse models pass W1 = A L_uu^-1 and W2 = B L_s^-1, SoR only W2)
// Thread t takes i = t, t + DX_NT, ... in order, then every coordinate is summed over the threads by one fixed tree, so a
// row's result does not depend on the launch it belongs to.  The d-vector accumulators are indexed by the leaves' input
// dimensions at run time and live in local memory.
constexpr int DX_NT = 128;
__global__ void __launch_bounds__(DX_NT) crossgram_dx_kernel(const __grid_constant__ KProg P, const double* __restrict__ xs,
                                                             long long ldxs, const double* __restrict__ z, long long ldz,
                                                             long long n, int d, const double* __restrict__ a,
                                                             const double* __restrict__ W1, const double* __restrict__ W2,
                                                             long long ldw, double c,
                                                             double* __restrict__ dmu, double* __restrict__ dvar) {
    __shared__ double sx[GPB200_MAX_DIMS];
    __shared__ double red[DX_NT];
    const long long m = blockIdx.x;
    const int t = threadIdx.x;
    for (int k = t; k < d; k += DX_NT) sx[k] = xs[m * ldxs + k];
    __syncthreads();
    double gm[GPB200_MAX_DIMS], gv[GPB200_MAX_DIMS];
    for (int k = 0; k < d; ++k) { gm[k] = 0.0; gv[k] = 0.0; }
    const bool W = W1 || W2;
    const double* w1 = W1 ? W1 + m * ldw : nullptr;
    const double* w2 = W2 ? W2 + m * ldw : nullptr;
    // the k(x*, x*) term enters thread 0's sum as -c dk(x*, x*)/dx*, so that dvar = -2 (sum)
    if (W && t == 0 && c != 0.0) kprog_eval_dx(P, sx, sx, 0.0, gm, -c, gv);
    for (long long i = t; i < n; i += DX_NT) {
        const double wi = (w1 ? w1[i] : 0.0) - (w2 ? w2[i] : 0.0);
        kprog_eval_dx(P, sx, z + i * ldz, a[i], gm, wi, W ? gv : nullptr);
    }
    for (int k = 0; k < d; ++k) {
        for (int which = 0; which < (W ? 2 : 1); ++which) {
            red[t] = which ? gv[k] : gm[k];
            __syncthreads();
            for (int s = DX_NT / 2; s > 0; s >>= 1) {
                if (t < s) red[t] += red[t + s];
                __syncthreads();
            }
            if (t == 0) {
                if (which) dvar[m * d + k] = -2.0 * red[0];
                else dmu[m * d + k] = red[0];
            }
            __syncthreads();
        }
    }
}

// inducing-point gradient of the sparse mll, one CTA per inducing point j (u_j staged in shared memory):
//   out[j, :] (=, or += when accumulate) sum_i W(i, j) dk(u_j, z_i)/du_j,   W(i, j) = W[i * ldw + j] (+ W[j * ldw + i] if sym)
// W is read in place down column j (the adjoint W_fu of a chunk, Nc x Mpad, or W_uu with sym = W_uu + W_uu').  Rows with
// mask[i] == 0 (FSA padding) are skipped, not weighted by 0.  Thread t takes i = t, t + DX_NT, ... in order and every
// coordinate is summed over the threads by one fixed tree (crossgram_dx_kernel's order), so a launch's sum does not
// depend on the grid; accumulate adds it to out in launch order.
__global__ void __launch_bounds__(DX_NT) inducing_dx_kernel(const __grid_constant__ KProg P, const double* __restrict__ u,
                                                            long long ldu, const double* __restrict__ z, long long ldz,
                                                            long long n, int d, const double* __restrict__ W, long long ldw,
                                                            int sym, const double* __restrict__ mask,
                                                            double* __restrict__ out, int accumulate) {
    __shared__ double su[GPB200_MAX_DIMS];
    __shared__ double red[DX_NT];
    const long long j = blockIdx.x;
    const int t = threadIdx.x;
    for (int k = t; k < d; k += DX_NT) su[k] = u[j * ldu + k];
    __syncthreads();
    double g[GPB200_MAX_DIMS];
    for (int k = 0; k < d; ++k) g[k] = 0.0;
    const double* wc = W + j;
    const double* wr = W + j * ldw;
    for (long long i = t; i < n; i += DX_NT) {
        if (mask && mask[i] == 0.0) continue;
        const double wi = sym ? wc[i * ldw] + wr[i] : wc[i * ldw];
        kprog_eval_dx(P, su, z + i * ldz, wi, g, 0.0, nullptr);
    }
    for (int k = 0; k < d; ++k) {
        red[t] = g[k];
        __syncthreads();
        for (int s = DX_NT / 2; s > 0; s >>= 1) {
            if (t < s) red[t] += red[t + s];
            __syncthreads();
        }
        if (t == 0) out[j * d + k] = accumulate ? out[j * d + k] + red[0] : red[0];
        __syncthreads();
    }
}

// training-input gradient over the stored lower triangle of a symmetric A (A_ij = a_i a_j - G[i * ldg + j], a = alpha or 0
// when alpha is null: A = alpha alpha' - K^-1 after grad_prepare, A = S after gpa_grad), one CTA per IX_PB points p0..:
//   out[i, :] = sum_{j <= i} A_ij d1k(x_i, x_j)  +  sum_{l > i} A_li d1k(x_i, x_l)
// (d1k: derivative in the first argument).  Row part: warp w takes rows p0 + w, p0 + w + 8, ..., its lanes run across the
// columns j <= i of row i (coalesced), then one fixed shuffle tree per coordinate.  Column part: lane t owns column p0 + t,
// warp w walks the rows l = w, w + 8, ... below it (each row's 32 columns are one coalesced read), then the 8 warps are
// summed in warp order.  Both parts of a CTA cover together N entries per point, so the CTAs are balanced although the
// triangle is not.  Only tile rows with ((tile / bm_div) % bm_mod) == bm_rem are read (trace_kernel's ownership); the
// others contribute 0 here and come from the other ranks.  Rows and columns >= N are never read.  Fixed order throughout.
// FAST: the single SEIso leaf with d <= 8, the d-vectors in registers; else kprog_eval_dx with a local-memory d-vector.
constexpr int IX_PB = 32;
template <bool FAST>
__global__ void __launch_bounds__(NT) inputs_dx_kernel(const __grid_constant__ KProg P, const double* __restrict__ x, long long ldx,
                                                       int d, long long N, const double* __restrict__ alpha,
                                                       const double* __restrict__ G, long long ldg, double* __restrict__ out,
                                                       int bm_mod, int bm_rem, int bm_div) {
    constexpr int DR = FAST ? 8 : GPB200_MAX_DIMS;
    __shared__ double red[NT / 32][IX_PB];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long p0 = (long long)blockIdx.x * IX_PB;
    auto owned = [&](long long row) { return bm_mod <= 1 || ((row / TB / bm_div) % bm_mod) == bm_rem; };
    double il2 = 0.0, mh = 0.0, s2 = 0.0;
    if (FAST) { il2 = 1.0 / P.par[0]; mh = -0.5 / P.par[0]; s2 = P.par[1]; }
    double acc[DR];
    const int dk = FAST ? 8 : d;                          // accumulated coordinates (FAST: zero beyond d)
    // A_ij d1k(x_i, x_j) into acc (xi: the point differentiated, xj: the other)
    auto add = [&](const double* xi, const double* xj, double A) {
        if (FAST) {
            double df[8], r2 = 0.0;
#pragma unroll
            for (int k = 0; k < 8; ++k) { df[k] = k < d ? xi[k] - xj[k] : 0.0; r2 += df[k] * df[k]; }
            const double f = -s2 * exp(mh * r2) * il2 * A;
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] += f * df[k];
        } else {
            kprog_eval_dx(P, xi, xj, A, acc, 0.0, nullptr);
        }
    };

    // ---- row part: j <= i in row i
#pragma unroll 1
    for (int rr = warp; rr < IX_PB; rr += NT / 32) {
        const long long i = p0 + rr;
        if (i >= N) break;
#pragma unroll
        for (int k = 0; k < dk; ++k) acc[k] = 0.0;
        if (owned(i)) {
            const double* xi = x + i * ldx;
            double xr[FAST ? 8 : 1];
            if (FAST) {
#pragma unroll
                for (int k = 0; k < 8; ++k) xr[k] = k < d ? xi[k] : 0.0;
            }
            const double ai = alpha ? alpha[i] : 0.0;
            const double* gr = G + i * ldg;
#pragma unroll 1
            for (long long j = lane; j <= i; j += 32) {
                const double A = (alpha ? ai * alpha[j] : 0.0) - gr[j];
                add(FAST ? xr : xi, x + j * ldx, A);
            }
        }
        for (int k = 0; k < dk; ++k) {
            double v = acc[k];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
            if (lane == 0 && k < d) out[i * d + k] = v;
        }
    }

    // ---- column part: l > j in column j = p0 + lane
    const long long j = p0 + lane;
#pragma unroll
    for (int k = 0; k < dk; ++k) acc[k] = 0.0;
    if (j < N) {
        const double* xj = x + j * ldx;
        double xc[FAST ? 8 : 1];
        if (FAST) {
#pragma unroll
            for (int k = 0; k < 8; ++k) xc[k] = k < d ? xj[k] : 0.0;
        }
        const double aj = alpha ? alpha[j] : 0.0;
        for (long long t0 = p0 / TB * TB; t0 < N; t0 += TB) {
            if (!owned(t0)) continue;
            const long long lend = t0 + TB < N ? t0 + TB : N;
#pragma unroll 1
            for (long long l = (t0 > p0 ? t0 : p0) + warp; l < lend; l += NT / 32) {
                if (l <= j) continue;
                const double A = (alpha ? alpha[l] * aj : 0.0) - G[l * ldg + j];
                add(FAST ? xc : xj, x + l * ldx, A);
            }
        }
    }
    __syncthreads();                                      // the row part's out[] stores are visible to the whole CTA
#pragma unroll
    for (int k = 0; k < dk; ++k) {
        if (k >= d) break;                                // uniform: the barriers below are reached by every thread
        red[warp][lane] = acc[k];
        __syncthreads();
        if (warp == 0 && j < N) {
            double v = 0.0;
#pragma unroll
            for (int w = 0; w < NT / 32; ++w) v += red[w][lane];
            out[j * d + k] += v;
        }
        __syncthreads();
    }
}

// training-input gradient of the sparse mll, one warp per training row i (RX_PB rows per CTA):
//   out[row(i), :] (=, or += when accumulate) sum_{j < M} W[i * ldw + j] d1k(x_i, u_j) + 2 c_i d1k(x_i, x_i)
// (d1k: derivative in the first argument; 2 d1k(x, x) is the derivative of k(x, x)).  W is the adjoint W_fu of a chunk
// (row-major, ld Mpad): the lanes run across row i, so its reads are coalesced.  Rows with mask[i] == 0 (FSA padding) are
// skipped, not weighted by 0: their output rows are neither read nor written.  row(i) = map[i] (the caller's order of an FSA
// row) or i.  The c term enters lane 0 before its columns; each coordinate is then reduced by one fixed shuffle tree, so the
// result does not depend on the grid.  FAST: the single SEIso leaf with d <= 8, the d-vectors in registers (its d1k(x, x)
// is 0 and the c term is left out); else kprog_eval_dx with a local-memory d-vector.
constexpr int RX_PB = NT / 32;
template <bool FAST>
__global__ void __launch_bounds__(NT) rows_dx_kernel(const __grid_constant__ KProg P, const double* __restrict__ x, long long ldx,
                                                     long long n, const double* __restrict__ u, long long ldu, long long M, int d,
                                                     const double* __restrict__ W, long long ldw, const double* __restrict__ c,
                                                     const double* __restrict__ mask, const long long* __restrict__ map,
                                                     double* __restrict__ out, int accumulate) {
    constexpr int DR = FAST ? 8 : GPB200_MAX_DIMS;
    const int lane = threadIdx.x & 31;
    const long long i = (long long)blockIdx.x * RX_PB + (threadIdx.x >> 5);
    if (i >= n || (mask && mask[i] == 0.0)) return;      // whole warps: no barrier below
    const int dk = FAST ? 8 : d;
    double acc[DR];
#pragma unroll
    for (int k = 0; k < dk; ++k) acc[k] = 0.0;
    const double* xi = x + i * ldx;
    const double* wr = W + i * ldw;
    if (FAST) {
        const double il2 = 1.0 / P.par[0], mh = -0.5 / P.par[0], s2 = P.par[1];
        double xr[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) xr[k] = k < d ? xi[k] : 0.0;
#pragma unroll 1
        for (long long j = lane; j < M; j += 32) {
            const double* uj = u + j * ldu;
            double df[8], r2 = 0.0;
#pragma unroll
            for (int k = 0; k < 8; ++k) { df[k] = k < d ? xr[k] - uj[k] : 0.0; r2 += df[k] * df[k]; }
            const double f = -s2 * exp(mh * r2) * il2 * wr[j];
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] += f * df[k];
        }
    } else {
        if (c && lane == 0) kprog_eval_dx(P, xi, xi, 2.0 * c[i], acc, 0.0, nullptr);
#pragma unroll 1
        for (long long j = lane; j < M; j += 32) kprog_eval_dx(P, xi, u + j * ldu, wr[j], acc, 0.0, nullptr);
    }
    const long long r = map ? map[i] : i;
#pragma unroll
    for (int k = 0; k < dk; ++k) {
        double v = acc[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
        if (lane == 0 && k < d) out[r * d + k] = accumulate ? out[r * d + k] + v : v;
    }
}

// strict-upper tiles of the Npad x Npad matrix F <- transpose of its strict-lower tiles (diagonal tiles untouched)
__global__ void mirror_lower_tiles_kernel(double* __restrict__ F, long long ld) {
    __shared__ double tl[32][33];
    const int bx = blockIdx.x, by = blockIdx.y;             // 32 x 32 block (by, bx) of the lower source
    if ((bx * 32) / TB >= (by * 32) / TB) return;
    const long long r0 = (long long)by * 32, c0 = (long long)bx * 32;
    for (int r = threadIdx.y; r < 32; r += 8) tl[r][threadIdx.x] = F[(r0 + r) * ld + c0 + threadIdx.x];
    __syncthreads();
    for (int r = threadIdx.y; r < 32; r += 8) F[(c0 + r) * ld + r0 + threadIdx.x] = tl[threadIdx.x][r];
}

size_t xtile_smem(int d) { return (size_t)2 * TB * (d | 1) * sizeof(double); }

// Dynamic shared memory of a tile kernel: the two staged point tiles plus `extra` bytes of scratch when that fits the
// device's opt-in limit per block (staged = 1), else the scratch alone, the points then being read in place (staged = 0).
template <typename K>
cudaError_t tile_smem(K kern, int d, size_t extra, size_t& bytes, int& staged) {
    int dev = 0, optin = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    if (e != cudaSuccess) return e;
    staged = xtile_smem(d) + extra <= (size_t)optin;
    bytes = (staged ? xtile_smem(d) : 0) + extra;
    if (bytes > 48 * 1024) return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    return cudaSuccess;
}

}  // namespace

cudaError_t gram_lower_launch(const KProg& P, const double* x, int64_t ldx, int d, int64_t N, int64_t Npad,
                              const double* noise_var, int64_t n_noise, double nugget, double* G, int64_t ldg,
                              cudaStream_t st, int64_t* launches, int own_tiles, int nranks, int rank, int own_axis, int bm_min) {
    const int T = (int)(Npad / TB);
    if (T <= 0) return cudaSuccess;
    dim3 grid(T, T);
    size_t sm;
    int stg;
    cudaError_t e;
    if (kprog_fast(P, d)) {
        if ((e = tile_smem(gram_lower_kernel<true>, d, 0, sm, stg)) != cudaSuccess) return e;
        gram_lower_kernel<true><<<grid, NT, sm, st>>>(P, x, ldx, d, N, Npad, noise_var, n_noise, nugget, G, ldg, own_tiles, nranks, rank, own_axis, bm_min, stg);
    } else {
        if ((e = tile_smem(gram_lower_kernel<false>, d, 0, sm, stg)) != cudaSuccess) return e;
        gram_lower_kernel<false><<<grid, NT, sm, st>>>(P, x, ldx, d, N, Npad, noise_var, n_noise, nugget, G, ldg, own_tiles, nranks, rank, own_axis, bm_min, stg);
    }
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t crossgram_launch(const KProg& P, const double* xs, int64_t ldxs, int64_t M, int64_t Mpad, const double* x,
                             int64_t ldx, int64_t N, int64_t Npad, int d, double* Kst, int64_t ldk, cudaStream_t st, int64_t* launches) {
    if (Mpad < TB || Npad < TB) return cudaSuccess;
    dim3 grid((unsigned)(Npad / TB), (unsigned)(Mpad / TB));
    size_t sm;
    int stg;
    cudaError_t e;
    if (kprog_fast(P, d)) {
        if ((e = tile_smem(crossgram_kernel<true>, d, 0, sm, stg)) != cudaSuccess) return e;
        crossgram_kernel<true><<<grid, NT, sm, st>>>(P, xs, ldxs, M, x, ldx, N, d, Kst, ldk, stg);
    } else {
        if ((e = tile_smem(crossgram_kernel<false>, d, 0, sm, stg)) != cudaSuccess) return e;
        crossgram_kernel<false><<<grid, NT, sm, st>>>(P, xs, ldxs, M, x, ldx, N, d, Kst, ldk, stg);
    }
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t gram_full_launch(const KProg& P, const double* xs, int64_t ldxs, int64_t M, int64_t Mpad, int d,
                             double* Kss, int64_t ldk, cudaStream_t st, int64_t* launches) {
    if (Mpad < TB) return cudaSuccess;
    dim3 grid((unsigned)(Mpad / TB), (unsigned)(Mpad / TB));
    size_t sm;
    int stg;
    cudaError_t e;
    if (kprog_fast(P, d)) {
        if ((e = tile_smem(gram_full_kernel<true>, d, 0, sm, stg)) != cudaSuccess) return e;
        gram_full_kernel<true><<<grid, NT, sm, st>>>(P, xs, ldxs, M, d, Kss, ldk, stg);
    } else {
        if ((e = tile_smem(gram_full_kernel<false>, d, 0, sm, stg)) != cudaSuccess) return e;
        gram_full_kernel<false><<<grid, NT, sm, st>>>(P, xs, ldxs, M, d, Kss, ldk, stg);
    }
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t kdiag_launch(const KProg& P, const double* xs, int64_t ldxs, int64_t M, double* out, cudaStream_t st, int64_t* launches) {
    if (M <= 0) return cudaSuccess;
    kdiag_kernel<<<(unsigned)((M + 127) / 128), 128, 0, st>>>(P, xs, ldxs, M, out);
    if (launches) ++*launches;
    return cudaGetLastError();
}

int trace_num_acc(const KProg& P, int d) { return kprog_fast(P, d) ? 3 : P.n_theta + 1; }

cudaError_t trace_launch(const KProg& P, const double* x, int64_t ldx, int d, int64_t N, int64_t Npad,
                         const double* alpha, const double* Kinv, int64_t ldg, double* part, double* out,
                         cudaStream_t st, int64_t* launches, int bm_mod, int bm_rem, int bm_div) {
    if (bm_div < 1) bm_div = 1;
    const int T = (int)(Npad / TB);
    const int tiles = T * (T + 1) / 2;
    const int nacc = trace_num_acc(P, d);
    if (tiles <= 0) return cudaMemsetAsync(out, 0, sizeof(double) * nacc, st);
    const size_t extra = (size_t)(2 * TB + 8 * nacc) * sizeof(double);
    size_t sm;
    int stg;
    cudaError_t e;
    if (kprog_fast(P, d)) {
        if ((e = tile_smem(trace_kernel<true>, d, extra, sm, stg)) != cudaSuccess) return e;
        trace_kernel<true><<<tiles, NT, sm, st>>>(P, x, ldx, d, N, alpha, Kinv, ldg, part, tiles, bm_mod, bm_rem, bm_div, stg);
    } else {
        if ((e = tile_smem(trace_kernel<false>, d, extra, sm, stg)) != cudaSuccess) return e;
        trace_kernel<false><<<tiles, NT, sm, st>>>(P, x, ldx, d, N, alpha, Kinv, ldg, part, tiles, bm_mod, bm_rem, bm_div, stg);
    }
    if (launches) ++*launches;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    reduce_partials_kernel<<<nacc, 256, 0, st>>>(part, tiles, nacc, out);
    if (launches) ++*launches;
    return cudaGetLastError();
}

// acc_out[p] += sum over the N1 x N2 rectangle of W[i,m] dk(x1_i,x2_m)/dθ_p ; part: [tiles][n_theta] scratch
cudaError_t trace_rect_launch(const KProg& P, const double* x1, int64_t ldx1, int64_t N1, const double* x2, int64_t ldx2,
                              int64_t N2, int d, const double* W, int64_t ldw, double* part, double* tmp_out,
                              cudaStream_t st, int64_t* launches) {
    const int tm = (int)((N1 + TB - 1) / TB), tn = (int)((N2 + TB - 1) / TB);
    const int nacc = kprog_fast(P, d) ? 2 : P.n_theta;
    if (tm <= 0 || tn <= 0) return cudaMemsetAsync(tmp_out, 0, sizeof(double) * nacc, st);
    const size_t extra = (size_t)(8 * nacc) * sizeof(double);
    dim3 grid(tn, tm);
    size_t sm;
    int stg;
    cudaError_t e;
    if (kprog_fast(P, d)) {
        if ((e = tile_smem(trace_rect_kernel<true>, d, extra, sm, stg)) != cudaSuccess) return e;
        trace_rect_kernel<true><<<grid, NT, sm, st>>>(P, x1, ldx1, N1, x2, ldx2, N2, d, W, ldw, part, stg);
    } else {
        if ((e = tile_smem(trace_rect_kernel<false>, d, extra, sm, stg)) != cudaSuccess) return e;
        trace_rect_kernel<false><<<grid, NT, sm, st>>>(P, x1, ldx1, N1, x2, ldx2, N2, d, W, ldw, part, stg);
    }
    if (launches) ++*launches;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    reduce_partials_kernel<<<nacc, 256, 0, st>>>(part, tm * tn, nacc, tmp_out);
    if (launches) ++*launches;
    return cudaGetLastError();
}
cudaError_t kdiag_grad_launch(const KProg& P, const double* x, int64_t ldx, int64_t N, const double* gvec, double* out,
                              cudaStream_t st, int64_t* launches) {
    if (N <= 0) return cudaSuccess;
    kdiag_grad_kernel<<<(unsigned)((N + 127) / 128), 128, 0, st>>>(P, x, ldx, N, gvec, out);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t gram_grad_full_launch(const KProg& P, const double* x, int64_t ldx, int d, int64_t N, int64_t Npad, int j,
                                  double* D, int64_t ldd, cudaStream_t st, int64_t* launches, int64_t row0, int64_t rows) {
    if (j < 0 || j >= P.n_theta) return cudaErrorInvalidValue;
    if (rows < 0) rows = Npad - row0;
    if (row0 < 0 || row0 % TB || rows % TB || row0 + rows > Npad) return cudaErrorInvalidValue;
    if (rows == 0 || Npad < TB) return cudaSuccess;
    dim3 grid((unsigned)(Npad / TB), (unsigned)(rows / TB));
    size_t sm;
    int stg;
    cudaError_t e;
    if ((e = tile_smem(gram_grad_full_kernel, d, 0, sm, stg)) != cudaSuccess) return e;
    gram_grad_full_kernel<<<grid, NT, sm, st>>>(P, x, ldx, N, d, j, D, ldd, (int)(row0 / TB), stg);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t crossgram_grad_launch(const KProg& P, const double* x1, int64_t ldx1, int64_t N1, int64_t N1pad, const double* x2,
                                  int64_t ldx2, int64_t N2, int64_t N2pad, int d, int j, double* D, int64_t ldd, cudaStream_t st,
                                  int64_t* launches) {
    if (j < 0 || j >= P.n_theta || N1pad % TB || N2pad % TB) return cudaErrorInvalidValue;
    if (N1pad < TB || N2pad < TB) return cudaSuccess;
    dim3 grid((unsigned)(N2pad / TB), (unsigned)(N1pad / TB));
    size_t sm;
    int stg;
    cudaError_t e;
    if ((e = tile_smem(crossgram_grad_kernel, d, 0, sm, stg)) != cudaSuccess) return e;
    crossgram_grad_kernel<<<grid, NT, sm, st>>>(P, x1, ldx1, N1, x2, ldx2, N2, d, j, D, ldd, stg);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t crossgram_dx_launch(const KProg& P, const double* xs, int64_t ldxs, int64_t M, const double* z, int64_t ldz, int64_t n,
                                int d, const double* a, const double* W1, const double* W2, int64_t ldw, double c, double* dmu,
                                double* dvar, cudaStream_t st, int64_t* launches) {
    if (M <= 0) return cudaSuccess;
    if (d <= 0 || d > GPB200_MAX_DIMS || ((W1 || W2) && !dvar)) return cudaErrorInvalidValue;
    crossgram_dx_kernel<<<(unsigned)M, DX_NT, 0, st>>>(P, xs, ldxs, z, ldz, n, d, a, W1, W2, ldw, c, dmu, dvar);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t inducing_dx_launch(const KProg& P, const double* u, int64_t ldu, int64_t M, const double* z, int64_t ldz, int64_t n,
                               int d, const double* W, int64_t ldw, int sym, const double* mask, double* out, int accumulate,
                               cudaStream_t st, int64_t* launches) {
    if (M <= 0) return cudaSuccess;
    if (d <= 0 || d > GPB200_MAX_DIMS || n < 0) return cudaErrorInvalidValue;
    inducing_dx_kernel<<<(unsigned)M, DX_NT, 0, st>>>(P, u, ldu, z, ldz, n, d, W, ldw, sym, mask, out, accumulate);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t inputs_dx_launch(const KProg& P, bool fast, const double* x, int64_t ldx, int d, int64_t N, const double* alpha,
                             const double* G, int64_t ldg, double* out, cudaStream_t st, int64_t* launches, int bm_mod,
                             int bm_rem, int bm_div) {
    if (N <= 0) return cudaSuccess;
    if (d <= 0 || d > GPB200_MAX_DIMS || (fast && (!kprog_fast(P, d) || d > 8))) return cudaErrorInvalidValue;
    if (bm_div < 1) bm_div = 1;
    const unsigned grid = (unsigned)((N + IX_PB - 1) / IX_PB);
    if (fast) inputs_dx_kernel<true><<<grid, NT, 0, st>>>(P, x, ldx, d, N, alpha, G, ldg, out, bm_mod, bm_rem, bm_div);
    else inputs_dx_kernel<false><<<grid, NT, 0, st>>>(P, x, ldx, d, N, alpha, G, ldg, out, bm_mod, bm_rem, bm_div);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t rows_dx_launch(const KProg& P, const double* x, int64_t ldx, int64_t n, const double* u, int64_t ldu, int64_t M, int d,
                           const double* W, int64_t ldw, const double* c, const double* mask, const long long* map, double* out,
                           int accumulate, cudaStream_t st, int64_t* launches) {
    if (n <= 0) return cudaSuccess;
    if (d <= 0 || d > GPB200_MAX_DIMS || M < 0) return cudaErrorInvalidValue;
    const unsigned grid = (unsigned)((n + RX_PB - 1) / RX_PB);
    if (kprog_fast(P, d) && d <= 8) rows_dx_kernel<true><<<grid, NT, 0, st>>>(P, x, ldx, n, u, ldu, M, d, W, ldw, c, mask, map, out, accumulate);
    else rows_dx_kernel<false><<<grid, NT, 0, st>>>(P, x, ldx, n, u, ldu, M, d, W, ldw, c, mask, map, out, accumulate);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t mirror_lower_tiles_launch(double* F, int64_t ld, int64_t Npad, cudaStream_t st, int64_t* launches) {
    if (Npad <= TB) return cudaSuccess;
    dim3 grid((unsigned)(Npad / 32), (unsigned)(Npad / 32)), block(32, 8);
    mirror_lower_tiles_kernel<<<grid, block, 0, st>>>(F, ld);
    if (launches) ++*launches;
    return cudaGetLastError();
}
