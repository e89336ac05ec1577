// fitc_cv.cu -- row kernels of the sparse engine's cross-validation (see fitc_cv.cuh).  The O(N M^2) work of the schedule
// is DMMA GEMMs in fitc_engine.cu; these kernels are the O(N M) per-row epilogues between them.
#include "fitc_cv.cuh"

namespace {

constexpr int WARPS = 8;                       // rows per 256-thread CTA

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__global__ void __launch_bounds__(256) delta_kernel(int kind, const __grid_constant__ KProg P, const double* __restrict__ x,
                                                    long long ldx, int j, const double* __restrict__ G,
                                                    const double* __restrict__ C, long long ld, long long ncols,
                                                    long long nrows, long long rows_pad, const double* __restrict__ alpha,
                                                    double* __restrict__ delta, double* __restrict__ da) {
    const int lane = threadIdx.x & 31;
    const long long i = (long long)blockIdx.x * WARPS + (threadIdx.x >> 5);
    if (i >= rows_pad) return;
    if (i >= nrows) { if (lane == 0) da[i] = 0.0; return; }
    double dl;
    if (kind == 0) {
        const double* g = G + i * ld;
        const double* c = C + i * ld;
        double s = 0.0;
        for (long long m = lane; m < ncols; m += 32) s += g[m] * c[m];
        s = warp_sum(s);
        double dk = 0.0;
        if (lane == 0) {
            double gbuf[GPB200_MAX_THETA];
            const double* xi = x + i * ldx;
            kprog_eval<true>(P, xi, xi, gbuf);
            dk = gbuf[j];
        }
        dl = dk - 2.0 * s;
    } else {
        dl = kind == 1 ? 0.0 : 1.0;
    }
    if (lane == 0) { delta[i] = dl; da[i] = dl * alpha[i]; }
}

__global__ void __launch_bounds__(256) rows_kernel(const double* __restrict__ G, const double* __restrict__ Ch,
                                                   const double* __restrict__ K, const double* __restrict__ P, long long ld,
                                                   long long nrows, long long ncols, const double* __restrict__ lam,
                                                   const double* __restrict__ delta, const double* __restrict__ alpha,
                                                   const double* __restrict__ beta, const double* __restrict__ w,
                                                   double* __restrict__ zja, double* __restrict__ dg) {
    const int lane = threadIdx.x & 31;
    const long long i = (long long)blockIdx.x * WARPS + (threadIdx.x >> 5);
    if (i >= nrows) return;
    const double* c = Ch + i * ld;
    const double* k = K + i * ld;
    const double* p = P + i * ld;
    double gb = 0.0, cw = 0.0, gc = 0.0, kc = 0.0, pc = 0.0;
    if (G) {
        const double* g = G + i * ld;
        for (long long m = lane; m < ncols; m += 32) {
            const double cm = c[m], gm = g[m];
            gb += gm * beta[m]; gc += gm * cm;
            cw += cm * w[m]; kc += k[m] * cm; pc += p[m] * cm;
        }
    } else {
        for (long long m = lane; m < ncols; m += 32) {
            const double cm = c[m];
            cw += cm * w[m]; kc += k[m] * cm; pc += p[m] * cm;
        }
    }
    gb = warp_sum(gb); cw = warp_sum(cw); gc = warp_sum(gc); kc = warp_sum(kc); pc = warp_sum(pc);
    if (lane == 0) {
        const double il = 1.0 / lam[i], dl = delta[i];
        zja[i] = dl * alpha[i] * il + gb * il + cw;
        dg[i] = dl * il * il + 2.0 * gc * il - 2.0 * dl * kc * il * il + pc;
    }
}

__global__ void invdiag_kernel(long long n, const double* __restrict__ lam, const double* __restrict__ q, double* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { const double il = 1.0 / lam[i]; out[i] = il - q[i] * il * il; }
}

__global__ void eblock_kernel(double* __restrict__ E, const double* __restrict__ G, const double* __restrict__ K, long long ld,
                              long long nrows, long long ncols, const double* __restrict__ lam, const double* __restrict__ delta) {
    const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long i = blockIdx.y;
    if (m >= ncols || i >= nrows) return;
    const double il = 1.0 / lam[i];
    const long long o = i * ld + m;
    E[o] += (G ? G[o] * il : 0.0) - delta[i] * K[o] * il * il;
}

__global__ void qs_kernel(double* __restrict__ Q, const double* __restrict__ H, const double* __restrict__ R, long long ld, long long n) {
    const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long r = blockIdx.y;
    if (c < n && r < n) Q[r * ld + c] = H[r * ld + c] - R[r * ld + c] - R[c * ld + r];
}

__global__ void wvec_kernel(long long n, double* __restrict__ w, const double* __restrict__ a, const double* __restrict__ b,
                            const double* __restrict__ c) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) w[i] = a[i] - b[i] - c[i];
}

__global__ void gather_kernel(long long nv, const long long* __restrict__ idx, const double* __restrict__ x, long long ldx, int d,
                              double* __restrict__ xout, const double* __restrict__ lam, double* __restrict__ lamout,
                              const double* __restrict__ delta, double* __restrict__ delout) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nv) return;
    const long long s = idx[r];
    for (int k = 0; k < d; ++k) xout[r * d + k] = x[s * ldx + k];
    lamout[r] = lam[s];
    if (delta) delout[r] = delta[s];
}

__global__ void diag_kernel(double* __restrict__ out, long long ld, long long nv, int which, const double* __restrict__ lam,
                            const double* __restrict__ delta) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nv) return;
    const double il = 1.0 / lam[r];
    out[r * ld + r] += which == 0 ? il : delta[r] * il * il;
}

inline unsigned blocks(long long n, int per) { return (unsigned)((n + per - 1) / per); }

}  // namespace

cudaError_t fitc_cv_delta_launch(int kind, const KProg& P, const double* x, int64_t ldx, int j, const double* G, const double* C,
                                 int64_t ld, int64_t ncols, int64_t nrows, int64_t rows_pad, const double* alpha, double* delta,
                                 double* da, cudaStream_t st, int64_t* launches) {
    if (rows_pad <= 0) return cudaSuccess;
    delta_kernel<<<blocks(rows_pad, WARPS), 256, 0, st>>>(kind, P, x, ldx, j, G, C, ld, ncols, nrows, rows_pad, alpha, delta, da);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t fitc_cv_rows_launch(const double* G, const double* Ch, const double* K, const double* P, int64_t ld, int64_t nrows,
                                int64_t ncols, const double* lam, const double* delta, const double* alpha, const double* beta,
                                const double* w, double* zja, double* dg, cudaStream_t st, int64_t* launches) {
    if (nrows <= 0) return cudaSuccess;
    rows_kernel<<<blocks(nrows, WARPS), 256, 0, st>>>(G, Ch, K, P, ld, nrows, ncols, lam, delta, alpha, beta, w, zja, dg);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t fitc_cv_invdiag_launch(int64_t n, const double* lam, const double* q, double* out, cudaStream_t st, int64_t* launches) {
    if (n <= 0) return cudaSuccess;
    invdiag_kernel<<<blocks(n, 256), 256, 0, st>>>(n, lam, q, out);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t fitc_cv_eblock_launch(double* E, const double* G, const double* K, int64_t ld, int64_t nrows, int64_t ncols,
                                  const double* lam, const double* delta, cudaStream_t st, int64_t* launches) {
    if (nrows <= 0 || ncols <= 0) return cudaSuccess;
    dim3 grid(blocks(ncols, 256), (unsigned)nrows);
    eblock_kernel<<<grid, 256, 0, st>>>(E, G, K, ld, nrows, ncols, lam, delta);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t fitc_cv_qs_launch(double* Q, const double* H, const double* R, int64_t ld, int64_t n, cudaStream_t st, int64_t* launches) {
    if (n <= 0) return cudaSuccess;
    dim3 grid(blocks(n, 256), (unsigned)n);
    qs_kernel<<<grid, 256, 0, st>>>(Q, H, R, ld, n);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t fitc_cv_wvec_launch(int64_t n, double* w, const double* a, const double* b, const double* c, cudaStream_t st,
                                int64_t* launches) {
    if (n <= 0) return cudaSuccess;
    wvec_kernel<<<blocks(n, 256), 256, 0, st>>>(n, w, a, b, c);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t fitc_cv_gather_launch(int64_t nv, const long long* idx, const double* x, int64_t ldx, int d, double* xout,
                                  const double* lam, double* lamout, const double* delta, double* delout, cudaStream_t st,
                                  int64_t* launches) {
    if (nv <= 0) return cudaSuccess;
    gather_kernel<<<blocks(nv, 256), 256, 0, st>>>(nv, idx, x, ldx, d, xout, lam, lamout, delta, delout);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t fitc_cv_diag_launch(double* out, int64_t ld, int64_t nv, int which, const double* lam, const double* delta,
                                cudaStream_t st, int64_t* launches) {
    if (nv <= 0) return cudaSuccess;
    diag_kernel<<<blocks(nv, 256), 256, 0, st>>>(out, ld, nv, which, lam, delta);
    if (launches) ++*launches;
    return cudaGetLastError();
}
