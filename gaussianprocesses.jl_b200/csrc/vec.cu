// vec.cu -- bandwidth-bound helpers around the factor.
//
//  * trsv_lower_fwd / trsv_lower_bwd : alpha = K_y \ r  == dpotrs with one right-hand side
//    (/root/reference/src/GPE.jl:208, PDMats `\`).  Blocked by the 128-wide tiles of the factor:
//    step i multiplies the inverted diagonal tile (Dinv, produced by the Cholesky leaf kernel) and
//    immediately applies the 128-column panel update to the remaining right-hand side, one launch
//    per block step (every CTA recomputes the 128-vector y_i instead of waiting on a second kernel).
//    Out of place: the solution blocks go to a separate vector so that no CTA writes a block other
//    CTAs of the same launch still read.
//  * fixed-order reductions (dot, sum) so that mll / logdet are bitwise reproducible.
//  * predictive mean / variance epilogues (/root/reference/src/GP.jl:26, 51-54, 75).
#include "devbuf.cuh"
#include "vec.cuh"
#include <math.h>

namespace {
constexpr int T = 128;

// out[r] = sum_c M[r*ld + c] * v[c]   (128x128 tile, 256 threads, v/out in shared memory)
__device__ __forceinline__ void tile_matvec(const double* __restrict__ M, long long ld, const double* v, double* out) {
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    const double v0 = v[l], v1 = v[l + 32], v2 = v[l + 64], v3 = v[l + 96];
#pragma unroll 4
    for (int rr = 0; rr < 16; ++rr) {
        const int r = w * 16 + rr;
        const double* row = M + (long long)r * ld;
        double s = row[l] * v0 + row[l + 32] * v1 + row[l + 64] * v2 + row[l + 96] * v3;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (l == 0) out[r] = s;
    }
}
// out[c] = sum_r M[r*ld + c] * v[r]   (transposed), 256 threads: two row halves combined in smem
__device__ __forceinline__ void tile_matvec_t(const double* __restrict__ M, long long ld, const double* v, double* out, double* scratch) {
    const int c = threadIdx.x & 127, h = threadIdx.x >> 7;
    double s = 0.0;
#pragma unroll 8
    for (int r = h * 64; r < h * 64 + 64; ++r) s += M[(long long)r * ld + c] * v[r];
    if (h == 1) scratch[c] = s;
    __syncthreads();
    if (h == 0) out[c] = s + scratch[c];
}

__global__ void __launch_bounds__(256) trsv_fwd_step(const double* __restrict__ F, long long ldf, const double* __restrict__ Dinv,
                                                      double* __restrict__ r, double* __restrict__ yout, int i) {
    __shared__ double sr[T], sy[T], so[T];
    const long long p = (long long)i * T;
    if (threadIdx.x < T) sr[threadIdx.x] = r[p + threadIdx.x];
    __syncthreads();
    tile_matvec(Dinv + p * T, T, sr, sy);
    __syncthreads();
    const int b = blockIdx.x;
    if (b == 0) { if (threadIdx.x < T) yout[p + threadIdx.x] = sy[threadIdx.x]; return; }
    const long long q = (long long)(i + b) * T;
    tile_matvec(F + q * ldf + p, ldf, sy, so);
    __syncthreads();
    if (threadIdx.x < T) r[q + threadIdx.x] -= so[threadIdx.x];
}

__global__ void __launch_bounds__(256) trsv_bwd_step(const double* __restrict__ F, long long ldf, const double* __restrict__ DinvT,
                                                      double* __restrict__ z, double* __restrict__ aout, int i) {
    __shared__ double sz[T], sa[T], so[T], sc[T];
    const long long p = (long long)i * T;
    if (threadIdx.x < T) sz[threadIdx.x] = z[p + threadIdx.x];
    __syncthreads();
    tile_matvec(DinvT + p * T, T, sz, sa);         // a_i = W_ii' z_i
    __syncthreads();
    const int b = blockIdx.x;
    if (b == 0) { if (threadIdx.x < T) aout[p + threadIdx.x] = sa[threadIdx.x]; return; }
    const long long q = (long long)(b - 1) * T;    // column block q < i
    tile_matvec_t(F + p * ldf + q, ldf, sa, so, sc);   // L[i-block, q-block]' a_i
    __syncthreads();
    if (threadIdx.x < T) z[q + threadIdx.x] -= so[threadIdx.x];
}

__global__ void __launch_bounds__(1024) dot_kernel(const double* __restrict__ a, const double* __restrict__ b, long long n, double* __restrict__ out) {
    __shared__ double s[1024];
    double v = 0.0;
    for (long long i = threadIdx.x; i < n; i += 1024) v += a[i] * b[i];
    s[threadIdx.x] = v;
    __syncthreads();
    for (int o = 512; o > 0; o >>= 1) { if (threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) out[0] = s[0];
}
__global__ void __launch_bounds__(1024) sum_kernel(const double* __restrict__ a, long long n, double* __restrict__ out) {
    __shared__ double s[1024];
    double v = 0.0;
    for (long long i = threadIdx.x; i < n; i += 1024) v += a[i];
    s[threadIdx.x] = v;
    __syncthreads();
    for (int o = 512; o > 0; o >>= 1) { if (threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) out[0] = s[0];
}

// one CTA (256 threads) per row
__global__ void __launch_bounds__(256) rowdot_kernel(const double* __restrict__ K, long long ldk, const double* __restrict__ alpha,
                                                     long long N, double* __restrict__ mu) {
    __shared__ double s[256];
    const double* row = K + (long long)blockIdx.x * ldk;
    double v = 0.0;
    for (long long n = threadIdx.x; n < N; n += 256) v += row[n] * alpha[n];
    s[threadIdx.x] = v;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) { if (threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) mu[blockIdx.x] = s[0];
}
__global__ void __launch_bounds__(256) rowvar_kernel(const double* __restrict__ V, long long ldk, const double* __restrict__ kdiag,
                                                     long long N, double* __restrict__ var) {
    __shared__ double s[256];
    const double* row = V + (long long)blockIdx.x * ldk;
    double v = 0.0;
    for (long long n = threadIdx.x; n < N; n += 256) { const double t = row[n]; v += t * t; }
    s[threadIdx.x] = v;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) { if (threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) var[blockIdx.x] = kdiag[blockIdx.x] - s[0];
}
__global__ void exp2x_kernel(const double* __restrict__ ln, long long n, double* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = exp(2.0 * ln[i]);
}
}  // namespace

// ---- FP64 pipe calibration (roofline denominator): DMMA.16x8x16 (the GEMM's shape) / DFMA issue rates from registers ----
namespace {
__global__ void dmma_peak_kernel(double* out, int iters) {
    double c[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { c[i][0] = 0.0; c[i][1] = 0.0; c[i][2] = 0.0; c[i][3] = 0.0; }
    const double a = threadIdx.x * 1e-3, b = 1.0 + threadIdx.x * 1e-4;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 8; ++i)
            asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%4,%4,%4,%4,%4,%4,%4}, "
                         "{%5,%5,%5,%5}, {%0,%1,%2,%3};"
                         : "+d"(c[i][0]), "+d"(c[i][1]), "+d"(c[i][2]), "+d"(c[i][3]) : "d"(a), "d"(b));
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += c[i][0] + c[i][1] + c[i][2] + c[i][3];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
__global__ void dfma_peak_kernel(double* out, int iters) {
    double c[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) c[i] = i;
    const double a = 1.0 + threadIdx.x * 1e-9, b = 1e-9;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 16; ++i) c[i] = fma(c[i], a, b);
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < 16; ++i) s += c[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
}  // namespace

cudaError_t fp64_peak_measure(cudaStream_t st, int64_t* launches, double* tflops) {
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int warps = 8, iters = 10000;
    DevBuf<double> out;
    const cudaError_t e = out.alloc((size_t)sms * warps * 32);
    if (e != cudaSuccess) return e;
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    float best[2] = {1e30f, 1e30f};
    for (int rep = 0; rep < 3; ++rep) {
        cudaEventRecord(e0, st);
        dmma_peak_kernel<<<sms, warps * 32, 0, st>>>(out, iters);
        if (launches) ++*launches;
        cudaEventRecord(e1, st); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1); if (rep && ms < best[0]) best[0] = ms;
        cudaEventRecord(e0, st);
        dfma_peak_kernel<<<sms, warps * 32, 0, st>>>(out, iters);
        if (launches) ++*launches;
        cudaEventRecord(e1, st); cudaEventSynchronize(e1);
        cudaEventElapsedTime(&ms, e0, e1); if (rep && ms < best[1]) best[1] = ms;
    }
    tflops[0] = 2.0 * 2048 * 8.0 * iters * warps * sms / best[0] * 1e-9;    // 8 x (16*8*16 FMA) per warp and iteration
    tflops[1] = 2.0 * 32 * 16.0 * iters * warps * sms / best[1] * 1e-9;
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    out.reset();
    return cudaGetLastError();
}

// ---- small elementwise kernels used by the FITC path ----
namespace {
// op: 0 out=a+s  1 out=a/b  2 out+=a  3 out=(a-b)/c  4 out=log(a)  5 out=1/a  6 out=a-b
__global__ void ew_kernel(int op, long long n, double* __restrict__ out, const double* __restrict__ a,
                          const double* __restrict__ b, const double* __restrict__ c, double s) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    switch (op) {
    case 0: out[i] = a[i] + s; break;
    case 1: out[i] = a[i] / b[i]; break;
    case 2: out[i] += a[i]; break;
    case 3: out[i] = (a[i] - b[i]) / c[i]; break;
    case 4: out[i] = log(a[i]); break;
    case 5: out[i] = 1.0 / a[i]; break;
    case 6: out[i] = a[i] - b[i]; break;
    }
}
// A[r, j] *= f(v[j]) for j < ncols (mode 0: 1/sqrt(v), columns) ; A[r, :] *= 1/v[r] for r < nrows (mode 1, rows)
__global__ void scale_kernel(int mode, double* __restrict__ A, long long ld, long long nrows, long long ncols,
                             const double* __restrict__ v) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long r = blockIdx.y;
    if (j >= ncols || r >= nrows) return;
    const double f = mode == 0 ? 1.0 / sqrt(v[j]) : 1.0 / v[r];
    A[r * ld + j] *= f;
}
}  // namespace
namespace {
// q[r] = sum_c A[r,c] * B[r,c]
__global__ void __launch_bounds__(256) rowdot2_kernel(const double* __restrict__ A, const double* __restrict__ B, long long ld,
                                                      long long ncols, double* __restrict__ q) {
    __shared__ double s[256];
    const double* ra = A + (long long)blockIdx.x * ld;
    const double* rb = B + (long long)blockIdx.x * ld;
    double v = 0.0;
    for (long long c = threadIdx.x; c < ncols; c += 256) v += ra[c] * rb[c];
    s[threadIdx.x] = v;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) { if (threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) q[blockIdx.x] = s[0];
}
// g[i] = alpha_i^2 - (1/lam_i - q_i/lam_i^2)
__global__ void fitc_g_kernel(long long n, const double* __restrict__ alpha, const double* __restrict__ lam,
                              const double* __restrict__ q, double* __restrict__ g) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { const double il = 1.0 / lam[i]; g[i] = alpha[i] * alpha[i] - (il - q[i] * il * il); }
}
// P2[i,m] <- 2 alpha_i beta_m - (2/lam_i) P2[i,m] - 2 g_i P1[i,m]      (W_fu, in place on P2)
__global__ void fitc_wfu_kernel(double* __restrict__ P2, const double* __restrict__ P1, long long ld, long long nrows,
                                long long ncols, const double* __restrict__ alpha, const double* __restrict__ lam,
                                const double* __restrict__ g, const double* __restrict__ beta) {
    const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long i = blockIdx.y;
    if (m >= ncols || i >= nrows) return;
    const long long o = i * ld + m;
    P2[o] = 2.0 * alpha[i] * beta[m] - (2.0 / lam[i]) * P2[o] - 2.0 * g[i] * P1[o];
}
// A[r, j] *= v[j] (j < ncols)
__global__ void colscale_kernel(double* __restrict__ A, long long ld, long long nrows, long long ncols, const double* __restrict__ v) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long r = blockIdx.y;
    if (j < ncols && r < nrows) A[r * ld + j] *= v[j];
}
// mirror the lower triangle of an n x n matrix into its upper triangle
__global__ void symmetrize_kernel(double* __restrict__ A, long long ld, long long n) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long i = blockIdx.y;
    if (i < n && j < n && j > i) A[i * ld + j] = A[j * ld + i];
}
// Wuu[m,n] = T[m,n] - beta_m beta_n + Kinv[m,n] - Sinv[m,n]
__global__ void fitc_wuu_kernel(double* __restrict__ Wuu, const double* __restrict__ T, const double* __restrict__ Kinv,
                                const double* __restrict__ Sinv, long long ld, long long n, const double* __restrict__ beta) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long i = blockIdx.y;
    if (i < n && j < n) Wuu[i * ld + j] = T[i * ld + j] - beta[i] * beta[j] + Kinv[i * ld + j] - Sinv[i * ld + j];
}
}  // namespace
cudaError_t rowdot2_launch(const double* A, const double* B, int64_t ld, int64_t nrows, int64_t ncols, double* q, cudaStream_t st, int64_t* launches) {
    if (nrows <= 0) return cudaSuccess;
    rowdot2_kernel<<<(unsigned)nrows, 256, 0, st>>>(A, B, ld, ncols, q);
    if (launches) ++*launches;
    return cudaGetLastError();
}
cudaError_t fitc_g_launch(int64_t n, const double* alpha, const double* lam, const double* q, double* g, cudaStream_t st, int64_t* launches) {
    if (n <= 0) return cudaSuccess;
    fitc_g_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(n, alpha, lam, q, g);
    if (launches) ++*launches;
    return cudaGetLastError();
}
cudaError_t fitc_wfu_launch(double* P2, const double* P1, int64_t ld, int64_t nrows, int64_t ncols, const double* alpha,
                            const double* lam, const double* g, const double* beta, cudaStream_t st, int64_t* launches) {
    if (nrows <= 0 || ncols <= 0) return cudaSuccess;
    dim3 grid((unsigned)((ncols + 255) / 256), (unsigned)nrows);
    fitc_wfu_kernel<<<grid, 256, 0, st>>>(P2, P1, ld, nrows, ncols, alpha, lam, g, beta);
    if (launches) ++*launches;
    return cudaGetLastError();
}
cudaError_t colscale_launch(double* A, int64_t ld, int64_t nrows, int64_t ncols, const double* v, cudaStream_t st, int64_t* launches) {
    if (nrows <= 0 || ncols <= 0) return cudaSuccess;
    dim3 grid((unsigned)((ncols + 255) / 256), (unsigned)nrows);
    colscale_kernel<<<grid, 256, 0, st>>>(A, ld, nrows, ncols, v);
    if (launches) ++*launches;
    return cudaGetLastError();
}
cudaError_t symmetrize_launch(double* A, int64_t ld, int64_t n, cudaStream_t st, int64_t* launches) {
    if (n <= 0) return cudaSuccess;
    dim3 grid((unsigned)((n + 255) / 256), (unsigned)n);
    symmetrize_kernel<<<grid, 256, 0, st>>>(A, ld, n);
    if (launches) ++*launches;
    return cudaGetLastError();
}
cudaError_t fitc_wuu_launch(double* Wuu, const double* T, const double* Kinv, const double* Sinv, int64_t ld, int64_t n,
                            const double* beta, cudaStream_t st, int64_t* launches) {
    if (n <= 0) return cudaSuccess;
    dim3 grid((unsigned)((n + 255) / 256), (unsigned)n);
    fitc_wuu_kernel<<<grid, 256, 0, st>>>(Wuu, T, Kinv, Sinv, ld, n, beta);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t ew_launch(int op, int64_t n, double* out, const double* a, const double* b, const double* c, double s, cudaStream_t st, int64_t* launches) {
    if (n <= 0) return cudaSuccess;
    ew_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(op, n, out, a, b, c, s);
    if (launches) ++*launches;
    return cudaGetLastError();
}
cudaError_t scale_launch(int mode, double* A, int64_t ld, int64_t nrows, int64_t ncols, const double* v, cudaStream_t st, int64_t* launches) {
    if (nrows <= 0 || ncols <= 0) return cudaSuccess;
    dim3 grid((unsigned)((ncols + 255) / 256), (unsigned)nrows);
    scale_kernel<<<grid, 256, 0, st>>>(mode, A, ld, nrows, ncols, v);
    if (launches) ++*launches;
    return cudaGetLastError();
}

// ---- single-launch ("sync-free") triangular solves -------------------------------------------------
// One CTA per 128-row block; CTA b consumes the solution blocks y_i (i < b) as their ready-flags appear, then publishes y_b.
// The two tiles on the critical chain are RESIDENT before the CTA starts waiting: the inverted diagonal tile in registers
// (each thread keeps exactly the 16 x 4 entries its part of the tile mat-vec uses) and the neighbour tile L[b, b-1]
// (forward) / L[b+1, b] (backward) in shared memory.  Per block step the chain is then: flag -> 1 KB vector -> mat-vec out
// of shared memory -> mat-vec out of registers -> flag, instead of two 128 KB tile reads from L2 (19 us per step with the
// tiles only prefetched to L2).  128 KB of dynamic shared memory per CTA: one CTA per SM; later CTAs start as earlier ones
// retire, dependencies only point to lower blockIdx (in-order dispatch).  A watchdog turns a missing flag into an error
// code instead of a hang.
namespace {
__device__ __forceinline__ int ld_acquire(const int* p) {
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release(int* p, int v) {
    asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ bool wait_flag(const int* flag, int* err) {
    long long spins = 0;
    while (ld_acquire(flag) == 0) {
        if (++spins > (1LL << 26)) { atomicExch(err, 1); return false; }
        __nanosleep(20);
    }
    return true;
}

__device__ __forceinline__ void load_tile_regs(const double* __restrict__ M, long long ld, double (&t)[16][4]) {
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
#pragma unroll
    for (int rr = 0; rr < 16; ++rr) {
        const double* row = M + (long long)(w * 16 + rr) * ld;
        t[rr][0] = row[l]; t[rr][1] = row[l + 32]; t[rr][2] = row[l + 64]; t[rr][3] = row[l + 96];
    }
}
__device__ __forceinline__ void tile_matvec_regs(const double (&t)[16][4], const double* v, double* out) {
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    const double v0 = v[l], v1 = v[l + 32], v2 = v[l + 64], v3 = v[l + 96];
#pragma unroll
    for (int rr = 0; rr < 16; ++rr) {
        double s = t[rr][0] * v0 + t[rr][1] * v1 + t[rr][2] * v2 + t[rr][3] * v3;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (l == 0) out[w * 16 + rr] = s;
    }
}
__device__ __forceinline__ void stage_tile_smem(double* dst, const double* __restrict__ M, long long ld) {
    // 128 x 128 tile, row-major in shared memory with the same 128-double pitch (rows are read by consecutive lanes)
    for (int idx = threadIdx.x; idx < T * T / 2; idx += blockDim.x) {
        const int r = idx >> 6, c2 = (idx & 63) * 2;
        *reinterpret_cast<double2*>(dst + r * T + c2) = *reinterpret_cast<const double2*>(M + (long long)r * ld + c2);
    }
}

__global__ void __launch_bounds__(256, 1) trsv_fwd_persistent2(const double* __restrict__ F, long long ldf, const double* __restrict__ Dinv,
                                                               const double* __restrict__ r, double* __restrict__ y,
                                                               int* __restrict__ flags, int* __restrict__ err) {
    extern __shared__ __align__(16) double sTile[];            // L[b, b-1]
    __shared__ double sAcc[T], sY[T], sO[T];
    __shared__ int ok;
    const int b = blockIdx.x;
    const long long q = (long long)b * T;
    double dreg[16][4];
    load_tile_regs(Dinv + q * T, T, dreg);
    if (b > 0) stage_tile_smem(sTile, F + q * ldf + (q - T), ldf);
    if (threadIdx.x < T) sAcc[threadIdx.x] = r[q + threadIdx.x];
    __syncthreads();
    for (int i = 0; i < b; ++i) {
        if (threadIdx.x == 0) ok = wait_flag(flags + i, err) ? 1 : 0;
        __syncthreads();
        if (!ok) return;
        if (threadIdx.x < T) sY[threadIdx.x] = __ldcg(y + (long long)i * T + threadIdx.x);
        __syncthreads();
        if (i == b - 1) tile_matvec(sTile, T, sY, sO);
        else tile_matvec(F + q * ldf + (long long)i * T, ldf, sY, sO);
        __syncthreads();
        if (threadIdx.x < T) sAcc[threadIdx.x] -= sO[threadIdx.x];
        __syncthreads();
    }
    tile_matvec_regs(dreg, sAcc, sO);                         // y_b = W_bb (r_b - sum_i L_bi y_i)
    __syncthreads();
    if (threadIdx.x < T) y[q + threadIdx.x] = sO[threadIdx.x];
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) st_release(flags + b, 1);
}

__global__ void __launch_bounds__(256, 1) trsv_bwd_persistent2(const double* __restrict__ F, long long ldf, const double* __restrict__ DinvT,
                                                               const double* __restrict__ z, double* __restrict__ a,
                                                               int* __restrict__ flags, int* __restrict__ err, int nb) {
    extern __shared__ __align__(16) double sTile[];            // L[b+1, b]
    __shared__ double sAcc[T], sA[T], sO[T], sC[T];
    __shared__ int ok;
    const int b = nb - 1 - blockIdx.x;                     // dependencies (blocks > b) have lower blockIdx
    const long long q = (long long)b * T;
    double dreg[16][4];
    load_tile_regs(DinvT + q * T, T, dreg);
    if (b + 1 < nb) stage_tile_smem(sTile, F + (q + T) * ldf + q, ldf);
    if (threadIdx.x < T) sAcc[threadIdx.x] = z[q + threadIdx.x];
    __syncthreads();
    for (int i = nb - 1; i > b; --i) {
        if (threadIdx.x == 0) ok = wait_flag(flags + i, err) ? 1 : 0;
        __syncthreads();
        if (!ok) return;
        if (threadIdx.x < T) sA[threadIdx.x] = __ldcg(a + (long long)i * T + threadIdx.x);
        __syncthreads();
        if (i == b + 1) tile_matvec_t(sTile, T, sA, sO, sC);
        else tile_matvec_t(F + (long long)i * T * ldf + q, ldf, sA, sO, sC);     // L[i-block, b-block]' a_i
        __syncthreads();
        if (threadIdx.x < T) sAcc[threadIdx.x] -= sO[threadIdx.x];
        __syncthreads();
    }
    tile_matvec_regs(dreg, sAcc, sO);                         // a_b = W_bb' (z_b - sum_i L_ib' a_i)
    __syncthreads();
    if (threadIdx.x < T) a[q + threadIdx.x] = sO[threadIdx.x];
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) st_release(flags + b, 1);
}
bool g_trsv_attr = false;

cudaError_t trsv_set_smem_attr() {
    if (g_trsv_attr) return cudaSuccess;
    const int bytes = (int)(sizeof(double) * T * T);
    cudaError_t e = cudaFuncSetAttribute(trsv_fwd_persistent2, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(trsv_bwd_persistent2, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) g_trsv_attr = true;
    return e;
}
}  // namespace

// flags: int[Npad/128 + 1] scratch (last entry = watchdog error flag); returns cudaErrorLaunchFailure-free:
// the caller reads flags[nb] after the stream sync.
cudaError_t trsv_lower_fwd_fused(const double* F, int64_t ldf, const double* Dinv, const double* r, double* y, int64_t Npad,
                                 int* flags, cudaStream_t st, int64_t* launches) {
    const int nb = (int)(Npad / T);
    cudaError_t e = trsv_set_smem_attr();
    if (e != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(flags, 0, sizeof(int) * (nb + 1), st)) != cudaSuccess) return e;
    trsv_fwd_persistent2<<<nb, 256, sizeof(double) * T * T, st>>>(F, ldf, Dinv, r, y, flags, flags + nb);
    if (launches) ++*launches;
    return cudaGetLastError();
}
cudaError_t trsv_lower_bwd_fused(const double* F, int64_t ldf, const double* DinvT, const double* z, double* a, int64_t Npad,
                                 int* flags, cudaStream_t st, int64_t* launches) {
    const int nb = (int)(Npad / T);
    cudaError_t e = trsv_set_smem_attr();
    if (e != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(flags, 0, sizeof(int) * (nb + 1), st)) != cudaSuccess) return e;
    trsv_bwd_persistent2<<<nb, 256, sizeof(double) * T * T, st>>>(F, ldf, DinvT, z, a, flags, flags + nb, nb);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t trsv_lower_fwd(const double* F, int64_t ldf, const double* Dinv, double* r, double* y, int64_t Npad,
                           cudaStream_t st, int64_t* launches) {
    const int nb = (int)(Npad / T);
    for (int i = 0; i < nb; ++i) {
        trsv_fwd_step<<<nb - i, 256, 0, st>>>(F, ldf, Dinv, r, y, i);
        if (launches) ++*launches;
    }
    return cudaGetLastError();
}
cudaError_t trsv_lower_bwd(const double* F, int64_t ldf, const double* DinvT, double* z, double* a, int64_t Npad,
                           cudaStream_t st, int64_t* launches) {
    const int nb = (int)(Npad / T);
    for (int i = nb - 1; i >= 0; --i) {
        trsv_bwd_step<<<i + 1, 256, 0, st>>>(F, ldf, DinvT, z, a, i);
        if (launches) ++*launches;
    }
    return cudaGetLastError();
}
cudaError_t dot_launch(const double* a, const double* b, int64_t n, double* out, cudaStream_t st, int64_t* launches) {
    dot_kernel<<<1, 1024, 0, st>>>(a, b, n, out);
    if (launches) ++*launches;
    return cudaGetLastError();
}
cudaError_t sum_launch(const double* a, int64_t n, double* out, cudaStream_t st, int64_t* launches) {
    sum_kernel<<<1, 1024, 0, st>>>(a, n, out);
    if (launches) ++*launches;
    return cudaGetLastError();
}
cudaError_t rowdot_launch(const double* Kst, int64_t ldk, const double* alpha, int64_t M, int64_t N, double* mu, cudaStream_t st, int64_t* launches) {
    if (M <= 0) return cudaSuccess;
    rowdot_kernel<<<(unsigned)M, 256, 0, st>>>(Kst, ldk, alpha, N, mu);
    if (launches) ++*launches;
    return cudaGetLastError();
}
cudaError_t rowvar_launch(const double* Vt, int64_t ldk, const double* kdiag, int64_t M, int64_t N, double* var, cudaStream_t st, int64_t* launches) {
    if (M <= 0) return cudaSuccess;
    rowvar_kernel<<<(unsigned)M, 256, 0, st>>>(Vt, ldk, kdiag, N, var);
    if (launches) ++*launches;
    return cudaGetLastError();
}
cudaError_t exp2x_launch(const double* ln, int64_t n, double* out, cudaStream_t st, int64_t* launches) {
    exp2x_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ln, n, out);
    if (launches) ++*launches;
    return cudaGetLastError();
}

// ---- posterior sampling helpers (gpb200_rand) -------------------------------------------------------------------
namespace {
// lower tiles of dst (n_pad x n_pad, ld ldd) = src[:n, :n] + nugget I ; identity in the padding
__global__ void spd_from_cov_kernel(double* __restrict__ dst, long long ldd, const double* __restrict__ src, long long lds,
                                    long long n, long long npad, double nugget) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y;
    if (j >= npad || (j >> 7) > (i >> 7)) return;
    double v;
    if (i < n && j < n) v = src[i * lds + j] + (i == j ? nugget : 0.0);
    else v = (i == j) ? 1.0 : 0.0;
    dst[i * ldd + j] = v;
}
__global__ void add_rowvec_kernel(double* __restrict__ A, long long ld, const double* __restrict__ v, long long nrows, long long ncols) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y;
    if (j < ncols && i < nrows) A[i * ld + j] += v[j];
}
}  // namespace
cudaError_t spd_from_cov_launch(double* dst, int64_t ldd, const double* src, int64_t lds, int64_t n, int64_t npad, double nugget, cudaStream_t st, int64_t* launches) {
    dim3 grid((unsigned)((npad + 255) / 256), (unsigned)npad);
    spd_from_cov_kernel<<<grid, 256, 0, st>>>(dst, ldd, src, lds, n, npad, nugget);
    if (launches) ++*launches;
    return cudaGetLastError();
}
cudaError_t add_rowvec_launch(double* A, int64_t ld, const double* v, int64_t nrows, int64_t ncols, cudaStream_t st, int64_t* launches) {
    dim3 grid((unsigned)((ncols + 255) / 256), (unsigned)nrows);
    add_rowvec_kernel<<<grid, 256, 0, st>>>(A, ld, v, nrows, ncols);
    if (launches) ++*launches;
    return cudaGetLastError();
}

namespace {
__global__ void gather_block_kernel(double* __restrict__ out, const double* __restrict__ src, long long ld, const long long* __restrict__ idx, long long nv) {
    const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x, a = blockIdx.y;
    if (b < nv) out[a * nv + b] = src[idx[a] * ld + idx[b]];
}
}  // namespace
cudaError_t gather_block_launch(double* out, const double* src, int64_t ld, const long long* idx, int64_t nv, cudaStream_t st, int64_t* launches) {
    if (nv <= 0) return cudaSuccess;
    dim3 grid((unsigned)((nv + 255) / 256), (unsigned)nv);
    gather_block_kernel<<<grid, 256, 0, st>>>(out, src, ld, idx, nv);
    if (launches) ++*launches;
    return cudaGetLastError();
}
