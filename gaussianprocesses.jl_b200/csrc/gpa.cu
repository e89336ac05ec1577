// gpa.cu -- the O(N^2) pieces of the GPA gradient (src/GPA.jl:130-173, 200; src/chol_utils.jl:15-39).
//
// With K = L L', W = L^-1, f = L v + mu, g = dlog_dens_df(f) and u = L' g, the reference's reverse-mode Cholesky pass on
// Lbar = tril(g v') followed by dmll_kern! equals 1/2 sum_ij S_ij dK_ij with S = W' M_s W, M_s[i,j] = u[max(i,j)] v[min(i,j)].
// Only the lower triangle of S is needed:  S[a,b] = sum_{i>=a} W[i,a] Z[i,b]  (a >= b), where
//     Z[i,b] = u_i * sum_{b<=j<=i} v_j W[j,b]  +  v_i * sum_{j>i} u_j W[j,b]      (i >= b)
// is one prefix and one suffix scan along column b of W, i.e. along row b of W'.  That row is contiguous: its diagonal tile
// sits in DinvT, the rest in G's strict-upper tiles.  The product S = W' Z is then an NT GEMM (gpb200.cu).
//
// Every reduction runs in a fixed order, so repeated calls give bitwise-equal results.
#include "gpa.cuh"

namespace {
constexpr int T = 128;

// f[i] = sum_{j <= i} L[i,j] v[j]: one CTA (256 threads) per row, columns strided over the threads, fixed-order tree
__global__ void __launch_bounds__(256) trmv_lower_kernel(const double* __restrict__ F, long long ldf, const double* __restrict__ v,
                                                         double* __restrict__ f) {
    __shared__ double s[256];
    const long long i = blockIdx.x;
    const double* row = F + i * ldf;
    double acc = 0.0;
    for (long long j = threadIdx.x; j <= i; j += 256) acc += row[j] * v[j];
    s[threadIdx.x] = acc;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) { if (threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) f[i] = s[0];
}

// u[j] = sum_{i >= j} L[i,j] g[i]: one CTA (128 x 8 threads) per 128-column tile; thread (c, r) sums rows r, r+8, ... of
// column c (coalesced across c), the 8 partial sums are added in row order
__global__ void __launch_bounds__(1024) trmv_lower_t_kernel(const double* __restrict__ F, long long ldf, const double* __restrict__ g,
                                                            double* __restrict__ u, long long Npad) {
    __shared__ double s[8][T];
    const int c = threadIdx.x, r = threadIdx.y;
    const long long j = (long long)blockIdx.x * T + c;
    double acc = 0.0;
    long long i = (long long)blockIdx.x * T + r;
    for (; i < (long long)(blockIdx.x + 1) * T; i += 8)          // diagonal tile: rows i >= j only
        if (i >= j) acc += F[i * ldf + j] * g[i];
    for (; i < Npad; i += 8) acc += F[i * ldf + j] * g[i];
    s[r][c] = acc;
    __syncthreads();
    if (r == 0) {
        double t = s[0][c];
#pragma unroll
        for (int q = 1; q < 8; ++q) t += s[q][c];
        u[j] = t;
    }
}

constexpr int SCAN_T = 256, SCAN_E = 8, SCAN_CH = SCAN_T * SCAN_E;   // one chunk = 2048 consecutive entries of the row

// element c (global column, c >= b) of row b of W'
__device__ __forceinline__ double wt_at(const double* __restrict__ G, long long ld, const double* __restrict__ DinvT, int b, int tb0,
                                        long long c) {
    return c < tb0 + T ? DinvT[(long long)b * T + (c - tb0)] : G[(long long)b * ld + c];
}

// fixed-order block scans of one value per thread: apre = sum over threads < t of a, ssuf = sum over threads > t of s;
// atot / stot = the block totals.  sh: 16 doubles.
__device__ __forceinline__ void block_scan2(double a, double s, double& apre, double& ssuf, double& atot, double& stot, double* sh) {
    const int l = threadIdx.x & 31, w = threadIdx.x >> 5;
    double ai = a, si = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double ta = __shfl_up_sync(0xffffffffu, ai, o);
        const double ts = __shfl_down_sync(0xffffffffu, si, o);
        if (l >= o) ai += ta;
        if (l + o < 32) si += ts;
    }
    double ae = __shfl_up_sync(0xffffffffu, ai, 1);              // exclusive forms
    double se = __shfl_down_sync(0xffffffffu, si, 1);
    if (l == 0) ae = 0.0;
    if (l == 31) se = 0.0;
    if (l == 31) sh[w] = ai;
    if (l == 0) sh[8 + w] = si;
    __syncthreads();
    double aoff = 0.0, soff = 0.0, at = 0.0, st = 0.0;
#pragma unroll
    for (int q = 0; q < 8; ++q) { if (q < w) aoff += sh[q]; at += sh[q]; }
#pragma unroll
    for (int q = 7; q >= 0; --q) { if (q > w) soff += sh[8 + q]; st += sh[8 + q]; }
    __syncthreads();
    apre = aoff + ae; ssuf = soff + se; atot = at; stot = st;
}

// one CTA per row b of W'.  Pass 1: per-chunk totals of v_j w_j and u_j w_j.  Pass 2: per entry the inclusive prefix of v w
// and the exclusive suffix of u w (chunk carries + block scan + the thread's own run), Z = u_i P + v_i Q.
__global__ void __launch_bounds__(SCAN_T) gpa_scan_kernel(const double* __restrict__ G, long long ld, const double* __restrict__ DinvT,
                                                          const double* __restrict__ u, const double* __restrict__ v,
                                                          double* __restrict__ F, double* __restrict__ ZdT, long long Npad) {
    extern __shared__ double csum[];                           // [nch] totals of v w, [nch] of u w
    __shared__ double sh[16];
    const int b = blockIdx.x;
    const int tb0 = b & ~(T - 1);
    const long long len = Npad - b;
    const int nch = (int)((len + SCAN_CH - 1) / SCAN_CH);
    double* tv = csum;
    double* tu = csum + nch;
    for (int ch = 0; ch < nch; ++ch) {
        const long long j0 = (long long)ch * SCAN_CH + threadIdx.x * SCAN_E;
        double a = 0.0, s = 0.0;
#pragma unroll
        for (int k = 0; k < SCAN_E; ++k) {
            const long long j = j0 + k;
            if (j < len) {
                const long long c = b + j;
                const double w = wt_at(G, ld, DinvT, b, tb0, c);
                a += v[c] * w;
                s += u[c] * w;
            }
        }
        double apre, ssuf, atot, stot;
        block_scan2(a, s, apre, ssuf, atot, stot, sh);
        if (threadIdx.x == 0) { tv[ch] = atot; tu[ch] = stot; }
    }
    for (int k = threadIdx.x; k < b - tb0; k += SCAN_T) ZdT[(long long)b * T + k] = 0.0;   // clean upper diagonal tile
    __syncthreads();
    double carry_v = 0.0;
    for (int ch = 0; ch < nch; ++ch) {
        double carry_u = 0.0;
        for (int q = nch - 1; q > ch; --q) carry_u += tu[q];
        const long long j0 = (long long)ch * SCAN_CH + threadIdx.x * SCAN_E;
        double wk[SCAN_E], uk[SCAN_E], vk[SCAN_E];
        double a = 0.0, s = 0.0;
#pragma unroll
        for (int k = 0; k < SCAN_E; ++k) {
            const long long j = j0 + k;
            wk[k] = 0.0; uk[k] = 0.0; vk[k] = 0.0;
            if (j < len) {
                const long long c = b + j;
                wk[k] = wt_at(G, ld, DinvT, b, tb0, c);
                uk[k] = u[c]; vk[k] = v[c];
            }
            a += vk[k] * wk[k];
            s += uk[k] * wk[k];
        }
        double apre, ssuf, atot, stot;
        block_scan2(a, s, apre, ssuf, atot, stot, sh);
        double Q[SCAN_E];
        double q = carry_u + ssuf;
#pragma unroll
        for (int k = SCAN_E - 1; k >= 0; --k) { Q[k] = q; q += uk[k] * wk[k]; }
        double p = carry_v + apre;
#pragma unroll
        for (int k = 0; k < SCAN_E; ++k) {
            p += vk[k] * wk[k];
            const long long j = j0 + k;
            if (j < len) {
                const long long c = b + j;
                const double z = uk[k] * p + vk[k] * Q[k];
                if (c < tb0 + T) ZdT[(long long)b * T + (c - tb0)] = z;
                else F[(long long)b * ld + c] = z;
            }
        }
        carry_v += tv[ch];
    }
}
}  // namespace

cudaError_t gpa_trmv_launch(const double* F, int64_t ldf, const double* v, double* f, int64_t Npad, cudaStream_t st, int64_t* launches) {
    if (Npad <= 0) return cudaSuccess;
    trmv_lower_kernel<<<(unsigned)Npad, 256, 0, st>>>(F, ldf, v, f);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t gpa_trmv_t_launch(const double* F, int64_t ldf, const double* g, double* u, int64_t Npad, cudaStream_t st, int64_t* launches) {
    if (Npad <= 0) return cudaSuccess;
    trmv_lower_t_kernel<<<(unsigned)(Npad / T), dim3(T, 8), 0, st>>>(F, ldf, g, u, Npad);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t gpa_scan_launch(const double* G, int64_t ld, const double* DinvT, const double* u, const double* v, double* F,
                            double* ZdT, int64_t Npad, cudaStream_t st, int64_t* launches) {
    if (Npad <= 0) return cudaSuccess;
    const int64_t nch = (Npad + SCAN_CH - 1) / SCAN_CH;
    const size_t smem = sizeof(double) * 2 * (size_t)nch;
    if (smem > 48 * 1024) return cudaErrorInvalidValue;        // Npad > 6.2M: far beyond two N x N buffers on one device
    gpa_scan_kernel<<<(unsigned)Npad, SCAN_T, smem, st>>>(G, ld, DinvT, u, v, F, ZdT, Npad);
    if (launches) ++*launches;
    return cudaGetLastError();
}
