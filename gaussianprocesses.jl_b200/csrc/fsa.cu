// fsa.cu -- kernels of the Full Scale Approximation's block-diagonal Lambda (see fsa.cuh and fsa_engine.cu).
//
// The hot path is the grouped tile GEMM: every CTA reads one work item (tile pointers, leading dimensions, K, alpha, beta)
// from a device array, so one launch covers a list of aligned 128 x 128 tiles that belong to blocks of different sizes --
// the Schur update V_i V_i' of every block, the panels / trailing updates / inverse tiles of the batched block Cholesky,
// and the products against L_Lambda^-1.  Per-buffer TMA descriptors do not fit variable-size packed blocks, so operands
// are staged by cp.async (16-byte copies into the 128B-swizzled layout of gemm_nt.cu) through a 3-stage ring; the
// consumer warps, fragment loads and DMMA.16x8x16 issue order are those of gemm_nt.cu (dmma_tile.cuh).
#include "fsa.cuh"
#include <algorithm>
#include "dmma_tile.cuh"

namespace {

constexpr int TB = 128, KB = 16;
constexpr int GEMM_THREADS = 256;
constexpr int NSTAGE_G = 3;
constexpr int TILE_B = TB * KB * 8;                 // 16 KB per operand tile
constexpr int STAGE_B = 2 * TILE_B;
constexpr int SMEM_G = NSTAGE_G * STAGE_B;

template <int N>
__device__ __forceinline__ void cp_async_wait_group() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__global__ void __launch_bounds__(GEMM_THREADS, 1) fsa_gemm_kernel(const FsaGemmItem* __restrict__ items) {
    const FsaGemmItem it = items[blockIdx.x];
    extern __shared__ __align__(1024) unsigned char smem[];
    const uint32_t base = smem_u32(smem);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wm = warp & 1, wn = warp >> 1;
    const int g = lane >> 2, tq = lane & 3;
    int coff[4];
#pragma unroll
    for (int s = 0; s < 4; ++s) coff[s] = ((((tq >> 1) * 4 + s) ^ g) << 4) | ((tq & 1) << 3);
    double acc[8][4][2];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) { acc[i][j][0] = 0.0; acc[i][j][1] = 0.0; }

    auto gcopy = [&](int kt, int stage) {
        const uint32_t sA = base + stage * STAGE_B, sB = sA + TILE_B;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int chunk = threadIdx.x + i * GEMM_THREADS;
            const int row = chunk >> 3, c = chunk & 7;
            const int off = row * 128 + ((c ^ (row & 7)) << 4);
            cp_async16(sA + off, it.A + (long long)row * it.lda + kt * KB + c * 2);
            cp_async16(sB + off, it.B + (long long)row * it.ldb + kt * KB + c * 2);
        }
    };
    const int nk = it.K / KB;
#pragma unroll
    for (int s = 0; s < NSTAGE_G - 1; ++s) {
        if (s < nk) gcopy(s, s);
        cp_async_commit();
    }
    for (int kt = 0; kt < nk; ++kt) {
        cp_async_wait_group<NSTAGE_G - 2>();      // k-step kt has landed
        __syncthreads();                          // ... for every thread, and every warp is done with k-step kt-1's slot
        const int nxt = kt + NSTAGE_G - 1;
        if (nxt < nk) gcopy(nxt, nxt % NSTAGE_G);
        cp_async_commit();
        const uint32_t sA = base + (kt % NSTAGE_G) * STAGE_B;
        compute_stage(sA, sA + TILE_B, acc, wm, wn, g, coff);
    }

#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int r = wm * 64 + g + i * 8, c = wn * 32 + 2 * tq + j * 8;
            double* cp = it.C + (long long)r * it.ldc + c;
            double v0 = it.alpha * acc[i][j][0], v1 = it.alpha * acc[i][j][1];
            if (it.beta != 0.0) {
                // rounded as gemm_nt.cu's epilogue (alpha * acc, then one fma with beta * C): left to contraction, some
                // paths of this kernel became fma(alpha, acc, beta * C) and differed from the NT GEMM in the last bit
                const double2 old = *reinterpret_cast<const double2*>(cp);
                v0 = fma(it.beta, old.x, v0); v1 = fma(it.beta, old.y, v1);
            }
            if (!it.lower || c + 1 <= r) *reinterpret_cast<double2*>(cp) = make_double2(v0, v1);
            else if (c <= r) cp[0] = v0;
        }
    }
}

__global__ void __launch_bounds__(256) fsa_gram_kernel(const __grid_constant__ KProg P, const double* __restrict__ xb, int d,
                                                       const FsaGramItem* __restrict__ items, const double* __restrict__ mask,
                                                       double diag_add) {
    const FsaGramItem it = items[blockIdx.x];
    for (int e = threadIdx.x; e < TB * TB; e += blockDim.x) {
        const int li = e >> 7, lj = e & 127;
        if (it.diag && lj > li) continue;
        const long long gi = it.row_i + li, gj = it.row_j + lj;
        double v;
        if (mask[gi] == 0.0 || mask[gj] == 0.0) {
            v = (gi == gj) ? 1.0 : 0.0;
        } else {
            v = kprog_eval<false>(P, xb + gi * d, xb + gj * d, nullptr);
            if (gi == gj) v += diag_add;
        }
        it.dst[(long long)li * it.ld + lj] = v;
    }
}

__global__ void fsa_bdmv_kernel(int mode, const double* __restrict__ packed, const int* __restrict__ rblk,
                                const long long* __restrict__ bstart, const int* __restrict__ bsize,
                                const long long* __restrict__ boff, const double* __restrict__ v, double* __restrict__ y,
                                long long Np) {
    const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (r >= Np) return;
    const int b = rblk[r];
    const long long P = bstart[b];
    const int B = bsize[b], rl = (int)(r - P);
    const double* row = packed + boff[b] + (long long)rl * B;
    const int lo = (mode == 1) ? rl : 0, hi = (mode == 1) ? B : rl + 1;
    double s = 0.0;
    for (int k = lo + lane; k < hi; k += 32) {
        const double m = row[k];
        s = fma(m, (mode == 2) ? m : v[P + k], s);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) y[r] = s;
}

__global__ void fsa_mask_kernel(double* A, long long ld, long long nrows, long long ncols, const double* rowmask,
                                const double* colmask) {
    const long long i = blockIdx.y;
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < ncols; j += (long long)gridDim.x * blockDim.x) {
        if ((rowmask && rowmask[i] == 0.0) || (colmask && colmask[j] == 0.0)) A[i * ld + j] = 0.0;
    }
}

__global__ void fsa_permute_kernel(int scatter, const double* src, const long long* pos, long long n, double* dst) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (scatter) dst[pos[i]] = src[i];
    else dst[i] = src[pos[i]];
}

__global__ void fsa_resid_kernel(double* out, const double* a, const double* b, const double* mask, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = mask[i] * (a[i] - b[i]);
}

__global__ void __launch_bounds__(256) fsa_outer_kernel(const FsaGramItem* __restrict__ items, const double* __restrict__ a) {
    const FsaGramItem it = items[blockIdx.x];
    for (int e = threadIdx.x; e < TB * TB; e += blockDim.x) {
        const int li = e >> 7, lj = e & 127;
        it.dst[(long long)li * it.ld + lj] += a[it.row_i + li] * a[it.row_j + lj];
    }
}

__global__ void __launch_bounds__(256) fsa_trace_kernel(const __grid_constant__ KProg P, const double* __restrict__ xb, int d,
                                                        const FsaGramItem* __restrict__ items, const double* __restrict__ mask,
                                                        double* __restrict__ part) {
    __shared__ double red[256];
    const FsaGramItem it = items[blockIdx.x];
    const int np = P.n_theta;
    double acc[GPB200_MAX_THETA], g[GPB200_MAX_THETA];
    for (int p = 0; p < np; ++p) acc[p] = 0.0;
    for (int e = threadIdx.x; e < TB * TB; e += blockDim.x) {
        const int li = e >> 7, lj = e & 127;
        const long long gi = it.row_i + li, gj = it.row_j + lj;
        if (mask[gi] == 0.0 || mask[gj] == 0.0) continue;
        const double w = it.dst[(long long)li * it.ld + lj];
        kprog_eval<true>(P, xb + gi * d, xb + gj * d, g);
        for (int p = 0; p < np; ++p) acc[p] = fma(w, g[p], acc[p]);
    }
    for (int p = 0; p < np; ++p) {
        red[threadIdx.x] = acc[p];
        __syncthreads();
        for (int s = 128; s > 0; s >>= 1) {
            if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
            __syncthreads();
        }
        if (threadIdx.x == 0) part[(long long)blockIdx.x * np + p] = red[0];
        __syncthreads();
    }
}

// out[p] = sum_t part[t * np + p], t ascending
__global__ void fsa_trace_reduce_kernel(const double* __restrict__ part, int ntiles, int np, double* __restrict__ out) {
    const int p = blockIdx.x;
    __shared__ double red[256];
    double s = 0.0;
    for (int t = threadIdx.x; t < ntiles; t += blockDim.x) s += part[(long long)t * np + p];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int k = 128; k > 0; k >>= 1) {
        if (threadIdx.x < k) red[threadIdx.x] += red[threadIdx.x + k];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[p] = red[0];
}

__global__ void fsa_axpy_t_kernel(double* C, long long ldc, const double* A, long long lda, long long nrows, long long ncols,
                                  double alpha) {
    __shared__ double t[32][33];
    const long long i0 = (long long)blockIdx.y * 32, j0 = (long long)blockIdx.x * 32;
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {        // t[c][r] = A[j0 + r][i0 + c]
        const long long j = j0 + r, i = i0 + threadIdx.x;
        t[threadIdx.x][r] = (j < ncols && i < nrows) ? A[j * lda + i] : 0.0;
    }
    __syncthreads();
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const long long i = i0 + r, j = j0 + threadIdx.x;
        if (i < nrows && j < ncols) C[i * ldc + j] += alpha * t[r][threadIdx.x];
    }
}

__global__ void __launch_bounds__(256) fsa_crossgram_kernel(const __grid_constant__ KProg P, const double* __restrict__ xs,
                                                            const double* __restrict__ xb, int d,
                                                            const FsaGramItem* __restrict__ items, const double* __restrict__ mask) {
    const FsaGramItem it = items[blockIdx.x];
    for (int e = threadIdx.x; e < TB * TB; e += blockDim.x) {
        const int li = e >> 7, lj = e & 127;
        const long long gi = it.row_i + li, gj = it.row_j + lj;
        it.dst[(long long)li * it.ld + lj] = (mask[gj] == 0.0) ? 0.0 : kprog_eval<false>(P, xs + gi * d, xb + gj * d, nullptr);
    }
}

__global__ void __launch_bounds__(256) fsa_rowdot_kernel(const FsaRowItem* __restrict__ items) {
    const FsaRowItem it = items[blockIdx.x];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int r = warp; r < TB; r += 8) {
        const double* a = it.A + (long long)r * it.lda;
        double s = 0.0;
        for (int k = lane; k < it.K; k += 32) s = fma(a[k], it.sq ? a[k] : it.v[k], s);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) it.out[r] = s;
    }
}

__global__ void fsa_var_kernel(double* out, const double* q, const double* g2, const double* r2neg, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = q[i] - g2[i] - r2neg[i];
}

// Thread t takes the inducing points j = t, t + DX_NT, ..., then the block rows i = t, t + DX_NT, ..., in order; the d-vector
// accumulators are indexed by the leaves' input dimensions at run time and live in local memory (as crossgram_dx_kernel's).
constexpr int DX_NT = 128;
__global__ void __launch_bounds__(DX_NT) fsa_crossgram_dx_kernel(
        const __grid_constant__ KProg P, const double* __restrict__ xs, const double* __restrict__ z,
        const double* __restrict__ xb, int d, long long M, const double* __restrict__ u, const double* __restrict__ Wb,
        const double* __restrict__ S1, const double* __restrict__ S2, long long ldw, const double* __restrict__ mask,
        const double* __restrict__ alpha, const double* __restrict__ E, long long lde, const FsaDxItem* __restrict__ items,
        double* __restrict__ dmu, double* __restrict__ dvar) {
    __shared__ double sx[GPB200_MAX_DIMS];
    __shared__ double red[DX_NT];
    const FsaDxItem it = items[blockIdx.x];
    const int t = threadIdx.x;
    for (int k = t; k < d; k += DX_NT) sx[k] = xs[it.row * d + k];
    __syncthreads();
    double gm[GPB200_MAX_DIMS], gv[GPB200_MAX_DIMS];
    for (int k = 0; k < d; ++k) { gm[k] = 0.0; gv[k] = 0.0; }
    const bool V = dvar != nullptr;
    // dk(x*, x*)/dx* = 2 dk(x*, x')/dx* at x' = x*, into thread 0's variance sum only
    if (V && t == 0) kprog_eval_dx(P, sx, sx, 2.0, gv, 0.0, nullptr);
    const double* w = Wb ? Wb + it.row * ldw : nullptr;
    const double* s1 = V ? S1 + it.row * ldw : nullptr;
    const double* s2 = V ? S2 + it.row * ldw : nullptr;
    for (long long j = t; j < M; j += DX_NT)
        kprog_eval_dx(P, sx, z + j * d, u[j] - (w ? w[j] : 0.0), gm, V ? 2.0 * (s1[j] - s2[j]) : 0.0, V ? gv : nullptr);
    const double* e = V ? E + it.row * lde : nullptr;
    for (long long i = t; i < it.nb; i += DX_NT) {
        const long long gi = it.b0 + i;
        if (mask[gi] == 0.0) continue;
        kprog_eval_dx(P, sx, xb + gi * d, alpha[gi], gm, V ? e[i] : 0.0, V ? gv : nullptr);
    }
    for (int k = 0; k < d; ++k) {
        for (int which = 0; which < (V ? 2 : 1); ++which) {
            red[t] = which ? gv[k] : gm[k];
            __syncthreads();
            for (int s = DX_NT / 2; s > 0; s >>= 1) {
                if (t < s) red[t] += red[t + s];
                __syncthreads();
            }
            if (t == 0) (which ? dvar : dmu)[it.out * d + k] = red[0];
            __syncthreads();
        }
    }
}

// One CTA of TB threads per item (one 128-row tile row of a block), thread t owns row i = 128 tile + t of the block and walks
// l = 0 .. n-1 in order: G[i][l] along its own row (cached lines), G[l][i] down column i (coalesced over the threads), x_l
// the same for every thread.  No atomics and no cross-thread sums: a row's result does not depend on the launch.  FAST: the
// single SEIso leaf with d <= 8, the d-vectors in registers; else kprog_eval_dx with a local-memory d-vector.
template <bool FAST>
__global__ void __launch_bounds__(TB) fsa_block_dx_kernel(const __grid_constant__ KProg P, const double* __restrict__ xb, int d,
                                                         const FsaBlockDxItem* __restrict__ items, const long long* __restrict__ map,
                                                         double* __restrict__ out, int accumulate) {
    constexpr int DR = FAST ? 8 : GPB200_MAX_DIMS;
    const FsaBlockDxItem it = items[blockIdx.x];
    const long long i = (long long)it.tile * TB + threadIdx.x;
    if (i >= it.n) return;
    const int dk = FAST ? 8 : d;
    double acc[DR];
#pragma unroll
    for (int k = 0; k < dk; ++k) acc[k] = 0.0;
    const double* xi = xb + (it.row0 + i) * d;
    const double* gr = it.G + i * it.B;
    const double* gc = it.G + i;
    if (FAST) {
        const double il2 = 1.0 / P.par[0], mh = -0.5 / P.par[0], s2 = P.par[1];
        double xr[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) xr[k] = k < d ? xi[k] : 0.0;
#pragma unroll 1
        for (long long l = 0; l < it.n; ++l) {
            const double* xl = xb + (it.row0 + l) * d;
            double df[8], r2 = 0.0;
#pragma unroll
            for (int k = 0; k < 8; ++k) { df[k] = k < d ? xr[k] - xl[k] : 0.0; r2 += df[k] * df[k]; }
            const double f = -s2 * exp(mh * r2) * il2 * (gr[l] + gc[l * it.B]);
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] += f * df[k];
        }
    } else {
#pragma unroll 1
        for (long long l = 0; l < it.n; ++l) kprog_eval_dx(P, xi, xb + (it.row0 + l) * d, gr[l] + gc[l * it.B], acc, 0.0, nullptr);
    }
    const long long r = map ? map[it.row0 + i] : it.row0 + i;
#pragma unroll
    for (int k = 0; k < dk; ++k)
        if (k < d) out[r * d + k] = accumulate ? out[r * d + k] + acc[k] : acc[k];
}

bool g_gemm_attr = false;

}  // namespace

cudaError_t fsa_gemm_launch(const FsaGemmItem* items, int n, cudaStream_t st, int64_t* launches) {
    if (n <= 0) return cudaSuccess;
    if (!g_gemm_attr) {
        cudaError_t e = cudaFuncSetAttribute(fsa_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_G);
        if (e != cudaSuccess) return e;
        g_gemm_attr = true;
    }
    fsa_gemm_kernel<<<n, GEMM_THREADS, SMEM_G, st>>>(items);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t fsa_gram_launch(const KProg& P, const double* xb, int d, const FsaGramItem* items, int n, const double* mask,
                            double diag_add, cudaStream_t st, int64_t* launches) {
    if (n <= 0) return cudaSuccess;
    fsa_gram_kernel<<<n, 256, 0, st>>>(P, xb, d, items, mask, diag_add);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t fsa_bdmv_launch(int mode, const double* packed, const int* rblk, const long long* bstart, const int* bsize,
                            const long long* boff, const double* v, double* y, long long Np, cudaStream_t st, int64_t* launches) {
    if (Np <= 0) return cudaSuccess;
    fsa_bdmv_kernel<<<(unsigned)((Np + 7) / 8), 256, 0, st>>>(mode, packed, rblk, bstart, bsize, boff, v, y, Np);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t fsa_mask_launch(double* A, long long ld, long long nrows, long long ncols, const double* rowmask,
                            const double* colmask, cudaStream_t st, int64_t* launches) {
    if (nrows <= 0 || ncols <= 0) return cudaSuccess;
    const unsigned gx = (unsigned)std::min<long long>((ncols + 255) / 256, 64);
    fsa_mask_kernel<<<dim3(gx, (unsigned)nrows), 256, 0, st>>>(A, ld, nrows, ncols, rowmask, colmask);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t fsa_permute_launch(int scatter, const double* src, const long long* pos, long long n, double* dst, cudaStream_t st, int64_t* launches) {
    if (n <= 0) return cudaSuccess;
    fsa_permute_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(scatter, src, pos, n, dst);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t fsa_resid_launch(double* out, const double* a, const double* b, const double* mask, long long n, cudaStream_t st, int64_t* launches) {
    if (n <= 0) return cudaSuccess;
    fsa_resid_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(out, a, b, mask, n);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t fsa_outer_launch(const FsaGramItem* items, int n, const double* a, cudaStream_t st, int64_t* launches) {
    if (n <= 0) return cudaSuccess;
    fsa_outer_kernel<<<n, 256, 0, st>>>(items, a);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t fsa_trace_launch(const KProg& P, const double* xb, int d, const FsaGramItem* items, int n, const double* mask,
                             double* part, double* out, cudaStream_t st, int64_t* launches) {
    if (n <= 0) return cudaMemsetAsync(out, 0, sizeof(double) * P.n_theta, st);
    fsa_trace_kernel<<<n, 256, 0, st>>>(P, xb, d, items, mask, part);
    if (launches) ++*launches;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    fsa_trace_reduce_kernel<<<P.n_theta, 256, 0, st>>>(part, n, P.n_theta, out);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t fsa_axpy_t_launch(double* C, long long ldc, const double* A, long long lda, long long nrows, long long ncols,
                              double alpha, cudaStream_t st, int64_t* launches) {
    if (nrows <= 0 || ncols <= 0) return cudaSuccess;
    dim3 grid((unsigned)((ncols + 31) / 32), (unsigned)((nrows + 31) / 32));
    fsa_axpy_t_kernel<<<grid, dim3(32, 8), 0, st>>>(C, ldc, A, lda, nrows, ncols, alpha);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t fsa_crossgram_launch(const KProg& P, const double* xs, const double* xb, int d, const FsaGramItem* items, int n,
                                 const double* mask, cudaStream_t st, int64_t* launches) {
    if (n <= 0) return cudaSuccess;
    fsa_crossgram_kernel<<<n, 256, 0, st>>>(P, xs, xb, d, items, mask);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t fsa_rowdot_launch(const FsaRowItem* items, int n, cudaStream_t st, int64_t* launches) {
    if (n <= 0) return cudaSuccess;
    fsa_rowdot_kernel<<<n, 256, 0, st>>>(items);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t fsa_var_launch(double* out, const double* q, const double* g2, const double* r2neg, long long n, cudaStream_t st, int64_t* launches) {
    if (n <= 0) return cudaSuccess;
    fsa_var_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(out, q, g2, r2neg, n);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t fsa_crossgram_dx_launch(const KProg& P, const double* xs, const double* z, const double* xb, int d, long long M,
                                    const double* u, const double* Wb, const double* S1, const double* S2, long long ldw,
                                    const double* mask, const double* alpha, const double* E, long long lde,
                                    const FsaDxItem* items, int n, double* dmu, double* dvar, cudaStream_t st, int64_t* launches) {
    if (n <= 0) return cudaSuccess;
    fsa_crossgram_dx_kernel<<<n, DX_NT, 0, st>>>(P, xs, z, xb, d, M, u, Wb, S1, S2, ldw, mask, alpha, E, lde, items, dmu, dvar);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t fsa_block_dx_launch(const KProg& P, const double* xb, int d, const FsaBlockDxItem* items, int n, const long long* map,
                                double* out, int accumulate, cudaStream_t st, int64_t* launches) {
    if (n <= 0) return cudaSuccess;
    if (d <= 0 || d > GPB200_MAX_DIMS) return cudaErrorInvalidValue;
    if (kprog_fast(P, d) && d <= 8) fsa_block_dx_kernel<true><<<n, TB, 0, st>>>(P, xb, d, items, map, out, accumulate);
    else fsa_block_dx_kernel<false><<<n, TB, 0, st>>>(P, xb, d, items, map, out, accumulate);
    if (launches) ++*launches;
    return cudaGetLastError();
}
