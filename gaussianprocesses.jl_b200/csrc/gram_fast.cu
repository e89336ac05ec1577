// gram_fast.cu -- the SEIso Gram build and the fused gradient trace in the form the north-star asks for:
// tile-per-CTA, the two 128 x d input tiles staged in shared memory by TMA (cp.async.bulk.tensor.2d, SASS UTMALDG,
// out-of-range rows zero-filled by the hardware), only the T(T+1)/2 lower tiles launched, column points cached in
// registers, row points broadcast from shared memory, FP64 outputs stored as 16-byte vectors (512 contiguous bytes per
// warp and row half).
//
// Replaces cov!(cK, k, X, data) (/root/reference/src/kernels/kernels.jl:39-50) with the SEIso leaf
// k = sigma^2 exp(-r / (2 l^2)) (src/kernels/se_iso.jl:39) and dmll_kern! (src/GPE.jl:219-241) with the SEIso
// derivatives dk/dll = r / l^2 k (se_iso.jl:41), dk/dlsigma = 2 k (stationary.jl:28).  Distances are direct
// differences summed in dimension order, as src/kernels/distance.jl:43-56.
//
// Why a hand-written exp: the kernel is bound by the FP64 pipe, not by HBM (d = 8: 16 FP64 ops for the distance;
// CUDA's exp() adds ~30 more).  exp(x) = 2^z, z = r * c, c = -log2(e) / (2 l^2), is evaluated as
// T[k mod 64] * p(f) * 2^(k div 64)  with k = round(64 z), f = z - k/64 (|f| <= 1/128), p = degree-5 Taylor polynomial of 2^f
// (truncation 3.5e-17), T[j] = sigma^2 2^(j/64) rounded once on the host, the power of two applied by an integer add to the
// exponent field and underflow detected in the integer pipe: 9 FP64 instructions including the argument, < 2 ulp of the
// exponential of the rounded argument (the argument's own rounding, |x| eps relative, is what any exp(-r/2l^2) carries).
// 25 FP64 instructions per output instead of ~46.
#include "gram_fast.cuh"
#include "gemm_nt.cuh"
#include <math.h>
#include <stdint.h>

namespace {

constexpr int TB = 128;
constexpr int NT = 256;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    } while (!ok);
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
                 : "memory");
}

// sigma^2 * 2^z for z <= 0; exactly 0 below z = -960 (true values < 1e-289 sigma^2).
// 2^z = T[k mod 64] * p(f) * 2^(k div 64), k = round(64 z), f = z - k/64 (|f| <= 1/128), p = degree-5 Taylor polynomial of
// 2^f (truncation 3.5e-17); 8 FP64 instructions.  The 64-entry table is replicated 16 times in shared memory, entry j of copy
// c at word j*16 + c, and lane l reads copy l % 16: the 16 lanes of a half-warp always hit 16 different bank pairs, whatever
// their indices (a plain table cost ~9 extra LSU cycles per lookup: ncu l1tex__data_bank_conflicts 154 M per launch at C2).
constexpr int TABN = 64;
__device__ __forceinline__ double exp2_tab(double z, const double* __restrict__ tab) {
    const double MAGIC = 6755399441055744.0;                 // 1.5 * 2^52: the low mantissa bits hold round(64 z)
    const double zs = fma(z, 64.0, MAGIC);
    const int ki = __double2loint(zs);
    const double kf = zs - MAGIC;
    const double f = fma(kf, -0.015625, z);                   // exact
    double p = 1.3333558146428443423e-3;                      // ln2^5 / 120
    p = fma(p, f, 9.6181291076284771619e-3);                  // ln2^4 / 24
    p = fma(p, f, 5.5504108664821579953e-2);                  // ln2^3 / 6
    p = fma(p, f, 2.4022650695910071233e-1);                  // ln2^2 / 2
    p = fma(p, f, 6.9314718055994530942e-1);                  // ln2
    p = fma(p, f, 1.0);
    const double r = tab[(ki & (TABN - 1)) << 4] * p;         // tab already points at this lane's copy (bank pair lane % 16)
    const double v = __hiloint2double(__double2hiint(r) + ((ki >> 6) << 20), __double2loint(r));
    // underflow guard in the integer pipe: z <= -960 (high word compare; z <= 0 always) -> 0, whatever k wrapped to
    return ((unsigned)__double2hiint(z) > 0xC08E0000u) ? 0.0 : v;
}

__device__ __forceinline__ void tri_decode(int lin, int& bm, int& bn) {
    int m = (int)((sqrt(8.0 * (double)lin + 1.0) - 1.0) * 0.5);
    while (m * (m + 1) / 2 > lin) --m;
    while ((m + 1) * (m + 2) / 2 <= lin) ++m;
    bm = m; bn = lin - m * (m + 1) / 2;
}

// stage the two 128 x DX input tiles by TMA; returns true if every staged value is finite
// row tile sXi[r][k] from x (N x DX), column tile sXjT[k][c] from the transposed copy x' (DX x N): the per-lane register
// preload of column points then reads 16 consecutive bytes per lane (conflict-free), the row points are broadcast reads.
template <int DX>
__device__ __forceinline__ bool stage_tiles(const CUtensorMap* mapX, const CUtensorMap* mapXT, double* sXi, double* sXj, uint64_t* bar, int bm, int bn) {
    if (threadIdx.x == 0) {
        mbar_init(bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_expect_tx(bar, 2u * TB * DX * 8u);
        tma_load_2d(sXi, mapX, bar, 0, bm * TB);
        tma_load_2d(sXj, mapXT, bar, bn * TB, 0);
    }
    mbar_wait(bar, 0);
    int bad = 0;
    for (int i = threadIdx.x; i < TB * DX; i += NT) bad |= !(fabs(sXi[i]) <= 1.7e308) | !(fabs(sXj[i]) <= 1.7e308);
    return __syncthreads_or(bad) == 0;
}

template <int DX>
__global__ void __launch_bounds__(NT, 2)
gram_seiso_tma_kernel(const __grid_constant__ CUtensorMap mapX, const __grid_constant__ CUtensorMap mapXT,
                      const __grid_constant__ SeIsoFast sf, long long N,
                      const double* __restrict__ noise_var, long long n_noise, double nugget, double* __restrict__ G,
                      long long ldg, int own_tiles, int nranks, int rank, int own_axis) {
    __shared__ __align__(128) double sXi[TB * DX];
    __shared__ __align__(128) double sXj[TB * DX];
    __shared__ double sTabR[TABN * 16];
    __shared__ __align__(8) uint64_t bar;
    int bm, bn;
    tri_decode(blockIdx.x, bm, bn);
    if (own_tiles > 0 && (((own_axis ? bm : bn) / own_tiles) % nranks) != rank) return;
    for (int i = threadIdx.x; i < TABN * 16; i += NT) sTabR[i] = sf.tab[i >> 4];
    const double* sTab = sTabR + (threadIdx.x & 15);
    const bool finite = stage_tiles<DX>(&mapX, &mapXT, sXi, sXj, &bar, bm, bn);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double xj[4][DX];
#pragma unroll
    for (int k = 0; k < DX; ++k) {
        const double2 lo = *reinterpret_cast<const double2*>(sXj + k * TB + lane * 2);
        const double2 hi = *reinterpret_cast<const double2*>(sXj + k * TB + 64 + lane * 2);
        xj[0][k] = lo.x; xj[1][k] = lo.y; xj[2][k] = hi.x; xj[3][k] = hi.y;
    }
    const bool plain = finite && (bm != bn) && ((long long)(bm + 1) * TB <= N);
    const double c_hi = sf.c_hi;
    double* gbase = G + ((long long)bm * TB + warp * 16) * ldg + (long long)bn * TB + lane * 2;
    if (plain) {
#pragma unroll 2
        for (int rr = 0; rr < 16; ++rr) {
            const double2* xi2 = reinterpret_cast<const double2*>(sXi + (warp * 16 + rr) * DX);
            double xir[DX];
#pragma unroll
            for (int k = 0; k < DX / 2; ++k) { const double2 t2 = xi2[k]; xir[2 * k] = t2.x; xir[2 * k + 1] = t2.y; }
            double v[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                double r2 = 0.0;
#pragma unroll
                for (int k = 0; k < DX; ++k) { const double df = xir[k] - xj[q][k]; r2 = fma(df, df, r2); }
                v[q] = exp2_tab(r2 * c_hi, sTab);
            }
            double* row = gbase + (long long)rr * ldg;
            *reinterpret_cast<double2*>(row) = make_double2(v[0], v[1]);
            *reinterpret_cast<double2*>(row + 64) = make_double2(v[2], v[3]);
        }
        return;
    }
    // diagonal tiles (noise on the diagonal), tiles touching the padding (identity), non-finite inputs (libm exp)
#pragma unroll 1
    for (int rr = 0; rr < 16; ++rr) {
        const int r = warp * 16 + rr;
        const long long gi = (long long)bm * TB + r;
        const double* xi = sXi + r * DX;
        double v[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const long long gj = (long long)bn * TB + (q >> 1) * 64 + lane * 2 + (q & 1);
            double r2 = 0.0;
#pragma unroll
            for (int k = 0; k < DX; ++k) { const double df = xi[k] - xj[q][k]; r2 = fma(df, df, r2); }
            double kv = finite ? exp2_tab(r2 * c_hi, sTab) : sf.s2 * exp(-0.5 * r2 * sf.il2);
            if (gi >= N || gj >= N) kv = (gi == gj) ? 1.0 : 0.0;
            else if (gi == gj) kv += ((n_noise == 1) ? noise_var[0] : noise_var[gi]) + nugget;
            v[q] = kv;
        }
        double* row = gbase + (long long)rr * ldg;
        *reinterpret_cast<double2*>(row) = make_double2(v[0], v[1]);
        *reinterpret_cast<double2*>(row + 64) = make_double2(v[2], v[3]);
    }
}

// fused gradient trace, SEIso: part[tile][0..2] = { sum w r/l^2 k, sum w 2k, sum_diag A },  A = a_i a_j - Kinv_ij,
// w = A below the diagonal, A/2 on it  (GPE.jl:219-241, 273-275)
template <int DX>
__global__ void __launch_bounds__(NT, 2)
trace_seiso_tma_kernel(const __grid_constant__ CUtensorMap mapX, const __grid_constant__ CUtensorMap mapXT,
                       const __grid_constant__ SeIsoFast sf, long long N,
                       const double* __restrict__ alpha, const double* __restrict__ Kinv, long long ldg,
                       double* __restrict__ part, int bm_mod, int bm_rem, int bm_div) {
    __shared__ __align__(128) double sXi[TB * DX];
    __shared__ __align__(128) double sXj[TB * DX];
    __shared__ double sTabR[TABN * 16];
    __shared__ __align__(16) double sAi[TB];
    __shared__ __align__(16) double sAj[TB];
    __shared__ double sRed[8 * 3];
    __shared__ __align__(8) uint64_t bar;
    int bm, bn;
    tri_decode(blockIdx.x, bm, bn);
    const long long lin = blockIdx.x;
    if (bm_mod > 1 && ((bm / bm_div) % bm_mod) != bm_rem) {
        if (threadIdx.x < 3) part[lin * 3 + threadIdx.x] = 0.0;
        return;
    }
    for (int i = threadIdx.x; i < TABN * 16; i += NT) sTabR[i] = sf.tab[i >> 4];
    const double* sTab = sTabR + (threadIdx.x & 15);
    if (threadIdx.x < TB) {
        const long long gi = (long long)bm * TB + threadIdx.x, gj = (long long)bn * TB + threadIdx.x;
        sAi[threadIdx.x] = gi < N ? alpha[gi] : 0.0;
        sAj[threadIdx.x] = gj < N ? alpha[gj] : 0.0;
    }
    const bool finite = stage_tiles<DX>(&mapX, &mapXT, sXi, sXj, &bar, bm, bn);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double xj[4][DX], aj[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) aj[q] = sAj[(q >> 1) * 64 + lane * 2 + (q & 1)];
#pragma unroll
    for (int k = 0; k < DX; ++k) {
        const double2 lo = *reinterpret_cast<const double2*>(sXj + k * TB + lane * 2);
        const double2 hi = *reinterpret_cast<const double2*>(sXj + k * TB + 64 + lane * 2);
        xj[0][k] = lo.x; xj[1][k] = lo.y; xj[2][k] = hi.x; xj[3][k] = hi.y;
    }
    const bool plain = finite && (bm != bn) && ((long long)(bm + 1) * TB <= N);
    const double c_hi = sf.c_hi;
    double acc0 = 0.0, acc1 = 0.0, acc2 = 0.0;
    const double* kbase = Kinv + ((long long)bm * TB + warp * 16) * ldg + (long long)bn * TB + lane * 2;
    if (plain) {
        // the K^-1 values of a row are fetched two rows ahead (register double-buffer): the global-load latency (~1.5k cycles)
        // is covered by two rows of FP64 work instead of stalling every row (ncu: FP64 pipe 42% -> with the plain loop)
        double2 pa[2], pb[2];
#pragma unroll
        for (int s = 0; s < 2; ++s) {
            pa[s] = *reinterpret_cast<const double2*>(kbase + (long long)s * ldg);
            pb[s] = *reinterpret_cast<const double2*>(kbase + (long long)s * ldg + 64);
        }
#pragma unroll 2
        for (int rr = 0; rr < 16; ++rr) {
            const int r = warp * 16 + rr;
            const double2* xi2 = reinterpret_cast<const double2*>(sXi + r * DX);
            double xir[DX];
#pragma unroll
            for (int k = 0; k < DX / 2; ++k) { const double2 t2 = xi2[k]; xir[2 * k] = t2.x; xir[2 * k + 1] = t2.y; }
            const double ai = sAi[r];
            const double2 k01 = pa[rr & 1], k23 = pb[rr & 1];
            if (rr + 2 < 16) {
                pa[rr & 1] = *reinterpret_cast<const double2*>(kbase + (long long)(rr + 2) * ldg);
                pb[rr & 1] = *reinterpret_cast<const double2*>(kbase + (long long)(rr + 2) * ldg + 64);
            }
            const double kin[4] = {k01.x, k01.y, k23.x, k23.y};
            const double2 a01 = *reinterpret_cast<const double2*>(sAj + lane * 2);        // re-read per row: frees 8 registers
            const double2 a23 = *reinterpret_cast<const double2*>(sAj + 64 + lane * 2);
            const double ajr[4] = {a01.x, a01.y, a23.x, a23.y};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                double r2 = 0.0;
#pragma unroll
                for (int k = 0; k < DX; ++k) { const double df = xir[k] - xj[q][k]; r2 = fma(df, df, r2); }
                const double kv = exp2_tab(r2 * c_hi, sTab);
                const double t = fma(ai, ajr[q], -kin[q]) * kv;                // A k
                acc0 = fma(t, r2, acc0);                                       // * 1/l^2 at the end
                acc1 += t;                                                     // * 2 at the end
            }
        }
    } else {
#pragma unroll 1
        for (int rr = 0; rr < 16; ++rr) {
            const int r = warp * 16 + rr;
            const long long gi = (long long)bm * TB + r;
            if (gi >= N) continue;
            const double* xi = sXi + r * DX;
            const double ai = sAi[r];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const long long gj = (long long)bn * TB + (q >> 1) * 64 + lane * 2 + (q & 1);
                if (gj > gi || gj >= N) continue;
                const double kinv = kbase[(long long)rr * ldg + (q >> 1) * 64 + (q & 1)];
                double r2 = 0.0;
#pragma unroll
                for (int k = 0; k < DX; ++k) { const double df = xi[k] - xj[q][k]; r2 = fma(df, df, r2); }
                const double kv = finite ? exp2_tab(r2 * c_hi, sTab) : sf.s2 * exp(-0.5 * r2 * sf.il2);
                const double A = fma(ai, aj[q], -kinv);
                const double t = ((gi == gj) ? 0.5 * A : A) * kv;
                acc0 = fma(t, r2, acc0);
                acc1 += t;
                if (gi == gj) acc2 += A;
            }
        }
    }
    acc0 *= sf.il2;
    acc1 *= 2.0;
    // lane tree, then fixed warp order: bitwise reproducible
    double accs[3] = {acc0, acc1, acc2};
#pragma unroll
    for (int p = 0; p < 3; ++p) {
        double v = accs[p];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
        if (lane == 0) sRed[warp * 3 + p] = v;
    }
    __syncthreads();
    if (threadIdx.x < 3) {
        double v = 0.0;
        for (int w8 = 0; w8 < NT / 32; ++w8) v += sRed[w8 * 3 + threadIdx.x];
        part[lin * 3 + threadIdx.x] = v;
    }
}

__global__ void reduce_partials3_kernel(const double* __restrict__ part, int tiles, double* __restrict__ out) {
    const int p = blockIdx.x;
    __shared__ double s[256];
    double v = 0.0;
    for (int t = threadIdx.x; t < tiles; t += 256) v += part[(long long)t * 3 + p];
    s[threadIdx.x] = v;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[p] = s[0];
}

}  // namespace

bool seiso_fast_prepare(double l2, double s2, SeIsoFast* out) {
    if (!(l2 > 1e-20 && l2 < 1e20 && s2 > 1e-15 && s2 < 1e15)) return false;
    const long double c = (-0.5L / (long double)l2) * 1.442695040888963407359924681001892137L;      // -log2(e) / (2 l^2)
    out->c_hi = (double)c;
    out->c_lo = (double)(c - (long double)out->c_hi);
    out->il2 = 1.0 / l2;
    out->s2 = s2;
    for (int j = 0; j < 64; ++j) out->tab[j] = (double)((long double)s2 * exp2l((long double)j / 64.0L));
    return true;
}

bool seiso_make_x_maps(CUtensorMap* mapX, CUtensorMap* mapXT, const double* xp, const double* xpt, int dx, int64_t N, int64_t Npad) {
    return gemm_make_tensor_map_plain(mapX, xp, N, dx, dx, TB, dx) && gemm_make_tensor_map_plain(mapXT, xpt, dx, N, Npad, dx, TB);
}

cudaError_t gram_seiso_tma_launch(const CUtensorMap* mapX, const CUtensorMap* mapXT, int dx, const SeIsoFast& sf, int64_t N, int64_t Npad,
                                  const double* noise_var, int64_t n_noise, double nugget, double* G, int64_t ldg,
                                  cudaStream_t st, int64_t* launches, int own_tiles, int nranks, int rank, int own_axis) {
    const int T = (int)(Npad / TB);
    const int tiles = T * (T + 1) / 2;
    switch (dx) {
    case 2: gram_seiso_tma_kernel<2><<<tiles, NT, 0, st>>>(*mapX, *mapXT, sf, N, noise_var, n_noise, nugget, G, ldg, own_tiles, nranks, rank, own_axis); break;
    case 4: gram_seiso_tma_kernel<4><<<tiles, NT, 0, st>>>(*mapX, *mapXT, sf, N, noise_var, n_noise, nugget, G, ldg, own_tiles, nranks, rank, own_axis); break;
    case 6: gram_seiso_tma_kernel<6><<<tiles, NT, 0, st>>>(*mapX, *mapXT, sf, N, noise_var, n_noise, nugget, G, ldg, own_tiles, nranks, rank, own_axis); break;
    case 8: gram_seiso_tma_kernel<8><<<tiles, NT, 0, st>>>(*mapX, *mapXT, sf, N, noise_var, n_noise, nugget, G, ldg, own_tiles, nranks, rank, own_axis); break;
    default: return cudaErrorInvalidValue;
    }
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t trace_seiso_tma_launch(const CUtensorMap* mapX, const CUtensorMap* mapXT, int dx, const SeIsoFast& sf, int64_t N, int64_t Npad,
                                   const double* alpha, const double* Kinv, int64_t ldg, double* part, double* out,
                                   cudaStream_t st, int64_t* launches, int bm_mod, int bm_rem, int bm_div) {
    const int T = (int)(Npad / TB);
    const int tiles = T * (T + 1) / 2;
    if (bm_div < 1) bm_div = 1;
    switch (dx) {
    case 2: trace_seiso_tma_kernel<2><<<tiles, NT, 0, st>>>(*mapX, *mapXT, sf, N, alpha, Kinv, ldg, part, bm_mod, bm_rem, bm_div); break;
    case 4: trace_seiso_tma_kernel<4><<<tiles, NT, 0, st>>>(*mapX, *mapXT, sf, N, alpha, Kinv, ldg, part, bm_mod, bm_rem, bm_div); break;
    case 6: trace_seiso_tma_kernel<6><<<tiles, NT, 0, st>>>(*mapX, *mapXT, sf, N, alpha, Kinv, ldg, part, bm_mod, bm_rem, bm_div); break;
    case 8: trace_seiso_tma_kernel<8><<<tiles, NT, 0, st>>>(*mapX, *mapXT, sf, N, alpha, Kinv, ldg, part, bm_mod, bm_rem, bm_div); break;
    default: return cudaErrorInvalidValue;
    }
    if (launches) ++*launches;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    reduce_partials3_kernel<<<3, 256, 0, st>>>(part, tiles, out);
    if (launches) ++*launches;
    return cudaGetLastError();
}
