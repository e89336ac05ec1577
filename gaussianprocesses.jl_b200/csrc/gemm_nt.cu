// gemm_nt.cu -- FP64 tensor-core (DMMA) "NT" GEMM for sm_90a (H100).
//
// wgmma has no FP64 form; the FP64 tensor path on Hopper is warp-level mma.sync.f64.  On H100
// m8n8k4 (SASS DMMA.8x8x4) issues at half the FP64 rate of the m16n8k{4,8,16} shapes.  The kernel
// uses mma.sync.m16n8k16.f64 (DMMA.16x8x16): one instruction per 16-deep stage and fragment pair,
// 64 FMA per lane for 20 doubles of operand and accumulator traffic (m16n8k4: 16 FMA for 11), which
// matters because the GEMM runs at the card's power cap.  The A fragment holds rows g and g+8,
// so the accumulator layout is that of two stacked 8x8 tiles.  The kernel keeps the Hopper
// *data-movement* structure -- one producer warp driving TMA (cp.async.bulk.tensor.2d,
// 128B-swizzled 16x128 boxes) into a 5-stage shared-memory ring guarded by full/empty mbarriers --
// and feeds eight consumer warps that hold a 128x128 FP64 accumulator tile in registers (64x32
// per warp = 32 DMMA fragments).  The consumers load the first fragments of stage s+1 beside the
// last MMAs of stage s, so the tensor pipe does not idle at stage boundaries.
//
// Shared-memory layout per stage: A tile [128 rows][16 k] then B tile [128 rows][16 k], each row
// 128 bytes, TMA SWIZZLE_128B (16-byte chunk index ^= row & 7).  Lane (g, tq) feeds k slot q of
// the mma (logical k tq + 4q) from physical k 8*(tq>>1) + 2q + (tq&1): for each q the 16 lanes
// of a half-warp hit 16 distinct 8-byte bank pairs under the swizzle, so every fragment LDS.64 is
// conflict-free (any bijection of k indices to the mma's k slots is valid as long as A and B
// agree).
//
// Per CTA tile and k-step of 16: 32 KB staged for 128*128*16 FMAs = 2048 clk of DMMA at
// 128 FMA/clk/SM -> 16 B/clk/SM of L2 traffic; HBM traffic is a fraction of that thanks to the
// grouped rasterisation below.
#include "gemm_nt.cuh"
#include "dmma_tile.cuh"
#include <stdio.h>
#include <string.h>

namespace {

constexpr int BM = 128, BN = 128, BK = 16;
constexpr int NSTAGE = 5;
constexpr int TILE_BYTES = BM * BK * 8;           // 16 KB per operand tile
constexpr int STAGE_BYTES = 2 * TILE_BYTES;       // 32 KB
constexpr int TMA_THREADS = 12 * 32;              // 2 consumer warpgroups (8 warps) + 1 producer warpgroup
constexpr int SIMPLE_THREADS = 8 * 32;
constexpr int SMEM_TMA = NSTAGE * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
constexpr int SMEM_SIMPLE = 2 * STAGE_BYTES + 1024;
// rasterisation of triangular (GEMM_KLO_M) launches: group height in tile rows, k walked downwards (passed in GemmKP)
constexpr int GM_TRI = 4, K_DOWN = 1;

struct GemmKP {
    const double* A; const double* Asub; const double* B; const double* Bsub;
    long long lda, ldb;
    double* C; long long ldc;
    double* Ct; long long ldct;
    int a_row0, a_col0, b_row0, b_col0, c_row0, c_col0, ct_row0, ct_col0;
    int M, N, K;
    int flags, zstep, m_lim, n_lim, k_lim;
    int a_has_sub, b_has_sub;
    int klo_off, bm_mod, bm_rem, bn_mod, bn_rem;
    int bm_div, bm_off, bn_div, bn_off;
    int own_compact, n_own;      // row-ownership launches: the grid enumerates only the owned tile rows (n_own of them)
    long long own_first;         // global ordinal of the first owned tile row of this launch
    int gm_tri, k_down;          // rasterisation of triangular (GEMM_KLO_M) launches: group height, descending k
    int n_peer;                  // extra copies of C stored into peer GPUs' buffers (NVLink P2P), same ldc/offsets
    double* Cpeer[7];
    double alpha, beta;
};

struct TileCtx {
    int bm, bn, zoff;
    int kt_lo, kt_hi;
    bool valid;
};

__device__ __forceinline__ TileCtx decode_tile(const GemmKP& p) {
    TileCtx t;
    t.zoff = blockIdx.z * p.zstep;
    const int Mz = min(p.M, p.m_lim - t.zoff);
    const int Nz = min(p.N, p.n_lim - t.zoff);
    const int Kz = min(p.K, p.k_lim - t.zoff);
    {
        // L2-friendly rasterisation: the tm x tn tile rectangle is walked in groups of GROUP_M tile rows,
        // column by column inside a group, so the ~132 CTAs in flight cover ~16 rows x ~8 columns and every
        // k-slice of an operand row panel fetched from DRAM is reused out of L2 by its neighbours (the CTAs
        // march through k in near lock-step).  A plain row-major walk re-read the B panels once per tile.
        // Launches whose k range starts at the tile row (GEMM_KLO_M: triangular operand) have row-dependent
        // lengths; they walk k downwards (every tile starts at the common upper end) in narrower groups so
        // that neighbours stay within the L2 reuse window.
        const int GROUP_M = (p.flags & GEMM_KLO_M) ? p.gm_tri : 16;
        const int tm = p.M / BM, tn = p.N / BN;
        int rem = blockIdx.x;
        if (p.own_compact) {
            // multi-GPU launches that touch only the tile rows this rank owns (block-cyclic): enumerate exactly those rows,
            // 8 at a time, column by column inside a group -- no CTA is spent on a foreign row (at 8 ranks 7/8 of a plain
            // grid would start, decode and exit).  ordinal -> global tile row in closed form.
            constexpr int GO = 8;
            const int per_group = GO * tn;
            const int group = rem / per_group, in_group = rem - group * per_group;
            const int o = group * GO + in_group % GO;
            t.bn = in_group / GO;
            t.bm = 0;
            if (o < p.n_own) {
                const long long og = (long long)o + p.own_first;
                const long long tg = ((og / p.bm_div) * p.bm_mod + p.bm_rem) * p.bm_div + og % p.bm_div;
                t.bm = (int)(tg - p.bm_off);
            } else {
                t.bm = tm;                                     // -> invalid below
            }
        } else if (!(p.flags & GEMM_LOWER_ONLY)) {
            const int per_group = GROUP_M * tn;
            const int group = rem / per_group;
            const int first_m = group * GROUP_M;
            const int gsize = min(GROUP_M, tm - first_m);
            const int in_group = rem - group * per_group;
            t.bm = first_m + in_group % gsize;
            t.bn = in_group / gsize;
        } else {
            // lower trapezoid (tm >= tn): only tiles bn <= bm exist; same grouped walk, compactly enumerated
            int first_m = 0, gsize = 0;
            for (;;) {
                gsize = min(GROUP_M, tm - first_m);
                int cnt = 0;
                for (int r = first_m; r < first_m + gsize; ++r) cnt += min(r, tn - 1) + 1;
                if (rem < cnt || first_m + gsize >= tm) break;
                rem -= cnt; first_m += gsize;
            }
            const int full_cols = min(first_m, tn);             // columns every row of the group owns
            if (rem < full_cols * gsize) {
                t.bn = rem / gsize; t.bm = first_m + rem % gsize;
            } else {
                rem -= full_cols * gsize;
                int bn = full_cols;
                for (;;) {                                       // diagonal part of the group: rows >= bn
                    const int nrows = first_m + gsize - max(bn, first_m);
                    if (rem < nrows || bn + 1 >= tn) break;
                    rem -= nrows; ++bn;
                }
                t.bn = bn; t.bm = max(bn, first_m) + rem;
            }
        }
    }
    t.valid = (t.bm * BM < Mz) && (t.bn * BN < Nz) && (!(p.flags & GEMM_LOWER_ONLY) || t.bn <= t.bm) &&
              (!(p.flags & GEMM_SKIP_FIRST) || t.bm != 0 || t.bn != 0) &&
              (p.bm_mod <= 1 || (((t.bm + p.bm_off) / p.bm_div) % p.bm_mod) == p.bm_rem) &&
              (p.bn_mod <= 1 || (((t.bn + p.bn_off) / p.bn_div) % p.bn_mod) == p.bn_rem);
    t.kt_lo = (p.flags & GEMM_KLO_M) ? (p.klo_off + t.bm * BM) / BK : 0;
    if (p.flags & GEMM_KLO_N) t.kt_lo = max(t.kt_lo, t.bn * (BN / BK));
    int hi = Kz > 0 ? Kz / BK : 0;
    if (p.flags & GEMM_KHI_M) hi = min(hi, (t.bm + 1) * (BM / BK));
    if (p.flags & GEMM_KHI_N) hi = min(hi, (t.bn + 1) * (BN / BK));
    t.kt_hi = hi;
    return t;
}

__device__ __forceinline__ void epilogue(const GemmKP& p, const TileCtx& t, double (&acc)[8][4][2],
                                         int wm, int wn, int g, int tq) {
    const bool diag_mask = (p.flags & GEMM_LOWER_ONLY) && (t.bm == t.bn);
    const long long crow0 = (long long)p.c_row0 + t.zoff + t.bm * BM + wm * 64 + g;
    const long long ccol0 = (long long)p.c_col0 + t.zoff + t.bn * BN + wn * 32 + 2 * tq;
    const int lrow0 = wm * 64 + g, lcol0 = wn * 32 + 2 * tq;    // tile-local, for the diagonal mask
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const long long row = crow0 + i * 8, col = ccol0 + j * 8;
            double* cp = p.C + row * p.ldc + col;
            double v0 = p.alpha * acc[i][j][0], v1 = p.alpha * acc[i][j][1];
            if (p.beta != 0.0) {
                const double2 old = *reinterpret_cast<const double2*>(cp);
                v0 += p.beta * old.x; v1 += p.beta * old.y;
            }
            if (!diag_mask) {
                *reinterpret_cast<double2*>(cp) = make_double2(v0, v1);
                // fused panel broadcast: the same tile goes straight into every peer's copy of the factor
                for (int q = 0; q < p.n_peer; ++q)
                    *reinterpret_cast<double2*>(p.Cpeer[q] + row * p.ldc + col) = make_double2(v0, v1);
            } else {
                const int lr = lrow0 + i * 8, lc = lcol0 + j * 8;
                if (lc + 1 <= lr) *reinterpret_cast<double2*>(cp) = make_double2(v0, v1);
                else if (lc <= lr) cp[0] = v0;
            }
            if (p.Ct != nullptr) {
                const long long trow = (long long)p.ct_row0 + t.zoff + t.bn * BN + wn * 32 + 2 * tq + j * 8;
                const long long tcol = (long long)p.ct_col0 + t.zoff + t.bm * BM + wm * 64 + g + i * 8;
                p.Ct[trow * p.ldct + tcol] = v0;
                p.Ct[(trow + 1) * p.ldct + tcol] = v1;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// PTX wrappers: mbarrier + TMA
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
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

// ---------------------------------------------------------------------------------------------
// TMA / mbarrier warp-specialised kernel
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(TMA_THREADS, 1)
gpb200_dgemm_nt_tma(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapAsub,
                    const __grid_constant__ CUtensorMap mapB, const __grid_constant__ CUtensorMap mapBsub,
                    const GemmKP p) {
    const TileCtx t = decode_tile(p);
    if (!t.valid) return;

    extern __shared__ __align__(1024) unsigned char smem[];
    const uint32_t smem_base = smem_u32(smem);
    if (smem_base & 1023u) __trap();               // SWIZZLE_128B needs 1024-byte aligned tiles
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + NSTAGE * STAGE_BYTES);
    uint64_t* empty = full + NSTAGE;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
#pragma unroll
        for (int s = 0; s < NSTAGE; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();

    if (warp >= 8) {
        // ===== TMA producer warpgroup: give its registers to the consumers, one elected lane works =====
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == 8 && lane == 0) {
            const int ar = p.a_row0 + t.zoff + t.bm * BM;
            const int br = p.b_row0 + t.zoff + t.bn * BN;
            int stage = 0; uint32_t phase = 0;
            const bool down = (p.flags & GEMM_KLO_M) != 0 && p.k_down;
            for (int it = t.kt_lo; it < t.kt_hi; ++it) {
                const int kt = down ? (t.kt_hi - 1 - (it - t.kt_lo)) : it;
                mbar_wait(&empty[stage], phase ^ 1);
                mbar_expect_tx(&full[stage], STAGE_BYTES);
                unsigned char* sA = smem + stage * STAGE_BYTES;
                unsigned char* sB = sA + TILE_BYTES;
                const int ac = p.a_col0 + t.zoff + kt * BK;
                const int bc = p.b_col0 + t.zoff + kt * BK;
                if (p.a_has_sub && (ac >> 7) == (ar >> 7)) tma_load_2d(sA, &mapAsub, &full[stage], ac & 127, ar);
                else                                        tma_load_2d(sA, &mapA, &full[stage], ac, ar);
                if (p.b_has_sub && (bc >> 7) == (br >> 7)) tma_load_2d(sB, &mapBsub, &full[stage], bc & 127, br);
                else                                        tma_load_2d(sB, &mapB, &full[stage], bc, br);
                if (++stage == NSTAGE) { stage = 0; phase ^= 1; }
            }
        }
        return;
    }

    // ===== DMMA consumers =====
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
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

    // compute_stage's MMAs, pipelined across stages: the B and first A fragments of stage s+1 load beside the last
    // three MMAs of stage s, so no warp waits for a barrier or a fragment load at the top of a stage.  The consumers
    // wait on exactly the stages the producer fills, in its order (one per k-step).
    const uint32_t pa0 = smem_base + (wm * 64 + g) * 128;
    const uint32_t pb0 = smem_base + TILE_BYTES + (wn * 32 + g) * 128;
    const int nk = t.kt_hi - t.kt_lo;
    if (nk > 0) {
        int stage = 0; uint32_t phase = 0;
        double b[4][4], alo[4], ahi[4];
        mbar_wait(&full[0], 0);
#pragma unroll
        for (int j = 0; j < 4; ++j) load_b(pb0, j, coff, b[j]);
        load_a(pa0, 0, coff, alo, ahi);
        for (int it = 1;; ++it) {
            mma_pairs_0_to_4(pa0 + stage * STAGE_BYTES, coff, acc, b, alo, ahi);
            // This MMA consumes the last fragments loaded from the stage (B was consumed by pair 0).
            dmma16816(acc[6][0], acc[7][0], alo, ahi, b[0]);
            if (it == nk) {                              // the producer refills no slot after its last k-step
#pragma unroll
                for (int j = 1; j < 4; ++j) dmma16816(acc[6][j], acc[7][j], alo, ahi, b[j]);
                break;
            }
            const int done = stage;
            if (++stage == NSTAGE) { stage = 0; phase ^= 1; }
            mbar_wait(&full[stage], phase);
            // The slot goes back to the producer only here: an arrive does not wait for outstanding LDS, and the
            // wait loop above keeps the compiler from hoisting the arrive above the MMA that consumed them.
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[done]);
            const uint32_t pb = pb0 + stage * STAGE_BYTES;
            double nlo[4], nhi[4];
            load_b(pb, 0, coff, b[0]);
            load_a(pa0 + stage * STAGE_BYTES, 0, coff, nlo, nhi);
#pragma unroll
            for (int j = 1; j < 4; ++j) {
                dmma16816(acc[6][j], acc[7][j], alo, ahi, b[j]);
                load_b(pb, j, coff, b[j]);
            }
#pragma unroll
            for (int q = 0; q < 4; ++q) { alo[q] = nlo[q]; ahi[q] = nhi[q]; }
        }
    }
    epilogue(p, t, acc, wm, wn, g, tq);
}

// ---------------------------------------------------------------------------------------------
// Simple kernel: same tile math and the same swizzled smem layout, but filled by cp.async
// (16-byte global -> shared copies, no register staging next to the 128 accumulator registers)
// into two stages with __syncthreads.  Kept as the bring-up / cross-check path (option
// "gemm"=1) -- two independent loaders, one consumer.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SIMPLE_THREADS, 1) gpb200_dgemm_nt_simple(const GemmKP p) {
    const TileCtx t = decode_tile(p);
    if (!t.valid) return;
    extern __shared__ __align__(1024) unsigned char smem[];
    const uint32_t smem_base = smem_u32(smem);

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

    const int ar = p.a_row0 + t.zoff + t.bm * BM;
    const int br = p.b_row0 + t.zoff + t.bn * BN;

    // 16-byte global -> shared copies of one k-step into the swizzled layout, in flight while the other stage computes
    auto gcopy = [&](int kt, int stage) {
        const int ac = p.a_col0 + t.zoff + kt * BK;
        const int bc = p.b_col0 + t.zoff + kt * BK;
        const bool asub = p.a_has_sub && (ac >> 7) == (ar >> 7);
        const bool bsub = p.b_has_sub && (bc >> 7) == (br >> 7);
        const uint32_t sA = smem_base + stage * STAGE_BYTES;
        const uint32_t sB = sA + TILE_BYTES;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int chunk = threadIdx.x + i * SIMPLE_THREADS;
            const int row = chunk >> 3, c = chunk & 7;
            const int off = row * 128 + ((c ^ (row & 7)) << 4);
            const double* pa = asub ? p.Asub + (long long)(ar + row) * 128 + (ac & 127) + c * 2
                                    : p.A + (long long)(ar + row) * p.lda + ac + c * 2;
            const double* pb = bsub ? p.Bsub + (long long)(br + row) * 128 + (bc & 127) + c * 2
                                    : p.B + (long long)(br + row) * p.ldb + bc + c * 2;
            cp_async16(sA + off, pa);
            cp_async16(sB + off, pb);
        }
        cp_async_commit();
    };

    if (t.kt_lo < t.kt_hi) {
        const bool down = (p.flags & GEMM_KLO_M) != 0 && p.k_down;
        auto kmap = [&](int it) { return down ? (t.kt_hi - 1 - (it - t.kt_lo)) : it; };
        gcopy(kmap(t.kt_lo), 0);
        cp_async_wait_all();
        __syncthreads();
        int stage = 0;
        for (int kt = t.kt_lo; kt < t.kt_hi; ++kt) {
            if (kt + 1 < t.kt_hi) gcopy(kmap(kt + 1), stage ^ 1);
            const uint32_t sA = smem_base + stage * STAGE_BYTES;
            compute_stage(sA, sA + TILE_BYTES, acc, wm, wn, g, coff);
            cp_async_wait_all();
            __syncthreads();
            stage ^= 1;
        }
    }
    epilogue(p, t, acc, wm, wn, g, tq);
}

bool g_inited = false;
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;

}  // namespace

cudaError_t gemm_nt_init() {
    if (g_inited) return cudaSuccess;
    cudaError_t e = cudaFuncSetAttribute(gpb200_dgemm_nt_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_TMA);
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(gpb200_dgemm_nt_simple, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_SIMPLE);
    if (e != cudaSuccess) return e;
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) g_encode = reinterpret_cast<EncodeTiledFn>(fn);
    else (void)cudaGetLastError();
    g_inited = true;
    return cudaSuccess;
}

bool gemm_make_tensor_map(CUtensorMap* out, const double* base, int64_t rows, int64_t cols, int64_t ld) {
    memset(out, 0, sizeof(*out));
    if (!g_encode) return false;
    cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t gstride[1] = {(cuuint64_t)ld * sizeof(double)};
    cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)BM};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = g_encode(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, const_cast<double*>(base), gdim, gstride, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

bool gemm_make_tensor_map_plain(CUtensorMap* out, const double* base, int64_t rows, int64_t cols, int64_t ld, int box_rows, int box_cols) {
    memset(out, 0, sizeof(*out));
    if (!g_encode) return false;
    cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t gstride[1] = {(cuuint64_t)ld * sizeof(double)};
    cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = g_encode(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, const_cast<double*>(base), gdim, gstride, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

cudaError_t gemm_nt_launch(const GemmDesc& d, int impl, cudaStream_t stream, int64_t* launches) {
    GemmKP p;
    p.A = d.A.buf.base; p.Asub = d.A.sub.base; p.B = d.B.buf.base; p.Bsub = d.B.sub.base;
    p.lda = d.A.buf.ld; p.ldb = d.B.buf.ld;
    p.C = d.C; p.ldc = d.ldc; p.Ct = d.Ct; p.ldct = d.ldct;
    p.a_row0 = d.A.row0; p.a_col0 = d.A.col0; p.b_row0 = d.B.row0; p.b_col0 = d.B.col0;
    p.c_row0 = d.c_row0; p.c_col0 = d.c_col0; p.ct_row0 = d.ct_row0; p.ct_col0 = d.ct_col0;
    p.M = d.M; p.N = d.N; p.K = d.K;
    p.flags = d.flags; p.zstep = d.zstep; p.m_lim = d.m_lim; p.n_lim = d.n_lim; p.k_lim = d.k_lim;
    p.a_has_sub = d.A.sub.base != nullptr; p.b_has_sub = d.B.sub.base != nullptr;
    p.klo_off = d.klo_off; p.bm_mod = d.bm_mod; p.bm_rem = d.bm_rem; p.bn_mod = d.bn_mod; p.bn_rem = d.bn_rem;
    p.bm_div = d.bm_div > 0 ? d.bm_div : 1; p.bm_off = d.bm_off; p.bn_div = d.bn_div > 0 ? d.bn_div : 1; p.bn_off = d.bn_off;
    p.gm_tri = GM_TRI; p.k_down = K_DOWN;
    p.own_compact = 0; p.n_own = 0; p.own_first = 0;
    p.n_peer = d.n_peer;
    for (int q = 0; q < 7; ++q) p.Cpeer[q] = q < d.n_peer ? d.Cpeer[q] : nullptr;
    p.alpha = d.alpha; p.beta = d.beta;
    if (d.M <= 0 || d.N <= 0) return cudaSuccess;
    if ((d.M % BM) || (d.N % BN) || (d.K % BK)) return cudaErrorInvalidValue;
    // the diagonal mask applies to C only: a peer copy or Ct of a LOWER_ONLY launch would get the diagonal tiles' upper halves
    // wrong (peers) or written (Ct)
    if ((d.flags & GEMM_LOWER_ONLY) && (d.n_peer > 0 || d.Ct != nullptr)) return cudaErrorInvalidValue;
    // the TMA kernel reads a sub buffer through its own descriptor only
    if (impl == 0 && ((d.A.sub.base && !d.A.sub.map) || (d.B.sub.base && !d.B.sub.map))) return cudaErrorInvalidValue;
    const int tm = d.M / BM, tn = d.N / BN;
    if ((d.flags & GEMM_LOWER_ONLY) && tm < tn) return cudaErrorInvalidValue;
    // one CTA per tile (LOWER_ONLY: per tile of the lower trapezoid), walked in L2-friendly groups
    long long ntiles = (long long)tm * tn;
    if (d.flags & GEMM_LOWER_ONLY) { ntiles = 0; for (int r = 0; r < tm; ++r) ntiles += (r < tn - 1 ? r : tn - 1) + 1; }
    if (d.bm_mod > 1 && d.batch == 1) {
        // compact enumeration of the owned tile rows
        auto own_before = [&](long long t) {
            const long long cyc = (long long)p.bm_div * d.bm_mod, c = t / cyc, r = t % cyc;
            long long extra = r - (long long)d.bm_rem * p.bm_div;
            if (extra < 0) extra = 0;
            if (extra > p.bm_div) extra = p.bm_div;
            return c * p.bm_div + extra;
        };
        p.own_first = own_before(p.bm_off);
        p.n_own = (int)(own_before((long long)p.bm_off + tm) - p.own_first);
        p.own_compact = 1;
        if (p.n_own <= 0) return cudaSuccess;
        ntiles = (long long)((p.n_own + 7) / 8) * 8 * tn;
    }
    dim3 grid((unsigned)ntiles, 1, (unsigned)d.batch);
    if (impl == 0) {
        if (!d.A.buf.map || !d.B.buf.map) return cudaErrorInvalidValue;
        const CUtensorMap* ma = d.A.buf.map;
        const CUtensorMap* mas = d.A.sub.map ? d.A.sub.map : d.A.buf.map;
        const CUtensorMap* mb = d.B.buf.map;
        const CUtensorMap* mbs = d.B.sub.map ? d.B.sub.map : d.B.buf.map;
        gpb200_dgemm_nt_tma<<<grid, TMA_THREADS, SMEM_TMA, stream>>>(*ma, *mas, *mb, *mbs, p);
    } else {
        gpb200_dgemm_nt_simple<<<grid, SIMPLE_THREADS, SMEM_SIMPLE, stream>>>(p);
    }
    if (launches) ++*launches;
    return cudaGetLastError();
}
