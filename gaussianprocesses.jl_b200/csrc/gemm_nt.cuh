// gemm_nt.cuh -- host-side descriptor of the FP64 "NT" GEMM family used by every O(N^3) phase:
//     C[m,n] (+)= alpha * sum_{k in [klo,khi)} A[m,k] * B[n,k]          (all row-major)
// Cholesky trailing update (SYRK), panel TRSM through inverted diagonal blocks, the level-parallel
// triangular inverse, the LAUUM-like W'W product and the predictive TRSM are all instances.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

enum : int {
    GEMM_LOWER_ONLY = 1,   // M >= N: only tiles bm >= bn (lower trapezoid); diagonal tiles write i >= j only
    GEMM_KLO_M      = 2,   // k starts at bm*128        (A rows are upper-triangular in the frame)
    GEMM_KHI_M      = 4,   // k ends at (bm+1)*128      (A rows are lower-triangular)
    GEMM_KHI_N      = 8,   // k ends at (bn+1)*128      (B rows are lower-triangular)
    GEMM_SKIP_FIRST = 16,  // tile (0,0) is computed elsewhere (look-ahead of the next diagonal tile)
    GEMM_KLO_N      = 32,  // k starts at bn*128        (B rows are upper-triangular in the frame)
};

// A matrix living in a handle-owned buffer.  `map` is the TMA descriptor of the whole buffer
// (box 16 x 128 doubles, 128B swizzle); `base/ld` the same buffer for the non-TMA kernel.
struct GemmBuf {
    const CUtensorMap* map;
    const double* base;
    int64_t ld;
};

struct GemmOperand {
    GemmBuf buf;        // main buffer
    GemmBuf sub;        // compact [Npad x 128] buffer of clean diagonal tiles (or map == nullptr)
    int row0, col0;     // origin of the operand inside the buffer frame (multiples of 128)
};

struct GemmDesc {
    GemmOperand A, B;
    double* C; int64_t ldc; int c_row0, c_col0;
    double* Ct; int64_t ldct; int ct_row0, ct_col0;    // optional transposed copy: Ct[n, m] = C[m, n]
    int M, N, K;                                       // multiples of 128, 128, 16
    double alpha, beta;
    int flags;
    int batch;          // grid.z
    int zstep;          // added to every row0/col0 per batch index (diagonal stepping)
    int m_lim, n_lim, k_lim;   // per-batch clipping: M_z = min(M, m_lim - z*zstep) etc. (<=0: skip)
    int klo_off;        // GEMM_KLO_M: k starts at klo_off + bm*128 (row slice of a triangular operand)
    int bm_mod, bm_rem; // multi-GPU work split: only tile rows with ((bm + bm_off) / bm_div) % bm_mod == bm_rem (bm_mod <= 1: all)
    int bn_mod, bn_rem; // same for tile columns
    int bm_div, bm_off; // block-cyclic ownership: bm_div tiles per block (0/1: tile-cyclic), bm_off = global tile index of tile row 0
    int bn_div, bn_off;
    int n_peer;         // fused broadcast: C is additionally stored to these peer-mapped buffers (LOWER_ONLY: rejected, as Ct is)
    double* Cpeer[7];
};

static inline GemmDesc gemm_desc_default() {
    GemmDesc d{};
    d.alpha = 1.0; d.beta = 0.0; d.batch = 1; d.zstep = 0;
    d.m_lim = d.n_lim = d.k_lim = 1 << 30;
    return d;
}

// impl: 0 = TMA + mbarrier warp-specialised kernel, 1 = simple synchronous kernel.
// cudaErrorInvalidValue, nothing launched: M / N / K not multiples of 128 / 128 / 16, LOWER_ONLY with tm < tn, with n_peer > 0
// or with Ct; impl 0 without a main-buffer map or with a sub buffer that has no map.
cudaError_t gemm_nt_launch(const GemmDesc& d, int impl, cudaStream_t stream, int64_t* launches);
// one-time per process (sets max dynamic smem)
cudaError_t gemm_nt_init();
// Build a TMA descriptor for a row-major [rows x cols] FP64 buffer, box 16 x 128, swizzle 128B.
// Returns false (and leaves *out zeroed) if the driver entry point is unavailable.
bool gemm_make_tensor_map(CUtensorMap* out, const double* base, int64_t rows, int64_t cols, int64_t ld);

// Plain (un-swizzled) TMA descriptor of a row-major [rows x cols] FP64 buffer with a [box_rows x box_cols] box; rows past
// `rows` are zero-filled by the hardware (used for the 128 x d input tiles of the Gram / trace kernels).
// cols * 8 and ld * 8 must be multiples of 16 bytes.
bool gemm_make_tensor_map_plain(CUtensorMap* out, const double* base, int64_t rows, int64_t cols, int64_t ld, int box_rows, int box_cols);
