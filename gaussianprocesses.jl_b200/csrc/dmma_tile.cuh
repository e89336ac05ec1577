// dmma_tile.cuh -- device building blocks of the 128 x 128 FP64 DMMA tile shared by the NT GEMM (gemm_nt.cu) and the
// grouped block-diagonal tile GEMM (fsa.cu): mma.sync.m16n8k16.f64, the conflict-free fragment loads out of a
// 128B-swizzled [128 rows][16 k] stage, one 16-deep k-step of the 64 x 32 warp tile, and cp.async.
//
// Eight consumer warps: warp (wm = warp & 1, wn = warp >> 1) owns rows wm*64 .. +64 and columns wn*32 .. +32 of the tile;
// lane (g, tq) feeds k slot q from physical k coff[q] (see gemm_nt.cu's header for the bank analysis).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// D[16x8] += A[16x16] B[16x8]: a_lo / a_hi = rows g / g+8 of A, {c0,c1} / {c2,c3} = rows g / g+8 of D.  k slot q
// of lane (g, tq) is a_lo[q], a_hi[q] and b[q].
__device__ __forceinline__ void dmma16816(double (&c_lo)[2], double (&c_hi)[2], const double (&a_lo)[4],
                                          const double (&a_hi)[4], const double (&b)[4]) {
    asm("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
        "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
        : "+d"(c_lo[0]), "+d"(c_lo[1]), "+d"(c_hi[0]), "+d"(c_hi[1])
        : "d"(a_lo[0]), "d"(a_hi[0]), "d"(a_lo[1]), "d"(a_hi[1]), "d"(a_lo[2]), "d"(a_hi[2]), "d"(a_lo[3]), "d"(a_hi[3]),
          "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

__device__ __forceinline__ double lds_f64(uint32_t addr) {
    double v;
    asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(addr));
    return v;
}

// Fragment loads of one stage.  pa / pb point at row g of the warp's A / B rows in the stage; k slot q is physical k
// coff[q] (the same for A and B, so any bijection is valid; this one is bank-conflict free, see the header).
// A rows g + 8i and g + 8i + 8 (row pair i = 0, 2, 4, 6):
__device__ __forceinline__ void load_a(uint32_t pa, int i, const int (&coff)[4], double (&alo)[4], double (&ahi)[4]) {
#pragma unroll
    for (int q = 0; q < 4; ++q) { alo[q] = lds_f64(pa + i * 1024 + coff[q]); ahi[q] = lds_f64(pa + (i + 1) * 1024 + coff[q]); }
}
// B rows g + 8j:
__device__ __forceinline__ void load_b(uint32_t pb, int j, const int (&coff)[4], double (&b)[4]) {
#pragma unroll
    for (int q = 0; q < 4; ++q) b[q] = lds_f64(pb + j * 1024 + coff[q]);
}

// Row pairs 0, 2 and 4 of a stage whose B fragments and pair-0 A fragments are in registers; the A fragments of the
// next pair load beside each pair's MMAs.  Leaves pair 6's A fragments in alo / ahi.
__device__ __forceinline__ void mma_pairs_0_to_4(uint32_t pa, const int (&coff)[4], double (&acc)[8][4][2],
                                                 const double (&b)[4][4], double (&alo)[4], double (&ahi)[4]) {
#pragma unroll
    for (int i = 0; i < 6; i += 2) {
        double nlo[4], nhi[4];
        load_a(pa, i + 2, coff, nlo, nhi);
#pragma unroll
        for (int j = 0; j < 4; ++j) dmma16816(acc[i][j], acc[i + 1][j], alo, ahi, b[j]);
#pragma unroll
        for (int q = 0; q < 4; ++q) { alo[q] = nlo[q]; ahi[q] = nhi[q]; }
    }
}

// One 16-deep k-step of the 64x32 warp tile out of swizzled shared memory (32-bit shared addresses): one
// m16n8k16 per (row pair, column fragment).  The TMA consumer loop issues the same MMAs in the same order.
__device__ __forceinline__ void compute_stage(uint32_t sA, uint32_t sB,
                                              double (&acc)[8][4][2], int wm, int wn, int g, const int (&coff)[4]) {
    const uint32_t pa = sA + (wm * 64 + g) * 128;
    const uint32_t pb = sB + (wn * 32 + g) * 128;
    double b[4][4], alo[4], ahi[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) load_b(pb, j, coff, b[j]);
    load_a(pa, 0, coff, alo, ahi);
    mma_pairs_0_to_4(pa, coff, acc, b, alo, ahi);
#pragma unroll
    for (int j = 0; j < 4; ++j) dmma16816(acc[6][j], acc[7][j], alo, ahi, b[j]);
}

__device__ __forceinline__ void cp_async16(uint32_t smem_dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

}  // namespace
