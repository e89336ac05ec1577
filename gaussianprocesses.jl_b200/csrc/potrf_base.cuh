// potrf_base.cuh -- 128 x 128 diagonal-tile Cholesky + triangular inverse (see potrf_base.cu)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
// fused panel broadcast (multi-GPU): every output of the leaf is also stored into the peers' buffers (NVLink P2P)
struct PotrfPeers {
    int n;
    double* F[7];
    double* Dinv[7];
    double* DinvT[7];
    double* logd[7];
};
// tiles at diagonal offsets p0 + b*tile_stride, b < ntiles.  *info must be initialised to INT_MAX.
cudaError_t potrf128_launch(const double* G, int64_t ldg, double* F, int64_t ldf, double* Dinv, double* DinvT,
                            double* logd, int* info, int p0, int ntiles, int tile_stride, cudaStream_t st, int64_t* launches,
                            const PotrfPeers* peers = nullptr);
// pointer-table entry point (batched block-diagonal factorisation, fsa.cu): tile b of the launch reads the lower triangle of
// items[b].G and writes W = L^-1 (clean lower) to items[b].Dinv, W' (clean upper) to items[b].DinvT, all three with leading
// dimension items[b].ld, and 2 log L_jj to items[b].logd[j]; a non-positive pivot j records info_base + j + 1 (atomicMin,
// *info initialised to INT_MAX).  G may equal Dinv: the tile is read completely before anything is written.
struct Potrf128Item {
    const double* G;
    double* Dinv;
    double* DinvT;
    double* logd;
    long long ld;
    int info_base;
    int pad_;
};
cudaError_t potrf128_ptr_launch(const Potrf128Item* items, int n, int* info, cudaStream_t st, int64_t* launches);
