// gpb200.cu -- the dense engine (gpb200_handle) behind the C ABI of include/gpb200.h: device state, the blocked
// factorisation / inverse schedules, and their entry points.  The sparse handle (fitc_engine.cu, fsa_engine.cu) and the
// raw kernel entry points (kernel_contracts.cu) are separate units; engine.cuh lists what they share.
//
// Device layout (all FP64, row-major, leading dimension Npad = N rounded up to 128; the padding is
// an identity block, so L, L^-1, logdet and every solve are unaffected):
//   F     Npad x Npad   lower triangle: L (K_y = L L'; the reference's U = L', src/GP.jl:110).
//                       strict-upper tiles: scratch for the triangular-inverse merges.
//   G     Npad x Npad   lower tiles: K_y -> Schur complements during the factorisation ->
//                       W = L^-1 (strictly-lower tiles) ; strictly-upper tiles: W' ;
//                       after gpb200_grad_prepare the lower triangle holds K_y^-1.
//   Dinv / DinvT  Npad x 128   clean lower / upper copies of the inverted diagonal tiles.
//   x     N x d point-major (== Julia's d x N column-major), uploaded once (gpb200_set_data).
// The reference keeps four N x N host matrices per GPE (R, cK.mat, chol factors, ααinvcKI;
// test/memory.jl:14-19); this engine keeps two on the device and no distance cache.
//
// Every O(N^3) step is the NT DMMA GEMM of gemm_nt.cu:
//   Cholesky: recursive panel factorisation (chol_panel): leaf = potrf128 (tile factor + tile
//   inverse in one CTA) + a 128-wide TRSM GEMM through the inverted tile; every internal node is one
//   Schur-complement GEMM over a lower trapezoid with inner dimension = half the block, so ~98% of
//   the N^3/3 flops run with K >= 1024.  Option "nb" > 0 switches to a right-looking outer loop over
//   nb-wide panels (the form the multi-GPU block-column distribution uses).
//   Inverse: bottom-up *level-parallel* triangular inverse -- at level s every pair of adjacent
//   s x s diagonal blocks is merged independently, W21 = -W_C (L21 W_A), two batched GEMMs per
//   level, 2 log2(Npad/128) launches in total -- then K_y^-1 = W' W in ONE triangular SYRK launch.
//   N^3/3 + 2N^3/3 = N^3 flop per mll+gradient (the reference's potrs on the identity costs 7N^3/3).
#include <dlfcn.h>
#include <limits.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>

#include "engine.cuh"
#include "gram.cuh"
#include "gram_fast.cuh"
#include "potrf_base.cuh"
#include "shard_kernels.cuh"
#include "vec.cuh"
#include "gpa.cuh"

namespace engine __attribute__((visibility("hidden"))) {
std::string g_create_error;
NcclApi g_nccl;

bool nccl_load() {
    if (g_nccl.ok) return true;
    if (!g_nccl.lib) g_nccl.lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!g_nccl.lib) g_nccl.lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!g_nccl.lib) return false;
    void* L = g_nccl.lib;
    g_nccl.GetUniqueId = (decltype(g_nccl.GetUniqueId))dlsym(L, "ncclGetUniqueId");
    g_nccl.CommInitRank = (decltype(g_nccl.CommInitRank))dlsym(L, "ncclCommInitRank");
    g_nccl.CommDestroy = (decltype(g_nccl.CommDestroy))dlsym(L, "ncclCommDestroy");
    g_nccl.Broadcast = (decltype(g_nccl.Broadcast))dlsym(L, "ncclBroadcast");
    g_nccl.AllGather = (decltype(g_nccl.AllGather))dlsym(L, "ncclAllGather");
    g_nccl.AllReduce = (decltype(g_nccl.AllReduce))dlsym(L, "ncclAllReduce");
    g_nccl.GetErrorString = (decltype(g_nccl.GetErrorString))dlsym(L, "ncclGetErrorString");
    g_nccl.GroupStart = (decltype(g_nccl.GroupStart))dlsym(L, "ncclGroupStart");
    g_nccl.GroupEnd = (decltype(g_nccl.GroupEnd))dlsym(L, "ncclGroupEnd");
    g_nccl.ok = g_nccl.GetUniqueId && g_nccl.CommInitRank && g_nccl.CommDestroy && g_nccl.Broadcast &&
                g_nccl.AllGather && g_nccl.AllReduce && g_nccl.GetErrorString && g_nccl.GroupStart && g_nccl.GroupEnd;
    return g_nccl.ok;
}


// unmap every peer buffer imported by gpb200_ipc_import (a realloc or a re-import makes them stale)
void close_peer_maps(gpb200_handle* h) {
    for (int q = 0; q < h->n_peer; ++q) {
        cudaIpcCloseMemHandle(h->peer_F[q]); cudaIpcCloseMemHandle(h->peer_Dinv[q]);
        cudaIpcCloseMemHandle(h->peer_DinvT[q]); cudaIpcCloseMemHandle(h->peer_logd[q]);
        cudaIpcCloseMemHandle(h->peer_sig[q]);
        h->peer_F[q] = h->peer_Dinv[q] = h->peer_DinvT[q] = h->peer_logd[q] = nullptr; h->peer_sig[q] = nullptr;
    }
    (void)cudaGetLastError();
    h->p2p = false; h->n_peer = 0;
}

void free_FG(gpb200_handle* h);               // shard_impl.cuh: F / G are cudaMalloc'ed (replicated) or VMM ranges (row-sharded)

void free_data(gpb200_handle* h) {
    free_FG(h);
    h->xmap_ok = false;
    h->cvD.reset(); h->cvY.reset(); h->cvblk.reset(); h->cvidx.reset();
    h->g_sym = false; h->cv_m_ok = false;
    for (DevBuf<double>* b : {&h->x, &h->Dinv, &h->DinvT, &h->logd, &h->noise_var, &h->r0, &h->r1, &h->y1, &h->alpha, &h->scal,
                              &h->part, &h->trace_out, &h->xs, &h->Kst, &h->Kss, &h->pmu, &h->pvar, &h->pkdiag, &h->tblk, &h->xp,
                              &h->xpt, &h->ZdT, &h->pdx, &h->dxin})
        b->reset();
    h->info_dev.reset(); h->flags.reset();
    close_peer_maps(h);                        // peers' mappings refer to the old buffers whether or not p2p is switched on
    h->sig.reset(); h->peer_sig_dev.reset();
    h->pack[0].reset(); h->pack[1].reset();
    h->ag_send.reset(); h->ag_recv.reset();
    h->has_data = h->factored = h->inv_ready = h->s_ready = h->alpha_ready = false;
}


// flops the GEMM launch executes (tile-granular: whole 128x128 tiles, clipped k ranges)
double gemm_exec_flops(const GemmDesc& d) {
    double total = 0.0;
    for (int z = 0; z < d.batch; ++z) {
        const int zo = z * d.zstep;
        const int Mz = std::min(d.M, d.m_lim - zo), Nz = std::min(d.N, d.n_lim - zo), Kz = std::min(d.K, d.k_lim - zo);
        if (Mz <= 0 || Nz <= 0 || Kz <= 0) continue;
        const int tm = Mz / TILE, tn = Nz / TILE;
        for (int bm = 0; bm < tm; ++bm) {
            if (d.bm_mod > 1 && (((bm + d.bm_off) / (d.bm_div > 0 ? d.bm_div : 1)) % d.bm_mod) != d.bm_rem) continue;
            const int bn_hi = (d.flags & GEMM_LOWER_ONLY) ? std::min(bm + 1, tn) : tn;
            for (int bn = 0; bn < bn_hi; ++bn) {
                if (d.bn_mod > 1 && (((bn + d.bn_off) / (d.bn_div > 0 ? d.bn_div : 1)) % d.bn_mod) != d.bn_rem) continue;
                int lo = (d.flags & GEMM_KLO_M) ? d.klo_off + bm * TILE : 0;
                if (d.flags & GEMM_KLO_N) lo = std::max(lo, bn * TILE);
                int hi = Kz;
                if (d.flags & GEMM_KHI_M) hi = std::min(hi, (bm + 1) * TILE);
                if (d.flags & GEMM_KHI_N) hi = std::min(hi, (bn + 1) * TILE);
                if (hi > lo) total += 2.0 * TILE * TILE * (double)(hi - lo);
            }
        }
    }
    return total;
}

cudaError_t launch_gemm(gpb200_handle* h, const GemmDesc& d) {
    const int impl = h->tma_ok ? h->gemm_impl : 1;
    cudaStream_t stc = h->st_cur ? h->st_cur : h->st;
    if (!h->profile || stc != h->st) return gemm_nt_launch(d, impl, stc, &h->launches);
    if (h->pev_used + 2 > h->pev.size()) {
        const size_t old = h->pev.size();
        h->pev.resize(old + 512);
        for (size_t i = old; i < h->pev.size(); ++i) cudaEventCreate(&h->pev[i]);
    }
    cudaEventRecord(h->pev[h->pev_used++], h->st);
    cudaError_t e = gemm_nt_launch(d, impl, h->st, &h->launches);
    cudaEventRecord(h->pev[h->pev_used++], h->st);
    h->gemm_flops_exec += gemm_exec_flops(d);
    ++h->gemm_launches;
    return e;
}

cudaError_t gemm_whole(gpb200_handle* h, GemmBuf a, GemmBuf b, double* c, int64_t ldc, int64_t M, int64_t N, int64_t K,
                       double alpha, double beta, double* ct, int64_t ldct, int flags) {
    GemmDesc g = gemm_desc_default();
    g.A = GemmOperand{a, bufNone(), 0, 0};
    g.B = GemmOperand{b, bufNone(), 0, 0};
    g.C = c; g.ldc = ldc; g.M = (int)M; g.N = (int)N; g.K = (int)K;
    g.alpha = alpha; g.beta = beta;
    g.Ct = ct; g.ldct = ldct;
    g.flags = flags;
    return launch_gemm(h, g);
}

// after a stream sync: fold the recorded GEMM launch durations into ms[6..8] and reset
void profile_collect(gpb200_handle* h) {
    if (!h->profile) return;
    double tot = 0.0;
    for (size_t i = 0; i + 1 < h->pev_used; i += 2) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, h->pev[i], h->pev[i + 1]) == cudaSuccess) tot += ms;
    }
    h->ms[6] += (double)h->gemm_launches;
    h->ms[7] += tot;
    h->ms[8] += h->gemm_flops_exec;
    h->pev_used = 0; h->gemm_flops_exec = 0.0; h->gemm_launches = 0;
}

// ---- pieces of the factorisation --------------------------------------------------------------

// F[r0.., p..p+128) = G[r0.., p..p+128) * W_pp'   (leaf panel TRSM through the inverted diagonal tile)
cudaError_t panel_trsm_leaf(gpb200_handle* h, int r0, int rows, int p) {
    GemmDesc g = gemm_desc_default();
    g.A = GemmOperand{bufG(h), bufNone(), r0, p};
    g.B = GemmOperand{bufDinv(h), bufNone(), p, 0};
    g.C = h->F; g.ldc = h->ld; g.c_row0 = r0; g.c_col0 = p;
    g.M = rows; g.N = TILE; g.K = TILE;
    if (h->push_panel) {                       // fused broadcast: the epilogue also writes the peers' factor
        g.n_peer = h->n_peer;
        for (int q = 0; q < h->n_peer; ++q) g.Cpeer[q] = h->peer_F[q];
    }
    return launch_gemm(h, g);
}
// Schur update of the lower trapezoid G[r0.., r0..r0+cols) -= F[r0.., p..p+k) F[r0..r0+cols, p..p+k)'
// (rows >= cols; cols == rows gives the classical trailing SYRK)
cudaError_t schur_update(gpb200_handle* h, int r0, int rows, int cols, int p, int k, int extra_flags = 0) {
    GemmDesc g = gemm_desc_default();
    g.A = GemmOperand{bufF(h), bufNone(), r0, p};
    g.B = GemmOperand{bufF(h), bufNone(), r0, p};
    g.C = h->G; g.ldc = h->ld; g.c_row0 = r0; g.c_col0 = r0;
    g.M = rows; g.N = cols; g.K = k;
    g.alpha = -1.0; g.beta = 1.0;
    g.flags = GEMM_LOWER_ONLY | extra_flags;
    return launch_gemm(h, g);
}
// merge of the inverses of two adjacent diagonal blocks [p,p+n1) and [p+n1,p+n1+n2):
//   T' = Wt_A * L21'  -> F strict-upper block (p, p+n1)
//   W21 = -W_C * T    -> G (p+n1, p)  and its transpose -> G (p, p+n1)
// batched over `batch` problems stepping 2*n1 along the diagonal (clipped at Npad).
cudaError_t merge_inverse(gpb200_handle* h, int p, int n1, int n2, int batch) {
    const int lim = (int)h->Npad - p - n1;     // rows available below the first block of problem 0
    {
        GemmDesc g = gemm_desc_default();
        g.A = GemmOperand{bufG(h), bufDinvT(h), p, p};
        g.B = GemmOperand{bufF(h), bufNone(), p + n1, p};
        g.C = h->F; g.ldc = h->ld; g.c_row0 = p; g.c_col0 = p + n1;
        g.M = n1; g.N = n2; g.K = n1;
        g.flags = GEMM_KLO_M;
        g.batch = batch; g.zstep = 2 * n1;
        g.n_lim = lim;
        cudaError_t e = launch_gemm(h, g);
        if (e != cudaSuccess) return e;
    }
    {
        GemmDesc g = gemm_desc_default();
        g.A = GemmOperand{bufG(h), bufDinv(h), p + n1, p + n1};
        g.B = GemmOperand{bufF(h), bufNone(), p, p + n1};
        g.C = h->G; g.ldc = h->ld; g.c_row0 = p + n1; g.c_col0 = p;
        g.Ct = h->G; g.ldct = h->ld; g.ct_row0 = p; g.ct_col0 = p + n1;
        g.M = n2; g.N = n1; g.K = n2;
        g.alpha = -1.0;
        g.flags = GEMM_KHI_M;
        g.batch = batch; g.zstep = 2 * n1;
        g.m_lim = lim; g.k_lim = lim;
        return launch_gemm(h, g);
    }
}

// Recursive panel Cholesky: factor columns [p, p+n) for ALL rows below (n <= s, s = 128 * 2^k,
// p aligned to s).  Every Schur update inside is one NT GEMM whose inner dimension is the half
// block size, so ~98% of the flops run with K >= 1024 (near-peak DMMA activity); only the
// 128-wide leaves (tile factorisation + TRSM through the inverted tile) are latency bound.
cudaError_t leaf_launch(gpb200_handle* h, int p, cudaStream_t st) {
    PotrfPeers pp{};
    if (h->push_panel) {
        pp.n = h->n_peer;
        for (int q = 0; q < h->n_peer; ++q) { pp.F[q] = h->peer_F[q]; pp.Dinv[q] = h->peer_Dinv[q]; pp.DinvT[q] = h->peer_DinvT[q]; pp.logd[q] = h->peer_logd[q]; }
    }
    return potrf128_launch(h->G, h->ld, h->F, h->ld, h->Dinv, h->DinvT, h->logd, h->info_dev, p, 1, TILE, st, &h->launches, &pp);
}

// `leaf_done`: the tile at p was already factored by the look-ahead chain on the side stream (join it first).
// Look-ahead: once the left half of a node is done, the ONE tile of the Schur update the next leaf needs and
// that leaf run on a high-priority side stream while the main stream does the rest of the update -- the
// 125 us latency-bound leaf disappears behind the GEMM.
cudaError_t chol_panel(gpb200_handle* h, int p, int n, int s, bool leaf_done = false) {
    const int Np = h->row_lim > 0 ? h->row_lim : (int)h->Npad;
    cudaError_t e;
    if (s == TILE) {
        if (leaf_done) e = cudaStreamWaitEvent(h->st, h->ev_la2, 0);
        else e = leaf_launch(h, p, h->st);
        if (e != cudaSuccess) return e;
        const int below = Np - p - TILE;
        return below > 0 ? panel_trsm_leaf(h, p + TILE, below, p) : cudaSuccess;
    }
    const int hs = s / 2;
    if (n <= hs) return chol_panel(h, p, n, hs, leaf_done);
    if ((e = chol_panel(h, p, hs, hs, leaf_done)) != cudaSuccess) return e;
    const int rows = Np - p - hs, cols = n - hs;
    if (h->lookahead && h->st_side) {
        if ((e = cudaEventRecord(h->ev_la0, h->st)) != cudaSuccess) return e;
        if ((e = cudaStreamWaitEvent(h->st_side, h->ev_la0, 0)) != cudaSuccess) return e;
        h->st_cur = h->st_side;
        e = schur_update(h, p + hs, TILE, TILE, p, hs);                 // the next diagonal tile only
        h->st_cur = nullptr;
        if (e != cudaSuccess) return e;
        if ((e = leaf_launch(h, p + hs, h->st_side)) != cudaSuccess) return e;
        if ((e = cudaEventRecord(h->ev_la2, h->st_side)) != cudaSuccess) return e;
        if ((e = schur_update(h, p + hs, rows, cols, p, hs, GEMM_SKIP_FIRST)) != cudaSuccess) return e;
        return chol_panel(h, p + hs, cols, hs, true);
    }
    if ((e = schur_update(h, p + hs, rows, cols, p, hs)) != cudaSuccess) return e;
    return chol_panel(h, p + hs, cols, hs);
}

// right-looking outer loop over the columns from p0 on, `nb`-wide panels (0 = one panel spanning the rest: fully recursive)
cudaError_t cholesky(gpb200_handle* h, int p0, int nb) {
    const int Np = (int)h->Npad;
    int NB = TILE;
    const int want = nb > 0 ? nb : Np;
    while (NB < want && NB < Np) NB *= 2;
    cudaError_t e;
    for (int p = p0; p < Np; p += NB) {
        const int n = (Np - p < NB) ? Np - p : NB;
        if ((e = chol_panel(h, p, n, NB)) != cudaSuccess) return e;
        const int rem = Np - p - n;
        if (rem > 0 && (e = schur_update(h, p + n, rem, rem, p, n)) != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// W = L^-1 from the factor: level-parallel triangular inverse (all pairs of adjacent s x s diagonal blocks merged at once,
// s = 128, 256, ...: 2 batched GEMM launches per level).  Leaves W in G's strict-lower tiles and W' in its strict-upper tiles.
cudaError_t inverse_merges(gpb200_handle* h) {
    const int Np = (int)h->Npad;
    cudaError_t e;
    for (long long s = TILE; s < Np; s *= 2) {
        const int batch = (int)((Np + 2 * s - 1) / (2 * s));
        const int n2 = (int)((Np - s < s) ? Np - s : s);
        if ((e = merge_inverse(h, 0, (int)s, n2, batch)) != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// K_y^-1 from the factor: the merges, then W'W.
cudaError_t inverse_from_factor(gpb200_handle* h) {
    const int Np = (int)h->Npad;
    cudaError_t e;
    if ((e = inverse_merges(h)) != cudaSuccess) return e;
    GemmDesc g = gemm_desc_default();
    g.A = GemmOperand{bufG(h), bufDinvT(h), 0, 0};
    g.B = GemmOperand{bufG(h), bufDinvT(h), 0, 0};
    g.C = h->G; g.ldc = h->ld; g.c_row0 = 0; g.c_col0 = 0;
    g.M = Np; g.N = Np; g.K = Np;
    g.flags = GEMM_LOWER_ONLY | GEMM_KLO_M;
    return launch_gemm(h, g);
}


// ================================================================================================
// multi-GPU schedules (nranks > 1).  Storage is replicated (every rank holds full F, G, Dinv);
// WORK is partitioned:
//   Gram / Cholesky : 1-D block-cyclic ownership of dist_nb-wide block columns.  The owner factors
//                     its panel (chol_panel), the panel is broadcast (NCCL over NVLink, on a side
//                     stream, double-buffered), every rank applies it to the block columns it owns.
//                     The owner of the NEXT panel updates and factors that panel first and ships it
//                     before finishing its remaining updates (look-ahead), so the broadcast and the
//                     latency-bound panel factorisation hide behind the other ranks' updates.
//   inverse         : small levels of the level-parallel triangular inverse are recomputed on every
//                     rank; from block size 128*nranks upwards each merge is split by column slices
//                     of W21 (no exchange between its two GEMMs), then all-gathered.
//   W'W + trace     : tile rows dealt round-robin; only the P+1 partial sums are all-reduced, K^-1
//                     itself is never exchanged.
// ================================================================================================

int dist_block(gpb200_handle* h) {
    int NB = TILE;
    if (h->dist_nb > 0) { while (NB < h->dist_nb && NB < h->Npad) NB *= 2; return NB; }
    const long long target = h->Npad / (8LL * h->nranks);           // ~8 block columns per rank (measured best at 2/4/8 GPUs)
    while (NB * 2 <= target && NB < 4096) NB *= 2;
    return NB < 256 ? (h->Npad >= 256 ? 256 : TILE) : NB;
}

int dist_alloc(gpb200_handle* h) {
    const size_t Np = (size_t)h->Npad;
    const size_t nbw = (size_t)dist_block(h);
    const size_t need_pack = Np * nbw + 2 * nbw * TILE + nbw + 16;
    if (need_pack > h->pack[1].size())
        for (int i = 0; i < 2; ++i) CK(h->pack[i].alloc(need_pack));
    const size_t need_recv = Np * Np / 4 + Np * TILE;
    const size_t need_send = need_recv / h->nranks + Np * TILE;
    if (need_recv > h->ag_recv.size() || !h->ag_send) {  // ag_send, allocated last, is empty after any failure here
        h->ag_recv.reset(); h->ag_send.reset();
        CK(h->ag_recv.alloc(need_recv));
        CK(h->ag_send.alloc(need_send));
    }
    return GPB200_OK;
}

size_t panel_count(gpb200_handle* h, int p, int n) {
    return (size_t)(h->Npad - p) * n + 2 * (size_t)n * TILE + (size_t)n;
}
// F[p.., p..p+n) + Dinv/DinvT rows p..p+n + logd[p..p+n)  <->  contiguous staging buffer
cudaError_t panel_pack(gpb200_handle* h, int p, int n, double* buf, bool unpack) {
    const size_t rows = (size_t)(h->Npad - p);
    double* fpan = h->F + (size_t)p * h->ld + p;
    cudaError_t e;
    if (!unpack) e = cudaMemcpy2DAsync(buf, sizeof(double) * n, fpan, sizeof(double) * h->ld, sizeof(double) * n, rows, cudaMemcpyDeviceToDevice, h->st);
    else         e = cudaMemcpy2DAsync(fpan, sizeof(double) * h->ld, buf, sizeof(double) * n, sizeof(double) * n, rows, cudaMemcpyDeviceToDevice, h->st);
    if (e != cudaSuccess) return e;
    double* b1 = buf + rows * n;
    double* b2 = b1 + (size_t)n * TILE;
    double* b3 = b2 + (size_t)n * TILE;
    const size_t tb = sizeof(double) * (size_t)n * TILE;
    if (!unpack) {
        if ((e = cudaMemcpyAsync(b1, h->Dinv + (size_t)p * TILE, tb, cudaMemcpyDeviceToDevice, h->st)) != cudaSuccess) return e;
        if ((e = cudaMemcpyAsync(b2, h->DinvT + (size_t)p * TILE, tb, cudaMemcpyDeviceToDevice, h->st)) != cudaSuccess) return e;
        return cudaMemcpyAsync(b3, h->logd + p, sizeof(double) * n, cudaMemcpyDeviceToDevice, h->st);
    }
    if ((e = cudaMemcpyAsync(h->Dinv + (size_t)p * TILE, b1, tb, cudaMemcpyDeviceToDevice, h->st)) != cudaSuccess) return e;
    if ((e = cudaMemcpyAsync(h->DinvT + (size_t)p * TILE, b2, tb, cudaMemcpyDeviceToDevice, h->st)) != cudaSuccess) return e;
    return cudaMemcpyAsync(h->logd + p, b3, sizeof(double) * n, cudaMemcpyDeviceToDevice, h->st);
}

int cholesky_dist(gpb200_handle* h) {
    const int Np = (int)h->Npad, R = h->nranks, me = h->rank;
    const int NB = dist_block(h);
    const int nblk = (Np + NB - 1) / NB;
    auto bp = [&](int b) { return b * NB; };
    auto bn = [&](int b) { return std::min(NB, Np - b * NB); };
    auto owner = [&](int b) { return b % R; };
    auto update = [&](int jb, int b) {      // block column jb <- panel b
        const int r0 = bp(jb);
        return schur_update(h, r0, Np - r0, bn(jb), bp(b), bn(b));
    };
    // panel 0
    if (owner(0) == me) {
        CK(chol_panel(h, 0, bn(0), NB));
        CK(panel_pack(h, 0, bn(0), h->pack[0], false));
        CK(cudaEventRecord(h->ev_packed[0], h->st));
        CK(cudaStreamWaitEvent(h->st_comm, h->ev_packed[0], 0));
    }
    CKN(g_nccl.Broadcast(h->pack[0], h->pack[0], panel_count(h, 0, bn(0)), ncclDouble, owner(0), h->comm, h->st_comm));
    CK(cudaEventRecord(h->ev_bcast[0], h->st_comm));
    for (int b = 0; b < nblk; ++b) {
        const int cur = b & 1, nxt = cur ^ 1;
        CK(cudaStreamWaitEvent(h->st, h->ev_bcast[cur], 0));
        if (owner(b) != me) CK(panel_pack(h, bp(b), bn(b), h->pack[cur], true));
        CK(cudaEventRecord(h->ev_unpacked[cur], h->st));
        bool did_next = false;
        if (b + 1 < nblk) {
            if (owner(b + 1) == me) {                         // look-ahead: next panel first
                CK(update(b + 1, b));
                CK(chol_panel(h, bp(b + 1), bn(b + 1), NB));
                CK(panel_pack(h, bp(b + 1), bn(b + 1), h->pack[nxt], false));
                CK(cudaEventRecord(h->ev_packed[nxt], h->st));
                CK(cudaStreamWaitEvent(h->st_comm, h->ev_packed[nxt], 0));
                did_next = true;
            } else if (b >= 1) {
                CK(cudaStreamWaitEvent(h->st_comm, h->ev_unpacked[nxt], 0));   // staging buffer free again
            }
            CKN(g_nccl.Broadcast(h->pack[nxt], h->pack[nxt], panel_count(h, bp(b + 1), bn(b + 1)), ncclDouble,
                                 owner(b + 1), h->comm, h->st_comm));
            CK(cudaEventRecord(h->ev_bcast[nxt], h->st_comm));
        }
        for (int jb = b + 1 + (did_next ? 1 : 0); jb < nblk; ++jb)
            if (owner(jb) == me) CK(update(jb, b));
    }
    // first failing pivot over all ranks
    CK(cudaEventRecord(h->ev_x, h->st));
    CK(cudaStreamWaitEvent(h->st_comm, h->ev_x, 0));
    CKN(g_nccl.AllReduce(h->info_dev, h->info_dev, 1, ncclInt32, ncclMin, h->comm, h->st_comm));
    CK(cudaEventRecord(h->ev_y, h->st_comm));
    CK(cudaStreamWaitEvent(h->st, h->ev_y, 0));
    return GPB200_OK;
}

// Cholesky over block columns with the panel broadcast FUSED into the kernels that produce the panel:
// the tile leaf and the 128-wide TRSM GEMM store their outputs into every peer's F / Dinv / DinvT / logd
// through NVLink-mapped pointers (CUDA IPC), then one tiny kernel raises a flag word in each peer; the
// peers' streams wait on that word with a one-thread kernel.  No staging copy, no NCCL on the panel path.
int cholesky_dist_p2p(gpb200_handle* h) {
    const int Np = (int)h->Npad, R = h->nranks, me = h->rank;
    const int NB = dist_block(h);
    const int nblk = (Np + NB - 1) / NB;
    auto bp = [&](int b) { return b * NB; };
    auto bn = [&](int b) { return std::min(NB, Np - b * NB); };
    auto owner = [&](int b) { return b % R; };
    auto update = [&](int jb, int b) {
        const int r0 = bp(jb);
        return schur_update(h, r0, Np - r0, bn(jb), bp(b), bn(b));
    };
    // start barrier: no rank may push a new panel into a peer's factor while that peer still reads the
    // previous evaluation's factor (inverse / predict); also makes the rare epoch wrap safe
    if (++h->epoch >= 32000) { h->epoch = 1; CK(cudaMemsetAsync(h->sig, 0, sizeof(int) * 8, h->st)); }
    const int base = h->epoch * 65536;
    CK(cudaEventRecord(h->ev_x, h->st));
    CK(cudaStreamWaitEvent(h->st_comm, h->ev_x, 0));
    CKN(g_nccl.AllReduce(h->sig + 12, h->sig + 12, 1, ncclInt32, ncclSum, h->comm, h->st_comm));
    CK(cudaEventRecord(h->ev_y, h->st_comm));
    CK(cudaStreamWaitEvent(h->st, h->ev_y, 0));
    auto factor_and_publish = [&](int b) -> int {
        h->push_panel = true;
        cudaError_t e = chol_panel(h, bp(b), bn(b), NB);
        h->push_panel = false;
        CK(e);
        CK(shard_signal_peers(h->peer_sig_dev, h->n_peer, base + b + 1, h->st, &h->launches));
        return GPB200_OK;
    };
    if (owner(0) == me) { int rc = factor_and_publish(0); if (rc) return rc; }
    for (int b = 0; b < nblk; ++b) {
        if (owner(b) != me) {
            CK(shard_wait_signal(h->sig + owner(b), base + b + 1, h->sig + 8, h->st, &h->launches));
        }
        bool did_next = false;
        if (b + 1 < nblk && owner(b + 1) == me) {
            CK(update(b + 1, b));
            int rc = factor_and_publish(b + 1);
            if (rc) return rc;
            did_next = true;
        }
        for (int jb = b + 1 + (did_next ? 1 : 0); jb < nblk; ++jb)
            if (owner(jb) == me) CK(update(jb, b));
    }
    // first failing pivot over all ranks; also the barrier that keeps the next evaluation from overwriting
    // a panel a slower peer is still reading
    CK(cudaEventRecord(h->ev_x, h->st));
    CK(cudaStreamWaitEvent(h->st_comm, h->ev_x, 0));
    CKN(g_nccl.AllReduce(h->info_dev, h->info_dev, 1, ncclInt32, ncclMin, h->comm, h->st_comm));
    CK(cudaEventRecord(h->ev_y, h->st_comm));
    CK(cudaStreamWaitEvent(h->st, h->ev_y, 0));
    return GPB200_OK;
}

int inverse_dist(gpb200_handle* h) {
    const int Np = (int)h->Npad, R = h->nranks, me = h->rank;
    for (long long s = TILE; s < Np; s *= 2) {
        const int batch = (int)((Np + 2 * s - 1) / (2 * s));
        const int n2 = (int)((Np - s < s) ? Np - s : s);
        const int tiles = (int)(s / TILE);
        if (tiles < R || tiles % R) {                        // small level: recompute everywhere
            CK(merge_inverse(h, 0, (int)s, n2, batch));
            continue;
        }
        const int wr = (int)(s / R);
        const int lim = Np - (int)s;
        {   // T'[own tile rows, :] = Wt_A[own tile rows, :] * L21'
            GemmDesc g = gemm_desc_default();
            g.A = GemmOperand{bufG(h), bufDinvT(h), 0, 0};
            g.B = GemmOperand{bufF(h), bufNone(), (int)s, 0};
            g.C = h->F; g.ldc = h->ld; g.c_row0 = 0; g.c_col0 = (int)s;
            g.M = (int)s; g.N = n2; g.K = (int)s;
            g.flags = GEMM_KLO_M;
            g.bm_mod = R; g.bm_rem = me;
            g.batch = batch; g.zstep = 2 * (int)s; g.n_lim = lim;
            CK(launch_gemm(h, g));
        }
        {   // W21[:, own tile columns] = -W_C * (T'[own tile rows, :])'
            GemmDesc g = gemm_desc_default();
            g.A = GemmOperand{bufG(h), bufDinv(h), (int)s, (int)s};
            g.B = GemmOperand{bufF(h), bufNone(), 0, (int)s};
            g.C = h->G; g.ldc = h->ld; g.c_row0 = (int)s; g.c_col0 = 0;
            g.Ct = h->G; g.ldct = h->ld; g.ct_row0 = 0; g.ct_col0 = (int)s;
            g.M = n2; g.N = (int)s; g.K = n2;
            g.alpha = -1.0; g.flags = GEMM_KHI_M;
            g.bn_mod = R; g.bn_rem = me;
            g.batch = batch; g.zstep = 2 * (int)s; g.m_lim = lim; g.k_lim = lim;
            CK(launch_gemm(h, g));
        }
        // exchange the column slices
        long long rows_total = 0;                                   // sum over problems of n2_z (only the last is short)
        for (int z = 0; z < batch; ++z) rows_total += std::max(0LL, std::min((long long)s, (long long)Np - z * 2 * s - s));
        const long long per_rank = rows_total * wr;
        if ((size_t)per_rank > h->ag_send.size() || (size_t)per_rank * R > h->ag_recv.size())
            return fail(h, GPB200_ECUDA, "inverse_dist: exchange buffers too small");
        CK(shard_pack_slices(h->G, h->ld, h->ag_send, (int)s, R, me, Np, h->st, &h->launches));
        CK(cudaEventRecord(h->ev_x, h->st));
        CK(cudaStreamWaitEvent(h->st_comm, h->ev_x, 0));
        CKN(g_nccl.AllGather(h->ag_send, h->ag_recv, (size_t)per_rank, ncclDouble, h->comm, h->st_comm));
        CK(cudaEventRecord(h->ev_y, h->st_comm));
        CK(cudaStreamWaitEvent(h->st, h->ev_y, 0));
        CK(shard_unpack_slices(h->G, h->ld, h->ag_recv, per_rank, (int)s, R, me, Np, h->st, &h->launches));
    }
    // W'W on this rank's tile rows only (K^-1 stays distributed; the trace needs no more)
    GemmDesc g = gemm_desc_default();
    g.A = GemmOperand{bufG(h), bufDinvT(h), 0, 0};
    g.B = GemmOperand{bufG(h), bufDinvT(h), 0, 0};
    g.C = h->G; g.ldc = h->ld; g.c_row0 = 0; g.c_col0 = 0;
    g.M = Np; g.N = Np; g.K = Np;
    g.flags = GEMM_LOWER_ONLY | GEMM_KLO_M;
    g.bm_mod = R; g.bm_rem = me;
    CK(launch_gemm(h, g));
    return GPB200_OK;
}

// alpha-type solve on device vectors: out = K_y^-1 rhs ; rhs (Npad, zero padded) is destroyed
cudaError_t solve_device(gpb200_handle* h, double* rhs, double* tmp, double* out) {
    const int nb = (int)(h->Npad / TILE);
    // single-launch flag-synchronised solves: each CTA stages a 128 KB tile in dynamic shared memory, so one CTA fits per
    // SM.  Every wait points to a lower blockIdx, so for nb above the SM count correctness rests on in-order CTA dispatch
    // (a CTA waits only on CTAs dispatched before it, which run or have retired).  max_resident_ctas (TRSV_FUSED_CTAS_PER_SM
    // per SM) is a chosen limit on nb, not a residency count; above it the per-step schedule runs.
    if (h->trsv_fused && h->flags && nb <= h->max_resident_ctas) {
        cudaError_t e = trsv_lower_fwd_fused(h->F, h->ld, h->Dinv, rhs, tmp, h->Npad, h->flags, h->st, &h->launches);
        if (e != cudaSuccess) return e;
        return trsv_lower_bwd_fused(h->F, h->ld, h->DinvT, tmp, out, h->Npad, h->flags + nb + 1, h->st, &h->launches);
    }
    cudaError_t e = trsv_lower_fwd(h->F, h->ld, h->Dinv, rhs, tmp, h->Npad, h->st, &h->launches);
    if (e != cudaSuccess) return e;
    return trsv_lower_bwd(h->F, h->ld, h->DinvT, tmp, out, h->Npad, h->st, &h->launches);
}

// after a stream sync: did the watchdog of the single-launch solves fire?
int check_trsv_watchdog(gpb200_handle* h) {
    if (!h->trsv_fused || !h->flags) return GPB200_OK;
    const int nb = (int)(h->Npad / TILE);
    if (nb > h->max_resident_ctas) return GPB200_OK;
    int e[2] = {0, 0};
    CK(cudaMemcpy(&e[0], h->flags + nb, sizeof(int), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(&e[1], h->flags + 2 * nb + 1, sizeof(int), cudaMemcpyDeviceToHost));
    if (e[0] || e[1]) return fail(h, GPB200_ECUDA, "triangular solve watchdog fired (a ready-flag never arrived)");
    return GPB200_OK;
}

int upload_padded(gpb200_handle* h, double* dst, const double* src_host) {
    CK(cudaMemsetAsync(dst, 0, sizeof(double) * h->Npad, h->st));
    CK(cudaMemcpyAsync(dst, src_host, sizeof(double) * h->N, cudaMemcpyHostToDevice, h->st));
    return GPB200_OK;
}

int ensure_predict_ws(gpb200_handle* h, int64_t Mc, bool want_cov) {
    const int64_t Mpad = (Mc + TILE - 1) / TILE * TILE;
    if ((size_t)Mpad > h->pkdiag.size()) {          // pkdiag, allocated last, is empty after any failure here
        for (DevBuf<double>* b : {&h->xs, &h->pmu, &h->pvar, &h->pkdiag}) b->reset();
        CK(h->xs.alloc(Mpad * h->d));
        for (DevBuf<double>* b : {&h->pmu, &h->pvar, &h->pkdiag}) CK(b->alloc(Mpad));
    }
    if ((size_t)(Mpad * h->Npad) > h->Kst.size()) {
        CK(h->Kst.alloc(Mpad * h->Npad));
        if (h->tma_ok && !gemm_make_tensor_map(&h->mapKst, h->Kst, Mpad, h->Npad, h->Npad)) {
            h->Kst.reset();
            return fail(h, GPB200_ECUDA, "cuTensorMapEncodeTiled failed for the predict buffer");
        }
    }
    if (want_cov) CK(h->Kss.ensure(Mpad * Mpad));
    return GPB200_OK;
}

// Vt[:, c0..c0+n) <- solve against L[c0.., c0..] of handle h, in place on a row-major buffer
// (`rows` x h->Npad, leading dimension ldk): recursive blocked TRSM, leaves multiply by the inverted
// 128-tile, updates are NT GEMMs.  (whiten!, PDMats: x <- U^-T x.)
cudaError_t trsm_rec_buf(gpb200_handle* h, GemmBuf bk, int rows, int c0, int n) {
    double* kb = const_cast<double*>(bk.base);
    if (n == TILE) {
        GemmDesc g = gemm_desc_default();
        g.A = GemmOperand{bk, bufNone(), 0, c0};
        g.B = GemmOperand{bufDinv(h), bufNone(), c0, 0};
        g.C = kb; g.ldc = bk.ld; g.c_row0 = 0; g.c_col0 = c0;
        g.M = rows; g.N = TILE; g.K = TILE;
        return launch_gemm(h, g);
    }
    int n1 = TILE;
    while (n1 * 2 < n) n1 *= 2;
    const int n2 = n - n1;
    cudaError_t e;
    if ((e = trsm_rec_buf(h, bk, rows, c0, n1)) != cudaSuccess) return e;
    {
        GemmDesc g = gemm_desc_default();
        g.A = GemmOperand{bk, bufNone(), 0, c0};
        g.B = GemmOperand{bufF(h), bufNone(), c0 + n1, c0};
        g.C = kb; g.ldc = bk.ld; g.c_row0 = 0; g.c_col0 = c0 + n1;
        g.M = rows; g.N = n2; g.K = n1;
        g.alpha = -1.0; g.beta = 1.0;
        if ((e = launch_gemm(h, g)) != cudaSuccess) return e;
    }
    return trsm_rec_buf(h, bk, rows, c0 + n1, n2);
}
cudaError_t trsm_rec(gpb200_handle* h, int Mpad, int c0, int n) {
    const GemmBuf bk = gbuf(h, h->Kst, h->mapKst, h->Npad);
    return trsm_rec_buf(h, bk, Mpad, c0, n);
}

// Vt[:, c0..c0+n) <- Vt[:, c0..c0+n) L[c0.., c0..]^-1, the mirror of trsm_rec_buf: the second half is solved first, then
// X1 -= X2 L21 as an NT GEMM whose B operand is L21' -- rows of U = L' in F's strict-upper tiles, which the caller has filled
// (mirror_lower_tiles_launch) -- and the leaves multiply by DinvT = (L_tt^-1)'.
cudaError_t trsm_right_rec_buf(gpb200_handle* h, GemmBuf bk, int rows, int c0, int n) {
    double* kb = const_cast<double*>(bk.base);
    if (n == TILE) {
        GemmDesc g = gemm_desc_default();
        g.A = GemmOperand{bk, bufNone(), 0, c0};
        g.B = GemmOperand{bufDinvT(h), bufNone(), c0, 0};
        g.C = kb; g.ldc = bk.ld; g.c_row0 = 0; g.c_col0 = c0;
        g.M = rows; g.N = TILE; g.K = TILE;
        return launch_gemm(h, g);
    }
    int n1 = TILE;
    while (n1 * 2 < n) n1 *= 2;
    const int n2 = n - n1;
    cudaError_t e;
    if ((e = trsm_right_rec_buf(h, bk, rows, c0 + n1, n2)) != cudaSuccess) return e;
    {
        GemmDesc g = gemm_desc_default();
        g.A = GemmOperand{bk, bufNone(), 0, c0 + n1};
        g.B = GemmOperand{bufF(h), bufNone(), c0, c0 + n1};
        g.C = kb; g.ldc = bk.ld; g.c_row0 = 0; g.c_col0 = c0;
        g.M = rows; g.N = n1; g.K = n2;
        g.alpha = -1.0; g.beta = 1.0;
        if ((e = launch_gemm(h, g)) != cudaSuccess) return e;
    }
    return trsm_right_rec_buf(h, bk, rows, c0, n1);
}

float ev_ms(cudaEvent_t a, cudaEvent_t b) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, a, b);
    return ms;
}

// Gram build / gradient trace dispatch: the TMA-staged SEIso kernels (gram_fast.cu) when the kernel program is the single
// SEIso leaf over all (<= 8) input dimensions, else the generic kernel-program kernels (gram.cu)
bool use_seiso_fast(gpb200_handle* h, SeIsoFast* sf) {
    return h->gram_fast && kprog_fast(h->prog, h->d) && h->xmap_ok && h->xp && seiso_fast_prepare(h->prog.par[0], h->prog.par[1], sf);
}
cudaError_t launch_gram(gpb200_handle* h, double* G, int64_t ldg, int own_tiles, int nranks, int rank, int own_axis) {
    SeIsoFast sf;
    if (use_seiso_fast(h, &sf))
        return gram_seiso_tma_launch(&h->mapX, &h->mapXT, h->dxp, sf, h->N, h->Npad, h->noise_var, h->n_noise, h->nugget, G, ldg, h->st, &h->launches,
                                     own_tiles, nranks, rank, own_axis);
    return gram_lower_launch(h->prog, h->x, h->d, h->d, h->N, h->Npad, h->noise_var, h->n_noise, h->nugget, G, ldg, h->st, &h->launches,
                             own_tiles, nranks, rank, own_axis);
}
cudaError_t launch_trace(gpb200_handle* h, int bm_mod, int bm_rem, int bm_div) {
    SeIsoFast sf;
    if (use_seiso_fast(h, &sf))
        return trace_seiso_tma_launch(&h->mapX, &h->mapXT, h->dxp, sf, h->N, h->Npad, h->alpha, h->G, h->ld, h->part, h->trace_out, h->st, &h->launches,
                                      bm_mod, bm_rem, bm_div);
    return trace_launch(h->prog, h->x, h->d, h->d, h->N, h->Npad, h->alpha, h->G, h->ld, h->part, h->trace_out, h->st, &h->launches,
                        bm_mod, bm_rem, bm_div);
}

#include "shard_impl.cuh"

// collective entry points of a sharded handle: in an in-process group they must be called on the leader (it drives every
// virtual rank); per-rank state (host arguments) is replicated to every local handle here
int shard_entry(gpb200_handle* h, Locals& L) {
    L = locals(h);
    if (h->grp && L[0] != h) return fail(h, GPB200_ESTATE, "in-process group: call collective entry points on the leader (rank 0) handle");
    for (auto* q : L) q->err.clear();          // a message on any rank after this call comes from this call
    return GPB200_OK;
}
// debug getters with sharded storage: rows this rank owns, zeros elsewhere (the caller adds the ranks' pieces)
int copy_own_rows(gpb200_handle* h, double* dst_host, const double* src_dev) {
    const int64_t N = h->N;
    memset(dst_host, 0, sizeof(double) * (size_t)N * (size_t)N);
    for (int64_t t = 0; t * TILE < N; ++t) {
        if (owner_of_tile(h, t) != h->rank) continue;
        const int64_t r0 = t * TILE, nr = std::min<int64_t>(TILE, N - r0);
        CK(cudaMemcpy2DAsync(dst_host + r0 * N, sizeof(double) * N, src_dev + r0 * h->ld, sizeof(double) * h->ld, sizeof(double) * N, nr,
                             cudaMemcpyDeviceToHost, h->st));
    }
    return GPB200_OK;
}
int sync_all(const Locals& L) {
    for (auto* q : L) SCK(q, cudaStreamSynchronize(q->st));
    return GPB200_OK;
}

// Every factorisation schedule runs between these two.  factor_begin: no failing pivot yet on any rank (info = INT_MAX).
// factor_end: the first failing pivot is read on the leader once every rank has finished; `factored` of every rank follows
// it.  Returns GPB200_OK or the leading minor clipped to N, with "<what>matrix is not positive definite; ..." as the message.
int factor_begin(const Locals& L) {
    const int init = INT_MAX;
    for (auto* q : L) SCK(q, cudaMemcpyAsync(q->info_dev, &init, sizeof(int), cudaMemcpyHostToDevice, q->st));
    return GPB200_OK;
}
int factor_end(const Locals& L, const char* what, bool p2p_ran) {
    gpb200_handle* h = L[0];
    int info = 0;
    CK(cudaMemcpyAsync(&info, h->info_dev, sizeof(int), cudaMemcpyDeviceToHost, h->st));
    TRY(sync_all(L));
    for (auto* q : L) profile_collect(q);
    if (p2p_ran) {
        int wd = 0;
        CK(cudaMemcpy(&wd, h->sig + 8, sizeof(int), cudaMemcpyDeviceToHost));
        if (wd) return fail(h, GPB200_ECUDA, "panel signal watchdog fired (a peer never published its panel)");
    }
    for (auto* q : L) q->factored = info == INT_MAX;
    if (info == INT_MAX) return GPB200_OK;
    char buf[128];
    snprintf(buf, sizeof buf, "%smatrix is not positive definite; leading minor %d", what, info);
    h->err = buf;
    return info > h->N ? (int)h->N : info;
}

// factor whatever SPD matrix sits in the lower tiles of h->G (padding must be identity)
int chol_inplace(gpb200_handle* h) {
    h->factored = h->inv_ready = h->s_ready = h->alpha_ready = false;
    const Locals L{h};
    TRY(factor_begin(L));
    CK(cholesky(h, 0, h->nb));
    return factor_end(L, "", false);
}

// make_posdef!(Sigma; nugget), cholesky and unwhiten! of rand(gp, X, n) on h's stream, from Sigma (M x M, leading dimension
// ldc) and mu (M) on the device.  h owns the M x M sub-engine and the staging of the draws; the sub-engine's kernels are
// counted on h.  Events on h: ev0 before make_posdef!, ev1 after the Cholesky, ev3 / ev2 around unwhiten! + mu (the upload
// of z lies between ev1 and ev3).
int rand_from_cov(gpb200_handle* h, int64_t M, const double* cov, int64_t ldc, const double* mu, int64_t nsamp,
                  const double* z, double nugget, double* samples) {
    const int64_t Mpad = (M + TILE - 1) / TILE * TILE, Spad = (nsamp + TILE - 1) / TILE * TILE;
    int rc;
    // sub-engine of size M (shares this handle's stream)
    if (!h->sub) {
        rc = gpb200_create(&h->sub, h->device);
        if (rc) return fail(h, rc, "rand: could not create the M x M sub-engine");
        cudaStreamDestroy(h->sub->st);
        h->sub->own_stream = false;
    }
    gpb200_handle* sb = h->sub;
    sb->st = h->st;
    const int64_t sub_launches = sb->launches;
    if (!sb->has_data || sb->N != M) {
        std::vector<double> dummy((size_t)M, 0.0);
        rc = gpb200_set_data(sb, M, 1, dummy.data(), 1);
        if (rc) { h->err = "rand: " + sb->err; return rc; }
    }
    CK(cudaEventRecord(h->ev0, h->st));
    CK(spd_from_cov_launch(sb->G, sb->ld, cov, ldc, M, Mpad, nugget, h->st, &h->launches));
    rc = chol_inplace(sb);
    h->launches += sb->launches - sub_launches;                 // the sub-engine's kernels run for this call
    if (rc) { h->err = "rand: predictive covariance + nugget is not positive definite: " + sb->err; return rc; }
    CK(cudaEventRecord(h->ev1, h->st));
    // draws: Zt (nsamp x M, zero padded) on the device
    if (Spad > h->rz_rows || Mpad > h->rz_cols) {
        h->rz.reset(); h->rout.reset();
        h->rz_rows = h->rz_cols = 0;
        CK(h->rz.alloc(Spad * Mpad));
        CK(h->rout.alloc(Spad * Mpad));
        h->rz_rows = Spad; h->rz_cols = Mpad;
    }
    const int64_t ldz = h->rz_cols;
    if (h->tma_ok && !gemm_make_tensor_map(&h->mapRz, h->rz, h->rz_rows, ldz, ldz)) return fail(h, GPB200_ECUDA, "rand: tensor map");
    CK(cudaMemsetAsync(h->rz, 0, sizeof(double) * h->rz_rows * ldz, h->st));
    CK(cudaMemcpy2DAsync(h->rz, sizeof(double) * ldz, z, sizeof(double) * M, sizeof(double) * M, nsamp, cudaMemcpyHostToDevice, h->st));
    CK(cudaEventRecord(h->ev3, h->st));
    // out[s, m] = sum_{k <= m} Zt[s, k] L[m, k]       (unwhiten!: L Z)
    CK(gemm_whole(h, gbuf(h, h->rz, h->mapRz, ldz), bufF(sb), h->rout, ldz, Spad, Mpad, Mpad, 1.0, 0.0,
                  nullptr, 0, GEMM_KHI_N));
    CK(add_rowvec_launch(h->rout, ldz, mu, nsamp, M, h->st, &h->launches));                              // + mu
    CK(cudaEventRecord(h->ev2, h->st));
    CK(cudaMemcpy2DAsync(samples, sizeof(double) * M, h->rout, sizeof(double) * ldz, sizeof(double) * M, nsamp, cudaMemcpyDeviceToHost, h->st));
    CK(cudaStreamSynchronize(h->st));
    return GPB200_OK;
}

}  // namespace engine

using namespace engine;

// ================================================================================================
// C ABI
// ================================================================================================
extern "C" {

int gpb200_version(void) { return 100; }

const char* gpb200_last_error(gpb200_handle* h) { return h ? h->err.c_str() : g_create_error.c_str(); }

int gpb200_create(gpb200_handle** out, int device) {
    if (!out) return GPB200_EINVAL;
    *out = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count <= 0) {
        g_create_error = std::string("no CUDA device available (") + cudaGetErrorString(e) +
                         "); libgpb200 has no CPU fallback";
        (void)cudaGetLastError();
        return GPB200_ECUDA;
    }
    if (device < 0 || device >= count) { g_create_error = "device index out of range"; return GPB200_EINVAL; }
    gpb200_handle* h = new gpb200_handle();
    h->device = device;
    auto bail = [&](const char* what, cudaError_t ce) {
        g_create_error = std::string(what) + ": " + cudaGetErrorString(ce);
        delete h;
        return GPB200_ECUDA;
    };
    if ((e = cudaSetDevice(device)) != cudaSuccess) return bail("cudaSetDevice", e);
    if ((e = cudaStreamCreateWithFlags(&h->st, cudaStreamNonBlocking)) != cudaSuccess) return bail("cudaStreamCreate", e);
    cudaEventCreate(&h->ev0); cudaEventCreate(&h->ev1); cudaEventCreate(&h->ev2); cudaEventCreate(&h->ev3); cudaEventCreate(&h->ev4);
    cudaEventCreate(&h->ev5);
    {
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);
        if (cudaStreamCreateWithPriority(&h->st_side, cudaStreamNonBlocking, hi) != cudaSuccess) { h->st_side = nullptr; (void)cudaGetLastError(); }
        cudaEventCreateWithFlags(&h->ev_la0, cudaEventDisableTiming);
        cudaEventCreateWithFlags(&h->ev_la2, cudaEventDisableTiming);
    }
    if ((e = gemm_nt_init()) != cudaSuccess) return bail("gemm_nt_init", e);
    *out = h;
    return GPB200_OK;
}

void gpb200_destroy(gpb200_handle* h) {
    if (!h) return;
    cudaSetDevice(h->device);
    if (h->grp) {                              // a group dissolves with its first destroyed member
        gpb200_group* g = h->grp;
        for (auto* m : g->hs) { if (m->st) cudaStreamSynchronize(m->st); }
        for (auto* m : g->hs) {                 // the survivors become ordinary single-rank handles (storage re-allocated at their next factorize)
            m->grp = nullptr; m->nranks = 1; m->rank = 0;
            m->factored = m->inv_ready = m->s_ready = m->alpha_ready = false;
        }
        delete g;
    }
    if (h->st) cudaStreamSynchronize(h->st);
    if (h->sub) { h->sub->st = nullptr; h->sub->own_stream = false; gpb200_destroy(h->sub); h->sub = nullptr; }
    h->rz.reset(); h->rout.reset();
    free_data(h);
    for (auto e : h->evring) cudaEventDestroy(e);
    if (h->ev0) cudaEventDestroy(h->ev0);
    if (h->ev1) cudaEventDestroy(h->ev1);
    if (h->ev2) cudaEventDestroy(h->ev2);
    if (h->ev3) cudaEventDestroy(h->ev3);
    if (h->ev4) cudaEventDestroy(h->ev4);
    if (h->ev5) cudaEventDestroy(h->ev5);
    if (h->ev_la0) cudaEventDestroy(h->ev_la0);
    if (h->ev_la2) cudaEventDestroy(h->ev_la2);
    if (h->st_side) cudaStreamDestroy(h->st_side);
    for (auto e : h->pev) cudaEventDestroy(e);
    if (h->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(h->comm);
    for (int i = 0; i < 2; ++i) {
        if (h->ev_packed[i]) cudaEventDestroy(h->ev_packed[i]);
        if (h->ev_bcast[i]) cudaEventDestroy(h->ev_bcast[i]);
        if (h->ev_unpacked[i]) cudaEventDestroy(h->ev_unpacked[i]);
    }
    if (h->ev_x) cudaEventDestroy(h->ev_x);
    if (h->ev_y) cudaEventDestroy(h->ev_y);
    if (h->st_comm) cudaStreamDestroy(h->st_comm);
    if (h->st && h->own_stream) cudaStreamDestroy(h->st);
    delete h;
}

int gpb200_set_option(gpb200_handle* h, const char* key, int64_t value) {
    if (!h || !key) return GPB200_EINVAL;
    if (!strcmp(key, "nb")) {
        if (value != 0 && value != 128 && value != 256 && value != 512 && value != 1024 && value != 2048 && value != 4096)
            return fail(h, GPB200_EINVAL, "nb must be 0 (fully recursive) or 128 * 2^k <= 4096");
        h->nb = (int)value; h->factored = h->inv_ready = h->s_ready = false; return GPB200_OK;
    }
    if (!strcmp(key, "gemm")) { h->gemm_impl = value ? 1 : 0; return GPB200_OK; }
    if (!strcmp(key, "dist_nb")) {
        if (value != 0 && value != 128 && value != 256 && value != 512 && value != 1024 && value != 2048 && value != 4096)
            return fail(h, GPB200_EINVAL, "dist_nb must be 0 (auto) or 128 * 2^k <= 4096");
        h->dist_nb = (int)value; h->factored = h->inv_ready = h->s_ready = false; return GPB200_OK;
    }
    if (!strcmp(key, "lookahead")) { h->lookahead = value ? 1 : 0; return GPB200_OK; }
    if (!strcmp(key, "gram_fast")) { h->gram_fast = value ? 1 : 0; return GPB200_OK; }
    if (!strcmp(key, "capacity")) {             // rows reserved by the next gpb200_set_data (>= N): room for gpb200_append
        if (value < 0 || value > ((int64_t)1 << 30)) return fail(h, GPB200_EINVAL, "capacity out of range");
        h->capacity = value; return GPB200_OK;
    }
    if (!strcmp(key, "shard")) {                // storage of F / G with several ranks: -1 auto, 0 replicated, 1 row-sharded
        if (value < -1 || value > 1) return fail(h, GPB200_EINVAL, "shard must be -1 (auto), 0 or 1");
        h->shard_opt = (int)value; h->factored = h->inv_ready = h->s_ready = false; return GPB200_OK;
    }
    if (!strcmp(key, "shard_rb")) {             // ownership block of the row-sharded storage in 128-row tiles (panel = 128 * rb)
        if (value != 0 && value != 1 && value != 2 && value != 4 && value != 8) return fail(h, GPB200_EINVAL, "shard_rb must be 0 (auto), 1, 2, 4 or 8");
        h->shard_rb_opt = (int)value; h->factored = h->inv_ready = h->s_ready = false; return GPB200_OK;
    }
    if (!strcmp(key, "trsv_fused")) {            // 0: one launch per block step; 1 (default): single-launch kernels
        if (value != 0 && value != 1) return fail(h, GPB200_EINVAL, "trsv_fused must be 0 or 1");
        h->trsv_fused = (int)value; return GPB200_OK;
    }
    if (!strcmp(key, "p2p")) {                 // 0: NCCL panel broadcast even if peer memory is mapped
        if (value && h->n_peer == 0) return fail(h, GPB200_ESTATE, "p2p: ipc_import first");
        h->p2p = value != 0; return GPB200_OK;
    }
    if (!strcmp(key, "profile")) {
        h->profile = value ? 1 : 0;
        h->ms[6] = h->ms[7] = h->ms[8] = 0.0;
        h->pev_used = 0; h->gemm_flops_exec = 0.0; h->gemm_launches = 0;
        return GPB200_OK;
    }
    return fail(h, GPB200_EINVAL, "unknown option");
}

int64_t gpb200_launch_count(gpb200_handle* h) { return h ? h->launches : 0; }
int64_t gpb200_device_bytes(void) { return g_device_bytes.load(); }

int gpb200_set_stream(gpb200_handle* h, void* stream) {
    if (!h) return GPB200_EINVAL;
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->st));
    if (h->own_stream && h->st) cudaStreamDestroy(h->st);
    if (stream) { h->st = (cudaStream_t)stream; h->own_stream = false; }
    else {
        h->st = nullptr;
        CK(cudaStreamCreateWithFlags(&h->st, cudaStreamNonBlocking));
        h->own_stream = true;
    }
    return GPB200_OK;
}

int gpb200_get_timings(gpb200_handle* h, double* ms, int32_t n) {
    if (!h || !ms) return GPB200_EINVAL;
    for (int i = 0; i < n && i < 17; ++i) ms[i] = h->ms[i];
    return GPB200_OK;
}

int gpb200_set_data(gpb200_handle* h, int64_t N, int32_t d, const double* x, int64_t ldx) {
    if (!h) return GPB200_EINVAL;
    if (N <= 0 || d <= 0 || !x || ldx < d) return fail(h, GPB200_EINVAL, "set_data: bad N, d, x or ldx");
    if (d > GPB200_MAX_DIMS) return fail(h, GPB200_EINVAL, "set_data: d exceeds GPB200_MAX_DIMS");
    if (N > (int64_t)1 << 30) return fail(h, GPB200_EINVAL, "set_data: N too large");
    CK(cudaSetDevice(h->device));
    const int64_t Npad = (std::max<int64_t>(N, h->capacity) + TILE - 1) / TILE * TILE;
    const bool realloc = !h->has_data || Npad != h->Npad || d != h->d;
    if (realloc) {
        free_data(h);
        h->N = N; h->Npad = Npad; h->ld = Npad; h->d = d;
        CK(h->x.alloc(Npad * d));                    // Npad rows: N may grow up to Npad without realloc
        CK(h->Dinv.alloc(Npad * TILE));
        CK(h->DinvT.alloc(Npad * TILE));
        for (DevBuf<double>* b : {&h->logd, &h->noise_var, &h->r0, &h->r1, &h->y1, &h->alpha, &h->tblk}) CK(b->alloc(Npad));
        CK(h->scal.alloc(16));
        CK(h->info_dev.alloc(1));
        CK(h->flags.alloc(2 * (Npad / TILE + 1)));
        CK(h->sig.alloc(16));
        CK(cudaMemsetAsync(h->sig, 0, sizeof(int) * 16, h->st));
        {
            int sms = 0;
            CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device));
            // a chosen limit on the block count of the single-launch solves, not a residency count: one CTA fits per
            // SM, and above the SM count the schedule relies on in-order CTA dispatch (see solve_device)
            h->max_resident_ctas = sms * TRSV_FUSED_CTAS_PER_SM;
        }
        const int64_t T = Npad / TILE;
        CK(h->part.alloc((size_t)(T * (T + 1) / 2) * (GPB200_MAX_THETA + 1)));
        CK(h->trace_out.alloc(GPB200_MAX_THETA + 1));
        // F / G: replicated (cudaMalloc) or row-sharded (virtual range, owned rows mapped) -- decided by the communicator,
        // the problem size and option "shard"; re-checked at every factorize (the communicator may be joined later)
        int rc_fg = ensure_storage(h);
        if (rc_fg != GPB200_OK) return rc_fg;
    }
    h->N = N;
    // x arrives as Julia's d x N column-major (ld = ldx): point i is the contiguous run x[i*ldx .. +d)
    CK(cudaMemcpy2DAsync(h->x, sizeof(double) * d, x, sizeof(double) * ldx, sizeof(double) * d, N,
                         cudaMemcpyHostToDevice, h->st));
    // second copy with an even row length for the TMA-staged SEIso kernels (row pitch must be a multiple of 16 bytes)
    h->xmap_ok = false;
    if (d <= 8) {
        h->dxp = (d + 1) / 2 * 2;
        if (!h->xp) CK(h->xp.alloc(Npad * h->dxp));
        CK(cudaMemsetAsync(h->xp, 0, sizeof(double) * Npad * h->dxp, h->st));
        CK(cudaMemcpy2DAsync(h->xp, sizeof(double) * h->dxp, x, sizeof(double) * ldx, sizeof(double) * d, N,
                             cudaMemcpyHostToDevice, h->st));
        if (!h->xpt) CK(h->xpt.alloc(Npad * h->dxp));
        CK(shard_transpose(h->xpt, Npad, h->xp, h->dxp, Npad, h->dxp, h->st, &h->launches));
        h->xmap_ok = seiso_make_x_maps(&h->mapX, &h->mapXT, h->xp, h->xpt, h->dxp, N, Npad);
    }
    CK(cudaStreamSynchronize(h->st));
    h->has_data = true;
    h->factored = h->inv_ready = h->s_ready = h->alpha_ready = false;
    // a kernel program that reads a dimension the new points do not have is dropped: factorize then asks for set_kernel
    for (int i = 0; h->has_kernel && i < GPB200_MAX_DIMS; ++i)
        if (h->prog.dims[i] >= d) h->has_kernel = false;
    return GPB200_OK;
}

int gpb200_set_kernel(gpb200_handle* h, int32_t n_ops, const int32_t* ops, int32_t n_dims, const int32_t* dims,
                      int32_t n_theta) {
    if (!h) return GPB200_EINVAL;
    if (n_ops <= 0 || n_ops > GPB200_MAX_OPS || !ops) return fail(h, GPB200_EINVAL, "set_kernel: bad n_ops");
    if (n_theta < 0 || n_theta > GPB200_MAX_THETA) return fail(h, GPB200_EINVAL, "set_kernel: too many parameters");
    if (n_dims < 0 || n_dims > GPB200_MAX_DIMS || (n_dims > 0 && !dims)) return fail(h, GPB200_EINVAL, "set_kernel: bad dims");
    KProg P{};
    P.n_ops = n_ops; P.n_theta = n_theta;
    int stack[GPB200_MAX_OPS]; int sp = 0; int tcount = 0;
    for (int q = 0; q < n_ops; ++q) {
        const int32_t* o = ops + q * GPB200_OP_STRIDE;
        P.op[q] = o[0]; P.toff[q] = o[1]; P.nth[q] = o[2]; P.doff[q] = o[3]; P.nd[q] = o[4]; P.extra[q] = o[5];
        if (o[0] == GPB200_OP_SUM || o[0] == GPB200_OP_PROD) {
            if (sp < 2) return fail(h, GPB200_EINVAL, "set_kernel: malformed program (stack underflow)");
            const int right = stack[--sp]; const int left = stack[--sp];
            if (right != q - 1) return fail(h, GPB200_EINVAL, "set_kernel: program is not in post-order");
            P.left[q] = left; P.nth[q] = 0;
            stack[sp++] = q;
        } else {
            if (o[0] < GPB200_OP_SE_ISO || o[0] > GPB200_OP_CONST) return fail(h, GPB200_EINVAL, "set_kernel: unknown opcode");
            if (o[1] < 0 || o[2] < 0 || o[1] + o[2] > n_theta) return fail(h, GPB200_EINVAL, "set_kernel: theta range");
            if (o[3] < 0 || o[4] < 0 || o[3] + o[4] > n_dims) return fail(h, GPB200_EINVAL, "set_kernel: dims range");
            int expect = -1;
            switch (o[0]) {
            case GPB200_OP_SE_ISO: case GPB200_OP_MAT12_ISO: case GPB200_OP_MAT32_ISO: case GPB200_OP_MAT52_ISO:
            case GPB200_OP_POLY: expect = 2; break;
            case GPB200_OP_SE_ARD: case GPB200_OP_MAT12_ARD: case GPB200_OP_MAT32_ARD: case GPB200_OP_MAT52_ARD:
                expect = o[4] + 1; break;
            case GPB200_OP_RQ_ISO: case GPB200_OP_PERIODIC: expect = 3; break;
            case GPB200_OP_RQ_ARD: expect = o[4] + 2; break;
            case GPB200_OP_LIN_ISO: case GPB200_OP_NOISE: case GPB200_OP_CONST: expect = 1; break;
            case GPB200_OP_LIN_ARD: expect = o[4]; break;
            }
            if (o[2] != expect) return fail(h, GPB200_EINVAL, "set_kernel: wrong parameter count for a leaf");
            tcount += o[2];
            stack[sp++] = q;
        }
    }
    if (sp != 1 || tcount != n_theta) return fail(h, GPB200_EINVAL, "set_kernel: malformed program");
    for (int i = 0; i < n_dims; ++i) {
        if (dims[i] < 0 || (h->has_data && dims[i] >= h->d)) return fail(h, GPB200_EINVAL, "set_kernel: dim index out of range");
        P.dims[i] = dims[i];
    }
    // single SEIso leaf over dims 0..nd-1: specialised kernels whenever nd is the input dimension (kprog_fast)
    P.fast = 0;
    if (n_ops == 1 && P.op[0] == GPB200_OP_SE_ISO) {
        bool ident = true;
        for (int i = 0; i < P.nd[0]; ++i) ident = ident && (P.dims[P.doff[0] + i] == i);
        P.fast = ident ? 1 : 0;
    }
    h->prog = P;
    h->theta.assign(n_theta, 0.0);
    h->has_kernel = true;
    h->factored = h->inv_ready = h->s_ready = false;
    return GPB200_OK;
}

int gpb200_factorize(gpb200_handle* h, const double* theta, const double* log_noise, int64_t n_noise,
                     double extra_nugget) {
    if (!h) return GPB200_EINVAL;
    if (!h->has_data || !h->has_kernel) return fail(h, GPB200_ESTATE, "factorize: set_data and set_kernel first");
    if ((h->prog.n_theta > 0 && !theta) || !log_noise) return fail(h, GPB200_EINVAL, "factorize: null theta/log_noise");
    if (n_noise != 1 && n_noise != h->N) return fail(h, GPB200_EINVAL, "factorize: n_noise must be 1 or N");
    for (int i = 0; i < h->prog.n_theta; ++i)
        if (!isfinite(theta[i])) return fail(h, GPB200_EINVAL, "factorize: non-finite hyper-parameter");
    CK(cudaSetDevice(h->device));
    h->factored = h->inv_ready = h->s_ready = h->alpha_ready = false; h->g_sym = false; h->cv_m_ok = false;
    std::vector<double> nv((size_t)n_noise);
    for (int64_t i = 0; i < n_noise; ++i) {
        if (!isfinite(log_noise[i])) return fail(h, GPB200_EINVAL, "factorize: non-finite logNoise");
        nv[i] = exp(2.0 * log_noise[i]);
    }
    Locals L;
    { int rc = shard_entry(h, L); if (rc) return rc; }
    for (auto* q : L) TRY(rank_failed(q, ensure_storage(q)));
    for (auto* q : L) {                                    // (an in-process group: every virtual rank gets the arguments)
        if (!q->has_data || !q->has_kernel || q->prog.n_theta != h->prog.n_theta || q->N != h->N)
            return fail(h, GPB200_ESTATE, "factorize: every handle of the group needs the same set_data / set_kernel");
        q->factored = q->inv_ready = q->s_ready = q->alpha_ready = false;
        for (int i = 0; i < q->prog.n_theta; ++i) q->theta[i] = theta[i];
        kprog_set_theta(q->prog, theta);
        SCK(q, cudaMemcpyAsync(q->noise_var, nv.data(), sizeof(double) * n_noise, cudaMemcpyHostToDevice, q->st));
        q->n_noise = n_noise; q->nugget = extra_nugget;
    }
    TRY(factor_begin(L));
    CK(cudaEventRecord(h->ev0, h->st));
    if (h->sharded) {
        // row-sharded storage: own rows of the Gram matrix, then the all-gathered-panel Cholesky (shard_impl.cuh)
        for (auto* q : L) SCK(q, launch_gram(q, q->G, q->ld, q->rb, q->nranks, q->rank, 1));
        CK(cudaEventRecord(h->ev1, h->st));
        TRY(shard_cholesky_la(L));
    } else if (h->nranks > 1) {
        TRY(dist_alloc(h));
        CK(launch_gram(h, h->G, h->ld, dist_block(h) / TILE, h->nranks, h->rank, 0));
        CK(cudaEventRecord(h->ev1, h->st));
        TRY(h->p2p ? cholesky_dist_p2p(h) : cholesky_dist(h));
    } else {
        CK(launch_gram(h, h->G, h->ld, 0, 1, 0, 0));
        CK(cudaEventRecord(h->ev1, h->st));
        CK(cholesky(h, 0, h->nb));
    }
    CK(cudaEventRecord(h->ev2, h->st));
    const int rc = factor_end(L, "", !h->sharded && h->p2p);
    h->ms[0] = ev_ms(h->ev0, h->ev1);
    h->ms[1] = ev_ms(h->ev1, h->ev2);
    return rc;
}

int gpb200_logdet(gpb200_handle* h, double* logdet) {
    if (!h || !logdet) return GPB200_EINVAL;
    if (!h->factored) return fail(h, GPB200_ESTATE, "logdet: factorize first");
    CK(cudaSetDevice(h->device));
    CK(sum_launch(h->logd, h->Npad, h->scal, h->st, &h->launches));
    CK(cudaMemcpyAsync(logdet, h->scal, sizeof(double), cudaMemcpyDeviceToHost, h->st));
    CK(cudaStreamSynchronize(h->st));
    return GPB200_OK;
}

int gpb200_solve(gpb200_handle* h, const double* rhs, double* out) {
    if (!h || !rhs || !out) return GPB200_EINVAL;
    if (!h->factored) return fail(h, GPB200_ESTATE, "solve: factorize first");
    CK(cudaSetDevice(h->device));
    if (h->sharded) {
        Locals L;
        { int rc = shard_entry(h, L); if (rc) return rc; }
        for (auto* q : L) TRY(rank_failed(q, upload_padded(q, q->r1, rhs)));
        TRY(shard_solve(L, &gpb200_handle::r1, &gpb200_handle::y1, &gpb200_handle::r0));
        CK(cudaMemcpyAsync(out, h->r0, sizeof(double) * h->N, cudaMemcpyDeviceToHost, h->st));
        return sync_all(L);
    }
    int rc = upload_padded(h, h->r1, rhs);
    if (rc) return rc;
    CK(solve_device(h, h->r1, h->y1, h->r0));
    CK(cudaMemcpyAsync(out, h->r0, sizeof(double) * h->N, cudaMemcpyDeviceToHost, h->st));
    CK(cudaStreamSynchronize(h->st));
    return check_trsv_watchdog(h);
}

int gpb200_mll(gpb200_handle* h, const double* y_minus_mean, double* alpha, double* mll) {
    if (!h || !y_minus_mean || !mll) return GPB200_EINVAL;
    if (!h->factored) return fail(h, GPB200_ESTATE, "mll: factorize first");
    CK(cudaSetDevice(h->device));
    CK(cudaEventRecord(h->ev0, h->st));
    Locals Ls;
    if (h->sharded) { int rc = shard_entry(h, Ls); if (rc) return rc; }
    int rc = upload_padded(h, h->r0, y_minus_mean);
    if (rc) return rc;
    if (h->sharded) {
        for (auto* q : Ls) if (q != h) TRY(rank_failed(q, upload_padded(q, q->r0, y_minus_mean)));
        TRY(shard_solve(Ls, &gpb200_handle::r0, &gpb200_handle::y1, &gpb200_handle::alpha));
        for (auto* q : Ls) q->alpha_ready = true;
    } else {
        CK(cudaMemcpyAsync(h->r1, h->r0, sizeof(double) * h->Npad, cudaMemcpyDeviceToDevice, h->st));
        CK(solve_device(h, h->r1, h->y1, h->alpha));
    }
    CK(dot_launch(h->r0, h->alpha, h->Npad, h->scal + 0, h->st, &h->launches));
    CK(sum_launch(h->logd, h->Npad, h->scal + 1, h->st, &h->launches));
    double s[2];
    CK(cudaMemcpyAsync(s, h->scal, sizeof(double) * 2, cudaMemcpyDeviceToHost, h->st));
    if (alpha) CK(cudaMemcpyAsync(alpha, h->alpha, sizeof(double) * h->N, cudaMemcpyDeviceToHost, h->st));
    CK(cudaEventRecord(h->ev1, h->st));
    CK(cudaStreamSynchronize(h->st));
    if (h->sharded) TRY(sync_all(Ls));
    h->ms[2] = ev_ms(h->ev0, h->ev1);
    if (!h->sharded) { int rcw = check_trsv_watchdog(h); if (rcw) return rcw; }
    *mll = -(s[0] + s[1] + LOG2PI * (double)h->N) / 2.0;    // src/GPE.jl:210
    h->alpha_ready = true;
    return GPB200_OK;
}

int gpb200_grad_prepare(gpb200_handle* h) {
    if (!h) return GPB200_EINVAL;
    if (!h->factored) return fail(h, GPB200_ESTATE, "grad_prepare: factorize first");
    if (h->inv_ready) return GPB200_OK;
    h->g_sym = false; h->cv_m_ok = false; h->s_ready = false;
    CK(cudaSetDevice(h->device));
    CK(cudaEventRecord(h->ev0, h->st));
    if (h->sharded) {
        Locals L;
        { int rc = shard_entry(h, L); if (rc) return rc; }
        TRY(shard_inverse_la(L));
        CK(cudaEventRecord(h->ev1, h->st));
        TRY(sync_all(L));
        for (auto* q : L) { profile_collect(q); q->inv_ready = true; }
        h->ms[3] = ev_ms(h->ev0, h->ev1);
        return GPB200_OK;
    }
    if (h->nranks > 1) { int rc = inverse_dist(h); if (rc) return rc; }
    else CK(inverse_from_factor(h));
    CK(cudaEventRecord(h->ev1, h->st));
    CK(cudaStreamSynchronize(h->st));
    profile_collect(h);
    h->ms[3] = ev_ms(h->ev0, h->ev1);
    h->inv_ready = true;
    return GPB200_OK;
}

int gpb200_grad_kernel(gpb200_handle* h, const double* alpha, double* dmll_kernel, double* trA) {
    if (!h) return GPB200_EINVAL;
    if (!h->inv_ready) return fail(h, GPB200_ESTATE, "grad_kernel: grad_prepare first");
    if (!alpha && !h->alpha_ready) return fail(h, GPB200_ESTATE, "grad_kernel: no alpha (call mll or pass alpha)");
    CK(cudaSetDevice(h->device));
    Locals Lg;
    if (h->sharded) { int rc = shard_entry(h, Lg); if (rc) return rc; } else Lg = Locals{h};
    if (alpha) {
        for (auto* q : Lg) {
            TRY(rank_failed(q, upload_padded(q, q->alpha, alpha)));
            q->alpha_ready = true;
        }
    }
    CK(cudaEventRecord(h->ev0, h->st));
    if (h->sharded) {
        // fused trace over the own rows of K^-1 (block-cyclic tile rows), P+1 partial sums summed over the ranks
        for (auto* q : Lg) SCK(q, launch_trace(q, q->nranks, q->rank, q->rb));
        TRY(coll_allreduce_sum(Lg, [&](gpb200_handle* q) { return q->trace_out.data(); }, (size_t)trace_num_acc(h->prog, h->d)));
    } else {
        CK(launch_trace(h, h->nranks, h->rank, 1));
    }
    if (!h->sharded && h->nranks > 1) {                    // P+1 partial sums, summed over ranks
        CK(cudaEventRecord(h->ev_x, h->st));
        CK(cudaStreamWaitEvent(h->st_comm, h->ev_x, 0));
        CKN(g_nccl.AllReduce(h->trace_out, h->trace_out, (size_t)trace_num_acc(h->prog, h->d), ncclDouble, ncclSum, h->comm, h->st_comm));
        CK(cudaEventRecord(h->ev_y, h->st_comm));
        CK(cudaStreamWaitEvent(h->st, h->ev_y, 0));
    }
    CK(cudaEventRecord(h->ev1, h->st));
    const int np = h->prog.n_theta;
    std::vector<double> out((size_t)np + 1);
    CK(cudaMemcpyAsync(out.data(), h->trace_out, sizeof(double) * (np + 1), cudaMemcpyDeviceToHost, h->st));
    CK(cudaStreamSynchronize(h->st));
    if (h->sharded) TRY(sync_all(Lg));
    h->ms[4] = ev_ms(h->ev0, h->ev1);
    if (dmll_kernel) for (int p = 0; p < np; ++p) dmll_kernel[p] = out[p];
    if (trA) *trA = out[np];
    return GPB200_OK;
}

// ---- GPA (src/GPA.jl): whitened latent variables f = L v + mu, gradient through the Cholesky factor ------------------------
static int gpa_check(gpb200_handle* h, const char* who) {
    if (h->nranks > 1 || h->sharded || h->grp) return fail(h, GPB200_EINVAL, (std::string(who) + ": single-GPU handles only").c_str());
    if (!h->factored) return fail(h, GPB200_ESTATE, (std::string(who) + ": factorize first").c_str());
    return GPB200_OK;
}

int gpb200_unwhiten(gpb200_handle* h, const double* v, double* f) {
    if (!h) return GPB200_EINVAL;
    if (!v || !f) return fail(h, GPB200_EINVAL, "unwhiten: null v or f");
    int rc = gpa_check(h, "unwhiten");
    if (rc) return rc;
    CK(cudaSetDevice(h->device));
    if ((rc = upload_padded(h, h->r0, v))) return rc;
    CK(gpa_trmv_launch(h->F, h->ld, h->r0, h->y1, h->Npad, h->st, &h->launches));
    CK(cudaMemcpyAsync(f, h->y1, sizeof(double) * h->N, cudaMemcpyDeviceToHost, h->st));
    CK(cudaStreamSynchronize(h->st));
    return GPB200_OK;
}

// u = L' g; then, for the kernel gradient, W = L^-1 (the inverse merges), Z' by the scans of gpa.cu, G_lower = -S = -W' Z (one
// NT GEMM with the k range of K^-1 = W'W), and the trace kernels with alpha = 0 (A = alpha alpha' - G = S): 1/2 sum S dK.
int gpb200_gpa_grad(gpb200_handle* h, const double* v, const double* dl_df, double* dll_process, double* dll_kernel) {
    if (!h) return GPB200_EINVAL;
    if (!v || !dl_df) return fail(h, GPB200_EINVAL, "gpa_grad: null v or dl_df");
    int rc = gpa_check(h, "gpa_grad");
    if (rc) return rc;
    CK(cudaSetDevice(h->device));
    if ((rc = upload_padded(h, h->r0, v))) return rc;
    if ((rc = upload_padded(h, h->r1, dl_df))) return rc;
    CK(gpa_trmv_t_launch(h->F, h->ld, h->r1, h->y1, h->Npad, h->st, &h->launches));
    if (dll_process) CK(cudaMemcpyAsync(dll_process, h->y1, sizeof(double) * h->N, cudaMemcpyDeviceToHost, h->st));
    if (!dll_kernel) {
        CK(cudaStreamSynchronize(h->st));
        return GPB200_OK;
    }
    // G and F's strict-upper tiles are overwritten: K^-1, its mirror, M_j and alpha are gone
    h->inv_ready = h->s_ready = h->alpha_ready = false; h->g_sym = false; h->cv_m_ok = false;
    const int Np = (int)h->Npad;
    if (!h->ZdT) {
        CK(h->ZdT.alloc(h->Npad * TILE));
        if (h->tma_ok && !gemm_make_tensor_map(&h->mapZdT, h->ZdT, h->Npad, TILE, TILE)) {
            h->ZdT.reset();
            return fail(h, GPB200_ECUDA, "gpa_grad: cuTensorMapEncodeTiled failed for the diagonal tiles of Z'");
        }
    }
    CK(cudaEventRecord(h->ev0, h->st));
    CK(inverse_merges(h));
    CK(cudaEventRecord(h->ev1, h->st));
    CK(gpa_scan_launch(h->G, h->ld, h->DinvT, h->y1, h->r0, h->F, h->ZdT, h->Npad, h->st, &h->launches));
    CK(cudaEventRecord(h->ev2, h->st));
    {
        GemmDesc g = gemm_desc_default();                       // G[a,b] = -sum_{i >= a} W'[a,i] Z'[b,i]   (a >= b)
        g.A = GemmOperand{bufG(h), bufDinvT(h), 0, 0};
        g.B = GemmOperand{bufF(h), gbuf(h, h->ZdT, h->mapZdT, TILE), 0, 0};
        g.C = h->G; g.ldc = h->ld; g.c_row0 = 0; g.c_col0 = 0;
        g.M = Np; g.N = Np; g.K = Np;
        g.alpha = -1.0;
        g.flags = GEMM_LOWER_ONLY | GEMM_KLO_M;
        CK(launch_gemm(h, g));
    }
    CK(cudaEventRecord(h->ev3, h->st));
    CK(cudaMemsetAsync(h->alpha, 0, sizeof(double) * h->Npad, h->st));
    CK(launch_trace(h, 1, 0, 1));
    CK(cudaEventRecord(h->ev4, h->st));
    const int np = h->prog.n_theta;
    std::vector<double> out((size_t)np + 1);
    CK(cudaMemcpyAsync(out.data(), h->trace_out, sizeof(double) * (np + 1), cudaMemcpyDeviceToHost, h->st));
    CK(cudaStreamSynchronize(h->st));
    profile_collect(h);
    h->ms[3] = ev_ms(h->ev0, h->ev1);
    h->ms[9] = ev_ms(h->ev1, h->ev2);
    h->ms[10] = ev_ms(h->ev2, h->ev3);
    h->ms[4] = ev_ms(h->ev3, h->ev4);
    for (int p = 0; p < np; ++p) dll_kernel[p] = out[p];
    h->s_ready = true;
    return GPB200_OK;
}

// Training-input gradient: out[i, :] = sum_j A_ij dk(x_i, x_j)/dx_i over the resident lower triangle of A (the inputs_dx
// kernel of gram.cu reads each stored entry twice, once for its row point and once for its column point).  The tile rows
// are split as in gpb200_grad_kernel's trace: replicated multi-rank handles sum rows t % nranks == rank and all-reduce the
// N x d partials over NCCL; row-sharded handles sum their own rows and all-reduce through coll_allreduce_sum.  Reads F, G,
// alpha and the cross-validation work matrices only: a caller's alpha goes to the dxin scratch.  Timing slot 16.
int gpb200_grad_inputs(gpb200_handle* h, const double* alpha, double* dmll_x) {
    if (!h) return GPB200_EINVAL;
    if (!dmll_x) return fail(h, GPB200_EINVAL, "grad_inputs: null dmll_x");
    if (h->s_ready && alpha) return fail(h, GPB200_EINVAL, "grad_inputs: after gpa_grad the contraction is with S; alpha must be NULL");
    if (!h->s_ready && !h->inv_ready) return fail(h, GPB200_ESTATE, "grad_inputs: grad_prepare (or gpa_grad with the kernel gradient) first");
    if (!h->s_ready && !alpha && !h->alpha_ready) return fail(h, GPB200_ESTATE, "grad_inputs: no alpha (call mll or pass alpha)");
    CK(cudaSetDevice(h->device));
    Locals L;
    if (h->sharded) TRY(shard_entry(h, L)); else L = Locals{h};
    const int64_t N = h->N, Npad = h->Npad, nd = Npad * h->d;
    for (auto* q : L) {
        if (!q->dxin) SCK(q, q->dxin.alloc(Npad + nd * (1 + (q->grp ? q->nranks : 0))));
        if (alpha) TRY(rank_failed(q, upload_padded(q, q->dxin, alpha)));
    }
    auto res = [&](gpb200_handle* q) { return q->dxin + Npad; };
    CK(cudaEventRecord(h->ev0, h->st));
    for (auto* q : L) {
        SeIsoFast sf;
        const double* a = h->s_ready ? nullptr : alpha ? q->dxin.data() : q->alpha.data();     // S state: A = -G = S
        SCK(q, inputs_dx_launch(q->prog, use_seiso_fast(q, &sf), q->x, q->d, q->d, N, a, q->G, q->ld, res(q), q->st, &q->launches,
                                q->nranks, q->rank, q->sharded ? q->rb : 1));
    }
    if (h->sharded) {
        TRY(coll_allreduce_sum(L, res, (size_t)(N * h->d), [&](gpb200_handle* q) { return q->dxin + Npad + nd; }));
    } else if (h->nranks > 1) {                            // N x d partial sums, summed over ranks
        CK(cudaEventRecord(h->ev_x, h->st));
        CK(cudaStreamWaitEvent(h->st_comm, h->ev_x, 0));
        CKN(g_nccl.AllReduce(res(h), res(h), (size_t)(N * h->d), ncclDouble, ncclSum, h->comm, h->st_comm));
        CK(cudaEventRecord(h->ev_y, h->st_comm));
        CK(cudaStreamWaitEvent(h->st, h->ev_y, 0));
    }
    CK(cudaEventRecord(h->ev1, h->st));
    CK(cudaMemcpyAsync(dmll_x, res(h), sizeof(double) * (size_t)(N * h->d), cudaMemcpyDeviceToHost, h->st));
    CK(cudaStreamSynchronize(h->st));
    if (h->sharded) TRY(sync_all(L));
    h->ms[16] = ev_ms(h->ev0, h->ev1);
    return GPB200_OK;
}

// test points per chunk, so that the M_c x Npad workspace stays below ~16 GB; a full covariance needs all of V at once
static int64_t predict_chunk(const gpb200_handle* h, int64_t M, bool want_cov) {
    int64_t cap = (int64_t)(16.0e9 / (8.0 * (double)h->Npad)) / TILE * TILE;
    if (const char* env = getenv("GPB200_PREDICT_CHUNK")) {            // testing hook: force small chunks
        const int64_t v = atoll(env) / TILE * TILE;
        if (v >= TILE && v < cap) cap = v;
    }
    if (cap < TILE) cap = TILE;
    if (h->sharded && cap > h->Npad) cap = h->Npad;       // a block of V' travels through the Npad x NBp panel buffer
    if (want_cov) cap = (M + TILE - 1) / TILE * TILE;
    return cap;
}

// K*' of Mc test rows (xs, row stride ldxs) into Kst, on h's stream
static int predict_cross(gpb200_handle* h, const double* xs, int64_t ldxs, int64_t Mc) {
    const int64_t Mpad = (Mc + TILE - 1) / TILE * TILE;
    CK(cudaMemcpy2DAsync(h->xs, sizeof(double) * h->d, xs, sizeof(double) * ldxs, sizeof(double) * h->d, Mc,
                         cudaMemcpyHostToDevice, h->st));
    CK(crossgram_launch(h->prog, h->xs, h->d, Mc, Mpad, h->x, h->d, h->N, h->Npad, h->d, h->Kst, h->Npad, h->st, &h->launches));
    return GPB200_OK;
}

// mu = K*' alpha (GP.jl:26) into pmu and mu[0..Mc) on the host
static int predict_mean(gpb200_handle* h, int64_t Mc, double* mu) {
    CK(rowdot_launch(h->Kst, h->Npad, h->alpha, Mc, h->Npad, h->pmu, h->st, &h->launches));
    CK(cudaMemcpyAsync(mu, h->pmu, sizeof(double) * Mc, cudaMemcpyDeviceToHost, h->st));
    return GPB200_OK;
}

// V' = K*' L^-T in Kst (whiten!, GP.jl:27); with var, var = k** - |V'|^2 into pvar and var[0..Mc) on the host
static int predict_var(gpb200_handle* h, int64_t Mc, double* var) {
    CK(trsm_rec(h, (int)((Mc + TILE - 1) / TILE * TILE), 0, (int)h->Npad));
    if (!var) return GPB200_OK;
    CK(kdiag_launch(h->prog, h->xs, h->d, Mc, h->pkdiag, h->st, &h->launches));
    CK(rowvar_launch(h->Kst, h->Npad, h->pkdiag, Mc, h->Npad, h->pvar, h->st, &h->launches));
    CK(cudaMemcpyAsync(var, h->pvar, sizeof(double) * Mc, cudaMemcpyDeviceToHost, h->st));
    return GPB200_OK;
}

// gpb200_predict with Sigma* sent to cov_to (CovDest::host: cov, M x M).  *out, if given: pmu holds the last chunk's mu
// (all of mu* when Sigma* is formed, which takes one chunk) and Kss holds Sigma*.
static int predict_run(gpb200_handle* h, int64_t M, const double* xs, int64_t ldxs, const double* alpha, double* mu,
                       double* var, CovDest cov_to, double* cov, DevPrediction* out) {
    if (!h->factored) return fail(h, GPB200_ESTATE, "predict: factorize first");
    if (M <= 0 || !xs || ldxs < h->d || !mu) return fail(h, GPB200_EINVAL, "predict: bad M, xs, ldxs or mu");
    if (!alpha && !h->alpha_ready) return fail(h, GPB200_ESTATE, "predict: no alpha (call mll or pass alpha)");
    CK(cudaSetDevice(h->device));
    if (alpha) {
        TRY(upload_padded(h, h->alpha, alpha));
        h->alpha_ready = true;
    }
    const bool want_cov = cov_to != CovDest::none;
    const int64_t cap = predict_chunk(h, M, want_cov);
    if (want_cov && h->sharded && cap > h->Npad) return fail(h, GPB200_EINVAL, "predict: full covariance of more than Npad test points is not supported with sharded storage");
    const bool need_v = (var != nullptr) || want_cov;
    Locals Lp;
    if (h->sharded) {
        int rc = shard_entry(h, Lp); if (rc) return rc;
        if (alpha) for (auto* q : Lp) if (q != h) TRY(rank_failed(q, upload_padded(q, q->alpha, alpha)));
    }
    CK(cudaEventRecord(h->ev2, h->st));
    for (int64_t m0 = 0; h->sharded && m0 < M; m0 += cap) {
        // row-sharded factor: K*' on every rank, the triangular solve runs over column blocks owned like the rows of L
        const int64_t Mc = (M - m0 < cap) ? M - m0 : cap;
        const int64_t Mpad = (Mc + TILE - 1) / TILE * TILE;
        for (auto* q : Lp) {
            TRY(rank_failed(q, ensure_predict_ws(q, Mc, want_cov)));
            TRY(rank_failed(q, predict_cross(q, xs + m0 * ldxs, ldxs, Mc)));
            if (need_v) {
                SCK(q, kdiag_launch(q->prog, q->xs, q->d, Mc, q->pvar, q->st, &q->launches));           // running variance starts at k**
                if (want_cov) SCK(q, gram_full_launch(q->prog, q->xs, q->d, Mc, Mpad, q->d, q->Kss, Mpad, q->st, &q->launches));
            }
        }
        TRY(predict_mean(h, Mc, mu + m0));
        if (need_v) {
            TRY(shard_predict_solve(Lp, (int)Mpad, Mc, var != nullptr, want_cov));
            if (var) CK(cudaMemcpyAsync(var + m0, h->pvar, sizeof(double) * Mc, cudaMemcpyDeviceToHost, h->st));
            if (cov_to == CovDest::host) CK(cudaMemcpy2DAsync(cov, sizeof(double) * M, h->Kss, sizeof(double) * Mpad, sizeof(double) * M, M,
                                                              cudaMemcpyDeviceToHost, h->st));
        }
        TRY(sync_all(Lp));
    }
    for (int64_t m0 = 0; !h->sharded && m0 < M; m0 += cap) {
        const int64_t Mc = (M - m0 < cap) ? M - m0 : cap;
        const int64_t Mpad = (Mc + TILE - 1) / TILE * TILE;
        TRY(ensure_predict_ws(h, Mc, want_cov));
        TRY(predict_cross(h, xs + m0 * ldxs, ldxs, Mc));
        TRY(predict_mean(h, Mc, mu + m0));
        if (need_v) {
            TRY(predict_var(h, Mc, var ? var + m0 : nullptr));
            if (want_cov) {                                                                 // GP.jl:51-54
                CK(gram_full_launch(h->prog, h->xs, h->d, Mc, Mpad, h->d, h->Kss, Mpad, h->st, &h->launches));
                const GemmBuf bk = gbuf(h, h->Kst, h->mapKst, h->Npad);
                CK(gemm_whole(h, bk, bk, h->Kss, Mpad, Mpad, Mpad, h->Npad, -1.0, 1.0));
                if (cov_to == CovDest::host)
                    CK(cudaMemcpy2DAsync(cov, sizeof(double) * M, h->Kss, sizeof(double) * Mpad, sizeof(double) * M, M,
                                         cudaMemcpyDeviceToHost, h->st));
            }
        }
        CK(cudaStreamSynchronize(h->st));
    }
    CK(cudaEventRecord(h->ev3, h->st));
    CK(cudaStreamSynchronize(h->st));
    profile_collect(h);
    h->ms[5] = ev_ms(h->ev2, h->ev3);
    if (out) *out = DevPrediction{h->pmu, h->Kss, (M + TILE - 1) / TILE * TILE};
    return GPB200_OK;
}

int gpb200_predict(gpb200_handle* h, int64_t M, const double* xs, int64_t ldxs, const double* alpha,
                   double* mu, double* var, double* cov) {
    if (!h) return GPB200_EINVAL;
    return predict_run(h, M, xs, ldxs, alpha, mu, var, cov ? CovDest::host : CovDest::none, cov, nullptr);
}

// Predictive gradients (for ForwardDiff.Dual test inputs of predict_f): mu and var through gpb200_predict's chunk steps,
// then, with W' = V' L^-1 = K*' K^-1 (rows w_m' = (K^-1 k*_m)'),
//   dmu[m, :] = sum_i dk(x*_m, x_i)/dx*_m alpha_i,   dvar[m, :] = 2 dk(x*_m, x*_m)/dx*_m - 2 sum_i dk(x*_m, x_i)/dx*_m W'[m, i].
// F's strict-upper tiles are scratch between calls (inverse merges, GPA's Z'); every call that solves for W' first fills
// them with L' (one O(N^2) pass).  Timing slots 11..15: cross-Gram + mean, V' + variance, transpose, W', contraction.
int gpb200_predict_grad(gpb200_handle* h, int64_t M, const double* xs, int64_t ldxs, const double* alpha,
                        double* mu, double* var, double* dmu, double* dvar) {
    if (!h) return GPB200_EINVAL;
    if (h->nranks > 1 || h->sharded || h->grp) return fail(h, GPB200_EINVAL, "predict_grad: single GPU handles only");
    if (!h->factored) return fail(h, GPB200_ESTATE, "predict_grad: factorize first");
    if (M <= 0 || !xs || ldxs < h->d || !mu || !dmu) return fail(h, GPB200_EINVAL, "predict_grad: bad M, xs, ldxs, mu or dmu");
    if (!var != !dvar) return fail(h, GPB200_EINVAL, "predict_grad: var and dvar must be given together");
    if (!alpha && !h->alpha_ready) return fail(h, GPB200_ESTATE, "predict_grad: no alpha (call mll or pass alpha)");
    CK(cudaSetDevice(h->device));
    if (alpha) {
        TRY(upload_padded(h, h->alpha, alpha));
        h->alpha_ready = true;
    }
    const int64_t cap = predict_chunk(h, M, false);
    const int d = h->d;
    for (int i = 11; i < 16; ++i) h->ms[i] = 0.0;
    for (int64_t m0 = 0; m0 < M; m0 += cap) {
        const int64_t Mc = (M - m0 < cap) ? M - m0 : cap;
        const int64_t Mpad = (Mc + TILE - 1) / TILE * TILE;
        TRY(ensure_predict_ws(h, Mc, false));
        CK(h->pdx.ensure(2 * Mpad * d));
        double* ddmu = h->pdx;
        double* ddvar = h->pdx + h->pdx.size() / 2;             // dmu and dvar take one half each
        CK(cudaEventRecord(h->ev0, h->st));
        TRY(predict_cross(h, xs + m0 * ldxs, ldxs, Mc));
        TRY(predict_mean(h, Mc, mu + m0));
        CK(cudaEventRecord(h->ev1, h->st));
        if (var) TRY(predict_var(h, Mc, var + m0));                                        // V' = K*' L^-T
        CK(cudaEventRecord(h->ev2, h->st));
        if (var && m0 == 0) CK(mirror_lower_tiles_launch(h->F, h->ld, h->Npad, h->st, &h->launches));   // L' into F's upper tiles
        CK(cudaEventRecord(h->ev5, h->st));
        if (var) {
            const GemmBuf bk = gbuf(h, h->Kst, h->mapKst, h->Npad);
            CK(trsm_right_rec_buf(h, bk, (int)Mpad, 0, (int)h->Npad));                     // W' = V' L^-1
        }
        CK(cudaEventRecord(h->ev3, h->st));
        CK(crossgram_dx_launch(h->prog, h->xs, d, Mc, h->x, d, h->N, d, h->alpha, var ? h->Kst.data() : nullptr, nullptr, h->Npad, 1.0,
                               ddmu, ddvar, h->st, &h->launches));
        CK(cudaEventRecord(h->ev4, h->st));
        CK(cudaMemcpyAsync(dmu + m0 * d, ddmu, sizeof(double) * Mc * d, cudaMemcpyDeviceToHost, h->st));
        if (var) CK(cudaMemcpyAsync(dvar + m0 * d, ddvar, sizeof(double) * Mc * d, cudaMemcpyDeviceToHost, h->st));
        CK(cudaStreamSynchronize(h->st));
        h->ms[11] += ev_ms(h->ev0, h->ev1);
        h->ms[12] += ev_ms(h->ev1, h->ev2);
        h->ms[13] += ev_ms(h->ev2, h->ev5);
        h->ms[14] += ev_ms(h->ev5, h->ev3);
        h->ms[15] += ev_ms(h->ev3, h->ev4);
    }
    profile_collect(h);
    return GPB200_OK;
}

// rand(gp, X, n) (src/GP.jl:120-146): posterior draws  mu* + chol(Sigma* + nugget I) Z  entirely on the device: full predictive
// covariance (predictMVN), make_posdef!(Sigma; nugget) with the engine's own Cholesky on an M x M sub-engine, unwhiten! as one
// triangular NT GEMM.  z / samples are Julia's M x nsamp column-major matrices (== nsamp x M row-major).
int gpb200_rand(gpb200_handle* h, int64_t M, const double* xs, int64_t ldxs, const double* alpha, int64_t nsamp,
                const double* z, double nugget, double* mu_minus_mean, double* samples) {
    if (!h) return GPB200_EINVAL;
    if (M <= 0 || nsamp <= 0 || !z || !samples || !mu_minus_mean) return fail(h, GPB200_EINVAL, "rand: bad M, nsamp, z, mu or samples");
    if (!(nugget >= 0.0)) return fail(h, GPB200_EINVAL, "rand: nugget must be >= 0");
    DevPrediction p;
    TRY(predict_run(h, M, xs, ldxs, alpha, mu_minus_mean, nullptr, CovDest::device, nullptr, &p));
    return rand_from_cov(h, M, p.cov, p.ldc, p.mu, nsamp, z, nugget, samples);
}

// ---- ElasticGPE append! (src/GPEelastic.jl:13-22): extend the factor by k new observations -----------------------------
// The reference appends rows to an elastic Cholesky (ElasticPDMats.append!, a rank-k extension) and keeps the hyper-parameters
// (update_target!(gp, kern=false, noise=false)).  Here the rows live inside the capacity reserved at set_data (option
// "capacity"): only the block rows from the first touched 128-row tile on are rebuilt --
//   Gram rows r >= c0;  L[r, 0:c0] = K[r, 0:c0] L11^-T (whitening TRSM against the existing factor);
//   Schur complement of the trailing block (one GEMM with K = c0);  Cholesky of that small trailing block --
// i.e. O(k N^2) instead of O(N^3).  Returns GPB200_EINVAL if N + k exceeds the capacity (the caller refits).
// Row-sharded handles run the same steps over the ranks (shard_append in shard_impl.cuh).
static int append_inputs(gpb200_handle* h, int64_t k, const double* xnew, int64_t ldx) {
    const int64_t Nold = h->N, Nnew = Nold + k;
    const int d = h->d, Np = (int)h->Npad;
    CK(cudaMemcpy2DAsync(h->x + Nold * d, sizeof(double) * d, xnew, sizeof(double) * ldx, sizeof(double) * d, k, cudaMemcpyHostToDevice, h->st));
    h->xmap_ok = false;
    if (h->xp) {
        CK(cudaMemcpy2DAsync(h->xp + Nold * h->dxp, sizeof(double) * h->dxp, xnew, sizeof(double) * ldx, sizeof(double) * d, k, cudaMemcpyHostToDevice, h->st));
        CK(shard_transpose(h->xpt, Np, h->xp, h->dxp, Np, h->dxp, h->st, &h->launches));
        h->xmap_ok = seiso_make_x_maps(&h->mapX, &h->mapXT, h->xp, h->xpt, h->dxp, Nnew, Np);
    }
    h->N = Nnew;
    h->inv_ready = h->s_ready = h->alpha_ready = false; h->g_sym = false; h->cv_m_ok = false;
    return GPB200_OK;
}

int gpb200_append(gpb200_handle* h, int64_t k, const double* xnew, int64_t ldx) {
    if (!h) return GPB200_EINVAL;
    if (k <= 0 || !xnew || ldx < h->d) return fail(h, GPB200_EINVAL, "append: bad k, x or ldx");
    if (!h->factored) return fail(h, GPB200_ESTATE, "append: factorize first");
    if (h->nranks > 1 && !h->sharded)
        return fail(h, GPB200_ESTATE, "append: multi-rank handles need row-sharded storage (option \"shard\" = 1)");
    Locals L{h};
    if (h->sharded) { int rc = shard_entry(h, L); if (rc) return rc; }
    if (h->n_noise != 1) return fail(h, GPB200_ESTATE, "append: scalar logNoise only (per-point noise needs a refit)");
    if (h->N + k > h->Npad) return fail(h, GPB200_EINVAL, "append: capacity exceeded (set option \"capacity\" before set_data, or refit)");
    CK(cudaSetDevice(h->device));
    const int64_t Nold = h->N;
    if (h->sharded) {
        for (auto* q : L)
            if (!q->factored || q->N != Nold || q->Npad != h->Npad)
                return fail(h, GPB200_ESTATE, "append: every handle of the group needs the same factorized data");
        for (auto* q : L) TRY(rank_failed(q, append_inputs(q, k, xnew, ldx)));
        TRY(factor_begin(L));
        TRY(shard_append(L, Nold));
        return factor_end(L, "append: extended ", false);
    }
    TRY(append_inputs(h, k, xnew, ldx));
    const int64_t Nnew = h->N;
    const int d = h->d, Np = (int)h->Npad;
    const int c0 = (int)(Nold / TILE * TILE);                       // first tile row that changes
    TRY(factor_begin(L));
    // Gram rows >= c0 (columns <= row), identity beyond the new N
    CK(gram_lower_launch(h->prog, h->x, d, d, Nnew, Np, h->noise_var, 1, h->nugget, h->G, h->ld, h->st, &h->launches, 0, 1, 0, 0, c0 / TILE));
    cudaError_t e = cudaSuccess;
    if (c0 > 0) {
        // rows >= c0 of G against the existing factor: G[r, 0:c0] <- G[r, 0:c0] L11^-T, then keep them as rows of L
        CUtensorMap sub{};
        double* gsub = h->G + (size_t)c0 * h->ld;
        const bool tma = h->tma_ok && gemm_make_tensor_map(&sub, gsub, Np - c0, Np, h->ld);
        GemmBuf bk{tma ? &sub : nullptr, gsub, h->ld};
        const int impl_save = h->gemm_impl;
        if (!tma) h->gemm_impl = 1;
        e = trsm_rec_buf(h, bk, Np - c0, 0, c0);
        h->gemm_impl = impl_save;
        CK(e);
        CK(cudaMemcpy2DAsync(h->F + (size_t)c0 * h->ld, sizeof(double) * h->ld, gsub, sizeof(double) * h->ld, sizeof(double) * c0, Np - c0,
                             cudaMemcpyDeviceToDevice, h->st));
        // Schur complement of the trailing block:  G[r, c] -= sum_{k < c0} L[r, k] L[c, k],  r >= c >= c0
        CK(schur_update(h, c0, Np - c0, Np - c0, 0, c0));
    }
    // factor the trailing block tile by tile (right-looking, 128-wide panels)
    CK(cholesky(h, c0, TILE));
    return factor_end(L, "append: extended ", false);
}

// ---- cross-validation on the resident inverse (src/crossvalidation.jl) --------------------------------------------
// The reference forms inv(Sigma) and, per hyper-parameter j, Z_j = inv(Sigma) dK_j and Z_j inv(Sigma) on the host
// (crossvalidation.jl:86-108, 270-283).  Here K_y^-1 already sits on the device after gpb200_grad_prepare; per parameter:
// D = dK_j (recomputed from x), Y' = K^-1 D, M_j = Y' K^-1 -- two NT DMMA GEMMs -- and the two N-vectors every LOO / fold
// formula needs: Z_j alpha = Y' alpha and diag(M_j).  Fold formulas read principal sub-blocks through gpb200_cv_block.
// Row-sharded handles run the same steps over the ranks (shard_cv_* in shard_impl.cuh) and keep only the lower triangle of M_j.
static int cv_check(gpb200_handle* h) {
    if (!h->inv_ready) return fail(h, GPB200_ESTATE, "cv: grad_prepare first (K_y^-1 must be resident)");
    if (h->nranks > 1 && !h->sharded)
        return fail(h, GPB200_ESTATE, "cv: K^-1 is distributed over the ranks; multi-rank handles need row-sharded storage (option \"shard\" = 1)");
    return GPB200_OK;
}

static int cv_prepare(gpb200_handle* h) {
    TRY(cv_check(h));
    const size_t nn = (size_t)h->Npad * (size_t)h->Npad;
    if (!h->cvD || !h->cvY) {
        h->cvD.reset(); h->cvY.reset();
        h->cv_m_ok = false;
        if (h->cvD.alloc(nn) != cudaSuccess || h->cvY.alloc(nn) != cudaSuccess) {
            (void)cudaGetLastError();
            h->cvD.reset();
            return fail(h, GPB200_ECUDA, "cv: out of device memory for the two N x N work matrices");
        }
        if (h->tma_ok && !(gemm_make_tensor_map(&h->mapCvD, h->cvD, h->Npad, h->Npad, h->Npad) &&
                           gemm_make_tensor_map(&h->mapCvY, h->cvY, h->Npad, h->Npad, h->Npad)))
            return fail(h, GPB200_ECUDA, "cv: cuTensorMapEncodeTiled failed");
    }
    if (!h->g_sym) {
        CK(symmetrize_launch(h->G, h->ld, h->Npad, h->st, &h->launches));      // lower K^-1 -> full symmetric (the W' scratch above it is dead)
        h->g_sym = true;
    }
    return GPB200_OK;
}

// the N-vectors of the compact own-row values in Sbuf (`width` per row): all-gathered, read back on this rank, unpacked
static int shard_own_vectors(const Locals& L, size_t per, int width, double* out0, double* out1) {
    gpb200_handle* h = L[0];
    TRY(coll_allgather(L, [&](gpb200_handle* q) { return (void*)q->Sbuf; }, sizeof(double) * per));
    std::vector<double> buf(per * (size_t)h->nranks);
    CK(cudaMemcpyAsync(buf.data(), h->Sbuf, sizeof(double) * buf.size(), cudaMemcpyDeviceToHost, h->st));
    TRY(sync_all(L));
    unpack_own_rows(h, buf, per, width, 0, out0);
    if (out1) unpack_own_rows(h, buf, per, width, 1, out1);
    return GPB200_OK;
}

static int shard_cv_param(gpb200_handle* h, int32_t param, const double* alpha, double* Zj_alpha, double* diag_ZjSinv) {
    Locals L;
    TRY(shard_entry(h, L));
    TRY(cv_check(h));
    TRY(shard_cv_alloc(L));
    if (!h->g_sym) {
        TRY(shard_cv_symmetrize(L));
        h->g_sym = true;
    }
    if (alpha) {
        for (auto* q : L) {
            TRY(rank_failed(q, upload_padded(q, q->alpha, alpha)));
            q->alpha_ready = true;
        }
    }
    h->cv_m_ok = false;
    if (param >= 0) TRY(shard_cv_y(L, param));
    const size_t per = 2 * (size_t)shard_own_rows(h->N, ShardOwn{h->nranks, 0, h->rb});      // rank 0 owns the most rows
    for (auto* q : L)
        SCK(q, shard_rowdot_own(param >= 0 ? cv_y(q) : q->G, q->G, q->ld, q->Npad, q->alpha, q->N, own_of(q), q->Sbuf + (size_t)q->rank * per,
                                q->st, &q->launches));
    TRY(shard_cv_m(L, param < 0));
    TRY(shard_own_vectors(L, per, 2, Zj_alpha, diag_ZjSinv));
    for (auto* q : L) profile_collect(q);
    h->cv_m_ok = true;
    return GPB200_OK;
}

// principal sub-block workspace: nV indices, `elems` doubles
static int ensure_cv_block_ws(gpb200_handle* h, int64_t nV, int64_t elems) {
    if ((size_t)nV <= h->cvidx.size() && (size_t)elems <= h->cvblk.size()) return GPB200_OK;
    h->cvblk.reset(); h->cvidx.reset();
    CK(h->cvblk.alloc(elems));
    CK(h->cvidx.alloc(nV));
    return GPB200_OK;
}

int gpb200_cv_param(gpb200_handle* h, int32_t param, const double* alpha, double* Zj_alpha, double* diag_ZjSinv) {
    if (!h || !Zj_alpha || !diag_ZjSinv) return GPB200_EINVAL;
    if (param < -1 || param >= h->prog.n_theta) return fail(h, GPB200_EINVAL, "cv_param: parameter index out of range");
    if (!alpha && !h->alpha_ready) return fail(h, GPB200_ESTATE, "cv_param: no alpha (call mll or pass alpha)");
    CK(cudaSetDevice(h->device));
    if (h->sharded) return shard_cv_param(h, param, alpha, Zj_alpha, diag_ZjSinv);
    int rc = cv_prepare(h);
    if (rc) return rc;
    if (alpha) { rc = upload_padded(h, h->alpha, alpha); if (rc) return rc; h->alpha_ready = true; }
    const int Np = (int)h->Npad;
    const GemmBuf bD = gbuf(h, h->cvD, h->mapCvD, h->Npad), bY = gbuf(h, h->cvY, h->mapCvY, h->Npad);
    const double* Yt = h->cvY;
    if (param >= 0) {
        CK(gram_grad_full_launch(h->prog, h->x, h->d, h->d, h->N, h->Npad, param, h->cvD, h->Npad, h->st, &h->launches));
        CK(gemm_whole(h, bufG(h), bD, h->cvY, h->Npad, Np, Np, Np, 1.0, 0.0));    // Y' = K^-1 D   (both symmetric: NT form)
    } else {
        Yt = h->G;                                                  // noise: Z = K^-1 (crossvalidation.jl:124-126)
    }
    CK(rowdot_launch(Yt, h->Npad, h->alpha, h->N, h->Npad, h->r1, h->st, &h->launches));              // Z_j alpha
    CK(rowdot2_launch(h->G, Yt, h->Npad, h->N, h->Npad, h->y1, h->st, &h->launches));                 // diag(Z_j K^-1) = rowwise <K^-1_i, Y'_i>
    CK(gemm_whole(h, param >= 0 ? bY : bufG(h), bufG(h), h->cvD, h->Npad, Np, Np, Np, 1.0, 0.0));   // M_j = Y' K^-1 -> cvD (fold sub-blocks)
    h->cv_m_ok = true;
    CK(cudaMemcpyAsync(Zj_alpha, h->r1, sizeof(double) * h->N, cudaMemcpyDeviceToHost, h->st));
    CK(cudaMemcpyAsync(diag_ZjSinv, h->y1, sizeof(double) * h->N, cudaMemcpyDeviceToHost, h->st));
    CK(cudaStreamSynchronize(h->st));
    profile_collect(h);
    return GPB200_OK;
}

int gpb200_cv_block(gpb200_handle* h, int32_t which, int64_t nV, const int64_t* idx, double* out) {
    if (!h || !idx || !out || nV <= 0 || which < 0 || which > 1) return GPB200_EINVAL;
    CK(cudaSetDevice(h->device));
    static_assert(sizeof(long long) == sizeof(int64_t), "index width");
    if (h->sharded) {
        // every rank reads the entries whose row (of the stored lower triangle) it owns, zeros elsewhere; one sum over the ranks
        Locals L;
        TRY(shard_entry(h, L));
        TRY(cv_check(h));
        if (which == 1 && !h->cv_m_ok) return fail(h, GPB200_ESTATE, "cv_block: which = 1 reads M_j of the last cv_param call; call cv_param first");
        for (int64_t a = 0; a < nV; ++a)
            if (idx[a] < 0 || idx[a] >= h->N) return fail(h, GPB200_EINVAL, "cv_block: index out of range");
        const size_t nn = (size_t)nV * (size_t)nV;
        const int64_t elems = (int64_t)nn * (1 + (h->grp ? h->nranks : 0));       // + the group's all-reduce scratch
        for (auto* q : L) {
            TRY(rank_failed(q, ensure_cv_block_ws(q, nV, elems)));
            SCK(q, cudaMemcpyAsync(q->cvidx, idx, sizeof(long long) * nV, cudaMemcpyHostToDevice, q->st));
            SCK(q, shard_gather_block_own(q->cvblk, which == 0 ? q->G : cv_m(q), q->ld, q->cvidx, nV, own_of(q), q->st, &q->launches));
        }
        TRY(coll_allreduce_sum(L, [&](gpb200_handle* q) { return q->cvblk.data(); }, nn, [&](gpb200_handle* q) { return q->cvblk + nn; }));
        CK(cudaMemcpyAsync(out, h->cvblk, sizeof(double) * nn, cudaMemcpyDeviceToHost, h->st));
        return sync_all(L);
    }
    int rc = cv_prepare(h);
    if (rc) return rc;
    if (which == 1 && !h->cv_m_ok) return fail(h, GPB200_ESTATE, "cv_block: which = 1 reads M_j of the last cv_param call; call cv_param first");
    for (int64_t a = 0; a < nV; ++a)
        if (idx[a] < 0 || idx[a] >= h->N) return fail(h, GPB200_EINVAL, "cv_block: index out of range");
    TRY(ensure_cv_block_ws(h, nV, nV * nV));
    CK(cudaMemcpyAsync(h->cvidx, idx, sizeof(long long) * nV, cudaMemcpyHostToDevice, h->st));
    CK(gather_block_launch(h->cvblk, which == 0 ? h->G : h->cvD, h->Npad, h->cvidx, nV, h->st, &h->launches));
    CK(cudaMemcpyAsync(out, h->cvblk, sizeof(double) * nV * nV, cudaMemcpyDeviceToHost, h->st));
    CK(cudaStreamSynchronize(h->st));
    return GPB200_OK;
}

int gpb200_get_gram(gpb200_handle* h, double* K) {
    if (!h || !K) return GPB200_EINVAL;
    if (!h->has_data || !h->has_kernel) return fail(h, GPB200_ESTATE, "get_gram: set_data and set_kernel first");
    CK(cudaSetDevice(h->device));
    DevBuf<double> tmp;
    CK(tmp.alloc((size_t)h->Npad * (size_t)h->Npad));
    CK(launch_gram(h, tmp, h->Npad, 0, 1, 0, 0));
    CK(cudaMemcpy2DAsync(K, sizeof(double) * h->N, tmp, sizeof(double) * h->Npad, sizeof(double) * h->N, h->N,
                         cudaMemcpyDeviceToHost, h->st));
    CK(cudaStreamSynchronize(h->st));
    tmp.reset();
    const int64_t N = h->N;
    for (int64_t i = 0; i < N; ++i)
        for (int64_t j = i + 1; j < N; ++j) K[i * N + j] = K[j * N + i];
    return GPB200_OK;
}

int gpb200_get_factor(gpb200_handle* h, double* U) {
    if (!h || !U) return GPB200_EINVAL;
    if (!h->factored) return fail(h, GPB200_ESTATE, "get_factor: factorize first");
    CK(cudaSetDevice(h->device));
    const int64_t N = h->N;
    if (h->sharded) { int rc = copy_own_rows(h, U, h->F); if (rc) return rc; }
    else
    CK(cudaMemcpy2DAsync(U, sizeof(double) * N, h->F, sizeof(double) * h->ld, sizeof(double) * N, N,
                         cudaMemcpyDeviceToHost, h->st));
    CK(cudaStreamSynchronize(h->st));
    // row-major lower L == column-major upper U; clear the other triangle (scratch on the device)
    for (int64_t j = 0; j < N; ++j)
        for (int64_t i = j + 1; i < N; ++i) U[j * N + i] = 0.0;
    return GPB200_OK;
}

int gpb200_get_inverse(gpb200_handle* h, double* Kinv) {
    if (!h || !Kinv) return GPB200_EINVAL;
    if (!h->inv_ready) return fail(h, GPB200_ESTATE, "get_inverse: grad_prepare first");
    if (h->nranks > 1 && !h->sharded) return fail(h, GPB200_ESTATE, "get_inverse: K^-1 is distributed over the ranks (tile rows round-robin)");
    CK(cudaSetDevice(h->device));
    const int64_t N = h->N;
    if (h->sharded) { int rc = copy_own_rows(h, Kinv, h->G); if (rc) return rc; }     // own rows only (others zero): sum over the ranks
    else
    CK(cudaMemcpy2DAsync(Kinv, sizeof(double) * N, h->G, sizeof(double) * h->ld, sizeof(double) * N, N,
                         cudaMemcpyDeviceToHost, h->st));
    CK(cudaStreamSynchronize(h->st));
    for (int64_t i = 0; i < N; ++i)
        for (int64_t j = i + 1; j < N; ++j) Kinv[i * N + j] = Kinv[j * N + i];
    return GPB200_OK;
}

int gpb200_get_inverse_diag(gpb200_handle* h, double* diag) {
    if (!h || !diag) return GPB200_EINVAL;
    if (!h->inv_ready) return fail(h, GPB200_ESTATE, "get_inverse_diag: grad_prepare first");
    if (h->nranks > 1 && !h->sharded)
        return fail(h, GPB200_ESTATE, "get_inverse_diag: K^-1 is distributed over the ranks; multi-rank handles need row-sharded storage (option \"shard\" = 1)");
    CK(cudaSetDevice(h->device));
    if (h->sharded) {           // own diagonal entries (copies), all-gathered
        Locals L;
        TRY(shard_entry(h, L));
        const size_t per = (size_t)shard_own_rows(h->N, ShardOwn{h->nranks, 0, h->rb});
        for (auto* q : L) SCK(q, shard_diag_own(q->G, q->ld, q->N, own_of(q), q->Sbuf + (size_t)q->rank * per, q->st, &q->launches));
        return shard_own_vectors(L, per, 1, diag, nullptr);
    }
    // strided gather of G[i,i]: pitch (ld+1) doubles, one double per row
    CK(cudaMemcpy2DAsync(diag, sizeof(double), h->G, sizeof(double) * (h->ld + 1), sizeof(double), h->N,
                         cudaMemcpyDeviceToHost, h->st));
    CK(cudaStreamSynchronize(h->st));
    return GPB200_OK;
}

int gpb200_fp64_peak(gpb200_handle* h, double* tflops_dmma, double* tflops_dfma) {
    if (!h) return GPB200_EINVAL;
    CK(cudaSetDevice(h->device));
    double t[2] = {0, 0};
    CK(fp64_peak_measure(h->st, &h->launches, t));
    if (tflops_dmma) *tflops_dmma = t[0];
    if (tflops_dfma) *tflops_dfma = t[1];
    return GPB200_OK;
}


#define GPB200_IPC_BYTES 512
int gpb200_ipc_export(gpb200_handle* h, char* out) {
    if (!h || !out) return GPB200_EINVAL;
    if (!h->has_data) return fail(h, GPB200_ESTATE, "ipc_export: set_data first (buffers must exist)");
    CK(cudaSetDevice(h->device));
    memset(out, 0, GPB200_IPC_BYTES);
    cudaIpcMemHandle_t hd[5];
    CK(cudaIpcGetMemHandle(&hd[0], h->F));
    CK(cudaIpcGetMemHandle(&hd[1], h->Dinv));
    CK(cudaIpcGetMemHandle(&hd[2], h->DinvT));
    CK(cudaIpcGetMemHandle(&hd[3], h->logd));
    CK(cudaIpcGetMemHandle(&hd[4], h->sig));
    static_assert(5 * sizeof(cudaIpcMemHandle_t) + 16 <= GPB200_IPC_BYTES, "ipc blob too small");
    memcpy(out, hd, sizeof hd);
    const int64_t np = h->Npad;
    memcpy(out + sizeof hd, &np, sizeof np);
    return GPB200_OK;
}

int gpb200_ipc_import(gpb200_handle* h, int nranks, const char* all) {
    if (!h || !all) return GPB200_EINVAL;
    if (nranks != h->nranks || nranks < 2 || nranks > 8) return fail(h, GPB200_EINVAL, "ipc_import: call comm_init first; 2..8 ranks");
    CK(cudaSetDevice(h->device));
    close_peer_maps(h);                        // re-import: drop the previous mappings first
    int n = 0;
    for (int q = 0; q < nranks; ++q) {
        if (q == h->rank) continue;
        const char* blob = all + (size_t)q * GPB200_IPC_BYTES;
        cudaIpcMemHandle_t hd[5];
        memcpy(hd, blob, sizeof hd);
        int64_t np = 0;
        memcpy(&np, blob + sizeof hd, sizeof np);
        if (np != h->Npad) return fail(h, GPB200_EINVAL, "ipc_import: peers hold a different problem size");
        void* ptr[5];
        for (int k = 0; k < 5; ++k) CK(cudaIpcOpenMemHandle(&ptr[k], hd[k], cudaIpcMemLazyEnablePeerAccess));
        h->peer_rank[n] = q;
        h->peer_F[n] = (double*)ptr[0]; h->peer_Dinv[n] = (double*)ptr[1]; h->peer_DinvT[n] = (double*)ptr[2];
        h->peer_logd[n] = (double*)ptr[3]; h->peer_sig[n] = (int*)ptr[4];
        ++n;
    }
    h->n_peer = n;
    int* words[7];
    for (int q = 0; q < n; ++q) words[q] = h->peer_sig[q] + h->rank;
    if (!h->peer_sig_dev) CK(h->peer_sig_dev.alloc(8));
    CK(cudaMemcpy(h->peer_sig_dev, words, sizeof(int*) * n, cudaMemcpyHostToDevice));
    h->p2p = true;
    return GPB200_OK;
}

int gpb200_nccl_unique_id(char* id128) {
    if (!id128) return GPB200_EINVAL;
    if (!nccl_load()) { g_create_error = "libnccl.so.2 could not be loaded"; return GPB200_ENCCL; }
    ncclUniqueId id;
    if (g_nccl.GetUniqueId(&id) != ncclSuccess) { g_create_error = "ncclGetUniqueId failed"; return GPB200_ENCCL; }
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
    memcpy(id128, &id, 128);
    return GPB200_OK;
}

int gpb200_comm_init(gpb200_handle* h, int nranks, int rank, const char* id128) {
    if (!h || !id128 || nranks < 1 || rank < 0 || rank >= nranks) return GPB200_EINVAL;
    if (nranks & (nranks - 1)) return fail(h, GPB200_EINVAL, "comm_init: number of ranks must be a power of two");
    if (h->grp) return fail(h, GPB200_ESTATE, "comm_init: handle belongs to an in-process group");
    if (!nccl_load()) return fail(h, GPB200_ENCCL, "libnccl.so.2 could not be loaded");
    CK(cudaSetDevice(h->device));
    if (h->comm) { g_nccl.CommDestroy(h->comm); h->comm = nullptr; }
    ncclUniqueId id;
    memcpy(&id, id128, 128);
    CKN(g_nccl.CommInitRank(&h->comm, nranks, id, rank));
    if (!h->st_comm) CK(cudaStreamCreateWithFlags(&h->st_comm, cudaStreamNonBlocking));
    for (int i = 0; i < 2; ++i) {
        if (!h->ev_packed[i]) CK(cudaEventCreateWithFlags(&h->ev_packed[i], cudaEventDisableTiming));
        if (!h->ev_bcast[i]) CK(cudaEventCreateWithFlags(&h->ev_bcast[i], cudaEventDisableTiming));
        if (!h->ev_unpacked[i]) CK(cudaEventCreateWithFlags(&h->ev_unpacked[i], cudaEventDisableTiming));
    }
    if (!h->ev_x) CK(cudaEventCreateWithFlags(&h->ev_x, cudaEventDisableTiming));
    if (!h->ev_y) CK(cudaEventCreateWithFlags(&h->ev_y, cudaEventDisableTiming));
    h->nranks = nranks; h->rank = rank;
    h->factored = h->inv_ready = h->s_ready = false;
    return GPB200_OK;
}


int gpb200_storage_info(gpb200_handle* h, int64_t* out, int32_t n) {
    if (!h || !out) return GPB200_EINVAL;
    int64_t v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    v[6] = h->tma_ok ? 1 : 0;
    v[0] = h->sharded ? 1 : 0;
    v[1] = h->sharded ? (int64_t)vm_mapped_bytes(h->vmF) : (h->F ? (int64_t)sizeof(double) * h->Npad * h->Npad : 0);
    v[2] = h->sharded ? (int64_t)vm_mapped_bytes(h->vmG) : (h->G ? (int64_t)sizeof(double) * h->Npad * h->Npad : 0);
    v[3] = h->sharded ? h->rb : 0;
    v[4] = h->nranks;
    v[5] = h->rank;
    v[7] = h->sharded ? (int64_t)(vm_mapped_bytes(h->vmCvY) + vm_mapped_bytes(h->vmCvM))
                      : (h->cvD && h->cvY ? 2 * (int64_t)sizeof(double) * h->Npad * h->Npad : 0);
    for (int i = 0; i < n && i < 8; ++i) out[i] = v[i];
    return GPB200_OK;
}

int gpb200_group_create(gpb200_handle** hs, int n) {
    if (!hs || n < 1 || n > 8) return GPB200_EINVAL;
    for (int i = 0; i < n; ++i) {
        if (!hs[i]) return GPB200_EINVAL;
        if (hs[i]->grp || hs[i]->comm) return fail(hs[i], GPB200_ESTATE, "group_create: handle already belongs to a group / communicator");
        if (hs[i]->device != hs[0]->device) return fail(hs[i], GPB200_EINVAL, "group_create: all handles must live on one device");
        for (int j = 0; j < i; ++j) if (hs[j] == hs[i]) return fail(hs[i], GPB200_EINVAL, "group_create: duplicate handle");
    }
    gpb200_group* g = new gpb200_group();
    for (int i = 0; i < n; ++i) {
        g->hs.push_back(hs[i]);
        hs[i]->grp = g; hs[i]->nranks = n; hs[i]->rank = i;
        hs[i]->factored = hs[i]->inv_ready = hs[i]->s_ready = false;
    }
    return GPB200_OK;
}

}  // extern "C"
