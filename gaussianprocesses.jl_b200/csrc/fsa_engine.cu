// fsa_engine.cu -- the FSA schedule of the sparse handle gpb200_fitc (mode 3): training blocks, the packed
// block-diagonal factors, and the likelihood, gradient and block-paired prediction passes on top of fitc_engine.cu's
// K_uu, Sigma_QR and N-chunk streaming.
#include <limits.h>

#include <memory>

#include "engine.cuh"
#include "fsa.cuh"
#include "gram.cuh"
#include "potrf_base.cuh"
#include "vec.cuh"

using namespace engine;

// ================================================================================================
// FSA -- Full Scale Approximation (src/sparse/full_scale_approximation.jl), mode 3 of the sparse engine:
//   Sigma = Q_ff + Lambda,  Lambda = blockdiag(Lambda_i),  Lambda_i = K_ii - V_i V_i' + (sigma^2 + 1e-10) I  (:197-230).
// K_uu, Sigma_QR = K_uu + K_uf Lambda^-1 K_fu, alpha_u and the N-chunk streaming are FITC's.  gpb200_fitc_set_blocks
// reorders the training rows once so that every block is contiguous and starts on a 128-row boundary (padding rows are
// zero in K_fu, zero in r, identity in Lambda); a staging chunk then holds whole blocks, and every per-block product is a
// list of aligned 128 x 128 tiles -- one grouped-GEMM launch (fsa.cu) per operation and chunk, whatever the number of blocks.
// Per block, packed with leading dimension B_i (fsa.cuh):
//   X   Lambda_i in the lower tiles during the factorisation -> X = L_i^-1 in the lower tiles; the strictly-upper tiles are
//       scratch (T' of the inverse recurrence below) and are never read as X;
//   LT  L_i in the strictly-lower tiles (panels) and X' = L_i^-T in the upper tiles (diagonal tiles: clean upper X_ss').
// Batched right-looking block Cholesky + inverse, step s = 0 .. (largest block's tiles - 1), one launch each, over every
// block that still has a tile s:
//   leaf   X_ss = L_ss^-1, X_ss' and 2 log diag(L_ss) from the Schur-updated Lambda_ss (potrf128_ptr_launch)
//   panel  L_is = Lambda_is X_ss'                                        (i > s)
//   trail  Lambda_ij -= L_is L_js'                                        (i >= j > s)
//   inv1   T_sj' = sum_{j <= k < s} X_kj' L_sk'  -> X(j, s) scratch     (j < s)
//   inv2   X_sj = -X_ss T_sj ;  X_js' = -T_sj' X_ss'                     (j < s)
// ================================================================================================
static constexpr int FSA_MAX_BLOCK = 2048;
struct FsaLaunch { int64_t off = 0; int n = 0; };
struct FsaChunk {
    int64_t r0 = 0, rows = 0;                           // padded rows [r0, r0 + rows), whole blocks, rows <= Nc
    FsaLaunch gram, vv, wt, z;
    std::vector<FsaLaunch> leaf, panel, trail, inv1, inv2;
    // kernel gradient: G_i = alpha_i alpha_i' - Lambda_i^-1 + Y_i Y_i' as full tiles of the chunk's blocks in Gpk
    FsaLaunch gtiles;                                   // FsaGramItem list: every tile (r, c) of every block, dst in Gpk
    FsaLaunch ginv, gyy, gp1t;                          // -X_r' X_c tiles ; += Y_r Y_c' ; (K_uu^-1 K_uf G_bd) (bufA, Mpad x Nc)
    FsaLaunch bdx;                                      // training-input gradient: FsaBlockDxItem list, one per tile row of a block
};
// first use of gpb200_fitc_predict_fsa: V* = K_*u L_uu^-T, the C / G tiles of the test rows (Nc x 2048 each) and the
// per-row vectors
struct FsaPredWs {
    DevBuf<double> Vs, Cb, Gb, pvec;
    CUtensorMap mapVs{};
    bool ready = false;
};
// first use of gpb200_fitc_predict_fsa_grad with variances: the s K_ub' tiles of the test rows (Nc x 2048) and
// Z = K_*u + E K_fu / 2 (Nc x Mpad)
struct FsaGradWs {
    DevBuf<double> Tb, Zb;
    CUtensorMap mapZb{};
    bool ready = false;
};
// everything gpb200_fitc_set_blocks builds; it lives until the next set_blocks or set_data (fsa_free)
struct Fsa {
    int64_t nblocks = 0, Np = 0, n_pad = 0, packed = 0;
    int max_tiles = 0;
    std::vector<FsaChunk> chunks;
    DevBuf<double> xb, mask, X, LT, logd;
    DevBuf<double> r, a, t1, t2;
    DevBuf<long long> pos, bstart, boff;
    DevBuf<long long> ipos;                             // padded row -> caller index (-1 on padding): inverse of pos
    DevBuf<FsaBlockDxItem> bdx;
    std::vector<long long> pos_h;                       // pos on the host: gpb200_fitc_set_inputs rebuilds xb through it
    DevBuf<int> rblk, bsize, info;
    DevBuf<FsaGemmItem> gitems;
    DevBuf<Potrf128Item> litems;
    DevBuf<FsaGramItem> gramitems;
    CUtensorMap mapWt{};                                // bufA as Mpad x Nc (W' = K_uf L_Lambda^-T of a chunk)
    DevBuf<double> Gpk, gpart, ones;                    // kernel gradient: one chunk's G_i blocks, trace partials, 1s
    std::vector<long long> bstart_h, boff_h;
    std::vector<int> bsize_h, bchunk_h;                 // bchunk_h[b]: staging chunk of block b
    FsaPredWs pred;
    FsaGradWs pgrad;
    // per-call work lists of the predictions, grown on demand
    DevBuf<FsaGemmItem> pg; DevBuf<FsaGramItem> px; DevBuf<FsaRowItem> pr;
    // CovDest::device: Sigma* gathered into the caller's order (Ms x Ms, dense) through the test-point permutation pp
    DevBuf<double> Sc; DevBuf<long long> pp;
    // gpb200_fitc_predict_fsa_grad: dmu / dvar in the caller's order (2 x Ms x d) and the contraction's items
    DevBuf<double> pdx;
    DevBuf<FsaDxItem> pdi;
};

extern "C" {
int gpb200_fitc_set_blocks(gpb200_fitc* f, int64_t nblocks, const int64_t* block_ptr, const int64_t* idx) {
    if (!f) return GPB200_EINVAL;
    if (!f->has_data) return fail(f, GPB200_ESTATE, "fitc_set_blocks: set_data first");
    if (nblocks < 1 || !block_ptr || !idx) return fail(f, GPB200_EINVAL, "fitc_set_blocks: bad arguments");
    const int64_t N = f->N;
    if (block_ptr[0] != 0 || block_ptr[nblocks] != N)
        return fail(f, GPB200_EINVAL, "fitc_set_blocks: the blocks must partition the N training points (block_ptr[0] = 0, block_ptr[nblocks] = N)");
    int64_t Np = 0, packed = 0;
    int max_tiles = 0;
    for (int64_t b = 0; b < nblocks; ++b) {
        const int64_t n = block_ptr[b + 1] - block_ptr[b];
        if (n < 0) return fail(f, GPB200_EINVAL, "fitc_set_blocks: block_ptr must be non-decreasing");
        if (n > FSA_MAX_BLOCK) return fail(f, GPB200_EINVAL, "fitc_set_blocks: a block holds more than 2048 points");
        const int64_t B = (n + TILE - 1) / TILE * TILE;
        if (B > f->Nc) return fail(f, GPB200_EINVAL, "fitc_set_blocks: a block does not fit one staging chunk");
        Np += B; packed += B * B;
        max_tiles = std::max(max_tiles, (int)(B / TILE));
    }
    std::vector<char> seen((size_t)N, 0);
    for (int64_t k = 0; k < N; ++k) {
        const int64_t i = idx[k];
        if (i < 0 || i >= N || seen[(size_t)i])
            return fail(f, GPB200_EINVAL, "fitc_set_blocks: the blocks must partition 0..N-1 (an index is out of range or repeated)");
        seen[(size_t)i] = 1;
    }
    FCK(cudaSetDevice(f->device));
    fsa_free(f);
    fitc_invalidate(f);
    // set_data sizes the staging chunk to N; the padded blocks and the padded test groups of FSA predictions need the
    // full chunk, so grow it to the cap set_data applies to large N (with every workspace sized by the chunk)
    const int64_t cap = std::min<int64_t>((int64_t)(2.0e9 / (8.0 * (double)f->Mpad)) / TILE * TILE, 32768);
    if (cap > f->Nc) TRY(fitc_stage_alloc(f, cap, "fitc_set_blocks"));
    std::unique_ptr<Fsa> s(new Fsa());            // f->fsa once complete
    s->nblocks = nblocks; s->Np = Np; s->n_pad = Np - N; s->packed = packed; s->max_tiles = max_tiles;
    cudaStream_t st = f->eu->st;
    const int d = f->d;
    const int64_t Mp = f->Mpad, Nc = f->Nc;
    // host tables: padded layout, positions, the reordered inputs
    std::vector<long long> bstart((size_t)nblocks), boff((size_t)nblocks), pos((size_t)N), ipos;
    std::vector<int> bsize((size_t)nblocks), rblk((size_t)Np);
    std::vector<double> mask((size_t)Np, 0.0), xh((size_t)N * d), xb((size_t)Np * d, 0.0);
    FCK(cudaMemcpy(xh.data(), f->data.x, sizeof(double) * N * d, cudaMemcpyDeviceToHost));
    {
        int64_t P = 0, off = 0;
        for (int64_t b = 0; b < nblocks; ++b) {
            const int64_t n = block_ptr[b + 1] - block_ptr[b], B = (n + TILE - 1) / TILE * TILE;
            bstart[b] = P; bsize[b] = (int)B; boff[b] = off;
            for (int64_t j = 0; j < B; ++j) rblk[(size_t)(P + j)] = (int)b;
            for (int64_t j = 0; j < n; ++j) {
                const int64_t i = idx[block_ptr[b] + j];
                pos[(size_t)i] = P + j;
                mask[(size_t)(P + j)] = 1.0;
                memcpy(&xb[(size_t)(P + j) * d], &xh[(size_t)i * d], sizeof(double) * d);
            }
            P += B; off += B * B;
        }
    }
    FCK(s->xb.alloc((size_t)Np * d));
    for (DevBuf<double>* p : {&s->mask, &s->logd, &s->r, &s->a, &s->t1, &s->t2}) FCK(p->alloc(Np));
    FCK(s->X.alloc(packed));
    FCK(s->LT.alloc(packed));
    FCK(cudaMemsetAsync(s->X, 0, sizeof(double) * packed, st));
    FCK(cudaMemsetAsync(s->LT, 0, sizeof(double) * packed, st));
    FCK(s->pos.alloc(N));
    FCK(s->ipos.alloc(Np));
    FCK(s->bstart.alloc(nblocks));
    FCK(s->boff.alloc(nblocks));
    FCK(s->bsize.alloc(nblocks));
    FCK(s->rblk.alloc(Np));
    FCK(s->info.alloc(1));
    // a chunk holds sum B_i <= Nc rows of blocks of at most 2048 rows: its blocks' G_i take at most Nc * 2048 doubles
    FCK(s->Gpk.alloc(std::min<int64_t>(packed, Nc * FSA_MAX_BLOCK)));
    FCK(s->gpart.alloc((size_t)(Nc / TILE) * (FSA_MAX_BLOCK / TILE) * GPB200_MAX_THETA));
    {
        std::vector<double> ones((size_t)Nc, 1.0);
        FCK(s->ones.alloc(Nc));
        FCK(cudaMemcpy(s->ones, ones.data(), sizeof(double) * Nc, cudaMemcpyHostToDevice));
    }
    FCK(cudaMemcpy(s->xb, xb.data(), sizeof(double) * Np * d, cudaMemcpyHostToDevice));
    FCK(cudaMemcpy(s->mask, mask.data(), sizeof(double) * Np, cudaMemcpyHostToDevice));
    FCK(cudaMemcpy(s->pos, pos.data(), sizeof(long long) * N, cudaMemcpyHostToDevice));
    ipos.assign((size_t)Np, -1);
    for (int64_t i = 0; i < N; ++i) ipos[(size_t)pos[(size_t)i]] = i;
    FCK(cudaMemcpy(s->ipos, ipos.data(), sizeof(long long) * Np, cudaMemcpyHostToDevice));
    FCK(cudaMemcpy(s->bstart, bstart.data(), sizeof(long long) * nblocks, cudaMemcpyHostToDevice));
    FCK(cudaMemcpy(s->boff, boff.data(), sizeof(long long) * nblocks, cudaMemcpyHostToDevice));
    FCK(cudaMemcpy(s->bsize, bsize.data(), sizeof(int) * nblocks, cudaMemcpyHostToDevice));
    FCK(cudaMemcpy(s->rblk, rblk.data(), sizeof(int) * Np, cudaMemcpyHostToDevice));
    if (f->eu->tma_ok && !gemm_make_tensor_map(&s->mapWt, f->stage.bufA, Mp, Nc, Nc)) {
        return fail(f, GPB200_ECUDA, "fitc_set_blocks: cuTensorMapEncodeTiled failed");
    }
    s->bstart_h = bstart; s->boff_h = boff; s->bsize_h = bsize; s->pos_h = pos;
    s->bchunk_h.assign((size_t)nblocks, 0);
    // work lists: staging chunks of whole blocks, then every launch of factorize / grad_noise as a range of items
    std::vector<FsaGemmItem> gi;
    std::vector<Potrf128Item> li;
    std::vector<FsaGramItem> gr;
    std::vector<FsaBlockDxItem> bd;
    auto gemm = [&](double* C, long long ldc, const double* A, long long lda, const double* B, long long ldb, int64_t K,
                    double alpha, double beta, bool lower) {
        FsaGemmItem it{};
        it.C = C; it.A = A; it.B = B; it.ldc = ldc; it.lda = lda; it.ldb = ldb; it.K = (int)K;
        it.lower = lower ? 1 : 0; it.alpha = alpha; it.beta = beta;
        gi.push_back(it);
    };
    auto open_g = [&](FsaLaunch& l) { l.off = (int64_t)gi.size(); };
    auto close_g = [&](FsaLaunch& l) { l.n = (int)((int64_t)gi.size() - l.off); };
    for (int64_t b0 = 0; b0 < nblocks;) {
        FsaChunk ch;
        ch.r0 = bstart[b0];
        int64_t b1 = b0;
        while (b1 < nblocks && bstart[b1] + bsize[b1] - ch.r0 <= Nc) ++b1;
        ch.rows = (b1 < nblocks ? bstart[b1] : Np) - ch.r0;
        auto Xt = [&](int64_t b, int i, int j) { return s->X + boff[b] + (int64_t)i * TILE * bsize[b] + (int64_t)j * TILE; };
        auto Lt = [&](int64_t b, int i, int j) { return s->LT + boff[b] + (int64_t)i * TILE * bsize[b] + (int64_t)j * TILE; };
        // Gram tiles of Lambda_i (lower) and the Schur term -V_i V_j' (V = K_fu L_uu^-T of the chunk in bufA)
        ch.gram.off = (int64_t)gr.size();
        open_g(ch.vv);
        for (int64_t b = b0; b < b1; ++b) {
            const int T = bsize[b] / TILE;
            for (int i = 0; i < T; ++i)
                for (int j = 0; j <= i; ++j) {
                    FsaGramItem g{};
                    g.dst = Xt(b, i, j); g.ld = bsize[b]; g.row_i = bstart[b] + i * TILE; g.row_j = bstart[b] + j * TILE; g.diag = (i == j);
                    gr.push_back(g);
                    gemm(Xt(b, i, j), bsize[b], f->stage.bufA + (bstart[b] - ch.r0 + i * TILE) * Mp, Mp,
                         f->stage.bufA + (bstart[b] - ch.r0 + j * TILE) * Mp, Mp, Mp, -1.0, 1.0, i == j);
                }
        }
        ch.gram.n = (int)((int64_t)gr.size() - ch.gram.off);
        close_g(ch.vv);
        for (int k = 0; k < max_tiles; ++k) {
            FsaLaunch lf, pn, tr, i1, i2;
            lf.off = (int64_t)li.size();
            for (int64_t b = b0; b < b1; ++b) {
                if (bsize[b] / TILE <= k) continue;
                Potrf128Item it{};
                it.G = Xt(b, k, k); it.Dinv = Xt(b, k, k); it.DinvT = Lt(b, k, k);
                it.logd = s->logd + bstart[b] + k * TILE; it.ld = bsize[b]; it.info_base = (int)(bstart[b] + k * TILE);
                li.push_back(it);
            }
            lf.n = (int)((int64_t)li.size() - lf.off);
            open_g(pn);
            for (int64_t b = b0; b < b1; ++b)
                for (int i = k + 1; i < bsize[b] / TILE; ++i)
                    gemm(Lt(b, i, k), bsize[b], Xt(b, i, k), bsize[b], Xt(b, k, k), bsize[b], TILE, 1.0, 0.0, false);
            close_g(pn);
            open_g(tr);
            for (int64_t b = b0; b < b1; ++b)
                for (int i = k + 1; i < bsize[b] / TILE; ++i)
                    for (int j = k + 1; j <= i; ++j)
                        gemm(Xt(b, i, j), bsize[b], Lt(b, i, k), bsize[b], Lt(b, j, k), bsize[b], TILE, -1.0, 1.0, i == j);
            close_g(tr);
            open_g(i1);
            for (int64_t b = b0; b < b1; ++b)
                if (bsize[b] / TILE > k)
                    for (int j = 0; j < k; ++j)
                        gemm(Xt(b, j, k), bsize[b], Lt(b, j, j), bsize[b], Lt(b, k, j), bsize[b], (int64_t)(k - j) * TILE, 1.0, 0.0, false);
            close_g(i1);
            open_g(i2);
            for (int64_t b = b0; b < b1; ++b)
                if (bsize[b] / TILE > k)
                    for (int j = 0; j < k; ++j) {
                        gemm(Xt(b, k, j), bsize[b], Xt(b, k, k), bsize[b], Xt(b, j, k), bsize[b], TILE, -1.0, 0.0, false);
                        gemm(Lt(b, j, k), bsize[b], Xt(b, j, k), bsize[b], Xt(b, k, k), bsize[b], TILE, -1.0, 0.0, false);
                    }
            close_g(i2);
            ch.leaf.push_back(lf); ch.panel.push_back(pn); ch.trail.push_back(tr); ch.inv1.push_back(i1); ch.inv2.push_back(i2);
        }
        // W' = K_uf X' (bufB = K_uf chunk -> bufA as Mpad x Nc) and Z = X' W = Lambda^-1 K_fu (bufB as Nc x Mpad)
        open_g(ch.wt);
        for (int64_t b = b0; b < b1; ++b)
            for (int64_t u = 0; u < Mp / TILE; ++u)
                for (int r = 0; r < bsize[b] / TILE; ++r)
                    gemm(f->stage.bufA + u * TILE * Nc + (bstart[b] - ch.r0) + r * TILE, Nc, f->stage.bufB + u * TILE * Nc + (bstart[b] - ch.r0), Nc,
                         Xt(b, r, 0), bsize[b], (int64_t)(r + 1) * TILE, 1.0, 0.0, false);
        close_g(ch.wt);
        open_g(ch.z);
        for (int64_t b = b0; b < b1; ++b)
            for (int64_t u = 0; u < Mp / TILE; ++u)
                for (int r = 0; r < bsize[b] / TILE; ++r)
                    gemm(f->stage.bufB + (bstart[b] - ch.r0 + r * TILE) * Mp + u * TILE, Mp, Lt(b, r, r), bsize[b],
                         f->stage.bufA + u * TILE * Nc + (bstart[b] - ch.r0) + r * TILE, Nc, bsize[b] - (int64_t)r * TILE, 1.0, 0.0, false);
        close_g(ch.z);
        // kernel gradient: every tile of G_i (full, G is symmetric), in Gpk at the block's offset within the chunk
        auto Gt = [&](int64_t b, int i, int j) { return s->Gpk + (boff[b] - boff[b0]) + (int64_t)i * TILE * bsize[b] + (int64_t)j * TILE; };
        ch.gtiles.off = (int64_t)gr.size();
        for (int64_t b = b0; b < b1; ++b)
            for (int i = 0; i < bsize[b] / TILE; ++i)
                for (int j = 0; j < bsize[b] / TILE; ++j) {
                    FsaGramItem g{};
                    g.dst = Gt(b, i, j); g.ld = bsize[b]; g.row_i = bstart[b] + i * TILE; g.row_j = bstart[b] + j * TILE;
                    gr.push_back(g);
                }
        ch.gtiles.n = (int)((int64_t)gr.size() - ch.gtiles.off);
        open_g(ch.ginv);                                // (Lambda^-1)_ij = sum_k X'_ik X'_jk over k >= max(i, j)
        for (int64_t b = b0; b < b1; ++b)
            for (int i = 0; i < bsize[b] / TILE; ++i)
                for (int j = 0; j < bsize[b] / TILE; ++j) {
                    const int k0 = std::max(i, j);
                    gemm(Gt(b, i, j), bsize[b], Lt(b, i, k0), bsize[b], Lt(b, j, k0), bsize[b], bsize[b] - (int64_t)k0 * TILE, -1.0, 0.0, false);
                }
        close_g(ch.ginv);
        open_g(ch.gyy);                                 // Y = Lambda^-1 K_fu L_s^-T in bufB (Nc x Mpad)
        for (int64_t b = b0; b < b1; ++b)
            for (int i = 0; i < bsize[b] / TILE; ++i)
                for (int j = 0; j < bsize[b] / TILE; ++j)
                    gemm(Gt(b, i, j), bsize[b], f->stage.bufB + (bstart[b] - ch.r0 + i * TILE) * Mp, Mp,
                         f->stage.bufB + (bstart[b] - ch.r0 + j * TILE) * Mp, Mp, Mp, 1.0, 1.0, false);
        close_g(ch.gyy);
        open_g(ch.gp1t);                                // (P1' G_bd) with P1' = K_uu^-1 K_uf in bufB (Mpad x Nc) -> bufA (Mpad x Nc)
        for (int64_t b = b0; b < b1; ++b)
            for (int64_t u = 0; u < Mp / TILE; ++u)
                for (int r = 0; r < bsize[b] / TILE; ++r)
                    gemm(f->stage.bufA + u * TILE * Nc + (bstart[b] - ch.r0) + r * TILE, Nc, f->stage.bufB + u * TILE * Nc + (bstart[b] - ch.r0), Nc,
                         Gt(b, r, 0), bsize[b], bsize[b], 1.0, 0.0, false);
        close_g(ch.gp1t);
        ch.bdx.off = (int64_t)bd.size();                // the real tile rows of every block, G_b in Gpk as above
        for (int64_t b = b0; b < b1; ++b) {
            const int64_t n = block_ptr[b + 1] - block_ptr[b];
            for (int r = 0; (int64_t)r * TILE < n; ++r) bd.push_back(FsaBlockDxItem{Gt(b, 0, 0), bstart[b], bsize[b], (int)n, r, 0});
        }
        ch.bdx.n = (int)((int64_t)bd.size() - ch.bdx.off);
        for (int64_t b = b0; b < b1; ++b) s->bchunk_h[(size_t)b] = (int)s->chunks.size();
        s->chunks.push_back(std::move(ch));
        b0 = b1;
    }
    FCK(s->gitems.alloc(std::max<size_t>(gi.size(), 1)));
    FCK(s->litems.alloc(std::max<size_t>(li.size(), 1)));
    FCK(s->gramitems.alloc(std::max<size_t>(gr.size(), 1)));
    FCK(cudaMemcpy(s->gitems, gi.data(), sizeof(FsaGemmItem) * gi.size(), cudaMemcpyHostToDevice));
    FCK(cudaMemcpy(s->litems, li.data(), sizeof(Potrf128Item) * li.size(), cudaMemcpyHostToDevice));
    FCK(cudaMemcpy(s->gramitems, gr.data(), sizeof(FsaGramItem) * gr.size(), cudaMemcpyHostToDevice));
    FCK(s->bdx.alloc(std::max<size_t>(bd.size(), 1)));
    FCK(cudaMemcpy(s->bdx, bd.data(), sizeof(FsaBlockDxItem) * bd.size(), cudaMemcpyHostToDevice));
    FCK(cudaStreamSynchronize(st));
    f->fsa = s.release();
    return GPB200_OK;
}
}  // extern "C"

namespace engine __attribute__((visibility("hidden"))) {
size_t fsa_num_chunks(const gpb200_fitc* f) { return f->fsa ? f->fsa->chunks.size() : 0; }

void fsa_free(gpb200_fitc* f) {
    delete f->fsa;
    f->fsa = nullptr;
}

int fsa_check(gpb200_fitc* f, const char* who) {
    if (f->nranks > 1) return fail(f, GPB200_EINVAL, std::string(who) + ": FSA is single-GPU only");
    if (!f->fsa) return fail(f, GPB200_ESTATE, std::string(who) + ": FSA needs gpb200_fitc_set_blocks after set_data");
    return GPB200_OK;
}

// update_cK! (:197-230) once K_uu, its factor and Sigma_QR = K_uu (+ nuggets) are in place (gpb200_fitc_factorize)
int fsa_factorize(gpb200_fitc* f) {
    Fsa* s = f->fsa;
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int64_t Mp = f->Mpad, Nc = f->Nc;
    const int init = INT_MAX;
    FCK(cudaMemcpyAsync(s->info, &init, sizeof(int), cudaMemcpyHostToDevice, st));
    const GemmBuf bA = gbuf(eu, f->stage.bufA, f->stage.mapA, Mp);
    const GemmBuf bWt = gbuf(eu, f->stage.bufA, s->mapWt, Nc);
    for (const FsaChunk& ch : s->chunks) {
        const double* xr = s->xb + ch.r0 * f->d;
        // V = K_fu L_uu^-T (padding rows zero), then Lambda_i = K_ii + (sigma^2 + 1e-10) I - V_i V_i'
        FCK(fitc_kfu(f, xr, ch.rows));
        FCK(fsa_mask_launch(f->stage.bufA, Mp, ch.rows, Mp, s->mask + ch.r0, nullptr, st, &eu->launches));
        FCK(trsm_rec_buf(eu, bA, (int)Nc, 0, (int)Mp));
        FCK(fsa_gram_launch(eu->prog, s->xb, f->d, s->gramitems + ch.gram.off, ch.gram.n, s->mask, f->noise_var + 1e-10, st, &eu->launches));
        FCK(fsa_gemm_launch(s->gitems + ch.vv.off, ch.vv.n, st, &eu->launches));
        // batched block Cholesky + inverse
        for (int k = 0; k < s->max_tiles; ++k) {
            FCK(potrf128_ptr_launch(s->litems + ch.leaf[k].off, ch.leaf[k].n, s->info, st, &eu->launches));
            FCK(fsa_gemm_launch(s->gitems + ch.panel[k].off, ch.panel[k].n, st, &eu->launches));
            FCK(fsa_gemm_launch(s->gitems + ch.trail[k].off, ch.trail[k].n, st, &eu->launches));
            FCK(fsa_gemm_launch(s->gitems + ch.inv1[k].off, ch.inv1[k].n, st, &eu->launches));
            FCK(fsa_gemm_launch(s->gitems + ch.inv2[k].off, ch.inv2[k].n, st, &eu->launches));
        }
        // W' = K_uf L_Lambda^-T, Sigma_QR += W' W
        FCK(fitc_kuf(f, xr, ch.rows));
        FCK(fsa_mask_launch(f->stage.bufB, Nc, Mp, ch.rows, nullptr, s->mask + ch.r0, st, &eu->launches));
        FCK(fsa_gemm_launch(s->gitems + ch.wt.off, ch.wt.n, st, &eu->launches));
        FCK(gemm_whole(es, bWt, bWt, es->G, es->ld, Mp, Mp, ch.rows, 1.0, 1.0, nullptr, 0, GEMM_LOWER_ONLY));
    }
    int info = INT_MAX;
    FCK(cudaMemcpyAsync(&info, s->info, sizeof(int), cudaMemcpyDeviceToHost, st));
    FCK(cudaStreamSynchronize(st));
    if (info != INT_MAX)
        return fail(f, info, "fitc_factorize (FSA): a block of Lambda is not positive definite (padded row " + std::to_string(info) + ")");
    int rc = chol_inplace(es);
    if (rc != GPB200_OK) return fail(f, rc, "fitc_factorize (Sigma_QR): " + es->err);
    f->factored = true;
    return GPB200_OK;
}

// `\` (:105-108), logdet (:142), get_alpha_u (:366-373):  b = K_uf Lambda^-1 r,  u = Sigma_QR^-1 b,
// alpha = Lambda^-1 (r - K_fu u),  logdet = logdet Sigma_QR - logdet K_uu + sum_i logdet Lambda_i
int fsa_mll(gpb200_fitc* f, const double* y_minus_mean, double* alpha, double* mll, double* logdet) {
    Fsa* s = f->fsa;
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int64_t Np = s->Np, Mp = f->Mpad;
    FCK(cudaMemcpyAsync(f->data.y, y_minus_mean, sizeof(double) * f->N, cudaMemcpyHostToDevice, st));
    FCK(cudaMemsetAsync(s->r, 0, sizeof(double) * Np, st));
    FCK(fsa_permute_launch(1, f->data.y, s->pos, f->N, s->r, st, &eu->launches));
    FCK(fsa_bdmv_launch(0, s->X, s->rblk, s->bstart, s->bsize, s->boff, s->r, s->t1, Np, st, &eu->launches));
    FCK(fsa_bdmv_launch(1, s->LT, s->rblk, s->bstart, s->bsize, s->boff, s->t1, s->t2, Np, st, &eu->launches));     // t2 = Lambda^-1 r
    FCK(cudaMemsetAsync(f->data.bvec, 0, sizeof(double) * Mp, st));
    for (const FsaChunk& ch : s->chunks) {
        FCK(fitc_kuf(f, s->xb + ch.r0 * f->d, ch.rows));
        FCK(rowdot_launch(f->stage.bufB, f->Nc, s->t2 + ch.r0, f->M, ch.rows, f->data.tmpm, st, &eu->launches));
        FCK(ew_launch(2, f->M, f->data.bvec, f->data.tmpm, nullptr, nullptr, 0.0, st, &eu->launches));
    }
    FCK(cudaMemcpyAsync(f->data.rhsm, f->data.bvec, sizeof(double) * Mp, cudaMemcpyDeviceToDevice, st));
    FCK(solve_device(es, f->data.rhsm, f->data.tmpm, f->data.uvec));
    for (const FsaChunk& ch : s->chunks) {
        FCK(fitc_kfu(f, s->xb + ch.r0 * f->d, ch.rows));
        FCK(rowdot_launch(f->stage.bufA, Mp, f->data.uvec, ch.rows, Mp, s->t1 + ch.r0, st, &eu->launches));
    }
    FCK(fsa_resid_launch(s->t1, s->r, s->t1, s->mask, Np, st, &eu->launches));                                      // r - K_fu u, padding 0
    FCK(fsa_bdmv_launch(0, s->X, s->rblk, s->bstart, s->bsize, s->boff, s->t1, s->t2, Np, st, &eu->launches));
    FCK(fsa_bdmv_launch(1, s->LT, s->rblk, s->bstart, s->bsize, s->boff, s->t2, s->a, Np, st, &eu->launches));      // alpha (padded order)
    FCK(fsa_permute_launch(0, s->a, s->pos, f->N, f->data.alpha, st, &eu->launches));
    FCK(dot_launch(s->r, s->a, Np, f->data.scal + 0, st, &eu->launches));
    FCK(sum_launch(es->logd, es->Npad, f->data.scal + 1, st, &eu->launches));
    FCK(sum_launch(eu->logd, eu->Npad, f->data.scal + 2, st, &eu->launches));
    FCK(sum_launch(s->logd, Np, f->data.scal + 3, st, &eu->launches));
    double sc[4];
    FCK(cudaMemcpyAsync(sc, f->data.scal, sizeof(double) * 4, cudaMemcpyDeviceToHost, st));
    if (alpha) FCK(cudaMemcpyAsync(alpha, f->data.alpha, sizeof(double) * f->N, cudaMemcpyDeviceToHost, st));
    FCK(cudaStreamSynchronize(st));
    FSUB(check_trsv_watchdog(es), es);                                   // the solve for u above
    f->Ntotal = (double)f->N;
    const double ld = sc[1] - sc[2] + sc[3];
    if (logdet) *logdet = ld;
    *mll = -(sc[0] + ld + LOG2PI * f->Ntotal) / 2.0;
    f->alpha_ready = true;
    return GPB200_OK;
}

// dmll_noise (:328-363): sigma^2 (alpha'alpha - tr Lambda^-1 + |Lambda^-1 K_fu L_s^-T|_F^2),
// tr Lambda^-1 = |L_Lambda^-1|_F^2 over the real rows (every padding row of X is a unit row)
int fsa_grad_noise(gpb200_fitc* f, double* dmll_noise) {
    Fsa* s = f->fsa;
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int64_t Np = s->Np, Mp = f->Mpad, Nc = f->Nc;
    const GemmBuf bB2 = gbuf(eu, f->stage.bufB, f->stage.mapB2, Mp);
    for (const FsaChunk& ch : s->chunks) {
        FCK(fitc_kuf(f, s->xb + ch.r0 * f->d, ch.rows));
        FCK(fsa_mask_launch(f->stage.bufB, Nc, Mp, ch.rows, nullptr, s->mask + ch.r0, st, &eu->launches));
        FCK(fsa_gemm_launch(s->gitems + ch.wt.off, ch.wt.n, st, &eu->launches));  // W' = K_uf X'               (bufA, Mpad x Nc)
        FCK(fsa_gemm_launch(s->gitems + ch.z.off, ch.z.n, st, &eu->launches));    // Z = X' W = Lambda^-1 K_fu  (bufB, Nc x Mpad)
        FCK(trsm_rec_buf(es, bB2, (int)ch.rows, 0, (int)Mp));                 // Y = Z L_s^-T
        FCK(rowvar_launch(f->stage.bufB, Mp, f->stage.zeroc, ch.rows, Mp, s->t1 + ch.r0, st, &eu->launches));   // -|Y_r|^2
    }
    FCK(sum_launch(s->t1, Np, f->data.scal + 0, st, &eu->launches));
    FCK(dot_launch(s->a, s->a, Np, f->data.scal + 1, st, &eu->launches));
    FCK(fsa_bdmv_launch(2, s->X, s->rblk, s->bstart, s->bsize, s->boff, nullptr, s->t2, Np, st, &eu->launches));
    FCK(sum_launch(s->t2, Np, f->data.scal + 2, st, &eu->launches));
    double sc[3];
    FCK(cudaMemcpyAsync(sc, f->data.scal, sizeof(double) * 3, cudaMemcpyDeviceToHost, st));
    FCK(cudaStreamSynchronize(st));
    *dmll_noise = f->noise_var * (sc[1] - (sc[2] - (double)s->n_pad) - sc[0]);
    return GPB200_OK;
}

// dmll_kern! (:274-326 on top of subsetofregressors.jl:219-253): FITC's regrouping (gpb200_fitc_grad_kernel) with diag(g)
// replaced by the block-diagonal G_bd = blockdiag(alpha_i alpha_i' - Lambda_i^-1 + Y_i Y_i'), the blocks of alpha alpha' - Sigma^-1
// (Sigma^-1 = Lambda^-1 - Lambda^-1 K_fu S^-1 K_uf Lambda^-1, Y = Lambda^-1 K_fu L_s^-T):
//   dmll_p = 1/2 [ <W_fu, dK_fu/dθ_p> + <W_uu, dK_uu/dθ_p> + sum_i <G_i, dK_ii/dθ_p> ]
//   W_fu = 2 alpha beta' - 2 Lambda^-1 K_fu S^-1 - 2 G_bd K_fu K_uu^-1
//   W_uu = -beta beta' + K_uu^-1 - S^-1 + K_uu^-1 (K_uf G_bd K_fu) K_uu^-1
// since dSigma = dQ + blockdiag(dK - dQ) and <alpha alpha' - Sigma^-1, blockdiag(D)> = <G_bd, D>.  Called by
// gpb200_fitc_grad_kernel once K_uu^-1, S^-1 (full symmetric, sub-engines' G) and beta are in place, gacc and Hbuf zeroed.
int fsa_grad_kernel(gpb200_fitc* f, double* dmll_kernel, double* dmll_xu, double* dmll_x) {
    Fsa* s = f->fsa;
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int np = eu->prog.n_theta;
    const int64_t Mp = f->Mpad, Nc = f->Nc;
    const GemmBuf bA = gbuf(eu, f->stage.bufA, f->stage.mapA, Mp);          // bufA as Nc x Mpad
    const GemmBuf bAt = gbuf(eu, f->stage.bufA, s->mapWt, Nc);        // bufA as Mpad x Nc
    const GemmBuf bB2 = gbuf(eu, f->stage.bufB, f->stage.mapB2, Mp);        // bufB as Nc x Mpad
    const GemmBuf bBt = gbuf(eu, f->stage.bufB, f->stage.mapB, Nc);         // bufB as Mpad x Nc
    size_t xk = 0, rk = 0;                                        // inducing-point / training-input contractions so far
    for (const FsaChunk& ch : s->chunks) {
        const double* xr = s->xb + ch.r0 * f->d;
        const int64_t nc = ch.rows;
        FCK(fitc_kuf(f, xr, nc));
        FCK(fsa_mask_launch(f->stage.bufB, Nc, Mp, nc, nullptr, s->mask + ch.r0, st, &eu->launches));
        FCK(fsa_gemm_launch(s->gitems + ch.wt.off, ch.wt.n, st, &eu->launches));  // W' = K_uf X'                   (bufA, Mpad x Nc)
        FCK(fsa_gemm_launch(s->gitems + ch.z.off, ch.z.n, st, &eu->launches));    // Z = Lambda^-1 K_fu             (bufB, Nc x Mpad)
        FCK(gemm_whole(es, bB2, bufG(es), f->grad.bufC, Mp, nc, Mp, Mp, 1.0, 0.0));  // P2 = Z S^-1 -> bufC
        FCK(trsm_rec_buf(es, bB2, (int)nc, 0, (int)Mp));       // Y = Z L_s^-T                   (bufB)
        // G_i = -Lambda_i^-1 + Y_i Y_i' + alpha_i alpha_i'  (Gpk), then sum_i <G_i, dK_ii/dθ_p>
        FCK(fsa_gemm_launch(s->gitems + ch.ginv.off, ch.ginv.n, st, &eu->launches));
        FCK(fsa_gemm_launch(s->gitems + ch.gyy.off, ch.gyy.n, st, &eu->launches));
        FCK(fsa_outer_launch(s->gramitems + ch.gtiles.off, ch.gtiles.n, s->a, st, &eu->launches));
        FCK(fsa_trace_launch(eu->prog, s->xb, f->d, s->gramitems + ch.gtiles.off, ch.gtiles.n, s->mask, s->gpart, f->grad.gtmp, st, &eu->launches));
        FCK(ew_launch(2, np, f->grad.gacc, f->grad.gtmp, nullptr, nullptr, 0.0, st, &eu->launches));
        if (dmll_x) {                                               // the G_b part of dmll/dX, written in the caller's order
            ++rk;
            FCK(cudaEventRecord(f->x_ev[2 * rk], st));
            FCK(fsa_block_dx_launch(eu->prog, s->xb, f->d, s->bdx + ch.bdx.off, ch.bdx.n, s->ipos, f->dx, 0, st, &eu->launches));
            FCK(cudaEventRecord(f->x_ev[2 * rk + 1], st));
        }
        // P1' = K_uu^-1 K_uf (bufB, Mpad x Nc) from K_fu (bufA)
        FCK(fitc_kfu(f, xr, nc));
        FCK(fsa_mask_launch(f->stage.bufA, Mp, nc, Mp, s->mask + ch.r0, nullptr, st, &eu->launches));
        FCK(gemm_whole(eu, bufG(eu), bA, f->stage.bufB, Nc, Mp, nc, Mp, 1.0, 0.0));
        // W_fu = 2 alpha beta' - 2 P2 - 2 G_bd P1  (bufC); P1' G_bd -> bufA (Mpad x Nc)
        FCK(fitc_wfu_launch(f->grad.bufC, f->stage.bufA, Mp, nc, f->M, s->a + ch.r0, s->ones, f->stage.zeroc, f->grad.betav, st, &eu->launches));   // g = 0: P1 unused
        FCK(fsa_gemm_launch(s->gitems + ch.gp1t.off, ch.gp1t.n, st, &eu->launches));
        FCK(fsa_axpy_t_launch(f->grad.bufC, Mp, f->stage.bufA, Nc, nc, Mp, -2.0, st, &eu->launches));
        FCK(trace_rect_launch(eu->prog, xr, f->d, nc, eu->x, f->d, f->M, f->d, f->grad.bufC, Mp, f->grad.gpart, f->grad.gtmp, st, &eu->launches));
        FCK(ew_launch(2, np, f->grad.gacc, f->grad.gtmp, nullptr, nullptr, 0.0, st, &eu->launches));
        // dmll/dXu: the padding rows of the chunk are skipped (mask 0); Xu is in the caller's order (never permuted)
        if (dmll_xu) { TRY(xu_contract(f, xk + 1, xr, nc, f->grad.bufC, 0, s->mask + ch.r0, xk > 0)); ++xk; }
        if (dmll_x) { TRY(x_rows(f, rk + 1, xr, nc, f->grad.bufC, nullptr, s->mask + ch.r0, s->ipos + ch.r0, f->dx, 1)); ++rk; }
        FCK(gemm_whole(eu, bBt, bAt, f->grad.Hbuf, Mp, Mp, Mp, nc, 1.0, 1.0));   // H += P1' G_bd P1 = K_uu^-1 (K_uf G_bd K_fu) K_uu^-1
    }
    FCK(fitc_wuu_launch(f->grad.Wbuf, f->grad.Hbuf, eu->G, es->G, Mp, f->M, f->grad.betav, st, &eu->launches));
    FCK(trace_rect_launch(eu->prog, eu->x, f->d, f->M, eu->x, f->d, f->M, f->d, f->grad.Wbuf, Mp, f->grad.gpart, f->grad.gtmp, st, &eu->launches));
    FCK(ew_launch(2, np, f->grad.gacc, f->grad.gtmp, nullptr, nullptr, 0.0, st, &eu->launches));
    if (dmll_xu) {
        TRY(xu_contract(f, xk + 1, eu->x, f->M, f->grad.Wbuf, 1, nullptr, xk > 0)); ++xk;
        FCK(cudaEventRecord(f->xu_ev[1], st));
    }
    if (dmll_x) FCK(cudaEventRecord(f->x_ev[1], st));
    std::vector<double> out((size_t)std::max(np, 1));
    FCK(cudaMemcpyAsync(out.data(), f->grad.gacc, sizeof(double) * np, cudaMemcpyDeviceToHost, st));
    FCK(cudaStreamSynchronize(st));
    FSUB(check_trsv_watchdog(eu), eu);                                   // the solve for beta in gpb200_fitc_grad_kernel
    if (dmll_kernel) for (int p = 0; p < np; ++p) dmll_kernel[p] = 0.5 * out[p];
    if (dmll_xu) TRY(xu_finish(f, xk, dmll_xu));
    if (dmll_x) TRY(x_finish(f, rk, dmll_x));
    return GPB200_OK;
}

// gpb200_fitc_set_inputs: the padded inputs xb through the row map of gpb200_fitc_set_blocks, built as it builds them
int fsa_set_inputs(gpb200_fitc* f, const double* x, int64_t ldx) {
    Fsa* s = f->fsa;
    const int d = f->d;
    std::vector<double> xb((size_t)s->Np * d, 0.0);
    for (int64_t i = 0; i < f->N; ++i) memcpy(&xb[(size_t)s->pos_h[(size_t)i] * d], x + i * ldx, sizeof(double) * d);
    FCK(cudaMemcpy(s->xb, xb.data(), sizeof(double) * s->Np * d, cudaMemcpyHostToDevice));
    return GPB200_OK;
}

// predictMVN / predict_f with test blocks (:413-478): test block j is paired with training block j, Lambda_xf = K_xf - Q_xf on the
// paired blocks and 0 elsewhere.  With C = Lambda_xf, G = C L_Lambda^-T, W = L_Lambda^-1 K_fu and V_* = L_uu^-1 K_u*:
//   mu = K_*u u + C alpha ,   Sigma = K_** - V_*' V_* - G G' + R R' ,   R = (K_*u - G W) L_s^-T
// (from Sigma^-1 = Lambda^-1 - Lambda^-1 K_fu S^-1 K_uf Lambda^-1 and S = K_uu + K_uf Lambda^-1 K_fu; C = 0 is the FITC formula).
// G G' is block-diagonal in the test blocks.  Test points are grouped by paired block, each group padded to 128 rows, and
// streamed in chunks of at most Nc padded rows; per chunk, the training chunks of the paired blocks are revisited (V, K_uf).
//
// dmu != null (gpb200_fitc_predict_fsa_grad; no Sigma*): the same launches give mu and var, then per test chunk the
// gradients with respect to the test inputs.  With c = C row m, h = H row m, D_u / D_b / D_** the input derivatives of
// k(x*, u_j), k(x*, x_i) (i in the paired block b) and k(x*, x*), and s = S^-1 r~' (= R L_s^-1, r~ = K_*u - C Lambda_b^-1 K_bu):
//   dmu  = D_u (u - beta) + D_b alpha_b ,               beta = K_uu^-1 K_ub alpha_b
//   dvar = D_** + D_u 2 (s - K_uu^-1 Z) + D_b e ,       e = -2 (h + s K_ub Lambda_b^-1) ,  Z = k_u + K_ub e / 2
// (dc = D_b - D_u K_uu^-1 K_ub; c = 0 gives the FITC formula).  s comes from the right-side TRSM on es after R; a second
// sweep over the paired training chunks regenerates K_fu / K_uf and forms s K_ub' (the C tiles' shape, into Tb), its
// product with Lambda_b^-1 = X'X through Gb, e (over H, in the C tiles), then Z += e K_bu / 2 and alpha_b K_bu (A read
// with lda = 0, every row of a test tile the same alpha_b) into the Mpad-wide test rows of Zb and Vs; beta is formed per
// test row rather than once per block, so that it shares the row layout, the GEMM shape and the two K_uu^-1 TRSMs of Z.
// One fsa_crossgram_dx launch per chunk writes dmu / dvar into the caller's order.
// Sigma* (cov_to, into cov with CovDest::host) needs the padded test blocks in one staging chunk; CovDest::device leaves it
// in Sc and mu* in stage.tmpc, in the caller's order, as *out says.
int fsa_predict(gpb200_fitc* f, int64_t Ms, const double* xs, int64_t ldxs, const int64_t* block_of, double* mu, double* var,
                CovDest cov_to, double* cov, double* dmu, double* dvar, DevPrediction* out) {
    if (!f || Ms <= 0 || !xs || !block_of || !mu) return GPB200_EINVAL;
    if (f->mode != 3) return fail(f, GPB200_EINVAL, "fitc_predict_fsa: the handle is not in FSA mode (3)");
    if (!f->fsa || !f->factored || !f->alpha_ready) return fail(f, GPB200_ESTATE, "fitc_predict_fsa: set_blocks, factorize and mll first");
    if (ldxs < f->d) return fail(f, GPB200_EINVAL, "fitc_predict_fsa: ldxs < d");
    FCK(cudaSetDevice(f->device));
    Fsa* s = f->fsa;
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int d = f->d;
    const int64_t Mp = f->Mpad, Nc = f->Nc, nb = s->nblocks;
    const int64_t LDC = (int64_t)s->max_tiles * TILE;         // leading dimension of the C / G tile rows: the largest block
    // group by paired block (ascending, unpaired last), each group padded to whole tiles
    std::vector<int64_t> key((size_t)Ms), cnt((size_t)nb + 1, 0);
    for (int64_t i = 0; i < Ms; ++i) {
        const int64_t b = block_of[i];
        key[(size_t)i] = (b >= 0 && b < nb && s->bsize_h[(size_t)b] > 0) ? b : nb;
        ++cnt[(size_t)key[(size_t)i]];
    }
    std::vector<int64_t> gstart((size_t)nb + 1), fill((size_t)nb + 1, 0), tile_blk;
    int64_t Msp = 0;
    for (int64_t b = 0; b <= nb; ++b) {
        gstart[(size_t)b] = Msp;
        const int64_t tiles = (cnt[(size_t)b] + TILE - 1) / TILE;
        for (int64_t t = 0; t < tiles; ++t) tile_blk.push_back(b < nb ? b : -1);
        Msp += tiles * TILE;
    }
    const bool want_cov = cov_to != CovDest::none, cov_host = cov_to == CovDest::host;
    if (want_cov && Msp > Nc) return fail(f, GPB200_EINVAL, "fitc_predict_fsa: cov needs the padded test blocks in one staging chunk");
    if (want_cov) FCK(f->Kss.ensure((size_t)Msp * Msp));
    std::vector<int64_t> ppos((size_t)Ms);
    std::vector<double> xsp((size_t)Msp * d, 0.0);
    for (int64_t i = 0; i < Ms; ++i) {
        const int64_t k = key[(size_t)i], r = gstart[(size_t)k] + fill[(size_t)k]++;
        ppos[(size_t)i] = r;
        for (int q = 0; q < d; ++q) xsp[(size_t)r * d + q] = xs[i * ldxs + q];
    }
    if (!s->pred.ready) TRY(make_group(s->pred, [&] {
        FsaPredWs& g = s->pred;
        FCK(g.Vs.alloc((size_t)Nc * Mp));
        FCK(g.Cb.alloc((size_t)Nc * LDC));
        FCK(g.Gb.alloc((size_t)Nc * LDC));
        FCK(g.pvec.alloc((size_t)Nc * 6));
        if (eu->tma_ok && !gemm_make_tensor_map(&g.mapVs, g.Vs, Nc, Mp, Mp)) {
            return fail(f, GPB200_ECUDA, "fitc_predict_fsa: cuTensorMapEncodeTiled failed");
        }
        g.ready = true;
        return GPB200_OK;
    }));
    const bool grad = dmu != nullptr, gvar = grad && var;
    if (gvar && !s->pgrad.ready) TRY(make_group(s->pgrad, [&] {
        FsaGradWs& g = s->pgrad;
        FCK(g.Tb.alloc((size_t)Nc * LDC));
        FCK(g.Zb.alloc((size_t)Nc * Mp));
        if (eu->tma_ok && !gemm_make_tensor_map(&g.mapZb, g.Zb, Nc, Mp, Mp)) {
            return fail(f, GPB200_ECUDA, "fitc_predict_fsa_grad: cuTensorMapEncodeTiled failed");
        }
        g.ready = true;
        return GPB200_OK;
    }));
    if (grad) FCK(s->pdx.ensure((size_t)2 * Ms * d));
    double *mu1 = s->pred.pvec, *mu2 = mu1 + Nc, *q = mu2 + Nc, *g2 = q + Nc, *r2 = g2 + Nc, *vp = r2 + Nc;
    // work lists of every (test chunk, training chunk) pair; t1 .. ak: the gradient's second sweep
    struct Pass { int chunk; FsaLaunch xg, vv, gg, hh, kh; FsaLaunch mu2, g2; FsaLaunch t1, tx, ee, ek, ak; };
    struct Sub { int64_t t0, t1; std::vector<Pass> passes; FsaLaunch ggt, dx; };
    std::vector<Sub> subs;
    std::vector<FsaGemmItem> gi; std::vector<FsaGramItem> xi; std::vector<FsaRowItem> ri;
    auto gemm = [&](double* C, long long ldc, const double* A, long long lda, const double* B, long long ldb, int64_t K,
                    double alpha, double beta) {
        FsaGemmItem it{};
        it.C = C; it.A = A; it.B = B; it.ldc = ldc; it.lda = lda; it.ldb = ldb; it.K = (int)K; it.alpha = alpha; it.beta = beta;
        gi.push_back(it);
    };
    const int64_t ntiles = (int64_t)tile_blk.size();
    for (int64_t t0 = 0; t0 < ntiles;) {
        Sub sb;
        sb.t0 = t0;
        sb.t1 = std::min(ntiles, t0 + Nc / TILE);
        for (int64_t t = t0; t < sb.t1;) {
            if (tile_blk[(size_t)t] < 0) { ++t; continue; }
            Pass ps;
            ps.chunk = s->bchunk_h[(size_t)tile_blk[(size_t)t]];
            const FsaChunk& ch = s->chunks[(size_t)ps.chunk];
            int64_t te = t;
            while (te < sb.t1 && tile_blk[(size_t)te] >= 0 && s->bchunk_h[(size_t)tile_blk[(size_t)te]] == ps.chunk) ++te;
            auto each = [&](auto fn) {
                for (int64_t u = t; u < te; ++u) {
                    const int64_t b = tile_blk[(size_t)u], tl = u - t0;
                    fn(b, tl);
                }
            };
            ps.xg.off = (int64_t)xi.size();
            each([&](int64_t b, int64_t tl) {
                for (int c = 0; c < s->bsize_h[(size_t)b] / TILE; ++c) {
                    FsaGramItem g{};
                    g.dst = s->pred.Cb + tl * TILE * LDC + c * TILE; g.ld = LDC; g.row_i = tl * TILE; g.row_j = s->bstart_h[(size_t)b] + c * TILE;
                    xi.push_back(g);
                }
            });
            ps.xg.n = (int)((int64_t)xi.size() - ps.xg.off);
            ps.vv.off = (int64_t)gi.size();                     // C -= V_* V_b'
            each([&](int64_t b, int64_t tl) {
                for (int c = 0; c < s->bsize_h[(size_t)b] / TILE; ++c)
                    gemm(s->pred.Cb + tl * TILE * LDC + c * TILE, LDC, s->pred.Vs + tl * TILE * Mp, Mp,
                         f->stage.bufA + (s->bstart_h[(size_t)b] - ch.r0 + c * TILE) * Mp, Mp, Mp, -1.0, 1.0);
            });
            ps.vv.n = (int)((int64_t)gi.size() - ps.vv.off);
            ps.mu2.off = (int64_t)ri.size();                    // C alpha
            each([&](int64_t b, int64_t tl) {
                FsaRowItem r{};
                r.A = s->pred.Cb + tl * TILE * LDC; r.lda = LDC; r.v = s->a + s->bstart_h[(size_t)b]; r.out = mu2 + tl * TILE;
                r.K = s->bsize_h[(size_t)b]; r.sq = 0;
                ri.push_back(r);
            });
            ps.mu2.n = (int)((int64_t)ri.size() - ps.mu2.off);
            ps.gg.off = (int64_t)gi.size();                     // G = C X'
            each([&](int64_t b, int64_t tl) {
                const int B = s->bsize_h[(size_t)b];
                for (int c = 0; c < B / TILE; ++c)
                    gemm(s->pred.Gb + tl * TILE * LDC + c * TILE, LDC, s->pred.Cb + tl * TILE * LDC, LDC,
                         s->X + s->boff_h[(size_t)b] + (int64_t)c * TILE * B, B, (int64_t)(c + 1) * TILE, 1.0, 0.0);
            });
            ps.gg.n = (int)((int64_t)gi.size() - ps.gg.off);
            ps.g2.off = (int64_t)ri.size();                     // |G|^2
            each([&](int64_t b, int64_t tl) {
                FsaRowItem r{};
                r.A = s->pred.Gb + tl * TILE * LDC; r.lda = LDC; r.v = nullptr; r.out = g2 + tl * TILE; r.K = s->bsize_h[(size_t)b]; r.sq = 1;
                ri.push_back(r);
            });
            ps.g2.n = (int)((int64_t)ri.size() - ps.g2.off);
            ps.hh.off = (int64_t)gi.size();                     // H = G X = C Lambda^-1  (into the C tiles)
            each([&](int64_t b, int64_t tl) {
                const int B = s->bsize_h[(size_t)b];
                for (int c = 0; c < B / TILE; ++c)
                    gemm(s->pred.Cb + tl * TILE * LDC + c * TILE, LDC, s->pred.Gb + tl * TILE * LDC + c * TILE, LDC,
                         s->LT + s->boff_h[(size_t)b] + (int64_t)c * TILE * B + c * TILE, B, B - (int64_t)c * TILE, 1.0, 0.0);
            });
            ps.hh.n = (int)((int64_t)gi.size() - ps.hh.off);
            ps.kh.off = (int64_t)gi.size();                     // K_*u -= H K_fu  (= G W)
            each([&](int64_t b, int64_t tl) {
                for (int64_t u = 0; u < Mp / TILE; ++u)
                    gemm(f->stage.bufB + tl * TILE * Mp + u * TILE, Mp, s->pred.Cb + tl * TILE * LDC, LDC,
                         f->stage.bufA + u * TILE * Nc + (s->bstart_h[(size_t)b] - ch.r0), Nc, s->bsize_h[(size_t)b], -1.0, 1.0);
            });
            ps.kh.n = (int)((int64_t)gi.size() - ps.kh.off);
            if (gvar) {
                ps.t1.off = (int64_t)gi.size();                 // T = s K_ub'  (bufB = s, bufA = K_fu of the chunk)
                each([&](int64_t b, int64_t tl) {
                    for (int c = 0; c < s->bsize_h[(size_t)b] / TILE; ++c)
                        gemm(s->pgrad.Tb + tl * TILE * LDC + c * TILE, LDC, f->stage.bufB + tl * TILE * Mp, Mp,
                             f->stage.bufA + (s->bstart_h[(size_t)b] - ch.r0 + c * TILE) * Mp, Mp, Mp, 1.0, 0.0);
                });
                ps.t1.n = (int)((int64_t)gi.size() - ps.t1.off);
                ps.tx.off = (int64_t)gi.size();                 // T X'  (into the G tiles)
                each([&](int64_t b, int64_t tl) {
                    const int B = s->bsize_h[(size_t)b];
                    for (int c = 0; c < B / TILE; ++c)
                        gemm(s->pred.Gb + tl * TILE * LDC + c * TILE, LDC, s->pgrad.Tb + tl * TILE * LDC, LDC,
                             s->X + s->boff_h[(size_t)b] + (int64_t)c * TILE * B, B, (int64_t)(c + 1) * TILE, 1.0, 0.0);
                });
                ps.tx.n = (int)((int64_t)gi.size() - ps.tx.off);
                ps.ee.off = (int64_t)gi.size();                 // e = -2 (H + T X' X)  (over H in the C tiles)
                each([&](int64_t b, int64_t tl) {
                    const int B = s->bsize_h[(size_t)b];
                    for (int c = 0; c < B / TILE; ++c)
                        gemm(s->pred.Cb + tl * TILE * LDC + c * TILE, LDC, s->pred.Gb + tl * TILE * LDC + c * TILE, LDC,
                             s->LT + s->boff_h[(size_t)b] + (int64_t)c * TILE * B + c * TILE, B, B - (int64_t)c * TILE, -2.0, -2.0);
                });
                ps.ee.n = (int)((int64_t)gi.size() - ps.ee.off);
                ps.ek.off = (int64_t)gi.size();                 // Z += e K_bu / 2  (bufA = K_uf of the chunk)
                each([&](int64_t b, int64_t tl) {
                    for (int64_t u = 0; u < Mp / TILE; ++u)
                        gemm(s->pgrad.Zb + tl * TILE * Mp + u * TILE, Mp, s->pred.Cb + tl * TILE * LDC, LDC,
                             f->stage.bufA + u * TILE * Nc + (s->bstart_h[(size_t)b] - ch.r0), Nc, s->bsize_h[(size_t)b], 0.5, 1.0);
                });
                ps.ek.n = (int)((int64_t)gi.size() - ps.ek.off);
            }
            if (grad) {
                ps.ak.off = (int64_t)gi.size();                 // alpha_b K_bu on every row of the tile (into Vs)
                each([&](int64_t b, int64_t tl) {
                    for (int64_t u = 0; u < Mp / TILE; ++u)
                        gemm(s->pred.Vs + tl * TILE * Mp + u * TILE, Mp, s->a + s->bstart_h[(size_t)b], 0,
                             f->stage.bufA + u * TILE * Nc + (s->bstart_h[(size_t)b] - ch.r0), Nc, s->bsize_h[(size_t)b], 1.0, 0.0);
                });
                ps.ak.n = (int)((int64_t)gi.size() - ps.ak.off);
            }
            sb.passes.push_back(ps);
            t = te;
        }
        sb.ggt.off = (int64_t)gi.size();                        // cov: -G G' on the tile pairs of the same block
        if (want_cov) {
            const int64_t mq = (sb.t1 - sb.t0) * TILE;
            for (int64_t t = sb.t0; t < sb.t1; ++t)
                for (int64_t u = sb.t0; u < sb.t1; ++u) {
                    const int64_t b = tile_blk[(size_t)t];
                    if (b < 0 || tile_blk[(size_t)u] != b) continue;
                    gemm(f->Kss + (t - sb.t0) * TILE * mq + (u - sb.t0) * TILE, mq, s->pred.Gb + (t - sb.t0) * TILE * LDC, LDC,
                         s->pred.Gb + (u - sb.t0) * TILE * LDC, LDC, s->bsize_h[(size_t)b], -1.0, 1.0);
                }
        }
        sb.ggt.n = (int)((int64_t)gi.size() - sb.ggt.off);
        subs.push_back(std::move(sb));
        t0 = subs.back().t1;
    }
    std::vector<FsaDxItem> di;                                   // the contraction: one item per real test point
    if (grad) {
        std::vector<int64_t> at((size_t)Msp, -1);
        for (int64_t i = 0; i < Ms; ++i) at[(size_t)ppos[(size_t)i]] = i;
        for (Sub& sb : subs) {
            sb.dx.off = (int64_t)di.size();
            for (int64_t r = sb.t0 * TILE; r < sb.t1 * TILE; ++r) {
                const int64_t i = at[(size_t)r];
                if (i < 0) continue;
                const int64_t b = key[(size_t)i];
                di.push_back(FsaDxItem{r - sb.t0 * TILE, i, b < nb ? s->bstart_h[(size_t)b] : 0, b < nb ? s->bsize_h[(size_t)b] : 0});
            }
            sb.dx.n = (int)((int64_t)di.size() - sb.dx.off);
        }
    }
    auto upload = [&](auto& dst, const auto& v) -> cudaError_t {
        const cudaError_t e = dst.ensure(v.size());
        return e != cudaSuccess || v.empty() ? e : cudaMemcpy(dst, v.data(), sizeof(v[0]) * v.size(), cudaMemcpyHostToDevice);
    };
    FCK(upload(s->pg, gi));
    FCK(upload(s->px, xi));
    FCK(upload(s->pr, ri));
    if (grad) FCK(upload(s->pdi, di));
    const GemmBuf bA = gbuf(eu, f->stage.bufA, f->stage.mapA, Mp);
    const GemmBuf bB2 = gbuf(eu, f->stage.bufB, f->stage.mapB2, Mp);
    const GemmBuf bVs = gbuf(eu, s->pred.Vs, s->pred.mapVs, Mp);
    const GemmBuf bZb = gbuf(eu, s->pgrad.Zb, s->pgrad.mapZb, Mp);
    std::vector<double> mu_p((size_t)Msp), var_p(var ? (size_t)Msp : 0), cov_p(cov_host ? (size_t)Msp * Msp : 0);
    double* ddmu = grad ? s->pdx.data() : nullptr;
    double* ddvar = grad ? s->pdx + Ms * d : nullptr;
    if (grad) {
        for (double& t : f->fsag_ms) t = 0.0;
        FCK(mirror_lower_tiles_launch(eu->F, eu->ld, eu->Npad, st, &eu->launches));      // L' for the right-side TRSMs
        if (var) FCK(mirror_lower_tiles_launch(es->F, es->ld, es->Npad, st, &eu->launches));
    }
    for (const Sub& sb : subs) {
        const int64_t row0 = sb.t0 * TILE, mq = (sb.t1 - sb.t0) * TILE;
        if (grad) FCK(cudaEventRecord(eu->ev0, st));
        FCK(cudaMemcpyAsync(f->stage.xs, xsp.data() + row0 * d, sizeof(double) * mq * d, cudaMemcpyHostToDevice, st));
        FCK(crossgram_launch(eu->prog, f->stage.xs, d, mq, mq, eu->x, d, f->M, Mp, d, f->stage.bufB, Mp, st, &eu->launches));     // K_*u
        FCK(rowdot_launch(f->stage.bufB, Mp, f->data.uvec, mq, Mp, mu1, st, &eu->launches));                                       // K_*u u
        FCK(cudaMemcpyAsync(s->pred.Vs, f->stage.bufB, sizeof(double) * mq * Mp, cudaMemcpyDeviceToDevice, st));
        if (gvar) FCK(cudaMemcpyAsync(s->pgrad.Zb, f->stage.bufB, sizeof(double) * mq * Mp, cudaMemcpyDeviceToDevice, st));      // Z = K_*u
        FCK(trsm_rec_buf(eu, bVs, (int)mq, 0, (int)Mp));                                                 // V_*'
        FCK(kdiag_launch(eu->prog, f->stage.xs, d, mq, r2, st, &eu->launches));
        FCK(rowvar_launch(s->pred.Vs, Mp, r2, mq, Mp, q, st, &eu->launches));                                                 // k** - |V_*|^2
        FCK(cudaMemsetAsync(mu2, 0, sizeof(double) * mq, st));
        FCK(cudaMemsetAsync(g2, 0, sizeof(double) * mq, st));
        for (const Pass& ps : sb.passes) {
            const FsaChunk& ch = s->chunks[(size_t)ps.chunk];
            const double* xr = s->xb + ch.r0 * d;
            FCK(fitc_kfu(f, xr, ch.rows));                                                                 // V of the training chunk
            FCK(fsa_mask_launch(f->stage.bufA, Mp, ch.rows, Mp, s->mask + ch.r0, nullptr, st, &eu->launches));
            FCK(trsm_rec_buf(eu, bA, (int)Nc, 0, (int)Mp));
            FCK(fsa_crossgram_launch(eu->prog, f->stage.xs, s->xb, d, s->px + ps.xg.off, ps.xg.n, s->mask, st, &eu->launches));
            FCK(fsa_gemm_launch(s->pg + ps.vv.off, ps.vv.n, st, &eu->launches));
            FCK(fsa_rowdot_launch(s->pr + ps.mu2.off, ps.mu2.n, st, &eu->launches));
            FCK(fsa_gemm_launch(s->pg + ps.gg.off, ps.gg.n, st, &eu->launches));
            FCK(fsa_rowdot_launch(s->pr + ps.g2.off, ps.g2.n, st, &eu->launches));
            FCK(fsa_gemm_launch(s->pg + ps.hh.off, ps.hh.n, st, &eu->launches));
            FCK(crossgram_launch(eu->prog, eu->x, d, f->M, Mp, xr, d, ch.rows, Nc, d, f->stage.bufA, Nc, st, &eu->launches));   // K_uf of the chunk
            FCK(fsa_mask_launch(f->stage.bufA, Nc, Mp, ch.rows, nullptr, s->mask + ch.r0, st, &eu->launches));
            FCK(fsa_gemm_launch(s->pg + ps.kh.off, ps.kh.n, st, &eu->launches));
        }
        FCK(trsm_rec_buf(es, bB2, (int)mq, 0, (int)Mp));                                                  // R = (K_*u - G W) L_s^-T
        FCK(rowvar_launch(f->stage.bufB, Mp, f->stage.zeroc, mq, Mp, r2, st, &eu->launches));
        FCK(fsa_var_launch(vp, q, g2, r2, mq, st, &eu->launches));
        FCK(ew_launch(2, mq, mu1, mu2, nullptr, nullptr, 0.0, st, &eu->launches));
        FCK(cudaMemcpyAsync(mu_p.data() + row0, mu1, sizeof(double) * mq, cudaMemcpyDeviceToHost, st));
        if (var) FCK(cudaMemcpyAsync(var_p.data() + row0, vp, sizeof(double) * mq, cudaMemcpyDeviceToHost, st));
        if (grad) {
            FCK(cudaEventRecord(eu->ev1, st));
            if (var) FCK(trsm_right_rec_buf(es, bB2, (int)mq, 0, (int)Mp));                             // s = R L_s^-1
            FCK(cudaMemsetAsync(s->pred.Vs, 0, sizeof(double) * mq * Mp, st));
            for (const Pass& ps : sb.passes) {                                                           // second sweep
                const FsaChunk& ch = s->chunks[(size_t)ps.chunk];
                const double* xr = s->xb + ch.r0 * d;
                if (var) {
                    FCK(fitc_kfu(f, xr, ch.rows));                                                       // K_fu of the chunk
                    FCK(fsa_mask_launch(f->stage.bufA, Mp, ch.rows, Mp, s->mask + ch.r0, nullptr, st, &eu->launches));
                    FCK(fsa_gemm_launch(s->pg + ps.t1.off, ps.t1.n, st, &eu->launches));
                    FCK(fsa_gemm_launch(s->pg + ps.tx.off, ps.tx.n, st, &eu->launches));
                    FCK(fsa_gemm_launch(s->pg + ps.ee.off, ps.ee.n, st, &eu->launches));
                }
                FCK(crossgram_launch(eu->prog, eu->x, d, f->M, Mp, xr, d, ch.rows, Nc, d, f->stage.bufA, Nc, st, &eu->launches));
                FCK(fsa_mask_launch(f->stage.bufA, Nc, Mp, ch.rows, nullptr, s->mask + ch.r0, st, &eu->launches));
                if (var) FCK(fsa_gemm_launch(s->pg + ps.ek.off, ps.ek.n, st, &eu->launches));
                FCK(fsa_gemm_launch(s->pg + ps.ak.off, ps.ak.n, st, &eu->launches));
            }
            FCK(cudaEventRecord(eu->ev2, st));
            FCK(trsm_rec_buf(eu, bVs, (int)mq, 0, (int)Mp));                                             // beta
            FCK(trsm_right_rec_buf(eu, bVs, (int)mq, 0, (int)Mp));
            if (var) {
                FCK(trsm_rec_buf(eu, bZb, (int)mq, 0, (int)Mp));                                         // K_uu^-1 Z
                FCK(trsm_right_rec_buf(eu, bZb, (int)mq, 0, (int)Mp));
            }
            FCK(cudaEventRecord(eu->ev3, st));
            FCK(fsa_crossgram_dx_launch(eu->prog, f->stage.xs, eu->x, s->xb, d, f->M, f->data.uvec, s->pred.Vs, f->stage.bufB, s->pgrad.Zb, Mp, s->mask,
                                        s->a, s->pred.Cb, LDC, s->pdi + sb.dx.off, sb.dx.n, ddmu, var ? ddvar : nullptr, st,
                                        &eu->launches));
            FCK(cudaEventRecord(eu->ev4, st));
        }
        if (want_cov) {
            FCK(gram_full_launch(eu->prog, f->stage.xs, d, mq, mq, d, f->Kss, mq, st, &eu->launches));
            FCK(gemm_whole(eu, bVs, bVs, f->Kss, mq, mq, mq, Mp, -1.0, 1.0));                              // - V_*' V_*
            FCK(gemm_whole(es, bB2, bB2, f->Kss, mq, mq, mq, Mp, 1.0, 1.0));                               // + R R'
            FCK(fsa_gemm_launch(s->pg + sb.ggt.off, sb.ggt.n, st, &eu->launches));  // - G G'
            if (cov_host) FCK(cudaMemcpyAsync(cov_p.data(), f->Kss, sizeof(double) * mq * mq, cudaMemcpyDeviceToHost, st));
        }
        FCK(cudaStreamSynchronize(st));
        if (grad) {
            f->fsag_ms[0] += ev_ms(eu->ev0, eu->ev1);
            f->fsag_ms[1] += ev_ms(eu->ev1, eu->ev2);
            f->fsag_ms[2] += ev_ms(eu->ev2, eu->ev3);
            f->fsag_ms[3] += ev_ms(eu->ev3, eu->ev4);
        }
    }
    if (grad) {
        FCK(cudaMemcpyAsync(dmu, ddmu, sizeof(double) * Ms * d, cudaMemcpyDeviceToHost, st));
        if (var) FCK(cudaMemcpyAsync(dvar, ddvar, sizeof(double) * Ms * d, cudaMemcpyDeviceToHost, st));
        FCK(cudaStreamSynchronize(st));
    }
    if (cov_to == CovDest::device) {
        // Sigma* (one sub-chunk: leading dimension Msp) and mu in the caller's order on the device, as the host loop below
        // reorders them
        FCK(s->Sc.ensure((size_t)Ms * Ms));
        FCK(upload(s->pp, ppos));
        FCK(gather_block_launch(s->Sc, f->Kss, Msp, s->pp, Ms, st, &eu->launches));
        FCK(fsa_permute_launch(0, mu1, s->pp, Ms, f->stage.tmpc, st, &eu->launches));
        if (out) *out = DevPrediction{f->stage.tmpc, s->Sc, Ms};
    }
    for (int64_t i = 0; i < Ms; ++i) {
        const size_t r = (size_t)ppos[(size_t)i];
        mu[i] = mu_p[r];
        if (var) var[i] = var_p[r];
        if (cov_host)
            for (int64_t j = 0; j < Ms; ++j) cov[i * Ms + j] = cov_p[r * (size_t)Msp + (size_t)ppos[(size_t)j]];
    }
    return GPB200_OK;
}
}  // namespace engine

extern "C" {
int gpb200_fitc_predict_fsa(gpb200_fitc* f, int64_t Ms, const double* xs, int64_t ldxs, const int64_t* block_of,
                            double* mu, double* var, double* cov) {
    return fsa_predict(f, Ms, xs, ldxs, block_of, mu, var, cov ? CovDest::host : CovDest::none, cov, nullptr, nullptr, nullptr);
}

int gpb200_fitc_predict_fsa_grad(gpb200_fitc* f, int64_t Ms, const double* xs, int64_t ldxs, const int64_t* block_of,
                                 double* mu, double* var, double* dmu, double* dvar) {
    if (!f) return GPB200_EINVAL;
    if (f->mode != 3) return fail(f, GPB200_EINVAL, "fitc_predict_fsa_grad: the handle is not in FSA mode (3)");
    if (f->nranks > 1) return fail(f, GPB200_EINVAL, "fitc_predict_fsa_grad: single GPU handles only");
    if (!f->fsa || !f->factored || !f->alpha_ready) return fail(f, GPB200_ESTATE, "fitc_predict_fsa_grad: set_blocks, factorize and mll first");
    if (Ms <= 0 || !xs || ldxs < f->d || !block_of || !mu || !dmu) {
        return fail(f, GPB200_EINVAL, "fitc_predict_fsa_grad: bad Ms, xs, ldxs, block_of, mu or dmu");
    }
    if (!var != !dvar) return fail(f, GPB200_EINVAL, "fitc_predict_fsa_grad: var and dvar must be given together");
    return fsa_predict(f, Ms, xs, ldxs, block_of, mu, var, CovDest::none, nullptr, dmu, dvar, nullptr);
}
}  // extern "C"
