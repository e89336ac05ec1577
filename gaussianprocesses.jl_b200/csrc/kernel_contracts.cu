// kernel_contracts.cu -- the raw kernels exposed for the parity tests and the roofline bench (include/gpb200.h): each entry
// point launches one kernel family of the engine on caller buffers, so that tests hold it to its contract directly.
#include <limits.h>

#include "engine.cuh"
#include "fitc_cv.cuh"
#include "fsa.cuh"
#include "gpa.cuh"
#include "gram.cuh"
#include "gram_fast.cuh"
#include "potrf_base.cuh"
#include "shard_kernels.cuh"
#include "vec.cuh"

using namespace engine;

extern "C" {
int gpb200_dgemm_nt_device(gpb200_handle* h, int impl, int64_t M, int64_t N, int64_t K, double alpha,
                           const double* dA, int64_t lda, const double* dB, int64_t ldb, double beta, double* dC,
                           int64_t ldc, int lower_only, int reps, double* ms) {
    if (!h || !dA || !dB || !dC) return GPB200_EINVAL;
    if (M % TILE || N % TILE || K % 16 || M <= 0 || N <= 0 || K <= 0 || reps < 1)
        return fail(h, GPB200_EINVAL, "dgemm_nt: M,N multiples of 128, K multiple of 16");
    CK(cudaSetDevice(h->device));
    CUtensorMap ma{}, mb{};
    const bool tma = gemm_make_tensor_map(&ma, dA, M, K, lda) && gemm_make_tensor_map(&mb, dB, N, K, ldb);
    if (impl == 0 && !tma) return fail(h, GPB200_ECUDA, "dgemm_nt: TMA descriptors unavailable");
    GemmDesc g = gemm_desc_default();
    g.A = GemmOperand{GemmBuf{&ma, dA, lda}, bufNone(), 0, 0};
    g.B = GemmOperand{GemmBuf{&mb, dB, ldb}, bufNone(), 0, 0};
    g.C = dC; g.ldc = ldc; g.M = (int)M; g.N = (int)N; g.K = (int)K;
    g.alpha = alpha; g.beta = beta;
    g.flags = lower_only ? GEMM_LOWER_ONLY : 0;
    CK(cudaEventRecord(h->ev0, h->st));
    for (int r = 0; r < reps; ++r) CK(gemm_nt_launch(g, impl, h->st, &h->launches));
    CK(cudaEventRecord(h->ev1, h->st));
    CK(cudaStreamSynchronize(h->st));
    if (ms) *ms = ev_ms(h->ev0, h->ev1);
    return GPB200_OK;
}

int gpb200_gemm_nt_desc(gpb200_handle* h, int impl, const int64_t* desc, int32_t n, double alpha, double beta) {
    if (!h || !desc || n != GPB200_GEMM_DESC_LEN || (impl != 0 && impl != 1)) return GPB200_EINVAL;
    const int64_t* f = desc;
    const int64_t* bufs = desc + 27;                       // (pointer, rows, cols, ld): A, A.sub, B, B.sub, C, Ct, 7 peers
    for (int i = 0; i < 27; ++i)
        if (f[i] < INT_MIN || f[i] > INT_MAX) return fail(h, GPB200_EINVAL, "gemm_nt_desc: field out of int range");
    for (int b = 0; b < 13; ++b) {
        const int64_t* q = bufs + 4 * b;
        if (q[0] && ((q[0] & 15) || (q[3] & 1) || q[1] < 0 || q[2] < 0 || q[2] > q[3]))
            return fail(h, GPB200_EINVAL, "gemm_nt_desc: buffers need 16-byte aligned pointers, even ld >= cols");
    }
    const int64_t* qa = bufs; const int64_t* qas = bufs + 4; const int64_t* qb = bufs + 8; const int64_t* qbs = bufs + 12;
    if (!qa[0] || !qb[0] || !bufs[16]) return fail(h, GPB200_EINVAL, "gemm_nt_desc: A, B and C are required");
    if (f[1] % TILE || f[2] % TILE || f[3] % 16 || f[1] < 0 || f[2] < 0 || f[3] < 0)
        return fail(h, GPB200_EINVAL, "gemm_nt_desc: M, N multiples of 128, K multiple of 16");
    for (const int64_t* s : {qas, qbs})
        if (s[0] && (s[3] != TILE || ((s[1] || s[2]) && (s[1] % TILE || s[2] != TILE))))
            return fail(h, GPB200_EINVAL, "gemm_nt_desc: sub buffers are [Npad x 128] with ld 128");
    if (f[18] < 0 || f[18] > 7) return fail(h, GPB200_EINVAL, "gemm_nt_desc: n_peer in [0, 7]");
    CK(cudaSetDevice(h->device));
    // descriptors as the engine builds them: 16 x 128 boxes with 128B swizzle over the whole buffer; a sub buffer's map
    // covers [Npad x 128].  rows = cols = 0 passes a buffer without a map (the engine's buffers when TMA is unavailable).
    CUtensorMap maps[4];
    const int64_t* ops[4] = {qa, qas, qb, qbs};
    GemmBuf gb[4];
    for (int i = 0; i < 4; ++i) {
        const int64_t* q = ops[i];
        const double* base = reinterpret_cast<const double*>(q[0]);
        const bool want = q[0] && (q[1] > 0 || q[2] > 0);
        if (want && !gemm_make_tensor_map(&maps[i], base, q[1], q[2], q[3]))
            return fail(h, GPB200_ECUDA, "gemm_nt_desc: TMA descriptor could not be built");
        gb[i] = q[0] ? GemmBuf{want ? &maps[i] : nullptr, base, q[3]} : bufNone();
    }
    GemmDesc g = gemm_desc_default();
    g.A = GemmOperand{gb[0], gb[1], (int)f[19], (int)f[20]};
    g.B = GemmOperand{gb[2], gb[3], (int)f[21], (int)f[22]};
    g.C = reinterpret_cast<double*>(bufs[16]); g.ldc = bufs[19]; g.c_row0 = (int)f[23]; g.c_col0 = (int)f[24];
    g.Ct = reinterpret_cast<double*>(bufs[20]); g.ldct = bufs[23]; g.ct_row0 = (int)f[25]; g.ct_col0 = (int)f[26];
    g.flags = (int)f[0]; g.M = (int)f[1]; g.N = (int)f[2]; g.K = (int)f[3];
    g.batch = (int)f[4]; g.zstep = (int)f[5]; g.m_lim = (int)f[6]; g.n_lim = (int)f[7]; g.k_lim = (int)f[8];
    g.klo_off = (int)f[9]; g.bm_mod = (int)f[10]; g.bm_rem = (int)f[11]; g.bn_mod = (int)f[12]; g.bn_rem = (int)f[13];
    g.bm_div = (int)f[14]; g.bm_off = (int)f[15]; g.bn_div = (int)f[16]; g.bn_off = (int)f[17];
    g.n_peer = (int)f[18];
    for (int q = 0; q < g.n_peer; ++q) {
        const int64_t* pq = bufs + 4 * (6 + q);
        if (!pq[0]) return fail(h, GPB200_EINVAL, "gemm_nt_desc: missing peer buffer");
        g.Cpeer[q] = reinterpret_cast<double*>(pq[0]);
    }
    g.alpha = alpha; g.beta = beta;
    if (g.batch < 1) return fail(h, GPB200_EINVAL, "gemm_nt_desc: batch >= 1");
    if ((impl == 0 && (!gb[0].map || !gb[2].map)) || (g.flags & ~63))
        return fail(h, GPB200_EINVAL, "gemm_nt_desc: impl 0 needs maps of A and B; unknown flag");
    const cudaError_t e = gemm_nt_launch(g, impl, h->st, &h->launches);
    if (e == cudaErrorInvalidValue) { (void)cudaGetLastError(); return fail(h, GPB200_EINVAL, "gemm_nt_desc: rejected by gemm_nt_launch"); }
    CK(e);
    CK(cudaStreamSynchronize(h->st));
    return GPB200_OK;
}

int gpb200_fsa_gemm_items(gpb200_handle* h, const int64_t* items, const double* alpha_beta, int32_t n) {
    if (!h || n < 0 || (n > 0 && (!items || !alpha_beta))) return GPB200_EINVAL;
    std::vector<FsaGemmItem> v(n);
    for (int i = 0; i < n; ++i) {
        const int64_t* q = items + 8 * i;                  // C, A, B, ldc, lda, ldb, K, lower
        if (!q[0] || !q[1] || !q[2] || ((q[0] | q[1] | q[2]) & 15) || ((q[3] | q[4] | q[5]) & 1) || q[6] < 0 || q[6] % 16 ||
            q[6] > INT_MAX)
            return fail(h, GPB200_EINVAL, "fsa_gemm_items: 16-byte aligned pointers, even ld, K a multiple of 16");
        v[i] = FsaGemmItem{reinterpret_cast<double*>(q[0]), reinterpret_cast<const double*>(q[1]),
                           reinterpret_cast<const double*>(q[2]), q[3], q[4], q[5], (int)q[6], (int)(q[7] != 0),
                           alpha_beta[2 * i], alpha_beta[2 * i + 1]};
    }
    if (n == 0) return GPB200_OK;
    CK(cudaSetDevice(h->device));
    DevBuf<FsaGemmItem> d;
    CK(d.alloc(n));
    CK(cudaMemcpyAsync(d, v.data(), sizeof(FsaGemmItem) * n, cudaMemcpyHostToDevice, h->st));
    CK(fsa_gemm_launch(d, n, h->st, &h->launches));
    CK(cudaStreamSynchronize(h->st));
    return GPB200_OK;
}

int gpb200_potrf_tiles(gpb200_handle* h, int mode, const int64_t* args, int32_t n, int32_t* info) {
    if (!h || !args || !info || (mode != 0 && mode != 1)) return GPB200_EINVAL;
    if (mode == 0 && n != 39) return fail(h, GPB200_EINVAL, "potrf_tiles: mode 0 takes 39 arguments");
    if (mode == 1 && (n <= 0 || n % 6)) return fail(h, GPB200_EINVAL, "potrf_tiles: mode 1 takes 6 arguments per tile");
    CK(cudaSetDevice(h->device));
    DevBuf<int> dinfo;
    DevBuf<Potrf128Item> ditems;
    const int big = INT_MAX;
    CK(dinfo.alloc(1));
    CK(cudaMemcpyAsync(dinfo, &big, sizeof(int), cudaMemcpyHostToDevice, h->st));
    if (mode == 0) {
        // G, ldg, F, ldf, Dinv, DinvT, logd, p0, ntiles, tile_stride, n_peer, then per peer (F, Dinv, DinvT, logd)
        const int64_t* a = args;
        PotrfPeers pp{};
        pp.n = (int)std::min<int64_t>(std::max<int64_t>(a[10], 0), 7);
        for (int q = 0; q < pp.n; ++q) {
            pp.F[q] = reinterpret_cast<double*>(a[11 + 4 * q]); pp.Dinv[q] = reinterpret_cast<double*>(a[12 + 4 * q]);
            pp.DinvT[q] = reinterpret_cast<double*>(a[13 + 4 * q]); pp.logd[q] = reinterpret_cast<double*>(a[14 + 4 * q]);
        }
        if (a[8] > 0)
            CK(potrf128_launch(reinterpret_cast<const double*>(a[0]), a[1], reinterpret_cast<double*>(a[2]), a[3],
                                reinterpret_cast<double*>(a[4]), reinterpret_cast<double*>(a[5]), reinterpret_cast<double*>(a[6]),
                                dinfo, (int)a[7], (int)a[8], (int)a[9], h->st, &h->launches, &pp));
    } else {
        const int nt = n / 6;
        std::vector<Potrf128Item> v(nt);
        for (int i = 0; i < nt; ++i) {
            const int64_t* q = args + 6 * i;               // G, Dinv, DinvT, logd, ld, info_base
            v[i] = Potrf128Item{reinterpret_cast<const double*>(q[0]), reinterpret_cast<double*>(q[1]),
                                reinterpret_cast<double*>(q[2]), reinterpret_cast<double*>(q[3]), q[4], (int)q[5], 0};
        }
        CK(ditems.alloc(nt));
        CK(cudaMemcpyAsync(ditems, v.data(), sizeof(Potrf128Item) * nt, cudaMemcpyHostToDevice, h->st));
        CK(potrf128_ptr_launch(ditems, nt, dinfo, h->st, &h->launches));
    }
    int hinfo = big;
    CK(cudaMemcpyAsync(&hinfo, dinfo, sizeof(int), cudaMemcpyDeviceToHost, h->st));
    CK(cudaStreamSynchronize(h->st));
    *info = hinfo;
    return GPB200_OK;
}

int gpb200_trsv_tiles(gpb200_handle* h, int schedule, int direction, const int64_t* args, int32_t n, int32_t* watchdog) {
    if (!h || !args || !watchdog || (schedule != 0 && schedule != 1) || (direction != 0 && direction != 1)) return GPB200_EINVAL;
    if (n != 6) return fail(h, GPB200_EINVAL, "trsv_tiles: 6 arguments (F, ldf, Dinv or DinvT, rhs, out, Npad)");
    const int64_t ldf = args[1], Npad = args[5];
    if (!args[0] || !args[2] || !args[3] || !args[4] || ((args[0] | args[2] | args[3] | args[4]) & 15))
        return fail(h, GPB200_EINVAL, "trsv_tiles: 16-byte aligned device pointers");
    if (Npad <= 0 || Npad % TILE || ldf <= 0 || ldf % 2)
        return fail(h, GPB200_EINVAL, "trsv_tiles: Npad a positive multiple of 128, ldf positive and even");
    const int nb = (int)(Npad / TILE);
    CK(cudaSetDevice(h->device));
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device));
    if (schedule == 1 && nb > sms * TRSV_FUSED_CTAS_PER_SM)
        return fail(h, GPB200_EINVAL, "trsv_tiles: the single-launch schedule runs for Npad/128 <= 4 x SMs only");
    const double* F = reinterpret_cast<const double*>(args[0]);
    const double* D = reinterpret_cast<const double*>(args[2]);
    double* rhs = reinterpret_cast<double*>(args[3]);
    double* out = reinterpret_cast<double*>(args[4]);
    *watchdog = 0;
    if (schedule == 0) {
        CK(direction == 0 ? trsv_lower_fwd(F, ldf, D, rhs, out, Npad, h->st, &h->launches)
                          : trsv_lower_bwd(F, ldf, D, rhs, out, Npad, h->st, &h->launches));
        CK(cudaStreamSynchronize(h->st));
        return GPB200_OK;
    }
    DevBuf<int> flags;
    CK(flags.alloc(nb + 1));
    CK(direction == 0 ? trsv_lower_fwd_fused(F, ldf, D, rhs, out, Npad, flags, h->st, &h->launches)
                      : trsv_lower_bwd_fused(F, ldf, D, rhs, out, Npad, flags, h->st, &h->launches));
    int wd = 0;
    CK(cudaMemcpyAsync(&wd, flags + nb, sizeof(int), cudaMemcpyDeviceToHost, h->st));
    CK(cudaStreamSynchronize(h->st));
    *watchdog = wd;
    return GPB200_OK;
}

int gpb200_gpa_kernels(gpb200_handle* h, int which, const int64_t* args, int32_t n) {
    if (!h || !args || which < 0 || which > 2) return GPB200_EINVAL;
    const int want = which == 2 ? 8 : 5;
    if (n != want) return fail(h, GPB200_EINVAL, "gpa_kernels: 5 arguments (trmv, trmv_t) or 8 (scan)");
    const int64_t ld = args[1], Npad = args[want - 1];
    if (Npad <= 0 || Npad % TILE || ld < Npad) return fail(h, GPB200_EINVAL, "gpa_kernels: Npad a positive multiple of 128, ld >= Npad");
    for (int i = 0; i < want - 1; ++i)
        if (i != 1 && !args[i]) return fail(h, GPB200_EINVAL, "gpa_kernels: null device pointer");
    CK(cudaSetDevice(h->device));
    auto cp = [&](int i) { return reinterpret_cast<const double*>(args[i]); };
    auto mp = [&](int i) { return reinterpret_cast<double*>(args[i]); };
    cudaError_t e;
    if (which == 0) e = gpa_trmv_launch(cp(0), ld, cp(2), mp(3), Npad, h->st, &h->launches);
    else if (which == 1) e = gpa_trmv_t_launch(cp(0), ld, cp(2), mp(3), Npad, h->st, &h->launches);
    else e = gpa_scan_launch(cp(0), ld, cp(2), cp(3), cp(4), mp(5), mp(6), Npad, h->st, &h->launches);
    if (e == cudaErrorInvalidValue) { (void)cudaGetLastError(); return fail(h, GPB200_EINVAL, "gpa_kernels: rejected by the launch"); }
    CK(e);
    CK(cudaStreamSynchronize(h->st));
    return GPB200_OK;
}

int gpb200_row_reductions(gpb200_handle* h, int which, const int64_t* args, int32_t n) {
    if (!h || !args || which < 0 || which > 4) return GPB200_EINVAL;
    static const int want[5] = {4, 3, 6, 6, 6};
    if (n != want[which]) return fail(h, GPB200_EINVAL, "row_reductions: dot 4, sum 3, rowdot / rowvar / rowdot2 6 arguments");
    auto cp = [&](int i) { return reinterpret_cast<const double*>(args[i]); };
    auto mp = [&](int i) { return reinterpret_cast<double*>(args[i]); };
    cudaError_t e;
    if (which <= 1) {
        const int64_t len = args[which == 0 ? 2 : 1];
        const int outi = which == 0 ? 3 : 2;
        if (len < 0 || !args[0] || !args[outi] || (which == 0 && !args[1]))
            return fail(h, GPB200_EINVAL, "row_reductions: n >= 0 and non-null pointers");
        CK(cudaSetDevice(h->device));
        e = which == 0 ? dot_launch(cp(0), cp(1), len, mp(3), h->st, &h->launches) : sum_launch(cp(0), len, mp(2), h->st, &h->launches);
    } else {
        // rowdot (K, ldk, alpha, M, N, mu), rowvar (V, ldk, kdiag, M, N, var), rowdot2 (A, B, ld, M, N, q)
        const int64_t ld = which == 4 ? args[2] : args[1], M = args[3], N = args[4];
        if (M < 0 || N < 0 || ld < N || !args[0] || !args[which == 4 ? 1 : 2] || !args[5])
            return fail(h, GPB200_EINVAL, "row_reductions: M, N >= 0, ld >= N and non-null pointers");
        CK(cudaSetDevice(h->device));
        if (which == 2) e = rowdot_launch(cp(0), ld, cp(2), M, N, mp(5), h->st, &h->launches);
        else if (which == 3) e = rowvar_launch(cp(0), ld, cp(2), M, N, mp(5), h->st, &h->launches);
        else e = rowdot2_launch(cp(0), cp(1), ld, M, N, mp(5), h->st, &h->launches);
    }
    CK(e);
    CK(cudaStreamSynchronize(h->st));
    return GPB200_OK;
}

// A local copy of the handle's kernel program at log-scale theta (the handle's own theta and factor stay as they are).
// The program must exist, theta must have n_theta entries and every input dimension the program reads must be < d.
static int local_prog(gpb200_handle* h, const char* what, const double* theta, int32_t ntheta, int64_t d, KProg& P) {
    if (!h->has_kernel) return fail(h, GPB200_ESTATE, (std::string(what) + ": set_kernel first").c_str());
    if (ntheta != h->prog.n_theta || (ntheta > 0 && !theta)) return fail(h, GPB200_EINVAL, (std::string(what) + ": theta has n_theta entries").c_str());
    if (d < 1) return fail(h, GPB200_EINVAL, (std::string(what) + ": d >= 1").c_str());
    P = h->prog;
    for (int q = 0; q < P.n_ops; ++q)
        if (P.op[q] != GPB200_OP_SUM && P.op[q] != GPB200_OP_PROD)
            for (int k = 0; k < P.nd[q]; ++k)
                if (P.dims[P.doff[q] + k] >= d) return fail(h, GPB200_EINVAL, (std::string(what) + ": the program reads a dimension >= d").c_str());
    kprog_set_theta(P, theta);
    return GPB200_OK;
}

int gpb200_fsa_kernels(gpb200_handle* h, int which, const int64_t* args, int32_t n, const double* fargs, int32_t nf) {
    if (!h || (n > 0 && !args) || which < 0 || which > 12 || nf < 0 || (nf > 0 && !fargs)) return GPB200_EINVAL;
    // fixed arguments before the flattened items, and the item stride (0: no items)
    static const int head[13] = {3, 9, 6, 5, 5, 1, 5, 6, 4, 0, 5, 16, 5};
    static const int stride[13] = {5, 0, 0, 0, 0, 5, 5, 0, 5, 6, 0, 4, 5};
    const int hd = head[which], sd = stride[which];
    if (sd ? (n < hd || (n - hd) % sd) : n != hd) return fail(h, GPB200_EINVAL, "fsa_kernels: wrong argument count for this kernel");
    const int ni = sd ? (n - hd) / sd : 0;
    auto ptr = [&](int i) { return reinterpret_cast<double*>(args[i]); };
    const bool bdx = which == 12;                        // block_dx items share the Gram items' stride
    std::vector<FsaGramItem> gitems(sd == 5 && !bdx ? ni : 0);
    std::vector<FsaBlockDxItem> bitems(bdx ? ni : 0);
    std::vector<FsaRowItem> ritems(sd == 6 ? ni : 0);
    std::vector<FsaDxItem> ditems(sd == 4 ? ni : 0);
    int64_t max_nb = 0;
    for (int k = 0; k < ni; ++k) {
        const int64_t* q = args + hd + sd * k;
        if (bdx) {                                       // G, row0, B, n, tile
            if (!q[0] || q[1] < 0 || q[2] < TILE || q[2] % TILE || q[2] > INT_MAX || q[3] < 0 || q[3] > q[2] || q[4] < 0 ||
                q[4] * TILE >= q[2])
                return fail(h, GPB200_EINVAL, "fsa_kernels: block_dx item with a null G, a negative row0, B not a positive "
                                              "multiple of 128, n outside [0, B] or a tile row past B");
            bitems[k] = FsaBlockDxItem{reinterpret_cast<const double*>(q[0]), q[1], (int)q[2], (int)q[3], (int)q[4], 0};
        } else if (sd == 4) {                            // row, out, b0, nb
            if (q[0] < 0 || q[1] < 0 || q[2] < 0 || q[3] < 0)
                return fail(h, GPB200_EINVAL, "fsa_kernels: crossgram_dx item with a negative row, out, b0 or nb");
            ditems[k] = FsaDxItem{q[0], q[1], q[2], q[3]};
            max_nb = std::max(max_nb, q[3]);
        } else if (sd == 5) {                            // dst, ld, row_i, row_j, diag
            if (!q[0] || q[1] < TILE || q[2] < 0 || q[3] < 0)
                return fail(h, GPB200_EINVAL, "fsa_kernels: item with a null dst, ld < 128 or a negative row");
            gitems[k] = FsaGramItem{reinterpret_cast<double*>(q[0]), q[1], q[2], q[3], (int)(q[4] != 0), 0};
        } else {                                         // A, v, out, lda, K, sq
            if (!q[0] || !q[2] || (!q[5] && !q[1]) || q[4] < 0 || q[4] > INT_MAX || q[3] < q[4])
                return fail(h, GPB200_EINVAL, "fsa_kernels: row item with a null pointer, K < 0 or lda < K");
            ritems[k] = FsaRowItem{reinterpret_cast<const double*>(q[0]), reinterpret_cast<const double*>(q[1]),
                                   reinterpret_cast<double*>(q[2]), q[3], (int)q[4], (int)(q[5] != 0)};
        }
    }
    auto need = [&](std::initializer_list<int> idx) {
        for (int i : idx) if (!args[i]) return false;
        return true;
    };
    KProg P{};
    const bool prog = which == 0 || which == 6 || which == 8 || which == 11 || which == 12;
    if (prog) {
        const int64_t d = args[which == 8 ? 2 : which == 11 ? 3 : 1];
        if ((which == 11 || which == 12) && d > GPB200_MAX_DIMS) return fail(h, GPB200_EINVAL, "fsa_kernels: d above GPB200_MAX_DIMS");
        const int32_t want = h->prog.n_theta + (which == 0 ? 1 : 0);
        if (h->has_kernel && nf != want) return fail(h, GPB200_EINVAL, "fsa_kernels: fargs = theta (+ diag_add for fsa_gram)");
        TRY(local_prog(h, "fsa_kernels", fargs, h->prog.n_theta, d, P));
    } else if (nf != (which == 7 ? 1 : 0)) {
        return fail(h, GPB200_EINVAL, "fsa_kernels: fargs = alpha for fsa_axpy_t, none otherwise");
    }
    bool ok = true;
    switch (which) {
    case 0: ok = need({0, 2}); break;                                        // xb, d, mask | items
    case 1: ok = need({1, 2, 3, 4, 5, 7}) && (args[0] == 2 || args[6]) && args[0] >= 0 && args[0] <= 2 && args[8] >= 0; break;
    case 2: ok = need({0}) && args[1] >= args[3] && args[2] >= 0 && args[3] >= 0; break;     // A, ld, nrows, ncols, rowmask, colmask
    case 3: ok = need({1, 2, 4}) && (args[0] == 0 || args[0] == 1) && args[3] >= 0; break;   // scatter, src, pos, n, dst
    case 4: ok = need({0, 1, 2, 3}) && args[4] >= 0; break;                  // out, a, b, mask, n
    case 5: ok = need({0}); break;                                           // a | items
    case 6: ok = need({0, 2, 4}) && (ni == 0 || args[3]); break;             // xb, d, mask, part, out | items
    case 7: ok = need({0, 2}) && args[4] >= 0 && args[5] >= 0 && args[1] >= args[5] && args[3] >= args[4]; break;  // C, ldc, A, lda, nrows, ncols
    case 8: ok = need({0, 1, 3}); break;                                     // xs, xb, d, mask | items
    case 9: break;                                                           // items only
    case 10: ok = need({0, 1, 2, 3}) && args[4] >= 0; break;                 // out, q, g2, r2neg, n
    case 11:    // xs, z, xb, d, M, u, Wb, S1, S2, ldw, mask, alpha, E, lde, dmu, dvar | items
        ok = need({0, 14}) && args[4] >= 0 && (args[4] == 0 || (args[1] && args[5])) && (max_nb == 0 || need({2, 10, 11})) &&
             (!args[6] || args[9] >= args[4]) &&
             (!args[15] || (need({7, 8}) && args[9] >= args[4] && (max_nb == 0 || (args[12] && args[13] >= max_nb))));
        break;
    case 12: ok = need({0, 3}) && (args[4] == 0 || args[4] == 1); break;    // xb, d, map, out, accumulate | items
    }
    if (!ok) return fail(h, GPB200_EINVAL, "fsa_kernels: a null pointer, a negative size, a bad mode or ld below the row width");
    CK(cudaSetDevice(h->device));
    cudaStream_t st = h->st;
    int64_t* L = &h->launches;
    DevBuf<FsaGramItem> dg;
    DevBuf<FsaRowItem> dr;
    DevBuf<FsaDxItem> dd;
    DevBuf<FsaBlockDxItem> db;
    auto items_to_device = [&](const auto& v, auto& d) -> cudaError_t {     // none for an empty list
        if (v.empty()) return cudaSuccess;
        const cudaError_t e = d.alloc(v.size());
        return e != cudaSuccess ? e : cudaMemcpyAsync(d, v.data(), sizeof(v[0]) * v.size(), cudaMemcpyHostToDevice, st);
    };
    CK(bdx ? items_to_device(bitems, db) : sd == 6 ? items_to_device(ritems, dr)
                                         : sd == 4 ? items_to_device(ditems, dd) : items_to_device(gitems, dg));
    cudaError_t e = cudaSuccess;
    switch (which) {
    case 0: e = fsa_gram_launch(P, ptr(0), (int)args[1], dg, ni, ptr(2), fargs[nf - 1], st, L); break;
    case 1: e = fsa_bdmv_launch((int)args[0], ptr(1), reinterpret_cast<const int*>(args[2]), reinterpret_cast<const long long*>(args[3]),
                                reinterpret_cast<const int*>(args[4]), reinterpret_cast<const long long*>(args[5]), ptr(6), ptr(7),
                                args[8], st, L); break;
    case 2: e = fsa_mask_launch(ptr(0), args[1], args[2], args[3], ptr(4), ptr(5), st, L); break;
    case 3: e = fsa_permute_launch((int)args[0], ptr(1), reinterpret_cast<const long long*>(args[2]), args[3], ptr(4), st, L); break;
    case 4: e = fsa_resid_launch(ptr(0), ptr(1), ptr(2), ptr(3), args[4], st, L); break;
    case 5: e = fsa_outer_launch(dg, ni, ptr(0), st, L); break;
    case 6: e = fsa_trace_launch(P, ptr(0), (int)args[1], dg, ni, ptr(2), ptr(3), ptr(4), st, L); break;
    case 7: e = fsa_axpy_t_launch(ptr(0), args[1], ptr(2), args[3], args[4], args[5], fargs[0], st, L); break;
    case 8: e = fsa_crossgram_launch(P, ptr(0), ptr(1), (int)args[2], dg, ni, ptr(3), st, L); break;
    case 9: e = fsa_rowdot_launch(dr, ni, st, L); break;
    case 10: e = fsa_var_launch(ptr(0), ptr(1), ptr(2), ptr(3), args[4], st, L); break;
    case 11: e = fsa_crossgram_dx_launch(P, ptr(0), ptr(1), ptr(2), (int)args[3], args[4], ptr(5), ptr(6), ptr(7), ptr(8),
                                         args[9], ptr(10), ptr(11), ptr(12), args[13], dd, ni, ptr(14), ptr(15), st, L); break;
    case 12: e = fsa_block_dx_launch(P, ptr(0), (int)args[1], db, ni, reinterpret_cast<const long long*>(args[2]), ptr(3),
                                     (int)args[4], st, L); break;
    }
    CK(e);
    CK(cudaStreamSynchronize(st));
    return GPB200_OK;
}

int gpb200_gram_kernels(gpb200_handle* h, int which, const int64_t* args, int32_t n, const double* fargs, int32_t nf) {
    if (!h || (n > 0 && !args) || which < 0 || which > 13 || nf < 0 || (nf > 0 && !fargs)) return GPB200_EINVAL;
    static const int want[14] = {14, 11, 7, 5, 10, 12, 13, 11, 6, 13, 3, 12, 14, 14};
    if (n != want[which]) return fail(h, GPB200_EINVAL, "gram_kernels: wrong argument count for this kernel");
    const int64_t* a = args;
    auto ptr = [&](int i) { return reinterpret_cast<double*>(a[i]); };
    // every argument pointer non-null; a buffer accessed as double2 16-byte aligned with an even leading dimension
    auto need = [&](std::initializer_list<int> idx) {
        for (int i : idx) if (!a[i]) return false;
        return true;
    };
    auto vec2 = [&](int p, int ld) { return a[p] % 16 == 0 && a[ld] % 2 == 0; };
    auto padded = [&](int size, int pad) { return a[size] >= 0 && a[pad] >= a[size] && a[pad] % TILE == 0; };
    KProg P{};
    int64_t d = 1;
    if (which != 10) {
        static const int dpos[14] = {2, 8, 4, 2, 2, 8, 2, 6, 2, 6, 0, 2, 2, 2};
        d = a[dpos[which]];
        if (d < 1 || d > GPB200_MAX_DIMS) return fail(h, GPB200_EINVAL, "gram_kernels: d outside 1 .. GPB200_MAX_DIMS");
        const int32_t extra = (which == 0 || which == 9 || which == 12) ? 1 : 0;       // nugget / c after theta
        if (h->has_kernel && nf != h->prog.n_theta + extra)
            return fail(h, GPB200_EINVAL, "gram_kernels: fargs = theta (+ nugget for gram_lower, c for crossgram_dx)");
        TRY(local_prog(h, "gram_kernels", fargs, h->prog.n_theta, d, P));
    } else if (nf != 0) {
        return fail(h, GPB200_EINVAL, "gram_kernels: mirror_lower_tiles takes no fargs");
    }
    const int np = P.n_theta;
    auto jok = [&](int i) { return a[i] >= 0 && a[i] < np; };
    // the TMA-staged SEIso kernels (12, 13): the single SEIso leaf over d <= 8 dimensions with constants the fast exp accepts,
    // 16-byte aligned inputs xp [N x dx] and xpt [dx x Npad], dx = d rounded up to even
    const bool tma = which == 12 || which == 13;
    SeIsoFast sf{};
    if (tma && !(kprog_fast(P, (int)d) && d <= 8 && seiso_fast_prepare(P.par[0], P.par[1], &sf) && need({0, 1}) &&
                 a[0] % 16 == 0 && a[1] % 16 == 0 && a[3] >= 1))
        return fail(h, GPB200_EINVAL, "gram_kernels: the TMA kernels take a single SEIso leaf over d <= 8 dimensions whose "
                                      "constants seiso_fast_prepare accepts, N >= 1 and 16-byte aligned xp and xpt");
    bool ok = true;
    switch (which) {
    case 0:     // x, ldx, d, N, Npad, noise_var, n_noise, G, ldg, own_tiles, nranks, rank, own_axis, bm_min
        ok = need({0, 5, 7}) && a[1] >= d && padded(3, 4) && (a[6] == 1 || a[6] == a[3]) && vec2(7, 8) && a[8] >= a[4] &&
             a[9] >= 0 && a[10] >= 1 && a[11] >= 0 && a[11] < a[10] && (a[12] == 0 || a[12] == 1) && a[13] >= 0;
        break;
    case 1:     // xs, ldxs, M, Mpad, x, ldx, N, Npad, d, Kst, ldk
        ok = need({0, 4, 9}) && a[1] >= d && a[5] >= d && padded(2, 3) && padded(6, 7) && vec2(9, 10) && a[10] >= a[7];
        break;
    case 2:     // xs, ldxs, M, Mpad, d, Kss, ldk
        ok = need({0, 5}) && a[1] >= d && padded(2, 3) && vec2(5, 6) && a[6] >= a[3];
        break;
    case 3:     // xs, ldxs, d, M, out
        ok = need({0, 4}) && a[1] >= d && a[3] >= 0;
        break;
    case 4:     // x, ldx, d, N, Npad, j, D, ldd, row0, rows
        ok = need({0, 6}) && a[1] >= d && padded(3, 4) && jok(5) && a[7] >= a[4] && a[8] >= 0 && a[8] % TILE == 0 &&
             a[9] >= 0 && a[9] % TILE == 0 && a[8] + a[9] <= a[4];
        break;
    case 5:     // x1, ldx1, N1, N1pad, x2, ldx2, N2, N2pad, d, j, D, ldd
        ok = need({0, 4, 10}) && a[1] >= d && a[5] >= d && padded(2, 3) && padded(6, 7) && jok(9) && a[11] >= a[7];
        break;
    case 6:     // x, ldx, d, N, Npad, alpha, Kinv, ldg, part, out, bm_mod, bm_rem, bm_div
        ok = need({0, 5, 6, 8, 9}) && a[1] >= d && padded(3, 4) && vec2(6, 7) && a[7] >= a[4] && a[10] >= 1 &&
             a[11] >= 0 && a[11] < a[10] && a[12] >= 1;
        break;
    case 7:     // x1, ldx1, N1, x2, ldx2, N2, d, W, ldw, part, out
        ok = need({0, 3, 7, 9, 10}) && a[1] >= d && a[4] >= d && a[2] >= 0 && a[5] >= 0 && vec2(7, 8) && a[8] >= a[5];
        break;
    case 8:     // x, ldx, d, N, g, out
        ok = need({0, 4, 5}) && a[1] >= d && a[3] >= 0;
        break;
    case 9:     // xs, ldxs, M, z, ldz, n, d, a, W1, W2, ldw, dmu, dvar
        ok = need({0, 3, 7, 11}) && a[1] >= d && a[4] >= d && a[2] >= 0 && a[5] >= 0 && ((!a[8] && !a[9]) || (a[12] && a[10] >= a[5]));
        break;
    case 10:    // F, ld, Npad
        ok = need({0}) && a[2] >= 0 && a[2] % TILE == 0 && a[1] >= a[2];
        break;
    case 11:    // x, ldx, d, N, alpha, G, ldg, out, bm_mod, bm_rem, bm_div, fast
        ok = need({0, 5, 7}) && a[1] >= d && a[3] >= 0 && a[6] >= a[3] && a[8] >= 1 && a[9] >= 0 && a[9] < a[8] && a[10] >= 1 &&
             (a[11] == 0 || (a[11] == 1 && kprog_fast(P, (int)d) && d <= 8));
        break;
    case 12:    // xp, xpt, d, N, Npad, noise_var, n_noise, G, ldg, own_tiles, nranks, rank, own_axis, sf
        ok = need({5, 7}) && padded(3, 4) && (a[6] == 1 || a[6] == a[3]) && vec2(7, 8) && a[8] >= a[4] && a[9] >= 0 &&
             a[10] >= 1 && a[11] >= 0 && a[11] < a[10] && (a[12] == 0 || a[12] == 1);
        break;
    case 13:    // xp, xpt, d, N, Npad, alpha, Kinv, ldg, part, out, bm_mod, bm_rem, bm_div, sf
        ok = need({5, 6, 8, 9}) && padded(3, 4) && vec2(6, 7) && a[7] >= a[4] && a[10] >= 1 && a[11] >= 0 && a[11] < a[10] &&
             a[12] >= 1;
        break;
    }
    if (!ok) return fail(h, GPB200_EINVAL, "gram_kernels: a null pointer, a negative size, a bad padding, leading dimension or "
                                           "alignment, j outside [0, n_theta) or a bad ownership argument");
    CK(cudaSetDevice(h->device));
    cudaStream_t st = h->st;
    int64_t* L = &h->launches;
    const int id = (int)d;
    const int dx = (id + 1) / 2 * 2;
    CUtensorMap mx, mxt;
    if (tma) {
        if (!seiso_make_x_maps(&mx, &mxt, ptr(0), ptr(1), dx, a[3], a[4]))
            return fail(h, GPB200_ECUDA, "gram_kernels: TMA descriptors of xp / xpt could not be built");
        if (a[13]) {                                     // the prepared constants: c_hi, il2, s2, tab[64]
            double* o = reinterpret_cast<double*>(a[13]);
            o[0] = sf.c_hi; o[1] = sf.il2; o[2] = sf.s2;
            for (int j = 0; j < 64; ++j) o[3 + j] = sf.tab[j];
        }
    }
    cudaError_t e = cudaSuccess;
    switch (which) {
    case 0: e = gram_lower_launch(P, ptr(0), a[1], id, a[3], a[4], ptr(5), a[6], fargs[nf - 1], ptr(7), a[8], st, L, (int)a[9],
                                  (int)a[10], (int)a[11], (int)a[12], (int)a[13]); break;
    case 1: e = crossgram_launch(P, ptr(0), a[1], a[2], a[3], ptr(4), a[5], a[6], a[7], id, ptr(9), a[10], st, L); break;
    case 2: e = gram_full_launch(P, ptr(0), a[1], a[2], a[3], id, ptr(5), a[6], st, L); break;
    case 3: e = kdiag_launch(P, ptr(0), a[1], a[3], ptr(4), st, L); break;
    case 4: e = gram_grad_full_launch(P, ptr(0), a[1], id, a[3], a[4], (int)a[5], ptr(6), a[7], st, L, a[8], a[9]); break;
    case 5: e = crossgram_grad_launch(P, ptr(0), a[1], a[2], a[3], ptr(4), a[5], a[6], a[7], id, (int)a[9], ptr(10), a[11], st, L); break;
    case 6: e = trace_launch(P, ptr(0), a[1], id, a[3], a[4], ptr(5), ptr(6), a[7], ptr(8), ptr(9), st, L, (int)a[10], (int)a[11],
                             (int)a[12]); break;
    case 7: e = trace_rect_launch(P, ptr(0), a[1], a[2], ptr(3), a[4], a[5], id, ptr(7), a[8], ptr(9), ptr(10), st, L); break;
    case 8: e = kdiag_grad_launch(P, ptr(0), a[1], a[3], ptr(4), ptr(5), st, L); break;
    case 9: e = crossgram_dx_launch(P, ptr(0), a[1], a[2], ptr(3), a[4], a[5], id, ptr(7), ptr(8), ptr(9), a[10], fargs[nf - 1],
                                    ptr(11), ptr(12), st, L); break;
    case 10: e = mirror_lower_tiles_launch(ptr(0), a[1], a[2], st, L); break;
    case 11: e = inputs_dx_launch(P, a[11] != 0, ptr(0), a[1], id, a[3], ptr(4), ptr(5), a[6], ptr(7), st, L, (int)a[8], (int)a[9],
                                  (int)a[10]); break;
    case 12: e = gram_seiso_tma_launch(&mx, &mxt, dx, sf, a[3], a[4], ptr(5), a[6], fargs[nf - 1], ptr(7), a[8], st, L, (int)a[9],
                                       (int)a[10], (int)a[11], (int)a[12]); break;
    case 13: e = trace_seiso_tma_launch(&mx, &mxt, dx, sf, a[3], a[4], ptr(5), ptr(6), a[7], ptr(8), ptr(9), st, L, (int)a[10],
                                        (int)a[11], (int)a[12]); break;
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    CK(e);
    return GPB200_OK;
}

int gpb200_vec_kernels(gpb200_handle* h, int which, const int64_t* args, int32_t n, const double* fargs, int32_t nf) {
    if (!h || !args || which < 0 || which > 3 || nf < 0 || (nf > 0 && !fargs)) return GPB200_EINVAL;
    static const int want[4] = {6, 6, 5, 5};
    static const int wantf[4] = {1, 1, 0, 0};
    if (n != want[which] || nf != wantf[which])
        return fail(h, GPB200_EINVAL, "vec_kernels: wrong argument count for this kernel (fargs = s for ew, nugget for spd_from_cov)");
    const int64_t* a = args;
    auto ptr = [&](int i) { return reinterpret_cast<double*>(a[i]); };
    auto need = [&](std::initializer_list<int> idx) {
        for (int i : idx) if (!a[i]) return false;
        return true;
    };
    bool ok = true;
    switch (which) {
    case 0: {   // op, n, out, a, b, c: b for ops 1, 3, 6; c for op 3
        const int64_t op = a[0];
        ok = op >= 0 && op <= 6 && a[1] >= 0 && need({2, 3}) && (!(op == 1 || op == 3 || op == 6) || a[4]) && (op != 3 || a[5]);
        break;
    }
    case 1: ok = need({0, 2}) && a[4] >= 0 && a[5] >= a[4] && a[5] >= TILE && a[5] % TILE == 0 && a[1] >= a[5] && a[3] >= a[4]; break;   // dst, ldd, src, lds, n, npad
    case 2: ok = need({0, 2}) && a[3] >= 0 && a[4] >= 0 && a[1] >= a[4]; break;                  // A, ld, v, nrows, ncols
    case 3: ok = need({0, 1, 3}) && a[4] >= 0 && a[2] >= 0; break;                               // out, src, ld, idx, nv
    }
    if (!ok) return fail(h, GPB200_EINVAL, "vec_kernels: a null pointer, a negative size, a bad op, a bad padding or ld below the row width");
    CK(cudaSetDevice(h->device));
    cudaStream_t st = h->st;
    int64_t* L = &h->launches;
    cudaError_t e = cudaSuccess;
    switch (which) {
    case 0: e = ew_launch((int)a[0], a[1], ptr(2), ptr(3), ptr(4), ptr(5), fargs[0], st, L); break;
    case 1: e = spd_from_cov_launch(ptr(0), a[1], ptr(2), a[3], a[4], a[5], fargs[0], st, L); break;
    case 2: e = add_rowvec_launch(ptr(0), a[1], ptr(2), a[3], a[4], st, L); break;
    case 3: e = gather_block_launch(ptr(0), ptr(1), a[2], reinterpret_cast<const long long*>(a[3]), a[4], st, L); break;
    }
    CK(e);
    CK(cudaStreamSynchronize(st));
    return GPB200_OK;
}

int gpb200_fitc_cv_kernels(gpb200_handle* h, int which, const int64_t* args, int32_t n, const double* fargs, int32_t nf) {
    if (!h || !args || which < 0 || which > 15 || nf < 0 || (nf > 0 && !fargs)) return GPB200_EINVAL;
    static const int want[16] = {14, 14, 4, 8, 5, 5, 10, 6, 5, 6, 5, 9, 7, 3, 13, 14};
    if (n != want[which]) return fail(h, GPB200_EINVAL, "fitc_cv_kernels: wrong argument count for this kernel");
    const int64_t* a = args;
    auto ptr = [&](int i) { return reinterpret_cast<double*>(a[i]); };
    auto need = [&](std::initializer_list<int> idx) {
        for (int i : idx) if (!a[i]) return false;
        return true;
    };
    KProg P{};
    if (which == 0) {
        // kind, x, ldx, d, j, G, C, ld, ncols, nrows, rows_pad, alpha, delta, da
        TRY(local_prog(h, "fitc_cv_kernels", fargs, nf, a[3], P));
    } else if (which == 14) {
        // u, ldu, M, z, ldz, n, d, W, ldw, sym, mask, out, accumulate
        if (a[6] > GPB200_MAX_DIMS) return fail(h, GPB200_EINVAL, "fitc_cv_kernels: d exceeds GPB200_MAX_DIMS");
        TRY(local_prog(h, "fitc_cv_kernels", fargs, nf, a[6], P));
    } else if (which == 15) {
        // x, ldx, n, u, ldu, M, d, W, ldw, c, mask, map, out, accumulate
        if (a[6] > GPB200_MAX_DIMS) return fail(h, GPB200_EINVAL, "fitc_cv_kernels: d exceeds GPB200_MAX_DIMS");
        TRY(local_prog(h, "fitc_cv_kernels", fargs, nf, a[6], P));
    } else if (nf != 0) {
        return fail(h, GPB200_EINVAL, "fitc_cv_kernels: fargs = theta for delta, inducing_dx and rows_dx, none otherwise");
    }
    bool ok = true;
    switch (which) {
    case 0: ok = a[0] >= 0 && a[0] <= 2 && a[9] >= 0 && a[10] >= 0 && need({11, 12, 13}) &&
                 (a[0] != 0 || (need({1, 5, 6}) && a[2] >= a[3] && a[4] >= 0 && a[4] < P.n_theta && a[8] >= 0 && a[7] >= a[8]));
            break;
    // G, Ch, K, P, ld, nrows, ncols, lam, delta, alpha, beta, w, zja, dg   (G = 0: beta unread)
    case 1: ok = need({1, 2, 3, 7, 8, 9, 11, 12, 13}) && (!a[0] || a[10]) && a[5] >= 0 && a[6] >= 0 && a[4] >= a[6]; break;
    case 2: ok = need({1, 2, 3}) && a[0] >= 0; break;                                  // n, lam, q, out
    case 3: ok = need({0, 2, 6, 7}) && a[4] >= 0 && a[5] >= 0 && a[3] >= a[5]; break;   // E, G, K, ld, nrows, ncols, lam, delta
    case 4: ok = need({0, 1, 2}) && a[4] >= 0 && a[3] >= a[4]; break;                  // Q, H, R, ld, n
    case 5: ok = need({1, 2, 3, 4}) && a[0] >= 0; break;                               // n, w, a, b, c
    // nv, idx, x, ldx, d, xout, lam, lamout, delta, delout   (delta = 0: delout unwritten)
    case 6: ok = need({1, 2, 5, 6, 7}) && (!a[8] || a[9]) && a[0] >= 0 && a[4] >= 0 && a[4] <= INT_MAX && a[3] >= a[4]; break;
    case 7: ok = need({0, 4}) && (a[3] == 0 || (a[3] == 1 && a[5])) && a[2] >= 0 && a[1] >= a[2]; break;   // out, ld, nv, which, lam, delta
    case 8: ok = need({0, 4}) && a[2] >= 0 && a[3] >= 0 && a[1] >= a[3]; break;       // colscale: A, ld, nrows, ncols, v
    case 9: ok = need({1, 5}) && (a[0] == 0 || a[0] == 1) && a[3] >= 0 && a[4] >= 0 && a[2] >= a[4]; break;   // scale: mode, A, ld, nrows, ncols, v
    case 10: ok = need({1, 2, 3, 4}) && a[0] >= 0; break;                             // fitc_g: n, alpha, lam, q, g
    case 11: ok = need({0, 1, 5, 6, 7, 8}) && a[3] >= 0 && a[4] >= 0 && a[2] >= a[4]; break;   // fitc_wfu: P2, P1, ld, nrows, ncols, alpha, lam, g, beta
    case 12: ok = need({0, 1, 2, 3, 6}) && a[5] >= 0 && a[4] >= a[5]; break;          // fitc_wuu: Wuu, T, Kinv, Sinv, ld, n, beta
    case 13: ok = need({0}) && a[2] >= 0 && a[1] >= a[2]; break;                       // symmetrize: A, ld, n
    case 14: ok = need({0, 3, 7, 11}) && a[2] >= 0 && a[5] >= 0 && a[1] >= a[6] && a[4] >= a[6] && a[8] >= a[2] &&
                  (a[9] == 0 || (a[9] == 1 && a[5] == a[2])) && (a[12] == 0 || a[12] == 1); break;
    case 15: ok = need({0, 3, 7, 12}) && a[2] >= 0 && a[5] >= 0 && a[1] >= a[6] && a[4] >= a[6] && a[8] >= a[5] &&
                  (a[13] == 0 || a[13] == 1); break;
    }
    if (!ok) return fail(h, GPB200_EINVAL, "fitc_cv_kernels: a null pointer, a negative size, a bad mode or ld below the row width");
    CK(cudaSetDevice(h->device));
    cudaStream_t st = h->st;
    int64_t* L = &h->launches;
    cudaError_t e = cudaSuccess;
    switch (which) {
    case 0: e = fitc_cv_delta_launch((int)a[0], P, ptr(1), a[2], (int)a[4], ptr(5), ptr(6), a[7], a[8], a[9], a[10], ptr(11), ptr(12),
                                     ptr(13), st, L); break;
    case 1: e = fitc_cv_rows_launch(ptr(0), ptr(1), ptr(2), ptr(3), a[4], a[5], a[6], ptr(7), ptr(8), ptr(9), ptr(10), ptr(11), ptr(12),
                                    ptr(13), st, L); break;
    case 2: e = fitc_cv_invdiag_launch(a[0], ptr(1), ptr(2), ptr(3), st, L); break;
    case 3: e = fitc_cv_eblock_launch(ptr(0), ptr(1), ptr(2), a[3], a[4], a[5], ptr(6), ptr(7), st, L); break;
    case 4: e = fitc_cv_qs_launch(ptr(0), ptr(1), ptr(2), a[3], a[4], st, L); break;
    case 5: e = fitc_cv_wvec_launch(a[0], ptr(1), ptr(2), ptr(3), ptr(4), st, L); break;
    case 6: e = fitc_cv_gather_launch(a[0], reinterpret_cast<const long long*>(a[1]), ptr(2), a[3], (int)a[4], ptr(5), ptr(6), ptr(7),
                                      ptr(8), ptr(9), st, L); break;
    case 7: e = fitc_cv_diag_launch(ptr(0), a[1], a[2], (int)a[3], ptr(4), ptr(5), st, L); break;
    case 8: e = colscale_launch(ptr(0), a[1], a[2], a[3], ptr(4), st, L); break;
    case 9: e = scale_launch((int)a[0], ptr(1), a[2], a[3], a[4], ptr(5), st, L); break;
    case 10: e = fitc_g_launch(a[0], ptr(1), ptr(2), ptr(3), ptr(4), st, L); break;
    case 11: e = fitc_wfu_launch(ptr(0), ptr(1), a[2], a[3], a[4], ptr(5), ptr(6), ptr(7), ptr(8), st, L); break;
    case 12: e = fitc_wuu_launch(ptr(0), ptr(1), ptr(2), ptr(3), a[4], a[5], ptr(6), st, L); break;
    case 13: e = symmetrize_launch(ptr(0), a[1], a[2], st, L); break;
    case 14: e = inducing_dx_launch(P, ptr(0), a[1], a[2], ptr(3), a[4], a[5], (int)a[6], ptr(7), a[8], (int)a[9], ptr(10), ptr(11),
                                    (int)a[12], st, L); break;
    case 15: e = rows_dx_launch(P, ptr(0), a[1], a[2], ptr(3), a[4], a[5], (int)a[6], ptr(7), a[8], ptr(9), ptr(10),
                                reinterpret_cast<const long long*>(a[11]), ptr(12), (int)a[13], st, L); break;
    }
    CK(e);
    CK(cudaStreamSynchronize(st));
    return GPB200_OK;
}

int gpb200_shard_kernels(gpb200_handle* h, int which, const int64_t* args, int32_t n) {
    if (!h || !args || which < 0 || which > 14) return GPB200_EINVAL;
    static const int want[15] = {5, 12, 10, 6, 7, 5, 3, 9, 10, 7, 8, 7, 8, 3, 3};
    if (n != want[which]) return fail(h, GPB200_EINVAL, "shard_kernels: wrong argument count for this kernel");
    const int64_t* a = args;
    auto ptr = [&](int i) { return reinterpret_cast<double*>(a[i]); };
    auto need = [&](std::initializer_list<int> idx) {
        for (int i : idx) if (!a[i]) return false;
        return true;
    };
    auto in_int = [&](std::initializer_list<int> idx) {           // sizes the wrappers take as int: in [0, INT_MAX]
        for (int i : idx) if (a[i] < 0 || a[i] > INT_MAX) return false;
        return true;
    };
    const int64_t YMAX = 65535;                                    // grid.y / grid.z limit
    // the ownership {R, me, rb} at a[i], a[i + 1], a[i + 2]
    auto own_ok = [&](int i) { return a[i] >= 1 && a[i] <= INT_MAX && a[i + 1] >= 0 && a[i + 1] < a[i] && a[i + 2] >= 1 && a[i + 2] <= INT_MAX; };
    auto own_at = [&](int i) { return ShardOwn{(int)a[i], (int)a[i + 1], (int)a[i + 2]}; };
    // rows r >= 128 t1 of Npad: Npad a multiple of 128, t1 in [0, Npad / 128], at most 65 535 tiles past t1
    auto panel_ok = [&](int npad, int t1) {
        return a[npad] >= 0 && a[npad] % TILE == 0 && a[npad] / TILE <= INT_MAX && a[t1] >= 0 && a[t1] <= a[npad] / TILE &&
               a[npad] / TILE - a[t1] <= YMAX;
    };
    // a level s that inverse_dist splits over R ranks: s a positive multiple of 128 R below Np, grid.y and grid.z in range
    auto level_ok = [&](int s, int np, int r, int me, int ld) {
        if (a[r] < 1 || a[r] > INT_MAX || a[me] < 0 || a[me] >= a[r] || a[np] <= 0 || a[np] % TILE || a[np] > INT_MAX) return false;
        if (a[s] <= 0 || a[s] % (TILE * a[r]) || a[s] >= a[np] || (a[s] + 31) / 32 > YMAX || a[ld] < a[np]) return false;
        return (a[np] + 2 * a[s] - 1) / (2 * a[s]) * (which == 12 ? a[r] : 1) <= YMAX;
    };
    bool ok = true;
    switch (which) {
    case 0: ok = need({0, 2}) && in_int({4}) && a[4] <= YMAX && a[1] >= a[4] && a[3] >= a[4]; break;      // dst, ldd, src, lds, n
    case 1:     // G, F, ld, Npad, c0, nb, t1, S_me, nbp, R, me, rb
        ok = need({0, 1, 7}) && in_int({4, 5, 8}) && panel_ok(3, 6) && a[5] <= a[8] && a[2] >= a[4] + a[5] && own_ok(9);
        break;
    case 2:     // P, nbp, Npad, nb, t1, S, per_rank, R, me, rb; every rank's region holds its rows >= 128 t1
        ok = need({0, 5}) && in_int({1, 3}) && panel_ok(2, 4) && a[3] <= a[1] && own_ok(7) && a[6] >= 0;
        if (ok) {
            const ShardOwn o = own_at(7);
            for (int q = 0; q < o.R && ok; ++q)
                ok = a[6] >= (shard_own_before(a[2] / TILE, q, o.rb, o.R) - shard_own_before(a[4], q, o.rb, o.R)) * TILE * a[1];
        }
        break;
    case 3:     // dst, ldd, src, lds, rows, cols
    case 7:     // dst, ldd, src, lds, rows, cols, R, me, rb
        ok = need({0, 2}) && a[4] >= 0 && a[5] >= 0 && a[4] <= 32 * YMAX && a[1] >= a[4] && a[3] >= a[5] && (which == 3 || own_ok(6));
        break;
    case 4:     // P, nbp, G, ld, Dinv, j0, nb: j0, nb multiples of 128 (the panels of shard_inverse_la)
        ok = need({0, 2, 4}) && in_int({1, 5, 6}) && a[5] % TILE == 0 && a[6] % TILE == 0 && a[6] <= a[1] && a[6] <= YMAX &&
             a[3] >= a[5] + a[6];
        break;
    case 5: ok = need({0, 1}) && a[3] >= 1 && a[3] <= INT_MAX && a[4] >= 0 && a[2] >= a[4]; break;     // out, in, stride, nranks, n
    case 6: ok = need({0, 1}) && a[2] >= 1 && a[2] <= INT_MAX; break;                                  // out, in, nranks
    case 8:     // Y, G, ld, ncols, alpha, N, out, R, me, rb
        ok = need({0, 1, 4, 6}) && a[3] >= 0 && a[5] >= 0 && a[2] >= a[3] && own_ok(7);
        break;
    case 9:     // G, ld, N, out, R, me, rb: the diagonal of every row of the tiles covering 0 .. N
        ok = need({0, 3}) && a[2] >= 0 && a[1] >= (a[2] + TILE - 1) / TILE * TILE && own_ok(4);
        break;
    case 10: ok = need({0, 1, 3}) && a[2] >= 1 && a[4] >= 0 && a[4] <= YMAX && own_ok(5); break;       // out, src, ld, idx, nv, R, me, rb
    case 11: ok = need({0, 2}) && level_ok(3, 4, 5, 6, 1); break;                                      // G, ld, out, s, Np, R, me
    case 12:    // G, ld, in, per_rank, s, Np, R, me: per_rank = sum_z n2_z * wr, as inverse_dist computes it
        ok = need({0, 2}) && level_ok(4, 5, 6, 7, 1);
        if (ok) {
            int64_t rows = 0;
            for (int64_t p = 0; p < a[5]; p += 2 * a[4]) rows += std::max<int64_t>(0, std::min(a[4], a[5] - p - a[4]));
            ok = a[3] >= rows * (a[4] / a[6]);
        }
        break;
    case 13: ok = need({0}) && a[1] >= 0 && a[1] <= 7 && a[2] >= INT_MIN && a[2] <= INT_MAX; break;   // words, n_peer, value
    case 14: ok = need({0, 2}) && a[1] >= INT_MIN && a[1] <= INT_MAX; break;                           // word, target, err
    }
    if (!ok) return fail(h, GPB200_EINVAL, "shard_kernels: a null pointer, a negative size, a bad ownership, padding or level, a leading "
                                           "dimension below the row width, a region too small or a grid dimension past 65 535");
    CK(cudaSetDevice(h->device));
    cudaStream_t st = h->st;
    int64_t* L = &h->launches;
    cudaError_t e = cudaSuccess;
    switch (which) {
    case 0: e = shard_copy_lower(ptr(0), a[1], ptr(2), a[3], (int)a[4], st, L); break;
    case 1: e = shard_scatter_rows(ptr(0), ptr(1), a[2], a[3], (int)a[4], (int)a[5], (int)a[6], ptr(7), (int)a[8], own_at(9), st, L); break;
    case 2: e = shard_unpack_panel(ptr(0), (int)a[1], a[2], (int)a[3], (int)a[4], ptr(5), a[6], own_at(7), st, L); break;
    case 3: e = shard_transpose(ptr(0), a[1], ptr(2), a[3], a[4], a[5], st, L); break;
    case 4: e = shard_pack_wblock(ptr(0), (int)a[1], ptr(2), a[3], ptr(4), (int)a[5], (int)a[6], st, L); break;
    case 5: e = shard_sum_ranks(ptr(0), ptr(1), a[2], (int)a[3], a[4], st, L); break;
    case 6: e = shard_min_ranks(reinterpret_cast<int*>(a[0]), reinterpret_cast<const int*>(a[1]), (int)a[2], st, L); break;
    case 7: e = shard_transpose_own(ptr(0), a[1], ptr(2), a[3], a[4], a[5], own_at(6), st, L); break;
    case 8: e = shard_rowdot_own(ptr(0), ptr(1), a[2], a[3], ptr(4), a[5], own_at(7), ptr(6), st, L); break;
    case 9: e = shard_diag_own(ptr(0), a[1], a[2], own_at(4), ptr(3), st, L); break;
    case 10: e = shard_gather_block_own(ptr(0), ptr(1), a[2], reinterpret_cast<const long long*>(a[3]), a[4], own_at(5), st, L); break;
    case 11: e = shard_pack_slices(ptr(0), a[1], ptr(2), (int)a[3], (int)a[5], (int)a[6], (int)a[4], st, L); break;
    case 12: e = shard_unpack_slices(ptr(0), a[1], ptr(2), a[3], (int)a[4], (int)a[6], (int)a[7], (int)a[5], st, L); break;
    case 13: e = shard_signal_peers(reinterpret_cast<int* const*>(a[0]), (int)a[1], (int)a[2], st, L); break;
    case 14: e = shard_wait_signal(reinterpret_cast<const int*>(a[0]), (int)a[1], reinterpret_cast<int*>(a[2]), st, L); break;
    }
    CK(e);
    CK(cudaStreamSynchronize(st));
    return GPB200_OK;
}
}  // extern "C"
