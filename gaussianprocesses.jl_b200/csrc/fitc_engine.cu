// fitc_engine.cu -- the sparse handle gpb200_fitc behind include/gpb200.h: FITC, DTC and SoR (modes 0-2), their
// cross-validation, posterior draws and append.  The FSA schedule of the same handle (mode 3) is fsa_engine.cu.
#include "engine.cuh"
#include "fitc_cv.cuh"
#include "gram.cuh"
#include "vec.cuh"

using namespace engine;

extern "C" {
// ================================================================================================
// FITC -- Fully Independent Training Conditional (src/sparse/fully_indep_train_conditional.jl)
//   update_cK! (:134-156), `\` (:33-36), logdet (:77), dmll_noise (:243-257), predictMVN (:324-332 ->
//   determ_train_conditional.jl:41-59 -> subsetofregressors.jl:302-321).
// The reference materialises K_uf (M x N) and several copies; here N is streamed in chunks through two
// staging buffers and only M x M state persists (H7 of SURVEY.md §7.2): per chunk a cross-Gram, a
// recursive TRSM against L_uu for diag(Q_ff), and one rank-Nc SYRK into Sigma_QR -- all on the DMMA GEMM.
// ================================================================================================
// in-place sum over the ranks of a device vector (no-op on one rank)
static int fitc_allreduce(gpb200_fitc* f, double* v, size_t n) {
    if (f->nranks <= 1 || n == 0) return GPB200_OK;
    FCKN(g_nccl.AllReduce(v, v, n, ncclDouble, ncclSum, f->comm, f->eu->st));
    return GPB200_OK;
}

// every buffer that depends on the observations or the inducing points; the FSA blocks refer to the old observations too
static void fitc_free_data(gpb200_fitc* f) {
    f->data = {}; f->stage = {}; f->grad = {}; f->app = {};
    f->pdx.reset(); f->dxu.reset(); f->dx.reset();
    fsa_free(f);
    f->cv = {};
}

int gpb200_fitc_comm_init(gpb200_fitc* f, int nranks, int rank, const char* id128) {
    if (!f || !id128 || nranks < 1 || rank < 0 || rank >= nranks) return GPB200_EINVAL;
    if (!nccl_load()) return fail(f, GPB200_ENCCL, "libnccl.so.2 could not be loaded");
    FCK(cudaSetDevice(f->device));
    if (f->comm) { g_nccl.CommDestroy(f->comm); f->comm = nullptr; }
    ncclUniqueId id;
    memcpy(&id, id128, 128);
    FCKN(g_nccl.CommInitRank(&f->comm, nranks, id, rank));
    f->nranks = nranks; f->rank = rank;
    fitc_invalidate(f);
    return GPB200_OK;
}

void gpb200_fitc_destroy(gpb200_fitc* f) {
    if (!f) return;
    cudaSetDevice(f->device);
    if (f->eu && f->eu->st) cudaStreamSynchronize(f->eu->st);
    fitc_free_data(f);
    f->Kss.reset();
    for (cudaEvent_t e : f->xu_ev) cudaEventDestroy(e);
    for (cudaEvent_t e : f->x_ev) cudaEventDestroy(e);
    if (f->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(f->comm);
    if (f->es) { f->es->st = nullptr; f->es->own_stream = false; gpb200_destroy(f->es); }
    if (f->eu) gpb200_destroy(f->eu);
    delete f;
}

int gpb200_fitc_create(gpb200_fitc** out, int device) {
    if (!out) return GPB200_EINVAL;
    *out = nullptr;
    gpb200_fitc* f = new gpb200_fitc();
    f->device = device;
    int rc = gpb200_create(&f->eu, device);
    if (rc == GPB200_OK) rc = gpb200_create(&f->es, device);
    if (rc != GPB200_OK) { if (f->eu) gpb200_destroy(f->eu); delete f; return rc; }
    // one stream for both sub-engines
    cudaStreamDestroy(f->es->st);
    f->es->st = f->eu->st; f->es->own_stream = false;
    *out = f;
    return GPB200_OK;
}

const char* gpb200_fitc_last_error(gpb200_fitc* f) { return f ? f->err.c_str() : g_create_error.c_str(); }

int gpb200_fitc_set_data(gpb200_fitc* f, int64_t N, int32_t d, const double* x, int64_t ldx, int64_t M,
                         const double* xu, int64_t ldxu) {
    if (!f) return GPB200_EINVAL;
    if (N <= 0 || M <= 0 || d <= 0 || !x || !xu || ldx < d || ldxu < d) return fail(f, GPB200_EINVAL, "fitc_set_data: bad arguments");
    FCK(cudaSetDevice(f->device));
    FSUB(gpb200_set_data(f->eu, M, d, xu, ldxu), f->eu);
    FSUB(gpb200_set_data(f->es, M, d, xu, ldxu), f->es);
    cudaStream_t st = f->eu->st;
    fitc_free_data(f);
    f->has_data = false;
    f->N = N; f->M = M; f->d = d; f->Mpad = f->eu->Npad;
    // chunk of data rows: two staging buffers of ~2 GB each at most
    int64_t nc = (int64_t)(2.0e9 / (8.0 * (double)f->Mpad)) / TILE * TILE;
    const int64_t Nceil = (N + TILE - 1) / TILE * TILE;
    if (nc > 32768) nc = 32768;                       // grid.y limit of the row-scaling kernel
    if (nc > Nceil) nc = Nceil;
    if (nc < TILE) nc = TILE;
    TRY(make_group(f->data, [&] {
        FitcData& g = f->data;
        FCK(g.x.alloc((size_t)N * d));
        for (DevBuf<double>* p : {&g.lam, &g.y, &g.alpha, &g.tmpn}) FCK(p->alloc(N + TILE));
        for (DevBuf<double>* p : {&g.bvec, &g.uvec, &g.tmpm, &g.rhsm}) FCK(p->alloc(f->Mpad));
        FCK(g.scal.alloc(16));
        return GPB200_OK;
    }));
    TRY(fitc_stage_alloc(f, nc, "fitc_set_data"));
    FCK(cudaMemcpy2DAsync(f->data.x, sizeof(double) * d, x, sizeof(double) * ldx, sizeof(double) * d, N, cudaMemcpyHostToDevice, st));
    FCK(cudaStreamSynchronize(st));
    f->Ncap = N;
    f->has_data = true; fitc_invalidate(f);
    return GPB200_OK;
}

int gpb200_fitc_set_kernel(gpb200_fitc* f, int32_t n_ops, const int32_t* ops, int32_t n_dims, const int32_t* dims,
                           int32_t n_theta) {
    if (!f) return GPB200_EINVAL;
    FSUB(gpb200_set_kernel(f->eu, n_ops, ops, n_dims, dims, n_theta), f->eu);
    FSUB(gpb200_set_kernel(f->es, n_ops, ops, n_dims, dims, n_theta), f->es);
    f->has_kernel = true; fitc_invalidate(f);
    return GPB200_OK;
}
}  // extern "C"

namespace engine __attribute__((visibility("hidden"))) {
// (re)makes the staging chunk for nc rows, with its tensor maps; the workspaces sized by Nc are freed with the old chunk
int fitc_stage_alloc(gpb200_fitc* f, int64_t nc, const char* who) {
    f->grad = {}; f->cv = {}; f->pdx.reset();
    f->stage = {};
    f->Nc = nc;
    return make_group(f->stage, [&] {
        FitcStage& g = f->stage;
        FCK(g.xs.alloc((size_t)nc * f->d));
        for (DevBuf<double>* p : {&g.w, &g.tmpc, &g.zeroc, &g.tmpc2}) FCK(p->alloc(nc));
        FCK(g.bufA.alloc((size_t)nc * f->Mpad));
        FCK(g.bufB.alloc((size_t)nc * f->Mpad));
        FCK(cudaMemsetAsync(g.zeroc, 0, sizeof(double) * nc, f->eu->st));
        if (f->eu->tma_ok) {
            const bool ok = gemm_make_tensor_map(&g.mapA, g.bufA, nc, f->Mpad, f->Mpad) &&
                            gemm_make_tensor_map(&g.mapB, g.bufB, f->Mpad, nc, nc) &&
                            gemm_make_tensor_map(&g.mapB2, g.bufB, nc, f->Mpad, f->Mpad);
            if (!ok) return fail(f, GPB200_ECUDA, std::string(who) + ": cuTensorMapEncodeTiled failed");
        }
        return GPB200_OK;
    });
}

// K_fu chunk (rows r0..r0+nc of x against the inducing points) into bufA [Nc x Mpad]
cudaError_t fitc_kfu(gpb200_fitc* f, const double* xrows, int64_t nc) {
    return crossgram_launch(f->eu->prog, xrows, f->d, nc, f->Nc, f->eu->x, f->d, f->M, f->Mpad, f->d, f->stage.bufA, f->Mpad, f->eu->st, &f->eu->launches);
}
// K_uf chunk into bufB [Mpad x Nc]
cudaError_t fitc_kuf(gpb200_fitc* f, const double* xrows, int64_t nc) {
    return crossgram_launch(f->eu->prog, f->eu->x, f->d, f->M, f->Mpad, xrows, f->d, nc, f->Nc, f->d, f->stage.bufB, f->Nc, f->eu->st, &f->eu->launches);
}

// Lambda of data rows r0 .. r0+nc into data.lam.  FITC: Lambda_i = sigma^2 + K_ii - |L_uu^-1 K_ui|^2 (fitc.jl:146-148), the
// whitening TRSM over trsm_rows rows of bufA; SoR / DTC: Lambda = sigma^2 I (subsetofregressors.jl:100: exp(-2 logNoise) *
// Kuf * Kfu + Kuu)
static int fitc_lambda(gpb200_fitc* f, int64_t r0, int64_t nc, int64_t trsm_rows) {
    gpb200_handle* eu = f->eu;
    cudaStream_t st = eu->st;
    const double* xr = f->data.x + r0 * f->d;
    if (f->mode == 0) {
        FCK(fitc_kfu(f, xr, nc));
        FCK(trsm_rec_buf(eu, gbuf(eu, f->stage.bufA, f->stage.mapA, f->Mpad), (int)trsm_rows, 0, (int)f->Mpad));
        FCK(kdiag_launch(eu->prog, xr, f->d, nc, f->stage.tmpc, st, &eu->launches));
        FCK(rowvar_launch(f->stage.bufA, f->Mpad, f->stage.tmpc, nc, f->Mpad, f->stage.tmpc2, st, &eu->launches));
        FCK(ew_launch(0, nc, f->data.lam + r0, f->stage.tmpc2, nullptr, nullptr, f->noise_var, st, &eu->launches));
    } else {
        FCK(ew_launch(0, nc, f->data.lam + r0, f->stage.zeroc, nullptr, nullptr, f->noise_var, st, &eu->launches));
    }
    return GPB200_OK;
}

// b += K_uf Lambda^-1 r over data rows r0 .. r0+nc (r in data.y), with their K_uf in bufB (fitc_kuf)
static int fitc_b_add(gpb200_fitc* f, int64_t r0, int64_t nc, double* b) {
    gpb200_handle* eu = f->eu;
    cudaStream_t st = eu->st;
    FCK(cudaMemsetAsync(f->stage.w, 0, sizeof(double) * f->Nc, st));
    FCK(ew_launch(1, nc, f->stage.w, f->data.y + r0, f->data.lam + r0, nullptr, 0.0, st, &eu->launches));
    FCK(rowdot_launch(f->stage.bufB, f->Nc, f->stage.w, f->M, f->Nc, f->data.tmpm, st, &eu->launches));
    FCK(ew_launch(2, f->M, b, f->data.tmpm, nullptr, nullptr, 0.0, st, &eu->launches));
    return GPB200_OK;
}

// S += K_uf Lambda^-1 K_fu (fitc.jl:150) over data rows r0 .. r0+nc, as (K_uf Lambda^-1/2)(K_uf Lambda^-1/2)': bufB (their
// K_uf) is scaled in place, then a lower-only SYRK over its first k columns into S (Mpad x Mpad, leading dimension lds)
static int fitc_syrk_add(gpb200_fitc* f, int64_t r0, int64_t nc, double* S, int64_t lds, int64_t k) {
    gpb200_handle *eu = f->eu, *es = f->es;
    const GemmBuf bB = gbuf(eu, f->stage.bufB, f->stage.mapB, f->Nc);
    FCK(scale_launch(0, f->stage.bufB, f->Nc, f->Mpad, nc, f->data.lam + r0, eu->st, &eu->launches));
    FCK(gemm_whole(es, bB, bB, S, lds, f->Mpad, f->Mpad, k, 1.0, 1.0, nullptr, 0, GEMM_LOWER_ONLY));
    return GPB200_OK;
}

// one contraction launch (slot k >= 1 of f->xu_ev) over n rows z against W (ld Mpad) into f->dxu
int xu_contract(gpb200_fitc* f, size_t k, const double* z, int64_t n, const double* W, int sym, const double* mask,
                int accumulate) {
    gpb200_handle* eu = f->eu;
    FCK(cudaEventRecord(f->xu_ev[2 * k], eu->st));
    FCK(inducing_dx_launch(eu->prog, eu->x, f->d, f->M, z, f->d, n, f->d, W, f->Mpad, sym, mask, f->dxu, accumulate, eu->st,
                           &eu->launches));
    FCK(cudaEventRecord(f->xu_ev[2 * k + 1], eu->st));
    return GPB200_OK;
}

// after the final synchronize: device times of the call and of its k_used contractions; dmll_xu = dxu / 2
int xu_finish(gpb200_fitc* f, size_t k_used, double* dmll_xu) {
    std::vector<double> h((size_t)f->M * f->d);
    FCK(cudaMemcpy(h.data(), f->dxu, sizeof(double) * h.size(), cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < h.size(); ++i) dmll_xu[i] = 0.5 * h[i];
    double c = 0.0;
    for (size_t k = 1; k <= k_used; ++k) c += ev_ms(f->xu_ev[2 * k], f->xu_ev[2 * k + 1]);
    f->xu_ms[0] = c;
    f->xu_ms[1] = ev_ms(f->xu_ev[0], f->xu_ev[1]);
    return GPB200_OK;
}

// one row-contraction launch (slot k >= 1 of f->x_ev) over n rows xr against the W_fu rows W (ld Mpad): rows_dx_launch
int x_rows(gpb200_fitc* f, size_t k, const double* xr, int64_t n, const double* W, const double* c, const double* mask,
           const long long* map, double* out, int accumulate) {
    gpb200_handle* eu = f->eu;
    FCK(cudaEventRecord(f->x_ev[2 * k], eu->st));
    FCK(rows_dx_launch(eu->prog, xr, f->d, n, eu->x, f->d, f->M, f->d, W, f->Mpad, c, mask, map, out, accumulate, eu->st,
                       &eu->launches));
    FCK(cudaEventRecord(f->x_ev[2 * k + 1], eu->st));
    return GPB200_OK;
}

// after the final synchronize: device times of the call and of its k_used contractions; dmll_x = dx / 2
int x_finish(gpb200_fitc* f, size_t k_used, double* dmll_x) {
    const size_t n = (size_t)f->N * f->d;
    FCK(cudaMemcpy(dmll_x, f->dx, sizeof(double) * n, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < n; ++i) dmll_x[i] *= 0.5;
    double c = 0.0;
    for (size_t k = 1; k <= k_used; ++k) c += ev_ms(f->x_ev[2 * k], f->x_ev[2 * k + 1]);
    f->x_ms[0] = c;
    f->x_ms[1] = ev_ms(f->x_ev[0], f->x_ev[1]);
    return GPB200_OK;
}
}  // namespace engine

extern "C" {
int gpb200_fitc_factorize(gpb200_fitc* f, const double* theta, double log_noise) {
    if (!f) return GPB200_EINVAL;
    if (!f->has_data || !f->has_kernel) return fail(f, GPB200_ESTATE, "fitc_factorize: set_data and set_kernel first");
    if (!isfinite(log_noise)) return fail(f, GPB200_EINVAL, "fitc_factorize: non-finite logNoise");
    if (f->mode == 3) TRY(fsa_check(f, "fitc_factorize"));
    FCK(cudaSetDevice(f->device));
    fitc_invalidate(f); f->cv.m_ok = false;
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    // K_uu + 1e-10 I and its factor (fitc.jl:139-141)
    const double ln_off = -1000.0;                          // exp(2*ln) == 0: no noise on K_uu
    FSUB(gpb200_factorize(eu, theta, &ln_off, 1, 1e-10), eu);
    // Sigma_QR starts as K_uu (+ the second 1e-10 nugget of make_posdef!, fitc.jl:153)
    kprog_set_theta(es->prog, theta);
    for (int i = 0; i < es->prog.n_theta; ++i) es->theta[i] = theta[i];
    const double zero = 0.0;
    FCK(cudaMemcpyAsync(es->noise_var, &zero, sizeof(double), cudaMemcpyHostToDevice, st));
    es->n_noise = 1; es->nugget = 2e-10;
    if (f->rank == 0) FCK(gram_lower_launch(es->prog, es->x, f->d, f->d, f->M, f->Mpad, es->noise_var, 1, 2e-10, es->G, es->ld, st, &es->launches));
    else FCK(cudaMemsetAsync(es->G, 0, sizeof(double) * (size_t)f->Mpad * (size_t)f->Mpad, st));     // K_uu (+ nuggets, identity padding) enters the sum once
    f->noise_var = exp(2.0 * log_noise);
    if (f->mode == 3) return fsa_factorize(f);
    for (int64_t r0 = 0; r0 < f->N; r0 += f->Nc) {
        const int64_t nc = std::min(f->Nc, f->N - r0);
        TRY(fitc_lambda(f, r0, nc, f->Nc));
        FCK(fitc_kuf(f, f->data.x + r0 * f->d, nc));
        TRY(fitc_syrk_add(f, r0, nc, es->G, es->ld, f->Nc));                 // Sigma_QR += K_uf Lambda^-1 K_fu
    }
    // multi-GPU: Sigma_QR = K_uu + sum over ranks of K_uf L^-1 K_fu  -- the one M x M exchange of the FITC likelihood
    TRY(fitc_allreduce(f, es->G, (size_t)f->Mpad * (size_t)f->Mpad));
    int rc = chol_inplace(es);
    if (rc != GPB200_OK) return fail(f, rc, "fitc_factorize (Sigma_QR): " + es->err);
    f->factored = true;
    return GPB200_OK;
}

// alpha = Sigma^-1 r (fitc.jl:33-36), logdet (fitc.jl:77), mll (GPE.jl:210)
int gpb200_fitc_mll(gpb200_fitc* f, const double* y_minus_mean, double* alpha, double* mll, double* logdet) {
    if (!f || !y_minus_mean || !mll) return GPB200_EINVAL;
    if (!f->factored) return fail(f, GPB200_ESTATE, "fitc_mll: factorize first");
    if (f->mode == 3) { FCK(cudaSetDevice(f->device)); return fsa_mll(f, y_minus_mean, alpha, mll, logdet); }
    FCK(cudaSetDevice(f->device));
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    FCK(cudaMemcpyAsync(f->data.y, y_minus_mean, sizeof(double) * f->N, cudaMemcpyHostToDevice, st));
    // b = K_uf Lambda^-1 r
    FCK(cudaMemsetAsync(f->data.bvec, 0, sizeof(double) * f->Mpad, st));
    for (int64_t r0 = 0; r0 < f->N; r0 += f->Nc) {
        const int64_t nc = std::min(f->Nc, f->N - r0);
        FCK(fitc_kuf(f, f->data.x + r0 * f->d, nc));
        TRY(fitc_b_add(f, r0, nc, f->data.bvec));
    }
    TRY(fitc_allreduce(f, f->data.bvec, (size_t)f->Mpad));              // b summed over the ranks' rows
    // u = Sigma_QR^-1 b   (== get_alpha_u, fitc.jl:279-286)
    FCK(cudaMemcpyAsync(f->data.rhsm, f->data.bvec, sizeof(double) * f->Mpad, cudaMemcpyDeviceToDevice, st));
    FCK(solve_device(es, f->data.rhsm, f->data.tmpm, f->data.uvec));
    // alpha = Lambda^-1 (r - K_fu u)
    for (int64_t r0 = 0; r0 < f->N; r0 += f->Nc) {
        const int64_t nc = std::min(f->Nc, f->N - r0);
        FCK(fitc_kfu(f, f->data.x + r0 * f->d, nc));
        FCK(rowdot_launch(f->stage.bufA, f->Mpad, f->data.uvec, nc, f->Mpad, f->stage.tmpc, st, &eu->launches));
        FCK(ew_launch(3, nc, f->data.alpha + r0, f->data.y + r0, f->stage.tmpc, f->data.lam + r0, 0.0, st, &eu->launches));
    }
    FCK(dot_launch(f->data.y, f->data.alpha, f->N, f->data.scal + 0, st, &eu->launches));
    FCK(sum_launch(es->logd, es->Npad, f->data.scal + 1, st, &eu->launches));
    FCK(sum_launch(eu->logd, eu->Npad, f->data.scal + 2, st, &eu->launches));
    FCK(ew_launch(4, f->N, f->data.tmpn, f->data.lam, nullptr, nullptr, 0.0, st, &eu->launches));
    FCK(sum_launch(f->data.tmpn, f->N, f->data.scal + 3, st, &eu->launches));
    double s[5];
    if (f->nranks > 1) {
        // r'alpha, sum log Lambda and N are sums over the ranks' rows; the two M x M log-determinants are replicated
        const double nloc = (double)f->N;
        FCK(cudaMemcpyAsync(f->data.scal + 8, f->data.scal + 0, sizeof(double), cudaMemcpyDeviceToDevice, st));
        FCK(cudaMemcpyAsync(f->data.scal + 9, f->data.scal + 3, sizeof(double), cudaMemcpyDeviceToDevice, st));
        FCK(cudaMemcpyAsync(f->data.scal + 10, &nloc, sizeof(double), cudaMemcpyHostToDevice, st));
        TRY(fitc_allreduce(f, f->data.scal + 8, 3));
        FCK(cudaMemcpyAsync(f->data.scal + 0, f->data.scal + 8, sizeof(double), cudaMemcpyDeviceToDevice, st));
        FCK(cudaMemcpyAsync(f->data.scal + 3, f->data.scal + 9, sizeof(double), cudaMemcpyDeviceToDevice, st));
        FCK(cudaMemcpyAsync(f->data.scal + 4, f->data.scal + 10, sizeof(double), cudaMemcpyDeviceToDevice, st));
    }
    FCK(cudaMemcpyAsync(s, f->data.scal, sizeof(double) * 5, cudaMemcpyDeviceToHost, st));
    if (alpha) FCK(cudaMemcpyAsync(alpha, f->data.alpha, sizeof(double) * f->N, cudaMemcpyDeviceToHost, st));
    FCK(cudaStreamSynchronize(st));
    FSUB(check_trsv_watchdog(es), es);                                   // the solve for u above
    f->Ntotal = f->nranks > 1 ? s[4] : (double)f->N;
    const double ld = s[1] - s[2] + s[3];
    if (logdet) *logdet = ld;
    *mll = -(s[0] + ld + LOG2PI * f->Ntotal) / 2.0;
    f->alpha_ready = true;
    f->app.sums_ok = false;                                              // the residuals may have changed
    return GPB200_OK;
}

// dmll_noise (fitc.jl:243-257): sigma^2 * (alpha.alpha - sum 1/Lambda + |L_s^-1 K_uf Lambda^-1|_F^2)
int gpb200_fitc_grad_noise(gpb200_fitc* f, double* dmll_noise) {
    if (!f || !dmll_noise) return GPB200_EINVAL;
    if (!f->factored || !f->alpha_ready) return fail(f, GPB200_ESTATE, "fitc_grad_noise: factorize and mll first");
    if (f->mode == 3) { FCK(cudaSetDevice(f->device)); return fsa_grad_noise(f, dmll_noise); }
    FCK(cudaSetDevice(f->device));
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const GemmBuf bA = gbuf(eu, f->stage.bufA, f->stage.mapA, f->Mpad);
    for (int64_t r0 = 0; r0 < f->N; r0 += f->Nc) {
        const int64_t nc = std::min(f->Nc, f->N - r0);
        FCK(fitc_kfu(f, f->data.x + r0 * f->d, nc));
        FCK(scale_launch(1, f->stage.bufA, f->Mpad, nc, f->Mpad, f->data.lam + r0, st, &eu->launches));
        FCK(trsm_rec_buf(es, bA, (int)f->Nc, 0, (int)f->Mpad));
        FCK(rowvar_launch(f->stage.bufA, f->Mpad, f->stage.zeroc, nc, f->Mpad, f->data.tmpn + r0, st, &eu->launches));     // = -|row|^2
    }
    FCK(sum_launch(f->data.tmpn, f->N, f->data.scal + 0, st, &eu->launches));
    FCK(dot_launch(f->data.alpha, f->data.alpha, f->N, f->data.scal + 1, st, &eu->launches));
    FCK(ew_launch(5, f->N, f->data.tmpn, f->data.lam, nullptr, nullptr, 0.0, st, &eu->launches));
    FCK(sum_launch(f->data.tmpn, f->N, f->data.scal + 2, st, &eu->launches));
    TRY(fitc_allreduce(f, f->data.scal, 3));                             // sums over the ranks' rows
    double s[3];
    FCK(cudaMemcpyAsync(s, f->data.scal, sizeof(double) * 3, cudaMemcpyDeviceToHost, st));
    FCK(cudaStreamSynchronize(st));
    *dmll_noise = f->noise_var * (s[1] - s[2] - s[0]);
    return GPB200_OK;
}

// predictive mean / variance of mc <= Nc test rows (xs, row stride ldxs; fitc.jl:324-332 -> dtc.jl:41-59 -> sor.jl:302-321):
//   mu = K_xu u ;  var = k_xx - |L_uu^-1 k_ux|^2 + |L_s^-1 k_ux|^2   (SoR: |L_s^-1 k_ux|^2 only)
// The rows are left in stage.xs and mu in stage.tmpc; without var, K*u in bufA; with var, A = K*u L_uu^-T in bufA and
// B = K*u L_s^-T in bufB
static int fitc_predict_chunk(gpb200_fitc* f, const double* xs, int64_t ldxs, int64_t mc, double* mu, double* var) {
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    FCK(cudaMemcpy2DAsync(f->stage.xs, sizeof(double) * f->d, xs, sizeof(double) * ldxs, sizeof(double) * f->d, mc,
                          cudaMemcpyHostToDevice, st));
    FCK(fitc_kfu(f, f->stage.xs, mc));
    FCK(rowdot_launch(f->stage.bufA, f->Mpad, f->data.uvec, mc, f->Mpad, f->stage.tmpc, st, &eu->launches));
    FCK(cudaMemcpyAsync(mu, f->stage.tmpc, sizeof(double) * mc, cudaMemcpyDeviceToHost, st));
    if (!var) return GPB200_OK;
    FCK(cudaMemcpyAsync(f->stage.bufB, f->stage.bufA, sizeof(double) * f->Nc * f->Mpad, cudaMemcpyDeviceToDevice, st));
    FCK(trsm_rec_buf(eu, gbuf(eu, f->stage.bufA, f->stage.mapA, f->Mpad), (int)f->Nc, 0, (int)f->Mpad));
    FCK(trsm_rec_buf(es, gbuf(eu, f->stage.bufB, f->stage.mapB2, f->Mpad), (int)f->Nc, 0, (int)f->Mpad));
    FCK(kdiag_launch(eu->prog, f->stage.xs, f->d, mc, f->stage.tmpc, st, &eu->launches));
    FCK(rowvar_launch(f->stage.bufA, f->Mpad, f->stage.tmpc, mc, f->Mpad, f->stage.tmpc2, st, &eu->launches));       // k_xx - q
    FCK(rowvar_launch(f->stage.bufB, f->Mpad, f->stage.zeroc, mc, f->Mpad, f->stage.w, st, &eu->launches));          // -s
    if (f->mode == 2) FCK(cudaMemsetAsync(f->stage.tmpc2, 0, sizeof(double) * mc, st));
    FCK(ew_launch(6, mc, f->stage.tmpc, f->stage.tmpc2, f->stage.w, nullptr, 0.0, st, &eu->launches));               // [k_xx - q] + s
    FCK(cudaMemcpyAsync(var, f->stage.tmpc, sizeof(double) * mc, cudaMemcpyDeviceToHost, st));
    return GPB200_OK;
}

int gpb200_fitc_predict(gpb200_fitc* f, int64_t Ms, const double* xs, int64_t ldxs, double* mu, double* var) {
    if (!f || Ms <= 0 || !xs || ldxs < f->d || !mu) return GPB200_EINVAL;
    if (!f->factored || !(f->alpha_ready || f->u_ready)) return fail(f, GPB200_ESTATE, "fitc_predict: factorize and mll first");
    if (f->mode == 3) return fail(f, GPB200_EINVAL, "fitc_predict: FSA predictions need test blocks");
    FCK(cudaSetDevice(f->device));
    for (int64_t m0 = 0; m0 < Ms; m0 += f->Nc) {
        TRY(fitc_predict_chunk(f, xs + m0 * ldxs, ldxs, std::min(f->Nc, Ms - m0), mu + m0, var ? var + m0 : nullptr));
        FCK(cudaStreamSynchronize(f->eu->st));
    }
    return GPB200_OK;
}

// Predictive gradients of the sparse models (predict_f with ForwardDiff.Dual inputs): mu and var through
// gpb200_fitc_predict's chunk step (A = K*u L_uu^-T in bufA, B = K*u L_s^-T in bufB), then W' = A L_uu^-1 - B L_s^-1
// (= K*u K_uu^-1 - K*u Sigma_QR^-1; SoR: - B L_s^-1) by the right-side TRSM on the two M x M sub-engines, whose F holds L'
// in its strict-upper tiles for the call, and the contraction over the inducing points with alpha = u:
//   dmu[m, :] = sum_j dk(x*_m, u_j)/dx*_m u_j,   dvar[m, :] = 2c dk(x*_m, x*_m)/dx*_m - 2 sum_j dk(x*_m, u_j)/dx*_m W'[m, j]
// with c = 1 (FITC, DTC) or 0 (SoR, whose variance has no k_xx).  Single GPU, modes 0-2.
int gpb200_fitc_predict_grad(gpb200_fitc* f, int64_t Ms, const double* xs, int64_t ldxs, double* mu, double* var,
                             double* dmu, double* dvar) {
    if (!f) return GPB200_EINVAL;
    if (!f->factored || !(f->alpha_ready || f->u_ready)) return fail(f, GPB200_ESTATE, "fitc_predict_grad: factorize and mll first");
    if (f->mode == 3) return fail(f, GPB200_EINVAL, "fitc_predict_grad: not available for FSA");
    if (f->nranks > 1) return fail(f, GPB200_EINVAL, "fitc_predict_grad: single GPU handles only");
    if (Ms <= 0 || !xs || ldxs < f->d || !mu || !dmu) return fail(f, GPB200_EINVAL, "fitc_predict_grad: bad Ms, xs, ldxs, mu or dmu");
    if (!var != !dvar) return fail(f, GPB200_EINVAL, "fitc_predict_grad: var and dvar must be given together");
    FCK(cudaSetDevice(f->device));
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int d = f->d;
    FCK(f->pdx.ensure((size_t)2 * f->Nc * d));
    double* ddmu = f->pdx;
    double* ddvar = f->pdx + f->Nc * d;
    const GemmBuf bA = gbuf(eu, f->stage.bufA, f->stage.mapA, f->Mpad);
    const GemmBuf bB2 = gbuf(eu, f->stage.bufB, f->stage.mapB2, f->Mpad);
    if (var) {
        FCK(mirror_lower_tiles_launch(eu->F, eu->ld, eu->Npad, st, &eu->launches));
        FCK(mirror_lower_tiles_launch(es->F, es->ld, es->Npad, st, &eu->launches));
    }
    for (int64_t m0 = 0; m0 < Ms; m0 += f->Nc) {
        const int64_t mc = std::min(f->Nc, Ms - m0);
        TRY(fitc_predict_chunk(f, xs + m0 * ldxs, ldxs, mc, mu + m0, var ? var + m0 : nullptr));
        if (var) {
            if (f->mode != 2) FCK(trsm_right_rec_buf(eu, bA, (int)f->Nc, 0, (int)f->Mpad));      // A L_uu^-1
            FCK(trsm_right_rec_buf(es, bB2, (int)f->Nc, 0, (int)f->Mpad));                        // B L_s^-1
        }
        FCK(crossgram_dx_launch(eu->prog, f->stage.xs, d, mc, eu->x, d, f->M, d, f->data.uvec, (var && f->mode != 2) ? f->stage.bufA.data() : nullptr,
                                var ? f->stage.bufB.data() : nullptr, f->Mpad, f->mode == 2 ? 0.0 : 1.0, ddmu, ddvar, st, &eu->launches));
        FCK(cudaMemcpyAsync(dmu + m0 * d, ddmu, sizeof(double) * mc * d, cudaMemcpyDeviceToHost, st));
        if (var) FCK(cudaMemcpyAsync(dvar + m0 * d, ddvar, sizeof(double) * mc * d, cudaMemcpyDeviceToHost, st));
        FCK(cudaStreamSynchronize(st));
    }
    return GPB200_OK;
}

// predictMVN with the FULL predictive covariance (fitc.jl:324-332 -> determ_train_conditional.jl:41-59 ->
// subsetofregressors.jl:302-321):  Sigma* = K** - K*u K_uu^-1 Ku* + K*u S^-1 Ku*   (FITC, DTC);   K*u S^-1 Ku*   (SoR)
// = K** - A A' + B B' with A = K*u L_uu^-T, B = K*u L_s^-T: two whitening TRSMs and two NT GEMMs.  Ms <= one staging chunk.
// mu into mu[Ms]; mu* and Sigma* left on the device (stage.tmpc, Kss) as *out says, on eu's stream; Ms <= Nc
static int fitc_cov_build(gpb200_fitc* f, int64_t Ms, const double* xs, int64_t ldxs, double* mu, DevPrediction* out) {
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int64_t Mspad = (Ms + TILE - 1) / TILE * TILE;
    FCK(f->Kss.ensure((size_t)Mspad * Mspad));
    const GemmBuf bA = gbuf(eu, f->stage.bufA, f->stage.mapA, f->Mpad);
    const GemmBuf bB2 = gbuf(eu, f->stage.bufB, f->stage.mapB2, f->Mpad);
    TRY(fitc_predict_chunk(f, xs, ldxs, Ms, mu, nullptr));                    // bufA = K*u  (Ms x Mpad, zero padded rows)
    FCK(cudaMemcpyAsync(f->stage.bufB, f->stage.bufA, sizeof(double) * f->Nc * f->Mpad, cudaMemcpyDeviceToDevice, st));
    FCK(trsm_rec_buf(es, bB2, (int)Mspad, 0, (int)f->Mpad));             // B = K*u L_s^-T
    if (f->mode != 2) {
        FCK(trsm_rec_buf(eu, bA, (int)Mspad, 0, (int)f->Mpad));         // A = K*u L_uu^-T
        FCK(gram_full_launch(eu->prog, f->stage.xs, f->d, Ms, Mspad, f->d, f->Kss, Mspad, st, &eu->launches));
        FCK(gemm_whole(eu, bA, bA, f->Kss, Mspad, Mspad, Mspad, f->Mpad, -1.0, 1.0));
    } else {
        FCK(cudaMemsetAsync(f->Kss, 0, sizeof(double) * Mspad * Mspad, st));
    }
    FCK(gemm_whole(es, bB2, bB2, f->Kss, Mspad, Mspad, Mspad, f->Mpad, 1.0, 1.0));
    *out = DevPrediction{f->stage.tmpc, f->Kss, Mspad};
    return GPB200_OK;
}

int gpb200_fitc_predict_cov(gpb200_fitc* f, int64_t Ms, const double* xs, int64_t ldxs, double* mu, double* cov) {
    if (!f || Ms <= 0 || !xs || ldxs < f->d || !mu || !cov) return GPB200_EINVAL;
    if (!f->factored || !(f->alpha_ready || f->u_ready)) return fail(f, GPB200_ESTATE, "fitc_predict_cov: factorize and mll first");
    if (f->mode == 3) return fail(f, GPB200_EINVAL, "fitc_predict_cov: FSA predictions need test blocks");
    if (Ms > f->Nc) return fail(f, GPB200_EINVAL, "fitc_predict_cov: too many test points for one staging chunk");
    FCK(cudaSetDevice(f->device));
    DevPrediction p;
    TRY(fitc_cov_build(f, Ms, xs, ldxs, mu, &p));
    FCK(cudaMemcpy2DAsync(cov, sizeof(double) * Ms, p.cov, sizeof(double) * p.ldc, sizeof(double) * Ms, Ms, cudaMemcpyDeviceToHost, f->eu->st));
    FCK(cudaStreamSynchronize(f->eu->st));
    return GPB200_OK;
}

// Kernel-parameter gradient of the FITC mll: dmll_kern!(::FullyIndepStrat) (fitc.jl:200-234) on top of
// dmll_kern!(::SubsetOfRegsStrategy) (subsetofregressors.jl:219-253), regrouped so that every
// parameter shares the same three weighted traces (kernel derivatives recomputed on the fly):
//   dmll_p = 1/2 [ <W_fu, dK_fu/dθ_p> + <W_uu, dK_uu/dθ_p> + sum_i g_i dK_ii/dθ_p ]
//   g_i   = alpha_i^2 - (Sigma^-1)_ii ,  (Sigma^-1)_ii = 1/L_i - K_fu,i S^-1 K_uf,i / L_i^2      (trinvAB, fitc.jl:63-67)
//   W_fu  = 2 alpha beta' - 2 L^-1 K_fu S^-1 - 2 diag(g) K_fu K_uu^-1 ,  beta = K_uu^-1 K_uf alpha   (sor.jl:147)
//   W_uu  = -beta beta' + K_uu^-1 - S^-1 + K_uu^-1 (K_uf diag(g) K_fu) K_uu^-1
// with S = Sigma_QR, L = Lambda; uses Sigma^-1 K_fu K_uu^-1 = L^-1 K_fu S^-1 and
// K_uu^-1 K_uf Sigma^-1 K_fu K_uu^-1 = K_uu^-1 - S^-1 (both follow from S = K_uu + K_uf L^-1 K_fu).
// All O(M^2 N) work is NT GEMMs against the explicit M x M inverses (grad_prepare of the sub-engines).
//
// Inducing points (dmll_xu != null, gpb200_fitc_grad_kernel_inducing): moving u_j changes K_fu and K_uu only (k_ii and the
// FSA blocks K_bb do not depend on Xu), so the same adjoints give
//   dmll/du_j = 1/2 [ sum_i W_fu[i, j] dk(u_j, x_i)/du_j + sum_l (W_uu[j, l] + W_uu[l, j]) dk(u_j, u_l)/du_j ]
// (W_uu is not exactly symmetric: it comes from two GEMMs).  One inducing_dx launch per chunk reads W_fu where
// trace_rect reads it and accumulates into f->dxu in chunk order; one more after the chunk loop contracts W_uu + W_uu'.
// Without dmll_xu the launches are exactly those of the kernel gradient alone; with it, they are the same launches plus
// the contractions (and, on several ranks, one all-reduce of the M x d partial), which read and write nothing else.
//
// Training inputs (dmll_x != null, gpb200_fitc_grad_kernel_inputs): x_i enters row i of K_fu, K_ii (FITC) and row and
// column i of its FSA block K_bb, never K_uu, so with d1k the derivative in the first argument
//   FITC:      dmll/dx_i = 1/2 [ sum_j W_fu[i, j] d1k(x_i, u_j) + 2 g_i d1k(x_i, x_i) ]
//   DTC, SoR:  dmll/dx_i = 1/2   sum_j W_fu[i, j] d1k(x_i, u_j)
//   FSA:       dmll/dx_i = 1/2 [ sum_j W_fu[i, j] d1k(x_i, u_j) + sum_{l in b(i)} (G_b[i, l] + G_b[l, i]) d1k(x_i, x_l) ]
// (2 d1k(x, x) is the derivative of k(x, x): 0 for the stationary leaves; G_b is not exactly symmetric, it comes from GEMMs).
// The mean's part alpha_i dm(x_i)/dx_i is the caller's.  One rows_dx launch per chunk reads W_fu where trace_rect reads it
// (FITC with c = g); FSA adds one fsa_block_dx launch per chunk over the G_b tiles in Gpk, after fsa_outer completes them
// and before the next chunk overwrites them, and writes in the caller's order through the inverse row map.  The rows are
// the rank's own, so nothing is exchanged.  Without dmll_x the launch sequence is unchanged.
static int event_pairs(gpb200_fitc* f, std::vector<cudaEvent_t>& ev, size_t pairs) {
    while (ev.size() < 2 * pairs) {
        cudaEvent_t e;
        FCK(cudaEventCreate(&e));
        ev.push_back(e);
    }
    return GPB200_OK;
}


static int fitc_grad(gpb200_fitc* f, double* dmll_kernel, double* dmll_xu, double* dmll_x, const char* who) {
    if (!f->factored || !f->alpha_ready) return fail(f, GPB200_ESTATE, std::string(who) + ": factorize and mll first");
    FCK(cudaSetDevice(f->device));
    const size_t chunks = f->mode == 3 ? fsa_num_chunks(f) : (size_t)((f->N + f->Nc - 1) / f->Nc);
    if (dmll_xu) {
        TRY(event_pairs(f, f->xu_ev, chunks + 2));
        FCK(f->dxu.ensure((size_t)f->M * f->d));
        FCK(cudaEventRecord(f->xu_ev[0], f->eu->st));
    }
    if (dmll_x) {
        TRY(event_pairs(f, f->x_ev, 2 * chunks + 1));
        FCK(f->dx.ensure((size_t)f->N * f->d));
        FCK(cudaEventRecord(f->x_ev[0], f->eu->st));
    }
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int np = eu->prog.n_theta;
    const int64_t Mp = f->Mpad, Nc = f->Nc;
    if (!f->grad.ready) TRY(make_group(f->grad, [&] {
        FitcGradWs& g = f->grad;
        FCK(g.bufC.alloc((size_t)Nc * Mp));
        for (DevBuf<double>* p : {&g.Hbuf, &g.Wbuf, &g.Tbuf}) FCK(p->alloc((size_t)Mp * Mp));
        FCK(g.gvec.alloc(f->Ncap + TILE));
        FCK(g.betav.alloc(Mp));
        const size_t tiles = (size_t)std::max((Nc / TILE) * (Mp / TILE), (Mp / TILE) * (Mp / TILE));
        FCK(g.gpart.alloc(tiles * GPB200_MAX_THETA));
        FCK(g.gacc.alloc(GPB200_MAX_THETA));
        FCK(g.gtmp.alloc(GPB200_MAX_THETA));
        if (eu->tma_ok) {
            const bool ok = gemm_make_tensor_map(&g.mapAt, f->stage.bufA, Mp, Nc, Nc) && gemm_make_tensor_map(&g.mapC, g.bufC, Nc, Mp, Mp) &&
                            gemm_make_tensor_map(&g.mapCt, g.bufC, Mp, Nc, Nc) && gemm_make_tensor_map(&g.mapH, g.Hbuf, Mp, Mp, Mp) &&
                            gemm_make_tensor_map(&g.mapT, g.Tbuf, Mp, Mp, Mp);
            if (!ok) return fail(f, GPB200_ECUDA, "fitc_grad_kernel: cuTensorMapEncodeTiled failed");
        }
        g.ready = true;
        return GPB200_OK;
    }));
    // explicit K_uu^-1 and Sigma_QR^-1 (full symmetric) in the sub-engines' G buffers
    FSUB(gpb200_grad_prepare(eu), eu);
    FSUB(gpb200_grad_prepare(es), es);
    FCK(symmetrize_launch(eu->G, eu->ld, Mp, st, &eu->launches));
    FCK(symmetrize_launch(es->G, es->ld, Mp, st, &eu->launches));
    const GemmBuf bA = gbuf(eu, f->stage.bufA, f->stage.mapA, Mp), bAt = gbuf(eu, f->stage.bufA, f->grad.mapAt, Nc);
    const GemmBuf bCt = gbuf(eu, f->grad.bufC, f->grad.mapCt, Nc);
    const GemmBuf bH = gbuf(eu, f->grad.Hbuf, f->grad.mapH, Mp), bT = gbuf(eu, f->grad.Tbuf, f->grad.mapT, Mp);
    // beta = K_uu^-1 (K_uf alpha)
    FCK(cudaMemsetAsync(f->data.rhsm, 0, sizeof(double) * Mp, st));
    for (int64_t r0 = 0; r0 < f->N; r0 += Nc) {
        const int64_t nc = std::min(Nc, f->N - r0);
        FCK(fitc_kuf(f, f->data.x + r0 * f->d, nc));
        FCK(cudaMemsetAsync(f->stage.w, 0, sizeof(double) * Nc, st));
        FCK(cudaMemcpyAsync(f->stage.w, f->data.alpha + r0, sizeof(double) * nc, cudaMemcpyDeviceToDevice, st));
        FCK(rowdot_launch(f->stage.bufB, Nc, f->stage.w, f->M, Nc, f->data.tmpm, st, &eu->launches));
        FCK(ew_launch(2, f->M, f->data.rhsm, f->data.tmpm, nullptr, nullptr, 0.0, st, &eu->launches));
    }
    TRY(fitc_allreduce(f, f->data.rhsm, (size_t)Mp));                    // K_uf alpha over all rows
    FCK(solve_device(eu, f->data.rhsm, f->data.tmpm, f->grad.betav));
    FCK(cudaMemsetAsync(f->grad.gacc, 0, sizeof(double) * GPB200_MAX_THETA, st));
    FCK(cudaMemsetAsync(f->grad.Hbuf, 0, sizeof(double) * Mp * Mp, st));
    if (f->mode == 3) return fsa_grad_kernel(f, dmll_kernel, dmll_xu, dmll_x);
    size_t xk = 0, rk = 0;                                                // Xu / X contraction launches so far
    for (int64_t r0 = 0; r0 < f->N; r0 += Nc) {
        const int64_t nc = std::min(Nc, f->N - r0);
        const double* xr = f->data.x + r0 * f->d;
        FCK(fitc_kfu(f, xr, nc));                                         // bufA = K_fu chunk
        FCK(gemm_whole(es, bA, bufG(es), f->stage.bufB, Mp, Nc, Mp, Mp, 1.0, 0.0));         // P2 = K_fu S^-1 -> bufB (as Nc x Mpad)
        FCK(rowdot2_launch(f->stage.bufA, f->stage.bufB, Mp, nc, Mp, f->stage.tmpc, st, &eu->launches));
        if (f->mode == 0) FCK(fitc_g_launch(nc, f->data.alpha + r0, f->data.lam + r0, f->stage.tmpc, f->grad.gvec + r0, st, &eu->launches));
        else FCK(cudaMemsetAsync(f->grad.gvec + r0, 0, sizeof(double) * nc, st));       // SoR part only (sor.jl:219-253)
        FCK(gemm_whole(eu, bA, bufG(eu), f->grad.bufC, Mp, Nc, Mp, Mp, 1.0, 0.0));         // P1 = K_fu K_uu^-1 -> bufC
        FCK(fitc_wfu_launch(f->stage.bufB, f->grad.bufC, Mp, nc, f->M, f->data.alpha + r0, f->data.lam + r0, f->grad.gvec + r0, f->grad.betav, st, &eu->launches));
        FCK(trace_rect_launch(eu->prog, xr, f->d, nc, eu->x, f->d, f->M, f->d, f->stage.bufB, Mp, f->grad.gpart, f->grad.gtmp, st, &eu->launches));
        FCK(ew_launch(2, np, f->grad.gacc, f->grad.gtmp, nullptr, nullptr, 0.0, st, &eu->launches));
        if (dmll_xu) { TRY(xu_contract(f, xk + 1, xr, nc, f->stage.bufB, 0, nullptr, xk > 0)); ++xk; }
        if (dmll_x) {
            TRY(x_rows(f, rk + 1, xr, nc, f->stage.bufB, f->mode == 0 ? f->grad.gvec + r0 : nullptr, nullptr, nullptr, f->dx + r0 * f->d, 0));
            ++rk;
        }
        if (f->mode != 0) continue;                                       // no Lambda-derivative terms for SoR / DTC
        // diagonal term sum_i g_i dK_ii/dθ_p (scratch: bufC as np x nc)
        FCK(kdiag_grad_launch(eu->prog, xr, f->d, nc, f->grad.gvec + r0, f->grad.bufC, st, &eu->launches));
        for (int p = 0; p < np; ++p) FCK(sum_launch(f->grad.bufC + (size_t)p * nc, nc, f->grad.gtmp + p, st, &eu->launches));
        FCK(ew_launch(2, np, f->grad.gacc, f->grad.gtmp, nullptr, nullptr, 0.0, st, &eu->launches));
        // H += K_uf diag(g) K_fu
        FCK(crossgram_launch(eu->prog, eu->x, f->d, f->M, Mp, xr, f->d, nc, Nc, f->d, f->stage.bufA, Nc, st, &eu->launches));   // bufA = K_uf chunk (Mpad x Nc)
        FCK(cudaMemcpyAsync(f->grad.bufC, f->stage.bufA, sizeof(double) * Mp * Nc, cudaMemcpyDeviceToDevice, st));
        FCK(colscale_launch(f->grad.bufC, Nc, Mp, nc, f->grad.gvec + r0, st, &eu->launches));
        FCK(gemm_whole(eu, bAt, bCt, f->grad.Hbuf, Mp, Mp, Mp, Nc, 1.0, 1.0));
    }
    // multi-GPU: the per-row traces and H = K_uf diag(g) K_fu are sums over the ranks' rows; the M x M part below is replicated
    TRY(fitc_allreduce(f, f->grad.gacc, (size_t)np));
    TRY(fitc_allreduce(f, f->grad.Hbuf, (size_t)Mp * (size_t)Mp));
    if (dmll_xu) TRY(fitc_allreduce(f, f->dxu, (size_t)f->M * f->d));   // W_fu part over all rows
    // T = K_uu^-1 H ; Wbuf = K_uu^-1 T' = K_uu^-1 H K_uu^-1
    FCK(gemm_whole(eu, bufG(eu), bH, f->grad.Tbuf, Mp, Mp, Mp, Mp, 1.0, 0.0));
    FCK(gemm_whole(eu, bufG(eu), bT, f->grad.Wbuf, Mp, Mp, Mp, Mp, 1.0, 0.0));
    FCK(fitc_wuu_launch(f->grad.Wbuf, f->grad.Wbuf, eu->G, es->G, Mp, f->M, f->grad.betav, st, &eu->launches));
    FCK(trace_rect_launch(eu->prog, eu->x, f->d, f->M, eu->x, f->d, f->M, f->d, f->grad.Wbuf, Mp, f->grad.gpart, f->grad.gtmp, st, &eu->launches));
    FCK(ew_launch(2, np, f->grad.gacc, f->grad.gtmp, nullptr, nullptr, 0.0, st, &eu->launches));
    if (dmll_xu) {
        TRY(xu_contract(f, xk + 1, eu->x, f->M, f->grad.Wbuf, 1, nullptr, 1)); ++xk;
        FCK(cudaEventRecord(f->xu_ev[1], st));
    }
    if (dmll_x) FCK(cudaEventRecord(f->x_ev[1], st));
    std::vector<double> out((size_t)std::max(np, 1));
    FCK(cudaMemcpyAsync(out.data(), f->grad.gacc, sizeof(double) * np, cudaMemcpyDeviceToHost, st));
    FCK(cudaStreamSynchronize(st));
    FSUB(check_trsv_watchdog(eu), eu);                                   // the solve for beta above
    if (dmll_kernel) for (int p = 0; p < np; ++p) dmll_kernel[p] = 0.5 * out[p];
    if (dmll_xu) TRY(xu_finish(f, xk, dmll_xu));
    if (dmll_x) TRY(x_finish(f, rk, dmll_x));
    return GPB200_OK;
}

int gpb200_fitc_grad_kernel(gpb200_fitc* f, double* dmll_kernel) {
    if (!f || !dmll_kernel) return GPB200_EINVAL;
    return fitc_grad(f, dmll_kernel, nullptr, nullptr, "fitc_grad_kernel");
}

int gpb200_fitc_grad_kernel_inducing(gpb200_fitc* f, double* dmll_kernel, double* dmll_xu) {
    if (!f) return GPB200_EINVAL;
    if (!dmll_xu) return fail(f, GPB200_EINVAL, "fitc_grad_kernel_inducing: dmll_xu is required");
    return fitc_grad(f, dmll_kernel, dmll_xu, nullptr, "fitc_grad_kernel_inducing");
}

int gpb200_fitc_grad_kernel_inputs(gpb200_fitc* f, double* dmll_kernel, double* dmll_xu, double* dmll_x) {
    if (!f) return GPB200_EINVAL;
    if (!dmll_x) return fail(f, GPB200_EINVAL, "fitc_grad_kernel_inputs: dmll_x is required");
    return fitc_grad(f, dmll_kernel, dmll_xu, dmll_x, "fitc_grad_kernel_inputs");
}

// Replaces the inducing inputs of both sub-engines in place (same M and d: no buffer is reallocated); the training inputs,
// the kernel program, the FSA blocks and every workspace are kept.  The factorisation, alpha and the cross-validation state
// refer to the old Xu and are invalidated.
int gpb200_fitc_set_inducing(gpb200_fitc* f, int64_t M, const double* xu, int64_t ldxu) {
    if (!f) return GPB200_EINVAL;
    if (!f->has_data) return fail(f, GPB200_ESTATE, "fitc_set_inducing: set_data first");
    if (M != f->M || !xu || ldxu < f->d) {
        return fail(f, GPB200_EINVAL, "fitc_set_inducing: M must be set_data's, xu non-null and ldxu >= d");
    }
    FCK(cudaSetDevice(f->device));
    fitc_invalidate(f); f->cv.m_ok = false;
    FSUB(gpb200_set_data(f->eu, M, f->d, xu, ldxu), f->eu);
    FSUB(gpb200_set_data(f->es, M, f->d, xu, ldxu), f->es);
    return GPB200_OK;
}

// Replaces the training inputs in place (same N and d: no buffer is reallocated); FSA rebuilds its padded copy through the
// kept row map, so the blocks, their work lists and every workspace stay.  The factorisation, alpha and the cross-validation
// state refer to the old inputs and are invalidated.
int gpb200_fitc_set_inputs(gpb200_fitc* f, int64_t N, const double* x, int64_t ldx) {
    if (!f) return GPB200_EINVAL;
    if (!f->has_data) return fail(f, GPB200_ESTATE, "fitc_set_inputs: set_data first");
    if (N != f->N || !x || ldx < f->d) return fail(f, GPB200_EINVAL, "fitc_set_inputs: N must be set_data's, x non-null and ldx >= d");
    FCK(cudaSetDevice(f->device));
    fitc_invalidate(f); f->cv.m_ok = false;
    cudaStream_t st = f->eu->st;
    FCK(cudaMemcpy2DAsync(f->data.x, sizeof(double) * f->d, x, sizeof(double) * ldx, sizeof(double) * f->d, N, cudaMemcpyHostToDevice, st));
    if (f->fsa) TRY(fsa_set_inputs(f, x, ldx));
    FCK(cudaStreamSynchronize(st));
    return GPB200_OK;
}
}  // extern "C"

// the N-sized buffers hold at least n rows: capacity doubles (at least to n), x, Lambda and r are copied, and the
// gradient and cross-validation workspaces, sized by the capacity, are freed to be remade at the next use
static int fitc_grow(gpb200_fitc* f, int64_t n) {
    if (n <= f->Ncap) return GPB200_OK;
    const int64_t cap = std::max(n, 2 * f->Ncap);
    cudaStream_t st = f->eu->st;
    FitcData g;
    FCK(g.x.alloc((size_t)cap * f->d));
    for (DevBuf<double>* p : {&g.lam, &g.y, &g.alpha, &g.tmpn}) {
        FCK(p->alloc(cap + TILE));
        FCK(cudaMemsetAsync(*p, 0, sizeof(double) * (cap + TILE), st));
    }
    FCK(cudaMemcpyAsync(g.x, f->data.x, sizeof(double) * f->N * f->d, cudaMemcpyDeviceToDevice, st));
    FCK(cudaMemcpyAsync(g.lam, f->data.lam, sizeof(double) * f->N, cudaMemcpyDeviceToDevice, st));
    FCK(cudaMemcpyAsync(g.y, f->data.y, sizeof(double) * f->N, cudaMemcpyDeviceToDevice, st));
    FCK(cudaStreamSynchronize(st));                                      // before the old buffers are freed
    f->data.x = std::move(g.x); f->data.lam = std::move(g.lam); f->data.y = std::move(g.y);
    f->data.alpha = std::move(g.alpha); f->data.tmpn = std::move(g.tmpn);
    f->grad = {}; f->cv = {};
    f->Ncap = cap;
    return GPB200_OK;
}

extern "C" {
// ================================================================================================
// append! for FITC, DTC and SoR: k new observations with the hyper-parameters and Xu fixed.  K_uu, L_uu and the old rows'
// Lambda_i do not change; Sigma_QR and b change by one rank-k term and one M-vector, so the cost is O(k M^2 + M^3) whatever
// N is.  With K_nu (k x M) the cross-Gram of the new rows, Lambda_n their diagonal terms (FITC: sigma^2 + k_ii -
// |L_uu^-1 k_ui|^2; DTC / SoR: sigma^2) and r_n their residuals, with the chunk steps factorize and mll run (fitc_lambda,
// fitc_syrk_add, fitc_b_add):
//   Sigma_QR <- Sigma_QR + K_un Lambda_n^-1 K_nu       (lower-only SYRK on the DMMA GEMM)
//   b        <- b + K_un Lambda_n^-1 r_n
//   s        <- s + sum r_n^2 / Lambda_n               (s = r'Lambda^-1 r)
//   l        <- l + sum log Lambda_n                   (l = sum log Lambda_i)
//   L_s = chol(Sigma_QR),  u = Sigma_QR^-1 b
//   mll = -1/2 ( s - b'u + logdet Sigma_QR - logdet K_uu + l + N log 2 pi )
// using r'alpha = r'Lambda^-1 r - b'Sigma_QR^-1 b: the mll of gpb200_fitc_mll on the concatenated data, without alpha.
// The unfactored Sigma_QR is kept in f->app.sqr.  factorize leaves only its factor, so the first append after it rebuilds
// Sigma_QR once as L_s L_s' (one lower-only NT product; GEMM_KHI_N stops each tile's k range at its diagonal tile, so the
// strict-upper tiles of F, which other schedules use as scratch, are never read, and the diagonal tiles of F are clean above
// their diagonal: the leaf writes i >= j only).  Later appends add to the kept copy, which is copied into es and factored.
// s and l are summed over all rows (O(N), no kernel evaluation) on the first append after a mll and carried from then on.
// On several ranks the call is collective: the M x M increment (accumulated in es->G, which the refactor overwrites
// anyway), the b increment and the three scalars (s, l, N) are summed with one all-reduce each.
// ================================================================================================
int gpb200_fitc_append(gpb200_fitc* f, int64_t k, const double* xnew, int64_t ldx, const double* r_new, double* mll,
                       double* logdet) {
    if (!f) return GPB200_EINVAL;
    if (f->mode == 3) return fail(f, GPB200_EINVAL, "fitc_append: not available for FSA (mode 3); new rows would need new blocks, refit with set_data");
    const bool multi = f->nranks > 1;
    if (k < (multi ? 0 : 1)) return fail(f, GPB200_EINVAL, multi ? "fitc_append: k must be >= 0" : "fitc_append: k must be >= 1");
    if (ldx < f->d) return fail(f, GPB200_EINVAL, "fitc_append: ldx must be >= d");
    if (!mll || (k > 0 && (!xnew || !r_new))) return fail(f, GPB200_EINVAL, "fitc_append: xnew, r_new and mll must be non-null");
    for (int64_t i = 0; i < k; ++i)
        if (!std::isfinite(r_new[i])) return fail(f, GPB200_EINVAL, "fitc_append: non-finite r_new");
    if (!f->factored || !(f->alpha_ready || f->u_ready)) return fail(f, GPB200_ESTATE, "fitc_append: factorize and mll first");
    FCK(cudaSetDevice(f->device));
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int64_t Mp = f->Mpad, Nc = f->Nc, N0 = f->N, N1 = N0 + k;
    const int d = f->d;
    if (!f->app.sqr_ok) {                                                // Sigma_QR = L_s L_s', once per factorize
        FCK(f->app.sqr.ensure((size_t)Mp * Mp));
        FCK(cudaMemsetAsync(f->app.sqr, 0, sizeof(double) * Mp * Mp, st));           // clean above the diagonal
        FCK(gemm_whole(es, bufF(es), bufF(es), f->app.sqr, Mp, Mp, Mp, Mp, 1.0, 0.0, nullptr, 0, GEMM_LOWER_ONLY | GEMM_KHI_N));
        f->app.sqr_ok = true;
    }
    TRY(fitc_grow(f, N1));
    fsa_free(f);                                                         // FSA blocks partition the old rows only
    // until the refactor below succeeds, the handle holds no factorisation of its data
    f->factored = f->alpha_ready = f->u_ready = f->cv.m_ok = false;
    es->inv_ready = false;                                               // es->G is scratch from here on
    if (k > 0) {
        FCK(cudaMemcpy2DAsync(f->data.x + N0 * d, sizeof(double) * d, xnew, sizeof(double) * ldx, sizeof(double) * d, k,
                              cudaMemcpyHostToDevice, st));
        FCK(cudaMemcpyAsync(f->data.y + N0, r_new, sizeof(double) * k, cudaMemcpyHostToDevice, st));
    }
    f->N = N1;
    // one rank: the increment goes straight into the kept Sigma_QR; several: into es->G (ld Mpad, as in factorize), summed
    // over the ranks below
    double* dS = multi ? es->G : f->app.sqr.data();
    if (multi) FCK(cudaMemsetAsync(es->G, 0, sizeof(double) * Mp * Mp, st));
    FCK(cudaMemsetAsync(f->data.rhsm, 0, sizeof(double) * Mp, st));     // b increment
    for (int64_t r0 = N0; r0 < N1; r0 += Nc) {
        const int64_t nc = std::min(Nc, N1 - r0);
        const int64_t ncp = (nc + TILE - 1) / TILE * TILE;              // the TRSM and the SYRK stop at the chunk's padded rows
        TRY(fitc_lambda(f, r0, nc, ncp));
        FCK(fitc_kuf(f, f->data.x + r0 * d, nc));
        TRY(fitc_b_add(f, r0, nc, f->data.rhsm));                        // b += K_un Lambda_n^-1 r_n
        TRY(fitc_syrk_add(f, r0, nc, dS, Mp, ncp));                      // Sigma_QR += K_un Lambda_n^-1 K_nu
    }
    // s and l over the new rows, or over every row on the first append after a mll; and the row count
    const int64_t s0 = f->app.sums_ok ? N0 : 0;
    const double ns = (double)(N1 - s0);
    FCK(cudaMemsetAsync(f->data.scal + 8, 0, sizeof(double) * 2, st));
    if (N1 > s0) {
        FCK(ew_launch(1, N1 - s0, f->data.tmpn + s0, f->data.y + s0, f->data.lam + s0, nullptr, 0.0, st, &eu->launches));
        FCK(dot_launch(f->data.tmpn + s0, f->data.y + s0, N1 - s0, f->data.scal + 8, st, &eu->launches));
        FCK(ew_launch(4, N1 - s0, f->data.tmpn + s0, f->data.lam + s0, nullptr, nullptr, 0.0, st, &eu->launches));
        FCK(sum_launch(f->data.tmpn + s0, N1 - s0, f->data.scal + 9, st, &eu->launches));
    }
    FCK(cudaMemcpyAsync(f->data.scal + 10, &ns, sizeof(double), cudaMemcpyHostToDevice, st));
    if (multi) {
        TRY(fitc_allreduce(f, es->G, (size_t)Mp * Mp));
        FCK(ew_launch(2, Mp * Mp, f->app.sqr, es->G, nullptr, nullptr, 0.0, st, &eu->launches));
        TRY(fitc_allreduce(f, f->data.rhsm, (size_t)Mp));
        TRY(fitc_allreduce(f, f->data.scal + 8, 3));
    }
    FCK(ew_launch(2, f->M, f->data.bvec, f->data.rhsm, nullptr, nullptr, 0.0, st, &eu->launches));
    double sums[3];
    FCK(cudaMemcpyAsync(sums, f->data.scal + 8, sizeof(double) * 3, cudaMemcpyDeviceToHost, st));
    FCK(cudaStreamSynchronize(st));
    if (f->app.sums_ok) { f->app.s += sums[0]; f->app.l += sums[1]; f->app.n += sums[2]; }
    else { f->app.s = sums[0]; f->app.l = sums[1]; f->app.n = sums[2]; f->app.sums_ok = true; }
    // refactor the kept Sigma_QR; u = Sigma_QR^-1 b
    FCK(cudaMemcpyAsync(es->G, f->app.sqr, sizeof(double) * Mp * Mp, cudaMemcpyDeviceToDevice, st));
    const int rc = chol_inplace(es);
    if (rc != GPB200_OK) {
        fitc_invalidate(f);                                              // the grown data stays; factorize to go on
        return fail(f, rc, "fitc_append (Sigma_QR): " + es->err);
    }
    FCK(cudaMemcpyAsync(f->data.rhsm, f->data.bvec, sizeof(double) * Mp, cudaMemcpyDeviceToDevice, st));
    FCK(solve_device(es, f->data.rhsm, f->data.tmpm, f->data.uvec));
    FCK(dot_launch(f->data.bvec, f->data.uvec, f->M, f->data.scal + 0, st, &eu->launches));
    FCK(sum_launch(es->logd, es->Npad, f->data.scal + 1, st, &eu->launches));
    FCK(sum_launch(eu->logd, eu->Npad, f->data.scal + 2, st, &eu->launches));
    double s[3];
    FCK(cudaMemcpyAsync(s, f->data.scal, sizeof(double) * 3, cudaMemcpyDeviceToHost, st));
    FCK(cudaStreamSynchronize(st));
    FSUB(check_trsv_watchdog(es), es);                                   // the solve for u above
    f->Ntotal = f->app.n;
    f->factored = f->u_ready = true;
    const double ld = s[1] - s[2] + f->app.l;
    if (logdet) *logdet = ld;
    *mll = -(f->app.s - s[0] + ld + LOG2PI * f->app.n) / 2.0;
    return GPB200_OK;
}

// ================================================================================================
// Cross-validation on the sparse engine (src/crossvalidation.jl with cK a FITC / DTC / SoR covariance), one GPU.
// Sigma = Lambda + K_fu K_uu^-1 K_uf is the matrix gpb200_fitc_mll inverts; nothing N x N is formed.  With S = Sigma_QR,
// L = Lambda and the explicit K_uu^-1, S^-1 of the sub-engines (grad_prepare, as gpb200_fitc_grad_kernel):
//   Sigma^-1 = L^-1 - Ch K_uf L^-1,   Ch = L^-1 K_fu S^-1 = Sigma^-1 K_fu K_uu^-1   (row-local)
//   [Sigma^-1]_ii = 1/L_i - k_i S^-1 k_i' / L_i^2
// Per hyper-parameter j: dSigma_j = Delta + G C' + C G',  C = K_fu K_uu^-1,  G = dK_fu - 1/2 K_fu Dp,  Dp = dK_uu K_uu^-1,
// Delta = diag(dk_ii - 2 G_i.C_i) (FITC), 0 (SoR / DTC kernel parameters), I (noise variance; G = 0).  Then
//   Sigma^-1 dSigma_j Sigma^-1 = diag(Delta / L^2) + E Ch' + Ch E',   E = L^-1 G - L^-2 Delta K_fu + 1/2 Ch Q,
//   Q = H - R - R',  R = K_uf L^-1 G,  H = K_uf L^-1 Delta L^-1 K_fu      (both M x M)
//   Z_j alpha = Delta alpha / L + L^-1 G beta + Ch w,   beta = K_uu^-1 K_uf alpha,  w = G'alpha - K_uf L^-1 Delta alpha - R beta
// Pass 1 streams the chunks once to accumulate R, H and the M-vectors, pass 2 streams them again for the two N-vectors; a
// fold block reads the same quantities on the gathered rows V only.
// ================================================================================================
static int fitc_cv_check(gpb200_fitc* f, const char* who) {
    if (f->mode == 3) return fail(f, GPB200_EINVAL, std::string(who) + ": cross-validation is not available for FSA (mode 3)");
    if (f->nranks > 1)
        return fail(f, GPB200_EINVAL, std::string(who) + ": cross-validation runs on one GPU; this handle has " + std::to_string(f->nranks) + " ranks");
    if (!f->factored || !f->alpha_ready) return fail(f, GPB200_ESTATE, std::string(who) + ": factorize and mll first");
    return GPB200_OK;
}

// workspace on first use; K_uu^-1 and S^-1 as full symmetric matrices in the sub-engines' G (the state grad_kernel builds)
static int fitc_cv_prepare(gpb200_fitc* f) {
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int64_t Mp = f->Mpad, Nc = f->Nc, Ncap = f->Ncap;
    if (!f->cv.ready) TRY(make_group(f->cv, [&] {
        FitcCvWs& g = f->cv;
        for (DevBuf<double>* p : {&g.G, &g.Gt, &g.Ch, &g.P}) FCK(p->alloc((size_t)Nc * Mp));
        for (DevBuf<double>* p : {&g.Duu, &g.Dp, &g.R, &g.H, &g.Q}) FCK(p->alloc((size_t)Mp * Mp));
        for (DevBuf<double>* p : {&g.alpha, &g.del, &g.ilam, &g.za, &g.dg}) FCK(p->alloc(Ncap + Nc));
        for (DevBuf<double>* p : {&g.da, &g.q, &g.lamV, &g.delV}) FCK(p->alloc(Nc));
        FCK(g.xs.alloc((size_t)Nc * f->d));
        FCK(g.m.alloc(8 * Mp));
        FCK(g.idx.alloc(Nc));
        FCK(cudaMemsetAsync(g.alpha, 0, sizeof(double) * (Ncap + Nc), st));      // zero tail: chunk vectors are read Nc wide
        if (eu->tma_ok) {
            const bool ok = gemm_make_tensor_map(&g.mapGt, g.Gt, Mp, Nc, Nc) && gemm_make_tensor_map(&g.mapCh, g.Ch, Nc, Mp, Mp) &&
                            gemm_make_tensor_map(&g.mapP, g.P, Nc, Mp, Mp) && gemm_make_tensor_map(&g.mapDuu, g.Duu, Mp, Mp, Mp) &&
                            gemm_make_tensor_map(&g.mapDp, g.Dp, Mp, Mp, Mp) && gemm_make_tensor_map(&g.mapQ, g.Q, Mp, Mp, Mp);
            if (!ok) return fail(f, GPB200_ECUDA, "fitc_cv: cuTensorMapEncodeTiled failed");
        }
        g.ready = true;
        return GPB200_OK;
    }));
    FSUB(gpb200_grad_prepare(eu), eu);
    FSUB(gpb200_grad_prepare(es), es);
    FCK(symmetrize_launch(eu->G, eu->ld, Mp, st, &eu->launches));
    FCK(symmetrize_launch(es->G, es->ld, Mp, st, &eu->launches));
    return GPB200_OK;
}

int gpb200_fitc_get_inverse_diag(gpb200_fitc* f, double* diag) {
    if (!f || !diag) return GPB200_EINVAL;
    TRY(fitc_cv_check(f, "fitc_get_inverse_diag"));
    FCK(cudaSetDevice(f->device));
    TRY(fitc_cv_prepare(f));
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int64_t Mp = f->Mpad, Nc = f->Nc;
    const GemmBuf bA = gbuf(eu, f->stage.bufA, f->stage.mapA, Mp);
    for (int64_t r0 = 0; r0 < f->N; r0 += Nc) {
        const int64_t nc = std::min(Nc, f->N - r0);
        FCK(fitc_kfu(f, f->data.x + r0 * f->d, nc));                                                   // bufA = K_fu
        FCK(gemm_whole(f->eu, bA, bufG(es), f->cv.Ch, Mp, Nc, Mp, Mp, 1.0, 0.0));                      // K_fu S^-1
        FCK(rowdot2_launch(f->stage.bufA, f->cv.Ch, Mp, nc, Mp, f->cv.q, st, &eu->launches));
        FCK(fitc_cv_invdiag_launch(nc, f->data.lam + r0, f->cv.q, f->cv.dg + r0, st, &eu->launches));
    }
    FCK(cudaMemcpyAsync(diag, f->cv.dg, sizeof(double) * f->N, cudaMemcpyDeviceToHost, st));
    FCK(cudaStreamSynchronize(st));
    return GPB200_OK;
}

int gpb200_fitc_cv_param(gpb200_fitc* f, int32_t param, const double* alpha, double* Zj_alpha, double* diag_ZjSinv) {
    if (!f || !Zj_alpha || !diag_ZjSinv) return GPB200_EINVAL;
    TRY(fitc_cv_check(f, "fitc_cv_param"));
    const int np = f->eu->prog.n_theta;
    if (param < -1 || param >= np)
        return fail(f, GPB200_EINVAL, "fitc_cv_param: param must be -1 (noise variance) or a kernel parameter index below " + std::to_string(np));
    FCK(cudaSetDevice(f->device));
    TRY(fitc_cv_prepare(f));
    f->cv.m_ok = false;
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int64_t Mp = f->Mpad, Nc = f->Nc, N = f->N, M = f->M;
    const int d = f->d;
    const bool noise = param < 0;
    const int kind = noise ? 2 : (f->mode == 0 ? 0 : 1);
    const GemmBuf bA = gbuf(eu, f->stage.bufA, f->stage.mapA, Mp), bB = gbuf(eu, f->stage.bufB, f->stage.mapB, Nc);
    const GemmBuf bGt = gbuf(eu, f->cv.Gt, f->cv.mapGt, Nc), bCh = gbuf(eu, f->cv.Ch, f->cv.mapCh, Mp);
    const GemmBuf bDuu = gbuf(eu, f->cv.Duu, f->cv.mapDuu, Mp), bDp = gbuf(eu, f->cv.Dp, f->cv.mapDp, Mp);
    const GemmBuf bQ = gbuf(eu, f->cv.Q, f->cv.mapQ, Mp);
    double *kta = f->cv.m, *gta = f->cv.m + Mp, *uD = f->cv.m + 2 * Mp, *beta = f->cv.m + 3 * Mp;
    double *rb = f->cv.m + 4 * Mp, *w = f->cv.m + 5 * Mp, *tmp = f->cv.m + 6 * Mp;
    if (alpha) FCK(cudaMemcpyAsync(f->cv.alpha, alpha, sizeof(double) * N, cudaMemcpyHostToDevice, st));
    else FCK(cudaMemcpyAsync(f->cv.alpha, f->data.alpha, sizeof(double) * N, cudaMemcpyDeviceToDevice, st));
    FCK(ew_launch(5, N, f->cv.ilam, f->data.lam, nullptr, nullptr, 0.0, st, &eu->launches));              // 1 / Lambda
    FCK(cudaMemsetAsync(f->cv.m, 0, sizeof(double) * 8 * Mp, st));
    FCK(cudaMemsetAsync(f->cv.R, 0, sizeof(double) * Mp * Mp, st));
    FCK(cudaMemsetAsync(f->cv.H, 0, sizeof(double) * Mp * Mp, st));
    if (!noise) {   // Dp = dK_uu K_uu^-1
        FCK(gram_grad_full_launch(eu->prog, eu->x, d, d, M, Mp, param, f->cv.Duu, Mp, st, &eu->launches));
        FCK(gemm_whole(f->eu, bDuu, bufG(eu), f->cv.Dp, Mp, Mp, Mp, Mp, 1.0, 0.0));
    }
    // pass 1: Delta, R, H, K_uf alpha, G'alpha, K_uf L^-1 Delta alpha
    for (int64_t r0 = 0; r0 < N; r0 += Nc) {
        const int64_t nc = std::min(Nc, N - r0);
        const double* xr = f->data.x + r0 * d;
        FCK(fitc_kfu(f, xr, nc));                                                                     // bufA = K_fu
        if (!noise) {
            FCK(crossgram_grad_launch(eu->prog, xr, d, nc, Nc, eu->x, d, M, Mp, d, param, f->cv.G, Mp, st, &eu->launches));
            if (kind == 0) FCK(gemm_whole(f->eu, bA, bufG(eu), f->stage.bufB, Mp, Nc, Mp, Mp, 1.0, 0.0));     // bufB = C (Nc x Mpad)
            FCK(gemm_whole(f->eu, bA, bDp, f->cv.G, Mp, Nc, Mp, Mp, -0.5, 1.0, f->cv.Gt, Nc));              // G and G'
        }
        FCK(fitc_cv_delta_launch(kind, eu->prog, xr, d, param, f->cv.G, f->stage.bufB, Mp, Mp, nc, Nc, f->cv.alpha + r0, f->cv.del + r0,
                                 f->cv.da, st, &eu->launches));
        FCK(fitc_kuf(f, xr, nc));                                                                     // bufB = K_uf
        FCK(rowdot_launch(f->stage.bufB, Nc, f->cv.alpha + r0, M, Nc, tmp, st, &eu->launches));
        FCK(ew_launch(2, M, kta, tmp, nullptr, nullptr, 0.0, st, &eu->launches));
        FCK(colscale_launch(f->stage.bufB, Nc, Mp, nc, f->cv.ilam + r0, st, &eu->launches));                // K_uf L^-1
        FCK(rowdot_launch(f->stage.bufB, Nc, f->cv.da, M, Nc, tmp, st, &eu->launches));
        FCK(ew_launch(2, M, uD, tmp, nullptr, nullptr, 0.0, st, &eu->launches));
        if (!noise) {
            FCK(rowdot_launch(f->cv.Gt, Nc, f->cv.alpha + r0, M, Nc, tmp, st, &eu->launches));
            FCK(ew_launch(2, M, gta, tmp, nullptr, nullptr, 0.0, st, &eu->launches));
            FCK(gemm_whole(f->eu, bB, bGt, f->cv.R, Mp, Mp, Mp, Nc, 1.0, 1.0));                           // R += K_uf L^-1 G
        }
        if (kind != 1) {                                                                              // H += K_uf L^-1 Delta L^-1 K_fu
            FCK(cudaMemcpyAsync(f->cv.Gt, f->stage.bufB, sizeof(double) * Mp * Nc, cudaMemcpyDeviceToDevice, st));
            FCK(colscale_launch(f->cv.Gt, Nc, Mp, nc, f->cv.del + r0, st, &eu->launches));
            FCK(gemm_whole(f->eu, bB, bGt, f->cv.H, Mp, Mp, Mp, Nc, 1.0, 1.0));
        }
    }
    FCK(rowdot_launch(eu->G, eu->ld, kta, M, Mp, beta, st, &eu->launches));                         // beta = K_uu^-1 K_uf alpha
    FCK(rowdot_launch(f->cv.R, Mp, beta, M, Mp, rb, st, &eu->launches));
    FCK(fitc_cv_wvec_launch(M, w, gta, uD, rb, st, &eu->launches));
    FCK(fitc_cv_qs_launch(f->cv.Q, f->cv.H, f->cv.R, Mp, Mp, st, &eu->launches));
    // pass 2: the two N-vectors
    for (int64_t r0 = 0; r0 < N; r0 += Nc) {
        const int64_t nc = std::min(Nc, N - r0);
        const double* xr = f->data.x + r0 * d;
        FCK(fitc_kfu(f, xr, nc));
        if (!noise) {
            FCK(crossgram_grad_launch(eu->prog, xr, d, nc, Nc, eu->x, d, M, Mp, d, param, f->cv.G, Mp, st, &eu->launches));
            FCK(gemm_whole(f->eu, bA, bDp, f->cv.G, Mp, Nc, Mp, Mp, -0.5, 1.0));
        }
        FCK(gemm_whole(f->eu, bA, bufG(es), f->cv.Ch, Mp, Nc, Mp, Mp, 1.0, 0.0));
        FCK(scale_launch(1, f->cv.Ch, Mp, nc, Mp, f->data.lam + r0, st, &eu->launches));                  // Ch = L^-1 K_fu S^-1
        FCK(gemm_whole(f->eu, bCh, bQ, f->cv.P, Mp, Nc, Mp, Mp, 1.0, 0.0));                                // Ch Q
        FCK(fitc_cv_rows_launch(noise ? nullptr : f->cv.G.data(), f->cv.Ch, f->stage.bufA, f->cv.P, Mp, nc, Mp, f->data.lam + r0, f->cv.del + r0,
                                f->cv.alpha + r0, beta, w, f->cv.za + r0, f->cv.dg + r0, st, &eu->launches));
    }
    FCK(cudaMemcpyAsync(Zj_alpha, f->cv.za, sizeof(double) * N, cudaMemcpyDeviceToHost, st));
    FCK(cudaMemcpyAsync(diag_ZjSinv, f->cv.dg, sizeof(double) * N, cudaMemcpyDeviceToHost, st));
    FCK(cudaStreamSynchronize(st));
    f->cv_param = param;
    f->cv.m_ok = true;
    return GPB200_OK;
}

int gpb200_fitc_cv_block(gpb200_fitc* f, int32_t which, int64_t nV, const int64_t* idx, double* out) {
    if (!f || !idx || !out) return GPB200_EINVAL;
    TRY(fitc_cv_check(f, "fitc_cv_block"));
    if (which != 0 && which != 1) return fail(f, GPB200_EINVAL, "fitc_cv_block: which must be 0 (Sigma^-1) or 1 (the last cv_param's M_j)");
    if (nV < 1 || nV > f->Nc)
        return fail(f, GPB200_EINVAL, "fitc_cv_block: nV must lie in 1.." + std::to_string(f->Nc) + " (one staging chunk)");
    for (int64_t r = 0; r < nV; ++r)
        if (idx[r] < 0 || idx[r] >= f->N) return fail(f, GPB200_EINVAL, "fitc_cv_block: index out of range");
    if (which == 1 && !f->cv.m_ok) return fail(f, GPB200_ESTATE, "fitc_cv_block: which = 1 needs a fitc_cv_param since the last factorize");
    FCK(cudaSetDevice(f->device));
    TRY(fitc_cv_prepare(f));
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int64_t Mp = f->Mpad, M = f->M;
    const int d = f->d;
    const int64_t nVp = (nV + TILE - 1) / TILE * TILE;
    FCK(f->cv.out.ensure((size_t)nVp * nVp));
    const GemmBuf bA = gbuf(eu, f->stage.bufA, f->stage.mapA, Mp), bB2 = gbuf(eu, f->stage.bufB, f->stage.mapB2, Mp);
    const GemmBuf bCh = gbuf(eu, f->cv.Ch, f->cv.mapCh, Mp), bP = gbuf(eu, f->cv.P, f->cv.mapP, Mp);
    const GemmBuf bDp = gbuf(eu, f->cv.Dp, f->cv.mapDp, Mp), bQ = gbuf(eu, f->cv.Q, f->cv.mapQ, Mp);
    FCK(cudaMemcpyAsync(f->cv.idx, idx, sizeof(long long) * nV, cudaMemcpyHostToDevice, st));
    FCK(fitc_cv_gather_launch(nV, f->cv.idx, f->data.x, d, d, f->cv.xs, f->data.lam, f->cv.lamV, which == 1 ? f->cv.del.data() : nullptr, f->cv.delV,
                              st, &eu->launches));
    FCK(crossgram_launch(eu->prog, f->cv.xs, d, nV, nVp, eu->x, d, M, Mp, d, f->stage.bufA, Mp, st, &eu->launches));   // K_V
    FCK(gemm_whole(f->eu, bA, bufG(es), f->cv.Ch, Mp, nVp, Mp, Mp, 1.0, 0.0));
    FCK(scale_launch(1, f->cv.Ch, Mp, nV, Mp, f->cv.lamV, st, &eu->launches));                       // Ch_V
    if (which == 0) {   // Sigma^-1[V,V] = diag(1/L_V) - Ch_V (L_V^-1 K_V)'
        FCK(cudaMemcpyAsync(f->stage.bufB, f->stage.bufA, sizeof(double) * nVp * Mp, cudaMemcpyDeviceToDevice, st));
        FCK(scale_launch(1, f->stage.bufB, Mp, nV, Mp, f->cv.lamV, st, &eu->launches));
        FCK(gemm_whole(f->eu, bCh, bB2, f->cv.out, nVp, nVp, nVp, Mp, -1.0, 0.0));
    } else {            // (Sigma^-1 dSigma_j Sigma^-1)[V,V] = diag(Delta_V / L_V^2) + E_V Ch_V' + Ch_V E_V'
        const bool noise = f->cv_param < 0;
        if (!noise) {
            FCK(crossgram_grad_launch(eu->prog, f->cv.xs, d, nV, nVp, eu->x, d, M, Mp, d, f->cv_param, f->cv.G, Mp, st, &eu->launches));
            FCK(gemm_whole(f->eu, bA, bDp, f->cv.G, Mp, nVp, Mp, Mp, -0.5, 1.0));
        }
        FCK(gemm_whole(f->eu, bCh, bQ, f->cv.P, Mp, nVp, Mp, Mp, 0.5, 0.0));
        FCK(fitc_cv_eblock_launch(f->cv.P, noise ? nullptr : f->cv.G.data(), f->stage.bufA, Mp, nV, Mp, f->cv.lamV, f->cv.delV, st, &eu->launches));
        FCK(gemm_whole(f->eu, bP, bCh, f->cv.out, nVp, nVp, nVp, Mp, 1.0, 0.0));
        FCK(gemm_whole(f->eu, bCh, bP, f->cv.out, nVp, nVp, nVp, Mp, 1.0, 1.0));
    }
    FCK(fitc_cv_diag_launch(f->cv.out, nVp, nV, which, f->cv.lamV, f->cv.delV, st, &eu->launches));
    FCK(cudaMemcpy2DAsync(out, sizeof(double) * nV, f->cv.out, sizeof(double) * nVp, sizeof(double) * nV, nV, cudaMemcpyDeviceToHost, st));
    FCK(cudaStreamSynchronize(st));
    return GPB200_OK;
}

// rand(gp, X, n) (src/GP.jl:120-146) with a sparse cK: Sigma* is the covariance predict_cov (modes 0-2) or predict_fsa
// (mode 3) returns, built on the device and kept there; make_posdef!, the Cholesky and unwhiten! are gpb200_rand's
// (rand_from_cov on eu, whose Ms x Ms sub-engine shares the handle's stream).  The likelihood, gradient, prediction and
// cross-validation state is only read.
int gpb200_fitc_rand(gpb200_fitc* f, int64_t Ms, const double* xs, int64_t ldxs, const int64_t* block_of, int64_t nsamp,
                     const double* z, double nugget, double* mu_minus_mean, double* samples) {
    if (!f) return GPB200_EINVAL;
    if (Ms <= 0 || nsamp <= 0 || !xs || ldxs < f->d || !z || !mu_minus_mean || !samples) {
        return fail(f, GPB200_EINVAL, "fitc_rand: bad Ms, nsamp, xs, ldxs, z, mu or samples");
    }
    if (!(nugget >= 0.0)) return fail(f, GPB200_EINVAL, "fitc_rand: nugget must be >= 0");
    if ((f->mode == 3) != (block_of != nullptr)) {
        return fail(f, GPB200_EINVAL, "fitc_rand: block_of is required in FSA mode (3) and must be NULL otherwise");
    }
    if (!f->factored || !(f->alpha_ready || f->u_ready)) return fail(f, GPB200_ESTATE, "fitc_rand: factorize and mll first");
    if (f->mode != 3 && Ms > f->Nc) return fail(f, GPB200_EINVAL, "fitc_rand: too many test points for one staging chunk");
    FCK(cudaSetDevice(f->device));
    gpb200_handle* eu = f->eu;
    cudaEvent_t ev_start = eu->ev4;                      // rand_from_cov records ev0 .. ev3
    FCK(cudaEventRecord(ev_start, eu->st));
    DevPrediction p;
    if (f->mode == 3) TRY(fsa_predict(f, Ms, xs, ldxs, block_of, mu_minus_mean, nullptr, CovDest::device, nullptr, nullptr, nullptr, &p));
    else TRY(fitc_cov_build(f, Ms, xs, ldxs, mu_minus_mean, &p));
    FSUB(rand_from_cov(eu, Ms, p.cov, p.ldc, p.mu, nsamp, z, nugget, samples), eu);
    f->rand_ms[0] = ev_ms(ev_start, eu->ev0);
    f->rand_ms[1] = ev_ms(eu->ev0, eu->ev1);
    f->rand_ms[2] = ev_ms(eu->ev3, eu->ev2);
    return GPB200_OK;
}

int gpb200_fitc_get_timings(gpb200_fitc* f, double* ms, int32_t n) {
    if (!f || !ms || n < 0) return GPB200_EINVAL;
    for (int32_t i = 0; i < n && i < 3; ++i) ms[i] = f->rand_ms[i];
    for (int32_t i = 3; i < n && i < 7; ++i) ms[i] = f->fsag_ms[i - 3];
    for (int32_t i = 7; i < n && i < 9; ++i) ms[i] = f->xu_ms[i - 7];
    for (int32_t i = 9; i < n && i < 11; ++i) ms[i] = f->x_ms[i - 9];
    return GPB200_OK;
}

int gpb200_fitc_set_mode(gpb200_fitc* f, int mode) {
    if (!f || mode < 0 || mode > 3) return GPB200_EINVAL;
    f->mode = mode; fitc_invalidate(f);
    return GPB200_OK;
}

int64_t gpb200_fitc_launch_count(gpb200_fitc* f) { return f ? f->eu->launches + f->es->launches : 0; }
}  // extern "C"
