/*
 * gpb200.h -- C ABI of libgpb200.so: the H100-native exact-GP hot path behind the
 * GaussianProcesses.jl `CovarianceStrategy` seam.
 *
 * There is no FFI in the reference (pure Julia); the boundary this library slots into is the
 * reference's own strategy-dispatch API (src/GP.jl:10 `abstract type CovarianceStrategy`).  Each
 * entry point below names the reference method (file:line under /root/reference) it replaces;
 * INTEGRATION.md shows the Julia `ccall` shim (`B200Covariance <: CovarianceStrategy`) and the
 * Python ctypes binding that drive exactly these symbols.
 *
 * Conventions
 *   - all matrices FP64.  `x` is Julia's d x N column-major Matrix{Float64} (== N x d row-major,
 *     one observation per column), passed with its leading dimension `ldx` (>= d).
 *   - caller owns every host buffer for the duration of the call only; the library owns all
 *     device memory behind the opaque handle.  Calls are synchronous.
 *   - return value: 0 OK;  k > 0 = LAPACK-style "leading minor k is not positive definite"
 *     (shim throws LinearAlgebra.PosDefException(k), cf. src/GP.jl:110, src/optimize.jl:46-61);
 *     GPB200_EINVAL (<0) invalid argument (-> ArgumentError);  GPB200_ECUDA / GPB200_ENCCL
 *     runtime failure, message via gpb200_last_error().  A failed factorisation leaves the
 *     handle reusable with new hyper-parameters.
 *   - one handle must not be used from two threads at once; distinct handles may be.
 *   - there is NO CPU fallback: without a CUDA device gpb200_create fails with GPB200_ECUDA.
 */
#ifndef GPB200_H
#define GPB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct gpb200_handle gpb200_handle;

#define GPB200_OK        0
#define GPB200_EINVAL   (-1)
#define GPB200_ECUDA    (-2)
#define GPB200_ENCCL    (-3)
#define GPB200_ESTATE   (-4)   /* call order violated (e.g. solve before factorize) */

/* ---- kernel program: post-order (RPN) list of ops; 6 int32 per op ------------------------
 *   {opcode, theta_off, n_theta, dims_off, n_dims, extra}
 * leaves read theta[theta_off .. theta_off+n_theta) (log-scale, exactly get_params(kernel) order,
 * src/kernels/pair_kernel.jl:15, src/common.jl:98-104) and the active input dimensions
 * dims[dims_off .. dims_off+n_dims) (0-based; `Masked`, src/kernels/masked_kernel.jl:23, is
 * resolved into this list by the shim).  `extra` = polynomial degree for GPB200_OP_POLY.
 * SUM / PROD pop two values (src/kernels/sum_kernel.jl:15-16, prod_kernel.jl:14-15).
 * FixedKernel (src/kernels/fixed_kernel.jl:64-69) is resolved in the shim: pass the full
 * parameter vector of the wrapped kernel, select gradient entries `free` on the host.        */
#define GPB200_OP_SE_ISO     1   /* src/kernels/se_iso.jl:39-50     theta = [ll, lsigma]          */
#define GPB200_OP_SE_ARD     2   /* src/kernels/se_ard.jl:43-50     theta = [ll_1..ll_nd, lsigma] */
#define GPB200_OP_MAT12_ISO  3   /* src/kernels/mat12_iso.jl:41-43                                */
#define GPB200_OP_MAT32_ISO  4   /* src/kernels/mat32_iso.jl:41-45                                */
#define GPB200_OP_MAT52_ISO  5   /* src/kernels/mat52_iso.jl:40-44                                */
#define GPB200_OP_MAT12_ARD  6   /* src/kernels/mat12_ard.jl:43-45, mat.jl:5-18                   */
#define GPB200_OP_MAT32_ARD  7   /* src/kernels/mat32_ard.jl:43-46                                */
#define GPB200_OP_MAT52_ARD  8   /* src/kernels/mat52_ard.jl:43-47                                */
#define GPB200_OP_RQ_ISO     9   /* src/kernels/rq_iso.jl:44-52     theta = [ll, lsigma, lalpha]  */
#define GPB200_OP_RQ_ARD    10   /* src/kernels/rq_ard.jl:47-54     theta = [ll.., lsigma, lalpha]*/
#define GPB200_OP_PERIODIC  11   /* src/kernels/periodic.jl:45-51   theta = [ll, lsigma, lp]      */
#define GPB200_OP_LIN_ISO   12   /* src/kernels/lin_iso.jl:42,71    theta = [ll]                  */
#define GPB200_OP_LIN_ARD   13   /* src/kernels/lin_ard.jl:69-92    theta = [ll_1..ll_nd]         */
#define GPB200_OP_POLY      14   /* src/kernels/poly.jl:44,69-70    theta = [lc, lsigma]          */
#define GPB200_OP_NOISE     15   /* src/kernels/noise.jl:31-52      theta = [lsigma]              */
#define GPB200_OP_CONST     16   /* src/kernels/const.jl:41         theta = [lsigma]              */
#define GPB200_OP_SUM       32
#define GPB200_OP_PROD      33

#define GPB200_MAX_OPS     16
#define GPB200_MAX_THETA   96
#define GPB200_MAX_DIMS   128
#define GPB200_OP_STRIDE    6

/* ---- lifetime ------------------------------------------------------------------------- */
/* replaces alloc_cK(covstrat, nobs) (src/GP.jl:14-20): creates the engine on CUDA device
 * `device`; device buffers are sized at gpb200_set_data.                                   */
int  gpb200_create(gpb200_handle** out, int device);
/* Julia finalizer on B200PDMat */
void gpb200_destroy(gpb200_handle* h);
/* message of the last failure on this handle (h == NULL: last create failure) */
const char* gpb200_last_error(gpb200_handle* h);
int  gpb200_version(void);

/* ---- data + model ---------------------------------------------------------------------- */
/* GPE ctor / fit! (src/GPE.jl:63-69, 128-136): upload the d x N inputs once; hyper-parameter
 * independent.  No N x N distance matrix is precomputed (cf. IsotropicData,
 * src/kernels/stationary.jl:34-40): distances are recomputed from x inside the Gram kernel. */
int  gpb200_set_data(gpb200_handle* h, int64_t N, int32_t d, const double* x, int64_t ldx);
/* flattened kernel tree (see opcodes above) */
int  gpb200_set_kernel(gpb200_handle* h, int32_t n_ops, const int32_t* ops,
                       int32_t n_dims, const int32_t* dims, int32_t n_theta);

/* ---- update_cK! (src/GPE.jl:169-186) + make_posdef! (src/GP.jl:101-112) ------------------
 * Gram build cov!(...) (src/kernels/kernels.jl:39-50) with K_ii += exp(2*log_noise) (n_noise==1)
 * or += exp(2*log_noise[i]) (n_noise==N), plus `extra_nugget`, then the Cholesky factorisation.
 * Returns k>0 if the leading minor k is not positive definite.                              */
int  gpb200_factorize(gpb200_handle* h, const double* theta, const double* log_noise,
                      int64_t n_noise, double extra_nugget);
/* logdet(cK) (src/GPE.jl:210; PDMats: 2*sum(log(diag(U)))) */
int  gpb200_logdet(gpb200_handle* h, double* logdet);
/* cK \ rhs (src/GPE.jl:208; PDMats `\` == dpotrs): out = K_y^-1 rhs, both length N on host */
int  gpb200_solve(gpb200_handle* h, const double* rhs, double* out);
/* update_mll! body (src/GPE.jl:206-210): alpha = K_y^-1 r, mll = -(r'alpha + logdet + N log 2pi)/2;
 * alpha stays resident on the device for grad/predict.                                      */
int  gpb200_mll(gpb200_handle* h, const double* y_minus_mean, double* alpha, double* mll);

/* ---- gradient -------------------------------------------------------------------------- */
/* precompute!(precomp, gp) -> get_ααinvcKI! (src/GPE.jl:151-164, 262-264): builds K_y^-1 from
 * the factor (triangular inverse + W'W, N^3*2/3 flop instead of the reference's 2N^3 potrs on
 * the identity).  The factor is kept: predict after grad needs no refactorisation.           */
int  gpb200_grad_prepare(gpb200_handle* h);
/* dmll_kern! (src/GPE.jl:219-241) + dmll_noise's tr(A) (src/GPE.jl:273-275), fused:
 * dmll_kernel[p] = 1/2 sum_ij A_ij dK_ij/dtheta_p, A = alpha alpha' - K_y^-1;  *trA = tr(A).
 * `alpha` may be NULL to use the alpha left resident by gpb200_mll.                          */
int  gpb200_grad_kernel(gpb200_handle* h, const double* alpha, double* dmll_kernel, double* trA);
/* dmll/dX (N x d, point-major == Julia's d x N column-major) of the kernel part: sum_j A_ij dk(x_i, x_j)/dx_i.
 * After gpb200_grad_prepare: A = alpha alpha' - K_y^-1 (alpha as in gpb200_grad_kernel: given, or the resident one).
 * After gpb200_gpa_grad with dll_kernel != NULL: A = S (alpha must be NULL).  Otherwise GPB200_ESTATE.
 * Collective on multi-rank and row-sharded handles; every rank returns the full array.
 * Not in the reference (which differentiates its Julia cov! automatically).  The noise terms do not depend on x; the mean's
 * part alpha_i dm(x_i)/dx_i (GPA: (dl_df)_i dm(x_i)/dx_i) is the caller's.  At coincident inputs the stationary kernels
 * contribute the limit of their derivative (0), as in gpb200_predict_grad.  Each stored entry of A's lower triangle is read
 * twice, nothing else of G; the tile rows are split over the ranks as by gpb200_grad_kernel and the N x d partials are
 * summed once.  Sums run in a fixed order: repeated calls are bitwise equal.  GPB200_EINVAL for a NULL dmll_x or an alpha
 * in the S state.  Reads F, G and alpha only (a given alpha is not kept): every later call behaves as without this one.
 * Device memory grows by (N + N d) doubles on the first call (in-process groups: + nranks N d for the sum).  Timing slot 16. */
int  gpb200_grad_inputs(gpb200_handle* h, const double* alpha, double* dmll_x);

/* ---- predictMVN / predict_f (src/GP.jl:25-79) ---------------------------------------------
 * xs: d x M column-major test inputs (leading dim ldxs).  mu_minus_mean[M] = K*' alpha;
 * var[M] (may be NULL) = k** - |L^-1 k*|^2, NOT clamped (the shim applies max(.,0) as
 * src/GP.jl:75 does only on the diagonal path); cov[M*M] (may be NULL) = K** - V'V, symmetric.
 * Batched: one cross-Gram + one blocked triangular solve for all M points (the reference loops
 * over test points, src/GP.jl:72-76).                                                       */
int  gpb200_predict(gpb200_handle* h, int64_t M, const double* xs, int64_t ldxs,
                    const double* alpha, double* mu_minus_mean, double* var, double* cov);

/* Predictive gradients with respect to the test inputs (predict_f with ForwardDiff.Dual inputs): mu_minus_mean[M] and var[M]
 * bitwise equal to gpb200_predict's on the same handle, and dmu / dvar (M x d point-major == Julia's d x M column-major)
 *   dmu[m, p]  = sum_i dk(x*_m, x_i)/dx*_{m,p} alpha_i                     (the mean's own gradient is the caller's)
 *   dvar[m, p] = 2 dk(x*_m, x*_m)/dx*_{m,p} - 2 sum_i dk(x*_m, x_i)/dx*_{m,p} (K^-1 k*_m)_i     (var NOT clamped)
 * var and dvar are given together or both NULL (then only the cross-Gram and the contraction run, no solve).  Where x*_m
 * coincides with a training input the stationary kernels contribute the limit of their derivative (0) rather than the NaN
 * of differentiating through sqrt(0).  Single-GPU handles only (GPB200_EINVAL otherwise); chunked as gpb200_predict.
 * Uses F's strict-upper tiles as scratch (they hold L' during the call).                                                 */
int  gpb200_predict_grad(gpb200_handle* h, int64_t M, const double* xs, int64_t ldxs, const double* alpha,
                         double* mu_minus_mean, double* var, double* dmu, double* dvar);

/* rand(gp, X, n) (src/GP.jl:120-146): n posterior draws at the M test points, on the device: predictMVN's full covariance,
 * make_posdef!(Sigma; nugget) (Cholesky of the M x M matrix), unwhiten!(Sigma, Z) and + mu.  z and samples are M x nsamp
 * column-major (Julia `randn(M, n)` / the returned matrix); mu_minus_mean[M] as in gpb200_predict (the shim adds mean(x*) to
 * it and to every draw).  Returns k > 0 if Sigma + nugget I is not positive definite (PosDefException).               */
int  gpb200_rand(gpb200_handle* h, int64_t M, const double* xs, int64_t ldxs, const double* alpha, int64_t nsamp,
                 const double* z, double nugget, double* mu_minus_mean, double* samples);

/* append!(gp::ElasticGPE, x, y) (src/GPEelastic.jl:13-22): k more observations (xnew: d x k column-major) with UNCHANGED
 * hyper-parameters; the factor is extended in place (rows from the first touched tile on are rebuilt: O(k N^2)), alpha / mll are
 * then refreshed with gpb200_mll on the longer y.  Needs room reserved by option "capacity" (ElasticGPE's capacity) before
 * gpb200_set_data; GPB200_EINVAL when the capacity is exceeded (the shim refits, like ElasticPDMats.resize!).
 * Row-sharded handles extend the distributed factor: an in-process group through its leader, NCCL ranks (option "shard" = 1)
 * collectively; the rebuild starts at the ownership block of the first touched tile.  Replicated multi-rank handles and
 * vector logNoise return GPB200_ESTATE; a non-positive-definite extension returns the leading minor and clears the factor. */
int  gpb200_append(gpb200_handle* h, int64_t k, const double* xnew, int64_t ldx);

/* ---- GPA: GP with a non-Gaussian likelihood (src/GPA.jl), latent f = L v + mu over K = L L' ---------------------------------
 * The likelihood stays on the host (O(N)); the handle supplies the O(N^2) / O(N^3) pieces.  Call gpb200_factorize first
 * (update_cK!(::GPA), GPA.jl:111-114: log_noise = -20).  Single GPU: GPB200_EINVAL on multi-rank, row-sharded and grouped
 * handles; GPB200_ESTATE before factorize.                                                                                  */
/* unwhiten(cK, v) (src/GPA.jl:106,125,159,294): f[N] = L v, L the factor of the last gpb200_factorize */
int  gpb200_unwhiten(gpb200_handle* h, const double* v, double* f);
/* GPA gradient (src/GPA.jl:164-173,200; src/chol_utils.jl:15-39), after gpb200_factorize:
 * dll_process[N] = L' dl_df (may be NULL); dll_kernel[P] = dll_kern! for Lbar = tril(dl_df v') (may be NULL: no O(N^3) work).
 * The kernel gradient is 1/2 sum_ij S_ij dK_ij/dtheta_p with S = W' M_s W, W = L^-1, M_s[i,j] = u[max(i,j)] v[min(i,j)],
 * u = L' dl_df: the inverse merges, two scans and one triangular NT GEMM (N^3/3 + N^3/3 flop) instead of the reference's
 * level-2 reverse pass.  It overwrites K_y^-1 and the resident alpha: grad_kernel / cv_* then need grad_prepare / mll again
 * (GPB200_ESTATE otherwise).  The factor, logdet, solve, mll, predict, rand and append are unaffected.                   */
int  gpb200_gpa_grad(gpb200_handle* h, const double* v, const double* dl_df, double* dll_process, double* dll_kernel);

/* ---- cross-validation on the resident inverse (src/crossvalidation.jl; after gpb200_grad_prepare) ------------------------
 * Per hyper-parameter the reference forms Z_j = inv(Sigma) dK_j and Z_j inv(Sigma) as host matrices (crossvalidation.jl:86-108,
 * 270-283).  gpb200_cv_param does the two N^3 products on the device and returns the two vectors the LOO formulas need:
 * Zj_alpha[N] = Z_j alpha and diag_ZjSinv[N] = diag(Z_j inv(Sigma)); `param` indexes the kernel's full parameter vector, -1 is the
 * noise variance (Z = inv(Sigma), crossvalidation.jl:124-126).  M_j = Z_j inv(Sigma) stays resident for gpb200_cv_block.
 * Row-sharded handles (in-process groups, or NCCL ranks with option "shard" = 1) run the same steps over the ranks: every rank
 * keeps its own rows of Z_j and of the lower triangle of M_j (3 N^3 flop split over the ranks instead of 4 N^3); call the
 * leader of a group.  Replicated multi-rank handles return GPB200_ESTATE.  Repeated calls return bitwise equal vectors.      */
int  gpb200_cv_param(gpb200_handle* h, int32_t param, const double* alpha, double* Zj_alpha, double* diag_ZjSinv);
/* principal sub-matrix on the index set idx[nV] (0-based) of inv(Sigma) (which = 0) or of the last M_j (which = 1), row-major
 * nV x nV: `Matrix(invΣ)[V,V]` / `ZjΣinv[V,V]` of predict_CVfold / gradient_fold (crossvalidation.jl:180-191, 248-262).
 * which = 1 before a gpb200_cv_param since the last factorize / append / grad_prepare: GPB200_ESTATE.  Row-sharded handles read
 * every entry from the stored lower triangle and sum the ranks' pieces: the block is exactly symmetric.                    */
int  gpb200_cv_block(gpb200_handle* h, int32_t which, int64_t nV, const int64_t* idx, double* out);

/* ---- debug / introspection (Base.Matrix(::P), mat(::P), tests) ----------------------------- */
int  gpb200_get_gram(gpb200_handle* h, double* K);        /* N x N, K_y rebuilt from x, theta   */
int  gpb200_get_factor(gpb200_handle* h, double* U);      /* N x N column-major upper U, K_y=U'U */
int  gpb200_get_inverse(gpb200_handle* h, double* Kinv);  /* N x N, after gpb200_grad_prepare    */
/* diag(K_y^-1)[N] after gpb200_grad_prepare: all predict_LOO / logp_LOO need besides alpha
 * (src/crossvalidation.jl:8-13, 37-49: sigma_i^2 = 1/[K^-1]_ii, mu_i = y_i - alpha_i sigma_i^2).  Row-sharded handles copy
 * the own diagonal entries and all-gather them; replicated multi-rank handles return GPB200_ESTATE.                         */
int  gpb200_get_inverse_diag(gpb200_handle* h, double* diag);
/* per-phase device times (ms) of the last calls:
 * [0] gram  [1] cholesky  [2] solve+mll  [3] inverse (trtri+lauum; gpb200_gpa_grad: the merges only)  [4] trace  [5] predict
 * [9] gpb200_gpa_grad's scans  [10] its S = W'Z GEMM
 * gpb200_predict_grad (summed over chunks): [11] cross-Gram + mean  [12] V' = K*' L^-T + variance  [13] L' into F's upper
 * tiles  [14] W' = V' L^-1  [15] gradient contraction
 * [16] gpb200_grad_inputs (contraction and, on several ranks, the sum of the partials)
 * with option "profile"=1, accumulated since the option was set:
 * [6] number of DMMA GEMM launches  [7] sum of their device durations (ms, CUDA events around
 * every launch)  [8] FP64 flops those launches executed (tile-granular)                       */
int  gpb200_get_timings(gpb200_handle* h, double* ms, int32_t n);   /* writes min(n, 17) entries */
/* number of kernels enqueued by calls on this handle since creation (gpb200_rand includes its M x M sub-engine's
 * Cholesky); cudaMemsetAsync and copies are not counted */
int64_t gpb200_launch_count(gpb200_handle* h);
/* bytes of device memory the library's own buffers hold right now, over every handle of the process (diagnostics; the
 * virtual-memory ranges of row-sharded storage and IPC peer mappings are not counted) */
int64_t gpb200_device_bytes(void);
/* tuning knobs (string key):
 *   "nb"         outer Cholesky block: 0 (default) = fully recursive, else 128*2^k <= 4096 (right-looking panels)
 *   "gemm"       0 = TMA/mbarrier DMMA kernel (default), 1 = simple-loader kernel (bring-up / cross-check)
 *   "lookahead"  1 (default) = next diagonal tile factored on a side stream behind the Schur update
 *   "trsv_fused" 1 (default) = single-launch flag-synchronised triangular solves, 0 = one launch per block step
 *   "profile"    1 = CUDA events around every GEMM launch (see gpb200_get_timings)
 *   "dist_nb"    multi-GPU: width of an owned block column, 0 = auto (~N/(8*ranks))
 *   "p2p"        multi-GPU: 1 = fused panel push over peer memory (after gpb200_ipc_import), 0 = NCCL broadcast
 *   "gram_fast"  1 (default) = TMA-staged SEIso Gram / trace kernels (gram_fast.cu) when the kernel is one SEIso leaf over
 *                <= 8 dimensions, 0 = always the generic kernel-program kernels (cross-check)
 *   "capacity"   rows reserved by the next gpb200_set_data (>= N) so that gpb200_append can extend the factor in place
 *   "shard"      multi-GPU storage of the two N x N buffers: 1 = row-sharded (each rank maps only its own block rows),
 *                0 = replicated, -1 (default) = sharded only when the replicated form would not fit the device
 *   "shard_rb"   row-sharded ownership block in 128-row tiles (panel width 128*rb): 0 auto, 1, 2, 4, 8
 * Returns GPB200_EINVAL for unknown keys or values.                                           */
int  gpb200_set_option(gpb200_handle* h, const char* key, int64_t value);

/* run all work of this handle on the caller's CUDA stream (cudaStream_t; NULL = a private
 * stream again), so that the caller's events bracket it (bench.py: torch.cuda.Event).         */
int  gpb200_set_stream(gpb200_handle* h, void* cuda_stream);
/* FP64 roofline denominators measured on this device: DMMA.16x8x16 (mma.sync f64, the FP64 tensor
 * path on sm_90a, the shape the GEMM issues) and DFMA issue rates, TFLOP/s.                  */
int  gpb200_fp64_peak(gpb200_handle* h, double* tflops_dmma, double* tflops_dfma);

/* ---- raw kernels exposed for the parity tests and the roofline bench ----------------------
 * C[M x N] = alpha * A[M x K] * B[N x K]' + beta * C   (all row-major, device pointers,
 * M,N multiples of 128, K multiple of 16, leading dims multiples of 2); runs the same DMMA
 * kernel the factorisation uses.  `impl` 0 = TMA/mbarrier kernel, 1 = simple kernel.
 * Returns the device time of `reps` launches in *ms (reps>=1).                               */
int  gpb200_dgemm_nt_device(gpb200_handle* h, int impl, int64_t M, int64_t N, int64_t K,
                            double alpha, const double* dA, int64_t lda,
                            const double* dB, int64_t ldb, double beta,
                            double* dC, int64_t ldc, int lower_only, int reps, double* ms);
/* One launch of the NT GEMM from a complete descriptor (csrc/gemm_nt.cuh GemmDesc), synchronous.  desc holds
 * GPB200_GEMM_DESC_LEN int64 (n must equal it):
 *   [0] flags  [1] M  [2] N  [3] K  [4] batch  [5] zstep  [6] m_lim  [7] n_lim  [8] k_lim  [9] klo_off
 *   [10] bm_mod  [11] bm_rem  [12] bn_mod  [13] bn_rem  [14] bm_div  [15] bm_off  [16] bn_div  [17] bn_off  [18] n_peer
 *   [19] A.row0  [20] A.col0  [21] B.row0  [22] B.col0  [23] c_row0  [24] c_col0  [25] ct_row0  [26] ct_col0
 *   [27 + 4 b ..] buffer b = (device pointer, rows, cols, ld) for b = 0 A, 1 A.sub, 2 B, 3 B.sub, 4 C, 5 Ct, 6..12 peers;
 *                 pointer 0 = absent.  A, A.sub, B, B.sub get TMA descriptors as the engine builds them (whole buffer,
 *                 16 x 128 box, 128B swizzle; a sub buffer is [Npad x 128] with ld 128); rows = cols = 0 passes the
 *                 buffer without one.
 * GPB200_EINVAL, nothing launched: M, N not multiples of 128, K not a multiple of 16, an odd ld or unaligned pointer,
 * impl 0 with a buffer that has no descriptor, and every descriptor gemm_nt_launch rejects (LOWER_ONLY with tm < tn,
 * with n_peer > 0 or with Ct).                                                                                       */
#define GPB200_GEMM_DESC_LEN 79
int  gpb200_gemm_nt_desc(gpb200_handle* h, int impl, const int64_t* desc, int32_t n, double alpha, double beta);
/* One launch of the grouped tile GEMM of the FSA strategy (csrc/fsa.cuh FsaGemmItem) over n items, synchronous:
 * items[8 i ..] = (C, A, B, ldc, lda, ldb, K, lower), alpha_beta[2 i ..] = (alpha, beta).                            */
int  gpb200_fsa_gemm_items(gpb200_handle* h, const int64_t* items, const double* alpha_beta, int32_t n);
/* One launch of the 128 x 128 diagonal-tile leaf (csrc/potrf_base.cuh), synchronous; *info = the device info word
 * (INT_MAX: every pivot positive).
 *   mode 0 (potrf128_launch), n = 39: G, ldg, F, ldf, Dinv, DinvT, logd, p0, ntiles, tile_stride, n_peer, then
 *          (F, Dinv, DinvT, logd) for each of the 7 peer sets;
 *   mode 1 (potrf128_ptr_launch), n = 6 per tile: G, Dinv, DinvT, logd, ld, info_base.                                */
int  gpb200_potrf_tiles(gpb200_handle* h, int mode, const int64_t* args, int32_t n, int32_t* info);
/* The blocked triangular solves (csrc/vec.cuh) on caller buffers, synchronous, launched as the engine launches them.
 * args (n = 6): F, ldf, Dinv (direction 0: out = L^-1 rhs) or DinvT (direction 1: out = L^-T rhs), rhs, out, Npad.
 * schedule 0: one launch per 128-block step (rhs is overwritten); schedule 1: the single-launch flag-synchronised kernel
 * (rhs is only read), Npad/128 <= 4 x SMs.  *watchdog = the watchdog word of the single-launch kernel (a flags buffer
 * owned by the call; 0 for schedule 0 and for every run in which each ready-flag arrived).
 * GPB200_EINVAL, nothing launched: bad schedule / direction / n, Npad not a positive multiple of 128, ldf odd or not
 * positive, a null or not 16-byte aligned pointer, schedule 1 above its block limit.                                  */
int  gpb200_trsv_tiles(gpb200_handle* h, int schedule, int direction, const int64_t* args, int32_t n, int32_t* watchdog);
/* The GPA kernels (csrc/gpa.cuh), synchronous, launched as the engine launches them:
 *   which 0 gpa_trmv_launch   (n = 5): F, ldf, v, f, Npad
 *   which 1 gpa_trmv_t_launch (n = 5): F, ldf, g, u, Npad
 *   which 2 gpa_scan_launch   (n = 8): G, ld, DinvT, u, v, F, ZdT, Npad
 * GPB200_EINVAL, nothing launched: bad which / n, Npad not a positive multiple of 128, ld < Npad, a null pointer.      */
int  gpb200_gpa_kernels(gpb200_handle* h, int which, const int64_t* args, int32_t n);
/* The fixed-order reductions (csrc/vec.cuh), synchronous, launched as the engine launches them:
 *   which 0 dot (n = 4): a, b, len, out     which 1 sum (n = 3): a, len, out
 *   which 2 rowdot (n = 6): K, ldk, alpha, M, N, mu     which 3 rowvar (n = 6): V, ldk, kdiag, M, N, var
 *   which 4 rowdot2 (n = 6): A, B, ld, M, N, q
 * GPB200_EINVAL, nothing launched: bad which / n, a negative length, ld < N, a null pointer.                           */
int  gpb200_row_reductions(gpb200_handle* h, int which, const int64_t* args, int32_t n);
/* The FSA block-diagonal kernels (csrc/fsa.cuh) on caller buffers, synchronous, each through its launch wrapper (one
 * launch, two for fsa_trace; sizes <= 0 launch nothing, as the wrappers do).  Item lists follow the fixed arguments,
 * flattened: FsaGramItem = (dst, ld, row_i, row_j, diag), FsaRowItem = (A, v, out, lda, K, sq).  The kernels that
 * evaluate the kernel program use the program of the last gpb200_set_kernel at fargs = log-scale theta (n_theta
 * entries); the handle's own theta and factor are left alone.
 *   which 0  fsa_gram      : xb, d, mask | Gram items        fargs = theta, diag_add
 *   which 1  fsa_bdmv      : mode, packed, rblk (int32), bstart, bsize (int32), boff, v (mode 2: unused), y, Np
 *   which 2  fsa_mask      : A, ld, nrows, ncols, rowmask, colmask (either may be 0)
 *   which 3  fsa_permute   : scatter, src, pos, n, dst
 *   which 4  fsa_resid     : out, a, b, mask, n
 *   which 5  fsa_outer     : a | Gram items
 *   which 6  fsa_trace     : xb, d, mask, part (items x n_theta), out | Gram items      fargs = theta
 *                            (no items: out[0 .. n_theta) is zeroed and nothing is launched)
 *   which 7  fsa_axpy_t    : C, ldc, A, lda, nrows, ncols                             fargs = alpha
 *   which 8  fsa_crossgram : xs, xb, d, mask | Gram items                             fargs = theta
 *   which 9  fsa_rowdot    : | row items (v unused when sq != 0)
 *   which 10 fsa_var       : out, q, g2, r2neg, n
 *   which 11 crossgram_dx  : xs, z, xb, d, M, u, Wb (0 = none), S1, S2, ldw, mask, alpha, E, lde, dmu, dvar (0: dmu only)
 *                            | items (row, out, b0, nb)                                 fargs = theta
 *                            (fsa_crossgram_dx, csrc/fsa.cuh: one CTA per item; xs, z, xb of leading dimension d)
 *   which 12 block_dx      : xb, d, map (0 = none), out, accumulate | items (G, row0, B, n, tile)   fargs = theta
 *                            out[row(i), :] (+)= sum_{l < n} (G[i B + l] + G[l B + i]) dk(x_i, x_l)/dx_i for the real rows
 *                            i = 128 tile .. min(n, 128 tile + 128) - 1 of each item, x_i = xb row row0 + i (leading
 *                            dimension d), row(i) = map[row0 + i] or row0 + i; out point-major (fsa_block_dx, csrc/fsa.cuh)
 * GPB200_EINVAL, nothing launched: bad which / n / nf, theta not of n_theta entries, a program dimension >= d, a null
 * pointer the kernel dereferences, a negative size or row, a bad mode, an item ld < 128, lda < K, ld < ncols.
 * GPB200_ESTATE: a kernel-program call before gpb200_set_kernel.                                                    */
int  gpb200_fsa_kernels(gpb200_handle* h, int which, const int64_t* args, int32_t n, const double* fargs, int32_t nf);
/* The dense Gram-family kernels (csrc/gram.cuh), synchronous, one call of the existing launch wrapper each, on device
 * buffers (row-major, leading dimensions in doubles).  The kernels that evaluate the kernel program use the program of
 * the last gpb200_set_kernel at fargs = log-scale theta (n_theta entries); the handle's own theta and factor are left
 * alone.  A size of 0 launches nothing (trace and trace_rect then zero their outputs).
 *   which 0  gram_lower         : x, ldx, d, N, Npad, noise_var, n_noise, G, ldg, own_tiles, nranks, rank, own_axis, bm_min
 *                                 fargs = theta, nugget
 *   which 1  crossgram          : xs, ldxs, M, Mpad, x, ldx, N, Npad, d, Kst, ldk
 *   which 2  gram_full          : xs, ldxs, M, Mpad, d, Kss, ldk
 *   which 3  kdiag              : xs, ldxs, d, M, out
 *   which 4  gram_grad_full     : x, ldx, d, N, Npad, j, D, ldd, row0, rows
 *   which 5  crossgram_grad     : x1, ldx1, N1, N1pad, x2, ldx2, N2, N2pad, d, j, D, ldd
 *   which 6  trace (+ reduce)   : x, ldx, d, N, Npad, alpha, Kinv, ldg, part, out, bm_mod, bm_rem, bm_div
 *                                 (out: n_theta + 1 entries, 3 for a single SEIso leaf over all d dimensions)
 *   which 7  trace_rect         : x1, ldx1, N1, x2, ldx2, N2, d, W, ldw, part, out
 *                                 (out: n_theta entries, 2 for a single SEIso leaf over all d dimensions)
 *   which 8  kdiag_grad         : x, ldx, d, N, g, out                                   (out[p * N + i])
 *   which 9  crossgram_dx       : xs, ldxs, M, z, ldz, n, d, a, W1 (0 = none), W2 (0 = none), ldw, dmu, dvar
 *                                 fargs = theta, c
 *   which 10 mirror_lower_tiles : F, ld, Npad                                            (no fargs)
 *   which 11 inputs_dx          : x, ldx, d, N, alpha (0 = none), G, ldg, out, bm_mod, bm_rem, bm_div, fast
 *                                 out[i, :] = sum_j A_ij dk(x_i, x_j)/dx_i over the lower triangle of A = alpha alpha' - G
 *                                 mirrored (A = -G without alpha); N x d point-major (inputs_dx_launch, csrc/gram.cuh).
 *                                 fast = 1: the SEIso specialisation, only for a single SEIso leaf over all d <= 8 dims
 *   which 12 gram_seiso_tma     : xp, xpt, d, N, Npad, noise_var, n_noise, G, ldg, own_tiles, nranks, rank, own_axis, sf
 *                                 fargs = theta, nugget
 *   which 13 trace_seiso_tma    : xp, xpt, d, N, Npad, alpha, Kinv, ldg, part, out, bm_mod, bm_rem, bm_div, sf
 *                                 (+ reduce; part: 3 per lower tile, out: 3 entries)      fargs = theta
 *                                 12 and 13 are the TMA-staged kernels of csrc/gram_fast.cuh on the engine's descriptors
 *                                 (seiso_make_x_maps): xp is [N x dx] with row pitch dx, xpt is [dx x N] with row pitch
 *                                 Npad, dx = d rounded up to even (a pad column, if any, must be zero in both).  sf, a HOST
 *                                 pointer or 0, receives the prepared constants c_hi, il2, s2, tab[64] (67 doubles).
 * GPB200_EINVAL, nothing launched: bad which / n / nf, theta not of n_theta entries, d outside 1 .. GPB200_MAX_DIMS, a
 * program dimension >= d, a null pointer (W1, W2 and, without them, dvar may be null), a negative size, a padded size
 * that is not a multiple of 128 or is below its size, a leading dimension below the row width, an odd leading dimension
 * or a pointer not 16-byte aligned for G, Kst, Kss, Kinv and W, j outside [0, n_theta), bad ownership arguments
 * (nranks >= 1, 0 <= rank < nranks, own_axis 0 or 1; bm_mod, bm_div >= 1, 0 <= bm_rem < bm_mod), row0 or rows not a
 * multiple of 128 or past Npad, fast = 1 without the single SEIso leaf over d <= 8 dims; for 12 and 13 also a program that
 * is not that leaf, d > 8, constants seiso_fast_prepare rejects, N < 1, or xp / xpt not 16-byte aligned.
 * GPB200_ECUDA: the TMA descriptors of 12 and 13 cannot be built.
 * GPB200_ESTATE: a kernel-program call before gpb200_set_kernel.                                                    */
int  gpb200_gram_kernels(gpb200_handle* h, int which, const int64_t* args, int32_t n, const double* fargs, int32_t nf);
/* The elementwise and sampling helpers (csrc/vec.cuh), synchronous, one launch each through its wrapper (sizes <= 0
 * launch nothing):
 *   which 0 ew           : op, n, out, a, b, c                  fargs = s
 *                          op 0 out = a + s, 1 out = a / b, 2 out += a, 3 out = (a - b) / c, 4 out = log(a), 5 out = 1 / a,
 *                          6 out = a - b
 *   which 1 spd_from_cov : dst, ldd, src, lds, n, npad          fargs = nugget
 *                          lower 128-tiles of dst (npad x npad) = src[:n, :n] + nugget I, identity in the padding
 *   which 2 add_rowvec   : A, ld, v, nrows, ncols               A[i, j] += v[j] for i < nrows, j < ncols
 *   which 3 gather_block : out, src, ld, idx, nv                out[a nv + b] = src[idx[a] ld + idx[b]] (idx: int64)
 * GPB200_EINVAL, nothing launched: bad which / n / nf, a bad op, a null pointer the kernel dereferences, a negative size,
 * npad not a positive multiple of 128 or below n, a leading dimension below the row width.                          */
int  gpb200_vec_kernels(gpb200_handle* h, int which, const int64_t* args, int32_t n, const double* fargs, int32_t nf);
/* The sparse cross-validation row kernels (csrc/fitc_cv.cuh) and the FITC element kernels that run between the same
 * GEMMs (csrc/vec.cuh), synchronous, one launch each through its wrapper (sizes <= 0 launch nothing):
 *   which 0  delta      : kind, x, ldx, d, j, G, C, ld, ncols, nrows, rows_pad, alpha, delta, da   fargs = theta
 *                         (the program of the last gpb200_set_kernel; x, G, C and j are read for kind 0 only)
 *   which 1  rows       : G (0 = none), Ch, K, P, ld, nrows, ncols, lam, delta, alpha, beta, w, zja, dg
 *   which 2  invdiag    : n, lam, q, out
 *   which 3  eblock     : E, G (0 = none), K, ld, nrows, ncols, lam, delta
 *   which 4  qs         : Q, H, R, ld, n
 *   which 5  wvec       : n, w, a, b, c
 *   which 6  gather     : nv, idx, x, ldx, d, xout, lam, lamout, delta (0 = none), delout
 *   which 7  diag       : out, ld, nv, which (0: 1/lam, 1: delta/lam^2), lam, delta
 *   which 8  colscale   : A, ld, nrows, ncols, v
 *   which 9  scale      : mode, A, ld, nrows, ncols, v
 *   which 10 fitc_g     : n, alpha, lam, q, g
 *   which 11 fitc_wfu   : P2, P1, ld, nrows, ncols, alpha, lam, g, beta
 *   which 12 fitc_wuu   : Wuu, T, Kinv, Sinv, ld, n, beta
 *   which 13 symmetrize : A, ld, n
 *   which 14 inducing_dx: u, ldu, M, z, ldz, n, d, W, ldw, sym, mask (0 = none), out, accumulate   fargs = theta
 *                         out[j, :] (+)= sum_{i < n, mask[i] != 0} W(i, j) dk(u_j, z_i)/du_j, W(i, j) = W[i ldw + j]
 *                         (+ W[j ldw + i] when sym = 1, which needs n = M); out is M x d point-major
 *   which 15 rows_dx    : x, ldx, n, u, ldu, M, d, W, ldw, c (0 = none), mask (0 = none), map (0 = none), out, accumulate
 *                         fargs = theta
 *                         out[row(i), :] (+)= sum_{j < M} W[i ldw + j] dk(x_i, u_j)/dx_i + 2 c_i dk(x_i, x')/dx_i at x' = x_i
 *                         over the rows i < n with mask[i] != 0 (the others are not written), row(i) = map[i] or i; out
 *                         point-major (rows_dx_launch, csrc/gram.cuh)
 * GPB200_EINVAL, nothing launched: as gpb200_fsa_kernels, plus j outside [0, n_theta) and ldx < d.                   */
int  gpb200_fitc_cv_kernels(gpb200_handle* h, int which, const int64_t* args, int32_t n, const double* fargs, int32_t nf);
/* The data-movement kernels of the multi-rank schedules (csrc/shard_kernels.cuh) on caller buffers, synchronous, one
 * launch each through its wrapper (nothing to do: no launch, as the wrappers do).  An ownership (R, me, rb) is the
 * block-cyclic layout of 128-row tiles, tile t owned by rank (t / rb) % R; one device can act as any rank of any layout.
 *   which 0  copy_lower      : dst, ldd, src, lds, n                                     (n <= 65 535)
 *   which 1  scatter_rows    : G, F, ld, Npad, c0, nb, t1, S_me, nbp, R, me, rb
 *   which 2  unpack_panel    : P, nbp, Npad, nb, t1, S, per_rank, R, me, rb             (per_rank holds every rank's rows)
 *   which 3  transpose       : dst, ldd, src, lds, rows, cols                            (rows <= 65 535 * 32)
 *   which 4  pack_wblock     : P, nbp, G, ld, Dinv, j0, nb                               (j0, nb multiples of 128)
 *   which 5  sum_ranks       : out, in, stride, nranks, n
 *   which 6  min_ranks       : out, in, nranks                                           (int32 words)
 *   which 7  transpose_own   : dst, ldd, src, lds, rows, cols, R, me, rb
 *   which 8  rowdot_own      : Y, G, ld, ncols, alpha, N, out, R, me, rb
 *   which 9  diag_own        : G, ld, N, out, R, me, rb
 *   which 10 gather_block_own: out, src, ld, idx, nv, R, me, rb                          (idx int64, nv <= 65 535)
 *   which 11 pack_slices     : G, ld, out, s, Np, R, me                                  (inverse_dist's slice exchange)
 *   which 12 unpack_slices   : G, ld, in, per_rank, s, Np, R, me
 *   which 13 signal_peers    : words (device array of int32 pointers), n_peer, value     (n_peer <= 7)
 *   which 14 wait_signal     : word, target, err                                         (spins until *word >= target)
 * The slice kernels take a level inverse_dist splits: s a multiple of 128 R below Np, Np a multiple of 128, ld >= Np, and
 * for unpack_slices per_rank >= sum_z n2_z s / R.
 * GPB200_EINVAL, nothing launched: bad which / n, a null pointer, a negative size, R < 1, me outside [0, R), rb < 1, Npad
 * not a multiple of 128, t1 past the last tile, nb > nbp, a leading dimension below the row width, a region too small
 * or a grid dimension past 65 535.                                                                                  */
int  gpb200_shard_kernels(gpb200_handle* h, int which, const int64_t* args, int32_t n);

/* ---- multi-GPU (one process per GPU; NCCL over NVLink) -------------------------------------- */
/* rank 0 obtains a 128-byte NCCL unique id, the host side broadcasts it (torch.distributed /
 * Julia Distributed), every rank then joins.                                                */
int  gpb200_nccl_unique_id(char* id128);
int  gpb200_comm_init(gpb200_handle* h, int nranks, int rank, const char* id128);
/* Fused panel broadcast over NVLink peer memory (optional, after comm_init and set_data): every rank
 * exports CUDA-IPC handles of its factor buffers (GPB200_IPC_BYTES bytes), the host layer all-gathers
 * the blobs (rank order) and every rank imports them.  From then on the kernels that PRODUCE a panel
 * (tile leaf, 128-wide TRSM GEMM) store it straight into all peers' buffers and raise a device-side
 * flag; NCCL stays on the small collectives only.  Re-export after a gpb200_set_data that changes N. */
#define GPB200_IPC_BYTES 512
int  gpb200_ipc_export(gpb200_handle* h, char* out);
int  gpb200_ipc_import(gpb200_handle* h, int nranks, const char* all_blobs);

/* In-process group of `n` (<= 8) handles on ONE device acting as n ranks of the ROW-SHARDED schedules (the storage
 * layout of config C4: each rank keeps only its own block rows of the N x N factor / inverse; see csrc/shard_impl.cuh).
 * Collectives become event-ordered device copies, so a single-GPU box exercises exactly the multi-rank code.  Every
 * handle needs the same gpb200_set_data / gpb200_set_kernel; factorize / mll / solve / grad_* / predict are then called
 * on hs[0] only.  (One process per GPU uses gpb200_comm_init instead and option "shard".)                       */
int  gpb200_group_create(gpb200_handle** hs, int n);
/* storage of the two N x N buffers of this handle: out[0] = 1 if row-sharded, out[1] / out[2] = bytes of F / G physically
 * backed on this device, out[3] = ownership block (tiles), out[4] = ranks, out[5] = rank, out[6] = 1 if the GEMMs run on
 * TMA descriptors (0: plain-load fallback), out[7] = bytes of the cross-validation work matrices physically backed on this
 * device (0 before the first gpb200_cv_param; 2 Npad^2 8 on one GPU, the own rows of two such matrices when row-sharded)
 * (cf. test/memory.jl:14-19)                                                                                         */
int  gpb200_storage_info(gpb200_handle* h, int64_t* out, int32_t n);

/* ---- sparse FITC strategy (src/sparse/fully_indep_train_conditional.jl) ------------------------
 * FITC(x, Xu, y, mean, kern, logNoise) (fitc.jl:335-338) == GPE(..., FullyIndepStrat(Xu)).
 * Covers update_cK!(::FullyIndepPDMat) (fitc.jl:134-156), `\` (fitc.jl:33-36), logdet (fitc.jl:77),
 * dmll_noise (fitc.jl:243-257), get_alpha_u (fitc.jl:279-286) and predictMVN (fitc.jl:324-332 ->
 * determ_train_conditional.jl:41-59 -> subsetofregressors.jl:302-321) and the kernel-parameter
 * gradient dmll_kern! (fitc.jl:200-234 on top of subsetofregressors.jl:140-151, 219-253).
 * N is streamed in chunks; only M x M matrices and O(N) vectors persist on the device.          */
typedef struct gpb200_fitc gpb200_fitc;
int  gpb200_fitc_create(gpb200_fitc** out, int device);
void gpb200_fitc_destroy(gpb200_fitc* f);
const char* gpb200_fitc_last_error(gpb200_fitc* f);
/* multi-GPU (one process per GPU): after gpb200_nccl_unique_id / broadcast of the id, every rank joins; each rank then passes
 * ITS OWN slice of the observations to gpb200_fitc_set_data / _mll (alpha is returned for that slice) and the same inducing points
 * and hyper-parameters.  Exchanged over NCCL: one all-reduce of the M x M accumulator Sigma_QR per factorisation (0.54 GB at
 * M = 8192), one of H per kernel gradient, M-vectors and scalars; K_uu / Sigma_QR factorisations and predictions are replicated. */
int  gpb200_fitc_comm_init(gpb200_fitc* f, int nranks, int rank, const char* id128);
/* x: d x N training inputs, xu: d x M inducing inputs (both column-major, one point per column) */
int  gpb200_fitc_set_data(gpb200_fitc* f, int64_t N, int32_t d, const double* x, int64_t ldx,
                          int64_t M, const double* xu, int64_t ldxu);
int  gpb200_fitc_set_kernel(gpb200_fitc* f, int32_t n_ops, const int32_t* ops, int32_t n_dims,
                            const int32_t* dims, int32_t n_theta);
/* update_cK!: K_uu (+1e-10 I), Lambda, Sigma_QR (+1e-10 I) and both Cholesky factors */
int  gpb200_fitc_factorize(gpb200_fitc* f, const double* theta, double log_noise);
/* alpha = Sigma^-1 r, logdet(Sigma), mll = -(r'alpha + logdet + N log 2pi)/2 */
int  gpb200_fitc_mll(gpb200_fitc* f, const double* y_minus_mean, double* alpha, double* mll, double* logdet);
int  gpb200_fitc_grad_noise(gpb200_fitc* f, double* dmll_noise);
/* dmll_kernel[n_theta], full parameter vector of the un-fixed kernel tree (as gpb200_grad_kernel) */
int  gpb200_fitc_grad_kernel(gpb200_fitc* f, double* dmll_kernel);
/* Gradient of the mll with respect to the inducing inputs (not in the reference; Snelson & Ghahramani's pseudo-inputs),
 * all four modes.  One sweep gives dmll_kernel[n_theta] (may be NULL; when given, bitwise equal to gpb200_fitc_grad_kernel
 * on the same handle: the same launches) and dmll_xu[M x d], point-major (Julia's d x M column-major):
 *   dmll/du_j = 1/2 [ sum_i W_fu[i, j] dk(u_j, x_i)/du_j + sum_l (W_uu[j, l] + W_uu[l, j]) dk(u_j, u_l)/du_j ]
 * with W_fu, W_uu the adjoints of the mll with respect to K_fu and K_uu that the kernel gradient already builds.  It adds one
 * contraction launch per staging chunk and one for W_uu (FSA padding rows are skipped); with several ranks the W_fu part is
 * all-reduced once (M d doubles).  Sums are in a fixed order: repeated calls are bitwise equal.  Device memory grows by
 * M d doubles on the first call.  GPB200_ESTATE before factorize + mll; GPB200_EINVAL for a NULL dmll_xu.
 * gpb200_fitc_get_timings slots 7-8 hold the last call's device times: the contractions, the whole call.            */
int  gpb200_fitc_grad_kernel_inducing(gpb200_fitc* f, double* dmll_kernel, double* dmll_xu);
/* Replaces the inducing inputs (xu: d x M column-major, ld = ldxu) of both M x M sub-engines in place (not in the
 * reference).  M must be gpb200_fitc_set_data's and ldxu >= d (GPB200_EINVAL otherwise); GPB200_ESTATE before set_data.
 * The training inputs, the kernel program, the FSA blocks and their work lists and every workspace are kept; the
 * factorisation, alpha and the cross-validation state are cleared.  After factorize + mll, alpha, mll and logdet are
 * bitwise those of a fresh handle given the same xu to gpb200_fitc_set_data (and the same gpb200_fitc_set_blocks).
 * With several ranks every rank passes the same xu.                                                                   */
int  gpb200_fitc_set_inducing(gpb200_fitc* f, int64_t M, const double* xu, int64_t ldxu);
/* Gradient of the mll with respect to the training inputs (not in the reference; latent-input and input-warping models),
 * all four modes.  One sweep gives dmll_x[N x d], point-major (Julia's d x N column-major; on several ranks the rank's own
 * rows), and optionally dmll_kernel[n_theta] and dmll_xu[M x d] (either may be NULL; when given, bitwise equal to those of
 * gpb200_fitc_grad_kernel and gpb200_fitc_grad_kernel_inducing: the same launches).  With W_fu, g and G_b the adjoints of
 * the mll with respect to K_fu, the FITC diagonal K_ii and the FSA blocks K_bb that the kernel gradient builds, and d1k the
 * derivative of k in its first argument:
 *   FITC:      dmll/dx_i = 1/2 [ sum_j W_fu[i, j] d1k(x_i, u_j) + 2 g_i d1k(x_i, x_i) ]
 *   DTC, SoR:  dmll/dx_i = 1/2   sum_j W_fu[i, j] d1k(x_i, u_j)
 *   FSA:       dmll/dx_i = 1/2 [ sum_j W_fu[i, j] d1k(x_i, u_j) + sum_{l in b(i)} (G_b[i, l] + G_b[l, i]) d1k(x_i, x_l) ]
 * The mean's part alpha_i dm(x_i)/dx_i is left to the caller.  It adds one row-contraction launch per staging chunk (FSA:
 * two, the block contraction and the row contraction); these read the adjoints and write nothing else, and nothing is
 * exchanged between ranks for X.  Sums are in a fixed order: repeated calls are bitwise equal.  Device memory grows by
 * N d doubles on the first call.  GPB200_ESTATE before factorize + mll; GPB200_EINVAL for a NULL dmll_x.
 * gpb200_fitc_get_timings slots 9-10 hold the last call's device times: the X contractions summed, the whole call.   */
int  gpb200_fitc_grad_kernel_inputs(gpb200_fitc* f, double* dmll_kernel, double* dmll_xu, double* dmll_x);
/* Replaces the training inputs (x: d x N column-major, ld = ldx) in place (not in the reference).  N must be
 * gpb200_fitc_set_data's and ldx >= d (GPB200_EINVAL otherwise); GPB200_ESTATE before set_data.  FSA keeps its blocks (by
 * index), their work lists and every workspace, and rebuilds its reordered copy of the inputs.  The factorisation, alpha
 * and the cross-validation state are cleared.  After factorize + mll, alpha, mll and logdet are bitwise those of a fresh
 * handle given the same x to gpb200_fitc_set_data (and the same gpb200_fitc_set_blocks).  With several ranks every rank
 * passes its own slice.  No kernel is launched.                                                                        */
int  gpb200_fitc_set_inputs(gpb200_fitc* f, int64_t N, const double* x, int64_t ldx);
/* append! for FITC, DTC and SoR (modes 0-2; not in the reference for the sparse strategies): k new observations (xnew:
 * d x k column-major, ld = ldx; r_new[k] = y - m(x) of the new rows) with the hyper-parameters and Xu of the last
 * factorize.  Sigma_QR, b = K_uf Lambda^-1 r and the mll's scalars are updated by the new rows only and Sigma_QR is
 * refactored: O(k M^2 + M^3) whatever N is; no pass over the old rows' kernel values.  mll (and logdet, may be NULL) are
 * those gpb200_fitc_mll gives on the concatenated data.  Needs factorize + mll, or an earlier successful append
 * (GPB200_ESTATE otherwise).  GPB200_EINVAL, nothing changed: mode 3 (FSA), k < 1 (k < 0 on several ranks), ldx < d, a NULL
 * xnew, r_new or mll, a non-finite r_new.  Afterwards u, L_uu and L_s match the data: gpb200_fitc_predict, _predict_cov,
 * _predict_grad and _rand accept the handle; grad_noise, the kernel gradients and cross-validation need alpha and return
 * GPB200_ESTATE until gpb200_fitc_mll is called with the full residuals (the last cv_param's state is cleared).  The
 * N-sized buffers grow geometrically; FSA blocks set earlier are dropped.  A Sigma_QR that is not positive definite
 * returns its leading minor (> 0): the factorisation is cleared, the grown data stays.  On several ranks the call is
 * collective: each rank passes its own rows (k may be 0 on some ranks).                                               */
int  gpb200_fitc_append(gpb200_fitc* f, int64_t k, const double* xnew, int64_t ldx, const double* r_new, double* mll,
                        double* logdet);
/* mu_minus_mean[Ms], var[Ms] (may be NULL; not clamped) */
int  gpb200_fitc_predict(gpb200_fitc* f, int64_t Ms, const double* xs, int64_t ldxs, double* mu_minus_mean, double* var);
/* Predictive gradients of FITC / DTC / SoR with respect to the test inputs, as gpb200_predict_grad (same layouts, var and
 * dvar together or both NULL): mu_minus_mean and var bitwise equal to gpb200_fitc_predict's, and
 *   dvar[m, p] = 2c dk(x*_m, x*_m)/dx*_{m,p} - 2 sum_j dk(x*_m, u_j)/dx*_{m,p} W'[m, j],  W' = K*u K_uu^-1 - K*u Sigma_QR^-1
 * (c = 1; SoR: W' = -K*u Sigma_QR^-1, c = 0), dmu[m, p] = sum_j dk(x*_m, u_j)/dx*_{m,p} (Sigma_QR^-1 K_uf Lambda^-1 y)_j.
 * GPB200_ESTATE before factorize + mll; GPB200_EINVAL for multi-rank handles ("single GPU") and in mode 3, whose
 * gradients need test blocks (gpb200_fitc_predict_fsa_grad).                                                          */
int  gpb200_fitc_predict_grad(gpb200_fitc* f, int64_t Ms, const double* xs, int64_t ldxs, double* mu_minus_mean,
                              double* var, double* dmu, double* dvar);
/* predictMVN with the full covariance cov[Ms x Ms] (fitc.jl:324-332, dtc.jl:41-59, sor.jl:302-321); Ms <= 32768 */
int  gpb200_fitc_predict_cov(gpb200_fitc* f, int64_t Ms, const double* xs, int64_t ldxs, double* mu_minus_mean, double* cov);
/* 0 = FITC (default), 1 = DTC (src/sparse/determ_train_conditional.jl), 2 = SoR
 * (src/sparse/subsetofregressors.jl): the two share Lambda = sigma^2 I (sor.jl:96-106, `\` sor.jl:50,
 * logdet sor.jl:53, dmll_noise sor.jl:159-166, dmll_kern! sor.jl:219-253); SoR's predictive covariance is
 * K_xu S^-1 K_ux (sor.jl:302-321), DTC's adds K_xx - Q_xx (dtc.jl:41-59).
 * 3 = FSA (src/sparse/full_scale_approximation.jl): Lambda = blockdiag(K_ii - Q_ii + (sigma^2 + 1e-10) I) over the
 * training blocks of gpb200_fitc_set_blocks (update_cK! :197-230).  gpb200_fitc_mll (`\` :105-108, logdet :142) and
 * gpb200_fitc_grad_noise (dmll_noise :328-363) return the FSA results, alpha in the caller's order; factorize returns
 * k > 0 when a block of Lambda is not positive definite (k = 1 + the row of the first bad pivot in the padded block
 * layout).  gpb200_fitc_grad_kernel returns the FSA kernel-parameter gradient (dmll_kern! :274-326).
 * gpb200_fitc_predict / _predict_cov return GPB200_EINVAL (FSA predictions need test blocks: gpb200_fitc_predict_fsa).
 * Single GPU only: after gpb200_fitc_comm_init with more than one rank, factorize returns GPB200_EINVAL.          */
int  gpb200_fitc_set_mode(gpb200_fitc* f, int mode);
/* FSA training blocks in CSR form: block b is idx[block_ptr[b] .. block_ptr[b+1]) (0-based), nblocks >= 1.  Call after
 * gpb200_fitc_set_data (which clears them) and before gpb200_fitc_factorize (mode 3 without blocks: GPB200_ESTATE).  The
 * blocks must partition 0..N-1 (GPB200_EINVAL otherwise); empty blocks are allowed; a block holds at most 2048 points
 * (GPB200_EINVAL otherwise), which bounds the tile steps of the batched block factorisation.  The rows are reordered once
 * so that every block starts on a 128-row boundary; device memory grows by 2 * sum_i B_i^2 doubles (the factor and its
 * inverse, B_i = the block size rounded up to 128), one staging chunk's G_i blocks for the kernel gradient (at most
 * 32768 * 2048 doubles), O(N) vectors and the work lists, and the staging chunk is grown to its full size.            */
int  gpb200_fitc_set_blocks(gpb200_fitc* f, int64_t nblocks, const int64_t* block_ptr, const int64_t* idx);
/* FSA predictMVN / predict_f with test blocks (full_scale_approximation.jl:413-478), mode 3 after gpb200_fitc_mll.
 * block_of[Ms] is the training block each test point is paired with (test block j pairs with training block j, as the
 * reference's `zip`); -1 or a block id >= nblocks contributes no Lambda_xf term.  mu_minus_mean[Ms] = K_xu alpha_u +
 * Lambda_xf alpha;  var[Ms] (may be NULL; not clamped) = the diagonal of Sigma_FSA = K_xx - (Q_xf + Lambda_xf) Sigma^-1
 * (Q_xf + Lambda_xf)' (each point's variance does not depend on the other test points);  cov[Ms x Ms] (may be NULL) =
 * Sigma_FSA, row-major.  Test blocks have no size limit (test rows are streamed in chunks); cov needs the test points,
 * grouped by block and each group padded to a multiple of 128, to fit one staging chunk (GPB200_EINVAL otherwise).      */
int  gpb200_fitc_predict_fsa(gpb200_fitc* f, int64_t Ms, const double* xs, int64_t ldxs, const int64_t* block_of,
                             double* mu_minus_mean, double* var, double* cov);
/* Predictive gradients of FSA with respect to the test inputs (predict_f(gp, x, blockindpred) with ForwardDiff.Dual
 * inputs), block_of and layouts as gpb200_fitc_predict_fsa and gpb200_fitc_predict_grad: mu_minus_mean[Ms] and var[Ms]
 * bitwise equal to gpb200_fitc_predict_fsa's (same launches), dmu and dvar Ms x d point-major, var and dvar given together
 * or both NULL.  With c = Lambda_xf row m (0 when unpaired), u = alpha_u, S = Sigma_QR, h = c Lambda_b^-1,
 * s = S^-1 (k_u - K_ub h') and D_u, D_b, D_** the input derivatives of k(x*, u_j), k(x*, x_i) over the paired block and k(x*, x*):
 *   dmu  = D_u (u - K_uu^-1 K_ub alpha_b) + D_b alpha_b
 *   dvar = D_** + D_u (2 s - 2 K_uu^-1 k_u - K_uu^-1 K_ub e) + D_b e,   e = -2 Lambda_b^-1 (c' + K_bu s)
 * Test points are streamed (no size limit).  Device memory grows on the first call with var by one staging chunk of
 * test-row x block tiles (Nc x 128 * the largest block's tiles doubles) and one Nc x Mpad matrix, and by 2 Ms d doubles
 * for the outputs.  GPB200_ESTATE before set_blocks + factorize + mll; GPB200_EINVAL outside mode 3, for multi-rank
 * handles and for bad arguments.  gpb200_fitc_get_timings slots 3-6 hold its device-event split, summed over the test
 * chunks: predict_fsa's launches, s and the second block sweep, the K_uu^-1 TRSMs, the contraction.                   */
int  gpb200_fitc_predict_fsa_grad(gpb200_fitc* f, int64_t Ms, const double* xs, int64_t ldxs, const int64_t* block_of,
                                  double* mu_minus_mean, double* var, double* dmu, double* dvar);
/* rand(gp, X, n) (src/GP.jl:120-146) with a sparse cK, on the device, with gpb200_rand's conventions: z and samples are
 * Ms x nsamp column-major, mu_minus_mean[Ms] is the predictive mean without mean(x*).  Sigma* is exactly the covariance of
 * gpb200_fitc_predict_cov (modes 0-2; block_of must be NULL; Ms <= one staging chunk) or of gpb200_fitc_predict_fsa (mode 3;
 * block_of[Ms] required, as there; the grouped, padded test blocks must fit one staging chunk); it stays on the device.
 * (FSA's Sigma* is positive semi-definite when all test points pair with one training block; over several blocks it is in
 * general indefinite, and k > 0 is returned as the reference's cholesky would.)
 * make_posdef!(Sigma*; nugget), its Cholesky on an Ms x Ms sub-engine of the handle (created on first use), unwhiten! as one
 * NT GEMM and + mu follow gpb200_rand; the sub-engine's kernels count in gpb200_fitc_launch_count.  After factorize + mll
 * (GPB200_ESTATE otherwise).  GPB200_EINVAL: bad Ms, nsamp or ldxs, a NULL xs, z, mu_minus_mean or samples, nugget < 0,
 * block_of given in modes 0-2 or missing in mode 3, too many test points.  Returns k > 0 when Sigma* + nugget I is not
 * positive definite; the handle stays usable.  The likelihood, gradient, prediction and cross-validation results of the
 * handle are unchanged (bitwise).  With several ranks (gpb200_fitc_comm_init) every rank holds the replicated M x M state
 * and draws on its own, as predict_cov does; that case has not been run on more than one GPU.                          */
int  gpb200_fitc_rand(gpb200_fitc* f, int64_t Ms, const double* xs, int64_t ldxs, const int64_t* block_of,
                      int64_t nsamp, const double* z, double nugget, double* mu_minus_mean, double* samples);
/* device times (ms) of the last successful gpb200_fitc_rand: [0] Sigma* build (with mu), [1] make_posdef! + Cholesky,
 * [2] unwhiten! GEMM + mu; of the last gpb200_fitc_predict_fsa_grad, summed over its test chunks: [3] predict_fsa's
 * launches, [4] s = R L_s^-1 and the second block sweep, [5] the K_uu^-1 TRSMs, [6] the contraction; of the last
 * gpb200_fitc_grad_kernel_inducing: [7] its dmll/dXu contractions summed, [8] the whole call; of the last
 * gpb200_fitc_grad_kernel_inputs: [9] its dmll/dX contractions summed, [10] the whole call (CUDA events; n <= 11 entries
 * are written)                                                                                                          */
int  gpb200_fitc_get_timings(gpb200_fitc* f, double* ms, int32_t n);
/* ---- cross-validation on the sparse engine (src/crossvalidation.jl with cK a FITC / DTC / SoR covariance) ---------------
 * The dense entry points gpb200_get_inverse_diag / gpb200_cv_param / gpb200_cv_block for modes 0 (FITC), 1 (DTC: SoR's
 * covariance) and 2 (SoR), after gpb200_fitc_factorize and gpb200_fitc_mll.  Sigma = Lambda + K_fu K_uu^-1 K_uf is the matrix
 * gpb200_fitc_mll inverts; nothing N x N is formed: every quantity comes from K_uu^-1, Sigma_QR^-1 (M x M) and the rows of
 * K_fu and dK_fu regenerated chunk by chunk.  gpb200_fitc_cv_param costs two streaming passes over the N rows (~14 N M^2
 * flop on the DMMA GEMM for a FITC kernel parameter), a fold block O(nV M^2 + nV^2 M).  The likelihood, gradient and
 * prediction state of the handle is not touched: their results stay bitwise equal.  Repeated calls are bitwise equal.
 * GPB200_ESTATE before factorize + mll; GPB200_EINVAL for mode 3 (FSA), for a handle with more than one rank
 * (gpb200_fitc_comm_init), for a bad `param`, `which` or index, and for nV above one staging chunk.                    */
/* diag(Sigma^-1)[N]: all predict_LOO / logp_LOO need besides alpha (crossvalidation.jl:8-49) */
int  gpb200_fitc_get_inverse_diag(gpb200_fitc* f, double* diag);
/* Zj_alpha[N] = Z_j alpha and diag_ZjSinv[N] = diag(Z_j Sigma^-1) with Z_j = Sigma^-1 dSigma/dtheta_j; `param` indexes the
 * kernel's full parameter vector, -1 is the noise variance (dSigma = I).  alpha[N] may be NULL: the alpha of the last
 * gpb200_fitc_mll.  The M x M state of this parameter stays resident for gpb200_fitc_cv_block(which = 1).                */
int  gpb200_fitc_cv_param(gpb200_fitc* f, int32_t param, const double* alpha, double* Zj_alpha, double* diag_ZjSinv);
/* principal sub-matrix on idx[nV] (0-based), row-major nV x nV, of Sigma^-1 (which = 0) or of Z_j Sigma^-1 for the parameter
 * of the last gpb200_fitc_cv_param (which = 1; GPB200_ESTATE without one since the last factorize).  nV <= the staging chunk
 * (32768 rows at most, fewer for large M: 2e9 / (8 Mpad) rounded down to 128).                                            */
int  gpb200_fitc_cv_block(gpb200_fitc* f, int32_t which, int64_t nV, const int64_t* idx, double* out);
/* number of kernels enqueued by calls on this handle since creation, on both M x M sub-engines; cudaMemsetAsync and
 * copies are not counted */
int64_t gpb200_fitc_launch_count(gpb200_fitc* f);

#ifdef __cplusplus
}
#endif
#endif /* GPB200_H */
