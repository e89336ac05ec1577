// engine.cuh -- private to the engine's translation units; not installed and not part of the ABI.
//   gpb200.cu            the dense engine (gpb200_handle) and its C ABI: schedules, IPC / NCCL, in-process groups
//   kernel_contracts.cu  the raw kernels exposed for the parity tests and the roofline bench (include/gpb200.h)
//   fitc_engine.cu       the sparse handle (gpb200_fitc): FITC / DTC / SoR, sparse cross-validation, rand, append
//   fsa_engine.cu        the FSA schedule of the sparse handle (mode 3)
// It holds the handle structs, the error path, and the declarations of what one unit uses from another.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <nccl.h>
#include <stdio.h>
#include <string>
#include <vector>

#include "../../include/gpb200.h"
#include "devbuf.cuh"
#include "gemm_nt.cuh"
#include "kprog.cuh"

// a virtual address range backed by physical memory only where `runs` say so (CUDA VMM: cuMemAddressReserve / cuMemMap)
struct VmBuf {
    CUdeviceptr base = 0;
    size_t va_size = 0;
    std::vector<std::pair<size_t, size_t>> runs;          // (offset, bytes) of every mapped run
    std::vector<CUmemGenericAllocationHandle> handles;    // one physical allocation per run
};

struct gpb200_handle {
    int device = 0;
    cudaStream_t st = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr, ev3 = nullptr, ev4 = nullptr, ev5 = nullptr;
    int64_t N = 0, Npad = 0, ld = 0;
    int d = 0;
    DevBuf<double> x;
    KProg prog{};
    std::vector<double> theta;
    bool has_data = false, has_kernel = false, factored = false, inv_ready = false, alpha_ready = false;
    bool s_ready = false;                      // G's lower triangle holds -S of gpb200_gpa_grad (A = S for gpb200_grad_inputs)
    double *F = nullptr, *G = nullptr;         // Frep / Grep (replicated) or the VMM ranges vmF / vmG (row-sharded)
    DevBuf<double> Frep, Grep;
    DevBuf<double> Dinv, DinvT, logd;
    DevBuf<double> noise_var, r0, r1, y1, alpha, scal;
    DevBuf<double> part, trace_out;
    DevBuf<double> tblk;                       // Npad scratch vector (block right-hand sides of the sharded solves)
    DevBuf<double> ZdT;                        // gpb200_gpa_grad: Npad x 128 clean upper diagonal tiles of Z' (allocated on first use)
    CUtensorMap mapZdT{};
    // TMA-staged SEIso kernels (gram_fast.cu): inputs stored [Npad x dxp] with an even, zero-padded dxp <= 8
    DevBuf<double> xp, xpt;                    // [Npad x dxp] and its transpose [dxp x Npad]
    int dxp = 0;
    CUtensorMap mapX{}, mapXT{};
    bool xmap_ok = false;
    int64_t capacity = 0;                      // option "capacity": rows reserved for gpb200_append (ElasticGPE's capacity)
    int gram_fast = 1;                         // option "gram_fast": 0 = always the generic kernels of gram.cu
    // cross-validation (gpb200_cv_*): K_y^-1 mirrored to a full symmetric matrix in G; two N x N temporaries
    bool g_sym = false;
    bool cv_m_ok = false;                                       // cvD holds M_j = Z_j K^-1 of the last cv_param call
    DevBuf<double> cvD, cvY;
    CUtensorMap mapCvD{}, mapCvY{};
    DevBuf<double> cvblk; DevBuf<long long> cvidx;   // principal sub-blocks of gpb200_cv_block (grown on demand)
    // posterior sampling (gpb200_rand): M x M sub-engine for chol(Sigma* + nugget I), normal draws / samples staging
    gpb200_handle* sub = nullptr;
    DevBuf<double> rz, rout;                   // rz_rows x rz_cols each
    int64_t rz_rows = 0, rz_cols = 0;
    CUtensorMap mapRz{};
    DevBuf<int> info_dev;
    DevBuf<int> flags;                         // ready-flags of the single-launch triangular solves (2 x (Npad/128 + 1))
    int trsv_fused = 1;
    int max_resident_ctas = 0;
    int64_t n_noise = 1;
    double nugget = 0.0;
    CUtensorMap mapF{}, mapG{}, mapDinv{}, mapDinvT{};
    bool tma_ok = false;
    // predict workspace
    DevBuf<double> xs, Kst, Kss, pmu, pvar, pkdiag;   // grown on demand
    DevBuf<double> pdx;                        // gpb200_predict_grad: dmu (Mpad x d), then dvar (Mpad x d)
    // gpb200_grad_inputs (first use, freed with the data): a caller's alpha (Npad), the N x d result (Npad x d), and in an
    // in-process group the gathered ranks' results (nranks x Npad x d)
    DevBuf<double> dxin;
    CUtensorMap mapKst{};
    // options
    int nb = 0;                 // outer Cholesky block; 0 = fully recursive (one panel)
    int gemm_impl = 0;
    int lookahead = 1;          // factor the next diagonal tile on a side stream while the Schur update runs
    cudaStream_t st_side = nullptr;            // high-priority stream of the look-ahead chain
    cudaStream_t st_cur = nullptr;             // stream launch_gemm / the leaf use right now (st or st_side)
    cudaEvent_t ev_la0 = nullptr, ev_la2 = nullptr;
    // stats
    double ms[17] = {};
    int64_t launches = 0;
    bool own_stream = true;
    // per-launch GEMM profiling (option "profile"): event pairs + executed flops of every GEMM launch
    int profile = 0;
    std::vector<cudaEvent_t> pev;
    size_t pev_used = 0;
    double gemm_flops_exec = 0.0;
    int64_t gemm_launches = 0;
    // multi-GPU (one process per GPU): replicated F/G, block-column ownership, NCCL over NVLink
    int nranks = 1, rank = 0;
    ncclComm_t comm = nullptr;
    cudaStream_t st_comm = nullptr;
    int dist_nb = 0;                           // width of an owned block column; 0 = auto (~Npad/(8*nranks))
    DevBuf<double> pack[2];                    // panel staging (double buffered)
    cudaEvent_t ev_packed[2] = {nullptr, nullptr}, ev_bcast[2] = {nullptr, nullptr}, ev_unpacked[2] = {nullptr, nullptr};
    cudaEvent_t ev_x = nullptr, ev_y = nullptr;
    DevBuf<double> ag_send, ag_recv;
    // fused panel broadcast over NVLink peer memory (CUDA IPC): peers' F / Dinv / DinvT / logd / signal words
    bool p2p = false;
    int n_peer = 0;
    int peer_rank[7] = {0, 0, 0, 0, 0, 0, 0};
    double *peer_F[7] = {}, *peer_Dinv[7] = {}, *peer_DinvT[7] = {}, *peer_logd[7] = {};
    int* peer_sig[7] = {};
    DevBuf<int> sig;                           // sig[q] = last panel published by rank q (epoch * 65536 + b + 1); sig[8] = watchdog
    int epoch = 0;
    DevBuf<int*> peer_sig_dev;                 // device array: &peer_sig[q][rank]
    bool push_panel = false;                   // set while the owner factors a panel: leaf + leaf TRSM also store to the peers
    // ---- row-sharded storage (shard_impl.cuh): F / G are virtual address ranges, physical pages exist for owned rows only ----
    int shard_opt = -1;                        // option "shard": -1 auto (when replicated F+G would not fit), 0 never, 1 always
    int shard_rb_opt = 0;                      // option "shard_rb": ownership block in 128-row tiles (0 = auto)
    bool sharded = false;                      // current storage mode of F / G
    int rb = 4;                                // effective ownership block (tiles); panel width NBp = 128 * rb
    int row_lim = 0;                           // chol_panel: rows below this limit only (diagonal block of a sharded panel); 0 = Npad
    VmBuf vmF, vmG;
    VmBuf vmCvY, vmCvM;                        // cross-validation work matrices (Y' = K^-1 dK_j, lower triangle of M_j), own rows only
    CUtensorMap mapShCvY{}, mapShCvM{};
    DevBuf<double> P[4];                                   // panel buffers, Npad x NBp (global row order); P[1], P[3] double as NBp x Npad row panels
    DevBuf<double> Sbuf;                       // all-gather staging: nranks regions of S_per_rank doubles; scratch of the inverse sweep
    size_t S_per_rank = 0;
    CUtensorMap mapP[4] = {}, mapXR[2] = {}, mapS{};
    DevBuf<double> XRbig[2];                   // row-panel forms X_J of a BATCH of panels (inverse sweep: batched LAUUM part)
    int xr_batch = 1;                          // panels per batch
    CUtensorMap mapXRbig[2] = {};
    DevBuf<double> red;                        // small reduction scratch (local group all-reduce)
    DevBuf<int> redi;
    struct gpb200_group* grp = nullptr;        // in-process group of virtual ranks on one device (gpb200_group_create)
    std::vector<cudaEvent_t> evring;
    size_t evring_next = 0;
    std::string err;
};

// in-process "communicator": R handles on one device acting as R ranks of the sharded schedules, driven in lock step by
// one host thread.  Collectives are device-to-device copies ordered by events (shard_impl.cuh).
struct gpb200_group {
    std::vector<gpb200_handle*> hs;
};


// ---- FITC (sparse/fully_indep_train_conditional.jl): two dense M x M sub-engines + N-chunk streaming ----
// The sparse handle's device buffers, grouped by lifetime; assigning {} to a group frees it.
struct FitcData {                    // the observations: N (+ 128 padding) and Mpad vectors
    DevBuf<double> x, lam, y, alpha, tmpn;
    DevBuf<double> bvec, uvec, tmpm, rhsm, scal;
};
struct FitcStage {                   // one staging chunk of Nc rows (fitc_stage_alloc)
    DevBuf<double> xs, w, tmpc, zeroc, tmpc2;
    DevBuf<double> bufA, bufB;       // Nc x Mpad (K_fu chunk) ; Mpad x Nc (K_uf chunk)
    CUtensorMap mapA{}, mapB{}, mapB2{};
};
struct FitcGradWs {                  // kernel-gradient workspace; sized by N, Nc and Mpad
    DevBuf<double> bufC, Hbuf, Wbuf, Tbuf, gvec, betav, gpart, gacc, gtmp;
    CUtensorMap mapAt{}, mapC{}, mapCt{}, mapH{}, mapT{};
    bool ready = false;
};
// cross-validation (gpb200_fitc_get_inverse_diag / _cv_param / _cv_block), apart from every buffer the likelihood,
// gradient and prediction schedules keep; sized by N, Nc and Mpad:
//   G Nc x Mpad: G = dK_fu - 1/2 K_fu Dp of a chunk;  Gt Mpad x Nc: G' (pass 1), then the Delta-scaled K_uf L^-1;
//   Ch Nc x Mpad: Ch = L^-1 K_fu S^-1;  P Nc x Mpad: Ch Q (pass 2) or E (fold blocks)
//   Mpad x Mpad: Duu = dK_uu, Dp = dK_uu K_uu^-1, R = K_uf L^-1 G, H = K_uf L^-1 Delta L^-1 K_fu, Q = H - R - R'
struct FitcCvWs {
    DevBuf<double> G, Gt, Ch, P;
    DevBuf<double> Duu, Dp, R, H, Q;
    DevBuf<double> alpha, del, ilam, za, dg;         // N + Nc
    DevBuf<double> da, q, lamV, delV, xs;            // Nc (xs: Nc x d)
    DevBuf<double> m;                                // 8 x Mpad: K_uf alpha, G' alpha, K_uf L^-1 Delta alpha, beta, R beta, w, tmp
    DevBuf<double> out;                              // fold block (padded nV x padded nV), grown on demand
    DevBuf<long long> idx;
    CUtensorMap mapG{}, mapGt{}, mapCh{}, mapP{}, mapDuu{}, mapDp{}, mapQ{};
    bool ready = false;
    bool m_ok = false;                               // Dp / Q / del hold the state of the last cv_param since factorize
};
// gpb200_fitc_append: the unfactored Sigma_QR (Mpad x Mpad, lower tiles; allocated on first use, rebuilt once as L_s L_s'
// after each factorize) and the running sums of the mll over all ranks: r'Lambda^-1 r, sum log Lambda, N
struct FitcAppend {
    DevBuf<double> sqr;
    bool sqr_ok = false;             // sqr is Sigma_QR of the current data
    bool sums_ok = false;            // s, l, n are those of the current data and residuals
    double s = 0.0, l = 0.0, n = 0.0;
};

struct gpb200_fitc {
    gpb200_handle* eu = nullptr;     // K_uu  (+1e-10 I)            -> L_uu
    gpb200_handle* es = nullptr;     // Sigma_QR = K_uf L^-1 K_fu + K_uu (+1e-10 I) -> L_s
    int device = 0;
    int64_t N = 0, M = 0, Mpad = 0, Nc = 0;
    int d = 0;
    FitcData data;                   // per data set
    FitcStage stage;                 // per staging chunk
    FitcGradWs grad;                 // kernel-gradient workspace (first use)
    DevBuf<double> Kss;                               // full predictive covariance (gpb200_fitc_predict_cov)
    DevBuf<double> pdx;                               // gpb200_fitc_predict_grad: dmu, dvar of a chunk (2 x Nc x d; first use)
    // posterior sampling (gpb200_fitc_rand): the Ms x Ms sub-engine and the staging of the draws are eu's (rand_from_cov)
    double rand_ms[3] = {0, 0, 0};                    // device times of the last rand: Sigma* build, Cholesky, unwhiten!
    double fsag_ms[4] = {0, 0, 0, 0};                 // last predict_fsa_grad, summed over test chunks: predict_fsa's
                                                      // launches, s + second sweep, K_uu^-1 TRSMs, contraction
    // inducing-point gradient (gpb200_fitc_grad_kernel_inducing; first use): dmll/dXu accumulator (M x d), the events
    // around the call (0, 1) and around each contraction launch (2k, 2k + 1 for k >= 1), and the device times of the last
    // call: the contractions summed, the whole call
    DevBuf<double> dxu;
    std::vector<cudaEvent_t> xu_ev;
    double xu_ms[2] = {0, 0};
    // training-input gradient (gpb200_fitc_grad_kernel_inputs; first use): dmll/dX accumulator (N x d, this rank's rows in
    // the caller's order), the events around the call and its contractions (as xu_ev) and the device times of the last call
    DevBuf<double> dx;
    std::vector<cudaEvent_t> x_ev;
    double x_ms[2] = {0, 0};
    FitcCvWs cv;                     // cross-validation workspace (first use)
    int cv_param = 0;
    // rows the N-sized buffers hold (data, grad.gvec, the cross-validation N-vectors): N after set_data, grown
    // geometrically by gpb200_fitc_append
    int64_t Ncap = 0;
    FitcAppend app;
    bool u_ready = false;            // after gpb200_fitc_append: u, L_uu and L_s match the data, alpha does not (predictions only)
    // multi-GPU (gpb200_fitc_comm_init): the N observations are sharded over the ranks, every M x M object is replicated;
    // exchanged: one all-reduce of the M x M accumulator Sigma_QR (and of H for the kernel gradient), M-vectors, scalars
    ncclComm_t comm = nullptr;
    int nranks = 1, rank = 0;
    double Ntotal = 0.0;                              // observations over all ranks (mll's N log 2 pi)
    int mode = 0;                    // 0 FITC, 1 DTC, 2 SoR (Lambda = sigma^2 I; SoR also drops K_xx - Q_xx from the predictive variance)
    double noise_var = 0.0;
    bool has_data = false, has_kernel = false, factored = false, alpha_ready = false;
    std::string err;
    struct Fsa* fsa = nullptr;       // mode 3 (FSA): training blocks and the packed block-diagonal factors (gpb200_fitc_set_blocks)
};

// shared by the units, not exported from libgpb200.so (each `namespace engine` block of the units repeats the attribute)
namespace engine __attribute__((visibility("hidden"))) {

constexpr int TILE = 128;
constexpr int TRSV_FUSED_CTAS_PER_SM = 4;      // single-launch solves run for Npad/128 <= this x SMs (see solve_device)
constexpr double LOG2PI = 1.8378770664093453;
extern std::string g_create_error;     // message of the last failed gpb200_create (one instance, in gpb200.cu)

// ---- NCCL, bound at run time (dlopen) so that single-GPU use has no NCCL dependency -------------
struct NcclApi {
    void* lib = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    bool ok = false;
};
extern NcclApi g_nccl;                 // one instance, in gpb200.cu
bool nccl_load();

// "<call> failed at file:line: reason" into `err`; a CUDA failure also clears the error the runtime keeps for the next
// cudaGetLastError.  Returns `code`.
inline int check_failed(std::string& err, int code, const char* call, const char* file, int line, const char* reason) {
    char buf[512];
    snprintf(buf, sizeof buf, "%s failed at %s:%d: %s", call, file, line, reason);
    err = buf;
    if (code == GPB200_ECUDA) (void)cudaGetLastError();
    return code;
}
inline int cuda_rc(std::string& err, cudaError_t e, const char* call, const char* file, int line) {
    return e == cudaSuccess ? GPB200_OK : check_failed(err, GPB200_ECUDA, call, file, line, cudaGetErrorString(e));
}
inline int nccl_rc(std::string& err, ncclResult_t r, const char* call, const char* file, int line) {
    return r == ncclSuccess ? GPB200_OK
                            : check_failed(err, GPB200_ENCCL, call, file, line, g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "nccl error");
}
// a failure on rank q: in an in-process group the caller holds the leader (shard_entry), so q's message is copied there
inline int rank_failed(gpb200_handle* q, int rc) {
    if (rc && q->grp && q != q->grp->hs[0]) q->grp->hs[0]->err = q->err;
    return rc;
}

#define TRY(rc)        do { if (int rc_ = (rc)) return rc_; } while (0)
#define CK(call)       TRY(cuda_rc(h->err, (call), #call, __FILE__, __LINE__))
#define CKN(call)      TRY(nccl_rc(h->err, (call), #call, __FILE__, __LINE__))
#define SCK(q, call)   TRY(rank_failed(q, cuda_rc((q)->err, (call), #call, __FILE__, __LINE__)))
#define SCKN(q, call)  TRY(rank_failed(q, nccl_rc((q)->err, (call), #call, __FILE__, __LINE__)))
#define FCK(call)      TRY(cuda_rc(f->err, (call), #call, __FILE__, __LINE__))
#define FCKN(call)     TRY(nccl_rc(f->err, (call), #call, __FILE__, __LINE__))

// all-or-nothing workspace: make() allocates the buffers of `group`; if any step fails, the whole group is freed
template <class Group, class Make>
int make_group(Group& group, Make make) {
    const int rc = make();
    if (rc != GPB200_OK) group = {};
    return rc;
}

inline int fail(gpb200_handle* h, int code, const char* msg) {
    if (h) h->err = msg;
    return code;
}
inline int fail(gpb200_fitc* f, int code, const std::string& msg) {
    if (f) f->err = msg;
    return code;
}
#define FSUB(call, who)                                                                            \
    do {                                                                                           \
        int rc_ = (call);                                                                          \
        if (rc_ != GPB200_OK) { f->err = std::string(#call) + ": " + (who)->err; return rc_; }     \
    } while (0)

// a GEMM operand: buffer p with leading dimension ld, read through its tensor map when h's GEMM runs on TMA descriptors
inline GemmBuf gbuf(const gpb200_handle* h, const double* p, const CUtensorMap& map, int64_t ld) {
    return GemmBuf{h->tma_ok ? &map : nullptr, p, ld};
}
// the factorisation, u and the kept append state no longer match the data, the kernel or the inducing points
inline void fitc_invalidate(gpb200_fitc* f) {
    f->factored = f->alpha_ready = f->u_ready = false;
    f->app.sqr_ok = f->app.sums_ok = false;
}

inline GemmBuf bufF(gpb200_handle* h) { return gbuf(h, h->F, h->mapF, h->ld); }
inline GemmBuf bufG(gpb200_handle* h) { return gbuf(h, h->G, h->mapG, h->ld); }
inline GemmBuf bufDinv(gpb200_handle* h) { return gbuf(h, h->Dinv, h->mapDinv, TILE); }
inline GemmBuf bufDinvT(gpb200_handle* h) { return gbuf(h, h->DinvT, h->mapDinvT, TILE); }
inline GemmBuf bufNone() { return GemmBuf{nullptr, nullptr, 0}; }

// where a prediction puts the full covariance Sigma*: nowhere, the caller's host array, or the device (for rand_from_cov)
enum class CovDest { none, host, device };
// mu* (M) and Sigma* (M x M, leading dimension ldc) where a prediction left them on the device
struct DevPrediction { const double *mu, *cov; int64_t ldc; };

// ---- dense engine (gpb200.cu) -------------------------------------------------------------------------------------
cudaError_t launch_gemm(gpb200_handle* h, const GemmDesc& d);
// C[M x N] (+)= alpha A B' on h's DMMA GEMM, A and B whole buffers from (0, 0), C (and the optional transposed copy Ct)
// from (0, 0)
cudaError_t gemm_whole(gpb200_handle* h, GemmBuf a, GemmBuf b, double* c, int64_t ldc, int64_t M, int64_t N, int64_t K,
                       double alpha, double beta, double* ct = nullptr, int64_t ldct = 0, int flags = 0);
cudaError_t trsm_rec_buf(gpb200_handle* h, GemmBuf bk, int rows, int c0, int n);
cudaError_t trsm_right_rec_buf(gpb200_handle* h, GemmBuf bk, int rows, int c0, int n);
cudaError_t solve_device(gpb200_handle* h, double* rhs, double* tmp, double* out);
int check_trsv_watchdog(gpb200_handle* h);
int chol_inplace(gpb200_handle* h);
int rand_from_cov(gpb200_handle* h, int64_t M, const double* cov, int64_t ldc, const double* mu, int64_t nsamp,
                  const double* z, double nugget, double* samples);
float ev_ms(cudaEvent_t a, cudaEvent_t b);

// ---- FSA schedule of the sparse handle (fsa_engine.cu), called by the FITC entry points -----------------------------
void fsa_free(gpb200_fitc* f);
int fsa_check(gpb200_fitc* f, const char* who);
int fsa_factorize(gpb200_fitc* f);
int fsa_mll(gpb200_fitc* f, const double* y_minus_mean, double* alpha, double* mll, double* logdet);
int fsa_grad_noise(gpb200_fitc* f, double* dmll_noise);
int fsa_grad_kernel(gpb200_fitc* f, double* dmll_kernel, double* dmll_xu, double* dmll_x);
int fsa_set_inputs(gpb200_fitc* f, const double* x, int64_t ldx);
size_t fsa_num_chunks(const gpb200_fitc* f);
int fsa_predict(gpb200_fitc* f, int64_t Ms, const double* xs, int64_t ldxs, const int64_t* block_of, double* mu, double* var,
                CovDest cov_to, double* cov, double* dmu, double* dvar, DevPrediction* out);

// ---- FITC (fitc_engine.cu), shared with the FSA schedule --------------------------------------------------------------
int fitc_stage_alloc(gpb200_fitc* f, int64_t nc, const char* who);
cudaError_t fitc_kfu(gpb200_fitc* f, const double* xrows, int64_t nc);
cudaError_t fitc_kuf(gpb200_fitc* f, const double* xrows, int64_t nc);
int xu_contract(gpb200_fitc* f, size_t k, const double* z, int64_t n, const double* W, int sym, const double* mask,
                int accumulate);
int xu_finish(gpb200_fitc* f, size_t k_used, double* dmll_xu);
int x_rows(gpb200_fitc* f, size_t k, const double* xr, int64_t n, const double* W, const double* c, const double* mask,
           const long long* map, double* out, int accumulate);
int x_finish(gpb200_fitc* f, size_t k_used, double* dmll_x);

}  // namespace engine
