// gpb200.cu -- the engine behind the C ABI of include/gpb200.h: device state, the blocked
// factorisation / inverse schedules, and the entry points the reference-side shim binds.
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
#include <cuda.h>
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <limits.h>
#include <nccl.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <string>
#include <vector>

#include "../../include/gpb200.h"
#include "gemm_nt.cuh"
#include "gram.cuh"
#include "gram_fast.cuh"
#include "kprog.cuh"
#include "potrf_base.cuh"
#include "shard_kernels.cuh"
#include "vec.cuh"
#include "fsa.cuh"
#include "gpa.cuh"
#include "fitc_cv.cuh"

namespace {
constexpr int TILE = 128;
constexpr int TRSV_FUSED_CTAS_PER_SM = 4;      // single-launch solves run for Npad/128 <= this x SMs (see solve_device)
constexpr double LOG2PI = 1.8378770664093453;
std::string g_create_error;
}  // namespace

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
    double* x = nullptr;
    KProg prog{};
    std::vector<double> theta;
    bool has_data = false, has_kernel = false, factored = false, inv_ready = false, alpha_ready = false;
    bool s_ready = false;                      // G's lower triangle holds -S of gpb200_gpa_grad (A = S for gpb200_grad_inputs)
    double *F = nullptr, *G = nullptr, *Dinv = nullptr, *DinvT = nullptr, *logd = nullptr;
    double *noise_var = nullptr, *r0 = nullptr, *r1 = nullptr, *y1 = nullptr, *alpha = nullptr, *scal = nullptr;
    double *part = nullptr, *trace_out = nullptr;
    double* tblk = nullptr;                    // Npad scratch vector (block right-hand sides of the sharded solves)
    double* ZdT = nullptr;                     // gpb200_gpa_grad: Npad x 128 clean upper diagonal tiles of Z' (allocated on first use)
    CUtensorMap mapZdT{};
    // TMA-staged SEIso kernels (gram_fast.cu): inputs stored [Npad x dxp] with an even, zero-padded dxp <= 8
    double *xp = nullptr, *xpt = nullptr;      // [Npad x dxp] and its transpose [dxp x Npad]
    int dxp = 0;
    CUtensorMap mapX{}, mapXT{};
    bool xmap_ok = false;
    int64_t capacity = 0;                      // option "capacity": rows reserved for gpb200_append (ElasticGPE's capacity)
    int gram_fast = 1;                         // option "gram_fast": 0 = always the generic kernels of gram.cu
    // cross-validation (gpb200_cv_*): K_y^-1 mirrored to a full symmetric matrix in G; two N x N temporaries
    bool g_sym = false;
    bool cv_m_ok = false;                                       // cvD holds M_j = Z_j K^-1 of the last cv_param call
    double *cvD = nullptr, *cvY = nullptr;
    CUtensorMap mapCvD{}, mapCvY{};
    double* cvblk = nullptr; long long* cvidx = nullptr; int64_t cvblk_cap = 0, cvidx_cap = 0;   // capacities in elements
    // posterior sampling (gpb200_rand): M x M sub-engine for chol(Sigma* + nugget I), normal draws / samples staging
    gpb200_handle* sub = nullptr;
    bool cov_keep_device = false;              // predict: leave the full covariance in Kss (no D2H)
    double *rz = nullptr, *rout = nullptr;
    int64_t rz_rows = 0, rz_cols = 0;
    CUtensorMap mapRz{};
    int* info_dev = nullptr;
    int* flags = nullptr;                      // ready-flags of the single-launch triangular solves (2 x (Npad/128 + 1))
    int trsv_fused = 1;
    int max_resident_ctas = 0;
    int64_t n_noise = 1;
    double nugget = 0.0;
    CUtensorMap mapF{}, mapG{}, mapDinv{}, mapDinvT{};
    bool tma_ok = false;
    // predict workspace
    double *xs = nullptr, *Kst = nullptr, *Kss = nullptr, *pmu = nullptr, *pvar = nullptr, *pkdiag = nullptr;
    int64_t xs_cap = 0, Kst_rows = 0, Kss_rows = 0;
    double* pdx = nullptr; int64_t pdx_rows = 0;   // gpb200_predict_grad: dmu (Mpad x d), then dvar (Mpad x d)
    // gpb200_grad_inputs (first use, freed with the data): a caller's alpha (Npad), the N x d result (Npad x d), and in an
    // in-process group the gathered ranks' results (nranks x Npad x d)
    double* dxin = nullptr;
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
    double* pack[2] = {nullptr, nullptr};      // panel staging (double buffered)
    size_t pack_elems = 0;
    cudaEvent_t ev_packed[2] = {nullptr, nullptr}, ev_bcast[2] = {nullptr, nullptr}, ev_unpacked[2] = {nullptr, nullptr};
    cudaEvent_t ev_x = nullptr, ev_y = nullptr;
    double *ag_send = nullptr, *ag_recv = nullptr;
    size_t ag_send_elems = 0, ag_recv_elems = 0;
    // fused panel broadcast over NVLink peer memory (CUDA IPC): peers' F / Dinv / DinvT / logd / signal words
    bool p2p = false;
    int n_peer = 0;
    int peer_rank[7] = {0, 0, 0, 0, 0, 0, 0};
    double *peer_F[7] = {}, *peer_Dinv[7] = {}, *peer_DinvT[7] = {}, *peer_logd[7] = {};
    int* peer_sig[7] = {};
    int* sig = nullptr;                        // sig[q] = last panel published by rank q (epoch * 65536 + b + 1); sig[8] = watchdog
    int epoch = 0;
    int** peer_sig_dev = nullptr;              // device array: &peer_sig[q][rank]
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
    double* P[4] = {nullptr, nullptr, nullptr, nullptr};   // panel buffers, Npad x NBp (global row order); P[1], P[3] double as NBp x Npad row panels
    double* Sbuf = nullptr;                    // all-gather staging: nranks regions of S_per_rank doubles; scratch of the inverse sweep
    size_t S_per_rank = 0;
    CUtensorMap mapP[4] = {}, mapXR[2] = {}, mapS{};
    double* XRbig[2] = {nullptr, nullptr};     // row-panel forms X_J of a BATCH of panels (inverse sweep: batched LAUUM part)
    int xr_batch = 1;                          // panels per batch
    CUtensorMap mapXRbig[2] = {};
    double* red = nullptr;                     // small reduction scratch (local group all-reduce)
    int* redi = nullptr;
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
struct gpb200_fitc {
    gpb200_handle* eu = nullptr;     // K_uu  (+1e-10 I)            -> L_uu
    gpb200_handle* es = nullptr;     // Sigma_QR = K_uf L^-1 K_fu + K_uu (+1e-10 I) -> L_s
    int device = 0;
    int64_t N = 0, M = 0, Mpad = 0, Nc = 0;
    int d = 0;
    double *x = nullptr, *xs = nullptr, *lam = nullptr, *y = nullptr, *alpha = nullptr, *tmpn = nullptr;
    double *w = nullptr, *tmpc = nullptr, *zeroc = nullptr, *tmpc2 = nullptr;          // Nc
    double *bvec = nullptr, *uvec = nullptr, *tmpm = nullptr, *rhsm = nullptr, *scal = nullptr;   // Mpad
    double *bufA = nullptr, *bufB = nullptr;   // Nc x Mpad (K_fu chunk) ; Mpad x Nc (K_uf chunk)
    CUtensorMap mapA{}, mapB{}, mapB2{};
    // kernel-gradient workspace (allocated on first use)
    double *bufC = nullptr, *Hbuf = nullptr, *Wbuf = nullptr, *Tbuf = nullptr, *gvec = nullptr, *betav = nullptr;
    double *gpart = nullptr, *gacc = nullptr, *gtmp = nullptr;
    CUtensorMap mapAt{}, mapC{}, mapCt{}, mapH{}, mapT{};
    bool grad_ws = false;
    double* Kss = nullptr; int64_t Kss_rows = 0;      // full predictive covariance (gpb200_fitc_predict_cov)
    double* pdx = nullptr;                            // gpb200_fitc_predict_grad: dmu, dvar of a chunk (2 x Nc x d; first use)
    // posterior sampling (gpb200_fitc_rand): the Ms x Ms sub-engine and the staging of the draws are eu's (rand_from_cov)
    bool cov_keep_device = false;                     // predict_fsa: leave Sigma* in caller order on the device (fsa->Sc)
    double rand_ms[3] = {0, 0, 0};                    // device times of the last rand: Sigma* build, Cholesky, unwhiten!
    double fsag_ms[4] = {0, 0, 0, 0};                 // last predict_fsa_grad, summed over test chunks: predict_fsa's
                                                      // launches, s + second sweep, K_uu^-1 TRSMs, contraction
    // inducing-point gradient (gpb200_fitc_grad_kernel_inducing; first use): dmll/dXu accumulator (M x d), the events
    // around the call (0, 1) and around each contraction launch (2k, 2k + 1 for k >= 1), and the device times of the last
    // call: the contractions summed, the whole call
    double* dxu = nullptr;
    std::vector<cudaEvent_t> xu_ev;
    double xu_ms[2] = {0, 0};
    // cross-validation (gpb200_fitc_get_inverse_diag / _cv_param / _cv_block; allocated on first use, apart from every
    // buffer the likelihood, gradient and prediction schedules keep):
    //   cvG Nc x Mpad: G = dK_fu - 1/2 K_fu Dp of a chunk;  cvGt Mpad x Nc: G' (pass 1), then the Delta-scaled K_uf L^-1;
    //   cvCh Nc x Mpad: Ch = L^-1 K_fu S^-1;  cvP Nc x Mpad: Ch Q (pass 2) or E (fold blocks)
    //   Mpad x Mpad: cvDuu = dK_uu, cvDp = dK_uu K_uu^-1, cvR = K_uf L^-1 G, cvH = K_uf L^-1 Delta L^-1 K_fu, cvQ = H - R - R'
    double *cvG = nullptr, *cvGt = nullptr, *cvCh = nullptr, *cvP = nullptr;
    double *cvDuu = nullptr, *cvDp = nullptr, *cvR = nullptr, *cvH = nullptr, *cvQ = nullptr;
    double *cvalpha = nullptr, *cvdel = nullptr, *cvilam = nullptr, *cvza = nullptr, *cvdg = nullptr;   // N + Nc
    double *cvda = nullptr, *cvq = nullptr, *cvlamV = nullptr, *cvdelV = nullptr, *cvxs = nullptr;     // Nc (cvxs: Nc x d)
    double* cvm = nullptr;                            // 8 x Mpad: K_uf alpha, G' alpha, K_uf L^-1 Delta alpha, beta, R beta, w, tmp
    double* cvout = nullptr; int64_t cvout_rows = 0;  // fold block (padded nV x padded nV)
    long long* cvidx = nullptr;
    CUtensorMap mapCvG{}, mapCvGt{}, mapCvCh{}, mapCvP{}, mapCvDuu{}, mapCvDp{}, mapCvQ{};
    bool cv_ws = false;
    bool cv_m_ok = false;                             // cvDp / cvQ / cvdel hold the state of the last cv_param since factorize
    int cv_param = 0;
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

namespace {

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
} g_nccl;

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

// "<call> failed at file:line: reason" into `err`; a CUDA failure also clears the error the runtime keeps for the next
// cudaGetLastError.  Returns `code`.
int check_failed(std::string& err, int code, const char* call, const char* file, int line, const char* reason) {
    char buf[512];
    snprintf(buf, sizeof buf, "%s failed at %s:%d: %s", call, file, line, reason);
    err = buf;
    if (code == GPB200_ECUDA) (void)cudaGetLastError();
    return code;
}
int cuda_rc(std::string& err, cudaError_t e, const char* call, const char* file, int line) {
    return e == cudaSuccess ? GPB200_OK : check_failed(err, GPB200_ECUDA, call, file, line, cudaGetErrorString(e));
}
int nccl_rc(std::string& err, ncclResult_t r, const char* call, const char* file, int line) {
    return r == ncclSuccess ? GPB200_OK
                            : check_failed(err, GPB200_ENCCL, call, file, line, g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "nccl error");
}
// a failure on rank q: in an in-process group the caller holds the leader (shard_entry), so q's message is copied there
int rank_failed(gpb200_handle* q, int rc) {
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

int fail(gpb200_handle* h, int code, const char* msg) {
    if (h) h->err = msg;
    return code;
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
    double** ptrs[] = {&h->x, &h->Dinv, &h->DinvT, &h->logd, &h->noise_var, &h->r0, &h->r1,
                       &h->y1, &h->alpha, &h->scal, &h->part, &h->trace_out, &h->xs, &h->Kst, &h->Kss,
                       &h->pmu, &h->pvar, &h->pkdiag, &h->tblk, &h->xp, &h->xpt, &h->ZdT, &h->pdx, &h->dxin};
    h->xmap_ok = false;
    if (h->cvD) cudaFree(h->cvD);
    if (h->cvY) cudaFree(h->cvY);
    if (h->cvblk) cudaFree(h->cvblk);
    if (h->cvidx) cudaFree(h->cvidx);
    h->cvD = h->cvY = h->cvblk = nullptr; h->cvidx = nullptr; h->cvblk_cap = h->cvidx_cap = 0; h->g_sym = false; h->cv_m_ok = false;
    for (auto pp : ptrs) { if (*pp) cudaFree(*pp); *pp = nullptr; }
    if (h->info_dev) { cudaFree(h->info_dev); h->info_dev = nullptr; }
    if (h->flags) { cudaFree(h->flags); h->flags = nullptr; }
    close_peer_maps(h);                        // peers' mappings refer to the old buffers whether or not p2p is switched on
    if (h->sig) { cudaFree(h->sig); h->sig = nullptr; }
    if (h->peer_sig_dev) { cudaFree(h->peer_sig_dev); h->peer_sig_dev = nullptr; }
    for (int i = 0; i < 2; ++i) { if (h->pack[i]) cudaFree(h->pack[i]); h->pack[i] = nullptr; }
    if (h->ag_send) cudaFree(h->ag_send);
    if (h->ag_recv) cudaFree(h->ag_recv);
    h->ag_send = h->ag_recv = nullptr; h->pack_elems = h->ag_send_elems = h->ag_recv_elems = 0;
    h->xs_cap = h->Kst_rows = h->Kss_rows = h->pdx_rows = 0;
    h->has_data = h->factored = h->inv_ready = h->s_ready = h->alpha_ready = false;
}

GemmBuf bufF(gpb200_handle* h) { return GemmBuf{h->tma_ok ? &h->mapF : nullptr, h->F, h->ld}; }
GemmBuf bufG(gpb200_handle* h) { return GemmBuf{h->tma_ok ? &h->mapG : nullptr, h->G, h->ld}; }
GemmBuf bufDinv(gpb200_handle* h) { return GemmBuf{h->tma_ok ? &h->mapDinv : nullptr, h->Dinv, TILE}; }
GemmBuf bufDinvT(gpb200_handle* h) { return GemmBuf{h->tma_ok ? &h->mapDinvT : nullptr, h->DinvT, TILE}; }
GemmBuf bufNone() { return GemmBuf{nullptr, nullptr, 0}; }

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
// rank q owns the 128-wide tile columns t with t % nranks == q of every W21 block; its "slice" is
// the concatenation of those tile columns (local column jl <-> global column ((jl/128)*nranks+q)*128 + jl%128)
__global__ void pack_slices_kernel(const double* __restrict__ G, long long ld, double* __restrict__ out,
                                   int s, int wr, int nranks, int self, int Np) {
    const int z = blockIdx.z;
    const int p = z * 2 * s;
    const int n2 = min(s, Np - p - s);
    const int i = blockIdx.y * 32 + threadIdx.y, jl = blockIdx.x * 32 + threadIdx.x;
    if (n2 <= 0 || i >= n2 || jl >= wr) return;
    const int gj = ((jl >> 7) * nranks + self) * 128 + (jl & 127);
    out[(long long)z * s * wr + (long long)i * wr + jl] = G[(long long)(p + s + i) * ld + p + gj];
}
// scatter the gathered W21 slices of all other ranks into G (lower block) and, transposed, into
// G's strict-upper block
__global__ void unpack_slices_kernel(double* __restrict__ G, long long ld, const double* __restrict__ in,
                                     long long per_rank, int s, int wr, int Np, int nranks, int self) {
    __shared__ double tile[32][33];
    const int batch = (Np + 2 * s - 1) / (2 * s);
    const int z = blockIdx.z % batch;
    const int q = blockIdx.z / batch;
    if (q == self) return;
    const int p = z * 2 * s;
    const int n2 = min(s, Np - p - s);
    if (n2 <= 0) return;
    const double* src = in + (long long)q * per_rank + (long long)z * s * wr;
    const int i0 = blockIdx.y * 32, j0 = blockIdx.x * 32;            // 32 | 128: a block never straddles tiles
    if (i0 >= n2 || j0 >= wr) return;
    const int i = i0 + threadIdx.y, jl = j0 + threadIdx.x;
    double v = 0.0;
    if (i < n2 && jl < wr) {
        v = src[(long long)i * wr + jl];
        const int gj = ((jl >> 7) * nranks + q) * 128 + (jl & 127);
        G[(long long)(p + s + i) * ld + p + gj] = v;
    }
    tile[threadIdx.y][threadIdx.x] = v;
    __syncthreads();
    const int ti = i0 + threadIdx.x, tjl = j0 + threadIdx.y;
    if (ti < n2 && tjl < wr) {
        const int gj = ((tjl >> 7) * nranks + q) * 128 + (tjl & 127);
        G[(long long)(p + gj) * ld + p + s + ti] = tile[threadIdx.x][threadIdx.y];
    }
}

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
    if (need_pack > h->pack_elems) {
        for (int i = 0; i < 2; ++i) {
            if (h->pack[i]) cudaFree(h->pack[i]);
            h->pack[i] = nullptr;
            CK(cudaMalloc(&h->pack[i], sizeof(double) * need_pack));
        }
        h->pack_elems = need_pack;
    }
    const size_t need_recv = Np * Np / 4 + Np * TILE;
    const size_t need_send = need_recv / h->nranks + Np * TILE;
    if (need_recv > h->ag_recv_elems) {
        if (h->ag_recv) cudaFree(h->ag_recv);
        if (h->ag_send) cudaFree(h->ag_send);
        h->ag_recv = h->ag_send = nullptr;
        CK(cudaMalloc(&h->ag_recv, sizeof(double) * need_recv));
        CK(cudaMalloc(&h->ag_send, sizeof(double) * need_send));
        h->ag_recv_elems = need_recv; h->ag_send_elems = need_send;
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


// ---- device-side signalling for the fused (peer-memory) panel broadcast --------------------------
__global__ void signal_peers_kernel(int* const* peer_sig_words, int n_peer, int value) {
    // all panel stores of the preceding kernels are complete (stream order); make them visible
    // system-wide before the flag
    __threadfence_system();
    if ((int)threadIdx.x < n_peer)
        asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(peer_sig_words[threadIdx.x]), "r"(value) : "memory");
}
__global__ void wait_signal_kernel(const int* word, int target, int* err) {
    long long spins = 0;
    int v;
    do {
        asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(word) : "memory");
        if (v >= target) break;
        if (++spins > (1LL << 27)) { atomicExch(err, 1); break; }
        __nanosleep(100);
    } while (true);
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
        signal_peers_kernel<<<1, 32, 0, h->st>>>(h->peer_sig_dev, h->n_peer, base + b + 1);
        ++h->launches;
        CK(cudaGetLastError());
        return GPB200_OK;
    };
    if (owner(0) == me) { int rc = factor_and_publish(0); if (rc) return rc; }
    for (int b = 0; b < nblk; ++b) {
        if (owner(b) != me) {
            wait_signal_kernel<<<1, 1, 0, h->st>>>(h->sig + owner(b), base + b + 1, h->sig + 8);
            ++h->launches;
            CK(cudaGetLastError());
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
        if ((size_t)per_rank > h->ag_send_elems || (size_t)per_rank * R > h->ag_recv_elems)
            return fail(h, GPB200_ECUDA, "inverse_dist: exchange buffers too small");
        dim3 blk(32, 32), grd((wr + 31) / 32, (unsigned)((s + 31) / 32), (unsigned)batch);
        pack_slices_kernel<<<grd, blk, 0, h->st>>>(h->G, h->ld, h->ag_send, (int)s, wr, R, me, Np);
        ++h->launches;
        CK(cudaGetLastError());
        CK(cudaEventRecord(h->ev_x, h->st));
        CK(cudaStreamWaitEvent(h->st_comm, h->ev_x, 0));
        CKN(g_nccl.AllGather(h->ag_send, h->ag_recv, (size_t)per_rank, ncclDouble, h->comm, h->st_comm));
        CK(cudaEventRecord(h->ev_y, h->st_comm));
        CK(cudaStreamWaitEvent(h->st, h->ev_y, 0));
        dim3 grd2((wr + 31) / 32, (unsigned)((s + 31) / 32), (unsigned)(batch * R));
        unpack_slices_kernel<<<grd2, blk, 0, h->st>>>(h->G, h->ld, h->ag_recv, per_rank, (int)s, wr, Np, R, me);
        ++h->launches;
        CK(cudaGetLastError());
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
    if (Mpad > h->xs_cap) {
        if (h->xs) cudaFree(h->xs);
        if (h->pmu) cudaFree(h->pmu);
        if (h->pvar) cudaFree(h->pvar);
        if (h->pkdiag) cudaFree(h->pkdiag);
        h->xs = h->pmu = h->pvar = h->pkdiag = nullptr; h->xs_cap = 0;
        CK(cudaMalloc(&h->xs, sizeof(double) * Mpad * h->d));
        CK(cudaMalloc(&h->pmu, sizeof(double) * Mpad));
        CK(cudaMalloc(&h->pvar, sizeof(double) * Mpad));
        CK(cudaMalloc(&h->pkdiag, sizeof(double) * Mpad));
        h->xs_cap = Mpad;
    }
    if (Mpad > h->Kst_rows) {
        if (h->Kst) cudaFree(h->Kst);
        h->Kst = nullptr; h->Kst_rows = 0;
        CK(cudaMalloc(&h->Kst, sizeof(double) * Mpad * h->Npad));
        h->Kst_rows = Mpad;
        if (h->tma_ok && !gemm_make_tensor_map(&h->mapKst, h->Kst, Mpad, h->Npad, h->Npad))
            return fail(h, GPB200_ECUDA, "cuTensorMapEncodeTiled failed for the predict buffer");
    }
    if (want_cov && Mpad > h->Kss_rows) {
        if (h->Kss) cudaFree(h->Kss);
        h->Kss = nullptr; h->Kss_rows = 0;
        CK(cudaMalloc(&h->Kss, sizeof(double) * Mpad * Mpad));
        h->Kss_rows = Mpad;
    }
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
    GemmBuf bk{h->tma_ok ? &h->mapKst : nullptr, h->Kst, h->Npad};
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
        if (h->rz) cudaFree(h->rz);
        if (h->rout) cudaFree(h->rout);
        h->rz = h->rout = nullptr; h->rz_rows = h->rz_cols = 0;
        CK(cudaMalloc(&h->rz, sizeof(double) * Spad * Mpad));
        CK(cudaMalloc(&h->rout, sizeof(double) * Spad * Mpad));
        h->rz_rows = Spad; h->rz_cols = Mpad;
    }
    const int64_t ldz = h->rz_cols;
    if (h->tma_ok && !gemm_make_tensor_map(&h->mapRz, h->rz, h->rz_rows, ldz, ldz)) return fail(h, GPB200_ECUDA, "rand: tensor map");
    CK(cudaMemsetAsync(h->rz, 0, sizeof(double) * h->rz_rows * ldz, h->st));
    CK(cudaMemcpy2DAsync(h->rz, sizeof(double) * ldz, z, sizeof(double) * M, sizeof(double) * M, nsamp, cudaMemcpyHostToDevice, h->st));
    CK(cudaEventRecord(h->ev3, h->st));
    {   // out[s, m] = sum_{k <= m} Zt[s, k] L[m, k]       (unwhiten!: L Z)
        GemmDesc g = gemm_desc_default();
        g.A = GemmOperand{GemmBuf{h->tma_ok ? &h->mapRz : nullptr, h->rz, ldz}, bufNone(), 0, 0};
        g.B = GemmOperand{bufF(sb), bufNone(), 0, 0};
        g.C = h->rout; g.ldc = ldz; g.M = (int)Spad; g.N = (int)Mpad; g.K = (int)Mpad;
        g.flags = GEMM_KHI_N;
        CK(launch_gemm(h, g));
    }
    CK(add_rowvec_launch(h->rout, ldz, mu, nsamp, M, h->st, &h->launches));                              // + mu
    CK(cudaEventRecord(h->ev2, h->st));
    CK(cudaMemcpy2DAsync(samples, sizeof(double) * M, h->rout, sizeof(double) * ldz, sizeof(double) * M, nsamp, cudaMemcpyDeviceToHost, h->st));
    CK(cudaStreamSynchronize(h->st));
    return GPB200_OK;
}

}  // namespace

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
    if (h->rz) cudaFree(h->rz);
    if (h->rout) cudaFree(h->rout);
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
        CK(cudaMalloc(&h->x, sizeof(double) * Npad * d));      // Npad rows: N may grow up to Npad without realloc
        CK(cudaMalloc(&h->Dinv, sizeof(double) * Npad * TILE));
        CK(cudaMalloc(&h->DinvT, sizeof(double) * Npad * TILE));
        const size_t nv = sizeof(double) * Npad;
        CK(cudaMalloc(&h->logd, nv)); CK(cudaMalloc(&h->noise_var, nv)); CK(cudaMalloc(&h->r0, nv));
        CK(cudaMalloc(&h->r1, nv)); CK(cudaMalloc(&h->y1, nv)); CK(cudaMalloc(&h->alpha, nv)); CK(cudaMalloc(&h->tblk, nv));
        CK(cudaMalloc(&h->scal, sizeof(double) * 16));
        CK(cudaMalloc(&h->info_dev, sizeof(int)));
        CK(cudaMalloc(&h->flags, sizeof(int) * 2 * (Npad / TILE + 1)));
        CK(cudaMalloc(&h->sig, sizeof(int) * 16));
        CK(cudaMemsetAsync(h->sig, 0, sizeof(int) * 16, h->st));
        {
            int sms = 0;
            CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device));
            // a chosen limit on the block count of the single-launch solves, not a residency count: one CTA fits per
            // SM, and above the SM count the schedule relies on in-order CTA dispatch (see solve_device)
            h->max_resident_ctas = sms * TRSV_FUSED_CTAS_PER_SM;
        }
        const int64_t T = Npad / TILE;
        CK(cudaMalloc(&h->part, sizeof(double) * (size_t)(T * (T + 1) / 2) * (GPB200_MAX_THETA + 1)));
        CK(cudaMalloc(&h->trace_out, sizeof(double) * (GPB200_MAX_THETA + 1)));
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
        if (!h->xp) CK(cudaMalloc(&h->xp, sizeof(double) * Npad * h->dxp));
        CK(cudaMemsetAsync(h->xp, 0, sizeof(double) * Npad * h->dxp, h->st));
        CK(cudaMemcpy2DAsync(h->xp, sizeof(double) * h->dxp, x, sizeof(double) * ldx, sizeof(double) * d, N,
                             cudaMemcpyHostToDevice, h->st));
        if (!h->xpt) CK(cudaMalloc(&h->xpt, sizeof(double) * Npad * h->dxp));
        CK(shard_transpose(h->xpt, Npad, h->xp, h->dxp, Npad, h->dxp, h->st, &h->launches));
        h->xmap_ok = gemm_make_tensor_map_plain(&h->mapX, h->xp, N, h->dxp, h->dxp, TILE, h->dxp) &&
                     gemm_make_tensor_map_plain(&h->mapXT, h->xpt, h->dxp, N, Npad, h->dxp, TILE);
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
        TRY(coll_allreduce_sum(Lg, [&](gpb200_handle* q) { return q->trace_out; }, (size_t)trace_num_acc(h->prog, h->d)));
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
        CK(cudaMalloc(&h->ZdT, sizeof(double) * h->Npad * TILE));
        if (h->tma_ok && !gemm_make_tensor_map(&h->mapZdT, h->ZdT, h->Npad, TILE, TILE)) {
            cudaFree(h->ZdT); h->ZdT = nullptr;
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
        g.B = GemmOperand{bufF(h), GemmBuf{h->tma_ok ? &h->mapZdT : nullptr, h->ZdT, TILE}, 0, 0};
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
        if (!q->dxin) SCK(q, cudaMalloc(&q->dxin, sizeof(double) * (size_t)(Npad + nd * (1 + (q->grp ? q->nranks : 0)))));
        if (alpha) TRY(rank_failed(q, upload_padded(q, q->dxin, alpha)));
    }
    auto res = [&](gpb200_handle* q) { return q->dxin + Npad; };
    CK(cudaEventRecord(h->ev0, h->st));
    for (auto* q : L) {
        SeIsoFast sf;
        const double* a = h->s_ready ? nullptr : alpha ? q->dxin : q->alpha;     // S state: A = -G = S
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

int gpb200_predict(gpb200_handle* h, int64_t M, const double* xs, int64_t ldxs, const double* alpha,
                   double* mu, double* var, double* cov) {
    if (!h) return GPB200_EINVAL;
    if (!h->factored) return fail(h, GPB200_ESTATE, "predict: factorize first");
    if (M <= 0 || !xs || ldxs < h->d || !mu) return fail(h, GPB200_EINVAL, "predict: bad M, xs, ldxs or mu");
    if (!alpha && !h->alpha_ready) return fail(h, GPB200_ESTATE, "predict: no alpha (call mll or pass alpha)");
    CK(cudaSetDevice(h->device));
    if (alpha) {
        int rc = upload_padded(h, h->alpha, alpha);
        if (rc) return rc;
        h->alpha_ready = true;
    }
    // chunk the test points so that the M_c x Npad workspace stays below ~16 GB
    int64_t cap = (int64_t)(16.0e9 / (8.0 * (double)h->Npad)) / TILE * TILE;
    if (const char* env = getenv("GPB200_PREDICT_CHUNK")) {            // testing hook: force small chunks
        const int64_t v = atoll(env) / TILE * TILE;
        if (v >= TILE && v < cap) cap = v;
    }
    if (cap < TILE) cap = TILE;
    if (h->sharded && cap > h->Npad) cap = h->Npad;       // a block of V' travels through the Npad x NBp panel buffer
    if (cov) cap = (M + TILE - 1) / TILE * TILE;          // full covariance needs all of V at once
    if (cov && h->sharded && cap > h->Npad) return fail(h, GPB200_EINVAL, "predict: full covariance of more than Npad test points is not supported with sharded storage");
    const bool need_v = (var != nullptr) || (cov != nullptr);
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
            TRY(rank_failed(q, ensure_predict_ws(q, Mc, cov != nullptr)));
            SCK(q, cudaMemcpy2DAsync(q->xs, sizeof(double) * q->d, xs + m0 * ldxs, sizeof(double) * ldxs, sizeof(double) * q->d, Mc,
                                     cudaMemcpyHostToDevice, q->st));
            SCK(q, crossgram_launch(q->prog, q->xs, q->d, Mc, Mpad, q->x, q->d, q->N, q->Npad, q->d, q->Kst, q->Npad, q->st, &q->launches));
            if (need_v) {
                SCK(q, kdiag_launch(q->prog, q->xs, q->d, Mc, q->pvar, q->st, &q->launches));           // running variance starts at k**
                if (cov) SCK(q, gram_full_launch(q->prog, q->xs, q->d, Mc, Mpad, q->d, q->Kss, Mpad, q->st, &q->launches));
            }
        }
        CK(rowdot_launch(h->Kst, h->Npad, h->alpha, Mc, h->Npad, h->pmu, h->st, &h->launches));          // GP.jl:26
        CK(cudaMemcpyAsync(mu + m0, h->pmu, sizeof(double) * Mc, cudaMemcpyDeviceToHost, h->st));
        if (need_v) {
            TRY(shard_predict_solve(Lp, (int)Mpad, Mc, var != nullptr, cov != nullptr));
            if (var) CK(cudaMemcpyAsync(var + m0, h->pvar, sizeof(double) * Mc, cudaMemcpyDeviceToHost, h->st));
            if (cov && !h->cov_keep_device) CK(cudaMemcpy2DAsync(cov, sizeof(double) * M, h->Kss, sizeof(double) * Mpad, sizeof(double) * M, M,
                                          cudaMemcpyDeviceToHost, h->st));
        }
        TRY(sync_all(Lp));
    }
    for (int64_t m0 = 0; !h->sharded && m0 < M; m0 += cap) {
        const int64_t Mc = (M - m0 < cap) ? M - m0 : cap;
        const int64_t Mpad = (Mc + TILE - 1) / TILE * TILE;
        int rc = ensure_predict_ws(h, Mc, cov != nullptr);
        if (rc) return rc;
        CK(cudaMemcpy2DAsync(h->xs, sizeof(double) * h->d, xs + m0 * ldxs, sizeof(double) * ldxs,
                             sizeof(double) * h->d, Mc, cudaMemcpyHostToDevice, h->st));
        CK(crossgram_launch(h->prog, h->xs, h->d, Mc, Mpad, h->x, h->d, h->N, h->Npad, h->d, h->Kst, h->Npad, h->st, &h->launches));
        CK(rowdot_launch(h->Kst, h->Npad, h->alpha, Mc, h->Npad, h->pmu, h->st, &h->launches));          // GP.jl:26
        CK(cudaMemcpyAsync(mu + m0, h->pmu, sizeof(double) * Mc, cudaMemcpyDeviceToHost, h->st));
        if (need_v) {
            CK(trsm_rec(h, (int)Mpad, 0, (int)h->Npad));                                   // whiten!, GP.jl:27
            if (var) {
                CK(kdiag_launch(h->prog, h->xs, h->d, Mc, h->pkdiag, h->st, &h->launches));
                CK(rowvar_launch(h->Kst, h->Npad, h->pkdiag, Mc, h->Npad, h->pvar, h->st, &h->launches));
                CK(cudaMemcpyAsync(var + m0, h->pvar, sizeof(double) * Mc, cudaMemcpyDeviceToHost, h->st));
            }
            if (cov) {                                                                      // GP.jl:51-54
                CK(gram_full_launch(h->prog, h->xs, h->d, Mc, Mpad, h->d, h->Kss, Mpad, h->st, &h->launches));
                GemmBuf bk{h->tma_ok ? &h->mapKst : nullptr, h->Kst, h->Npad};
                GemmDesc g = gemm_desc_default();
                g.A = GemmOperand{bk, bufNone(), 0, 0};
                g.B = GemmOperand{bk, bufNone(), 0, 0};
                g.C = h->Kss; g.ldc = Mpad; g.M = (int)Mpad; g.N = (int)Mpad; g.K = (int)h->Npad;
                g.alpha = -1.0; g.beta = 1.0;
                CK(launch_gemm(h, g));
                if (!h->cov_keep_device)
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
    return GPB200_OK;
}

// Predictive gradients (for ForwardDiff.Dual test inputs of predict_f): mu and var through the same launches as gpb200_predict,
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
        int rc = upload_padded(h, h->alpha, alpha);
        if (rc) return rc;
        h->alpha_ready = true;
    }
    int64_t cap = (int64_t)(16.0e9 / (8.0 * (double)h->Npad)) / TILE * TILE;       // as gpb200_predict
    if (const char* env = getenv("GPB200_PREDICT_CHUNK")) {
        const int64_t v = atoll(env) / TILE * TILE;
        if (v >= TILE && v < cap) cap = v;
    }
    if (cap < TILE) cap = TILE;
    const int d = h->d;
    for (int i = 11; i < 16; ++i) h->ms[i] = 0.0;
    for (int64_t m0 = 0; m0 < M; m0 += cap) {
        const int64_t Mc = (M - m0 < cap) ? M - m0 : cap;
        const int64_t Mpad = (Mc + TILE - 1) / TILE * TILE;
        int rc = ensure_predict_ws(h, Mc, false);
        if (rc) return rc;
        if (Mpad > h->pdx_rows) {
            if (h->pdx) cudaFree(h->pdx);
            h->pdx = nullptr; h->pdx_rows = 0;
            CK(cudaMalloc(&h->pdx, sizeof(double) * 2 * Mpad * d));
            h->pdx_rows = Mpad;
        }
        double* ddmu = h->pdx;
        double* ddvar = h->pdx + h->pdx_rows * d;
        CK(cudaEventRecord(h->ev0, h->st));
        CK(cudaMemcpy2DAsync(h->xs, sizeof(double) * d, xs + m0 * ldxs, sizeof(double) * ldxs, sizeof(double) * d, Mc,
                             cudaMemcpyHostToDevice, h->st));
        CK(crossgram_launch(h->prog, h->xs, d, Mc, Mpad, h->x, d, h->N, h->Npad, d, h->Kst, h->Npad, h->st, &h->launches));
        CK(rowdot_launch(h->Kst, h->Npad, h->alpha, Mc, h->Npad, h->pmu, h->st, &h->launches));
        CK(cudaMemcpyAsync(mu + m0, h->pmu, sizeof(double) * Mc, cudaMemcpyDeviceToHost, h->st));
        CK(cudaEventRecord(h->ev1, h->st));
        if (var) {
            CK(trsm_rec(h, (int)Mpad, 0, (int)h->Npad));                                   // V' = K*' L^-T
            CK(kdiag_launch(h->prog, h->xs, d, Mc, h->pkdiag, h->st, &h->launches));
            CK(rowvar_launch(h->Kst, h->Npad, h->pkdiag, Mc, h->Npad, h->pvar, h->st, &h->launches));
            CK(cudaMemcpyAsync(var + m0, h->pvar, sizeof(double) * Mc, cudaMemcpyDeviceToHost, h->st));
        }
        CK(cudaEventRecord(h->ev2, h->st));
        if (var && m0 == 0) CK(mirror_lower_tiles_launch(h->F, h->ld, h->Npad, h->st, &h->launches));   // L' into F's upper tiles
        CK(cudaEventRecord(h->ev5, h->st));
        if (var) {
            GemmBuf bk{h->tma_ok ? &h->mapKst : nullptr, h->Kst, h->Npad};
            CK(trsm_right_rec_buf(h, bk, (int)Mpad, 0, (int)h->Npad));                     // W' = V' L^-1
        }
        CK(cudaEventRecord(h->ev3, h->st));
        CK(crossgram_dx_launch(h->prog, h->xs, d, Mc, h->x, d, h->N, d, h->alpha, var ? h->Kst : nullptr, nullptr, h->Npad, 1.0,
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
    CK(cudaSetDevice(h->device));
    static double cov_flag;                                     // non-null marker: the covariance stays in h->Kss
    h->cov_keep_device = true;
    int rc = gpb200_predict(h, M, xs, ldxs, alpha, mu_minus_mean, nullptr, &cov_flag);
    h->cov_keep_device = false;
    if (rc) return rc;
    return rand_from_cov(h, M, h->Kss, (M + TILE - 1) / TILE * TILE, h->pmu, nsamp, z, nugget, samples);
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
        h->xmap_ok = gemm_make_tensor_map_plain(&h->mapX, h->xp, Nnew, h->dxp, h->dxp, TILE, h->dxp) &&
                     gemm_make_tensor_map_plain(&h->mapXT, h->xpt, h->dxp, Nnew, Np, h->dxp, TILE);
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
    const size_t nn = sizeof(double) * (size_t)h->Npad * (size_t)h->Npad;
    if (!h->cvD || !h->cvY) {
        if (h->cvD) { cudaFree(h->cvD); h->cvD = nullptr; }
        if (h->cvY) { cudaFree(h->cvY); h->cvY = nullptr; }
        h->cv_m_ok = false;
        if (cudaMalloc(&h->cvD, nn) != cudaSuccess || cudaMalloc(&h->cvY, nn) != cudaSuccess) {
            (void)cudaGetLastError();
            if (h->cvD) { cudaFree(h->cvD); h->cvD = nullptr; }
            h->cvY = nullptr;
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
    if (nV <= h->cvidx_cap && elems <= h->cvblk_cap) return GPB200_OK;
    if (h->cvblk) cudaFree(h->cvblk);
    if (h->cvidx) cudaFree(h->cvidx);
    h->cvblk = nullptr; h->cvidx = nullptr; h->cvblk_cap = h->cvidx_cap = 0;
    CK(cudaMalloc(&h->cvblk, sizeof(double) * elems));
    CK(cudaMalloc(&h->cvidx, sizeof(long long) * nV));
    h->cvblk_cap = elems; h->cvidx_cap = nV;
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
    GemmBuf bD{h->tma_ok ? &h->mapCvD : nullptr, h->cvD, h->Npad}, bY{h->tma_ok ? &h->mapCvY : nullptr, h->cvY, h->Npad};
    const double* Yt = h->cvY;
    if (param >= 0) {
        CK(gram_grad_full_launch(h->prog, h->x, h->d, h->d, h->N, h->Npad, param, h->cvD, h->Npad, h->st, &h->launches));
        GemmDesc g = gemm_desc_default();                           // Y' = K^-1 D   (both symmetric: NT form)
        g.A = GemmOperand{bufG(h), bufNone(), 0, 0};
        g.B = GemmOperand{bD, bufNone(), 0, 0};
        g.C = h->cvY; g.ldc = h->Npad; g.M = Np; g.N = Np; g.K = Np;
        CK(launch_gemm(h, g));
    } else {
        Yt = h->G;                                                  // noise: Z = K^-1 (crossvalidation.jl:124-126)
    }
    CK(rowdot_launch(Yt, h->Npad, h->alpha, h->N, h->Npad, h->r1, h->st, &h->launches));              // Z_j alpha
    CK(rowdot2_launch(h->G, Yt, h->Npad, h->N, h->Npad, h->y1, h->st, &h->launches));                 // diag(Z_j K^-1) = rowwise <K^-1_i, Y'_i>
    {   // M_j = Y' K^-1  -> cvD (fold sub-blocks)
        GemmDesc g = gemm_desc_default();
        g.A = GemmOperand{param >= 0 ? bY : bufG(h), bufNone(), 0, 0};
        g.B = GemmOperand{bufG(h), bufNone(), 0, 0};
        g.C = h->cvD; g.ldc = h->Npad; g.M = Np; g.N = Np; g.K = Np;
        CK(launch_gemm(h, g));
    }
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
        TRY(coll_allreduce_sum(L, [&](gpb200_handle* q) { return q->cvblk; }, nn, [&](gpb200_handle* q) { return q->cvblk + nn; }));
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
    double* tmp = nullptr;
    const size_t nn = sizeof(double) * (size_t)h->Npad * (size_t)h->Npad;
    CK(cudaMalloc(&tmp, nn));
    cudaError_t e = launch_gram(h, tmp, h->Npad, 0, 1, 0, 0);
    if (e == cudaSuccess)
        e = cudaMemcpy2DAsync(K, sizeof(double) * h->N, tmp, sizeof(double) * h->Npad, sizeof(double) * h->N, h->N,
                              cudaMemcpyDeviceToHost, h->st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->st);
    cudaFree(tmp);
    CK(e);
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
    FsaGemmItem* d = nullptr;
    CK(cudaMalloc(&d, sizeof(FsaGemmItem) * n));
    cudaError_t e = cudaMemcpyAsync(d, v.data(), sizeof(FsaGemmItem) * n, cudaMemcpyHostToDevice, h->st);
    if (e == cudaSuccess) e = fsa_gemm_launch(d, n, h->st, &h->launches);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->st);
    cudaFree(d);
    CK(e);
    return GPB200_OK;
}

int gpb200_potrf_tiles(gpb200_handle* h, int mode, const int64_t* args, int32_t n, int32_t* info) {
    if (!h || !args || !info || (mode != 0 && mode != 1)) return GPB200_EINVAL;
    if (mode == 0 && n != 39) return fail(h, GPB200_EINVAL, "potrf_tiles: mode 0 takes 39 arguments");
    if (mode == 1 && (n <= 0 || n % 6)) return fail(h, GPB200_EINVAL, "potrf_tiles: mode 1 takes 6 arguments per tile");
    CK(cudaSetDevice(h->device));
    int* dinfo = nullptr;
    Potrf128Item* ditems = nullptr;
    const int big = INT_MAX;
    CK(cudaMalloc(&dinfo, sizeof(int)));
    cudaError_t e = cudaMemcpyAsync(dinfo, &big, sizeof(int), cudaMemcpyHostToDevice, h->st);
    if (mode == 0) {
        // G, ldg, F, ldf, Dinv, DinvT, logd, p0, ntiles, tile_stride, n_peer, then per peer (F, Dinv, DinvT, logd)
        const int64_t* a = args;
        PotrfPeers pp{};
        pp.n = (int)std::min<int64_t>(std::max<int64_t>(a[10], 0), 7);
        for (int q = 0; q < pp.n; ++q) {
            pp.F[q] = reinterpret_cast<double*>(a[11 + 4 * q]); pp.Dinv[q] = reinterpret_cast<double*>(a[12 + 4 * q]);
            pp.DinvT[q] = reinterpret_cast<double*>(a[13 + 4 * q]); pp.logd[q] = reinterpret_cast<double*>(a[14 + 4 * q]);
        }
        if (e == cudaSuccess && a[8] > 0)
            e = potrf128_launch(reinterpret_cast<const double*>(a[0]), a[1], reinterpret_cast<double*>(a[2]), a[3],
                                reinterpret_cast<double*>(a[4]), reinterpret_cast<double*>(a[5]), reinterpret_cast<double*>(a[6]),
                                dinfo, (int)a[7], (int)a[8], (int)a[9], h->st, &h->launches, &pp);
    } else {
        const int nt = n / 6;
        std::vector<Potrf128Item> v(nt);
        for (int i = 0; i < nt; ++i) {
            const int64_t* q = args + 6 * i;               // G, Dinv, DinvT, logd, ld, info_base
            v[i] = Potrf128Item{reinterpret_cast<const double*>(q[0]), reinterpret_cast<double*>(q[1]),
                                reinterpret_cast<double*>(q[2]), reinterpret_cast<double*>(q[3]), q[4], (int)q[5], 0};
        }
        if (e == cudaSuccess) e = cudaMalloc(&ditems, sizeof(Potrf128Item) * nt);
        if (e == cudaSuccess) e = cudaMemcpyAsync(ditems, v.data(), sizeof(Potrf128Item) * nt, cudaMemcpyHostToDevice, h->st);
        if (e == cudaSuccess) e = potrf128_ptr_launch(ditems, nt, dinfo, h->st, &h->launches);
    }
    int hinfo = big;
    if (e == cudaSuccess) e = cudaMemcpyAsync(&hinfo, dinfo, sizeof(int), cudaMemcpyDeviceToHost, h->st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->st);
    cudaFree(dinfo);
    if (ditems) cudaFree(ditems);
    CK(e);
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
    int* flags = nullptr;
    CK(cudaMalloc(&flags, sizeof(int) * (nb + 1)));
    cudaError_t e = direction == 0 ? trsv_lower_fwd_fused(F, ldf, D, rhs, out, Npad, flags, h->st, &h->launches)
                                   : trsv_lower_bwd_fused(F, ldf, D, rhs, out, Npad, flags, h->st, &h->launches);
    int wd = 0;
    if (e == cudaSuccess) e = cudaMemcpyAsync(&wd, flags + nb, sizeof(int), cudaMemcpyDeviceToHost, h->st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->st);
    cudaFree(flags);
    CK(e);
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

// Copies a host item list to a new device array (the caller frees it after the synchronize); none for an empty list.
static cudaError_t items_to_device(const void* src, size_t bytes, void** d, cudaStream_t st) {
    *d = nullptr;
    if (!bytes) return cudaSuccess;
    cudaError_t e = cudaMalloc(d, bytes);
    if (e == cudaSuccess) e = cudaMemcpyAsync(*d, src, bytes, cudaMemcpyHostToDevice, st);
    return e;
}

int gpb200_fsa_kernels(gpb200_handle* h, int which, const int64_t* args, int32_t n, const double* fargs, int32_t nf) {
    if (!h || (n > 0 && !args) || which < 0 || which > 11 || nf < 0 || (nf > 0 && !fargs)) return GPB200_EINVAL;
    // fixed arguments before the flattened items, and the item stride (0: no items)
    static const int head[12] = {3, 9, 6, 5, 5, 1, 5, 6, 4, 0, 5, 16};
    static const int stride[12] = {5, 0, 0, 0, 0, 5, 5, 0, 5, 6, 0, 4};
    const int hd = head[which], sd = stride[which];
    if (sd ? (n < hd || (n - hd) % sd) : n != hd) return fail(h, GPB200_EINVAL, "fsa_kernels: wrong argument count for this kernel");
    const int ni = sd ? (n - hd) / sd : 0;
    auto ptr = [&](int i) { return reinterpret_cast<double*>(args[i]); };
    std::vector<FsaGramItem> gitems(sd == 5 ? ni : 0);
    std::vector<FsaRowItem> ritems(sd == 6 ? ni : 0);
    std::vector<FsaDxItem> ditems(sd == 4 ? ni : 0);
    int64_t max_nb = 0;
    for (int k = 0; k < ni; ++k) {
        const int64_t* q = args + hd + sd * k;
        if (sd == 4) {                                   // row, out, b0, nb
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
    const bool prog = which == 0 || which == 6 || which == 8 || which == 11;
    if (prog) {
        const int64_t d = args[which == 8 ? 2 : which == 11 ? 3 : 1];
        if (which == 11 && d > GPB200_MAX_DIMS) return fail(h, GPB200_EINVAL, "fsa_kernels: d above GPB200_MAX_DIMS");
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
    }
    if (!ok) return fail(h, GPB200_EINVAL, "fsa_kernels: a null pointer, a negative size, a bad mode or ld below the row width");
    CK(cudaSetDevice(h->device));
    cudaStream_t st = h->st;
    int64_t* L = &h->launches;
    FsaGramItem* dg = nullptr;
    FsaRowItem* dr = nullptr;
    FsaDxItem* dd = nullptr;
    cudaError_t e = sd == 6   ? items_to_device(ritems.data(), sizeof(FsaRowItem) * ritems.size(), reinterpret_cast<void**>(&dr), st)
                    : sd == 4 ? items_to_device(ditems.data(), sizeof(FsaDxItem) * ditems.size(), reinterpret_cast<void**>(&dd), st)
                              : items_to_device(gitems.data(), sizeof(FsaGramItem) * gitems.size(), reinterpret_cast<void**>(&dg), st);
    if (e == cudaSuccess) {
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
        }
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (dg) cudaFree(dg);
    if (dr) cudaFree(dr);
    if (dd) cudaFree(dd);
    CK(e);
    return GPB200_OK;
}

int gpb200_gram_kernels(gpb200_handle* h, int which, const int64_t* args, int32_t n, const double* fargs, int32_t nf) {
    if (!h || (n > 0 && !args) || which < 0 || which > 10 || nf < 0 || (nf > 0 && !fargs)) return GPB200_EINVAL;
    static const int want[11] = {14, 11, 7, 5, 10, 12, 13, 11, 6, 13, 3};
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
        static const int dpos[10] = {2, 8, 4, 2, 2, 8, 2, 6, 2, 6};
        d = a[dpos[which]];
        if (d < 1 || d > GPB200_MAX_DIMS) return fail(h, GPB200_EINVAL, "gram_kernels: d outside 1 .. GPB200_MAX_DIMS");
        const int32_t extra = (which == 0 || which == 9) ? 1 : 0;       // nugget / c after theta
        if (h->has_kernel && nf != h->prog.n_theta + extra)
            return fail(h, GPB200_EINVAL, "gram_kernels: fargs = theta (+ nugget for gram_lower, c for crossgram_dx)");
        TRY(local_prog(h, "gram_kernels", fargs, h->prog.n_theta, d, P));
    } else if (nf != 0) {
        return fail(h, GPB200_EINVAL, "gram_kernels: mirror_lower_tiles takes no fargs");
    }
    const int np = P.n_theta;
    auto jok = [&](int i) { return a[i] >= 0 && a[i] < np; };
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
    }
    if (!ok) return fail(h, GPB200_EINVAL, "gram_kernels: a null pointer, a negative size, a bad padding, leading dimension or "
                                           "alignment, j outside [0, n_theta) or a bad ownership argument");
    CK(cudaSetDevice(h->device));
    cudaStream_t st = h->st;
    int64_t* L = &h->launches;
    const int id = (int)d;
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
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    CK(e);
    return GPB200_OK;
}

int gpb200_fitc_cv_kernels(gpb200_handle* h, int which, const int64_t* args, int32_t n, const double* fargs, int32_t nf) {
    if (!h || !args || which < 0 || which > 14 || nf < 0 || (nf > 0 && !fargs)) return GPB200_EINVAL;
    static const int want[15] = {14, 14, 4, 8, 5, 5, 10, 6, 5, 6, 5, 9, 7, 3, 13};
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
    } else if (nf != 0) {
        return fail(h, GPB200_EINVAL, "fitc_cv_kernels: fargs = theta for delta and inducing_dx, none otherwise");
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
    }
    CK(e);
    CK(cudaStreamSynchronize(st));
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
    if (!h->peer_sig_dev) CK(cudaMalloc(&h->peer_sig_dev, sizeof(int*) * 8));
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

// ================================================================================================
// FITC -- Fully Independent Training Conditional (src/sparse/fully_indep_train_conditional.jl)
//   update_cK! (:134-156), `\` (:33-36), logdet (:77), dmll_noise (:243-257), predictMVN (:324-332 ->
//   determ_train_conditional.jl:41-59 -> subsetofregressors.jl:302-321).
// The reference materialises K_uf (M x N) and several copies; here N is streamed in chunks through two
// staging buffers and only M x M state persists (H7 of SURVEY.md §7.2): per chunk a cross-Gram, a
// recursive TRSM against L_uu for diag(Q_ff), and one rank-Nc SYRK into Sigma_QR -- all on the DMMA GEMM.
// ================================================================================================
#define FSUB(call, who)                                                                            \
    do {                                                                                           \
        int rc_ = (call);                                                                          \
        if (rc_ != GPB200_OK) { f->err = std::string(#call) + ": " + (who)->err; return rc_; }     \
    } while (0)
// in-place sum over the ranks of a device vector (no-op on one rank)
static int fitc_allreduce(gpb200_fitc* f, double* v, size_t n) {
    if (f->nranks <= 1 || n == 0) return GPB200_OK;
    FCKN(g_nccl.AllReduce(v, v, n, ncclDouble, ncclSum, f->comm, f->eu->st));
    return GPB200_OK;
}

// FSA (mode 3), defined below the FITC entry points
static void fsa_free(gpb200_fitc* f);
static int fsa_check(gpb200_fitc* f, const char* who);
static int fsa_factorize(gpb200_fitc* f);
static int fsa_mll(gpb200_fitc* f, const double* y_minus_mean, double* alpha, double* mll, double* logdet);
static int fsa_grad_noise(gpb200_fitc* f, double* dmll_noise);
static int fsa_grad_kernel(gpb200_fitc* f, double* dmll_kernel, double* dmll_xu);
static size_t fsa_num_chunks(const gpb200_fitc* f);

// cross-validation workspace (gpb200_fitc_cv_*): it depends on N, Nc and Mpad only
static void fitc_cv_free(gpb200_fitc* f) {
    double** ptrs[] = {&f->cvG, &f->cvGt, &f->cvCh, &f->cvP, &f->cvDuu, &f->cvDp, &f->cvR, &f->cvH, &f->cvQ, &f->cvalpha,
                       &f->cvdel, &f->cvilam, &f->cvza, &f->cvdg, &f->cvda, &f->cvq, &f->cvlamV, &f->cvdelV, &f->cvxs,
                       &f->cvm, &f->cvout};
    for (auto pp : ptrs) { if (*pp) cudaFree(*pp); *pp = nullptr; }
    if (f->cvidx) cudaFree(f->cvidx);
    f->cvidx = nullptr; f->cvout_rows = 0;
    f->cv_ws = f->cv_m_ok = false;
}

int gpb200_fitc_comm_init(gpb200_fitc* f, int nranks, int rank, const char* id128) {
    if (!f || !id128 || nranks < 1 || rank < 0 || rank >= nranks) return GPB200_EINVAL;
    if (!nccl_load()) { f->err = "libnccl.so.2 could not be loaded"; return GPB200_ENCCL; }
    FCK(cudaSetDevice(f->device));
    if (f->comm) { g_nccl.CommDestroy(f->comm); f->comm = nullptr; }
    ncclUniqueId id;
    memcpy(&id, id128, 128);
    FCKN(g_nccl.CommInitRank(&f->comm, nranks, id, rank));
    f->nranks = nranks; f->rank = rank;
    f->factored = f->alpha_ready = false;
    return GPB200_OK;
}

void gpb200_fitc_destroy(gpb200_fitc* f) {
    if (!f) return;
    cudaSetDevice(f->device);
    if (f->eu && f->eu->st) cudaStreamSynchronize(f->eu->st);
    double** ptrs[] = {&f->x, &f->xs, &f->lam, &f->y, &f->alpha, &f->tmpn, &f->w, &f->tmpc, &f->zeroc, &f->tmpc2,
                       &f->bvec, &f->uvec, &f->tmpm, &f->rhsm, &f->scal, &f->bufA, &f->bufB,
                       &f->bufC, &f->Hbuf, &f->Wbuf, &f->Tbuf, &f->gvec, &f->betav, &f->gpart, &f->gacc, &f->gtmp, &f->pdx,
                       &f->dxu};
    for (auto pp : ptrs) { if (*pp) cudaFree(*pp); *pp = nullptr; }
    if (f->Kss) cudaFree(f->Kss);
    for (cudaEvent_t e : f->xu_ev) cudaEventDestroy(e);
    fsa_free(f);
    fitc_cv_free(f);
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
    if (N <= 0 || M <= 0 || d <= 0 || !x || !xu || ldx < d || ldxu < d) { f->err = "fitc_set_data: bad arguments"; return GPB200_EINVAL; }
    FCK(cudaSetDevice(f->device));
    FSUB(gpb200_set_data(f->eu, M, d, xu, ldxu), f->eu);
    FSUB(gpb200_set_data(f->es, M, d, xu, ldxu), f->es);
    cudaStream_t st = f->eu->st;
    double** ptrs[] = {&f->x, &f->xs, &f->lam, &f->y, &f->alpha, &f->tmpn, &f->w, &f->tmpc, &f->zeroc, &f->tmpc2,
                       &f->bvec, &f->uvec, &f->tmpm, &f->rhsm, &f->scal, &f->bufA, &f->bufB,
                       &f->bufC, &f->Hbuf, &f->Wbuf, &f->Tbuf, &f->gvec, &f->betav, &f->gpart, &f->gacc, &f->gtmp, &f->pdx,
                       &f->dxu};
    for (auto pp : ptrs) { if (*pp) cudaFree(*pp); *pp = nullptr; }
    f->grad_ws = false;
    fsa_free(f);                                      // the FSA blocks refer to the old observations
    fitc_cv_free(f);
    f->N = N; f->M = M; f->d = d; f->Mpad = f->eu->Npad;
    // chunk of data rows: two staging buffers of ~2 GB each at most
    int64_t nc = (int64_t)(2.0e9 / (8.0 * (double)f->Mpad)) / TILE * TILE;
    const int64_t Nceil = (N + TILE - 1) / TILE * TILE;
    if (nc > 32768) nc = 32768;                       // grid.y limit of the row-scaling kernel
    if (nc > Nceil) nc = Nceil;
    if (nc < TILE) nc = TILE;
    f->Nc = nc;
    FCK(cudaMalloc(&f->x, sizeof(double) * N * d));
    FCK(cudaMalloc(&f->xs, sizeof(double) * nc * d));
    for (double** p : {&f->lam, &f->y, &f->alpha, &f->tmpn}) FCK(cudaMalloc(p, sizeof(double) * (N + TILE)));
    for (double** p : {&f->w, &f->tmpc, &f->zeroc, &f->tmpc2}) FCK(cudaMalloc(p, sizeof(double) * nc));
    for (double** p : {&f->bvec, &f->uvec, &f->tmpm, &f->rhsm}) FCK(cudaMalloc(p, sizeof(double) * f->Mpad));
    FCK(cudaMalloc(&f->scal, sizeof(double) * 16));
    FCK(cudaMalloc(&f->bufA, sizeof(double) * nc * f->Mpad));
    FCK(cudaMalloc(&f->bufB, sizeof(double) * nc * f->Mpad));
    FCK(cudaMemsetAsync(f->zeroc, 0, sizeof(double) * nc, st));
    FCK(cudaMemcpy2DAsync(f->x, sizeof(double) * d, x, sizeof(double) * ldx, sizeof(double) * d, N, cudaMemcpyHostToDevice, st));
    if (f->eu->tma_ok) {
        const bool ok = gemm_make_tensor_map(&f->mapA, f->bufA, nc, f->Mpad, f->Mpad) &&
                        gemm_make_tensor_map(&f->mapB, f->bufB, f->Mpad, nc, nc) &&
                        gemm_make_tensor_map(&f->mapB2, f->bufB, nc, f->Mpad, f->Mpad);
        if (!ok) { f->err = "fitc_set_data: cuTensorMapEncodeTiled failed"; return GPB200_ECUDA; }
    }
    FCK(cudaStreamSynchronize(st));
    f->has_data = true; f->factored = f->alpha_ready = false;
    return GPB200_OK;
}

int gpb200_fitc_set_kernel(gpb200_fitc* f, int32_t n_ops, const int32_t* ops, int32_t n_dims, const int32_t* dims,
                           int32_t n_theta) {
    if (!f) return GPB200_EINVAL;
    FSUB(gpb200_set_kernel(f->eu, n_ops, ops, n_dims, dims, n_theta), f->eu);
    FSUB(gpb200_set_kernel(f->es, n_ops, ops, n_dims, dims, n_theta), f->es);
    f->has_kernel = true; f->factored = f->alpha_ready = false;
    return GPB200_OK;
}

// K_fu chunk (rows r0..r0+nc of x against the inducing points) into bufA [Nc x Mpad]
static cudaError_t fitc_kfu(gpb200_fitc* f, const double* xrows, int64_t nc) {
    return crossgram_launch(f->eu->prog, xrows, f->d, nc, f->Nc, f->eu->x, f->d, f->M, f->Mpad, f->d, f->bufA, f->Mpad, f->eu->st, &f->eu->launches);
}
// K_uf chunk into bufB [Mpad x Nc]
static cudaError_t fitc_kuf(gpb200_fitc* f, const double* xrows, int64_t nc) {
    return crossgram_launch(f->eu->prog, f->eu->x, f->d, f->M, f->Mpad, xrows, f->d, nc, f->Nc, f->d, f->bufB, f->Nc, f->eu->st, &f->eu->launches);
}

int gpb200_fitc_factorize(gpb200_fitc* f, const double* theta, double log_noise) {
    if (!f) return GPB200_EINVAL;
    if (!f->has_data || !f->has_kernel) { f->err = "fitc_factorize: set_data and set_kernel first"; return GPB200_ESTATE; }
    if (!isfinite(log_noise)) { f->err = "fitc_factorize: non-finite logNoise"; return GPB200_EINVAL; }
    if (f->mode == 3) { int rc3 = fsa_check(f, "fitc_factorize"); if (rc3) return rc3; }
    FCK(cudaSetDevice(f->device));
    f->factored = f->alpha_ready = f->cv_m_ok = false;
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
    GemmBuf bA{eu->tma_ok ? &f->mapA : nullptr, f->bufA, f->Mpad};
    GemmBuf bB{eu->tma_ok ? &f->mapB : nullptr, f->bufB, f->Nc};
    for (int64_t r0 = 0; r0 < f->N; r0 += f->Nc) {
        const int64_t nc = std::min(f->Nc, f->N - r0);
        const double* xr = f->x + r0 * f->d;
        if (f->mode == 0) {
            // Lambda_i = sigma^2 + K_ii - |L_uu^-1 K_ui|^2   (fitc.jl:146-148)
            FCK(fitc_kfu(f, xr, nc));
            FCK(trsm_rec_buf(eu, bA, (int)f->Nc, 0, (int)f->Mpad));
            FCK(kdiag_launch(eu->prog, xr, f->d, nc, f->tmpc, st, &eu->launches));
            FCK(rowvar_launch(f->bufA, f->Mpad, f->tmpc, nc, f->Mpad, f->tmpc2, st, &eu->launches));
            FCK(ew_launch(0, nc, f->lam + r0, f->tmpc2, nullptr, nullptr, f->noise_var, st, &eu->launches));
        } else {
            // SoR / DTC: Lambda = sigma^2 I   (subsetofregressors.jl:100: exp(-2 logNoise) * Kuf * Kfu + Kuu)
            FCK(ew_launch(0, nc, f->lam + r0, f->zeroc, nullptr, nullptr, f->noise_var, st, &eu->launches));
        }
        // Sigma_QR += K_uf Lambda^-1 K_fu   (fitc.jl:150), as (K_uf Lambda^-1/2)(K_uf Lambda^-1/2)'
        FCK(fitc_kuf(f, xr, nc));
        FCK(scale_launch(0, f->bufB, f->Nc, f->Mpad, nc, f->lam + r0, st, &eu->launches));
        GemmDesc g = gemm_desc_default();
        g.A = GemmOperand{bB, bufNone(), 0, 0};
        g.B = GemmOperand{bB, bufNone(), 0, 0};
        g.C = es->G; g.ldc = es->ld; g.M = (int)f->Mpad; g.N = (int)f->Mpad; g.K = (int)f->Nc;
        g.alpha = 1.0; g.beta = 1.0; g.flags = GEMM_LOWER_ONLY;
        FCK(launch_gemm(es, g));
    }
    // multi-GPU: Sigma_QR = K_uu + sum over ranks of K_uf L^-1 K_fu  -- the one M x M exchange of the FITC likelihood
    { int rca = fitc_allreduce(f, es->G, (size_t)f->Mpad * (size_t)f->Mpad); if (rca) return rca; }
    int rc = chol_inplace(es);
    if (rc != GPB200_OK) { f->err = "fitc_factorize (Sigma_QR): " + es->err; return rc; }
    f->factored = true;
    return GPB200_OK;
}

// alpha = Sigma^-1 r (fitc.jl:33-36), logdet (fitc.jl:77), mll (GPE.jl:210)
int gpb200_fitc_mll(gpb200_fitc* f, const double* y_minus_mean, double* alpha, double* mll, double* logdet) {
    if (!f || !y_minus_mean || !mll) return GPB200_EINVAL;
    if (!f->factored) { f->err = "fitc_mll: factorize first"; return GPB200_ESTATE; }
    if (f->mode == 3) { FCK(cudaSetDevice(f->device)); return fsa_mll(f, y_minus_mean, alpha, mll, logdet); }
    FCK(cudaSetDevice(f->device));
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    FCK(cudaMemcpyAsync(f->y, y_minus_mean, sizeof(double) * f->N, cudaMemcpyHostToDevice, st));
    // b = K_uf Lambda^-1 r
    FCK(cudaMemsetAsync(f->bvec, 0, sizeof(double) * f->Mpad, st));
    for (int64_t r0 = 0; r0 < f->N; r0 += f->Nc) {
        const int64_t nc = std::min(f->Nc, f->N - r0);
        FCK(fitc_kuf(f, f->x + r0 * f->d, nc));
        FCK(cudaMemsetAsync(f->w, 0, sizeof(double) * f->Nc, st));
        FCK(ew_launch(1, nc, f->w, f->y + r0, f->lam + r0, nullptr, 0.0, st, &eu->launches));
        FCK(rowdot_launch(f->bufB, f->Nc, f->w, f->M, f->Nc, f->tmpm, st, &eu->launches));
        FCK(ew_launch(2, f->M, f->bvec, f->tmpm, nullptr, nullptr, 0.0, st, &eu->launches));
    }
    { int rca = fitc_allreduce(f, f->bvec, (size_t)f->Mpad); if (rca) return rca; }              // b summed over the ranks' rows
    // u = Sigma_QR^-1 b   (== get_alpha_u, fitc.jl:279-286)
    FCK(cudaMemcpyAsync(f->rhsm, f->bvec, sizeof(double) * f->Mpad, cudaMemcpyDeviceToDevice, st));
    FCK(solve_device(es, f->rhsm, f->tmpm, f->uvec));
    // alpha = Lambda^-1 (r - K_fu u)
    for (int64_t r0 = 0; r0 < f->N; r0 += f->Nc) {
        const int64_t nc = std::min(f->Nc, f->N - r0);
        FCK(fitc_kfu(f, f->x + r0 * f->d, nc));
        FCK(rowdot_launch(f->bufA, f->Mpad, f->uvec, nc, f->Mpad, f->tmpc, st, &eu->launches));
        FCK(ew_launch(3, nc, f->alpha + r0, f->y + r0, f->tmpc, f->lam + r0, 0.0, st, &eu->launches));
    }
    FCK(dot_launch(f->y, f->alpha, f->N, f->scal + 0, st, &eu->launches));
    FCK(sum_launch(es->logd, es->Npad, f->scal + 1, st, &eu->launches));
    FCK(sum_launch(eu->logd, eu->Npad, f->scal + 2, st, &eu->launches));
    FCK(ew_launch(4, f->N, f->tmpn, f->lam, nullptr, nullptr, 0.0, st, &eu->launches));
    FCK(sum_launch(f->tmpn, f->N, f->scal + 3, st, &eu->launches));
    double s[5];
    if (f->nranks > 1) {
        // r'alpha, sum log Lambda and N are sums over the ranks' rows; the two M x M log-determinants are replicated
        const double nloc = (double)f->N;
        FCK(cudaMemcpyAsync(f->scal + 8, f->scal + 0, sizeof(double), cudaMemcpyDeviceToDevice, st));
        FCK(cudaMemcpyAsync(f->scal + 9, f->scal + 3, sizeof(double), cudaMemcpyDeviceToDevice, st));
        FCK(cudaMemcpyAsync(f->scal + 10, &nloc, sizeof(double), cudaMemcpyHostToDevice, st));
        { int rca = fitc_allreduce(f, f->scal + 8, 3); if (rca) return rca; }
        FCK(cudaMemcpyAsync(f->scal + 0, f->scal + 8, sizeof(double), cudaMemcpyDeviceToDevice, st));
        FCK(cudaMemcpyAsync(f->scal + 3, f->scal + 9, sizeof(double), cudaMemcpyDeviceToDevice, st));
        FCK(cudaMemcpyAsync(f->scal + 4, f->scal + 10, sizeof(double), cudaMemcpyDeviceToDevice, st));
    }
    FCK(cudaMemcpyAsync(s, f->scal, sizeof(double) * 5, cudaMemcpyDeviceToHost, st));
    if (alpha) FCK(cudaMemcpyAsync(alpha, f->alpha, sizeof(double) * f->N, cudaMemcpyDeviceToHost, st));
    FCK(cudaStreamSynchronize(st));
    FSUB(check_trsv_watchdog(es), es);                                   // the solve for u above
    f->Ntotal = f->nranks > 1 ? s[4] : (double)f->N;
    const double ld = s[1] - s[2] + s[3];
    if (logdet) *logdet = ld;
    *mll = -(s[0] + ld + LOG2PI * f->Ntotal) / 2.0;
    f->alpha_ready = true;
    return GPB200_OK;
}

// dmll_noise (fitc.jl:243-257): sigma^2 * (alpha.alpha - sum 1/Lambda + |L_s^-1 K_uf Lambda^-1|_F^2)
int gpb200_fitc_grad_noise(gpb200_fitc* f, double* dmll_noise) {
    if (!f || !dmll_noise) return GPB200_EINVAL;
    if (!f->factored || !f->alpha_ready) { f->err = "fitc_grad_noise: factorize and mll first"; return GPB200_ESTATE; }
    if (f->mode == 3) { FCK(cudaSetDevice(f->device)); return fsa_grad_noise(f, dmll_noise); }
    FCK(cudaSetDevice(f->device));
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    GemmBuf bA{eu->tma_ok ? &f->mapA : nullptr, f->bufA, f->Mpad};
    for (int64_t r0 = 0; r0 < f->N; r0 += f->Nc) {
        const int64_t nc = std::min(f->Nc, f->N - r0);
        FCK(fitc_kfu(f, f->x + r0 * f->d, nc));
        FCK(scale_launch(1, f->bufA, f->Mpad, nc, f->Mpad, f->lam + r0, st, &eu->launches));
        FCK(trsm_rec_buf(es, bA, (int)f->Nc, 0, (int)f->Mpad));
        FCK(rowvar_launch(f->bufA, f->Mpad, f->zeroc, nc, f->Mpad, f->tmpn + r0, st, &eu->launches));     // = -|row|^2
    }
    FCK(sum_launch(f->tmpn, f->N, f->scal + 0, st, &eu->launches));
    FCK(dot_launch(f->alpha, f->alpha, f->N, f->scal + 1, st, &eu->launches));
    FCK(ew_launch(5, f->N, f->tmpn, f->lam, nullptr, nullptr, 0.0, st, &eu->launches));
    FCK(sum_launch(f->tmpn, f->N, f->scal + 2, st, &eu->launches));
    { int rca = fitc_allreduce(f, f->scal, 3); if (rca) return rca; }                             // sums over the ranks' rows
    double s[3];
    FCK(cudaMemcpyAsync(s, f->scal, sizeof(double) * 3, cudaMemcpyDeviceToHost, st));
    FCK(cudaStreamSynchronize(st));
    *dmll_noise = f->noise_var * (s[1] - s[2] - s[0]);
    return GPB200_OK;
}

// predictive mean / variance (fitc.jl:324-332 -> dtc.jl:41-59 -> sor.jl:302-321):
//   mu = K_xu u ;  var = k_xx - |L_uu^-1 k_ux|^2 + |L_s^-1 k_ux|^2
int gpb200_fitc_predict(gpb200_fitc* f, int64_t Ms, const double* xs, int64_t ldxs, double* mu, double* var) {
    if (!f || Ms <= 0 || !xs || ldxs < f->d || !mu) return GPB200_EINVAL;
    if (!f->factored || !f->alpha_ready) { f->err = "fitc_predict: factorize and mll first"; return GPB200_ESTATE; }
    if (f->mode == 3) { f->err = "fitc_predict: FSA predictions need test blocks"; return GPB200_EINVAL; }
    FCK(cudaSetDevice(f->device));
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    GemmBuf bA{eu->tma_ok ? &f->mapA : nullptr, f->bufA, f->Mpad};
    GemmBuf bB2{eu->tma_ok ? &f->mapB2 : nullptr, f->bufB, f->Mpad};
    for (int64_t m0 = 0; m0 < Ms; m0 += f->Nc) {
        const int64_t mc = std::min(f->Nc, Ms - m0);
        FCK(cudaMemcpy2DAsync(f->xs, sizeof(double) * f->d, xs + m0 * ldxs, sizeof(double) * ldxs, sizeof(double) * f->d,
                              mc, cudaMemcpyHostToDevice, st));
        FCK(fitc_kfu(f, f->xs, mc));
        FCK(rowdot_launch(f->bufA, f->Mpad, f->uvec, mc, f->Mpad, f->tmpc, st, &eu->launches));
        FCK(cudaMemcpyAsync(mu + m0, f->tmpc, sizeof(double) * mc, cudaMemcpyDeviceToHost, st));
        if (var) {
            FCK(cudaMemcpyAsync(f->bufB, f->bufA, sizeof(double) * f->Nc * f->Mpad, cudaMemcpyDeviceToDevice, st));
            FCK(trsm_rec_buf(eu, bA, (int)f->Nc, 0, (int)f->Mpad));
            FCK(trsm_rec_buf(es, bB2, (int)f->Nc, 0, (int)f->Mpad));
            FCK(kdiag_launch(eu->prog, f->xs, f->d, mc, f->tmpc, st, &eu->launches));
            FCK(rowvar_launch(f->bufA, f->Mpad, f->tmpc, mc, f->Mpad, f->tmpc2, st, &eu->launches));       // k_xx - q
            FCK(rowvar_launch(f->bufB, f->Mpad, f->zeroc, mc, f->Mpad, f->w, st, &eu->launches));          // -s
            if (f->mode == 2) {                                                             // SoR: K_xu S^-1 K_ux only (sor.jl:302-321)
                FCK(cudaMemsetAsync(f->tmpc2, 0, sizeof(double) * mc, st));
            }
            FCK(ew_launch(6, mc, f->tmpc, f->tmpc2, f->w, nullptr, 0.0, st, &eu->launches));               // [k_xx - q] + s
            FCK(cudaMemcpyAsync(var + m0, f->tmpc, sizeof(double) * mc, cudaMemcpyDeviceToHost, st));
        }
        FCK(cudaStreamSynchronize(st));
    }
    return GPB200_OK;
}

// Predictive gradients of the sparse models (predict_f with ForwardDiff.Dual inputs): mu and var through
// gpb200_fitc_predict's launches (A = K*u L_uu^-T in bufA, B = K*u L_s^-T in bufB), then W' = A L_uu^-1 - B L_s^-1
// (= K*u K_uu^-1 - K*u Sigma_QR^-1; SoR: - B L_s^-1) by the right-side TRSM on the two M x M sub-engines, whose F holds L'
// in its strict-upper tiles for the call, and the contraction over the inducing points with alpha = u:
//   dmu[m, :] = sum_j dk(x*_m, u_j)/dx*_m u_j,   dvar[m, :] = 2c dk(x*_m, x*_m)/dx*_m - 2 sum_j dk(x*_m, u_j)/dx*_m W'[m, j]
// with c = 1 (FITC, DTC) or 0 (SoR, whose variance has no k_xx).  Single GPU, modes 0-2.
int gpb200_fitc_predict_grad(gpb200_fitc* f, int64_t Ms, const double* xs, int64_t ldxs, double* mu, double* var,
                             double* dmu, double* dvar) {
    if (!f) return GPB200_EINVAL;
    if (!f->factored || !f->alpha_ready) { f->err = "fitc_predict_grad: factorize and mll first"; return GPB200_ESTATE; }
    if (f->mode == 3) { f->err = "fitc_predict_grad: not available for FSA"; return GPB200_EINVAL; }
    if (f->nranks > 1) { f->err = "fitc_predict_grad: single GPU handles only"; return GPB200_EINVAL; }
    if (Ms <= 0 || !xs || ldxs < f->d || !mu || !dmu) { f->err = "fitc_predict_grad: bad Ms, xs, ldxs, mu or dmu"; return GPB200_EINVAL; }
    if (!var != !dvar) { f->err = "fitc_predict_grad: var and dvar must be given together"; return GPB200_EINVAL; }
    FCK(cudaSetDevice(f->device));
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int d = f->d;
    if (!f->pdx) FCK(cudaMalloc(&f->pdx, sizeof(double) * 2 * f->Nc * d));
    double* ddmu = f->pdx;
    double* ddvar = f->pdx + f->Nc * d;
    GemmBuf bA{eu->tma_ok ? &f->mapA : nullptr, f->bufA, f->Mpad};
    GemmBuf bB2{eu->tma_ok ? &f->mapB2 : nullptr, f->bufB, f->Mpad};
    if (var) {
        FCK(mirror_lower_tiles_launch(eu->F, eu->ld, eu->Npad, st, &eu->launches));
        FCK(mirror_lower_tiles_launch(es->F, es->ld, es->Npad, st, &eu->launches));
    }
    for (int64_t m0 = 0; m0 < Ms; m0 += f->Nc) {
        const int64_t mc = std::min(f->Nc, Ms - m0);
        FCK(cudaMemcpy2DAsync(f->xs, sizeof(double) * d, xs + m0 * ldxs, sizeof(double) * ldxs, sizeof(double) * d,
                              mc, cudaMemcpyHostToDevice, st));
        FCK(fitc_kfu(f, f->xs, mc));
        FCK(rowdot_launch(f->bufA, f->Mpad, f->uvec, mc, f->Mpad, f->tmpc, st, &eu->launches));
        FCK(cudaMemcpyAsync(mu + m0, f->tmpc, sizeof(double) * mc, cudaMemcpyDeviceToHost, st));
        if (var) {                                                          // as gpb200_fitc_predict
            FCK(cudaMemcpyAsync(f->bufB, f->bufA, sizeof(double) * f->Nc * f->Mpad, cudaMemcpyDeviceToDevice, st));
            FCK(trsm_rec_buf(eu, bA, (int)f->Nc, 0, (int)f->Mpad));
            FCK(trsm_rec_buf(es, bB2, (int)f->Nc, 0, (int)f->Mpad));
            FCK(kdiag_launch(eu->prog, f->xs, d, mc, f->tmpc, st, &eu->launches));
            FCK(rowvar_launch(f->bufA, f->Mpad, f->tmpc, mc, f->Mpad, f->tmpc2, st, &eu->launches));
            FCK(rowvar_launch(f->bufB, f->Mpad, f->zeroc, mc, f->Mpad, f->w, st, &eu->launches));
            if (f->mode == 2) FCK(cudaMemsetAsync(f->tmpc2, 0, sizeof(double) * mc, st));
            FCK(ew_launch(6, mc, f->tmpc, f->tmpc2, f->w, nullptr, 0.0, st, &eu->launches));
            FCK(cudaMemcpyAsync(var + m0, f->tmpc, sizeof(double) * mc, cudaMemcpyDeviceToHost, st));
            if (f->mode != 2) FCK(trsm_right_rec_buf(eu, bA, (int)f->Nc, 0, (int)f->Mpad));      // A L_uu^-1
            FCK(trsm_right_rec_buf(es, bB2, (int)f->Nc, 0, (int)f->Mpad));                        // B L_s^-1
        }
        FCK(crossgram_dx_launch(eu->prog, f->xs, d, mc, eu->x, d, f->M, d, f->uvec, (var && f->mode != 2) ? f->bufA : nullptr,
                                var ? f->bufB : nullptr, f->Mpad, f->mode == 2 ? 0.0 : 1.0, ddmu, ddvar, st, &eu->launches));
        FCK(cudaMemcpyAsync(dmu + m0 * d, ddmu, sizeof(double) * mc * d, cudaMemcpyDeviceToHost, st));
        if (var) FCK(cudaMemcpyAsync(dvar + m0 * d, ddvar, sizeof(double) * mc * d, cudaMemcpyDeviceToHost, st));
        FCK(cudaStreamSynchronize(st));
    }
    return GPB200_OK;
}

// predictMVN with the FULL predictive covariance (fitc.jl:324-332 -> determ_train_conditional.jl:41-59 ->
// subsetofregressors.jl:302-321):  Sigma* = K** - K*u K_uu^-1 Ku* + K*u S^-1 Ku*   (FITC, DTC);   K*u S^-1 Ku*   (SoR)
// = K** - A A' + B B' with A = K*u L_uu^-T, B = K*u L_s^-T: two whitening TRSMs and two NT GEMMs.  Ms <= one staging chunk.
// Sigma* into f->Kss (leading dimension Ms rounded up to 128) and mu into f->tmpc and mu[Ms], on eu's stream; Ms <= Nc
static int fitc_cov_build(gpb200_fitc* f, int64_t Ms, const double* xs, int64_t ldxs, double* mu) {
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int64_t Mspad = (Ms + TILE - 1) / TILE * TILE;
    if (Mspad > f->Kss_rows) {
        if (f->Kss) cudaFree(f->Kss);
        f->Kss = nullptr; f->Kss_rows = 0;
        FCK(cudaMalloc(&f->Kss, sizeof(double) * Mspad * Mspad));
        f->Kss_rows = Mspad;
    }
    GemmBuf bA{eu->tma_ok ? &f->mapA : nullptr, f->bufA, f->Mpad};
    GemmBuf bB2{eu->tma_ok ? &f->mapB2 : nullptr, f->bufB, f->Mpad};
    FCK(cudaMemcpy2DAsync(f->xs, sizeof(double) * f->d, xs, sizeof(double) * ldxs, sizeof(double) * f->d, Ms, cudaMemcpyHostToDevice, st));
    FCK(fitc_kfu(f, f->xs, Ms));                                         // bufA = K*u  (Ms x Mpad, zero padded rows)
    FCK(rowdot_launch(f->bufA, f->Mpad, f->uvec, Ms, f->Mpad, f->tmpc, st, &eu->launches));
    FCK(cudaMemcpyAsync(mu, f->tmpc, sizeof(double) * Ms, cudaMemcpyDeviceToHost, st));
    FCK(cudaMemcpyAsync(f->bufB, f->bufA, sizeof(double) * f->Nc * f->Mpad, cudaMemcpyDeviceToDevice, st));
    FCK(trsm_rec_buf(es, bB2, (int)Mspad, 0, (int)f->Mpad));             // B = K*u L_s^-T
    if (f->mode != 2) {
        FCK(trsm_rec_buf(eu, bA, (int)Mspad, 0, (int)f->Mpad));         // A = K*u L_uu^-T
        FCK(gram_full_launch(eu->prog, f->xs, f->d, Ms, Mspad, f->d, f->Kss, Mspad, st, &eu->launches));
        GemmDesc g = gemm_desc_default();
        g.A = GemmOperand{bA, bufNone(), 0, 0};
        g.B = GemmOperand{bA, bufNone(), 0, 0};
        g.C = f->Kss; g.ldc = Mspad; g.M = (int)Mspad; g.N = (int)Mspad; g.K = (int)f->Mpad;
        g.alpha = -1.0; g.beta = 1.0;
        FCK(launch_gemm(eu, g));
    } else {
        FCK(cudaMemsetAsync(f->Kss, 0, sizeof(double) * Mspad * Mspad, st));
    }
    {
        GemmDesc g = gemm_desc_default();
        g.A = GemmOperand{bB2, bufNone(), 0, 0};
        g.B = GemmOperand{bB2, bufNone(), 0, 0};
        g.C = f->Kss; g.ldc = Mspad; g.M = (int)Mspad; g.N = (int)Mspad; g.K = (int)f->Mpad;
        g.alpha = 1.0; g.beta = 1.0;
        FCK(launch_gemm(es, g));
    }
    return GPB200_OK;
}

int gpb200_fitc_predict_cov(gpb200_fitc* f, int64_t Ms, const double* xs, int64_t ldxs, double* mu, double* cov) {
    if (!f || Ms <= 0 || !xs || ldxs < f->d || !mu || !cov) return GPB200_EINVAL;
    if (!f->factored || !f->alpha_ready) { f->err = "fitc_predict_cov: factorize and mll first"; return GPB200_ESTATE; }
    if (f->mode == 3) { f->err = "fitc_predict_cov: FSA predictions need test blocks"; return GPB200_EINVAL; }
    if (Ms > f->Nc) { f->err = "fitc_predict_cov: too many test points for one staging chunk"; return GPB200_EINVAL; }
    FCK(cudaSetDevice(f->device));
    TRY(fitc_cov_build(f, Ms, xs, ldxs, mu));
    const int64_t Mspad = (Ms + TILE - 1) / TILE * TILE;
    FCK(cudaMemcpy2DAsync(cov, sizeof(double) * Ms, f->Kss, sizeof(double) * Mspad, sizeof(double) * Ms, Ms, cudaMemcpyDeviceToHost, f->eu->st));
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
static int xu_event_pairs(gpb200_fitc* f, size_t pairs) {
    while (f->xu_ev.size() < 2 * pairs) {
        cudaEvent_t e;
        FCK(cudaEventCreate(&e));
        f->xu_ev.push_back(e);
    }
    return GPB200_OK;
}

// one contraction launch (slot k >= 1 of f->xu_ev) over n rows z against W (ld Mpad) into f->dxu
static int xu_contract(gpb200_fitc* f, size_t k, const double* z, int64_t n, const double* W, int sym, const double* mask,
                       int accumulate) {
    gpb200_handle* eu = f->eu;
    FCK(cudaEventRecord(f->xu_ev[2 * k], eu->st));
    FCK(inducing_dx_launch(eu->prog, eu->x, f->d, f->M, z, f->d, n, f->d, W, f->Mpad, sym, mask, f->dxu, accumulate, eu->st,
                           &eu->launches));
    FCK(cudaEventRecord(f->xu_ev[2 * k + 1], eu->st));
    return GPB200_OK;
}

// after the final synchronize: device times of the call and of its k_used contractions; dmll_xu = dxu / 2
static int xu_finish(gpb200_fitc* f, size_t k_used, double* dmll_xu) {
    std::vector<double> h((size_t)f->M * f->d);
    FCK(cudaMemcpy(h.data(), f->dxu, sizeof(double) * h.size(), cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < h.size(); ++i) dmll_xu[i] = 0.5 * h[i];
    double c = 0.0;
    for (size_t k = 1; k <= k_used; ++k) c += ev_ms(f->xu_ev[2 * k], f->xu_ev[2 * k + 1]);
    f->xu_ms[0] = c;
    f->xu_ms[1] = ev_ms(f->xu_ev[0], f->xu_ev[1]);
    return GPB200_OK;
}

static int fitc_grad(gpb200_fitc* f, double* dmll_kernel, double* dmll_xu, const char* who) {
    if (!f->factored || !f->alpha_ready) { f->err = std::string(who) + ": factorize and mll first"; return GPB200_ESTATE; }
    FCK(cudaSetDevice(f->device));
    if (dmll_xu) {
        const size_t chunks = f->mode == 3 ? fsa_num_chunks(f) : (size_t)((f->N + f->Nc - 1) / f->Nc);
        TRY(xu_event_pairs(f, chunks + 2));
        if (!f->dxu) FCK(cudaMalloc(&f->dxu, sizeof(double) * f->M * f->d));
        FCK(cudaEventRecord(f->xu_ev[0], f->eu->st));
    }
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int np = eu->prog.n_theta;
    const int64_t Mp = f->Mpad, Nc = f->Nc;
    if (!f->grad_ws) {
        FCK(cudaMalloc(&f->bufC, sizeof(double) * Nc * Mp));
        for (double** p : {&f->Hbuf, &f->Wbuf, &f->Tbuf}) FCK(cudaMalloc(p, sizeof(double) * Mp * Mp));
        FCK(cudaMalloc(&f->gvec, sizeof(double) * (f->N + TILE)));
        FCK(cudaMalloc(&f->betav, sizeof(double) * Mp));
        const size_t tiles = (size_t)std::max((Nc / TILE) * (Mp / TILE), (Mp / TILE) * (Mp / TILE));
        FCK(cudaMalloc(&f->gpart, sizeof(double) * tiles * GPB200_MAX_THETA));
        FCK(cudaMalloc(&f->gacc, sizeof(double) * GPB200_MAX_THETA));
        FCK(cudaMalloc(&f->gtmp, sizeof(double) * GPB200_MAX_THETA));
        if (eu->tma_ok) {
            const bool ok = gemm_make_tensor_map(&f->mapAt, f->bufA, Mp, Nc, Nc) && gemm_make_tensor_map(&f->mapC, f->bufC, Nc, Mp, Mp) &&
                            gemm_make_tensor_map(&f->mapCt, f->bufC, Mp, Nc, Nc) && gemm_make_tensor_map(&f->mapH, f->Hbuf, Mp, Mp, Mp) &&
                            gemm_make_tensor_map(&f->mapT, f->Tbuf, Mp, Mp, Mp);
            if (!ok) { f->err = "fitc_grad_kernel: cuTensorMapEncodeTiled failed"; return GPB200_ECUDA; }
        }
        f->grad_ws = true;
    }
    // explicit K_uu^-1 and Sigma_QR^-1 (full symmetric) in the sub-engines' G buffers
    FSUB(gpb200_grad_prepare(eu), eu);
    FSUB(gpb200_grad_prepare(es), es);
    FCK(symmetrize_launch(eu->G, eu->ld, Mp, st, &eu->launches));
    FCK(symmetrize_launch(es->G, es->ld, Mp, st, &eu->launches));
    const bool tma = eu->tma_ok;
    GemmBuf bA{tma ? &f->mapA : nullptr, f->bufA, Mp}, bAt{tma ? &f->mapAt : nullptr, f->bufA, Nc};
    GemmBuf bCt{tma ? &f->mapCt : nullptr, f->bufC, Nc};
    GemmBuf bH{tma ? &f->mapH : nullptr, f->Hbuf, Mp}, bT{tma ? &f->mapT : nullptr, f->Tbuf, Mp};
    // beta = K_uu^-1 (K_uf alpha)
    FCK(cudaMemsetAsync(f->rhsm, 0, sizeof(double) * Mp, st));
    for (int64_t r0 = 0; r0 < f->N; r0 += Nc) {
        const int64_t nc = std::min(Nc, f->N - r0);
        FCK(fitc_kuf(f, f->x + r0 * f->d, nc));
        FCK(cudaMemsetAsync(f->w, 0, sizeof(double) * Nc, st));
        FCK(cudaMemcpyAsync(f->w, f->alpha + r0, sizeof(double) * nc, cudaMemcpyDeviceToDevice, st));
        FCK(rowdot_launch(f->bufB, Nc, f->w, f->M, Nc, f->tmpm, st, &eu->launches));
        FCK(ew_launch(2, f->M, f->rhsm, f->tmpm, nullptr, nullptr, 0.0, st, &eu->launches));
    }
    { int rca = fitc_allreduce(f, f->rhsm, (size_t)Mp); if (rca) return rca; }                    // K_uf alpha over all rows
    FCK(solve_device(eu, f->rhsm, f->tmpm, f->betav));
    FCK(cudaMemsetAsync(f->gacc, 0, sizeof(double) * GPB200_MAX_THETA, st));
    FCK(cudaMemsetAsync(f->Hbuf, 0, sizeof(double) * Mp * Mp, st));
    if (f->mode == 3) return fsa_grad_kernel(f, dmll_kernel, dmll_xu);
    size_t xk = 0;                                                        // contraction launches so far
    for (int64_t r0 = 0; r0 < f->N; r0 += Nc) {
        const int64_t nc = std::min(Nc, f->N - r0);
        const double* xr = f->x + r0 * f->d;
        FCK(fitc_kfu(f, xr, nc));                                         // bufA = K_fu chunk
        {   // P2 = K_fu S^-1 -> bufB (as Nc x Mpad)
            GemmDesc g = gemm_desc_default();
            g.A = GemmOperand{bA, bufNone(), 0, 0};
            g.B = GemmOperand{bufG(es), bufNone(), 0, 0};
            g.C = f->bufB; g.ldc = Mp; g.M = (int)Nc; g.N = (int)Mp; g.K = (int)Mp;
            FCK(launch_gemm(es, g));
        }
        FCK(rowdot2_launch(f->bufA, f->bufB, Mp, nc, Mp, f->tmpc, st, &eu->launches));
        if (f->mode == 0) FCK(fitc_g_launch(nc, f->alpha + r0, f->lam + r0, f->tmpc, f->gvec + r0, st, &eu->launches));
        else FCK(cudaMemsetAsync(f->gvec + r0, 0, sizeof(double) * nc, st));       // SoR part only (sor.jl:219-253)
        {   // P1 = K_fu K_uu^-1 -> bufC
            GemmDesc g = gemm_desc_default();
            g.A = GemmOperand{bA, bufNone(), 0, 0};
            g.B = GemmOperand{bufG(eu), bufNone(), 0, 0};
            g.C = f->bufC; g.ldc = Mp; g.M = (int)Nc; g.N = (int)Mp; g.K = (int)Mp;
            FCK(launch_gemm(eu, g));
        }
        FCK(fitc_wfu_launch(f->bufB, f->bufC, Mp, nc, f->M, f->alpha + r0, f->lam + r0, f->gvec + r0, f->betav, st, &eu->launches));
        FCK(trace_rect_launch(eu->prog, xr, f->d, nc, eu->x, f->d, f->M, f->d, f->bufB, Mp, f->gpart, f->gtmp, st, &eu->launches));
        FCK(ew_launch(2, np, f->gacc, f->gtmp, nullptr, nullptr, 0.0, st, &eu->launches));
        if (dmll_xu) { TRY(xu_contract(f, xk + 1, xr, nc, f->bufB, 0, nullptr, xk > 0)); ++xk; }
        if (f->mode != 0) continue;                                       // no Lambda-derivative terms for SoR / DTC
        // diagonal term sum_i g_i dK_ii/dθ_p (scratch: bufC as np x nc)
        FCK(kdiag_grad_launch(eu->prog, xr, f->d, nc, f->gvec + r0, f->bufC, st, &eu->launches));
        for (int p = 0; p < np; ++p) FCK(sum_launch(f->bufC + (size_t)p * nc, nc, f->gtmp + p, st, &eu->launches));
        FCK(ew_launch(2, np, f->gacc, f->gtmp, nullptr, nullptr, 0.0, st, &eu->launches));
        // H += K_uf diag(g) K_fu
        FCK(crossgram_launch(eu->prog, eu->x, f->d, f->M, Mp, xr, f->d, nc, Nc, f->d, f->bufA, Nc, st, &eu->launches));   // bufA = K_uf chunk (Mpad x Nc)
        FCK(cudaMemcpyAsync(f->bufC, f->bufA, sizeof(double) * Mp * Nc, cudaMemcpyDeviceToDevice, st));
        FCK(colscale_launch(f->bufC, Nc, Mp, nc, f->gvec + r0, st, &eu->launches));
        {
            GemmDesc g = gemm_desc_default();
            g.A = GemmOperand{bAt, bufNone(), 0, 0};
            g.B = GemmOperand{bCt, bufNone(), 0, 0};
            g.C = f->Hbuf; g.ldc = Mp; g.M = (int)Mp; g.N = (int)Mp; g.K = (int)Nc;
            g.alpha = 1.0; g.beta = 1.0;
            FCK(launch_gemm(eu, g));
        }
    }
    // multi-GPU: the per-row traces and H = K_uf diag(g) K_fu are sums over the ranks' rows; the M x M part below is replicated
    { int rca = fitc_allreduce(f, f->gacc, (size_t)np); if (rca) return rca; }
    { int rca = fitc_allreduce(f, f->Hbuf, (size_t)Mp * (size_t)Mp); if (rca) return rca; }
    if (dmll_xu) { int rca = fitc_allreduce(f, f->dxu, (size_t)f->M * f->d); if (rca) return rca; }   // W_fu part over all rows
    {   // T = K_uu^-1 H ; Wbuf = K_uu^-1 T' = K_uu^-1 H K_uu^-1
        GemmDesc g = gemm_desc_default();
        g.A = GemmOperand{bufG(eu), bufNone(), 0, 0};
        g.B = GemmOperand{bH, bufNone(), 0, 0};
        g.C = f->Tbuf; g.ldc = Mp; g.M = (int)Mp; g.N = (int)Mp; g.K = (int)Mp;
        FCK(launch_gemm(eu, g));
        g.B = GemmOperand{bT, bufNone(), 0, 0};
        g.C = f->Wbuf;
        FCK(launch_gemm(eu, g));
    }
    FCK(fitc_wuu_launch(f->Wbuf, f->Wbuf, eu->G, es->G, Mp, f->M, f->betav, st, &eu->launches));
    FCK(trace_rect_launch(eu->prog, eu->x, f->d, f->M, eu->x, f->d, f->M, f->d, f->Wbuf, Mp, f->gpart, f->gtmp, st, &eu->launches));
    FCK(ew_launch(2, np, f->gacc, f->gtmp, nullptr, nullptr, 0.0, st, &eu->launches));
    if (dmll_xu) {
        TRY(xu_contract(f, xk + 1, eu->x, f->M, f->Wbuf, 1, nullptr, 1)); ++xk;
        FCK(cudaEventRecord(f->xu_ev[1], st));
    }
    std::vector<double> out((size_t)std::max(np, 1));
    FCK(cudaMemcpyAsync(out.data(), f->gacc, sizeof(double) * np, cudaMemcpyDeviceToHost, st));
    FCK(cudaStreamSynchronize(st));
    FSUB(check_trsv_watchdog(eu), eu);                                   // the solve for beta above
    if (dmll_kernel) for (int p = 0; p < np; ++p) dmll_kernel[p] = 0.5 * out[p];
    if (dmll_xu) TRY(xu_finish(f, xk, dmll_xu));
    return GPB200_OK;
}

int gpb200_fitc_grad_kernel(gpb200_fitc* f, double* dmll_kernel) {
    if (!f || !dmll_kernel) return GPB200_EINVAL;
    return fitc_grad(f, dmll_kernel, nullptr, "fitc_grad_kernel");
}

int gpb200_fitc_grad_kernel_inducing(gpb200_fitc* f, double* dmll_kernel, double* dmll_xu) {
    if (!f) return GPB200_EINVAL;
    if (!dmll_xu) { f->err = "fitc_grad_kernel_inducing: dmll_xu is required"; return GPB200_EINVAL; }
    return fitc_grad(f, dmll_kernel, dmll_xu, "fitc_grad_kernel_inducing");
}

// Replaces the inducing inputs of both sub-engines in place (same M and d: no buffer is reallocated); the training inputs,
// the kernel program, the FSA blocks and every workspace are kept.  The factorisation, alpha and the cross-validation state
// refer to the old Xu and are invalidated.
int gpb200_fitc_set_inducing(gpb200_fitc* f, int64_t M, const double* xu, int64_t ldxu) {
    if (!f) return GPB200_EINVAL;
    if (!f->has_data) { f->err = "fitc_set_inducing: set_data first"; return GPB200_ESTATE; }
    if (M != f->M || !xu || ldxu < f->d) {
        f->err = "fitc_set_inducing: M must be set_data's, xu non-null and ldxu >= d"; return GPB200_EINVAL;
    }
    FCK(cudaSetDevice(f->device));
    f->factored = f->alpha_ready = f->cv_m_ok = false;
    FSUB(gpb200_set_data(f->eu, M, f->d, xu, ldxu), f->eu);
    FSUB(gpb200_set_data(f->es, M, f->d, xu, ldxu), f->es);
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
    if (f->mode == 3) { f->err = std::string(who) + ": cross-validation is not available for FSA (mode 3)"; return GPB200_EINVAL; }
    if (f->nranks > 1) {
        f->err = std::string(who) + ": cross-validation runs on one GPU; this handle has " + std::to_string(f->nranks) + " ranks";
        return GPB200_EINVAL;
    }
    if (!f->factored || !f->alpha_ready) { f->err = std::string(who) + ": factorize and mll first"; return GPB200_ESTATE; }
    return GPB200_OK;
}

// workspace on first use; K_uu^-1 and S^-1 as full symmetric matrices in the sub-engines' G (the state grad_kernel builds)
static int fitc_cv_prepare(gpb200_fitc* f) {
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int64_t Mp = f->Mpad, Nc = f->Nc, N = f->N;
    if (!f->cv_ws) {
        for (double** p : {&f->cvG, &f->cvGt, &f->cvCh, &f->cvP}) FCK(cudaMalloc(p, sizeof(double) * Nc * Mp));
        for (double** p : {&f->cvDuu, &f->cvDp, &f->cvR, &f->cvH, &f->cvQ}) FCK(cudaMalloc(p, sizeof(double) * Mp * Mp));
        for (double** p : {&f->cvalpha, &f->cvdel, &f->cvilam, &f->cvza, &f->cvdg}) FCK(cudaMalloc(p, sizeof(double) * (N + Nc)));
        for (double** p : {&f->cvda, &f->cvq, &f->cvlamV, &f->cvdelV}) FCK(cudaMalloc(p, sizeof(double) * Nc));
        FCK(cudaMalloc(&f->cvxs, sizeof(double) * Nc * f->d));
        FCK(cudaMalloc(&f->cvm, sizeof(double) * 8 * Mp));
        FCK(cudaMalloc(&f->cvidx, sizeof(long long) * Nc));
        FCK(cudaMemsetAsync(f->cvalpha, 0, sizeof(double) * (N + Nc), st));      // zero tail: chunk vectors are read Nc wide
        if (eu->tma_ok) {
            const bool ok = gemm_make_tensor_map(&f->mapCvGt, f->cvGt, Mp, Nc, Nc) && gemm_make_tensor_map(&f->mapCvCh, f->cvCh, Nc, Mp, Mp) &&
                            gemm_make_tensor_map(&f->mapCvP, f->cvP, Nc, Mp, Mp) && gemm_make_tensor_map(&f->mapCvDuu, f->cvDuu, Mp, Mp, Mp) &&
                            gemm_make_tensor_map(&f->mapCvDp, f->cvDp, Mp, Mp, Mp) && gemm_make_tensor_map(&f->mapCvQ, f->cvQ, Mp, Mp, Mp);
            if (!ok) { f->err = "fitc_cv: cuTensorMapEncodeTiled failed"; return GPB200_ECUDA; }
        }
        f->cv_ws = true;
    }
    FSUB(gpb200_grad_prepare(eu), eu);
    FSUB(gpb200_grad_prepare(es), es);
    FCK(symmetrize_launch(eu->G, eu->ld, Mp, st, &eu->launches));
    FCK(symmetrize_launch(es->G, es->ld, Mp, st, &eu->launches));
    return GPB200_OK;
}

// C[M x N] (+)= alpha A B' on the engine's DMMA GEMM
static cudaError_t fitc_gemm(gpb200_fitc* f, GemmBuf a, GemmBuf b, double* c, int64_t ldc, int64_t M, int64_t N, int64_t K,
                             double alpha, double beta, double* ct = nullptr, int64_t ldct = 0) {
    GemmDesc g = gemm_desc_default();
    g.A = GemmOperand{a, bufNone(), 0, 0};
    g.B = GemmOperand{b, bufNone(), 0, 0};
    g.C = c; g.ldc = ldc; g.M = (int)M; g.N = (int)N; g.K = (int)K;
    g.alpha = alpha; g.beta = beta;
    g.Ct = ct; g.ldct = ldct;
    return launch_gemm(f->eu, g);
}

int gpb200_fitc_get_inverse_diag(gpb200_fitc* f, double* diag) {
    if (!f || !diag) return GPB200_EINVAL;
    TRY(fitc_cv_check(f, "fitc_get_inverse_diag"));
    FCK(cudaSetDevice(f->device));
    TRY(fitc_cv_prepare(f));
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int64_t Mp = f->Mpad, Nc = f->Nc;
    const bool tma = eu->tma_ok;
    GemmBuf bA{tma ? &f->mapA : nullptr, f->bufA, Mp};
    for (int64_t r0 = 0; r0 < f->N; r0 += Nc) {
        const int64_t nc = std::min(Nc, f->N - r0);
        FCK(fitc_kfu(f, f->x + r0 * f->d, nc));                                                   // bufA = K_fu
        FCK(fitc_gemm(f, bA, bufG(es), f->cvCh, Mp, Nc, Mp, Mp, 1.0, 0.0));                      // K_fu S^-1
        FCK(rowdot2_launch(f->bufA, f->cvCh, Mp, nc, Mp, f->cvq, st, &eu->launches));
        FCK(fitc_cv_invdiag_launch(nc, f->lam + r0, f->cvq, f->cvdg + r0, st, &eu->launches));
    }
    FCK(cudaMemcpyAsync(diag, f->cvdg, sizeof(double) * f->N, cudaMemcpyDeviceToHost, st));
    FCK(cudaStreamSynchronize(st));
    return GPB200_OK;
}

int gpb200_fitc_cv_param(gpb200_fitc* f, int32_t param, const double* alpha, double* Zj_alpha, double* diag_ZjSinv) {
    if (!f || !Zj_alpha || !diag_ZjSinv) return GPB200_EINVAL;
    TRY(fitc_cv_check(f, "fitc_cv_param"));
    const int np = f->eu->prog.n_theta;
    if (param < -1 || param >= np) {
        f->err = "fitc_cv_param: param must be -1 (noise variance) or a kernel parameter index below " + std::to_string(np);
        return GPB200_EINVAL;
    }
    FCK(cudaSetDevice(f->device));
    TRY(fitc_cv_prepare(f));
    f->cv_m_ok = false;
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int64_t Mp = f->Mpad, Nc = f->Nc, N = f->N, M = f->M;
    const int d = f->d;
    const bool tma = eu->tma_ok, noise = param < 0;
    const int kind = noise ? 2 : (f->mode == 0 ? 0 : 1);
    GemmBuf bA{tma ? &f->mapA : nullptr, f->bufA, Mp}, bB{tma ? &f->mapB : nullptr, f->bufB, Nc};
    GemmBuf bGt{tma ? &f->mapCvGt : nullptr, f->cvGt, Nc}, bCh{tma ? &f->mapCvCh : nullptr, f->cvCh, Mp};
    GemmBuf bDuu{tma ? &f->mapCvDuu : nullptr, f->cvDuu, Mp}, bDp{tma ? &f->mapCvDp : nullptr, f->cvDp, Mp};
    GemmBuf bQ{tma ? &f->mapCvQ : nullptr, f->cvQ, Mp};
    double *kta = f->cvm, *gta = f->cvm + Mp, *uD = f->cvm + 2 * Mp, *beta = f->cvm + 3 * Mp;
    double *rb = f->cvm + 4 * Mp, *w = f->cvm + 5 * Mp, *tmp = f->cvm + 6 * Mp;
    if (alpha) FCK(cudaMemcpyAsync(f->cvalpha, alpha, sizeof(double) * N, cudaMemcpyHostToDevice, st));
    else FCK(cudaMemcpyAsync(f->cvalpha, f->alpha, sizeof(double) * N, cudaMemcpyDeviceToDevice, st));
    FCK(ew_launch(5, N, f->cvilam, f->lam, nullptr, nullptr, 0.0, st, &eu->launches));              // 1 / Lambda
    FCK(cudaMemsetAsync(f->cvm, 0, sizeof(double) * 8 * Mp, st));
    FCK(cudaMemsetAsync(f->cvR, 0, sizeof(double) * Mp * Mp, st));
    FCK(cudaMemsetAsync(f->cvH, 0, sizeof(double) * Mp * Mp, st));
    if (!noise) {   // Dp = dK_uu K_uu^-1
        FCK(gram_grad_full_launch(eu->prog, eu->x, d, d, M, Mp, param, f->cvDuu, Mp, st, &eu->launches));
        FCK(fitc_gemm(f, bDuu, bufG(eu), f->cvDp, Mp, Mp, Mp, Mp, 1.0, 0.0));
    }
    // pass 1: Delta, R, H, K_uf alpha, G'alpha, K_uf L^-1 Delta alpha
    for (int64_t r0 = 0; r0 < N; r0 += Nc) {
        const int64_t nc = std::min(Nc, N - r0);
        const double* xr = f->x + r0 * d;
        FCK(fitc_kfu(f, xr, nc));                                                                     // bufA = K_fu
        if (!noise) {
            FCK(crossgram_grad_launch(eu->prog, xr, d, nc, Nc, eu->x, d, M, Mp, d, param, f->cvG, Mp, st, &eu->launches));
            if (kind == 0) FCK(fitc_gemm(f, bA, bufG(eu), f->bufB, Mp, Nc, Mp, Mp, 1.0, 0.0));     // bufB = C (Nc x Mpad)
            FCK(fitc_gemm(f, bA, bDp, f->cvG, Mp, Nc, Mp, Mp, -0.5, 1.0, f->cvGt, Nc));              // G and G'
        }
        FCK(fitc_cv_delta_launch(kind, eu->prog, xr, d, param, f->cvG, f->bufB, Mp, Mp, nc, Nc, f->cvalpha + r0, f->cvdel + r0,
                                 f->cvda, st, &eu->launches));
        FCK(fitc_kuf(f, xr, nc));                                                                     // bufB = K_uf
        FCK(rowdot_launch(f->bufB, Nc, f->cvalpha + r0, M, Nc, tmp, st, &eu->launches));
        FCK(ew_launch(2, M, kta, tmp, nullptr, nullptr, 0.0, st, &eu->launches));
        FCK(colscale_launch(f->bufB, Nc, Mp, nc, f->cvilam + r0, st, &eu->launches));                // K_uf L^-1
        FCK(rowdot_launch(f->bufB, Nc, f->cvda, M, Nc, tmp, st, &eu->launches));
        FCK(ew_launch(2, M, uD, tmp, nullptr, nullptr, 0.0, st, &eu->launches));
        if (!noise) {
            FCK(rowdot_launch(f->cvGt, Nc, f->cvalpha + r0, M, Nc, tmp, st, &eu->launches));
            FCK(ew_launch(2, M, gta, tmp, nullptr, nullptr, 0.0, st, &eu->launches));
            FCK(fitc_gemm(f, bB, bGt, f->cvR, Mp, Mp, Mp, Nc, 1.0, 1.0));                           // R += K_uf L^-1 G
        }
        if (kind != 1) {                                                                              // H += K_uf L^-1 Delta L^-1 K_fu
            FCK(cudaMemcpyAsync(f->cvGt, f->bufB, sizeof(double) * Mp * Nc, cudaMemcpyDeviceToDevice, st));
            FCK(colscale_launch(f->cvGt, Nc, Mp, nc, f->cvdel + r0, st, &eu->launches));
            FCK(fitc_gemm(f, bB, bGt, f->cvH, Mp, Mp, Mp, Nc, 1.0, 1.0));
        }
    }
    FCK(rowdot_launch(eu->G, eu->ld, kta, M, Mp, beta, st, &eu->launches));                         // beta = K_uu^-1 K_uf alpha
    FCK(rowdot_launch(f->cvR, Mp, beta, M, Mp, rb, st, &eu->launches));
    FCK(fitc_cv_wvec_launch(M, w, gta, uD, rb, st, &eu->launches));
    FCK(fitc_cv_qs_launch(f->cvQ, f->cvH, f->cvR, Mp, Mp, st, &eu->launches));
    // pass 2: the two N-vectors
    for (int64_t r0 = 0; r0 < N; r0 += Nc) {
        const int64_t nc = std::min(Nc, N - r0);
        const double* xr = f->x + r0 * d;
        FCK(fitc_kfu(f, xr, nc));
        if (!noise) {
            FCK(crossgram_grad_launch(eu->prog, xr, d, nc, Nc, eu->x, d, M, Mp, d, param, f->cvG, Mp, st, &eu->launches));
            FCK(fitc_gemm(f, bA, bDp, f->cvG, Mp, Nc, Mp, Mp, -0.5, 1.0));
        }
        FCK(fitc_gemm(f, bA, bufG(es), f->cvCh, Mp, Nc, Mp, Mp, 1.0, 0.0));
        FCK(scale_launch(1, f->cvCh, Mp, nc, Mp, f->lam + r0, st, &eu->launches));                  // Ch = L^-1 K_fu S^-1
        FCK(fitc_gemm(f, bCh, bQ, f->cvP, Mp, Nc, Mp, Mp, 1.0, 0.0));                                // Ch Q
        FCK(fitc_cv_rows_launch(noise ? nullptr : f->cvG, f->cvCh, f->bufA, f->cvP, Mp, nc, Mp, f->lam + r0, f->cvdel + r0,
                                f->cvalpha + r0, beta, w, f->cvza + r0, f->cvdg + r0, st, &eu->launches));
    }
    FCK(cudaMemcpyAsync(Zj_alpha, f->cvza, sizeof(double) * N, cudaMemcpyDeviceToHost, st));
    FCK(cudaMemcpyAsync(diag_ZjSinv, f->cvdg, sizeof(double) * N, cudaMemcpyDeviceToHost, st));
    FCK(cudaStreamSynchronize(st));
    f->cv_param = param;
    f->cv_m_ok = true;
    return GPB200_OK;
}

int gpb200_fitc_cv_block(gpb200_fitc* f, int32_t which, int64_t nV, const int64_t* idx, double* out) {
    if (!f || !idx || !out) return GPB200_EINVAL;
    TRY(fitc_cv_check(f, "fitc_cv_block"));
    if (which != 0 && which != 1) { f->err = "fitc_cv_block: which must be 0 (Sigma^-1) or 1 (the last cv_param's M_j)"; return GPB200_EINVAL; }
    if (nV < 1 || nV > f->Nc) {
        f->err = "fitc_cv_block: nV must lie in 1.." + std::to_string(f->Nc) + " (one staging chunk)";
        return GPB200_EINVAL;
    }
    for (int64_t r = 0; r < nV; ++r)
        if (idx[r] < 0 || idx[r] >= f->N) { f->err = "fitc_cv_block: index out of range"; return GPB200_EINVAL; }
    if (which == 1 && !f->cv_m_ok) { f->err = "fitc_cv_block: which = 1 needs a fitc_cv_param since the last factorize"; return GPB200_ESTATE; }
    FCK(cudaSetDevice(f->device));
    TRY(fitc_cv_prepare(f));
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int64_t Mp = f->Mpad, M = f->M;
    const int d = f->d;
    const int64_t nVp = (nV + TILE - 1) / TILE * TILE;
    const bool tma = eu->tma_ok;
    if (nVp > f->cvout_rows) {
        if (f->cvout) cudaFree(f->cvout);
        f->cvout = nullptr; f->cvout_rows = 0;
        FCK(cudaMalloc(&f->cvout, sizeof(double) * nVp * nVp));
        f->cvout_rows = nVp;
    }
    GemmBuf bA{tma ? &f->mapA : nullptr, f->bufA, Mp}, bB2{tma ? &f->mapB2 : nullptr, f->bufB, Mp};
    GemmBuf bCh{tma ? &f->mapCvCh : nullptr, f->cvCh, Mp}, bP{tma ? &f->mapCvP : nullptr, f->cvP, Mp};
    GemmBuf bDp{tma ? &f->mapCvDp : nullptr, f->cvDp, Mp}, bQ{tma ? &f->mapCvQ : nullptr, f->cvQ, Mp};
    FCK(cudaMemcpyAsync(f->cvidx, idx, sizeof(long long) * nV, cudaMemcpyHostToDevice, st));
    FCK(fitc_cv_gather_launch(nV, f->cvidx, f->x, d, d, f->cvxs, f->lam, f->cvlamV, which == 1 ? f->cvdel : nullptr, f->cvdelV,
                              st, &eu->launches));
    FCK(crossgram_launch(eu->prog, f->cvxs, d, nV, nVp, eu->x, d, M, Mp, d, f->bufA, Mp, st, &eu->launches));   // K_V
    FCK(fitc_gemm(f, bA, bufG(es), f->cvCh, Mp, nVp, Mp, Mp, 1.0, 0.0));
    FCK(scale_launch(1, f->cvCh, Mp, nV, Mp, f->cvlamV, st, &eu->launches));                       // Ch_V
    if (which == 0) {   // Sigma^-1[V,V] = diag(1/L_V) - Ch_V (L_V^-1 K_V)'
        FCK(cudaMemcpyAsync(f->bufB, f->bufA, sizeof(double) * nVp * Mp, cudaMemcpyDeviceToDevice, st));
        FCK(scale_launch(1, f->bufB, Mp, nV, Mp, f->cvlamV, st, &eu->launches));
        FCK(fitc_gemm(f, bCh, bB2, f->cvout, nVp, nVp, nVp, Mp, -1.0, 0.0));
    } else {            // (Sigma^-1 dSigma_j Sigma^-1)[V,V] = diag(Delta_V / L_V^2) + E_V Ch_V' + Ch_V E_V'
        const bool noise = f->cv_param < 0;
        if (!noise) {
            FCK(crossgram_grad_launch(eu->prog, f->cvxs, d, nV, nVp, eu->x, d, M, Mp, d, f->cv_param, f->cvG, Mp, st, &eu->launches));
            FCK(fitc_gemm(f, bA, bDp, f->cvG, Mp, nVp, Mp, Mp, -0.5, 1.0));
        }
        FCK(fitc_gemm(f, bCh, bQ, f->cvP, Mp, nVp, Mp, Mp, 0.5, 0.0));
        FCK(fitc_cv_eblock_launch(f->cvP, noise ? nullptr : f->cvG, f->bufA, Mp, nV, Mp, f->cvlamV, f->cvdelV, st, &eu->launches));
        FCK(fitc_gemm(f, bP, bCh, f->cvout, nVp, nVp, nVp, Mp, 1.0, 0.0));
        FCK(fitc_gemm(f, bCh, bP, f->cvout, nVp, nVp, nVp, Mp, 1.0, 1.0));
    }
    FCK(fitc_cv_diag_launch(f->cvout, nVp, nV, which, f->cvlamV, f->cvdelV, st, &eu->launches));
    FCK(cudaMemcpy2DAsync(out, sizeof(double) * nV, f->cvout, sizeof(double) * nVp, sizeof(double) * nV, nV, cudaMemcpyDeviceToHost, st));
    FCK(cudaStreamSynchronize(st));
    return GPB200_OK;
}

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
};
struct Fsa {
    int64_t nblocks = 0, Np = 0, n_pad = 0, packed = 0;
    int max_tiles = 0;
    std::vector<FsaChunk> chunks;
    double *xb = nullptr, *mask = nullptr, *X = nullptr, *LT = nullptr, *logd = nullptr;
    double *r = nullptr, *a = nullptr, *t1 = nullptr, *t2 = nullptr;
    long long *pos = nullptr, *bstart = nullptr, *boff = nullptr;
    int *rblk = nullptr, *bsize = nullptr, *info = nullptr;
    FsaGemmItem* gitems = nullptr;
    Potrf128Item* litems = nullptr;
    FsaGramItem* gramitems = nullptr;
    CUtensorMap mapWt{};                                // bufA as Mpad x Nc (W' = K_uf L_Lambda^-T of a chunk)
    double *Gpk = nullptr, *gpart = nullptr, *ones = nullptr;   // kernel gradient: one chunk's G_i blocks, trace partials, 1s
    std::vector<long long> bstart_h, boff_h;
    std::vector<int> bsize_h, bchunk_h;                 // bchunk_h[b]: staging chunk of block b
    // predictions (gpb200_fitc_predict_fsa, allocated on first use): V* = K_*u L_uu^-T, the C / G tiles of the test rows
    // (Nc x 2048 each), the per-row vectors, and the per-call work lists
    double *Vs = nullptr, *Cb = nullptr, *Gb = nullptr, *pvec = nullptr;
    CUtensorMap mapVs{};
    FsaGemmItem* pg = nullptr; FsaGramItem* px = nullptr; FsaRowItem* pr = nullptr;
    size_t pg_cap = 0, px_cap = 0, pr_cap = 0;
    // gpb200_fitc_rand: Sigma* gathered into the caller's order (Ms x Ms, dense) through the test-point permutation pp
    double* Sc = nullptr; long long* pp = nullptr;
    size_t Sc_cap = 0, pp_cap = 0;
    // gpb200_fitc_predict_fsa_grad (first use): the s K_ub' tiles of the test rows (Nc x 2048), Z = K_*u + E K_fu / 2
    // (Nc x Mpad), dmu / dvar in the caller's order (2 x Ms x d) and the contraction's items
    double *Tb = nullptr, *Zb = nullptr, *pdx = nullptr;
    CUtensorMap mapZb{};
    FsaDxItem* pdi = nullptr;
    size_t pdx_cap = 0, pdi_cap = 0;
};

static size_t fsa_num_chunks(const gpb200_fitc* f) { return f->fsa ? f->fsa->chunks.size() : 0; }

static void fsa_free(gpb200_fitc* f) {
    if (!f->fsa) return;
    Fsa* s = f->fsa;
    void* ptrs[] = {s->xb, s->mask, s->X, s->LT, s->logd, s->r, s->a, s->t1, s->t2, s->pos, s->bstart, s->boff,
                    s->rblk, s->bsize, s->info, s->gitems, s->litems, s->gramitems, s->Gpk, s->gpart, s->ones,
                    s->Vs, s->Cb, s->Gb, s->pvec, s->pg, s->px, s->pr, s->Sc, s->pp, s->Tb, s->Zb, s->pdx, s->pdi};
    for (void* p : ptrs) if (p) cudaFree(p);
    delete s;
    f->fsa = nullptr;
}

int gpb200_fitc_set_blocks(gpb200_fitc* f, int64_t nblocks, const int64_t* block_ptr, const int64_t* idx) {
    if (!f) return GPB200_EINVAL;
    if (!f->has_data) { f->err = "fitc_set_blocks: set_data first"; return GPB200_ESTATE; }
    if (nblocks < 1 || !block_ptr || !idx) { f->err = "fitc_set_blocks: bad arguments"; return GPB200_EINVAL; }
    const int64_t N = f->N;
    if (block_ptr[0] != 0 || block_ptr[nblocks] != N) {
        f->err = "fitc_set_blocks: the blocks must partition the N training points (block_ptr[0] = 0, block_ptr[nblocks] = N)";
        return GPB200_EINVAL;
    }
    int64_t Np = 0, packed = 0;
    int max_tiles = 0;
    for (int64_t b = 0; b < nblocks; ++b) {
        const int64_t n = block_ptr[b + 1] - block_ptr[b];
        if (n < 0) { f->err = "fitc_set_blocks: block_ptr must be non-decreasing"; return GPB200_EINVAL; }
        if (n > FSA_MAX_BLOCK) { f->err = "fitc_set_blocks: a block holds more than 2048 points"; return GPB200_EINVAL; }
        const int64_t B = (n + TILE - 1) / TILE * TILE;
        if (B > f->Nc) { f->err = "fitc_set_blocks: a block does not fit one staging chunk"; return GPB200_EINVAL; }
        Np += B; packed += B * B;
        max_tiles = std::max(max_tiles, (int)(B / TILE));
    }
    std::vector<char> seen((size_t)N, 0);
    for (int64_t k = 0; k < N; ++k) {
        const int64_t i = idx[k];
        if (i < 0 || i >= N || seen[(size_t)i]) {
            f->err = "fitc_set_blocks: the blocks must partition 0..N-1 (an index is out of range or repeated)";
            return GPB200_EINVAL;
        }
        seen[(size_t)i] = 1;
    }
    FCK(cudaSetDevice(f->device));
    fsa_free(f);
    f->factored = f->alpha_ready = false;
    {
        // set_data sizes the staging chunk to N; the padded blocks and the padded test groups of FSA predictions need the
        // full chunk, so grow it to the cap set_data applies to large N (the buffers are re-made, the gradient workspace freed)
        const int64_t cap = std::min<int64_t>((int64_t)(2.0e9 / (8.0 * (double)f->Mpad)) / TILE * TILE, 32768);
        if (cap > f->Nc) {
            double** ptrs[] = {&f->xs, &f->w, &f->tmpc, &f->zeroc, &f->tmpc2, &f->bufA, &f->bufB, &f->bufC, &f->Hbuf, &f->Wbuf,
                               &f->Tbuf, &f->gvec, &f->betav, &f->gpart, &f->gacc, &f->gtmp, &f->pdx};
            for (auto pp : ptrs) { if (*pp) cudaFree(*pp); *pp = nullptr; }
            f->grad_ws = false;
            const int64_t nc = cap;
            f->Nc = nc;
            FCK(cudaMalloc(&f->xs, sizeof(double) * nc * f->d));
            for (double** q : {&f->w, &f->tmpc, &f->zeroc, &f->tmpc2}) FCK(cudaMalloc(q, sizeof(double) * nc));
            FCK(cudaMalloc(&f->bufA, sizeof(double) * nc * f->Mpad));
            FCK(cudaMalloc(&f->bufB, sizeof(double) * nc * f->Mpad));
            FCK(cudaMemset(f->zeroc, 0, sizeof(double) * nc));
            if (f->eu->tma_ok) {
                const bool ok = gemm_make_tensor_map(&f->mapA, f->bufA, nc, f->Mpad, f->Mpad) &&
                                gemm_make_tensor_map(&f->mapB, f->bufB, f->Mpad, nc, nc) &&
                                gemm_make_tensor_map(&f->mapB2, f->bufB, nc, f->Mpad, f->Mpad);
                if (!ok) { f->err = "fitc_set_blocks: cuTensorMapEncodeTiled failed"; return GPB200_ECUDA; }
            }
        }
    }
    Fsa* s = new Fsa();
    f->fsa = s;
    s->nblocks = nblocks; s->Np = Np; s->n_pad = Np - N; s->packed = packed; s->max_tiles = max_tiles;
    cudaStream_t st = f->eu->st;
    const int d = f->d;
    const int64_t Mp = f->Mpad, Nc = f->Nc;
    // host tables: padded layout, positions, the reordered inputs
    std::vector<long long> bstart((size_t)nblocks), boff((size_t)nblocks), pos((size_t)N);
    std::vector<int> bsize((size_t)nblocks), rblk((size_t)Np);
    std::vector<double> mask((size_t)Np, 0.0), xh((size_t)N * d), xb((size_t)Np * d, 0.0);
    FCK(cudaMemcpy(xh.data(), f->x, sizeof(double) * N * d, cudaMemcpyDeviceToHost));
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
    FCK(cudaMalloc(&s->xb, sizeof(double) * Np * d));
    for (double** p : {&s->mask, &s->logd, &s->r, &s->a, &s->t1, &s->t2}) FCK(cudaMalloc(p, sizeof(double) * Np));
    FCK(cudaMalloc(&s->X, sizeof(double) * packed));
    FCK(cudaMalloc(&s->LT, sizeof(double) * packed));
    FCK(cudaMemsetAsync(s->X, 0, sizeof(double) * packed, st));
    FCK(cudaMemsetAsync(s->LT, 0, sizeof(double) * packed, st));
    FCK(cudaMalloc(&s->pos, sizeof(long long) * N));
    FCK(cudaMalloc(&s->bstart, sizeof(long long) * nblocks));
    FCK(cudaMalloc(&s->boff, sizeof(long long) * nblocks));
    FCK(cudaMalloc(&s->bsize, sizeof(int) * nblocks));
    FCK(cudaMalloc(&s->rblk, sizeof(int) * Np));
    FCK(cudaMalloc(&s->info, sizeof(int)));
    // a chunk holds sum B_i <= Nc rows of blocks of at most 2048 rows: its blocks' G_i take at most Nc * 2048 doubles
    const int64_t gpk_elems = std::min<int64_t>(packed, Nc * FSA_MAX_BLOCK);
    FCK(cudaMalloc(&s->Gpk, sizeof(double) * gpk_elems));
    FCK(cudaMalloc(&s->gpart, sizeof(double) * (Nc / TILE) * (FSA_MAX_BLOCK / TILE) * GPB200_MAX_THETA));
    {
        std::vector<double> ones((size_t)Nc, 1.0);
        FCK(cudaMalloc(&s->ones, sizeof(double) * Nc));
        FCK(cudaMemcpy(s->ones, ones.data(), sizeof(double) * Nc, cudaMemcpyHostToDevice));
    }
    FCK(cudaMemcpy(s->xb, xb.data(), sizeof(double) * Np * d, cudaMemcpyHostToDevice));
    FCK(cudaMemcpy(s->mask, mask.data(), sizeof(double) * Np, cudaMemcpyHostToDevice));
    FCK(cudaMemcpy(s->pos, pos.data(), sizeof(long long) * N, cudaMemcpyHostToDevice));
    FCK(cudaMemcpy(s->bstart, bstart.data(), sizeof(long long) * nblocks, cudaMemcpyHostToDevice));
    FCK(cudaMemcpy(s->boff, boff.data(), sizeof(long long) * nblocks, cudaMemcpyHostToDevice));
    FCK(cudaMemcpy(s->bsize, bsize.data(), sizeof(int) * nblocks, cudaMemcpyHostToDevice));
    FCK(cudaMemcpy(s->rblk, rblk.data(), sizeof(int) * Np, cudaMemcpyHostToDevice));
    if (f->eu->tma_ok && !gemm_make_tensor_map(&s->mapWt, f->bufA, Mp, Nc, Nc)) {
        f->err = "fitc_set_blocks: cuTensorMapEncodeTiled failed"; return GPB200_ECUDA;
    }
    s->bstart_h = bstart; s->boff_h = boff; s->bsize_h = bsize;
    s->bchunk_h.assign((size_t)nblocks, 0);
    // work lists: staging chunks of whole blocks, then every launch of factorize / grad_noise as a range of items
    std::vector<FsaGemmItem> gi;
    std::vector<Potrf128Item> li;
    std::vector<FsaGramItem> gr;
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
                    gemm(Xt(b, i, j), bsize[b], f->bufA + (bstart[b] - ch.r0 + i * TILE) * Mp, Mp,
                         f->bufA + (bstart[b] - ch.r0 + j * TILE) * Mp, Mp, Mp, -1.0, 1.0, i == j);
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
                    gemm(f->bufA + u * TILE * Nc + (bstart[b] - ch.r0) + r * TILE, Nc, f->bufB + u * TILE * Nc + (bstart[b] - ch.r0), Nc,
                         Xt(b, r, 0), bsize[b], (int64_t)(r + 1) * TILE, 1.0, 0.0, false);
        close_g(ch.wt);
        open_g(ch.z);
        for (int64_t b = b0; b < b1; ++b)
            for (int64_t u = 0; u < Mp / TILE; ++u)
                for (int r = 0; r < bsize[b] / TILE; ++r)
                    gemm(f->bufB + (bstart[b] - ch.r0 + r * TILE) * Mp + u * TILE, Mp, Lt(b, r, r), bsize[b],
                         f->bufA + u * TILE * Nc + (bstart[b] - ch.r0) + r * TILE, Nc, bsize[b] - (int64_t)r * TILE, 1.0, 0.0, false);
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
                    gemm(Gt(b, i, j), bsize[b], f->bufB + (bstart[b] - ch.r0 + i * TILE) * Mp, Mp,
                         f->bufB + (bstart[b] - ch.r0 + j * TILE) * Mp, Mp, Mp, 1.0, 1.0, false);
        close_g(ch.gyy);
        open_g(ch.gp1t);                                // (P1' G_bd) with P1' = K_uu^-1 K_uf in bufB (Mpad x Nc) -> bufA (Mpad x Nc)
        for (int64_t b = b0; b < b1; ++b)
            for (int64_t u = 0; u < Mp / TILE; ++u)
                for (int r = 0; r < bsize[b] / TILE; ++r)
                    gemm(f->bufA + u * TILE * Nc + (bstart[b] - ch.r0) + r * TILE, Nc, f->bufB + u * TILE * Nc + (bstart[b] - ch.r0), Nc,
                         Gt(b, r, 0), bsize[b], bsize[b], 1.0, 0.0, false);
        close_g(ch.gp1t);
        for (int64_t b = b0; b < b1; ++b) s->bchunk_h[(size_t)b] = (int)s->chunks.size();
        s->chunks.push_back(std::move(ch));
        b0 = b1;
    }
    FCK(cudaMalloc(&s->gitems, sizeof(FsaGemmItem) * std::max<size_t>(gi.size(), 1)));
    FCK(cudaMalloc(&s->litems, sizeof(Potrf128Item) * std::max<size_t>(li.size(), 1)));
    FCK(cudaMalloc(&s->gramitems, sizeof(FsaGramItem) * std::max<size_t>(gr.size(), 1)));
    FCK(cudaMemcpy(s->gitems, gi.data(), sizeof(FsaGemmItem) * gi.size(), cudaMemcpyHostToDevice));
    FCK(cudaMemcpy(s->litems, li.data(), sizeof(Potrf128Item) * li.size(), cudaMemcpyHostToDevice));
    FCK(cudaMemcpy(s->gramitems, gr.data(), sizeof(FsaGramItem) * gr.size(), cudaMemcpyHostToDevice));
    FCK(cudaStreamSynchronize(st));
    return GPB200_OK;
}

static int fsa_check(gpb200_fitc* f, const char* who) {
    if (f->nranks > 1) { f->err = std::string(who) + ": FSA is single-GPU only"; return GPB200_EINVAL; }
    if (!f->fsa) { f->err = std::string(who) + ": FSA needs gpb200_fitc_set_blocks after set_data"; return GPB200_ESTATE; }
    return GPB200_OK;
}

// update_cK! (:197-230) once K_uu, its factor and Sigma_QR = K_uu (+ nuggets) are in place (gpb200_fitc_factorize)
static int fsa_factorize(gpb200_fitc* f) {
    Fsa* s = f->fsa;
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int64_t Mp = f->Mpad, Nc = f->Nc;
    const int init = INT_MAX;
    FCK(cudaMemcpyAsync(s->info, &init, sizeof(int), cudaMemcpyHostToDevice, st));
    GemmBuf bA{eu->tma_ok ? &f->mapA : nullptr, f->bufA, Mp};
    GemmBuf bWt{eu->tma_ok ? &s->mapWt : nullptr, f->bufA, Nc};
    for (const FsaChunk& ch : s->chunks) {
        const double* xr = s->xb + ch.r0 * f->d;
        // V = K_fu L_uu^-T (padding rows zero), then Lambda_i = K_ii + (sigma^2 + 1e-10) I - V_i V_i'
        FCK(fitc_kfu(f, xr, ch.rows));
        FCK(fsa_mask_launch(f->bufA, Mp, ch.rows, Mp, s->mask + ch.r0, nullptr, st, &eu->launches));
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
        FCK(fsa_mask_launch(f->bufB, Nc, Mp, ch.rows, nullptr, s->mask + ch.r0, st, &eu->launches));
        FCK(fsa_gemm_launch(s->gitems + ch.wt.off, ch.wt.n, st, &eu->launches));
        GemmDesc g = gemm_desc_default();
        g.A = GemmOperand{bWt, bufNone(), 0, 0};
        g.B = GemmOperand{bWt, bufNone(), 0, 0};
        g.C = es->G; g.ldc = es->ld; g.M = (int)Mp; g.N = (int)Mp; g.K = (int)ch.rows;
        g.alpha = 1.0; g.beta = 1.0; g.flags = GEMM_LOWER_ONLY;
        FCK(launch_gemm(es, g));
    }
    int info = INT_MAX;
    FCK(cudaMemcpyAsync(&info, s->info, sizeof(int), cudaMemcpyDeviceToHost, st));
    FCK(cudaStreamSynchronize(st));
    if (info != INT_MAX) {
        f->err = "fitc_factorize (FSA): a block of Lambda is not positive definite (padded row " + std::to_string(info) + ")";
        return info;
    }
    int rc = chol_inplace(es);
    if (rc != GPB200_OK) { f->err = "fitc_factorize (Sigma_QR): " + es->err; return rc; }
    f->factored = true;
    return GPB200_OK;
}

// `\` (:105-108), logdet (:142), get_alpha_u (:366-373):  b = K_uf Lambda^-1 r,  u = Sigma_QR^-1 b,
// alpha = Lambda^-1 (r - K_fu u),  logdet = logdet Sigma_QR - logdet K_uu + sum_i logdet Lambda_i
static int fsa_mll(gpb200_fitc* f, const double* y_minus_mean, double* alpha, double* mll, double* logdet) {
    Fsa* s = f->fsa;
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int64_t Np = s->Np, Mp = f->Mpad;
    FCK(cudaMemcpyAsync(f->y, y_minus_mean, sizeof(double) * f->N, cudaMemcpyHostToDevice, st));
    FCK(cudaMemsetAsync(s->r, 0, sizeof(double) * Np, st));
    FCK(fsa_permute_launch(1, f->y, s->pos, f->N, s->r, st, &eu->launches));
    FCK(fsa_bdmv_launch(0, s->X, s->rblk, s->bstart, s->bsize, s->boff, s->r, s->t1, Np, st, &eu->launches));
    FCK(fsa_bdmv_launch(1, s->LT, s->rblk, s->bstart, s->bsize, s->boff, s->t1, s->t2, Np, st, &eu->launches));     // t2 = Lambda^-1 r
    FCK(cudaMemsetAsync(f->bvec, 0, sizeof(double) * Mp, st));
    for (const FsaChunk& ch : s->chunks) {
        FCK(fitc_kuf(f, s->xb + ch.r0 * f->d, ch.rows));
        FCK(rowdot_launch(f->bufB, f->Nc, s->t2 + ch.r0, f->M, ch.rows, f->tmpm, st, &eu->launches));
        FCK(ew_launch(2, f->M, f->bvec, f->tmpm, nullptr, nullptr, 0.0, st, &eu->launches));
    }
    FCK(cudaMemcpyAsync(f->rhsm, f->bvec, sizeof(double) * Mp, cudaMemcpyDeviceToDevice, st));
    FCK(solve_device(es, f->rhsm, f->tmpm, f->uvec));
    for (const FsaChunk& ch : s->chunks) {
        FCK(fitc_kfu(f, s->xb + ch.r0 * f->d, ch.rows));
        FCK(rowdot_launch(f->bufA, Mp, f->uvec, ch.rows, Mp, s->t1 + ch.r0, st, &eu->launches));
    }
    FCK(fsa_resid_launch(s->t1, s->r, s->t1, s->mask, Np, st, &eu->launches));                                      // r - K_fu u, padding 0
    FCK(fsa_bdmv_launch(0, s->X, s->rblk, s->bstart, s->bsize, s->boff, s->t1, s->t2, Np, st, &eu->launches));
    FCK(fsa_bdmv_launch(1, s->LT, s->rblk, s->bstart, s->bsize, s->boff, s->t2, s->a, Np, st, &eu->launches));      // alpha (padded order)
    FCK(fsa_permute_launch(0, s->a, s->pos, f->N, f->alpha, st, &eu->launches));
    FCK(dot_launch(s->r, s->a, Np, f->scal + 0, st, &eu->launches));
    FCK(sum_launch(es->logd, es->Npad, f->scal + 1, st, &eu->launches));
    FCK(sum_launch(eu->logd, eu->Npad, f->scal + 2, st, &eu->launches));
    FCK(sum_launch(s->logd, Np, f->scal + 3, st, &eu->launches));
    double sc[4];
    FCK(cudaMemcpyAsync(sc, f->scal, sizeof(double) * 4, cudaMemcpyDeviceToHost, st));
    if (alpha) FCK(cudaMemcpyAsync(alpha, f->alpha, sizeof(double) * f->N, cudaMemcpyDeviceToHost, st));
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
static int fsa_grad_noise(gpb200_fitc* f, double* dmll_noise) {
    Fsa* s = f->fsa;
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int64_t Np = s->Np, Mp = f->Mpad, Nc = f->Nc;
    GemmBuf bB2{eu->tma_ok ? &f->mapB2 : nullptr, f->bufB, Mp};
    for (const FsaChunk& ch : s->chunks) {
        FCK(fitc_kuf(f, s->xb + ch.r0 * f->d, ch.rows));
        FCK(fsa_mask_launch(f->bufB, Nc, Mp, ch.rows, nullptr, s->mask + ch.r0, st, &eu->launches));
        FCK(fsa_gemm_launch(s->gitems + ch.wt.off, ch.wt.n, st, &eu->launches));  // W' = K_uf X'               (bufA, Mpad x Nc)
        FCK(fsa_gemm_launch(s->gitems + ch.z.off, ch.z.n, st, &eu->launches));    // Z = X' W = Lambda^-1 K_fu  (bufB, Nc x Mpad)
        FCK(trsm_rec_buf(es, bB2, (int)ch.rows, 0, (int)Mp));                 // Y = Z L_s^-T
        FCK(rowvar_launch(f->bufB, Mp, f->zeroc, ch.rows, Mp, s->t1 + ch.r0, st, &eu->launches));   // -|Y_r|^2
    }
    FCK(sum_launch(s->t1, Np, f->scal + 0, st, &eu->launches));
    FCK(dot_launch(s->a, s->a, Np, f->scal + 1, st, &eu->launches));
    FCK(fsa_bdmv_launch(2, s->X, s->rblk, s->bstart, s->bsize, s->boff, nullptr, s->t2, Np, st, &eu->launches));
    FCK(sum_launch(s->t2, Np, f->scal + 2, st, &eu->launches));
    double sc[3];
    FCK(cudaMemcpyAsync(sc, f->scal, sizeof(double) * 3, cudaMemcpyDeviceToHost, st));
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
static int fsa_grad_kernel(gpb200_fitc* f, double* dmll_kernel, double* dmll_xu) {
    Fsa* s = f->fsa;
    gpb200_handle *eu = f->eu, *es = f->es;
    cudaStream_t st = eu->st;
    const int np = eu->prog.n_theta;
    const int64_t Mp = f->Mpad, Nc = f->Nc;
    const bool tma = eu->tma_ok;
    GemmBuf bA{tma ? &f->mapA : nullptr, f->bufA, Mp};          // bufA as Nc x Mpad
    GemmBuf bAt{tma ? &s->mapWt : nullptr, f->bufA, Nc};        // bufA as Mpad x Nc
    GemmBuf bB2{tma ? &f->mapB2 : nullptr, f->bufB, Mp};        // bufB as Nc x Mpad
    GemmBuf bBt{tma ? &f->mapB : nullptr, f->bufB, Nc};         // bufB as Mpad x Nc
    size_t xk = 0;                                                // inducing-point contractions so far
    for (const FsaChunk& ch : s->chunks) {
        const double* xr = s->xb + ch.r0 * f->d;
        const int64_t nc = ch.rows;
        FCK(fitc_kuf(f, xr, nc));
        FCK(fsa_mask_launch(f->bufB, Nc, Mp, nc, nullptr, s->mask + ch.r0, st, &eu->launches));
        FCK(fsa_gemm_launch(s->gitems + ch.wt.off, ch.wt.n, st, &eu->launches));  // W' = K_uf X'                   (bufA, Mpad x Nc)
        FCK(fsa_gemm_launch(s->gitems + ch.z.off, ch.z.n, st, &eu->launches));    // Z = Lambda^-1 K_fu             (bufB, Nc x Mpad)
        {   // P2 = Z S^-1 -> bufC
            GemmDesc g = gemm_desc_default();
            g.A = GemmOperand{bB2, bufNone(), 0, 0};
            g.B = GemmOperand{bufG(es), bufNone(), 0, 0};
            g.C = f->bufC; g.ldc = Mp; g.M = (int)nc; g.N = (int)Mp; g.K = (int)Mp;
            FCK(launch_gemm(es, g));
        }
        FCK(trsm_rec_buf(es, bB2, (int)nc, 0, (int)Mp));       // Y = Z L_s^-T                   (bufB)
        // G_i = -Lambda_i^-1 + Y_i Y_i' + alpha_i alpha_i'  (Gpk), then sum_i <G_i, dK_ii/dθ_p>
        FCK(fsa_gemm_launch(s->gitems + ch.ginv.off, ch.ginv.n, st, &eu->launches));
        FCK(fsa_gemm_launch(s->gitems + ch.gyy.off, ch.gyy.n, st, &eu->launches));
        FCK(fsa_outer_launch(s->gramitems + ch.gtiles.off, ch.gtiles.n, s->a, st, &eu->launches));
        FCK(fsa_trace_launch(eu->prog, s->xb, f->d, s->gramitems + ch.gtiles.off, ch.gtiles.n, s->mask, s->gpart, f->gtmp, st, &eu->launches));
        FCK(ew_launch(2, np, f->gacc, f->gtmp, nullptr, nullptr, 0.0, st, &eu->launches));
        // P1' = K_uu^-1 K_uf (bufB, Mpad x Nc) from K_fu (bufA)
        FCK(fitc_kfu(f, xr, nc));
        FCK(fsa_mask_launch(f->bufA, Mp, nc, Mp, s->mask + ch.r0, nullptr, st, &eu->launches));
        {
            GemmDesc g = gemm_desc_default();
            g.A = GemmOperand{bufG(eu), bufNone(), 0, 0};
            g.B = GemmOperand{bA, bufNone(), 0, 0};
            g.C = f->bufB; g.ldc = Nc; g.M = (int)Mp; g.N = (int)nc; g.K = (int)Mp;
            FCK(launch_gemm(eu, g));
        }
        // W_fu = 2 alpha beta' - 2 P2 - 2 G_bd P1  (bufC); P1' G_bd -> bufA (Mpad x Nc)
        FCK(fitc_wfu_launch(f->bufC, f->bufA, Mp, nc, f->M, s->a + ch.r0, s->ones, f->zeroc, f->betav, st, &eu->launches));   // g = 0: P1 unused
        FCK(fsa_gemm_launch(s->gitems + ch.gp1t.off, ch.gp1t.n, st, &eu->launches));
        FCK(fsa_axpy_t_launch(f->bufC, Mp, f->bufA, Nc, nc, Mp, -2.0, st, &eu->launches));
        FCK(trace_rect_launch(eu->prog, xr, f->d, nc, eu->x, f->d, f->M, f->d, f->bufC, Mp, f->gpart, f->gtmp, st, &eu->launches));
        FCK(ew_launch(2, np, f->gacc, f->gtmp, nullptr, nullptr, 0.0, st, &eu->launches));
        // dmll/dXu: the padding rows of the chunk are skipped (mask 0); Xu is in the caller's order (never permuted)
        if (dmll_xu) { TRY(xu_contract(f, xk + 1, xr, nc, f->bufC, 0, s->mask + ch.r0, xk > 0)); ++xk; }
        {   // H += P1' G_bd P1 = K_uu^-1 (K_uf G_bd K_fu) K_uu^-1
            GemmDesc g = gemm_desc_default();
            g.A = GemmOperand{bBt, bufNone(), 0, 0};
            g.B = GemmOperand{bAt, bufNone(), 0, 0};
            g.C = f->Hbuf; g.ldc = Mp; g.M = (int)Mp; g.N = (int)Mp; g.K = (int)nc;
            g.alpha = 1.0; g.beta = 1.0;
            FCK(launch_gemm(eu, g));
        }
    }
    FCK(fitc_wuu_launch(f->Wbuf, f->Hbuf, eu->G, es->G, Mp, f->M, f->betav, st, &eu->launches));
    FCK(trace_rect_launch(eu->prog, eu->x, f->d, f->M, eu->x, f->d, f->M, f->d, f->Wbuf, Mp, f->gpart, f->gtmp, st, &eu->launches));
    FCK(ew_launch(2, np, f->gacc, f->gtmp, nullptr, nullptr, 0.0, st, &eu->launches));
    if (dmll_xu) {
        TRY(xu_contract(f, xk + 1, eu->x, f->M, f->Wbuf, 1, nullptr, xk > 0)); ++xk;
        FCK(cudaEventRecord(f->xu_ev[1], st));
    }
    std::vector<double> out((size_t)std::max(np, 1));
    FCK(cudaMemcpyAsync(out.data(), f->gacc, sizeof(double) * np, cudaMemcpyDeviceToHost, st));
    FCK(cudaStreamSynchronize(st));
    FSUB(check_trsv_watchdog(eu), eu);                                   // the solve for beta in gpb200_fitc_grad_kernel
    if (dmll_kernel) for (int p = 0; p < np; ++p) dmll_kernel[p] = 0.5 * out[p];
    if (dmll_xu) TRY(xu_finish(f, xk, dmll_xu));
    return GPB200_OK;
}

// predictMVN / predict_f with test blocks (:413-478): test block j is paired with training block j, Lambda_xf = K_xf - Q_xf on the
// paired blocks and 0 elsewhere.  With C = Lambda_xf, G = C L_Lambda^-T, W = L_Lambda^-1 K_fu and V_* = L_uu^-1 K_u*:
//   mu = K_*u u + C alpha ,   Sigma = K_** - V_*' V_* - G G' + R R' ,   R = (K_*u - G W) L_s^-T
// (from Sigma^-1 = Lambda^-1 - Lambda^-1 K_fu S^-1 K_uf Lambda^-1 and S = K_uu + K_uf Lambda^-1 K_fu; C = 0 is the FITC formula).
// G G' is block-diagonal in the test blocks.  Test points are grouped by paired block, each group padded to 128 rows, and
// streamed in chunks of at most Nc padded rows; per chunk, the training chunks of the paired blocks are revisited (V, K_uf).
//
// dmu != null (gpb200_fitc_predict_fsa_grad; cov null): the same launches give mu and var, then per test chunk the
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
static int fsa_predict(gpb200_fitc* f, int64_t Ms, const double* xs, int64_t ldxs, const int64_t* block_of, double* mu,
                       double* var, double* cov, double* dmu, double* dvar) {
    if (!f || Ms <= 0 || !xs || !block_of || !mu) return GPB200_EINVAL;
    if (f->mode != 3) { f->err = "fitc_predict_fsa: the handle is not in FSA mode (3)"; return GPB200_EINVAL; }
    if (!f->fsa || !f->factored || !f->alpha_ready) { f->err = "fitc_predict_fsa: set_blocks, factorize and mll first"; return GPB200_ESTATE; }
    if (ldxs < f->d) { f->err = "fitc_predict_fsa: ldxs < d"; return GPB200_EINVAL; }
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
    if (cov && Msp > Nc) { f->err = "fitc_predict_fsa: cov needs the padded test blocks in one staging chunk"; return GPB200_EINVAL; }
    if (cov && Msp > f->Kss_rows) {
        if (f->Kss) cudaFree(f->Kss);
        f->Kss = nullptr; f->Kss_rows = 0;
        FCK(cudaMalloc(&f->Kss, sizeof(double) * Msp * Msp));
        f->Kss_rows = Msp;
    }
    std::vector<int64_t> ppos((size_t)Ms);
    std::vector<double> xsp((size_t)Msp * d, 0.0);
    for (int64_t i = 0; i < Ms; ++i) {
        const int64_t k = key[(size_t)i], r = gstart[(size_t)k] + fill[(size_t)k]++;
        ppos[(size_t)i] = r;
        for (int q = 0; q < d; ++q) xsp[(size_t)r * d + q] = xs[i * ldxs + q];
    }
    if (!s->Vs) {
        FCK(cudaMalloc(&s->Vs, sizeof(double) * Nc * Mp));
        FCK(cudaMalloc(&s->Cb, sizeof(double) * Nc * LDC));
        FCK(cudaMalloc(&s->Gb, sizeof(double) * Nc * LDC));
        FCK(cudaMalloc(&s->pvec, sizeof(double) * Nc * 6));
        if (eu->tma_ok && !gemm_make_tensor_map(&s->mapVs, s->Vs, Nc, Mp, Mp)) {
            f->err = "fitc_predict_fsa: cuTensorMapEncodeTiled failed"; return GPB200_ECUDA;
        }
    }
    const bool grad = dmu != nullptr, gvar = grad && var;
    if (gvar && !s->Zb) {
        FCK(cudaMalloc(&s->Tb, sizeof(double) * Nc * LDC));
        FCK(cudaMalloc(&s->Zb, sizeof(double) * Nc * Mp));
        if (eu->tma_ok && !gemm_make_tensor_map(&s->mapZb, s->Zb, Nc, Mp, Mp)) {
            f->err = "fitc_predict_fsa_grad: cuTensorMapEncodeTiled failed"; return GPB200_ECUDA;
        }
    }
    if (grad && (size_t)(2 * Ms * d) > s->pdx_cap) {
        if (s->pdx) cudaFree(s->pdx);
        s->pdx = nullptr; s->pdx_cap = 0;
        FCK(cudaMalloc(&s->pdx, sizeof(double) * 2 * Ms * d));
        s->pdx_cap = (size_t)(2 * Ms * d);
    }
    double *mu1 = s->pvec, *mu2 = mu1 + Nc, *q = mu2 + Nc, *g2 = q + Nc, *r2 = g2 + Nc, *vp = r2 + Nc;
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
                    g.dst = s->Cb + tl * TILE * LDC + c * TILE; g.ld = LDC; g.row_i = tl * TILE; g.row_j = s->bstart_h[(size_t)b] + c * TILE;
                    xi.push_back(g);
                }
            });
            ps.xg.n = (int)((int64_t)xi.size() - ps.xg.off);
            ps.vv.off = (int64_t)gi.size();                     // C -= V_* V_b'
            each([&](int64_t b, int64_t tl) {
                for (int c = 0; c < s->bsize_h[(size_t)b] / TILE; ++c)
                    gemm(s->Cb + tl * TILE * LDC + c * TILE, LDC, s->Vs + tl * TILE * Mp, Mp,
                         f->bufA + (s->bstart_h[(size_t)b] - ch.r0 + c * TILE) * Mp, Mp, Mp, -1.0, 1.0);
            });
            ps.vv.n = (int)((int64_t)gi.size() - ps.vv.off);
            ps.mu2.off = (int64_t)ri.size();                    // C alpha
            each([&](int64_t b, int64_t tl) {
                FsaRowItem r{};
                r.A = s->Cb + tl * TILE * LDC; r.lda = LDC; r.v = s->a + s->bstart_h[(size_t)b]; r.out = mu2 + tl * TILE;
                r.K = s->bsize_h[(size_t)b]; r.sq = 0;
                ri.push_back(r);
            });
            ps.mu2.n = (int)((int64_t)ri.size() - ps.mu2.off);
            ps.gg.off = (int64_t)gi.size();                     // G = C X'
            each([&](int64_t b, int64_t tl) {
                const int B = s->bsize_h[(size_t)b];
                for (int c = 0; c < B / TILE; ++c)
                    gemm(s->Gb + tl * TILE * LDC + c * TILE, LDC, s->Cb + tl * TILE * LDC, LDC,
                         s->X + s->boff_h[(size_t)b] + (int64_t)c * TILE * B, B, (int64_t)(c + 1) * TILE, 1.0, 0.0);
            });
            ps.gg.n = (int)((int64_t)gi.size() - ps.gg.off);
            ps.g2.off = (int64_t)ri.size();                     // |G|^2
            each([&](int64_t b, int64_t tl) {
                FsaRowItem r{};
                r.A = s->Gb + tl * TILE * LDC; r.lda = LDC; r.v = nullptr; r.out = g2 + tl * TILE; r.K = s->bsize_h[(size_t)b]; r.sq = 1;
                ri.push_back(r);
            });
            ps.g2.n = (int)((int64_t)ri.size() - ps.g2.off);
            ps.hh.off = (int64_t)gi.size();                     // H = G X = C Lambda^-1  (into the C tiles)
            each([&](int64_t b, int64_t tl) {
                const int B = s->bsize_h[(size_t)b];
                for (int c = 0; c < B / TILE; ++c)
                    gemm(s->Cb + tl * TILE * LDC + c * TILE, LDC, s->Gb + tl * TILE * LDC + c * TILE, LDC,
                         s->LT + s->boff_h[(size_t)b] + (int64_t)c * TILE * B + c * TILE, B, B - (int64_t)c * TILE, 1.0, 0.0);
            });
            ps.hh.n = (int)((int64_t)gi.size() - ps.hh.off);
            ps.kh.off = (int64_t)gi.size();                     // K_*u -= H K_fu  (= G W)
            each([&](int64_t b, int64_t tl) {
                for (int64_t u = 0; u < Mp / TILE; ++u)
                    gemm(f->bufB + tl * TILE * Mp + u * TILE, Mp, s->Cb + tl * TILE * LDC, LDC,
                         f->bufA + u * TILE * Nc + (s->bstart_h[(size_t)b] - ch.r0), Nc, s->bsize_h[(size_t)b], -1.0, 1.0);
            });
            ps.kh.n = (int)((int64_t)gi.size() - ps.kh.off);
            if (gvar) {
                ps.t1.off = (int64_t)gi.size();                 // T = s K_ub'  (bufB = s, bufA = K_fu of the chunk)
                each([&](int64_t b, int64_t tl) {
                    for (int c = 0; c < s->bsize_h[(size_t)b] / TILE; ++c)
                        gemm(s->Tb + tl * TILE * LDC + c * TILE, LDC, f->bufB + tl * TILE * Mp, Mp,
                             f->bufA + (s->bstart_h[(size_t)b] - ch.r0 + c * TILE) * Mp, Mp, Mp, 1.0, 0.0);
                });
                ps.t1.n = (int)((int64_t)gi.size() - ps.t1.off);
                ps.tx.off = (int64_t)gi.size();                 // T X'  (into the G tiles)
                each([&](int64_t b, int64_t tl) {
                    const int B = s->bsize_h[(size_t)b];
                    for (int c = 0; c < B / TILE; ++c)
                        gemm(s->Gb + tl * TILE * LDC + c * TILE, LDC, s->Tb + tl * TILE * LDC, LDC,
                             s->X + s->boff_h[(size_t)b] + (int64_t)c * TILE * B, B, (int64_t)(c + 1) * TILE, 1.0, 0.0);
                });
                ps.tx.n = (int)((int64_t)gi.size() - ps.tx.off);
                ps.ee.off = (int64_t)gi.size();                 // e = -2 (H + T X' X)  (over H in the C tiles)
                each([&](int64_t b, int64_t tl) {
                    const int B = s->bsize_h[(size_t)b];
                    for (int c = 0; c < B / TILE; ++c)
                        gemm(s->Cb + tl * TILE * LDC + c * TILE, LDC, s->Gb + tl * TILE * LDC + c * TILE, LDC,
                             s->LT + s->boff_h[(size_t)b] + (int64_t)c * TILE * B + c * TILE, B, B - (int64_t)c * TILE, -2.0, -2.0);
                });
                ps.ee.n = (int)((int64_t)gi.size() - ps.ee.off);
                ps.ek.off = (int64_t)gi.size();                 // Z += e K_bu / 2  (bufA = K_uf of the chunk)
                each([&](int64_t b, int64_t tl) {
                    for (int64_t u = 0; u < Mp / TILE; ++u)
                        gemm(s->Zb + tl * TILE * Mp + u * TILE, Mp, s->Cb + tl * TILE * LDC, LDC,
                             f->bufA + u * TILE * Nc + (s->bstart_h[(size_t)b] - ch.r0), Nc, s->bsize_h[(size_t)b], 0.5, 1.0);
                });
                ps.ek.n = (int)((int64_t)gi.size() - ps.ek.off);
            }
            if (grad) {
                ps.ak.off = (int64_t)gi.size();                 // alpha_b K_bu on every row of the tile (into Vs)
                each([&](int64_t b, int64_t tl) {
                    for (int64_t u = 0; u < Mp / TILE; ++u)
                        gemm(s->Vs + tl * TILE * Mp + u * TILE, Mp, s->a + s->bstart_h[(size_t)b], 0,
                             f->bufA + u * TILE * Nc + (s->bstart_h[(size_t)b] - ch.r0), Nc, s->bsize_h[(size_t)b], 1.0, 0.0);
                });
                ps.ak.n = (int)((int64_t)gi.size() - ps.ak.off);
            }
            sb.passes.push_back(ps);
            t = te;
        }
        sb.ggt.off = (int64_t)gi.size();                        // cov: -G G' on the tile pairs of the same block
        if (cov) {
            const int64_t mq = (sb.t1 - sb.t0) * TILE;
            for (int64_t t = sb.t0; t < sb.t1; ++t)
                for (int64_t u = sb.t0; u < sb.t1; ++u) {
                    const int64_t b = tile_blk[(size_t)t];
                    if (b < 0 || tile_blk[(size_t)u] != b) continue;
                    gemm(f->Kss + (t - sb.t0) * TILE * mq + (u - sb.t0) * TILE, mq, s->Gb + (t - sb.t0) * TILE * LDC, LDC,
                         s->Gb + (u - sb.t0) * TILE * LDC, LDC, s->bsize_h[(size_t)b], -1.0, 1.0);
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
    auto upload = [&](auto*& dst, size_t& cap, const auto& v) -> cudaError_t {
        using T = typename std::decay_t<decltype(v)>::value_type;
        if (v.size() > cap) {
            if (dst) cudaFree(dst);
            dst = nullptr; cap = 0;
            cudaError_t e = cudaMalloc(&dst, sizeof(T) * v.size());
            if (e != cudaSuccess) return e;
            cap = v.size();
        }
        return v.empty() ? cudaSuccess : cudaMemcpy(dst, v.data(), sizeof(T) * v.size(), cudaMemcpyHostToDevice);
    };
    FCK(upload(s->pg, s->pg_cap, gi));
    FCK(upload(s->px, s->px_cap, xi));
    FCK(upload(s->pr, s->pr_cap, ri));
    if (grad) FCK(upload(s->pdi, s->pdi_cap, di));
    GemmBuf bA{eu->tma_ok ? &f->mapA : nullptr, f->bufA, Mp};
    GemmBuf bB2{eu->tma_ok ? &f->mapB2 : nullptr, f->bufB, Mp};
    GemmBuf bVs{eu->tma_ok ? &s->mapVs : nullptr, s->Vs, Mp};
    GemmBuf bZb{eu->tma_ok ? &s->mapZb : nullptr, s->Zb, Mp};
    const bool cov_host = cov && !f->cov_keep_device;
    std::vector<double> mu_p((size_t)Msp), var_p(var ? (size_t)Msp : 0), cov_p(cov_host ? (size_t)Msp * Msp : 0);
    double* ddmu = grad ? s->pdx : nullptr;
    double* ddvar = grad ? s->pdx + Ms * d : nullptr;
    if (grad) {
        for (double& t : f->fsag_ms) t = 0.0;
        FCK(mirror_lower_tiles_launch(eu->F, eu->ld, eu->Npad, st, &eu->launches));      // L' for the right-side TRSMs
        if (var) FCK(mirror_lower_tiles_launch(es->F, es->ld, es->Npad, st, &eu->launches));
    }
    for (const Sub& sb : subs) {
        const int64_t row0 = sb.t0 * TILE, mq = (sb.t1 - sb.t0) * TILE;
        if (grad) FCK(cudaEventRecord(eu->ev0, st));
        FCK(cudaMemcpyAsync(f->xs, xsp.data() + row0 * d, sizeof(double) * mq * d, cudaMemcpyHostToDevice, st));
        FCK(crossgram_launch(eu->prog, f->xs, d, mq, mq, eu->x, d, f->M, Mp, d, f->bufB, Mp, st, &eu->launches));     // K_*u
        FCK(rowdot_launch(f->bufB, Mp, f->uvec, mq, Mp, mu1, st, &eu->launches));                                       // K_*u u
        FCK(cudaMemcpyAsync(s->Vs, f->bufB, sizeof(double) * mq * Mp, cudaMemcpyDeviceToDevice, st));
        if (gvar) FCK(cudaMemcpyAsync(s->Zb, f->bufB, sizeof(double) * mq * Mp, cudaMemcpyDeviceToDevice, st));      // Z = K_*u
        FCK(trsm_rec_buf(eu, bVs, (int)mq, 0, (int)Mp));                                                 // V_*'
        FCK(kdiag_launch(eu->prog, f->xs, d, mq, r2, st, &eu->launches));
        FCK(rowvar_launch(s->Vs, Mp, r2, mq, Mp, q, st, &eu->launches));                                                 // k** - |V_*|^2
        FCK(cudaMemsetAsync(mu2, 0, sizeof(double) * mq, st));
        FCK(cudaMemsetAsync(g2, 0, sizeof(double) * mq, st));
        for (const Pass& ps : sb.passes) {
            const FsaChunk& ch = s->chunks[(size_t)ps.chunk];
            const double* xr = s->xb + ch.r0 * d;
            FCK(fitc_kfu(f, xr, ch.rows));                                                                 // V of the training chunk
            FCK(fsa_mask_launch(f->bufA, Mp, ch.rows, Mp, s->mask + ch.r0, nullptr, st, &eu->launches));
            FCK(trsm_rec_buf(eu, bA, (int)Nc, 0, (int)Mp));
            FCK(fsa_crossgram_launch(eu->prog, f->xs, s->xb, d, s->px + ps.xg.off, ps.xg.n, s->mask, st, &eu->launches));
            FCK(fsa_gemm_launch(s->pg + ps.vv.off, ps.vv.n, st, &eu->launches));
            FCK(fsa_rowdot_launch(s->pr + ps.mu2.off, ps.mu2.n, st, &eu->launches));
            FCK(fsa_gemm_launch(s->pg + ps.gg.off, ps.gg.n, st, &eu->launches));
            FCK(fsa_rowdot_launch(s->pr + ps.g2.off, ps.g2.n, st, &eu->launches));
            FCK(fsa_gemm_launch(s->pg + ps.hh.off, ps.hh.n, st, &eu->launches));
            FCK(crossgram_launch(eu->prog, eu->x, d, f->M, Mp, xr, d, ch.rows, Nc, d, f->bufA, Nc, st, &eu->launches));   // K_uf of the chunk
            FCK(fsa_mask_launch(f->bufA, Nc, Mp, ch.rows, nullptr, s->mask + ch.r0, st, &eu->launches));
            FCK(fsa_gemm_launch(s->pg + ps.kh.off, ps.kh.n, st, &eu->launches));
        }
        FCK(trsm_rec_buf(es, bB2, (int)mq, 0, (int)Mp));                                                  // R = (K_*u - G W) L_s^-T
        FCK(rowvar_launch(f->bufB, Mp, f->zeroc, mq, Mp, r2, st, &eu->launches));
        FCK(fsa_var_launch(vp, q, g2, r2, mq, st, &eu->launches));
        FCK(ew_launch(2, mq, mu1, mu2, nullptr, nullptr, 0.0, st, &eu->launches));
        FCK(cudaMemcpyAsync(mu_p.data() + row0, mu1, sizeof(double) * mq, cudaMemcpyDeviceToHost, st));
        if (var) FCK(cudaMemcpyAsync(var_p.data() + row0, vp, sizeof(double) * mq, cudaMemcpyDeviceToHost, st));
        if (grad) {
            FCK(cudaEventRecord(eu->ev1, st));
            if (var) FCK(trsm_right_rec_buf(es, bB2, (int)mq, 0, (int)Mp));                             // s = R L_s^-1
            FCK(cudaMemsetAsync(s->Vs, 0, sizeof(double) * mq * Mp, st));
            for (const Pass& ps : sb.passes) {                                                           // second sweep
                const FsaChunk& ch = s->chunks[(size_t)ps.chunk];
                const double* xr = s->xb + ch.r0 * d;
                if (var) {
                    FCK(fitc_kfu(f, xr, ch.rows));                                                       // K_fu of the chunk
                    FCK(fsa_mask_launch(f->bufA, Mp, ch.rows, Mp, s->mask + ch.r0, nullptr, st, &eu->launches));
                    FCK(fsa_gemm_launch(s->pg + ps.t1.off, ps.t1.n, st, &eu->launches));
                    FCK(fsa_gemm_launch(s->pg + ps.tx.off, ps.tx.n, st, &eu->launches));
                    FCK(fsa_gemm_launch(s->pg + ps.ee.off, ps.ee.n, st, &eu->launches));
                }
                FCK(crossgram_launch(eu->prog, eu->x, d, f->M, Mp, xr, d, ch.rows, Nc, d, f->bufA, Nc, st, &eu->launches));
                FCK(fsa_mask_launch(f->bufA, Nc, Mp, ch.rows, nullptr, s->mask + ch.r0, st, &eu->launches));
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
            FCK(fsa_crossgram_dx_launch(eu->prog, f->xs, eu->x, s->xb, d, f->M, f->uvec, s->Vs, f->bufB, s->Zb, Mp, s->mask,
                                        s->a, s->Cb, LDC, s->pdi + sb.dx.off, sb.dx.n, ddmu, var ? ddvar : nullptr, st,
                                        &eu->launches));
            FCK(cudaEventRecord(eu->ev4, st));
        }
        if (cov) {
            FCK(gram_full_launch(eu->prog, f->xs, d, mq, mq, d, f->Kss, mq, st, &eu->launches));
            GemmDesc g = gemm_desc_default();
            g.A = GemmOperand{bVs, bufNone(), 0, 0};
            g.B = GemmOperand{bVs, bufNone(), 0, 0};
            g.C = f->Kss; g.ldc = mq; g.M = (int)mq; g.N = (int)mq; g.K = (int)Mp;
            g.alpha = -1.0; g.beta = 1.0;
            FCK(launch_gemm(eu, g));                                                                      // - V_*' V_*
            g.A = GemmOperand{bB2, bufNone(), 0, 0};
            g.B = GemmOperand{bB2, bufNone(), 0, 0};
            g.alpha = 1.0;
            FCK(launch_gemm(es, g));                                                                      // + R R'
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
    if (cov && !cov_host) {
        // Sigma* (one sub-chunk: leading dimension Msp) and mu in the caller's order on the device, as the host loop below
        // reorders them
        if ((size_t)(Ms * Ms) > s->Sc_cap) {
            if (s->Sc) cudaFree(s->Sc);
            s->Sc = nullptr; s->Sc_cap = 0;
            FCK(cudaMalloc(&s->Sc, sizeof(double) * Ms * Ms));
            s->Sc_cap = (size_t)(Ms * Ms);
        }
        FCK(upload(s->pp, s->pp_cap, ppos));
        FCK(gather_block_launch(s->Sc, f->Kss, Msp, s->pp, Ms, st, &eu->launches));
        FCK(fsa_permute_launch(0, mu1, s->pp, Ms, f->tmpc, st, &eu->launches));
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

int gpb200_fitc_predict_fsa(gpb200_fitc* f, int64_t Ms, const double* xs, int64_t ldxs, const int64_t* block_of,
                            double* mu, double* var, double* cov) {
    return fsa_predict(f, Ms, xs, ldxs, block_of, mu, var, cov, nullptr, nullptr);
}

int gpb200_fitc_predict_fsa_grad(gpb200_fitc* f, int64_t Ms, const double* xs, int64_t ldxs, const int64_t* block_of,
                                 double* mu, double* var, double* dmu, double* dvar) {
    if (!f) return GPB200_EINVAL;
    if (f->mode != 3) { f->err = "fitc_predict_fsa_grad: the handle is not in FSA mode (3)"; return GPB200_EINVAL; }
    if (f->nranks > 1) { f->err = "fitc_predict_fsa_grad: single GPU handles only"; return GPB200_EINVAL; }
    if (!f->fsa || !f->factored || !f->alpha_ready) { f->err = "fitc_predict_fsa_grad: set_blocks, factorize and mll first"; return GPB200_ESTATE; }
    if (Ms <= 0 || !xs || ldxs < f->d || !block_of || !mu || !dmu) {
        f->err = "fitc_predict_fsa_grad: bad Ms, xs, ldxs, block_of, mu or dmu"; return GPB200_EINVAL;
    }
    if (!var != !dvar) { f->err = "fitc_predict_fsa_grad: var and dvar must be given together"; return GPB200_EINVAL; }
    return fsa_predict(f, Ms, xs, ldxs, block_of, mu, var, nullptr, dmu, dvar);
}

// rand(gp, X, n) (src/GP.jl:120-146) with a sparse cK: Sigma* is the covariance predict_cov (modes 0-2) or predict_fsa
// (mode 3) returns, built on the device and kept there; make_posdef!, the Cholesky and unwhiten! are gpb200_rand's
// (rand_from_cov on eu, whose Ms x Ms sub-engine shares the handle's stream).  The likelihood, gradient, prediction and
// cross-validation state is only read.
int gpb200_fitc_rand(gpb200_fitc* f, int64_t Ms, const double* xs, int64_t ldxs, const int64_t* block_of, int64_t nsamp,
                     const double* z, double nugget, double* mu_minus_mean, double* samples) {
    if (!f) return GPB200_EINVAL;
    if (Ms <= 0 || nsamp <= 0 || !xs || ldxs < f->d || !z || !mu_minus_mean || !samples) {
        f->err = "fitc_rand: bad Ms, nsamp, xs, ldxs, z, mu or samples"; return GPB200_EINVAL;
    }
    if (!(nugget >= 0.0)) { f->err = "fitc_rand: nugget must be >= 0"; return GPB200_EINVAL; }
    if ((f->mode == 3) != (block_of != nullptr)) {
        f->err = "fitc_rand: block_of is required in FSA mode (3) and must be NULL otherwise"; return GPB200_EINVAL;
    }
    if (!f->factored || !f->alpha_ready) { f->err = "fitc_rand: factorize and mll first"; return GPB200_ESTATE; }
    if (f->mode != 3 && Ms > f->Nc) { f->err = "fitc_rand: too many test points for one staging chunk"; return GPB200_EINVAL; }
    FCK(cudaSetDevice(f->device));
    gpb200_handle* eu = f->eu;
    cudaEvent_t ev_start = eu->ev4;                      // rand_from_cov records ev0 .. ev3
    FCK(cudaEventRecord(ev_start, eu->st));
    const double* cov;
    int64_t ldc;
    if (f->mode == 3) {
        static double cov_flag;                          // non-null marker: Sigma* stays on the device
        f->cov_keep_device = true;
        const int rc = gpb200_fitc_predict_fsa(f, Ms, xs, ldxs, block_of, mu_minus_mean, nullptr, &cov_flag);
        f->cov_keep_device = false;
        if (rc) return rc;
        cov = f->fsa->Sc; ldc = Ms;
    } else {
        TRY(fitc_cov_build(f, Ms, xs, ldxs, mu_minus_mean));
        cov = f->Kss; ldc = (Ms + TILE - 1) / TILE * TILE;
    }
    FSUB(rand_from_cov(eu, Ms, cov, ldc, f->tmpc, nsamp, z, nugget, samples), eu);
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
    return GPB200_OK;
}

int gpb200_fitc_set_mode(gpb200_fitc* f, int mode) {
    if (!f || mode < 0 || mode > 3) return GPB200_EINVAL;
    f->mode = mode; f->factored = f->alpha_ready = false;
    return GPB200_OK;
}

int64_t gpb200_fitc_launch_count(gpb200_fitc* f) { return f ? f->eu->launches + f->es->launches : 0; }

}  // extern "C"
