// shard_impl.cuh -- ROW-SHARDED multi-GPU schedules (included by gpb200.cu inside namespace engine).
//
// North-star: "for N beyond one GPU's HBM the Gram matrix is row-block sharded across the 8 GPUs and a 1-D block
// Cholesky exchanges panels over NVLink with NCCL" (config C4: Mat32Iso N=131072 d=16, 137 GB per N x N matrix).
// Reference memory contract being replaced: four N x N host matrices per GPE (test/memory.jl:14-19, src/GP.jl:14-20).
//
// Storage: F and G keep their GLOBAL row-major addressing (ld = Npad) -- every kernel of the replicated engine works
// unchanged -- but they are CUDA virtual-memory ranges (cuMemAddressReserve) in which only the pages holding this rank's
// rows are backed by physical memory (cuMemCreate / cuMemMap).  Ownership is block-cyclic over 128-row tiles:
// tile t -> rank (t / rb) % R, panel width NBp = 128 * rb, so a diagonal block lives on one rank.  A stray access to a
// row another rank owns faults instead of silently reading stale data.  Per rank: 2 * Npad^2 * 8 / R bytes (+ panels).
//   F own rows:  lower part = rows of L;  beyond the row's diagonal block = rows of U = L' (the transposed column panel,
//                kept by the block owner when the panel is gathered) -> both triangular solves are fan-OUT only.
//   G own rows:  Gram rows -> Schur complements -> (inverse sweep) upper part: rows of L^-T, lower part: rows of K_y^-1.
//
// Schedules (tests/test_shard_model.py is their executable numpy specification, NaN-poisoned outside owned rows):
//   Cholesky   per panel k: owner factors the NBp x NBp diagonal block (the single-GPU recursive chol_panel restricted to
//              the block), broadcasts it with its inverted tiles; EVERY rank solves its own rows of the panel (TRSM split
//              R ways), the panel is all-gathered, every rank applies it to its own rows of the trailing matrix.
//   solves     forward on L rows, backward on U rows: per block one row-block GEMV, a 4-tile triangular solve, one broadcast.
//   inverse    one backward sweep over row panels J of X = L^-T:  owner finalises X_J = -W_JJ' acc_J and broadcasts it;
//              every rank adds U[i,J] X_J to the accumulators of its rows i < J (TRTRI part, N^3/3 flop in total) and
//              forms K^-1[i, J] = X_i X_J' for its rows i >= J (LAUUM part, N^3/3): the same 2N^3/3 as the single-GPU
//              path, K^-1 never leaves the rank that owns the row.
//   predict    V' = K*' L^-T with the columns of V' (training rows) owned like the rows of L; variance accumulated from
//              the broadcast blocks, identical on every rank.
//   append     rebuild from the ownership block b0 of the first touched tile: own Gram rows >= b0; V = K[b0.., :b0] L11^-T
//              solved like the predict (the block owner also keeps each block's transpose as U rows of its old rows); own
//              rows of V into L; Schur complement of the own rows (K = b0); the Cholesky above from block b0 / NBp on.
//   CV         own rows of K^-1 completed to full rows once, then per parameter own rows of Y' = K^-1 dK_j and of the lower
//              triangle of M_j = Y' K^-1 (see the section at the end; tests/test_shard_cv_model.py).
// Collectives: NCCL (one process per GPU) or, for an in-process group of virtual ranks on ONE device
// (gpb200_group_create: lets a 1-GPU box run the multi-rank schedules), event-ordered device-to-device copies.

// ---- CUDA VMM through the runtime's driver entry points (no link-time libcuda dependency: the library must dlopen on
// GPU-less build hosts) -------------------------------------------------------------------------------------------
struct VmApi {
    CUresult (*GetGranularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags) = nullptr;
    CUresult (*AddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
    CUresult (*AddressFree)(CUdeviceptr, size_t) = nullptr;
    CUresult (*Create)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long) = nullptr;
    CUresult (*Release)(CUmemGenericAllocationHandle) = nullptr;
    CUresult (*Map)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long) = nullptr;
    CUresult (*Unmap)(CUdeviceptr, size_t) = nullptr;
    CUresult (*SetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t) = nullptr;
    bool tried = false, ok = false;
} g_vm;

bool vm_load() {
    if (g_vm.tried) return g_vm.ok;
    g_vm.tried = true;
    auto get = [](const char* name) -> void* {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint(name, &fn, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
            (void)cudaGetLastError();
            return nullptr;
        }
        return fn;
    };
    g_vm.GetGranularity = (decltype(g_vm.GetGranularity))get("cuMemGetAllocationGranularity");
    g_vm.AddressReserve = (decltype(g_vm.AddressReserve))get("cuMemAddressReserve");
    g_vm.AddressFree = (decltype(g_vm.AddressFree))get("cuMemAddressFree");
    g_vm.Create = (decltype(g_vm.Create))get("cuMemCreate");
    g_vm.Release = (decltype(g_vm.Release))get("cuMemRelease");
    g_vm.Map = (decltype(g_vm.Map))get("cuMemMap");
    g_vm.Unmap = (decltype(g_vm.Unmap))get("cuMemUnmap");
    g_vm.SetAccess = (decltype(g_vm.SetAccess))get("cuMemSetAccess");
    g_vm.ok = g_vm.GetGranularity && g_vm.AddressReserve && g_vm.AddressFree && g_vm.Create && g_vm.Release && g_vm.Map &&
              g_vm.Unmap && g_vm.SetAccess;
    return g_vm.ok;
}

void vm_free(VmBuf& b) {
    if (!b.base) return;
    for (size_t i = 0; i < b.runs.size(); ++i) {
        g_vm.Unmap(b.base + b.runs[i].first, b.runs[i].second);
        if (i < b.handles.size()) g_vm.Release(b.handles[i]);
    }
    g_vm.AddressFree(b.base, b.va_size);
    b = VmBuf{};
}

// reserve `total` bytes of address space and back the byte ranges `want` (rounded out to the allocation granularity,
// merged) with device memory, zero-filled
int vm_alloc(gpb200_handle* h, VmBuf& b, size_t total, const std::vector<std::pair<size_t, size_t>>& want) {
    if (!vm_load()) return fail(h, GPB200_ECUDA, "CUDA virtual memory management entry points unavailable");
    CUmemAllocationProp prop{};
    prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    prop.location.id = h->device;
    size_t gran = 0;
    if (g_vm.GetGranularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM) != CUDA_SUCCESS || gran == 0)
        return fail(h, GPB200_ECUDA, "cuMemGetAllocationGranularity failed");
    b = VmBuf{};
    b.va_size = (total + gran - 1) / gran * gran;
    if (g_vm.AddressReserve(&b.base, b.va_size, 0, 0, 0) != CUDA_SUCCESS) { b = VmBuf{}; return fail(h, GPB200_ECUDA, "cuMemAddressReserve failed"); }
    // page runs
    std::vector<std::pair<size_t, size_t>> pages;         // [first page, last page]
    for (auto& w : want) {
        if (w.second == 0) continue;
        const size_t p0 = w.first / gran, p1 = (w.first + w.second - 1) / gran;
        if (!pages.empty() && p0 <= pages.back().second + 1) pages.back().second = std::max(pages.back().second, p1);
        else pages.push_back({p0, p1});
    }
    CUmemAccessDesc acc{};
    acc.location = prop.location;
    acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    for (auto& pr : pages) {
        const size_t off = pr.first * gran, bytes = (pr.second - pr.first + 1) * gran;
        CUmemGenericAllocationHandle mh;
        if (g_vm.Create(&mh, bytes, &prop, 0) != CUDA_SUCCESS) { vm_free(b); return fail(h, GPB200_ECUDA, "cuMemCreate failed (out of device memory?)"); }
        if (g_vm.Map(b.base + off, bytes, 0, mh, 0) != CUDA_SUCCESS) { g_vm.Release(mh); vm_free(b); return fail(h, GPB200_ECUDA, "cuMemMap failed"); }
        b.runs.push_back({off, bytes});
        b.handles.push_back(mh);
        if (g_vm.SetAccess(b.base + off, bytes, &acc, 1) != CUDA_SUCCESS) { vm_free(b); return fail(h, GPB200_ECUDA, "cuMemSetAccess failed"); }
        CK(cudaMemsetAsync((void*)(b.base + off), 0, bytes, h->st));
    }
    return GPB200_OK;
}

size_t vm_mapped_bytes(const VmBuf& b) {
    size_t s = 0;
    for (auto& r : b.runs) s += r.second;
    return s;
}

// ---- group / rank helpers ------------------------------------------------------------------------------------------
using Locals = std::vector<gpb200_handle*>;
Locals locals(gpb200_handle* h) { return h->grp ? h->grp->hs : Locals{h}; }
bool multi_rank(gpb200_handle* h) { return h->nranks > 1; }
ShardOwn own_of(gpb200_handle* h) { return ShardOwn{h->nranks, h->rank, h->rb}; }
int owner_of_tile(gpb200_handle* h, long long t) { return (int)((t / h->rb) % h->nranks); }

cudaEvent_t ring_event(gpb200_handle* h) {
    if (h->evring.empty()) {
        h->evring.resize(128);
        for (auto& e : h->evring) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
    }
    cudaEvent_t e = h->evring[h->evring_next];
    h->evring_next = (h->evring_next + 1) % h->evring.size();
    return e;
}

// ---- collectives: NCCL for one-process-per-GPU, event-ordered copies for an in-process group ----------------------
// `buf(q)` is the address of the (identically laid out) buffer in rank q's memory; all on the ranks' main streams.
template <class BufFn>
int coll_bcast(const Locals& L, int root, BufFn buf, size_t bytes) {
    if (bytes == 0) return GPB200_OK;
    gpb200_handle* h0 = L[0];
    if (h0->nranks <= 1) return GPB200_OK;
    if (!h0->grp) {
        SCKN(h0, g_nccl.Broadcast(buf(h0), buf(h0), bytes, ncclChar, root, h0->comm, h0->st));
        return GPB200_OK;
    }
    gpb200_handle* hr = L[root];
    cudaEvent_t e = ring_event(hr);
    SCK(hr, cudaEventRecord(e, hr->st));
    for (auto* q : L) {
        if (q == hr) continue;
        SCK(q, cudaStreamWaitEvent(q->st, e, 0));
        SCK(q, cudaMemcpyAsync(buf(q), buf(hr), bytes, cudaMemcpyDeviceToDevice, q->st));
        cudaEvent_t d = ring_event(q);
        SCK(q, cudaEventRecord(d, q->st));
        SCK(hr, cudaStreamWaitEvent(hr->st, d, 0));      // the root may not overwrite its buffer before every copy is done
    }
    return GPB200_OK;
}
int coll_group_begin(const Locals& L) {
    if (L[0]->nranks > 1 && !L[0]->grp) SCKN(L[0], g_nccl.GroupStart());
    return GPB200_OK;
}
int coll_group_end(const Locals& L) {
    if (L[0]->nranks > 1 && !L[0]->grp) SCKN(L[0], g_nccl.GroupEnd());
    return GPB200_OK;
}
// every rank holds [R][per_bytes]; rank q's contribution sits in region q of its own buffer
template <class BufFn>
int coll_allgather(const Locals& L, BufFn base, size_t per_bytes) {
    if (per_bytes == 0) return GPB200_OK;
    gpb200_handle* h0 = L[0];
    const int R = h0->nranks;
    if (R <= 1) return GPB200_OK;
    if (!h0->grp) {
        char* b = (char*)base(h0);
        SCKN(h0, g_nccl.AllGather(b + (size_t)h0->rank * per_bytes, b, per_bytes, ncclChar, h0->comm, h0->st));
        return GPB200_OK;
    }
    std::vector<cudaEvent_t> ready(R), done(R);
    for (int q = 0; q < R; ++q) { ready[q] = ring_event(L[q]); SCK(L[q], cudaEventRecord(ready[q], L[q]->st)); }
    for (int q = 0; q < R; ++q) {
        for (int p = 0; p < R; ++p) {
            if (p == q) continue;
            SCK(L[q], cudaStreamWaitEvent(L[q]->st, ready[p], 0));
            SCK(L[q], cudaMemcpyAsync((char*)base(L[q]) + (size_t)p * per_bytes, (char*)base(L[p]) + (size_t)p * per_bytes, per_bytes,
                                      cudaMemcpyDeviceToDevice, L[q]->st));
        }
        done[q] = ring_event(L[q]);
        SCK(L[q], cudaEventRecord(done[q], L[q]->st));
    }
    for (int p = 0; p < R; ++p)
        for (int q = 0; q < R; ++q)
            if (q != p) SCK(L[p], cudaStreamWaitEvent(L[p]->st, done[q], 0));
    return GPB200_OK;
}
// vec(q)[0..n) <- sum over ranks; local groups gather the R vectors into scratch(q) (R * n doubles) and sum them in rank
// order (deterministic)
template <class BufFn, class ScratchFn>
int coll_allreduce_sum(const Locals& L, BufFn vec, size_t n, ScratchFn scratch) {
    gpb200_handle* h0 = L[0];
    const int R = h0->nranks;
    if (R <= 1 || n == 0) return GPB200_OK;
    if (!h0->grp) {
        SCKN(h0, g_nccl.AllReduce(vec(h0), vec(h0), n, ncclDouble, ncclSum, h0->comm, h0->st));
        return GPB200_OK;
    }
    std::vector<cudaEvent_t> ready(R), copied(R);
    for (int q = 0; q < R; ++q) { ready[q] = ring_event(L[q]); SCK(L[q], cudaEventRecord(ready[q], L[q]->st)); }
    for (int q = 0; q < R; ++q) {
        for (int p = 0; p < R; ++p) {
            if (p != q) SCK(L[q], cudaStreamWaitEvent(L[q]->st, ready[p], 0));
            SCK(L[q], cudaMemcpyAsync(scratch(L[q]) + (size_t)p * n, vec(L[p]), sizeof(double) * n, cudaMemcpyDeviceToDevice, L[q]->st));
        }
        copied[q] = ring_event(L[q]);
        SCK(L[q], cudaEventRecord(copied[q], L[q]->st));
    }
    for (int q = 0; q < R; ++q) {
        for (int p = 0; p < R; ++p)
            if (p != q) SCK(L[q], cudaStreamWaitEvent(L[q]->st, copied[p], 0));
        SCK(L[q], shard_sum_ranks(vec(L[q]), scratch(L[q]), (int64_t)n, R, (int64_t)n, L[q]->st, &L[q]->launches));
    }
    return GPB200_OK;
}
// the same through the group scratch `red` (n <= 4096)
template <class BufFn>
int coll_allreduce_sum(const Locals& L, BufFn vec, size_t n) {
    if (L[0]->grp && n > 4096) return fail(L[0], GPB200_EINVAL, "coll_allreduce_sum: vector too long for the group scratch");
    return coll_allreduce_sum(L, vec, n, [](gpb200_handle* q) { return q->red.data(); });
}
int coll_allreduce_min_info(const Locals& L) {
    gpb200_handle* h0 = L[0];
    const int R = h0->nranks;
    if (R <= 1) return GPB200_OK;
    if (!h0->grp) {
        SCKN(h0, g_nccl.AllReduce(h0->info_dev, h0->info_dev, 1, ncclInt32, ncclMin, h0->comm, h0->st));
        return GPB200_OK;
    }
    std::vector<cudaEvent_t> ready(R), copied(R);
    for (int q = 0; q < R; ++q) { ready[q] = ring_event(L[q]); SCK(L[q], cudaEventRecord(ready[q], L[q]->st)); }
    for (int q = 0; q < R; ++q) {
        for (int p = 0; p < R; ++p) {
            if (p != q) SCK(L[q], cudaStreamWaitEvent(L[q]->st, ready[p], 0));
            SCK(L[q], cudaMemcpyAsync(L[q]->redi + p, L[p]->info_dev, sizeof(int), cudaMemcpyDeviceToDevice, L[q]->st));
        }
        copied[q] = ring_event(L[q]);
        SCK(L[q], cudaEventRecord(copied[q], L[q]->st));
    }
    for (int q = 0; q < R; ++q) {
        for (int p = 0; p < R; ++p)
            if (p != q) SCK(L[q], cudaStreamWaitEvent(L[q]->st, copied[p], 0));
        SCK(L[q], shard_min_ranks(L[q]->info_dev, L[q]->redi, R, L[q]->st, &L[q]->launches));
    }
    return GPB200_OK;
}

// ---- storage ---------------------------------------------------------------------------------------------------
int shard_panel_width(gpb200_handle* h) { return h->rb * TILE; }

int shard_pick_rb(gpb200_handle* h) {
    if (h->shard_rb_opt > 0) return h->shard_rb_opt;
    // ~>= 8 panels per rank, panel width 512 (K = 512 GEMMs) up to 1024 for very large N
    const long long tiles = h->Npad / TILE;
    int rb = 4;
    if (tiles / (8LL * h->nranks) >= 16) rb = 8;
    while (rb > 1 && tiles / ((long long)rb * h->nranks) < 2) rb /= 2;
    return rb;
}

void shard_free_buffers(gpb200_handle* h) {
    for (DevBuf<double>& b : h->P) b.reset();
    for (DevBuf<double>& b : h->XRbig) b.reset();
    h->Sbuf.reset(); h->red.reset(); h->redi.reset();
    h->S_per_rank = 0;
}

// free F / G whatever their mode (with the row-sharded cross-validation work matrices, which share their layout)
void free_FG(gpb200_handle* h) {
    if (h->sharded) {
        vm_free(h->vmF); vm_free(h->vmG);
        vm_free(h->vmCvY); vm_free(h->vmCvM);
        h->g_sym = h->cv_m_ok = false;
        shard_free_buffers(h);
    } else {
        h->Frep.reset(); h->Grep.reset();
    }
    h->F = h->G = nullptr;
    h->sharded = false;
    h->factored = h->inv_ready = h->s_ready = false;
}

bool make_FG_maps(gpb200_handle* h) {
    return gemm_make_tensor_map(&h->mapF, h->F, h->Npad, h->Npad, h->Npad) &&
           gemm_make_tensor_map(&h->mapG, h->G, h->Npad, h->Npad, h->Npad) &&
           gemm_make_tensor_map(&h->mapDinv, h->Dinv, h->Npad, TILE, TILE) &&
           gemm_make_tensor_map(&h->mapDinvT, h->DinvT, h->Npad, TILE, TILE);
}

int alloc_FG_replicated(gpb200_handle* h) {
    const size_t nn = (size_t)h->Npad * (size_t)h->Npad;
    CK(h->Frep.alloc(nn));
    h->F = h->Frep;
    CK(h->Grep.alloc(nn));
    h->G = h->Grep;
    CK(cudaMemsetAsync(h->F, 0, sizeof(double) * nn, h->st));
    CK(cudaMemsetAsync(h->G, 0, sizeof(double) * nn, h->st));
    h->sharded = false;
    h->tma_ok = make_FG_maps(h);
    return GPB200_OK;
}

// byte ranges of the own 128-row tiles of an Npad x Npad row-major matrix
std::vector<std::pair<size_t, size_t>> own_row_runs(gpb200_handle* h) {
    const size_t rowb = (size_t)h->Npad * sizeof(double);
    std::vector<std::pair<size_t, size_t>> want;
    for (long long t = 0; t < h->Npad / TILE; ++t)
        if (owner_of_tile(h, t) == h->rank) want.push_back({(size_t)t * TILE * rowb, (size_t)TILE * rowb});
    return want;
}

int alloc_FG_sharded(gpb200_handle* h) {
    const size_t Np = (size_t)h->Npad;
    const size_t rowb = Np * sizeof(double);
    h->rb = shard_pick_rb(h);
    const auto want = own_row_runs(h);
    const long long tiles = (long long)(Np / TILE);
    h->sharded = true;                                          // so that a failure below is cleaned up by free_FG
    TRY(vm_alloc(h, h->vmF, Np * rowb, want));
    TRY(vm_alloc(h, h->vmG, Np * rowb, want));
    h->F = (double*)h->vmF.base;
    h->G = (double*)h->vmG.base;
    const size_t nbp = (size_t)shard_panel_width(h);
    const size_t pelems = Np * nbp;
    for (DevBuf<double>& b : h->P) CK(b.alloc(pelems));
    // all-gather staging: every rank's rows below a panel, padded to the largest per-rank count
    const size_t max_own_tiles = (size_t)shard_own_before(tiles, 0, h->rb, h->nranks);      // rank 0 owns the most
    h->S_per_rank = max_own_tiles * TILE * nbp;
    const size_t selems = std::max(h->S_per_rank * (size_t)h->nranks, pelems);
    CK(h->Sbuf.alloc(selems));
    // batched LAUUM part of the inverse sweep: up to 4096 columns of row panels at a time (two buffers: look-ahead)
    h->xr_batch = std::max<int>(1, (int)(4096 / nbp));
    for (DevBuf<double>& b : h->XRbig) CK(b.alloc((size_t)h->xr_batch * nbp * Np));
    CK(h->red.alloc(4096 * 8));
    CK(h->redi.alloc(16));
    h->tma_ok = make_FG_maps(h) &&
                gemm_make_tensor_map(&h->mapP[0], h->P[0], Np, nbp, nbp) &&
                gemm_make_tensor_map(&h->mapP[1], h->P[1], Np, nbp, nbp) &&
                gemm_make_tensor_map(&h->mapP[2], h->P[2], Np, nbp, nbp) &&
                gemm_make_tensor_map(&h->mapP[3], h->P[3], Np, nbp, nbp) &&
                gemm_make_tensor_map(&h->mapXR[0], h->P[1], nbp, Np, Np) &&
                gemm_make_tensor_map(&h->mapXR[1], h->P[3], nbp, Np, Np) &&
                gemm_make_tensor_map(&h->mapS, h->Sbuf, Np, nbp, nbp) &&
                gemm_make_tensor_map(&h->mapXRbig[0], h->XRbig[0], (int64_t)h->xr_batch * nbp, Np, Np) &&
                gemm_make_tensor_map(&h->mapXRbig[1], h->XRbig[1], (int64_t)h->xr_batch * nbp, Np, Np);
    // without TMA descriptors the GEMMs fall back to the plain-load kernel (launch_gemm), storage_info reports it
    return GPB200_OK;
}

// should F / G of this handle be row-sharded?  (identical decision on every rank: depends on sizes and options only)
bool want_sharded(gpb200_handle* h) {
    if (h->nranks <= 1) return false;
    if (h->grp) return true;                                     // an in-process group exists only for the sharded schedules
    if (h->shard_opt == 0) return false;
    if (h->shard_opt == 1) return true;
    size_t fr = 0, tot = 0;
    if (cudaMemGetInfo(&fr, &tot) != cudaSuccess) { (void)cudaGetLastError(); return false; }
    const double need = 2.0 * 8.0 * (double)h->Npad * (double)h->Npad * 1.12;      // F + G + panels / workspaces
    return need > 0.9 * (double)tot;
}

// (re)allocate F / G in the mode the current communicator / options ask for
int ensure_storage(gpb200_handle* h) {
    const bool want = want_sharded(h);
    const bool ok_now = h->F && h->G && h->sharded == want && (!want || h->rb == shard_pick_rb(h));
    if (ok_now) return GPB200_OK;
    CK(cudaStreamSynchronize(h->st));
    close_peer_maps(h);                                       // peers' IPC views of the old buffers die with them (every rank re-allocates)
    if (h->F || h->G) free_FG(h);
    return want ? alloc_FG_sharded(h) : alloc_FG_replicated(h);
}

GemmBuf bufP(gpb200_handle* h, int i) { return GemmBuf{&h->mapP[i], h->P[i], (int64_t)shard_panel_width(h)}; }
GemmBuf bufXR(gpb200_handle* h, int set = 0) { return GemmBuf{&h->mapXR[set], h->P[2 * set + 1], h->Npad}; }
GemmBuf bufS(gpb200_handle* h) { return GemmBuf{&h->mapS, h->Sbuf, (int64_t)shard_panel_width(h)}; }

void own_rows_filter(gpb200_handle* h, GemmDesc& g, int row0) {
    g.bm_mod = h->nranks; g.bm_rem = h->rank; g.bm_div = h->rb; g.bm_off = row0 / TILE;
}
void own_cols_filter(gpb200_handle* h, GemmDesc& g, int row0_of_B) {
    g.bn_mod = h->nranks; g.bn_rem = h->rank; g.bn_div = h->rb; g.bn_off = row0_of_B / TILE;
}

// ---- Cholesky -------------------------------------------------------------------------------------------------
// G[r1.., c0+off .. c0+off+n) <- (same) * L_kk[off.., off..]^-T  on this rank's rows >= r1 (L_kk sits in P[pb] rows c0..)
cudaError_t shard_trsm_rows(gpb200_handle* h, int c0, int r1, int off, int n, int pb) {
    const int rows = (int)h->Npad - r1;
    if (n == TILE) {
        GemmDesc g = gemm_desc_default();
        g.A = GemmOperand{bufG(h), bufNone(), r1, c0 + off};
        g.B = GemmOperand{bufDinv(h), bufNone(), c0 + off, 0};
        g.C = h->G; g.ldc = h->ld; g.c_row0 = r1; g.c_col0 = c0 + off;
        g.M = rows; g.N = TILE; g.K = TILE;
        own_rows_filter(h, g, r1);
        return launch_gemm(h, g);
    }
    int n1 = TILE;
    while (n1 * 2 < n) n1 *= 2;
    const int n2 = n - n1;
    cudaError_t e;
    if ((e = shard_trsm_rows(h, c0, r1, off, n1, pb)) != cudaSuccess) return e;
    {
        GemmDesc g = gemm_desc_default();
        g.A = GemmOperand{bufG(h), bufNone(), r1, c0 + off};
        g.B = GemmOperand{bufP(h, pb), bufNone(), c0 + off + n1, off};                 // L21 of the diagonal block
        g.C = h->G; g.ldc = h->ld; g.c_row0 = r1; g.c_col0 = c0 + off + n1;
        g.M = rows; g.N = n2; g.K = n1;
        g.alpha = -1.0; g.beta = 1.0;
        own_rows_filter(h, g, r1);
        if ((e = launch_gemm(h, g)) != cudaSuccess) return e;
    }
    return shard_trsm_rows(h, c0, r1, off + n1, n2, pb);
}

// Per panel (see the file head) with LOOK-AHEAD: the latency-bound chain of a panel (diagonal-block factorisation, its broadcast, the
// R-way split TRSM, the all-gather) runs on the high-priority side stream while the main stream applies the PREVIOUS panel
// to the bulk of the trailing matrix.  Per panel the main stream first updates only the columns of the next block ("narrow"
// update, K = NBp, a few hundred tiles), hands over to the chain, then does the rest.  Panel buffers alternate (P[k & 1]).
// `kb0` > 0 factors only the trailing matrix from block kb0 on (append: the blocks before it are already factored).
int shard_cholesky_la(const Locals& L, int kb0 = 0) {
    gpb200_handle* h0 = L[0];
    const int Np = (int)h0->Npad, R = h0->nranks, NBp = shard_panel_width(h0);
    const int nblk = (Np + NBp - 1) / NBp;
    const long long tiles = Np / TILE;
    for (auto* q : L) {
        if (!q->st_side) return rank_failed(q, fail(q, GPB200_ECUDA, "sharded look-ahead needs the side stream"));
        cudaEvent_t e = ring_event(q);                       // the chain starts after the Gram build
        SCK(q, cudaEventRecord(e, q->st));
        SCK(q, cudaStreamWaitEvent(q->st_side, e, 0));
    }
    std::vector<cudaEvent_t> ev_panel(L.size());
    for (int k = kb0; k < nblk; ++k) {
        const int c0 = k * NBp, nb = std::min(NBp, Np - c0), o = k % R, r1 = c0 + nb, pb = k & 1;
        const int t1 = r1 / TILE;
        // ---------------- chain of panel k, on the side streams ----------------
        for (auto* q : L) std::swap(q->st, q->st_side);
        int rc = GPB200_OK;
        do {
            for (auto* q : L) {
                if (q->rank != o) continue;
                const int la = q->lookahead;
                q->lookahead = 0; q->row_lim = r1;
                cudaError_t e = chol_panel(q, c0, nb, NBp);
                q->row_lim = 0; q->lookahead = la;
                if (e != cudaSuccess) { q->err = std::string("chol_panel: ") + cudaGetErrorString(e); rc = rank_failed(q, GPB200_ECUDA); break; }
                e = shard_copy_lower(q->P[pb] + (size_t)c0 * NBp, NBp, q->F + (size_t)c0 * q->ld + c0, q->ld, nb, q->st, &q->launches);
                if (e != cudaSuccess) { q->err = cudaGetErrorString(e); rc = rank_failed(q, GPB200_ECUDA); break; }
            }
            if (rc) break;
            if ((rc = coll_group_begin(L))) break;
            if ((rc = coll_bcast(L, o, [&](gpb200_handle* q) { return (void*)(q->P[pb] + (size_t)c0 * NBp); }, sizeof(double) * (size_t)nb * NBp))) break;
            if ((rc = coll_bcast(L, o, [&](gpb200_handle* q) { return (void*)(q->Dinv + (size_t)c0 * TILE); }, sizeof(double) * (size_t)nb * TILE))) break;
            if ((rc = coll_bcast(L, o, [&](gpb200_handle* q) { return (void*)(q->DinvT + (size_t)c0 * TILE); }, sizeof(double) * (size_t)nb * TILE))) break;
            if ((rc = coll_bcast(L, o, [&](gpb200_handle* q) { return (void*)(q->logd + c0); }, sizeof(double) * (size_t)nb))) break;
            if ((rc = coll_group_end(L))) break;
            if (r1 >= Np) break;
            long long maxown = 0;
            for (int q = 0; q < R; ++q)
                maxown = std::max(maxown, shard_own_before(tiles, q, h0->rb, R) - shard_own_before(t1, q, h0->rb, R));
            const size_t per = (size_t)maxown * TILE * NBp;
            for (auto* q : L) {
                cudaError_t e = shard_trsm_rows(q, c0, r1, 0, nb, pb);
                if (e == cudaSuccess) e = shard_scatter_rows(q->G, q->F, q->ld, Np, c0, nb, t1, q->Sbuf + (size_t)q->rank * per, NBp, own_of(q), q->st, &q->launches);
                if (e != cudaSuccess) { q->err = cudaGetErrorString(e); rc = rank_failed(q, GPB200_ECUDA); break; }
            }
            if (rc) break;
            if ((rc = coll_allgather(L, [&](gpb200_handle* q) { return (void*)q->Sbuf; }, sizeof(double) * per))) break;
            for (auto* q : L) {
                cudaError_t e = shard_unpack_panel(q->P[pb], NBp, Np, nb, t1, q->Sbuf, (int64_t)per, own_of(q), q->st, &q->launches);
                if (e == cudaSuccess && q->rank == o) {
                    e = shard_transpose(q->F + (size_t)c0 * q->ld + r1, q->ld, q->P[pb] + (size_t)r1 * NBp, NBp, Np - r1, nb, q->st, &q->launches);
                }
                if (e != cudaSuccess) { q->err = cudaGetErrorString(e); rc = rank_failed(q, GPB200_ECUDA); break; }
            }
        } while (false);
        if (!rc) {
            for (size_t i = 0; i < L.size(); ++i) {
                ev_panel[i] = ring_event(L[i]);
                if (cudaEventRecord(ev_panel[i], L[i]->st) != cudaSuccess) { L[i]->err = "cudaEventRecord failed"; rc = rank_failed(L[i], GPB200_ECUDA); }
            }
        }
        for (auto* q : L) std::swap(q->st, q->st_side);           // back to the main streams
        if (rc) return rc;
        if (r1 >= Np) {
            for (size_t i = 0; i < L.size(); ++i) SCK(L[i], cudaStreamWaitEvent(L[i]->st, ev_panel[i], 0));
            break;
        }
        // ---------------- main streams: apply panel k ----------------
        const int nb1 = std::min(NBp, Np - r1), r2 = r1 + nb1;
        for (size_t i = 0; i < L.size(); ++i) {
            gpb200_handle* q = L[i];
            SCK(q, cudaStreamWaitEvent(q->st, ev_panel[i], 0));
            {   // narrow: the columns of the next block, own rows >= r1 (lower trapezoid)
                GemmDesc g = gemm_desc_default();
                g.A = GemmOperand{bufP(q, pb), bufNone(), r1, 0};
                g.B = GemmOperand{bufP(q, pb), bufNone(), r1, 0};
                g.C = q->G; g.ldc = q->ld; g.c_row0 = r1; g.c_col0 = r1;
                g.M = Np - r1; g.N = nb1; g.K = nb;
                g.alpha = -1.0; g.beta = 1.0;
                g.flags = GEMM_LOWER_ONLY;
                own_rows_filter(q, g, r1);
                SCK(q, launch_gemm(q, g));
            }
            cudaEvent_t e = ring_event(q);
            SCK(q, cudaEventRecord(e, q->st));
            SCK(q, cudaStreamWaitEvent(q->st_side, e, 0));           // the chain of panel k+1 may start
            if (r2 < Np) {   // the rest of the trailing matrix
                GemmDesc g = gemm_desc_default();
                g.A = GemmOperand{bufP(q, pb), bufNone(), r2, 0};
                g.B = GemmOperand{bufP(q, pb), bufNone(), r2, 0};
                g.C = q->G; g.ldc = q->ld; g.c_row0 = r2; g.c_col0 = r2;
                g.M = Np - r2; g.N = Np - r2; g.K = nb;
                g.alpha = -1.0; g.beta = 1.0;
                g.flags = GEMM_LOWER_ONLY;
                own_rows_filter(q, g, r2);
                SCK(q, launch_gemm(q, g));
            }
        }
    }
    return coll_allreduce_min_info(L);
}

// ---- triangular solves (one right-hand side) ---------------------------------------------------------------------
// out = K_y^-1 rhs on every rank; rhs (device, Npad, zero padded) identical on every rank; tmp/y scratch vectors
int shard_solve(const Locals& L, DevBuf<double> gpb200_handle::*rhs, DevBuf<double> gpb200_handle::*ybuf, DevBuf<double> gpb200_handle::*out) {
    gpb200_handle* h0 = L[0];
    const int Np = (int)h0->Npad, R = h0->nranks, NBp = shard_panel_width(h0);
    const int nblk = (Np + NBp - 1) / NBp;
    // forward: L y = r on the rows of L
    for (int k = 0; k < nblk; ++k) {
        const int c0 = k * NBp, nb = std::min(NBp, Np - c0), o = k % R;
        for (auto* q : L) {
            if (q->rank != o) continue;
            double* r = q->*rhs; double* y = q->*ybuf;
            double* t = q->tblk;                     // nb-vector scratch
            if (c0 > 0) {
                SCK(q, rowdot_launch(q->F + (size_t)c0 * q->ld, q->ld, y, nb, c0, t, q->st, &q->launches));
                SCK(q, ew_launch(6, nb, t, r + c0, t, nullptr, 0.0, q->st, &q->launches));                 // t = r_k - L[k, <k] y
            } else {
                SCK(q, cudaMemcpyAsync(t, r, sizeof(double) * nb, cudaMemcpyDeviceToDevice, q->st));
            }
            SCK(q, trsv_lower_fwd(q->F + (size_t)c0 * q->ld + c0, q->ld, q->Dinv + (size_t)c0 * TILE, t, y + c0, nb, q->st, &q->launches));
        }
        TRY(coll_bcast(L, o, [&](gpb200_handle* q) { return (void*)(q->*ybuf + c0); }, sizeof(double) * (size_t)nb));
    }
    // backward: U a = y on the rows of U = L' (upper part of F)
    for (int k = nblk - 1; k >= 0; --k) {
        const int c0 = k * NBp, nb = std::min(NBp, Np - c0), o = k % R, r1 = c0 + nb;
        for (auto* q : L) {
            if (q->rank != o) continue;
            double* y = q->*ybuf; double* a = q->*out;
            double* t = q->tblk;
            if (r1 < Np) {
                SCK(q, rowdot_launch(q->F + (size_t)c0 * q->ld + r1, q->ld, a + r1, nb, Np - r1, t, q->st, &q->launches));
                SCK(q, ew_launch(6, nb, t, y + c0, t, nullptr, 0.0, q->st, &q->launches));                 // t = y_k - U[k, >k] a
            } else {
                SCK(q, cudaMemcpyAsync(t, y + c0, sizeof(double) * nb, cudaMemcpyDeviceToDevice, q->st));
            }
            SCK(q, trsv_lower_bwd(q->F + (size_t)c0 * q->ld + c0, q->ld, q->DinvT + (size_t)c0 * TILE, t, a + c0, nb, q->st, &q->launches));
        }
        TRY(coll_bcast(L, o, [&](gpb200_handle* q) { return (void*)(q->*out + c0); }, sizeof(double) * (size_t)nb));
    }
    return GPB200_OK;
}

// ---- inverse: backward sweep over row panels (see the file head) with LOOK-AHEAD ---------------------------------------
// Chain of panel J (side stream): finalise X_J, broadcast, transpose, and the part of the TRTRI update that the NEXT
// finalisation needs (rows of block J-1 only); main stream: the bulk TRTRI update (rows before block J-1) and the LAUUM
// part of panel J.  Panel buffers alternate between two sets {P[2s], P[2s+1]}.  Dependencies:
//   chain(K) starts after main(K+2) finished (its accumulators received panel K+2's contribution; buffer set K&1 is free),
//   its narrow update waits for main(K+1)'s TRTRI part (both add into the rows of block K-1), main(K) waits for chain(K).
int shard_inverse_la(const Locals& L) {
    gpb200_handle* h0 = L[0];
    const int Np = (int)h0->Npad, R = h0->nranks, NBp = shard_panel_width(h0);
    const int nblk = (Np + NBp - 1) / NBp;
    const size_t nl = L.size();
    for (auto* q : L) {
        if (!q->st_side) return rank_failed(q, fail(q, GPB200_ECUDA, "sharded look-ahead needs the side stream"));
        for (auto& run : q->vmG.runs) SCK(q, cudaMemsetAsync((char*)q->G + run.first, 0, run.second, q->st));
        // W_kk = L_kk^-1 of the own diagonal blocks, level by level (strictly-lower tiles -> G lower, transposed -> G upper;
        // the diagonal tiles stay in Dinv / DinvT, substituted by the GEMM producer)
        for (int k = q->rank; k < nblk; k += R) {
            const int c0 = k * NBp, nb = std::min(NBp, Np - c0);
            for (int s = TILE; s < nb; s *= 2) {
                const int batch = (nb + 2 * s - 1) / (2 * s);
                const int n2 = (nb - s < s) ? nb - s : s;
                SCK(q, merge_inverse(q, c0, s, n2, batch));
            }
        }
        cudaEvent_t e = ring_event(q);
        SCK(q, cudaEventRecord(e, q->st));
        SCK(q, cudaStreamWaitEvent(q->st_side, e, 0));
    }
    // per local rank: events of the two previous main steps
    std::vector<cudaEvent_t> ev_full1(nl, nullptr), ev_full2(nl, nullptr), ev_trtri1(nl, nullptr), ev_panel(nl, nullptr);
    // The LAUUM part is applied per BATCH of gB consecutive panels: one panel alone gives N = NBp output columns, i.e. fewer
    // tiles than SMs with inner dimensions up to Npad -- measured at C2 on 8 GPUs: 200 ms for the sweep, bound by the
    // duration of a single long-K tile per panel.  The row-panel forms X_J of a batch are collected in XRbig[batch & 1].
    const int gB = h0->xr_batch;
    for (int k = nblk - 1; k >= 0; --k) {
        const int j0 = k * NBp, nb = std::min(NBp, Np - j0), o = k % R, r1 = j0 + nb;
        const int ncols = Np - r1, set = k & 1;
        const int bidx = (nblk - 1 - k) / gB;                        // batch of this panel
        const int k_first = nblk - 1 - bidx * gB, k_low = std::max(0, k_first - gB + 1);
        const int j0L = k_low * NBp, xb = bidx & 1;
        const int batch_cols = std::min(Np, (k_first + 1) * NBp) - j0L;
        const int j0p = (k > 0) ? (k - 1) * NBp : 0;                 // start of block k-1 (size NBp)
        // ---------------- chain of panel k ----------------
        for (size_t i = 0; i < nl; ++i) {
            gpb200_handle* q = L[i];
            if (ev_full2[i]) SCK(q, cudaStreamWaitEvent(q->st_side, ev_full2[i], 0));       // main(k+2) done
            std::swap(q->st, q->st_side);
        }
        int rc = GPB200_OK;
        do {
            // owner: finalise X_J.  Beyond the block: Xt[c, i] = -sum_k accT[c, k] Wt_JJ[i, k]  (accT = transposed accumulator),
            // written as the column panel and, through the transposed-copy epilogue, as rows of X in place (G upper);
            // inside the block: Xt = W_JJ
            for (auto* q : L) {
                if (q->rank != o) continue;
                cudaError_t e = cudaSuccess;
                if (ncols > 0) {
                    e = shard_transpose(q->Sbuf + (size_t)r1 * NBp, NBp, q->G + (size_t)j0 * q->ld + r1, q->ld, nb, ncols, q->st, &q->launches);
                    GemmDesc g = gemm_desc_default();
                    g.A = GemmOperand{bufS(q), bufNone(), r1, 0};
                    g.B = GemmOperand{bufG(q), bufDinvT(q), j0, j0};
                    g.C = q->P[2 * set]; g.ldc = NBp; g.c_row0 = r1; g.c_col0 = 0;
                    g.Ct = q->G; g.ldct = q->ld; g.ct_row0 = j0; g.ct_col0 = r1;
                    g.M = ncols; g.N = nb; g.K = nb;
                    g.alpha = -1.0;
                    g.flags = GEMM_KLO_N;
                    if (e == cudaSuccess) e = launch_gemm(q, g);
                }
                if (e == cudaSuccess) e = shard_pack_wblock(q->P[2 * set], NBp, q->G, q->ld, q->Dinv, j0, nb, q->st, &q->launches);
                if (e != cudaSuccess) { q->err = cudaGetErrorString(e); rc = rank_failed(q, GPB200_ECUDA); break; }
            }
            if (rc) break;
            if ((rc = coll_bcast(L, o, [&](gpb200_handle* q) { return (void*)(q->P[2 * set] + (size_t)j0 * NBp); },
                                 sizeof(double) * (size_t)(Np - j0) * NBp))) break;
            for (size_t i = 0; i < nl; ++i) {
                gpb200_handle* q = L[i];
                cudaError_t e = shard_transpose(q->XRbig[xb] + (size_t)(j0 - j0L) * Np + j0, Np, q->P[2 * set] + (size_t)j0 * NBp, NBp,
                                                Np - j0, nb, q->st, &q->launches);
                if (e == cudaSuccess && k > 0 && q->rank == (k - 1) % R) {
                    // narrow TRTRI update: the accumulator rows of block k-1 (the next panel to be finalised)
                    if (ev_trtri1[i]) e = cudaStreamWaitEvent(q->st, ev_trtri1[i], 0);           // main(k+1)'s TRTRI part adds into the same rows
                    GemmDesc g = gemm_desc_default();
                    g.A = GemmOperand{bufF(q), bufNone(), j0p, j0};
                    g.B = GemmOperand{bufP(q, 2 * set), bufNone(), j0, 0};
                    g.C = q->G; g.ldc = q->ld; g.c_row0 = j0p; g.c_col0 = j0;
                    g.M = NBp; g.N = Np - j0; g.K = nb;
                    g.alpha = 1.0; g.beta = 1.0;
                    if (e == cudaSuccess) e = launch_gemm(q, g);
                }
                if (e != cudaSuccess) { q->err = cudaGetErrorString(e); rc = rank_failed(q, GPB200_ECUDA); break; }
            }
        } while (false);
        if (!rc) {
            for (size_t i = 0; i < nl; ++i) {
                ev_panel[i] = ring_event(L[i]);
                if (cudaEventRecord(ev_panel[i], L[i]->st) != cudaSuccess) { L[i]->err = "cudaEventRecord failed"; rc = rank_failed(L[i], GPB200_ECUDA); }
            }
        }
        for (auto* q : L) std::swap(q->st, q->st_side);
        if (rc) return rc;
        // ---------------- main streams: bulk of panel k ----------------
        for (size_t i = 0; i < nl; ++i) {
            gpb200_handle* q = L[i];
            SCK(q, cudaStreamWaitEvent(q->st, ev_panel[i], 0));
            if (j0p > 0) {   // TRTRI part for the own rows before block k-1
                GemmDesc g = gemm_desc_default();
                g.A = GemmOperand{bufF(q), bufNone(), 0, j0};
                g.B = GemmOperand{bufP(q, 2 * set), bufNone(), j0, 0};
                g.C = q->G; g.ldc = q->ld; g.c_row0 = 0; g.c_col0 = j0;
                g.M = j0p; g.N = Np - j0; g.K = nb;
                g.alpha = 1.0; g.beta = 1.0;
                own_rows_filter(q, g, 0);
                SCK(q, launch_gemm(q, g));
            }
            cudaEvent_t et = ring_event(q);
            SCK(q, cudaEventRecord(et, q->st));
            if (k == k_low) {   // LAUUM part of the whole batch [k_low, k_first] for the own rows >= j0L
                GemmDesc g = gemm_desc_default();
                g.A = GemmOperand{bufG(q), bufDinvT(q), j0L, j0L};
                g.B = GemmOperand{GemmBuf{&q->mapXRbig[xb], q->XRbig[xb], q->Npad}, bufNone(), 0, j0L};
                g.C = q->G; g.ldc = q->ld; g.c_row0 = j0L; g.c_col0 = j0L;
                g.M = Np - j0L; g.N = batch_cols; g.K = Np - j0L;
                g.flags = GEMM_LOWER_ONLY | GEMM_KLO_M;
                own_rows_filter(q, g, j0L);
                SCK(q, launch_gemm(q, g));
            }
            cudaEvent_t ef = ring_event(q);
            SCK(q, cudaEventRecord(ef, q->st));
            ev_full2[i] = ev_full1[i]; ev_full1[i] = ef; ev_trtri1[i] = et;
        }
    }
    return GPB200_OK;
}

// ---- predict: V' = K*' L^-T over column blocks (columns = training rows, owned like the rows of L) ----------------------
// Kst (Mpad x Npad) holds K*' on every rank; on return pvar = kdiag - sum_n V'[m, n]^2 (if want_var), Kss -= V'V (if cov)
int shard_predict_solve(const Locals& L, int Mpad, int64_t Mc, bool want_var, bool want_cov) {
    gpb200_handle* h0 = L[0];
    const int Np = (int)h0->Npad, R = h0->nranks, NBp = shard_panel_width(h0);
    const int nblk = (Np + NBp - 1) / NBp;
    for (int k = 0; k < nblk; ++k) {
        const int c0 = k * NBp, nb = std::min(NBp, Np - c0), o = k % R, r1 = c0 + nb;
        for (auto* q : L) {
            if (q->rank != o) continue;
            GemmBuf bk{&q->mapKst, q->Kst, q->Npad};
            SCK(q, trsm_rec_buf(q, bk, Mpad, c0, nb));
            SCK(q, cudaMemcpy2DAsync(q->P[0], sizeof(double) * NBp, q->Kst + c0, sizeof(double) * q->Npad, sizeof(double) * nb,
                                     (size_t)Mpad, cudaMemcpyDeviceToDevice, q->st));
        }
        TRY(coll_bcast(L, o, [&](gpb200_handle* q) { return (void*)q->P[0]; }, sizeof(double) * (size_t)Mpad * NBp));
        for (auto* q : L) {
            if (want_var) SCK(q, rowvar_launch(q->P[0], NBp, q->pvar, Mc, nb, q->pvar, q->st, &q->launches));
            if (r1 < Np) {
                GemmDesc g = gemm_desc_default();
                g.A = GemmOperand{bufP(q, 0), bufNone(), 0, 0};
                g.B = GemmOperand{bufF(q), bufNone(), r1, c0};
                g.C = q->Kst; g.ldc = q->Npad; g.c_row0 = 0; g.c_col0 = r1;
                g.M = Mpad; g.N = Np - r1; g.K = nb;
                g.alpha = -1.0; g.beta = 1.0;
                own_cols_filter(q, g, r1);
                SCK(q, launch_gemm(q, g));
            }
            if (want_cov) {
                GemmDesc g = gemm_desc_default();
                g.A = GemmOperand{bufP(q, 0), bufNone(), 0, 0};
                g.B = GemmOperand{bufP(q, 0), bufNone(), 0, 0};
                g.C = q->Kss; g.ldc = Mpad; g.M = Mpad; g.N = Mpad; g.K = nb;
                g.alpha = -1.0; g.beta = 1.0;
                SCK(q, launch_gemm(q, g));
            }
        }
    }
    return GPB200_OK;
}

// ---- append: V = K[b0.., 0..b0) L11^-T for the Mv rows from b0 on, solved like the test points of shard_predict_solve -------
// Kst (Mv x Npad) holds K[b0.., 0..b0) on every rank.  Per old column block the owner solves it, keeps its transpose as the
// U part of its own old rows (F[c0.., b0..b0+Mv)) and broadcasts it; every rank copies the block into its Kst, which ends
// as the replicated V, and applies it to its own later columns below b0.
int shard_append_solve(const Locals& L, int b0, int Mv) {
    gpb200_handle* h0 = L[0];
    const int R = h0->nranks, NBp = shard_panel_width(h0);
    for (int k = 0; k * NBp < b0; ++k) {
        const int c0 = k * NBp, o = k % R, r1 = c0 + NBp;
        for (auto* q : L) {
            if (q->rank != o) continue;
            const GemmBuf bk = gbuf(q, q->Kst, q->mapKst, q->Npad);
            SCK(q, trsm_rec_buf(q, bk, Mv, c0, NBp));
            SCK(q, cudaMemcpy2DAsync(q->P[0], sizeof(double) * NBp, q->Kst + c0, sizeof(double) * q->Npad, sizeof(double) * NBp,
                                     (size_t)Mv, cudaMemcpyDeviceToDevice, q->st));
            SCK(q, shard_transpose(q->F + (size_t)c0 * q->ld + b0, q->ld, q->P[0], NBp, Mv, NBp, q->st, &q->launches));
        }
        TRY(coll_bcast(L, o, [&](gpb200_handle* q) { return (void*)q->P[0]; }, sizeof(double) * (size_t)Mv * NBp));
        for (auto* q : L) {
            if (q->rank != o)
                SCK(q, cudaMemcpy2DAsync(q->Kst + c0, sizeof(double) * q->Npad, q->P[0], sizeof(double) * NBp, sizeof(double) * NBp,
                                         (size_t)Mv, cudaMemcpyDeviceToDevice, q->st));
            if (r1 < b0) {
                GemmDesc g = gemm_desc_default();
                g.A = GemmOperand{bufP(q, 0), bufNone(), 0, 0};
                g.B = GemmOperand{bufF(q), bufNone(), r1, c0};
                g.C = q->Kst; g.ldc = q->Npad; g.c_row0 = 0; g.c_col0 = r1;
                g.M = Mv; g.N = b0 - r1; g.K = NBp;
                g.alpha = -1.0; g.beta = 1.0;
                own_cols_filter(q, g, r1);
                SCK(q, launch_gemm(q, g));
            }
        }
    }
    return GPB200_OK;
}

// Extend the factor by the points the caller placed at rows Nold..N of x on every rank (gpb200_append).  The rebuild starts at
// the ownership block b0 holding row Nold, so every panel factored again is one whole block with one owner; rows < b0 of L,
// their Dinv / DinvT / logd and their U part left of b0 stay.  Rows >= N up to Npad keep identity rows of L, so only the Mv
// rows b0 .. N (rounded up to a tile) carry V.
int shard_append(const Locals& L, int64_t Nold) {
    gpb200_handle* h0 = L[0];
    const int Np = (int)h0->Npad, NBp = shard_panel_width(h0);
    const int b0 = (int)(Nold / NBp * NBp);
    const int Mv = (int)((h0->N + TILE - 1) / TILE * TILE) - b0;
    for (auto* q : L)        // own Gram rows >= b0 (columns <= row), identity beyond the new N
        SCK(q, gram_lower_launch(q->prog, q->x, q->d, q->d, q->N, Np, q->noise_var, 1, q->nugget, q->G, q->ld, q->st, &q->launches,
                                 q->rb, q->nranks, q->rank, 1, b0 / TILE));
    if (b0 > 0) {
        for (auto* q : L) {
            TRY(rank_failed(q, ensure_predict_ws(q, Mv, false)));
            SCK(q, crossgram_launch(q->prog, q->x + (size_t)b0 * q->d, q->d, q->N - b0, Mv, q->x, q->d, b0, b0, q->d, q->Kst, q->Npad,
                                    q->st, &q->launches));
        }
        TRY(shard_append_solve(L, b0, Mv));
        for (auto* q : L) {
            // own rows of V are the rows of L left of b0
            for (long long t = b0 / TILE; t < (b0 + Mv) / TILE; ++t)
                if (owner_of_tile(q, t) == q->rank)
                    SCK(q, cudaMemcpy2DAsync(q->F + (size_t)t * TILE * q->ld, sizeof(double) * q->ld, q->Kst + (size_t)(t * TILE - b0) * q->Npad,
                                             sizeof(double) * q->Npad, sizeof(double) * b0, TILE, cudaMemcpyDeviceToDevice, q->st));
            // Schur complement of the own rows: G[r, c] -= V_r V_c',  r >= c >= b0
            const GemmBuf bv = gbuf(q, q->Kst, q->mapKst, q->Npad);
            GemmDesc g = gemm_desc_default();
            g.A = GemmOperand{bv, bufNone(), 0, 0};
            g.B = GemmOperand{bv, bufNone(), 0, 0};
            g.C = q->G; g.ldc = q->ld; g.c_row0 = b0; g.c_col0 = b0;
            g.M = Mv; g.N = Mv; g.K = b0;
            g.alpha = -1.0; g.beta = 1.0;
            g.flags = GEMM_LOWER_ONLY;
            own_rows_filter(q, g, b0);
            SCK(q, launch_gemm(q, g));
        }
    }
    return shard_cholesky_la(L, b0 / NBp);
}

// ---- cross-validation (gpb200_cv_param / cv_block / get_inverse_diag) ------------------------------------------------------
// After the inverse sweep the lower part of an own row of G holds K^-1; its upper part is dead scratch.  Per grad_prepare the
// rows are completed once (shard_cv_symmetrize); per parameter j (tests/test_shard_cv_model.py is the numpy specification):
//   Y' own rows = K^-1[own, :] dK_j, dK_j generated by every rank itself in row batches of up to xr_batch * NBp rows (NT:
//   dK_j is symmetric), no communication; Z_j alpha and diag(Z_j K^-1) are row-local (<Y'_i, alpha>, <K^-1_i, Y'_i>);
//   M_j = Y' K^-1 own rows, lower triangle only (symmetric): the K^-1 row panels are broadcast batch by batch.
// Communication: N^2 / 2 doubles once per grad_prepare, N^2 per cv_param, plus the N-vectors.
double* cv_y(gpb200_handle* h) { return (double*)h->vmCvY.base; }
double* cv_m(gpb200_handle* h) { return (double*)h->vmCvM.base; }
GemmBuf bufCvY(gpb200_handle* h) { return gbuf(h, cv_y(h), h->mapShCvY, h->Npad); }
GemmBuf bufXRbig(gpb200_handle* h, int set) { return gbuf(h, h->XRbig[set], h->mapXRbig[set], h->Npad); }

// Y' and M_j of every rank, backed on the own rows like F and G; all ranks or none
int shard_cv_alloc(const Locals& L) {
    bool have = true;
    for (auto* q : L) have = have && q->vmCvY.base && q->vmCvM.base;
    if (have) return GPB200_OK;
    for (auto* q : L) { SCK(q, cudaStreamSynchronize(q->st)); vm_free(q->vmCvY); vm_free(q->vmCvM); }
    for (auto* q : L) {
        const size_t total = sizeof(double) * (size_t)q->Npad * (size_t)q->Npad;
        const auto want = own_row_runs(q);
        int rc = vm_alloc(q, q->vmCvY, total, want);
        if (!rc) rc = vm_alloc(q, q->vmCvM, total, want);
        if (!rc && q->tma_ok && !(gemm_make_tensor_map(&q->mapShCvY, cv_y(q), q->Npad, q->Npad, q->Npad) &&
                                  gemm_make_tensor_map(&q->mapShCvM, cv_m(q), q->Npad, q->Npad, q->Npad)))
            rc = fail(q, GPB200_ECUDA, "cv: cuTensorMapEncodeTiled failed");
        if (rc) {
            for (auto* p : L) { vm_free(p->vmCvY); vm_free(p->vmCvM); }
            return rank_failed(q, rc);
        }
    }
    return GPB200_OK;
}

// every own row of G <- the full row of K^-1: the owner of panel k broadcasts K^-1[k, 0..c0) (staged in XRbig[0]); every rank
// writes its transpose into the upper part of its own rows < c0; the owner mirrors inside the diagonal block
int shard_cv_symmetrize(const Locals& L) {
    gpb200_handle* h0 = L[0];
    const int Np = (int)h0->Npad, R = h0->nranks, NBp = shard_panel_width(h0);
    for (int k = 0; k * NBp < Np; ++k) {
        const int c0 = k * NBp, nb = std::min(NBp, Np - c0), o = k % R;
        if (c0 > 0) {
            for (auto* q : L)
                if (q->rank == o)
                    SCK(q, cudaMemcpy2DAsync(q->XRbig[0], sizeof(double) * c0, q->G + (size_t)c0 * q->ld, sizeof(double) * q->ld,
                                             sizeof(double) * c0, nb, cudaMemcpyDeviceToDevice, q->st));
            TRY(coll_bcast(L, o, [&](gpb200_handle* q) { return (void*)q->XRbig[0]; }, sizeof(double) * (size_t)nb * c0));
            for (auto* q : L)
                SCK(q, shard_transpose_own(q->G + c0, q->ld, q->XRbig[0], c0, nb, c0, own_of(q), q->st, &q->launches));
        }
        for (auto* q : L)
            if (q->rank == o) SCK(q, symmetrize_launch(q->G + (size_t)c0 * q->ld + c0, q->ld, nb, q->st, &q->launches));
    }
    return GPB200_OK;
}

// own rows of Y' = K^-1 dK_param, dK generated row batch by row batch into XRbig[0]
int shard_cv_y(const Locals& L, int param) {
    gpb200_handle* h0 = L[0];
    const int Np = (int)h0->Npad, rows_b = h0->xr_batch * shard_panel_width(h0);
    for (int n0 = 0; n0 < Np; n0 += rows_b) {
        const int nr = std::min(rows_b, Np - n0);
        for (auto* q : L) {
            SCK(q, gram_grad_full_launch(q->prog, q->x, q->d, q->d, q->N, q->Npad, param, q->XRbig[0], q->Npad, q->st, &q->launches, n0, nr));
            GemmDesc g = gemm_desc_default();
            g.A = GemmOperand{bufG(q), bufNone(), 0, 0};
            g.B = GemmOperand{bufXRbig(q, 0), bufNone(), 0, 0};
            g.C = cv_y(q); g.ldc = q->Npad; g.c_row0 = 0; g.c_col0 = n0;
            g.M = Np; g.N = nr; g.K = Np;
            own_rows_filter(q, g, 0);
            SCK(q, launch_gemm(q, g));
        }
    }
    return GPB200_OK;
}

// own rows of the lower triangle of M_j = Y' K^-1 (Y' = K^-1 itself for the noise): per batch of K^-1 row panels (rows n0 ..
// n0 + nr) the owners broadcast them into XRbig[b & 1] on the side streams, then one lower-trapezoid GEMM on the main streams.
// The broadcast of batch b + 1 may run while the GEMM of batch b does; batch b + 2 reuses the set once GEMM b is done.
int shard_cv_m(const Locals& L, bool noise) {
    gpb200_handle* h0 = L[0];
    const int Np = (int)h0->Npad, R = h0->nranks, NBp = shard_panel_width(h0), rows_b = h0->xr_batch * NBp;
    const size_t nl = L.size();
    // [set * nl + i]: the GEMM of the last batch that read XRbig[set] is done.  A ring event: between its record and its wait
    // each rank takes at most 2 * (xr_batch + 1) <= 66 of the 128 ring events (one per panel broadcast, one per batch)
    std::vector<cudaEvent_t> ev_free(2 * nl, nullptr);
    int rc = GPB200_OK;
    for (auto* q : L) {                                        // the side streams start after the main streams' work so far
        cudaEvent_t e = ring_event(q);
        if (cudaEventRecord(e, q->st) != cudaSuccess || cudaStreamWaitEvent(q->st_side, e, 0) != cudaSuccess) {
            q->err = "cudaEventRecord failed"; rc = rank_failed(q, GPB200_ECUDA); break;
        }
    }
    std::vector<cudaEvent_t> ev_ready(nl);
    for (int b = 0, n0 = 0; !rc && n0 < Np; ++b, n0 += rows_b) {
        const int nr = std::min(rows_b, Np - n0), set = b & 1;
        for (size_t i = 0; i < nl; ++i) std::swap(L[i]->st, L[i]->st_side);
        rc = [&]() -> int {
            for (size_t i = 0; i < nl; ++i)
                if (ev_free[set * nl + i]) SCK(L[i], cudaStreamWaitEvent(L[i]->st, ev_free[set * nl + i], 0));
            for (int k = n0 / NBp; k * NBp < n0 + nr; ++k) {
                const int c0 = k * NBp, nb = std::min(NBp, Np - c0), o = k % R;
                for (auto* q : L)
                    if (q->rank == o)
                        SCK(q, cudaMemcpyAsync(q->XRbig[set] + (size_t)(c0 - n0) * Np, q->G + (size_t)c0 * q->ld,
                                               sizeof(double) * (size_t)nb * Np, cudaMemcpyDeviceToDevice, q->st));
                TRY(coll_bcast(L, o, [&](gpb200_handle* q) { return (void*)(q->XRbig[set] + (size_t)(c0 - n0) * Np); },
                               sizeof(double) * (size_t)nb * Np));
            }
            for (size_t i = 0; i < nl; ++i) {
                ev_ready[i] = ring_event(L[i]);
                SCK(L[i], cudaEventRecord(ev_ready[i], L[i]->st));
            }
            return GPB200_OK;
        }();
        for (size_t i = 0; i < nl; ++i) std::swap(L[i]->st, L[i]->st_side);
        if (rc) break;
        rc = [&]() -> int {
            for (size_t i = 0; i < nl; ++i) {
                gpb200_handle* q = L[i];
                SCK(q, cudaStreamWaitEvent(q->st, ev_ready[i], 0));
                GemmDesc g = gemm_desc_default();
                g.A = GemmOperand{noise ? bufG(q) : bufCvY(q), bufNone(), n0, 0};
                g.B = GemmOperand{bufXRbig(q, set), bufNone(), 0, 0};
                g.C = cv_m(q); g.ldc = q->Npad; g.c_row0 = n0; g.c_col0 = n0;
                g.M = Np - n0; g.N = nr; g.K = Np;
                g.flags = GEMM_LOWER_ONLY;
                own_rows_filter(q, g, n0);
                SCK(q, launch_gemm(q, g));
                ev_free[set * nl + i] = ring_event(q);
                SCK(q, cudaEventRecord(ev_free[set * nl + i], q->st));
            }
            return GPB200_OK;
        }();
    }
    return rc;
}

// own rows r < N of the tiles covering 0 .. N, compact (shard_kernels.cuh) in region q of the all-gathered buffer -> out[r]
void unpack_own_rows(gpb200_handle* h, const std::vector<double>& buf, size_t per, int width, int k, double* out) {
    for (int64_t i = 0; i < h->N; ++i) {
        const long long t = i / TILE;
        const int q = owner_of_tile(h, t);
        const long long li = shard_own_before(t, q, h->rb, h->nranks) * TILE + i % TILE;
        out[i] = buf[(size_t)q * per + (size_t)li * width + k];
    }
}
