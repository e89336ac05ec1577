// shard_kernels.cu -- see shard_kernels.cuh
#include "shard_kernels.cuh"

namespace {
constexpr int T = 128;

__global__ void copy_lower_kernel(double* __restrict__ dst, long long ldd, const double* __restrict__ src, long long lds, int n) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y;
    if (j >= n) return;
    dst[(long long)i * ldd + j] = (j <= i) ? src[(long long)i * lds + j] : 0.0;
}

// grid: (ceil(nb/128), own tile ordinal); block 128 threads x 1; each block moves one 128-row tile x 128 columns
__global__ void __launch_bounds__(256) scatter_rows_kernel(const double* __restrict__ G, double* __restrict__ F, long long ld,
                                                           int c0, int nb, long long t1, double* __restrict__ S_me, int nbp,
                                                           ShardOwn own, long long own_before_t1, long long n_tiles) {
    // blockIdx.y enumerates ALL tiles t >= t1; non-owned ones exit (cheap: a few thousand CTAs at most)
    const long long t = t1 + blockIdx.y;
    if (t >= n_tiles || (int)((t / own.rb) % own.R) != own.me) return;
    const long long li = shard_own_before(t, own.me, own.rb, own.R) - own_before_t1;     // local tile index
    const int cb = blockIdx.x * 128;
    const int c = cb + (threadIdx.x & 127);
    if (c >= nb) return;
    for (int rr = threadIdx.x >> 7; rr < T; rr += 2) {
        const long long r = t * T + rr;
        const double v = G[r * ld + c0 + c];
        F[r * ld + c0 + c] = v;
        S_me[(li * T + rr) * nbp + c] = v;
    }
}

__global__ void __launch_bounds__(256) unpack_panel_kernel(double* __restrict__ P, int nbp, int nb, long long t1,
                                                           const double* __restrict__ S, long long per_rank, ShardOwn own,
                                                           long long n_tiles) {
    const long long t = t1 + blockIdx.y;
    if (t >= n_tiles) return;
    const int q = (int)((t / own.rb) % own.R);
    const long long li = shard_own_before(t, q, own.rb, own.R) - shard_own_before(t1, q, own.rb, own.R);
    const int c = blockIdx.x * 128 + (threadIdx.x & 127);
    if (c >= nb) return;
    const double* src = S + (long long)q * per_rank;
    for (int rr = threadIdx.x >> 7; rr < T; rr += 2)
        P[(t * T + rr) * nbp + c] = src[(li * T + rr) * nbp + c];
}

__global__ void transpose_kernel(double* __restrict__ dst, long long ldd, const double* __restrict__ src, long long lds,
                                 long long rows, long long cols) {
    __shared__ double tile[32][33];
    const long long i0 = (long long)blockIdx.y * 32, j0 = (long long)blockIdx.x * 32;
    for (int y = threadIdx.y; y < 32; y += 8) {
        const long long i = i0 + y, j = j0 + threadIdx.x;
        tile[y][threadIdx.x] = (i < rows && j < cols) ? src[i * lds + j] : 0.0;
    }
    __syncthreads();
    for (int y = threadIdx.y; y < 32; y += 8) {
        const long long j = j0 + y, i = i0 + threadIdx.x;
        if (i < rows && j < cols) dst[j * ldd + i] = tile[threadIdx.x][y];
    }
}

__global__ void pack_wblock_kernel(double* __restrict__ P, int nbp, const double* __restrict__ G, long long ld,
                                   const double* __restrict__ Dinv, int j0, int nb) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x, c = blockIdx.y;       // P[(j0+c), i]
    if (i >= nb) return;
    double v = 0.0;
    if ((c >> 7) > (i >> 7)) v = G[(long long)(j0 + c) * ld + j0 + i];        // strictly-lower tile of W_JJ
    else if ((c >> 7) == (i >> 7) && c >= i) v = Dinv[(long long)(j0 + c) * T + (i & 127)];   // lower half of the diagonal tile
    P[(long long)(j0 + c) * nbp + i] = v;
}

__global__ void sum_ranks_kernel(double* __restrict__ out, const double* __restrict__ in, long long stride, int nranks, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double s = 0.0;
    for (int q = 0; q < nranks; ++q) s += in[(long long)q * stride + i];
    out[i] = s;
}
__global__ void min_ranks_kernel(int* __restrict__ out, const int* __restrict__ in, int nranks) {
    int m = in[0];
    for (int q = 1; q < nranks; ++q) m = min(m, in[q]);
    out[0] = m;
}

// global tile index of this rank's lt-th own tile
__device__ __forceinline__ long long own_tile(long long lt, const ShardOwn& own) {
    return (lt / own.rb) * ((long long)own.rb * own.R) + (long long)own.me * own.rb + lt % own.rb;
}

// 32 x 32 blocks as in transpose_kernel; a block whose destination rows lie in another rank's tile exits (32 | 128: uniform)
__global__ void transpose_own_kernel(double* __restrict__ dst, long long ldd, const double* __restrict__ src, long long lds,
                                     long long rows, long long cols, ShardOwn own) {
    __shared__ double tile[32][33];
    const long long i0 = (long long)blockIdx.y * 32, j0 = (long long)blockIdx.x * 32;
    if ((int)((j0 / T / own.rb) % own.R) != own.me) return;
    for (int y = threadIdx.y; y < 32; y += 8) {
        const long long i = i0 + y, j = j0 + threadIdx.x;
        tile[y][threadIdx.x] = (i < rows && j < cols) ? src[i * lds + j] : 0.0;
    }
    __syncthreads();
    for (int y = threadIdx.y; y < 32; y += 8) {
        const long long j = j0 + y, i = i0 + threadIdx.x;
        if (i < rows && j < cols) dst[j * ldd + i] = tile[threadIdx.x][y];
    }
}

// one CTA per own row (compact index li): the reduction order of rowdot_kernel / rowdot2_kernel (vec.cu), so every value is
// bitwise the one a single-GPU handle computes from the same rows
__global__ void __launch_bounds__(256) rowdot_own_kernel(const double* __restrict__ Y, const double* __restrict__ G, long long ld,
                                                         long long ncols, const double* __restrict__ alpha, long long N, ShardOwn own,
                                                         double* __restrict__ out) {
    __shared__ double s[256], s2[256];
    const long long li = blockIdx.x;
    const long long r = own_tile(li / T, own) * T + li % T;
    double v = 0.0, v2 = 0.0;
    if (r < N) {
        const double* ry = Y + r * ld;
        const double* rg = G + r * ld;
        for (long long c = threadIdx.x; c < ncols; c += 256) v += ry[c] * alpha[c];
        for (long long c = threadIdx.x; c < ncols; c += 256) v2 += rg[c] * ry[c];
    }
    s[threadIdx.x] = v; s2[threadIdx.x] = v2;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) { s[threadIdx.x] += s[threadIdx.x + o]; s2[threadIdx.x] += s2[threadIdx.x + o]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { out[2 * li] = s[0]; out[2 * li + 1] = s2[0]; }
}

__global__ void diag_own_kernel(const double* __restrict__ G, long long ld, long long n_own_rows, ShardOwn own, double* __restrict__ out) {
    const long long li = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (li >= n_own_rows) return;
    const long long r = own_tile(li / T, own) * T + li % T;
    out[li] = G[r * ld + r];
}

__global__ void gather_block_own_kernel(double* __restrict__ out, const double* __restrict__ src, long long ld,
                                        const long long* __restrict__ idx, long long nv, ShardOwn own) {
    const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x, a = blockIdx.y;
    if (b >= nv) return;
    const long long r = max(idx[a], idx[b]), c = min(idx[a], idx[b]);
    out[a * nv + b] = ((int)((r / T / own.rb) % own.R) == own.me) ? src[r * ld + c] : 0.0;
}

// ---- replicated storage (inverse_dist): rank q owns the 128-wide tile columns t with t % nranks == q of every W21 block; its
// "slice" is the concatenation of those tile columns (local column jl <-> global column ((jl/128)*nranks+q)*128 + jl%128)
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

// ---- device-side signalling for the fused (peer-memory) panel broadcast of cholesky_dist_p2p ----------------------
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
}  // namespace

cudaError_t shard_copy_lower(double* dst, int64_t ldd, const double* src, int64_t lds, int n, cudaStream_t st, int64_t* launches) {
    if (n <= 0) return cudaSuccess;
    dim3 grid((n + 127) / 128, n);
    copy_lower_kernel<<<grid, 128, 0, st>>>(dst, ldd, src, lds, n);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t shard_scatter_rows(const double* G, double* F, int64_t ld, int64_t Npad, int c0, int nb, int t1, double* S_me,
                               int nbp, ShardOwn own, cudaStream_t st, int64_t* launches) {
    const long long n_tiles = Npad / T;
    if (t1 >= n_tiles || nb <= 0) return cudaSuccess;
    dim3 grid((nb + 127) / 128, (unsigned)(n_tiles - t1));
    scatter_rows_kernel<<<grid, 256, 0, st>>>(G, F, ld, c0, nb, t1, S_me, nbp, own,
                                              shard_own_before(t1, own.me, own.rb, own.R), n_tiles);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t shard_unpack_panel(double* P, int nbp, int64_t Npad, int nb, int t1, const double* S, int64_t per_rank,
                               ShardOwn own, cudaStream_t st, int64_t* launches) {
    const long long n_tiles = Npad / T;
    if (t1 >= n_tiles || nb <= 0) return cudaSuccess;
    dim3 grid((nb + 127) / 128, (unsigned)(n_tiles - t1));
    unpack_panel_kernel<<<grid, 256, 0, st>>>(P, nbp, nb, t1, S, per_rank, own, n_tiles);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t shard_transpose(double* dst, int64_t ldd, const double* src, int64_t lds, int64_t rows, int64_t cols, cudaStream_t st, int64_t* launches) {
    if (rows <= 0 || cols <= 0) return cudaSuccess;
    // grid.y is limited to 65535 blocks of 32 rows: rows <= 65535 * 32 = 2 097 120 (32 short of 2^21)
    dim3 grid((unsigned)((cols + 31) / 32), (unsigned)((rows + 31) / 32)), block(32, 8);
    transpose_kernel<<<grid, block, 0, st>>>(dst, ldd, src, lds, rows, cols);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t shard_pack_wblock(double* P, int nbp, const double* G, int64_t ld, const double* Dinv, int j0, int nb, cudaStream_t st, int64_t* launches) {
    if (nb <= 0) return cudaSuccess;
    dim3 grid((nb + 127) / 128, nb);
    pack_wblock_kernel<<<grid, 128, 0, st>>>(P, nbp, G, ld, Dinv, j0, nb);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t shard_sum_ranks(double* out, const double* in, int64_t stride, int nranks, int64_t n, cudaStream_t st, int64_t* launches) {
    if (n <= 0) return cudaSuccess;
    sum_ranks_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(out, in, stride, nranks, n);
    if (launches) ++*launches;
    return cudaGetLastError();
}
cudaError_t shard_min_ranks(int* out, const int* in, int nranks, cudaStream_t st, int64_t* launches) {
    min_ranks_kernel<<<1, 1, 0, st>>>(out, in, nranks);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t shard_transpose_own(double* dst, int64_t ldd, const double* src, int64_t lds, int64_t rows, int64_t cols, ShardOwn own,
                                cudaStream_t st, int64_t* launches) {
    if (rows <= 0 || cols <= 0) return cudaSuccess;
    dim3 grid((unsigned)((cols + 31) / 32), (unsigned)((rows + 31) / 32)), block(32, 8);
    transpose_own_kernel<<<grid, block, 0, st>>>(dst, ldd, src, lds, rows, cols, own);
    if (launches) ++*launches;
    return cudaGetLastError();
}

int64_t shard_own_rows(int64_t n, ShardOwn own) {
    return shard_own_before((n + T - 1) / T, own.me, own.rb, own.R) * T;
}

cudaError_t shard_rowdot_own(const double* Y, const double* G, int64_t ld, int64_t ncols, const double* alpha, int64_t N, ShardOwn own,
                             double* out, cudaStream_t st, int64_t* launches) {
    const int64_t n = shard_own_rows(N, own);
    if (n <= 0) return cudaSuccess;
    rowdot_own_kernel<<<(unsigned)n, 256, 0, st>>>(Y, G, ld, ncols, alpha, N, own, out);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t shard_diag_own(const double* G, int64_t ld, int64_t N, ShardOwn own, double* out, cudaStream_t st, int64_t* launches) {
    const int64_t n = shard_own_rows(N, own);
    if (n <= 0) return cudaSuccess;
    diag_own_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(G, ld, n, own, out);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t shard_gather_block_own(double* out, const double* src, int64_t ld, const long long* idx, int64_t nv, ShardOwn own,
                                   cudaStream_t st, int64_t* launches) {
    if (nv <= 0) return cudaSuccess;
    dim3 grid((unsigned)((nv + 255) / 256), (unsigned)nv);
    gather_block_own_kernel<<<grid, 256, 0, st>>>(out, src, ld, idx, nv, own);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t shard_pack_slices(const double* G, int64_t ld, double* out, int s, int nranks, int self, int Np, cudaStream_t st,
                              int64_t* launches) {
    const int wr = s / nranks, batch = (Np + 2 * s - 1) / (2 * s);
    dim3 blk(32, 32), grd((wr + 31) / 32, (unsigned)((s + 31) / 32), (unsigned)batch);
    pack_slices_kernel<<<grd, blk, 0, st>>>(G, ld, out, s, wr, nranks, self, Np);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t shard_unpack_slices(double* G, int64_t ld, const double* in, int64_t per_rank, int s, int nranks, int self, int Np,
                                cudaStream_t st, int64_t* launches) {
    const int wr = s / nranks, batch = (Np + 2 * s - 1) / (2 * s);
    dim3 blk(32, 32), grd((wr + 31) / 32, (unsigned)((s + 31) / 32), (unsigned)(batch * nranks));
    unpack_slices_kernel<<<grd, blk, 0, st>>>(G, ld, in, per_rank, s, wr, Np, nranks, self);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t shard_signal_peers(int* const* peer_sig_words, int n_peer, int value, cudaStream_t st, int64_t* launches) {
    signal_peers_kernel<<<1, 32, 0, st>>>(peer_sig_words, n_peer, value);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t shard_wait_signal(const int* word, int target, int* err, cudaStream_t st, int64_t* launches) {
    wait_signal_kernel<<<1, 1, 0, st>>>(word, target, err);
    if (launches) ++*launches;
    return cudaGetLastError();
}
