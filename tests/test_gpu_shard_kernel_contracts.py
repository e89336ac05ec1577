"""GPU: the data-movement kernels of the multi-rank schedules (csrc/shard_kernels.cuh), one at a time through
gpb200_shard_kernels, against the index model tests/shard_kernels_model.py.

* Row-sharded storage: copy_lower, scatter_rows, unpack_panel, transpose, pack_wblock, sum_ranks, min_ranks,
  transpose_own, rowdot_own, diag_own and gather_block_own.  One device acts as every rank of every layout (R, rb) in
  sm.LAYOUTS, at tile counts that leave ranks without a tile and end on a partial cycle.
* Replicated storage: inverse_dist's column-slice exchange (pack_slices, all-gather, unpack_slices) and the flag words of
  cholesky_dist_p2p (signal_peers, wait_signal).

These kernels copy data, or reduce in an order the model replays, so every expected value is exact and compared bit for
bit.  Every element a kernel must not read holds a NaN, and every element it must not write holds a NaN with its own
payload that must come back unchanged.  A virtual rank's input holds values only in the rows that rank owns, NaN in the
rows of the others (on sharded storage those rows are not mapped): a wrong read poisons the output instead of faulting.

The file sorts after every file that opens a torch.profiler session (torch.profiler records no device activity in a
session started about a minute or more after the process's first one); it opens none itself."""
import itertools

import numpy as np
import pytest

import shard_kernels_model as sm

pytestmark = pytest.mark.gpu

T = sm.T
IMAX = 2 ** 31 - 1
_tags = itertools.count(1)


def nan_fill(shape):
    """NaNs with a payload unique to the element and to the call: 'never read' and 'never written'"""
    n = int(np.prod(shape))
    tag = np.uint64((next(_tags) & 0x7FFFF) << 32)
    bits = np.uint64(0x7FF8_0000_0000_0000) | tag | np.arange(n, dtype=np.uint64)
    return bits.view(np.float64).reshape(shape)


def _raw(a):
    return np.ascontiguousarray(a).view(np.uint64)


def _same(got, want, what):
    bad = _raw(got) != _raw(want)
    assert not bad.any(), (what, int(bad.sum()), np.argwhere(bad)[:3].tolist())


def _torch():
    import torch
    return torch


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _host(t):
    _torch().cuda.synchronize()
    return t.cpu().numpy()


def _call(engine, name, args, launches):
    n0 = engine.launch_count()
    engine.shard_kernels(name, args)
    assert engine.launch_count() - n0 == launches, (name, engine.launch_count() - n0, launches)


def _masked_rows(dfull, mask):
    """device copy of dfull with NaN in the rows where mask is False (a rank's view of row-sharded storage)"""
    torch = _torch()
    m = torch.from_numpy(mask).to(dfull.device).reshape((-1,) + (1,) * (dfull.dim() - 1))
    return torch.where(m, dfull, torch.full_like(dfull, float("nan"))).contiguous()


def _max_own(n_tiles, t1, R, rb):
    return max(sm.own_before(n_tiles, q, R, rb) - sm.own_before(t1, q, R, rb) for q in range(R))


# ---- panel scatter and all-gather unpack (shard_cholesky_la) -----------------------------------------------------------

# (nb, nbp, c0): panel widths at and around a tile, an odd row pitch, both panel offsets
COMBOS = [(1, 1, 0), (127, 128, 128), (128, 128, 0), (129, 131, 128), (384, 385, 0), (384, 384, 128)]


@pytest.mark.parametrize("R,rb", sm.LAYOUTS)
def test_scatter_rows_unpack_panel_round_trip(engine, R, rb):
    """scatter_rows on every rank into its region of the all-gather buffer, then unpack_panel: the panel rows >= 128 t1
    of G bitwise, F gets exactly the own rows, and nothing else is written."""
    rng = np.random.default_rng(100 * R + rb)
    k = 0
    for n_tiles in sm.tile_counts(R, rb):
        Npad = n_tiles * T
        for t1 in sorted({0, 1, rb, n_tiles - 1, n_tiles} & set(range(n_tiles + 1))):
            nb, nbp, c0 = COMBOS[k % len(COMBOS)]
            k += 1
            ld = c0 + nb + 3
            Gfull = rng.standard_normal((Npad, ld))
            per = _max_own(n_tiles, t1, R, rb) * T * nbp
            launch = 1 if t1 < n_tiles else 0
            regions = []
            for me in range(R):
                mine = sm.compact_rows(n_tiles, me, R, rb)
                G = nan_fill((Npad, ld))
                G[mine, c0:c0 + nb] = Gfull[mine, c0:c0 + nb]
                F0, S0 = nan_fill((Npad, ld)), nan_fill(R * per + 7)
                dG, dF, dS = _dev(G), _dev(F0), _dev(S0)
                _call(engine, "scatter_rows", [dG.data_ptr(), dF.data_ptr(), ld, Npad, c0, nb, t1, dS.data_ptr() + 8 * me * per, nbp,
                                               R, me, rb], launch)
                what = (R, rb, n_tiles, t1, nb, nbp, c0, me)
                _same(_host(dG), G, ("G read only",) + what)
                rows = sm.compact_rows(n_tiles, me, R, rb, t1)
                wantF = F0.copy()
                wantF[rows, c0:c0 + nb] = Gfull[rows, c0:c0 + nb]
                _same(_host(dF), wantF, ("F",) + what)
                S, wantS = _host(dS), S0.copy()
                wantS[me * per:me * per + rows.size * nbp].reshape(rows.size, nbp)[:, :nb] = Gfull[rows, c0:c0 + nb]
                _same(S, wantS, ("S_me",) + what)
                regions.append(S[me * per:(me + 1) * per])
            dSall = _dev(np.concatenate(regions + [nan_fill(7)]))
            for me in sorted({0, R - 1}):                    # unpack_panel reads every rank's region: the same on every rank
                P0 = nan_fill((Npad, nbp))
                dP = _dev(P0)
                _call(engine, "unpack_panel", [dP.data_ptr(), nbp, Npad, nb, t1, dSall.data_ptr(), per, R, me, rb], launch)
                want = P0.copy()
                want[t1 * T:, :nb] = Gfull[t1 * T:, c0:c0 + nb]
                _same(_host(dP), want, ("P", R, rb, n_tiles, t1, nb, nbp, c0, me))


# ---- transposes ------------------------------------------------------------------------------------------------------

SIZES = [1, 31, 32, 33, 127, 128, 129, 1000]


def _transpose_case(engine, name, rows, cols, rng, own=None, src=None):
    lds, ldd = cols + 3, rows + 5
    if src is None:
        src = nan_fill((rows, lds))
        src[:, :cols] = rng.standard_normal((rows, cols))
    dst0 = nan_fill((cols, ldd))
    dsrc, ddst = _dev(src), _dev(dst0)
    _call(engine, name, [ddst.data_ptr(), ldd, dsrc.data_ptr(), lds, rows, cols] + (list(own) if own else []), 1)
    _same(_host(dsrc), src, (name, "src read only", rows, cols, own))
    return src, dst0, _host(ddst)


def test_transpose_every_shape(engine):
    rng = np.random.default_rng(3)
    for rows in SIZES:
        for cols in SIZES:
            src, dst0, got = _transpose_case(engine, "transpose", rows, cols, rng)
            want = dst0.copy()
            want[:, :rows] = src[:, :cols].T
            _same(got, want, ("transpose", rows, cols))


def test_transpose_grid_y_edge_65535_x_32_rows(engine):
    rows = 65535 * 32
    rng = np.random.default_rng(4)
    src = rng.standard_normal((rows, 1))
    dst0 = nan_fill(rows + 5)
    dsrc, ddst = _dev(src), _dev(dst0)
    _call(engine, "transpose", [ddst.data_ptr(), rows, dsrc.data_ptr(), 1, rows, 1], 1)
    want = dst0.copy()
    want[:rows] = src[:, 0]
    _same(_host(ddst), want, "tall transpose")


@pytest.mark.parametrize("R,rb", sm.LAYOUTS)
def test_transpose_own_writes_own_destination_rows_only(engine, R, rb):
    """every rank writes exactly the destination rows of its own tiles; the union over the ranks is the transpose"""
    rng = np.random.default_rng(10 * R + rb)
    c = R * rb
    for rows, cols in ((33, T * (3 * c + 2) - 5), (129, T * (c + 1)), (1000, 1000), (1, 1)):
        src = nan_fill((rows, cols + 3))
        src[:, :cols] = rng.standard_normal((rows, cols))
        union = np.full((cols, rows), np.nan)
        for me in range(R):
            _, dst0, got = _transpose_case(engine, "transpose_own", rows, cols, rng, own=(R, me, rb), src=src)
            mine = sm.own_row_mask(cols, me, R, rb)
            want = dst0.copy()
            want[mine, :rows] = src[:, :cols].T[mine]
            _same(got, want, ("transpose_own", R, rb, rows, cols, me))
            union[mine] = got[mine, :rows]
        _same(union, src[:, :cols].T, ("transpose_own union", R, rb, rows, cols))


# ---- diagonal-block copies -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n,ldd,lds", [(128, 128, 128), (256, 384, 300), (384, 512, 385), (512, 512, 1000)])
def test_copy_lower_zeros_above_upper_unread(engine, n, ldd, lds):
    rng = np.random.default_rng(n + ldd)
    low = np.tril(np.ones((n, n), bool))
    src = nan_fill((n, lds))
    src[:, :n][low] = rng.standard_normal(int(low.sum()))
    dst0 = nan_fill((n, ldd))
    dsrc, ddst = _dev(src), _dev(dst0)
    _call(engine, "copy_lower", [ddst.data_ptr(), ldd, dsrc.data_ptr(), lds, n], 1)
    want = dst0.copy()
    want[:, :n] = 0.0
    want[:, :n][low] = src[:, :n][low]
    _same(_host(ddst), want, ("copy_lower", n, ldd, lds))
    _same(_host(dsrc), src, "src read only")


@pytest.mark.parametrize("j0,nb,nbp", [(0, 128, 128), (128, 256, 256), (256, 384, 512), (384, 512, 640)])
def test_pack_wblock_from_lower_tiles_and_lower_diagonal_tiles(engine, j0, nb, nbp):
    """P[j0 + c, i] = W_JJ[c, i] for c >= i (strictly-lower tiles of G, the lower half of Dinv's diagonal tiles), 0 above;
    G's diagonal and upper tiles, everything outside W_JJ and Dinv's upper triangle are poisoned"""
    rng = np.random.default_rng(j0 + nb)
    Nr = j0 + nb + T
    ld = Nr + 7
    c, i = np.meshgrid(np.arange(nb), np.arange(nb), indexing="ij")
    strict = (c // T) > (i // T)
    diag = ((c // T) == (i // T)) & (c >= i)
    G = nan_fill((Nr, ld))
    blk = G[j0:j0 + nb, j0:j0 + nb]
    blk[strict] = rng.standard_normal(int(strict.sum()))
    Dinv = nan_fill((Nr, T))
    lowt = np.arange(T)[None, :] <= (np.arange(nb) % T)[:, None]
    Dinv[j0:j0 + nb][lowt] = rng.standard_normal(int(lowt.sum()))
    P0 = nan_fill((Nr, nbp))
    dP, dG, dD = _dev(P0), _dev(G), _dev(Dinv)
    _call(engine, "pack_wblock", [dP.data_ptr(), nbp, dG.data_ptr(), ld, dD.data_ptr(), j0, nb], 1)
    W = np.zeros((nb, nb))
    W[strict] = blk[strict]
    W[diag] = Dinv[j0 + c[diag], i[diag] % T]
    want = P0.copy()
    want[j0:j0 + nb, :nb] = W
    _same(_host(dP), want, ("pack_wblock", j0, nb, nbp))
    _same(_host(dG), G, "G read only")
    _same(_host(dD), Dinv, "Dinv read only")


# ---- reductions over the ranks ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("nranks", [1, 2, 3, 8])
def test_sum_ranks_left_to_right_in_rank_order(engine, nranks):
    rng = np.random.default_rng(nranks)
    for n in (1, 255, 256, 257, 100000):
        stride = n + 3
        x = rng.standard_normal((nranks, stride)) * 10.0 ** rng.integers(-12, 13, (nranks, stride))
        inb = nan_fill((nranks, stride))
        inb[:, :n] = x[:, :n]
        out0 = nan_fill(n + 4)
        din, dout = _dev(np.concatenate([inb.ravel(), nan_fill(5)])), _dev(out0)
        _call(engine, "sum_ranks", [dout.data_ptr(), din.data_ptr(), stride, nranks, n], 1)
        acc = np.zeros(n)
        for q in range(nranks):
            acc = acc + x[q, :n]
        want = out0.copy()
        want[:n] = acc
        _same(_host(dout), want, ("sum_ranks", nranks, n))
        if nranks >= 3 and n >= 255:
            rev = np.zeros(n)
            for q in reversed(range(nranks)):
                rev = rev + x[q, :n]
            assert (rev != acc).any()                    # the data tells the rank order apart


def test_min_ranks_with_no_failing_pivot_values(engine):
    torch = _torch()
    for vals in ([IMAX], [IMAX, IMAX], [IMAX, 5], [5, IMAX], [IMAX, IMAX, IMAX], [7, 0, IMAX], [IMAX] * 7 + [3],
                 [9, 4, 4, 100, IMAX, 2, IMAX, 6]):
        din = torch.tensor(vals + [-1, -2], dtype=torch.int32, device="cuda:0")   # past nranks: never read
        dout = torch.tensor([-7, -8], dtype=torch.int32, device="cuda:0")
        _call(engine, "min_ranks", [dout.data_ptr(), din.data_ptr(), len(vals)], 1)
        assert _host(dout).tolist() == [min(vals), -8], vals


# ---- compact per-row vectors (cross-validation on row-sharded storage) ------------------------------------------------

MAXROWS = T * max(max(sm.tile_counts(R, rb)) for R, rb in sm.LAYOUTS)


def _row_counts(R, rb):
    """N per tile count: a partial last tile (padding rows) except for the largest, which ends on a tile boundary"""
    tcs = sm.tile_counts(R, rb)
    return [T * tc - 37 for tc in tcs[:-1]] + [T * tcs[-1]]


@pytest.mark.parametrize("ncols", [1, 255, 256, 257, 1000])
def test_rowdot_own_compact_layout_bitwise_the_single_gpu_reductions(engine, ncols):
    """out[2 li], out[2 li + 1] of own row r = rowdot (<Y_r, alpha>) and rowdot2 (<G_r, Y_r>) of gpb200_row_reductions on
    the same rows, bitwise (Gaussian data: the shared reduction order is what is tested); 0 in padding rows r >= N"""
    torch = _torch()
    rng = np.random.default_rng(ncols)
    ld = ncols + 5
    Y, G = nan_fill((MAXROWS, ld)), nan_fill((MAXROWS, ld))
    Y[:, :ncols] = rng.standard_normal((MAXROWS, ncols))
    G[:, :ncols] = rng.standard_normal((MAXROWS, ncols))
    alpha = np.concatenate([rng.standard_normal(ncols), nan_fill(3)])
    dY, dG, da = _dev(Y), _dev(G), _dev(alpha)
    mu, q2 = (torch.full((MAXROWS,), float("nan"), dtype=torch.float64, device="cuda:0") for _ in range(2))
    engine.row_reductions(2, [dY.data_ptr(), ld, da.data_ptr(), MAXROWS, ncols, mu.data_ptr()])
    engine.row_reductions(4, [dG.data_ptr(), dY.data_ptr(), ld, MAXROWS, ncols, q2.data_ptr()])
    mu, q2 = _host(mu), _host(q2)
    for R, rb in sm.LAYOUTS:
        for N in _row_counts(R, rb):
            n_tiles = -(-N // T)
            for me in range(R):
                valid = sm.own_row_mask(n_tiles * T, me, R, rb) & (np.arange(n_tiles * T) < N)
                dYm, dGm = _masked_rows(dY[:n_tiles * T], valid), _masked_rows(dG[:n_tiles * T], valid)
                nown = sm.own_rows(N, me, R, rb)
                out0 = nan_fill(2 * nown + 3)
                dout = _dev(out0)
                _call(engine, "rowdot_own", [dYm.data_ptr(), dGm.data_ptr(), ld, ncols, da.data_ptr(), N, dout.data_ptr(), R, me, rb],
                      1 if nown else 0)
                rows = sm.compact_rows(n_tiles, me, R, rb)
                want = out0.copy()
                want[0:2 * nown:2] = np.where(rows < N, mu[rows], 0.0)
                want[1:2 * nown:2] = np.where(rows < N, q2[rows], 0.0)
                _same(_host(dout), want, ("rowdot_own", ncols, R, rb, N, me))


@pytest.mark.parametrize("R,rb", sm.LAYOUTS)
def test_diag_own_compact_layout_reads_padding_rows(engine, R, rb):
    torch = _torch()
    rng = np.random.default_rng(20 * R + rb)
    for N in _row_counts(R, rb):
        Npad = -(-N // T) * T
        ld = Npad + 3
        d = rng.standard_normal(Npad)
        for me in range(R):
            rows = sm.compact_rows(Npad // T, me, R, rb)
            dG = torch.full((Npad * ld,), float("nan"), dtype=torch.float64, device="cuda:0")
            if rows.size:
                dG[torch.from_numpy(rows * (ld + 1)).to("cuda:0")] = torch.from_numpy(d[rows]).to("cuda:0")
            nown = rows.size
            out0 = nan_fill(nown + 3)
            dout = _dev(out0)
            _call(engine, "diag_own", [dG.data_ptr(), ld, N, dout.data_ptr(), R, me, rb], 1 if nown else 0)
            want = out0.copy()
            want[:nown] = d[rows]                            # padding rows r >= N included
            _same(_host(dout), want, ("diag_own", R, rb, N, me))


@pytest.mark.parametrize("R,rb", sm.LAYOUTS)
def test_gather_block_own_sums_to_the_exactly_symmetric_block(engine, R, rb):
    """each rank: the entries whose row max(ia, ib) it owns, 0 elsewhere; summed over the ranks, gather_block of the
    mirrored lower triangle, exactly symmetric (compared with ==: a sum turns -0 into +0)"""
    torch = _torch()
    rng = np.random.default_rng(30 * R + rb)
    n_tiles = R * rb + 1
    Ns = n_tiles * T
    ld = Ns + 3
    low = np.tril(np.ones((Ns, Ns), bool))
    L = nan_fill((Ns, ld))
    L[:, :Ns][low] = rng.standard_normal(int(low.sum()))
    Sym = np.zeros((Ns, ld))
    Sym[:, :Ns] = np.where(low, L[:, :Ns], L[:, :Ns].T)
    dL, dSym = _dev(L), _dev(Sym)
    for nv in (1, 2, 255, 256, 257, 700):
        idx = rng.integers(0, Ns, nv)
        if nv == 2:
            idx = np.array([Ns - 1, 0])
        elif nv > 2:
            idx[-1] = idx[0]
            idx[nv // 2] = idx[1]
        assert nv < 3 or len(set(sm.owner(idx // T, R, rb))) >= min(R, 2)
        didx = _dev(idx.astype(np.int64))
        ref = torch.full((nv * nv,), float("nan"), dtype=torch.float64, device="cuda:0")
        engine.vec_kernels("gather_block", [ref.data_ptr(), dSym.data_ptr(), ld, didx.data_ptr(), nv])
        ref = _host(ref).reshape(nv, nv)
        r, c = np.maximum.outer(idx, idx), np.minimum.outer(idx, idx)
        acc = np.zeros((nv, nv))
        for me in range(R):
            dLm = _masked_rows(dL, sm.own_row_mask(Ns, me, R, rb))
            out0 = nan_fill(nv * nv + 3)
            dout = _dev(out0)
            _call(engine, "gather_block_own", [dout.data_ptr(), dLm.data_ptr(), ld, didx.data_ptr(), nv, R, me, rb], 1)
            got = _host(dout)
            want = out0.copy()
            want[:nv * nv] = np.where(sm.owner(r // T, R, rb) == me, L[r, c], 0.0).ravel()
            _same(got, want, ("gather_block_own", R, rb, nv, me))
            acc = acc + got[:nv * nv].reshape(nv, nv)
        assert (acc == ref).all() and (acc == acc.T).all(), (R, rb, nv)


# ---- replicated storage: inverse_dist's slice exchange, cholesky_dist_p2p's flags -------------------------------------

@pytest.mark.parametrize("R", [2, 4, 8])
@pytest.mark.parametrize("tiles", [2, 3, 5, 8, 9, 12, 17])
def test_pack_unpack_slices_round_trip_every_split_level(engine, R, tiles):
    """each rank starts with its own tile columns of every W21 block (as after the filtered GEMM); after pack, the
    all-gather (regions per_rank apart) and unpack, every rank holds all of W21 and the transposes of the other ranks'
    slices, while its own transposed slice (the GEMM's Ct epilogue writes it) and everything else keep their payloads"""
    Np = tiles * T
    ld = Np + 4
    levels = sm.split_levels(Np, R)
    if not levels:
        assert tiles < 2 * R                              # inverse_dist recomputes every level of so small a matrix
        return
    rng = np.random.default_rng(tiles * 10 + R)
    W = np.zeros((Np, ld))
    W[:, :Np] = rng.standard_normal((Np, Np))
    WT = np.zeros((Np, ld))
    WT[:, :Np] = W[:, :Np].T
    for s in levels:
        wr, per = s // R, sm.per_rank(s, Np, R)
        w21 = np.zeros((Np, ld), bool)
        own = [np.zeros((Np, ld), bool) for _ in range(R)]
        up = [np.zeros((Np, ld), bool) for _ in range(R)]
        for z, p, n2 in sm.problems(s, Np):
            w21[p + s:p + s + n2, p:p + s] = True
            for q in range(R):
                gj = p + sm.slice_cols(s, R, q)
                own[q][p + s:p + s + n2, gj] = True
                up[q][gj, p + s:p + s + n2] = True
        G0 = []
        packs = []
        for q in range(R):
            g = nan_fill((Np, ld))
            g[own[q]] = W[own[q]]
            G0.append(g)
            out0 = nan_fill(per + 5)
            dG, dout = _dev(g), _dev(out0)
            _call(engine, "pack_slices", [dG.data_ptr(), ld, dout.data_ptr(), s, Np, R, q], 1)
            _same(_host(dG), g, ("pack_slices G read only", R, Np, s, q))
            want = out0.copy()
            for z, p, n2 in sm.problems(s, Np):
                want[z * s * wr:z * s * wr + n2 * wr] = W[p + s:p + s + n2, p + sm.slice_cols(s, R, q)].ravel()
            got = _host(dout)
            _same(got, want, ("pack_slices", R, Np, s, q))
            packs.append(got[:per])
        din = _dev(np.concatenate(packs + [nan_fill(5)]))
        for q in range(R):
            dG = _dev(G0[q])
            _call(engine, "unpack_slices", [dG.data_ptr(), ld, din.data_ptr(), per, s, Np, R, q], 1)
            want = G0[q].copy()
            want[w21] = W[w21]
            for q2 in range(R):
                if q2 != q:
                    want[up[q2]] = WT[up[q2]]
            _same(_host(dG), want, ("unpack_slices", R, Np, s, q))


def test_signal_peers_and_wait_signal_on_local_flag_words(engine):
    torch = _torch()
    init = -100 - torch.arange(16, dtype=torch.int32, device="cuda:0")
    words = init.clone()
    slots = [3, 0, 9, 5, 12, 1, 7]                      # one flag word per peer, scattered
    ptrs = torch.tensor([words.data_ptr() + 4 * k for k in slots], dtype=torch.int64, device="cuda:0")
    for n_peer in (0, 1, 7):
        words.copy_(init)
        value = 65536 * 3 + n_peer
        _call(engine, "signal_peers", [ptrs.data_ptr(), n_peer, value], 1)
        want = _host(init).copy()
        want[slots[:n_peer]] = value
        assert _host(words).tolist() == want.tolist(), n_peer
    err = torch.zeros(2, dtype=torch.int32, device="cuda:0")
    words.copy_(init)
    words[4] = 65536 * 5 + 2
    for target in (65536 * 5 + 2, 65536 * 5 + 1, -5):    # already at or above the target: returns at once
        _call(engine, "wait_signal", [words.data_ptr() + 16, target, err.data_ptr()], 1)
        assert _host(err).tolist() == [0, 0], target
    assert _host(words)[4] == 65536 * 5 + 2


# ---- misuse -----------------------------------------------------------------------------------------------------------

def test_rejections_launch_nothing(engine):
    buf = _dev(np.zeros(1024))
    p = buf.data_ptr()
    big = 128 * 65536
    BASE = {
        "copy_lower": [p, 128, p, 128, 128],
        "scatter_rows": [p, p, 256, 1024, 0, 128, 0, p, 128, 2, 0, 1],
        "unpack_panel": [p, 128, 1024, 128, 0, p, 4 * T * 128, 2, 0, 1],
        "transpose": [p, 64, p, 64, 64, 64],
        "pack_wblock": [p, 256, p, 512, p, 128, 256],
        "sum_ranks": [p, p, 100, 2, 100],
        "min_ranks": [p, p, 2],
        "transpose_own": [p, 64, p, 64, 64, 64, 2, 1, 1],
        "rowdot_own": [p, p, 64, 64, p, 64, p, 2, 0, 1],
        "diag_own": [p, 256, 200, p, 2, 0, 1],
        "gather_block_own": [p, p, 64, p, 64, 2, 0, 1],
        "pack_slices": [p, 1024, p, 256, 1024, 2, 0],
        "unpack_slices": [p, 1024, p, sm.per_rank(256, 1024, 2), 256, 1024, 2, 0],
        "signal_peers": [p, 7, 1],
        "wait_signal": [p, 0, p],
    }
    # (kernel, {position: value}): each a single rejection named in include/gpb200.h
    BAD = [
        ("copy_lower", {0: 0}), ("copy_lower", {2: 0}), ("copy_lower", {4: -1}), ("copy_lower", {1: 127}), ("copy_lower", {3: 127}),
        ("copy_lower", {1: 65536, 3: 65536, 4: 65536}),
        ("scatter_rows", {0: 0}), ("scatter_rows", {1: 0}), ("scatter_rows", {7: 0}), ("scatter_rows", {3: 1000}),
        ("scatter_rows", {3: -128}), ("scatter_rows", {5: 129}), ("scatter_rows", {5: -1}), ("scatter_rows", {4: -1}),
        ("scatter_rows", {6: -1}), ("scatter_rows", {6: 9}), ("scatter_rows", {2: 127}), ("scatter_rows", {9: 0}),
        ("scatter_rows", {10: 2}), ("scatter_rows", {10: -1}), ("scatter_rows", {11: 0}), ("scatter_rows", {3: big}),
        ("unpack_panel", {0: 0}), ("unpack_panel", {5: 0}), ("unpack_panel", {3: 129}), ("unpack_panel", {2: 1000}),
        ("unpack_panel", {6: 4 * T * 128 - 1}), ("unpack_panel", {7: 0}), ("unpack_panel", {8: 2}), ("unpack_panel", {9: 0}),
        ("unpack_panel", {4: 9}), ("unpack_panel", {2: big, 6: big * 128, 7: 1}),
        ("transpose", {0: 0}), ("transpose", {4: -1}), ("transpose", {5: -1}), ("transpose", {1: 63}), ("transpose", {3: 63}),
        ("transpose", {1: 65535 * 32 + 1, 4: 65535 * 32 + 1}),
        ("pack_wblock", {4: 0}), ("pack_wblock", {5: 64}), ("pack_wblock", {6: 200}), ("pack_wblock", {6: 384}),
        ("pack_wblock", {3: 383}), ("pack_wblock", {1: 65536, 3: 2 * 65536, 6: 65536}),
        ("sum_ranks", {0: 0}), ("sum_ranks", {3: 0}), ("sum_ranks", {4: -1}), ("sum_ranks", {2: 99}),
        ("min_ranks", {1: 0}), ("min_ranks", {2: 0}),
        ("transpose_own", {6: 0}), ("transpose_own", {7: 2}), ("transpose_own", {7: -1}), ("transpose_own", {8: 0}),
        ("transpose_own", {1: 65535 * 32 + 1, 4: 65535 * 32 + 1}),
        ("rowdot_own", {2: 63}), ("rowdot_own", {3: -1}), ("rowdot_own", {5: -1}), ("rowdot_own", {4: 0}), ("rowdot_own", {7: 0}),
        ("rowdot_own", {8: 5}),
        ("diag_own", {1: 255}), ("diag_own", {2: -1}), ("diag_own", {3: 0}), ("diag_own", {6: 0}),
        ("gather_block_own", {4: 65536}), ("gather_block_own", {4: -1}), ("gather_block_own", {3: 0}), ("gather_block_own", {6: 2}),
        ("pack_slices", {3: 384}), ("pack_slices", {3: 128}), ("pack_slices", {3: 1024}), ("pack_slices", {4: 1000}),
        ("pack_slices", {1: 1000}), ("pack_slices", {5: 0}), ("pack_slices", {6: 2}), ("pack_slices", {2: 0}),
        ("pack_slices", {3: 2 ** 21, 4: 2 ** 22, 1: 2 ** 22}), ("pack_slices", {4: 256 * 2 * 65536, 1: 256 * 2 * 65536}),
        ("unpack_slices", {3: sm.per_rank(256, 1024, 2) - 1}), ("unpack_slices", {4: 128}), ("unpack_slices", {7: -1}),
        ("unpack_slices", {5: 256 * 65536, 1: 256 * 65536, 3: sm.per_rank(256, 256 * 65536, 2)}),
        ("signal_peers", {0: 0}), ("signal_peers", {1: 8}), ("signal_peers", {1: -1}),
        ("wait_signal", {0: 0}), ("wait_signal", {2: 0}),
    ]
    n0 = engine.launch_count()
    for name, change in BAD:
        args = list(BASE[name])
        for k, v in change.items():
            args[k] = v
        with pytest.raises(ValueError):
            engine.shard_kernels(name, args)
            pytest.fail("accepted: %s %r" % (name, change))
    for name, args in BASE.items():                      # a wrong argument count
        with pytest.raises(ValueError):
            engine.shard_kernels(name, args + [0])
    assert engine.launch_count() == n0
