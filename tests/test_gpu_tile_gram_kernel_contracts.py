"""GPU: the dense Gram-family kernels (csrc/gram.cu) tested directly against the model tests/gram_model.py, through
gpb200_gram_kernels (one call of the production launch wrapper each).

* Pointwise edge table: values from the diagonal of crossgram on paired points, theta-partials from the diagonal of
  crossgram_grad for every j, x-partials from crossgram_dx with c = 0, a = 0 and a one-hot W row per point (so that
  dvar[m] = -2 dk(xs_m, z_m)/dxs_m exactly), each within the model's componentwise bound of the long-double result.
* Layouts bit for bit on exact dyadic operands (LinIso + Const at theta = 0): elements a kernel must not read hold NaN,
  elements it must not write hold a NaN with its own payload that must come back unchanged.
* Cross-kernel agreement, fixed-order reductions, every input dimension up to GPB200_MAX_DIMS, empty sizes and misuse.

The name puts the file after every file that opens a torch.profiler session (test_gpu_gpa.py, the launch-count files,
test_gpu_shard_cv.py): torch.profiler records no device activity in a session started about a minute or more after the
process's first one (see test_gpu_tile_kernel_contracts.py), so this file's run time must not fall between them.  It
opens no session itself, and uses engines of its own because it calls set_kernel."""
import zlib

import numpy as np
import pytest

import gram_model as gm
from conftest import kernel_zoo
from oracle import gp_oracle as orc

pytestmark = pytest.mark.gpu

T = gm.T
POISON = np.array([0x7FF8_DEAD_0000_0005], dtype=np.uint64).view(np.float64)[0]   # "never read, never written"
NAN = np.nan                                                                         # "never read"


def _raw(a):
    return np.ascontiguousarray(a).view(np.uint64)


def _same(got, want):
    """bitwise, with POISON payloads compared raw and every other value up to the sign of zero"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape
    g, w = np.where(got == 0, 0.0, got), np.where(want == 0, 0.0, want)
    bad = _raw(g) != _raw(w)
    assert not bad.any(), (int(bad.sum()), np.argwhere(bad)[:3].tolist(), got[bad][:3], want[bad][:3])


def _torch():
    import torch
    return torch


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to("cuda:0")


def _host(t):
    _torch().cuda.synchronize()
    return t.cpu().numpy()


def _need_longdouble():
    if np.finfo(np.longdouble).nmant < 63:
        pytest.skip("needs an 80-bit or wider np.longdouble")


@pytest.fixture(scope="module")
def eng():
    import gpb200
    e = gpb200.Engine(0)
    yield e
    e.close()


def _program(e, kernel, d):
    import gpb200 as g
    ops, dims, theta, _ = g.flatten(kernel, d)
    e.set_kernel(ops, dims, theta.size)
    return gm.Prog(kernel, d), theta


def _run(e, name, args, fargs=(), launches=1):
    n0 = e.launch_count()
    e.gram_kernels(name, [int(a) for a in args], fargs)
    assert e.launch_count() - n0 == launches, (name, e.launch_count() - n0)


def _pad(n):
    return -(-n // T) * T


def _dyadic(rng, shape):
    return rng.integers(-64, 65, size=shape) / 16.0


def _exact(e, d=3):
    import gpb200 as g
    return _program(e, g.LinIso(0.0) + g.Const(0.0), d)


RATIOS = {}


def _ratio(key, err, bound):
    r = float(np.max(np.where(err == 0, 0.0, err / np.maximum(bound, 1e-320)))) if np.size(err) else 0.0
    RATIOS[key] = max(RATIOS.get(key, 0.0), r)
    return r


# ---- pointwise edge table ---------------------------------------------------------------------------------------------

EDGE = gm.edge_table()
REGIMES = sorted(set(e[0] for e in EDGE), key=[e[0] for e in EDGE].index)


def _pointwise(e, P, theta, A, B, d):
    """(k, g (n_theta, n), dx (n, d)) of the device on the pairs (A[m], B[m])."""
    n = A.shape[0]
    npad = _pad(n)
    ldx = d + 1
    xa = np.full((npad, ldx), NAN)
    xa[:n, :d] = A
    xb = np.full((npad, ldx), NAN)
    xb[:n, :d] = B
    da, db = _dev(xa), _dev(xb)
    K = _dev(np.full((npad, npad), POISON))
    _run(e, "crossgram", [da.data_ptr(), ldx, n, npad, db.data_ptr(), ldx, n, npad, d, K.data_ptr(), npad], theta)
    k = np.diag(_host(K))[:n].copy()
    g = np.zeros((P.n_theta, n))
    for j in range(P.n_theta):
        _run(e, "crossgram_grad", [da.data_ptr(), ldx, n, npad, db.data_ptr(), ldx, n, npad, d, j, K.data_ptr(), npad], theta)
        g[j] = np.diag(_host(K))[:n]
    Wd = _dev(np.eye(n, npad))                        # one-hot rows: W[m, m] = 1
    zero = _dev(np.zeros(npad))
    dmu, dvar = _dev(np.full((n, d), POISON)), _dev(np.full((n, d), POISON))
    _run(e, "crossgram_dx", [da.data_ptr(), ldx, n, db.data_ptr(), ldx, n, d, zero.data_ptr(), Wd.data_ptr(), 0, npad,
                             dmu.data_ptr(), dvar.data_ptr()], list(theta) + [0.0])
    assert np.all(_host(dmu) == 0)
    return k, g, -0.5 * _host(dvar)


@pytest.mark.parametrize("regime", REGIMES)
def test_pointwise_edge_regimes_within_bounds_of_long_double(eng, regime):
    _need_longdouble()
    for reg, name, kernel, d, A, B in EDGE:
        if reg != regime:
            continue
        P, theta = _program(eng, kernel, d)
        k, g, dx = _pointwise(eng, P, theta, A, B, d)
        with np.errstate(all="ignore"):
            kl, bk, _, _ = gm.evaluate(P, A, B, gm.LD, False)
            _, _, gl, bg = gm.evaluate(P, A, B, gm.LD, True)
            dl, bdx = gm.evaluate_dx(P, A, B, gm.LD)
        ek, eg, ed = (np.abs((k - kl).astype(float)), np.abs((g - gl).astype(float)), np.abs((dx - dl).astype(float)))
        rk, rg, rd = _ratio(("value", reg), ek, bk), _ratio(("theta", reg), eg, bg), _ratio(("x", reg), ed, bdx)
        print("RATIO %-40s %-22s value %.3f theta %.3f x %.3f" % (reg, name, rk, rg, rd))
        assert np.all(ek <= bk) and np.all(eg <= bg) and np.all(ed <= bdx), (reg, name, rk, rg, rd)


# ---- layouts, bitwise on exact operands -------------------------------------------------------------------------------

NS = [1, 127, 128, 129, 257, 1000]


@pytest.mark.parametrize("N", NS)
def test_gram_lower_ownership_filters_bitwise(eng, N):
    rng = np.random.default_rng(N)
    P, theta = _exact(eng)
    d, ldx = 3, 5
    Npad = _pad(N)
    ld = Npad + 6
    x = np.full((Npad, ldx), NAN)
    x[:N, :d] = _dyadic(rng, (N, d))
    nv = np.full(Npad, NAN)
    nv[:N] = rng.integers(1, 8, N) / 4.0
    dx_, dn = _dev(x), _dev(nv)
    kf = lambda a, b: gm.kmat(P, a, b)
    Tn = Npad // T
    combos = [(0, 1, 0, 0, 0), (0, 1, 0, 0, Tn - 1), (1, 2, 1, 0, 0), (1, 3, 2, 1, 0), (2, 2, 0, 1, 1 if Tn > 1 else 0)]
    for own_tiles, nranks, rank, axis, bm_min in combos:
        for n_noise in (1, N):
            G0 = np.full(Npad * ld, POISON)
            dG = _dev(G0)
            _run(eng, "gram_lower", [dx_.data_ptr(), ldx, d, N, Npad, dn.data_ptr(), n_noise, dG.data_ptr(), ld, own_tiles,
                                     nranks, rank, axis, bm_min], list(theta) + [0.125])
            want = gm.gram_lower(kf, x.ravel(), ldx, d, N, Npad, nv if n_noise > 1 else nv[:1], n_noise, 0.125, G0, ld,
                                 own_tiles, nranks, rank, axis, bm_min)
            _same(_host(dG), want)


@pytest.mark.parametrize("N", NS)
def test_crossgram_gram_full_kdiag_bitwise(eng, N):
    rng = np.random.default_rng(N + 1)
    P, theta = _exact(eng)
    d, ldx = 3, 4
    M = max(N // 3, 1)
    Npad, Mpad = _pad(N), _pad(M)
    xs = np.full((Mpad, ldx), NAN)
    xs[:M, :d] = _dyadic(rng, (M, d))
    x = np.full((Npad, ldx), NAN)
    x[:N, :d] = _dyadic(rng, (N, d))
    dxs, dx_ = _dev(xs), _dev(x)
    kf = lambda a, b: gm.kmat(P, a, b)
    ld = Npad + 2
    K0 = np.full(Mpad * ld, POISON)
    dK = _dev(K0)
    _run(eng, "crossgram", [dxs.data_ptr(), ldx, M, Mpad, dx_.data_ptr(), ldx, N, Npad, d, dK.data_ptr(), ld], theta)
    _same(_host(dK), gm.crossgram(kf, xs.ravel(), ldx, M, Mpad, x.ravel(), ldx, N, Npad, d, K0, ld))
    ld = Npad + 4
    S0 = np.full(Npad * ld, POISON)
    dS = _dev(S0)
    _run(eng, "gram_full", [dx_.data_ptr(), ldx, N, Npad, d, dS.data_ptr(), ld], theta)
    _same(_host(dS), gm.gram_full(kf, x.ravel(), ldx, N, Npad, d, S0, ld))
    out = _dev(np.full(N + 3, POISON))
    _run(eng, "kdiag", [dx_.data_ptr(), ldx, d, N, out.data_ptr()], theta)
    want = np.full(N + 3, POISON)
    want[:N] = gm.kdiag(lambda a, b: gm.evaluate(P, a, b)[0], x.ravel(), ldx, d, N)
    _same(_host(out), want)


@pytest.mark.parametrize("N", [129, 1000])
def test_gradient_grams_row_batches_and_rectangles_bitwise(eng, N):
    rng = np.random.default_rng(N + 2)
    P, theta = _exact(eng)
    d, ldx = 3, 5
    Npad = _pad(N)
    x = np.full((Npad, ldx), NAN)
    x[:N, :d] = _dyadic(rng, (N, d))
    dx_ = _dev(x)
    ld = Npad + 2
    Tn = Npad // T
    for j in range(P.n_theta):
        gf = lambda a, b, j=j: gm.gmat(P, a, b)[j]
        for row0, rows in ((0, T), (T * (Tn // 2), T), ((Tn - 1) * T, T), (0, Npad)):
            D0 = np.full(rows * ld, POISON)
            dD = _dev(D0)
            _run(eng, "gram_grad_full", [dx_.data_ptr(), ldx, d, N, Npad, j, dD.data_ptr(), ld, row0, rows], theta)
            _same(_host(dD), gm.gram_grad_full(gf, x.ravel(), ldx, d, N, Npad, D0, ld, row0, rows))
        N2 = N // 2 + 3
        N2pad = _pad(N2)
        x2 = np.full((N2pad, 4), NAN)
        x2[:N2, :d] = _dyadic(rng, (N2, d))
        dx2 = _dev(x2)
        ld2 = N2pad + 2
        D0 = np.full(Npad * ld2, POISON)
        dD = _dev(D0)
        _run(eng, "crossgram_grad", [dx_.data_ptr(), ldx, N, Npad, dx2.data_ptr(), 4, N2, N2pad, d, j, dD.data_ptr(), ld2],
             theta)
        _same(_host(dD), gm.crossgram_grad(gf, x.ravel(), ldx, N, Npad, x2.ravel(), 4, N2, N2pad, d, D0, ld2))


@pytest.mark.parametrize("N", [1, 129, 1000])
def test_traces_and_kdiag_grad_bitwise_and_repeatable(eng, N):
    rng = np.random.default_rng(N + 3)
    P, theta = _exact(eng)
    d, ldx = 3, 5
    Npad = _pad(N)
    ld = Npad + 2
    x = np.full((Npad, ldx), NAN)
    x[:N, :d] = _dyadic(rng, (N, d))
    alpha = np.full(Npad, NAN)
    alpha[:N] = _dyadic(rng, N)
    Kinv = np.full((Npad, ld), NAN)
    Kinv[:N, :N] = np.tril(_dyadic(rng, (N, N)))
    # (i, i + 1) of an even row i is read as the pair of (i, i) and discarded: NaN is harmless there
    dx_, da, dK = _dev(x), _dev(alpha), _dev(Kinv)
    gall = lambda a, b: gm.gmat(P, a, b)
    nacc = P.n_theta + 1
    tiles = (Npad // T) * (Npad // T + 1) // 2
    for bm_mod, bm_rem, bm_div in ((1, 0, 1), (2, 1, 1), (3, 0, 2)):
        part, out = _dev(np.full(tiles * nacc, POISON)), _dev(np.full(nacc, POISON))
        args = [dx_.data_ptr(), ldx, d, N, Npad, da.data_ptr(), dK.data_ptr(), ld, part.data_ptr(), out.data_ptr(), bm_mod,
                bm_rem, bm_div]
        _run(eng, "trace", args, theta, launches=2)
        wp, wo = gm.trace_out(gm.trace(gall, x.ravel(), ldx, d, N, Npad, alpha, Kinv.ravel(), ld, bm_mod, bm_rem, bm_div),
                              P.n_theta)
        o1 = _host(out).copy()
        _same(_host(part), wp)
        _same(o1, wo)
        _run(eng, "trace", args, theta, launches=2)
        _same(_host(out), o1)
    N2 = max(N // 2, 1) | 1                                   # odd: a partial tile and a discarded pair column
    ldw = N2 + 3
    W = np.full((N, ldw), NAN)
    W[:, :N2] = _dyadic(rng, (N, N2))
    dW = _dev(W)
    tr = -(-N // T) * -(-N2 // T)
    part, out = _dev(np.full(tr * P.n_theta, POISON)), _dev(np.full(P.n_theta, POISON))
    args = [dx_.data_ptr(), ldx, N, dx_.data_ptr(), ldx, N2, d, dW.data_ptr(), ldw, part.data_ptr(), out.data_ptr()]
    _run(eng, "trace_rect", args, theta, launches=2)
    wp, wo = gm.trace_rect(gall, x.ravel(), ldx, N, x.ravel(), ldx, N2, d, W.ravel(), ldw, P.n_theta)
    _same(_host(part), wp)
    _same(_host(out), wo)
    gv = _dyadic(rng, N)
    dg, out = _dev(gv), _dev(np.full(P.n_theta * N + 2, POISON))
    _run(eng, "kdiag_grad", [dx_.data_ptr(), ldx, d, N, dg.data_ptr(), out.data_ptr()], theta)
    want = np.full(P.n_theta * N + 2, POISON)
    want[:P.n_theta * N] = gm.kdiag_grad(lambda a, b: np.stack([np.diag(m) for m in gm.gmat(P, a, b)]), x.ravel(), ldx, d,
                                         N, gv, P.n_theta)
    _same(_host(out), want)


@pytest.mark.parametrize("Npad", [128, 256, 384, 4096])
def test_mirror_lower_tiles_bitwise(eng, Npad):
    rng = np.random.default_rng(Npad)
    ld = Npad + 2
    F = rng.standard_normal(Npad * ld)
    dF = _dev(F)
    _run(eng, "mirror_lower_tiles", [dF.data_ptr(), ld, Npad], launches=0 if Npad == T else 1)
    _same(_host(dF), gm.mirror_lower_tiles(F, ld, Npad))


# ---- cross-kernel agreement and zoo reductions ------------------------------------------------------------------------

ZOO = [(n, k, 3) for n, k in kernel_zoo(3)]


@pytest.mark.parametrize("name,kernel,d", ZOO, ids=[z[0] for z in ZOO])
def test_zoo_kernels_agree_and_traces_within_bounds(eng, name, kernel, d):
    _need_longdouble()
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    N = 300
    Npad = _pad(N)
    X = rng.standard_normal((N, d))
    X[7] = X[3]
    x = np.full((Npad, d), NAN)
    x[:N] = X
    P, theta = _program(eng, kernel, d)
    dx_, dn = _dev(x), _dev(np.zeros(1))
    G, S, C = (_dev(np.full((Npad, Npad), POISON)) for _ in range(3))
    _run(eng, "gram_lower", [dx_.data_ptr(), d, d, N, Npad, dn.data_ptr(), 1, G.data_ptr(), Npad, 0, 1, 0, 0, 0],
         list(theta) + [0.0])
    _run(eng, "gram_full", [dx_.data_ptr(), d, N, Npad, d, S.data_ptr(), Npad], theta)
    _run(eng, "crossgram", [dx_.data_ptr(), d, N, Npad, dx_.data_ptr(), d, N, Npad, d, C.data_ptr(), Npad], theta)
    Gh, Sh, Ch = _host(G)[:N, :N], _host(S)[:N, :N], _host(C)[:N, :N]
    low = np.tril_indices(N, -1)
    _same(Sh[low], Gh[low])
    _same(Ch, Sh)
    Kl = gm.kmat(P, X, X, gm.LD)
    kb = gm.evaluate(P, np.repeat(X, N, 0), np.tile(X, (N, 1)), gm.LD)[1].reshape(N, N)
    _ratio(("gram", "zoo"), np.abs((Gh[low] - Kl[low]).astype(float)), kb[low])
    assert np.all(np.abs((Gh[low] - Kl[low]).astype(float)) <= kb[low]), name
    # trace: repeated calls bitwise; within gamma_m sum |w||g| + sum |w| bound_g of the long-double model
    alpha = rng.standard_normal(N)
    Kinv = rng.standard_normal((N, N))
    Kinv = Kinv + Kinv.T
    kv = np.full((Npad, Npad), NAN)
    kv[:N, :N] = Kinv
    a_ = np.full(Npad, NAN)
    a_[:N] = alpha
    fast = P.fast()
    nacc = 3 if fast else P.n_theta + 1
    tiles = (Npad // T) * (Npad // T + 1) // 2
    da, dK = _dev(a_), _dev(kv)
    part, out = _dev(np.zeros(tiles * nacc)), _dev(np.zeros(nacc))
    args = [dx_.data_ptr(), d, d, N, Npad, da.data_ptr(), dK.data_ptr(), Npad, part.data_ptr(), out.data_ptr(), 1, 0, 1]
    _run(eng, "trace", args, theta, launches=2)
    o1 = _host(out).copy()
    _run(eng, "trace", args, theta, launches=2)
    _same(_host(out), o1)
    A = np.outer(alpha, alpha) - Kinv
    Wt = np.tril(A, -1) + 0.5 * np.diag(np.diag(A))
    _, _, gl, bgl = gm.evaluate(P, np.repeat(X, N, 0), np.tile(X, (N, 1)), gm.LD, True)
    gl, bgl = gl.reshape(P.n_theta, N, N), bgl.reshape(P.n_theta, N, N)
    m = N * (N + 1) // 2
    for p in range(P.n_theta):
        want = np.sum(Wt.astype(gm.LD) * gl[p])
        bound = gm.gamma(m + 4) * np.sum(np.abs(Wt) * np.abs(gl[p].astype(float))) + np.sum(np.abs(Wt) * bgl[p]) + 1e-300
        err = abs(float(o1[p] - want))
        _ratio(("trace", "zoo"), np.array(err), np.array(bound))
        assert err <= bound, (name, p, err, bound)
    # trace_rect over a partial rectangle, repeated bitwise, within the same bound
    N2 = 131
    W = rng.standard_normal((N, N2 + 1))
    dW = _dev(W)
    nr = 2 if fast else P.n_theta
    part, out = _dev(np.zeros(3 * 2 * nr)), _dev(np.zeros(nr))
    args = [dx_.data_ptr(), d, N, dx_.data_ptr(), d, N2, d, dW.data_ptr(), N2 + 1, part.data_ptr(), out.data_ptr()]
    _run(eng, "trace_rect", args, theta, launches=2)
    o1 = _host(out).copy()
    _run(eng, "trace_rect", args, theta, launches=2)
    _same(_host(out), o1)
    _, _, gr, bgr = gm.evaluate(P, np.repeat(X, N2, 0), np.tile(X[:N2], (N, 1)), gm.LD, True)
    gr, bgr = gr.reshape(P.n_theta, N, N2), bgr.reshape(P.n_theta, N, N2)
    for p in range(nr):
        want = np.sum(W[:, :N2].astype(gm.LD) * gr[p])
        bound = gm.gamma(N * N2 + 4) * np.sum(np.abs(W[:, :N2]) * np.abs(gr[p].astype(float))) + \
            np.sum(np.abs(W[:, :N2]) * bgr[p]) + 1e-300
        err = abs(float(o1[p] - want))
        _ratio(("trace_rect", "zoo"), np.array(err), np.array(bound))
        assert err <= bound, (name, p, err, bound)


def test_gram_lower_matches_fsa_gram_off_the_diagonal(eng):
    import sparse_model as sm
    rng = np.random.default_rng(11)
    for name, kernel in kernel_zoo(3):
        if name == "SEIso":                           # the dense kernels' specialised formula: compared by bound above
            continue
        N, d = 200, 3
        X = rng.standard_normal((N, d))
        P, theta = _program(eng, kernel, d)
        lay = sm.Layout([N])
        xb = np.zeros((lay.Np, d))
        xb[:N] = X
        dst = _dev(np.full(lay.packed, POISON))
        dxb, dm = _dev(xb), _dev(lay.mask)
        items = lay.gram_items()
        flat = [v for off, ld, ri, rj, dg in items for v in (dst.data_ptr() + 8 * off, ld, ri, rj, dg)]
        eng.fsa_kernels("gram", [dxb.data_ptr(), d, dm.data_ptr()] + flat, list(theta) + [0.0])
        F = np.tril(lay.block(_host(dst), 0))[:N, :N]
        Npad = _pad(N)
        G = _dev(np.full((Npad, Npad), POISON))
        _run(eng, "gram_lower", [dxb.data_ptr(), d, d, N, Npad, dm.data_ptr(), 1, G.data_ptr(), Npad, 0, 1, 0, 0, 0],
             list(theta) + [0.0])
        low = np.tril_indices(N, -1)
        _same(_host(G)[:N, :N][low], F[low])


# ---- every input dimension --------------------------------------------------------------------------------------------

DIMS = [1, 2, 9, 31, 109, 110, 113, 114, 128]


def _masked_ard(g, leaf, d, w, *args):
    """an ARD leaf over the last min(d, w) input dimensions: a program holds at most GPB200_MAX_THETA = 96 parameters and
    GPB200_MAX_DIMS = 128 leaf dimensions in all"""
    dw = min(d, w)
    k = leaf(list(np.linspace(-0.3, 0.3, dw) + 0.5 * np.log(dw)), *args)
    return k if dw == d else g.Masked(k, list(range(d - dw, d)))


def _masked_iso(g, k, d, w):
    return k if d <= w else g.Masked(k, list(range(d - w, d)))


def _dim_kernels(d):
    import gpb200 as g
    out = [("SEIso", g.SEIso(0.5 * np.log(d) + 0.3, 0.1)), ("SEArd", _masked_ard(g, g.SEArd, d, 95, 0.1))]
    if d >= 2:
        out.append(("MaunaLoa-like", _masked_ard(g, g.SEArd, d, 25, 0.0) + g.Masked(g.Periodic(0.0, 0.0, 0.3), [0]) *
                    _masked_ard(g, g.SEArd, d, 25, 0.0) + _masked_iso(g, g.RQIso(0.5 * np.log(min(d, 25)), 0.0, -1.0), d, 25) +
                    _masked_ard(g, g.SEArd, d, 25, -1.0)))
    return out


@pytest.mark.parametrize("d", DIMS)
def test_every_kernel_at_input_dimension(eng, d):
    _need_longdouble()
    rng = np.random.default_rng(d)
    N = 200
    Npad = _pad(N)
    X = rng.standard_normal((N, d))
    x = np.full((Npad, d + 1), NAN)
    x[:N, :d] = X
    dx_, dn = _dev(x), _dev(np.full(1, 0.5))
    ldx = d + 1
    for name, kernel in _dim_kernels(d):
        P, theta = _program(eng, kernel, d)
        Kl = gm.kmat(P, X, X, gm.LD)
        kb = gm.evaluate(P, np.repeat(X, N, 0), np.tile(X, (N, 1)), gm.LD)[1].reshape(N, N)
        G, S, C = (_dev(np.full((Npad, Npad), POISON)) for _ in range(3))
        _run(eng, "gram_lower", [dx_.data_ptr(), ldx, d, N, Npad, dn.data_ptr(), 1, G.data_ptr(), Npad, 0, 1, 0, 0, 0],
             list(theta) + [0.0])
        _run(eng, "gram_full", [dx_.data_ptr(), ldx, N, Npad, d, S.data_ptr(), Npad], theta)
        _run(eng, "crossgram", [dx_.data_ptr(), ldx, N, Npad, dx_.data_ptr(), ldx, N, Npad, d, C.data_ptr(), Npad], theta)
        Gh, Sh, Ch = _host(G), _host(S), _host(C)
        low = np.tril_indices(N, -1)
        _same(Sh[:N, :N][low], Gh[:N, :N][low])
        _same(Ch, Sh)
        err = np.abs((Sh[:N, :N] - Kl).astype(float))
        assert np.all(err <= kb), (d, name, _ratio(("dim", d), err, kb))
        _ratio(("dim", d), err, kb)
        assert np.all(np.diag(Gh)[:N] == np.diag(Sh)[:N] + 0.5)
        assert np.all(Gh[N:, N:] == np.eye(Npad - N)) and np.all(Sh[N:] == 0) and np.all(Sh[:, N:] == 0)
        j = P.n_theta - 1
        D = _dev(np.full((Npad, Npad), POISON))
        _run(eng, "gram_grad_full", [dx_.data_ptr(), ldx, d, N, Npad, j, D.data_ptr(), Npad, 0, Npad], theta)
        _, _, gl, bgl = gm.evaluate(P, np.repeat(X, N, 0), np.tile(X, (N, 1)), gm.LD, True)
        gl, bgl = gl[j].reshape(N, N), bgl[j].reshape(N, N)
        assert np.all(np.abs((_host(D)[:N, :N] - gl).astype(float)) <= bgl), (d, name)
        fast = P.fast()
        nacc = 3 if fast else P.n_theta + 1
        tiles = (Npad // T) * (Npad // T + 1) // 2
        alpha = np.zeros(Npad)
        alpha[:N] = rng.standard_normal(N)
        Ki = np.zeros((Npad, Npad))
        da, dK = _dev(alpha), _dev(Ki)
        part, out = _dev(np.zeros(tiles * nacc)), _dev(np.zeros(nacc))
        _run(eng, "trace", [dx_.data_ptr(), ldx, d, N, Npad, da.data_ptr(), dK.data_ptr(), Npad, part.data_ptr(),
                            out.data_ptr(), 1, 0, 1], theta, launches=2)
        Wt = np.tril(np.outer(alpha[:N], alpha[:N]), -1) + 0.5 * np.diag(alpha[:N] ** 2)
        want = np.sum(Wt.astype(gm.LD) * gl)
        bound = gm.gamma(N * N) * np.sum(np.abs(Wt) * np.abs(gl.astype(float))) + np.sum(np.abs(Wt) * bgl) + 1e-300
        got = _host(out)[1 if fast else j]
        assert abs(float(got - want)) <= bound, (d, name, got, want)


def test_dense_gpe_at_128_input_dimensions_matches_the_oracle():
    import gpb200
    rng = np.random.default_rng(128)
    N, d = 1000, 128
    X = rng.standard_normal((N, d))
    y = np.sin(X[:, :4].sum(axis=1)) + 0.1 * rng.standard_normal(N)
    Xs = rng.standard_normal((20, d))
    kernel = _masked_ard(gpb200, gpb200.SEArd, d, 95, 0.0)         # dimensions 33 .. 127
    gp = gpb200.GPE(X.T, y, gpb200.MeanZero(), kernel, -1.0)
    gp.update_target_and_dtarget()
    mu, s2 = gp.predict_f(Xs.T)
    spec = kernel.spec()
    o = orc.mll_and_dmll(spec, X, y, -1.0)
    mo, vo = orc.predict_f(spec, X, o, Xs)
    assert abs(gp.mll - o["mll"]) <= 1e-10 * abs(o["mll"]), (gp.mll, o["mll"])
    assert np.allclose(gp.dmll, o["dmll"], rtol=1e-8, atol=1e-10)
    assert np.max(np.abs(mu - mo)) <= 1e-10 * np.max(np.abs(mo))
    assert np.max(np.abs(s2 - vo)) <= 1e-10 * np.max(np.abs(vo)) + 1e-13


# ---- empty sizes, misuse, and the SEIso fast flag ---------------------------------------------------------------------

def test_empty_sizes_launch_nothing(eng):
    P, theta = _exact(eng)
    buf = _dev(np.full(4 * T * T, POISON))
    z = _dev(np.full(16, POISON))
    b, o = buf.data_ptr(), z.data_ptr()
    f = list(theta)
    calls = [("gram_lower", [b, 3, 3, 0, 0, b, 1, b, 128, 0, 1, 0, 0, 0], f + [0.0]),
             ("crossgram", [b, 3, 0, 0, b, 3, 5, 128, 3, b, 128], f), ("crossgram", [b, 3, 5, 128, b, 3, 0, 0, 3, b, 128], f),
             ("gram_full", [b, 3, 0, 0, 3, b, 128], f), ("kdiag", [b, 3, 3, 0, b], f),
             ("gram_grad_full", [b, 3, 3, 0, 0, 0, b, 128, 0, 0], f),
             ("gram_grad_full", [b, 3, 3, 5, 128, 0, b, 128, 128, 0], f),
             ("crossgram_grad", [b, 3, 0, 0, b, 3, 5, 128, 3, 0, b, 128], f),
             ("trace", [b, 3, 3, 0, 0, b, b, 128, b, o, 1, 0, 1], f), ("trace_rect", [b, 3, 0, b, 3, 5, 3, b, 128, b, o], f),
             ("trace_rect", [b, 3, 5, b, 3, 0, 3, b, 128, b, o], f), ("kdiag_grad", [b, 3, 3, 0, b, b], f),
             ("crossgram_dx", [b, 3, 0, b, 3, 5, 3, b, b, 0, 128, b, b], f + [0.0]), ("mirror_lower_tiles", [b, 128, 0], ())]
    before = _host(buf).copy()
    for name, args, fa in calls:
        _run(eng, name, args, fa, launches=0)
    _same(_host(buf), before)
    got = _host(z)
    assert np.all(got[:P.n_theta + 1] == 0) and _raw(got[P.n_theta + 1:]).tolist() == _raw(np.full(15 - P.n_theta, POISON)).tolist()


def test_misuse_returns_einval_or_estate_and_launches_nothing(eng):
    import gpb200
    fresh = gpb200.Engine(0)
    try:
        buf = _dev(np.zeros(4 * T * T))
        b = buf.data_ptr()
        with pytest.raises(ValueError, match="set_kernel first"):
            fresh.gram_kernels("crossgram", [b, 3, 5, 128, b, 3, 5, 128, 3, b, 128], [0.0, 0.0])
    finally:
        fresh.close()
    P, theta = _exact(eng)
    f = list(theta)
    good = [b, 3, 5, 128, b, 3, 5, 128, 3, b, 128]
    _run(eng, "crossgram", good, f)

    def sub(i, v, base=good):
        a = list(base)
        a[i] = v
        return a
    gl = [b, 3, 3, 5, 128, b, 1, b, 128, 0, 1, 0, 0, 0]
    tr = [b, 3, 3, 5, 128, b, b, 128, b, b, 1, 0, 1]
    trr = [b, 3, 5, b, 3, 5, 3, b, 128, b, b]
    gg = [b, 3, 3, 5, 128, 0, b, 128, 0, 128]
    bad = [("crossgram", good[:-1], f), ("crossgram", good, f[:-1]), ("crossgram", good, f + [0.0]),
           ("crossgram", sub(8, 0), f), ("crossgram", sub(8, 129), f), ("crossgram", sub(8, 2), f),   # d; program reads dim 2
           ("crossgram", sub(0, 0), f), ("crossgram", sub(9, 0), f), ("crossgram", sub(2, -1), f),
           ("crossgram", sub(3, 64), f), ("crossgram", sub(3, 0), f), ("crossgram", sub(7, 130), f),
           ("crossgram", sub(10, 129), f), ("crossgram", sub(9, b + 8), f), ("crossgram", sub(10, 127), f),
           ("crossgram", sub(1, 2), f),
           ("gram_lower", sub(7, b + 8, gl), f + [0.0]), ("gram_lower", sub(8, 129, gl), f + [0.0]), ("gram_lower", sub(8, 126, gl), f + [0.0]),
           ("gram_lower", sub(11, 1, gl), f + [0.0]), ("gram_lower", sub(12, 2, gl), f + [0.0]),
           ("gram_lower", sub(6, 3, gl), f + [0.0]), ("gram_lower", sub(10, 0, gl), f + [0.0]),
           ("gram_full", [b, 3, 5, 128, 3, b + 8, 128], f), ("gram_full", [b, 3, 5, 128, 3, b, 129], f),
           ("trace", sub(6, b + 8, tr), f), ("trace", sub(7, 129, tr), f), ("trace", sub(10, 0, tr), f),
           ("trace", sub(11, 1, tr), f), ("trace", sub(12, 0, tr), f),
           ("trace_rect", sub(7, b + 8, trr), f), ("trace_rect", sub(8, 127, trr), f), ("trace_rect", sub(5, -1, trr), f),
           ("gram_grad_full", sub(5, P.n_theta, gg), f), ("gram_grad_full", sub(5, -1, gg), f),
           ("gram_grad_full", sub(8, 64, gg), f), ("gram_grad_full", sub(9, 256, gg), f),
           ("crossgram_grad", [b, 3, 5, 128, b, 3, 5, 128, 3, P.n_theta, b, 128], f),
           ("kdiag", [b, 2, 3, 5, b], f), ("kdiag_grad", [b, 3, 3, -1, b, b], f),
           ("crossgram_dx", [b, 3, 5, b, 3, 5, 3, b, b, 0, 128, b, 0], f + [0.0]),
           ("crossgram_dx", [b, 3, 5, b, 3, 5, 3, b, b, 0, 4, b, b], f + [0.0]),
           ("mirror_lower_tiles", [b, 128, 64], ()), ("mirror_lower_tiles", [b, 127, 128], ()),
           ("mirror_lower_tiles", [b, 128, 128], [0.0])]
    n0 = eng.launch_count()
    for name, args, fa in bad:
        with pytest.raises(ValueError):
            eng.gram_kernels(name, [int(a) for a in args], fa)
    for which in (-1, 11):
        a = np.zeros(3, dtype=np.int64)
        rc = eng._lib.gpb200_gram_kernels(eng._h, which, a.ctypes.data_as(gpb200.capi._lp), 3, None, 0)
        assert rc == gpb200.capi.EINVAL
    assert eng.launch_count() == n0


def test_seiso_fast_flag_follows_the_data_dimension():
    import gpb200
    rng = np.random.default_rng(5)
    X3 = rng.standard_normal((300, 3))
    k3 = gpb200.SEIso(0.3, 0.2)
    grams = []
    for order in ("data first", "kernel first"):
        e = gpb200.Engine(0)
        try:
            e.set_option("gram_fast", 0)
            ops, dims, theta, _ = gpb200.flatten(k3, 3)
            if order == "data first":
                e.set_data(X3)
                e.set_kernel(ops, dims, theta.size)
            else:
                e.set_kernel(ops, dims, theta.size)
                e.set_data(X3)
            e.factorize(theta, -1.0)
            grams.append(e.gram())
        finally:
            e.close()
    _same(grams[1], grams[0])
    # a program that reads a dimension the new data lacks is dropped: factorize asks for set_kernel
    e = gpb200.Engine(0)
    try:
        ops, dims, theta, _ = gpb200.flatten(k3, 3)
        e.set_data(X3)
        e.set_kernel(ops, dims, theta.size)
        e.set_data(X3[:, :2])
        with pytest.raises(ValueError, match="set_kernel"):
            e.factorize(theta, -1.0)
        # a two-dimensional SEIso program set on three-dimensional data becomes the specialised one at d = 2
        ops2, dims2, theta2, _ = gpb200.flatten(gpb200.SEIso(0.3, 0.2), 2)
        e.set_data(X3)
        e.set_kernel(ops2, dims2, theta2.size)
        e.set_option("gram_fast", 0)
        e.set_data(X3[:, :2])
        e.factorize(theta2, -1.0)
        G2 = e.gram()
    finally:
        e.close()
    f = gpb200.Engine(0)
    try:
        f.set_option("gram_fast", 0)
        f.set_data(X3[:, :2])
        f.set_kernel(ops2, dims2, theta2.size)
        f.factorize(theta2, -1.0)
        _same(G2, f.gram())
    finally:
        f.close()


def test_print_ratio_table():
    for key in sorted(RATIOS, key=str):
        print("RATIO-TABLE %-50s %.3e" % (key, RATIOS[key]))
