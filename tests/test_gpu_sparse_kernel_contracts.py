"""GPU: the sparse engine's non-GEMM kernels, tested directly against the model tests/sparse_model.py.

* FSA block-diagonal kernels (csrc/fsa.cu) through gpb200_fsa_kernels: Gram tiles, block-diagonal row products, masks,
  permutations, the gradient trace, the cross-Gram and the row products of predictions, on the tile lists the engine
  builds (sparse_model.Layout restates gpb200_fitc_set_blocks).
* Sparse cross-validation row kernels (csrc/fitc_cv.cu) and the FITC element kernels of csrc/vec.cu through
  gpb200_fitc_cv_kernels.

Exact cases use dyadic operands j / 256 (or j / 16 where many products are summed), small integers, powers of two for
lambda, and kernel programs whose values and theta-gradients are exact in binary64 for such inputs (LinIso + Const,
LinArd and Poly of degree 2 at theta = 0; sparse_model.kprog, checked against the oracle on the CPU).  Every product and
partial sum is then exact, so the kernels match the model bit for bit whatever their summation order.  Elements a
kernel must not read hold NaN; elements it must not write hold a NaN with its own payload that must come back unchanged.

Transcendental leaves (the kernel zoo of conftest.kernel_zoo) are checked against the oracle:
* fsa_gram / fsa_crossgram values within 4 ulp of the largest entry (the dense Gram's bound, DESIGN section 1), and
  fsa_gram's off-diagonal entries bitwise equal to the dense generic Gram (both evaluate kprog_eval<false>(P, x_i, x_j)),
  except for the single SEIso leaf, which the dense Gram evaluates through its own specialised formula;
* delta (kind 0) and fsa_trace gradients within gamma_m sum |w| |g| + 1e-12 max |g_p| sum |w|: the summation bound of
  sparse_model plus an allowance of 1e-12 of the largest entry of dK/dtheta_p per evaluated leaf gradient.

The file sorts after every file that opens a torch.profiler session; it opens none itself, and uses engines of its own
because it calls set_kernel."""
import zlib

import numpy as np
import pytest

import sparse_model as sm
import vec_model as vm
from conftest import kernel_zoo
from oracle import gp_oracle as orc

pytestmark = pytest.mark.gpu

T = sm.T
POISON = np.array([0x7FF8_DEAD_0000_0003], dtype=np.uint64).view(np.float64)[0]   # "never read, never written"
NAN = np.nan                                                                         # "never read"


def _bits(a):
    a = np.where(a == 0, 0.0, a)                 # +0 and -0 are the same result of an exact sum
    return np.ascontiguousarray(a).view(np.uint64)


def _raw(a):
    return np.ascontiguousarray(a).view(np.uint64)


def _same(got, want):
    """bitwise, with POISON payloads compared raw and every other value up to the sign of zero"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape
    bad = _bits(got) != _bits(want)
    assert not bad.any(), (int(bad.sum()), np.argwhere(bad)[:3].tolist(), got[bad][:3], want[bad][:3])


def _torch():
    import torch
    return torch


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a)).to("cuda:0")


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
    spec = kernel.spec()
    return theta, (spec[1] if spec[0] == "Fixed" else spec)


def _run(e, fn, name, args, fargs=(), launches=1):
    n0 = e.launch_count()
    getattr(e, fn)(name, [int(a) for a in args], fargs)
    assert e.launch_count() - n0 == launches, (name, e.launch_count() - n0)


def _items(base, items):
    return [v for off, ld, ri, rj, dg in items for v in (base.data_ptr() + 8 * off, ld, ri, rj, dg)]


def _exact_kernels(d):
    import gpb200 as g
    return [("LinIso+Const", g.LinIso(0.0) + g.Const(0.0)), ("LinArd", g.LinArd([0.0] * d)), ("Poly2", g.Poly(0.0, 0.0, 2))]


def _kf(spec):
    return lambda X1, X2: sm.kprog(spec, X1, X2)[0]


def _gf(spec):
    return lambda X1, X2: sm.kprog(spec, X1, X2, grad=True)[1]


# ---- fsa_gram ------------------------------------------------------------------------------------------------------------

BLOCKS = [1, 127, 128, 129, 2048]


@pytest.mark.parametrize("kname", ["LinIso+Const", "LinArd", "Poly2"])
def test_fsa_gram_exact_blocks_padding_and_diagonal_tiles(eng, kname):
    d = 3
    rng = np.random.default_rng(len(kname))
    lay = sm.Layout(BLOCKS)
    theta, spec = _program(eng, dict(_exact_kernels(d))[kname], d)
    xb = np.where(lay.mask[:, None] != 0, vm.dyadic(rng, (lay.Np, d)), NAN)          # padding rows are never evaluated
    dst = np.full(lay.packed, POISON)
    ddst, dx, dm = _dev(dst), _dev(xb), _dev(lay.mask)
    items = lay.gram_items()
    _run(eng, "fsa_kernels", "gram", [dx.data_ptr(), d, dm.data_ptr()] + _items(ddst, items), list(theta) + [0.5])
    got = _host(ddst)
    _same(got, sm.gram(_kf(spec), xb, items, lay.mask, 0.5, dst))
    for b, (n, B) in enumerate(zip(BLOCKS, lay.bsize)):
        blk = lay.block(got, b)
        assert np.array_equal(_raw(blk[np.triu_indices(B, 1)]), _raw(np.full(B * (B - 1) // 2, POISON)))   # upper: untouched
        pad = np.arange(n, B)
        assert np.all(blk[pad, pad] == 1.0) and np.all(np.tril(blk, -1)[n:] == 0) and np.all(blk[n:, :n] == 0)
        Kd = np.diag(sm.kprog(spec, xb[lay.bstart[b]:lay.bstart[b] + n], xb[lay.bstart[b]:lay.bstart[b] + n])[0])
        assert np.array_equal(np.diag(blk)[:n], Kd + 0.5)


def _zoo():
    out = [(n, k, 3) for n, k in kernel_zoo(3)]
    out += [(n + "(d=8)", k, 8) for n, k in kernel_zoo(8) if "Ard" in n]
    return out


ZOO = _zoo()


@pytest.mark.parametrize("name,kernel,d", ZOO, ids=[z[0] for z in ZOO])
def test_fsa_gram_and_crossgram_zoo_against_oracle_and_dense_gram(name, kernel, d):
    import gpb200 as g
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    N, Ms = 200, 130
    X = rng.standard_normal((N, d))
    X[7] = X[3]                                                                     # a duplicated input (Noise)
    Xs = rng.standard_normal((Ms, d))
    e = g.Engine(0)
    try:
        e.set_data(X)
        theta, spec = _program(e, kernel, d)
        e.set_option("gram_fast", 0)
        e.factorize(theta, 0.0)
        Kd = e.gram()                                                               # dense generic Gram + noise on the diagonal
        lay = sm.Layout([N])
        xb = np.zeros((lay.Np, d))
        xb[:N] = X
        dst = np.full(lay.packed, POISON)
        ddst, dx, dm = _dev(dst), _dev(xb), _dev(lay.mask)
        items = lay.gram_items()
        _run(e, "fsa_kernels", "gram", [dx.data_ptr(), d, dm.data_ptr()] + _items(ddst, items), list(theta) + [0.0])
        G = np.tril(lay.block(_host(ddst), 0))[:N, :N]
        Ko = orc.cov(spec, X)
        bound = 4 * np.spacing(np.max(np.abs(Ko)))
        low = np.tril_indices(N, -1)
        # a single SEIso leaf over every dimension takes the dense Gram's specialised path (csrc/gram.cu FAST:
        # s2 exp(mh r2) with mh = -1/(2 l^2) precomputed), a different rounding of the same value; every other program
        # runs kprog_eval<false> in both kernels
        if name != "SEIso":
            assert np.array_equal(_raw(G[low]), _raw(Kd[low])), (name, int(np.sum(G[low] != Kd[low])))
        err = np.max(np.abs(np.tril(G) - np.tril(Ko)))
        print("RATIO fsa_gram %s max|err|/(4 ulp of max|K|) = %.3e" % (name, err / bound))
        assert err <= bound, (name, err / bound)
        # cross-Gram: two test tiles against the training block; padding columns are 0
        Msp = 2 * T
        xs = np.full((Msp, d), NAN)
        xs[:Ms] = Xs
        xs[Ms:] = 0.0
        ld = lay.bsize[0] + 8
        cdst = np.full(Msp * ld, POISON)
        dcd, dxs = _dev(cdst), _dev(xs)
        citems = [(i * T * ld + j * T, ld, i * T, j * T, 0) for i in range(2) for j in range(lay.bsize[0] // T)]
        _run(e, "fsa_kernels", "crossgram", [dxs.data_ptr(), dx.data_ptr(), d, dm.data_ptr()] + _items(dcd, citems), theta)
        C = _host(dcd).reshape(Msp, ld)
        assert np.array_equal(_raw(C[:, lay.bsize[0]:]), _raw(np.full((Msp, 8), POISON)))
        assert np.all(C[:, N:lay.bsize[0]] == 0)
        Co = orc.cov(spec, Xs, X)
        err = np.max(np.abs(C[:Ms, :N] - Co))
        bound = 4 * np.spacing(np.max(np.abs(Co)))
        print("RATIO fsa_crossgram %s max|err|/(4 ulp of max|K|) = %.3e" % (name, err / bound))
        assert err <= bound, (name, err / bound)
    finally:
        e.close()


# ---- fsa_bdmv, mask, permute, resid, outer, var ----------------------------------------------------------------------------

LAYOUT_SIZES = [0, 1, 127, 128, 129, 300, 1100, 2048]


def _layout_dev(lay):
    return [_dev(lay.rblk), _dev(lay.bstart), _dev(np.array(lay.bsize, np.int32)), _dev(lay.boff)]


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_fsa_bdmv_exact_every_row_length_other_triangle_poisoned(eng, mode):
    rng = np.random.default_rng(10 + mode)
    lay = sm.Layout(LAYOUT_SIZES)
    pk = vm.dyadic(rng, lay.packed)
    for b, B in enumerate(lay.bsize):
        blk = lay.block(pk, b)
        blk[np.tril_indices(B, -1) if mode == 1 else np.triu_indices(B, 1)] = NAN
    v = np.concatenate([rng.integers(-4, 5, lay.Np).astype(np.float64), np.full(64, NAN)])
    y = np.full(lay.Np + 64, POISON)
    dp, dv, dy = _dev(pk), _dev(v), _dev(y)
    rb, bs, bz, bo = _layout_dev(lay)
    _run(eng, "fsa_kernels", "bdmv", [mode, dp.data_ptr(), rb.data_ptr(), bs.data_ptr(), bz.data_ptr(), bo.data_ptr(),
                                      dv.data_ptr() if mode != 2 else 0, dy.data_ptr(), lay.Np])
    got = _host(dy)
    _same(got, np.concatenate([sm.bdmv(mode, pk, lay, None if mode == 2 else v), y[lay.Np:]]))


def test_fsa_bdmv_gaussian_within_bound(eng):
    _need_longdouble()
    rng = np.random.default_rng(13)
    lay = sm.Layout([1, 129, 2048])
    pk, v = rng.standard_normal(lay.packed), rng.standard_normal(lay.Np)
    rb, bs, bz, bo = _layout_dev(lay)
    dp, dv = _dev(pk), _dev(v)
    for mode in (0, 1, 2):
        dy = _dev(np.full(lay.Np, POISON))
        _run(eng, "fsa_kernels", "bdmv", [mode, dp.data_ptr(), rb.data_ptr(), bs.data_ptr(), bz.data_ptr(), bo.data_ptr(),
                                          dv.data_ptr(), dy.data_ptr(), lay.Np])
        got = _host(dy)
        err = np.abs(got - sm.bdmv(mode, pk, lay, v, np.longdouble))
        bnd = sm.bdmv_bound(mode, pk, lay, v)
        print("RATIO bdmv mode=%d max|err|/bound = %.3e" % (mode, float(np.max(err / bnd))))
        assert np.all(err <= bnd), mode


@pytest.mark.parametrize("ncols", [1, 255, 16384, 16385, 40000])
def test_fsa_mask_rows_columns_and_both_past_the_grid_cap(eng, ncols):
    rng = np.random.default_rng(ncols)
    nrows, ld = 3, ncols + 3
    A = np.full((nrows + 1, ld), POISON)
    A[:nrows, :ncols] = vm.dyadic(rng, (nrows, ncols))
    rm = np.array([1.0, 0.0, 1.0, NAN])
    cm = np.concatenate([(rng.random(ncols) < 0.7).astype(np.float64), np.full(5, NAN)])
    cm[-6] = 0.0                                                      # the last column is masked
    drm, dcm = _dev(rm), _dev(cm)
    for r, c in ((drm, None), (None, dcm), (drm, dcm)):
        dA = _dev(A)
        _run(eng, "fsa_kernels", "mask", [dA.data_ptr(), ld, nrows, ncols, r.data_ptr() if r is not None else 0,
                                          c.data_ptr() if c is not None else 0])
        want = sm.mask(A, nrows, ncols, rm if r is not None else None, cm if c is not None else None)
        assert np.array_equal(_raw(_host(dA)), _raw(want))


def test_fsa_permute_resid_outer_var_exact(eng):
    rng = np.random.default_rng(21)
    lay = sm.Layout([1, 129, 300], rng.permutation(430))
    N = lay.N
    src = vm.dyadic(rng, lay.Np)
    dpos = _dev(lay.pos)
    for scatter in (1, 0):
        s = np.concatenate([src[:N] if scatter else src, np.full(7, NAN)]) if scatter else src
        dst = np.full(lay.Np + 7, POISON)
        ds, dd = _dev(s), _dev(dst)
        _run(eng, "fsa_kernels", "permute", [scatter, ds.data_ptr(), dpos.data_ptr(), N, dd.data_ptr()])
        assert np.array_equal(_raw(_host(dd)), _raw(sm.permute(scatter, s, lay.pos, N, dst)))
    a, b = vm.dyadic(rng, lay.Np + 5), vm.dyadic(rng, lay.Np + 5)
    a[lay.Np:] = b[lay.Np:] = NAN
    m = np.concatenate([lay.mask, np.full(5, NAN)])
    out = np.full(lay.Np + 5, POISON)
    da_, db_, dm, do = _dev(a), _dev(b), _dev(m), _dev(out)
    _run(eng, "fsa_kernels", "resid", [do.data_ptr(), da_.data_ptr(), db_.data_ptr(), dm.data_ptr(), lay.Np])
    _same(_host(do), sm.resid(a, b, m, lay.Np, out))
    do = _dev(out)
    _run(eng, "fsa_kernels", "var", [do.data_ptr(), da_.data_ptr(), db_.data_ptr(), dm.data_ptr(), lay.Np - 3])
    _same(_host(do), sm.var(a, b, m, lay.Np - 3, out))
    W = vm.dyadic(rng, lay.packed)
    dW = _dev(W)
    items = lay.gtiles()
    _run(eng, "fsa_kernels", "outer", [da_.data_ptr()] + _items(dW, items))
    _same(_host(dW), sm.outer(items, a, W))


# ---- fsa_trace -------------------------------------------------------------------------------------------------------------

TRACE_CASES = [(1, 1), (1, 256), (1, 257), (1, 4096), (33, 256), (33, 257), (96, 1), (96, 257)]


def _trace_setup(rng, d, ntiles, exact):
    Np = 8 * T
    msk = np.ones(Np)
    msk[::7] = 0.0
    msk[T - 1] = 0.0
    if exact:
        xb = rng.integers(-16, 17, (Np, d)).astype(np.float64) / 16
        W = rng.integers(-4, 5, 4 * T * T).astype(np.float64)
    else:
        xb = rng.standard_normal((Np, d))
        W = rng.standard_normal(4 * T * T)
    xb[msk == 0] = NAN                                                 # masked rows are never evaluated
    items = [((t % 4) * T * T, T, T * (t % 8), T * ((3 * t + 1) % 8), 0) for t in range(ntiles)]
    return xb, msk, W, items


def _trace_call(e, theta, xb, msk, W, items, P):
    dx, dm, dW = _dev(xb), _dev(msk), _dev(W)
    part = _dev(np.full(max(len(items), 1) * P, POISON))
    out = _dev(np.full(P + 1, POISON))
    _run(e, "fsa_kernels", "trace", [dx.data_ptr(), xb.shape[1], dm.data_ptr(), part.data_ptr(), out.data_ptr()]
         + _items(dW, items), theta, launches=2 if items else 0)
    got = _host(out)
    assert np.array_equal(_raw(got[P:]), _raw(np.full(1, POISON)))
    assert np.array_equal(_raw(_host(dW)), _raw(W))
    return got[:P]


@pytest.mark.parametrize("P,ntiles", TRACE_CASES)
def test_fsa_trace_exact_parameters_tiles_and_repeats(eng, P, ntiles):
    import gpb200 as g
    rng = np.random.default_rng(P * 10000 + ntiles)
    d = {1: 3, 33: 32, 96: 96}[P]
    kernel = {1: g.LinIso(0.0), 33: g.LinArd([0.0] * d) + g.Const(0.0), 96: g.LinArd([0.0] * d)}[P]
    theta, spec = _program(eng, kernel, d)
    assert theta.size == P
    xb, msk, W, items = _trace_setup(rng, d, ntiles, exact=True)
    got = _trace_call(eng, theta, xb, msk, W, items, P)
    _same(got, sm.trace(_gf(spec), xb, items, msk, W, P))
    assert np.array_equal(_raw(_trace_call(eng, theta, xb, msk, W, items, P)), _raw(got))


def test_fsa_trace_no_items_zeroes_out_and_launches_nothing(eng):
    import gpb200 as g
    theta, _ = _program(eng, g.LinArd([0.0] * 4) + g.Const(0.0), 4)
    got = _trace_call(eng, theta, np.zeros((T, 4)), np.ones(T), np.zeros(T * T), [], 5)
    assert np.array_equal(_raw(got), np.zeros(5, np.uint64))


TRACE_ZOO = [z for z in ZOO if z[2] == 3] + [("SEArd(d=95)", None, 95)]


def _leaf_allowance(gfun, xb, items, msk, W, P):
    """1e-12 max |dK/dtheta_p| sum |w| over the evaluated entries"""
    gmax, wsum = np.zeros(P), 0.0
    for w, g, real in sm.trace_terms(gfun, xb, items, msk, W):
        gmax = np.maximum(gmax, [np.max(np.abs(np.where(real, gp, 0))) for gp in g])
        wsum += float(np.sum(np.abs(w)))
    return 1e-12 * gmax * wsum


@pytest.mark.parametrize("name,kernel,d", TRACE_ZOO, ids=[z[0] for z in TRACE_ZOO])
def test_fsa_trace_zoo_within_bound(eng, name, kernel, d):
    import gpb200 as g
    _need_longdouble()
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    if kernel is None:
        kernel = g.SEArd([0.5 + 0.01 * i for i in range(d)], 0.1)
    theta, spec = _program(eng, kernel, d)
    P = theta.size
    xb, msk, W, items = _trace_setup(rng, d, 12, exact=False)
    xb[3] = xb[9]                                                      # a duplicated input (Noise)
    gfun = lambda X1, X2: orc.cov_and_grads(spec, X1, X2, True)[1]
    got = _trace_call(eng, theta, xb, msk, W, items, P)
    ref = sm.trace(gfun, xb, items, msk, W, P, np.longdouble)
    bnd = sm.trace_bound(gfun, xb, items, msk, W, P) + _leaf_allowance(gfun, xb, items, msk, W, P)
    err = np.abs(got - ref)
    assert np.all(np.isfinite(got)), name
    print("RATIO fsa_trace %s max|err|/bound = %.3e" % (name, float(np.max(err / np.where(bnd > 0, bnd, np.inf)))))
    assert np.all(err <= bnd), (name, err, bnd)


# ---- fsa_axpy_t, fsa_rowdot ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("nrows,ncols", [(1, 1), (31, 33), (129, 4097)])
def test_fsa_axpy_t_exact_edges(eng, nrows, ncols):
    rng = np.random.default_rng(nrows * ncols)
    ldc, lda = ncols + 3, nrows + 5
    C = np.full((nrows + 1, ldc), POISON)
    C[:nrows, :ncols] = vm.dyadic(rng, (nrows, ncols))
    A = np.full((ncols + 1, lda), NAN)
    A[:ncols, :nrows] = vm.dyadic(rng, (ncols, nrows))
    dC, dA = _dev(C), _dev(A)
    _run(eng, "fsa_kernels", "axpy_t", [dC.data_ptr(), ldc, dA.data_ptr(), lda, nrows, ncols], [-2.0])
    assert np.array_equal(_raw(_host(dC)), _raw(sm.axpy_t(C, A, nrows, ncols, -2.0)))


@pytest.mark.parametrize("K", [0, 1, 31, 32, 33, 4096])
def test_fsa_rowdot_exact_both_modes_lda_above_k(eng, K):
    rng = np.random.default_rng(K + 3)
    lda = K + 5
    As = [np.full((T, lda), NAN) for _ in range(2)]
    for A in As:
        A[:, :K] = vm.dyadic(rng, (T, K))
    v = np.concatenate([vm.dyadic(rng, K), np.full(4, NAN)])
    dA, dv = [_dev(A) for A in As], _dev(v)
    for sq in (0, 1):
        outs = [_dev(np.full(T + 1, POISON)) for _ in As]
        items = [x for A, o in zip(dA, outs) for x in (A.data_ptr(), dv.data_ptr() if not sq else 0, o.data_ptr(), lda, K, sq)]
        _run(eng, "fsa_kernels", "rowdot", items)
        for A, o in zip(As, outs):
            _same(_host(o), np.concatenate([sm.rowdot(A, v, K, sq), [POISON]]))


# ---- delta -----------------------------------------------------------------------------------------------------------------

def _delta_call(e, kind, theta, x, ldx, d, j, G, C, ld, ncols, nrows, rows_pad, alpha, d0, a0):
    dx, dG, dC, dal, dd, dda = _dev(x), _dev(G), _dev(C), _dev(alpha), _dev(d0), _dev(a0)
    _run(e, "fitc_cv_kernels", "delta", [kind, dx.data_ptr(), ldx, d, j, dG.data_ptr(), dC.data_ptr(), ld, ncols, nrows,
                                          rows_pad, dal.data_ptr(), dd.data_ptr(), dda.data_ptr()], theta)
    return _host(dd), _host(dda)


@pytest.mark.parametrize("kname", ["LinIso+Const", "LinArd", "Poly2"])
def test_delta_exact_every_parameter_padding_rows_and_kinds(eng, kname):
    d, nrows, rows_pad, ncols, ld, ldx = 3, 50, 64, 37, 41, 5
    rng = np.random.default_rng(len(kname) + 100)
    theta, spec = _program(eng, dict(_exact_kernels(d))[kname], d)
    x = np.full((rows_pad + 2, ldx), NAN)
    x[:nrows, :d] = vm.dyadic(rng, (nrows, d))
    G, C = np.full((rows_pad, ld), NAN), np.full((rows_pad, ld), NAN)
    G[:nrows, :ncols], C[:nrows, :ncols] = vm.dyadic(rng, (nrows, ncols)), vm.dyadic(rng, (nrows, ncols))
    alpha = np.concatenate([vm.dyadic(rng, nrows), np.full(rows_pad - nrows + 2, NAN)])
    d0, a0 = np.full(rows_pad + 2, POISON), np.full(rows_pad + 2, POISON)
    _, gd = sm.kprog(spec, x[:nrows, :d], x[:nrows, :d], grad=True)
    for kind in (0, 1, 2):
        for j in (range(theta.size) if kind == 0 else [0]):
            got = _delta_call(eng, kind, theta, x, ldx, d, j, G, C, ld, ncols, nrows, rows_pad, alpha, d0, a0)
            want = sm.delta(kind, np.diag(gd[j]), G, C, ncols, nrows, rows_pad, alpha, d0, a0)
            for g_, w_ in zip(got, want):
                _same(g_, w_)


DELTA_ZOO = ZOO


@pytest.mark.parametrize("name,kernel,d", DELTA_ZOO, ids=[z[0] for z in DELTA_ZOO])
def test_delta_zoo_finite_and_within_bound(eng, name, kernel, d):
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    nrows, rows_pad = 40, 48
    theta, spec = _program(eng, kernel, d)
    X = rng.standard_normal((nrows, d))
    X[5] = X[2]                                                       # duplicated training inputs
    x = np.full((rows_pad, d), NAN)
    x[:nrows] = X
    G = C = np.zeros((rows_pad, 32))                                  # ncols = 0: delta_i = dk(x_i, x_i)/dtheta_j
    alpha = np.concatenate([np.ones(nrows), np.full(rows_pad - nrows, NAN)])
    z = np.full(rows_pad, POISON)
    gK = orc.cov_and_grads(spec, X, X, True)[1]
    for j in range(theta.size):
        dl, da = _delta_call(eng, 0, theta, x, d, d, j, G, C, 32, 0, nrows, rows_pad, alpha, z, z)
        assert np.all(np.isfinite(dl[:nrows])) and np.all(da[nrows:] == 0), (name, j)
        err = np.max(np.abs(dl[:nrows] - np.diag(gK[j])))
        bound = 1e-12 * np.max(np.abs(gK[j]))
        print("RATIO delta %s j=%d max|err|/(1e-12 max|dK_j|) = %.3e" % (name, j, err / bound if bound else 0.0))
        assert err <= bound, (name, j, err, bound)


# ---- the other cross-validation row kernels and the FITC element kernels ---------------------------------------------------

def _lam(rng, n):
    return 2.0 ** rng.integers(-2, 3, n).astype(np.float64)


def test_rows_eblock_invdiag_qs_wvec_diag_exact(eng):
    rng = np.random.default_rng(31)
    nrows, ncols, ld = 50, 37, 41
    mat = lambda: np.where(np.arange(ld)[None, :] < ncols, vm.dyadic(rng, (nrows + 1, ld)), NAN)
    G, Ch, K, P = mat(), mat(), mat(), mat()
    lam = np.concatenate([_lam(rng, nrows), [NAN]])
    dl, alpha = np.concatenate([vm.dyadic(rng, nrows), [NAN]]), np.concatenate([vm.dyadic(rng, nrows), [NAN]])
    beta, w = np.concatenate([vm.dyadic(rng, ncols), [NAN] * 4]), np.concatenate([vm.dyadic(rng, ncols), [NAN] * 4])
    dev = {k: _dev(v) for k, v in dict(G=G, Ch=Ch, K=K, P=P, lam=lam, dl=dl, alpha=alpha, beta=beta, w=w).items()}
    p = lambda k: dev[k].data_ptr()
    for withG in (True, False):
        zja, dg = _dev(np.full(nrows + 1, POISON)), _dev(np.full(nrows + 1, POISON))
        _run(eng, "fitc_cv_kernels", "rows", [p("G") if withG else 0, p("Ch"), p("K"), p("P"), ld, nrows, ncols, p("lam"),
                                              p("dl"), p("alpha"), p("beta") if withG else 0, p("w"), zja.data_ptr(), dg.data_ptr()])
        wz, wd = sm.rows(G if withG else None, Ch, K, P, nrows, ncols, lam, dl, alpha, beta, w)
        _same(_host(zja), np.concatenate([wz, [POISON]]))
        _same(_host(dg), np.concatenate([wd, [POISON]]))
        E = np.full((nrows + 1, ld), POISON)
        E[:nrows, :ncols] = vm.dyadic(rng, (nrows, ncols))
        dE = _dev(E)
        _run(eng, "fitc_cv_kernels", "eblock", [dE.data_ptr(), p("G") if withG else 0, p("K"), ld, nrows, ncols, p("lam"), p("dl")])
        _same(_host(dE), sm.eblock(E, G if withG else None, K, nrows, ncols, lam, dl))
    out = np.full(nrows + 1, POISON)
    do = _dev(out)
    _run(eng, "fitc_cv_kernels", "invdiag", [nrows, p("lam"), p("alpha"), do.data_ptr()])
    _same(_host(do), sm.invdiag(lam, alpha, nrows, out))
    n = 37
    H, R = np.full((n + 1, ld), NAN), np.full((n + 1, ld), NAN)
    H[:n, :n], R[:n, :n] = vm.dyadic(rng, (n, n)), vm.dyadic(rng, (n, n))
    Q = np.full((n + 1, ld), POISON)
    dQ, dH, dR = _dev(Q), _dev(H), _dev(R)
    _run(eng, "fitc_cv_kernels", "qs", [dQ.data_ptr(), dH.data_ptr(), dR.data_ptr(), ld, n])
    _same(_host(dQ), sm.qs(H, R, n, Q))
    wv = np.full(n + 1, POISON)
    dw = _dev(wv)
    _run(eng, "fitc_cv_kernels", "wvec", [n, dw.data_ptr(), p("beta"), p("w"), p("alpha")])
    _same(_host(dw), sm.wvec(beta, w, alpha, n, wv))
    nv, ldo = 45, 53
    for which in (0, 1):
        O = np.full((nv + 1, ldo), POISON)
        O[:nv, :nv] = vm.dyadic(rng, (nv, nv))
        dO = _dev(O)
        _run(eng, "fitc_cv_kernels", "diag", [dO.data_ptr(), ldo, nv, which, p("lam"), p("dl") if which else 0])
        _same(_host(dO), sm.diag(O, nv, which, lam, dl))


def test_gather_duplicate_unsorted_indices(eng):
    rng = np.random.default_rng(41)
    N, d, ldx = 300, 3, 5
    x = np.full((N, ldx), NAN)
    x[:, :d] = vm.dyadic(rng, (N, d))
    lam, dl = vm.dyadic(rng, N), vm.dyadic(rng, N)
    idx = np.array([299, 3, 17, 3, 250, 0, 128, 127, 17, 299, 5], np.int64)
    nv = idx.size
    dix, dx, dlam, ddl = _dev(idx), _dev(x), _dev(lam), _dev(dl)
    for withd in (True, False):
        xo, lo, do = np.full((nv + 1, d), POISON), np.full(nv + 1, POISON), np.full(nv + 1, POISON)
        dxo, dlo, ddo = _dev(xo), _dev(lo), _dev(do)
        _run(eng, "fitc_cv_kernels", "gather", [nv, dix.data_ptr(), dx.data_ptr(), ldx, d, dxo.data_ptr(), dlam.data_ptr(),
                                                dlo.data_ptr(), ddl.data_ptr() if withd else 0, ddo.data_ptr()])
        wx, wl, wd = sm.gather(idx, x, d, lam, dl if withd else None, nv, xo, lo, do)
        assert np.array_equal(_raw(_host(dxo)), _raw(wx)) and np.array_equal(_raw(_host(dlo)), _raw(wl))
        assert np.array_equal(_raw(_host(ddo)), _raw(wd if withd else do))


def test_fitc_element_kernels_exact(eng):
    rng = np.random.default_rng(51)
    nrows, ncols, ld = 50, 37, 41
    full = lambda: np.where(np.arange(ld)[None, :] < ncols, vm.dyadic(rng, (nrows + 1, ld)), POISON)
    vpos = np.concatenate([_lam(rng, max(nrows, ncols)), [NAN]])
    v4 = np.concatenate([4.0 ** rng.integers(-1, 3, max(nrows, ncols)).astype(np.float64), [NAN]])
    dvp, dv4 = _dev(vpos), _dev(v4)
    A = full()
    A[nrows] = POISON
    dA = _dev(A)
    _run(eng, "fitc_cv_kernels", "colscale", [dA.data_ptr(), ld, nrows, ncols, dvp.data_ptr()])
    _same(_host(dA), sm.colscale(A, nrows, ncols, vpos))
    for mode, v, dv in ((0, v4, dv4), (1, vpos, dvp)):
        dA = _dev(A)
        _run(eng, "fitc_cv_kernels", "scale", [mode, dA.data_ptr(), ld, nrows, ncols, dv.data_ptr()])
        _same(_host(dA), sm.scale(mode, A, nrows, ncols, v))
    al, q = np.concatenate([vm.dyadic(rng, nrows), [NAN]]), np.concatenate([vm.dyadic(rng, nrows), [NAN]])
    g0 = np.full(nrows + 1, POISON)
    dal, dq, dg = _dev(al), _dev(q), _dev(g0)
    _run(eng, "fitc_cv_kernels", "fitc_g", [nrows, dal.data_ptr(), dvp.data_ptr(), dq.data_ptr(), dg.data_ptr()])
    gv = _host(dg)
    _same(gv, sm.fitc_g(al, vpos, q, nrows, g0))
    P1 = np.where(np.arange(ld)[None, :] < ncols, vm.dyadic(rng, (nrows + 1, ld)), NAN)
    beta = np.concatenate([vm.dyadic(rng, ncols), [NAN]])
    P2 = A.copy()
    dP2, dP1, db = _dev(P2), _dev(P1), _dev(beta)
    _run(eng, "fitc_cv_kernels", "fitc_wfu", [dP2.data_ptr(), dP1.data_ptr(), ld, nrows, ncols, dal.data_ptr(), dvp.data_ptr(),
                                              dg.data_ptr(), db.data_ptr()])
    _same(_host(dP2), sm.fitc_wfu(P2, P1, nrows, ncols, al, vpos, gv, beta))
    n = 37
    sq = lambda: np.where((np.arange(ld)[None, :] < n) & (np.arange(n + 1)[:, None] < n), vm.dyadic(rng, (n + 1, ld)), NAN)
    Tm, Ki, Si = sq(), sq(), sq()
    Wuu = np.full((n + 1, ld), POISON)
    dW, dT, dK, dS = _dev(Wuu), _dev(Tm), _dev(Ki), _dev(Si)
    _run(eng, "fitc_cv_kernels", "fitc_wuu", [dW.data_ptr(), dT.data_ptr(), dK.data_ptr(), dS.data_ptr(), ld, n, db.data_ptr()])
    _same(_host(dW), sm.fitc_wuu(Tm, Ki, Si, n, beta, Wuu))
    S = np.full((n + 1, ld), POISON)
    S[np.tril_indices(n)] = vm.dyadic(rng, n * (n + 1) // 2)
    dS = _dev(S)
    _run(eng, "fitc_cv_kernels", "symmetrize", [dS.data_ptr(), ld, n])
    assert np.array_equal(_raw(_host(dS)), _raw(sm.symmetrize(S, n)))


# ---- empty sizes, launch counts and rejections -------------------------------------------------------------------------------

def test_empty_sizes_launch_nothing(eng):
    import gpb200 as g
    theta, _ = _program(eng, g.LinIso(0.0) + g.Const(0.0), 3)
    buf = _dev(np.full(4 * T * T, POISON))
    ib = _dev(np.zeros(T, np.int64))
    p, q = buf.data_ptr(), ib.data_ptr()
    calls = [("fsa_kernels", "gram", [p, 3, p], list(theta) + [0.0]), ("fsa_kernels", "bdmv", [0, p, q, q, q, q, p, p, 0], ()),
             ("fsa_kernels", "mask", [p, 8, 0, 8, p, p], ()), ("fsa_kernels", "mask", [p, 8, 3, 0, p, p], ()),
             ("fsa_kernels", "permute", [1, p, q, 0, p], ()), ("fsa_kernels", "resid", [p, p, p, p, 0], ()),
             ("fsa_kernels", "outer", [p], ()), ("fsa_kernels", "axpy_t", [p, 8, p, 8, 0, 8], [1.0]),
             ("fsa_kernels", "crossgram", [p, p, 3, p], theta), ("fsa_kernels", "rowdot", [], ()),
             ("fsa_kernels", "var", [p, p, p, p, 0], ()),
             ("fitc_cv_kernels", "delta", [0, p, 3, 3, 0, p, p, 8, 8, 0, 0, p, p, p], theta),
             ("fitc_cv_kernels", "rows", [p, p, p, p, 8, 0, 8, p, p, p, p, p, p, p], ()),
             ("fitc_cv_kernels", "invdiag", [0, p, p, p], ()), ("fitc_cv_kernels", "eblock", [p, p, p, 8, 0, 8, p, p], ()),
             ("fitc_cv_kernels", "qs", [p, p, p, 8, 0], ()), ("fitc_cv_kernels", "wvec", [0, p, p, p, p], ()),
             ("fitc_cv_kernels", "gather", [0, q, p, 3, 3, p, p, p, p, p], ()), ("fitc_cv_kernels", "diag", [p, 8, 0, 0, p, p], ()),
             ("fitc_cv_kernels", "colscale", [p, 8, 0, 8, p], ()), ("fitc_cv_kernels", "colscale", [p, 8, 8, 0, p], ()),
             ("fitc_cv_kernels", "scale", [0, p, 8, 0, 8, p], ()), ("fitc_cv_kernels", "fitc_g", [0, p, p, p, p], ()),
             ("fitc_cv_kernels", "fitc_wfu", [p, p, 8, 0, 8, p, p, p, p], ()),
             ("fitc_cv_kernels", "fitc_wfu", [p, p, 8, 8, 0, p, p, p, p], ()),
             ("fitc_cv_kernels", "fitc_wuu", [p, p, p, p, 8, 0, p], ()), ("fitc_cv_kernels", "symmetrize", [p, 8, 0], ())]
    for fn, name, args, fargs in calls:
        _run(eng, fn, name, args, fargs, launches=0)
    assert np.array_equal(_raw(_host(buf)), _raw(np.full(4 * T * T, POISON)))


def test_rejections_launch_nothing(eng):
    import ctypes as C
    import gpb200 as g
    theta, _ = _program(eng, g.LinIso(0.0) + g.Const(0.0), 3)
    buf = _dev(np.zeros(4 * T * T))
    ib = _dev(np.zeros(T, np.int64))
    p, q = buf.data_ptr(), ib.data_ptr()
    th, th1 = list(theta), list(theta) + [0.0]
    item = [p, T, 0, 0, 1]
    bad = [("fsa_kernels", "gram", [p, 3, p] + item, th),                       # no diag_add
           ("fsa_kernels", "gram", [p, 3, p] + item[:4], th1),                  # n not 3 + 5 k
           ("fsa_kernels", "gram", [p, 3, p, p, 127, 0, 0, 1], th1),            # item ld < 128
           ("fsa_kernels", "gram", [p, 3, p, 0, T, 0, 0, 1], th1),              # null dst
           ("fsa_kernels", "gram", [p, 3, p, p, T, -128, 0, 1], th1),           # negative row
           ("fsa_kernels", "gram", [0, 3, p] + item, th1),                      # null xb
           ("fsa_kernels", "gram", [p, 2, p] + item, th1),                      # the program reads dimension 2
           ("fsa_kernels", "gram", [p, 0, p] + item, th1),                      # d < 1
           ("fsa_kernels", "bdmv", [3, p, q, q, q, q, p, p, 8], ()),            # mode
           ("fsa_kernels", "bdmv", [0, p, q, q, q, q, 0, p, 8], ()),            # mode 0 without v
           ("fsa_kernels", "bdmv", [0, p, q, q, q, q, p, p, -1], ()),           # negative Np
           ("fsa_kernels", "mask", [p, 7, 2, 8, p, p], ()),                     # ld < ncols
           ("fsa_kernels", "mask", [p, 8, -1, 8, p, p], ()),
           ("fsa_kernels", "permute", [2, p, q, 8, p], ()), ("fsa_kernels", "permute", [1, p, 0, 8, p], ()),
           ("fsa_kernels", "resid", [p, p, p, p, -1], ()), ("fsa_kernels", "resid", [p, p, 0, p, 8], ()),
           ("fsa_kernels", "outer", [0] + item, ()),
           ("fsa_kernels", "trace", [p, 3, p, 0, p] + item, th),                # null part with items
           ("fsa_kernels", "trace", [p, 3, p, p, p] + item, th1),               # theta length
           ("fsa_kernels", "axpy_t", [p, 7, p, 8, 8, 8], [1.0]),                # ldc < ncols
           ("fsa_kernels", "axpy_t", [p, 8, p, 7, 8, 8], [1.0]),                # lda < nrows
           ("fsa_kernels", "axpy_t", [p, 8, p, 8, 8, 8], ()),                   # no alpha
           ("fsa_kernels", "crossgram", [p, p, 3, 0] + item, th),               # null mask
           ("fsa_kernels", "rowdot", [p, p, p, 7, 8, 0], ()),                   # lda < K
           ("fsa_kernels", "rowdot", [p, 0, p, 8, 8, 0], ()),                   # null v with sq = 0
           ("fsa_kernels", "rowdot", [p, p, p, 8, -1, 0], ()),
           ("fsa_kernels", "var", [p, p, p, p, -2], ()),
           ("fitc_cv_kernels", "delta", [0, p, 3, 3, 0, p, p, 8, 8, 4, 8, p, p, p], th1),     # theta length
           ("fitc_cv_kernels", "delta", [0, p, 3, 3, 2, p, p, 8, 8, 4, 8, p, p, p], th),      # j >= n_theta
           ("fitc_cv_kernels", "delta", [0, p, 2, 3, 0, p, p, 8, 8, 4, 8, p, p, p], th),      # ldx < d
           ("fitc_cv_kernels", "delta", [0, p, 3, 3, 0, p, p, 7, 8, 4, 8, p, p, p], th),      # ld < ncols
           ("fitc_cv_kernels", "delta", [0, p, 3, 3, 0, 0, p, 8, 8, 4, 8, p, p, p], th),      # null G
           ("fitc_cv_kernels", "delta", [3, p, 3, 3, 0, p, p, 8, 8, 4, 8, p, p, p], th),      # kind
           ("fitc_cv_kernels", "delta", [1, p, 3, 3, 0, p, p, 8, 8, -4, 8, p, p, p], th),
           ("fitc_cv_kernels", "rows", [p, p, p, p, 7, 4, 8, p, p, p, p, p, p, p], ()),
           ("fitc_cv_kernels", "rows", [p, p, p, p, 8, 4, 8, p, p, p, 0, p, p, p], ()),       # G without beta
           ("fitc_cv_kernels", "invdiag", [-1, p, p, p], ()),
           ("fitc_cv_kernels", "eblock", [p, p, p, 7, 4, 8, p, p], ()), ("fitc_cv_kernels", "eblock", [p, p, 0, 8, 4, 8, p, p], ()),
           ("fitc_cv_kernels", "qs", [p, p, p, 7, 8], ()), ("fitc_cv_kernels", "wvec", [8, p, p, 0, p], ()),
           ("fitc_cv_kernels", "gather", [4, q, p, 2, 3, p, p, p, p, p], ()),                 # ldx < d
           ("fitc_cv_kernels", "gather", [4, q, p, 3, 3, p, p, p, p, 0], ()),                 # delta without delout
           ("fitc_cv_kernels", "diag", [p, 7, 8, 0, p, p], ()), ("fitc_cv_kernels", "diag", [p, 8, 8, 1, p, 0], ()),
           ("fitc_cv_kernels", "diag", [p, 8, 8, 2, p, p], ()),
           ("fitc_cv_kernels", "colscale", [p, 7, 4, 8, p], ()), ("fitc_cv_kernels", "scale", [2, p, 8, 4, 8, p], ()),
           ("fitc_cv_kernels", "fitc_g", [-1, p, p, p, p], ()), ("fitc_cv_kernels", "fitc_wfu", [p, p, 7, 4, 8, p, p, p, p], ()),
           ("fitc_cv_kernels", "fitc_wuu", [p, p, p, p, 7, 8, p], ()), ("fitc_cv_kernels", "symmetrize", [p, 7, 8], ()),
           ("fitc_cv_kernels", "wvec", [8, p, p, p], ()),                                     # n
           ("fitc_cv_kernels", "qs", [p, p, p, 8, 8], [1.0])]                                 # fargs where none are taken
    n0 = eng.launch_count()
    for fn, name, args, fargs in bad:
        with pytest.raises(ValueError):
            getattr(eng, fn)(name, args, fargs)
        assert eng.launch_count() == n0, (fn, name, args)
    lib = eng._lib
    a = np.zeros(16, np.int64)
    f = np.zeros(4)
    for fn, which in (("gpb200_fsa_kernels", 11), ("gpb200_fsa_kernels", -1), ("gpb200_fitc_cv_kernels", 14)):
        rc = getattr(lib, fn)(eng._h, which, a.ctypes.data_as(C.POINTER(C.c_int64)), 5, f.ctypes.data_as(C.POINTER(C.c_double)), 0)
        assert rc == g.capi.EINVAL
    assert eng.launch_count() == n0
    fresh = g.Engine(0)
    try:
        with pytest.raises(ValueError, match="set_kernel"):
            fresh.fsa_kernels("gram", [p, 3, p] + item, th1)
        assert fresh.launch_count() == 0
    finally:
        fresh.close()
