"""GPU: the TMA-staged SEIso Gram and trace kernels (csrc/gram_fast.cu), the training-input gradient inputs_dx (csrc/gram.cu)
and the elementwise and sampling helpers (csrc/vec.cu), each tested directly through gpb200_gram_kernels (which 11 - 13) and
gpb200_vec_kernels against tests/seiso_model.py and numpy.

* TMA Gram: bit for bit against the fma-exact model on dyadic points for d = 1 .. 8 (odd d with a zero pad column), on the
  device's own prepared constants; ownership filters; rows past N never read; long-double bounds at the numerical edges
  (length scales e^-6 / e^6, sigma^2 at the limits seiso_fast_prepare accepts, coincident points, the -960 underflow guard);
  the libm fallback of a tile with a non-finite input; agreement with the generic gram_lower.
* TMA trace and inputs_dx: within the long-double model's componentwise bound, unread elements NaN, ownership partitions,
  repeatability, and agreement with the generic kernels.
* ew, spd_from_cov, add_rowvec (up to 70 000 rows: more than gridDim.y allows), gather_block: bit for bit.
Elements a kernel must not read hold NaN, elements it must not write hold a NaN with its own payload (POISON).

The name puts the file after test_gpu_shard_cv.py, the last file that opens a torch.profiler session: a session started
about a minute or more after the process's first one records no device activity (see test_gpu_tile_kernel_contracts.py)."""
import zlib

import numpy as np
import pytest

import gram_model as gm
import seiso_model as sm
import test_gpu_tile_gram_kernel_contracts as tg
from conftest import kernel_zoo
from test_gpu_tile_gram_kernel_contracts import NAN, POISON, _dev, _dyadic, _host, _need_longdouble, _pad, _ratio, _raw, _same

pytestmark = pytest.mark.gpu

T = gm.T
NS = [1, 127, 128, 129, 257, 1000]


@pytest.fixture(scope="module")
def eng():
    import gpb200
    e = gpb200.Engine(0)
    yield e
    e.close()


def _run(e, name, args, fargs=(), launches=1):
    tg._run(e, name, args, fargs, launches)


def _seiso(e, d, ll, ls):
    import gpb200 as g
    return tg._program(e, g.SEIso(ll, ls), d)


def _xp(X, N, Npad, d):
    """the engine's two copies of the inputs: xp [Npad x dx] and xpt [dx x Npad], dx = d rounded up to even, the pad column
    zero, everything at or past row N NaN (outside the maps)"""
    dx = (d + 1) // 2 * 2
    xp = np.full((Npad, dx), NAN)
    xp[:N, :d] = X[:N]
    xp[:N, d:] = 0.0
    xpt = np.full((dx, Npad), NAN)
    xpt[:, :N] = xp[:N].T
    return xp, _dev(xp), _dev(xpt), dx


def _gram_tma(e, dxp, dxt, d, N, Npad, dn, n_noise, G0, ld, theta, nugget, own=(0, 1, 0, 0)):
    sf = np.zeros(67)
    dG = _dev(G0)
    _run(e, "gram_seiso_tma", [dxp.data_ptr(), dxt.data_ptr(), d, N, Npad, dn.data_ptr(), n_noise, dG.data_ptr(), ld, *own,
                               sf.ctypes.data], list(theta) + [nugget])
    return _host(dG), sm.from_device(sf)


# ---- TMA Gram ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("d", list(range(1, 9)))
def test_tma_gram_bitwise_on_dyadic_points(eng, d):
    rng = np.random.default_rng(100 + d)
    P, theta = _seiso(eng, d, 0.3, -0.2)
    for N in NS:
        Npad = _pad(N)
        ld = Npad + 2 * (d % 3)
        X = _dyadic(rng, (N, d))
        xp, dxp, dxt, dx = _xp(X, N, Npad, d)
        nv = np.full(Npad, NAN)
        nv[:N] = rng.integers(1, 8, N) / 4.0
        dn = _dev(nv)
        G0 = np.full(Npad * ld, POISON)
        for n_noise in (1, N):
            G, sf = _gram_tma(eng, dxp, dxt, d, N, Npad, dn, n_noise, G0, ld, theta, 0.125)
            want = sm.gram_seiso(xp[:N].ravel(), dx, N, Npad, sf, nv[:N] if n_noise > 1 else nv[:1], n_noise, 0.125, G0, ld)
            _same(G, want)
        assert sf["c_hi"] < 0 and sf["tab"][0] == sf["s2"]


def test_tma_gram_ownership_filters_bitwise(eng):
    rng = np.random.default_rng(7)
    d, N = 3, 1000
    Npad, ld = _pad(N), _pad(N) + 4
    P, theta = _seiso(eng, d, 0.1, 0.2)
    X = _dyadic(rng, (N, d))
    xp, dxp, dxt, dx = _xp(X, N, Npad, d)
    dn = _dev(np.full(1, 0.5))
    G0 = np.full(Npad * ld, POISON)
    full, sf = _gram_tma(eng, dxp, dxt, d, N, Npad, dn, 1, G0, ld, theta, 0.0)
    _same(full, sm.gram_seiso(xp[:N].ravel(), dx, N, Npad, sf, [0.5], 1, 0.0, G0, ld))
    for own_tiles in (1, 2):
        for nranks in (1, 2, 3):
            for axis in (0, 1):
                acc = np.array(G0)
                for rank in range(nranks):
                    G, _ = _gram_tma(eng, dxp, dxt, d, N, Npad, dn, 1, G0, ld, theta, 0.0, (own_tiles, nranks, rank, axis))
                    _same(G, sm.gram_seiso(xp[:N].ravel(), dx, N, Npad, sf, [0.5], 1, 0.0, G0, ld, own_tiles, nranks, rank, axis))
                    mine = _raw(G) != _raw(G0)
                    assert not np.any(mine & (_raw(acc) != _raw(G0)))          # no tile written by two ranks
                    acc = np.where(mine, G, acc)
                _same(acc, full)


def _edge_points(rng, d, ll):
    N = 300
    X = rng.standard_normal((N, d)) * np.exp(ll) * rng.uniform(0.2, 4.0, (N, 1))
    X[7] = X[3]
    X[200] = X[150]
    return X


@pytest.mark.parametrize("d", [3, 8])
@pytest.mark.parametrize("ll,ls", [(-6.0, 0.1), (6.0, 0.1), (0.2, 0.5 * np.log(1.0001e-15)), (0.2, 0.5 * np.log(9.9e14))])
def test_tma_gram_within_long_double_bound_and_the_generic_kernel(eng, d, ll, ls):
    _need_longdouble()
    rng = np.random.default_rng(zlib.crc32(("%d %g %g" % (d, ll, ls)).encode()))
    P, theta = _seiso(eng, d, ll, ls)
    X = _edge_points(rng, d, ll)
    N = X.shape[0]
    Npad = _pad(N)
    xp, dxp, dxt, dx = _xp(X, N, Npad, d)
    dn = _dev(np.zeros(1))
    G, sf = _gram_tma(eng, dxp, dxt, d, N, Npad, dn, 1, np.full(Npad * Npad, POISON), Npad, theta, 0.0)
    G = G.reshape(Npad, Npad)[:N, :N]
    l2, s2 = float(P.par[0]), float(P.par[1])
    _, k, kb = sm.k_ld(X, X, l2, s2)
    low = np.tril_indices(N, -1)
    err = np.abs((G[low] - k[low]).astype(float))
    _ratio(("tma gram", "edges"), err, kb[low])
    assert np.all(err <= kb[low]), float(np.max(err / kb[low]))
    assert G[7, 3] == sf["s2"] and G[200, 150] == sf["s2"] and np.all(np.diag(G) == sf["s2"])    # coincident: sigma^2
    xg = np.full((Npad, d + 1), NAN)
    xg[:N, :d] = X
    Gg = _dev(np.full((Npad, Npad), POISON))
    _run(eng, "gram_lower", [_dev(xg).data_ptr(), d + 1, d, N, Npad, dn.data_ptr(), 1, Gg.data_ptr(), Npad, 0, 1, 0, 0, 0],
         list(theta) + [0.0])
    Gg = _host(Gg)[:N, :N]
    kbg = gm.evaluate(P, np.repeat(X, N, 0), np.tile(X, (N, 1)), gm.LD)[1].reshape(N, N)
    assert np.all(np.abs(G[low] - Gg[low]) <= kb[low] + kbg[low])


def test_tma_gram_underflow_guard(eng):
    _need_longdouble()
    d = 3
    P, theta = _seiso(eng, d, 0.0, 0.0)
    zs = [-959.5, -960.0, -960.0004, -960.0006, -1000.0]
    sfh = sm.prepare(1.0, 1.0)
    X = np.zeros((len(zs) + 1, d))
    for i, z in enumerate(zs):
        X[i + 1, 0] = np.sqrt(z / sfh["c_hi"])
    N = X.shape[0]
    Npad = _pad(N)
    xp, dxp, dxt, dx = _xp(X, N, Npad, d)
    G0 = np.full(Npad * Npad, POISON)
    G, sf = _gram_tma(eng, dxp, dxt, d, N, Npad, _dev(np.zeros(1)), 1, G0, Npad, theta, 0.0)
    _same(G, sm.gram_seiso(xp[:N].ravel(), dx, N, Npad, sf, [0.0], 1, 0.0, G0, Npad))
    col = G.reshape(Npad, Npad)[1:N, 0]
    z = sm.r2_fma(X[1:], X[:1])[:, 0] * sf["c_hi"]
    assert np.allclose(z, zs, rtol=1e-15, atol=0)
    assert np.all(col[:3] > 2.0 ** -961) and np.all(col[3:] == 0.0)      # the guard: high word of z past that of -960
    _, k, kb = sm.k_ld(X, X, 1.0, 1.0)
    assert np.all(np.abs((col - k[1:, 0]).astype(float)) <= kb[1:, 0])


def test_tma_gram_nonfinite_tile_takes_the_libm_path(eng):
    _need_longdouble()
    rng = np.random.default_rng(21)
    d = 5
    P, theta = _seiso(eng, d, 0.4, 0.1)
    N = 300
    Npad = _pad(N)
    X = rng.standard_normal((N, d))
    xp, dxp, dxt, dx = _xp(X, N, Npad, d)
    dn = _dev(np.full(1, 0.25))
    G0 = np.full(Npad * Npad, POISON)
    clean, sf = _gram_tma(eng, dxp, dxt, d, N, Npad, dn, 1, G0, Npad, theta, 0.0)
    _same(clean, sm.gram_seiso(xp[:N].ravel(), dx, N, Npad, sf, [0.25], 1, 0.0, G0, Npad))
    bad = 200                                              # tile row / column 1
    Xn = X.copy()
    Xn[bad, 2] = np.nan
    _, dxp2, dxt2, _ = _xp(Xn, N, Npad, d)
    G, _ = _gram_tma(eng, dxp2, dxt2, d, N, Npad, dn, 1, G0, Npad, theta, 0.0)
    G, C = G.reshape(Npad, Npad), clean.reshape(Npad, Npad)
    hit = np.zeros((Npad, Npad), bool)
    for bm, bn in ((1, 0), (1, 1), (2, 1)):
        hit[bm * T:(bm + 1) * T, bn * T:(bn + 1) * T] = True
    _same(G[~hit], C[~hit])                                # every other tile: bitwise the clean run
    assert np.all(np.isnan(G[bad, :bad + 1])) and np.all(np.isnan(G[bad:N, bad]))
    _, k, kb = sm.k_ld(X, X, float(P.par[0]), float(P.par[1]))
    i, j = np.tril_indices(N, -1)
    sel = hit[i, j] & (i != bad) & (j != bad)
    i, j = i[sel], j[sel]
    err = np.abs((G[i, j] - k[i, j]).astype(float))
    _ratio(("tma gram", "libm tile"), err, kb[i, j])
    assert np.all(err <= kb[i, j])
    on = np.arange(T, 2 * T)
    on = on[on != bad]
    assert np.all(np.abs((G[on, on] - (k[on, on] + 0.25)).astype(float)) <= kb[on, on] + 2 * gm.U * (0.25 + float(P.par[1])))
    assert np.array_equal(G[N:, N:], np.eye(Npad - N))


# ---- TMA trace --------------------------------------------------------------------------------------------------------

def _trace_inputs(rng, N, Npad, d, ld):
    X = rng.standard_normal((N, d))
    alpha = np.full(Npad, NAN)
    alpha[:N] = rng.standard_normal(N)
    S = rng.standard_normal((N, N))
    Kinv = np.full((Npad, ld), NAN)                       # strict upper triangle, rows and columns past N: never read
    Kinv[:N, :N] = np.where(np.tril(np.ones((N, N), bool)), S + S.T, NAN)
    return X, alpha, Kinv


def _trace_tma(e, dxp, dxt, d, N, Npad, da, dK, ld, theta, bm=(1, 0, 1)):
    tiles = (Npad // T) * (Npad // T + 1) // 2
    part, out = _dev(np.full(tiles * 3 + 2, POISON)), _dev(np.full(5, POISON))
    _run(e, "trace_seiso_tma", [dxp.data_ptr(), dxt.data_ptr(), d, N, Npad, da.data_ptr(), dK.data_ptr(), ld, part.data_ptr(),
                                out.data_ptr(), *bm, 0], theta, launches=2)
    p, o = _host(part), _host(out)
    assert _raw(p[tiles * 3:]).tolist() == _raw(np.full(2, POISON)).tolist()
    assert _raw(o[3:]).tolist() == _raw(np.full(2, POISON)).tolist()
    return p[:tiles * 3].reshape(tiles, 3), o[:3]


@pytest.mark.parametrize("N", NS)
def test_tma_trace_within_long_double_bound(eng, N):
    _need_longdouble()
    rng = np.random.default_rng(300 + N)
    d = 3 if N != 257 else 8
    P, theta = _seiso(eng, d, 0.2, -0.1)
    Npad = _pad(N)
    ld = Npad + 2
    X, alpha, Kinv = _trace_inputs(rng, N, Npad, d, ld)
    _, dxp, dxt, _ = _xp(X, N, Npad, d)
    da, dK = _dev(alpha), _dev(Kinv)
    part, out = _trace_tma(eng, dxp, dxt, d, N, Npad, da, dK, ld, theta)
    l2, s2 = float(P.par[0]), float(P.par[1])
    Kl = np.nan_to_num(Kinv[:N, :N])
    wp, bp, wo, bo = sm.trace_seiso(X, N, Npad, l2, s2, alpha, Kl)
    ep, eo = np.abs((part - wp).astype(float)), np.abs((out - wo).astype(float))
    _ratio(("tma trace", "part"), ep, bp)
    _ratio(("tma trace", "out"), eo, bo)
    assert np.all(ep <= bp) and np.all(eo <= bo), (float(np.max(ep / np.maximum(bp, 1e-300))), eo / bo)
    p2, o2 = _trace_tma(eng, dxp, dxt, d, N, Npad, da, dK, ld, theta)
    _same(p2, part)
    _same(o2, out)
    # ownership: unowned partials exactly 0, owned ones bitwise the single-rank ones, the ranks' outputs sum to the total
    for bm_mod, bm_div in ((2, 1), (3, 1), (2, 2), (3, 2)):
        tot = np.zeros(3)
        for rem in range(bm_mod):
            pr, orr = _trace_tma(eng, dxp, dxt, d, N, Npad, da, dK, ld, theta, (bm_mod, rem, bm_div))
            own = np.array([(sm.tri_decode(t)[0] // bm_div) % bm_mod == rem for t in range(part.shape[0])])
            assert np.all(pr[~own] == 0)
            _same(pr[own], part[own])
            tot = tot + orr
        assert np.all(np.abs((tot - wo).astype(float)) <= bo + gm.gamma(bm_mod) * np.sum(np.abs(part), axis=0))
    # the generic trace kernel (three accumulators for the single SEIso leaf) on the same operands
    xg = np.full((Npad, d), NAN)
    xg[:N] = X
    tiles = part.shape[0]
    gp, go = _dev(np.zeros(tiles * 3)), _dev(np.zeros(3))
    _run(eng, "trace", [_dev(xg).data_ptr(), d, d, N, Npad, da.data_ptr(), dK.data_ptr(), ld, gp.data_ptr(), go.data_ptr(), 1, 0, 1],
         theta, launches=2)
    assert np.all(np.abs(_host(go) - out) <= 2 * bo)


# ---- inputs_dx --------------------------------------------------------------------------------------------------------

def _inputs_dx(e, X, N, d, alpha, G, ldg, theta, fast, bm=(1, 0, 1)):
    Npad = _pad(N)
    x = np.full((Npad, d + 1), NAN)
    x[:N, :d] = X
    out = _dev(np.full((Npad + 1) * d, POISON))
    da = _dev(alpha) if alpha is not None else None
    dG = _dev(G)
    _run(e, "inputs_dx", [_dev(x).data_ptr(), d + 1, d, N, da.data_ptr() if da is not None else 0, dG.data_ptr(), ldg,
                          out.data_ptr(), *bm, int(fast)], theta)
    o = _host(out)
    assert _raw(o[N * d:]).tolist() == _raw(np.full((Npad + 1 - N) * d, POISON)).tolist()
    return o[:N * d].reshape(N, d)


def _dx_operands(rng, N, d):
    Npad = _pad(N)
    ldg = Npad + 3
    X = rng.standard_normal((N, d))
    alpha = np.full(Npad, NAN)
    alpha[:N] = rng.standard_normal(N)
    S = rng.standard_normal((N, N))
    G = np.full((Npad, ldg), NAN)                          # strict upper triangle and everything past N: never read
    G[:N, :N] = np.where(np.tril(np.ones((N, N), bool)), S, NAN)
    return X, alpha, G, ldg


@pytest.mark.parametrize("N", [1, 31, 32, 33, 127, 128, 129, 257, 1000])
def test_inputs_dx_fast_and_generic_within_long_double_bound(eng, N):
    _need_longdouble()
    rng = np.random.default_rng(500 + N)
    d = 3
    P, theta = _seiso(eng, d, 0.1, 0.2)
    X, alpha, G, ldg = _dx_operands(rng, N, d)
    Gl = np.nan_to_num(G[:N, :N])
    models = {id(a): sm.inputs_dx(P, X, a, Gl) for a in (alpha, None)}
    for a in (alpha, None):
        want, bound = models[id(a)]
        outs = []
        for fast in (1, 0):
            o = _inputs_dx(eng, X, N, d, a, G, ldg, theta, fast)
            err = np.abs((o - want).astype(float))
            _ratio(("inputs_dx", "fast" if fast else "generic"), err, bound)
            assert np.all(err <= bound), (fast, a is None, float(np.max(err / bound)))
            _same(_inputs_dx(eng, X, N, d, a, G, ldg, theta, fast), o)
            outs.append(o)
        assert np.all(np.abs(outs[0] - outs[1]) <= 2 * bound)
    # ownership: each rank adds the rows of its tile rows; the ranks' results sum to the whole
    for bm_mod, bm_div in ((2, 1), (3, 1), (2, 2), (3, 2)):
        parts = [_inputs_dx(eng, X, N, d, alpha, G, ldg, theta, 1, (bm_mod, r, bm_div)) for r in range(bm_mod)]
        want, bound = models[id(alpha)]
        tot = sum(parts)
        assert np.all(np.abs((tot - want).astype(float)) <= bound + gm.gamma(bm_mod) * sum(np.abs(p) for p in parts))


ZOO = [(n, k) for n, k in kernel_zoo(3)]


def _dx_generic_case(eng, kernel, d, N, seed):
    rng = np.random.default_rng(seed)
    P, theta = tg._program(eng, kernel, d)
    X, alpha, G, ldg = _dx_operands(rng, N, d)
    X[5] = X[2]
    want, bound = sm.inputs_dx(P, X, alpha, np.nan_to_num(G[:N, :N]))
    o = _inputs_dx(eng, X, N, d, alpha, G, ldg, theta, 0)
    err = np.abs((o - want).astype(float))
    return err, bound


@pytest.mark.parametrize("name,kernel", ZOO, ids=[z[0] for z in ZOO])
def test_inputs_dx_generic_over_the_kernel_zoo(eng, name, kernel):
    _need_longdouble()
    err, bound = _dx_generic_case(eng, kernel, 3, 150, zlib.crc32(name.encode()))
    _ratio(("inputs_dx", "zoo"), err, bound)
    assert np.all(err <= bound), (name, float(np.max(err / bound)))


@pytest.mark.parametrize("d", [9, 31, 128])
def test_inputs_dx_generic_at_input_dimension(eng, d):
    _need_longdouble()
    for name, kernel in tg._dim_kernels(d):
        err, bound = _dx_generic_case(eng, kernel, d, 100, d)
        _ratio(("inputs_dx", "dim %d" % d), err, bound)
        assert np.all(err <= bound), (d, name, float(np.max(err / bound)))


# ---- vector kernels ---------------------------------------------------------------------------------------------------

def _vrun(e, name, args, fargs=(), launches=1):
    n0 = e.launch_count()
    e.vec_kernels(name, [int(a) for a in args], fargs)
    assert e.launch_count() - n0 == launches, (name, e.launch_count() - n0)


@pytest.mark.parametrize("n", [0, 1, 255, 256, 257, 10 ** 6])
def test_ew_ops_bitwise(eng, n):
    rng = np.random.default_rng(n)
    a = np.full(n + 3, NAN)
    b, c = a.copy(), a.copy()
    a[:n] = rng.uniform(0.5, 4.0, n) * np.where(rng.random(n) < 0.5, 1, 1e-300)
    b[:n] = rng.standard_normal(n)
    c[:n] = rng.uniform(0.5, 4.0, n)
    da, db, dc = _dev(a), _dev(b), _dev(c)
    s = 0.1
    o0 = np.full(n + 3, POISON)
    o0[:n] = rng.standard_normal(n)
    with np.errstate(all="ignore"):
        want = {0: a[:n] + s, 1: a[:n] / b[:n], 2: o0[:n] + a[:n], 3: (a[:n] - b[:n]) / c[:n], 4: np.log(a[:n]),
                5: 1.0 / a[:n], 6: a[:n] - b[:n]}
    for op in range(7):
        out = _dev(o0)
        _vrun(eng, "ew", [op, n, out.data_ptr(), da.data_ptr(), db.data_ptr(), dc.data_ptr()], [s], launches=int(n > 0))
        got = _host(out)
        assert _raw(got[n:]).tolist() == _raw(o0[n:]).tolist()
        if op == 4:                                        # log: within one ulp of the long-double logarithm
            assert np.all(np.abs((got[:n] - np.log(a[:n].astype(gm.LD))).astype(float)) <= np.spacing(np.abs(want[4])))
        else:
            _same(got[:n], want[op])


@pytest.mark.parametrize("n", [1, 100, 128, 129, 300])
def test_spd_from_cov_bitwise(eng, n):
    rng = np.random.default_rng(n)
    npad = _pad(n)
    ldd, lds = npad + 2, n + 5
    src = np.full((n, lds), NAN)
    S = rng.standard_normal((n, n))
    tri = (np.arange(n)[None, :] >> 7) <= (np.arange(n)[:, None] >> 7)        # lower 128-tiles: read whole
    src[:, :n] = np.where(tri, S, NAN)
    D0 = np.full((npad, ldd), POISON)
    dD = _dev(D0)
    _vrun(eng, "spd_from_cov", [dD.data_ptr(), ldd, _dev(src).data_ptr(), lds, n, npad], [1e-3])
    want = D0.copy()
    i, j = np.arange(npad)[:, None], np.arange(npad)[None, :]
    v = np.where((i == j), 1.0, 0.0)
    v[:n, :n] = S + 1e-3 * np.eye(n)
    want[:, :npad] = np.where((j >> 7) <= (i >> 7), v, D0[:, :npad])
    _same(_host(dD), want)


@pytest.mark.parametrize("nv", [0, 1, 5, 300])
def test_gather_block_bitwise(eng, nv):
    rng = np.random.default_rng(nv)
    M, ld = 400, 411
    src = rng.standard_normal((M, ld))
    src[:, M:] = NAN
    idx = rng.integers(0, M, nv).astype(np.int64)
    if nv > 2:
        idx[2] = idx[0]                                    # unsorted, with a repeated index
    out = _dev(np.full(nv * nv + 3, POISON))
    di = _torch_long(np.concatenate([idx, [0]]))         # one spare entry, never read: an empty tensor has a null pointer
    _vrun(eng, "gather_block", [out.data_ptr(), _dev(src).data_ptr(), ld, di.data_ptr(), nv], launches=int(nv > 0))
    want = np.full(nv * nv + 3, POISON)
    want[:nv * nv] = src[np.ix_(idx, idx)].ravel()
    _same(_host(out), want)


def _torch_long(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64)).to("cuda:0")


@pytest.mark.parametrize("nrows", [1, 65535, 65536, 70000])
def test_add_rowvec_bitwise_at_any_row_count(eng, nrows):
    rng = np.random.default_rng(nrows)
    ncols, ld = 8, 10
    A = rng.standard_normal((nrows, ld))
    A[:, ncols:] = POISON
    v = rng.standard_normal(ncols)
    dA = _dev(A)
    _vrun(eng, "add_rowvec", [dA.data_ptr(), ld, _dev(v).data_ptr(), nrows, ncols])
    want = A.copy()
    want[:, :ncols] += v[None, :]
    _same(_host(dA), want)


# ---- misuse -----------------------------------------------------------------------------------------------------------

def test_misuse_returns_einval_and_launches_nothing(eng):
    import gpb200
    P, theta = _seiso(eng, 3, 0.1, 0.2)
    f = list(theta)
    buf = _dev(np.zeros(8 * T * T))
    b = buf.data_ptr()
    gt = [b, b, 3, 5, 128, b, 1, b, 128, 0, 1, 0, 0, 0]
    tt = [b, b, 3, 5, 128, b, b, 128, b, b, 1, 0, 1, 0]
    dx = [b, 4, 3, 5, b, b, 5, b, 1, 0, 1, 1]

    def sub(base, i, v):
        a = list(base)
        a[i] = v
        return a
    bad = [("gram_seiso_tma", sub(gt, 0, b + 8), f + [0.0]), ("gram_seiso_tma", sub(gt, 1, 0), f + [0.0]),
           ("gram_seiso_tma", sub(gt, 3, 0), f + [0.0]), ("gram_seiso_tma", sub(gt, 4, 64), f + [0.0]),
           ("gram_seiso_tma", sub(gt, 8, 127), f + [0.0]), ("gram_seiso_tma", sub(gt, 6, 3), f + [0.0]),
           ("gram_seiso_tma", sub(gt, 11, 1), f + [0.0]), ("gram_seiso_tma", gt, f),
           ("gram_seiso_tma", gt, [-24.0, 0.0, 0.0]),                           # l2 = e^-48 < 1e-20: the fast exp's range
           ("gram_seiso_tma", gt, [0.0, 18.0, 0.0]),                            # s2 = e^36 > 1e15
           ("trace_seiso_tma", sub(tt, 1, b + 8), f), ("trace_seiso_tma", sub(tt, 6, b + 8), f),
           ("trace_seiso_tma", sub(tt, 7, 129), f), ("trace_seiso_tma", sub(tt, 10, 0), f), ("trace_seiso_tma", sub(tt, 12, 0), f),
           ("inputs_dx", sub(dx, 1, 2), f), ("inputs_dx", sub(dx, 6, 4), f), ("inputs_dx", sub(dx, 9, 1), f),
           ("inputs_dx", sub(dx, 11, 2), f), ("inputs_dx", sub(dx, 5, 0), f)]
    n0 = eng.launch_count()
    for name, args, fa in bad:
        with pytest.raises(ValueError):
            eng.gram_kernels(name, [int(a) for a in args], fa)
    # the fast paths need the single SEIso leaf over every dimension, at most 8 of them
    import gpb200 as g
    tg._program(eng, g.SEIso(0.1, 0.2) + g.Const(0.0), 3)
    for name, args, fa in (("gram_seiso_tma", gt, f + [0.0, 0.0]), ("trace_seiso_tma", tt, f + [0.0]), ("inputs_dx", dx, f + [0.0])):
        with pytest.raises(ValueError):
            eng.gram_kernels(name, [int(a) for a in args], fa)
    _seiso(eng, 9, 0.1, 0.2)
    with pytest.raises(ValueError):
        eng.gram_kernels("gram_seiso_tma", [int(a) for a in sub(gt, 2, 9)], f + [0.0])
    with pytest.raises(ValueError):
        eng.gram_kernels("inputs_dx", [int(a) for a in sub(sub(dx, 2, 9), 1, 9)], f)
    vbad = [("ew", [7, 5, b, b, b, b], [0.0]), ("ew", [1, 5, b, b, 0, b], [0.0]), ("ew", [3, 5, b, b, b, 0], [0.0]),
            ("ew", [0, -1, b, b, b, b], [0.0]), ("ew", [0, 5, b, b, b, b], []),
            ("spd_from_cov", [b, 128, b, 5, 5, 64], [0.0]), ("spd_from_cov", [b, 127, b, 5, 5, 128], [0.0]),
            ("spd_from_cov", [b, 128, b, 4, 5, 128], [0.0]), ("spd_from_cov", [b, 128, b, 5, 5, 0], [0.0]),
            ("add_rowvec", [b, 7, b, 5, 8], []), ("add_rowvec", [b, 8, 0, 5, 8], []), ("add_rowvec", [b, 8, b, -1, 8], []),
            ("gather_block", [b, b, 5, 0, 3], []), ("gather_block", [b, b, 5, b, -1], []), ("add_rowvec", [b, 8, b, 5, 8], [1.0])]
    for name, args, fa in vbad:
        with pytest.raises(ValueError):
            eng.vec_kernels(name, args, fa)
    for which in (-1, 4):
        a = np.zeros(6, dtype=np.int64)
        assert eng._lib.gpb200_vec_kernels(eng._h, which, a.ctypes.data_as(gpb200.capi._lp), 6, None, 0) == gpb200.capi.EINVAL
    for which in (-1, 14):
        a = np.zeros(14, dtype=np.int64)
        assert eng._lib.gpb200_gram_kernels(eng._h, which, a.ctypes.data_as(gpb200.capi._lp), 14, None, 0) == gpb200.capi.EINVAL
    assert eng.launch_count() == n0


def test_print_ratio_table():
    for key in sorted(k for k in tg.RATIOS if k[0] in ("tma gram", "tma trace", "inputs_dx")):
        print("RATIO-TABLE %-50s %.3e" % (key, tg.RATIOS[key]))
